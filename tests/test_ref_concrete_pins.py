"""tests/golden/ref_concrete.npz (made by tests/golden/make_ref_concrete_golden.py): samples,
log-densities and gradients of the reference's own ExpConcrete and Concrete.  The committed arrays
must match their digests, and float64 restatements must reproduce them: the sample from the
recorded uniforms, oracle/distributions.py's exp_concrete_log_prob / concrete_log_prob for the
values, and float64 autograd of the same formula for the gradients.  CPU only."""
import hashlib
import json
import math
import os

import numpy as np
import pytest
import torch

from oracle import distributions as OD

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KEYS = [(p, c) for p in ("exp_", "con_") for c in (0, 1)]


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_concrete.npz"))


def test_fixture_matches_digests(g):
    with open(os.path.join(GOLD, "ref_concrete_digests.json")) as f:
        want = json.load(f)
    got = {}
    for k in g.files:
        a = np.ascontiguousarray(g[k])
        got["ref_concrete/" + k] = [str(a.dtype), list(a.shape),
                                    hashlib.sha256(a.tobytes()).hexdigest()]
    assert got == want


@pytest.mark.parametrize("p,c", KEYS)
def test_sample_from_recorded_uniforms(g, p, c):
    l, t, u = (g[p + k + "_%d" % c].astype(np.float64) for k in ("logits", "t", "u"))
    a = (l - np.log(-np.log(u))) / t
    a = a - a.max(-1, keepdims=True)
    lsm = a - np.log(np.exp(a).sum(-1, keepdims=True))
    want = lsm if p == "exp_" else np.exp(lsm)
    np.testing.assert_allclose(g[p + "sample_%d" % c], want, rtol=1e-5, atol=1e-5)


@pytest.mark.parametrize("p,c", KEYS)
def test_oracle_reproduces_log_prob_and_gradients(g, p, c):
    fn = OD.exp_concrete_log_prob if p == "exp_" else OD.concrete_log_prob
    x, l, t = g[p + "sample_%d" % c], g[p + "logits_%d" % c], g[p + "t_%d" % c]
    for gnd in (0, 1):
        want = fn(x, float(t), l, group_ndims=gnd, dtype=np.float64)
        np.testing.assert_allclose(g[p + "lp%d_%d" % (gnd, c)], want, rtol=1e-5, atol=1e-4)
        xt, lt, tt = (torch.tensor(np.asarray(v, np.float64), requires_grad=True)
                      for v in (x, l, t))
        xx = xt if p == "exp_" else torch.log(xt)
        temp = lt - tt * xx
        C = l.shape[-1]
        lp = math.lgamma(C) + (C - 1) * torch.log(tt) + temp.sum(-1) - \
            C * torch.logsumexp(temp, -1)
        if p == "con_":
            lp = lp - xx.sum(-1)
        lp = lp.sum(-1) if gnd else lp
        grads = torch.autograd.grad((lp * torch.tensor(g[p + "w%d_%d" % (gnd, c)],
                                                       dtype=torch.float64)).sum(), [xt, lt, tt])
        for name, r in zip(("dgiven", "dlogits", "dt"), grads):
            rec = g[p + "%s%d_%d" % (name, gnd, c)]
            r = r.numpy()
            np.testing.assert_allclose(rec, r, rtol=1e-4, atol=1e-4 * (np.abs(r).max() + 1))
