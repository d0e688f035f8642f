"""tests/golden/ref_sbn.npz (made by tests/golden/make_ref_sbn_golden.py): the sigmoid belief nets of
sbn_vimco.py / sbn_adaptive_is.py on the reference's own BayesianNet, Bernoulli, vimco() and
klpq(...).importance().  The committed arrays must match their digests, and the float64 oracle of
tests/sbn_oracle.py must reproduce the recorded samples, IW bound, costs and every gradient.  CPU
only."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import sbn_oracle as SO

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
Q_NAMES = ["q_h1", "q_h2", "q_h3"]
M_NAMES = ["m_h2", "m_h1", "m_x"]


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_sbn.npz"))


def test_fixture_matches_digests(g):
    with open(os.path.join(GOLD, "ref_sbn_digests.json")) as f:
        want = json.load(f)
    got = {}
    for k in g.files:
        a = np.ascontiguousarray(g[k])
        got["ref_sbn/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    assert got == want


def _layers(g, names):
    return [tuple(torch.tensor(g[p + n], dtype=torch.float64).requires_grad_(True)
                  for p in ("W_", "b_")) for n in names]


def _close(got, want, what):
    want = np.asarray(want, np.float64)
    np.testing.assert_allclose(got, want, rtol=2e-4, atol=2e-5 * max(1.0, np.abs(want).max()),
                               err_msg=what)


def test_recorded_samples_are_the_draws_on_float64_logits(g):
    x = torch.tensor(g["x"], dtype=torch.float64)
    q = _layers(g, Q_NAMES)
    h = x
    for name, layer, u in zip(("h1", "h2", "h3"), q, (g["u_h1"], g["u_h2"][0], g["u_h3"][0])):
        p = torch.sigmoid(SO.dense(h, layer)).detach().numpy()
        want = (u < p).astype(np.float32)
        np.testing.assert_array_equal(g[name], want, err_msg=name)
        assert np.abs(u - p).min() >= 1e-3
        h = torch.tensor(want)


def test_oracle_reproduces_vimco_step(g):
    x = torch.tensor(g["x"], dtype=torch.float64)
    hs = [torch.tensor(g[n], dtype=torch.float64) for n in ("h1", "h2", "h3")]
    q, m = _layers(g, Q_NAMES), _layers(g, M_NAMES)
    lq, lp = SO.log_q(x, hs, q), SO.log_joint(x, hs, m)
    bound = SO.iw_bound(lp, lq)
    np.testing.assert_allclose(bound.detach().numpy(), g["iw_bound"], rtol=2e-6)
    cost = SO.vimco_cost(lp, lq).mean()
    np.testing.assert_allclose(cost.item(), float(g["vimco_cost"]), rtol=2e-6)
    params = [p for l in q + m for p in l]
    grads = torch.autograd.grad(cost, params)
    for name, gW, gb in zip(Q_NAMES + M_NAMES, grads[0::2], grads[1::2]):
        _close(gW.numpy(), g["vimco_grad_W_" + name], "vimco W " + name)
        _close(gb.numpy(), g["vimco_grad_b_" + name], "vimco b " + name)


def test_oracle_reproduces_reweighted_wake_sleep_step(g):
    x = torch.tensor(g["x"], dtype=torch.float64)
    hs = [torch.tensor(g[n], dtype=torch.float64) for n in ("h1", "h2", "h3")]
    q, m = _layers(g, Q_NAMES), _layers(g, M_NAMES)
    lq, lp = SO.log_q(x, hs, q), SO.log_joint(x, hs, m)
    gm = torch.autograd.grad(-SO.iw_bound(lp, lq).mean(), [p for l in m for p in l],
                             retain_graph=True)
    for name, gW, gb in zip(M_NAMES, gm[0::2], gm[1::2]):
        _close(gW.numpy(), g["rws_grad_W_" + name], "model W " + name)
        _close(gb.numpy(), g["rws_grad_b_" + name], "model b " + name)
    cost = SO.importance_cost(lp, lq).mean()
    np.testing.assert_allclose(cost.item(), float(g["rws_klpq_cost"]), rtol=2e-6)
    gq = torch.autograd.grad(cost, [p for l in q for p in l])
    for name, gW, gb in zip(Q_NAMES, gq[0::2], gq[1::2]):
        _close(gW.numpy(), g["rws_grad_W_" + name], "proposal W " + name)
        _close(gb.numpy(), g["rws_grad_b_" + name], "proposal b " + name)
