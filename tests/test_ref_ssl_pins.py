"""tests/golden/ref_ssl.npz (made by tests/golden/make_ref_ssl_golden.py): one training step of the
semi-supervised VAE of vae_ssl.py on the reference's own BayesianNet, distributions and elbo().  The
committed arrays must match their digests, and the float64 oracle of tests/ssl_oracle.py must
reproduce every recorded bound, cost and gradient.  CPU only."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import ssl_oracle as SS

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_ssl.npz"))


def test_fixture_matches_digests(g):
    with open(os.path.join(GOLD, "ref_ssl_digests.json")) as f:
        want = json.load(f)
    got = {}
    for k in g.files:
        a = np.ascontiguousarray(g[k])
        got["ref_ssl/" + k] = [str(a.dtype), list(a.shape), hashlib.sha256(a.tobytes()).hexdigest()]
    assert got == want


def test_oracle_reproduces_the_step(g):
    L = {n: tuple(torch.tensor(g[p + n], dtype=torch.float64).requires_grad_(True)
                  for p in ("W_", "b_")) for n in SS.NAMES}
    T = lambda k: torch.tensor(g[k], dtype=torch.float64)          # noqa: E731
    out = SS.ssl_step(T("x_l"), T("y_l"), T("x_u"), T("eps_l"), T("eps_u"), L)
    for k in ("labeled_lb", "lb_z", "unlabeled_lb", "classifier_cost", "cost", "acc"):
        np.testing.assert_allclose(out[k].detach().numpy(), g[k], rtol=2e-5, atol=1e-5, err_msg=k)
    params = [p for n in SS.NAMES for p in L[n]]
    grads = torch.autograd.grad(out["cost"], params)
    for n, gW, gb in zip(SS.NAMES, grads[0::2], grads[1::2]):
        for what, got in (("W_", gW), ("b_", gb)):
            want = g["grad_" + what + n].astype(np.float64)
            np.testing.assert_allclose(got.numpy(), want, rtol=2e-4,
                                       atol=2e-5 * max(1.0, np.abs(want).max()),
                                       err_msg="grad " + what + n)
