"""tests/golden/ref_ssl_ais.npz (made by tests/golden/make_ref_ssl_ais_golden.py): one training step
and one test batch of the semi-supervised VAE of vae_ssl_adaptive_is.py on the reference's own
BayesianNet, distributions, klpq and importance_weighted_objective.  The committed arrays must match
their digests, and the float64 oracle of tests/ssl_ais_oracle.py must reproduce every recorded
bound, cost, accuracy and gradient.  CPU only."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import ssl_ais_oracle as SA

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
KEYS = ("labeled_lb", "unlabeled_lb", "labeled_q_cost", "unlabeled_q_cost", "classifier_cost",
        "acc")


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_ssl_ais.npz"))


def _layers(g):
    return {n: tuple(torch.tensor(g[p + n], dtype=torch.float64).requires_grad_(True)
                     for p in ("W_", "b_")) for n in SA.NAMES}


def test_fixture_matches_digests(g):
    with open(os.path.join(GOLD, "ref_ssl_ais_digests.json")) as f:
        want = json.load(f)
    got = {}
    for k in g.files:
        a = np.ascontiguousarray(g[k])
        got["ref_ssl_ais/" + k] = [str(a.dtype), list(a.shape),
                                   hashlib.sha256(a.tobytes()).hexdigest()]
    assert got == want


def test_oracle_reproduces_the_step(g):
    L = _layers(g)
    T = lambda k: torch.tensor(g[k], dtype=torch.float64)          # noqa: E731
    x_l = (T("u_l") < T("xp_l")).to(torch.float64)
    x_u = (T("u_u") < T("xp_u")).to(torch.float64)
    out = SA.ais_step(x_l, T("y_l"), x_u, T("eps_l"), T("eps_u"), torch.tensor(g["y_u"]), L)
    for k in KEYS:
        np.testing.assert_allclose(out[k].detach().numpy(), g[k], rtol=2e-5, atol=1e-5, err_msg=k)
    grads = SA.step_grads(out, L)
    for n in SA.NAMES:
        for what, got in zip(("W_", "b_"), grads[n]):
            want = g["grad_" + what + n].astype(np.float64)
            np.testing.assert_allclose(got.numpy(), want, rtol=2e-4,
                                       atol=2e-5 * max(1.0, np.abs(want).max()),
                                       err_msg="grad " + what + n)


def test_oracle_reproduces_the_test_batch(g):
    L = _layers(g)
    T = lambda k: torch.tensor(g[k], dtype=torch.float64)          # noqa: E731
    x = T("test_x")
    out = SA.ais_step(x, T("test_y"), x, T("test_eps_l"), T("test_eps_u"),
                      torch.tensor(g["test_y_u"]), L)
    for k in ("labeled_lb", "unlabeled_lb", "acc"):
        np.testing.assert_allclose(out[k].detach().numpy(), g["test_" + k], rtol=2e-5, atol=1e-5,
                                   err_msg=k)
