"""tests/golden/ref_lntm_mcem.npz (made by tests/golden/make_ref_lntm_mcem_golden.py): one epoch of
the logistic-normal topic model trained by Monte-Carlo EM (examples/topic_models/lntm_mcem.py) and
a short AIS evaluation, on the reference's own BayesianNet, distributions, HMC, tf.gradients and AIS.
The committed arrays must match their digests, and the float64 oracle of tests/lntm_mcem_oracle.py
must reproduce every HMC iteration, M-step gradient and Adam update, the eta-prior update, the
perplexity and the AIS run.  CPU only."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import lntm_mcem_oracle as LO
from oracle import evaluation as OE
from oracle import hmc as OH
from ssl_ais_models import Adam

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_lntm_mcem.npz"))


def _batches(g):
    C, B = g["noise_u"].shape[1:]
    n_iters = g["x_train"].shape[0] // B
    e_steps = g["acc"].shape[0] // n_iters
    return B, n_iters, e_steps


def test_fixture_matches_digests(g):
    with open(os.path.join(GOLD, "ref_lntm_mcem_digests.json")) as f:
        want = json.load(f)
    got = {}
    for k in g.files:
        a = np.ascontiguousarray(g[k])
        got["ref_lntm_mcem/" + k] = [str(a.dtype), list(a.shape),
                                     hashlib.sha256(a.tobytes()).hexdigest()]
    assert got == want


def test_oracle_reproduces_the_epoch(g):
    B, n_iters, e_steps = _batches(g)
    K = g["beta0"].shape[0]
    mean0, logstd0 = np.zeros(K), np.zeros(K)
    hmc = OH.HMC(step_size=0.05, n_leapfrogs=3, adapt_step_size=True, target_acceptance_rate=0.6)
    beta = torch.tensor(g["beta0"], dtype=torch.float64)
    opt = Adam({"beta": [beta]}, lr=float(g["lr"]))
    Eta = np.zeros_like(g["Eta"])
    for t in range(n_iters):
        ids = g["perm"][t * B:(t + 1) * B]
        m = LO.LNTM(g["x_train"], beta.numpy(), mean0, logstd0, doc_ids=ids)
        q = [Eta[:, ids]]
        for j in range(e_steps):
            i = t * e_steps + j
            q, info = hmc.step(q, m.logp, m.grad, [g["noise_p"][i]], g["noise_u"][i], True)
            np.testing.assert_allclose(info.orig_log_prob, g["lp0"][i], rtol=1e-5, atol=1e-3)
            np.testing.assert_allclose(info.acceptance_rate, g["acc"][i], rtol=2e-3, atol=2e-4)
            np.testing.assert_allclose(info.updated_step_size, g["step_size"][i], rtol=1e-4)
            near = np.abs(g["noise_u"][i] - g["acc"][i]) < 2e-3
            np.testing.assert_allclose(q[0][~near], g["eta"][i][~near], rtol=1e-4, atol=1e-5)
            q = [g["eta"][i]]                        # continue from the reference's state
        Eta[:, ids] = q[0]
        grad, log_px = LO.m_step_grad(g["x_train"], beta.numpy(), mean0, logstd0, q[0], ids)
        np.testing.assert_allclose(log_px, g["log_px"][t], rtol=1e-5)
        want = g["grad_beta"][t]
        np.testing.assert_allclose(grad, want, rtol=1e-4, atol=1e-5 * np.abs(want).max())
        opt.step({"beta": [torch.tensor(want, dtype=torch.float64)]})
        np.testing.assert_allclose(beta.numpy(), g["beta"][t], rtol=1e-5, atol=1e-6)
        beta.copy_(torch.tensor(g["beta"][t]))
    np.testing.assert_array_equal(Eta, g["Eta"])
    np.testing.assert_allclose(Eta.mean((0, 1)), g["Eta_mean"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(np.log(Eta.astype(np.float64).std((0, 1)) + 1e-6),
                               g["Eta_logstd"], rtol=1e-5, atol=1e-5)
    perplexity = np.exp(-np.sum(g["log_px"].astype(np.float64)) / g["x_train"].sum())
    np.testing.assert_allclose(perplexity, g["perplexity"], rtol=1e-6)


def test_oracle_reproduces_the_ais_run(g):
    m = LO.LNTM(g["x_test"], g["beta"][-1], g["Eta_mean"], g["Eta_logstd"])
    hmc = OH.HMC(step_size=0.01, n_leapfrogs=3, adapt_step_size=True, target_acceptance_rate=0.6)
    n_t = g["ais_schedule"].shape[0] - 1
    n_adapt = g["ais_noise_u"].shape[0] - n_t
    ais = OE.AIS(lambda q: m.log_prior(q[0]), lambda q: m.grad_t(q, 0.0), m.logp, m.grad, hmc,
                 n_temperatures=n_t, n_adapt=n_adapt, dtype=np.float64)
    np.testing.assert_allclose([ais.schedule(t) for t in range(n_t + 1)], g["ais_schedule"],
                               rtol=1e-12)
    bound, log_w = ais.run([[g["ais_init"][0]], [g["ais_init"][1]]],
                           lambda k: ([g["ais_noise_p"][k]], g["ais_noise_u"][k]),
                           adapt_flags=(True, False))
    np.testing.assert_allclose(log_w, g["ais_log_weights"], rtol=1e-4, atol=1e-3)
    assert abs(bound - float(g["ais_bound"])) < 1e-3
