"""tests/golden/ref_blvae.npz (made by tests/golden/make_ref_blvae_golden.py): one REINFORCE
training step and one evaluation of the Bernoulli-latent VAE of bernoulli_latent_vae.py on the reference's
own BayesianNet, Bernoulli, elbo().reinforce(baseline=cx) and is_loglikelihood.  The committed
arrays must match their digests, and the float64 oracle of tests/blvae_oracle.py must reproduce
every recorded value on the recorded draws.  CPU only."""
import hashlib
import json
import os

import numpy as np
import pytest
import torch

import blvae_oracle as BO

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
Q_NAMES = ["W_q0", "gamma_q0", "beta_q0", "W_q1", "gamma_q1", "beta_q1", "W_qz", "b_qz"]
P_NAMES = ["W_p0", "gamma_p0", "beta_p0", "W_p1", "gamma_p1", "beta_p1", "W_px", "b_px"]
C_NAMES = ["W_c0", "b_c0", "W_c1", "b_c1"]
BN_LAYERS = ["q0", "q1", "p0", "p1"]


@pytest.fixture(scope="module")
def g():
    return np.load(os.path.join(GOLD, "ref_blvae.npz"))


def test_fixture_matches_digests(g):
    with open(os.path.join(GOLD, "ref_blvae_digests.json")) as f:
        want = json.load(f)
    got = {}
    for k in g.files:
        a = np.ascontiguousarray(g[k])
        got["ref_blvae/" + k] = [str(a.dtype), list(a.shape),
                                 hashlib.sha256(a.tobytes()).hexdigest()]
    assert got == want


def _T(g, k):
    return torch.tensor(g[k], dtype=torch.float64)


def _run(g, training, stats, zkey):
    """The oracle on the fixture's data and draws: (params, log q, log p, cx, new stats)."""
    q, p, c = ([_T(g, k).requires_grad_(True) for k in names]
               for names in (Q_NAMES, P_NAMES, C_NAMES))
    x, z = _T(g, "x"), _T(g, zkey)
    logits, nq = BO.encoder(x, q, stats[:2], training)
    log_qz = BO.bern_lp(logits, z)
    log_pxz, np_ = BO.decoder_log_joint(x, z, p, stats[2:], training)
    return q, p, c, log_qz, log_pxz, BO.baseline(x, c).unsqueeze(0), nq + np_


def test_binarisation_and_draws(g):
    np.testing.assert_array_equal(g["x"], (g["u_x"] < g["x_input"]).astype(np.int32))
    for zk, uk, training, stats in (("z", "u_z", True, None), ("eval_z", "eval_u_z", False, 1)):
        W1, g1, b1, W2, g2, b2, Wz, bz = (_T(g, k) for k in Q_NAMES)
        if training:
            st = [(torch.zeros(20, dtype=torch.float64), torch.ones(20, dtype=torch.float64))] * 2
        else:
            st = [(_T(g, "moving_mean_" + n), _T(g, "moving_variance_" + n)) for n in ("q0", "q1")]
        logits, _ = BO.encoder(_T(g, "x"), (W1, g1, b1, W2, g2, b2, Wz, bz), st, training)
        prob = torch.sigmoid(logits).numpy()
        u = g[uk]
        far = np.abs(u - prob) > 1e-6
        assert far.all()
        np.testing.assert_array_equal(g[zk], (u < prob).astype(np.float32))


def test_oracle_reproduces_the_training_step(g):
    J = int(g["W_q0"].shape[0])
    fresh = [(torch.zeros(J, dtype=torch.float64), torch.ones(J, dtype=torch.float64))] * 4
    q, p, c, lq, lp, cx, new = _run(g, True, fresh, "z")
    cost, bound, bc = BO.reinforce(lp, lq, cx, 0.0)
    np.testing.assert_allclose(float(cost.detach()), g["cost"], rtol=2e-5)
    np.testing.assert_allclose(float(bound), g["bound"], rtol=2e-5)
    np.testing.assert_allclose(BO.baseline_cost(lp, lq, cx).detach().numpy(), g["baseline_cost"],
                               rtol=2e-5)
    # REINFORCE's moving mean starts at 0; its zero-debiased first update is bc itself
    np.testing.assert_allclose(float(bc), g["rf_moving_mean"], rtol=2e-5)
    for name, (m, v) in zip(BN_LAYERS, new):
        np.testing.assert_allclose(m.detach().numpy(), g["moving_mean_" + name], rtol=1e-5,
                                   atol=1e-6, err_msg=name)
        np.testing.assert_allclose(v.detach().numpy(), g["moving_variance_" + name], rtol=1e-5,
                                   atol=1e-6, err_msg=name)
    grads = torch.autograd.grad(cost, q + p + c)
    for name, got in zip(Q_NAMES + P_NAMES + C_NAMES, grads):
        want = g["grad_" + name].astype(np.float64)
        np.testing.assert_allclose(got.numpy(), want, rtol=1e-3,
                                   atol=1e-4 * max(1.0, np.abs(want).max()), err_msg=name)


def test_oracle_reproduces_the_evaluation(g):
    stats = [(_T(g, "moving_mean_" + n), _T(g, "moving_variance_" + n)) for n in BN_LAYERS]
    _, _, _, lq, lp, _, new = _run(g, False, stats, "eval_z")
    np.testing.assert_allclose(float((lp - lq).mean()), g["eval_bound"], rtol=2e-5)
    np.testing.assert_allclose(float(BO.is_loglikelihood(lp, lq)), g["eval_is_ll"], rtol=2e-5)
    for (m, v), (m0, v0) in zip(new, stats):
        assert m is m0 and v is v0
