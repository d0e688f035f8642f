"""CPU tests of the HMC / SG-MCMC oracle: it reproduces the committed golden
vectors, and it passes the reference's own statistical tests
(tests/test_mcmc.py) re-stated with SciPy KDE."""
import os

import numpy as np
import pytest
from scipy import stats

from oracle import hmc as OH
from oracle import sgmcmc as OS
from oracle import models as OM

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _replay_hmc(g, model):
    cfg = {k[4:]: g[k] for k in g.files if k.startswith("cfg_")}
    h = OH.HMC(step_size=float(cfg["step_size"]),
               n_leapfrogs=int(cfg["n_leapfrogs"]), adapt_step_size=True,
               target_acceptance_rate=float(cfg["target_acceptance_rate"]),
               adapt_mass=True,
               mass_collect_iters=int(cfg["mass_collect_iters"]),
               mass_decay=float(cfg["mass_decay"]))
    q = [g["q0"].copy()]
    for i in range(g["q"].shape[0]):
        adapt = i < int(g["n_adapt"])
        q, info = h.step(q, model.logp, model.grad, [g["noise_p"][i]],
                         g["noise_u"][i], adapt, adapt)
        np.testing.assert_array_equal(info.if_accept.astype(np.int32),
                                      g["accept"][i])
        np.testing.assert_allclose(q[0], g["q"][i], rtol=1e-6, atol=1e-7)
        np.testing.assert_allclose(info.updated_step_size, g["step_size"][i],
                                   rtol=1e-6)
    assert h.n_search_iters == int(g["n_search_iters"])


def test_oracle_reproduces_hmc_diag_golden():
    g = np.load(os.path.join(GOLD, "hmc_diag.npz"))
    D = g["std"].shape[0]
    _replay_hmc(g, OM.DiagGaussian(np.zeros(D, np.float32), g["std"]))


def test_oracle_reproduces_hmc_dense_golden():
    g = np.load(os.path.join(GOLD, "hmc_dense.npz"))
    model = OM.DenseGaussian(g["P"].astype(np.float32), g["mu"],
                             float(g["const"]))
    _replay_hmc(g, model)


def test_dense_gaussian_matches_mvn_logpdf():
    P, const = OM.make_dense_gaussian_problem(16, seed=5)
    m = OM.DenseGaussian(P, None, const, dtype=np.float64)
    x = np.random.RandomState(0).standard_normal((5, 16))
    ref = stats.multivariate_normal.logpdf(x, np.zeros(16), np.linalg.inv(P))
    np.testing.assert_allclose(m.logp([x]), ref, rtol=1e-9)
    h = 1e-6
    xp = x.copy(); xp[:, 3] += h
    fd = (m.logp([xp]) - m.logp([x])) / h
    np.testing.assert_allclose(m.grad([x])[0][:, 3], fd, rtol=1e-4, atol=1e-5)


def test_bnn_oracle_gradient_matches_finite_difference():
    rng = np.random.RandomState(3)
    x = rng.standard_normal((7, 4)); y = rng.standard_normal(7)
    m = OM.BNN(x, y, n_train=100, dtype=np.float64)
    w0 = rng.standard_normal((3, 5, 5)); w1 = rng.standard_normal((3, 1, 6))
    g0, g1 = m.grad([w0, w1])
    h = 1e-6
    for (arr, grad, idx) in [(w0, g0, (1, 2, 3)), (w1, g1, (2, 0, 4))]:
        a2 = arr.copy(); a2[idx] += h
        args = [a2, w1] if arr is w0 else [w0, a2]
        fd = (m.logp(args) - m.logp([w0, w1]))[idx[0]] / h
        np.testing.assert_allclose(grad[idx], fd, rtol=1e-4, atol=1e-4)


def _kde_error(samples):
    """tests/test_mcmc.py:44-50."""
    A = 3
    xs = np.linspace(-A, A, 1000)
    pdfs = np.exp(2 * (xs ** 2) - xs ** 4)
    pdfs = pdfs / pdfs.mean() / A / 2
    est = stats.gaussian_kde(samples.reshape(-1))(xs)
    return np.abs(est - pdfs).mean()


def test_hmc_double_well_statistical():
    """tests/test_mcmc.py:53-62: step 0.01, L=10, 100 chains x 1000 iters,
    NOISY log-joint (fresh N(0, 2^2) per evaluation, zero gradient), burn-in
    2/3, thinning 50; KDE mean-abs error <= 0.030."""
    rng = np.random.RandomState(0)
    base = OM.DoubleWell(np.float32)

    def logp(q):
        return base.logp(q) + (2.0 * rng.standard_normal(q[0].shape)).astype(
            np.float32)
    h = OH.HMC(step_size=0.01, n_leapfrogs=10)
    q = [np.zeros(100, np.float32)]
    samples = []
    n_iters = 1000
    for t in range(n_iters):
        q, _ = h.step(q, logp, base.grad,
                      [rng.standard_normal(100).astype(np.float32)],
                      rng.random_sample(100).astype(np.float32))
        if t >= n_iters * 2 // 3 and t % 50 == 0:
            samples.append(q[0].copy())
    assert _kde_error(np.array(samples)) <= 0.030


@pytest.mark.parametrize("second_order", [False, True])
def test_sghmc_double_well_statistical(second_order):
    """tests/test_mcmc.py:72-88 (SGHMC 1st / 2nd order, threshold 0.016;
    iterations cut 8000 -> 3000 for CPU time, thresholds relaxed to 0.03)."""
    rng = np.random.RandomState(1)
    base = OM.DoubleWell(np.float32)
    s = OS.SGHMC(learning_rate=0.01, n_iter_resample_v=50, friction=0.3,
                 variance_estimate=0.02, second_order=second_order)
    n = lambda: rng.standard_normal(100).astype(np.float32)
    s.init_v([n()])
    q = [np.zeros(100, np.float32)]
    samples = []
    n_iters = 3000
    for t in range(n_iters):
        q, _ = s.step(q, base.grad, [n()], [n()])
        if t >= n_iters * 2 // 3 and t % 50 == 0:
            samples.append(q[0].copy())
    assert _kde_error(np.array(samples)) <= 0.03


def test_sgmcmc_golden_replay():
    import sys
    sys.path.insert(0, GOLD)
    g = np.load(os.path.join(GOLD, "sgmcmc.npz"))
    model = OM.DiagGaussian(g["mean"], g["std"])
    s = OS.SGHMC(learning_rate=0.01, friction=0.3, variance_estimate=0.02,
                 n_iter_resample_v=3, second_order=True)
    s.init_v([g["sghmc2_v0"]])
    q = [g["q0"].copy()]
    for t in range(g["sghmc2_q"].shape[0]):
        q, info = s.step(q, model.grad, [g["sghmc2_resample"][t]],
                         [g["sghmc2_noise"][t]])
        np.testing.assert_allclose(q[0], g["sghmc2_q"][t], rtol=1e-6,
                                   atol=1e-7)


def test_hmc_constructor_errors():
    with pytest.raises(ValueError, match="adapt mass"):
        OH.HMC(adapt_mass=True)
    h = OH.HMC()
    with pytest.raises(ValueError):
        h.step([np.zeros(3, np.float32)], lambda q: np.float32(0.0),
               lambda q: q, [np.zeros(3, np.float32)], np.float32(0.5))


@pytest.mark.parametrize("name", ["hmc_dense64", "hmc_dense1024"])
def test_oracle_reproduces_big_dense_golden(name):
    """The L = 50 adaptive fixtures of the tensor-core kernels (make_golden.py BIG): the float32
    oracle, fed the re-generated states / Philox noise and the stored (guard-pushed) uniforms,
    reproduces the stored decisions / step sizes, and the stored float64 re-evaluation bounds its
    error."""
    import sys
    sys.path.insert(0, GOLD)
    import make_golden as MG
    g = np.load(os.path.join(GOLD, name + ".npz"))
    cfg = MG.BIG[name]
    P, const, mu, chol = MG.big_problem(cfg)
    np.testing.assert_allclose(np.abs(P).sum(), float(g["P_checksum"]), rtol=1e-12)
    model = OM.DenseGaussian(P.astype(np.float32), mu, const)
    h = OH.HMC(step_size=cfg["eps0"], n_leapfrogs=cfg["L"], adapt_step_size=True,
               adapt_mass=True, mass_collect_iters=cfg["mci"])
    n_iters = cfg["iters"] if cfg["D"] <= 64 else 9     # keep the CPU suite short
    with np.errstate(all="ignore"):
        for i in range(n_iters):
            adapt = i < cfg["n_adapt"]
            q, info = h.step([MG.big_state(cfg, i)], model.logp, model.grad,
                             [MG.big_noise(cfg, i)], g["noise_u"][i], adapt, adapt)
            np.testing.assert_array_equal(info.if_accept.astype(np.int32), g["accept"][i])
            np.testing.assert_allclose(info.acceptance_rate, g["acc"][i], rtol=1e-5, atol=1e-6)
            np.testing.assert_allclose(info.updated_step_size, g["step_size"][i], rtol=1e-6)
            # every stored uniform sits >= u_guard / 2 away from the acceptance probability
            assert np.all(np.abs(g["noise_u"][i] - info.acceptance_rate) >= cfg["u_guard"] / 2)
    floor = np.abs(g["acc"] - g["acc64"]).max()
    assert floor < cfg["u_guard"] / 8
    live = g["acc64"] > 1e-6
    assert np.abs(g["h1"][live] / g["h1_64"][live] - 1).max() < 2e-6
    assert (~np.isfinite(g["h1"])).any() and live.any()   # diverging and healthy trajectories


@pytest.mark.parametrize("ls0_shape,ls1_shape", [((5, 1), ()), ((3, 5, 5), (3, 1, 6)), ((5,), (1, 6))])
def test_bnn_oracle_gradient_with_broadcast_prior_scales(ls0_shape, ls1_shape):
    """The BNN oracle with array prior log-stddevs (per hidden unit, per chain, ...) broadcast
    against the weights, and a non-default y_logstd: analytic gradient vs finite differences."""
    rng = np.random.RandomState(4)
    x = rng.standard_normal((7, 4)); y = rng.standard_normal(7)
    ls0 = rng.uniform(-0.7, 0.3, ls0_shape); ls1 = rng.uniform(-0.7, 0.3, ls1_shape)
    m = OM.BNN(x, y, 100, ls0, ls1, dtype=np.float64, y_logstd=-0.3)
    w0 = rng.standard_normal((3, 5, 5)); w1 = rng.standard_normal((3, 1, 6))
    g0, g1 = m.grad([w0, w1])
    h = 1e-6
    for (arr, grad, idx) in [(w0, g0, (1, 2, 3)), (w0, g0, (2, 4, 0)), (w1, g1, (2, 0, 4)),
                             (w1, g1, (0, 0, 5))]:
        a2 = arr.copy(); a2[idx] += h
        args = [a2, w1] if arr is w0 else [w0, a2]
        fd = (m.logp(args) - m.logp([w0, w1]))[idx[0]] / h
        np.testing.assert_allclose(grad[idx], fd, rtol=1e-4, atol=1e-4)
