"""GPU parity of the dense-Gaussian HMC paths when the chains move far from where the trajectory
started: chains initialised at zero or at a small scale, chains of very different magnitudes in
one batch, and a step size beyond the leapfrog's stability limit.

The fp16-split paths (dense_impl 2, 5) hold q inside a trajectory as fp16 hi/lo planes of
q * sq with one power-of-two sq per pass for all chains.  These tests pin that the plane scale
follows the trajectory: every path must give the decisions, Hamiltonians and positions of the
float64 oracle, with the injected momentum and uniforms of test_gpu_hmc.py."""
import numpy as np
import pytest
import torch

from oracle import hmc as OH
from oracle import models as OM

pytestmark = pytest.mark.gpu

# the suite's tolerances after a long trajectory (test_gpu_hmc.py): Hamiltonian and log-prob
H1_RTOL = 1e-5
LP1_RTOL = 5e-5
WIDE = 40.0            # marginal std of the wide target (precision / WIDE^2)


def T(a, dtype=torch.float32):
    return torch.tensor(np.asarray(a), dtype=dtype, device="cuda")


def N(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


_PROBLEMS = {}


def _problem(D, wide=False):
    """(P float64, const) of the unit-marginal test target, or of the same target widened to
    marginal std WIDE."""
    key = (D, wide)
    if key not in _PROBLEMS:
        P, const = OM.make_dense_gaussian_problem(D, seed=4)
        if wide:
            P = P / WIDE ** 2
            const = const - D * np.log(WIDE)
        _PROBLEMS[key] = (P, const)
    return _PROBLEMS[key]


def _log_joint(zs, P, const):
    D = P.shape[0]
    return zs.fused.GaussianLogJoint(P, log_det_cov=-2 * const - D * np.log(2 * np.pi))


def _oracle64(P, const, q0, npz, u, eps, L):
    om = OM.DenseGaussian(P, None, const, dtype=np.float64)
    oq, oi = OH.HMC(step_size=eps, n_leapfrogs=L, dtype=np.float64).step(
        [q0.astype(np.float64)], om.logp, om.grad, [npz.astype(np.float64)],
        u.astype(np.float64))
    return oq[0], oi


def _run(zs, impl, P, const, q0, npz, u, eps, L):
    x = T(q0)
    h = zs.HMC(step_size=eps, n_leapfrogs=L, dense_impl=impl)
    op, info = h.sample(_log_joint(zs, P, const), {}, {"x": x})
    op(noise={"p": {"x": T(npz)}, "u": T(u)})
    op.synchronize()
    if impl == 5 and L >= 1:
        assert h._res
    return N(x), {k: N(getattr(info, k)) for k in
                  ("acceptance_rate", "orig_hamiltonian", "hamiltonian", "orig_log_prob",
                   "log_prob")}


def _check_vs_oracle(got_q, got, oq, oi, q0, u, what):
    acc64, h0, h1 = oi.acceptance_rate, oi.orig_hamiltonian, oi.hamiltonian
    acc = got["acceptance_rate"]
    # acc = exp(min(H0 - H1, 0)): an error dH on H0 - H1 moves it by acc * dH
    dH = H1_RTOL * (np.abs(h0) + np.abs(h1)) + 1e-4
    band = acc64 * dH + 2e-5
    bad = np.abs(acc - acc64) > band
    assert not bad.any(), (
        "%s: acceptance_rate differs from the float64 oracle on %d of %d chains "
        "(mean %.4f vs oracle %.4f; first bad chain: %.6g vs %.6g)"
        % (what, bad.sum(), bad.size, acc.mean(), acc64.mean(), acc[bad][0], acc64[bad][0]))
    for k in ("orig_hamiltonian", "hamiltonian", "orig_log_prob", "log_prob"):
        assert np.isfinite(got[k]).all(), "%s: non-finite %s" % (what, k)
    np.testing.assert_allclose(got["orig_hamiltonian"], h0, rtol=H1_RTOL, atol=1e-4,
                               err_msg=what)
    np.testing.assert_allclose(got["hamiltonian"], h1, rtol=H1_RTOL, atol=1e-4, err_msg=what)
    np.testing.assert_allclose(got["orig_log_prob"], oi.orig_log_prob, rtol=H1_RTOL, atol=1e-4,
                               err_msg=what)
    # decisions: identical except where u is within the error band of the acceptance
    near = np.abs(u - acc64) < band
    accept, accept64 = u < acc, u < acc64
    flips = (accept != accept64) & ~near
    assert not flips.any(), "%s: %d decisions differ from the oracle" % (what, flips.sum())
    lp_scale = np.abs(oi.log_prob).max()
    np.testing.assert_allclose(got["log_prob"][~near], oi.log_prob[~near], rtol=LP1_RTOL,
                               atol=LP1_RTOL * lp_scale, err_msg=what)
    take = accept64 & ~near
    q_scale = max(float(np.abs(oq).max()), 1e-30)
    np.testing.assert_allclose(got_q[take], oq[take], rtol=1e-4, atol=1e-4 * q_scale,
                               err_msg=what)
    keep = ~accept64 & ~near
    np.testing.assert_array_equal(got_q[keep], q0[keep], err_msg=what)


_ORACLE = {}


def _case(D, init, wide, L, eps):
    """Injected draws and the float64 oracle of one iteration, shared by every impl."""
    key = (D, init, wide, L, eps)
    if key not in _ORACLE:
        P, const = _problem(D, wide)
        C = 130                              # two chain tiles, the second ragged
        rng = np.random.RandomState(D + L + int(wide))
        q0 = (init * rng.standard_normal((C, D))).astype(np.float32)
        if init == 0:
            q0 = np.zeros((C, D), np.float32)          # +0.0 everywhere, as torch.zeros
        npz = rng.standard_normal((C, D)).astype(np.float32)
        u = rng.random_sample(C).astype(np.float32)
        oq, oi = _oracle64(P, const, q0, npz, u, eps, L)
        _ORACLE[key] = (P, const, q0, npz, u, oq, oi)
    return _ORACLE[key]


_IMPL_D = [(i, 64) for i in (0, 1, 2, 5)] + [(i, 1024) for i in (0, 1, 2, 5)]


@pytest.mark.parametrize("L", [1, 10, 50])
@pytest.mark.parametrize("init,wide", [(0.0, False), (0.0, True), (1e-3, False),
                                       (1e-6, False)])
@pytest.mark.parametrize("impl,D", _IMPL_D)
def test_small_and_zero_initial_state_vs_oracle(zs, impl, D, init, wide, L):
    """One iteration from q0 = init * N(0, 1) (exact zeros for init 0).  From a small state the
    first leapfrog step already moves q by ~eps * p, orders of magnitude beyond max|q0|; on the
    wide target q must also cross 16 from zero.  eps is scaled with the target's width."""
    eps = 0.15 * (WIDE if wide else 1.0)
    P, const, q0, npz, u, oq, oi = _case(D, init, wide, L, eps)
    got_q, got = _run(zs, impl, P, const, q0, npz, u, eps, L)
    _check_vs_oracle(got_q, got, oq, oi, q0, u,
                     "impl %d D %d init %g%s L %d" % (impl, D, init, " wide" if wide else "", L))


@pytest.mark.parametrize("D", [64, 1024])
def test_single_half_kick_pass_from_a_small_state(zs, D):
    """n_leapfrogs = 0 runs one per-pass fp16-split launch (impl 2, the default for L = 0)."""
    P, const, q0, npz, u, oq, oi = _case(D, 1e-3, False, 0, 0.15)
    x = T(q0)
    h = zs.HMC(step_size=0.15, n_leapfrogs=0)
    op, info = h.sample(_log_joint(zs, P, const), {}, {"x": x})
    assert h._impl == 2 and not h._res
    op(noise={"p": {"x": T(npz)}, "u": T(u)})
    op.synchronize()
    got = {k: N(getattr(info, k)) for k in ("acceptance_rate", "orig_hamiltonian",
                                            "hamiltonian", "orig_log_prob", "log_prob")}
    _check_vs_oracle(N(x), got, oq, oi, q0, u, "impl 2 D %d L 0" % D)


@pytest.mark.parametrize("impl", [0, 5])
def test_adaptive_warmup_from_a_small_state(zs, impl):
    """30 adaptive iterations (step-size search at t = 1 and t = mass_collect_iters, dual
    averaging, mass adaptation) from 1e-3 * N(0, 1) with identical injected noise.  The search
    probes are L = 1 trajectories from the small state, so the plane scale matters there first."""
    D, C, L, iters = 64, 200, 10, 30
    P, const = _problem(D)
    rng = np.random.RandomState(17)
    q0 = (1e-3 * rng.standard_normal((C, D))).astype(np.float32)
    noise_p = rng.standard_normal((iters, C, D)).astype(np.float32)
    noise_u = rng.random_sample((iters, C)).astype(np.float32)
    cfg = dict(step_size=0.1, n_leapfrogs=L, adapt_step_size=True, adapt_mass=True,
               target_acceptance_rate=0.8, mass_collect_iters=10, mass_decay=0.99)
    om = OM.DenseGaussian(P.astype(np.float32), None, const)
    oh = OH.HMC(**cfg)
    oq = [q0]
    _, oi = oh.step(oq, om.logp, om.grad, [noise_p[0]], noise_u[0], True, True)
    eps0_oracle = float(oi.step_size_used)

    def run(im):
        x = T(q0)
        h = zs.HMC(dense_impl=im, **cfg)
        op, info = h.sample(_log_joint(zs, P, const), {}, {"x": x})
        eps, acc = [], []
        for i in range(iters):
            op(adapt_step_size=True, adapt_mass=True,
               noise={"p": {"x": T(noise_p[i])}, "u": T(noise_u[i])})
            eps.append(float(h._state[7]))
            acc.append(float(info.acceptance_rate.mean()))
        op.synchronize()
        assert np.isfinite(N(x)).all()
        return np.array(eps), np.array(acc)
    eps_i, acc_i = run(impl)
    np.testing.assert_allclose(eps_i[0], eps0_oracle, rtol=1e-4,
                               err_msg="step size after the initial search, impl %d" % impl)
    if impl != 0:
        eps_0, acc_0 = run(0)
        np.testing.assert_allclose(eps_i[-1], eps_0[-1], rtol=0.1)
        assert abs(acc_i[-10:].mean() - acc_0[-10:].mean()) < 0.05, (acc_i, acc_0)


@pytest.mark.parametrize("impl,D", [(2, 64), (5, 64), (2, 1024), (5, 1024)])
def test_chains_of_very_different_magnitude_in_one_batch(zs, impl, D):
    """Half the chains at 1e-4 * N(0, 1), half at 1e2 * N(0, 1): the plane scale is set by the
    large chains, and the small ones must keep fp32 accuracy in every Hamiltonian."""
    P, const = _problem(D)
    C, L, eps = 128, 10, 0.1
    rng = np.random.RandomState(D + impl)
    mag = np.where(np.arange(C) % 2 == 0, 1e-4, 1e2)[:, None]
    q0 = (mag * rng.standard_normal((C, D))).astype(np.float32)
    npz = rng.standard_normal((C, D)).astype(np.float32)
    u = rng.random_sample(C).astype(np.float32)
    oq, oi = _oracle64(P, const, q0, npz, u, eps, L)
    got_q, got = _run(zs, impl, P, const, q0, npz, u, eps, L)
    np.testing.assert_allclose(got["orig_hamiltonian"], oi.orig_hamiltonian, rtol=1e-5, atol=0)
    np.testing.assert_allclose(got["hamiltonian"], oi.hamiltonian, rtol=1e-5, atol=0)


@pytest.mark.parametrize("impl,D", _IMPL_D)
def test_unstable_step_rejects_cleanly(zs, impl, D):
    """eps * sqrt(lambda_max(P)) = 4: the trajectory diverges (x ~14 per leapfrog step) but stays
    finite in fp32.  Every path must reject every chain with finite Hamiltonians and leave the
    chains where they were."""
    P, const = _problem(D)
    eps = float(4.0 / np.sqrt(np.linalg.eigvalsh(P).max()))
    C, L = 130, 10
    rng = np.random.RandomState(D + 3)
    q0 = rng.standard_normal((C, D)).astype(np.float32)
    npz = rng.standard_normal((C, D)).astype(np.float32)
    u = rng.random_sample(C).astype(np.float32)
    oq, oi = _oracle64(P, const, q0, npz, u, eps, L)
    assert np.isfinite(oi.hamiltonian).all() and (oi.acceptance_rate == 0).all()
    got_q, got = _run(zs, impl, P, const, q0, npz, u, eps, L)
    assert (got["acceptance_rate"] == 0).all()
    for k, v in got.items():
        assert np.isfinite(v).all(), "non-finite %s" % k
    np.testing.assert_array_equal(got_q, q0)


@pytest.mark.parametrize("bad", [np.inf, -np.inf, np.nan])
def test_linear_non_finite_row_stays_local(zs, bad):
    """zs.fused.linear takes its operand scale from max|h| ignoring NaN / inf: one non-finite
    row of h changes no bit of any other row of y."""
    rng = np.random.RandomState(8)
    R, K, J = 300, 64, 128
    h = rng.standard_normal((R, K)).astype(np.float32)
    W = (rng.standard_normal((J, K)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(J).astype(np.float32)
    clean = N(zs.fused.linear(T(h), T(W), T(b)))
    hb = h.copy()
    hb[7, 5] = bad
    y = N(zs.fused.linear(T(hb), T(W), T(b)))
    rows = np.arange(R) != 7
    np.testing.assert_array_equal(y[rows], clean[rows])
    assert not np.isfinite(y[7]).all()


def test_linear_all_zero_input_gives_the_bias(zs):
    rng = np.random.RandomState(9)
    R, K, J = 200, 64, 96
    W = (rng.standard_normal((J, K)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(J).astype(np.float32)
    y = N(zs.fused.linear(T(np.zeros((R, K), np.float32)), T(W), T(b)))
    np.testing.assert_array_equal(y, np.broadcast_to(b, (R, J)))


def _dense_pass_reference(q, p, P, b, mu, mass, eps, scale):
    """float64 restatement of one leapfrog pass (hmc.py:38-43, 352-364)."""
    g = b - q @ P
    pn = p + scale * eps * g
    qn = q + eps * pn / mass
    lp = 0.5 * ((q - mu) * g).sum(-1)
    k = 0.5 * (pn * pn / mass).sum(-1)
    return pn, qn, lp, k


@pytest.mark.parametrize("C,D,init", [(300, 512, 1.0), (1000, 1024, 1.0), (130, 64, 1.0),
                                      (515, 192, 1.0), (130, 64, 1e-3), (300, 1024, 1e-3)])
def test_trajectory_form_pass_vs_float64(zs, C, D, init):
    """One pass of impl 2's trajectory form through the C ABI against float64: the momentum, the
    position, the log-prob and kinetic partials, the planes of q_next, and plane-scale record 1
    (from a small state the planes of q_next must be written at a lower scale)."""
    from zhusuan_b200._lib import lib, ptr, stream
    rng = np.random.RandomState(C + D)
    P64, _ = OM.make_dense_gaussian_problem(D, seed=4)
    q = init * rng.standard_normal((C, D)); p = rng.standard_normal((C, D))
    mu = 0.3 * rng.standard_normal(D)
    mass = 0.5 + rng.random_sample(D)
    eps, scale = 0.07, 0.5
    P32 = P64.astype(np.float32)
    b = (P32.astype(np.float64) @ mu).astype(np.float32)
    qt, pt, mt, mut, bt = T(q), T(p), T(mass), T(mu), T(b)
    lj = zs.fused.GaussianLogJoint(P64, device="cuda")._zsb_fused
    state = torch.zeros(16, device="cuda"); state[7] = eps
    nt = lib.load().zsb_hmc_dense_ntiles(D, 1)
    qn = torch.empty_like(qt); pn = torch.empty_like(pt)
    lpp = torch.zeros(nt * C, device="cuda"); kp = torch.zeros(nt * C, device="cuda")
    lp = torch.empty(C, device="cuda"); k = torch.empty(C, device="cuda")
    planes = torch.empty(2, C, D, dtype=torch.float16, device="cuda")
    nplanes = torch.empty_like(planes)
    scales = torch.zeros(8 + 4 * 3, device="cuda")
    scales[3], scales[4], scales[5] = lj["sP"], lj["P_inf"], float(np.abs(b).max())
    s = stream()
    lib.call("zsb_hmc_dense_traj_prepare_f32", ptr(qt), ptr(pt), ptr(mt), ptr(planes),
             ptr(scales), C, D, s)
    lib.call("zsb_hmc_dense_leapfrog_h16_pass_f32", ptr(qt), ptr(planes), ptr(qn), ptr(nplanes),
             ptr(pt), ptr(pn), ptr(lj["P_h16"]), ptr(lj["P_l16"]), ptr(scales), 0, ptr(bt),
             ptr(mut), ptr(mt), ptr(state), scale, ptr(lpp), ptr(kp), C, D, s)
    lib.call("zsb_hmc_dense_finish_f32", ptr(lpp), ptr(kp), nt, C, 0.0, ptr(lp), ptr(k), s)
    torch.cuda.synchronize()
    q32 = q.astype(np.float32).astype(np.float64)
    p32 = p.astype(np.float32).astype(np.float64)
    rpn, rqn, rlp, rk = _dense_pass_reference(
        q32, p32, P32.astype(np.float64), b.astype(np.float64),
        mu.astype(np.float32).astype(np.float64), mass.astype(np.float32).astype(np.float64),
        np.float32(eps), scale)
    gscale = np.abs(q32 @ P32.astype(np.float64)).max() + np.abs(b).max()
    np.testing.assert_allclose(N(pn), rpn, rtol=1e-5, atol=1e-5 * gscale)
    np.testing.assert_allclose(N(qn), rqn, rtol=1e-5, atol=1e-5 * max(gscale, np.abs(rqn).max()))
    np.testing.assert_allclose(N(lp), rlp, rtol=1e-5, atol=1e-5 * np.abs(rlp).max())
    np.testing.assert_allclose(N(k), rk, rtol=1e-5)
    sc = N(scales)
    sq0, sq1 = float(sc[8]), float(sc[12])
    assert sq0 == float(sc[0]) and 2 ** 11 <= np.abs(q32).max() * sq0 < 2 ** 12
    rec = (N(nplanes[0]).astype(np.float64) + N(nplanes[1]).astype(np.float64)) / sq1
    np.testing.assert_allclose(rec, N(qn).astype(np.float64), rtol=1e-6,
                               atol=1e-6 * np.abs(N(qn)).max())
    assert np.abs(N(qn)).max() * sq1 < 65520                    # q_next fits its planes
    assert sc[14] == np.abs(N(qn)).max()                        # record 1: max|q_next|
    if init < 1:
        assert sq1 < sq0
    else:
        assert sq1 == sq0


def _records(h, L):
    sc = N(h._scales)
    rec = sc[8:8 + 4 * (L + 1)].reshape(L + 1, 4)
    return rec[:, 0], rec[:, 1], rec[1:, 3].view(np.uint32)


@pytest.mark.parametrize("init,eps", [(1.0, 0.55), (1e-3, 0.15)])
def test_resident_spare_planes_only_where_the_planes_overflow(zs, init, eps):
    """dense_impl 5 keeps one plane scale as long as the planes fit, even where the a-priori bound
    asks for a spare copy: from posterior-scale states with a step near the stability limit
    (eps * sqrt(lambda_max) = 1.8) the bound is reached but nothing overflows, so every pass reads
    planes at the prepare's scale.  From a small state the planes do overflow and the next pass
    reads the spare copy.  Both against the float64 oracle."""
    D, C, L = 1024, 130, 10
    P, const = _problem(D)
    rng = np.random.RandomState(21)
    q0 = (init * rng.standard_normal((C, D))).astype(np.float32)
    npz = rng.standard_normal((C, D)).astype(np.float32)
    u = rng.random_sample(C).astype(np.float32)
    oq, oi = _oracle64(P, const, q0, npz, u, eps, L)
    x = T(q0)
    h = zs.HMC(step_size=eps, n_leapfrogs=L, dense_impl=5)
    op, info = h.sample(_log_joint(zs, P, const), {}, {"x": x})
    op(noise={"p": {"x": T(npz)}, "u": T(u)})
    op.synchronize()
    sq, sq_alt, flag = _records(h, L)
    assert (sq_alt < sq).any()                                  # a spare copy was written
    if init == 1.0:
        assert not flag.any() and (sq == sq[0]).all()
    else:
        assert flag.any()
    got = {k: N(getattr(info, k)) for k in ("acceptance_rate", "orig_hamiltonian",
                                            "hamiltonian", "orig_log_prob", "log_prob")}
    _check_vs_oracle(N(x), got, oq, oi, q0, u, "impl 5 init %g eps %g" % (init, eps))
