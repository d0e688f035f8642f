"""GPU parity: HMC through the drop-in API vs the CPU oracle / committed
golden vectors (injected noise).  Bar (north_star): accept/reject decisions
identical given identical uniforms, per-chain log-prob within 1e-5 relative."""
import os

import numpy as np
import pytest
import torch

from oracle import hmc as OH
from oracle import models as OM

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def T(a, dtype=torch.float32):
    return torch.tensor(np.asarray(a), dtype=dtype, device="cuda")


def N(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def _cfg(g):
    return dict(step_size=float(g["cfg_step_size"]),
                n_leapfrogs=int(g["cfg_n_leapfrogs"]), adapt_step_size=True,
                target_acceptance_rate=float(g["cfg_target_acceptance_rate"]),
                adapt_mass=True,
                mass_collect_iters=int(g["cfg_mass_collect_iters"]),
                mass_decay=float(g["cfg_mass_decay"]))


def _replay(zs, g, model, expect_kind, q_tol=2e-5, **hmc_kw):
    x = T(g["q0"])
    h = zs.HMC(**_cfg(g), **hmc_kw)
    op, info = h.sample(model, {}, {"x": x})
    kind = h._fused["kind"] if h._fused else "generic"
    assert kind == expect_kind
    n_mismatch = 0
    for i in range(g["q"].shape[0]):
        adapt = i < int(g["n_adapt"])
        op(adapt_step_size=adapt, adapt_mass=adapt,
           noise={"p": {"x": T(g["noise_p"][i])}, "u": T(g["noise_u"][i])})
        acc = N(info.acceptance_rate)
        accept = (g["noise_u"][i] < acc).astype(np.int32)
        bad = accept != g["accept"][i]
        # a flip is only tolerable when u sits within rounding of acc
        assert np.all(np.abs(g["noise_u"][i] - g["acc"][i])[bad] < 1e-5)
        n_mismatch += int(bad.sum())
        np.testing.assert_allclose(acc, g["acc"][i], rtol=1e-4, atol=2e-5)
        np.testing.assert_allclose(N(info.orig_log_prob), g["lp0"][i],
                                   rtol=1e-5, atol=1e-4)
        np.testing.assert_allclose(N(info.log_prob), g["lp"][i], rtol=1e-5,
                                   atol=1e-4)
        np.testing.assert_allclose(N(info.orig_hamiltonian), g["h0"][i],
                                   rtol=1e-5, atol=1e-4)
        np.testing.assert_allclose(N(info.init_momentum["x"]), g["p0"][i],
                                   rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(N(x), g["q"][i], rtol=q_tol, atol=q_tol)
        np.testing.assert_allclose(float(info.updated_step_size),
                                   g["step_size"][i], rtol=1e-4)
        if "eps_used" in g.files:       # internals the reference's HMCInfo does not expose
            np.testing.assert_allclose(float(h._state[7]), g["eps_used"][i],
                                       rtol=1e-5)
            np.testing.assert_allclose(N(h._mass[0]), g["mass"][i], rtol=1e-3)
    op.synchronize()
    assert n_mismatch == 0
    if "n_search_iters" in g.files:
        assert h.n_search_iters == int(g["n_search_iters"])
    return h


# ---- vectors written by the reference's own hmc.py (oracle/tf_shim/make_ref_golden.py) ----------
def test_reference_run_diag_fused(zs):
    g = np.load(os.path.join(GOLD, "ref_hmc_diag.npz"))
    D = g["std"].shape[0]

    @zs.meta_bayesian_net()
    def gaussian(n_x, stdev, n_particles):
        bn = zs.BayesianNet()
        bn.normal('x', torch.zeros(n_x, device="cuda"), std=stdev,
                  n_samples=n_particles, group_ndims=1)
        return bn
    _replay(zs, g, gaussian(D, T(g["std"]), g["q0"].shape[0]), "diag_normal")


@pytest.mark.parametrize("name,impl,q_tol", [
    ("ref_hmc_dense32", 0, 5e-5), ("ref_hmc_dense32", 1, 5e-5),
    ("ref_hmc_dense64", 0, 5e-5), ("ref_hmc_dense64", 1, 5e-5),
    ("ref_hmc_dense64", 2, 1e-4), ("ref_hmc_dense64", 5, 1e-4)])
def test_reference_run_dense(zs, name, impl, q_tol):
    """16 chained adaptive iterations of the reference's HMC (step-size search, dual averaging,
    mass adaptation, diverging and healthy iterations) replayed on each dense kernel."""
    g = np.load(os.path.join(GOLD, name + ".npz"))
    lj = zs.fused.GaussianLogJoint(g["P"], mean=g["mu"],
                                   log_det_cov=-2 * float(g["const"])
                                   - g["P"].shape[0] * np.log(2 * np.pi))
    _replay(zs, g, lj, "dense_gaussian", q_tol=q_tol, dense_impl=impl)


def test_golden_diag_fused_through_bayesian_net(zs):
    g = np.load(os.path.join(GOLD, "hmc_diag.npz"))
    D = g["std"].shape[0]

    @zs.meta_bayesian_net()
    def gaussian(n_x, stdev, n_particles):     # toy_examples/gaussian.py:15-20
        bn = zs.BayesianNet()
        bn.normal('x', torch.zeros(n_x, device="cuda"), std=stdev,
                  n_samples=n_particles, group_ndims=1)
        return bn
    _replay(zs, g, gaussian(D, T(g["std"]), g["q0"].shape[0]), "diag_normal")


def test_golden_diag_generic_callable(zs):
    g = np.load(os.path.join(GOLD, "hmc_diag.npz"))
    std = T(g["std"])

    def log_joint(obs):
        return zs.distributions.Normal(torch.zeros_like(std), std=std,
                                       group_ndims=1).log_prob(obs['x'])
    _replay(zs, g, log_joint, "generic")


def test_golden_dense_fused_simt(zs):
    g = np.load(os.path.join(GOLD, "hmc_dense.npz"))
    lj = zs.fused.GaussianLogJoint(g["P"], mean=g["mu"],
                                   log_det_cov=-2 * float(g["const"])
                                   - g["P"].shape[0] * np.log(2 * np.pi))
    _replay(zs, g, lj, "dense_gaussian", q_tol=5e-5, dense_impl=0)


def test_golden_dense_generic(zs):
    g = np.load(os.path.join(GOLD, "hmc_dense.npz"))
    lj = zs.fused.GaussianLogJoint(g["P"], mean=g["mu"],
                                   log_det_cov=-2 * float(g["const"])
                                   - g["P"].shape[0] * np.log(2 * np.pi))
    _replay(zs, g, lambda obs: lj(obs), "generic", q_tol=5e-5)


def test_multi_latent_two_chain_axes_generic(zs):
    """Two latents, chain axes [3, 5], data axes [4] and [2, 3]."""
    rng = np.random.RandomState(0)
    s1 = (0.5 + rng.random_sample(4)).astype(np.float32)
    s2 = (0.5 + rng.random_sample((2, 3))).astype(np.float32)
    a0 = rng.standard_normal((3, 5, 4)).astype(np.float32)
    b0 = rng.standard_normal((3, 5, 2, 3)).astype(np.float32)

    class Two(object):
        def logp(self, q):
            from oracle import distributions as OD
            return (OD.normal_log_prob(q[0], 0, np.log(s1), 1)
                    + OD.normal_log_prob(q[1], 1.0, np.log(s2), 2))

        def grad(self, q):
            return [(-q[0] / s1 ** 2).astype(np.float32),
                    (-(q[1] - 1.0) / s2 ** 2).astype(np.float32)]

    @zs.meta_bayesian_net()
    def model():
        bn = zs.BayesianNet()
        bn.normal('a', torch.zeros(4, device="cuda"), std=T(s1), group_ndims=1,
                  n_samples=None)
        bn.normal('b', torch.ones(2, 3, device="cuda"), std=T(s2),
                  group_ndims=2)
        return bn
    oh = OH.HMC(step_size=0.05, n_leapfrogs=4, adapt_step_size=True,
                adapt_mass=True, mass_collect_iters=2)
    h = zs.HMC(step_size=0.05, n_leapfrogs=4, adapt_step_size=True,
               adapt_mass=True, mass_collect_iters=2)
    a, b = T(a0), T(b0)
    op, info = h.sample(model(), {}, {"a": a, "b": b})
    assert h._fused is None
    oq = [a0, b0]
    m = Two()
    for i in range(6):
        na = rng.standard_normal(a0.shape).astype(np.float32)
        nb = rng.standard_normal(b0.shape).astype(np.float32)
        u = rng.random_sample((3, 5)).astype(np.float32)
        oq, oi = oh.step(oq, m.logp, m.grad, [na, nb], u, True, True)
        op(adapt_step_size=True, adapt_mass=True,
           noise={"p": {"a": T(na), "b": T(nb)}, "u": T(u)})
        np.testing.assert_allclose(N(info.acceptance_rate),
                                   oi.acceptance_rate, rtol=1e-4, atol=2e-5)
        np.testing.assert_allclose(N(a), oq[0], rtol=2e-5, atol=2e-5)
        np.testing.assert_allclose(N(b), oq[1], rtol=2e-5, atol=2e-5)
        np.testing.assert_allclose(float(info.updated_step_size),
                                   oi.updated_step_size, rtol=1e-4)
    assert tuple(info.acceptance_rate.shape) == (3, 5)


def test_error_contract(zs):
    with pytest.raises(ValueError, match="If adapt mass is set"):
        zs.HMC(adapt_mass=True)
    h = zs.HMC()
    with pytest.raises(TypeError, match=r"latent\['x'\] is not a"):
        h.sample(lambda o: o['x'].sum(-1), {}, {"x": np.zeros((2, 3))})
    h = zs.HMC()
    with pytest.raises(ValueError, match="log joint"):
        h.sample(lambda o: o['x'].sum(), {}, {"x": torch.zeros(2, 3,
                                                               device="cuda")})
    # check_numerics (hmc.py:51-53): non-finite old log-prob
    x = torch.full((4, 3), float("inf"), device="cuda")
    h = zs.HMC(step_size=0.1, n_leapfrogs=2)
    op, _ = h.sample(lambda o: -(o['x'] ** 2).sum(-1), {}, {"x": x})
    op()
    with pytest.raises(FloatingPointError, match="old_log_prob has numeric"):
        op.synchronize()


def test_non_finite_new_state_is_rejected(zs):
    """hmc.py:56-59: non-finite acceptance / new log-prob -> acc = 0."""
    x = T(np.ones((8, 2)))
    h = zs.HMC(step_size=1e6, n_leapfrogs=3)
    op, info = h.sample(lambda o: -(o['x'] ** 4).sum(-1), {}, {"x": x})
    op()
    op.synchronize()
    assert float(info.acceptance_rate.max()) == 0.0
    np.testing.assert_array_equal(N(x), np.ones((8, 2), np.float32))


def test_philox_sampling_recovers_target_std(zs):
    """gaussian.py end-to-end with in-kernel RNG: per-dimension sample std
    within 5% of the target after adaptation (statistical)."""
    D, C = 10, 2000
    std = (1.0 / (1.0 + np.arange(D))).astype(np.float32)

    @zs.meta_bayesian_net()
    def gaussian():
        bn = zs.BayesianNet()
        bn.normal('x', torch.zeros(D, device="cuda"), std=T(std),
                  n_samples=C, group_ndims=1)
        return bn
    x = torch.zeros(C, D, device="cuda")
    h = zs.HMC(step_size=1e-3, n_leapfrogs=5, adapt_step_size=True,
               adapt_mass=True, target_acceptance_rate=0.9, seed=42)
    op, info = h.sample(gaussian(), {}, {"x": x})
    samples = []
    for i in range(200):
        op(adapt_step_size=i < 50, adapt_mass=i < 50)
        if i >= 100:
            samples.append(x.clone())
    s = torch.cat(samples).std(0).cpu().numpy()
    np.testing.assert_allclose(s, std, rtol=0.05)
    assert 0.5 < float(info.acceptance_rate.mean()) <= 1.0


def test_dense_full_size_energy_conservation(zs):
    """BASELINE config-2 size (65 536 chains x 1024 dims) property test: with
    a small step the leapfrog integrator conserves H (|dH| << 1), the chain
    moves, and two identical runs are bit-identical (determinism)."""
    D, C = 1024, 65536
    P, const = OM.make_dense_gaussian_problem(D, seed=2)
    lj = zs.fused.GaussianLogJoint(P)
    outs = []
    for rep in range(2):
        torch.manual_seed(3)
        x = torch.randn(C, D, device="cuda")
        x0 = x.clone()
        h = zs.HMC(step_size=0.01, n_leapfrogs=3, seed=7, dense_impl=0)
        op, info = h.sample(lj, {}, {"x": x})
        op()
        op.synchronize()
        dH = (info.hamiltonian - info.orig_hamiltonian).abs()
        assert float(dH.max()) < 0.05
        assert float(info.acceptance_rate.min()) > 0.9
        assert float((x - x0).abs().max()) > 1e-3
        outs.append((x.clone(), info.acceptance_rate.clone()))
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.equal(outs[0][1], outs[1][1])
    # log-prob of the new state equals a float64 evaluation on a chain subset
    xs = outs[0][0][:64].double().cpu().numpy()
    ref = -0.5 * np.einsum('ci,ij,cj->c', xs, P, xs) + const
    op()   # one more iteration: orig_log_prob now describes outs' state
    op.synchronize()
    np.testing.assert_allclose(N(info.orig_log_prob[:64]), ref, rtol=1e-5)


def _dense_pass_reference(q, p, P, b, mu, mass, eps, scale):
    """float64 restatement of one pass of the leapfrog loop body for the dense
    Gaussian (hmc.py:38-43, 352-364): g = b - qP; p' = p + scale*eps*g;
    q' = q + eps*p'/m; lp = 1/2 (q-mu).g; K = 1/2 sum p'^2/m."""
    g = b - q @ P
    pn = p + scale * eps * g
    qn = q + eps * pn / mass
    lp = 0.5 * ((q - mu) * g).sum(-1)
    k = 0.5 * (pn * pn / mass).sum(-1)
    return pn, qn, lp, k


@pytest.mark.parametrize("impl", [0, 1, 2])
@pytest.mark.parametrize("C,D", [(300, 512), (24, 32), (129, 288), (1000, 1024),
                                 (130, 64), (515, 192)])
def test_dense_single_pass_vs_float64(zs, impl, C, D):
    """One fused GEMM+leapfrog pass through the C ABI vs float64, for the SIMT
    (impl 0) and wgmma 3xTF32 (impl 1) kernels, including ragged M / N tiles.
    Bar: per-evaluation log-prob and gradient-derived p within 1e-5 relative."""
    from zhusuan_b200._lib import lib, ptr, stream
    if impl >= 2 and D % 64:
        pytest.skip("fp16-split path needs D % 64 == 0")
    rng = np.random.RandomState(C + D)
    P64, _ = OM.make_dense_gaussian_problem(D, seed=4)
    q = rng.standard_normal((C, D)); p = rng.standard_normal((C, D))
    mu = 0.3 * rng.standard_normal(D)
    mass = 0.5 + rng.random_sample(D)
    eps, scale = 0.07, 0.5
    P32 = P64.astype(np.float32)
    hi = (P32.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
    lo = (P32 - hi).astype(np.float32)
    b = (P32.astype(np.float64) @ mu).astype(np.float32)
    qt, pt, mt, mut, bt = T(q), T(p), T(mass), T(mu), T(b)
    Pt, Pl = (T(hi), T(lo)) if impl == 1 else (T(P32), None)
    state = torch.zeros(16, device="cuda"); state[7] = eps
    nt = lib.load().zsb_hmc_dense_ntiles(D, min(impl, 1))
    qn = torch.empty_like(qt); pn = torch.empty_like(pt)
    qlo = torch.empty_like(qt); qnlo = torch.empty_like(qt)
    lpp = torch.zeros(nt * C, device="cuda"); kp = torch.zeros(nt * C, device="cuda")
    lp = torch.empty(C, device="cuda"); k = torch.empty(C, device="cuda")
    s = stream()
    if impl == 2:   # pass 0 of a trajectory, plane-scale records laid out as HMC._plane_scales
        lj = zs.fused.GaussianLogJoint(P64, device="cuda")._zsb_fused
        planes = torch.empty(2, C, D, dtype=torch.float16, device="cuda")
        nplanes = torch.empty_like(planes)
        scales = torch.zeros(8 + 4 * 3, device="cuda")
        scales[3], scales[4], scales[5] = lj["sP"], lj["P_inf"], float(np.abs(b).max())
        lib.call("zsb_hmc_dense_traj_prepare_f32", ptr(qt), ptr(pt), ptr(mt), ptr(planes),
                 ptr(scales), C, D, s)
        lib.call("zsb_hmc_dense_leapfrog_h16_pass_f32", ptr(qt), ptr(planes), ptr(qn),
                 ptr(nplanes), ptr(pt), ptr(pn), ptr(lj["P_h16"]),
                 ptr(lj["P_l16"]), ptr(scales), 0, ptr(bt), ptr(mut), ptr(mt),
                 ptr(state), scale, ptr(lpp), ptr(kp), C, D, s)
    else:
        if impl == 1:
            lib.call("zsb_hmc_dense_split_lo_f32", ptr(qt), ptr(qlo),
                     qt.numel(), s)
        lib.call("zsb_hmc_dense_leapfrog_f32", ptr(qt), ptr(qlo), ptr(qn),
                 ptr(qnlo), ptr(pt), ptr(pn), ptr(Pt), ptr(Pl), ptr(bt),
                 ptr(mut), ptr(mt), ptr(state), scale, ptr(lpp), ptr(kp), C, D,
                 impl, s)
    lib.call("zsb_hmc_dense_finish_f32", ptr(lpp), ptr(kp), nt, C, 0.0,
             ptr(lp), ptr(k), s)
    torch.cuda.synchronize()
    q32 = q.astype(np.float32).astype(np.float64)
    p32 = p.astype(np.float32).astype(np.float64)
    rpn, rqn, rlp, rk = _dense_pass_reference(
        q32, p32, P32.astype(np.float64), b.astype(np.float64),
        mu.astype(np.float32).astype(np.float64),
        mass.astype(np.float32).astype(np.float64), np.float32(eps), scale)
    gscale = np.abs(q32 @ P32.astype(np.float64)).max()
    np.testing.assert_allclose(N(pn), rpn, rtol=1e-5, atol=1e-5 * gscale)
    np.testing.assert_allclose(N(qn), rqn, rtol=1e-5, atol=1e-5 * gscale)
    np.testing.assert_allclose(N(lp), rlp, rtol=1e-5, atol=1e-5 * np.abs(rlp).max())
    np.testing.assert_allclose(N(k), rk, rtol=1e-5)
    if impl == 1:   # q_next_lo is exactly the TF32 residual of q_next
        qn32 = N(qn)
        res = qn32 - (qn32.view(np.uint32) & np.uint32(0xFFFFE000)).view(np.float32)
        np.testing.assert_array_equal(N(qnlo), res)
    if impl == 2:   # the planes reconstruct q_next * sq_1 to ~2^-22 relative
        sq = float(scales[8 + 4])     # record 1: the scale of q_next's planes
        rec = (N(nplanes[0]).astype(np.float64) + N(nplanes[1]).astype(np.float64)) / sq
        np.testing.assert_allclose(rec, N(qn).astype(np.float64), rtol=1e-6,
                                   atol=1e-6 * np.abs(N(qn)).max())
        sq0 = float(scales[8])        # record 0: the scale of q's planes
        assert 2 ** 11 <= np.abs(q).max() * sq0 < 2 ** 12


def test_golden_dense_fused_tc(zs):
    g = np.load(os.path.join(GOLD, "hmc_dense.npz"))
    lj = zs.fused.GaussianLogJoint(g["P"], mean=g["mu"],
                                   log_det_cov=-2 * float(g["const"])
                                   - g["P"].shape[0] * np.log(2 * np.pi))
    _replay(zs, g, lj, "dense_gaussian", q_tol=1e-4, dense_impl=1)


# Tolerances after a 50-step trajectory (measured in round 2 on every kernel, restart protocol):
# the Hamiltonian of the proposal stays within 5e-6 of float64 on all kernels (energy is conserved
# to first order, so position errors cancel between log p and the kinetic term) -> 1e-5 as for a
# single evaluation; the log-prob ALONE does not enjoy that cancellation (a position error dq
# moves it by g.dq): up to 1.5e-5 of max|log p| at D = 64 -> 5e-5.
H1_RTOL = 1e-5
LP1_RTOL = 5e-5


def _replay_big(zs, name, impl):
    """Replay tests/golden/<name>.npz (L = 50, adaptive, mass != 1, both step-size searches,
    diverging and healthy iterations; protocol in make_golden.py BIG: every iteration starts
    from a prescribed, re-generated state, the sampler's adaptation state carries over).

    Budget: the fixture carries the float32 oracle's outputs and a float64 re-evaluation of each
    iteration.  The CUDA path must keep |acc - acc64| below u_guard -- every stored uniform sits
    >= u_guard (pushed ones 2 x u_guard) away from acc64, so EVERY accept decision must then be
    reproduced -- the Hamiltonians / log-probs of a single evaluation within 1e-5, after the
    trajectory within H1_RTOL (log-prob alone: LP1_RTOL).  All iterations are tabulated first (stdout, run with -s), then
    asserted."""
    import sys
    sys.path.insert(0, GOLD)
    import make_golden as MG
    g = np.load(os.path.join(GOLD, name + ".npz"))
    cfg = dict(MG.BIG[name])
    for k, v in cfg.items():
        assert float(g["cfg_" + k]) == float(v), "fixture made with another BIG config"
    D, C, L = cfg["D"], cfg["C"], cfg["L"]
    P, const, mu, chol = MG.big_problem(cfg)
    np.testing.assert_allclose(np.abs(P).sum(), float(g["P_checksum"]), rtol=1e-12)
    np.testing.assert_allclose(np.abs(MG.big_state(cfg, 0).astype(np.float64)).sum(),
                               float(g["q0_checksum"]), rtol=1e-9)
    lj = zs.fused.GaussianLogJoint(P, mean=mu, log_det_cov=-2 * const - D * np.log(2 * np.pi))
    x = T(MG.big_state(cfg, 0))
    h = zs.HMC(step_size=cfg["eps0"], n_leapfrogs=L, adapt_step_size=True, adapt_mass=True,
               mass_collect_iters=cfg["mci"], dense_impl=impl)
    op, info = h.sample(lj, {}, {"x": x})
    assert h._fused["kind"] == "dense_gaussian"
    floor = float(np.abs(g["acc"] - g["acc64"]).max())
    stride = D // 16
    rel = lambda a, b: float(np.abs(a / b - 1).max()) if a.size else 0.0
    rows = []
    for i in range(cfg["iters"]):
        adapt = i < cfg["n_adapt"]
        x.copy_(T(MG.big_state(cfg, i)))        # the caller assigns the latent variable
        op(adapt_step_size=adapt, adapt_mass=adapt,
           noise={"p": {"x": T(MG.big_noise(cfg, i))}, "u": T(g["noise_u"][i])})
        acc = N(info.acceptance_rate)
        live = g["acc64"][i] > 1e-6              # chains whose proposal is not hopeless
        xq = N(x)
        lpmax = np.abs(g["lp0"][i]).max()
        rows.append(dict(
            i=i, eps=float(h._state[7]), eps_err=abs(float(h._state[7]) / g["eps_used"][i] - 1),
            acc_err=float(np.abs(acc - g["acc64"][i]).max()),
            flips=int(((g["noise_u"][i] < acc).astype(np.int32) != g["accept"][i]).sum()),
            h0_err=rel(N(info.orig_hamiltonian), g["h0_64"][i]),
            h1_err=rel(N(info.hamiltonian)[live], g["h1_64"][i][live]),
            lp0_err=float(np.abs(N(info.orig_log_prob) - g["lp0"][i]).max() / lpmax),
            lp_err=float(np.abs(N(info.log_prob) - g["lp"][i]).max() / lpmax),
            q_err=float(np.abs(xq[:, ::stride] - g["q_sub"][i]).max()),
            qsum_err=float(np.abs(xq.astype(np.float64).sum(1) - g["q_rowsum"][i]).max()),
            step_err=abs(float(info.updated_step_size) / g["step_size"][i] - 1),
            mass_err=rel(N(h._mass[0]), g["mass"][i]), n_live=int(live.sum())))
    op.synchronize()
    print("\nreplay %s impl %d (float32-oracle acceptance floor %.2e, u_guard %.1e)" % (
        name, impl, floor, cfg["u_guard"]))
    print(" it   eps     eps_err  acc_err  flips live h0_err   h1_err   lp0_err  lp_err   "
          "q_err    step_err mass_err")
    for r in rows:
        print(" %2d %7.4f %8.1e %8.1e %3d  %4d %8.1e %8.1e %8.1e %8.1e %8.1e %8.1e %8.1e" % (
            r["i"], r["eps"], r["eps_err"], r["acc_err"], r["flips"], r["n_live"], r["h0_err"],
            r["h1_err"], r["lp0_err"], r["lp_err"], r["q_err"], r["step_err"], r["mass_err"]))
    for r in rows:
        msg = "%s impl %d iteration %d: %r" % (name, impl, r["i"], r)
        assert r["eps_err"] < 1e-4, msg
        assert r["acc_err"] <= cfg["u_guard"], msg
        assert r["flips"] == 0, msg
        assert r["h0_err"] < 1e-5 and r["lp0_err"] < 1e-5, msg
        assert r["h1_err"] < H1_RTOL and r["lp_err"] < LP1_RTOL, msg
        assert r["q_err"] < 2e-4 * max(1.0, float(np.abs(g["q_sub"][r["i"]]).max())), msg
        assert r["step_err"] < 1e-3 and r["mass_err"] < 2e-4, msg
    assert h.n_search_iters == int(g["n_search_iters"])
    return h


@pytest.mark.parametrize("impl", [0, 1, 2, 5])
def test_golden_dense64_l50_adaptive(zs, impl):
    """D = 64, 160 chains (ragged tile), L = 50, 24 adaptive iterations on the SIMT, 3xTF32 and
    fp16-split (the benchmarked) kernels vs the oracle."""
    _replay_big(zs, "hmc_dense64", impl)


@pytest.mark.parametrize("impl", [2, 5])
def test_golden_dense1024_l50_adaptive(zs, impl):
    """The benchmark configuration's shape (D = 1024, L = 50, step + mass adaptation) at 320
    chains on the benchmarked kernels: impl 2 (fp16-split, one launch per pass) and impl 5 (the
    whole trajectory on the plane state) vs the oracle -- accept decisions, Hamiltonians, step
    sizes, mass."""
    _replay_big(zs, "hmc_dense1024", impl)


def test_dense_tc_vs_simt_full_size(zs):
    """65 536 x 1024, L=3: the tensor-core and SIMT paths agree on the
    per-chain Hamiltonians to 1e-5 relative and make identical MH decisions
    except where u is within rounding of acc."""
    D, C = 1024, 65536
    P, const = OM.make_dense_gaussian_problem(D, seed=2)
    res = []
    for impl in (0, 1, 2):
        lj = zs.fused.GaussianLogJoint(P)
        torch.manual_seed(3)
        x = torch.randn(C, D, device="cuda")
        h = zs.HMC(step_size=0.2, n_leapfrogs=3, seed=7, dense_impl=impl)
        op, info = h.sample(lj, {}, {"x": x})
        op()
        op.synchronize()
        res.append((N(info.hamiltonian), N(info.orig_hamiltonian),
                    N(info.acceptance_rate), N(x)))
    for k in (1, 2):
        np.testing.assert_allclose(res[k][1], res[0][1], rtol=1e-5)
        np.testing.assert_allclose(res[k][0], res[0][0], rtol=1e-5)
        np.testing.assert_allclose(res[k][2], res[0][2], rtol=0, atol=2e-3)
        moved0 = np.abs(res[0][3]).sum(1); moved1 = np.abs(res[k][3]).sum(1)
        frac_diff = np.mean(np.abs(moved0 - moved1) > 1e-2 * np.abs(moved0))
        assert frac_diff < 1e-3


@pytest.mark.parametrize("L", [0, 1, 2])
def test_leapfrog_count_edges_all_paths(zs, L):
    """n_leapfrogs = 0 / 1 / 2 (hmc.py:352-364: L+1 passes, half kicks first and
    last; L = 0 is a single half-kick pass) on the fused-diag, generic, SIMT-dense
    and tensor-core dense paths vs the oracle."""
    rng = np.random.RandomState(10 + L)
    # diagonal
    D, C = 12, 20
    std = (0.5 + rng.random_sample(D)).astype(np.float32)
    q0 = rng.standard_normal((C, D)).astype(np.float32)
    npz = rng.standard_normal((C, D)).astype(np.float32)
    u = rng.random_sample(C).astype(np.float32)
    om = OM.DiagGaussian(np.zeros(D, np.float32), std)
    oq, oi = OH.HMC(step_size=0.1, n_leapfrogs=L).step([q0], om.logp, om.grad, [npz], u)

    @zs.meta_bayesian_net()
    def gaussian():
        bn = zs.BayesianNet()
        bn.normal('x', torch.zeros(D, device="cuda"), std=T(std), group_ndims=1)
        return bn

    def lj(obs):
        return zs.distributions.Normal(torch.zeros(D, device="cuda"), std=T(std),
                                       group_ndims=1).log_prob(obs['x'])
    for model, kind in ((gaussian(), "diag_normal"), (lj, "generic")):
        x = T(q0)
        h = zs.HMC(step_size=0.1, n_leapfrogs=L)
        op, info = h.sample(model, {}, {"x": x})
        assert (h._fused["kind"] if h._fused else "generic") == kind
        op(noise={"p": {"x": T(npz)}, "u": T(u)})
        np.testing.assert_allclose(N(info.acceptance_rate), oi.acceptance_rate, rtol=1e-4, atol=1e-5)
        np.testing.assert_allclose(N(x), oq[0], rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(N(info.log_prob), oi.log_prob, rtol=1e-5, atol=1e-4)
    # dense: D = 64 so that all three kernels are legal
    D, C = 64, 40
    P, const = OM.make_dense_gaussian_problem(D, seed=6)
    q0 = rng.standard_normal((C, D)).astype(np.float32)
    npz = rng.standard_normal((C, D)).astype(np.float32)
    u = rng.random_sample(C).astype(np.float32)
    om = OM.DenseGaussian(P.astype(np.float32), None, const)
    oq, oi = OH.HMC(step_size=0.15, n_leapfrogs=L).step([q0], om.logp, om.grad, [npz], u)
    for impl in (0, 1, 2, 5):
        x = T(q0)
        h = zs.HMC(step_size=0.15, n_leapfrogs=L, dense_impl=impl)
        op, info = h.sample(zs.fused.GaussianLogJoint(P), {}, {"x": x})
        op(noise={"p": {"x": T(npz)}, "u": T(u)})
        np.testing.assert_allclose(N(info.acceptance_rate), oi.acceptance_rate, rtol=2e-4, atol=2e-5)
        np.testing.assert_allclose(N(x), oq[0], rtol=2e-5, atol=2e-5)
        np.testing.assert_allclose(N(info.hamiltonian), oi.hamiltonian, rtol=1e-5, atol=1e-4)


def test_single_chain_and_tiny_shapes(zs):
    """1 chain x 1 dim (generic) and 1 chain x 16 dims (SIMT dense): nothing
    assumes a multiple of the tile size."""
    x = torch.zeros(1, 1, device="cuda")
    h = zs.HMC(step_size=0.3, n_leapfrogs=3, seed=1)
    op, info = h.sample(lambda o: -0.5 * (o['x'] ** 2).sum(-1), {}, {"x": x})
    for _ in range(5):
        op()
    op.synchronize()
    assert tuple(info.acceptance_rate.shape) == (1,) and torch.isfinite(x).all()
    P, _ = OM.make_dense_gaussian_problem(16, seed=1)
    y = torch.randn(1, 16, device="cuda")
    h = zs.HMC(step_size=0.1, n_leapfrogs=2, seed=2)
    op, info = h.sample(zs.fused.GaussianLogJoint(P), {}, {"x": y})
    assert h._impl == 0
    op(); op.synchronize()
    ref = -0.5 * N(y).astype(np.float64) @ P @ N(y).astype(np.float64).T
    assert torch.isfinite(info.log_prob).all()


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["diag", "dense0", "dense1", "dense2", "dense5"])
def test_cuda_graph_replay_is_bitwise_eager(zs, path):
    """Device-driven iterations replayed from a CUDA graph (use_cuda_graph=True)
    give bit-identical chains, step sizes and mass estimates to the eager
    launches, across the step-size search iterations (t == 1 and
    t == mass_collect_iters, which always run eagerly), adaptation on -> off,
    and a mid-run switch of the adaptation flags (second captured graph)."""
    rng = np.random.RandomState(3)
    if path == "diag":
        D, C = 100, 64
        std = (0.5 + rng.random_sample(D)).astype(np.float32)
        q0 = rng.standard_normal((C, D)).astype(np.float32)

        def model():
            @zs.meta_bayesian_net()
            def gaussian():
                bn = zs.BayesianNet()
                bn.normal('x', torch.zeros(D, device="cuda"), std=T(std), group_ndims=1)
                return bn
            return gaussian()
        kw = {}
    else:
        D, C = 64, 48
        P, _ = OM.make_dense_gaussian_problem(D, seed=2)
        q0 = rng.standard_normal((C, D)).astype(np.float32)
        model = lambda: zs.fused.GaussianLogJoint(P)
        kw = {"dense_impl": int(path[-1])}
    runs = []
    for graph in (False, True):
        x = T(q0)
        h = zs.HMC(step_size=0.05, n_leapfrogs=5, adapt_step_size=True, adapt_mass=True,
                   mass_collect_iters=4, seed=11, use_cuda_graph=graph, **kw)
        op, info = h.sample(model(), {}, {"x": x})
        trace = []
        for i in range(14):
            adapt = i < 9
            op(adapt_step_size=adapt, adapt_mass=adapt)
            trace.append((N(x).copy(), float(h._state[1].item()), N(h._mass[0]).copy(),
                          N(info.acceptance_rate).copy()))
        op.synchronize()
        assert len(h._graphs) == (2 if graph else 0)
        runs.append((trace, h._t, h._ewmv_t, N(h._state).copy()))
    (ta, t_a, e_a, st_a), (tb, t_b, e_b, st_b) = runs
    assert (t_a, e_a) == (t_b, e_b)
    for i, (a, b) in enumerate(zip(ta, tb)):
        assert a[1] == b[1], "step size differs at iteration %d" % i
        np.testing.assert_array_equal(a[0], b[0], err_msg="q, iteration %d" % i)
        np.testing.assert_array_equal(a[2], b[2], err_msg="mass, iteration %d" % i)
        np.testing.assert_array_equal(a[3], b[3])
    np.testing.assert_array_equal(st_a, st_b)


@pytest.mark.gpu
@pytest.mark.parametrize("impl", [5])
@pytest.mark.parametrize("C,L", [(300, 3), (2048, 5), (8192, 2), (9472 + 256 + 40, 4)])
def test_trajectory_kernels_match_per_pass_kernel(zs, impl, C, L):
    """dense_impl=5 (the whole trajectory on the fp16 plane state, clusters of 2 x 2 CTAs where
    the units tile by them; the last shape ends in a ragged chain block) against dense_impl=2
    (fp32 q between passes): same operands and products, so the chains must agree to fp32
    rounding."""
    D = 1024
    P, _ = OM.make_dense_gaussian_problem(D, seed=2)
    res = []
    for im in (2, impl):
        torch.manual_seed(5)
        x = torch.randn(C, D, device="cuda")
        h = zs.HMC(step_size=0.1, n_leapfrogs=L, seed=7, dense_impl=im)
        op, info = h.sample(zs.fused.GaussianLogJoint(P), {}, {"x": x})
        for _ in range(2):
            op()
        op.synchronize()
        res.append((N(x), N(info.hamiltonian), N(info.acceptance_rate)))
    np.testing.assert_allclose(res[1][1], res[0][1], rtol=1e-5)
    # acc = exp(H0 - H1) with |H| ~ 3000: 1e-7 relative on H is 3e-4 absolute on acc
    np.testing.assert_allclose(res[1][2], res[0][2], rtol=0, atol=2e-3)
    same = np.abs(res[1][2] - res[0][2]) < 1e-6      # chains whose decision cannot have flipped
    np.testing.assert_allclose(res[1][0][same], res[0][0][same], rtol=1e-4, atol=1e-4)


@pytest.mark.gpu
@pytest.mark.parametrize("D,C,L", [(64, 40, 1), (64, 300, 3), (192, 70, 2), (512, 260, 3),
                                   (1024, 1, 1)])
def test_resident_kernel_shapes_vs_oracle(zs, D, C, L):
    """dense_impl=5 on ragged / tiny shapes (D not a multiple of 256, one chain, a single
    dimension tile) with a mean vector and a non-unit mass, one iteration vs the oracle."""
    rng = np.random.RandomState(D + C + L)
    P, const = OM.make_dense_gaussian_problem(D, seed=4)
    mu = (0.3 * rng.standard_normal(D)).astype(np.float32)
    q0 = rng.standard_normal((C, D)).astype(np.float32)
    npz = rng.standard_normal((C, D)).astype(np.float32)
    u = rng.random_sample(C).astype(np.float32)
    om = OM.DenseGaussian(P.astype(np.float32), mu, const)
    oq, oi = OH.HMC(step_size=0.12, n_leapfrogs=L).step([q0], om.logp, om.grad, [npz], u)
    x = T(q0)
    h = zs.HMC(step_size=0.12, n_leapfrogs=L, dense_impl=5)
    lj = zs.fused.GaussianLogJoint(P, mean=mu, log_det_cov=-2 * const - D * np.log(2 * np.pi))
    op, info = h.sample(lj, {}, {"x": x})
    assert h._res
    op(noise={"p": {"x": T(npz)}, "u": T(u)})
    op.synchronize()
    np.testing.assert_allclose(N(info.orig_hamiltonian), oi.orig_hamiltonian, rtol=1e-5, atol=1e-4)
    np.testing.assert_allclose(N(info.hamiltonian), oi.hamiltonian, rtol=1e-5, atol=1e-4)
    np.testing.assert_allclose(N(info.acceptance_rate), oi.acceptance_rate, rtol=2e-4, atol=1e-4)
    near = np.abs(u - oi.acceptance_rate) < 1e-3
    np.testing.assert_allclose(N(x)[~near], oq[0][~near], rtol=2e-5, atol=2e-5)


@pytest.mark.gpu
@pytest.mark.parametrize("path", ["diag", "dense5", "generic"])
def test_hmc_state_dict_round_trip_resumes_bitwise(zs, path):
    """HMC.state_dict() / load_state_dict(): a sampler rebuilt from a checkpoint (latents +
    state dict) continues EXACTLY like the uninterrupted one -- step size, dual-averaging state,
    EWMV mean / variance, iteration counter (Philox stream) -- across a mass_collect_iters
    boundary.  The check_numerics flag is not part of the checkpoint."""
    rng = np.random.RandomState(5)
    if path == "dense5":
        D, C = 64, 80
        P, _ = OM.make_dense_gaussian_problem(D, seed=2)
        model = lambda: zs.fused.GaussianLogJoint(P)
        kw = {"dense_impl": 5}
    else:
        D, C = 24, 40
        std = (0.5 + rng.random_sample(D)).astype(np.float32)

        def model():
            if path == "generic":
                return lambda o: zs.distributions.Normal(
                    torch.zeros(D, device="cuda"), std=T(std), group_ndims=1).log_prob(o['x'])

            @zs.meta_bayesian_net()
            def gaussian():
                bn = zs.BayesianNet()
                bn.normal('x', torch.zeros(D, device="cuda"), std=T(std), group_ndims=1)
                return bn
            return gaussian()
        kw = {}
    q0 = rng.standard_normal((C, D)).astype(np.float32)

    def build(x):
        h = zs.HMC(step_size=0.05, n_leapfrogs=5, adapt_step_size=True, adapt_mass=True,
                   mass_collect_iters=6, seed=21, **kw)
        op, info = h.sample(model(), {}, {"x": x})
        return h, op, info
    xa = T(q0)
    ha, opa, _ = build(xa)
    for _ in range(4):
        opa(adapt_step_size=True, adapt_mass=True)
    opa.synchronize()
    ckpt, x_ckpt = ha.state_dict(), xa.clone()
    ha._state[9] = float("nan")                 # a raised flag must not travel in a checkpoint
    assert float(ha.state_dict()["state"][9]) == 0.0
    ha._state[9] = 0.0
    for _ in range(5):
        opa(adapt_step_size=True, adapt_mass=True)
    opa.synchronize()
    xb = x_ckpt.clone()
    hb, opb, _ = build(xb)
    hb.load_state_dict(ckpt)
    for _ in range(5):
        opb(adapt_step_size=True, adapt_mass=True)
    opb.synchronize()
    assert (ha._t, ha._ewmv_t) == (hb._t, hb._ewmv_t) == (9, 9)
    np.testing.assert_array_equal(N(xa), N(xb))
    np.testing.assert_array_equal(N(ha._state)[:9], N(hb._state)[:9])
    np.testing.assert_array_equal(N(ha._mass[0]), N(hb._mass[0]))
    np.testing.assert_array_equal(N(ha._ew_var[0]), N(hb._ew_var[0]))
