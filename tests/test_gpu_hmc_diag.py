"""GPU parity of the fused diagonal-Gaussian HMC iteration (config 1: one Normal node whose
group_ndims cover the data axes, csrc/hmc.cu diag_normal_traj_kernel<E>) and of the mass-adaptation
kernels every HMC path shares, against the float64 oracle (oracle/hmc.py), across their shape
ranges.

The fused kernel runs one warp per chain with E columns per lane: E = 4 for D <= 128, 8 up to 256,
16 up to 512 and 32 up to 1024; longer rows take the generic path.  Its grid is capped at 132 * 8
blocks of 8 warps, so above 8448 chains the persistent row loop takes a second round.

A lock-step run steps the samplers and the oracle on the same noise and compares, after every
iteration, the acceptance rates, both log-probs and Hamiltonians, the initial momentum, the new
latent, the step size used and the updated one, the mass and the number of step-size search passes.
It then copies the oracle's state -- latent, dual-averaging tuner and EWMV mean / variance, rounded
to float32 -- into every sampler, so each comparison measures one iteration's float32 error instead
of accumulated drift.  With adapt_step_size, adapt_mass and mass_collect_iters = 2 the search runs
at t = 1 (unit mass) and t = 2 (adapted mass), t = 3 adapts without a search, and the last iteration
runs the non-adaptive branches of the tuner and of the EWMV.

Tolerances.  The log-std lies in [-0.6, 0.5], above -log sqrt(2 pi), so every summand of log p is
negative and every kinetic term positive: |log p| and H are the L1 norms of their sums, and holding
them to a relative 1e-6 (2e-6 and 2e-5 absolute after the trajectory, whose end point carries
(L + 1) roundings per column) is a tolerance that grows with D -- about 1.5e-3 for log p at
D = 1024, 2e-6 at D = 1.  One column read with a wrong mean or log-std moves a chain's log p by
O(0.1); one chain the kernel skips keeps the previous iteration's values.  A proposal the oracle
accepts with probability below 1e-6 comes from a diverging trajectory, whose rounding errors grow
with it: its Hamiltonian is held to 1e-4."""
import numpy as np
import pytest
import torch

from oracle import hmc as OH
from oracle import philox

pytestmark = pytest.mark.gpu

F64 = np.float64
SEED = 0x5EED1234ABCD
ROW0 = 12345
MCI = 2                                   # mass_collect_iters
# the tuner's mu is 10 * step_size (hmc.py:79), so a small initial step keeps the adapted step
# near 1 and leaves later iterations a visible share of accepted proposals
STEP0 = 1.0 / 128
DECAY = float(np.float32(0.99))           # the decay the kernel is given, as float64
ITERS = 4


def T(a):
    return torch.tensor(np.asarray(a), dtype=torch.float32, device="cuda")


def N(t):
    return t.detach().cpu().numpy()


def f32(a):
    """Round to float32, keep float64."""
    return np.asarray(a, np.float32).astype(F64)


def r32(x):
    return F64(np.float32(x))


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def _param_shape(spec, shape):
    """'full': the data shape; 'row': [1, data shape]; 'scalar': []; 'period': the last data axis
    (read with a period shorter than the row); 'col': the data shape with its last axis 1 (not a
    suffix of the data shape, so not fused)."""
    return {"full": shape, "row": (1,) + shape, "scalar": (), "period": shape[-1:],
            "col": shape[:-1] + (1,)}[spec]


class Problem(object):
    """A seeded diagonal-Normal target on data shape `shape` with chain shape `chains`: mean in
    [-1, 1] and log-std in [-0.6, 0.5] of the given parameter shapes, initial state drawn from the
    target, all rounded to float32.  logp / grad are the float64 model the oracle steps."""

    def __init__(self, shape, chains, mean_spec, ls_spec, seed):
        self.rng = np.random.RandomState(seed)
        self.shape, self.chains = tuple(shape), tuple(chains)
        self.C, self.D = int(np.prod(chains)), int(np.prod(shape))
        self.mean = f32(self.rng.uniform(-1, 1, _param_shape(mean_spec, self.shape)))
        self.logstd = f32(self.rng.uniform(-0.6, 0.5, _param_shape(ls_spec, self.shape)))
        self.q0 = f32(self.mean + np.exp(self.logstd)
                      * self.rng.standard_normal(self.chains + self.shape))
        self.axes = tuple(range(-len(self.shape), 0))

    def logp(self, qs):
        d = qs[0] - self.mean
        return (-0.5 * np.log(2 * np.pi) - self.logstd
                - 0.5 * np.exp(-2 * self.logstd) * d * d).sum(self.axes)

    def grad(self, qs):
        return [-np.exp(-2 * self.logstd) * (qs[0] - self.mean)]

    def fused_model(self, zs):
        mean, ls, g = T(self.mean), T(self.logstd), len(self.shape)

        @zs.meta_bayesian_net()
        def gaussian():
            bn = zs.BayesianNet()
            bn.normal('x', mean, logstd=ls, group_ndims=g)
            return bn
        return gaussian()

    def generic_model(self, zs):
        mean, ls, g = T(self.mean), T(self.logstd), len(self.shape)
        return lambda obs: zs.distributions.Normal(mean, logstd=ls,
                                                   group_ndims=g).log_prob(obs['x'])

    def injected(self):
        def draws(t):
            nz = f32(self.rng.standard_normal(self.chains + self.shape))
            u = f32(self.rng.random_sample(self.chains))
            if self.C == 1 and t == 1:
                # one chain's EWMV variance after the first update is exactly 0: the chain has to
                # move at t = 1 for the precision mass of t = 2 to be finite
                u *= 0.01
            return nz, u, True
        return draws

    def philox(self):
        def draws(t):
            nz = philox.normal_matrix(SEED, 1, t, ROW0, self.C, self.D).astype(F64)
            u = philox.uniform_vector(SEED, 2, t, ROW0, self.C).astype(F64)
            return nz.reshape(self.chains + self.shape), u.reshape(self.chains), False
        return draws


def _sampler(zs, model, prob, L, **kw):
    x = T(prob.q0)
    h = zs.HMC(step_size=STEP0, n_leapfrogs=L, adapt_step_size=True, adapt_mass=True,
               mass_collect_iters=MCI, **kw)
    op, info = h.sample(model, {}, {"x": x})
    return h, op, info, x


def _oracle(L):
    return OH.HMC(step_size=STEP0, n_leapfrogs=L, adapt_step_size=True, adapt_mass=True,
                  mass_collect_iters=MCI, mass_decay=DECAY, dtype=F64)


def _compare(tag, h, info, x, new_q, oi, u, n_search):
    """One iteration of one sampler against the float64 oracle (tolerances: module docstring)."""
    from zhusuan_b200.hmc import ST_EPS
    h0, h1, acc64 = oi.orig_hamiltonian, oi.hamiltonian, oi.acceptance_rate
    acc = N(info.acceptance_rate)
    # |d(h0 - h1)| <= t0 + t1, so |d acc| <= acc * (t0 + t1) to first order (x2, plus expf's ulp)
    tol_acc = 2 * acc64 * ((1e-6 * np.abs(h0) + 1e-6) + (2e-6 * np.abs(h1) + 2e-5)) + 1e-6
    assert np.all(np.abs(acc - acc64) <= tol_acc), \
        "%s: acceptance, max err %g" % (tag, np.abs(acc - acc64).max())
    # chains whose uniform lies within rounding of acc may decide either way
    near = np.abs(u - acc64) <= tol_acc
    assert near.sum() <= 1 + 0.02 * near.size, "%s: %d chains near u" % (tag, near.sum())
    np.testing.assert_array_equal((u < acc)[~near], oi.if_accept[~near], err_msg=tag + ": accept")
    np.testing.assert_allclose(N(info.orig_log_prob), oi.orig_log_prob, rtol=1e-6, atol=1e-6,
                               err_msg=tag + ": orig_log_prob")
    np.testing.assert_allclose(N(info.orig_hamiltonian), h0, rtol=1e-6, atol=1e-6,
                               err_msg=tag + ": orig_hamiltonian")
    live = acc64 > 1e-6
    np.testing.assert_allclose(N(info.hamiltonian)[live], h1[live], rtol=2e-6, atol=2e-5,
                               err_msg=tag + ": hamiltonian")
    np.testing.assert_allclose(N(info.hamiltonian)[~live], h1[~live], rtol=1e-4,
                               err_msg=tag + ": hamiltonian of a diverged proposal")
    np.testing.assert_allclose(N(info.log_prob)[~near], oi.log_prob[~near], rtol=2e-6, atol=2e-5,
                               err_msg=tag + ": log_prob")
    np.testing.assert_allclose(N(info.init_momentum["x"]), oi.init_momentum[0], rtol=1e-5,
                               atol=2e-6, err_msg=tag + ": init_momentum")
    np.testing.assert_allclose(N(x)[~near], new_q[~near], rtol=1e-5, atol=1e-5,
                               err_msg=tag + ": q")
    np.testing.assert_allclose(float(h._state[ST_EPS]), oi.step_size_used, rtol=1e-5,
                               err_msg=tag + ": eps_used")
    np.testing.assert_allclose(float(info.updated_step_size), oi.updated_step_size, rtol=1e-4,
                               err_msg=tag + ": updated_step_size")
    np.testing.assert_allclose(N(h._mass[0]), oi.mass[0].reshape(-1), rtol=2e-5,
                               err_msg=tag + ": mass")
    assert h.n_search_iters == n_search, "%s: %d search passes, oracle %d" % (
        tag, h.n_search_iters, n_search)


def _lockstep(tag, runs, prob, L, draws, check=None):
    """Step every (h, op, info, x) in `runs` and the oracle ITERS times; `draws(t)` gives the
    standard normals, the uniforms and whether to inject them; `check(t, nz, u)` runs after every
    sampler has stepped.  Then the oracle's state, rounded to float32, goes into every sampler."""
    from zhusuan_b200.hmc import ST_STEP, ST_TSTEP, ST_LEB, ST_HBAR
    oh = _oracle(L)
    oh.tuner.mu = r32(oh.tuner.mu)
    oq = prob.q0
    for t in range(1, ITERS + 1):
        adapt = t < ITERS
        nz, u, inject = draws(t)
        new_q, oi = oh.step([oq], prob.logp, prob.grad, [nz], u, adapt, adapt)
        for i, (h, op, info, x) in enumerate(runs):
            kw = {"noise": {"p": {"x": T(nz)}, "u": T(u)}} if inject else {}
            op(adapt_step_size=adapt, adapt_mass=adapt, **kw)
            _compare("%s run %d t=%d" % (tag, i, t), h, info, x, new_q[0], oi, u,
                     oh.n_search_iters)
        if check is not None:
            check(t, nz, u)
        oq = f32(new_q[0])
        tu, ew = oh.tuner, oh.ewmv
        oh.step_size = r32(oh.step_size)
        tu.step, tu.h_bar, tu.log_epsilon_bar = r32(tu.step), r32(tu.h_bar), r32(tu.log_epsilon_bar)
        ew.mean, ew.var = [f32(ew.mean[0])], [f32(ew.var[0])]
        for h, op, info, x in runs:
            x.copy_(T(oq))
            for k, v in ((ST_STEP, oh.step_size), (ST_TSTEP, tu.step), (ST_LEB, tu.log_epsilon_bar),
                         (ST_HBAR, tu.h_bar)):
                h._state[k] = float(v)
            h._ew_mean[0].copy_(T(ew.mean[0].reshape(-1)))
            h._ew_var[0].copy_(T(ew.var[0].reshape(-1)))
    for h, op, info, x in runs:
        op.synchronize()


# (data shape, chain shape, L, mean shape, log-std shape, also run the generic path, what it covers)
SWEEP = [
    ((1,), (1,), 4, "full", "full", True, "one column, one chain: E = 4, 31 idle lanes"),
    ((5,), (9,), 1, "scalar", "full", True, "D % 4 = 1, scalar mean"),
    ((127,), (9,), 0, "full", "row", False, "L = 0 (one half kick), [1, D] log-std"),
    ((128,), (1,), 4, "full", "scalar", True, "E = 4 at its top, scalar log-std"),
    ((129,), (3, 3), 4, "row", "full", False, "E = 8 at its bottom, two chain axes"),
    ((255,), (9,), 1, "full", "full", False, "E = 8, D % 4 = 3"),
    ((256,), (9,), 5, "scalar", "scalar", True, "E = 8 at its top, scalar parameters"),
    ((257,), (8448 + 37,), 4, "full", "full", True,
     "E = 16 at its bottom; the row loop's second round (37 chains)"),
    ((100,), (8448 + 37,), 1, "full", "row", True,
     "E = 4 over two rounds; the generic vec4 kernels at 8485 chains"),
    ((511,), (9,), 0, "full", "row", False, "E = 16, L = 0"),
    ((512,), (1,), 4, "full", "full", False, "E = 16 at its top"),
    ((513,), (9,), 4, "full", "scalar", False, "E = 32 at its bottom"),
    ((1023,), (9,), 1, "row", "full", True, "E = 32, D % 4 = 3"),
    ((1024,), (9,), 6, "full", "full", False, "E = 32 at its top"),
    ((4, 256), (9,), 4, "period", "period", True, "[256] parameters on [4, 256] rows (D = 1024)"),
    ((3, 43), (9,), 4, "period", "full", False, "period 43 mean at E = 8"),
    ((2, 200), (1,), 1, "scalar", "period", False, "period 200 log-std at E = 16"),
]
SWEEP_CASES = [pytest.param(*c[:6], id="%s-%s-L%d-%s-%s" % ("x".join(map(str, c[0])),
                                                            "x".join(map(str, c[1])), c[2], c[3],
                                                            c[4]))
               for c in SWEEP]


@pytest.mark.parametrize("shape,chains,L,mean_spec,ls_spec,generic", SWEEP_CASES)
def test_fused_diag_matches_oracle_across_shapes(zs, shape, chains, L, mean_spec, ls_spec,
                                                 generic):
    """The fused iteration at every E boundary from both sides, at D % 4 != 0, at 1, 9 and
    8448 + 37 chains, L = 0, 1 and >= 4, and with [D], [1, D], scalar and periodic ([b] on
    [a, b] rows) parameters, in lock-step with the float64 oracle on injected noise.  Where
    `generic` is set the same log-joint as a plain callable (the generic path's momentum,
    leapfrog, kinetic, MH and select kernels) steps alongside."""
    prob = Problem(shape, chains, mean_spec, ls_spec,
                   seed=int(np.prod(shape)) * 31 + int(np.prod(chains)) * 7 + L)
    runs = [_sampler(zs, prob.fused_model(zs), prob, L)]
    assert runs[0][0]._fused is not None and runs[0][0]._fused["kind"] == "diag_normal"
    if generic:
        runs.append(_sampler(zs, prob.generic_model(zs), prob, L))
        assert runs[1][0]._fused is None
    _lockstep(str(shape), runs, prob, L, prob.injected())


@pytest.mark.parametrize("shape,mean_spec,ls_spec", [
    ((1025,), "full", "full"),           # one column past the fused kernel's row
    ((4, 256), "col", "period"),         # a [4, 1] mean is not a suffix of the [4, 256] row
])
def test_generic_past_the_fused_kernel(zs, shape, mean_spec, ls_spec):
    """Models the fused kernel cannot take run on the generic path and still match the oracle."""
    prob = Problem(shape, (9,), mean_spec, ls_spec, seed=int(np.prod(shape)))
    run = _sampler(zs, prob.fused_model(zs), prob, 3)
    assert run[0]._fused is None
    _lockstep(str(shape), [run], prob, 3, prob.injected())


@pytest.mark.parametrize("D", [1, 33, 129, 257, 513, 1023, 1024])
def test_in_kernel_philox_matches_oracle_and_generic(zs, D):
    """No injected noise, seed SEED, chains starting at global row ROW0: every iteration's
    momentum is the oracle's Philox normals (stream 1, iteration t, one row per global chain) times
    sqrt(mass) to float32 rounding and, bit for bit, the generic path's momentum; every accept
    decision is u < acc for the oracle's stream-2 uniforms; and the lock-step against the oracle
    holds on those draws.  D = 1024 puts 8 Philox blocks on every lane (E = 32)."""
    prob = Problem((D,), (40,), "full", "full", seed=D + 3)
    runs = [_sampler(zs, prob.fused_model(zs), prob, 3, seed=SEED, chain_offset=ROW0),
            _sampler(zs, prob.generic_model(zs), prob, 3, seed=SEED, chain_offset=ROW0)]
    assert runs[0][0]._fused["kind"] == "diag_normal" and runs[1][0]._fused is None

    def check(t, nz, u):
        p = [N(info.init_momentum["x"]) for _, _, info, _ in runs]
        np.testing.assert_array_equal(p[0], p[1], err_msg="t=%d: fused vs generic momentum" % t)
        np.testing.assert_allclose(p[0], nz * np.sqrt(N(runs[0][0]._mass[0]).astype(F64)),
                                   rtol=1e-5, atol=2e-6, err_msg="t=%d: momentum" % t)
        for h, _, info, _ in runs:
            np.testing.assert_array_equal(N(h._accept),
                                          (u.astype(np.float32) < N(info.acceptance_rate)),
                                          err_msg="t=%d: accept" % t)
    _lockstep("philox D=%d" % D, runs, prob, 3, prob.philox(), check)


@pytest.mark.parametrize("D", [129, 1023])
def test_chain_split_is_bitwise(zs, D):
    """Without step-size adaptation nothing couples the chains: two samplers over the halves
    (chain_offset 0 and C / 2, one round of the row loop each) follow the sampler over all 8486
    chains (two rounds) bit for bit."""
    C, C1 = 8486, 4243
    prob = Problem((D,), (C,), "full", "full", seed=D)
    model = prob.fused_model(zs)

    def run(lo, hi, offset):
        x = T(prob.q0[lo:hi])
        h = zs.HMC(step_size=0.1, n_leapfrogs=4, seed=SEED, chain_offset=offset)
        op, info = h.sample(model, {}, {"x": x})
        assert h._fused["kind"] == "diag_normal"
        for _ in range(4):
            op()
        op.synchronize()
        return N(x), N(info.acceptance_rate), N(info.hamiltonian), N(info.init_momentum["x"])
    whole = run(0, C, None)
    parts = [run(0, C1, 0), run(C1, C, C1)]
    for k, name in enumerate(("q", "acc", "hamiltonian", "init_momentum")):
        np.testing.assert_array_equal(np.concatenate([parts[0][k], parts[1][k]]), whole[k],
                                      err_msg=name)
    assert (whole[0] != prob.q0).any(axis=1).mean() > 0.5


# ---- mass statistics and update through the C ABI (hmc.py:130-159) ---------------------------
def _mass_stats(q, mean):
    from zhusuan_b200._lib import lib, ptr, stream
    C, D = q.shape
    part = torch.empty(lib.load().zsb_hmc_mass_parts() * 2 * D, device="cuda")
    stats = torch.empty(2 * D, device="cuda")
    lib.call("zsb_hmc_mass_stats_f32", ptr(q), ptr(mean), C, D, ptr(part), ptr(stats), stream())
    return stats


def _mass_update(mean, var, stats, C, tt, adapt, use_ones, state):
    """Run zsb_hmc_mass_update_f32 on copies; returns (mean, var, mass)."""
    from zhusuan_b200._lib import lib, ptr, stream
    m, v = mean.clone(), var.clone()
    mass = torch.full_like(mean, float("nan"))
    lib.call("zsb_hmc_mass_update_f32", ptr(m), ptr(v), ptr(mass), ptr(stats), float(C),
             mean.numel(), DECAY, float(tt), int(adapt), int(use_ones), ptr(state), stream())
    return N(m), N(v), N(mass)


def _ewmv_oracle(q, mean, var, tt):
    """The oracle's EWMV (float64) from the state (mean, var, t = tt - 1) updated with q."""
    ew = OH.ExponentialWeightedMovingVariance(DECAY, [(1, q.shape[1])], 1, F64)
    ew.t = F64(tt - 1)
    ew.mean, ew.var = [N(mean).astype(F64)[None]], [N(var).astype(F64)[None]]
    ew.update([N(q).astype(F64)])
    return ew.mean[0][0], ew.var[0][0]


def _mass_problem(C, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    mu = torch.randn(D, generator=g, device="cuda")
    q = mu + torch.randn(C, D, generator=g, device="cuda") * (
        0.5 + torch.rand(D, generator=g, device="cuda"))
    mean = mu + 0.3 * torch.randn(D, generator=g, device="cuda")
    var = 0.5 + torch.rand(D, generator=g, device="cuda")
    return q, mean, var


@pytest.mark.parametrize("D", [1, 3, 4, 12, 100, 1024, 1030, 4096])
@pytest.mark.parametrize("C", [1, 7, 528, 529, 1585, 2113, 65536])
def test_mass_stats_and_update_match_float64(C, D):
    """S1 = sum_c (q - mean), S2 = sum_c (q - mean)^2 against float64 sums, at chain counts that
    do and do not fill the 528 stage-1 blocks, run the 4-way unrolled chain loop (from 1585 on)
    and its tail, and at D that take the scalar kernel (D % 4 != 0, or a misaligned q) and the
    vec4 kernel, with one or more column blocks on each (scalar above 256 columns, vec4 above
    1024).  Each sum is held to 4e-6 of the L1 norm of its summands.  The vec4 and scalar kernels
    give the same bits.  Where the float64 EWMV fits the host (C * D <= 2^22) the adaptive update
    of mean, variance and precision mass matches it too."""
    q, mean, var = _mass_problem(C, D, seed=C * 10007 + D)
    stats = _mass_stats(q, mean)
    x = q.double() - mean.double()
    s1, s2, l1 = x.sum(0), (x * x).sum(0), x.abs().sum(0)
    got = stats.double()
    err1 = float(((got[:D] - s1).abs() / l1).max())
    err2 = float(((got[D:] - s2).abs() / s2).max())
    assert err1 <= 4e-6 and err2 <= 4e-6, (err1, err2)
    if D % 4 == 0:
        buf = torch.empty(C * D + 4, device="cuda")
        q_mis = buf[1:1 + C * D].view(C, D)
        q_mis.copy_(q)
        assert q.data_ptr() % 16 == 0 and q_mis.data_ptr() % 16 != 0
        assert torch.equal(_mass_stats(q_mis, mean).view(torch.int32), stats.view(torch.int32))
    del x
    if C * D <= 1 << 22:
        tt = 3
        state = torch.zeros(16, device="cuda")
        m, v, mass = _mass_update(mean, var, stats, C, tt, 1, 0, state)
        om, ov = _ewmv_oracle(q, mean, var, tt)
        np.testing.assert_allclose(m, om, rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(v, ov, rtol=2e-5)
        np.testing.assert_allclose(mass, 1 / ov, rtol=2e-5)
        assert float(state[6]) == tt                    # the EWMV count in the state block


@pytest.mark.parametrize("adapt,use_ones,t,ewmv_t", [
    (0, 0, 7, 6), (0, 1, 7, 6), (1, 1, 7, 6), (1, 0, 7, 6),
    # device-driven iterations: use_ones = -(mass_collect_iters + 1), t and the EWMV count are
    # read from the state block
    (1, -3, 1, 0), (1, -3, 2, 1), (1, -3, 5, 4), (0, -3, 1, 4), (0, -3, 2, 4)])
def test_mass_update_gating(adapt, use_ones, t, ewmv_t):
    """hmc.py:283-305.  adapt = 0 leaves the EWMV alone; the mass is ones while t <
    mass_collect_iters (use_ones = 1 on the host, or t read from the state block when use_ones < 0)
    and the precision otherwise.  The host-driven update writes the EWMV count it was given into
    the state block; a device-driven one reads count + 1 from it, ignores the count argument and
    writes nothing."""
    C, D, mci = 7, 1030, 2
    q, mean, var = _mass_problem(C, D, seed=99)
    stats = _mass_stats(q, mean)
    state = torch.zeros(16, device="cuda")
    state[0], state[6] = float(t), float(ewmv_t)
    before = N(state).copy()
    device = use_ones < 0
    tt = ewmv_t + 1 if device else 7
    m, v, mass = _mass_update(mean, var, stats, C, 1000 if device else tt, adapt, use_ones, state)
    ones = (t < mci) if device else bool(use_ones)
    if adapt:
        om, ov = _ewmv_oracle(q, mean, var, tt)
        np.testing.assert_allclose(m, om, rtol=1e-6, atol=1e-6)
        np.testing.assert_allclose(v, ov, rtol=2e-5)
    else:
        np.testing.assert_array_equal(m, N(mean))
        np.testing.assert_array_equal(v, N(var))
        ov = N(var).astype(F64)
    if ones:
        np.testing.assert_array_equal(mass, np.ones(D, np.float32))
    else:
        np.testing.assert_allclose(mass, 1 / ov, rtol=2e-5)
    after = N(state)
    if adapt and not device:
        before[6] = tt
    np.testing.assert_array_equal(after, before)
