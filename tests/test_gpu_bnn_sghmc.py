"""GPU parity of SGHMC on the [n_in, H, 1] Bayesian neural net (config 4) against the float64 oracle
(oracle/models.py::BNN + oracle/sgmcmc.py::SGHMC), across the shape range of the fused one-launch
kernel (csrc/sgmcmc_bnn.cu) and the generic path it falls back to.

Each lock-step run compares w0, w1, the momenta and mean_k after every step, then copies the
oracle's state (rounded to float32) into both samplers, so every comparison measures one step's
float32 error instead of accumulated drift."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

F64 = np.float64
SEED = 1234


def T(a):
    return torch.tensor(np.asarray(a), dtype=torch.float32, device="cuda")


def N(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def _ls_shape(spec, n_in, H, C, layer):
    """Prior log-stddev shape from a short name: 'full' ([H, n_in+1] / [1, H+1]), 'hidden'
    ([H, 1], one scale per hidden unit), 'input' ([n_in+1]), 'scalar' ([]), 'chain' (one full
    set per chain), 'chain_hidden' ([C, H, 1])."""
    full = (H, n_in + 1) if layer == 0 else (1, H + 1)
    return {"full": full, "hidden": (H, 1), "input": (n_in + 1,), "scalar": (),
            "chain": (C,) + full, "chain_hidden": (C, H, 1)}[spec]


class Problem(object):
    """A seeded BNN problem: data, prior scales, initial state, and the float64 oracle."""

    def __init__(self, n_in, H, B, C, ls=("full", "full"), n_train=300, y_logstd=-0.4,
                 seed=0, B_all=None):
        rng = np.random.RandomState(seed)
        self.rng = rng
        self.n_in, self.H, self.B, self.C = n_in, H, B, C
        self.n_train, self.y_logstd = n_train, y_logstd
        n_rows = B_all or B
        self.x_all = rng.standard_normal((n_rows, n_in))
        self.y_all = np.sin(self.x_all.sum(1)) + 0.3 * rng.standard_normal(n_rows)
        # log-stddevs in [-0.7, 0.3]: prior precisions from 0.55 to 4, so the prior term of the
        # gradient is a visible share of it
        self.ls = [rng.uniform(-0.7, 0.3, _ls_shape(ls[k], n_in, H, C, k)) for k in (0, 1)]
        self.w0 = rng.uniform(-2, 2, (C, H, n_in + 1))
        self.w1 = rng.uniform(-2, 2, (C, 1, H + 1))
        # round everything the device sees to float32 so both sides start from the same numbers
        self.x_all, self.y_all, self.w0, self.w1 = (
            a.astype(np.float32).astype(F64) for a in (self.x_all, self.y_all, self.w0, self.w1))
        self.ls = [a.astype(np.float32).astype(F64) for a in self.ls]

    def oracle(self, rows=slice(None)):
        from oracle import models as OM
        return OM.BNN(self.x_all[rows], self.y_all[rows], self.n_train, self.ls[0], self.ls[1],
                      dtype=F64, y_logstd=self.y_logstd)

    def log_joint(self, zs, rows=slice(None)):
        return zs.fused.BNNRegressionLogJoint(T(self.x_all[rows]), T(self.y_all[rows]),
                                              [T(l) for l in self.ls], self.n_train,
                                              y_logstd=self.y_logstd)

    def normals(self):
        return [self.rng.standard_normal(s).astype(np.float32).astype(F64)
                for s in (self.w0.shape, self.w1.shape)]


def _count_fused(sg):
    """Record the steps that ran the fused kernel."""
    calls = []
    run = sg._update_fused_bnn

    def spy(obj, noise):
        calls.append(sg.t)
        return run(obj, noise)
    sg._update_fused_bnn = spy
    return calls


def _sampler(zs, lj, prob, use_fused=True, **kw):
    w0, w1 = T(prob.w0), T(prob.w1)
    sg = zs.SGHMC(use_fused=use_fused, **kw)
    op, info = sg.sample(lj, {}, {"w0": w0, "w1": w1})
    return sg, op, info, [w0, w1]


def _relu_ties(om, w0):
    """[C, H] mask of the hidden units whose pre-activation, at the weights the gradient was taken
    at, is within float32 rounding of 0 for some data point.  There the float32 and the float64
    ReLU may take different sides, and that unit's w0 gradient differs by one data point's
    term: such units (about 1% at B = 512) are left out of the tight comparison."""
    x = om.x
    h0 = np.concatenate([x, np.ones((x.shape[0], 1))], -1)
    s = h0 @ w0.transpose(0, 2, 1)                                  # [C, B, H]
    bound = np.abs(h0) @ np.abs(w0).transpose(0, 2, 1)
    return (np.abs(s) <= 3e-6 * bound).any(axis=1)


def _compare(tag, sg, info, ws, oq, osg, oinfo, ties):
    """One step's float32 result against the float64 oracle.  Weights are O(1) and move by
    O(1e-2) per step, so they are held to a few float32 ulps; momenta, whose magnitude is set by
    lr, to a relative error scaled by their largest entry."""
    assert ties.mean() < 0.05, "%s: %d ReLU ties" % (tag, ties.sum())
    for k, name in enumerate(("w0", "w1")):
        got_w, got_v, want_w, want_v = N(ws[k]), N(sg.vs[k]), oq[k], osg.vs[k]
        if k == 0:
            got_w, got_v, want_w, want_v = (a[~ties] for a in (got_w, got_v, want_w, want_v))
        np.testing.assert_allclose(got_w, want_w, rtol=2e-6, atol=2e-6,
                                   err_msg="%s: %s" % (tag, name))
        np.testing.assert_allclose(got_v, want_v, rtol=1e-5,
                                   atol=1e-5 * float(np.abs(want_v).max()),
                                   err_msg="%s: v of %s" % (tag, name))
        np.testing.assert_allclose(float(info.mean_k[name]), oinfo["mean_k"][k], rtol=1e-4,
                                   err_msg="%s: mean_k of %s" % (tag, name))


def _lockstep(tag, runs, prob, osg, om_of_step, steps, draws, observed_of_step=None):
    """Step every (sg, op, info, ws) in ``runs`` and the oracle together; ``draws(t)`` gives the
    (noise, resample) standard normals of step t and whether to inject them.  After each step
    the oracle's state, rounded to float32, is copied into every run and kept by the oracle."""
    oq = [prob.w0, prob.w1]
    for t in range(steps):
        nz, rs, inject = draws(t)
        om, at = om_of_step(t), []

        def grad(qs):
            at.append(qs[0])
            return om.grad(qs)
        oq, oinfo = osg.step(oq, grad, rs, nz)
        ties = _relu_ties(om, at[0])
        for i, (sg, op, info, ws) in enumerate(runs):
            kw = {}
            if inject:
                kw["noise"] = {"noise": {"w0": T(nz[0]), "w1": T(nz[1])},
                               "resample": {"w0": T(rs[0]), "w1": T(rs[1])}}
            if observed_of_step is not None:
                kw["observed"] = observed_of_step(t)
            op(**kw)
            _compare("%s run %d step %d" % (tag, i, t), sg, info, ws, oq, osg, oinfo, ties)
        oq = [q.astype(np.float32).astype(F64) for q in oq]
        osg.vs = [v.astype(np.float32).astype(F64) for v in osg.vs]
        for sg, op, info, ws in runs:
            for dst, src in zip(ws + list(sg.vs), oq + osg.vs):
                dst.copy_(T(src))


def _oracle_sampler(v0, **kw):
    from oracle import sgmcmc as OS
    osg = OS.SGHMC(dtype=F64, **kw)
    osg.init_v(v0)
    return osg


def _injected(prob):
    def draws(t):
        return prob.normals(), prob.normals(), True
    return draws


def _sgkw(second_order, lr=2e-5):
    return dict(learning_rate=lr, friction=0.2, variance_estimate=0.01, n_iter_resample_v=3,
                second_order=second_order)


# (n_in, H, B, C), the edge each covers, and prior-scale shapes crossed with it
SWEEP = [
    ((1, 1, 1, 3), "n_in+1 = 2, one hidden unit, one data point",
     [("full", "full"), ("scalar", "scalar"), ("input", "full")]),
    ((10, 32, 97, 70), "no lane's second unit; B % 4 = 1",
     [("hidden", "full"), ("input", "scalar")]),
    ((10, 33, 98, 70), "only lane 0's second unit",
     [("hidden", "scalar"), ("full", "full")]),
    ((15, 64, 512, 40), "n_in+1 = 16, H and B at their maxima: ~109 KB of shared memory",
     [("hidden", "full"), ("scalar", "scalar")]),
    ((7, 63, 130, 5000), "more than one persistent round (2112 chains), ragged",
     [("hidden", "full")]),
    ((10, 50, 100, 8192), "the benchmark shape", [("full", "full")]),
]
SWEEP_CASES = [pytest.param(shape, ls, id="%d-%d-%d-%d-%s-%s" % (shape + ls))
               for shape, _, lss in SWEEP for ls in lss]


@pytest.mark.parametrize("second_order", [True, False], ids=["2nd", "1st"])
@pytest.mark.parametrize("shape,ls", SWEEP_CASES)
def test_fused_step_matches_oracle_across_shapes(zs, shape, ls, second_order):
    n_in, H, B, C = shape
    prob = Problem(n_in, H, B, C, ls=ls, n_train=50 * B + 17, y_logstd=-0.4, seed=sum(shape))
    # the 5000- and 8192-chain oracles are the slow part: 4 steps still cover t = 0 and t = 3
    steps = 4 if C > 1000 else 6
    kw = _sgkw(second_order)
    sg, op, info, ws = _sampler(zs, prob.log_joint(zs), prob, **kw)
    assert sg._fused_bnn() is not None
    fused_steps = _count_fused(sg)
    v0 = prob.normals()
    sg.init_momentum({"w0": T(v0[0]), "w1": T(v0[1])})
    osg = _oracle_sampler(v0, **kw)
    om = prob.oracle()
    _lockstep("%s %s" % (shape, ls), [(sg, op, info, ws)], prob, osg, lambda t: om, steps,
              _injected(prob))
    assert fused_steps == list(range(steps))


@pytest.mark.parametrize("n_in,H,B,fused", [
    (15, 64, 512, True),       # every limit reached: still fused
    (16, 64, 512, False),      # n_in + 1 = 17
    (15, 65, 512, False),      # H = 65
    (15, 64, 513, False),      # B = 513
    (16, 65, 513, False),
])
def test_fused_path_boundaries(zs, n_in, H, B, fused):
    """Past any of the kernel's limits the step takes the generic path, which still matches the
    oracle; at the limits it stays on the fused kernel."""
    prob = Problem(n_in, H, B, 6, ls=("hidden", "full"), n_train=2000, seed=n_in + H + B)
    kw = _sgkw(True)
    sg, op, info, ws = _sampler(zs, prob.log_joint(zs), prob, **kw)
    assert (sg._fused_bnn() is not None) == fused
    fused_steps = _count_fused(sg)
    v0 = prob.normals()
    sg.init_momentum({"w0": T(v0[0]), "w1": T(v0[1])})
    osg = _oracle_sampler(v0, **kw)
    om = prob.oracle()
    _lockstep("boundary", [(sg, op, info, ws)], prob, osg, lambda t: om, 4, _injected(prob))
    assert fused_steps == (list(range(4)) if fused else [])


def _philox_draws(prob, row0):
    """The in-kernel draws, rebuilt: Philox stream 3 (update noise) and 4 (momentum resample) at
    iteration t, seed SEED for w0 and SEED + 1 for w1, one row per global chain row0 + c, the
    flat element index of one chain's weights as the column."""
    from oracle.philox import normal_matrix
    C = prob.C
    shapes = [prob.w0.shape, prob.w1.shape]

    def at(stream, it):
        return [normal_matrix(SEED + k, stream, it, row0, C, int(np.prod(s[1:])))
                .astype(F64).reshape(s) for k, s in enumerate(shapes)]

    def draws(t):
        return at(3, t), at(4, t), False
    return at, draws


@pytest.mark.parametrize("second_order", [True, False], ids=["2nd", "1st"])
@pytest.mark.parametrize("fused", [True, False], ids=["fused", "generic"])
def test_in_kernel_philox_matches_oracle(zs, fused, second_order):
    """No injected noise: the oracle is fed the Philox draws rebuilt in NumPy, for a sampler over
    more chains than one persistent round whose rows start at a non-zero chain offset.  The
    initial momentum drawn in sample() (stream 4, iteration 0xFFFFFFFF) is checked too."""
    row0 = 12345
    # H + 1 = 21 and H (n_in + 1) = 60 are not multiples of 4: the last Philox block is partial
    prob = Problem(4, 20, 24, 2300, ls=("hidden", "full"), n_train=1000, seed=5)
    kw = _sgkw(second_order)
    sg, op, info, ws = _sampler(zs, prob.log_joint(zs), prob, use_fused=fused, seed=SEED,
                                chain_offset=row0, **kw)
    fused_steps = _count_fused(sg)
    at, draws = _philox_draws(prob, row0)
    v0 = at(4, 0xFFFFFFFF)
    for k in range(2):
        np.testing.assert_allclose(N(sg.vs[k]), v0[k] * np.sqrt(kw["learning_rate"]),
                                   rtol=1e-5, atol=1e-7)
    osg = _oracle_sampler(v0, **kw)
    osg.vs = [N(v).astype(F64) for v in sg.vs]
    om = prob.oracle()
    _lockstep("philox", [(sg, op, info, ws)], prob, osg, lambda t: om, 5, draws)
    assert fused_steps == (list(range(5)) if fused else [])


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "generic"])
def test_chain_sharding_is_bitwise(zs, fused):
    """Chains split over two samplers (chain_offset = 0 and C1) follow the single sampler bit for
    bit: the in-kernel noise is keyed by the global chain, and nothing couples chains."""
    C, C1 = 4500, 2213
    prob = Problem(5, 40, 64, C, ls=("hidden", "full"), n_train=1000, seed=9)
    lj = prob.log_joint(zs)
    kw = dict(_sgkw(True), seed=SEED, use_fused=fused)

    def run(lo, hi, offset):
        w0, w1 = T(prob.w0[lo:hi]), T(prob.w1[lo:hi])
        sg = zs.SGHMC(chain_offset=offset, **kw)
        op, _ = sg.sample(lj, {}, {"w0": w0, "w1": w1})
        fused_steps = _count_fused(sg)
        for _ in range(5):
            op()
        assert len(fused_steps) == (5 if fused else 0)
        return [N(w0), N(w1), N(sg.vs[0]), N(sg.vs[1])]
    whole = run(0, C, None)
    parts = [run(0, C1, 0), run(C1, C, C1)]
    for k, name in enumerate(("w0", "w1", "v0", "v1")):
        np.testing.assert_array_equal(np.concatenate([parts[0][k], parts[1][k]]), whole[k],
                                      err_msg=name)
    assert np.isfinite(whole[0]).all()


def test_minibatch_switching(zs):
    """Minibatches fed through sample_op(observed=...): one larger than the kernel stages runs on
    the generic path, the next returns to the fused kernel, and every step matches the oracle.
    A minibatch that does not fit the weights is refused on the host, before any launch."""
    rows = [slice(0, 100), slice(100, 137), slice(0, 600), slice(137, 237), slice(300, 400)]
    prob = Problem(6, 40, 100, 50, ls=("hidden", "full"), n_train=5000, seed=3, B_all=600)
    kw = _sgkw(True)
    sg, op, info, ws = _sampler(zs, prob.log_joint(zs, rows[0]), prob, **kw)
    fused_steps = _count_fused(sg)
    v0 = prob.normals()
    sg.init_momentum({"w0": T(v0[0]), "w1": T(v0[1])})
    osg = _oracle_sampler(v0, **kw)
    oms = [prob.oracle(r) for r in rows]
    _lockstep("minibatch", [(sg, op, info, ws)], prob, osg, lambda t: oms[t], len(rows),
              _injected(prob),
              lambda t: {"x": T(prob.x_all[rows[t]]), "y": T(prob.y_all[rows[t]])})
    assert fused_steps == [0, 1, 3, 4]

    before = [N(w) for w in ws] + [N(v) for v in sg.vs]
    t = sg.t
    xb, yb = prob.x_all[:40], prob.y_all[:40]
    bad = [({"x": T(np.concatenate([xb, xb[:, :1]], 1)), "y": T(yb)}, "minibatch x"),
           ({"x": T(xb[:, :-1]), "y": T(yb)}, "minibatch x"),
           ({"x": T(xb), "y": T(yb[:-1])}, "minibatch y")]
    for obs, msg in bad:
        with pytest.raises(ValueError, match=msg):
            op(observed=obs)
    torch.cuda.synchronize()
    assert sg.t == t and fused_steps == [0, 1, 3, 4]
    for a, b in zip(before, [N(w) for w in ws] + [N(v) for v in sg.vs]):
        np.testing.assert_array_equal(a, b)


@pytest.mark.parametrize("second_order", [True, False], ids=["2nd", "1st"])
@pytest.mark.parametrize("ls", [("hidden", "full"), ("hidden", "scalar"), ("chain", "chain"),
                                ("chain_hidden", "scalar"), ("full", "chain")],
                         ids=lambda ls: "-".join(ls))
def test_prior_scale_shapes_fused_generic_oracle(zs, ls, second_order):
    """Prior log-stddevs that broadcast to one chain's weights without being a suffix of their
    shape (per hidden unit) run fused and read the right scale for every weight; ones with chain
    axes take the generic path.  Both paths match the oracle step for step."""
    prob = Problem(4, 45, 50, 24, ls=ls, n_train=400, seed=11)
    kw = _sgkw(second_order)
    per_chain = "chain" in ls[0] or "chain" in ls[1]
    v0 = prob.normals()
    runs, counts = [], []
    for use_fused in (True, False):
        sg, op, info, ws = _sampler(zs, prob.log_joint(zs), prob, use_fused=use_fused, **kw)
        if use_fused:
            assert (sg._fused_bnn() is None) == per_chain
        counts.append(_count_fused(sg))
        sg.init_momentum({"w0": T(v0[0]), "w1": T(v0[1])})
        runs.append((sg, op, info, ws))
    osg = _oracle_sampler(v0, **kw)
    om = prob.oracle()
    _lockstep("prior %s" % (ls,), runs, prob, osg, lambda t: om, 5, _injected(prob))
    assert counts == [[] if per_chain else list(range(5)), []]
