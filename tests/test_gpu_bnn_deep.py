"""GPU tests of the BNN regression log-joint with L >= 3 weight layers (csrc/bnn_deep.cu) against
the float64 oracle (tests/bnn_deep_oracle.py) and the generic path: the log-joint kernel over a
shape grid and every output subset, the fused SG-MCMC step of every method, the variational
objectives, HMC's provider, and the shapes past the limits that stay generic."""
import numpy as np
import pytest
import torch

from bnn_deep_oracle import DeepBNN

pytestmark = pytest.mark.gpu

F64 = np.float64


def T(a):
    return torch.as_tensor(np.ascontiguousarray(a, np.float32), device="cuda")


def N(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


class Problem(object):
    """sizes = [n_0, ..., n_{L-1}, 1]; ls: per layer "scalar", "full", "row" (one per output
    unit, [n_{i+1}, 1]) or "col" ([n_i + 1])."""

    def __init__(self, sizes, B, K, ls="scalar", n_train=500, y_logstd=-0.7, seed=0):
        rng = np.random.RandomState(seed)
        self.sizes, self.B, self.K = list(sizes), B, K
        L = len(sizes) - 1
        self.x = rng.standard_normal((B, sizes[0])).astype(np.float32)
        self.y = rng.standard_normal(B).astype(np.float32)
        self.ws = [rng.standard_normal((K, sizes[i + 1], sizes[i] + 1)).astype(np.float32)
                   for i in range(L)]
        forms = [ls] * L if isinstance(ls, str) else list(ls)
        shape_of = {"scalar": lambda i: (), "full": lambda i: (sizes[i + 1], sizes[i] + 1),
                    "row": lambda i: (sizes[i + 1], 1), "col": lambda i: (sizes[i] + 1,)}
        self.ls = [rng.uniform(-1.0, 0.5, shape_of[f](i)).astype(np.float32)
                   for i, f in enumerate(forms)]
        self.n_train, self.y_logstd = n_train, y_logstd
        self.names = ["w%d" % i for i in range(L)]

    def log_joint(self, zs, **kw):
        return zs.fused.BNNRegressionLogJoint(T(self.x), T(self.y), [T(l) for l in self.ls],
                                              self.n_train, y_logstd=self.y_logstd,
                                              names=self.names, **kw)

    def oracle(self, x=None, y=None):
        return DeepBNN(self.x if x is None else x, self.y if y is None else y, self.n_train,
                       self.ls, y_logstd=self.y_logstd)

    def obs(self, ws=None):
        return dict(zip(self.names, ws if ws is not None else [T(w) for w in self.ws]))


def _close(got, want, tol, msg, frac=0.999):
    """|got - want| <= tol * max|want| for at least ``frac`` of the entries (float32 may take
    the other side of a ReLU at a tie) and <= 100 tol * max|want| for all of them."""
    want = np.asarray(want, F64)
    got = np.asarray(got, F64).reshape(want.shape)
    scale = max(float(np.abs(want).max()), 1e-30)
    err = np.abs(got - want)
    assert np.isfinite(got).all(), msg
    assert (err <= tol * scale).mean() >= frac, "%s: max err %g (scale %g)" % (msg, err.max(), scale)
    assert err.max() <= 100 * tol * scale, "%s: max err %g (scale %g)" % (msg, err.max(), scale)


OUTS = ("lp", "g", "gys", "ym", "ll")


def _launch(lj, prob, want, ws=None):
    ws = ws if ws is not None else [T(w) for w in prob.ws]
    lp, gs, gys, ym, ll = lj._launch_deep(ws, lj.x, lj.y, lj._y_logstd_dev(ws[0].device),
                                          lp="lp" in want, gs=[("g" in want)] * len(ws),
                                          gys="gys" in want, ym="ym" in want, ll="ll" in want)
    return dict(lp=lp, g=gs if "g" in want else None, gys=gys, ym=ym, ll=ll)


def _check(tag, got, prob):
    om = prob.oracle()
    q = [w.astype(F64) for w in prob.ws]
    if got["lp"] is not None:
        np.testing.assert_allclose(N(got["lp"]), om.logp(q), rtol=2e-5,
                                   atol=2e-5 * float(np.abs(om.logp(q)).max()), err_msg=tag)
    if got["g"] is not None:
        keep = ~om.relu_ties(q)
        assert keep.mean() >= 0.25, "%s: %d of %d particles with ReLU ties" % (
            tag, (~keep).sum(), keep.size)
        for i, (g, want) in enumerate(zip(got["g"], om.grad(q))):
            _close(N(g)[keep], want[keep], 2e-5, "%s grad %d" % (tag, i))
    ym, ll = om.predictive(q)
    if got["ym"] is not None:
        _close(N(got["ym"]), ym, 1e-5, tag + " y_mean")
    if got["ll"] is not None:
        _close(N(got["ll"]), ll, 2e-5, tag + " log_lik")
    if got["gys"] is not None:
        _close(N(got["gys"]), om.grad_y_logstd(q), 2e-5, tag + " g_ylogstd")


# sizes, B, K, prior forms: depth 3-4 and the depth limit; widths 1, odd, 32, 50, 64, 65, 100 and
# the width limit 128; n_0 + 1 on both sides of 16 and at the limit; B = 1, 31-33, the tile of 64
# +- 1 and several tiles; K from 1 to over 2 x 132 CTAs; every prior broadcast form
GRID = [
    ([3, 1, 5, 1], 1, 1, "scalar"),
    ([15, 7, 32, 1], 31, 3, "full"),
    ([16, 50, 50, 1], 32, 5, "row"),
    ([10, 64, 65, 1], 33, 7, "col"),
    ([90, 100, 100, 1], 63, 4, ("full", "row", "col")),
    ([13, 50, 50, 50, 1], 64, 300, "scalar"),
    ([4, 33, 17, 9, 1], 65, 2, ("row", "scalar", "full", "col")),
    ([128, 128, 2, 1], 130, 3, "full"),
    ([90, 100, 100, 100, 1], 100, 270, "row"),
    ([5, 6, 7, 8, 9, 10, 11, 12, 1], 200, 6, "col"),
    ([2, 128, 128, 1], 17, 2, "scalar"),
    ([125, 128, 127, 1], 70, 2, "row"),          # 32639 weights: the largest net of this form
    ([3, 4, 3, 1], 40, 1500, "row"),             # more particles than any grid has CTAs
]


@pytest.mark.parametrize("sizes,B,K,ls", GRID, ids=lambda v: str(v).replace(" ", ""))
def test_logjoint_matches_oracle_across_shapes(zs, sizes, B, K, ls):
    prob = Problem(sizes, B, K, ls=ls, seed=len(sizes) + B + K)
    lj = prob.log_joint(zs)
    assert lj.fused_inputs(prob.obs()) is not None
    _check("%s B=%d K=%d" % (sizes, B, K), _launch(lj, prob, OUTS), prob)


def test_every_output_subset(zs):
    prob = Problem([6, 20, 11, 1], 70, 9, ls="row", seed=4)
    lj = prob.log_joint(zs)
    full = {k: v for k, v in _launch(lj, prob, OUTS).items()}
    for r in range(1, len(OUTS) + 1):
        import itertools
        for want in itertools.combinations(OUTS, r):
            got = _launch(lj, prob, want)
            for k in OUTS:
                if k in want:
                    a, b = got[k], full[k]
                    if k == "g":
                        for x, z in zip(a, b):
                            np.testing.assert_array_equal(N(x), N(z), err_msg=str(want))
                    else:
                        np.testing.assert_array_equal(N(a), N(b), err_msg="%s %s" % (want, k))
                else:
                    assert got[k] is None


def test_deterministic(zs):
    prob = Problem([10, 50, 50, 1], 150, 40, seed=8)
    lj = prob.log_joint(zs)
    a, b = _launch(lj, prob, OUTS), _launch(lj, prob, OUTS)
    for k in ("lp", "gys", "ym", "ll"):
        np.testing.assert_array_equal(N(a[k]), N(b[k]))
    for x, z in zip(a["g"], b["g"]):
        np.testing.assert_array_equal(N(x), N(z))


def test_call_with_three_names_matches_oracle(zs):
    """__call__ runs every layer and prior (the generic path of deeper nets)."""
    prob = Problem([5, 12, 8, 1], 20, 4, ls=("full", "row", "scalar"), seed=2)
    lj = prob.log_joint(zs)
    q = [w.astype(F64) for w in prob.ws]
    np.testing.assert_allclose(N(lj(prob.obs())), prob.oracle().logp(q), rtol=1e-5)


def test_constructor_rejects_mismatched_layers(zs):
    prob = Problem([5, 12, 8, 1], 20, 4, seed=2)
    with pytest.raises(ValueError):
        zs.fused.BNNRegressionLogJoint(T(prob.x), T(prob.y), [T(l) for l in prob.ls],
                                       prob.n_train, names=("w0", "w1"))
    with pytest.raises(ValueError):
        zs.fused.BNNRegressionLogJoint(T(prob.x), T(prob.y), [T(prob.ls[0])], prob.n_train,
                                       names=("w0",))


def test_fused_log_joint_autograd_and_no_grad(zs):
    prob = Problem([7, 30, 20, 1], 90, 6, ls="row", seed=5)
    ys = torch.tensor(-0.6, device="cuda", requires_grad=True)
    prob.y_logstd = -0.6
    lj = zs.fused.BNNRegressionLogJoint(T(prob.x), T(prob.y), [T(l) for l in prob.ls],
                                        prob.n_train, y_logstd=ys, names=prob.names)
    ws = [T(w).requires_grad_(True) for w in prob.ws]
    obs = prob.obs(ws)
    up = torch.linspace(0.5, 1.5, prob.K, device="cuda")
    lp = lj.fused_log_joint(obs)
    grads = torch.autograd.grad((lp * up).sum(), ws + [ys])
    om = prob.oracle()
    q = [w.astype(F64) for w in prob.ws]
    np.testing.assert_allclose(N(lp), om.logp(q), rtol=2e-5)
    for i, (g, want) in enumerate(zip(grads[:-1], om.grad(q))):
        _close(N(g), want * N(up)[:, None, None], 2e-5, "grad %d" % i)
    np.testing.assert_allclose(float(grads[-1]), float((om.grad_y_logstd(q) * N(up)).sum()),
                               rtol=2e-5)
    asked = []
    run = lj._launch_deep
    lj._launch_deep = lambda *a, **kw: asked.append(kw) or run(*a, **kw)
    with torch.no_grad():
        lp0 = lj.fused_log_joint(obs)
    assert lp0.grad_fn is None and asked == [{"lp": True}]
    np.testing.assert_array_equal(N(lp0), N(lp))


def test_predictive_over_many_rows(zs):
    prob = Problem([13, 50, 50, 1], 700, 12, seed=6)
    lj = prob.log_joint(zs)
    ym, ll = lj.predictive(prob.obs())
    want_ym, want_ll = prob.oracle().predictive([w.astype(F64) for w in prob.ws])
    _close(N(ym), want_ym, 1e-5, "y_mean")
    _close(N(ll), want_ll, 2e-5, "log_lik")


# ---------------------------------------------------------------- past the limits
@pytest.mark.parametrize("sizes", [[129, 4, 4, 1], [4, 129, 4, 1], [3, 2, 2, 2, 2, 2, 2, 2, 2, 1],
                                   [125, 128, 128, 1]],
                         ids=["n_in129", "hidden129", "depth9", "weights32769"])
def test_past_limits_take_generic_path(zs, sizes):
    prob = Problem(sizes, 10, 2, seed=9)
    prob.ws = [w * 0.5 for w in prob.ws]
    lj = prob.log_joint(zs)
    obs = prob.obs()
    assert lj.fused_inputs(obs) is None
    with pytest.raises(ValueError):
        lj.predictive(obs)
    np.testing.assert_allclose(N(lj(obs)), prob.oracle().logp([w.astype(F64) for w in prob.ws]),
                               rtol=1e-4)
    sg = zs.SGLD(learning_rate=1e-5)
    sg.sample(lj, {}, obs)
    assert sg._fused_bnn() is None


# ---------------------------------------------------------------- SG-MCMC
LR = 2e-5
_SGNHT = dict(learning_rate=LR, variance_extra=0.1, tune_rate=50., n_iter_resample_v=2)
METHODS = {
    "sghmc-2nd": ("SGHMC", dict(learning_rate=LR, friction=0.2, n_iter_resample_v=2)),
    "sghmc-1st": ("SGHMC", dict(learning_rate=LR, friction=0.2, n_iter_resample_v=2,
                                second_order=False)),
    "sgld": ("SGLD", dict(learning_rate=LR)),
    "psgld": ("PSGLD", dict(learning_rate=LR)),
    "sgnht-vec-2nd": ("SGNHT", dict(_SGNHT, second_order=True, use_vector_alpha=True)),
    "sgnht-vec-1st": ("SGNHT", dict(_SGNHT, second_order=False, use_vector_alpha=True)),
    "sgnht-scalar-2nd": ("SGNHT", dict(_SGNHT, second_order=True, use_vector_alpha=False)),
    "sgnht-scalar-1st": ("SGNHT", dict(_SGNHT, second_order=False, use_vector_alpha=False)),
}


def _sampler(zs, name, lj, prob, use_fused=True, lo=0, hi=None, **extra):
    cls, kw = METHODS[name]
    ws = [T(w[lo:hi]) for w in prob.ws]
    sg = getattr(zs, cls)(use_fused=use_fused, **dict(kw, **extra))
    op, info = sg.sample(lj, {}, dict(zip(prob.names, ws)))
    return sg, op, info, ws


def _state(sg):
    out = {}
    for key in ("vs", "alphas"):
        if hasattr(sg, key):
            out[key] = getattr(sg, key)
    return out


def _oracle_sampler(name, v0):
    from oracle import sgmcmc as OS
    cls, kw = METHODS[name]
    osg = getattr(OS, cls)(dtype=F64, **kw)
    if hasattr(osg, "init_v"):
        osg.init_v(v0)
    return osg


@pytest.mark.parametrize("name", list(METHODS))
def test_sgmcmc_lockstep_with_generic_and_oracle(zs, name):
    """Fused and generic samplers and the float64 oracle from the same state with every draw
    injected; v is re-drawn at t = 0 and 2.  After each step the oracle's state, rounded to
    float32, is copied into both samplers, so each comparison is one step's error."""
    prob = Problem([6, 20, 15, 1], 48, 10, ls=("row", "full", "scalar"), seed=11)
    prob.ws = [w * 0.5 for w in prob.ws]
    lj = prob.log_joint(zs)
    runs = [_sampler(zs, name, lj, prob, use_fused=f) for f in (True, False)]
    assert runs[0][0]._fused_bnn() is lj and runs[1][0]._use_fused is False
    rng = np.random.RandomState(3)
    v0 = [rng.standard_normal(w.shape).astype(np.float32) for w in prob.ws]
    for sg, _, _, _ in runs:
        if hasattr(sg, "init_momentum"):
            sg.init_momentum(dict(zip(prob.names, [T(v) for v in v0])))
    osg = _oracle_sampler(name, [v.astype(F64) for v in v0])
    om = prob.oracle()
    oq = [w.astype(F64) for w in prob.ws]
    for t in range(3):
        nz = [rng.standard_normal(w.shape).astype(np.float32) for w in prob.ws]
        rs = [rng.standard_normal(w.shape).astype(np.float32) for w in prob.ws]
        if hasattr(osg, "vs") or hasattr(osg, "alphas"):
            oq, oinfo = osg.step(oq, om.grad, [r.astype(F64) for r in rs],
                                 [n.astype(F64) for n in nz])
        else:
            oq, oinfo = osg.step(oq, om.grad, [n.astype(F64) for n in nz])
        noise = {"noise": dict(zip(prob.names, [T(n) for n in nz])),
                 "resample": dict(zip(prob.names, [T(r) for r in rs]))}
        for i, (sg, op, info, ws) in enumerate(runs):
            op(noise=noise)
            for k, w in enumerate(ws):
                _close(N(w), oq[k], 2e-6, "%s run %d step %d w%d" % (name, i, t, k))
            if "mean_k" in oinfo:
                for k, n in enumerate(prob.names):
                    _close(N(info.mean_k[n]), oinfo["mean_k"][k], 1e-4,
                           "%s run %d step %d mean_k %d" % (name, i, t, k))
        for k in range(len(prob.ws)):
            _close(N(runs[0][3][k]), N(runs[1][3][k]), 2e-6, "%s fused vs generic" % name)
        oq = [q.astype(np.float32).astype(F64) for q in oq]
        ost = {}
        if hasattr(osg, "vs") and osg.vs is not None:
            osg.vs = [np.asarray(v, np.float32).astype(F64) for v in osg.vs]
            ost["vs"] = osg.vs
        if hasattr(osg, "alphas") and osg.alphas is not None:
            osg.alphas = [np.asarray(a, np.float32).astype(F64) for a in osg.alphas]
            ost["alphas"] = osg.alphas
        if hasattr(osg, "aux") and osg.aux is not None:
            osg.aux = [np.asarray(a, np.float32).astype(F64) for a in osg.aux]
            ost["vs"] = osg.aux
        for sg, _, _, ws in runs:
            for dst, src in zip(ws, oq):
                dst.copy_(T(src))
            for key, vals in ost.items():
                for dst, src in zip(getattr(sg, key), vals):
                    dst.copy_(T(np.reshape(src, tuple(dst.shape))))


@pytest.mark.parametrize("name", ["sghmc-2nd", "sgld", "psgld", "sgnht-vec-2nd",
                                  "sgnht-scalar-1st"])
def test_in_kernel_philox_matches_generic(zs, name):
    """Without injected draws the fused step draws the generic path's numbers (latent k keyed
    seed + k), so both stay together over several steps, with v re-drawn on the way."""
    prob = Problem([8, 24, 12, 1], 40, 33, ls="row", seed=12)
    prob.ws = [w * 0.5 for w in prob.ws]
    lj = prob.log_joint(zs)
    runs = [_sampler(zs, name, lj, prob, use_fused=f, seed=1234) for f in (True, False)]
    for t in range(4):
        for _, op, _, _ in runs:
            op()
        for k in range(len(prob.ws)):
            _close(N(runs[0][3][k]), N(runs[1][3][k]), 1e-5, "%s step %d w%d" % (name, t, k))


MANY = 1200      # chains: more than zsb_sgmcmc_parts() = 1056, the step kernel's grid cap


@pytest.mark.parametrize("name", ["sghmc-2nd", "sgnht-scalar-2nd", "sgnht-scalar-1st", "sgld",
                                  "sgnht-vec-2nd"])
def test_many_chains_per_cta_match_generic(zs, name):
    """More chains than the step's grid can hold: each CTA walks several chains, so the chain
    loop, the per-thread v^2 sums behind mean_k, and the reuse of the staged weights, the gradient
    workspace and the staged minibatch across chains are all exercised.  Lock-step with the
    generic path from the same in-kernel draws (v re-drawn at t = 0 and 2)."""
    from zhusuan_b200._lib import lib
    assert MANY > lib.load().zsb_sgmcmc_parts()
    prob = Problem([3, 4, 3, 1], 20, MANY, ls="row", seed=21)
    prob.ws = [w * 0.5 for w in prob.ws]
    lj = prob.log_joint(zs)
    runs = [_sampler(zs, name, lj, prob, use_fused=f, seed=99) for f in (True, False)]
    assert runs[0][0]._fused_bnn() is lj
    for t in range(4):
        for _, op, _, _ in runs:
            op()
        for k in range(len(prob.ws)):
            _close(N(runs[0][3][k]), N(runs[1][3][k]), 1e-5, "%s step %d w%d" % (name, t, k))
        if hasattr(runs[0][2], "mean_k"):
            for n in prob.names:
                _close(N(runs[0][2].mean_k[n]), N(runs[1][2].mean_k[n]), 1e-5,
                       "%s step %d mean_k %s" % (name, t, n))
        if hasattr(runs[0][0], "alphas"):
            for k in range(len(prob.ws)):
                _close(N(runs[0][0].alphas[k]), N(runs[1][0].alphas[k]), 1e-5,
                       "%s step %d alpha %d" % (name, t, k))


@pytest.mark.parametrize("name", ["sghmc-2nd", "sgnht-vec-1st", "psgld"])
def test_chain_sharding_is_bitwise(zs, name):
    """Two samplers over chains [0, 500) and [500, 1200) with chain_offset give the bits of one
    sampler over all 1200: more chains than zsb_sgmcmc_parts(), the step's grid cap, so every
    CTA walks several chains whatever the occupancy."""
    prob = Problem([3, 4, 3, 1], 20, MANY, seed=13)
    prob.ws = [w * 0.3 for w in prob.ws]
    lj = prob.log_joint(zs)
    full = _sampler(zs, name, lj, prob, seed=77)
    parts = [_sampler(zs, name, lj, prob, lo=lo, hi=hi, seed=77, chain_offset=lo)
             for lo, hi in ((0, 500), (500, MANY))]
    for _ in range(3):
        for _, op, _, _ in [full] + parts:
            op()
    for k in range(len(prob.ws)):
        got = np.concatenate([N(p[3][k]) for p in parts])
        np.testing.assert_array_equal(got, N(full[3][k]))


def test_minibatch_switching(zs):
    """sample_op(observed=...) feeds minibatches of different sizes, one over several tiles; the
    fused step follows the generic one."""
    prob = Problem([6, 20, 20, 1], 30, 12, seed=14)
    prob.ws = [w * 0.5 for w in prob.ws]
    lj = prob.log_joint(zs)
    runs = [_sampler(zs, "sghmc-2nd", lj, prob, use_fused=f, seed=5) for f in (True, False)]
    rng = np.random.RandomState(0)
    for B in (30, 7, 200, 64, 65):
        xb = T(rng.standard_normal((B, 6)))
        yb = T(rng.standard_normal(B))
        for _, op, _, _ in runs:
            op(observed={"x": xb, "y": yb})
        assert runs[0][0]._fused_bnn() is lj
        for k in range(len(prob.ws)):
            _close(N(runs[0][3][k]), N(runs[1][3][k]), 1e-5, "B=%d w%d" % (B, k))


# ---------------------------------------------------------------- objectives and HMC
def test_objectives_match_generic(zs):
    prob = Problem([13, 20, 20, 1], 40, 8, ls="scalar", n_train=455, seed=15)
    rng = np.random.RandomState(1)
    eps = [rng.standard_normal(w.shape).astype(np.float32) for w in prob.ws]

    class InjectedNormal(zs.distributions.Normal):
        def __init__(self, *a, **kw):
            self._eps = kw.pop("eps")
            super(InjectedNormal, self).__init__(*a, **kw)

        def _sample(self, n_samples):
            return super(InjectedNormal, self)._sample(n_samples, eps=self._eps)

    res = []
    for fused in (True, False):
        means = [T(0.3 * rng.standard_normal(w.shape[1:])).requires_grad_(True) for w in prob.ws] \
            if not res else [m.detach().clone().requires_grad_(True) for m in res[0][0]]
        ys = torch.tensor(-0.3, device="cuda", requires_grad=True)
        lj = zs.fused.BNNRegressionLogJoint(T(prob.x), T(prob.y),
                                            [torch.zeros((), device="cuda")] * 3, prob.n_train,
                                            y_logstd=ys, names=prob.names)
        model = lj if fused else (lambda o: lj(o))

        def variational():
            bn = zs.BayesianNet()
            for i, n in enumerate(prob.names):
                bn.stochastic(n, InjectedNormal(means[i], logstd=torch.full_like(means[i], -2.),
                                                group_ndims=2, eps=T(eps[i])), n_samples=prob.K)
            return bn
        obs = {"x": T(prob.x), "y": T(prob.y)}
        lb = zs.variational.elbo(model, obs, variational=variational(), axis=0)
        g_lb = torch.autograd.grad(lb.sgvb(), means + [ys])
        iw = zs.variational.iw_objective(model, obs, variational=variational(), axis=0)
        g_iw = torch.autograd.grad(iw.sgvb(), means + [ys])
        with torch.no_grad():
            ll = zs.is_loglikelihood(model, obs, proposal=variational(), axis=0)
        res.append((means, float(lb.tensor.detach()), [N(g) for g in g_lb],
                    float(iw.tensor.detach()),
                    [N(g) for g in g_iw], float(ll)))
    a, b = res
    for i in (1, 3, 5):
        np.testing.assert_allclose(a[i], b[i], rtol=1e-5)
    for i in (2, 4):
        for x, z in zip(a[i], b[i]):
            np.testing.assert_allclose(x, z, rtol=1e-4, atol=1e-4 * float(np.abs(z).max()))


def test_hmc_provider_matches_oracle(zs):
    """zs.HMC on a depth-3 net over 150 rows (three tiles) takes the fused provider; one
    iteration with injected momenta and uniforms matches the oracle's."""
    from oracle import hmc as OH
    prob = Problem([13, 30, 20, 1], 150, 16, ls="row", n_train=150, y_logstd=-0.4, seed=16)
    prob.ws = [w * 0.3 for w in prob.ws]
    lj = prob.log_joint(zs)
    ws = [T(w) for w in prob.ws]
    h = zs.HMC(step_size=1e-3, n_leapfrogs=5)
    op, info = h.sample(lj, {}, dict(zip(prob.names, ws)))
    assert type(h._provider).__name__ == "_BNNProvider"
    om = prob.oracle()
    oh = OH.HMC(step_size=1e-3, n_leapfrogs=5)
    oq = [w.astype(F64) for w in prob.ws]
    rng = np.random.RandomState(2)
    npz = [rng.standard_normal(w.shape).astype(np.float32) for w in prob.ws]
    nu = rng.random_sample(prob.K).astype(np.float32)
    acc_o = oh.step(oq, om.logp, om.grad, npz, nu)[1].acceptance_rate
    nu = np.where(np.abs(nu - acc_o) < 1e-2, np.clip(acc_o + 0.05, 0, 1), nu).astype(np.float32)
    oq_new, oi = oh.step(oq, om.logp, om.grad, npz, nu)
    op(noise={"p": dict(zip(prob.names, [T(p) for p in npz])), "u": T(nu)})
    np.testing.assert_array_equal(N(info.acceptance_rate) > nu, oi.if_accept)
    np.testing.assert_allclose(N(info.orig_log_prob), oi.orig_log_prob, rtol=1e-5)
    for got, want in zip(ws, oq_new):
        _close(N(got), want, 1e-4, "hmc")


# ---------------------------------------------------------------- reference replays
GOLD_NETS = ["h2", "h3"]
GOLD_TAGS = {"sghmc": "SGHMC", "sgld": "SGLD", "psgld": "PSGLD", "sgnht_vec_2nd": "SGNHT",
             "sgnht_vec_1st": "SGNHT", "sgnht_scalar_2nd": "SGNHT", "sgnht_scalar_1st": "SGNHT"}


@pytest.fixture(scope="module")
def gold():
    import os
    return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                                "ref_bnn_deep.npz"))


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "generic"])
@pytest.mark.parametrize("tag", list(GOLD_TAGS))
@pytest.mark.parametrize("net", GOLD_NETS)
def test_sgmcmc_replays_reference(zs, gold, net, tag, fused):
    """The reference's own samplers on build_bnn with two and three hidden layers
    (tests/golden/make_ref_bnn_deep_golden.py): four steps with every draw injected, on the fused
    step (three and four weight layers) and on the generic path."""
    from test_ref_bnn_deep_pins import config, n_layers
    g, p = gold, "%s/%s/" % (net, tag)
    L = n_layers(g, net)
    names = ["w%d" % i for i in range(L)]
    lj = zs.fused.BNNRegressionLogJoint(T(g[net + "/x"]), T(g[net + "/y"]),
                                        [T(g["%s/logstd%d" % (net, i)]) for i in range(L)],
                                        int(g[net + "/n_train"]), names=names)
    kw = {k: v.item() for k, v in config(g, net, tag).items()}
    for k in ("n_iter_resample_v",):
        if k in kw:
            kw[k] = int(kw[k])
    for k in ("second_order", "use_vector_alpha"):
        if k in kw:
            kw[k] = bool(kw[k])
    ws = [T(g["%s/w%d_init" % (net, i)]) for i in range(L)]
    sg = getattr(zs, GOLD_TAGS[tag])(use_fused=fused, **kw)
    op, info = sg.sample(lj, {}, dict(zip(names, ws)))
    assert sg._fused_bnn() is lj and sg._use_fused == fused
    if hasattr(sg, "init_momentum"):
        sg.init_momentum({n: T(g["%s/v0_%d" % (net, i)]) for i, n in enumerate(names)})
    for t in range(g[p + "w0"].shape[0]):
        op(noise={"noise": {n: T(g[p + "noise%d" % i][t]) for i, n in enumerate(names)},
                  "resample": {n: T(g[p + "resample%d" % i][t]) for i, n in enumerate(names)}})
        for i, n in enumerate(names):
            want = g[p + "w%d" % i][t]
            np.testing.assert_allclose(N(ws[i]), want, rtol=1e-4, atol=1e-5,
                                       err_msg="%s step %d %s" % (p, t, n))
            if p + "mean_k%d" % i in g.files:
                mk = np.asarray(g[p + "mean_k%d" % i][t])
                np.testing.assert_allclose(np.asarray(N(info.mean_k[n])).reshape(mk.shape), mk,
                                           rtol=1e-3, atol=1e-3 * float(np.abs(mk).max()))
            if p + "alpha%d" % i in g.files:
                al = np.asarray(g[p + "alpha%d" % i][t])
                np.testing.assert_allclose(np.asarray(N(info.alpha[n])).reshape(al.shape), al,
                                           rtol=1e-4, atol=1e-6)


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "generic"])
@pytest.mark.parametrize("net", GOLD_NETS)
def test_bnn_vi_replays_reference(zs, gold, net, fused):
    """bnn_vi.py's lower bound, cost and gradients at the reference's injected draws, and its
    prediction fetches, on the fused log-joint and on the generic callable."""
    from test_ref_bnn_deep_pins import n_layers
    g, p = gold, net + "/vi/"
    L = n_layers(g, net)
    names = ["w%d" % i for i in range(L)]
    vars_ = ["w_mean_%d" % i for i in range(L)] + ["w_logstd_%d" % i for i in range(L)] + \
        ["y_logstd"]
    V = {n: T(g[p + "var_" + n]).reshape(g[p + "grad_" + n].shape).requires_grad_(True)
         for n in vars_}

    class InjectedNormal(zs.distributions.Normal):
        def __init__(self, *a, **kw):
            self._eps = kw.pop("eps")
            super(InjectedNormal, self).__init__(*a, **kw)

        def _sample(self, n_samples):
            return super(InjectedNormal, self)._sample(n_samples, eps=self._eps)

    def setup(x, y, eps):
        zero = torch.zeros((), device="cuda")
        lj = zs.fused.BNNRegressionLogJoint(T(x), T(y), [zero] * L, int(g[p + "n_train"]),
                                            y_logstd=V["y_logstd"], names=names)

        def variational():
            bn = zs.BayesianNet()
            for i, n in enumerate(names):
                bn.stochastic(n, InjectedNormal(V["w_mean_%d" % i], logstd=V["w_logstd_%d" % i],
                                                group_ndims=2, eps=T(eps[i])),
                              n_samples=eps[i].shape[0])
            return bn
        return (lj if fused else (lambda o: lj(o))), lj, variational

    model, lj, variational = setup(g[p + "x"], g[p + "y"], [g[p + "eps%d" % i] for i in range(L)])
    lb = zs.variational.elbo(model, {"y": T(g[p + "y"])}, variational=variational(), axis=0)
    cost = lb.sgvb()
    grads = torch.autograd.grad(cost, [V[n] for n in vars_])
    np.testing.assert_allclose(float(lb.tensor.detach()), float(g[p + "lower_bound"]), rtol=1e-5)
    np.testing.assert_allclose(float(cost.detach()), float(g[p + "cost"]), rtol=1e-5)
    for n, gr in zip(vars_, grads):
        ref = g[p + "grad_" + n]
        np.testing.assert_allclose(N(gr), ref, rtol=1e-4, atol=1e-4 * float(np.abs(ref).max()),
                                   err_msg=n)
    # prediction fetches (bnn_vi.py:98-103): predictive on the fused arm; on the generic arm the
    # callable's value at the test rows, whose likelihood term is the fetched log_py_xw
    _, lj_t, variational_t = setup(g[p + "x_test"], g[p + "y_test"],
                                   [g[p + "eps_ll%d" % i] for i in range(L)])
    bn = variational_t()
    obs = {n: getattr(bn[n], "tensor", bn[n]).detach() for n in names}
    if fused:
        ym, ll = lj_t.predictive(obs)
        np.testing.assert_allclose(N(ym), g[p + "ll_y_mean"], rtol=1e-5, atol=1e-5)
        np.testing.assert_allclose(N(ll), g[p + "ll_log_py_xw"], rtol=1e-5, atol=1e-5)
    else:
        from oracle import distributions as D
        with torch.no_grad():
            lp = N(lj_t(obs))
        prior = sum(D.normal_log_prob(N(obs[n]).astype(F64), 0, 0, 2, F64) for n in names)
        want = prior + g[p + "ll_log_py_xw"].astype(F64).mean(1) * int(g[p + "n_train"])
        np.testing.assert_allclose(lp, want, rtol=1e-5)
