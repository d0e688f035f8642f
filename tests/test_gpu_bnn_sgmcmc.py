"""GPU parity of SGLD, PSGLD and SGNHT (vector and scalar thermostat, 1st and 2nd order) on the
[n_in, H, 1] Bayesian neural net (config 4) against the float64 oracle (oracle/models.py::BNN +
oracle/sgmcmc.py), through the fused one-launch step (csrc/sgmcmc_bnn.cu) and the generic path it
falls back to.  The problems, shape sweep and ReLU-tie mask are the SGHMC test's.

Each lock-step run compares the weights, the method's state (PSGLD's aux, SGNHT's v and alpha) and
mean_k after every step, then copies the oracle's state (rounded to float32) into the samplers, so
every comparison measures one step's float32 error instead of accumulated drift."""
import os

import numpy as np
import pytest
import torch

from test_gpu_bnn_sghmc import (F64, SEED, SWEEP, N, Problem, T, _count_fused, _philox_draws,
                                _relu_ties)

pytestmark = pytest.mark.gpu

LR = 2e-5
_SGNHT = dict(learning_rate=LR, variance_extra=0.1, tune_rate=50., n_iter_resample_v=3)
# name -> (class in zhusuan_b200 and in oracle.sgmcmc, constructor keywords)
VARIANTS = {
    "sgld": ("SGLD", dict(learning_rate=LR)),
    "psgld": ("PSGLD", dict(learning_rate=LR)),
    "sgnht-vec-2nd": ("SGNHT", dict(_SGNHT, second_order=True, use_vector_alpha=True)),
    "sgnht-vec-1st": ("SGNHT", dict(_SGNHT, second_order=False, use_vector_alpha=True)),
    "sgnht-scalar-2nd": ("SGNHT", dict(_SGNHT, second_order=True, use_vector_alpha=False)),
    "sgnht-scalar-1st": ("SGNHT", dict(_SGNHT, second_order=False, use_vector_alpha=False)),
}
NAMES = list(VARIANTS)


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def _sampler(zs, name, lj, prob, use_fused=True, lo=0, hi=None, **extra):
    cls, kw = VARIANTS[name]
    w0, w1 = T(prob.w0[lo:hi]), T(prob.w1[lo:hi])
    sg = getattr(zs, cls)(use_fused=use_fused, **dict(kw, **extra))
    op, info = sg.sample(lj, {}, {"w0": w0, "w1": w1})
    return sg, op, info, [w0, w1]


def _init_v(sg, v0):
    if hasattr(sg, "init_momentum"):
        sg.init_momentum({"w0": T(v0[0]), "w1": T(v0[1])})


def _oracle_sampler(name, v0):
    from oracle import sgmcmc as OS
    cls, kw = VARIANTS[name]
    osg = getattr(OS, cls)(dtype=F64, **kw)
    if cls == "SGNHT":
        osg.init_v(v0)
    return osg


def _ostep(osg, oq, grad, rs, nz):
    if hasattr(osg, "alphas"):
        return osg.step(oq, grad, rs, nz)
    return osg.step(oq, grad, nz)


def _dev_state(sg):
    """The method's state tensors per latent, by name (PSGLD keeps its aux in ``vs``)."""
    if hasattr(sg, "alphas"):
        return {"v": sg.vs, "alpha": sg.alphas}
    if hasattr(sg, "vs"):
        return {"aux": sg.vs}
    return {}


def _oracle_state(osg):
    if hasattr(osg, "alphas"):
        return {"v": osg.vs, "alpha": osg.alphas}
    if hasattr(osg, "aux"):
        return {"aux": osg.aux}
    return {}


def _set_oracle_state(osg, st):
    for key, vals in st.items():
        setattr(osg, {"v": "vs", "alpha": "alphas", "aux": "aux"}[key], vals)


# relative tolerance of each state, scaled by its largest entry as for the momenta of the SGHMC
# test: aux ~ g^2 carries twice the gradient's relative error, k = v^2 twice v's
_STATE_RTOL = {"v": 1e-5, "aux": 1e-4, "alpha": 2e-5, "k": 2e-5}


def _close(got, want, rtol, msg):
    want = np.asarray(want, F64)
    got = np.asarray(got, F64).reshape(want.shape)
    np.testing.assert_allclose(got, want, rtol=rtol,
                               atol=rtol * float(np.abs(want).max()) if want.size else 0.,
                               err_msg=msg)


def _skip_masks(sg, ties, gs):
    """Per-weight masks of [w0, w1] left out of the tight comparison: w0's ReLU ties and, for
    PSGLD, the weights whose gradient nearly cancels over the minibatch (|g| under 1e-3 of the
    largest in that chain and layer).  There the preconditioner 1 / (eps + sqrt(aux)) turns the
    float32 gradient's relative rounding error into weight differences well above a few ulps
    (0.02% of the weights at the benchmark shape, up to ~3e-3 apart); every weight is held to
    1e-2 instead."""
    skip = [np.broadcast_to(ties[:, :, None], gs[0].shape), np.zeros(gs[1].shape, bool)]
    if not hasattr(sg, "alphas") and hasattr(sg, "vs"):
        skip = [m | (np.abs(g) < 1e-3 * np.abs(g).max(axis=(1, 2), keepdims=True))
                for m, g in zip(skip, gs)]
    return skip


def _compare(tag, sg, info, ws, oq, ost, oinfo, ties, gs):
    assert ties.mean() < 0.05, "%s: %d ReLU ties" % (tag, ties.sum())
    dst = _dev_state(sg)
    skip = _skip_masks(sg, ties, gs)
    assert skip[0].mean() < 0.05 and skip[1].mean() < 0.05, tag
    for k, name in enumerate(("w0", "w1")):
        def sel(a):
            a = np.asarray(a)
            return a[~skip[k]] if a.shape == skip[k].shape else a
        np.testing.assert_allclose(sel(N(ws[k])), sel(oq[k]), rtol=2e-6, atol=2e-6,
                                   err_msg="%s: %s" % (tag, name))
        np.testing.assert_allclose(N(ws[k]), oq[k], rtol=0, atol=1e-2,
                                   err_msg="%s: %s, every weight" % (tag, name))
        for key, vals in dst.items():
            _close(sel(N(vals[k]).reshape(np.shape(ost[key][k]))), sel(ost[key][k]),
                   _STATE_RTOL[key], "%s: %s of %s" % (tag, key, name))
        if "mean_k" in oinfo:
            mk, want = N(info.mean_k[name]), oinfo["mean_k"][k]
            if np.ndim(want) == 0:
                np.testing.assert_allclose(float(mk), want, rtol=1e-4,
                                           err_msg="%s: mean_k of %s" % (tag, name))
            else:
                _close(sel(mk), sel(want), _STATE_RTOL["k"], "%s: k of %s" % (tag, name))


def _lockstep(tag, runs, prob, osg, om_of_step, steps, draws, observed_of_step=None,
              cross=False):
    """Step every (sg, op, info, ws) in ``runs`` and the oracle together; ``draws(t)`` gives the
    (noise, resample) standard normals of step t and whether to inject them.  After each step
    the oracle's state, rounded to float32, is copied into every run and kept by the oracle.
    ``cross``: the runs are also held to each other (fused against generic)."""
    oq = [prob.w0, prob.w1]
    for t in range(steps):
        nz, rs, inject = draws(t)
        om, at, gs = om_of_step(t), [], []

        def grad(qs):
            at.append(qs[0])
            gs.extend(om.grad(qs))
            return gs
        oq, oinfo = _ostep(osg, oq, grad, rs, nz)
        ost = _oracle_state(osg)
        ties = _relu_ties(om, at[0])
        for i, (sg, op, info, ws) in enumerate(runs):
            kw = {}
            if inject:
                kw["noise"] = {"noise": {"w0": T(nz[0]), "w1": T(nz[1])},
                               "resample": {"w0": T(rs[0]), "w1": T(rs[1])}}
            if observed_of_step is not None:
                kw["observed"] = observed_of_step(t)
            op(**kw)
            _compare("%s run %d step %d" % (tag, i, t), sg, info, ws, oq, ost, oinfo, ties, gs)
        if cross:
            ref = runs[0]
            ref_st = {key: [N(x) for x in v] for key, v in _dev_state(ref[0]).items()}
            for i, (sg, op, info, ws) in enumerate(runs[1:], 1):
                ref_info = ({"mean_k": [N(ref[2].mean_k[n]) for n in ("w0", "w1")]}
                            if hasattr(ref[2], "mean_k") else {})
                _compare("%s run %d against run 0, step %d" % (tag, i, t), sg, info, ws,
                         [N(w) for w in ref[3]], ref_st, ref_info, ties, gs)
        oq = [q.astype(np.float32).astype(F64) for q in oq]
        ost = {key: [np.asarray(x, np.float32).astype(F64) for x in v]
               for key, v in ost.items()}
        _set_oracle_state(osg, ost)
        for sg, op, info, ws in runs:
            for dst, src in zip(ws, oq):
                dst.copy_(T(src))
            for key, vals in _dev_state(sg).items():
                for dst, src in zip(vals, ost[key]):
                    dst.copy_(T(np.reshape(src, tuple(dst.shape))))


def _injected(prob):
    def draws(t):
        return prob.normals(), prob.normals(), True
    return draws


SHAPES = [pytest.param(shape, lss[0], id="%d-%d-%d-%d" % shape) for shape, _, lss in SWEEP]


@pytest.mark.parametrize("shape,ls", SHAPES)
@pytest.mark.parametrize("name", NAMES)
def test_fused_step_matches_oracle_across_shapes(zs, name, shape, ls):
    n_in, H, B, C = shape
    prob = Problem(n_in, H, B, C, ls=ls, n_train=50 * B + 17, y_logstd=-0.4, seed=sum(shape))
    # the 5000- and 8192-chain oracles are the slow part: 4 steps still cover t = 0 and t = 3
    steps = 4 if C > 1000 else 6
    sg, op, info, ws = _sampler(zs, name, prob.log_joint(zs), prob)
    assert sg._fused_bnn() is not None
    fused_steps = _count_fused(sg)
    v0 = prob.normals()
    _init_v(sg, v0)
    osg = _oracle_sampler(name, v0)
    om = prob.oracle()
    _lockstep("%s %s %s" % (name, shape, ls), [(sg, op, info, ws)], prob, osg, lambda t: om,
              steps, _injected(prob))
    assert fused_steps == list(range(steps))


@pytest.mark.parametrize("name", NAMES)
def test_in_kernel_philox_fused_and_generic_match_oracle(zs, name):
    """No injected noise: the oracle is fed the Philox draws rebuilt in NumPy (stream 3 for the
    update noise, 4 for re-draws of v, seed + k per latent), for samplers over more chains than
    one persistent round whose rows start at a non-zero chain offset.  The fused and the
    generic sampler run side by side and also agree with each other step for step."""
    row0 = 12345
    # H + 1 = 21 and H (n_in + 1) = 60 are not multiples of 4: the last Philox block is partial
    prob = Problem(4, 20, 24, 2300, ls=("hidden", "full"), n_train=1000, seed=5)
    lj = prob.log_joint(zs)
    runs, counts = [], []
    for use_fused in (True, False):
        run = _sampler(zs, name, lj, prob, use_fused=use_fused, seed=SEED, chain_offset=row0)
        counts.append(_count_fused(run[0]))
        runs.append(run)
    at, draws = _philox_draws(prob, row0)
    v0 = at(4, 0xFFFFFFFF)
    osg = _oracle_sampler(name, v0)
    if hasattr(osg, "vs"):
        for sg, _, _, _ in runs:
            for k in range(2):
                np.testing.assert_allclose(N(sg.vs[k]), v0[k] * np.sqrt(LR), rtol=1e-5,
                                           atol=1e-7)
        osg.vs = [N(v).astype(F64) for v in runs[0][0].vs]
    om = prob.oracle()
    _lockstep("philox " + name, runs, prob, osg, lambda t: om, 5, draws, cross=True)
    assert counts == [list(range(5)), []]


@pytest.mark.parametrize("n_in,H,B,fused", [
    (15, 64, 512, True),       # every limit reached: still fused
    (16, 64, 512, False),      # n_in + 1 = 17
    (15, 65, 512, False),      # H = 65
    (15, 64, 513, False),      # B = 513
])
@pytest.mark.parametrize("name", NAMES)
def test_fused_path_boundaries(zs, name, n_in, H, B, fused):
    """Past any of the kernel's limits the step takes the generic path, which still matches the
    oracle; at the limits it stays on the fused kernel (the most shared memory per warp)."""
    prob = Problem(n_in, H, B, 6, ls=("hidden", "full"), n_train=2000, seed=n_in + H + B)
    sg, op, info, ws = _sampler(zs, name, prob.log_joint(zs), prob)
    assert (sg._fused_bnn() is not None) == fused
    fused_steps = _count_fused(sg)
    v0 = prob.normals()
    _init_v(sg, v0)
    osg = _oracle_sampler(name, v0)
    om = prob.oracle()
    _lockstep("boundary " + name, [(sg, op, info, ws)], prob, osg, lambda t: om, 4,
              _injected(prob))
    assert fused_steps == (list(range(4)) if fused else [])


@pytest.mark.parametrize("name", ["sgld", "psgld", "sgnht-vec-2nd"])
def test_chain_sharding_is_bitwise(zs, name):
    """Chains split over two samplers (chain_offset = 0 and C1) follow the single sampler bit for
    bit: the in-kernel noise is keyed by the global chain, and nothing couples chains (scalar
    SGNHT is left out: its thermostat couples all chains by design)."""
    C, C1 = 4500, 2213
    prob = Problem(5, 40, 64, C, ls=("hidden", "full"), n_train=1000, seed=9)
    lj = prob.log_joint(zs)

    def run(lo, hi, offset):
        sg, op, info, ws = _sampler(zs, name, lj, prob, lo=lo, hi=hi, seed=SEED,
                                    chain_offset=offset)
        fused_steps = _count_fused(sg)
        for _ in range(5):
            op()
        assert len(fused_steps) == 5
        st = _dev_state(sg)
        return [N(w) for w in ws] + [N(x) for key in sorted(st) for x in st[key]]
    whole = run(0, C, None)
    parts = [run(0, C1, 0), run(C1, C, C1)]
    for k in range(len(whole)):
        np.testing.assert_array_equal(np.concatenate([parts[0][k], parts[1][k]]), whole[k],
                                      err_msg="array %d" % k)
    assert np.isfinite(whole[0]).all()


@pytest.mark.parametrize("name", NAMES)
def test_minibatch_switching_and_resume(zs, name):
    """Minibatches fed through sample_op(observed=...): one larger than the kernel stages runs on
    the generic path, the next returns to the fused kernel, and every step matches the oracle
    (the paths share every state tensor).  A state_dict() taken on the fused path, loaded into a
    fresh sampler, continues bit for bit."""
    rows = [slice(0, 100), slice(100, 137), slice(0, 600), slice(137, 237), slice(300, 400)]
    prob = Problem(6, 40, 100, 50, ls=("hidden", "full"), n_train=5000, seed=3, B_all=600)
    sg, op, info, ws = _sampler(zs, name, prob.log_joint(zs, rows[0]), prob)
    fused_steps = _count_fused(sg)
    v0 = prob.normals()
    _init_v(sg, v0)
    osg = _oracle_sampler(name, v0)
    oms = [prob.oracle(r) for r in rows]

    def obs(t):
        return {"x": T(prob.x_all[rows[t]]), "y": T(prob.y_all[rows[t]])}
    _lockstep("minibatch " + name, [(sg, op, info, ws)], prob, osg, lambda t: oms[t], len(rows),
              _injected(prob), obs)
    assert fused_steps == [0, 1, 3, 4]

    # resume: checkpoint, run three more fused steps with in-kernel noise, then replay them on a
    # fresh sampler restored from the checkpoint
    sg._seed = SEED
    ck = sg.state_dict()
    w_ck = [w.clone() for w in ws]
    tail = [slice(400, 500), slice(10, 90), slice(200, 300)]

    def go(op_):
        for r in tail:
            op_(observed={"x": T(prob.x_all[r]), "y": T(prob.y_all[r])})
        torch.cuda.synchronize()
    go(op)
    assert fused_steps == [0, 1, 3, 4, 5, 6, 7]
    want = [N(w) for w in ws] + [N(x) for v in _dev_state(sg).values() for x in v]
    sg2, op2, _, ws2 = _sampler(zs, name, prob.log_joint(zs, rows[0]), prob, seed=SEED)
    sg2.load_state_dict(ck)
    for dst, src in zip(ws2, w_ck):
        dst.copy_(src)
    n2 = _count_fused(sg2)
    go(op2)
    assert n2 == [5, 6, 7]
    got = [N(w) for w in ws2] + [N(x) for v in _dev_state(sg2).values() for x in v]
    for k, (a, b) in enumerate(zip(got, want)):
        np.testing.assert_array_equal(a, b, err_msg="array %d" % k)


_REF_TAGS = {"sgld": "sgld", "psgld": "psgld", "sgnht-vec-2nd": "sgnht_vec_2nd",
             "sgnht-vec-1st": "sgnht_vec_1st", "sgnht-scalar-2nd": "sgnht_scalar_2nd",
             "sgnht-scalar-1st": "sgnht_scalar_1st"}


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "generic"])
@pytest.mark.parametrize("name", NAMES)
def test_matches_reference_run(zs, name, fused):
    """tests/golden/ref_bnn_sgmcmc.npz: config 4's model run on the reference's own SGLD, PSGLD
    and SGNHT classes (tests/golden/make_ref_bnn_sgmcmc_golden.py).  The fused one-launch step
    and the generic path must follow it step for step."""
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                             "ref_bnn_sgmcmc.npz"))
    tag = _REF_TAGS[name]
    cfg = {k[len(tag) + 5:]: g[k] for k in g.files if k.startswith(tag + "/cfg_")}
    lj = zs.fused.BNNRegressionLogJoint(T(g["x"]), T(g["y"]), [T(g["logstd0"]), T(g["logstd1"])],
                                        int(g["n_train"]))
    w0, w1 = T(g["w0_init"]), T(g["w1_init"])
    cls, _ = VARIANTS[name]
    kw = {k: (bool(v) if k in ("second_order", "use_vector_alpha") else
              int(v) if k == "n_iter_resample_v" else float(v)) for k, v in cfg.items()}
    sg = getattr(zs, cls)(use_fused=fused, **kw)
    op, info = sg.sample(lj, {}, {"w0": w0, "w1": w1})
    assert sg._fused_bnn() is lj
    fused_steps = _count_fused(sg)
    _init_v(sg, [g["v0_0"], g["v0_1"]])
    steps = g[tag + "/w0"].shape[0]
    for t in range(steps):
        op(noise={"noise": {"w0": T(g[tag + "/noise0"][t]), "w1": T(g[tag + "/noise1"][t])},
                  "resample": {"w0": T(g[tag + "/resample0"][t]),
                               "w1": T(g[tag + "/resample1"][t])}})
        for k, (n, w) in enumerate((("w0", w0), ("w1", w1))):
            np.testing.assert_allclose(N(w), g[tag + "/w%d" % k][t], rtol=2e-4, atol=2e-5,
                                       err_msg="%s step %d %s" % (name, t, n))
            if cls == "SGNHT":
                mk = g[tag + "/mean_k%d" % k][t]
                np.testing.assert_allclose(N(info.mean_k[n]), mk, rtol=1e-3,
                                           atol=1e-3 * float(np.abs(mk).max()))
                np.testing.assert_allclose(N(info.alpha[n]), g[tag + "/alpha%d" % k][t],
                                           rtol=1e-4, atol=1e-6)
    assert fused_steps == (list(range(steps)) if fused else [])
