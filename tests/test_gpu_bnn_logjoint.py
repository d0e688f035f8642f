"""GPU tests of the fused BNN regression log-joint (csrc/bnn_logjoint.cu, zsb_bnn_logjoint_f32) and
the consumers that recognise zs.fused.BNNRegressionLogJoint through it: the variational objectives
(elbo / iw_objective / is_loglikelihood), HMC and ``predictive``.

The kernel is checked against the float64 oracle (oracle/models.py::BNN + tests/bnn_oracle.py)
over the shape range of the SG-MCMC sweep and over row counts that need several 512-row tiles;
bnn_vi.py's training step is replayed against the reference's own run (ref_bnn_vi.npz) on the
fused and the generic path."""
import itertools
import math
import os

import numpy as np
import pytest
import torch

from bnn_oracle import BNN
from test_gpu_bnn_sghmc import SWEEP, Problem, T, N, _relu_ties

pytestmark = pytest.mark.gpu

F64 = np.float64
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
OUTS = ("lp", "g0", "g1", "gys", "ym", "ll")


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def _oracle(prob):
    return BNN(prob.x_all, prob.y_all, prob.n_train, prob.ls[0], prob.ls[1], dtype=F64,
               y_logstd=prob.y_logstd)


def _launch(lj, prob, want):
    w0, w1 = T(prob.w0), T(prob.w1)
    x, y = lj.x, lj.y
    return dict(zip(OUTS, lj._launch(w0, w1, x, y, lj._y_logstd_dev(w0.device),
                                     **{k: True for k in want})))


def _check(tag, got, prob, om, ties=None):
    """Every output in ``got`` that is not None against the float64 oracle."""
    B = prob.x_all.shape[0]
    gtol = 1e-5 if B <= 512 else 1e-4
    q = [prob.w0, prob.w1]
    if ties is None:
        ties = _relu_ties(om, prob.w0)
    assert ties.mean() < 0.05, "%s: %d ReLU ties" % (tag, ties.sum())
    ym, ll = om.predictive(q)
    want = {"lp": om.logp(q), "gys": om.grad_y_logstd(q), "ym": ym, "ll": ll}
    want["g0"], want["g1"] = om.grad(q)
    for k, v in got.items():
        if v is None:
            continue
        a, b = N(v).astype(F64), want[k]
        assert a.shape == b.shape, (tag, k, a.shape, b.shape)
        if k in ("g0", "g1"):
            scale = np.abs(b).reshape(b.shape[0], -1).max(1)[:, None, None]
            err = np.abs(a - b) / scale
            if k == "g0":
                err = err[~ties]
            assert err.max() <= gtol, "%s: %s max err %.3g of the particle's largest entry" % (
                tag, k, err.max())
        elif k == "lp":
            np.testing.assert_allclose(a, b, rtol=1e-5, err_msg="%s: lp" % tag)
        elif k == "gys":
            # d lp / d y_logstd = n_train (mean prec r^2 - 1): relative to its two terms
            np.testing.assert_allclose(a, b, rtol=0, atol=1e-5 * float(np.abs(b).max() +
                                                                        prob.n_train),
                                       err_msg="%s: gys" % tag)
        else:
            scale = np.abs(b).max(1, keepdims=True)
            err = np.abs(a - b) / scale
            assert err.max() <= 1e-5, "%s: %s max err %.3g" % (tag, k, err.max())


# (n_in, H, B, K) rows tiled over several 512-row tiles, K not a multiple of 8 warps per block
TILED = [((13, 50, 513, 37), ("hidden", "full")), ((9, 50, 2000, 20), ("input", "scalar")),
         ((10, 64, 4096, 9), ("full", "full")), ((15, 33, 1100, 3), ("scalar", "full"))]
# shapes whose dynamic shared memory lies just under 48 KB but over 48 KB minus the kernel's
# static shared memory: they launch only with the opt-in
SMEM_EDGE = [((10, 50, 482, 13), ("full", "full")), ((15, 64, 130, 5), ("hidden", "scalar")),
             ((13, 64, 194, 6), ("input", "full"))]
CASES = [pytest.param(shape, ls, id="%d-%d-%d-%d-%s-%s" % (shape + ls))
         for shape, _, lss in SWEEP for ls in lss] + \
    [pytest.param(shape, ls, id="tiled-%d-%d-%d-%d-%s-%s" % (shape + ls)) for shape, ls in TILED] + \
    [pytest.param(shape, ls, id="smem-%d-%d-%d-%d-%s-%s" % (shape + ls))
     for shape, ls in SMEM_EDGE]


@pytest.mark.parametrize("shape,ls", CASES)
def test_kernel_matches_oracle(zs, shape, ls):
    n_in, H, B, K = shape
    prob = Problem(n_in, H, B, K, ls=ls, n_train=50 * B + 17, y_logstd=-0.4, seed=sum(shape) + 1)
    lj = prob.log_joint(zs)
    om = _oracle(prob)
    _check("%s %s all" % (shape, ls), _launch(lj, prob, OUTS), prob, om)
    # value only (no backward pass compiled in), gradient only, predictions only
    for want in (("lp",), ("g0", "g1"), ("gys", "ym", "ll")):
        got = _launch(lj, prob, want)
        assert all((got[k] is None) == (k not in want) for k in OUTS)
        _check("%s %s %s" % (shape, ls, want), got, prob, om)


def test_every_output_subset(zs):
    """All 64 subsets of the six outputs: the requested ones are written and right, and a
    requested output does not depend on which others are requested."""
    prob = Problem(6, 40, 700, 11, ls=("hidden", "full"), n_train=900, seed=21)
    lj = prob.log_joint(zs)
    om = _oracle(prob)
    full = {k: N(v) for k, v in _launch(lj, prob, OUTS).items()}
    _check("full", _launch(lj, prob, OUTS), prob, om)
    for r in range(len(OUTS) + 1):
        for want in itertools.combinations(OUTS, r):
            got = _launch(lj, prob, want)
            for k in OUTS:
                if k not in want:
                    assert got[k] is None
                    continue
                np.testing.assert_allclose(N(got[k]), full[k], rtol=1e-6,
                                           atol=1e-6 * float(np.abs(full[k]).max()),
                                           err_msg="%s of %s" % (k, want))


def test_kernel_is_deterministic(zs):
    prob = Problem(10, 50, 2000, 300, ls=("hidden", "full"), n_train=5000, seed=4)
    lj = prob.log_joint(zs)
    a = [N(v) for v in _launch(lj, prob, OUTS).values()]
    b = [N(v) for v in _launch(lj, prob, OUTS).values()]
    for u, v in zip(a, b):
        assert u.tobytes() == v.tobytes()


def test_fused_log_joint_autograd(zs):
    """Backward with a non-uniform upstream [K] gradient against the oracle and against
    torch.autograd through __call__ (w0, w1 and a tensor y_logstd)."""
    prob = Problem(8, 30, 150, 12, ls=("hidden", "scalar"), n_train=700, y_logstd=-0.4, seed=8)
    om = _oracle(prob)
    up = np.random.RandomState(1).uniform(-1, 2, prob.C)
    grads = []
    for fused in (True, False):
        ys = torch.tensor(prob.y_logstd, dtype=torch.float32, device="cuda", requires_grad=True)
        lj = zs.fused.BNNRegressionLogJoint(T(prob.x_all), T(prob.y_all), [T(l) for l in prob.ls],
                                            prob.n_train, y_logstd=ys)
        w0 = T(prob.w0).requires_grad_(True)
        w1 = T(prob.w1).requires_grad_(True)
        obs = {"w0": w0, "w1": w1}
        lp = lj.fused_log_joint(obs) if fused else lj(obs)
        np.testing.assert_allclose(N(lp), om.logp([prob.w0, prob.w1]), rtol=1e-5)
        grads.append([N(g) for g in torch.autograd.grad((lp * T(up)).sum(), [w0, w1, ys])])
    g0, g1 = om.grad([prob.w0, prob.w1])
    want = [(g0 * up[:, None, None]), (g1 * up[:, None, None]),
            (om.grad_y_logstd([prob.w0, prob.w1]) * up).sum()]
    ties = _relu_ties(om, prob.w0)
    for tag, got in zip(("fused", "torch"), grads):
        for k, (a, b) in enumerate(zip(got, want)):
            scale = float(np.abs(b).max())
            if k == 2:                     # n_train (mean prec r^2 - 1): relative to its terms
                scale += prob.n_train * float(np.abs(up).sum())
            if k == 0:
                a, b = a[~ties], b[~ties]
            np.testing.assert_allclose(a, b, rtol=0, atol=(1e-5 if tag == "fused" else 1e-4) *
                                       scale, err_msg="%s grad %d" % (tag, k))


def test_no_grad_takes_value_only_launch_and_no_double_backward(zs):
    """Under torch.no_grad() fused_log_joint launches without any gradient output, even for
    inputs that require one; with gradients recorded, the gradient is first order only."""
    prob = Problem(5, 20, 40, 6, ls=("hidden", "full"), n_train=300, seed=3)
    lj = prob.log_joint(zs)
    w0, w1 = T(prob.w0).requires_grad_(True), T(prob.w1).requires_grad_(True)
    obs = {"w0": w0, "w1": w1}
    asked = []
    run = lj._launch
    lj._launch = lambda *a, **kw: asked.append(sorted(k for k, v in kw.items() if v)) or \
        run(*a, **kw)
    with torch.no_grad():
        lp0 = lj.fused_log_joint(obs)
    lp1 = lj.fused_log_joint(obs)
    assert asked == [["lp"], ["g0", "g1", "lp"]]
    assert lp0.grad_fn is None
    np.testing.assert_array_equal(N(lp0), N(lp1))
    g0, = torch.autograd.grad(lp1.sum(), [w0], create_graph=True)
    with pytest.raises(RuntimeError):
        g0.sum().backward()


# ---------------------------------------------------------------- bnn_vi.py replay
def _injected_normal(zs):
    class InjectedNormal(zs.distributions.Normal):
        def __init__(self, *a, **kw):
            self._eps = kw.pop("eps")
            super(InjectedNormal, self).__init__(*a, **kw)

        def _sample(self, n_samples):
            return super(InjectedNormal, self)._sample(n_samples, eps=self._eps)
    return InjectedNormal


VARS = ["w_mean_0", "w_logstd_0", "w_mean_1", "w_logstd_1", "y_logstd"]


def _vi_setup(zs, g, eps, x, y):
    """bnn_vi.py's model and mean-field variational net at the fixture's variables."""
    InjectedNormal = _injected_normal(zs)
    V = {n: T(g["var_" + n]).requires_grad_(True) for n in VARS}
    zero = torch.zeros((), device="cuda")
    lj = zs.fused.BNNRegressionLogJoint(T(x), T(y), [zero, zero], int(g["n_train"]),
                                        y_logstd=V["y_logstd"])
    K = eps[0].shape[0]

    def variational():
        bn = zs.BayesianNet()
        for i in range(2):
            bn.stochastic("w%d" % i, InjectedNormal(V["w_mean_%d" % i], logstd=V["w_logstd_%d" % i],
                                                    group_ndims=2, eps=T(eps[i])), n_samples=K)
        return bn
    return lj, V, variational


@pytest.mark.parametrize("fused", [True, False], ids=["fused", "generic"])
def test_bnn_vi_elbo_replays_reference(zs, fused):
    g = np.load(os.path.join(GOLD, "ref_bnn_vi.npz"))
    lj, V, variational = _vi_setup(zs, g, [g["eps0"], g["eps1"]], g["x"], g["y"])
    model = lj if fused else (lambda o: lj(o))
    obs = {"x": T(g["x"]), "y": T(g["y"])}
    lb = zs.variational.elbo(model, obs, variational=variational(), axis=0)
    calls = []
    run = lj.fused_log_joint
    lj.fused_log_joint = lambda o: calls.append(1) or run(o)
    np.testing.assert_allclose(float(lb.tensor.detach()), float(g["lower_bound"]), rtol=1e-5)
    assert len(calls) == (1 if fused else 0)
    cost = lb.sgvb()
    np.testing.assert_allclose(float(cost.detach()), float(g["cost"]), rtol=1e-5)
    grads = torch.autograd.grad(cost, [V[n] for n in VARS])
    for n, gr in zip(VARS, grads):
        ref = g["grad_" + n]
        np.testing.assert_allclose(N(gr), ref, rtol=1e-4, atol=1e-4 * float(np.abs(ref).max()),
                                   err_msg="%s fused=%s" % (n, fused))


def test_bnn_vi_prediction_replays_reference(zs):
    """bnn_vi.py:98-103 (rmse and the test log-likelihood over ll_samples particles) from one
    predictive() launch."""
    g = np.load(os.path.join(GOLD, "ref_bnn_vi.npz"))
    eps = [g["eps_ll0"], g["eps_ll1"]]
    lj, V, variational = _vi_setup(zs, g, eps, g["x_test"], g["y_test"])
    net = variational()
    ws = {n: net.nodes[n].tensor.detach() for n in ("w0", "w1")}
    y_mean, log_lik = lj.predictive(ws)
    np.testing.assert_allclose(N(y_mean), g["ll_y_mean"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(N(log_lik), g["ll_log_py_xw"], rtol=1e-5, atol=1e-5)
    std = float(g["std_y_train"])
    yt = T(g["y_test"])
    rmse = ((y_mean.mean(0) - yt) ** 2).mean().sqrt() * std
    ll = (torch.logsumexp(log_lik, 0) - math.log(log_lik.shape[0])).mean() - math.log(std)
    np.testing.assert_allclose(float(rmse), float(g["ll_rmse"]), rtol=1e-5)
    np.testing.assert_allclose(float(ll), float(g["ll_log_likelihood"]), rtol=1e-5)


def test_iw_objective_and_is_loglikelihood_match_generic(zs):
    """Non-uniform upstream weights (the normalised importance weights) through the fused
    backward, against the generic path on the same draws."""
    g = np.load(os.path.join(GOLD, "ref_bnn_vi.npz"))
    obs = {"x": T(g["x"]), "y": T(g["y"])}
    res = []
    for fused in (True, False):
        lj, V, variational = _vi_setup(zs, g, [g["eps0"], g["eps1"]], g["x"], g["y"])
        model = lj if fused else (lambda o: lj(o))
        iw = zs.variational.iw_objective(model, obs, variational=variational(), axis=0)
        cost = iw.sgvb()
        grads = torch.autograd.grad(cost, [V[n] for n in VARS])
        with torch.no_grad():
            ll = zs.is_loglikelihood(model, obs, proposal=variational(), axis=0)
        res.append((float(iw.tensor), float(cost), [N(x) for x in grads], float(ll)))
    (b0, c0, g0, l0), (b1, c1, g1, l1) = res
    np.testing.assert_allclose(b0, b1, rtol=1e-5)
    np.testing.assert_allclose(c0, c1, rtol=1e-5)
    np.testing.assert_allclose(l0, l1, rtol=1e-5)
    for n, a, b in zip(VARS, g0, g1):
        np.testing.assert_allclose(a, b, rtol=1e-4, atol=1e-4 * float(np.abs(b).max()), err_msg=n)


# ---------------------------------------------------------------- HMC
def test_hmc_provider_matches_oracle(zs):
    from oracle import hmc as OH
    prob = Problem(5, 20, 60, 24, ls=("hidden", "full"), n_train=60, y_logstd=-0.4, seed=31)
    prob.w0 *= 0.3
    prob.w1 *= 0.3
    lj = prob.log_joint(zs)
    om = _oracle(prob)
    w0, w1 = T(prob.w0), T(prob.w1)
    h = zs.HMC(step_size=2e-3, n_leapfrogs=5)
    op, info = h.sample(lj, {}, {"w0": w0, "w1": w1})
    assert type(h._provider).__name__ == "_BNNProvider" and h._fused is None
    oh = OH.HMC(step_size=2e-3, n_leapfrogs=5)
    oq = [prob.w0, prob.w1]
    rng = np.random.RandomState(5)
    n_acc = 0
    for i in range(4):
        npz = [rng.standard_normal(q.shape).astype(np.float32) for q in oq]
        nu = rng.random_sample(prob.C).astype(np.float32)
        # keep the uniforms away from the acceptance probabilities, so float32 and float64
        # take the same decisions (no adaptation: a repeated oracle step is the same step)
        acc_o = oh.step(oq, om.logp, om.grad, npz, nu)[1].acceptance_rate
        nu = np.where(np.abs(nu - acc_o) < 1e-2, np.clip(acc_o + 0.05, 0, 1), nu)
        nu = nu.astype(np.float32)
        oq_new, oi = oh.step(oq, om.logp, om.grad, npz, nu)
        op(noise={"p": {"w0": T(npz[0]), "w1": T(npz[1])}, "u": T(nu)})
        acc = N(info.acceptance_rate)
        np.testing.assert_array_equal(acc > nu, oi.if_accept)
        np.testing.assert_allclose(acc, oi.acceptance_rate, rtol=2e-3, atol=2e-4)
        np.testing.assert_allclose(N(info.orig_log_prob), oi.orig_log_prob, rtol=1e-5)
        for got, want in zip((w0, w1), oq_new):
            np.testing.assert_allclose(N(got), want, rtol=1e-4, atol=1e-4)
        n_acc += int(oi.if_accept.sum())
        oq = [N(w0).astype(F64), N(w1).astype(F64)]
    assert 0 < n_acc


def test_hmc_full_batch_over_512_rows(zs):
    """Full-batch HMC over 700 rows (two tiles) with the in-kernel draws: the provider is taken,
    and the log-probability it reports is the oracle's at the final state."""
    prob = Problem(13, 50, 700, 64, ls=("scalar", "scalar"), n_train=700, y_logstd=-0.4, seed=2)
    prob.w0 *= 0.2
    prob.w1 *= 0.2
    lj = prob.log_joint(zs)
    w0, w1 = T(prob.w0), T(prob.w1)
    h = zs.HMC(step_size=1e-3, n_leapfrogs=10)
    op, info = h.sample(lj, {}, {"w0": w0, "w1": w1})
    assert h._provider is not None
    for _ in range(3):
        op()
    op.synchronize()
    acc = N(info.acceptance_rate)
    assert np.all(np.isfinite(acc)) and np.all((acc >= 0) & (acc <= 1)) and acc.mean() > 0
    om = _oracle(prob)
    q = [N(w0).astype(F64), N(w1).astype(F64)]
    np.testing.assert_allclose(N(lj.hmc_provider(["w0", "w1"], {}, [w0, w1]).logp([w0, w1])),
                               om.logp(q), rtol=1e-5)
    np.testing.assert_allclose(N(info.log_prob), om.logp(q), rtol=1e-5)


# ---------------------------------------------------------------- fallback
@pytest.mark.parametrize("case", ["H65", "n_in16", "latent4d", "chain_prior", "prior_grad"])
def test_ineligible_inputs_take_generic_path(zs, case):
    n_in, H = {"H65": (4, 65), "n_in16": (16, 20)}.get(case, (4, 20))
    ls = ("chain", "full") if case == "chain_prior" else ("hidden", "full")
    prob = Problem(n_in, H, 40, 6, ls=ls, n_train=300, seed=17)
    lj = prob.log_joint(zs)
    if case == "prior_grad":
        lj.logstds[0].requires_grad_(True)
    w0, w1 = T(prob.w0), T(prob.w1)
    if case == "latent4d":
        w0, w1 = w0.view((2, 3) + w0.shape[1:]), w1.view((2, 3) + w1.shape[1:])
    obs = {"w0": w0, "w1": w1}
    assert lj.fused_inputs(obs) is None
    assert lj.hmc_provider(["w0", "w1"], {}, [w0, w1]) is None
    w0.requires_grad_(True)
    seen = []

    class Spy(object):
        _zsb_fused = lj._zsb_fused

        def __call__(self, o):
            seen.append(1)
            return lj(o)
    zero = torch.zeros(w0.shape[:-2], device="cuda")
    with pytest.warns(FutureWarning):           # the deprecated latent= dictionary
        lb = zs.variational.elbo(Spy(), {}, latent={"w0": [w0, zero], "w1": [w1, zero]},
                                 axis=0)
    if case == "latent4d":
        # __call__ (the example's einsum "imk,ijk->ijm") is defined for one chain axis: the
        # objective hands the latents to it and reports exactly what it reports
        with pytest.raises(RuntimeError) as generic:
            lj(obs)
        with pytest.raises(RuntimeError) as got:
            lb.tensor
        assert seen == [1] and str(got.value) == str(generic.value)
        return
    val = lb.tensor
    assert seen == [1]
    np.testing.assert_allclose(float(val), float(lj(obs).mean()), rtol=1e-6)
    om = _oracle(prob)
    np.testing.assert_allclose(N(lj(obs)), om.logp([prob.w0, prob.w1]), rtol=1e-4)


def test_float64_prior_or_foreign_device_is_ineligible(zs):
    """The kernel reads the scales as float32 on the latents' device: anything else is left to
    the generic path."""
    prob = Problem(4, 20, 40, 6, ls=("hidden", "full"), n_train=300, seed=17)
    lj = prob.log_joint(zs)
    obs = {"w0": T(prob.w0), "w1": T(prob.w1)}
    assert lj.fused_inputs(obs) is not None
    lj.logstds[0] = lj.logstds[0].double()
    assert lj.fused_inputs(obs) is None
    lj.logstds[0] = T(prob.ls[0])
    lj.logstds[1] = lj.logstds[1].cpu()
    assert lj.fused_inputs(obs) is None
    lj.logstds[1] = T(prob.ls[1])
    assert lj.fused_inputs(dict(obs, x=lj.x.cpu())) is None


def test_hmc_provider_falls_back_per_call(zs):
    """HMC picks the provider in sample(); an iteration whose inputs the kernel no longer accepts
    (here a prior scale that starts requiring a gradient) runs the generic path and matches an HMC
    on the generic path itself."""
    prob = Problem(5, 20, 60, 8, ls=("hidden", "full"), n_train=60, seed=19)
    prob.w0 *= 0.3
    prob.w1 *= 0.3
    rng = np.random.RandomState(2)
    npz = [rng.standard_normal(w.shape).astype(np.float32) for w in (prob.w0, prob.w1)]
    nu = rng.random_sample(prob.C).astype(np.float32)
    res = []
    for fused in (True, False):
        lj = prob.log_joint(zs)
        w0, w1 = T(prob.w0), T(prob.w1)
        h = zs.HMC(step_size=2e-3, n_leapfrogs=3)
        op, info = h.sample(lj if fused else (lambda o: lj(o)), {}, {"w0": w0, "w1": w1})
        assert (h._provider is not None) == fused
        lj.logstds[0].requires_grad_(True)
        op(noise={"p": {"w0": T(npz[0]), "w1": T(npz[1])}, "u": T(nu)})
        res.append([N(w0), N(w1), N(info.acceptance_rate)])
    for a, b in zip(*res):
        np.testing.assert_allclose(a, b, rtol=1e-6, atol=1e-6)


def test_tensor_y_logstd_sghmc_takes_generic_path(zs):
    """SG-MCMC's fused step takes y_logstd by value: with a tensor y_logstd the sampler runs its
    generic path, which follows the float-y_logstd fused step."""
    prob = Problem(6, 30, 64, 16, ls=("hidden", "full"), n_train=500, y_logstd=-0.4, seed=13)
    runs = []
    for ys in (prob.y_logstd, torch.tensor(prob.y_logstd, dtype=torch.float32, device="cuda")):
        lj = zs.fused.BNNRegressionLogJoint(T(prob.x_all), T(prob.y_all), [T(l) for l in prob.ls],
                                            prob.n_train, y_logstd=ys)
        w0, w1 = T(prob.w0), T(prob.w1)
        sg = zs.SGHMC(learning_rate=2e-5, friction=0.2, variance_estimate=0.01,
                      n_iter_resample_v=3, second_order=True)
        op, _ = sg.sample(lj, {}, {"w0": w0, "w1": w1})
        assert (sg._fused_bnn() is None) == isinstance(ys, torch.Tensor)
        runs.append((sg, op, [w0, w1]))
    rng = np.random.RandomState(0)
    v0 = [rng.standard_normal(s).astype(np.float32) for s in (prob.w0.shape, prob.w1.shape)]
    for sg, _, _ in runs:
        sg.init_momentum({"w0": T(v0[0]), "w1": T(v0[1])})
    for t in range(4):
        nz = [rng.standard_normal(s).astype(np.float32) for s in (prob.w0.shape, prob.w1.shape)]
        rs = [rng.standard_normal(s).astype(np.float32) for s in (prob.w0.shape, prob.w1.shape)]
        for sg, op, _ in runs:
            op(noise={"noise": {"w0": T(nz[0]), "w1": T(nz[1])},
                      "resample": {"w0": T(rs[0]), "w1": T(rs[1])}})
    for a, b in zip(runs[0][2], runs[1][2]):
        np.testing.assert_allclose(N(b), N(a), rtol=1e-5, atol=1e-5)


# ---------------------------------------------------------------- C ABI
def test_c_abi_rejects_bad_arguments(zs):
    from zhusuan_b200._lib import lib, ptr, stream
    prob = Problem(4, 10, 20, 3, seed=1)
    lj = prob.log_joint(zs)
    w0, w1, x, y = T(prob.w0), T(prob.w1), lj.x, lj.y
    ls0, ls1 = lj.logstds
    ys = lj._y_logstd_dev(w0.device)
    lp = torch.empty(3, device="cuda")
    dll = lib.load()

    def call(K=3, B=20, n_in=4, H=10, w0_p=ptr(w0), x_p=ptr(x), ys_p=ptr(ys), ls0_n=ls0.numel()):
        return dll.zsb_bnn_logjoint_f32(w0_p, ptr(w1), x_p, ptr(y), B, n_in, H, ptr(ls0), ls0_n,
                                        ptr(ls1), ls1.numel(), ys_p, 300.0, ptr(lp), None, None,
                                        None, None, None, K, stream())
    assert call() == 0
    torch.cuda.synchronize()
    for bad in (dict(K=0), dict(B=0), dict(n_in=0), dict(n_in=16), dict(H=0), dict(H=65),
                dict(w0_p=None), dict(x_p=None), dict(ys_p=None), dict(ls0_n=0),
                dict(ls0_n=10 ** 6)):
        assert call(**bad) != 0, bad
        assert "zsb_bnn_logjoint_f32" in lib.last_error()
    call(H=65)
    assert "H = 65" in lib.last_error()
    torch.cuda.synchronize()
