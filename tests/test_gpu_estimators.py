"""GPU parity: the score-function / self-normalised estimators (SURVEY 8f row 2) --
VIMCO (monte_carlo.py:166-227), importance / RWS (inclusive_kl.py:119-151) and
REINFORCE (exclusive_kl.py:161-231) -- against the CPU oracle and the reference's
own seeded gradient tests (tests/variational/test_monte_carlo.py:104-142,
test_inclusive_kl.py:26-92, test_exclusive_kl.py:80-122)."""
import os
import warnings

import numpy as np
import pytest
import torch

from oracle import variational as OV

pytestmark = pytest.mark.gpu


def T(a, dtype=torch.float32):
    return torch.tensor(np.asarray(a), dtype=dtype, device="cuda")


def N(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


@pytest.mark.parametrize("shape,axis", [((64, 300), 0), ((7, 33), 1), ((3, 5, 11), 1),
                                        ((2, 1), 0), ((1000, 4), 0)])
def test_vimco_signal_and_weights_vs_oracle(zs, shape, axis):
    rng = np.random.RandomState(sum(shape) + axis)
    l = (rng.standard_normal(shape) * 4).astype(np.float32)
    sig, lme = zs.ops.vimco_signal(T(l), axis)
    want = OV.vimco_signal(l, axis, np.float64)
    np.testing.assert_allclose(N(sig), want, rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(N(lme), OV.log_mean_exp(l, axis, keepdims=True, dtype=np.float64),
                               rtol=1e-6, atol=1e-6)
    w = zs.ops.normalized_weights(T(l), axis)
    np.testing.assert_allclose(N(w), OV.normalized_weights(l, axis, np.float64), rtol=1e-5,
                               atol=1e-9)
    np.testing.assert_allclose(N(w.sum(axis)), 1.0, rtol=1e-5)


def test_vimco_signal_extremes(zs):
    """One dominant weight (the leave-one-out sum for the arg-max must not cancel), exact ties,
    and very negative entries."""
    K, n = 16, 8
    l = np.full((K, n), -3.0, np.float32)
    l[3, 0] = 60.0                    # dominant
    l[:, 1] = 1.5                     # all tied
    l[5, 2] = l[9, 2] = 20.0          # two-way tie for the maximum
    l[2, 3] = -1e4                    # exp underflows
    l[:, 4] = np.linspace(-80, 80, K)
    sig, _ = zs.ops.vimco_signal(T(l), 0)
    want = OV.vimco_signal(l, 0, np.float64)
    np.testing.assert_allclose(N(sig), want, rtol=2e-5, atol=2e-5)
    assert np.isfinite(N(sig)).all()
    with pytest.raises(ValueError, match="larger than 1"):
        zs.ops.vimco_signal(T(l[:1]), 0)


@pytest.mark.parametrize("x_mean,x_std,thr", [(0., 1., 1e-2), (2., 3., 1e-6)])
def test_vimco_reference_test(zs, x_mean, x_std, thr):
    """tests/variational/test_monte_carlo.py:104-142: VIMCO gradient == SGVB gradient."""
    rng = np.random.RandomState(1)
    rng.standard_normal(size=(1, 1000))
    eps = T(rng.standard_normal(1000).astype(np.float32))
    mu = T(2.).requires_grad_(True)
    sigma = T(3.).requires_grad_(True)
    Normal = zs.distributions.Normal
    qx = eps * sigma + mu
    log_qx = Normal(mean=mu, std=sigma).log_prob(qx)
    v_qx = eps * sigma.detach() + mu.detach()
    v_log_qx = Normal(mean=mu, std=sigma).log_prob(v_qx)

    def log_joint(observed):
        return Normal(mean=x_mean, std=x_std).log_prob(observed['x'])
    with pytest.warns(FutureWarning):
        lb = zs.variational.importance_weighted_objective(
            log_joint, observed={}, latent={'x': [qx, log_qx]}, axis=0)
        v_lb = zs.variational.importance_weighted_objective(
            log_joint, observed={}, latent={'x': [v_qx, v_log_qx]}, axis=0)
    g1 = torch.autograd.grad(torch.mean(v_lb.vimco()), [mu, sigma])
    g2 = torch.autograd.grad(torch.mean(lb.sgvb()), [mu, sigma])
    np.testing.assert_allclose([float(g1[0]), float(g1[1])], [float(g2[0]), float(g2[1])],
                               rtol=thr, atol=thr)
    # the cost itself against the oracle
    c = OV.vimco_cost(N(log_joint({'x': v_qx})), N(v_log_qx), 0, np.float64)
    np.testing.assert_allclose(float(v_lb.vimco()), c, rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("x_mean,x_std,thr", [(0., 1., 0.01), (2., 3., 0.02)])
def test_importance_reference_test(zs, x_mean, x_std, thr):
    """tests/variational/test_inclusive_kl.py:44-72."""
    eps = T(np.random.RandomState(1).standard_normal(100000).astype(np.float32))
    mu = T(2.).requires_grad_(True)
    sigma = T(3.).requires_grad_(True)
    Normal = zs.distributions.Normal
    qx = (eps * sigma + mu).detach()
    log_qx = Normal(mean=mu, std=sigma).log_prob(qx)

    def log_joint(observed):
        return Normal(mean=x_mean, std=x_std).log_prob(observed['x'])
    with pytest.warns(FutureWarning):
        obj = zs.variational.klpq(log_joint, observed={}, latent={'x': [qx, log_qx]}, axis=0)
    cost = obj.importance()
    g = torch.autograd.grad(cost, [mu, sigma])
    true = (-(x_mean - 2.) / 9., 1. / 3. - (x_std ** 2 + (x_mean - 2.) ** 2) / 27.)
    np.testing.assert_allclose([float(g[0]), float(g[1])], true, rtol=thr, atol=thr)
    want = OV.importance_cost(N(log_joint({'x': qx})), N(log_qx), 0, np.float64)
    np.testing.assert_allclose(float(cost), want, rtol=1e-4)


def test_klpq_contract(zs):
    """test_inclusive_kl.py:26-42, 74-92: not evaluable; rws() deprecation; single-sample warning."""
    Normal = zs.distributions.Normal
    x = T(np.random.RandomState(0).standard_normal(10))
    log_q = Normal(mean=0., std=1.).log_prob(x)

    def log_joint(observed):
        return Normal(std=1.).log_prob(observed['x'])
    with pytest.warns(FutureWarning):
        obj = zs.variational.klpq(log_joint, observed={}, latent={'x': [x, log_q]}, axis=0)
    with pytest.raises(NotImplementedError, match="can only be optimized instead of being evaluated"):
        obj.tensor
    with pytest.raises(NotImplementedError):
        obj + 1.
    with pytest.warns(FutureWarning, match="renamed to `importance\\(\\)`"):
        obj.rws()
    with pytest.warns(FutureWarning):
        single = zs.variational.klpq(log_joint, observed={}, latent={'x': [x[0], log_q[0]]})
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        single.importance()
        assert issubclass(w[-1].category, UserWarning)
        assert "biased and inaccurate when you're using only a single sample" in str(w[-1].message)


@pytest.mark.parametrize("x_mean,x_std,rtol,atol", [(0., 1., 1e-2, 1e-6), (2., 3., 1e-6, 1e-6)])
def test_reinforce_reference_test(zs, x_mean, x_std, rtol, atol):
    """tests/variational/test_exclusive_kl.py:80-112."""
    rng = np.random.RandomState(1)
    rng.standard_normal(100000)
    eps = T(rng.standard_normal(1000000).astype(np.float32))
    mu = T(2.).requires_grad_(True)
    sigma = T(3.).requires_grad_(True)
    Normal = zs.distributions.Normal
    qx = (eps * sigma + mu).detach()
    log_qx = Normal(mean=mu, std=sigma).log_prob(qx)

    def log_joint(observed):
        return Normal(mean=x_mean, std=x_std).log_prob(observed['x'])
    with pytest.warns(FutureWarning):
        lb = zs.variational.elbo(log_joint, observed={}, latent={'x': [qx, log_qx]}, axis=0)
    cost = lb.reinforce(variance_reduction=False)
    g = torch.autograd.grad(cost, [mu, sigma])
    true = ((2. - x_mean) / x_std ** 2, -1 / 3. + 3. / x_std ** 2)
    np.testing.assert_allclose([float(g[0]), float(g[1])], true, rtol=rtol, atol=atol)
    want = OV.reinforce_cost(N(log_joint({'x': qx})), N(log_qx), 0, np.float64)
    np.testing.assert_allclose(float(cost), want, rtol=1e-4, atol=1e-5)
    # variance-reduced variants: moving-mean baseline, and a learned baseline with its own cost
    with pytest.warns(FutureWarning):
        lb2 = zs.variational.elbo(log_joint, observed={}, latent={'x': [qx, log_qx]}, axis=0)
    c2 = lb2.reinforce()
    assert torch.isfinite(c2)
    b = T(0.1).requires_grad_(True)
    c3, bc = lb2.reinforce(baseline=b)
    assert torch.isfinite(c3) and torch.isfinite(bc)
    assert torch.autograd.grad(bc, [b])[0] is not None
    # the moving-mean baseline is ONE persistent variable (tf.get_variable('moving_mean'),
    # exclusive_kl.py:209-216): it keeps averaging across objective instances / training steps
    from zhusuan_b200.variational import exclusive_kl as EK
    EK.reset_moving_mean()
    # update rule: TF's assign_moving_average with its default zero_debias=True (restated in
    # oracle/variational.py::zero_debiased_moving_average); pinned to the reference's own
    # exclusive_kl.py run on the TF stand-in by test_vae_objectives_match_reference_run below
    signal = float((log_joint({'x': qx}) - log_qx).mean())
    decay, state = 0.8, None
    for step in range(4):
        with pytest.warns(FutureWarning):
            lbk = zs.variational.elbo(log_joint, observed={}, latent={'x': [qx, log_qx]}, axis=0)
        lbk.reinforce(decay=decay)
        mm, state = OV.zero_debiased_moving_average(state, signal * (1 + 0.0 * step), decay)
        np.testing.assert_allclose(float(lbk._moving_mean), mm, rtol=1e-5)
    own = torch.zeros((), device="cuda")
    lbk.reinforce(decay=decay, moving_mean=own)              # caller-held variable, in place
    np.testing.assert_allclose(float(own), signal, rtol=1e-5)   # first debiased update = the value


def test_effective_sample_size_vs_oracle(zs):
    """zhusuan/diagnostics.py:17-64 on the device vs the NumPy oracle, on the reference test's
    two chains (tests/test_diagnostics.py:14-42) and a many-dimension AR(1) family."""
    from oracle import diagnostics as OG
    from test_oracle_diagnostics import make_chains
    iid, mcmc = make_chains()
    for chain in (iid, mcmc):
        got = N(zs.diagnostics.effective_sample_size_per_dim(T(chain), burn_in=100))
        np.testing.assert_allclose(got, OG.ess_per_dim(chain.astype(np.float32), 100), rtol=2e-3)
    assert zs.diagnostics.effective_sample_size(iid, burn_in=100) >= 2000
    assert zs.diagnostics.effective_sample_size(T(mcmc), burn_in=100) <= 1000
    rng = np.random.RandomState(5)
    M, D = 3000, 70                       # 3 blocks of 32 dimensions, last one ragged
    phi = np.linspace(0.0, 0.95, D)
    x = np.zeros((M, D), np.float32)
    e = rng.standard_normal((M, D)).astype(np.float32)
    for i in range(1, M):
        x[i] = phi * x[i - 1] + e[i]
    got = N(zs.diagnostics.effective_sample_size_per_dim(T(x), burn_in=0))
    np.testing.assert_allclose(got, OG.ess_per_dim(x, 0), rtol=2e-3)
    assert abs(zs.diagnostics.effective_sample_size_1d(T(x[:, 3])) - OG.ess_1d(x[:, 3])) < 1.0


@pytest.mark.parametrize("fused", [False, True])
def test_vae_objectives_match_reference_run(zs, fused):
    """tests/golden/ref_vae.npz: the VAE of examples/variational_autoencoders/iwae.py:23-44 run on
    the REFERENCE'S OWN BayesianNet / Normal / Bernoulli / importance_weighted_objective / elbo /
    .sgvb() / .reinforce() (executed on the NumPy TF stand-in, oracle/tf_shim/make_ref_golden.py).
    The same model written against this package -- generic path (registry kernels + torch linear)
    and the K8 path (wgmma dense layers, Bernoulli epilogue) -- must reproduce the per-datum
    bounds, the costs and the gradient of every weight; the injected eps enters through a
    user-defined Distribution subclass (the plugin contract, bn.stochastic)."""
    import torch.nn.functional as F
    from zhusuan_b200.variational import exclusive_kl as EK
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "ref_vae.npz"))
    names = [str(n) for n in g["names"]]
    K, N, z_dim = g["eps"].shape
    x = T(g["x"]).to(torch.int32)

    def weights():
        # TF kernels are [in, out]; torch linear weights [out, in]
        return {n: (T(g["w_" + n].T.copy()) if n.endswith("_w") else T(g["w_" + n]))
                .requires_grad_(True) for n in names}

    class InjectedNormal(zs.distributions.Normal):
        def __init__(self, *a, **kw):
            self._eps = kw.pop("eps")
            super(InjectedNormal, self).__init__(*a, **kw)

        def _sample(self, n_samples):
            return super(InjectedNormal, self)._sample(n_samples, eps=self._eps)

    if fused:
        lin = lambda h, w, b, relu=False: zs.fused.linear(h, w, b, relu=relu)
    else:
        lin = lambda h, w, b, relu=False: (F.relu(F.linear(h, w, b)) if relu
                                           else F.linear(h, w, b))

    def nets(W, eps, reparameterized=True):
        @zs.meta_bayesian_net(scope="gen", reuse_variables=True)
        def build_gen(n, n_particles):
            bn = zs.BayesianNet()
            z = bn.normal("z", torch.zeros(n, z_dim, device="cuda"), std=1., group_ndims=1,
                          n_samples=n_particles)
            h = lin(z.tensor, W["g0_w"], W["g0_b"], True)
            h = lin(h, W["g1_w"], W["g1_b"], True)
            if fused:
                bn.stochastic("x", zs.fused.LinearBernoulli(h, W["g2_w"], W["g2_b"]))
            else:
                bn.bernoulli("x", F.linear(h, W["g2_w"], W["g2_b"]), group_ndims=1)
            return bn

        def build_q_net(xx, n_particles):
            bn = zs.BayesianNet()
            h = lin(xx.float(), W["q0_w"], W["q0_b"], True)
            h = lin(h, W["q1_w"], W["q1_b"], True)
            bn.stochastic("z", InjectedNormal(lin(h, W["q2_w"], W["q2_b"]),
                                              logstd=lin(h, W["q3_w"], W["q3_b"]), group_ndims=1,
                                              is_reparameterized=reparameterized, eps=T(eps)),
                          n_samples=n_particles)
            return bn
        return build_gen(N, K), build_q_net(x, K)

    def check_grads(cost, W, key, which, rtol, atol, t=None):
        grads = torch.autograd.grad(cost, [W[n] for n in which], allow_unused=True)
        for n, gr in zip(which, grads):
            want = g[key + n] if t is None else g[key + n][t]
            want = want.T if n.endswith("_w") else want
            np.testing.assert_allclose(N_(gr), want, rtol=rtol, atol=atol,
                                       err_msg="%s%s fused=%s" % (key, n, fused))

    N_ = lambda t: t.detach().cpu().numpy()
    tol = 2e-4 if fused else 5e-5
    W = weights()
    model, variational = nets(W, g["eps"])
    lb = zs.variational.iw_objective(model, {'x': x}, variational=variational, axis=0)
    np.testing.assert_allclose(N_(lb.tensor), g["iw_bound"], rtol=1e-5, atol=1e-5)
    cost = torch.mean(lb.sgvb())
    np.testing.assert_allclose(float(cost.detach()), float(g["iw_cost"]), rtol=1e-5)
    check_grads(cost, W, "iw_grad_", names, tol * 5, tol)
    W = weights()
    model, variational = nets(W, g["eps"])
    el = zs.variational.elbo(model, {'x': x}, variational=variational, axis=0)
    np.testing.assert_allclose(N_(el.tensor), g["elbo_bound"], rtol=1e-5, atol=1e-5)
    cost = torch.mean(el.sgvb())
    np.testing.assert_allclose(float(cost.detach()), float(g["elbo_cost"]), rtol=1e-5)
    check_grads(cost, W, "elbo_grad_", names, tol * 5, tol)
    # REINFORCE with the moving-mean baseline over three steps (exclusive_kl.py:161-231)
    EK.reset_moving_mean()
    for t in range(3):
        W = weights()
        model, variational = nets(W, g["rf_eps"][t], reparameterized=False)
        el = zs.variational.elbo(model, {'x': x}, variational=variational, axis=0)
        cost = torch.mean(el.reinforce())
        np.testing.assert_allclose(float(cost.detach()), float(g["rf_cost"][t]), rtol=5e-5)
        np.testing.assert_allclose(float(el._moving_mean), float(g["rf_moving_mean"][t]),
                                   rtol=1e-5)
        check_grads(cost, W, "rf_grad_", names[:8], 2e-3, 2e-4, t)
    EK.reset_moving_mean()
    # VIMCO (monte_carlo.py:166-227) and the inclusive-KL importance estimator
    # (inclusive_kl.py:119-151) on the non-reparameterised q-net
    W = weights()
    model, variational = nets(W, g["eps"], reparameterized=False)
    lb = zs.variational.iw_objective(model, {'x': x}, variational=variational, axis=0)
    cost = torch.mean(lb.vimco())
    np.testing.assert_allclose(float(cost.detach()), float(g["vimco_cost"]), rtol=2e-5)
    check_grads(cost, W, "vimco_grad_", names, 2e-3, 2e-4)
    W = weights()
    model, variational = nets(W, g["eps"], reparameterized=False)
    kl = zs.variational.klpq(model, {'x': x}, variational=variational, axis=0)
    cost = torch.mean(kl.importance())
    np.testing.assert_allclose(float(cost.detach()), float(g["importance_cost"]), rtol=2e-5)
    check_grads(cost, W, "importance_grad_", names[:8], 2e-3, 2e-4)
