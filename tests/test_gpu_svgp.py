"""zs.fused.gp_conditional and RBFKernel on the kernels of csrc/gp.cu, and the sparse variational GP
of examples/gaussian_process/svgp.py on them: the moments and their gradients against float64
across the kernel's shape range, bitwise repeatability, empty shapes, laziness, sampling, the
generic fallback, the example's bound at the Protein training shape, and the C ABI's checks.

Rounding bounds: the kernel and the float64 side get the same float32 Li = chol^-1 and V = fz Li^T,
so only the kernel's rounding is measured.  Each tolerance is 4 eps32 (n + 8) times the sum of
the absolute terms of the quantity (svgp_oracle.moment_terms / grad_terms), n the longest sum.
Kzz_chol is chol(Kzz + 0.1 I), so cond(Kzz + 0.1 I) <= 1 + 10 M and var >= 0.1 / 1.1.

The end-to-end checks (through gp_conditional, the fallback, the example's bound and the reference
replay) also run float32 Cholesky factors and triangular solves in torch, whose error grows with
cond(Kzz) and is not the kernel's; they compare against float64 or the fixture with stated
relative tolerances instead."""
import numpy as np
import pytest
import torch

import svgp_oracle as O

pytestmark = pytest.mark.gpu

EPS = float(np.finfo(np.float32).eps)


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def D(t):
    return t.detach().double()


def _within(got, want, terms, n, what):
    tol = 4.0 * EPS * (n + 8) * D(terms) + 1e-30
    err = (D(got) - D(want)).abs()
    bad = err > tol
    assert not bool(bad.any()), "%s: max err/tol %.3g" % (what, float((err / tol).max()))


def _problem(zs, rng, M, d, B, K, jitter=0.1):
    z = torch.tensor(rng.uniform(-1.5, 1.5, (M, d)), dtype=torch.float32, device="cuda")
    x = torch.tensor(rng.standard_normal((B, d)), dtype=torch.float32, device="cuda")
    fz = torch.tensor(rng.standard_normal((K, M)), dtype=torch.float32, device="cuda")
    kern = zs.fused.RBFKernel(d)
    with torch.no_grad():
        kern.k_raw_scale.copy_(torch.tensor(rng.uniform(-0.5, 1.5, d)))
    s64 = O.softplus(D(kern.k_raw_scale))
    Kzz = O.rbf(D(z), D(z), s64) + jitter * torch.eye(M, dtype=torch.float64, device="cuda")
    L = torch.linalg.cholesky(Kzz).float()
    return z, x, fz, kern, L


def _factors(zs, z, fz, kern, L):
    Li, V = zs.fused._gp_factors(z, fz, kern, L)
    return kern.k_scale, Li, V


MOMENT_CASES = [(1, 1, 1, 1), (100, 9, 65, 20), (255, 13, 64, 100), (256, 64, 200, 1),
                (256, 1, 63, 20), (100, 64, 129, 100), (255, 9, 1, 20), (1, 64, 130, 100),
                (100, 13, 455, 20)]


@pytest.mark.parametrize("M,d,B,K", MOMENT_CASES)
def test_moments_against_float64(zs, M, d, B, K):
    rng = np.random.default_rng(M * 1000 + d * 10 + B)
    z, x, fz, kern, L = _problem(zs, rng, M, d, B, K)
    with torch.no_grad():
        s, Li, V = _factors(zs, z, fz, kern, L)
        mean, std = zs.fused._GPCondMoments.apply(x, z, s, Li, V, False)
    args = [D(t) for t in (x, z, s, Li, V)]
    m64, std64 = O.moments_from_factors(*args)
    mt, vt = O.moment_terms(*args)
    _within(mean, m64, mt, M + d, "mean")
    _within(D(std) ** 2, std64 ** 2, vt, M + d, "var")
    dist = zs.fused.gp_conditional(z, fz, x, False, kern, Kzz_chol=L)
    assert isinstance(dist, zs.fused.GPConditionalNormal)
    assert isinstance(dist, zs.distributions.Normal)
    assert torch.equal(dist.mean, mean) and torch.equal(dist.std, std)


@pytest.mark.parametrize("wired", ["both", "mean", "std"])
@pytest.mark.parametrize("M,d,B,K", [(100, 9, 200, 20), (256, 64, 65, 3), (7, 3, 11, 4),
                                     (129, 1, 64, 33), (100, 9, 20000, 20)])
def test_gradients_against_float64(zs, M, d, B, K, wired):
    rng = np.random.default_rng(7 * M + d + B)
    z, x, fz, kern, L = _problem(zs, rng, M, d, B, K)
    s, Li, V = _factors(zs, z, fz, kern, L)
    ins = [t.detach().clone().requires_grad_(True) for t in (z, s, Li, V)]
    wm = torch.tensor(rng.standard_normal((K, B)), dtype=torch.float32, device="cuda")
    ws = torch.tensor(rng.standard_normal(B), dtype=torch.float32, device="cuda")
    mean, std = zs.fused._GPCondMoments.apply(x, *ins, True)
    if wired == "mean":
        f = (mean * wm).sum()
    elif wired == "std":
        f = (std * ws).sum()
    else:
        f = (mean * wm).sum() + (std * ws).sum()
    got = torch.autograd.grad(f, ins)
    ins64 = [D(t).requires_grad_(True) for t in ins]
    m64, std64 = O.moments_from_factors(D(x), *ins64)
    gm = D(wm) if wired != "std" else None
    gs = D(ws) if wired != "mean" else None
    f64 = (m64 * gm).sum() if gm is not None else 0.0
    f64 = f64 + ((std64 * gs).sum() if gs is not None else 0.0)
    want = torch.autograd.grad(f64, ins64, allow_unused=True)
    want = [torch.zeros_like(t) if w is None else w for t, w in zip(ins64, want)]
    with torch.no_grad():
        A = O.rbf(D(x), ins64[0], ins64[1]) @ torch.tril(ins64[2]).t()
        terms = O.grad_terms(D(x), *[D(t) for t in ins64], A, std64, gm, gs)
    n = M + d + K + B
    for nm, g, w, t in zip(("z", "s", "Li", "V"), got, want, terms):
        if nm == "Li":
            w = torch.tril(w)
        _within(g, w, t, n, "d " + nm)


def test_gradients_through_gp_conditional(zs):
    """The torch side (cholesky_ex, solve_triangular, V = fz Li^T, softplus) carries the kernel's
    gradients to z, k_raw_scale, Kzz_chol and fz: the same as the generic path's, to float32."""
    rng = np.random.default_rng(3)
    z, x, fz, kern, L = _problem(zs, rng, 50, 5, 300, 8)
    wm = torch.tensor(rng.standard_normal((8, 300)), dtype=torch.float32, device="cuda")
    ws = torch.tensor(rng.standard_normal(300), dtype=torch.float32, device="cuda")
    grads = []
    for fused in (True, False):
        leaves = [t.detach().clone().requires_grad_(True) for t in (z, L, fz)]
        kern.k_raw_scale.grad = None
        dist = (zs.fused.gp_conditional if fused else zs.fused._gp_conditional_generic)(
            leaves[0], leaves[2], x, False, kern, leaves[1])
        assert isinstance(dist, zs.fused.GPConditionalNormal) == fused
        f = (dist.mean * wm).sum() + (dist.std * ws).sum()
        grads.append(torch.autograd.grad(f, leaves + [kern.k_raw_scale]))
    for nm, a, b in zip(("z", "Kzz_chol", "fz", "k_raw_scale"), *grads):
        scale = float(D(b).abs().max())
        assert float((D(a) - D(b)).abs().max()) <= 2e-3 * scale, nm


@pytest.mark.parametrize("mode", ["no_grad", "inference_mode"])
def test_no_grad_keeps_nothing(zs, mode):
    rng = np.random.default_rng(5)
    z, x, fz, kern, L = _problem(zs, rng, 30, 4, 100, 5)
    z.requires_grad_(True)
    ctx = torch.no_grad() if mode == "no_grad" else torch.inference_mode()
    with ctx:
        dist = zs.fused.gp_conditional(z, fz, x, False, kern, Kzz_chol=L)
        mean, std = dist.mean, dist.std
    assert mean.grad_fn is None and std.grad_fn is None
    assert not mean.requires_grad


@pytest.mark.parametrize("B", [5000, 20000])
def test_deterministic(zs, B):
    """B = 20000 gives 313 tiles on 132 CTAs: the sweep adds later tiles to each CTA's slice."""
    from zhusuan_b200._lib import lib
    assert (lib.load().zsb_gp_cond_parts(B, 100, 9, 20) < (B + 63) // 64) == (B > 5000)
    rng = np.random.default_rng(9)
    z, x, fz, kern, L = _problem(zs, rng, 100, 9, B, 20)
    outs = []
    for _ in range(2):
        ins = [t.detach().clone().requires_grad_(True) for t in _factors(zs, z, fz, kern, L)]
        zz = z.detach().clone().requires_grad_(True)
        mean, std = zs.fused._GPCondMoments.apply(x, zz, *ins, True)
        g = torch.autograd.grad(mean.sum() + (std * 3).sum(), [zz] + ins)
        outs.append([mean, std] + list(g))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


@pytest.mark.parametrize("mode", ["no_grad", "inference_mode"])
def test_first_read_without_grad_then_with_grad(zs, mode):
    """Moments first read without a gradient are computed again when read with one."""
    rng = np.random.default_rng(6)
    z, x, fz, kern, L = _problem(zs, rng, 30, 4, 100, 5)
    z.requires_grad_(True)
    dist = zs.fused.gp_conditional(z, fz, x, False, kern, Kzz_chol=L)
    with (torch.no_grad() if mode == "no_grad" else torch.inference_mode()):
        first = dist.mean.clone()
    lp = dist.log_prob(dist.mean.detach() + 0.1)
    gz, = torch.autograd.grad(lp.sum(), z)
    assert torch.equal(dist.mean.detach(), first)
    assert bool(gz.abs().sum() > 0)


def test_empty_shapes(zs):
    rng = np.random.default_rng(11)
    z, x, fz, kern, L = _problem(zs, rng, 20, 3, 0, 4)
    zz = z.clone().requires_grad_(True)
    dist = zs.fused.gp_conditional(zz, fz, x, False, kern, Kzz_chol=L)
    assert dist.mean.shape == (4, 0) and dist.std.shape == (0,)
    (dist.mean.sum() + dist.std.sum()).backward()
    assert torch.equal(zz.grad, torch.zeros_like(zz))
    z, x, fz, kern, L = _problem(zs, rng, 20, 3, 70, 0)
    dist = zs.fused.gp_conditional(z, fz, x, False, kern, Kzz_chol=L)
    assert dist.mean.shape == (0, 70)
    s, Li, V = _factors(zs, z, fz, kern, L)
    _, std64 = O.moments_from_factors(*[D(t) for t in (x, z, s, Li, V)])
    _, vt = O.moment_terms(*[D(t) for t in (x, z, s, Li, V)])
    _within(D(dist.std) ** 2, std64 ** 2, vt, 23, "var")


def _cuda_kernels(fn):
    from torch.profiler import profile, ProfilerActivity
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    return out, [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]


def test_construction_launches_nothing(zs):
    from zhusuan_b200._lib import lib
    rng = np.random.default_rng(13)
    z, x, fz, kern, _ = _problem(zs, rng, 40, 3, 100, 6)
    z.requires_grad_(True)
    before = lib.launches
    dist, kernels = _cuda_kernels(lambda: zs.fused.gp_conditional(z, fz, x, False, kern))
    assert lib.launches == before and kernels == []
    assert dist.batch_shape == (6, 100)
    dist.mean
    assert lib.launches == before + 1


def _svgp(zs, params, x, y, n_train, eps_fz, eps_fx, fused=True):
    """svgp.py:49-139 on zs with injected draws: build_model, the variational fz and fx, and elbo
    with fx's log-prob replaced by zeros.  Returns (lower bound object, model-side fx dists)."""
    K, M = eps_fz.shape
    kern = params["kernel"]
    z_pos = params["z_pos"]
    cond = zs.fused.gp_conditional if fused else zs.fused._gp_conditional_generic
    model_fx = []

    @zs.meta_bayesian_net(scope="model", reuse_variables=True)
    def build_model(n_particles):
        bn = zs.BayesianNet()
        Kzz_chol = torch.linalg.cholesky(kern(z_pos, z_pos))
        fz = bn.multivariate_normal_cholesky("fz", torch.zeros(M, device="cuda"), Kzz_chol,
                                             n_samples=n_particles)
        fx = bn.stochastic("fx", cond(z_pos, fz, x, False, kern, Kzz_chol))
        model_fx.append(fx.dist)
        bn.normal("y", mean=fx, std=torch.nn.functional.softplus(params["noise_level"]),
                  group_ndims=1)
        return bn

    raw = params["z_cov_raw"]
    tril = torch.tril(raw, -1) + torch.diag(torch.nn.functional.softplus(torch.diagonal(raw)))
    fz = params["z_mean"] + eps_fz @ tril.t()
    log_qfz = zs.distributions.MultivariateNormalCholesky(params["z_mean"], tril).log_prob(fz)
    qfx = cond(z_pos, fz, x, False, kern)
    fx = qfx.mean + qfx.std * eps_fx
    model = build_model(K)
    B = x.shape[0]

    def log_joint(bn):
        prior, log_py = bn.cond_log_prob(["fz", "y"])
        return prior + log_py / B * n_train

    model.log_joint = log_joint
    lb = zs.variational.elbo(model, {"y": y}, latent={"fz": [fz, log_qfz],
                                                       "fx": [fx, torch.zeros_like(log_qfz)]},
                             axis=0)
    return lb, model_fx


def _svgp_params(zs, rng, M, d):
    kern = zs.fused.RBFKernel(d)
    with torch.no_grad():
        kern.k_raw_scale.copy_(torch.tensor(rng.uniform(-0.5, 1.0, d)))
    T = lambda a: torch.tensor(a, dtype=torch.float32, device="cuda").requires_grad_(True)
    raw = np.eye(M) * 0.5 + np.tril(rng.standard_normal((M, M)) * 0.05, -1)
    return {"kernel": kern, "z_pos": T(rng.uniform(-1, 1, (M, d))),
            "z_mean": T(rng.standard_normal(M) * 0.3), "z_cov_raw": T(raw),
            "noise_level": T(np.float32(-1.0))}


@pytest.mark.parametrize("B,d", [(5000, 9), (455, 13)])
def test_example_bound_and_gradients(zs, B, d):
    """svgp.py's training objective at its Protein (B = 5000, d = 9) and Boston (455, 13) shapes,
    M = 100, K = 20: the bound and every gradient against the float64 oracle.  The model-side fx
    node, observed by the variational sample, computes nothing."""
    M, K = 100, 20
    rng = np.random.default_rng(B + d)
    params = _svgp_params(zs, rng, M, d)
    x = torch.tensor(rng.standard_normal((B, d)), dtype=torch.float32, device="cuda")
    y = torch.tensor(rng.standard_normal(B), dtype=torch.float32, device="cuda")
    eps_fz = torch.tensor(rng.standard_normal((K, M)), dtype=torch.float32, device="cuda")
    eps_fx = torch.tensor(rng.standard_normal((K, B)), dtype=torch.float32, device="cuda")
    names = ["z_pos", "z_mean", "z_cov_raw", "noise_level"]
    leaves = [params[n] for n in names] + [params["kernel"].k_raw_scale]
    lb, model_fx = _svgp(zs, params, x, y, 10 * B, eps_fz, eps_fx)
    cost = lb.sgvb().mean()
    got = torch.autograd.grad(cost, leaves)
    assert all(dist._moments is None for dist in model_fx)
    p64 = {n: D(params[n]).requires_grad_(True) for n in names}
    p64["k_raw_scale"] = D(params["kernel"].k_raw_scale).requires_grad_(True)
    obj = O.svgp_bound(p64, D(x), D(y), 10 * B, D(eps_fz), D(eps_fx))
    want = torch.autograd.grad(-obj.mean(), [p64[n] for n in names + ["k_raw_scale"]])
    ref_bound = float(obj.mean())
    assert abs(float(lb.tensor.mean()) - ref_bound) <= 2e-4 * abs(ref_bound)
    assert abs(float(cost) + ref_bound) <= 2e-4 * abs(ref_bound)
    for nm, g, w in zip(names + ["k_raw_scale"], got, want):
        err = float((D(g) - w).abs().max())
        assert err <= 2e-3 * float(w.abs().max()) + 1e-6, (nm, err, float(w.abs().max()))


def test_sample_is_mean_plus_std_eps(zs):
    rng = np.random.default_rng(17)
    z, x, fz, kern, L = _problem(zs, rng, 60, 5, 300, 7)
    dist = zs.fused.gp_conditional(z, fz, x, False, kern, Kzz_chol=L)
    zs.set_random_seed(1234)
    smp = dist.sample()
    mean, std = dist.mean, dist.std
    zs.set_random_seed(1234)
    eps = zs.distributions.Normal(torch.zeros_like(mean), std=torch.ones_like(mean)).sample()
    want = D(mean) + D(std) * D(eps)
    assert float((D(smp) - want).abs().max()) <= 1e-5 * float(want.abs().max())


class _LinearKernel(object):
    def __call__(self, x, y):
        return x @ y.transpose(-1, -2) + 1.0

    def Kdiag(self, x):
        return (x * x).sum(-1) + 1.0


@pytest.mark.parametrize("case", ["M257", "d65", "full_cov", "float64", "non_rbf", "x_grad"])
def test_fallback_matches_oracle(zs, case):
    M, d, B, K = {"M257": (257, 3), "d65": (20, 65)}.get(case, (30, 4)) + (90, 5)
    rng = np.random.default_rng(23)
    dt = torch.float64 if case == "float64" else torch.float32
    z = torch.tensor(rng.uniform(-1.5, 1.5, (M, d)), dtype=dt, device="cuda")
    x = torch.tensor(rng.standard_normal((B, d)), dtype=dt, device="cuda")
    fz = torch.tensor(rng.standard_normal((K, M)), dtype=dt, device="cuda")
    kern = zs.fused.RBFKernel(d, dtype=dt)
    s64 = O.softplus(D(kern.k_raw_scale))
    Kzz = O.rbf(D(z), D(z), s64) + 0.1 * torch.eye(M, dtype=torch.float64, device="cuda")
    L = torch.linalg.cholesky(Kzz).to(dt)
    if case == "non_rbf":
        kern = _LinearKernel()
        L = torch.linalg.cholesky(D(z) @ D(z).t() + 1.0 + torch.eye(M, device="cuda",
                                                                 dtype=torch.float64)).float()
    if case == "x_grad":
        x.requires_grad_(True)
    dist = zs.fused.gp_conditional(z, fz, x, case == "full_cov", kern, Kzz_chol=L)
    assert not isinstance(dist, zs.fused.GPConditionalNormal)
    if case == "non_rbf":
        Li = torch.linalg.solve_triangular(D(L), torch.eye(M, dtype=torch.float64, device="cuda"),
                                           upper=False)
        Kxz = D(x) @ D(z).t() + 1.0
        m64 = D(fz) @ (Kxz @ Li.t() @ Li).t()
        s64v = torch.sqrt((D(x) ** 2).sum(-1) + 1.0 - ((Kxz @ Li.t()) ** 2).sum(-1))
        tol = 1e-3
        assert float((D(dist.mean) - m64).abs().max()) <= tol * float(m64.abs().max())
        assert float((D(dist.std) - s64v).abs().max()) <= tol * float(s64v.abs().max())
        return
    m64, second = O.gp_conditional(D(z), D(fz), D(x), s64, case == "full_cov", D(L))
    tol = 1e-9 if dt == torch.float64 else 2e-3
    assert float((D(dist.mean) - m64).abs().max()) <= tol * max(1.0, float(m64.abs().max()))
    if case == "full_cov":
        assert isinstance(dist, zs.distributions.MultivariateNormalCholesky)
        assert dist.cov_tril.shape == (K, B, B)
        got = D(dist.cov_tril[0])
        assert float((got - second).abs().max()) <= 2e-2 * float(second.abs().max())
    else:
        assert float((D(dist.std) - second).abs().max()) <= tol * float(second.abs().max())


def test_shape_errors(zs):
    kern = zs.fused.RBFKernel(3)
    z = torch.zeros(5, 3, device="cuda")
    x = torch.zeros(7, 3, device="cuda")
    fz = torch.zeros(2, 5, device="cuda")
    for args in [(z[0], fz, x), (z, fz, x[0]), (z, fz[:, :4], x), (z, fz, x[:, :2])]:
        with pytest.raises(ValueError):
            zs.fused.gp_conditional(args[0], args[1], args[2], False, kern)
    with pytest.raises(ValueError):
        zs.fused.gp_conditional(z, fz, x, False, kern, Kzz_chol=torch.eye(4, device="cuda"))
    with pytest.raises(ValueError):
        zs.fused.gp_conditional(z, fz, x, False, zs.fused.RBFKernel(4))


def test_c_abi_argument_checks(zs):
    from zhusuan_b200._lib import lib, ptr, stream
    dll = lib.load()
    t = torch.zeros(4096, device="cuda")
    p = ptr(t)
    fwd, bwd = dll.zsb_gp_cond_fwd_f32, dll.zsb_gp_cond_bwd_f32
    for B, M, d, K in [(8, 0, 3, 2), (8, 257, 3, 2), (8, 4, 0, 2), (8, 4, 65, 2), (-1, 4, 3, 2),
                       (8, 4, 3, -1)]:
        assert fwd(p, p, p, p, p, p, p, None, B, M, d, K, stream()) == -1
        assert bwd(p, p, p, p, p, p, p, p, p, p, p, p, p, p, B, M, d, K, stream()) == -1
    assert fwd(None, p, p, p, p, p, p, None, 8, 4, 3, 2, stream()) == -1
    assert bwd(p, p, p, p, p, p, p, p, p, None, p, p, p, p, 8, 4, 3, 2, stream()) == -1
    assert fwd(None, None, None, None, None, None, None, None, 0, 4, 3, 2, stream()) == 0
    assert dll.zsb_gp_cond_parts(0, 4, 3, 2) == 0 and dll.zsb_gp_cond_parts(100, 4, 3, 2) == 2


def _replay_predict(zs, params, x, y, std_y, eps_fz, eps_fx, fused):
    """svgp.py:143-150: the model observes the variational fx; log_likelihood and pred_mse."""
    kern = params["kernel"]
    cond = zs.fused.gp_conditional if fused else zs.fused._gp_conditional_generic
    raw = params["z_cov_raw"]
    tril = torch.tril(raw, -1) + torch.diag(torch.nn.functional.softplus(torch.diagonal(raw)))
    fz = params["z_mean"] + eps_fz @ tril.t()
    qfx = cond(params["z_pos"], fz, x, False, kern)
    assert isinstance(qfx, zs.fused.GPConditionalNormal) == fused
    fx = qfx.mean + qfx.std * eps_fx
    noise = torch.nn.functional.softplus(params["noise_level"])
    ll = zs.distributions.Normal(fx, std=noise, group_ndims=1).log_prob(y)
    ll = zs.log_mean_exp(ll, 0) / x.shape[0] - float(np.log(std_y))
    mse = ((fx.mean(0) - y) ** 2).mean() * std_y ** 2
    return ll, mse


@pytest.mark.parametrize("fused", [True, False])
def test_reference_replay(zs, fused):
    """tests/golden/ref_svgp.npz: the reference's svgp.py graph on its own utils.py, replayed with
    the same draws: the bound, the cost, the cost's gradient w.r.t. every variable, and the two
    prediction fetches."""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                             "ref_svgp.npz"))
    T = lambda a: torch.tensor(np.asarray(a), dtype=torch.float32, device="cuda")  # noqa: E731
    kern = zs.fused.RBFKernel(g["x"].shape[1])
    with torch.no_grad():
        kern.k_raw_scale.copy_(T(g["param/k_raw_scale"]))
    names = ["z_pos", "z_mean", "z_cov_raw", "noise_level"]
    params = {n: T(g["param/" + n]).requires_grad_(True) for n in names}
    params["kernel"] = kern
    x, y = T(g["x"]), T(g["y"])
    lb, _ = _svgp(zs, params, x, y, float(g["n_train"]), T(g["train/eps_fz"]),
                  T(g["train/eps_fx"]), fused=fused)
    cost = lb.sgvb().mean()
    leaves = [params[n] for n in names] + [kern.k_raw_scale]
    grads = torch.autograd.grad(cost, leaves)
    rel = lambda a, b: abs(float(a) - float(b)) / max(1.0, abs(float(b)))  # noqa: E731
    assert rel(lb.tensor.mean(), g["train/bound"]) <= 2e-5
    assert rel(cost, g["train/cost"]) <= 2e-5
    for n, gr in zip(names + ["k_raw_scale"], grads):
        want = g["train/grad_" + n]
        err = float(np.abs(gr.detach().cpu().numpy() - want).max())
        assert err <= 1e-3 * max(1.0, float(np.abs(want).max())), (n, err)
    with torch.no_grad():
        ll, mse = _replay_predict(zs, params, x, y, float(g["std_y_train"]),
                                  T(g["pred/eps_fz"]), T(g["pred/eps_fx"]), fused)
    assert rel(ll, g["pred/log_likelihood"]) <= 2e-5
    assert rel(mse, g["pred/pred_mse"]) <= 2e-5
