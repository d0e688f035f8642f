"""GPU tests of zs.fused.bn_linear (dense layer + batch norm with a learned scale) and of the
Bernoulli-latent VAE of examples/variational_autoencoders/bernoulli_latent_vae.py trained by
REINFORCE on it, against the float64 restatement of tests/blvae_oracle.py."""
import os

import numpy as np
import pytest
import torch

import blvae_oracle as BO

pytestmark = pytest.mark.gpu


def T(a, dtype=torch.float32):
    return torch.tensor(np.asarray(a), dtype=dtype, device="cuda")


def N64(t):
    return torch.tensor(t.detach().cpu().numpy(), dtype=torch.float64)


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def _layer(rng, J, K, gamma="random"):
    W = T(rng.standard_normal((J, K)) / np.sqrt(K))
    g = rng.standard_normal(J) + 1.0
    if gamma == "special":            # zero and negative entries
        g[::3] = 0.0
        g[1::3] = -np.abs(g[1::3])
    return W, T(g), T(0.3 * rng.standard_normal(J))


def _stats(rng, J):
    return T(0.1 * rng.standard_normal(J)), T(0.5 + rng.random_sample(J))


def _bound(y64, *terms):
    """Allowed |error| of a float32 result: relative 3e-5 of the summed magnitudes involved."""
    s = y64.abs()
    for t in terms:
        s = s + t.abs()
    return 3e-5 * (s + 1.0)


# (lead shape of h, K, J): J and K odd, unaligned and 1; rows around 128; 2-D and 3-D h
SHAPES = [((127,), 1, 1), ((128,), 30, 7), ((129,), 33, 129), ((3, 43), 784, 500),
          ((2, 100), 500, 40), ((1,), 5, 3), ((4, 257), 64, 200)]


@pytest.mark.parametrize("lead,K,J", SHAPES)
@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("relu", [True, False])
def test_forward_against_float64(zs, lead, K, J, training, relu):
    rng = np.random.RandomState(K * 7 + J + len(lead))
    h = T(rng.standard_normal(lead + (K,)))
    W, g, b = _layer(rng, J, K, gamma="special")
    mm, mv = _stats(rng, J)
    mm64, mv64 = N64(mm), N64(mv)
    y = zs.fused.bn_linear(h, W, g, b, mm, mv, training, relu=relu)
    assert y.shape == lead + (J,)
    y64, nm, nv = BO.bn_layer(N64(h), N64(W), N64(g), N64(b), mm64, mv64, training, relu=relu)
    err = (N64(y) - y64).abs()
    assert (err <= _bound(y64, N64(b))).all(), float(err.max())
    if training:
        np.testing.assert_allclose(mm.cpu().numpy(), nm.numpy(), rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(mv.cpu().numpy(), nv.numpy(), rtol=1e-5, atol=1e-6)
    if not training:
        assert torch.equal(mm.cpu(), mm64.float()) and torch.equal(mv.cpu(), mv64.float())


@pytest.mark.parametrize("training", [True, False])
def test_binary_sample_gives_the_bits_of_its_float_values(zs, training):
    """A LinearBernoulli sample (one 0/1 operand plane) and the same values as a float tensor."""
    rng = np.random.RandomState(5)
    x = T(rng.standard_normal((200, 30)))
    Wq, bq = T(rng.standard_normal((40, 30))), T(rng.standard_normal(40))
    z = zs.fused.LinearBernoulli(x, Wq, bq, dtype=torch.float32).sample(3)
    assert z._zsb_pl.binary
    W, g, b = _layer(rng, 500, 40, gamma="special")
    outs = []
    for h in (z, z.detach().clone()):
        mm, mv = _stats(np.random.RandomState(1), 500)
        Wr, gr, br = (t.clone().requires_grad_(True) for t in (W, g, b))
        y = zs.fused.bn_linear(h, Wr, gr, br, mm, mv, training)
        gy = T(np.random.RandomState(2).standard_normal(tuple(y.shape)))
        grads = torch.autograd.grad(y, (Wr, gr, br), gy)
        outs.append((y, mm, mv) + tuple(grads))
    for a, c in zip(*outs):
        assert torch.equal(a, c)


def test_moving_statistics_over_two_training_calls(zs):
    rng = np.random.RandomState(3)
    W, g, b = _layer(rng, 70, 50)
    mm, mv = _stats(rng, 70)
    m64, v64 = N64(mm), N64(mv)
    for step in range(2):
        h = T(rng.standard_normal((2, 300, 50)) + step)
        zs.fused.bn_linear(h, W, g, b, mm, mv, True, momentum=0.9)
        _, m64, v64 = BO.bn_layer(N64(h), N64(W), N64(g), N64(b), m64, v64, True, momentum=0.9)
        np.testing.assert_allclose(mm.cpu().numpy(), m64.numpy(), rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(mv.cpu().numpy(), v64.numpy(), rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("lead,K,J", [((129,), 33, 129), ((3, 43), 784, 500), ((1000,), 1, 1),
                                      ((2, 100), 500, 40)])
@pytest.mark.parametrize("training", [True, False])
@pytest.mark.parametrize("gamma", ["random", "special"])
@pytest.mark.parametrize("relu", [True, False])
def test_gradients_against_float64(zs, lead, K, J, training, gamma, relu):
    rng = np.random.RandomState(K + J + 11)
    h = T(rng.standard_normal(lead + (K,))).requires_grad_(True)
    W, g, b = (t.requires_grad_(True) for t in _layer(rng, J, K, gamma=gamma))
    mm, mv = _stats(rng, J)
    m64, v64 = N64(mm), N64(mv)
    y = zs.fused.bn_linear(h, W, g, b, mm, mv, training, relu=relu)
    gy = T(rng.standard_normal(tuple(y.shape)))
    got = torch.autograd.grad(y, (h, W, g, b), gy)
    p64 = [N64(t).requires_grad_(True) for t in (h, W, g, b)]
    y64, _, _ = BO.bn_layer(*p64[:2], p64[2], p64[3], m64, v64, training, relu=relu)
    # the ReLU mask of the fused output, so that rows at the kink are not compared across it
    if relu:
        y64 = torch.where(N64(y) > 0, y64, torch.zeros_like(y64))
    want = torch.autograd.grad(y64, p64, N64(gy))
    for name, a, e in zip(("h", "W", "gamma", "beta"), got, want):
        a = N64(a)
        tol = 1e-4 * max(1.0, float(e.abs().max()))
        assert (a - e).abs().max() <= tol + 1e-4 * e.abs().max(), (name, float((a - e).abs().max()))


def test_gamma_gradient_at_gamma_zero_in_evaluation(zs):
    """d gamma needs xhat, kept as the pre-activation: not recoverable from y at gamma = 0."""
    rng = np.random.RandomState(8)
    h = T(rng.standard_normal((256, 20)))
    W = T(rng.standard_normal((9, 20)))
    g = torch.zeros(9, device="cuda", requires_grad=True)
    b = T(rng.standard_normal(9)).requires_grad_(True)
    mm, mv = _stats(rng, 9)
    y = zs.fused.bn_linear(h, W, g, b, mm, mv, False, relu=False)
    dg, = torch.autograd.grad(y.sum(), g)
    a64 = N64(h) @ N64(W).t()
    want = ((a64 - N64(mm)) * torch.rsqrt(N64(mv) + 1e-3)).sum(0)
    np.testing.assert_allclose(dg.cpu().numpy(), want.numpy(), rtol=1e-4,
                               atol=1e-4 * float(want.abs().max()))


@pytest.mark.parametrize("training", [True, False])
def test_two_identical_calls_give_identical_bits(zs, training):
    rng = np.random.RandomState(9)
    h0 = T(rng.standard_normal((3, 700, 300)))
    W0, g0, b0 = _layer(rng, 200, 300, gamma="special")
    outs = []
    for _ in range(2):
        h, W, g, b = (t.clone().requires_grad_(True) for t in (h0, W0, g0, b0))
        mm, mv = _stats(np.random.RandomState(4), 200)
        y = zs.fused.bn_linear(h, W, g, b, mm, mv, training)
        grads = torch.autograd.grad((y * y).sum(), (h, W, g, b))
        outs.append((y, mm, mv) + grads)
    for a, c in zip(*outs):
        assert torch.equal(a, c)


def test_inference_mode_and_amax_tag(zs):
    rng = np.random.RandomState(10)
    h = T(rng.standard_normal((300, 64)))
    W, g, b = _layer(rng, 100, 64)
    mm, mv = _stats(rng, 100)
    y0 = zs.fused.bn_linear(h, W, g, b, mm.clone(), mv.clone(), False)
    assert float(y0._zsb_amax[2]) == float(y0.abs().max())
    want = y0.detach()
    with torch.inference_mode():
        y = zs.fused.bn_linear(h, W, g, b, mm, mv, False)
        yt = zs.fused.bn_linear(h, W, g, b, mm, mv, True)
        nxt = zs.fused.linear(yt, T(rng.standard_normal((10, 100))))
    assert torch.equal(y, want)
    assert torch.isfinite(nxt).all()


def test_value_errors(zs):
    dev = "cuda"
    h = torch.zeros(10, 8, device=dev)
    W = torch.zeros(4, 8, device=dev)
    g, b = torch.ones(4, device=dev), torch.zeros(4, device=dev)
    mm, mv = torch.zeros(4, device=dev), torch.ones(4, device=dev)
    bad = [
        (h[:, :7], W, g, b, mm, mv),                                  # K mismatch
        (h.double(), W, g, b, mm, mv),                                # float64 h
        (h, W.double(), g, b, mm, mv),
        (h, W, g[:3], b, mm, mv),
        (h, W, g, b.cpu(), mm, mv),
        (h, W, g, b, mm.double(), mv),
        (h, W, g, b, mm, torch.ones(8, device=dev)[::2]),             # not contiguous
        (h.cpu(), W, g, b, mm, mv),
        (h, W.cpu(), g.cpu(), b.cpu(), mm.cpu(), mv.cpu()),           # not on CUDA
        (torch.zeros(0, 8, device=dev), W, g, b, mm, mv),
        (h, torch.zeros(4, 8, 1, device=dev), g, b, mm, mv),
    ]
    for args in bad:
        with pytest.raises(ValueError):
            zs.fused.bn_linear(*args, training=True)


# ---- the example -------------------------------------------------------------------------------
X_DIM, H_DIM, Z_DIM, C_DIM = 784, 500, 40, 100


def _params(rng):
    def bn(J, K):
        return [T(rng.standard_normal((J, K)) * np.sqrt(2.0 / K)),
                T(1.0 + 0.1 * rng.standard_normal(J)), T(0.1 * rng.standard_normal(J))]

    def dense(J, K):
        return [T(rng.standard_normal((J, K)) / np.sqrt(K)), T(0.1 * rng.standard_normal(J))]
    q = bn(H_DIM, X_DIM) + bn(H_DIM, H_DIM) + dense(Z_DIM, H_DIM)
    p = bn(H_DIM, Z_DIM) + bn(H_DIM, H_DIM) + dense(X_DIM, H_DIM)
    c = dense(C_DIM, X_DIM) + dense(1, C_DIM)
    return [[t.requires_grad_(True) for t in ps] for ps in (q, p, c)]


def _fresh_stats():
    return [[(torch.zeros(H_DIM, device="cuda"), torch.ones(H_DIM, device="cuda"))
             for _ in range(2)] for _ in range(2)]


def fused_blvae(zs, x, q, p, c, stats, training, S, u_z=None):
    """bernoulli_latent_vae.py:18-55 on fused layers: the z sample [S, n, z_dim], its log q, the
    model's log_joint and the baseline cx [1, n].  ``u_z``: injected uniforms of the z draw, else
    the zs.random stream."""
    qs, ps = stats
    xf = x.to(torch.float32)                                    # tf.cast(x, tf.float32)
    q_bn = zs.BayesianNet()
    h = zs.fused.bn_linear(xf, *q[0:3], *qs[0], training)
    h = zs.fused.bn_linear(h, *q[3:6], *qs[1], training)
    if u_z is None:
        z = q_bn.stochastic("z", zs.fused.LinearBernoulli(h, q[6], q[7], dtype=torch.float32),
                            n_samples=S)
        z, log_qz = z.tensor, z.cond_log_p
    else:
        dist = zs.fused.LinearBernoulli(h, q[6], q[7], dtype=torch.float32)
        z = dist.sample(S, u=u_z)
        log_qz = dist.log_prob(z)

    def log_joint(obs):
        bn = zs.BayesianNet(observed=obs)
        zn = bn.bernoulli("z", torch.zeros(x.shape[0], q[6].shape[0], device="cuda"),
                          group_ndims=1, n_samples=S, dtype=torch.float32)
        hh = zs.fused.bn_linear(zn.tensor, *p[0:3], *ps[0], training)
        hh = zs.fused.bn_linear(hh, *p[3:6], *ps[1], training)
        bn.stochastic("x", zs.fused.LinearBernoulli(hh, p[6], p[7]))
        return bn.log_joint()

    cx = zs.fused.linear(zs.fused.linear(xf, c[0], c[1], relu=True), c[2], c[3]).squeeze(-1)
    return z, log_qz, log_joint, cx.unsqueeze(0)


def _oracle(x, z, q, p, c, stats, training):
    q64, p64, c64 = ([N64(t).requires_grad_(True) for t in ps] for ps in (q, p, c))
    st = [[(N64(m), N64(v)) for m, v in s] for s in stats]
    lq_logits, nq = BO.encoder(N64(x), q64, st[0], training)
    log_qz = BO.bern_lp(lq_logits, N64(z))
    log_pxz, np_ = BO.decoder_log_joint(N64(x), N64(z), p64, st[1], training)
    cx = BO.baseline(N64(x), c64).unsqueeze(0)
    return q64, p64, c64, log_qz, log_pxz, cx, (nq, np_)


def _binarize(rng, n):
    xin = T(rng.random_sample((n, X_DIM)) ** 3)            # MNIST-like: mostly near 0
    u = T(rng.random_sample((n, X_DIM)))
    return (u < xin).to(torch.int32)


def test_training_step_at_the_example_shape(zs):
    """128 rows, S = 1, [784, 500, 500], z 40: the REINFORCE cost, bound, every gradient and the
    moving statistics of one step against float64 on the GPU's own sample; then Adam moves every
    parameter."""
    from zhusuan_b200.variational import exclusive_kl
    rng = np.random.RandomState(21)
    n, S = 128, 1
    x = _binarize(rng, n)
    q, p, c = _params(rng)
    stats = _fresh_stats()
    u_z = T(rng.random_sample((S, n, Z_DIM)))
    mmean = torch.full((), -3.0, device="cuda")
    exclusive_kl._SHADOW.pop(mmean, None)
    params = q + p + c
    z, log_qz, log_joint, cx = fused_blvae(zs, x, q, p, c, stats, True, S, u_z)
    assert z._zsb_pl.binary
    lb = zs.variational.elbo(log_joint, {"x": x}, latent={"z": [z, log_qz]}, axis=0)
    cost, baseline_cost = lb.reinforce(baseline=cx, moving_mean=mmean)
    cost = (cost + baseline_cost).mean()
    bound = lb.tensor.mean()
    grads = torch.autograd.grad(cost, params)
    q64, p64, c64, lq, lp, cx64, new_stats = _oracle(x, z, q, p, c, _fresh_stats(), True)
    cost64, bound64, bc64 = BO.reinforce(lp, lq, cx64, -3.0)
    np.testing.assert_allclose(float(cost.detach()), float(cost64), rtol=2e-5)
    np.testing.assert_allclose(float(bound), float(bound64), rtol=2e-5)
    np.testing.assert_allclose(float(mmean), float(bc64), rtol=2e-5)     # first update: bc itself
    want = torch.autograd.grad(cost64, q64 + p64 + c64)
    for i, (a, e) in enumerate(zip(grads, want)):
        a = N64(a)
        tol = 2e-4 * float(e.abs().max()) + 1e-6
        assert (a - e).abs().max() <= tol, (i, float((a - e).abs().max()), tol)
    for side in range(2):
        for k in range(2):
            for a, e in zip(stats[side][k], new_stats[side][k]):
                np.testing.assert_allclose(a.cpu().numpy(), e.numpy(), rtol=1e-5, atol=1e-6)
    opt = torch.optim.Adam(params, lr=1e-3)
    before = [t.detach().clone() for t in params]
    for t, gr in zip(params, grads):
        t.grad = gr
    opt.step()
    for t, b0 in zip(params, before):
        assert torch.isfinite(t).all() and not torch.equal(t.detach(), b0)


def _eval_stats(rng):
    return [[(T(0.2 * rng.standard_normal(H_DIM)), T(0.5 + rng.random_sample(H_DIM)))
             for _ in range(2)] for _ in range(2)]


def test_test_bound_at_400_rows(zs):
    rng = np.random.RandomState(22)
    n = 400
    x = _binarize(rng, n)
    q, p, c = _params(rng)
    stats = _eval_stats(rng)
    kept = [[(m.clone(), v.clone()) for m, v in s] for s in stats]
    u_z = T(rng.random_sample((1, n, Z_DIM)))
    with torch.no_grad():
        z, log_qz, log_joint, _ = fused_blvae(zs, x, q, p, c, stats, False, 1, u_z)
        bound = zs.variational.elbo(log_joint, {"x": x}, latent={"z": [z, log_qz]},
                                    axis=0).tensor.mean()
    for s, k in zip(stats, kept):
        for (m, v), (m0, v0) in zip(s, k):
            assert torch.equal(m, m0) and torch.equal(v, v0)
    *_, lq, lp, _, _ = _oracle(x, z, q, p, c, stats, False)
    np.testing.assert_allclose(float(bound), float((lp - lq).mean()), rtol=2e-5)


def test_is_loglikelihood_at_1000_particles(zs):
    rng = np.random.RandomState(23)
    n, S = 400, 1000
    x = _binarize(rng, n)
    q, p, c = _params(rng)
    stats = _eval_stats(rng)
    with torch.no_grad():
        z, log_qz, log_joint, _ = fused_blvae(zs, x, q, p, c, stats, False, S)
        ll = zs.is_loglikelihood(log_joint, {"x": x}, latent={"z": [z, log_qz]}, axis=0).mean()
    assert z.shape == (S, n, Z_DIM)
    *_, lq, lp, _, _ = _oracle(x, z, q, p, c, stats, False)
    np.testing.assert_allclose(float(ll), float(BO.is_loglikelihood(lp, lq)), rtol=2e-5)


def test_reference_run_replays(zs):
    """tests/golden/ref_blvae.npz, the reference's own graph on the NumPy TF stand-in, replayed on
    the fused layers with its draws: the z samples, the REINFORCE training step (bound, cost,
    REINFORCE's moving mean, every gradient, the moving statistics) and the evaluation bound and
    IS log-likelihood on the updated statistics."""
    from zhusuan_b200.variational import exclusive_kl
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden",
                             "ref_blvae.npz"))
    names = [["W_q0", "gamma_q0", "beta_q0", "W_q1", "gamma_q1", "beta_q1", "W_qz", "b_qz"],
             ["W_p0", "gamma_p0", "beta_p0", "W_p1", "gamma_p1", "beta_p1", "W_px", "b_px"],
             ["W_c0", "b_c0", "W_c1", "b_c1"]]
    q, p, c = ([T(g[k]).requires_grad_(True) for k in ns] for ns in names)
    x = T(g["x"], torch.int32)
    J = int(g["W_q0"].shape[0])
    stats = [[(torch.zeros(J, device="cuda"), torch.ones(J, device="cuda")) for _ in range(2)]
             for _ in range(2)]
    mmean = torch.zeros((), device="cuda")
    exclusive_kl._SHADOW.pop(mmean, None)
    S = int(g["u_z"].shape[0])
    z, log_qz, log_joint, cx = fused_blvae(zs, x, q, p, c, stats, True, S, T(g["u_z"]))
    np.testing.assert_array_equal(z.cpu().numpy(), g["z"])
    lb = zs.variational.elbo(log_joint, {"x": x}, latent={"z": [z, log_qz]}, axis=0)
    cost, baseline_cost = lb.reinforce(baseline=cx, moving_mean=mmean)
    np.testing.assert_allclose(baseline_cost.detach().cpu().numpy(), g["baseline_cost"],
                               rtol=2e-5)
    cost = (cost + baseline_cost).mean()
    np.testing.assert_allclose(float(cost.detach()), g["cost"], rtol=2e-5)
    np.testing.assert_allclose(float(lb.tensor.detach().mean()), g["bound"], rtol=2e-5)
    np.testing.assert_allclose(float(mmean), g["rf_moving_mean"], rtol=2e-5)
    grads = torch.autograd.grad(cost, q + p + c)
    for name, got in zip(sum(names, []), grads):
        want = g["grad_" + name]
        np.testing.assert_allclose(got.cpu().numpy(), want, rtol=1e-3,
                                   atol=1e-4 * max(1.0, np.abs(want).max()), err_msg=name)
    for (m, v), name in zip(stats[0] + stats[1], ("q0", "q1", "p0", "p1")):
        np.testing.assert_allclose(m.cpu().numpy(), g["moving_mean_" + name], rtol=1e-5,
                                   atol=1e-6, err_msg=name)
        np.testing.assert_allclose(v.cpu().numpy(), g["moving_variance_" + name], rtol=1e-5,
                                   atol=1e-6, err_msg=name)
    S_EVAL = int(g["eval_u_z"].shape[0])
    with torch.no_grad():
        z, log_qz, log_joint, _ = fused_blvae(zs, x, q, p, c, stats, False, S_EVAL,
                                              T(g["eval_u_z"]))
        np.testing.assert_array_equal(z.cpu().numpy(), g["eval_z"])
        latent = {"z": [z, log_qz]}
        bound = zs.variational.elbo(log_joint, {"x": x}, latent=latent, axis=0).tensor.mean()
        ll = zs.is_loglikelihood(log_joint, {"x": x}, latent=latent, axis=0).mean()
    np.testing.assert_allclose(float(bound), g["eval_bound"], rtol=2e-5)
    np.testing.assert_allclose(float(ll), g["eval_is_ll"], rtol=2e-5)
