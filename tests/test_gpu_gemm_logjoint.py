"""GPU parity: K8 dense-layer kernels on wgmma (gemm_logjoint_tc.cu) -- the decoder output layer
of examples/variational_autoencoders/iwae.py:23-32 with the Bernoulli likelihood
(univariate.py:398-403, group_ndims=1) fused into the GEMM epilogue -- against float64 matmul,
the NumPy oracle and the unfused path of this repo."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import distributions as OD

pytestmark = pytest.mark.gpu


def T(a, dtype=torch.float32):
    return torch.tensor(np.asarray(a), dtype=dtype, device="cuda")


def N(t):
    return t.detach().cpu().numpy()


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


@pytest.mark.parametrize("R,K,J,relu", [(300, 40, 500, True), (1000, 500, 784, False),
                                        (256, 64, 128, False), (77, 1, 5, True)])
def test_linear_forward_fp32_accuracy(zs, R, K, J, relu):
    """h W^T + b from the 3-product fp16 split is fp32-accurate: ragged rows, K not a multiple
    of 64 (zero padded), J not a multiple of 128 (TMA zero fill + masked stores)."""
    rng = np.random.RandomState(R + K + J)
    h = np.maximum(rng.standard_normal((R, K)), 0).astype(np.float32) * 3
    W = (rng.standard_normal((J, K)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(J).astype(np.float32)
    y = N(zs.fused.linear(T(h), T(W), T(b), relu=relu))
    want = h.astype(np.float64) @ W.astype(np.float64).T + b
    if relu:
        want = np.maximum(want, 0)
    scale = np.abs(h).astype(np.float64) @ np.abs(W).astype(np.float64).T + np.abs(b)
    assert y.shape == (R, J)
    # error relative to sum_k |h||W|: dropped lo*lo term (2^-22) + fp16 lo rounding (2^-22) +
    # fp32 accumulation -- the level of an fp32 SIMT GEMM (K * 2^-24 worst case), far below TF32
    assert np.max(np.abs(y - want) / scale) < 2e-6


@pytest.mark.parametrize("R,K,J,relu", [(5000, 500, 784, True), (300, 40, 500, False),
                                        (70000, 64, 50, True)])
def test_linear_backward_on_tensor_cores(zs, R, K, J, relu):
    """dh = g W and dW = g^T h (row-major operand planes read MN-major, split-K over the CTA pairs,
    ragged contraction length) and db against float64."""
    rng = np.random.RandomState(R + J)
    h = rng.standard_normal((R, K)).astype(np.float32)
    W = (rng.standard_normal((J, K)) / np.sqrt(K)).astype(np.float32)
    b = (0.1 * rng.standard_normal(J)).astype(np.float32)
    gy = rng.standard_normal((R, J)).astype(np.float32)
    th, tW, tb = (T(v).requires_grad_(True) for v in (h, W, b))
    y = zs.fused.linear(th, tW, tb, relu=relu)
    dh, dW, db = torch.autograd.grad((y * T(gy)).sum(), [th, tW, tb])
    pre = h.astype(np.float64) @ W.astype(np.float64).T + b
    g = gy.astype(np.float64) * ((pre > 0) if relu else 1.0)
    # mask decided in fp32 on the device: drop the (measure-zero) rows where pre ~ 0 disagrees
    for got, want, scale in [(dh, g @ W.astype(np.float64), np.abs(g) @ np.abs(W).astype(np.float64)),
                             (dW, g.T @ h.astype(np.float64),
                              np.abs(g).T @ np.abs(h).astype(np.float64)),
                             (db, g.sum(0), np.abs(g).sum(0))]:
        err = np.abs(N(got) - want) / (scale + 1e-30)
        assert np.quantile(err, 0.999) < 3e-6 and got.shape == want.shape


def test_bias_gradient_alone(zs):
    """Only the bias asks for a gradient: the split pass of the backward still runs, and its column
    sums are db, for the ReLU dense layer and for the Bernoulli likelihood layer."""
    rng = np.random.RandomState(11)
    R, K, J = 300, 40, 64
    h = rng.standard_normal((R, K)).astype(np.float32)
    W = (rng.standard_normal((J, K)) / np.sqrt(K)).astype(np.float32)
    b = (0.1 * rng.standard_normal(J)).astype(np.float32)
    gy = rng.standard_normal((R, J)).astype(np.float32)
    x = (rng.random_sample((R, J)) < 0.3).astype(np.float32)
    w = rng.standard_normal(R).astype(np.float32)
    pre = h.astype(np.float64) @ W.astype(np.float64).T + b
    tb = T(b).requires_grad_(True)
    db, = torch.autograd.grad((zs.fused.linear(T(h), T(W), tb, relu=True) * T(gy)).sum(), [tb])
    g = gy * (pre > 0)
    np.testing.assert_allclose(N(db), g.sum(0), rtol=0, atol=3e-6 * np.abs(g).sum(0).max())
    lp = zs.fused.linear_bernoulli_log_prob(T(h), T(W), tb, T(x))
    db, = torch.autograd.grad((lp * T(w)).sum(), [tb])
    g = w[:, None] * (x - 1 / (1 + np.exp(-pre)))
    np.testing.assert_allclose(N(db), g.sum(0), rtol=0, atol=3e-6 * np.abs(g).sum(0).max())


@pytest.mark.parametrize("R,K,J", [(1000, 500, 784), (63, 1, 5), (4097, 130, 257), (64, 64, 128),
                                   (20000, 40, 500)])
def test_weight_gradient_from_row_major_planes_vs_forward_product(zs, R, K, J):
    """zsb_linear_tc_wgrad_f32: dW = g^T h with both operands read as MN-major wgmma operands
    from the ROW-MAJOR planes (no transposed copy) against float64 and against the K-major forward
    product of zsb_linear_tc_f32 on the planes of explicit transposes; ragged contraction length
    (TMA zero fill of the last 64-row box), odd / tiny widths, feature counts that are not
    multiples of the 64-column box."""
    from zhusuan_b200 import fused
    from zhusuan_b200._lib import lib, ptr, stream
    rng = np.random.RandomState(R + K + J)
    h = rng.standard_normal((R, K)).astype(np.float32) * 2
    g = rng.standard_normal((R, J)).astype(np.float32) * 1e-3
    hp, hs = fused._tc_split(T(h))
    gp, gs = fused._tc_split(T(g))
    slices = lib.load().zsb_linear_tc_slices(J, K, R)
    part = torch.empty(max(slices, 1) * J * K, device="cuda")
    out = torch.full((J, K), float("nan"), device="cuda")
    lib.call("zsb_linear_tc_wgrad_f32", ptr(hp), ptr(hs), K, ptr(gp), ptr(gs), J, R, ptr(out),
             ptr(part) if slices > 1 else None, stream())
    want = g.astype(np.float64).T @ h.astype(np.float64)
    scale = np.abs(g).astype(np.float64).T @ np.abs(h).astype(np.float64)
    assert np.max(np.abs(N(out) - want) / (scale + 1e-30)) < 3e-6
    # the forward product on the planes of g^T [J, R] and h^T [K, R] is dW^T [K, J]
    fwd = fused._tc_linear(0, *fused._tc_split(T(g).t()), *fused._tc_split(T(h).t()), None, None,
                           None, K, J, R)
    np.testing.assert_allclose(N(out), N(fwd).T, rtol=0, atol=3e-6 * float(scale.max()))


@pytest.mark.parametrize("P,Nb,K,J", [(3, 100, 500, 784), (1, 64, 40, 20), (2, 257, 96, 130)])
def test_linear_bernoulli_log_prob_and_grads(zs, P, Nb, K, J):
    """[P particles, Nb data] activations against x [Nb, J]: value vs the oracle on float64
    logits; gradients wrt h, W, b vs float64 autograd of the unfused formula."""
    rng = np.random.RandomState(P * 1000 + Nb + J)
    h = np.maximum(rng.standard_normal((P, Nb, K)), 0).astype(np.float32)
    W = (rng.standard_normal((J, K)) * 2 / np.sqrt(K)).astype(np.float32)
    b = (0.3 * rng.standard_normal(J)).astype(np.float32)
    x = (rng.random_sample((Nb, J)) < 0.3).astype(np.float32)
    th, tW, tb = (T(v).requires_grad_(True) for v in (h, W, b))
    lp = zs.fused.linear_bernoulli_log_prob(th, tW, tb, T(x))
    assert tuple(lp.shape) == (P, Nb)
    logits = h.astype(np.float64) @ W.astype(np.float64).T + b
    want = OD.bernoulli_log_prob(np.broadcast_to(x, logits.shape), logits, group_ndims=1,
                                 dtype=np.float64)
    np.testing.assert_allclose(N(lp), want, rtol=1e-5, atol=1e-4)
    w = rng.standard_normal((P, Nb)).astype(np.float32)
    got = torch.autograd.grad((lp * T(w)).sum(), [th, tW, tb])
    rh, rW, rb = (torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in (h, W, b))
    rl = -F.binary_cross_entropy_with_logits(
        F.linear(rh, rW, rb), torch.tensor(x, dtype=torch.float64).expand(P, Nb, J),
        reduction="none").sum(-1)
    exp = torch.autograd.grad((rl * torch.tensor(w, dtype=torch.float64)).sum(), [rh, rW, rb])
    for g, e in zip(got, exp):
        e = e.numpy()
        assert np.max(np.abs(N(g) - e)) < 2e-4 * max(1.0, np.max(np.abs(e)))


@pytest.mark.parametrize("R,K,J", [(1000, 500, 784), (77, 1, 5), (300, 130, 257), (256, 64, 128),
                                   (5000, 40, 500)])
def test_input_gradient_from_the_forward_weight_planes(zs, R, K, J):
    """zsb_linear_tc_dgrad_f32: dh = g W with operand A = the forward planes of W [J, K] read
    MN-major (contraction over W's rows; no W^T copy) and B = the planes of g, against float64
    and against the K-major product on the planes of W^T; ragged J (TMA zero fill of the last
    64-row box of W), odd / tiny K, K not a multiple of the 64-column box."""
    from zhusuan_b200 import fused
    from zhusuan_b200._lib import lib, ptr, stream
    rng = np.random.RandomState(R + K + J)
    W = (rng.standard_normal((J, K)) / np.sqrt(K)).astype(np.float32)
    g = rng.standard_normal((R, J)).astype(np.float32) * 1e-2
    tW = T(W)
    wp, ws = fused._tc_split(tW)
    gp, gs = fused._tc_split(T(g))
    out = torch.full((R, K), float("nan"), device="cuda")
    amax = torch.zeros(4, device="cuda")
    lib.call("zsb_linear_tc_dgrad_f32", ptr(wp), ptr(ws), ptr(gp), ptr(gs), R, J, K, ptr(out),
             ptr(amax), stream())
    want = g.astype(np.float64) @ W.astype(np.float64)
    scale = np.abs(g).astype(np.float64) @ np.abs(W).astype(np.float64)
    assert np.max(np.abs(N(out) - want) / (scale + 1e-30)) < 3e-6
    got_max = float(amax.view(torch.int32)[2:3].view(torch.float32)[0])
    np.testing.assert_allclose(got_max, np.abs(N(out)).max(), rtol=1e-6)
    wtp, wts = fused._tc_split(tW.t())
    old = fused._tc_linear(0, wtp, wts, gp, gs, None, None, None, R, K, J)
    np.testing.assert_allclose(N(out), N(old), rtol=0, atol=3e-6 * float(scale.max()))


def test_linear_bernoulli_as_distribution_plugin(zs):
    """bn.stochastic('x', LinearBernoulli(h, W, b)) == bn.bernoulli('x', dense(h), group_ndims=1)
    inside an IWAE objective: same bound, same SGVB gradients."""
    rng = np.random.RandomState(7)
    Kp, Nb, Z, H, X = 8, 96, 10, 64, 50
    x = T((rng.random_sample((Nb, X)) < 0.2).astype(np.int32), torch.int32)
    W1 = T(rng.standard_normal((H, Z)) / 3).requires_grad_(True)
    W2 = T(rng.standard_normal((X, H)) / 8).requires_grad_(True)
    b2 = T(0.1 * rng.standard_normal(X)).requires_grad_(True)
    eps = T(rng.standard_normal((Kp, Nb, Z)))
    mu = T(0.3 * rng.standard_normal((Nb, Z))).requires_grad_(True)

    def bound(fused):
        def build(observed):
            bn = zs.BayesianNet(observed=observed)
            z = bn.normal("z", torch.zeros(Nb, Z, device="cuda"), std=1., group_ndims=1,
                          n_samples=Kp)
            hh = F.relu(F.linear(z.tensor, W1))
            if fused:
                bn.stochastic("x", zs.fused.LinearBernoulli(hh, W2, b2))
            else:
                bn.bernoulli("x", F.linear(hh, W2, b2), group_ndims=1)
            return bn
        z = mu + eps                      # q(z | x) = N(mu, 1), reparameterised
        log_q = zs.distributions.Normal(mu, std=1., group_ndims=1).log_prob(z)
        lj = lambda obs: build(obs).log_joint()
        import warnings
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            lb = zs.variational.iw_objective(lj, {"x": x}, latent={"z": [z, log_q]}, axis=0)
        cost = lb.sgvb().mean()
        return cost, torch.autograd.grad(cost, [W1, W2, b2, mu])
    c0, g0 = bound(False)
    c1, g1 = bound(True)
    np.testing.assert_allclose(float(c1), float(c0), rtol=2e-6)
    for a, b in zip(g1, g0):
        np.testing.assert_allclose(N(a), N(b), rtol=2e-4, atol=2e-6)
    d = zs.fused.LinearBernoulli(F.relu(F.linear(mu, W1)), W2, b2)
    s = d.sample(3)
    assert tuple(s.shape) == (3, Nb, X) and s.dtype == torch.int32
