"""The 3x3 SAME convolutions (zs.fused.conv2d, zs.fused.conv2d_transpose) and the convolutional
VAE of examples/variational_autoencoders/vae_conv.py on them: the forward of both against float64
across channels, image sizes, strides, bias / residual / ReLU and leading shapes, gradients
against float64 autograd (up to 1024 images of 28 x 28 x 16), bitwise repeatability, inference
mode, non-contiguous inputs, the errors raised before any launch, the reference run of
tests/golden/ref_vae_conv.npz replayed on the fused layers, and the example's training step and
test bound at its own shape against the float64 oracle of tests/vae_conv_oracle.py."""
import itertools
import math

import numpy as np
import pytest
import torch

import vae_conv_oracle as VC

pytestmark = pytest.mark.gpu

CHANNELS = [1, 3, 16, 32, 33, 64]
SIZES = [(1, 1), (2, 2), (5, 9), (7, 7), (14, 14), (28, 28)]
LEADS = [(), (3,), (2, 5)]


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def T(a, dtype=torch.float32):
    return torch.as_tensor(np.asarray(a), dtype=dtype, device="cuda")


def D(t):
    return t.detach().double()


def _close(got, want, what, rtol=1e-5, atol=1e-5):
    want = want.detach().double().cpu().numpy() if isinstance(want, torch.Tensor) else want
    np.testing.assert_allclose(got.detach().double().cpu().numpy(), want, rtol=rtol,
                               atol=atol * max(1.0, float(np.abs(want).max(initial=0.0))),
                               err_msg=what)


def _ref(x, W, b, res, relu, stride, transpose, out_hw):
    """Float64 oracle over any leading shape (differentiable in its inputs)."""
    lead = tuple(x.shape[:-3])
    x4 = x.double().reshape((-1,) + tuple(x.shape[-3:]))
    if transpose:
        y = VC.conv2d_transpose(x4, W.double(), tuple(out_hw) + (int(W.shape[2]),), stride)
    else:
        y = VC.conv2d(x4, W.double(), stride=stride)
    y = y.reshape(lead + tuple(y.shape[1:]))
    if b is not None:
        y = y + b.double()
    if res is not None:
        y = y + res.double()
    return torch.relu(y) if relu else y


def _out_sizes(H, Wd, stride, transpose):
    """Output sizes to test: conv2d has one; a stride-2 transpose has both valid ones."""
    if not transpose:
        return [(-(-H // stride), -(-Wd // stride))]
    if stride == 1:
        return [(H, Wd)]
    return [(2 * H, 2 * Wd), (2 * H - 1, 2 * Wd - 1)]


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("Cout", CHANNELS)
@pytest.mark.parametrize("Cin", CHANNELS)
def test_forward_matches_float64(zs, Cin, Cout, stride, transpose):
    rng = np.random.default_rng(Cin * 1000 + Cout * 10 + stride + 5 * transpose)
    flags = list(itertools.product([False, True], repeat=3))
    for si, (H, Wd) in enumerate(SIZES):
        for oi, (Ho, Wo) in enumerate(_out_sizes(H, Wd, stride, transpose)):
            if Ho < 1 or Wo < 1:
                continue
            for fi, (has_b, has_r, relu) in enumerate(flags):
                lead = LEADS[(si + oi + fi) % len(LEADS)]
                x = T(rng.standard_normal(lead + (H, Wd, Cin)))
                b = T(rng.standard_normal(Cout)) if has_b else None
                if transpose:
                    W = T(rng.standard_normal((3, 3, Cout, Cin)) / math.sqrt(9 * Cin))
                    res = T(rng.standard_normal(lead + (Ho, Wo, Cout))) if has_r else None
                    y = zs.fused.conv2d_transpose(x, W, (Ho, Wo, Cout), stride, b=b, relu=relu,
                                                  residual=res)
                    out_hw = (Ho, Wo)
                else:
                    W = T(rng.standard_normal((3, 3, Cin, Cout)) / math.sqrt(9 * Cin))
                    res = T(rng.standard_normal(lead + (Ho, Wo, Cout))) if has_r else None
                    y = zs.fused.conv2d(x, W, b, stride, relu, res)
                    out_hw = (Ho, Wo)
                want = _ref(x, W, b, res, relu, stride, transpose, out_hw)
                assert tuple(y.shape) == tuple(want.shape)
                _close(y, want, "%s H %d W %d -> %dx%d b %d r %d relu %d lead %s" % (
                    "transpose" if transpose else "conv", H, Wd, Ho, Wo, has_b, has_r, relu,
                    lead))


def test_worked_4x4_example(zs):
    """1..16 row-major, all-ones weights, stride 2: SAME gives [[54, 45], [72, 54]]."""
    x = T(np.arange(1, 17).reshape(1, 4, 4, 1))
    y = zs.fused.conv2d(x, T(np.ones((3, 3, 1, 1))), stride=2)
    np.testing.assert_array_equal(y[0, :, :, 0].cpu().numpy(), [[54, 45], [72, 54]])


def test_empty_batch_launches_nothing(zs):
    from zhusuan_b200._lib import lib
    W = T(np.ones((3, 3, 4, 5)))
    n = lib.launches
    for lead in [(0,), (2, 0)]:
        x = T(np.zeros(lead + (7, 7, 4))).requires_grad_(True)
        y = zs.fused.conv2d(x, W, stride=2)
        assert tuple(y.shape) == lead + (4, 4, 5)
        yt = zs.fused.conv2d_transpose(T(np.zeros(lead + (7, 7, 5))), W, (13, 13, 4), 2)
        assert tuple(yt.shape) == lead + (13, 13, 4)
    assert lib.launches == n


def _grad_case(zs, rng, lead, H, Wd, Cin, Cout, stride, transpose, relu, Ho=None):
    """Gradients of <y, G> w.r.t. x, W, b and residual, fused and float64."""
    if transpose:
        Ho = Ho or stride * H
        Wo = stride * Wd
        out = (Ho, Wo)
        Wt = rng.standard_normal((3, 3, Cout, Cin)) / math.sqrt(9 * Cin)
    else:
        out = (-(-H // stride), -(-Wd // stride))
        Wt = rng.standard_normal((3, 3, Cin, Cout)) / math.sqrt(9 * Cin)
    x = T(rng.standard_normal(lead + (H, Wd, Cin))).requires_grad_(True)
    W = T(Wt).requires_grad_(True)
    b = T(rng.standard_normal(Cout)).requires_grad_(True)
    res = T(rng.standard_normal(lead + out + (Cout,))).requires_grad_(True)
    G = T(rng.standard_normal(lead + out + (Cout,)))
    if transpose:
        y = zs.fused.conv2d_transpose(x, W, out + (Cout,), stride, b=b, relu=relu, residual=res)
    else:
        y = zs.fused.conv2d(x, W, b, stride, relu, res)
    got = torch.autograd.grad((y * G).sum(), (x, W, b, res))
    ins = [D(t).requires_grad_(True) for t in (x, W, b, res)]
    # float64 with the fused output's ReLU mask: where fp32 and float64 pre-activations straddle
    # 0 (a few in 1e5 at 1024 images) the masks would differ, and with them the gradients
    want_y = _ref(ins[0], ins[1], ins[2], ins[3], False, stride, transpose, out)
    if relu:
        want_y = want_y * (y > 0).double()
    want = torch.autograd.grad((want_y * D(G)).sum(), ins)
    for name, a, w in zip(("x", "W", "b", "residual"), got, want):
        _close(a, w, "d%s (%s, stride %d, relu %d, lead %s, %dx%d, %d->%d)" % (
            name, "transpose" if transpose else "conv", stride, relu, lead, H, Wd, Cin, Cout),
            rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("lead,H,Wd,Cin,Cout", [((3,), 7, 7, 16, 32), ((2, 5), 14, 14, 32, 16),
                                                ((2,), 5, 9, 3, 33), ((4,), 28, 28, 1, 16),
                                                ((), 2, 2, 64, 64), ((5,), 1, 1, 33, 3)])
def test_gradients_match_float64(zs, lead, H, Wd, Cin, Cout, stride, transpose, relu):
    rng = np.random.default_rng(H * 7 + Cin * 3 + Cout + stride * 11 + transpose * 5 + relu)
    _grad_case(zs, rng, lead, H, Wd, Cin, Cout, stride, transpose, relu)
    if transpose and stride == 2:
        _grad_case(zs, rng, lead, H, Wd, Cin, Cout, stride, transpose, relu, Ho=2 * H - 1)


@pytest.mark.parametrize("transpose", [False, True])
def test_gradients_at_1024_images(zs, transpose):
    """28 x 28 x 16 over 1024 images: dW sums 8e5 terms per entry."""
    rng = np.random.default_rng(1024 + transpose)
    _grad_case(zs, rng, (1024,), 28, 28, 16, 16, 1, transpose, True)


@pytest.mark.parametrize("transpose", [False, True])
def test_bias_gradient_without_a_weight_gradient(zs, transpose):
    """W needs no gradient: only the bias sums run, and db (and dx) still match float64."""
    rng = np.random.default_rng(11 + transpose)
    x = T(rng.standard_normal((6, 14, 14, 16))).requires_grad_(True)
    W = T(rng.standard_normal((3, 3, 16, 32)) / 12)
    b = T(rng.standard_normal(32 if not transpose else 16)).requires_grad_(True)
    if transpose:
        x = T(rng.standard_normal((6, 7, 7, 32))).requires_grad_(True)
        y = zs.fused.conv2d_transpose(x, W, (14, 14, 16), 2, b=b, relu=True)
    else:
        y = zs.fused.conv2d(x, W, b, 2, True)
    G = T(rng.standard_normal(tuple(y.shape)))
    gx, gb = torch.autograd.grad((y * G).sum(), (x, b))
    xd, bd = D(x).requires_grad_(True), D(b).requires_grad_(True)
    want_y = _ref(xd, W, bd, None, False, 2, transpose, (14, 14)) * (y > 0).double()
    wx, wb = torch.autograd.grad((want_y * D(G)).sum(), (xd, bd))
    _close(gx, wx, "dx", 1e-4, 1e-4)
    _close(gb, wb, "db", 1e-4, 1e-4)


def test_two_identical_calls_are_bitwise_equal(zs):
    rng = np.random.default_rng(7)
    x = T(rng.standard_normal((256, 28, 28, 16))).requires_grad_(True)
    W = T(rng.standard_normal((3, 3, 16, 32)) / 12).requires_grad_(True)
    Wt = T(rng.standard_normal((3, 3, 16, 32)) / 12).requires_grad_(True)
    b = T(rng.standard_normal(32)).requires_grad_(True)
    bt = T(rng.standard_normal(16)).requires_grad_(True)

    def run():
        y = zs.fused.conv2d(x, W, b, 2, True)
        z = zs.fused.conv2d_transpose(y, Wt, (28, 28, 16), 2, b=bt, relu=True, residual=x)
        gs = torch.autograd.grad((z * z).sum(), (x, W, b, Wt, bt))
        return [y.detach().clone(), z.detach().clone()] + [g.clone() for g in gs]

    a, c = run(), run()
    for u, v in zip(a, c):
        assert torch.equal(u, v)


def test_inference_mode_and_non_contiguous_inputs(zs):
    rng = np.random.default_rng(3)
    base = T(rng.standard_normal((2, 9, 7, 3)))
    x = base.transpose(1, 2)                          # [2, 7, 9, 3], non-contiguous
    assert not x.is_contiguous()
    W = T(rng.standard_normal((3, 3, 3, 8))).requires_grad_(True)
    Wt = T(rng.standard_normal((3, 3, 3, 8)))
    with torch.inference_mode():
        y = zs.fused.conv2d(x, W, stride=2, relu=True)
        z = zs.fused.conv2d_transpose(y, Wt, (7, 9, 3), 2)
    assert not y.requires_grad and y.grad_fn is None
    _close(y, _ref(x, W, None, None, True, 2, False, None), "conv2d under inference_mode")
    _close(z, _ref(y, Wt, None, None, False, 2, True, (7, 9)), "transpose under inference_mode")
    xg = base.clone().requires_grad_(True)
    y = zs.fused.conv2d(xg.transpose(1, 2), W, stride=1)
    (gx,) = torch.autograd.grad(y.sum(), (xg,))
    xr = D(base).requires_grad_(True)
    (wx,) = torch.autograd.grad(_ref(xr.transpose(1, 2), W, None, None, False, 1, False,
                                     None).sum(), (xr,))
    _close(gx, wx, "gradient through a non-contiguous x", rtol=1e-4, atol=1e-4)


def test_errors_raise_before_any_launch(zs):
    from zhusuan_b200._lib import lib
    x = T(np.zeros((2, 7, 7, 4)))
    W = T(np.zeros((3, 3, 4, 5)))
    Wt = T(np.zeros((3, 3, 5, 4)))
    bad_conv = [
        dict(x=x.double(), W=W),
        dict(x=x.cpu(), W=W),
        dict(x=x[0, 0], W=W),
        dict(x=x, W=T(np.zeros((5, 5, 4, 5)))),
        dict(x=x, W=T(np.zeros((3, 3, 3, 5)))),
        dict(x=x, W=W, stride=3),
        dict(x=x, W=W, stride=0),
        dict(x=x, W=W, b=T(np.zeros(4))),
        dict(x=x, W=W, residual=T(np.zeros((2, 7, 7, 4)))),
        dict(x=x, W=W, stride=2, residual=T(np.zeros((2, 7, 7, 5)))),
        dict(x=T(np.zeros((2, 7, 7, 65))), W=T(np.zeros((3, 3, 65, 5)))),
        dict(x=x, W=T(np.zeros((3, 3, 4, 65)))),
        dict(x=T(np.zeros((2, 0, 7, 4))), W=W),
    ]
    bad_transpose = [
        dict(x=x, W=Wt, out_shape=(15, 15, 5), stride=2),
        dict(x=x, W=Wt, out_shape=(12, 12, 5), stride=2),
        dict(x=x, W=Wt, out_shape=(8, 7, 5), stride=1),
        dict(x=x, W=Wt, out_shape=(7, 7, 4), stride=1),
        dict(x=x, W=Wt, out_shape=(7, 7), stride=1),
        dict(x=x, W=W, out_shape=(7, 7, 5), stride=1),
        dict(x=x, W=Wt, out_shape=(14, 14, 5), stride=2, b=T(np.zeros(4))),
        dict(x=x, W=Wt, out_shape=(14, 14, 5), stride=2, residual=T(np.zeros((2, 7, 7, 5)))),
    ]
    n = lib.launches
    for kw in bad_conv:
        with pytest.raises(ValueError):
            zs.fused.conv2d(**kw)
    for kw in bad_transpose:
        with pytest.raises(ValueError):
            zs.fused.conv2d_transpose(**kw)
    assert lib.launches == n
    torch.cuda.synchronize()


# ---- vae_conv.py on zs ---------------------------------------------------------------------------

class Layers(object):
    """zs.fused.conv2d / conv2d_transpose / linear that keep, in order, the ReLU masks (y > 0) of
    the layers with ReLU, for the float64 oracle to replay."""

    def __init__(self, zs):
        self.zs, self.masks = zs, []

    def _keep(self, y, relu):
        if relu:
            self.masks.append((y > 0).detach())
        return y

    def conv(self, h, W, b, stride=1, relu=False, residual=None):
        return self._keep(self.zs.fused.conv2d(h, W, b, stride, relu, residual), relu)

    def deconv(self, h, W, out_shape, stride=1, b=None, relu=False, residual=None):
        return self._keep(self.zs.fused.conv2d_transpose(h, W, out_shape, stride, b, relu,
                                                         residual), relu)

    def linear(self, h, W, b, relu=False):
        return self._keep(self.zs.fused.linear(h, W, b, relu=relu), relu)

    def replay(self):
        """A relu for the oracle that applies the kept masks in order."""
        masks = list(self.masks)
        return lambda t: t * masks.pop(0).reshape(t.shape).double()


def conv_resnet_block(L, h, ps, resize):
    """vae_conv.py:39-53: one launch per convolution, the residual add and ReLU fused."""
    if not resize:
        t = L.conv(h, ps[0], ps[1], relu=True)
        return L.conv(t, ps[2], ps[3], relu=True, residual=h)
    t = L.conv(h, ps[0], ps[1], stride=2, relu=True)
    r = L.conv(h, ps[4], ps[5], stride=2)
    return L.conv(t, ps[2], ps[3], relu=True, residual=r)


def deconv_resnet_block(L, h, ps, out_shape, resize):
    """vae_conv.py:20-36 with conv2d_transpose of examples/utils/utils.py:74-113."""
    if not resize:
        t = L.deconv(h, ps[0], out_shape, b=ps[1], relu=True)
        return L.deconv(t, ps[2], out_shape, b=ps[3], relu=True, residual=h)
    t = L.deconv(h, ps[0], tuple(h.shape[1:]), b=ps[1], relu=True)
    r = L.deconv(h, ps[4], out_shape, 2, b=ps[5])
    return L.deconv(t, ps[2], out_shape, 2, b=ps[3], relu=True, residual=r)


def example(L, x, eps, q, p, nf):
    """vae_conv.py:56-114 on zs: build_q_net, build_gen and elbo with latent={'z': [qz, log_qz]}
    (the q-net's draw injected).  Returns the elbo object and the model."""
    zs = L.zs
    S, n, z_dim = (int(v) for v in eps.shape)

    @zs.meta_bayesian_net(scope="gen", reuse_variables=True)
    def build_gen(n, z_dim, n_particles):
        bn = zs.BayesianNet()
        z = bn.normal("z", torch.zeros(n, z_dim, device="cuda"), std=1., group_ndims=1,
                      n_samples=n_particles)
        h = L.linear(z, p[0], p[1], relu=True).reshape(-1, 7, 7, 2 * nf)
        i = 2
        for out, resize in VC.dec_blocks(nf):
            k = 6 if resize else 4
            h = deconv_resnet_block(L, h, p[i:i + k], out, resize)
            i += k
        h = L.deconv(h, p[i], (28, 28, 1), b=p[i + 1])
        x_logits = h.reshape(n_particles, -1, 784)
        bn.deterministic("x_mean", torch.sigmoid(x_logits))
        bn.bernoulli("x", x_logits, group_ndims=1, dtype=torch.float32)
        return bn

    h = (2 * x - 1).reshape(-1, 28, 28, 1)
    h = L.conv(h, q[0], q[1], relu=True)
    i = 2
    for co, resize in VC.enc_blocks(nf):
        k = 6 if resize else 4
        h = conv_resnet_block(L, h, q[i:i + k], resize)
        i += k
    h = L.linear(h.reshape(h.shape[0], -1), q[i], q[i + 1], relu=True)
    mean, logstd = zs.fused.linear(h, q[i + 2], q[i + 3]), zs.fused.linear(h, q[i + 4], q[i + 5])
    qz = mean + torch.exp(logstd) * eps
    log_qz = zs.distributions.Normal(mean, logstd=logstd, group_ndims=1).log_prob(qz)
    model = build_gen(n, z_dim, S)
    lb = zs.variational.elbo(model, {"x": x}, latent={"z": [qz, log_qz]}, axis=0)
    return lb, model


def test_reference_run_replays(zs):
    """tests/golden/ref_vae_conv.npz: the reference's own elbo().sgvb() on vae_conv.py's graph at
    nf 2, z_dim 4, 3 images, replayed on the fused layers."""
    from test_ref_vae_conv_pins import golden, golden_grad_checks
    g, mk, q, p = golden()
    q = [T(a).requires_grad_(True) for a in q]
    p = [T(a).requires_grad_(True) for a in p]
    lb, _ = example(Layers(zs), T(g["x"]), T(g["eps"]), q, p, mk.NF)
    cost = lb.sgvb().mean()
    _close(lb.tensor.mean(), g["bound"].astype(np.float64), "bound", 2e-5, 2e-6)
    _close(cost, g["cost"].astype(np.float64), "cost", 2e-5, 2e-6)
    grads = [t.detach().double().cpu().numpy() for t in torch.autograd.grad(cost, q + p)]
    golden_grad_checks(g, mk, grads, lambda a, w, what: _close(
        torch.as_tensor(a), np.asarray(w, np.float64), what, 2e-3, 2e-4))


def _params(rng, nf, z_dim):
    q, p = VC.init_params(rng, nf, z_dim)
    return ([T(a).requires_grad_(True) for a in q], [T(a).requires_grad_(True) for a in p])


def test_training_step_and_test_bound_at_the_example_shape_match_the_oracle(zs):
    """vae_conv.py at its own shape: one training step (128 images, nf 16, z_dim 32, 1 particle,
    Adam(1e-4, beta1 0.5)) and the test bound over 400 images, against float64."""
    nf, z_dim = 16, 32
    rng = np.random.default_rng(2027)
    q, p = _params(rng, nf, z_dim)
    params = q + p
    before = [D(t) for t in params]
    x = T(rng.random((128, 784)) < 0.3)
    eps = T(rng.standard_normal((1, 128, z_dim)))
    L = Layers(zs)
    lb, _ = example(L, x, eps, q, p, nf)
    bound = lb.tensor.mean()
    cost = lb.sgvb().mean()
    opt = torch.optim.Adam(params, lr=1e-4, betas=(0.5, 0.999))
    opt.zero_grad()
    cost.backward()
    grads = [t.grad.detach().clone() for t in params]
    opt.step()
    p64 = [t.clone().requires_grad_(True) for t in before]
    # float64 with the fused forward's ReLU masks, so that units whose fp32 and float64
    # pre-activations straddle 0 do not make the gradients differ
    lw, _ = VC.vae_conv(D(x), D(eps), p64[:len(q)], p64[len(q):], nf, L.replay())
    bound64, cost64 = VC.bound_and_cost(lw)
    _close(bound, bound64, "bound", 1e-5, 1e-6)
    _close(cost, cost64, "cost", 1e-5, 1e-6)
    for i, (a, w) in enumerate(zip(grads, torch.autograd.grad(cost64, p64))):
        _close(a, w, "grad %d" % i, 2e-3, 1e-3)
    assert all(torch.isfinite(t).all() for t in params)
    # the test bound over 400 images on the updated parameters
    x = T(rng.random((400, 784)) < 0.3)
    eps = T(rng.standard_normal((1, 400, z_dim)))
    with torch.no_grad():
        lb, model = example(Layers(zs), x, eps, q, p, nf)
        got = lb.tensor.mean()
        P = [D(t) for t in params]
        lw, x_mean = VC.vae_conv(D(x), D(eps), P[:len(q)], P[len(q):], nf)
    _close(got, VC.bound_and_cost(lw)[0], "test bound", 1e-5, 1e-6)
