"""The biased convolutions on the tensor-core products -- zs.fused.conv2d_tc and
conv2d_transpose_tc, relu?(conv(x) + b + residual) -- against float64: the forward across kernel
sizes 1 to 7, strides 1 and 2, SAME and VALID, odd and even sizes, 1 to 256 channels, every
combination of bias, residual and ReLU, with and without leading axes; the gradients w.r.t. x, W,
b and residual (up to 1024 images of 28 x 28 x 16); agreement with the FFMA conv2d /
conv2d_transpose inside their range; bitwise repeatability, inference mode, non-contiguous inputs,
zero images, the errors raised before any launch and the max |.| hand-off between layers; and the
convolutional VAE of vae_conv.py on these layers: the reference run of tests/golden/ref_vae_conv.npz
and one training step at nf 16 and nf 64 against the float64 oracle of tests/vae_conv_oracle.py."""
import itertools

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import gan_oracle as GO
import vae_conv_oracle as VC
from test_gpu_vae_conv import Layers, example

pytestmark = pytest.mark.gpu

CHANNELS = [1, 3, 16, 64, 65, 128, 256]
LEADS = [(), (2,), (2, 3)]
FLAGS = list(itertools.product([False, True], repeat=3))     # (bias, residual, relu)


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def T(a):
    return torch.tensor(np.asarray(a), dtype=torch.float32, device="cuda")


def N64(t):
    return t.detach().double()


def conv_t64(x, W, out_hw, s, pad):
    """Float64 tf.nn.conv2d_transpose(x, W, [N, Ho, Wo, Cout], s, pad) on x [N, Hi, Wi, Cin], W [k,
    k, Cout, Cin]: the full transposed convolution, then TF's pads before cropped and rows no tap
    reaches zero-filled (written out independently of gan_oracle's fixed output size)."""
    k = int(W.shape[0])
    Hi, Wi = int(x.shape[1]), int(x.shape[2])
    Ho, Wo = out_hw
    pt, pl = GO.tf_pads(Ho, Hi, k, s, pad)[0], GO.tf_pads(Wo, Wi, k, s, pad)[0]
    y = F.conv_transpose2d(x.permute(0, 3, 1, 2), W.permute(3, 2, 0, 1).contiguous(), stride=s)
    y = F.pad(y, (0, max(pl + Wo - int(y.shape[3]), 0), 0, max(pt + Ho - int(y.shape[2]), 0)))
    return y[:, :, pt:pt + Ho, pl:pl + Wo].permute(0, 2, 3, 1)


def ref(x, W, b, res, relu, s, pad, transpose, out_hw=None):
    """Float64 relu?(conv(x) + b + residual) over any leading shape, and sum |x| |W| (the summed
    magnitudes of the product) of the same shape."""
    lead = tuple(x.shape[:-3])
    x4 = x.double().reshape((-1,) + tuple(x.shape[-3:]))
    W = W.double()
    if transpose:
        y, m = conv_t64(x4, W, out_hw, s, pad), conv_t64(x4.abs(), W.abs(), out_hw, s, pad)
    else:
        y, m = GO.conv2d(x4, W, s, pad), GO.conv2d(x4.abs(), W.abs(), s, pad)
    y, m = y.reshape(lead + tuple(y.shape[1:])), m.reshape(lead + tuple(m.shape[1:]))
    if b is not None:
        y, m = y + b.double(), m + b.double().abs()
    if res is not None:
        y, m = y + res.double(), m + res.double().abs()
    return (torch.relu(y) if relu else y), m


def out_sizes(H, Wd, k, s, pad, transpose):
    """conv2d_tc: tf.layers' output size.  conv2d_transpose_tc: the largest output height and the
    smallest output width TF accepts for the input (odd and even ones among them)."""
    if not transpose:
        return GO.conv_out_size(H, k, s, pad), GO.conv_out_size(Wd, k, s, pad)
    if pad == "SAME":
        return s * H, s * (Wd - 1) + 1
    return s * H + k - 1, s * (Wd - 1) + k


def call(zs, transpose, x, W, b, res, relu, s, pad, out_hw):
    if transpose:
        return zs.fused.conv2d_transpose_tc(x, W, tuple(out_hw) + (int(W.shape[2]),), s, b, relu,
                                            res, padding=pad)
    return zs.fused.conv2d_tc(x, W, b, s, relu, res, padding=pad)


def params(rng, k, cin, cout, transpose):
    shape = (k, k, cout, cin) if transpose else (k, k, cin, cout)
    return T(rng.standard_normal(shape) / np.sqrt(k * k * cin)), T(0.3 * rng.standard_normal(cout))


def _cases():
    """Every (k, stride, padding, H parity); channels rotate over the cases."""
    out = []
    for i, (k, s, pad, H) in enumerate(itertools.product([1, 2, 3, 4, 5, 7], [1, 2],
                                                         ["SAME", "VALID"], [7, 8])):
        out.append((k, s, pad, H, CHANNELS[i % 7], CHANNELS[(3 * i + 2) % 7]))
    return out


CASES = _cases()
IDS = ["k%d-s%d-%s-H%d-%dto%d" % c for c in CASES]


def _bound_ok(y, y64, m64, what):
    err = (N64(y) - y64).abs()
    bound = 3e-5 * (y64.abs() + m64 + 1.0)
    assert (err <= bound).all(), (what, float((err - bound).max()))


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("k,s,pad,H,cin,cout", CASES, ids=IDS)
def test_forward_against_float64(zs, k, s, pad, H, cin, cout, transpose):
    """Every combination of bias, residual and ReLU on each geometry, the leading shape rotating."""
    rng = np.random.RandomState(k * 1000 + s * 100 + H * 10 + cin % 7 + cout % 5 + 3 * transpose)
    W, b = params(rng, k, cin, cout, transpose)
    for fi, (has_b, has_r, relu) in enumerate(FLAGS):
        lead = LEADS[fi % 3]
        if transpose:
            Hi, Wi = max(H // (2 * s), 1), max(H // (2 * s), 1) + 1
        else:
            Hi, Wi = (max(H, k), max(H, k) - 1 if max(H, k) - 1 >= k else max(H, k)) \
                if pad == "VALID" else (H, H - 1)
        x = T(rng.standard_normal(lead + (Hi, Wi, cin)))
        out_hw = out_sizes(Hi, Wi, k, s, pad, transpose)
        res = T(rng.standard_normal(lead + tuple(out_hw) + (cout,))) if has_r else None
        y = call(zs, transpose, x, W, b if has_b else None, res, relu, s, pad, out_hw)
        y64, m64 = ref(x, W, b if has_b else None, res, relu, s, pad, transpose, out_hw)
        assert tuple(y.shape) == tuple(y64.shape), (tuple(y.shape), tuple(y64.shape))
        _bound_ok(y, y64, m64, (has_b, has_r, relu, lead))


def _grad_ok(name, got, want):
    """The gradient tolerance of test_gpu_gan_layers.py."""
    a = N64(got)
    tol = 1e-4 * max(1.0, float(want.abs().max()))
    err = float((a - want).abs().max())
    assert err <= tol + 1e-4 * float(want.abs().max()), (name, err)


def _grad_case(zs, rng, transpose, lead, H, Wd, k, s, pad, cin, cout, relu):
    """Gradients of <y, G> w.r.t. x, W, b and residual against float64 with the fused forward's
    ReLU mask replayed (where fp32 and float64 pre-activations straddle 0 the masks would differ)."""
    out_hw = out_sizes(H, Wd, k, s, pad, transpose)
    W, b = params(rng, k, cin, cout, transpose)
    x = T(rng.standard_normal(lead + (H, Wd, cin))).requires_grad_(True)
    res = T(rng.standard_normal(lead + tuple(out_hw) + (cout,))).requires_grad_(True)
    W.requires_grad_(True)
    b.requires_grad_(True)
    G = T(rng.standard_normal(lead + tuple(out_hw) + (cout,)))
    y = call(zs, transpose, x, W, b, res, relu, s, pad, out_hw)
    got = torch.autograd.grad((y * G).sum(), (x, W, b, res))
    ins = [N64(t).requires_grad_(True) for t in (x, W, b, res)]
    y64, _ = ref(ins[0], ins[1], ins[2], ins[3], False, s, pad, transpose, out_hw)
    if relu:
        y64 = y64 * (y > 0).double()
    want = torch.autograd.grad((y64 * N64(G)).sum(), ins)
    for name, a, w in zip(("x", "W", "b", "residual"), got, want):
        _grad_ok(name, a, w)


GRAD_CASES = [((3,), 7, 7, 3, 1, "SAME", 16, 32), ((2, 2), 9, 8, 5, 2, "SAME", 3, 65),
              ((2,), 8, 9, 4, 2, "VALID", 64, 16), ((), 6, 6, 1, 1, "VALID", 128, 1),
              ((4,), 10, 11, 7, 2, "SAME", 1, 16), ((2,), 14, 14, 2, 1, "VALID", 65, 256),
              ((2,), 7, 7, 3, 2, "SAME", 256, 128)]


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("lead,H,Wd,k,s,pad,cin,cout", GRAD_CASES,
                         ids=["%s-%dx%d-k%d-s%d-%s-%dto%d" % c for c in GRAD_CASES])
def test_gradients_against_float64(zs, lead, H, Wd, k, s, pad, cin, cout, transpose, relu):
    rng = np.random.RandomState(H * 7 + k * 3 + cin + cout % 11 + s * 13 + transpose * 5 + relu)
    if transpose:                                # x is the small grid: keep the output modest
        H, Wd = max(H // s, 1), max(Wd // s, 1)
    _grad_case(zs, rng, transpose, lead, H, Wd, k, s, pad, cin, cout, relu)


@pytest.mark.parametrize("transpose", [False, True])
def test_gradients_at_1024_images(zs, transpose):
    """28 x 28 x 16 over 1024 images: dW and db sum 8e5 terms per entry."""
    rng = np.random.RandomState(1024 + transpose)
    _grad_case(zs, rng, transpose, (1024,), 28, 28, 3, 1, "SAME", 16, 16, True)


@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("cin,cout", [(1, 16), (16, 32), (33, 3), (64, 64)])
def test_agrees_with_the_ffma_layers_in_their_range(zs, cin, cout, stride, transpose):
    """3 x 3 SAME, 1 to 64 channels: the same inputs through conv2d / conv2d_transpose and the
    tensor-core layers agree within fp32 tolerance, forward and every gradient."""
    rng = np.random.RandomState(cin * 100 + cout + stride * 7 + transpose)
    H, Wd = (7, 6) if transpose else (14, 13)
    out_hw = (2 * H - 1, 2 * Wd) if (transpose and stride == 2) else \
        ((H, Wd) if transpose else (-(-H // stride), -(-Wd // stride)))
    W, b = params(rng, 3, cin, cout, transpose)
    x = T(rng.standard_normal((5, H, Wd, cin)))
    res = T(rng.standard_normal((5,) + out_hw + (cout,)))
    G = T(rng.standard_normal((5,) + out_hw + (cout,)))
    outs = []
    for tc in (False, True):
        ins = [t.clone().requires_grad_(True) for t in (x, W, b, res)]
        if transpose:
            fn = zs.fused.conv2d_transpose_tc if tc else zs.fused.conv2d_transpose
            y = fn(ins[0], ins[1], out_hw + (cout,), stride, b=ins[2], relu=True, residual=ins[3])
        else:
            fn = zs.fused.conv2d_tc if tc else zs.fused.conv2d
            y = fn(ins[0], ins[1], ins[2], stride, True, ins[3])
        outs.append([y] + list(torch.autograd.grad((y * G).sum(), ins)))
    for name, a, c in zip(("y", "dx", "dW", "db", "dres"), *outs):
        a, c = a.detach(), c.detach()
        scale = max(1.0, float(c.abs().max()))
        tol = 2e-5 if name == "y" else 1e-4
        assert float((a - c).abs().max()) <= tol * scale, (name, float((a - c).abs().max()))


def _pair(rng, transpose, n=64, cin=64, cout=128, k=5):
    W, b = params(rng, k, cin, cout, transpose)
    if transpose:
        return T(rng.standard_normal((n, 8, 7, cin))), W, b, (16, 13)
    return T(rng.standard_normal((n, 16, 13, cin))), W, b, (8, 7)


@pytest.mark.parametrize("transpose", [False, True])
def test_two_identical_calls_give_identical_bits(zs, transpose):
    rng = np.random.RandomState(2)
    x0, W0, b0, out_hw = _pair(rng, transpose)
    r0 = T(rng.standard_normal((64,) + out_hw + (128,)))
    outs = []
    for _ in range(2):
        x, W, b, r = (t.clone().requires_grad_(True) for t in (x0, W0, b0, r0))
        y = call(zs, transpose, x, W, b, r, True, 2, "SAME", out_hw)
        outs.append([y] + list(torch.autograd.grad((y * y).sum(), (x, W, b, r))))
    for a, c in zip(*outs):
        assert torch.equal(a, c)


@pytest.mark.parametrize("transpose", [False, True])
def test_inference_mode_keeps_nothing(zs, transpose):
    rng = np.random.RandomState(4)
    x, W, b, out_hw = _pair(rng, transpose, n=3, cin=16, cout=32)
    r = T(rng.standard_normal((3,) + out_hw + (32,)))
    x0 = x
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with torch.inference_mode():          # first, on a fresh x: nothing may stay attached to it
        y = call(zs, transpose, x, W, b, r, True, 2, "SAME", out_hw)
    assert y.grad_fn is None and getattr(x, "_zsb_pl", None) is None
    got = y.cpu()
    del y
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == before
    x = x0.clone()
    want = call(zs, transpose, x, W.requires_grad_(True), b, r, True, 2, "SAME", out_hw)
    assert want.grad_fn is not None
    assert torch.equal(got, want.detach().cpu())
    assert float(want._zsb_amax[2]) == float(want.abs().max())


@pytest.mark.parametrize("transpose", [False, True])
def test_non_contiguous_inputs(zs, transpose):
    rng = np.random.RandomState(3)
    x, W, b, out_hw = _pair(rng, transpose, n=3, cin=16, cout=32)
    r = T(rng.standard_normal((3,) + out_hw + (32,)))
    xt = x.permute(0, 2, 1, 3).contiguous().permute(0, 2, 1, 3).requires_grad_(True)
    rt = r.permute(0, 2, 1, 3).contiguous().permute(0, 2, 1, 3).requires_grad_(True)
    Wt = W.permute(1, 0, 2, 3).contiguous().permute(1, 0, 2, 3).requires_grad_(True)
    assert not (xt.is_contiguous() or rt.is_contiguous() or Wt.is_contiguous())
    xc, rc, Wc = (t.clone().requires_grad_(True) for t in (x, r, W))
    ya = call(zs, transpose, xt, Wt, b, rt, True, 2, "SAME", out_hw)
    yb = call(zs, transpose, xc, Wc, b, rc, True, 2, "SAME", out_hw)
    assert torch.equal(ya, yb)
    gy = T(rng.standard_normal(tuple(ya.shape)))
    for a, c in zip(torch.autograd.grad(ya, (xt, Wt, rt), gy),
                    torch.autograd.grad(yb, (xc, Wc, rc), gy)):
        assert torch.equal(a, c)


def test_zero_images_launch_nothing(zs):
    from zhusuan_b200._lib import lib
    W, b = params(np.random.RandomState(0), 5, 4, 6, False)
    Wt, bt = params(np.random.RandomState(0), 5, 4, 6, True)
    n = lib.launches
    for lead in [(0,), (2, 0)]:
        x = T(np.zeros(lead + (7, 7, 4))).requires_grad_(True)
        y = zs.fused.conv2d_tc(x, W, b, 2, True, T(np.zeros(lead + (4, 4, 6))))
        assert tuple(y.shape) == lead + (4, 4, 6)
        y = zs.fused.conv2d_tc(x, W, padding="VALID")
        assert tuple(y.shape) == lead + (3, 3, 6)
        yt = zs.fused.conv2d_transpose_tc(T(np.zeros(lead + (7, 7, 4))), Wt, (13, 14, 6), 2, bt,
                                          True, T(np.zeros(lead + (13, 14, 6))))
        assert tuple(yt.shape) == lead + (13, 14, 6)
    assert lib.launches == n


def test_errors_raise_before_any_launch(zs):
    from zhusuan_b200._lib import lib
    x = T(np.zeros((2, 7, 7, 4)))
    W = T(np.zeros((5, 5, 4, 6)))
    Wt = T(np.zeros((5, 5, 6, 4)))
    b6 = T(np.zeros(6))
    bad_conv = [
        dict(x=x.double(), W=W), dict(x=x.cpu(), W=W), dict(x=x[0, 0], W=W),
        dict(x=x, W=W.double()), dict(x=x, W=T(np.zeros((5, 4, 4, 6)))),
        dict(x=x, W=T(np.zeros((8, 8, 4, 6)))), dict(x=x, W=T(np.zeros((3, 3, 5, 6)))),
        dict(x=x, W=T(np.zeros((3, 3, 4, 0)))), dict(x=x, W=W, stride=3),
        dict(x=x, W=W, stride=0), dict(x=x, W=W, stride=True), dict(x=x, W=W, padding="FULL"),
        dict(x=x, W=W, padding=None), dict(x=x, W=W, b=T(np.zeros(5))),
        dict(x=x, W=W, b=b6.double()), dict(x=x, W=W, b=b6.cpu()), dict(x=x, W=W, b=[0.0] * 6),
        dict(x=x, W=W, residual=T(np.zeros((2, 7, 7, 4)))),
        dict(x=x, W=W, stride=2, residual=T(np.zeros((2, 4, 4, 6))).double()),
        dict(x=x, W=W, stride=2, residual=T(np.zeros((8, 4, 6)))),
        dict(x=T(np.zeros((2, 0, 7, 4))), W=W), dict(x=T(np.zeros((2, 4, 4, 4))), W=W,
                                                     padding="VALID"),
    ]
    bad_transpose = [
        dict(x=x, W=Wt, out_shape=(15, 14, 6), stride=2),      # ceil(15 / 2) != 7
        dict(x=x, W=Wt, out_shape=(12, 14, 6), stride=2),
        dict(x=x, W=Wt, out_shape=(7, 8, 6)), dict(x=x, W=Wt, out_shape=(7, 7, 5)),
        dict(x=x, W=Wt, out_shape=(7, 7)), dict(x=x, W=Wt, out_shape=None),
        dict(x=x, W=Wt, out_shape=(10, 11, 6), padding="VALID"),   # Ho - k + 1 = 6 != 7
        dict(x=x, W=Wt, out_shape=(20, 19, 6), stride=2, padding="VALID"),
        dict(x=x, W=W, out_shape=(7, 7, 6)), dict(x=x, W=Wt, out_shape=(7, 7, 6), b=T(np.zeros(4))),
        dict(x=x, W=Wt, out_shape=(14, 14, 6), stride=2, residual=T(np.zeros((2, 7, 7, 6)))),
        dict(x=x.cpu(), W=Wt, out_shape=(7, 7, 6)), dict(x=x, W=Wt, out_shape=(7, 7, 6), stride=3),
    ]
    # index overflow: 2^31 entries in the im2col operand, shaped without allocating it
    big = torch.zeros(1, device="cuda").expand(4096, 64, 64, 64)
    bad_conv.append(dict(x=big, W=T(np.zeros((5, 5, 64, 6)))))
    bad_transpose.append(dict(x=big, W=T(np.zeros((5, 5, 6, 64))), out_shape=(128, 128, 6),
                              stride=2))
    n = lib.launches
    for kw in bad_conv:
        with pytest.raises(ValueError):
            zs.fused.conv2d_tc(**kw)
    for kw in bad_transpose:
        with pytest.raises(ValueError):
            zs.fused.conv2d_transpose_tc(**kw)
    # VALID sizes TF accepts are accepted: Ho - k + 1 in [s (Hi - 1) + 1, s Hi]
    assert lib.launches == n
    for Ho in (17, 18):
        y = zs.fused.conv2d_transpose_tc(x, Wt, (Ho, Ho, 6), 2, padding="VALID")
        assert tuple(y.shape) == (2, Ho, Ho, 6)
    torch.cuda.synchronize()


@pytest.mark.parametrize("first,second", [("conv", "conv"), ("conv", "deconv"),
                                          ("deconv", "conv"), ("deconv", "linear")])
def test_a_tagged_output_gives_the_bits_of_the_untagged_tensor(zs, first, second):
    """The max |.| tag a layer leaves is what the next fused layer's split would find: feeding the
    tagged output or an untagged copy gives the same bits, forward and backward."""
    rng = np.random.RandomState(9)
    x = T(rng.standard_normal((4, 9, 10, 16)))
    W1, b1 = params(rng, 3, 16, 32, first == "deconv")
    W2, b2 = params(rng, 4, 32, 24, second == "deconv")
    Wl = T(rng.standard_normal((10, 32)) / 6)

    def layer(kind, h, W, b):
        if kind == "conv":
            return zs.fused.conv2d_tc(h, W, b, 1, True)
        if kind == "deconv":
            Ho, Wo = 2 * int(h.shape[1]), 2 * int(h.shape[2])
            return zs.fused.conv2d_transpose_tc(h, W, (Ho, Wo, int(W.shape[2])), 2, b, True)
        return zs.fused.linear(h, Wl, None)                 # over the channel axis

    outs = []
    for tagged in (True, False):
        Wa = W1.clone().requires_grad_(True)
        y = layer(first, x, Wa, b1)
        assert getattr(y, "_zsb_amax", None) is not None
        h = y if tagged else y.clone()
        z = layer(second, h, W2, b2)
        assert getattr(h, "_zsb_amax", None) is None      # the split consumed the tag
        outs.append((z, torch.autograd.grad((z * z).sum(), Wa)[0]))
    for a, c in zip(*outs):
        assert torch.equal(a, c)


# ---- vae_conv.py on the tensor-core layers ---------------------------------------------------

class TCLayers(Layers):
    """Layers of test_gpu_vae_conv.py with conv / deconv routed to conv2d_tc /
    conv2d_transpose_tc; the dense layers stay zs.fused.linear."""

    def conv(self, h, W, b, stride=1, relu=False, residual=None):
        return self._keep(self.zs.fused.conv2d_tc(h, W, b, stride, relu, residual), relu)

    def deconv(self, h, W, out_shape, stride=1, b=None, relu=False, residual=None):
        return self._keep(self.zs.fused.conv2d_transpose_tc(h, W, out_shape, stride, b, relu,
                                                            residual), relu)


def _close(got, want, what, rtol, atol):
    want = want.detach().double().cpu().numpy() if isinstance(want, torch.Tensor) else want
    np.testing.assert_allclose(got.detach().double().cpu().numpy(), want, rtol=rtol,
                               atol=atol * max(1.0, float(np.abs(want).max(initial=0.0))),
                               err_msg=what)


def test_reference_run_replays(zs):
    """tests/golden/ref_vae_conv.npz replayed on the tensor-core layers at the tolerances of
    test_gpu_vae_conv.py::test_reference_run_replays."""
    from test_ref_vae_conv_pins import golden, golden_grad_checks
    g, mk, q, p = golden()
    q = [T(a).requires_grad_(True) for a in q]
    p = [T(a).requires_grad_(True) for a in p]
    lb, _ = example(TCLayers(zs), T(g["x"]), T(g["eps"]), q, p, mk.NF)
    cost = lb.sgvb().mean()
    _close(lb.tensor.mean(), g["bound"].astype(np.float64), "bound", 2e-5, 2e-6)
    _close(cost, g["cost"].astype(np.float64), "cost", 2e-5, 2e-6)
    grads = [t.detach().double().cpu().numpy() for t in torch.autograd.grad(cost, q + p)]
    golden_grad_checks(g, mk, grads, lambda a, w, what: _close(
        torch.as_tensor(a), np.asarray(w, np.float64), what, 2e-3, 2e-4))


@pytest.mark.parametrize("nf", [16, 64])
def test_training_step_and_test_bound_match_the_oracle(zs, nf):
    """vae_conv.py with 128 images, z_dim 32, 1 particle and Adam(1e-4, beta1 0.5): one training
    step and the test bound over 400 images against float64.  nf 16 is the example's shape; nf 64
    has the 64- and 128-channel layers the FFMA convolutions reject.  Each of its outputs sums four
    times as many products (3 x 3 x 128 against 3 x 3 x 32) through the same depth, and its fp32
    rounding of the bound is larger with them: 1.3e-5 relative on an H100, so the bound and cost
    get 3e-5 there; the gradients keep one tolerance."""
    z_dim = 32
    rtol = 1e-5 if nf == 16 else 3e-5
    rng = np.random.default_rng(2027 + nf)
    qa, pa = VC.init_params(rng, nf, z_dim)
    q = [T(a).requires_grad_(True) for a in qa]
    p = [T(a).requires_grad_(True) for a in pa]
    params_ = q + p
    before = [N64(t) for t in params_]
    x = T(rng.random((128, 784)) < 0.3)
    eps = T(rng.standard_normal((1, 128, z_dim)))
    L = TCLayers(zs)
    lb, _ = example(L, x, eps, q, p, nf)
    bound = lb.tensor.mean()
    cost = lb.sgvb().mean()
    opt = torch.optim.Adam(params_, lr=1e-4, betas=(0.5, 0.999))
    opt.zero_grad()
    cost.backward()
    grads = [t.grad.detach().clone() for t in params_]
    opt.step()
    p64 = [t.clone().requires_grad_(True) for t in before]
    lw, _ = VC.vae_conv(N64(x), N64(eps), p64[:len(q)], p64[len(q):], nf, L.replay())
    bound64, cost64 = VC.bound_and_cost(lw)
    _close(bound, bound64, "bound", rtol, 1e-6)
    _close(cost, cost64, "cost", rtol, 1e-6)
    for i, (a, w) in enumerate(zip(grads, torch.autograd.grad(cost64, p64))):
        _close(a, w, "grad %d" % i, 2e-3, 1e-3)
    assert all(torch.isfinite(t).all() for t in params_)
    x = T(rng.random((400, 784)) < 0.3)
    eps = T(rng.standard_normal((1, 400, z_dim)))
    with torch.no_grad():
        lb, _ = example(TCLayers(zs), x, eps, q, p, nf)
        got = lb.tensor.mean()
        P = [N64(t) for t in params_]
        lw, _ = VC.vae_conv(N64(x), N64(eps), P[:len(q)], P[len(q):], nf)
    _close(got, VC.bound_and_cost(lw)[0], "test bound", rtol, 1e-6)
