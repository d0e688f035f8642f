"""GPU tests of the GAN layers on the tensor-core products -- zs.fused.bn_conv2d,
bn_conv2d_transpose and sigmoid_conv2d_transpose -- against the float64 oracle of
tests/gan_oracle.py: forward, every gradient and the moving statistics across kernel sizes 1, 3,
4 and 5, strides 1 and 2, SAME and VALID, odd and even sizes, 1 to 512 channels, training and
evaluation, gamma given and None, ReLU on and off; then gamma=None against ones bit for bit,
bitwise repeatability, non-contiguous inputs, inference mode, one-pixel batch norm and the
errors raised before any launch."""
import itertools

import numpy as np
import pytest
import torch

import gan_oracle as GO

pytestmark = pytest.mark.gpu

CHANNELS = [1, 3, 16, 64, 128, 512]


def _cases():
    """Every (k, stride, padding, H parity); channels and flags rotate over the cases so that each
    value of each appears with several geometries."""
    out = []
    geoms = list(itertools.product([1, 3, 4, 5], [1, 2], ["SAME", "VALID"], [7, 8]))
    for i, (k, s, pad, H) in enumerate(geoms):
        cin, cout = CHANNELS[i % 6], CHANNELS[(5 * i + 2) % 6]
        # the three flags run through all 8 combinations on a rotation independent of the
        # geometry's index bits: (3 i + i // 8) % 8 takes every value once per 8 geometries and
        # shifts between the blocks, so each flag value meets each padding, stride and parity
        f = (3 * i + i // 8) % 8
        out.append((k, s, pad, H, cin, cout, bool(f & 1), bool(f & 2), bool(f & 4)))
    return out


CASES = _cases()
IDS = ["k%d-s%d-%s-H%d-%dto%d-%s-%s-%s" % (k, s, p, H, ci, co, "train" if t else "eval",
                                          "gamma" if g else "nogamma", "relu" if r else "lin")
       for k, s, p, H, ci, co, t, g, r in CASES]


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def T(a):
    return torch.tensor(np.asarray(a), dtype=torch.float32, device="cuda")


def N64(t):
    return torch.tensor(t.detach().cpu().numpy(), dtype=torch.float64)


def _bound(y64, *terms):
    """Allowed |error| of a float32 result: relative 3e-5 of the summed magnitudes involved."""
    s = y64.abs()
    for t in terms:
        s = s + t.abs()
    return 3e-5 * (s + 1.0)


def _grad_ok(name, got, want):
    a = N64(got)
    tol = 1e-4 * max(1.0, float(want.abs().max()))
    err = float((a - want).abs().max())
    assert err <= tol + 1e-4 * float(want.abs().max()), (name, err)


def _params(rng, k, cin, cout, transpose, gamma):
    shape = (k, k, cout, cin) if transpose else (k, k, cin, cout)
    W = T(rng.standard_normal(shape) / np.sqrt(k * k * cin))
    g = None
    if gamma:
        gv = rng.standard_normal(cout) + 1.0
        gv[::5] = 0.0
        g = T(gv)
    b = T(0.3 * rng.standard_normal(cout))
    mm, mv = T(0.1 * rng.standard_normal(cout)), T(0.5 + rng.random_sample(cout))
    return W, g, b, mm, mv


def _input(rng, k, s, pad, H, cin, transpose):
    if transpose:
        h = max(H // (2 * s), 1)
        return T(rng.standard_normal((2, h, h + 1, cin)))
    if pad == "VALID":
        H = max(H, k)
    return T(rng.standard_normal((2, H, H - 1 if H - 1 >= k else H, cin)))


def _run_bn(zs, fn, ofn, transpose, k, s, pad, H, cin, cout, training, gamma, relu):
    rng = np.random.RandomState(k * 1000 + s * 100 + H * 10 + cin % 7 + cout % 5)
    x = _input(rng, k, s, pad, H, cin, transpose).requires_grad_(True)
    W, g, b, mm, mv = _params(rng, k, cin, cout, transpose, gamma)
    W.requires_grad_(True)
    b.requires_grad_(True)
    if g is not None:
        g.requires_grad_(True)
    m64, v64 = N64(mm), N64(mv)
    y = fn(x, W, g, b, mm, mv, training, stride=s, padding=pad, relu=relu)
    p64 = [N64(t).requires_grad_(True) for t in (x, W, b)]
    g64 = N64(g).requires_grad_(True) if g is not None else None
    y64, nm, nv = ofn(p64[0], p64[1], g64, p64[2], m64, v64, training, s, pad, relu)
    assert tuple(y.shape) == tuple(y64.shape)
    # the summed magnitudes of the product, sum |x| |W|, carried through the normalisation
    conv = GO.conv2d_transpose if transpose else GO.conv2d
    with torch.no_grad():
        a64 = conv(p64[0], p64[1], s, pad)
        var = a64.var((0, 1, 2), unbiased=False) if training else v64
        gabs = g64.abs() if g64 is not None else 1.0
        term = conv(p64[0].abs(), p64[1].abs(), s, pad) * gabs / torch.sqrt(var + 1e-3)
    err = (N64(y) - y64.detach()).abs()
    assert (err <= _bound(y64.detach(), p64[2].detach(), term)).all(), float(err.max())
    if training:
        np.testing.assert_allclose(mm.cpu().numpy(), nm.detach().numpy(), rtol=1e-5, atol=1e-6)
        np.testing.assert_allclose(mv.cpu().numpy(), nv.detach().numpy(), rtol=1e-5, atol=1e-6)
    else:
        assert torch.equal(mm.cpu(), m64.float()) and torch.equal(mv.cpu(), v64.float())
    gy = T(rng.standard_normal(tuple(y.shape)))
    ins = [x, W, b] + ([g] if g is not None else [])
    got = torch.autograd.grad(y, ins, gy)
    if relu:        # the fused ReLU mask, so that entries at the kink are not compared across it
        y64 = torch.where(N64(y) > 0, y64, torch.zeros_like(y64))
    want = torch.autograd.grad(y64, p64 + ([g64] if g64 is not None else []), N64(gy))
    for name, a, e in zip(("x", "W", "beta", "gamma"), got, want):
        _grad_ok(name, a, e)


@pytest.mark.parametrize("k,s,pad,H,cin,cout,training,gamma,relu", CASES, ids=IDS)
def test_bn_conv2d_against_float64(zs, k, s, pad, H, cin, cout, training, gamma, relu):
    _run_bn(zs, zs.fused.bn_conv2d, GO.bn_conv2d, False, k, s, pad, H, cin, cout, training, gamma,
            relu)


@pytest.mark.parametrize("k,s,pad,H,cin,cout,training,gamma,relu", CASES, ids=IDS)
def test_bn_conv2d_transpose_against_float64(zs, k, s, pad, H, cin, cout, training, gamma, relu):
    _run_bn(zs, zs.fused.bn_conv2d_transpose, GO.bn_conv2d_transpose, True, k, s, pad, H, cin,
            cout, training, gamma, relu)


@pytest.mark.parametrize("k,s,pad,H,cin,cout,training,gamma,relu", CASES, ids=IDS)
def test_sigmoid_conv2d_transpose_against_float64(zs, k, s, pad, H, cin, cout, training, gamma,
                                                  relu):
    rng = np.random.RandomState(k * 999 + s * 99 + H + cin)
    x = _input(rng, k, s, pad, H, cin, True).requires_grad_(True)
    W, _, b, _, _ = _params(rng, k, cin, cout, True, False)
    W.requires_grad_(True)
    b = b.requires_grad_(True) if relu != training else None    # bias given / None, on its own
    y = zs.fused.sigmoid_conv2d_transpose(x, W, b, stride=s, padding=pad)
    p64 = [N64(t).requires_grad_(True) for t in (x, W)]
    b64 = N64(b).requires_grad_(True) if b is not None else None
    y64 = GO.sigmoid_conv2d_transpose(p64[0], p64[1], b64, s, pad)
    assert tuple(y.shape) == tuple(y64.shape)
    err = (N64(y) - y64.detach()).abs()
    assert (err <= _bound(y64.detach())).all(), float(err.max())
    gy = T(rng.standard_normal(tuple(y.shape)))
    ins = [x, W] + ([b] if b is not None else [])
    got = torch.autograd.grad(y, ins, gy)
    want = torch.autograd.grad(y64, p64 + ([b64] if b64 is not None else []), N64(gy))
    for name, a, e in zip(("x", "W", "b"), got, want):
        _grad_ok(name, a, e)


LAYERS = ["bn_conv2d", "bn_conv2d_transpose"]


def _bn_args(rng, name, k=5, cin=16, cout=32):
    transpose = name == "bn_conv2d_transpose"
    x = T(rng.standard_normal((3, 6, 8, cin) if transpose else (3, 13, 16, cin)))
    return (x,) + _params(rng, k, cin, cout, transpose, True)


@pytest.mark.parametrize("name", LAYERS)
@pytest.mark.parametrize("training", [True, False])
def test_gamma_none_gives_the_bits_of_ones(zs, name, training):
    rng = np.random.RandomState(1)
    x, W, _, b, mm0, mv0 = _bn_args(rng, name)
    outs = []
    for gamma in (None, torch.ones_like(b)):
        xx, WW, bb = (t.clone().requires_grad_(True) for t in (x, W, b))
        mm, mv = mm0.clone(), mv0.clone()
        y = getattr(zs.fused, name)(xx, WW, gamma, bb, mm, mv, training, stride=2)
        grads = torch.autograd.grad((y * y).sum(), (xx, WW, bb))
        outs.append((y, mm, mv) + grads)
    for a, c in zip(*outs):
        assert torch.equal(a, c)


@pytest.mark.parametrize("name", LAYERS + ["sigmoid_conv2d_transpose"])
@pytest.mark.parametrize("training", [True, False])
def test_two_identical_calls_give_identical_bits(zs, name, training):
    rng = np.random.RandomState(2)
    if name == "sigmoid_conv2d_transpose":
        x0 = T(rng.standard_normal((64, 16, 16, 64)))
        W0, b0 = T(0.05 * rng.standard_normal((5, 5, 3, 64))), T(rng.standard_normal(3))
    else:
        x0, W0, g0, b0, mm0, mv0 = _bn_args(rng, name, cin=64, cout=128)
        x0 = x0.repeat(20, 1, 1, 1)
    outs = []
    for _ in range(2):
        if name == "sigmoid_conv2d_transpose":
            x, W, b = (t.clone().requires_grad_(True) for t in (x0, W0, b0))
            y = zs.fused.sigmoid_conv2d_transpose(x, W, b, stride=2)
            grads = torch.autograd.grad((y * y).sum(), (x, W, b))
            outs.append((y,) + grads)
        else:
            x, W, g, b = (t.clone().requires_grad_(True) for t in (x0, W0, g0, b0))
            mm, mv = mm0.clone(), mv0.clone()
            y = getattr(zs.fused, name)(x, W, g, b, mm, mv, training, stride=2)
            grads = torch.autograd.grad((y * y).sum(), (x, W, g, b))
            outs.append((y, mm, mv) + grads)
    for a, c in zip(*outs):
        assert torch.equal(a, c)


@pytest.mark.parametrize("name", LAYERS)
def test_non_contiguous_x(zs, name):
    rng = np.random.RandomState(3)
    x, W, g, b, mm, mv = _bn_args(rng, name)
    xt = x.permute(0, 2, 1, 3).contiguous().permute(0, 2, 1, 3).requires_grad_(True)
    assert not xt.is_contiguous()
    xc = x.clone().requires_grad_(True)
    fn = getattr(zs.fused, name)
    ya = fn(xt, W, g, b, mm.clone(), mv.clone(), True, stride=2)
    yb = fn(xc, W, g, b, mm.clone(), mv.clone(), True, stride=2)
    assert torch.equal(ya, yb)
    gy = T(rng.standard_normal(tuple(ya.shape)))
    assert torch.equal(torch.autograd.grad(ya, xt, gy)[0], torch.autograd.grad(yb, xc, gy)[0])


@pytest.mark.parametrize("name", LAYERS + ["sigmoid_conv2d_transpose"])
def test_inference_mode_keeps_nothing(zs, name):
    rng = np.random.RandomState(4)
    x, W, g, b, mm, mv = _bn_args(rng, name)
    if name == "sigmoid_conv2d_transpose":
        W = T(rng.standard_normal((5, 5, 3, 16)))
        b = T(rng.standard_normal(3))
        call = lambda: zs.fused.sigmoid_conv2d_transpose(x, W, b, stride=2)      # noqa: E731
    else:
        call = lambda: getattr(zs.fused, name)(x, W, g, b, mm, mv, False, stride=2)  # noqa: E731
    x0 = x
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated()
    with torch.inference_mode():          # first, on a fresh x: nothing may stay attached to it
        y = call()
    assert y.grad_fn is None and getattr(x, "_zsb_pl", None) is None
    got = y.cpu()
    del y
    torch.cuda.synchronize()
    assert torch.cuda.memory_allocated() == before
    x = x0.clone()
    want = call()
    assert torch.equal(got, want.cpu())
    assert float(want._zsb_amax[2]) == float(want.abs().max())


@pytest.mark.parametrize("name", LAYERS)
def test_one_pixel_batch_norm(zs, name):
    """R = 1: the population variance is 0, so the output is act(beta); the moving variance moves
    towards 0 (Bessel factor 1) and the moving mean towards the one value."""
    rng = np.random.RandomState(5)
    cin, cout = 8, 6
    transpose = name == "bn_conv2d_transpose"
    x = T(rng.standard_normal((1, 1, 1, cin)))
    W, g, b, mm, mv = _params(rng, 1 if transpose else 3, cin, cout, transpose, True)
    m64, v64 = N64(mm), N64(mv)
    y = getattr(zs.fused, name)(x, W, g, b, mm, mv, True, relu=False, momentum=0.9)
    assert tuple(y.shape) == (1, 1, 1, cout)
    assert torch.equal(y.reshape(-1), b)
    ofn = GO.bn_conv2d_transpose if transpose else GO.bn_conv2d
    _, nm, nv = ofn(N64(x), N64(W), N64(g), N64(b), m64, v64, True, relu=False, momentum=0.9)
    np.testing.assert_allclose(mm.cpu().numpy(), nm.numpy(), rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(mv.cpu().numpy(), nv.numpy(), rtol=1e-6)
    np.testing.assert_allclose(mv.cpu().numpy(), 0.9 * v64.numpy(), rtol=1e-6)


def test_errors_raise_before_any_launch(zs):
    from zhusuan_b200._lib import lib
    x = T(np.zeros((2, 7, 7, 4)))
    W = T(np.zeros((5, 5, 4, 6)))
    Wt = T(np.zeros((5, 5, 6, 4)))
    c6 = T(np.zeros(6))
    st = (T(np.zeros(6)), T(np.ones(6)))

    def conv(**kw):
        a = dict(x=x, W=W, gamma=c6, beta=c6, moving_mean=st[0], moving_variance=st[1],
                 training=True)
        a.update(kw)
        return a

    bad_bn = [
        conv(x=x.double()), conv(x=x.cpu()), conv(x=x[0, 0]), conv(W=W.double()),
        conv(W=T(np.zeros((5, 4, 4, 6)))), conv(W=T(np.zeros((8, 8, 4, 6)))),
        conv(W=T(np.zeros((3, 3, 5, 6)))), conv(stride=3), conv(stride=0), conv(stride=True),
        conv(padding="same-ish"), conv(padding=None), conv(gamma=T(np.zeros(5))),
        conv(beta=None), conv(beta=T(np.zeros(7))), conv(moving_mean=T(np.zeros(5))),
        conv(moving_variance=T(np.zeros((6, 2)))[:, 0]), conv(moving_mean=st[0].double()),
        conv(x=T(np.zeros((2, 0, 7, 4)))), conv(x=T(np.zeros((0, 7, 7, 4)))),
        conv(x=T(np.zeros((2, 7, 7, 3)))),
    ]
    # index overflow: 2^31 entries in the im2col operand, shaped without allocating it
    big = torch.zeros(1, device="cuda").expand(4096, 64, 64, 64)
    bad_bn.append(conv(x=big, W=T(np.zeros((5, 5, 64, 6)))))
    n0 = lib.launches
    with pytest.raises(ValueError, match="2\\^31"):   # fails only on size: channels match
        zs.fused.bn_conv2d_transpose(**conv(x=big, W=T(np.zeros((5, 5, 6, 64))), stride=2))
    with pytest.raises(ValueError, match="2\\^31"):
        zs.fused.sigmoid_conv2d_transpose(big, T(np.zeros((5, 5, 3, 64))), stride=2)
    # 2^20 output or input channels, shaped without allocating them
    wide = torch.zeros(1, device="cuda").expand(1, 1, 2 ** 20, 4)
    with pytest.raises(ValueError, match="2\\^20"):
        zs.fused.sigmoid_conv2d_transpose(x, wide)
    with pytest.raises(ValueError, match="2\\^20"):       # x [1, 1, 4, 2^20], W [1, 1, 4, 2^20]
        zs.fused.sigmoid_conv2d_transpose(wide.permute(0, 1, 3, 2), wide.permute(0, 1, 3, 2))
    assert lib.launches == n0
    n = lib.launches
    with pytest.raises(ValueError):       # a VALID input smaller than the kernel
        zs.fused.bn_conv2d(**conv(x=T(np.zeros((2, 4, 4, 4))), padding="VALID"))
    for kw in bad_bn:
        with pytest.raises(ValueError):
            zs.fused.bn_conv2d(**kw)
        kt = dict(kw)
        if kt["W"] is W:
            kt["W"] = Wt
        with pytest.raises(ValueError):
            zs.fused.bn_conv2d_transpose(**kt)
    for kw in [dict(x=x, W=Wt, b=T(np.zeros(5))), dict(x=x, W=W), dict(x=x, W=Wt, stride=4),
               dict(x=x, W=Wt, padding="FULL"), dict(x=x.cpu(), W=Wt),
               dict(x=x, W=Wt, b=T(np.zeros(6)).double())]:
        with pytest.raises(ValueError):
            zs.fused.sigmoid_conv2d_transpose(**kw)
    assert lib.launches == n
    torch.cuda.synchronize()
