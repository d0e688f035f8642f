"""GPU parity of the kernels under the IWAE training step (scripts/bench_iwae.py) against float64,
at the edges where a tiled tensor-core product or a reduction goes wrong:

1. zs.fused.linear (EPI 0, the input- and weight-gradient products, the dual split pass of
   gemm_logjoint_tc.cu): y, dh, dW and db across a table of row, contraction and feature counts
   (partial last tiles, K off the 64-wide k-block, k-blocks that wrap the two-stage operand ring,
   unit counts on both sides of a multiple of the 132 SMs, split-K slice counts 1, 2 and the
   largest);
2. the max |.| tag a dense layer hands to its consumer, through the encoder and decoder chains;
3. the Bernoulli likelihood layer (EPI 1 and EPI 2) across the 32-lane groups of J, with
   broadcast and full, int32 and float32 observations and logits up to about +-80;
4. reduce.cu (log_mean_exp, log_sum_exp, mean, sum; forward and backward) on both kernels,
   across the column kernel's 4-way unrolled loop and its tail, with -inf / +inf / NaN entries
   and log-weights at realistic magnitudes;
5. the fused IWAE step at the benchmark's shape against a float64 twin, calibrated by the error
   of the same step on unfused fp32 torch layers.

Every comparison is scaled by the magnitude term of its operation, so a bound is a relative
accuracy of the operation rather than of the (possibly cancelling) result.  Each case records its
largest error-to-bound ratio as the junit property ``ratio_*``."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import variational as OV

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                 # unit roundoff of fp32
NUM_SMS = 132


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(g, *shape):
    return torch.randn(*shape, generator=g, device="cuda")


def _err_ratio(got, want, scale):
    """max |got - want| / scale over the elements (want, scale float64)."""
    d = (got.detach().double() - want).abs() / (scale + 1e-30)
    return float(d.max()) if d.numel() else 0.0


# ---------------------------------------------------------------------------------------------
# 1. zs.fused.linear against float64
# ---------------------------------------------------------------------------------------------
# Error bounds of the fp16 hi/lo three-product scheme, relative to the magnitude term of the
# product (sum_k |a_k| |b_k|): the dropped lo*lo product and the fp16 rounding of the lo planes
# (2^-22 each) plus fp32 accumulation.  FWD / GRAD are the bounds test_linear_forward_fp32_accuracy
# and test_linear_backward_on_tensor_cores use.  Beyond them the accumulation term is written
# out: a k-block is 4 k-steps x 3 products accumulated one after the other in the wgmma
# accumulator, so a worst-case rounding walk adds ACC_KB = 12 u per k-block (the tensor core's
# fp32 accumulation does not round to nearest: on partial sums of one sign it drifts toward zero
# by about 6 u per k-block on an H100).  The forward and input-gradient products run all n_kb
# k-blocks of their contraction in the accumulator.  The weight gradient adds its accumulator into
# the tile every PROMOTE_KB = 8 k-blocks (fp32 adds, u each), and its split-K slices are then
# added up in order (u each).  The bias gradient adds one partial column sum per 64-row tile of
# the split pass (u each).
FWD, GRAD = 2e-6, 3e-6
ACC_KB = 12
PROMOTE_KB = 8


def _n_kb(n):
    return (n + 63) // 64


def fwd_bound(K):
    return FWD + ACC_KB * U * _n_kb(K)


def grad_bound(n):
    """the input gradient, contraction length n"""
    return GRAD + ACC_KB * U * _n_kb(n)


def wgrad_bound(R, slices):
    kb_per = -(-_n_kb(R) // slices)
    return GRAD + U * (ACC_KB * min(kb_per, PROMOTE_KB) + -(-kb_per // PROMOTE_KB) + slices)


def db_bound(R):
    return GRAD + U * (_n_kb(R) + 16)


# (lead shape of h, K, J, relu, bias, note).  The unit count of the forward product is
# ceil(R / 128) * ceil(J / 128); a launch runs min(units, 132) CTAs that stride over the units.
LINEAR = [
    ((1,), 1, 1, False, True, "one row, K = 1, one feature"),
    ((127,), 2, 5, True, True, "K = 2: the dual split's kernel path at its smallest width"),
    ((129,), 3, 63, True, False, "K = 3 (odd: the split's torch branch), rows past one tile"),
    ((128,), 64, 128, False, True, "exactly one 128 x 128 tile, one k-block"),
    ((129,), 65, 129, True, True, "partial last row and column tile, K one past a k-block"),
    ((257,), 63, 127, False, True, "three row tiles, K one short of a k-block"),
    ((257,), 128, 255, True, True, "two k-blocks: the two-stage ring filled exactly"),
    ((127,), 129, 257, True, False, "three k-blocks: the ring wraps once, J past two blocks"),
    ((1,), 193, 65, False, True, "one row, four k-blocks"),
    ((256,), 500, 784, True, True, "IWAE d3 / e2 widths (K = 500), J = 784"),
    ((3, 129), 40, 500, True, True, "3-D [P, N, H] input as the decoder sees it (d1: 40 -> 500)"),
    ((2, 200), 500, 784, False, True, "3-D input, decoder output layer widths"),
    ((300,), 784, 500, True, True, "IWAE e1 (784 -> 500)"),
    ((257,), 2049, 129, False, True, "33 k-blocks, the last one a single column"),
    ((64,), 4096, 64, True, True, "64 k-blocks, the ring wraps 32 times"),
    ((16896,), 64, 127, False, True, "132 units: one full round over the SMs"),
    ((16897,), 64, 127, True, True, "133 units: one row tile into the second round"),
    ((33792,), 65, 64, False, False, "264 units: two full rounds"),
    ((33793,), 65, 64, True, True, "265 units: one unit into the third round"),
    ((4224,), 784, 500, True, True, "132 units over four feature blocks (IWAE e1 widths)"),
    ((19, 128), 500, 784, False, True, "133 units over seven feature blocks (decoder output)"),
    ((1000,), 784, 1, True, True, "J = 1: 127 idle features in every tile"),
]

LINEAR_CASES = [pytest.param(*c[:5], id="%s-K%d-J%d%s%s" % ("x".join(map(str, c[0])), c[1], c[2],
                                                           "-relu" if c[3] else "",
                                                           "" if c[4] else "-nobias"))
                for c in LINEAR]

# Split-K of the weight-gradient product dW [J, K] = g^T h over the R rows: zsb_linear_tc_slices
# gives min(132 // tiles, n_kb // 8) slices (>= 1), tiles = ceil(J / 128) * ceil(K / 128),
# n_kb = ceil(R / 64), rounded so that no slice is empty.  (R, K, J, expected slices, coherent,
# note); coherent: h >= 0 and g of mean 1, so every partial sum keeps its sign and the
# accumulation's drift adds up (the ReLU activations and the IWAE decoder's gradients are so)
SPLITK = [
    (960, 64, 64, 1, False, "n_kb = 15: one slice (n_kb // 8 = 1)"),
    (961, 64, 64, 2, False, "n_kb = 16: two slices of 8 k-blocks, the last one a single row"),
    (1024, 8448, 64, 2, False, "66 tiles: 132 // 66 = 2 slices (K = 8448)"),
    (1024, 8449, 64, 1, False, "67 tiles: 132 // 67 = 1 slice (K = 8449, odd)"),
    (67520, 64, 64, 118, False, "n_kb = 1055: 131 wanted, 118 slices of 9 k-blocks"),
    (67584, 64, 64, 132, False, "n_kb = 1056: the largest count, 132 slices of 8 k-blocks"),
    (67585, 63, 33, 118, False, "n_kb = 1057: 132 wanted, 9 k-blocks per slice, ragged last slice"),
    (127990, 63, 33, 125, False, "n_kb = 2000: 125 slices of 16 k-blocks, the last k-block ragged"),
    (32768, 500, 500, 8, True, "16 tiles: 8 slices of 64 k-blocks, coherent sums"),
    (65473, 500, 500, 8, True, "n_kb = 1023: 8 slices of 128 k-blocks, coherent, ragged"),
]


def _linear_check(zs, lead, K, J, relu, bias, seed, coherent=False):
    g = _gen(seed)
    h = _randn(g, *lead, K)
    if coherent:
        h = h.abs()
    W = _randn(g, J, K) / math.sqrt(K)
    b = 0.3 * _randn(g, J) if bias else None
    gy = _randn(g, *lead, J) + (1.0 if coherent else 0.0)
    th, tW = h.clone().requires_grad_(True), W.clone().requires_grad_(True)
    tb = b.clone().requires_grad_(True) if bias else None
    y = zs.fused.linear(th, tW, tb, relu=relu)
    assert tuple(y.shape) == tuple(lead) + (J,)
    grads = torch.autograd.grad(y, [th, tW] + ([tb] if bias else []), gy)
    h2, W64 = h.reshape(-1, K).double(), W.double()
    pre = h2 @ W64.T
    scale = h2.abs() @ W64.abs().T
    if bias:
        pre, scale = pre + b.double(), scale + b.double().abs()
    y2 = y.detach().reshape(-1, J)
    want = pre.clamp_min(0) if relu else pre
    r = {"y": _err_ratio(y2, want, scale) / fwd_bound(K)}
    # the mask of the backward is decided on the device from y; taking it from y makes the
    # reference the exact gradient of what the forward computed (a pre-activation within rounding
    # of 0 may fall either way), and the forward check above bounds y itself
    g64 = gy.reshape(-1, J).double() * ((y2 > 0) if relu else 1.0)
    R = h2.shape[0]
    slices = _slices(zs, J, K, R)
    r["dh"] = _err_ratio(grads[0].reshape(-1, K), g64 @ W64, g64.abs() @ W64.abs()) / grad_bound(J)
    r["dW"] = _err_ratio(grads[1], g64.T @ h2, g64.abs().T @ h2.abs()) / wgrad_bound(R, slices)
    if bias:
        r["db"] = _err_ratio(grads[2], g64.sum(0), g64.abs().sum(0)) / db_bound(R)
    return r, slices


def _slices(zs, J, K, R):
    from zhusuan_b200._lib import lib
    return int(lib.load().zsb_linear_tc_slices(J, K, R))


def _record(record_property, ratios):
    for k, v in ratios.items():
        record_property("ratio_" + k, "%.3g" % v)


@pytest.mark.parametrize("lead,K,J,relu,bias", LINEAR_CASES)
def test_linear_forward_and_gradients_vs_float64(zs, record_property, lead, K, J, relu, bias):
    """y against |h| |W|^T + |b|, dh against |g| |W|, dW against |g|^T |h| and db against
    sum |g|, each scaled by its bound: a dropped k-block, row, column or split-K slice, or a ReLU
    mask one row off, is off by orders of magnitude (the table's note says what each row
    covers)."""
    r, _ = _linear_check(zs, lead, K, J, relu, bias, seed=int(np.prod(lead)) * 7 + K * 3 + J)
    _record(record_property, r)
    assert max(r.values()) < 1.0, r


@pytest.mark.parametrize("R,K,J,slices,coherent",
                         [pytest.param(*c[:5], id="R%d-K%d-J%d-s%d%s" % (c[:4] + ("-coherent"
                                                                                  if c[4] else "",)))
                          for c in SPLITK])
def test_weight_gradient_split_k_vs_float64(zs, record_property, R, K, J, slices, coherent):
    """dW = g^T h on each side of the split-K thresholds: the case's slice count is asserted
    first, so the case stays on its edge if the heuristic changes."""
    assert _slices(zs, J, K, R) == slices
    r, got = _linear_check(zs, (R,), K, J, not coherent, True, seed=R + K + J, coherent=coherent)
    assert got == slices
    _record(record_property, r)
    assert max(r.values()) < 1.0, r


# ---------------------------------------------------------------------------------------------
# 2. The max |.| tag handed from one dense layer to the next
# ---------------------------------------------------------------------------------------------
def _tag_word(t):
    """max |t| as the producing GEMM folded it into word 2 of the scale slot it tagged t with
    (read before a consumer takes the slot: the consumer's split clears the word)."""
    amax = t._zsb_amax
    return float(amax.view(torch.int32)[2:3].view(torch.float32)[0])


def _peaked_chain_params(g, dims):
    """Weights and biases of a ReLU chain dims[0] -> dims[1] -> ... whose largest |y| of every
    layer sits in its last row and last feature, given a boosted last input row: the last
    feature's weights are positive and its bias large."""
    Ws, bs = [], []
    for i, o in zip(dims[:-1], dims[1:]):
        W = _randn(g, o, i) / math.sqrt(i)
        W[-1] = W[-1].abs() + 0.5 / math.sqrt(i)
        b = 0.1 * _randn(g, o)
        b[-1] = 4.0
        Ws.append(W)
        bs.append(b)
    return Ws, bs


def _leaves(ts):
    return [t.clone().requires_grad_(True) for t in ts]


def test_max_tag_handoff_encoder_chain(zs, record_property):
    """linear -> linear -> two heads (the IWAE encoder, 784-500-500-(40, 40)) at N = 257 (a
    partial last row tile) with the largest |y| of each layer in its last row and last, partial
    column: each tag equals max |y| exactly; the outputs and every parameter gradient match a
    float64 twin; each head gives the same bits through the shared split of its input as on its
    own (a fresh copy of the input, split with its own max pass)."""
    g = _gen(21)
    N, dims = 257, (784, 500, 500)
    x = (torch.rand(N, 784, generator=g, device="cuda") < 0.3).float()
    x[-1] = 1.0
    Ws, bs = _peaked_chain_params(g, dims)
    Wm, Ws_ = _randn(g, 40, 500) / math.sqrt(500), _randn(g, 40, 500) / math.sqrt(500)
    bm, bs_ = 0.1 * _randn(g, 40), 0.1 * _randn(g, 40)
    Wm[-1], bm[-1] = Wm[-1].abs() + 0.05, 3.0
    params = _leaves(Ws + bs + [Wm, bm, Ws_, bs_])
    W1, W2, b1, b2, tWm, tbm, tWs, tbs = params
    h1 = zs.fused.linear(x, W1, b1, relu=True)
    tags = [_tag_word(h1)]
    h2 = zs.fused.linear(h1, W2, b2, relu=True)
    tags.append(_tag_word(h2))
    m = zs.fused.linear(h2, tWm, tbm)
    tags.append(_tag_word(m))
    s = zs.fused.linear(h2, tWs, tbs)
    for t, tag in zip((h1, h2, m), tags):
        a = t.detach().abs()
        assert tag == float(a.max())
        assert int(a.argmax()) == a.numel() - 1, "the peak is not in the last row and column"
    # each head on its own: an untagged copy of its input takes the max pass
    h2c = h2.detach().clone()
    assert torch.equal(zs.fused.linear(h2c, tWm.detach(), tbm.detach()), m.detach())
    assert torch.equal(zs.fused.linear(h2.detach().clone(), tWs.detach(), tbs.detach()),
                       s.detach())
    gm, gs = _randn(g, N, 40), _randn(g, N, 40)
    grads = torch.autograd.grad((m * gm).sum() + (s * gs).sum(), params)
    # float64 twin, the ReLU masks taken from the fused forward (see _linear_check)
    P = [p.detach().double().requires_grad_(True) for p in params]
    d1 = (x.double() @ P[0].T + P[2]) * (h1.detach() > 0)
    d2 = (d1 @ P[1].T + P[3]) * (h2.detach() > 0)
    dm, ds = d2 @ P[4].T + P[5], d2 @ P[6].T + P[7]
    ref = torch.autograd.grad((dm * gm.double()).sum() + (ds * gs.double()).sum(), P)
    worst = 0.0
    for got, want in zip((h1, h2, m, s) + tuple(grads), (d1, d2, dm, ds) + tuple(ref)):
        e = float((got.detach().double() - want).abs().max() / want.abs().max())
        worst = max(worst, e)
        assert e < 2e-5, (tuple(want.shape), e)
    record_property("max_rel_err", "%.3g" % worst)


def test_max_tag_handoff_decoder_chain(zs, record_property):
    """linear -> linear -> LinearBernoulli (the IWAE decoder, 40-500-500-784) on z [3, 43, 40]
    (129 rows: a partial last row tile) with the largest |y| of each dense layer in its last row
    and last, partial column: the tags equal max |y| exactly; log p(x | z) and the gradients
    w.r.t. z and every parameter match a float64 twin; the likelihood gives the same bits through
    the tagged split as on an untagged copy of its input."""
    g = _gen(22)
    P_, N = 3, 43
    z = _randn(g, P_, N, 40)
    z[-1, -1] = z[-1, -1].abs() * 3 + 1
    x = (torch.rand(N, 784, generator=g, device="cuda") < 0.2).to(torch.int32)
    Ws, bs = _peaked_chain_params(g, (40, 500, 500))
    W3, b3 = _randn(g, 784, 500) * (2 / math.sqrt(500)), 0.3 * _randn(g, 784)
    params = _leaves([z] + Ws + bs + [W3, b3])
    tz, W1, W2, b1, b2, tW3, tb3 = params
    h1 = zs.fused.linear(tz, W1, b1, relu=True)
    tags = [_tag_word(h1)]
    h2 = zs.fused.linear(h1, W2, b2, relu=True)
    tags.append(_tag_word(h2))
    lp = zs.fused.LinearBernoulli(h2, tW3, tb3).log_prob(x)
    assert tuple(lp.shape) == (P_, N)
    for t, tag in zip((h1, h2), tags):
        a = t.detach().abs()
        assert tag == float(a.max())
        assert int(a.argmax()) == a.numel() - 1, "the peak is not in the last row and column"
    alone = zs.fused.LinearBernoulli(h2.detach().clone(), tW3.detach(), tb3.detach()).log_prob(x)
    assert torch.equal(alone, lp.detach())
    w = _randn(g, P_, N)
    grads = torch.autograd.grad((lp * w).sum(), params)
    P = [p.detach().double().requires_grad_(True) for p in params]
    d1 = (P[0] @ P[1].T + P[3]) * (h1.detach() > 0)
    d2 = (d1 @ P[2].T + P[4]) * (h2.detach() > 0)
    dl = -F.binary_cross_entropy_with_logits(d2 @ P[5].T + P[6], x.double().expand(P_, N, 784),
                                             reduction="none").sum(-1)
    ref = torch.autograd.grad((dl * w.double()).sum(), P)
    worst = 0.0
    for got, want in zip((h1, h2, lp) + tuple(grads), (d1, d2, dl) + tuple(ref)):
        e = float((got.detach().double() - want).abs().max() / want.abs().max())
        worst = max(worst, e)
        assert e < 2e-5, (tuple(want.shape), e)
    record_property("max_rel_err", "%.3g" % worst)


# ---------------------------------------------------------------------------------------------
# 3. The Bernoulli likelihood layer (EPI 1 value, EPI 2 gradient)
# ---------------------------------------------------------------------------------------------
# Per element, bern_lp = -(max(l, 0) - l x + __logf(1 + __expf(-|l|))).  For x in {0, 1} the
# first two terms are exact; __logf on [1, 2] is within 2^-21.41 absolute (CUDA C Programming
# Guide, intrinsic functions), the rounding of 1 + __expf(-|l|) and the error of __expf add at
# most 2^-23, and the final addition rounds by 2^-24 |lp|.  The row's value sums J such terms:
# 32-lane butterfly sums (5 levels), then nparts(J) = 4 ceil(J / 128) partial rows in order.
BERN_ELEM = 2.0 ** -21.41 + 2.0 ** -23


def _bern_value_tol(lp_elem, xs, scale_l, J):
    """Bound on |lp - lp64| per row: J per-element bounds + the rounding of the sum + the error
    of the fp32 logits (at most fwd_bound * scale_l each) times |d lp / dl| = |x - sigmoid(l)|."""
    nparts = 4 * ((J + 127) // 128)
    a = lp_elem.abs()
    return (J * BERN_ELEM + U * a.sum(-1) * (1 + 5 + nparts)
            + (xs * scale_l).sum(-1))


BERN = [
    (1, 1, 1, 1, "one row, one feature, K = 1"),
    (1, 127, 31, 40, "J = 31: one partial 32-lane group, rows one short of a tile"),
    (2, 64, 32, 64, "J = 32: one full group, exactly one row tile"),
    (3, 43, 33, 65, "J = 33: a second group with one lane, a partial second row tile"),
    (4, 64, 127, 500, "J = 127: four groups, the last one lane short"),
    (3, 129, 129, 500, "J = 129: a second feature block (nparts 8) with one lane"),
    (1, 16897, 1, 3, "J = 1 on 133 units: one tile into the second round"),
    (19, 128, 784, 500, "J = 784 on 133 units (7 feature blocks x 19 row tiles): the decoder"),
]
BERN_X = ["bcast-int32", "full-float32", "bcast-float32", "full-int32"]


@pytest.mark.parametrize("x_mode", BERN_X)
@pytest.mark.parametrize("P,N,J,K", [pytest.param(*c[:4], id="P%d-N%d-J%d-K%d" % c[:4])
                                     for c in BERN])
def test_linear_bernoulli_value_and_gradients_vs_float64(zs, record_property, P, N, J, K, x_mode):
    """linear_bernoulli_log_prob and LinearBernoulli(...).log_prob with x [N, J] broadcast over
    the P particles (row r reads x row r % N) or a full [P, N, J], int32 or float32, logits up to
    about +-80: the value within J per-element bounds of float64; the gradients w.r.t. h, W and b
    against float64 binary_cross_entropy_with_logits, each against its magnitude term plus the
    error the fp32 logits carry into d/dl."""
    g = _gen(P * 1000 + N + J)
    h = _randn(g, P, N, K)
    W = _randn(g, J, K) * (25.0 / math.sqrt(K))        # logits ~ N(0, 25^2): |l| up to ~80+
    b = 3.0 * _randn(g, J)
    full, dt = x_mode.startswith("full"), torch.int32 if x_mode.endswith("int32") else torch.float32
    xs = (torch.rand(*((P, N, J) if full else (N, J)), generator=g, device="cuda") < 0.4)
    x = xs.to(dt)
    wr = _randn(g, P, N)
    h64, W64, b64 = h.reshape(-1, K).double(), W.double(), b.double()
    l64 = h64 @ W64.T + b64
    scale_l = (h64.abs() @ W64.abs().T + b64.abs()) * fwd_bound(K)
    x64 = x.double().reshape(-1, J) if full else x.double().repeat(P, 1)
    elem = -F.binary_cross_entropy_with_logits(l64, x64, reduction="none")
    want = elem.sum(-1)
    sg = torch.sigmoid(l64)
    tol = _bern_value_tol(elem, (x64 - sg).abs(), scale_l, J)
    # d/dl = w (x - sigmoid(l)); its error per element: the fp32 logit error times sigmoid' <= 1/4,
    # and the rounding of sigmoid and of x - sigmoid
    gl = wr.reshape(-1, 1).double() * (x64 - sg)
    e_gl = wr.reshape(-1, 1).double().abs() * (0.25 * scale_l + 4 * U)
    ratios = {}
    for api in ("fn", "dist"):
        th, tW, tb = (t.clone().requires_grad_(True) for t in (h, W, b))
        if api == "fn":
            lp = zs.fused.linear_bernoulli_log_prob(th, tW, tb, x)
        else:
            lp = zs.fused.LinearBernoulli(th, tW, tb).log_prob(x)
        assert tuple(lp.shape) == (P, N)
        ratios[api + "_lp"] = float(((lp.detach().reshape(-1).double() - want).abs() / tol).max())
        dh, dW, db = torch.autograd.grad((lp * wr).sum(), [th, tW, tb])
        ratios[api + "_dh"] = _err_ratio(dh.reshape(-1, K), gl @ W64, grad_bound(J) * (gl.abs() @ W64.abs())
                                         + e_gl @ W64.abs())
        ratios[api + "_dW"] = _err_ratio(dW, gl.T @ h64, wgrad_bound(P * N, _slices(zs, J, K, P * N))
                                         * (gl.abs().T @ h64.abs()) + e_gl.T @ h64.abs())
        ratios[api + "_db"] = _err_ratio(db, gl.sum(0), db_bound(P * N) * gl.abs().sum(0)
                                         + e_gl.sum(0))
    _record(record_property, ratios)
    assert max(ratios.values()) < 1.0, ratios


def test_bern_lp_per_element_error(zs, record_property):
    """J = 1: the row's value is one bern_lp term, so its error against float64 on the very fp32
    logit the epilogue saw (EPI 0 over the same planes computes the same fmaf) is the error of
    bern_lp itself, over logits spread evenly on [-80, 80]."""
    R = 1 << 16
    g = _gen(5)
    h = (torch.rand(R, 1, generator=g, device="cuda") * 2 - 1) * 80
    W = torch.ones(1, 1, device="cuda")
    b = torch.zeros(1, device="cuda")
    x = (torch.rand(R, 1, generator=g, device="cuda") < 0.5).float()
    l32 = zs.fused.linear(h, W, b)
    lp = zs.fused.linear_bernoulli_log_prob(h, W, b, x)
    ref = -F.binary_cross_entropy_with_logits(l32.double(), x.double(), reduction="none")[:, 0]
    err = (lp.double() - ref).abs()
    small = l32[:, 0].abs() < 2
    record_property("max_abs_err", "%.3g" % float(err.max()))
    record_property("max_abs_err_small_logits", "%.3g" % float(err[small].max()))
    record_property("max_rel_err", "%.3g" % float((err / ref.abs().clamp_min(1e-30)).max()))
    assert bool((err <= BERN_ELEM + U * ref.abs()).all()), float(err.max())


# ---------------------------------------------------------------------------------------------
# 4. reduce.cu: log_mean_exp, log_sum_exp, mean, sum; forward and backward
# ---------------------------------------------------------------------------------------------
def _ulp(t):
    """ulp of float32 at |t| (t float64)."""
    e = torch.frexp(t.abs().clamp_min(2.0 ** -126).float())[1].double()
    return torch.pow(2.0, e - 24)


def _reduce_ref(op, x64, axis):
    if op == "lme":
        return torch.logsumexp(x64, axis) - math.log(_axis_len(x64, axis))
    if op == "lse":
        return torch.logsumexp(x64, axis)
    if op == "mean":
        return x64.mean(axis)
    return x64.sum(axis)


def _axis_len(x, axis):
    axes = axis if isinstance(axis, tuple) else (axis,)
    return int(np.prod([x.shape[a] for a in axes]))


def _reduce_call(zs, op, x, axis):
    from zhusuan_b200 import ops
    if op == "lme":
        return zs.log_mean_exp(x, axis)
    if op == "lse":
        return zs.log_sum_exp(x, axis)
    return ops.reduce_axes(x, ops.OP_MEAN if op == "mean" else ops.OP_SUM, axis)


def _reduce_check(zs, x, axis, ops_=("lme", "lse", "mean", "sum")):
    """Forward and backward of each op on x (float32, cuda) against float64.  Bounds:
    log-sum-exp: 2 ulp(|y|) (the final m + log s and log's own error) + (n + 4) u for the fp32 sum
    of n terms in [0, 1]; mean / sum: (n + 2) u sum |x| (/ n).  Backward: the softmax is
    exp(x - y) / n from the ROUNDED forward value, so its relative error is the forward bound on y
    (which holds ulp(|y|) ~ ulp(|x|) when the log-weights sit at |x| ~ 1e4: the conditioning of
    the inputs' own rounding, not a defect) plus exp's few ulp; mean / sum are exact up to 1/n."""
    n = _axis_len(x, axis)
    x64 = x.double()
    ratios = {}
    for op in ops_:
        xt = x.clone().requires_grad_(True)
        y = _reduce_call(zs, op, xt, axis)
        want = _reduce_ref(op, x64, axis)
        if op in ("lme", "lse"):
            tol = 2 * _ulp(want) + (n + 4) * U
        else:
            tol = (n + 2) * U * x64.abs().sum(axis) / (n if op == "mean" else 1) + 1e-30
        ratios[op] = float(((y.detach().double() - want).abs() / tol).max())
        gout = torch.rand(want.shape, device="cuda", dtype=torch.float64) + 0.5
        xr = x64.clone().requires_grad_(True)
        dref, = torch.autograd.grad((_reduce_ref(op, xr, axis) * gout).sum(), [xr])
        dx, = torch.autograd.grad((y * gout.float()).sum(), [xt])
        if op in ("lme", "lse"):
            ytol, yb = tol, want
            for a in (sorted(axis) if isinstance(axis, tuple) else [axis]):
                ytol, yb = ytol.unsqueeze(a), yb.unsqueeze(a)
            # + the rounding of x - y and exp's own error
            gtol = dref.abs() * (ytol + (x64 - yb).abs() * U + 8 * U) + 1e-37
        else:
            gtol = dref.abs() * 4 * U + 1e-37
        ratios["d" + op] = float(((dx.double() - dref).abs() / gtol).max())
    return ratios


REDUCE_K = [1, 2, 3, 4, 5, 7, 31, 32, 33, 64, 1000]
REDUCE_INNER = [1, 2, 255, 4096]


@pytest.mark.parametrize("inner", REDUCE_INNER)
@pytest.mark.parametrize("K", REDUCE_K)
def test_reduce_ops_vs_float64(zs, record_property, K, inner):
    """x [3, K, inner] reduced over axis 1: the row kernel (inner = 1, lanes striding K) and the
    column kernel (inner >= 2: its 4-way unrolled loop and the tail of K % 4), log-weights of
    spread 5 around 0."""
    g = _gen(K * 10007 + inner)
    x = 5 * _randn(g, 3, K, inner)
    r = _reduce_check(zs, x, 1)
    _record(record_property, r)
    assert max(r.values()) < 1.0, r


@pytest.mark.parametrize("offset", [-1e2, -1e3, -1e4])
@pytest.mark.parametrize("K,inner", [(64, 4096), (1000, 1), (33, 255)])
def test_reduce_log_weights_at_iwae_magnitudes(zs, record_property, K, inner, offset):
    """log-weights offset by -1e2 .. -1e4 with unit spread (the IWAE bound's log w): the forward
    keeps ulp(|x|) accuracy, the backward's softmax is bounded relative to ulp(|x|)."""
    g = _gen(K + inner + int(-offset))
    x = offset + _randn(g, 2, K, inner)
    r = _reduce_check(zs, x, 1, ops_=("lme", "lse"))
    _record(record_property, r)
    assert max(r.values()) < 1.0, r


def test_reduce_past_the_grid_cap_and_permuted_axes(zs, record_property):
    """More columns (2 x 300000) and rows (20000) than the 132 x 16 blocks of a launch cover in
    one sweep (grid-stride loops), and a reduction over axes (0, 2) of a 4-D tensor (the permute
    path)."""
    g = _gen(3)
    r = {}
    for name, x, axis in [("cols", 3 * _randn(g, 2, 3, 300000), 1),
                          ("rows", 3 * _randn(g, 20000, 33), 1),
                          ("perm", 3 * _randn(g, 4, 5, 6, 7), (0, 2))]:
        for k, v in _reduce_check(zs, x, axis).items():
            r[name + "_" + k] = v
    _record(record_property, r)
    assert max(r.values()) < 1.0, r


@pytest.mark.parametrize("kernel", ["rows", "cols"])
@pytest.mark.parametrize("K", [1, 2, 3, 5, 8, 9])
def test_reduce_non_finite_entries_match_the_oracle(zs, K, kernel):
    """Columns with some -inf entries, all -inf, one +inf and one NaN, the special entry at the
    first, a middle and the last position of K (inside and after the column kernel's unrolled
    groups; a NaN also among -inf entries followed by a finite one): log_mean_exp and log_sum_exp
    give the NaN / -inf / finite results of the reference (zhusuan/utils.py: x - max(x) with a
    NaN-propagating max), on the row kernel and on the column kernel, and the backward's softmax
    is 0 at -inf entries."""
    g = _gen(K * 31 + len(kernel))
    cols = []
    for p in sorted({0, K // 2, K - 1}):
        for kind in ("ninf", "pinf", "nan"):
            c = _randn(g, K)
            c[p] = {"ninf": -math.inf, "pinf": math.inf, "nan": math.nan}[kind]
            cols.append(c)
            if kind == "nan" and K > 1:
                c = torch.full((K,), -math.inf, device="cuda")
                c[p] = math.nan
                c[K - 1 if p != K - 1 else 0] = 0.5
                cols.append(c)
    cols.append(torch.full((K,), -math.inf, device="cuda"))
    x = torch.stack(cols, 1).unsqueeze(0).repeat(2, 1, 1)        # [2, K, C]: C columns of K
    if kernel == "rows":
        x = x.permute(0, 2, 1).contiguous().unsqueeze(-1)          # [2, C, K, 1]: rows of K
        axis = 2
    else:
        axis = 1
    xn = x.cpu().numpy().astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        want_lme = OV.log_mean_exp(xn, axis, dtype=np.float64)
        want_lse = OV.log_sum_exp(xn, axis, dtype=np.float64)
    for fn, want in ((zs.log_mean_exp, want_lme), (zs.log_sum_exp, want_lse)):
        got = fn(x, axis).cpu().numpy().astype(np.float64)
        np.testing.assert_array_equal(np.isnan(got), np.isnan(want))
        fin = ~np.isnan(want)
        np.testing.assert_array_equal(got[fin] == -np.inf, want[fin] == -np.inf)
        ok = np.isfinite(want)
        np.testing.assert_allclose(got[ok], want[ok], rtol=0, atol=1e-5)
    # backward on the columns whose value is finite: the softmax, 0 at the -inf entries
    xt = x.clone().requires_grad_(True)
    y = zs.log_mean_exp(xt, axis)
    keep = torch.isfinite(y.detach())
    dx, = torch.autograd.grad(torch.where(keep, y, torch.zeros_like(y)).sum(), [xt])
    sel = keep.unsqueeze(axis).expand_as(x)
    sm = torch.softmax(x.double().masked_fill(~sel, 0.0), axis)
    assert bool((dx[sel & torch.isinf(x)] == 0).all())
    assert torch.allclose(dx[sel].double(), sm[sel], rtol=1e-5, atol=1e-7)


# ---------------------------------------------------------------------------------------------
# 5. The fused IWAE step at the benchmark's shapes
# ---------------------------------------------------------------------------------------------
def _iwae_params(seed, x_dim=784, z_dim=40, h=500):
    """scripts/bench_iwae.py's parameters (glorot weights) with small nonzero biases, so the bias
    gradients are exercised at a generic point."""
    rng = np.random.Generator(np.random.PCG64(seed))
    W = {}
    for name, (i, o) in dict(e1=(x_dim, h), e2=(h, h), em=(h, z_dim), es=(h, z_dim),
                             d1=(z_dim, h), d2=(h, h), d3=(h, x_dim)).items():
        lim = np.sqrt(6.0 / (i + o))
        W[name] = torch.tensor(rng.uniform(-lim, lim, (o, i)), dtype=torch.float32, device="cuda")
        W[name + "_b"] = torch.tensor(0.05 * rng.standard_normal(o), dtype=torch.float32,
                                      device="cuda")
    return W


def _fused_iwae_step(zs, W, x, eps):
    """The fused step of scripts/bench_iwae.py (every dense layer on zs.fused.linear, the decoder
    output on LinearBernoulli), with the particles' noise injected through _sample(K, eps=...)."""
    K, n, z_dim = eps.shape
    Wd = {k: v.detach().requires_grad_(True) for k, v in W.items()}
    lin = zs.fused.linear

    @zs.meta_bayesian_net(scope="gen", reuse_variables=True)
    def build_gen(n, n_particles):
        bn = zs.BayesianNet()
        z = bn.normal("z", torch.zeros(n, z_dim, device="cuda"), std=1., group_ndims=1,
                      n_samples=n_particles)
        hh = lin(z.tensor, Wd["d1"], Wd["d1_b"], relu=True)
        hh = lin(hh, Wd["d2"], Wd["d2_b"], relu=True)
        bn.stochastic("x", zs.fused.LinearBernoulli(hh, Wd["d3"], Wd["d3_b"]))
        return bn

    def build_q_net(x, n_particles):
        bn = zs.BayesianNet()
        hh = lin(x.float(), Wd["e1"], Wd["e1_b"], relu=True)
        hh = lin(hh, Wd["e2"], Wd["e2_b"], relu=True)
        dist = zs.distributions.Normal(lin(hh, Wd["em"], Wd["em_b"]),
                                       logstd=lin(hh, Wd["es"], Wd["es_b"]), group_ndims=1)
        node = bn.stochastic("z", dist, n_samples=n_particles)
        node._samples = dist._sample(n_particles, eps=eps)
        return bn

    model = build_gen(n, K)
    variational = build_q_net(x, K)
    lb = zs.variational.iw_objective(model, {"x": x}, variational=variational, axis=0)
    cost = torch.mean(lb.sgvb())
    grads = torch.autograd.grad(cost, list(Wd.values()))
    return lb.tensor.detach(), grads


def _torch_iwae_step(W, x, eps, dtype):
    """The same graph op by op in torch at ``dtype`` (scripts/bench_iwae.py make_cpu_step)."""
    Wd = {k: v.detach().to(dtype).requires_grad_(True) for k, v in W.items()}
    xf = x.to(dtype)
    lin = lambda h, n: F.linear(h, Wd[n], Wd[n + "_b"])
    h = F.relu(lin(F.relu(lin(xf, "e1")), "e2"))
    zm, zl = lin(h, "em"), lin(h, "es")
    z = zm + torch.exp(zl) * eps.to(dtype)
    c = -0.5 * math.log(2 * math.pi)
    log_q = (c - zl - 0.5 * torch.exp(-2 * zl) * (z - zm) ** 2).sum(-1)
    log_pz = (c - 0.5 * z ** 2).sum(-1)
    h1 = F.relu(lin(z, "d1"))
    pre2 = lin(h1, "d2")
    logits = lin(F.relu(pre2), "d3")
    log_px = -F.binary_cross_entropy_with_logits(logits, xf.expand_as(logits),
                                                 reduction="none").sum(-1)
    lw = log_pz + log_px - log_q
    lb = torch.logsumexp(lw, 0) - math.log(eps.shape[0])
    out = torch.autograd.grad(-lb.mean(), list(Wd.values()) + [pre2, logits])
    grads, (g2, dl3) = out[:-2], out[-2:]
    # the magnitude terms through which the input-gradient product of d3 (dh = dl3 W3, 13
    # k-blocks) reaches the d2 gradients: |g2| <= mask |dl3| |W3| elementwise
    m2 = ((pre2 > 0) * (dl3.abs() @ Wd["d3"].detach().abs())).reshape(-1, pre2.shape[-1])
    mag = {"d2": float((m2.T @ h1.detach().reshape(-1, h1.shape[-1]).abs()).norm()),
           "d2_b": float(m2.sum(0).norm())}
    return lb.detach(), grads, mag


# the floor is one dense product's own accuracy bound: the fused step cannot be held closer to
# float64 than a single layer of it is
IWAE_FLOOR = GRAD


@pytest.mark.parametrize("K,N", [(64, 4096), (3, 129)], ids=["bench-K64-N4096", "ragged-K3-N129"])
def test_fused_iwae_step_vs_float64(zs, record_property, K, N):
    """The bound [N] and all 14 parameter gradients of the fused step against a float64 twin on
    the same eps, each as a norm-relative error: no more than twice the error of the same step on
    unfused fp32 torch layers (TF32 off), plus a floor of IWAE_FLOOR; for d2 and its bias plus the
    bound of the input-gradient product that feeds them, carried through its magnitude terms."""
    W = _iwae_params(5)
    rng = np.random.Generator(np.random.PCG64(4))
    x = torch.tensor(rng.random((N, 784)) < 0.13, dtype=torch.int32, device="cuda")
    eps = torch.randn(K, N, 40, generator=_gen(7), device="cuda")
    lb_f, g_f = _fused_iwae_step(zs, W, x, eps)
    prev = (torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32)
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    try:
        lb_32, g_32, _ = _torch_iwae_step(W, x, eps, torch.float32)
    finally:
        torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = prev
    lb_64, g_64, mag = _torch_iwae_step(W, x, eps, torch.float64)
    names = ["bound"] + list(W.keys())
    bad = []
    for name, a, b, ref in zip(names, (lb_f,) + tuple(g_f), (lb_32,) + tuple(g_32),
                               (lb_64,) + tuple(g_64)):
        ref_n = float(ref.norm())
        ef = float((a.double() - ref).norm()) / ref_n
        e32 = float((b.double() - ref).norm()) / ref_n
        record_property("err_" + name, "fused %.3g fp32 %.3g ratio %.3g"
                        % (ef, e32, ef / max(e32, 1e-300)))
        # d2 and its bias see the decoder output layer's input gradient, whose k-blocks the
        # tensor core accumulates with the drift toward zero of section 1 (13 k-blocks at J = 784):
        # that product's own bound, carried through its magnitude terms, is added for them
        carried = grad_bound(784) * mag[name] / ref_n if name in mag else 0.0
        record_property("carried_" + name, "%.3g" % carried)
        if ef > 2 * e32 + IWAE_FLOOR + carried:
            bad.append((name, ef, e32))
    assert not bad, bad
