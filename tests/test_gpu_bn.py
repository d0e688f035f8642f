"""The batch-norm path (gemm_logjoint_tc.cu EPI 9 - 11, bn_stats_kernel, bn_apply_kernel, the
three backward kernels, and conv_tc.cu's col2im epilogues 2 and 3) against float64, stage by
stage through the C ABI, then the four layers that run on it (bn_linear, noisy_bn_linear,
bn_conv2d, bn_conv2d_transpose) end to end against their oracles.

Each stage is fed its own fp32 inputs -- the kernel's own pre-activation ``a``, partials or stats
-- so a bound covers one stage's rounding, and an indexing or count error misses by a wide
margin.  u = 2^-24.  The rounding model of each stage, per column:

* Tile moments (EPI 9; col2im epi 2).  A tile of cnt rows sums its entries in fp32 and divides
  by cnt.  EPI 9 adds the cnt entries in one run, so its tile mean is off by at most
  (cnt + 1) u mean|a|.  col2im epi 2 adds runs of <= 16 rows per warp, then the 8 warp sums in
  turn: (min(cnt, 16) + 8 + 1) u mean|a|.  The M2 about the kernel's tile mean m~ = m + dm is
  sum (a - m~)^2 = M2 + cnt dm^2, each square off by 2 u (the rounded difference) and the run of
  fmas by its length: |M2~ - M2| <= (L + 3) u M2 + cnt dm^2, L the longest run as above.
* Merge (bn_stats_kernel).  Chan's formula in double over the fp32 partials: against a float64
  merge of the same partials, only the double rounding (< 1e-12 relative to the magnitudes) and
  the final fp32 casts remain: u |mean|, and for rstd = rsqrtf(var + eps) the cast and the add
  (u each, halved by the square root) and rsqrtf's 2 u: 3 u rstd.  Against the population
  moments of ``a`` the partials' errors add: the mean is the weighted mean of the tile means, so
  it is off by sum_t cnt_t dm_t / R; the variance gains sum_t [(L_t + 3) u M2_t + cnt_t dm_t^2 +
  4 cnt_t |m_t - mean| dm_t] / R + 4 dm^2 (the between-tile term with perturbed tile means).
* Moving statistics: m -= (m - batch) rate in fp32: rate times the batch's error, plus 3 u of
  |m| + rate |m - batch|.  Bessel's R / (R - 1) (R = 1: the factor 1, M2 = 0) is applied in double.
* Affine step (bn_apply_kernel, EPI 10 / 11, col2im epi 3): d = a - mean (u), then fma(d, rstd,
  beta) or fma(d rstd, gamma, beta) (u each): 3 u (|d| rstd |gamma| + |beta|).  ReLU is exact,
  and the amax slot holds max |out| exactly.  EPI 11's pre is the product, bounded as in
  test_gpu_iwae_kernels (2e-6 + 12 u per 64-wide k-block of sum |h| |W|).  col2im adds up to
  k^2 taps in a fixed order: (k^2 - 1) u sum |tap|.
* Backward sums.  dbeta = sum g' and dgamma = sum g' xhat run 16-row runs per warp, 8 warp sums in
  turn, then lane-strided runs of ceil(n_t / 32) tile sums and a 5-level shuffle tree:
  (16 + 8 + ceil(n_t / 32) + 5 + 2) u sum |term|; xhat = (a - mean) rstd adds 2 u |xhat| to each
  term of dgamma.  da = gamma rstd (g' - c1 - xhat c2) with c1 = dbeta / R and c2 = dgamma / R
  (u each beyond their sums' errors): |gamma| rstd (dc1 + |xhat| dc2 + 5 u (|g'| + |c1| +
  |xhat c2|) + 2 u |xhat c2|); in evaluation da = gamma rstd g' (two roundings: 2 u + u^2).  The planes hold hi + lo
  of da s at fp16: hi is off by 2^-11 of its value and lo by 2^-11 of that or half an fp16
  subnormal step, so (hi + lo) / s is within 2^-22 |da| + 2^-25 / s of da.
* End to end, the product's error e_a = (2e-6 + 12 u n_kb) sum |h| |W| moves xhat by rstd (e_a +
  mean e_a) + |xhat| drstd / rstd, with dvar <= 2 mean(|a - mean| e_a) + mean(e_a)^2 and drstd /
  rstd <= dvar / (2 (var + eps)); the stage bounds above come on top.  The gradient products add
  their own bound (2e-6 / 3e-6 + 12 u per k-block, test_gpu_iwae_kernels) on the magnitudes of
  the fp32 da.

Each GPU case records its largest error-to-bound ratio per quantity as the junit property
``ratio_*``.  The CPU tests at the end feed each comparator a float64 reference and copies of it
perturbed as a broken kernel would perturb it; the comparator must accept the first and reject
the others."""
import math

import numpy as np
import pytest
import torch

import blvae_oracle as BO
import gan_oracle as GO
import vardrop_oracle as VO

U = 2.0 ** -24
BN = 128                      # rows per moment partial and per backward tile
EPS = float(np.float32(1e-3))
FWD, GRAD, ACC_KB = 2e-6, 3e-6, 12


def _n_kb(n):
    return (n + 63) // 64


def fwd_bound(K):
    return FWD + ACC_KB * U * _n_kb(K)


def grad_bound(n):
    return GRAD + ACC_KB * U * _n_kb(n)


def wgrad_bound(R):
    # the weight-gradient product: 8 k-blocks per promotion, at most 132 split-K slices
    return GRAD + U * (ACC_KB * 8 + _n_kb(R) // 8 + 1 + 132)


# ---------------------------------------------------------------------------------------------
# float64 references and bounds (device-agnostic: the CPU tests run them on the CPU)
# ---------------------------------------------------------------------------------------------
def tile_counts(R, device="cpu"):
    n_t = -(-R // BN)
    c = torch.full((n_t,), float(BN), dtype=torch.float64, device=device)
    c[-1] = R - (n_t - 1) * BN
    return c


def _tiles(a64):
    """a64 [R, J] -> [n_t, 128, J] zero-padded, and the row mask of the same shape."""
    R, J = a64.shape
    n_t = -(-R // BN)
    pad = n_t * BN - R
    t = torch.cat([a64, a64.new_zeros(pad, J)]).reshape(n_t, BN, J)
    m = torch.cat([a64.new_ones(R, 1), a64.new_zeros(pad, 1)]).reshape(n_t, BN, 1)
    return t, m


def tile_moments(a64):
    """Per tile: (mean, M2 about it, mean |a|) [n_t, J], from the tile's true row count."""
    t, m = _tiles(a64)
    cnt = tile_counts(a64.shape[0], a64.device)[:, None]
    mean = t.sum(1) / cnt
    m2 = (((t - mean[:, None]) * m) ** 2).sum(1)
    return mean, m2, t.abs().sum(1) / cnt


def tile_run(cnt, col2im):
    """The longest fp32 run of a tile's sums (EPI 9: one run; col2im: 16-row runs + 8 warps)."""
    return torch.clamp(cnt, max=16) + 8 if col2im else cnt


def partial_bounds(a64, col2im=False):
    """Reference tile (mean, M2) and their bounds [n_t, J] by the model of the docstring."""
    mean, m2, mabs = tile_moments(a64)
    cnt = tile_counts(a64.shape[0], a64.device)[:, None]
    L = tile_run(cnt, col2im)
    dm = (L + 1) * U * mabs
    return mean, m2, dm + 1e-30, (L + 3) * U * m2 + cnt * dm ** 2 + 1e-30


def check_partials(part, a64, col2im=False):
    """Ratios (mean, M2) of the kernel's partials [n_t, 2, J] to their bounds."""
    mean, m2, bm, bq = partial_bounds(a64, col2im)
    p = part.double().reshape(-1, 2, a64.shape[1])
    return (float(((p[:, 0] - mean).abs() / bm).max()),
            float(((p[:, 1] - m2).abs() / bq).max()))


def merge64(part, R):
    """float64 merge of fp32 partials [n_t, 2, J] into (mean, var), and the magnitude of the
    merge's terms."""
    p = part.double()
    cnt = tile_counts(R, p.device)[:, None]
    mean = (cnt * p[:, 0]).sum(0) / R
    m2 = p[:, 1].sum(0) + (cnt * (p[:, 0] - mean) ** 2).sum(0)
    return mean, m2 / R, (cnt * p[:, 0].abs()).sum(0) / R


def rstd64(var):
    return 1.0 / torch.sqrt(var + EPS)


def check_merge(stats, part, R):
    """Ratios (mean, rstd) of stats [2, J] against the float64 merge of the kernel's partials.
    The kernel's double merge adds at most 2^-52 |mean| per step to its running mean, so over
    n_t steps the mean is off by n_t 2^-52 mag and M2 / R by twice that times the largest
    deviation of a tile mean, plus n_t 2^-52 var."""
    mean, var, mag = merge64(part, R)
    n_t = part.shape[0]
    dev = (part.double()[:, 0] - mean).abs().max(0).values
    dd = 2.0 ** -50 * n_t
    rs = rstd64(var)
    s = stats.double()
    b_rs = rs * (3 * U + 0.5 * dd * (mag * dev + var) / (var + EPS))
    return (float(((s[0] - mean).abs() / (U * mean.abs() + dd * mag + 1e-30)).max()),
            float(((s[1] - rs).abs() / b_rs).max()))


def population_bounds(a64, col2im=False):
    """(mean, var) of a64 over its rows and their bounds given the partials' model."""
    R = a64.shape[0]
    mean = a64.mean(0)
    var = ((a64 - mean) ** 2).mean(0)
    tm, m2, bm, _ = partial_bounds(a64, col2im)
    cnt = tile_counts(R, a64.device)[:, None]
    L = tile_run(cnt, col2im)
    b_mean = (cnt * bm).sum(0) / R + U * mean.abs()
    b_var = (((L + 3) * U * m2 + cnt * bm ** 2 + 4 * cnt * (tm - mean).abs() * bm).sum(0) / R
             + 4 * b_mean ** 2 + U * var + 1e-30)
    return mean, var, b_mean, b_var


def check_population(stats, a64, col2im=False):
    """Ratios (mean, rstd) of stats [2, J] against the population moments of a64."""
    mean, var, bm, bv = population_bounds(a64, col2im)
    rs = rstd64(var)
    b_rs = rs * (0.5 * bv / (var + EPS) + 3 * U)
    s = stats.double()
    return (float(((s[0] - mean).abs() / bm).max()), float(((s[1] - rs).abs() / b_rs).max()))


def moving64(mm, mv, mean, var, R, rate, bessel):
    """The moving statistics after one training step (float64), with Bessel's R / (R - 1)."""
    v = var * (R / (R - 1.0) if bessel and R > 1 else 1.0)
    return mm - (mm - mean) * rate, mv - (mv - v) * rate


def check_moving(new_mm, new_mv, mm, mv, a64, rate, bessel, col2im=False):
    R = a64.shape[0]
    rate = float(np.float32(rate))          # the rate the kernel is given
    mean, var, bm, bv = population_bounds(a64, col2im)
    f = R / (R - 1.0) if bessel and R > 1 else 1.0
    em, ev = moving64(mm.double(), mv.double(), mean, var, R, rate, bessel)
    b_m = rate * bm + 3 * U * (mm.double().abs() + rate * (mm.double() - mean).abs()) + 1e-30
    b_v = rate * f * bv + 3 * U * (mv.double().abs() + rate * (mv.double() - var * f).abs()) + \
        1e-30
    return (float(((new_mm.double() - em).abs() / b_m).max()),
            float(((new_mv.double() - ev).abs() / b_v).max()))


def affine64(a64, stats, gamma, beta, relu):
    """act(xhat * gamma + beta) from the kernel's own a and fp32 stats, and its bound."""
    s = stats.double()
    d = a64 - s[0]
    xh = d * s[1]
    gm = gamma.double() if gamma is not None else torch.ones_like(s[0])
    y = xh * gm + beta.double()
    b = 3 * U * (xh.abs() * gm.abs() + beta.double().abs()) + 1e-30
    return (y.clamp_min(0) if relu else y), b


def check_affine(out, a64, stats, gamma, beta, relu):
    want, b = affine64(a64, stats, gamma, beta, relu)
    return float(((out.double() - want).abs() / b).max())


def sums_len(R):
    return 16 + 8 + -(-(-(-R // BN)) // 32) + 5 + 2


def grad64(g, y, a, stats, gamma, relu, training):
    """dbeta, dgamma, da and their bounds in float64 from fp32 inputs."""
    R = g.shape[0]
    gg = g.double() * ((y > 0).double() if relu else 1.0)
    s = stats.double()
    xh = (a.double() - s[0]) * s[1] if a is not None else None
    L = sums_len(R)
    db = gg.sum(0)
    b_db = L * U * gg.abs().sum(0) + 1e-30
    dg = b_dg = None
    if xh is not None:
        dg = (gg * xh).sum(0)
        b_dg = (L + 3) * U * (gg * xh).abs().sum(0) + 1e-30
    gm = gamma.double().abs() if gamma is not None else torch.ones_like(s[1])
    gs = (gamma.double() if gamma is not None else 1.0) * s[1]
    if training:
        c1, c2 = db / R, dg / R
        dc1, dc2 = b_db / R + U * c1.abs(), b_dg / R + U * c2.abs()
        da = gs * (gg - c1 - xh * c2)
        b_da = gm * s[1] * (dc1 + xh.abs() * dc2 + 5 * U * (gg.abs() + c1.abs() +
                                                             (xh * c2).abs())
                            + 2 * U * (xh * c2).abs())
    else:
        da = gs * gg
        b_da = (2 * U + U * U) * da.abs()
    return db, b_db, dg, b_dg, da, b_da + 1e-30


def plane_scale(m):
    """pow2_plane_scale: 2^(12 - e) with m = f 2^e, f in [0.5, 1) (m = 0: 2^12)."""
    e = math.frexp(m)[1] if m > 0 else 0
    return math.ldexp(1.0, 12 - e)


def _ratio(got, want, b):
    if got.numel() == 0:
        return 0.0
    return float(((got.detach().double() - want.detach()).abs() / b.detach()).max())


# ---------------------------------------------------------------------------------------------
# GPU plumbing
# ---------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def _lib():
    from zhusuan_b200._lib import lib, ptr, stream
    return lib, ptr, stream


def _f32(*shape, fill=None):
    t = torch.empty(*shape, dtype=torch.float32, device="cuda")
    if fill is not None:
        t.fill_(fill)
    return t


def _split(t):
    lib, ptr, stream = _lib()
    rows, K = t.shape
    Kp = lib.load().zsb_linear_tc_kpad(K)
    planes = torch.empty((2, rows, Kp), dtype=torch.float16, device="cuda")
    scale = torch.zeros(4, dtype=torch.float32, device="cuda")
    lib.call("zsb_split16_pad_f32", ptr(t), rows, K, ptr(planes), ptr(scale), stream())
    return planes, scale


def _record(record_property, r):
    for k, v in r.items():
        record_property("ratio_" + k, "%.3g" % v)


def _assert_within(r):
    """Every ratio at most 1; a NaN ratio (an entry never written) fails too."""
    assert all(v <= 1.0 for v in r.values()), r


# Column kinds: |mean| / std of 0, 10 and 1e3; constant; std far below sqrt(eps); a linear trend
# over the rows, so that the tile means differ and the merge's between-tile term dominates; a
# generic offset column.
KINDS = 7


def _columns(R, J, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    z = torch.randn(R, J, generator=g, device="cuda")
    k = torch.arange(J, device="cuda") % KINDS
    r = (torch.arange(R, device="cuda", dtype=torch.float32) / max(R - 1, 1))[:, None]
    cols = torch.where(k == 0, z, z)
    cols = torch.where(k == 1, 10.0 + z, cols)
    cols = torch.where(k == 2, 1e3 + z, cols)
    cols = torch.where(k == 3, torch.full_like(z, 3.3), cols)
    cols = torch.where(k == 4, 1.0 + 1e-4 * z, cols)
    cols = torch.where(k == 5, 5.0 * r + 0.1 * z, cols)
    cols = torch.where(k == 6, 3.0 * z - 2.0, cols)
    return cols.contiguous()


def _params(J, seed, gamma="random"):
    g = torch.Generator(device="cuda").manual_seed(seed + 1)
    gm = torch.randn(J, generator=g, device="cuda") + 1.0
    if gamma == "special":
        gm[::3] = 0.0
        gm[1::3] = -gm[1::3].abs()
    beta = 0.3 * torch.randn(J, generator=g, device="cuda")
    mm = 0.1 * torch.randn(J, generator=g, device="cuda")
    mv = 0.5 + torch.rand(J, generator=g, device="cuda")
    return gm, beta, mm, mv


def _bn_call(training, bessel, wpl, hpl, gamma, beta, mm, mv, rate, R, J, K, relu, binary=0,
             a=None, part=None):
    lib, ptr, stream = _lib()
    stats, out, amax = _f32(2, J, fill=float("nan")), _f32(R, J, fill=float("nan")), _f32(4)
    amax.zero_()
    if training:
        a = _f32(R, J, fill=float("nan")) if a is None else a
        part = _f32(-(-R // BN) * 2 * J, fill=float("nan")) if part is None else part
    lib.call("zsb_linear_tc_bn_f32", int(training), int(bessel), ptr(wpl[0]), ptr(wpl[1]),
             ptr(hpl[0]), ptr(hpl[1]), int(binary), ptr(gamma), ptr(beta), ptr(mm), ptr(mv),
             float(rate), EPS, ptr(stats), ptr(a), ptr(part), ptr(out), R, J, K, int(relu),
             ptr(amax), stream())
    return stats, out, a, part, amax


# ---------------------------------------------------------------------------------------------
# 1-3. Training forward: partials, merge, moving statistics, affine step (zsb_linear_tc_bn_f32)
# ---------------------------------------------------------------------------------------------
# (R, J, note); h = the designed columns and W = I, so a is the columns up to the product's
# rounding, and every check reads the kernel's own a
TRAIN = [
    (1, 7, "one row: var = 0, Bessel's factor 1"),
    (2, 1, "two rows, one column"),
    (127, 31, "one partial tile"),
    (128, 32, "one full tile, one grad-sum block"),
    (129, 33, "a second tile of one row"),
    (255, 127, "two tiles, the last one row short"),
    (4095, 128, "32 tiles, the last one row short"),
    (4096, 129, "exactly 32 tiles: every lane one tile"),
    (4097, 500, "33 tiles: lane 0 takes a second tile of one row"),
    (32 * 4096 + 1, 33, "1025 tiles: every lane 32 or 33"),
    (802816, 64, "DCGAN conv3x3_64 rows (4096 images of 14 x 14): 6272 tiles"),
]


@pytest.mark.gpu
@pytest.mark.parametrize("R,J", [pytest.param(R, J, id="R%d-J%d" % (R, J)) for R, J, _ in TRAIN])
def test_training_forward_stages_vs_float64(zs, record_property, R, J):
    """Partials per tile, the merged stats against both the float64 merge of those partials and
    the population moments of a, the moving statistics (population variance, rate 1 and 0.1),
    and the affine step with and without gamma, ReLU on and off, with the exact amax tag."""
    h = _columns(R, J, seed=R + 7 * J)
    wpl = _split(torch.eye(J, device="cuda"))
    hpl = _split(h)
    gm, beta, mm, mv = _params(J, R + J)
    r = {}
    for i, (gamma, relu, rate) in enumerate(((gm, True, 1.0), (None, False, 0.1))):
        m1, v1 = mm.clone(), mv.clone()
        stats, out, a, part, amax = _bn_call(True, 0, wpl, hpl, gamma, beta, m1, v1, rate, R, J,
                                             J, relu)
        a64 = a.double()
        part3 = part.reshape(-1, 2, J)
        tag = "" if i == 0 else "_nogamma"
        if i == 0:
            r["tile_mean"], r["tile_m2"] = check_partials(part, a64)
            r["merge_mean"], r["merge_rstd"] = check_merge(stats, part3, R)
            r["pop_mean"], r["pop_rstd"] = check_population(stats, a64)
        r["mm" + tag], r["mv" + tag] = check_moving(m1, v1, mm, mv, a64, rate, False)
        r["out" + tag] = check_affine(out, a64, stats, gamma, beta, relu)
        assert float(amax[2]) == float(out.abs().max())
        if relu:
            assert bool((out >= 0).all())
    _record(record_property, r)
    _assert_within(r)


@pytest.mark.gpu
@pytest.mark.parametrize("R", [1, 2, 129, 4097, 32 * 4096 + 1])
def test_bessel_moving_variance(zs, record_property, R):
    """bessel = 1 of zsb_linear_tc_bn_f32 and zsb_bn_finish_fused_f32 on the same a and partials:
    the moving variance moves towards M2 / (R - 1) (R = 1: towards 0); rate 1 exposes the factor
    at full size.  The finish entry gives the bits of the fused call."""
    lib, ptr, stream = _lib()
    J = 40
    h = _columns(R, J, seed=3 * R + 1)
    wpl, hpl = _split(torch.eye(J, device="cuda")), _split(h)
    gm, beta, mm, mv = _params(J, R)
    m1, v1 = mm.clone(), mv.clone()
    stats, out, a, part, amax = _bn_call(True, 1, wpl, hpl, gm, beta, m1, v1, 1.0, R, J, J, True)
    a64 = a.double()
    r = {}
    r["mm"], r["mv"] = check_moving(m1, v1, mm, mv, a64, 1.0, True)
    m2, v2 = mm.clone(), mv.clone()
    stats2, out2, amax2 = _f32(2, J, fill=float("nan")), _f32(R, J, fill=float("nan")), _f32(4)
    amax2.zero_()
    lib.call("zsb_bn_finish_fused_f32", ptr(a), ptr(part), R, J, ptr(gm), ptr(beta), ptr(m2),
             ptr(v2), 1.0, EPS, ptr(stats2), ptr(out2), 1, ptr(amax2), stream())
    for x, y in ((m1, m2), (v1, v2), (stats, stats2), (out, out2), (amax, amax2)):
        assert torch.equal(x, y)
    if R == 1:
        # one row: M2 = 0, so the moving variance goes to exactly 0 at rate 1
        assert bool((v1 == 0).all())
    _record(record_property, r)
    _assert_within(r)


@pytest.mark.gpu
@pytest.mark.parametrize("R,J", [(1, 1), (129, 33), (4097, 129), (20000, 500)])
def test_evaluation_epilogues_vs_float64(zs, record_property, R, J):
    """EPI 10 (no gamma), EPI 11 with and without pre: stats from the moving statistics, which
    stay bit-for-bit; out against act(xhat gamma + beta) from the kernel's own a (EPI 11's pre,
    itself checked against the float64 product), ReLU on and off, and the exact amax tag."""
    g = torch.Generator(device="cuda").manual_seed(R + J)
    K = 3 * J + 5
    h = torch.randn(R, K, generator=g, device="cuda")
    W = torch.randn(J, K, generator=g, device="cuda") / math.sqrt(K)
    wpl, hpl = _split(W), _split(h)
    gm, beta, mm, mv = _params(J, R, gamma="special")
    mm0, mv0 = mm.clone(), mv.clone()
    r = {}
    pre = _f32(R, J, fill=float("nan"))
    stats, out11, _, _, amax = _bn_call(False, 0, wpl, hpl, gm, beta, mm, mv, 0.1, R, J, K, True,
                                        a=pre)
    assert torch.equal(mm, mm0) and torch.equal(mv, mv0)
    assert torch.equal(stats[0], mm)
    r["rstd"] = _ratio(stats[1], rstd64(mv.double()), 3 * U * rstd64(mv.double()))
    h64, W64 = h.double(), W.double()
    r["pre"] = _ratio(pre, h64 @ W64.T, fwd_bound(K) * (h64.abs() @ W64.abs().T) + 1e-30)
    a64 = pre.double()
    r["epi11"] = check_affine(out11, a64, stats, gm, beta, True)
    assert float(amax[2]) == float(out11.abs().max())
    _, out11b, _, _, _ = _bn_call(False, 0, wpl, hpl, gm, beta, mm, mv, 0.1, R, J, K, True)
    assert torch.equal(out11, out11b)
    stats10, out10, _, _, amax10 = _bn_call(False, 0, wpl, hpl, None, beta, mm, mv, 0.1, R, J, K,
                                            False)
    r["epi10"] = check_affine(out10, a64, stats10, None, beta, False)
    assert float(amax10[2]) == float(out10.abs().max())
    assert torch.equal(mm, mm0) and torch.equal(mv, mv0)
    _record(record_property, r)
    _assert_within(r)


@pytest.mark.gpu
@pytest.mark.parametrize("training", [True, False])
def test_binary_sample_plane(zs, record_property, training):
    """The Z = 2 instances: the one plane of a LinearBernoulli 0/1 sample.  Training: partials,
    merge and affine step from the kernel's own a; evaluation: pre against the exact product."""
    g = torch.Generator(device="cuda").manual_seed(11)
    x = torch.randn(1500, 30, generator=g, device="cuda")
    Wq, bq = torch.randn(40, 30, generator=g, device="cuda"), torch.randn(40, generator=g,
                                                                           device="cuda")
    z = zs.fused.LinearBernoulli(x, Wq, bq, dtype=torch.float32).sample(3)
    pl = z._zsb_pl
    assert pl.binary
    R, K, J = 4500, 40, 129
    W = torch.randn(J, K, generator=g, device="cuda") / math.sqrt(K)
    wpl = _split(W)
    gm, beta, mm, mv = _params(J, 5)
    m1, v1 = mm.clone(), mv.clone()
    r = {}
    pre = None if training else _f32(R, J, fill=float("nan"))
    stats, out, a, part, amax = _bn_call(training, 0, wpl, (pl.planes, pl.scale), gm, beta, m1,
                                         v1, 0.1, R, J, K, True, binary=1, a=pre)
    z64, W64 = z.reshape(R, K).double(), W.double()
    r["a"] = _ratio(a, z64 @ W64.T, fwd_bound(K) * (z64.abs() @ W64.abs().T) + 1e-30)
    a64 = a.double()
    if training:
        r["tile_mean"], r["tile_m2"] = check_partials(part, a64)
        r["merge_mean"], r["merge_rstd"] = check_merge(stats, part.reshape(-1, 2, J), R)
        r["mm"], r["mv"] = check_moving(m1, v1, mm, mv, a64, 0.1, False)
    else:
        assert torch.equal(m1, mm) and torch.equal(v1, mv)
    r["out"] = check_affine(out, a64, stats, gm, beta, True)
    assert float(amax[2]) == float(out.abs().max())
    _record(record_property, r)
    _assert_within(r)


# ---------------------------------------------------------------------------------------------
# col2im epilogues 2 (training: pre + partials) and 3 (evaluation) on transposed geometries
# ---------------------------------------------------------------------------------------------
def col2im64(cols, N, Hb, Wb, Hs, Ws, k, s, pt, pl, C):
    """float64 col2im of cols [N Hs Ws, k k C] onto [N Hb Wb, C]: the sum over the taps (kh, kw)
    of small pixel (i, j) landing on big pixel (s i + kh - pt, s j + kw - pl)."""
    c6 = cols.reshape(N, Hs, Ws, k, k, C)
    Hp, Wp = max(s * Hs + k, pt + Hb), max(s * Ws + k, pl + Wb)
    out = cols.new_zeros(N, Hp, Wp, C)
    for kh in range(k):
        for kw in range(k):
            out[:, kh:kh + s * Hs:s, kw:kw + s * Ws:s] += c6[:, :, :, kh, kw]
    return out[:, pt:pt + Hb, pl:pl + Wb].reshape(N * Hb * Wb, C)


# (N, Hs, k, s, C): the big grid is Hb = Hs s (SAME), pads by TF's rule
COL2IM = [(1, 1, 1, 1, 1), (1, 4, 3, 2, 7), (2, 8, 4, 2, 33), (3, 7, 5, 2, 64), (64, 7, 5, 2, 64),
          (5, 17, 3, 1, 129)]


@pytest.mark.gpu
@pytest.mark.parametrize("N,Hs,k,s,C", [pytest.param(*c, id="N%d-H%d-k%d-s%d-C%d" % c)
                                         for c in COL2IM])
def test_col2im_bn_epilogues_vs_float64(zs, record_property, N, Hs, k, s, C):
    """epi 2: pre against the float64 col2im of the columns, the partials per tile from the
    kernel's own pre, then zsb_bn_finish_fused_f32's merge and Bessel update; epi 3: the
    evaluation affine step with pre, stats and the exact amax tag, moving statistics unchanged."""
    lib, ptr, stream = _lib()
    from zhusuan_b200.fused import _tf_pad_before
    Hb = Wb = Hs * s
    pt = _tf_pad_before(Hb, Hs, k, s, "SAME")
    R = N * Hb * Wb
    g = torch.Generator(device="cuda").manual_seed(N * 131 + C)
    cols = torch.randn(N * Hs * Hs, k * k * C, generator=g, device="cuda")
    cols[:, ::KINDS] += 50.0              # channels with a large mean against their spread
    geo = (N, Hb, Wb, C, Hs, Hs, k, s, pt, pt)
    want = col2im64(cols.double(), N, Hb, Wb, Hs, Hs, k, s, pt, pt, C)
    mag = col2im64(cols.double().abs(), N, Hb, Wb, Hs, Hs, k, s, pt, pt, C)
    gm, beta, mm, mv = _params(C, N + C, gamma="special")
    pre, part = _f32(R, C, fill=float("nan")), _f32(-(-R // BN) * 2 * C, fill=float("nan"))
    nul = None
    lib.call("zsb_conv_col2im_f32", 2, ptr(cols), *geo, nul, nul, nul, nul, nul, nul, EPS, 0,
             nul, ptr(pre), ptr(part), nul, nul, stream())
    r = {"pre": _ratio(pre, want, (k * k) * U * mag + 1e-30)}
    a64 = pre.double()
    r["tile_mean"], r["tile_m2"] = check_partials(part, a64, col2im=True)
    m1, v1 = mm.clone(), mv.clone()
    stats, out, amax = _f32(2, C), _f32(R, C), _f32(4)
    amax.zero_()
    lib.call("zsb_bn_finish_fused_f32", ptr(pre), ptr(part), R, C, ptr(gm), ptr(beta), ptr(m1),
             ptr(v1), 0.5, EPS, ptr(stats), ptr(out), 1, ptr(amax), stream())
    r["merge_mean"], r["merge_rstd"] = check_merge(stats, part.reshape(-1, 2, C), R)
    r["pop_mean"], r["pop_rstd"] = check_population(stats, a64, col2im=True)
    r["mm"], r["mv"] = check_moving(m1, v1, mm, mv, a64, 0.5, True, col2im=True)
    r["out"] = check_affine(out, a64, stats, gm, beta, True)
    assert float(amax[2]) == float(out.abs().max())
    # epi 3
    m0, v0 = mm.clone(), mv.clone()
    pre3, stats3, out3, amax3 = _f32(R, C, fill=float("nan")), _f32(2, C), _f32(R, C), _f32(4)
    amax3.zero_()
    lib.call("zsb_conv_col2im_f32", 3, ptr(cols), *geo, nul, nul, ptr(gm), ptr(beta), ptr(mm),
             ptr(mv), EPS, 0, ptr(stats3), ptr(pre3), nul, ptr(out3), ptr(amax3), stream())
    assert torch.equal(mm, m0) and torch.equal(mv, v0)
    assert torch.equal(pre3, pre)
    assert torch.equal(stats3[0], mm)
    r["eval_rstd"] = _ratio(stats3[1], rstd64(mv.double()), 3 * U * rstd64(mv.double()))
    r["eval_out"] = check_affine(out3, a64, stats3, gm, beta, False)
    assert float(amax3[2]) == float(out3.abs().max())
    _record(record_property, r)
    _assert_within(r)


# ---------------------------------------------------------------------------------------------
# 4. Backward: zsb_bn_grad_f32out and zsb_bn_grad_f32 on synthetic inputs
# ---------------------------------------------------------------------------------------------
def _grad_inputs(R, J, seed, gamma):
    g_ = torch.Generator(device="cuda").manual_seed(seed)
    a = _columns(R, J, seed + 3)
    s = a.double()
    mean = s.mean(0)
    stats = torch.stack([mean, rstd64(((s - mean) ** 2).mean(0))]).float().contiguous()
    gy = torch.randn(R, J, generator=g_, device="cuda")
    k = torch.arange(J, device="cuda") % 3
    gy = torch.where(k == 1, 2.0 + 1e-3 * gy, gy)      # g' nearly constant: g' - mean(g') cancels
    y = torch.relu(torch.randn(R, J, generator=g_, device="cuda"))   # about half exact zeros
    gm = torch.randn(J, generator=g_, device="cuda") + 1.0
    if gamma == "zero":
        gm.zero_()
    elif gamma == "negative":
        gm = -gm.abs()
    elif gamma == "none":
        gm = None
    return gy.contiguous(), y, a, stats, gm


# (R, J): rows across the tile and lane-run edges, columns across the 32-column grad-sum blocks
# and the 8-column merge blocks
GRAD_SHAPES = [(1, 7), (2, 1), (128, 32), (129, 33), (4096, 31), (4097, 129), (32 * 4096 + 1, 8),
               (20000, 500)]


@pytest.mark.gpu
@pytest.mark.parametrize("R,J", [pytest.param(R, J, id="R%d-J%d" % (R, J))
                                 for R, J in GRAD_SHAPES])
@pytest.mark.parametrize("gamma", ["random", "zero", "negative", "none"])
def test_backward_vs_float64(zs, record_property, R, J, gamma):
    """dbeta, dgamma and da of the fp32 path in training and evaluation, ReLU on and off (y with
    exact zeros), dgamma requested and NULL (evaluation then passes no a); the planes path
    reproduces da within the fp16 lo plane, at exactly pow2_plane_scale(max |da|); the fp32
    path's amax slot is max |da| exactly."""
    lib, ptr, stream = _lib()
    gy, y, a, stats, gm = _grad_inputs(R, J, R * 3 + J, gamma)
    n_t = -(-R // BN)
    Jp = lib.load().zsb_linear_tc_kpad(J)
    r = {}
    for training, relu, want_dg in ((1, 1, True), (1, 0, False), (0, 1, True), (0, 0, False)):
        tag = "%s%s" % ("train" if training else "eval", "_relu" if relu else "")
        aa = a if (training or want_dg) else None
        part = _f32((n_t + 1) * 2 * J, fill=float("nan"))
        db, dg = _f32(J, fill=float("nan")), (_f32(J, fill=float("nan")) if want_dg else None)
        da, scale = _f32(R, J, fill=float("nan")), _f32(4)
        scale.zero_()
        lib.call("zsb_bn_grad_f32out", training, ptr(gy), ptr(y), ptr(aa), ptr(stats), ptr(gm),
                 relu, R, J, ptr(part), ptr(db), ptr(dg), ptr(da), ptr(scale), stream())
        e_db, b_db, e_dg, b_dg, e_da, b_da = grad64(gy, y, a, stats, gm, relu, training)
        r["dbeta_" + tag] = _ratio(db, e_db, b_db)
        if want_dg:
            r["dgamma_" + tag] = _ratio(dg, e_dg, b_dg)
        r["da_" + tag] = _ratio(da, e_da, b_da)
        m = float(da.abs().max())
        assert float(scale[2]) == m
        # the planes path: same da, split at the scale of its max
        part2 = _f32((n_t + 1) * 2 * J, fill=float("nan"))
        pl = torch.full((2, R, Jp), float("nan"), dtype=torch.float16, device="cuda")
        sc2 = _f32(4)
        sc2.zero_()
        lib.call("zsb_bn_grad_f32", training, ptr(gy), ptr(y), ptr(aa), ptr(stats), ptr(gm),
                 relu, R, J, ptr(part2), None, None, ptr(pl), ptr(sc2), stream())
        s0 = float(sc2[0])
        assert s0 == plane_scale(m), (s0, m)
        assert float(sc2[2]) == 0.0
        assert bool((pl[:, :, J:] == 0).all())
        back = (pl[0, :, :J].double() + pl[1, :, :J].double()) / s0
        r["planes_" + tag] = _ratio(back, da.double(),
                                    2.0 ** -22 * da.double().abs() + 2.0 ** -25 / s0 + 1e-30)
    _record(record_property, r)
    _assert_within(r)


# ---------------------------------------------------------------------------------------------
# 5. The four layers end to end against their oracles
# ---------------------------------------------------------------------------------------------
def _e2e_bounds(a64, P, coef, stats64, training, xh):
    """Bounds on xhat [R, J] and on rstd's relative error from the product's error e_a =
    coef P (P = sum |h| |W|), plus the batch moments' stage bounds (training)."""
    ea = coef * P
    if training:
        mean, var, bm, bv = population_bounds(a64)
        dmean = ea.mean(0) + bm
        dvar = 2 * ((a64 - mean).abs() * ea).mean(0) + ea.mean(0) ** 2 + bv
        drel = 0.5 * dvar / (var + EPS) + 3 * U
    else:
        dmean = torch.zeros_like(a64[0])
        drel = torch.full_like(a64[0], 3 * U)
    rs = stats64[1]
    dxh = rs * (ea + dmean) + xh.abs() * drel + 2 * U * xh.abs()
    return dxh, drel


def _e2e_compare(y, y64, dxh, gamma64, beta64):
    b = gamma64.abs() * dxh + 3 * U * (y64.abs() + beta64.abs()) + 1e-30
    return _ratio(y.reshape(y64.shape), y64, b)


def _da_bound(gg, xh, dxh, drel, gamma64, rs, training, R):
    """Bound on da [R, J] when xhat is known to within dxh and rstd to drel, on top of the
    backward's stage bound."""
    gm = gamma64.abs()
    if not training:
        return gm * rs * gg.abs() * drel
    c2 = (gg * xh).sum(0) / R
    dc2 = (gg.abs() * dxh).sum(0) / R
    da = gm * rs * (gg - gg.mean(0) - xh * c2)
    return gm * rs * (dxh * c2.abs() + xh.abs() * dc2) + da.abs() * drel


def _moments64(a64, training, mm, mv):
    if training:
        mean = a64.mean(0)
        return mean, ((a64 - mean) ** 2).mean(0)
    return mm.double(), mv.double()


# (lead, K, J, training, relu)
LINEAR_E2E = [((129,), 33, 129, True, True), ((4097,), 64, 500, True, False),
              ((2, 3000), 500, 100, True, True), ((300,), 784, 40, False, True),
              ((1,), 5, 7, True, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("lead,K,J,training,relu",
                         [pytest.param(*c, id="%s-K%d-J%d-%s%s" % (
                             "x".join(map(str, c[0])), c[1], c[2],
                             "train" if c[3] else "eval", "-relu" if c[4] else ""))
                          for c in LINEAR_E2E])
def test_bn_linear_end_to_end(zs, record_property, lead, K, J, training, relu):
    """y, the moving statistics and dh, dW, dgamma, dbeta against blvae_oracle.bn_layer;
    evaluation keeps the pre-activation for gamma's gradient."""
    g = torch.Generator(device="cuda").manual_seed(K + J)
    h = torch.randn(*lead, K, generator=g, device="cuda") + 0.5
    W = torch.randn(J, K, generator=g, device="cuda") / math.sqrt(K)
    gm, beta, mm, mv = _params(J, K, gamma="special")
    r = _layer_e2e(zs, "linear", h, W, gm, beta, mm, mv, training, relu, g)
    _record(record_property, r)
    _assert_within(r)


@pytest.mark.gpu
@pytest.mark.parametrize("training", [True, False])
def test_bn_linear_binary_end_to_end(zs, record_property, training):
    """bn_linear on a LinearBernoulli 0/1 sample (its one operand plane)."""
    g = torch.Generator(device="cuda").manual_seed(21)
    x = torch.randn(700, 30, generator=g, device="cuda")
    Wq, bq = torch.randn(64, 30, generator=g, device="cuda"), torch.randn(64, generator=g,
                                                                           device="cuda")
    z = zs.fused.LinearBernoulli(x, Wq, bq, dtype=torch.float32).sample(2)
    W = torch.randn(200, 64, generator=g, device="cuda") / 8.0
    gm, beta, mm, mv = _params(200, 64)
    r = _layer_e2e(zs, "linear", z, W, gm, beta, mm, mv, training, True, g, need_h=False)
    _record(record_property, r)
    _assert_within(r)


@pytest.mark.gpu
@pytest.mark.parametrize("training", [True, False])
def test_noisy_bn_linear_end_to_end(zs, record_property, training):
    """noisy_bn_linear against vardrop_oracle.bn_layer: h [n, K] broadcast over the particles of
    noise [S, n, K]."""
    g = torch.Generator(device="cuda").manual_seed(31)
    h = torch.randn(300, 100, generator=g, device="cuda")
    noise = 1.0 + 0.5 * torch.randn(10, 300, 100, generator=g, device="cuda")
    W = torch.randn(129, 100, generator=g, device="cuda") / 10.0
    _, beta, mm, mv = _params(129, 7)
    r = _layer_e2e(zs, "noisy", h, W, None, beta, mm, mv, training, True, g, noise=noise)
    _record(record_property, r)
    _assert_within(r)


# (N, H, k, stride, Cin, Cout, training, relu, gamma)
CONV_E2E = [(4, 14, 3, 1, 32, 64, True, True, True), (3, 7, 5, 2, 17, 33, True, False, False),
            (2, 8, 4, 2, 16, 128, False, True, True), (64, 14, 3, 1, 8, 64, True, True, True)]


@pytest.mark.gpu
@pytest.mark.parametrize("transpose", [False, True])
@pytest.mark.parametrize("N,H,k,s,Cin,Cout,training,relu,gamma",
                         [pytest.param(*c, id="N%d-H%d-k%d-s%d-%d-%d-%s%s%s" % (
                             c[:6] + ("train" if c[6] else "eval", "-relu" if c[7] else "",
                                      "" if c[8] else "-nogamma")))
                          for c in CONV_E2E])
def test_bn_conv_end_to_end(zs, record_property, transpose, N, H, k, s, Cin, Cout, training,
                            relu, gamma):
    """bn_conv2d / bn_conv2d_transpose against gan_oracle's layers: y, the Bessel-updated moving
    statistics and dx, dW, dgamma, dbeta."""
    g = torch.Generator(device="cuda").manual_seed(N * H + Cout)
    x = torch.randn(N, H, H, Cin, generator=g, device="cuda") + 0.3
    shape = (k, k, Cout, Cin) if transpose else (k, k, Cin, Cout)
    W = torch.randn(*shape, generator=g, device="cuda") / math.sqrt(k * k * Cin)
    gm, beta, mm, mv = _params(Cout, N + Cin, gamma="special")
    r = _layer_e2e(zs, "deconv" if transpose else "conv", x, W, gm if gamma else None, beta, mm,
                   mv, training, relu, g, conv=(k, s))
    _record(record_property, r)
    _assert_within(r)


def _layer_e2e(zs, kind, h, W, gm, beta, mm, mv, training, relu, g, noise=None, conv=None,
               need_h=True):
    """Runs one layer forward and backward, and its float64 oracle with the same inputs; returns
    the error-to-bound ratios of y, the moving statistics and every gradient."""
    m1, v1 = mm.clone(), mv.clone()
    th = h.detach().clone().requires_grad_(need_h) if kind != "linear" or need_h else h
    tW = W.clone().requires_grad_(True)
    tg = gm.clone().requires_grad_(True) if gm is not None else None
    tb = beta.clone().requires_grad_(True)
    if kind == "linear":
        y = zs.fused.bn_linear(th, tW, tg, tb, m1, v1, training, relu=relu)
    elif kind == "noisy":
        y = zs.fused.noisy_bn_linear(th, noise, tW, tb, m1, v1, training, relu=relu)
    elif kind == "conv":
        y = zs.fused.bn_conv2d(th, tW, tg, tb, m1, v1, training, stride=conv[1], relu=relu)
    else:
        y = zs.fused.bn_conv2d_transpose(th, tW, tg, tb, m1, v1, training, stride=conv[1],
                                         relu=relu)
    gy = torch.randn(*y.shape, generator=g, device="cuda")
    ins = ([th] if need_h else []) + [tW] + ([tg] if tg is not None else []) + [tb]
    got = torch.autograd.grad(y, ins, gy)
    # float64: the oracle and the magnitudes of its linear map
    p64 = [t.detach().double().requires_grad_(True) for t in ins]
    hd = p64[0] if need_h else h.detach().double()
    Wd = p64[1 if need_h else 0]
    gd = p64[2 if need_h else 1] if tg is not None else None
    bd = p64[-1]
    mm64, mv64 = mm.double(), mv.double()
    # the oracle without its ReLU: the gradients below take the fused output's mask, so that
    # entries within rounding of the kink are not compared across it
    if kind in ("linear", "noisy"):
        Kc = int(W.shape[1])
        coef, hcoef = fwd_bound(Kc), grad_bound(int(W.shape[0]))
        if kind == "linear":
            pre = pre_abs = lambda x, w: x @ w.t()
            y64, nm, nv = BO.bn_layer(hd, Wd, gd, bd, mm64, mv64, training, relu=False)
        else:
            nz = noise.double()
            pre = lambda x, w: (x * nz) @ w.t()
            pre_abs = lambda x, w: (x * nz.abs()) @ w.t()
            y64, nm, nv = VO.bn_layer(hd, nz, Wd, bd, mm64, mv64, training, relu=False)
            hcoef += U * int(nz.shape[0])       # dh adds the particles' rows in turn
        bessel = False
    else:
        k, s = conv
        op = GO.conv2d if kind == "conv" else GO.conv2d_transpose
        pre = pre_abs = lambda x, w: op(x, w, s)
        if kind == "conv":
            y64, nm, nv = GO.bn_conv2d(hd, Wd, gd, bd, mm64, mv64, training, s, relu=False)
            # the product over k k Cin; dx: the product over Cout, then up to k^2 taps
            coef = fwd_bound(k * k * int(W.shape[2]))
            hcoef = grad_bound(int(W.shape[3])) + k * k * U
        else:
            y64, nm, nv = GO.bn_conv2d_transpose(hd, Wd, gd, bd, mm64, mv64, training, s,
                                                 relu=False)
            # the product over Cin, then up to k^2 taps; dx: the product over k k Cout
            coef = fwd_bound(int(W.shape[3])) + k * k * U
            hcoef = grad_bound(k * k * int(W.shape[2]))
        bessel = True
    J = int(W.shape[0]) if kind in ("linear", "noisy") else int(W.shape[3 if kind == "conv" else 2])
    with torch.no_grad():
        a64 = pre(hd.detach(), Wd.detach()).reshape(-1, J)
        P = pre_abs(hd.detach().abs(), Wd.detach().abs()).reshape(-1, J)
        R = a64.shape[0]
        mean, var = _moments64(a64, training, mm, mv)
        rs = rstd64(var)
        xh = (a64 - mean) * rs
        g64 = gd.detach() if gd is not None else torch.ones_like(mean)
        dxh, drel = _e2e_bounds(a64, P, coef, torch.stack([mean, rs]), training, xh)
        y64r = y64.detach().reshape(-1, J)
        y64r = y64r.clamp_min(0) if relu else y64r
    r = {"y": _e2e_compare(y.detach(), y64r, dxh, g64, bd.detach())}
    if training:
        mean_b, var_b, bm, bv = population_bounds(a64)
        ea = coef * P
        f = R / (R - 1.0) if bessel and R > 1 else 1.0
        rate = float(np.float32(1.0 - (0.999 if kind == "noisy" else 0.99)))
        dmean = ea.mean(0) + bm
        dvar = 2 * ((a64 - mean).abs() * ea).mean(0) + ea.mean(0) ** 2 + bv
        r["mm"] = _ratio(m1, nm, rate * dmean + 3 * U * (mm64.abs() + rate * (mm64 - mean).abs()))
        r["mv"] = _ratio(v1, nv, rate * f * dvar + 3 * U * (mv64.abs() + rate * (mv64 - f * var)
                                                              .abs()))
    else:
        assert torch.equal(m1, mm) and torch.equal(v1, mv)
    # gradients: the fused y's ReLU mask, so that rows at the kink are not compared across it
    y2 = y.detach().reshape(-1, J)
    if relu:
        y64 = torch.where((y2 > 0).reshape(y64.shape), y64, torch.zeros_like(y64))
    want = torch.autograd.grad(y64, p64, gy.double())
    with torch.no_grad():
        gg = gy.double().reshape(-1, J) * ((y2 > 0).double() if relu else 1.0)
        _, b_db, _, b_dg, da, b_da = grad64(gy.reshape(-1, J), y2, a64.float(),
                                            torch.stack([mean, rs]).float(),
                                            gm if gm is not None else None, relu, training)
        b_da = b_da + _da_bound(gg, xh, dxh, drel, g64, rs, training, R)
        bounds = {}
        if tg is not None:
            bounds["dgamma"] = b_dg + (gg.abs() * dxh).sum(0)
        bounds["dbeta"] = b_db
        # the linear map's magnitudes at |da| and at its error bound, via vector-Jacobian products
        hm = hd.detach().abs().requires_grad_(True)
        Wm = Wd.detach().abs().requires_grad_(True)
    with torch.enable_grad():
        lin = pre_abs(hm, Wm).reshape(-1, J)
        vh_err, vW_err = torch.autograd.grad(lin, [hm, Wm], b_da, retain_graph=True)
        vh_mag, vW_mag = torch.autograd.grad(lin, [hm, Wm], da.abs())
    if need_h:
        bounds["h"] = vh_err + hcoef * vh_mag + 1e-30
    bounds["W"] = vW_err + wgrad_bound(R) * vW_mag + 1e-30
    names = (["h"] if need_h else []) + ["W"] + (["dgamma"] if tg is not None else []) + ["dbeta"]
    for nmx, a_, e_ in zip(names, got, want):
        r["d" + nmx if nmx in ("h", "W") else nmx] = _ratio(a_, e_.detach(), bounds[nmx])
    return r


# ---------------------------------------------------------------------------------------------
# The comparators on the CPU: each accepts a float64 reference and rejects copies perturbed as
# the mutations of a broken kernel would perturb them
# ---------------------------------------------------------------------------------------------
def _cpu_cols(R, J, seed):
    g = torch.Generator().manual_seed(seed)
    z = torch.randn(R, J, generator=g, dtype=torch.float64)
    k = torch.arange(J) % KINDS
    r = (torch.arange(R, dtype=torch.float64) / max(R - 1, 1))[:, None]
    base = [z, 10 + z, 1e3 + z, torch.full_like(z, 3.3), 1 + 1e-4 * z, 5 * r + 0.1 * z,
            3 * z - 2]
    out = torch.empty_like(z)
    for i in range(KINDS):
        out[:, k == i] = base[i][:, k == i]
    return out.float().double()


def _ref_partials(a64):
    mean, m2, _ = tile_moments(a64)
    return torch.stack([mean, m2], 1).float()


@pytest.mark.parametrize("R,J", [(129, 7), (4097, 14)])
def test_partials_comparator_rejects_mutations(R, J):
    a64 = _cpu_cols(R, J, 1)
    part = _ref_partials(a64)
    assert max(check_partials(part, a64)) <= 1.0
    # the last tile's count taken as 128
    t, m = _tiles(a64)
    bad = part.clone()
    bad[-1, 0] = (t[-1].sum(0) / BN).float()
    assert max(check_partials(bad, a64)) > 10.0
    # col2im: the same
    assert max(check_partials(part, a64, col2im=True)) <= 1.0
    assert max(check_partials(bad, a64, col2im=True)) > 10.0


@pytest.mark.parametrize("R,J", [(4096, 7), (4097, 7), (32 * 4096 + 1, 7)])
def test_merge_comparator_rejects_mutations(R, J):
    a64 = _cpu_cols(R, J, 2)
    part = _ref_partials(a64)
    mean, var, _ = merge64(part, R)
    stats = torch.stack([mean, rstd64(var)]).float()
    assert max(check_merge(stats, part, R)) <= 1.0
    assert max(check_population(stats, a64)) <= 1.0
    cnt = tile_counts(R)[:, None]
    p = part.double()

    def stats_of(mean_, m2_):
        return torch.stack([mean_, rstd64(m2_ / R)]).float()

    # a dropped tile (the shuffle tree started at 8 drops lanes 16-31)
    keep = torch.ones(p.shape[0], dtype=torch.bool)
    keep[16::32] = False
    n = cnt[keep].sum()
    mk = (cnt[keep] * p[keep, 0]).sum(0) / n
    m2k = p[keep, 1].sum(0) + (cnt[keep] * (p[keep, 0] - mk) ** 2).sum(0)
    bad = torch.stack([mk, rstd64(m2k / n)]).float()
    assert max(check_merge(bad, part, R)) > 10.0
    # the between-tile term dropped
    bad = stats_of(mean, p[:, 1].sum(0))
    assert max(check_merge(bad, part, R)) > 10.0
    assert max(check_population(bad, a64)) > 10.0
    # every tile counted as 128 rows (R off a multiple of 128 only)
    if R % BN:
        mb = (BN * p[:, 0]).sum(0) / (BN * p.shape[0])
        bad = torch.stack([mb, stats[1].double()]).float()
        assert max(check_merge(bad, part, R)) > 10.0


@pytest.mark.parametrize("R", [2, 129, 4096])
def test_moving_comparator_rejects_bessel_off_by_one(R):
    """Up to a few thousand rows; past about 2^14 rows 1 / R is below the merge's own rounding
    bound, so no comparator can see the factor there."""
    J = 7
    a64 = _cpu_cols(R, J, 3)
    mm, mv = torch.zeros(J).float(), torch.ones(J).float()
    mean, var = a64.mean(0), ((a64 - a64.mean(0)) ** 2).mean(0)
    em, ev = moving64(mm.double(), mv.double(), mean, var, R, 1.0, True)
    assert max(check_moving(em.float(), ev.float(), mm, mv, a64, 1.0, True)) <= 1.0
    # Bessel with n in place of n - 1, at rate 1; only the zero-mean columns carry a bound tight
    # enough to see R / (R - 1) at large R, so the check is on them
    bad = (var * (R / float(R))).float()
    k0 = torch.arange(J) % KINDS == 0
    assert check_moving(em.float()[k0], bad[k0], mm[k0], mv[k0], a64[:, k0], 1.0, True)[1] > 10.0


@pytest.mark.parametrize("R,J", [(129, 33), (4097, 8)])
def test_backward_comparator_rejects_mutations(R, J):
    g_ = torch.Generator().manual_seed(4)
    a = _cpu_cols(R, J, 5).float()
    s = a.double()
    mean = s.mean(0)
    stats = torch.stack([mean, rstd64(((s - mean) ** 2).mean(0))]).float()
    gy = torch.randn(R, J, generator=g_)
    y = torch.relu(torch.randn(R, J, generator=g_))
    gm = torch.randn(J, generator=g_) + 1.0
    db, b_db, dg, b_dg, da, b_da = grad64(gy, y, a, stats, gm, True, True)
    assert _ratio(db.float(), db, b_db) <= 1.0 and _ratio(da.float(), da, b_da) <= 1.0
    # the ReLU mask taken as y >= 0
    db2, _, _, _, da2, _ = grad64(gy, y + (y == 0) * 1.0, a, stats, gm, True, True)
    assert _ratio(db2.float(), db, b_db) > 10.0 and _ratio(da2.float(), da, b_da) > 10.0
    # coef from n_t 128 rows instead of R, and the xhat term dropped
    xh = (a.double() - stats.double()[0]) * stats.double()[1]
    gg = gy.double() * (y > 0)
    gs = gm.double() * stats.double()[1]
    n_t = -(-R // BN)
    bad = gs * (gg - db / (n_t * BN) - xh * dg / (n_t * BN))
    assert _ratio(bad.float(), da, b_da) > 10.0
    bad = gs * (gg - db / R)
    assert _ratio(bad.float(), da, b_da) > 10.0
    # planes: scale
    assert plane_scale(3.0) == 2.0 ** 10 and plane_scale(0.0) == 2.0 ** 12
    assert plane_scale(4.0) == 2.0 ** 9


def test_affine_comparator_rejects_a_missing_pre():
    a64 = _cpu_cols(300, 7, 6)
    stats = torch.stack([a64.mean(0), rstd64(a64.var(0, unbiased=False))]).float()
    gm, beta = torch.linspace(-1, 2, 7), torch.linspace(0.5, -0.5, 7)
    want, _ = affine64(a64, stats, gm, beta, True)
    assert check_affine(want.float(), a64, stats, gm, beta, True) <= 1.0
    bad = want.clone()
    bad[5] = 0.0                                     # a row never written
    assert check_affine(bad.float(), a64, stats, gm, beta, True) > 10.0
    # the GPU tests fill every output with NaN before the call: an entry never written must fail
    bad[5] = float("nan")
    r = {"pre": 0.5, "out": check_affine(bad.float(), a64, stats, gm, beta, True)}
    with pytest.raises(AssertionError):
        _assert_within(r)
