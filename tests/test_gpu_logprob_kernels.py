"""The distribution log-prob kernels (csrc/univariate_ext.cu and the Categorical,
UnnormalizedMultinomial, Dirichlet and MultivariateNormalCholesky row kernels of
csrc/distributions.cu) against float64 across lane counts, grid-stride passes, broadcast
patterns and the parameter values where lgamma, digamma and the log-sum-exp go wrong.

The reference is the same formula evaluated in float64 on the kernels' float32 inputs
(logprob_oracle.py).  Every bound is 4 eps32 (n + 8) times the sum of the absolute terms of the
quantity, n the length of its longest sum (the group size for grouped log-probs, the reduced
element count for broadcast gradients); the MultivariateNormalCholesky bounds come from the
componentwise error of a triangular solve instead.  Normal and Bernoulli have their own sweeps in
test_gpu_distributions.py.
"""
import numpy as np
import pytest
import torch

import logprob_oracle as O

pytestmark = pytest.mark.gpu

F32 = np.float32
EPS = O.EPS
# uni_row_kernel: 2112 blocks (ZSB_NUM_SMS * 16) of 256 threads; rows per block = 256 / lanes
GRID = 132 * 16
FAMILIES = ["fold_normal", "uniform", "gamma", "inverse_gamma", "beta", "poisson", "binomial",
            "laplace", "bin_concrete"]


@pytest.fixture(scope="module")
def zs():
    import zhusuan_b200 as zs
    return zs


def T(a, grad=False):
    t = torch.tensor(np.asarray(a, F32), device="cuda")
    return t.requires_grad_(True) if grad else t


def N(t):
    return t.detach().cpu().numpy()


# ---------------------------------------------------------------- univariate families
def _draw(fam, rng, xs, ps):
    """(x, a, b) float32 draws of shapes xs / ps inside each family's support."""
    lu = lambda lo, hi, s: np.exp(rng.uniform(np.log(lo), np.log(hi), s)).astype(F32)
    nrm = lambda s: rng.standard_normal(s).astype(F32)
    unit = lambda s: rng.uniform(0.02, 0.98, s).astype(F32)
    if fam == "fold_normal":
        return np.abs(2 * nrm(xs)), nrm(ps), (0.5 * nrm(ps)).astype(F32)
    if fam == "uniform":
        return rng.uniform(-0.9, 0.9, xs).astype(F32), (-1 - rng.random_sample(ps)).astype(F32), \
            (1 + rng.random_sample(ps)).astype(F32)
    if fam in ("gamma", "inverse_gamma"):
        return lu(0.05, 20, xs), lu(0.1, 10, ps), lu(0.1, 10, ps)
    if fam == "beta":
        return unit(xs), lu(0.1, 10, ps), lu(0.1, 10, ps)
    if fam == "poisson":
        return rng.poisson(3.0, xs).astype(F32), lu(0.1, 10, ps), None
    if fam == "binomial":
        return rng.binomial(12, 0.4, xs).astype(F32), nrm(ps), 12
    if fam == "laplace":
        return nrm(xs), nrm(ps), lu(0.3, 3, ps)
    return unit(xs), F32(0.7), nrm(ps)            # bin_concrete: the temperature is a scalar


def _dist(zs, fam, ta, tb, gnd):
    D = zs.distributions
    if fam == "fold_normal":
        return D.FoldNormal(ta, logstd=tb, group_ndims=gnd)
    if fam == "poisson":
        return D.Poisson(ta, group_ndims=gnd)
    if fam == "binomial":
        return D.Binomial(ta, int(tb), group_ndims=gnd)
    cls = dict(uniform="Uniform", gamma="Gamma", inverse_gamma="InverseGamma", beta="Beta",
               laplace="Laplace", bin_concrete="BinConcrete")[fam]
    return getattr(D, cls)(ta, tb, group_ndims=gnd)


def _check_uni(zs, fam, x, a, b, gnd, what, rng, grads=True):
    """log_prob through the public class and the gradients wrt every differentiable input,
    after the broadcast reduction, against the float64 oracle."""
    counts = fam in ("poisson", "binomial")
    tx = T(x, grad=grads and not counts)
    ta = T(a, grad=grads)
    tb = None if b is None else (b if fam == "binomial" else T(b, grad=grads))
    lp = _dist(zs, fam, ta, tb, gnd).log_prob(tx)
    full = np.broadcast_shapes(*[np.shape(v) for v in (x, a, b) if v is not None])
    X, A = np.broadcast_to(np.float64(x), full), np.broadcast_to(np.float64(a), full)
    B = None if b is None else np.broadcast_to(np.float64(b), full)
    ref = O.univariate(fam, X, A, B)
    axes = tuple(range(len(full) - gnd, len(full)))
    group = int(np.prod(full[len(full) - gnd:])) if gnd else 1
    val, terms = ref["lp"]
    O.within(N(lp), val.sum(axes), terms.sum(axes), group, what + " lp")
    if not grads:
        return
    w = rng.standard_normal(lp.shape).astype(F32)
    ins = [(n, t) for n, t in (("dx", tx), ("da", ta), ("db", tb))
           if isinstance(t, torch.Tensor) and t.requires_grad]
    got = torch.autograd.grad((lp * T(w)).sum(), [t for _, t in ins])
    W = np.broadcast_to(np.float64(w).reshape(w.shape + (1,) * gnd), full)
    digamma_in = fam in ("gamma", "inverse_gamma", "beta")
    for (name, t), g in zip(ins, got):
        v, tm = ref[name]
        m = int(np.prod(full)) // max(1, t.numel())
        n = m + (O.DIGAMMA_N if digamma_in and name != "dx" else 0)
        O.within(N(g), O.sum_to(v * W, t.shape), O.sum_to(np.abs(W) * tm, t.shape), n,
                 "%s %s" % (what, name))


@pytest.mark.parametrize("group", [1, 2, 3, 4, 7, 31, 32, 33, 64, 1000])
@pytest.mark.parametrize("fam", FAMILIES)
def test_univariate_every_lane_count(zs, fam, group):
    """uni_row_kernel picks 1 .. 32 lanes per row from the group size: each width, with a row
    count that leaves the last block part-full."""
    rng = np.random.RandomState(group * 31 + FAMILIES.index(fam))
    rows = 37
    x, a, b = _draw(fam, rng, (rows, group), (rows, group))
    _check_uni(zs, fam, x, a, b, 1, "%s group %d" % (fam, group), rng)


@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("group", [1, 64])
def test_univariate_grid_stride(zs, fam, group):
    """More rows than one pass of the capped grid covers: group 1 is 256 rows a block, groups of
    64 or more are 8 rows a block (32 lanes)."""
    rng = np.random.RandomState(7 + group + FAMILIES.index(fam))
    rows = GRID * 256 + 37 if group == 1 else GRID * 8 + 5
    x, a, b = _draw(fam, rng, (rows, group), (group,))
    _check_uni(zs, fam, x, a, b, 1, "%s %d rows of %d" % (fam, rows, group), rng)


BROADCASTS = {            # (given shape, parameter shape) against (5, 7, 6), group_ndims = 2
    "full": ((5, 7, 6), (5, 7, 6)),
    "suffix": ((5, 7, 6), (7, 6)),
    "scalar": ((5, 7, 6), ()),
    "leading_ones": ((5, 7, 6), (1, 1, 7, 6)),
    "wraps_in_row": ((5, 7, 6), (6,)),            # shorter than the 42-element group
    "materialised": ((5, 7, 6), (7, 1)),          # not a suffix: expanded by ops._prep
    "small_given": ((7, 6), (5, 7, 6)),
}


@pytest.mark.parametrize("pattern", sorted(BROADCASTS))
@pytest.mark.parametrize("fam", FAMILIES)
def test_univariate_broadcasts(zs, fam, pattern):
    xs, ps = BROADCASTS[pattern]
    rng = np.random.RandomState(len(pattern) * 13 + FAMILIES.index(fam))
    x, a, b = _draw(fam, rng, xs, ps)
    for gnd in (0, 2):
        _check_uni(zs, fam, x, a, b, gnd, "%s %s gnd %d" % (fam, pattern, gnd), rng)


def _grid(*axes):
    """float32 arrays of every combination of the given 1-D value lists."""
    return [np.asarray(v, F32) for v in np.meshgrid(*axes, indexing="ij")]


def test_gamma_and_inverse_gamma_parameter_edges(zs):
    rng = np.random.RandomState(11)
    x, a, b = _grid(np.logspace(-3, 3, 5), np.logspace(-3, 4, 8), np.logspace(-3, 4, 8))
    for fam in ("gamma", "inverse_gamma"):
        _check_uni(zs, fam, x, a, b, 0, fam + " edges", rng)
        _check_uni(zs, fam, x, a, b, 3, fam + " edges summed", rng)


def test_beta_and_bin_concrete_at_the_ends_of_the_unit_interval(zs):
    rng = np.random.RandomState(12)
    top = np.nextafter(F32(1), F32(0))
    xs = np.array([1e-6, 1e-3, 0.5, 0.999, top], F32)
    x, a, b = _grid(xs, np.logspace(-3, 3, 7), np.logspace(-3, 3, 7))
    _check_uni(zs, "beta", x, a, b, 0, "beta ends", rng)
    xl, logits = _grid(xs, [-30, -3, 0, 3, 30])
    for temp in (0.1, 0.7, 5.0):
        _check_uni(zs, "bin_concrete", xl, F32(temp), logits, 0, "bin_concrete T=%g" % temp, rng)


def test_poisson_large_counts_and_rates(zs):
    rng = np.random.RandomState(13)
    x, a = _grid([0, 1, 2, 10, 99, 1000, 5000, 10000], np.logspace(-3, 4, 15))
    _check_uni(zs, "poisson", x, a, None, 0, "poisson", rng)
    _check_uni(zs, "poisson", x, a, None, 1, "poisson summed", rng)


def test_binomial_counts_at_zero_and_n_and_saturated_logits(zs):
    rng = np.random.RandomState(14)
    for n in (1, 7, 10000):
        ks = sorted({0, 1, n // 2, n - 1, n})
        x, a = _grid(ks, [-30, -5, -1, 0, 1, 5, 30])
        _check_uni(zs, "binomial", x, a, n, 0, "binomial n=%d" % n, rng)


def test_laplace_gradient_at_the_location_is_zero(zs):
    """d|x - loc| at x == loc is 0, as TF's sign(0) gives."""
    rng = np.random.RandomState(15)
    loc = rng.standard_normal((4, 9)).astype(F32)
    x = loc.copy()
    x[:, ::2] += rng.standard_normal((4, 5)).astype(F32)
    scale = np.exp(rng.uniform(-3, 3, (4, 9))).astype(F32)
    _check_uni(zs, "laplace", x, loc, scale, 0, "laplace", rng)
    tx, tl = T(x, grad=True), T(loc, grad=True)
    lp = zs.distributions.Laplace(tl, T(scale)).log_prob(tx)
    gx, gl = torch.autograd.grad(lp.sum(), [tx, tl])
    at = x == loc
    assert at.sum() >= 16
    assert np.all(N(gx)[at] == 0) and np.all(N(gl)[at] == 0)


def test_uniform_outside_the_support(zs):
    """-inf log-prob outside [minval, maxval) and NaN parameter gradients: d log(mask / (b - a))
    is 0 / 0 there, as TF's tf.gradients gives."""
    rng = np.random.RandomState(16)
    lo = np.full((3, 8), -1, F32)
    hi = np.full((3, 8), 2, F32)
    x = np.tile(np.array([-1.5, -1.0, -0.999, 0.0, 1.999, 2.0, 2.5, 1e30], F32), (3, 1))
    _check_uni(zs, "uniform", x, lo, hi, 0, "uniform", rng)
    tl, th = T(lo, grad=True), T(hi, grad=True)
    lp = zs.distributions.Uniform(tl, th).log_prob(T(x))
    out = (x < lo) | (x >= hi)
    assert np.all(np.isneginf(N(lp)[out])) and np.all(np.isfinite(N(lp)[~out]))
    gl, gh = torch.autograd.grad(lp.sum(), [tl, th])
    assert np.all(np.isnan(N(gl)[out])) and np.all(np.isnan(N(gh)[out]))
    assert np.all(np.isfinite(N(gl)[~out])) and np.all(np.isfinite(N(gh)[~out]))


def test_fold_normal_below_zero(zs):
    rng = np.random.RandomState(17)
    x = rng.standard_normal((6, 10)).astype(F32) * 2
    mean = rng.standard_normal((6, 10)).astype(F32)
    logstd = (0.5 * rng.standard_normal((6, 10))).astype(F32)
    _check_uni(zs, "fold_normal", x, mean, logstd, 0, "fold_normal", rng)
    _check_uni(zs, "fold_normal", x, mean, logstd, 1, "fold_normal summed", rng)
    lp = zs.distributions.FoldNormal(T(mean), logstd=T(logstd)).log_prob(T(x))
    assert np.all(np.isneginf(N(lp)[x < 0])) and np.all(np.isfinite(N(lp)[x >= 0]))


# ---------------------------------------------------------------- digamma
def _digamma_via_gamma(zs, alpha):
    """Gamma(alpha, 1) at given = 1: d lp / d alpha = log 1 - psi(alpha) + log 1 = -psi(alpha)."""
    ta = T(alpha, grad=True)
    one = T(np.ones_like(alpha))
    lp = zs.distributions.Gamma(ta, one).log_prob(one)
    g, = torch.autograd.grad(lp.sum(), [ta])
    torch.cuda.synchronize()
    return -N(g)


def test_digamma_against_float64(zs):
    alpha = np.concatenate([np.logspace(-6, 6, 97), [5.999999, 6.0, 6.000001],
                            [-0.5, -3.7, -1000.5, -0.25, -7.9]]).astype(F32)
    got = _digamma_via_gamma(zs, alpha)
    want = torch.special.digamma(torch.tensor(alpha, dtype=torch.float64)).numpy()
    _, terms = O.digamma(alpha)
    O.within(got, want, terms, O.DIGAMMA_N, "digamma")


def test_digamma_returns_at_poles_and_infinities(zs):
    """0, the negative integers, -2^25 and -1e30 (where x + 1 == x in float32), -inf and NaN: the
    call returns and the result is non-finite wherever float64 digamma is."""
    from zhusuan_b200._lib import lib
    # the parent kernel's recurrence never ends at -2^25 or -inf: never run this against it
    if lib.load().zsb_version() < 102:
        pytest.skip("digamma recurrence of this library version is unbounded for x <= -2^24")
    alpha = np.array([0.0, -0.0, -1, -2, -7, -2.0 ** 25, -1e30, -np.inf, np.nan, np.inf], F32)
    want = torch.special.digamma(torch.tensor(alpha, dtype=torch.float64)).numpy()
    assert not np.isfinite(want).any()
    got = _digamma_via_gamma(zs, alpha)
    assert not np.isfinite(got).any(), got
    assert got[-1] == np.inf            # psi(+inf) = +inf
    # the other callers: InverseGamma alpha (its beta gradient has no digamma), Beta alpha and beta
    ta = T(alpha, grad=True)
    lp = zs.distributions.InverseGamma(ta, T(np.ones_like(alpha))).log_prob(T(np.ones_like(alpha)))
    ga, = torch.autograd.grad(lp.sum(), [ta])
    torch.cuda.synchronize()
    assert not np.isfinite(N(ga)).any()
    ta, tb = T(alpha, grad=True), T(alpha, grad=True)
    lp = zs.distributions.Beta(ta, tb).log_prob(T(np.full_like(alpha, 0.5)))
    ga, gb = torch.autograd.grad(lp.sum(), [ta, tb])
    torch.cuda.synchronize()
    assert not np.isfinite(N(ga)).any() and not np.isfinite(N(gb)).any()


# ---------------------------------------------------------------- Categorical
def _check_categorical(zs, k, l, gnd, what, rng, shared_logits_rows=None):
    tl = T(l, grad=True)
    lp = zs.distributions.Categorical(tl, group_ndims=gnd).log_prob(
        torch.tensor(k, dtype=torch.int32, device="cuda"))
    bshape = np.broadcast_shapes(k.shape, l.shape[:-1])
    L = np.broadcast_to(np.float64(l), bshape + l.shape[-1:])
    K = np.broadcast_to(k, bshape)
    v, vt, g, gt = O.categorical(K, L)
    C = l.shape[-1]
    axes = tuple(range(len(bshape) - gnd, len(bshape)))
    grp = int(np.prod(bshape[len(bshape) - gnd:])) if gnd else 1
    O.within(N(lp), v.sum(axes), vt.sum(axes), C + grp, what + " lp")
    w = rng.standard_normal(lp.shape).astype(F32)
    got, = torch.autograd.grad((lp * T(w)).sum(), [tl])
    W = np.broadcast_to(np.float64(w).reshape(w.shape + (1,) * gnd), bshape)[..., None]
    m = int(np.prod(bshape)) // max(1, int(np.prod(l.shape[:-1])))
    O.within(N(got), O.sum_to(g * W, l.shape), O.sum_to(np.abs(W) * gt, l.shape), C + m,
             what + " dlogits")


@pytest.mark.parametrize("C", [1, 2, 31, 32, 33, 1000, 10000])
def test_categorical_category_counts(zs, C):
    rng = np.random.RandomState(C)
    rows = 48 if C >= 1000 else 300
    l = (3 * rng.standard_normal((rows, C))).astype(F32)
    k = rng.randint(0, C, rows).astype(np.int32)
    _check_categorical(zs, k, l, 0, "C=%d" % C, rng)


def test_categorical_grid_stride_rows(zs):
    rng = np.random.RandomState(21)
    rows = GRID * 8 + 5
    l = (2 * rng.standard_normal((rows, 10))).astype(F32)
    _check_categorical(zs, rng.randint(0, 10, rows).astype(np.int32), l, 0, "rows", rng)


def test_categorical_extreme_logits(zs):
    """Logits of magnitude 1e3 (the log-sum-exp must subtract the max) and -inf on categories
    that are not chosen."""
    rng = np.random.RandomState(22)
    l = (1e3 * rng.standard_normal((64, 40))).astype(F32)
    k = rng.randint(0, 40, 64).astype(np.int32)
    _check_categorical(zs, k, l, 0, "1e3 logits", rng)
    l2 = rng.standard_normal((64, 40)).astype(F32)
    drop = rng.random_sample((64, 40)) < 0.5
    drop[np.arange(64), k] = False
    l2[drop] = -np.inf
    _check_categorical(zs, k, l2, 0, "-inf logits", rng)


@pytest.mark.parametrize("gnd", [0, 1, 2])
def test_categorical_shared_operands_and_groups(zs, gnd):
    rng = np.random.RandomState(23 + gnd)
    l = rng.standard_normal((6, 9, 35)).astype(F32)
    k_shared = rng.randint(0, 35, (6, 9)).astype(np.int32)
    _check_categorical(zs, np.broadcast_to(k_shared, (4, 6, 9)).copy(), l, gnd,
                       "logits shared gnd %d" % gnd, rng)
    l4 = rng.standard_normal((4, 6, 9, 35)).astype(F32)
    _check_categorical(zs, k_shared, l4, gnd, "given shared gnd %d" % gnd, rng)


def test_categorical_out_of_range_class_gives_a_nan_row(zs):
    """-1 and C give a NaN log-prob and a NaN gradient row, as the reference's
    sparse_softmax_cross_entropy_with_logits does on a GPU; the other rows are untouched."""
    rng = np.random.RandomState(24)
    C = 45
    l = rng.standard_normal((6, C)).astype(F32)
    k = rng.randint(0, C, 6).astype(np.int32)
    k[1], k[4] = -1, C
    tl = T(l, grad=True)
    lp = zs.distributions.Categorical(tl).log_prob(torch.tensor(k, device="cuda"))
    g, = torch.autograd.grad(lp.sum(), [tl])
    bad = np.array([False, True, False, False, True, False])
    assert np.isnan(N(lp)[bad]).all() and np.isfinite(N(lp)[~bad]).all()
    assert np.isnan(N(g)[bad]).all() and np.isfinite(N(g)[~bad]).all()
    _check_categorical(zs, k[~bad], l[~bad], 0, "in range", rng)


# ---------------------------------------------------------------- UnnormalizedMultinomial
def _check_multinomial(zs, x, l, normalize, what, rng):
    tl = T(l, grad=True)
    lp = zs.distributions.UnnormalizedMultinomial(tl, normalize_logits=normalize).log_prob(
        torch.tensor(x, dtype=torch.int32, device="cuda"))
    full = np.broadcast_shapes(x.shape, l.shape)
    X = np.broadcast_to(np.float64(x), full)
    L = np.broadcast_to(np.float64(l), full)
    V = full[-1]
    if normalize:
        lse, p, lt = O.lse_rows(L)
    else:
        lse, p, lt = np.zeros(full[:-1] + (1,)), np.zeros(full), np.zeros(full[:-1] + (1,))
    sx = X.sum(-1, keepdims=True)
    want = (X * (L - lse)).sum(-1)
    terms = (X * (np.abs(L) + np.abs(lse))).sum(-1) + (sx * lt)[..., 0]
    O.within(N(lp), want, terms, V, what + " lp")
    w = rng.standard_normal(lp.shape).astype(F32)
    got, = torch.autograd.grad((lp * T(w)).sum(), [tl])
    W = np.float64(w)[..., None]
    g = X - sx * p
    gt = X + sx * p * (np.abs(L) + np.abs(lse) + lt)
    m = int(np.prod(full)) // l.size
    O.within(N(got), O.sum_to(g * W, l.shape), O.sum_to(np.abs(W) * gt, l.shape), V + m,
             what + " dlogits")


@pytest.mark.parametrize("normalize", [True, False])
@pytest.mark.parametrize("V", [7, 33, 1000, 10000])
def test_unnormalized_multinomial(zs, V, normalize):
    rng = np.random.RandomState(V + normalize)
    docs = 6 if V >= 1000 else 40
    x = rng.poisson(rng.choice([0.1, 3.0, 300.0], (docs, 1)), (docs, V)).clip(0, 1000)
    x = x.astype(np.int32)
    x[0, :5] = 1000
    l = (2 * rng.standard_normal((3, docs, V))).astype(F32)      # [chains, docs, V]: LNTM shape
    _check_multinomial(zs, x, l, normalize, "V=%d norm=%d" % (V, normalize), rng)
    _check_multinomial(zs, x, l[0], normalize, "V=%d unshared" % V, rng)


# ---------------------------------------------------------------- Dirichlet
def _check_dirichlet(zs, x, a, what, rng):
    tx, ta = T(x, grad=True), T(a, grad=True)
    lp = zs.distributions.Dirichlet(ta).log_prob(tx)
    full = np.broadcast_shapes(x.shape, a.shape)
    X = np.broadcast_to(np.float64(x), full)
    A = np.broadcast_to(np.float64(a), full)
    C = full[-1]
    lg, lgt = O.lgamma(A)
    sa = A.sum(-1)
    ls, lst = O.lgamma(sa, rounded=True)
    with np.errstate(all="ignore"):
        xl = (A - 1) * np.log(X)
        want = -(lg.sum(-1) - ls) + xl.sum(-1)
        O.within(N(lp), want, lgt.sum(-1) + lst + np.abs(xl).sum(-1), C, what + " lp")
        w = rng.uniform(0.5, 1.5, lp.shape).astype(F32)
        gx, ga = torch.autograd.grad((lp * T(w)).sum(), [tx, ta])
        W = np.float64(w)[..., None]
        dx = (A - 1) / X
        mx = int(np.prod(full)) // x.size
        O.within(N(gx), O.sum_to(dx * W, x.shape), O.sum_to(np.abs(W * dx), x.shape), mx,
                 what + " dgiven")
        pa, pat = O.digamma(A)
        ps, pst = O.digamma(sa[..., None])
        da = ps - pa + np.log(X)
        ma = int(np.prod(full)) // a.size
        O.within(N(ga), O.sum_to(da * W, a.shape),
                 O.sum_to(np.abs(W) * (pst + pat + np.abs(np.log(X))), a.shape),
                 ma + C + O.DIGAMMA_N, what + " dalpha")


@pytest.mark.parametrize("C", [2, 3, 33, 1000])
def test_dirichlet(zs, C):
    rng = np.random.RandomState(30 + C)
    rows = 8 if C == 1000 else 40
    a = np.exp(rng.uniform(np.log(1e-3), np.log(1e3), (rows, C))).astype(F32)
    x = rng.dirichlet(np.full(C, 2.0), (5, rows)).astype(F32)
    _check_dirichlet(zs, x, a, "C=%d" % C, rng)                   # alpha shared across samples
    _check_dirichlet(zs, x[0], a[0], "C=%d alpha row" % C, rng)   # alpha shared across rows


def test_dirichlet_near_the_corners(zs):
    rng = np.random.RandomState(35)
    C = 4
    x = []
    for d in (1e-6, 1e-4, 1e-2):
        for c in range(C):
            r = np.full(C, d)
            r[c] = 1 - (C - 1) * d
            x.append(r)
    x = np.array(x, F32)
    a = np.exp(rng.uniform(np.log(1e-3), np.log(1e3), x.shape)).astype(F32)
    _check_dirichlet(zs, x, a, "corners", rng)


def test_dirichlet_zero_coordinate_with_unit_alpha_is_nan(zs):
    """x_j = 0 with alpha_j = 1: (alpha - 1) * log(given) is 0 * -inf = NaN, as in the
    reference; d lp / d x_j = 0 / 0."""
    rng = np.random.RandomState(36)
    x = np.array([[0.0, 0.4, 0.6], [0.3, 0.3, 0.4]], F32)
    a = np.array([[1.0, 2.0, 3.0], [1.0, 2.0, 3.0]], F32)
    tx, ta = T(x, grad=True), T(a, grad=True)
    lp = zs.distributions.Dirichlet(ta).log_prob(tx)
    gx, = torch.autograd.grad(lp.sum(), [tx])
    np.testing.assert_equal(np.isnan(N(lp)), [True, False])
    assert np.isnan(N(gx)[0, 0]) and np.isfinite(N(gx)[1]).all()
    _check_dirichlet(zs, x, a, "zero coordinate", rng)


# ---------------------------------------------------------------- MultivariateNormalCholesky
def _tril(rng, D, mats, cond=None):
    """float32 Cholesky factors of well-conditioned covariances, or with cond(L) ~ ``cond``."""
    out = []
    for _ in range(mats):
        Q, _ = np.linalg.qr(rng.standard_normal((D, D)))
        ev = np.logspace(0, -2 * np.log10(cond), D) if cond else rng.uniform(0.5, 2.0, D)
        out.append(np.linalg.cholesky((Q * ev) @ Q.T + 1e-12 * np.eye(D)))
    return np.array(out, F32)


def _check_mvn(zs, x, mu, L, what, rng, via_class=True):
    """lp and the gradients wrt given, mean and cov_tril.  Bounds: forward substitution gives
    (L + dL) y^ = b with |dL| <= gamma_D |L| (Higham, Thm 8.5), so |y^ - y| <= gamma_D |L^-1|
    (|L| |y| + |b|) (the |b| for rounding given - mean); back substitution adds the same for
    z = L^-T y, on top of |L^-T| |y^ - y|; products and the D-term sums add eps (D + 8)."""
    D = mu.shape[-1]
    tx, tm, tL = T(x, grad=True), T(mu, grad=True), T(L, grad=True)
    if via_class:
        lp = zs.distributions.MultivariateNormalCholesky(tm, tL).log_prob(tx)
    else:
        from zhusuan_b200 import ops
        lp = ops.mvn_cholesky_log_prob(tx, tm, tL)
    bshape = np.broadcast_shapes(x.shape[:-1], mu.shape[:-1], L.shape[:-2])
    X = np.broadcast_to(np.float64(x), bshape + (D,))
    M = np.broadcast_to(np.float64(mu), bshape + (D,))
    L64 = np.float64(L)
    Li = np.linalg.inv(L64)
    Lb = np.broadcast_to(L64, bshape + (D, D))
    Lib = np.broadcast_to(Li, bshape + (D, D))
    gam = D * EPS / (1 - D * EPS)
    b = X - M
    y = np.einsum("...ij,...j->...i", Lib, b)                     # L^-1 (given - mean)
    z = np.einsum("...ji,...j->...i", Lib, y)                     # L^-T y
    aLi, aL = np.abs(Lib), np.abs(Lb)
    ey = gam * np.einsum("...ij,...j->...i", aLi, np.einsum("...ij,...j->...i", aL, np.abs(y))
                         + np.abs(b))
    ez = np.einsum("...ji,...j->...i", aLi, ey) + gam * np.einsum(
        "...ji,...j->...i", aLi, np.einsum("...ji,...j->...i", aL, np.abs(z)))
    ldiag = np.log(np.diagonal(Lb, axis1=-2, axis2=-1))
    want = -D * O.HALF_LOG_2PI - ldiag.sum(-1) - 0.5 * (y * y).sum(-1)
    tol = 4 * ((np.abs(y) * ey).sum(-1) + EPS * (D + 8) * (
        D * O.HALF_LOG_2PI + np.abs(ldiag).sum(-1) + 0.5 * (y * y).sum(-1)))
    err = np.abs(N(lp) - want)
    assert (err <= tol).all(), "%s lp: max err/tol %.3g" % (what, (err / tol).max())
    w = rng.standard_normal(lp.shape).astype(F32)
    gx, gm, gL = torch.autograd.grad((lp * T(w)).sum(), [tx, tm, tL])
    W = np.float64(w)[..., None]
    # d lp / d given = -z, d lp / d mean = z, d lp / d L = tril(z y^T) - diag(1 / L_ii)
    for name, got, sign, shape in (("dgiven", gx, -1, x.shape), ("dmean", gm, 1, mu.shape)):
        m = int(np.prod(bshape)) // max(1, int(np.prod(shape[:-1])))
        ref = O.sum_to(sign * z * W, shape)
        tol = 4 * (O.sum_to(np.abs(W) * ez, shape)
                   + EPS * (m + 8) * O.sum_to(np.abs(W * z), shape))
        err = np.abs(N(got) - ref)
        assert (err <= tol).all(), "%s %s: max err/tol %.3g" % (what, name, (err / tol).max())
    Wm = W[..., None]
    idiag = np.eye(D) / np.diagonal(Lb, axis1=-2, axis2=-1)[..., None]
    full = np.tril(z[..., :, None] * y[..., None, :]) - idiag
    efull = np.tril(ez[..., :, None] * np.abs(y)[..., None, :]
                    + np.abs(z)[..., :, None] * ey[..., None, :])
    m = int(np.prod(bshape)) // max(1, int(np.prod(L.shape[:-2])))
    ref = O.sum_to(full * Wm, L.shape)
    tol = 4 * (O.sum_to(np.abs(Wm) * efull, L.shape) + EPS * (m + 8) * O.sum_to(
        np.abs(Wm) * (np.abs(np.tril(z[..., :, None] * y[..., None, :])) + np.abs(idiag)),
        L.shape))
    gL = N(gL)
    err = np.abs(gL - ref)
    assert (err <= tol).all(), "%s dtril: max err/tol %.3g" % (what, (err / tol).max())
    assert np.all(np.triu(gL, 1) == 0), what + ": upper triangle of dtril is not zero"


@pytest.mark.parametrize("D", [1, 2, 127, 128, 129, 512, 2000])
def test_mvn_cholesky_dimensions(zs, D):
    """Across the 128-thread block and the shared-memory forward / back substitution; at
    D = 2000 one L serves every row (one L per row would be 17 GB at realistic row counts)."""
    rng = np.random.RandomState(D)
    rows = 3 if D == 2000 else 6
    L = _tril(rng, D, 1 if D == 2000 else rows)
    mu = rng.standard_normal((rows, D)).astype(F32)
    x = (mu + rng.standard_normal((rows, D))).astype(F32)
    if D == 2000:
        _check_mvn(zs, x, mu, L[0], "D=%d" % D, rng, via_class=False)
    else:
        _check_mvn(zs, x, mu, L, "D=%d" % D, rng)


def test_mvn_cholesky_grid_stride_rows(zs):
    """More rows than the 1056-block grid (ZSB_NUM_SMS * 8), one factor per row."""
    rng = np.random.RandomState(40)
    rows, D = 132 * 8 + 13, 64
    L = _tril(rng, D, rows)
    mu = rng.standard_normal((rows, D)).astype(F32)
    x = (mu + rng.standard_normal((rows, D))).astype(F32)
    _check_mvn(zs, x, mu, L, "rows", rng)


def test_mvn_cholesky_ill_conditioned_factor(zs):
    rng = np.random.RandomState(41)
    D = 48
    L = _tril(rng, D, 3, cond=1e4)
    assert 3e3 < np.linalg.cond(np.float64(L[0])) < 3e4
    mu = rng.standard_normal((3, D)).astype(F32)
    x = (mu + rng.standard_normal((5, 3, D))).astype(F32)
    _check_mvn(zs, x, mu, L, "cond 1e4", rng)


@pytest.mark.parametrize("pattern", ["tril_shared", "mean_shared", "given_shared",
                                     "tril_materialised"])
def test_mvn_cholesky_broadcasts(zs, pattern):
    rng = np.random.RandomState(len(pattern))
    D = 33
    xs, ms, Ls = {"tril_shared": ((3, 5), (3, 5), ()),
                  "mean_shared": ((3, 5), (), (5,)),
                  "given_shared": ((5,), (3, 5), (3, 5)),
                  "tril_materialised": ((3, 5), (3, 5), (3, 1))}[pattern]
    nL = int(np.prod(Ls)) if Ls else 1
    L = _tril(rng, D, nL).reshape(Ls + (D, D))
    mu = rng.standard_normal(ms + (D,)).astype(F32)
    x = (rng.standard_normal(xs + (D,)) * 1.5).astype(F32)
    _check_mvn(zs, x, mu, L, pattern, rng, via_class=False)
