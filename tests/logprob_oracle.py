"""Float64 restatement of the distribution log-prob kernels (csrc/univariate_ext.cu,
csrc/distributions.cu) on the kernels' own float32 inputs, with the rounding terms each quantity
is bounded by.

Every function returns values together with ``terms``: the sum of the absolute values of the
additive components of the quantity, evaluated in float64.  A float32 evaluation of the same
formula is then within ``4 eps32 (n + 8) terms`` of the float64 value, ``n`` being the length of
the longest sum (Higham, Accuracy and Stability of Numerical Algorithms, 3.1-3.4).  Cancellation
already in the formula is not held against the kernel; a wrong special function or index is.

Besides the components themselves, a component f(u) of an intermediate u that the kernel rounds
(1 - x, a + b, x + 1) gets the extra term |u f'(u)|: the error one rounding of u moves it by.
"""
import numpy as np
from scipy import special

EPS = float(np.finfo(np.float32).eps)
TINY = float(np.finfo(np.float32).tiny)
HALF_LOG_2PI = 0.5 * np.log(2 * np.pi)


def within(got, want, terms, n, what):
    """|got - want| <= 4 eps32 (n + 8) terms elementwise.  Where ``want`` is not finite, ``got``
    must be the same non-finite value (NaN, +inf or -inf)."""
    got = np.asarray(got, np.float64)
    want = np.asarray(want, np.float64)
    terms = np.broadcast_to(np.asarray(terms, np.float64), want.shape)
    assert got.shape == want.shape, "%s: shape %s != %s" % (what, got.shape, want.shape)
    fin = np.isfinite(want)
    nf = ~fin
    if nf.any():
        g, w = got[nf], want[nf]
        same = (np.isnan(g) & np.isnan(w)) | (g == w)
        assert same.all(), "%s: %d non-finite reference values differ, first %r vs %r" % (
            what, int((~same).sum()), g[~same][0], w[~same][0])
    # + TINY: float32 cannot hold a result below 2^-126 to full relative precision (a softmax
    # entry of 1e-297 comes out as 0)
    tol = 4.0 * EPS * (n + 8) * terms[fin] + TINY
    err = np.abs(got[fin] - want[fin])
    bad = ~(err <= tol)
    if bad.any():
        i = int(np.argmax(np.where(bad, err / np.maximum(tol, 1e-300), 0)))
        raise AssertionError("%s: %d of %d values outside the rounding bound; worst got %r want "
                             "%r err %.3g tol %.3g" % (what, int(bad.sum()), bad.size,
                                                       got[fin][i], want[fin][i], err[i], tol[i]))


def sum_to(a, shape):
    """The broadcast reduction of autograd: sum ``a`` down to ``shape``."""
    shape = tuple(shape)
    while a.ndim > len(shape):
        a = a.sum(0)
    for ax, s in enumerate(shape):
        if s == 1 and a.shape[ax] != 1:
            a = a.sum(ax, keepdims=True)
    return a


def digamma(x):
    """(psi(x), terms) in the kernel's evaluation order: reflection psi(x) = psi(1 - x) -
    pi cot(pi x) for x <= 0, the recurrence up to 6, then log x - 1/(2x) - series."""
    x = np.asarray(x, np.float64)
    val = special.psi(x)
    terms = np.zeros_like(x)
    with np.errstate(all="ignore"):
        neg = x <= 0
        y = np.where(neg, 1.0 - x, x)
        refl = np.where(neg, np.pi / np.tan(np.pi * x), 0.0)
        # 1 - x is rounded: |y psi'(y)|
        terms += np.where(neg, np.abs(refl) + np.abs(y * special.polygamma(1, np.where(neg, y, 1.0))),
                          0.0)
        for _ in range(6):
            step = y < 6
            terms += np.where(step, 1.0 / np.abs(y), 0.0)
            y = np.where(step, y + 1, y)
        i = 1.0 / y
        terms += np.abs(np.log(y)) + 0.5 * i + i * i / 12
    return val, terms


DIGAMMA_N = 12          # 6 recurrence steps + log, 1/(2x) and the 3-term series


def lgamma(u, rounded=False):
    """(lgamma(u), terms); ``rounded``: u is a kernel-side sum (adds |u psi(u)|).

    No absolute floor under |lgamma(u)| near the roots 1 and 2: on an H100 (80GB HBM3, 700 W)
    -lgammaf(a) - 1 from the Gamma kernel at every float32 a in [0.9, 1.1] and [1.9, 2.1] was
    within 0.56 eps32 of float64, which is the rounding of the "- 1" itself."""
    u = np.asarray(u, np.float64)
    val = special.gammaln(u)
    terms = np.abs(val)
    if rounded:
        with np.errstate(all="ignore"):
            terms = terms + np.abs(u * special.psi(u))
    return val, terms


def softplus(t):
    return np.logaddexp(0.0, t)


def sigmoid(t):
    return special.expit(t)


def univariate(fam, x, a, b):
    """Elementwise log density and its gradients of one UNI_* family at broadcast float64 x, a,
    b.  Returns {"lp": (val, terms), "dx": ..., "da": ..., "db": ...} (absent entries are
    gradients the family does not have)."""
    x, a = np.asarray(x, np.float64), np.asarray(a, np.float64)
    b = None if b is None else np.asarray(b, np.float64)
    A = np.abs
    out = {}
    with np.errstate(all="ignore"):
        if fam == "fold_normal":                        # a = mean, b = logstd
            prec, d = np.exp(-2 * b), x - a
            t = -2 * a * x * prec
            s = sigmoid(t)
            mask = np.where(x >= 0, 0.0, -np.inf)
            out["lp"] = (-HALF_LOG_2PI - (b + 0.5 * prec * d * d) + softplus(t) + mask,
                         HALF_LOG_2PI + A(b) + A(0.5 * prec * d * d) + softplus(t) + s * A(t))
            # an error in t moves s by s (1 - s) |t| eps
            ds = s * (1 + (1 - s) * A(t))
            out["dx"] = (-prec * d + s * (-2 * a * prec), A(prec * d) + ds * A(2 * a * prec))
            out["da"] = (prec * d + s * (-2 * x * prec), A(prec * d) + ds * A(2 * x * prec))
            out["db"] = (-1 + prec * d * d - 2 * s * t, 1 + A(prec * d * d) + 2 * ds * A(t))
        elif fam == "uniform":                          # a = minval, b = maxval
            inside = (a <= x) & (x < b)
            nan = np.full(np.broadcast(x, a, b).shape, np.nan)
            w = b - a
            # b - a and 1 / (b - a) are rounded: 2 more terms of size 1 under the log
            out["lp"] = (np.where(inside, -np.log(w), -np.inf), A(np.log(w)) + 2)
            out["dx"] = (np.zeros(nan.shape), np.zeros(nan.shape))
            out["da"] = (np.where(inside, 1 / w, nan), A(1 / w))
            out["db"] = (np.where(inside, -1 / w, nan), A(1 / w))
        elif fam in ("gamma", "inverse_gamma"):         # a = alpha, b = beta
            lg, lgt = lgamma(a)
            ps, pst = digamma(a)
            lb, lx = np.log(b), np.log(x)
            if fam == "gamma":
                out["lp"] = (a * lb - lg + (a - 1) * lx - b * x,
                             A(a * lb) + lgt + A((a - 1) * lx) + A(b * x))
                out["dx"] = ((a - 1) / x - b, A((a - 1) / x) + A(b))
                out["da"] = (lb - ps + lx, A(lb) + pst + A(lx))
                out["db"] = (a / b - x, A(a / b) + A(x))
            else:
                out["lp"] = (a * lb - lg - (a + 1) * lx - b / x,
                             A(a * lb) + lgt + A((a + 1) * lx) + A(b / x))
                out["dx"] = (-(a + 1) / x + b / (x * x), A((a + 1) / x) + A(b / (x * x)))
                out["da"] = (lb - ps - lx, A(lb) + pst + A(lx))
                out["db"] = (a / b - 1 / x, A(a / b) + A(1 / x))
        elif fam == "beta":
            lx, l1x = np.log(x), np.log1p(-x)
            la, lat = lgamma(a)
            lb, lbt = lgamma(b)
            lab, labt = lgamma(a + b, rounded=True)
            pa, pat = digamma(a)
            pb, pbt = digamma(b)
            pab, pabt = digamma(a + b)
            # 1 - x is rounded: + |b - 1| under log(1 - x), + 1 in d/db
            out["lp"] = ((a - 1) * lx + (b - 1) * l1x - (la + lb - lab),
                         A((a - 1) * lx) + A((b - 1) * l1x) + A(b - 1) + lat + lbt + labt)
            out["dx"] = ((a - 1) / x - (b - 1) / (1 - x), A((a - 1) / x) + A((b - 1) / (1 - x)))
            # a + b is rounded: |s psi'(s)| <= the recurrence's 1/s + 1-ish, covered by pabt
            out["da"] = (lx - pa + pab, A(lx) + pat + pabt)
            out["db"] = (l1x - pb + pab, A(l1x) + 1 + pbt + pabt)
        elif fam == "poisson":                          # a = rate
            lg, lgt = lgamma(x + 1, rounded=True)
            out["lp"] = (x * np.log(a) - a - lg, A(x * np.log(a)) + A(a) + lgt)
            out["da"] = (x / a - 1, A(x / a) + 1)
        elif fam == "binomial":                         # a = logits, b = n
            l1, t1 = lgamma(b + 1, rounded=True)
            l2, t2 = lgamma(b - x + 1, rounded=True)
            l3, t3 = lgamma(x + 1, rounded=True)
            sp = softplus(a)
            out["lp"] = (l1 - l2 - l3 + x * a - b * sp,
                         t1 + t2 + t3 + A(x * a) + A(b * sp))
            sg = sigmoid(a)
            out["da"] = (x - b * sg, A(x) + A(b * sg))
        elif fam == "laplace":                          # a = loc, b = scale
            d = x - a
            sg = np.sign(d)
            out["lp"] = (-np.log(2.0) - np.log(b) - A(d) / b, np.log(2.0) + A(np.log(b)) + A(d) / b)
            out["dx"] = (-sg / b, A(1 / b))
            out["da"] = (sg / b, A(1 / b))
            out["db"] = (-1 / b + A(d) / (b * b), A(1 / b) + A(d) / (b * b))
        elif fam == "bin_concrete":                     # a = temperature, b = logits
            lx, l1x = np.log(x), np.log1p(-x)
            lg = lx - l1x
            t = a * lg - b
            u = 1 - 2 * sigmoid(t)
            # errors in t (|a| (|lx| + |l1x| + 1) + |b|, the 1 from rounding 1 - x) pass with
            # slope |1 - 2 sigmoid(t)| <= 1
            tt = A(a) * (A(lx) + A(l1x) + 1) + A(b)
            out["lp"] = (np.log(a) - lx - l1x + t - 2 * softplus(t),
                         A(np.log(a)) + A(lx) + A(l1x) + 1 + A(t) + 2 * softplus(t) + 2 * tt)
            r = 1 / x + 1 / (1 - x)
            out["dx"] = (-1 / x + 1 / (1 - x) + u * a * r,
                         r + A(a) * r * (1 + 2 * sigmoid(t) * (1 - sigmoid(t)) * tt))
            out["da"] = (1 / a + u * lg, A(1 / a) + A(lg) + 1 + 2 * A(lg) * tt)
            out["db"] = (-u, A(u) + tt)
        else:
            raise ValueError(fam)
    return out


# ---------------------------------------------------------------- multivariate rows
def lse_rows(l):
    """(lse, softmax, terms of lse) over the last axis, as the kernels evaluate it:
    m = max l, lse = log(sum exp(l - m)) + m.  Each l_j - m is rounded (p_j |l_j - m| in the
    sum), the sum of exponentials is a C-term sum >= 1 (the 1 under the log)."""
    l = np.asarray(l, np.float64)
    m = np.max(l, -1, keepdims=True)
    with np.errstate(all="ignore"):
        e = np.exp(l - m)
        s = e.sum(-1, keepdims=True)
        lse = m + np.log(s)
        p = e / s
        spread = np.where(p > 0, p * np.abs(l - m), 0.0).sum(-1, keepdims=True)
    return lse, p, np.abs(m) + np.abs(np.log(s)) + 1 + spread


def categorical(k, l):
    """Categorical rows: (lp, lp terms, d lp / d logits, its terms) for class index k [...]
    against logits [..., C]; a class outside [0, C) gives NaN."""
    l = np.asarray(l, np.float64)
    C = l.shape[-1]
    lse, p, lt = lse_rows(l)
    ok = (k >= 0) & (k < C)
    kk = np.where(ok, k, 0)
    lk = np.take_along_axis(l, kk[..., None], -1)
    lp = np.where(ok, (lk - lse)[..., 0], np.nan)
    lp_terms = (np.abs(lk) + np.abs(lse) + lt)[..., 0]
    onehot = (np.arange(C) == kk[..., None]).astype(np.float64)
    grad = np.where(ok[..., None], onehot - p, np.nan)
    with np.errstate(all="ignore"):
        al = np.where(p > 0, p * (np.abs(l) + np.abs(lse) + lt), 0.0)
    return lp, lp_terms, grad, onehot + al
