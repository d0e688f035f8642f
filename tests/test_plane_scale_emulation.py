"""NumPy emulation (CPU) of the fp16 plane state of the dense-Gaussian trajectory (dense_impl 5,
hmc_dense_res.cu; impl 2 writes its planes the same way): inside a trajectory q exists only
as fp16 hi / lo planes of q * sq.  Each pass rebuilds Q = hi + lo, kicks p with g = b - P q,
drifts Q by (eps / m) * sq * p and rounds the result into the next planes.

Two plane-scale rules:
  fixed  -- one sq per iteration from max|q0| (the power of two placing it in [2^11, 2^12)): the
            planes overflow once any element grows ~16x beyond max|q0|;
  bound  -- pass i writes its planes at sq_{i+1} = sq_i while the a-priori bound
              B_i = max|q_i| + drift_i + eps s2 max(1/m) (max|b| + ||P||_inf max|q_i|),
              drift_0 = eps max|p_0/m|,  drift_i = max|q_i| + max|q_{i-1}|  (i > 0),
            on |q_{i+1}| keeps B_i * sq_i below 2^16 - 2^8, else at the power of two placing B_i
            in [2^11, 2^12) (hmc_dense_epilogue.cuh; dense_impl 2);
  spare  -- (dense_impl 5) the planes are always written at sq_i; where the bound is reached a
            spare copy at the lowered scale is written too, and the next pass reads it only if
            some |q_{i+1}| * sq_i reached fp16's overflow."""
import itertools

import numpy as np

from oracle import hmc as OH
from oracle import models as OM

f16, f32 = np.float16, np.float32
KEEP = f32(65280.0)


def pow2_scale(m):
    e = np.frexp(f32(m))[1] if m > 0 else 0
    return f32(2.0) ** (12 - e)


def to_planes(x):
    with np.errstate(over="ignore", invalid="ignore"):
        h = x.astype(f16)
        l = (x - h.astype(f32)).astype(f16)
    return h, l


def finite_absmax(x):
    a = np.abs(x)
    a = a[np.isfinite(a)]
    return f32(a.max()) if a.size else f32(0)


def emulate(q0, p0, P, b, mass, eps, L, rule):
    """The L + 1 passes on the plane state; returns (q of the proposal, p, the scales used)."""
    P = P.astype(f32)
    eps = f32(eps)
    inv_m = (f32(1) / mass).astype(f32)
    p_inf, b_max, w = f32(np.abs(P).sum(1).max()), finite_absmax(b), f32(inv_m.max())
    sq = pow2_scale(finite_absmax(q0))
    hi, lo = to_planes((q0 * sq).astype(f32))
    mq, mq_prev, mv = finite_absmax(q0), None, finite_absmax(p0 * inv_m)
    p = p0.astype(f32)
    scales = [sq]
    with np.errstate(over="ignore", invalid="ignore"):
        for i in range(L + 1):
            Q = hi.astype(f32) + lo.astype(f32)
            q = (Q / sq).astype(f32)
            g = (b - q @ P).astype(f32)
            s2 = eps if 0 < i < L else eps / f32(2)
            p = (p + s2 * g).astype(f32)
            if i == L:
                return q, p, scales
            sq_next = sq
            if rule != "fixed":
                drift = eps * mv if i == 0 else mq + mq_prev
                bound = mq + drift + eps * s2 * w * (b_max + p_inf * mq)
                if not bound * sq < KEEP:
                    sq_next = pow2_scale(bound)
            Qm = (Q + (eps * inv_m * sq) * p).astype(f32)
            if rule == "spare" and not finite_absmax(Qm) >= 65520:
                sq_next = sq                           # the planes at sq fit: the spare is unused
            Qn = (Qm * (sq_next / sq)).astype(f32)
            hi, lo = to_planes(Qn)
            mq, mq_prev = finite_absmax(Qn / sq_next), mq
            sq = sq_next
            scales.append(sq)


def reference(q0, p0, P, b, mass, eps, L):
    """The fp32 leapfrog of the oracle (hmc.py:347-372)."""
    om = OM.DenseGaussian(P.astype(f32), np.linalg.solve(P, b).astype(f32))
    h = OH.HMC(step_size=eps, n_leapfrogs=L)
    q, p = [q0.astype(f32)], [p0.astype(f32)]
    for i in range(L + 1):
        s1 = f32(eps) if i > 0 else f32(0)
        s2 = f32(eps) if 0 < i < L else f32(eps) / f32(2)
        q, p = h._leapfrog_integrator(q, p, s1, s2, om.grad, [mass.astype(f32)])
    return q[0], p[0]


def _setup(init, D=64, C=24, seed=0):
    P, _ = OM.make_dense_gaussian_problem(D, seed=4)
    rng = np.random.RandomState(seed)
    q0 = (init * rng.standard_normal((C, D))).astype(f32)
    p0 = rng.standard_normal((C, D)).astype(f32)
    mass = np.ones(D, f32)
    return P, np.zeros(D, f32), mass, q0, p0


def test_one_scale_per_iteration_overflows_from_a_small_state():
    P, b, mass, q0, p0 = _setup(1e-3)
    q, p, scales = emulate(q0, p0, P, b, mass, 0.15, 10, "fixed")
    assert scales[0] == 2.0 ** 20                      # max|q0| ~ 3e-3
    assert not np.isfinite(q).all() and not np.isfinite(p).all()
    qr, _ = reference(q0, p0, P, b, mass, 0.15, 10)
    assert np.isfinite(qr).all() and np.abs(qr).max() > 65520 / 2.0 ** 20


def test_bound_rules_match_the_fp32_leapfrog_from_zero_and_small_states():
    for init, L, rule in itertools.product((0.0, 1e-3, 1e-6), (1, 10, 50), ("bound", "spare")):
            P, b, mass, q0, p0 = _setup(init, seed=L)
            q, p, scales = emulate(q0, p0, P, b, mass, 0.15, L, rule)
            qr, pr = reference(q0, p0, P, b, mass, 0.15, L)
            assert np.isfinite(q).all() and np.isfinite(p).all()
            if init > 0:                               # the scale followed the trajectory
                assert scales[-1] < scales[0]
            np.testing.assert_allclose(q, qr, rtol=0, atol=2e-6 * np.abs(qr).max())
            np.testing.assert_allclose(p, pr, rtol=0, atol=2e-6 * np.abs(pr).max())


def test_bound_rule_with_a_mean_and_a_mass_on_a_wide_target():
    D, C, L, eps = 64, 24, 20, 6.0
    P, _ = OM.make_dense_gaussian_problem(D, seed=4)
    P = P / 1600.0                                     # marginal std 40
    rng = np.random.RandomState(3)
    mu = (30 * rng.standard_normal(D)).astype(f32)
    b = (P.astype(f32).astype(np.float64) @ mu).astype(f32)
    mass = (0.5 + rng.random_sample(D)).astype(f32)
    q0 = np.zeros((C, D), f32)
    p0 = (rng.standard_normal((C, D)) * np.sqrt(mass)).astype(f32)
    q, p, scales = emulate(q0, p0, P, b, mass, eps, L, "bound")
    qr, pr = reference(q0, p0, P, b, mass, eps, L)
    assert np.abs(qr).max() > 16 and scales[-1] < 2.0 ** 12
    np.testing.assert_allclose(q, qr, rtol=0, atol=2e-6 * np.abs(qr).max())
    np.testing.assert_allclose(p, pr, rtol=0, atol=2e-6 * np.abs(pr).max())


def test_bound_rule_keeps_the_scale_when_the_trajectory_stays_in_range():
    """From posterior-scale states the bound never triggers: the planes, and so every result,
    are bit-identical to the one-scale rule."""
    P, b, mass, q0, p0 = _setup(1.0)
    for L in (1, 10, 50):
        qa, pa, sa = emulate(q0, p0, P, b, mass, 0.15, L, "bound")
        qb, pb, sb = emulate(q0, p0, P, b, mass, 0.15, L, "fixed")
        assert sa == sb
        np.testing.assert_array_equal(qa, qb)
        np.testing.assert_array_equal(pa, pb)


def test_spare_rule_is_the_one_scale_rule_wherever_that_one_fits():
    """A step size near the stability limit: the bound (loose by ~10x there) asks for a lower
    scale, but the planes at the one scale fit.  The spare rule then gives bit-identical results;
    the bound rule rescales, which changes the rounding."""
    P, b, mass, q0, p0 = _setup(1.0, D=1024, C=8, seed=3)
    eps = 0.55                                         # 2 / sqrt(lambda_max(P)) = 0.60
    qf, pf, sf = emulate(q0, p0, P, b, mass, eps, 10, "fixed")
    qs, ps, ss = emulate(q0, p0, P, b, mass, eps, 10, "spare")
    qb, pb, sb = emulate(q0, p0, P, b, mass, eps, 10, "bound")
    assert np.isfinite(qf).all() and min(sb) < sb[0]
    assert ss == sf
    np.testing.assert_array_equal(qs, qf)
    np.testing.assert_array_equal(ps, pf)
    assert not np.array_equal(qb, qf)


def test_the_bound_is_never_exceeded():
    """B_i >= max|q_{i+1}| on every pass, for an unstable step too (q grows ~14x per pass)."""
    for eps in (0.15, 4.0 / np.sqrt(11.3)):
        P, b, mass, q0, p0 = _setup(1.0, seed=7)
        P32 = P.astype(f32)
        p_inf = f32(np.abs(P32).sum(1).max())
        eps = f32(eps)
        q, p, q_prev = q0.copy(), p0.copy(), None
        for i in range(10):
            s2 = eps if i > 0 else eps / f32(2)
            mq = np.abs(q).max()
            drift = eps * np.abs(p).max() if i == 0 else mq + np.abs(q_prev).max()
            bound = mq + drift + eps * s2 * p_inf * mq
            p = (p + s2 * (b - q @ P32)).astype(f32)
            q, q_prev = (q + eps * p).astype(f32), q
            assert np.abs(q).max() <= bound
