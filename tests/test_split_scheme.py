"""Numerical design check (CPU, NumPy emulation) of the operand split the tensor-core kernels
use (hmc_dense_tc.cu impl 2/3, gemm_logjoint_tc.cu):  x * s = h + l with h = fp16_rn(x * s),
l = fp16_rn(x * s - h), s a power of two placing max|x| in [2^11, 2^12), and the product
approximated by  h_a h_b + h_a l_b + l_a h_b  accumulated in fp32.  The dropped l_a l_b term and
the rounding of l bound the error at ~2^-21 of sum_k |a_k b_k| -- fp32-GEMM level, three orders of
magnitude below a single TF32 / fp16 product -- which is what the GPU parity tests then observe."""
import numpy as np


def pow2_scale(x):
    m = np.abs(x).max()
    e = np.frexp(np.float32(m))[1] if m > 0 else 0          # m = f * 2^e, f in [0.5, 1)
    return np.float32(2.0) ** (12 - e)


def split(x):
    s = pow2_scale(x)
    xs = (x.astype(np.float32) * s).astype(np.float32)
    h = xs.astype(np.float16)
    l = (xs - h.astype(np.float32)).astype(np.float16)
    return h, l, s


def split_matmul(a, b):
    """a [M, K], b [N, K] -> a b^T the way the kernels compute it (fp32 accumulation)."""
    ah, al, sa = split(a)
    bh, bl, sb = split(b)
    f = lambda t: t.astype(np.float32)
    acc = f(al) @ f(bh).T + f(ah) @ f(bl).T + f(ah) @ f(bh).T
    return acc / (sa * sb)


def test_scale_places_the_maximum_in_2_11_2_12():
    rng = np.random.RandomState(0)
    for mag in (1e-6, 0.3, 1.0, 7.5, 4096.0, 3e7):
        x = (rng.standard_normal(1000) * mag).astype(np.float32)
        s = pow2_scale(x)
        assert 2 ** 11 <= np.abs(x).max() * s < 2 ** 12
        assert np.log2(s) == np.round(np.log2(s))            # exact power of two


def test_hi_plus_lo_reconstructs_to_22_bits_per_element():
    rng = np.random.RandomState(1)
    x = (rng.standard_normal(20000) * np.exp(rng.uniform(-6, 0, 20000))).astype(np.float32)
    h, l, s = split(x)
    rec = (h.astype(np.float64) + l.astype(np.float64)) / s
    big = np.abs(x) * s >= 2.0 ** -3           # lo plane still a normal fp16 number
    rel = np.abs(rec - x)[big] / np.abs(x)[big]
    assert rel.max() < 2.0 ** -21
    # tiny elements: absolute error bounded by the fp16 subnormal spacing of the lo plane
    assert (np.abs(rec - x)[~big] * s).max() <= 2.0 ** -24


def test_three_product_split_matmul_is_fp32_accurate():
    rng = np.random.RandomState(2)
    for (m, n, k) in ((64, 48, 500), (32, 32, 1024)):
        a = rng.standard_normal((m, k)).astype(np.float32)
        b = (rng.standard_normal((n, k)) / np.sqrt(k)).astype(np.float32)
        exact = a.astype(np.float64) @ b.astype(np.float64).T
        scale = np.abs(a).astype(np.float64) @ np.abs(b).astype(np.float64).T
        err_split = np.abs(split_matmul(a, b) - exact) / scale
        err_fp16 = np.abs(a.astype(np.float16).astype(np.float32)
                          @ b.astype(np.float16).astype(np.float32).T - exact) / scale
        err_fp32 = np.abs(a @ b.T - exact) / scale
        assert err_split.max() < 2.0 ** -20                   # ~1e-6 of sum |a||b|
        assert err_split.max() < 20 * max(err_fp32.max(), 2.0 ** -24)   # fp32-GEMM class
        assert err_fp16.max() > 50 * err_split.max()          # what one fp16 product would give


def test_overflow_headroom_of_the_hmc_scale():
    """sq places max|q| in [2^11, 2^12), so a scale kept fixed lets q grow at most ~16x before h
    overflows fp16 (65504 < 2^16 = 2^12 * 16).  The HMC trajectory therefore checks an a-priori
    bound on |q_next| every pass: where it would reach 2^16 - 2^8 at the current scale, the planes
    also get a copy at a lower scale (impl 5: kept as a spare, used only if the planes overflowed;
    impl 2: used directly) (hmc_dense_epilogue.cuh; emulated in
    test_plane_scale_emulation.py)."""
    x = np.array([1.0, -3.0], np.float32)
    s = pow2_scale(x)
    for growth in (1, 4, 8, 15):
        assert np.isfinite((x * growth * s).astype(np.float16)).all()
    with np.errstate(over="ignore"):
        assert not np.isfinite((x * 32 * s).astype(np.float16)).all()


def test_trajectory_kernel_buffer_schedule_matches_the_per_pass_host_loop():
    """Closed form of the buffer ping-pong of the per-pass host loop
    (zhusuan_b200/hmc.py::_iterate_dense, dense_impl 0 / 1 / 2): pass i reads traj_cur(i) and
    writes traj_nxt(i) with 0 = q0, 1 = qa, 2 = qb; the proposal ends in qa when L - 1 is even,
    else in qb."""
    traj_cur = lambda i: 0 if i == 0 else (1 if i & 1 else 2)
    traj_nxt = lambda i: 2 if i & 1 else 1
    for L in range(1, 12):
        cur, nxt = 0, 1                               # host loop: cur, nxt = q0, qa
        for i in range(L + 1):
            last = i == L
            assert traj_cur(i) == cur
            if not last:
                assert traj_nxt(i) == nxt
                cur, nxt = nxt, (2 if nxt == 1 else 1)
        assert cur == (1 if (L - 1) % 2 == 0 else 2)
