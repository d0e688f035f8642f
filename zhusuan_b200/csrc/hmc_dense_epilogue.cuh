// Fused leapfrog epilogue of the per-pass dense-Gaussian tensor-core kernel (hmc_dense_tc.cu), and
// the plane-scale records it shares with the trajectory kernel (hmc_dense_res.cu).  Velocity-Verlet
// update of zhusuan/hmc.py:38-43 on the accumulator tile: p += s2 * g, q_next = q + (eps / m) * p,
// plus the log p / kinetic partials of hamiltonian() (hmc.py:30-35) on the first / last pass.
#pragma once
#include "tc_common.cuh"

namespace {

// Plane scales of the fp16-split trajectory (impl 2, 5).  `scales` is a device float array of
// kScaleHdr + kScaleRec * (L + 2) words:
//   [0] sq of q0's planes, [1] 1/(sP*sq) (copies of record 0), [2] prepare scratch (max|q0| bits),
//   [3] sP, [4] ||P||_inf, [5] max|b| (the caller sets these three once), [6] prepare scratch
//   (max|p0/m| bits), [7] max(1/m) (prepare);
//   record i (pass i) at kScaleHdr + kScaleRec * i: {sq_i, sq_alt_i, max|q_i|, w}: the scale of
//   the planes of q_i, the scale of their spare copy (impl 5; = sq_i when there is none), an upper
//   bound of max|q_i|, and w = max|p_0/m| for record 0, else the flag "the planes of q_i
//   overflowed: read the spare copy" (impl 5).  Maxima and flags are uint bits.  Record 0 comes
//   from prepare, which also clears record 1; pass i writes record i + 1 and clears record i + 2.
//   So every trajectory, step-size probes included, starts with a prepare.
// Since g = b - P q and q_{i+1} = q_i + (eps/m) (p_i + s2 g_i),
//   B_i = max|q_i| + drift_i + eps * s2 * max(1/m) * (max|b| + ||P||_inf * max|q_i|)
// bounds |q_{i+1}| before any of it is computed, with drift_0 = eps * max|p_0/m| and, for i > 0,
// drift_i = max|q_i| + max|q_{i-1}| >= max|(eps/m) p_i| = max|q_i - q_{i-1}| (so a pass only
// reduces max|q|).  While B_i * sq_i stays below kPlaneKeep the planes of q_{i+1} cannot
// overflow at sq_i.  Otherwise sq_alt = the power of two that puts B_i in [2^11, 2^12):
//   impl 2 writes the next planes at sq_alt;
//   impl 5 writes them at sq_i, exactly as when the bound is not reached, plus a spare copy at
//   sq_alt, and flags the pass if any |q_{i+1}| * sq_i reached fp16's overflow (65520); the next
//   pass then reads the spare.  A bound is loose, so this keeps every trajectory whose planes fit
//   bit-identical to a fixed scale, and only the ones that would overflow change.
// B_i is a strict bound, so the only slack needed below 65520 is the rounding of B_i and q; scales
// are powers of two, so a rescaled copy is exact up to the fp16 rounding of its lo plane.
constexpr int kScaleHdr = 8, kScaleRec = 4;
constexpr float kPlaneKeep = 65280.f;   // 2^16 - 2^8
constexpr float kHalfOverflow = 65520.f;   // fp16 round-to-nearest gives inf from here on

__device__ __forceinline__ const float* scale_rec(const float* scales, int pass) {
  return scales + kScaleHdr + kScaleRec * pass;
}
// impl 5: pass `pass` reads the spare copy of its planes
__device__ __forceinline__ bool plane_spare_in(const float* scales, int pass) {
  return pass > 0 && __float_as_uint(scale_rec(scales, pass)[3]) != 0u;
}
// the scale of the planes pass `pass` reads
__device__ __forceinline__ float plane_scale_in(const float* scales, int pass) {
  return scale_rec(scales, pass)[plane_spare_in(scales, pass) ? 1 : 0];
}
// sq_alt of the planes pass `pass` writes (= sq when the bound keeps them inside fp16 at sq)
__device__ __forceinline__ float next_plane_scale(const float* __restrict__ scales, int pass,
                                                  float eps, float s2, float sq) {
  const float* r = scale_rec(scales, pass);
  const float mq = r[2];
  const float drift = pass == 0 ? eps * r[3] : mq + r[2 - kScaleRec];
  const float bound = mq + drift + eps * s2 * scales[7] * (scales[5] + scales[4] * mq);
  // a non-finite bound (an infinite q or p, or step size) keeps the scale: those proposals are
  // rejected
  if (bound * sq < kPlaneKeep || !(bound <= 3.0e38f)) return sq;
  return pow2_plane_scale(bound);
}
// end of a pass that wrote planes: the warp's bound of max|q_next| (and overflow flag) into record
// pass + 1; block 0 publishes the scales of those planes and clears record pass + 2
__device__ __forceinline__ void publish_plane_scale(float* __restrict__ scales, int pass,
                                                    float sq_next, float sq_alt, float qmax,
                                                    bool overflow, int quarter, int lane) {
  unsigned int* r = reinterpret_cast<unsigned int*>(scales + kScaleHdr + kScaleRec * (pass + 1));
  const float mq = warp_max(qmax);
  const bool any_overflow = __any_sync(0xffffffffu, overflow);
  if (lane == 0) {
    atomicMax(r + 2, __float_as_uint(mq));
    if (any_overflow) atomicOr(r + 3, 1u);
  }
  if (blockIdx.x == 0 && quarter == 0 && lane == 0) {
    reinterpret_cast<float*>(r)[0] = sq_next;
    reinterpret_cast<float*>(r)[1] = sq_alt;
    r[kScaleRec + 2] = 0u;
    r[kScaleRec + 3] = 0u;
  }
}

// Fused leapfrog epilogue for one warp's share of a tile: this thread's dimension `n` (accumulator
// row) against BN chains starting at c0 (`trow` = shared address of the row's first column).
// MODE 0: plain pass; 1: + log-prob partials (first pass); 2: + log-prob and kinetic partials
// (last pass).
struct EpiArgs {
  const float* __restrict__ q_cur; float* __restrict__ q_next; float* __restrict__ q_next_lo;
  const float* __restrict__ p_in; float* __restrict__ p_out;
  float* __restrict__ lp_part; float* __restrict__ k_part;
  int64_t chains; int D;
  // fp16-split operands (impl 2): q_next_lo is then a [2][chains][D] __half buffer (hi plane, lo
  // plane) of q_next * q_scale, and the accumulator holds (P*sP)(q_cur*sq): g = b - acc * acc_scale.
  float acc_scale; float q_scale;
};
// residual operand(s) of q_next for the next pass's MMA
template <int H16>   // 0: TF32 residual, 1: fp16 hi/lo planes
__device__ __forceinline__ void store_split(const EpiArgs& a, float* __restrict__ lo_f32,
                                            __half* __restrict__ hi_pl, __half* __restrict__ lo_pl,
                                            uint32_t off, float qn) {
  if (H16) {
    const float x = qn * a.q_scale;
    const __half h = __float2half_rn(x);
    hi_pl[off] = h;
    lo_pl[off] = __float2half_rn(x - __half2float(h));
  } else {
    lo_f32[off] = qn - __uint_as_float(__float_as_uint(qn) & 0xFFFFE000u);
  }
}
// MODE: see above.  q_next is written when a.q_next is set.  DC: the dimension count when known
// at compile time (all per-column offsets j*D then fold into the load/store immediates: ~15
// instead of ~40 instructions per element), 0 = run-time a.D.  H16: fp16-split planes (impl 2) vs
// TF32 residual (impl 1).  amax: running max of |q_next| (H16 1) over the elements this thread
// wrote (fmaxf drops NaN; an inf makes the plane-scale bound infinite, which keeps the scale).
template <int MODE, int DC, int H16>
__device__ __forceinline__ void epilogue_half_tile(const EpiArgs& a, uint32_t trow, int n,
                                                   bool n_ok, int64_t c0, int64_t part_row,
                                                   int lane, float s2, float eps_over_m,
                                                   float inv_m, float b_n, float mu_n,
                                                   float& amax) {
  constexpr int NCOL = BN;
  const uint32_t D = DC ? (uint32_t)DC : (uint32_t)a.D;
  const int64_t chains = a.chains;
  const bool has_next = a.q_next != nullptr;
  const bool warp_n_ok = __all_sync(0xffffffffu, n_ok);
  const bool fast_tile = warp_n_ok && (c0 + NCOL <= chains);

  // this thread's element of chain c0 in every array (the same element offset everywhere)
  const int64_t off_t = c0 * (int64_t)D + n;
  const float* __restrict__ pin0 = a.p_in + off_t;
  const float* __restrict__ qc0 = a.q_cur + off_t;
  float* __restrict__ po0 = a.p_out + off_t;
  float* __restrict__ qn0 = has_next ? a.q_next + off_t : nullptr;
  float* __restrict__ lo0 = (has_next && H16 == 0) ? a.q_next_lo + off_t : nullptr;
  __half* __restrict__ hi_pl0 =
      (has_next && H16 == 1) ? reinterpret_cast<__half*>(a.q_next_lo) + off_t : nullptr;
  __half* __restrict__ lo_pl0 = (has_next && H16 == 1) ? hi_pl0 + chains * (int64_t)D : nullptr;

  // `c`: first column of the 16-column block, relative to c0
  auto compute = [&](const uint32_t* v, const float* pe, const float* qe, int c) {
    const size_t cb = (size_t)c * D;
    float* __restrict__ po = po0 + cb;
    float* __restrict__ qn_p = has_next ? qn0 + cb : nullptr;
    float* __restrict__ lo_p = (has_next && H16 == 0) ? lo0 + cb : nullptr;
    __half* __restrict__ hp = (has_next && H16 == 1) ? hi_pl0 + cb : nullptr;
    __half* __restrict__ lp = (has_next && H16 == 1) ? lo_pl0 + cb : nullptr;
    float lpv[MODE >= 1 ? 16 : 1], kv[MODE >= 2 ? 16 : 1];
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const float g = b_n - a.acc_scale * __uint_as_float(v[j]);
      const float pn = fmaf(s2, g, pe[j]);
      po[(uint32_t)j * D] = pn;
      if (MODE >= 1) lpv[j] = (qe[j] - mu_n) * g;
      if (MODE >= 2) kv[j] = pn * pn * inv_m;
      if (has_next) {
        const float qn = fmaf(eps_over_m, pn, qe[j]);
        qn_p[(uint32_t)j * D] = qn;
        if (H16 == 1) amax = fmaxf(amax, fabsf(qn));
        store_split<H16>(a, lo_p, hp, lp, (uint32_t)j * D, qn);
      }
    }
    if (MODE >= 1) {
      const float sum = warp_transpose_sum16(lpv, lane);
      if (lane < 16) a.lp_part[part_row + c0 + c + lane] = sum;
    }
    if (MODE >= 2) {
      const float sum = warp_transpose_sum16(kv, lane);
      if (lane < 16) a.k_part[part_row + c0 + c + lane] = sum;
    }
  };
  auto load = [&](float* pe, float* qe, int c) {
    const float* __restrict__ pin = pin0 + (size_t)c * D;
    const float* __restrict__ qc = qc0 + (size_t)c * D;
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      pe[j] = __ldcs(pin + (uint32_t)j * D);       // p is streamed: evict-first
      qe[j] = __ldg(qc + (uint32_t)j * D);
    }
  };

  if (fast_tile) {
    // software-pipelined: the global loads of block i+1 are in flight while block i is computed
    // and stored (two register sets A/B, loop unrolled by two blocks)
    float pa[16], qa[16], pb[16], qb[16];
    uint32_t va[16], vb[16];
    load(pa, qa, 0);
#pragma unroll 1
    for (int c = 0; c < NCOL; c += 32) {
      load(pb, qb, c + 16);
      acc_ld16(trow + 4u * (uint32_t)c, va);
      compute(va, pa, qa, c);
      if (c + 32 < NCOL) load(pa, qa, c + 32);
      acc_ld16(trow + 4u * (uint32_t)(c + 16), vb);
      compute(vb, pb, qb, c + 16);
    }
  } else {
#pragma unroll 1
    for (int c = 0; c < NCOL; c += 16) {
      uint32_t v[16];
      acc_ld16(trow + 4u * (uint32_t)c, v);
      const int64_t cbase = c0 + c;
      if (cbase < chains) {
        const size_t cb = (size_t)c * D;
        float pe[16], qe[16];
        float lpv[MODE >= 1 ? 16 : 1], kv[MODE >= 2 ? 16 : 1];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const bool ok = n_ok && cbase + j < chains;
          pe[j] = ok ? pin0[cb + (uint32_t)j * D] : 0.f;
          qe[j] = ok ? qc0[cb + (uint32_t)j * D] : 0.f;
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const bool ok = n_ok && cbase + j < chains;
          const float g = b_n - a.acc_scale * __uint_as_float(v[j]);
          const float pn = fmaf(s2, g, pe[j]);
          if (MODE >= 1) lpv[j] = ok ? (qe[j] - mu_n) * g : 0.f;
          if (MODE >= 2) kv[j] = ok ? pn * pn * inv_m : 0.f;
          if (ok) {
            po0[cb + (uint32_t)j * D] = pn;
            if (has_next) {
              const float qn = fmaf(eps_over_m, pn, qe[j]);
              qn0[cb + (uint32_t)j * D] = qn;
              if (H16 == 1) amax = fmaxf(amax, fabsf(qn));
              store_split<H16>(a, lo0 + cb, hi_pl0 + cb, lo_pl0 + cb, (uint32_t)j * D, qn);
            }
          }
        }
        if (MODE >= 1) {
          const float sum = warp_transpose_sum16(lpv, lane);
          if (lane < 16 && cbase + lane < chains) a.lp_part[part_row + cbase + lane] = sum;
        }
        if (MODE >= 2) {
          const float sum = warp_transpose_sum16(kv, lane);
          if (lane < 16 && cbase + lane < chains) a.k_part[part_row + cbase + lane] = sum;
        }
      }
    }
  }
}

}  // namespace
