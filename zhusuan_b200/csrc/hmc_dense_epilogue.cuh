// Fused leapfrog epilogue shared by the dense-Gaussian tensor-core kernels (hmc_dense_tc.cu: one
// pass per launch; hmc_dense_traj.cu: a whole trajectory per launch).  Velocity-Verlet update of
// zhusuan/hmc.py:38-43 on the accumulator tile: p += s2 * g, q_next = q + (eps / m) * p, plus the
// log p / kinetic partials of hamiltonian() (hmc.py:30-35) on the first / last pass.
#pragma once
#include "tc_common.cuh"

namespace {

// Fused leapfrog epilogue for one warp's share of a tile: this thread's dimension `n` (accumulator
// row) against NCOL chains starting at c0 (`trow` = shared address of the row's first column).
// MODE 0: plain pass; 1: + log-prob partials (first pass); 2: + log-prob and kinetic partials
// (last pass).
struct EpiArgs {
  const float* __restrict__ q_cur; float* __restrict__ q_next; float* __restrict__ q_next_lo;
  const float* __restrict__ p_in; float* __restrict__ p_out;
  float* __restrict__ lp_part; float* __restrict__ k_part;
  int64_t chains; int D;
  // fp16-split operands (impl 2): q_next_lo is then a [2][chains][D] __half buffer (hi plane, lo
  // plane) of q_next * q_scale, and the accumulator holds (P*sP)(q*sq): g = b - acc * acc_scale.
  int h16; float q_scale; float acc_scale;
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
// MODE: see above.  NEXT: 1 / 0 = q_next is / is not written (compile time), -1 = decided at run
// time from a.q_next.  DC: the dimension count when known at compile time (all per-column offsets
// j*D then fold into the load/store immediates: ~15 instead of ~40 instructions per element), 0 =
// run-time a.D.  H16: fp16-split planes (impl 2) vs TF32 residual (impl 1).
// COHERENT: 1 when q_cur may have been written earlier in the SAME launch (trajectory kernel): the
// non-coherent ld.global.nc path of __ldg could then return a stale L1 line.
template <int MODE, int NEXT, int DC, int H16, int NCOL = BN, int COHERENT = 0>
__device__ __forceinline__ void epilogue_half_tile(const EpiArgs& a, uint32_t trow, int n,
                                                   bool n_ok, bool parts_ok, int64_t c0,
                                                   int64_t part_row, int lane, float s2,
                                                   float eps_over_m, float inv_m, float b_n,
                                                   float mu_n, bool skip, float& amax) {
  const uint32_t D = DC ? (uint32_t)DC : (uint32_t)a.D;
  const int64_t chains = a.chains;
  const bool has_next = NEXT < 0 ? (a.q_next != nullptr) : (NEXT != 0);
  const bool warp_n_ok = __all_sync(0xffffffffu, n_ok);
  const bool fast_tile = warp_n_ok && (c0 + NCOL <= chains) && !skip;

  // this thread's element of chain c0 in every array (the same element offset everywhere)
  const int64_t off_t = c0 * (int64_t)D + n;
  const float* __restrict__ pin0 = a.p_in + off_t;
  const float* __restrict__ qc0 = a.q_cur + off_t;
  float* __restrict__ po0 = a.p_out + off_t;
  float* __restrict__ qn0 = has_next ? a.q_next + off_t : nullptr;
  // H16 == 2: the next pass splits q_next itself (in-kernel conversion); only max|q_next| is
  // tracked here for its scale
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
        if (H16 == 2) {
          const float aq = fabsf(qn);
          amax = (aq <= 3.0e38f) ? fmaxf(amax, aq) : amax;      // ignores NaN / inf
        } else {
          store_split<H16>(a, lo_p, hp, lp, (uint32_t)j * D, qn);
        }
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
      qe[j] = COHERENT ? __ldcg(qc + (uint32_t)j * D) : __ldg(qc + (uint32_t)j * D);
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
      if (cbase < chains && !skip) {
        const size_t cb = (size_t)c * D;
        float pe[16], qe[16];
        float lpv[MODE >= 1 ? 16 : 1], kv[MODE >= 2 ? 16 : 1];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const bool ok = n_ok && cbase + j < chains;
          if (COHERENT) {     // written earlier in this launch: no ld.global.nc
            pe[j] = ok ? __ldcg(pin0 + cb + (uint32_t)j * D) : 0.f;
            qe[j] = ok ? __ldcg(qc0 + cb + (uint32_t)j * D) : 0.f;
          } else {
            pe[j] = ok ? pin0[cb + (uint32_t)j * D] : 0.f;
            qe[j] = ok ? qc0[cb + (uint32_t)j * D] : 0.f;
          }
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
              if (H16 == 2) {
                const float aq = fabsf(qn);
                amax = (aq <= 3.0e38f) ? fmaxf(amax, aq) : amax;
              } else {
                store_split<H16>(a, lo0 + cb, hi_pl0 + cb, lo_pl0 + cb, (uint32_t)j * D, qn);
              }
            }
          }
        }
        if (MODE >= 1) {
          const float sum = warp_transpose_sum16(lpv, lane);
          if (parts_ok && lane < 16 && cbase + lane < chains)
            a.lp_part[part_row + cbase + lane] = sum;
        }
        if (MODE >= 2) {
          const float sum = warp_transpose_sum16(kv, lane);
          if (parts_ok && lane < 16 && cbase + lane < chains)
            a.k_part[part_row + cbase + lane] = sum;
        }
      }
    }
  }
}

}  // namespace
