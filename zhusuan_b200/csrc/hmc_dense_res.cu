// Whole-trajectory dense-Gaussian HMC with the fp16 hi/lo planes of q as the chain state
// (dense_impl = 5).
//
// Replaces the L+1 iterations of the leapfrog `tf.while_loop` of zhusuan/hmc.py:347-372 (body =
// leapfrog_integrator, hmc.py:38-43) plus the log p / kinetic terms of hamiltonian(), hmc.py:30-35.
// Inside a trajectory the state of q is its fp16 hi/lo plane pair of q*sq (plus fp32 p): each
// pass reads the planes it wrote in the previous pass, reconstructs q = (hi + lo)/sq (within 2^-23
// of the fp32 value), and writes the next planes, so no fp32 copy of q travels: 16*D bytes per
// chain and pass, the algorithmic minimum.
//
// On H100 one pass of the benchmark shape (65 536 chains x 1024 dimensions) executes ~0.4 TFLOP of
// fp16 products against ~1 GB of operand and state traffic, so the pass is bound by the tensor
// cores, not by HBM: the passes run as L+1 launches of the persistent tensor-core kernel
// (tc_pipeline_kernel) on alternating plane buffers, and the sampler state never leaves the plane
// format between the prepare and the select.
#include "tc_common.cuh"

namespace {

struct ResEpi {
  const __half* __restrict__ hi_cur; const __half* __restrict__ lo_cur;   // planes of q (this pass)
  __half* __restrict__ hi_nxt; __half* __restrict__ lo_nxt;               // planes of q_next
  const float* __restrict__ p_in; float* __restrict__ p_out;
  float* __restrict__ lp_part; float* __restrict__ k_part;
  int64_t chains; int D;
  float sq, inv_sq, acc_scale;
};

// One warp's share of a unit: dimension n (accumulator row) against NCOL chains from c0.
//   Q   = hi + lo                      (q * sq, exact to 2^-24)
//   g   = b_n - acc_scale * acc        (acc = (P sP)(q sq) from the three products)
//   p  += s2 * g
//   Qn  = Q + (eps/m * sq) * p  -> hi' = fp16(Qn), lo' = fp16(Qn - hi')
// MODE 1 / 2 add the log-prob partial (q - mu) * g  (and the kinetic partial p^2 / m).
template <int MODE, int NEXT, int DC>
__device__ __forceinline__ void epilogue_planes(const ResEpi& a, uint32_t trow, int n, bool n_ok,
                                                bool parts_ok, int64_t c0, int64_t part_row,
                                                int lane, float s2, float eps_over_m_sq,
                                                float inv_m, float b_n, float mu_n, bool skip) {
  constexpr int NCOL = BN;
  const uint32_t D = DC ? (uint32_t)DC : (uint32_t)a.D;
  const int64_t chains = a.chains;
  const bool warp_n_ok = __all_sync(0xffffffffu, n_ok);
  const bool fast_tile = warp_n_ok && (c0 + NCOL <= chains) && !skip;
  const int64_t off_t = c0 * (int64_t)D + n;
  const float* __restrict__ pin0 = a.p_in + off_t;
  float* __restrict__ po0 = a.p_out + off_t;
  const unsigned short* __restrict__ hc0 =
      reinterpret_cast<const unsigned short*>(a.hi_cur) + off_t;
  const unsigned short* __restrict__ lc0 =
      reinterpret_cast<const unsigned short*>(a.lo_cur) + off_t;
  __half* __restrict__ hn0 = NEXT ? a.hi_nxt + off_t : nullptr;
  __half* __restrict__ ln0 = NEXT ? a.lo_nxt + off_t : nullptr;

  auto element = [&](float acc, float p, uint32_t hl, float& pn, float& lpv, float& kv,
                     __half& hh, __half& ll) {
    const float Q = __half2float(__ushort_as_half((unsigned short)(hl & 0xFFFFu))) +
                    __half2float(__ushort_as_half((unsigned short)(hl >> 16)));
    const float g = b_n - a.acc_scale * acc;
    pn = fmaf(s2, g, p);
    if (MODE >= 1) lpv = (Q * a.inv_sq - mu_n) * g;
    if (MODE >= 2) kv = pn * pn * inv_m;
    if (NEXT) {
      const float Qn = fmaf(eps_over_m_sq, pn, Q);
      hh = __float2half_rn(Qn);
      ll = __float2half_rn(Qn - __half2float(hh));
    }
  };

  if (fast_tile) {
    auto load = [&](float* pe, uint32_t* he, int c) {
      const size_t cb = (size_t)c * D;
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        pe[j] = __ldcg(pin0 + cb + (uint32_t)j * D);
        const uint32_t h = __ldcg(hc0 + cb + (uint32_t)j * D);
        const uint32_t l = __ldcg(lc0 + cb + (uint32_t)j * D);
        he[j] = h | (l << 16);
      }
    };
    auto compute = [&](const uint32_t* v, const float* pe, const uint32_t* he, int c) {
      const size_t cb = (size_t)c * D;
      float lpv[MODE >= 1 ? 16 : 1], kv[MODE >= 2 ? 16 : 1];
#pragma unroll
      for (int j = 0; j < 16; ++j) {
        float pn, lp1 = 0.f, k1 = 0.f;
        __half hh, ll;
        element(__uint_as_float(v[j]), pe[j], he[j], pn, lp1, k1, hh, ll);
        po0[cb + (uint32_t)j * D] = pn;
        if (MODE >= 1) lpv[j] = lp1;
        if (MODE >= 2) kv[j] = k1;
        if (NEXT) {
          hn0[cb + (uint32_t)j * D] = hh;
          ln0[cb + (uint32_t)j * D] = ll;
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
    // software pipeline: the global loads of block i+1 are in flight while block i is computed
    float pa[16], pb[16];
    uint32_t ha[16], hb[16], va[16], vb[16];
    load(pa, ha, 0);
#pragma unroll 1
    for (int c = 0; c < NCOL; c += 32) {
      load(pb, hb, c + 16);
      acc_ld16(trow + 4u * (uint32_t)c, va);
      compute(va, pa, ha, c);
      if (c + 32 < NCOL) load(pa, ha, c + 32);
      acc_ld16(trow + 4u * (uint32_t)(c + 16), vb);
      compute(vb, pb, hb, c + 16);
    }
  } else {
#pragma unroll 1
    for (int c = 0; c < NCOL; c += 16) {
      uint32_t v[16];
      acc_ld16(trow + 4u * (uint32_t)c, v);
      const int64_t cbase = c0 + c;
      if (cbase < chains && !skip) {
        const size_t cb = (size_t)c * D;
        float lpv[MODE >= 1 ? 16 : 1], kv[MODE >= 2 ? 16 : 1];
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const bool ok = n_ok && cbase + j < chains;
          float p = 0.f;
          uint32_t hl = 0u;
          if (ok) {
            p = __ldcg(pin0 + cb + (uint32_t)j * D);
            hl = (uint32_t)__ldcg(hc0 + cb + (uint32_t)j * D) |
                 ((uint32_t)__ldcg(lc0 + cb + (uint32_t)j * D) << 16);
          }
          float pn, lp1 = 0.f, k1 = 0.f;
          __half hh, ll;
          element(__uint_as_float(v[j]), p, hl, pn, lp1, k1, hh, ll);
          if (MODE >= 1) lpv[j] = ok ? lp1 : 0.f;
          if (MODE >= 2) kv[j] = ok ? k1 : 0.f;
          if (ok) {
            po0[cb + (uint32_t)j * D] = pn;
            if (NEXT) {
              hn0[cb + (uint32_t)j * D] = hh;
              ln0[cb + (uint32_t)j * D] = ll;
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


template <int MODE, int NEXT, int DC>
struct ResW {
  static constexpr int KIND = 1, RB = 128, MNA = 0, MNB = 0, CVT = 0;
  static constexpr int KE = RB / 2;
  static constexpr uint32_t TX = Cfg<RB>::STAGE;
  CUtensorMap m_phi, m_plo, m_qhi, m_qlo;
  ResEpi ea;
  const float* bvec; const float* mu; const float* mass; const float* state;
  const float* scales;
  float p_scale;
  int n_blk, D_rt;
  struct EpiState {};

  __device__ __forceinline__ int D() const { return DC ? DC : D_rt; }
  __host__ __device__ __forceinline__ int64_t units() const {
    return ((ea.chains + BN - 1) / BN) * (int64_t)n_blk;
  }
  __device__ __forceinline__ void kb_range(int64_t, int& kb0, int& kb1) const {
    kb0 = 0;
    kb1 = D() / KE;
  }
  __device__ __forceinline__ void prefetch() const {
    tma_prefetch_desc(&m_phi); tma_prefetch_desc(&m_plo);
    tma_prefetch_desc(&m_qhi); tma_prefetch_desc(&m_qlo);
  }
  __device__ __forceinline__ void load(int64_t u, int kb, uint32_t sa, uint32_t fb) const {
    using C = Cfg<RB>;
    const int n0 = (int)(u % n_blk) * BM;
    const int c0 = (int)(u / n_blk) * BN;
    tma_load_2d(sa, &m_phi, fb, kb * KE, n0);
    tma_load_2d(sa + C::A_TILE, &m_plo, fb, kb * KE, n0);
    tma_load_2d(sa + 2 * C::A_TILE, &m_qhi, fb, kb * KE, c0);
    tma_load_2d(sa + 2 * C::A_TILE + C::B_TILE, &m_qlo, fb, kb * KE, c0);
  }
  __device__ __forceinline__ void convert(int64_t, int, uint8_t*, int) const {}
  __device__ __forceinline__ void epilogue(int64_t u, uint32_t trow, int quarter, int lane,
                                           EpiState&) const {
    const int nb = (int)(u % n_blk);
    const int n = nb * BM + quarter * 32 + lane;
    const int64_t c0 = (u / n_blk) * BN;
    const bool n_ok = n < D();
    const float eps = state[ZSB_ST_EPS_USED];
    const float s2 = mul(eps, p_scale);
    const float sq = scales[0];
    const float m_n = n_ok ? mass[n] : 1.f;
    const float eps_over_m_sq = mul(fdiv(eps, m_n), sq);
    const float inv_m = fdiv(1.f, m_n);
    const float b_n = (n_ok && bvec) ? bvec[n] : 0.f;
    const float mu_n = (n_ok && mu) ? mu[n] : 0.f;
    const int64_t part_row = (int64_t)(nb * 4 + quarter) * ea.chains;
    ResEpi a = ea;
    a.sq = sq;
    a.inv_sq = fdiv(1.f, sq);
    a.acc_scale = scales[1];
    epilogue_planes<MODE, NEXT, DC>(a, trow, n, n_ok, true, c0, part_row, lane, s2,
                                    eps_over_m_sq, inv_m, b_n, mu_n, false);
  }
  __device__ __forceinline__ void epi_finish(EpiState&, int, int) const {}
};

template <int DC>
int res_pass(const CUtensorMap& phi, const CUtensorMap& plo, const CUtensorMap& qhi,
             const CUtensorMap& qlo, const ResEpi& ea, const float* bvec, const float* mu,
             const float* mass, const float* state, const float* scales, float p_scale, int n_blk,
             int D, int mode, cudaStream_t st) {
  if (mode == 1) {
    const ResW<1, 1, DC> w{phi, plo, qhi, qlo, ea, bvec, mu, mass, state, scales, p_scale, n_blk, D};
    return tc_launch(w, st, "hmc_dense_resident");
  }
  if (mode == 0) {
    const ResW<0, 1, DC> w{phi, plo, qhi, qlo, ea, bvec, mu, mass, state, scales, p_scale, n_blk, D};
    return tc_launch(w, st, "hmc_dense_resident");
  }
  const ResW<2, 0, DC> w{phi, plo, qhi, qlo, ea, bvec, mu, mass, state, scales, p_scale, n_blk, D};
  return tc_launch(w, st, "hmc_dense_resident");
}

// q[c, :] <- (hi + lo) / sq of the proposal planes where accept[c] (hmc.py:488-497).
// One warp per chain at a time (the accept flag is warp-uniform: a rejected chain costs one 4-byte
// load), 8 dimensions per lane and step: two 128-bit plane loads in, two 128-bit stores out, up to
// four steps' loads issued before the first use.  D % 8 == 0 (the dense kernels need D % 64 == 0).
__global__ void __launch_bounds__(256) select_planes_kernel(float* __restrict__ q,
                                                            const __half* __restrict__ planes,
                                                            const float* __restrict__ scales,
                                                            const int32_t* __restrict__ accept,
                                                            int64_t chains, int64_t D) {
  const float inv_sq = 1.f / scales[0];
  const int lane = threadIdx.x & 31;
  const int n8 = (int)(D >> 3);
  const int64_t wstride = (int64_t)gridDim.x * 8;
  for (int64_t c = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); c < chains; c += wstride) {
    if (!accept[c]) continue;
    const uint4* __restrict__ hi = reinterpret_cast<const uint4*>(planes + c * D);
    const uint4* __restrict__ lo = reinterpret_cast<const uint4*>(planes + (chains + c) * D);
    float4* __restrict__ qr = reinterpret_cast<float4*>(q + c * D);
    for (int i0 = lane; i0 < n8; i0 += 128) {
      uint4 h[4], l[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + 32 * u;
        if (i < n8) { h[u] = __ldcs(hi + i); l[u] = __ldcs(lo + i); }
      }
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int i = i0 + 32 * u;
        if (i < n8) {
          const uint32_t hw[4] = {h[u].x, h[u].y, h[u].z, h[u].w};
          const uint32_t lw[4] = {l[u].x, l[u].y, l[u].z, l[u].w};
          float o[8];
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float2 hf = __half22float2(*reinterpret_cast<const __half2*>(&hw[k]));
            const float2 lf = __half22float2(*reinterpret_cast<const __half2*>(&lw[k]));
            o[2 * k] = (hf.x + lf.x) * inv_sq;
            o[2 * k + 1] = (hf.y + lf.y) * inv_sq;
          }
          qr[2 * i] = make_float4(o[0], o[1], o[2], o[3]);
          qr[2 * i + 1] = make_float4(o[4], o[5], o[6], o[7]);
        }
      }
    }
  }
}

}  // namespace

// Chain blocks per scheduling group (one group = every chain: the passes run as separate launches)
int zsb_dense_res_group_blocks(int D) {
  (void)D;
  return 1 << 30;
}

// The L+1 passes of a trajectory for every chain (D % 64 == 0, L >= 1).
//   planes0: fp16 hi/lo planes of q * sq (zsb_hmc_dense_h16_prepare_f32), planes1: work buffer of
//   the same size (must differ from planes0: a pass reads every dimension of a chain block's planes
//   while other tiles of the same launch write the next ones); on return the proposal's planes are
//   in buffer (L & 1); p0 -> pw (final momentum); lp0_part / lp1_part / k_part as the per-pass
//   kernel writes them.  `flags` is not used.
int zsb_dense_res_h16_launch(void* planes0, void* planes1, const float* p0, float* pw,
                             const void* P_h16, const void* P_l16, const float* scales,
                             const float* bvec, const float* mu, const float* mass,
                             const float* state, float* lp0_part, float* lp1_part, float* k_part,
                             int* flags, int64_t chains, int D, int L, cudaStream_t st) {
  (void)flags;
  if (D % 64 != 0 || D < 64 || L < 1 || chains <= 0 || chains >= (1LL << 31)) {
    zsb_set_error("dense_res: needs D %% 64 == 0, n_leapfrogs >= 1");
    return ZSB_ERR_INVALID;
  }
  if (planes0 == planes1) {
    zsb_set_error("dense_res: planes1 must be a separate work buffer");
    return ZSB_ERR_INVALID;
  }
  CUtensorMap phi, plo, qhi[2], qlo[2];
  int rc;
  if ((rc = make_map(&phi, P_h16, (uint64_t)D, (uint64_t)D, BM, 128, 1))) return rc;
  if ((rc = make_map(&plo, P_l16, (uint64_t)D, (uint64_t)D, BM, 128, 1))) return rc;
  __half* pl[2] = {reinterpret_cast<__half*>(planes0), reinterpret_cast<__half*>(planes1)};
  const int64_t plane = chains * (int64_t)D;
  for (int b = 0; b < 2; ++b) {
    if ((rc = make_map(&qhi[b], pl[b], (uint64_t)chains, (uint64_t)D, BN, 128, 1))) return rc;
    if ((rc = make_map(&qlo[b], pl[b] + plane, (uint64_t)chains, (uint64_t)D, BN, 128, 1)))
      return rc;
  }
  const int n_blk = (D + BM - 1) / BM;
  for (int i = 0; i <= L; ++i) {
    const bool last = i == L;
    const int buf = i & 1;
    const ResEpi ea{pl[buf], pl[buf] + plane, pl[buf ^ 1], pl[buf ^ 1] + plane,
                    i == 0 ? p0 : pw, pw, i == 0 ? lp0_part : lp1_part, k_part, chains, D,
                    1.f, 1.f, 1.f};
    const int mode = last ? 2 : (i == 0 ? 1 : 0);
    const float p_scale = (i > 0 && !last) ? 1.f : 0.5f;
    rc = (D == 1024) ? res_pass<1024>(phi, plo, qhi[buf], qlo[buf], ea, bvec, mu, mass, state,
                                      scales, p_scale, n_blk, D, mode, st)
                     : res_pass<0>(phi, plo, qhi[buf], qlo[buf], ea, bvec, mu, mass, state,
                                   scales, p_scale, n_blk, D, mode, st);
    if (rc != ZSB_OK) return rc;
  }
  return ZSB_OK;
}

int zsb_dense_select_planes_launch(float* q, const void* planes, const float* scales,
                                   const int32_t* accept, int64_t chains, int64_t D,
                                   cudaStream_t st) {
  ZSB_REQUIRE(D % 8 == 0, "zsb_dense_select_planes: D must be a multiple of 8");
  int64_t blocks = zsb_ceil_div(chains, 8);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  if (blocks < 1) blocks = 1;
  select_planes_kernel<<<(unsigned)blocks, 256, 0, st>>>(
      q, reinterpret_cast<const __half*>(planes), scales, accept, chains, D);
  return zsb_check_launch("hmc_select_planes");
}
