// Whole-trajectory dense-Gaussian HMC with the fp16 hi/lo planes of q as the chain state
// (dense_impl = 5).
//
// Replaces the L+1 iterations of the leapfrog `tf.while_loop` of zhusuan/hmc.py:347-372 (body =
// leapfrog_integrator, hmc.py:38-43) plus the log p / kinetic terms of hamiltonian(), hmc.py:30-35.
// Inside a trajectory the state of q is its fp16 hi/lo plane pair of q*sq (plus fp32 p): each
// pass reads the planes it wrote in the previous pass, reconstructs q = (hi + lo)/sq_i (within
// 2^-23 of the fp32 value), and writes the next planes at sq_{i+1}, so no fp32 copy of q travels:
// 16*D bytes per chain and pass, the algorithmic minimum.  When an a-priori bound on |q_{i+1}|
// (hmc_dense_epilogue.cuh) says the planes might overflow at sq_i, the pass also writes a spare
// copy at a smaller scale, which the next pass reads if they did: a chain may move any distance
// from where it started without losing its planes.
//
// On H100 one pass of the benchmark shape (65 536 chains x 1024 dimensions) executes ~0.4 TFLOP of
// fp16 products against ~1 GB of state traffic, so the pass is compute-bound, not HBM-bound (on a
// card with a 400 W power limit it runs at the power cap, with the SM clock lowered to ~950 MHz;
// README has the numbers): the passes run as L+1 launches of the persistent tensor-core kernel
// (tc_pipeline_kernel) on alternating plane buffers, and the sampler state never leaves the plane
// format between the prepare and the select.
//
// Without sharing, every 128 x 128 unit pulls 1 MiB of operand planes from L2 (32 k-blocks of
// 32 KB), 4.3 GB per pass at the benchmark shape against 1.07 GB of HBM traffic.  Where the
// dimension blocks pair up (an even number of them) the pass runs on clusters of two CTAs on
// neighbouring dimension blocks of one chain block, which multicast that block's q planes: each
// CTA fetches half of its q tile, 3.2 GB per pass; the products and their order do not change, so
// neither do the results.  Clusters of two tile every GPC of an H100, so the pass runs on all 132
// SMs (clusters of four or eight leave 12 idle), and the benchmark card, at its power cap, does
// more work per joule on more SMs at a lower clock (README has the numbers).
#include "hmc_dense_epilogue.cuh"

namespace {

struct ResEpi {
  const __half* __restrict__ hi_cur; const __half* __restrict__ lo_cur;   // planes of q (this pass)
  __half* __restrict__ hi_nxt; __half* __restrict__ lo_nxt;               // planes of q_next
  const __half* __restrict__ hi_cur_s; const __half* __restrict__ lo_cur_s;   // spare copies
  __half* __restrict__ hi_nxt_s; __half* __restrict__ lo_nxt_s;
  const float* __restrict__ p_in; float* __restrict__ p_out;
  float* __restrict__ lp_part; float* __restrict__ k_part;
  int64_t chains; int D;
  float sq, inv_sq, acc_scale;
  float rescale;                                           // sq_alt / sq (a power of two)
};

// One warp's share of a unit: dimension n (accumulator row) against NCOL chains from c0.
//   Q   = hi + lo                      (q * sq, exact to 2^-24)
//   g   = b_n - acc_scale * acc        (acc = (P sP)(q sq) from the three products)
//   p  += s2 * g
//   Qn  = Q + (eps/m * sq) * p  -> hi' = fp16(Qn), lo' = fp16(Qn - hi')
// MODE 1 / 2 add the log-prob partial (q - mu) * g  (and the kinetic partial p^2 / m).
// SPARE: the bound says the next planes might overflow (uniform over the launch): also write the
// spare planes of Qn * rescale, and keep the exact max|Qn| (overflow iff >= 65520).
// qmax: running upper bound of |Qn| over the elements this thread wrote.  Without SPARE, on full
// tiles, it is the 2-norm of the thread's 128 elements (one FMA each; a max per element made the
// benchmark's pass ~3% slower at a 400 W power limit): >= their max, and for Gaussian-like states
// within ~2x of the max over the whole pass.  A NaN / inf element makes it infinite, which keeps
// the plane scale.
template <int MODE, int NEXT, int DC, bool SPARE>
__device__ __forceinline__ void epilogue_planes(const ResEpi& a, uint32_t trow, int n, bool n_ok,
                                                int64_t c0, int64_t part_row, int lane, float s2,
                                                float eps_over_m_sq, float inv_m, float b_n,
                                                float mu_n, float& qmax) {
  constexpr int NCOL = BN;
  const uint32_t D = DC ? (uint32_t)DC : (uint32_t)a.D;
  const int64_t chains = a.chains;
  const bool warp_n_ok = __all_sync(0xffffffffu, n_ok);
  const bool fast_tile = warp_n_ok && (c0 + NCOL <= chains);
  const int64_t off_t = c0 * (int64_t)D + n;
  const float* __restrict__ pin0 = a.p_in + off_t;
  float* __restrict__ po0 = a.p_out + off_t;
  const unsigned short* __restrict__ hc0 =
      reinterpret_cast<const unsigned short*>(a.hi_cur) + off_t;
  const unsigned short* __restrict__ lc0 =
      reinterpret_cast<const unsigned short*>(a.lo_cur) + off_t;
  __half* __restrict__ hn0 = NEXT ? a.hi_nxt + off_t : nullptr;
  __half* __restrict__ ln0 = NEXT ? a.lo_nxt + off_t : nullptr;
  __half* __restrict__ hs0 = SPARE ? a.hi_nxt_s + off_t : nullptr;
  __half* __restrict__ ls0 = SPARE ? a.lo_nxt_s + off_t : nullptr;

  auto element = [&](float acc, float p, uint32_t hl, float& pn, float& lpv, float& kv,
                     float& Qn) {
    const float Q = __half2float(__ushort_as_half((unsigned short)(hl & 0xFFFFu))) +
                    __half2float(__ushort_as_half((unsigned short)(hl >> 16)));
    const float g = b_n - a.acc_scale * acc;
    pn = fmaf(s2, g, p);
    if (MODE >= 1) lpv = (Q * a.inv_sq - mu_n) * g;
    if (MODE >= 2) kv = pn * pn * inv_m;
    if (NEXT) Qn = fmaf(eps_over_m_sq, pn, Q);
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
    // one sum of squares per software-pipeline half, so the two 16-column blocks in flight stay
    // independent
    float ss_a = 0.f, ss_b = 0.f;
    auto compute = [&](const uint32_t* v, const float* pe, const uint32_t* he, int c, float& ss) {
      const size_t cb = (size_t)c * D;
      float lpv[MODE >= 1 ? 16 : 1], kv[MODE >= 2 ? 16 : 1];
#pragma unroll
      for (int j = 0; j < 16; j += 2) {   // element pairs: one packed conversion per plane
        float pn[2], lp1[2] = {0.f, 0.f}, k1[2] = {0.f, 0.f}, Qn[2] = {0.f, 0.f};
#pragma unroll
        for (int t = 0; t < 2; ++t) {
          element(__uint_as_float(v[j + t]), pe[j + t], he[j + t], pn[t], lp1[t], k1[t], Qn[t]);
          po0[cb + (uint32_t)(j + t) * D] = pn[t];
          if (MODE >= 1) lpv[j + t] = lp1[t];
          if (MODE >= 2) kv[j + t] = k1[t];
          if (NEXT && !SPARE) ss = fmaf(Qn[t], Qn[t], ss);
          if (SPARE) qmax = fmaxf(qmax, fabsf(Qn[t]));
        }
        if (NEXT) {
          const __half2 h2 = __floats2half2_rn(Qn[0], Qn[1]);
          const float2 hf = __half22float2(h2);
          const __half2 l2 = __floats2half2_rn(Qn[0] - hf.x, Qn[1] - hf.y);
          hn0[cb + (uint32_t)j * D] = __low2half(h2);
          hn0[cb + (uint32_t)(j + 1) * D] = __high2half(h2);
          ln0[cb + (uint32_t)j * D] = __low2half(l2);
          ln0[cb + (uint32_t)(j + 1) * D] = __high2half(l2);
        }
        if (SPARE) {
          const float x0 = Qn[0] * a.rescale, x1 = Qn[1] * a.rescale;
          const __half2 h2 = __floats2half2_rn(x0, x1);
          const float2 hf = __half22float2(h2);
          const __half2 l2 = __floats2half2_rn(x0 - hf.x, x1 - hf.y);
          hs0[cb + (uint32_t)j * D] = __low2half(h2);
          hs0[cb + (uint32_t)(j + 1) * D] = __high2half(h2);
          ls0[cb + (uint32_t)j * D] = __low2half(l2);
          ls0[cb + (uint32_t)(j + 1) * D] = __high2half(l2);
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
      compute(va, pa, ha, c, ss_a);
      if (c + 32 < NCOL) load(pa, ha, c + 32);
      acc_ld16(trow + 4u * (uint32_t)(c + 16), vb);
      compute(vb, pb, hb, c + 16, ss_b);
    }
    if (NEXT && !SPARE) {
      const float norm = sqrtf(ss_a + ss_b) * (1.f + 0x1p-10f);   // covers the rounding
      qmax = fmaxf(qmax, norm == norm ? norm : INFINITY);
    }
  } else {
#pragma unroll 1
    for (int c = 0; c < NCOL; c += 16) {
      uint32_t v[16];
      acc_ld16(trow + 4u * (uint32_t)c, v);
      const int64_t cbase = c0 + c;
      if (cbase < chains) {
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
          float pn, lp1 = 0.f, k1 = 0.f, Qn = 0.f;
          element(__uint_as_float(v[j]), p, hl, pn, lp1, k1, Qn);
          const __half hh = __float2half_rn(Qn);
          const __half ll = __float2half_rn(Qn - __half2float(hh));
          if (NEXT && ok) qmax = fmaxf(qmax, fabsf(Qn));
          if (MODE >= 1) lpv[j] = ok ? lp1 : 0.f;
          if (MODE >= 2) kv[j] = ok ? k1 : 0.f;
          if (ok) {
            po0[cb + (uint32_t)j * D] = pn;
            if (NEXT) {
              hn0[cb + (uint32_t)j * D] = hh;
              ln0[cb + (uint32_t)j * D] = ll;
            }
            if (SPARE) {
              const float x = Qn * a.rescale;
              const __half hs = __float2half_rn(x);
              hs0[cb + (uint32_t)j * D] = hs;
              ls0[cb + (uint32_t)j * D] = __float2half_rn(x - __half2float(hs));
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


// What the TMA producer loads: whether this pass reads the spare planes (read from global memory
// once), and the first dimension and chain of its current unit, worked out before the unit's first
// k-block (kb_range starts every unit at 0).  The tensor cores wait on the one producer thread for
// every k-block, and tile()'s 64-bit division by the run-time number of dimension blocks, done per
// k-block, made the benchmark's pass about 6% slower on an H100 (README).
struct ProducerState {
  int spare_in, n0, c0;
};
__device__ __forceinline__ ProducerState& producer_state() {
  __shared__ ProducerState ps;
  return ps;
}

// CX x CY: a cluster takes CX dimension blocks of CY chain blocks.  Its CX CTAs on one chain block
// share that block's q planes and its CY CTAs on one dimension block share that block's P planes:
// each CTA loads 1/CX of the q tiles and 1/CY of the P tiles and multicasts them to the CTAs that
// share them, with maps whose boxes are that many rows high.
template <int MODE, int NEXT, int DC, int CX, int CY>
struct ResW {
  // 64-byte rows (32 fp16 of contraction per k-block): five 32 KB stages beside the accumulator
  // tile, so the TMA producer runs up to four k-blocks ahead of the tensor cores
  static constexpr int KIND = 1, RB = 64, MNA = 0, MNB = 0;
  static constexpr int CLUSTER = CX * CY;
  static constexpr int KE = RB / 2;
  static constexpr uint32_t TX = Cfg<RB>::STAGE;
  CUtensorMap m_phi, m_plo, m_qhi, m_qlo, m_shi, m_slo;   // m_s*: spare planes of q
  ResEpi ea;
  const float* bvec; const float* mu; const float* mass; const float* state;
  float* scales;                                           // plane-scale records
  float p_scale;
  int n_blk, D_rt, pass;
  struct EpiState { float qmax = 0.f; };

  __device__ __forceinline__ int D() const { return DC ? DC : D_rt; }
  __host__ __device__ __forceinline__ int64_t units() const {
    return ((ea.chains + BN - 1) / BN) * (int64_t)n_blk;
  }
  // unit u -> dimension block nb, chain block cb; the CTAs of a cluster take CLUSTER consecutive
  // units (n_blk % CX == 0, chain blocks % CY == 0)
  __device__ __forceinline__ void tile(int64_t u, int& nb, int64_t& cb) const {
    const uint64_t cu = (uint64_t)u / CLUSTER;
    const int r = (int)((uint64_t)u % CLUSTER);
    const uint32_t nbx = (uint32_t)(n_blk / CX);
    nb = (int)(cu % nbx) * CX + r % CX;
    cb = (int64_t)(cu / nbx) * CY + r / CX;
  }
  __device__ __forceinline__ void kb_range(int64_t, int& kb0, int& kb1) const {
    kb0 = 0;
    kb1 = D() / KE;
  }
  __device__ __forceinline__ void prefetch() const {
    tma_prefetch_desc(&m_phi); tma_prefetch_desc(&m_plo);
    tma_prefetch_desc(&m_qhi); tma_prefetch_desc(&m_qlo);
    tma_prefetch_desc(&m_shi); tma_prefetch_desc(&m_slo);
    producer_state().spare_in = plane_spare_in(scales, pass);   // prefetch runs on the producer
  }
  __device__ __forceinline__ void load(int64_t u, int kb, uint32_t sa, uint32_t fb) const {
    using C = Cfg<RB>;
    ProducerState& ps = producer_state();
    if (kb == 0) {
      int nb;
      int64_t cb;
      tile(u, nb, cb);
      ps.n0 = nb * BM;
      ps.c0 = (int)cb * BN;
    }
    const int n0 = ps.n0, c0 = ps.c0;
    const bool s = ps.spare_in != 0;
    const CUtensorMap* qh = s ? &m_shi : &m_qhi;
    const CUtensorMap* ql = s ? &m_slo : &m_qlo;
    const int r = (int)(u % CLUSTER), rx = r % CX, ry = r / CX;   // this CTA's cluster rank
    if constexpr (CY == 1) {
      tma_load_2d(sa, &m_phi, fb, kb * KE, n0);
      tma_load_2d(sa + C::A_TILE, &m_plo, fb, kb * KE, n0);
    } else {
      constexpr int rows = BM / CY;
      uint16_t mask = 0;                                   // the CTAs on dimension block nb
#pragma unroll
      for (int y = 0; y < CY; ++y) mask |= (uint16_t)(1u << (y * CX + rx));
      const uint32_t o = (uint32_t)(ry * rows * RB);
      tma_load_2d_mc(sa + o, &m_phi, fb, kb * KE, n0 + ry * rows, mask);
      tma_load_2d_mc(sa + C::A_TILE + o, &m_plo, fb, kb * KE, n0 + ry * rows, mask);
    }
    if constexpr (CX == 1) {
      tma_load_2d(sa + 2 * C::A_TILE, qh, fb, kb * KE, c0);
      tma_load_2d(sa + 2 * C::A_TILE + C::B_TILE, ql, fb, kb * KE, c0);
    } else {
      constexpr int rows = BN / CX;
      const uint16_t mask = (uint16_t)(((1u << CX) - 1u) << (ry * CX));   // on chain block cb
      const uint32_t o = (uint32_t)(rx * rows * RB);
      tma_load_2d_mc(sa + 2 * C::A_TILE + o, qh, fb, kb * KE, c0 + rx * rows, mask);
      tma_load_2d_mc(sa + 2 * C::A_TILE + C::B_TILE + o, ql, fb, kb * KE, c0 + rx * rows, mask);
    }
  }
  __device__ __forceinline__ float sq_alt(float eps, float sq) const {
    return next_plane_scale(scales, pass, eps, mul(eps, p_scale), sq);
  }
  __device__ __forceinline__ void epilogue(int64_t u, uint32_t trow, int quarter, int lane,
                                           EpiState& st) const {
    int nb;
    int64_t cb;
    tile(u, nb, cb);
    const int n = nb * BM + quarter * 32 + lane;
    const int64_t c0 = cb * BN;
    const bool n_ok = n < D();
    const float eps = state[ZSB_ST_EPS_USED];
    const float s2 = mul(eps, p_scale);
    const bool spare_in = plane_spare_in(scales, pass);
    const float sq = plane_scale_in(scales, pass);
    const float m_n = n_ok ? mass[n] : 1.f;
    const float eps_over_m_sq = mul(fdiv(eps, m_n), sq);
    const float inv_m = fdiv(1.f, m_n);
    const float b_n = (n_ok && bvec) ? bvec[n] : 0.f;
    const float mu_n = (n_ok && mu) ? mu[n] : 0.f;
    const int64_t part_row = (int64_t)(nb * 4 + quarter) * ea.chains;
    ResEpi a = ea;
    if (spare_in) {
      a.hi_cur = ea.hi_cur_s;
      a.lo_cur = ea.lo_cur_s;
    }
    a.sq = sq;
    a.inv_sq = fdiv(1.f, sq);
    a.acc_scale = 1.f / (scales[3] * sq);                   // powers of two: exact
    a.rescale = NEXT ? sq_alt(eps, sq) * a.inv_sq : 1.f;
    if (a.rescale == 1.f)
      epilogue_planes<MODE, NEXT, DC, false>(a, trow, n, n_ok, c0, part_row, lane, s2,
                                             eps_over_m_sq, inv_m, b_n, mu_n, st.qmax);
    else
      epilogue_planes<MODE, NEXT, DC, true>(a, trow, n, n_ok, c0, part_row, lane, s2,
                                            eps_over_m_sq, inv_m, b_n, mu_n, st.qmax);
  }
  __device__ __forceinline__ void epi_finish(EpiState& st, int quarter, int lane) const {
    if (!NEXT) return;
    const float sq = plane_scale_in(scales, pass);
    const float alt = sq_alt(state[ZSB_ST_EPS_USED], sq);
    // qmax is exact when there is a spare copy: the planes at sq overflowed iff it reached 65520
    publish_plane_scale(scales, pass, sq, alt, st.qmax * (1.f / sq),
                        alt != sq && !(st.qmax < kHalfOverflow), quarter, lane);
  }
};

// Cluster shape of the pass (CX dimension blocks x CY chain blocks) where the unit grid tiles by
// it; other shapes run without clusters.  On a 700 W H100 2 x 1 (or 1 x 2) ran the benchmark's
// pass faster than 1 x 1, 2 x 2, 2 x 4 and 4 x 2 (README).
constexpr int RES_CX = 2, RES_CY = 1;

template <int DC, int CX, int CY>
int res_pass(const CUtensorMap& phi, const CUtensorMap& plo, const CUtensorMap& qhi,
             const CUtensorMap& qlo, const CUtensorMap& shi, const CUtensorMap& slo,
             const ResEpi& ea, const float* bvec, const float* mu, const float* mass,
             const float* state, float* scales, int pass, float p_scale, int n_blk, int D,
             int mode, cudaStream_t st) {
  if (mode == 1) {
    const ResW<1, 1, DC, CX, CY> w{phi, plo, qhi, qlo, shi, slo, ea, bvec, mu, mass, state,
                                   scales, p_scale, n_blk, D, pass};
    return tc_launch(w, st, "hmc_dense_resident");
  }
  if (mode == 0) {
    const ResW<0, 1, DC, CX, CY> w{phi, plo, qhi, qlo, shi, slo, ea, bvec, mu, mass, state,
                                   scales, p_scale, n_blk, D, pass};
    return tc_launch(w, st, "hmc_dense_resident");
  }
  const ResW<2, 0, DC, CX, CY> w{phi, plo, qhi, qlo, shi, slo, ea, bvec, mu, mass, state, scales,
                                 p_scale, n_blk, D, pass};
  return tc_launch(w, st, "hmc_dense_resident");
}

template <int DC>
int res_pass(bool cluster, const CUtensorMap& phi, const CUtensorMap& plo, const CUtensorMap& qhi,
             const CUtensorMap& qlo, const CUtensorMap& shi, const CUtensorMap& slo,
             const ResEpi& ea, const float* bvec, const float* mu, const float* mass,
             const float* state, float* scales, int pass, float p_scale, int n_blk, int D,
             int mode, cudaStream_t st) {
  return cluster ? res_pass<DC, RES_CX, RES_CY>(phi, plo, qhi, qlo, shi, slo, ea, bvec, mu, mass,
                                                state, scales, pass, p_scale, n_blk, D, mode, st)
                 : res_pass<DC, 1, 1>(phi, plo, qhi, qlo, shi, slo, ea, bvec, mu, mass, state,
                                      scales, pass, p_scale, n_blk, D, mode, st);
}

// q[c, :] <- (hi + lo) / sq of the proposal planes where accept[c] (hmc.py:488-497).  `record` is
// the proposal's plane-scale record: the planes are in `planes` at record[0], or, when its
// overflow flag is set, in `spare` at record[1].
// One warp per chain at a time (the accept flag is warp-uniform: a rejected chain costs one 4-byte
// load), 8 dimensions per lane and step: two 128-bit plane loads in, two 128-bit stores out, up to
// four steps' loads issued before the first use.  D % 8 == 0 (the dense kernels need D % 64 == 0).
__global__ void __launch_bounds__(256) select_planes_kernel(float* __restrict__ q,
                                                            const __half* __restrict__ planes,
                                                            const __half* __restrict__ spare,
                                                            const float* __restrict__ record,
                                                            const int32_t* __restrict__ accept,
                                                            int64_t chains, int64_t D) {
  const bool use_spare = __float_as_uint(record[3]) != 0u;
  const float inv_sq = 1.f / record[use_spare ? 1 : 0];
  if (use_spare) planes = spare;
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

// The L+1 passes of a trajectory for every chain (D % 64 == 0, L >= 1).
//   planes0: fp16 hi/lo planes of q * sq_0 (zsb_hmc_dense_traj_prepare_f32), planes1: work buffer
//   of the same size (must differ from planes0: a pass reads every dimension of a chain block's
//   planes while other tiles of the same launch write the next ones); on return the proposal's
//   planes are in buffer (L & 1), or in spare buffer (L & 1) when record L flags them; spare0 / spare1: two
//   more buffers of that size for the spare copies; p0 -> pw (final momentum); lp0_part /
//   lp1_part / k_part as the per-pass kernel writes them; pass i writes plane-scale record i + 1.
int zsb_dense_res_h16_launch(void* planes0, void* planes1, void* spare0, void* spare1,
                             const float* p0, float* pw,
                             const void* P_h16, const void* P_l16, float* scales,
                             const float* bvec, const float* mu, const float* mass,
                             const float* state, float* lp0_part, float* lp1_part, float* k_part,
                             int64_t chains, int D, int L, cudaStream_t st) {
  if (D % 64 != 0 || D < 64 || L < 1 || chains <= 0 || chains >= (1LL << 31)) {
    zsb_set_error("dense_res: needs D %% 64 == 0, n_leapfrogs >= 1");
    return ZSB_ERR_INVALID;
  }
  if (planes0 == planes1 || !spare0 || !spare1 || spare0 == spare1) {
    zsb_set_error("dense_res: planes1, spare0 and spare1 must be separate work buffers");
    return ZSB_ERR_INVALID;
  }
  const int n_blk = (D + BM - 1) / BM;
  const int64_t c_blk = (chains + BN - 1) / BN;
  const bool cluster = n_blk % RES_CX == 0 && c_blk % RES_CY == 0;
  const uint32_t p_box = cluster ? BM / RES_CY : BM, q_box = cluster ? BN / RES_CX : BN;
  CUtensorMap phi, plo, qhi[2], qlo[2], shi[2], slo[2];
  int rc;
  constexpr int RB = ResW<0, 1, 0, 1, 1>::RB;
  if ((rc = make_map(&phi, P_h16, (uint64_t)D, (uint64_t)D, p_box, RB, 1))) return rc;
  if ((rc = make_map(&plo, P_l16, (uint64_t)D, (uint64_t)D, p_box, RB, 1))) return rc;
  __half* pl[2] = {reinterpret_cast<__half*>(planes0), reinterpret_cast<__half*>(planes1)};
  __half* sp[2] = {reinterpret_cast<__half*>(spare0), reinterpret_cast<__half*>(spare1)};
  const int64_t plane = chains * (int64_t)D;
  for (int b = 0; b < 2; ++b) {
    if ((rc = make_map(&qhi[b], pl[b], (uint64_t)chains, (uint64_t)D, q_box, RB, 1))) return rc;
    if ((rc = make_map(&qlo[b], pl[b] + plane, (uint64_t)chains, (uint64_t)D, q_box, RB, 1)))
      return rc;
    if ((rc = make_map(&shi[b], sp[b], (uint64_t)chains, (uint64_t)D, q_box, RB, 1))) return rc;
    if ((rc = make_map(&slo[b], sp[b] + plane, (uint64_t)chains, (uint64_t)D, q_box, RB, 1)))
      return rc;
  }
  for (int i = 0; i <= L; ++i) {
    const bool last = i == L;
    const int buf = i & 1;
    const ResEpi ea{pl[buf], pl[buf] + plane, pl[buf ^ 1], pl[buf ^ 1] + plane,
                    sp[buf], sp[buf] + plane, sp[buf ^ 1], sp[buf ^ 1] + plane,
                    i == 0 ? p0 : pw, pw, i == 0 ? lp0_part : lp1_part, k_part, chains, D,
                    1.f, 1.f, 1.f, 1.f};
    const int mode = last ? 2 : (i == 0 ? 1 : 0);
    const float p_scale = (i > 0 && !last) ? 1.f : 0.5f;
    rc = (D == 1024)
             ? res_pass<1024>(cluster, phi, plo, qhi[buf], qlo[buf], shi[buf], slo[buf], ea, bvec,
                              mu, mass, state, scales, i, p_scale, n_blk, D, mode, st)
             : res_pass<0>(cluster, phi, plo, qhi[buf], qlo[buf], shi[buf], slo[buf], ea, bvec, mu,
                           mass, state, scales, i, p_scale, n_blk, D, mode, st);
    if (rc != ZSB_OK) return rc;
  }
  return ZSB_OK;
}

#ifdef ZSB_PASS_PROFILE
// Stall accounting build only (tc_common.cuh): copy the per-CTA counters of the dense pass
// kernels, PASS_PROF_SLOTS per CTA for the first `ctas` CTAs, to `host` and clear them.
extern "C" int zsb_pass_profile_read(unsigned long long* host, int ctas) {
  if (ctas < 0 || ctas > PASS_PROF_CTAS) return ZSB_ERR_INVALID;
  const size_t bytes = sizeof(unsigned long long) * PASS_PROF_SLOTS * (size_t)ctas;
  if (cudaMemcpyFromSymbol(host, g_pass_prof, bytes) != cudaSuccess) return ZSB_ERR_CUDA;
  static unsigned long long zeros[PASS_PROF_CTAS * PASS_PROF_SLOTS];
  if (cudaMemcpyToSymbol(g_pass_prof, zeros, sizeof(zeros)) != cudaSuccess) return ZSB_ERR_CUDA;
  return ZSB_OK;
}
#endif

int zsb_dense_select_planes_launch(float* q, const void* planes, const void* spare,
                                   const float* record, const int32_t* accept, int64_t chains,
                                   int64_t D, cudaStream_t st) {
  ZSB_REQUIRE(D % 8 == 0, "zsb_dense_select_planes: D must be a multiple of 8");
  int64_t blocks = zsb_ceil_div(chains, 8);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  if (blocks < 1) blocks = 1;
  select_planes_kernel<<<(unsigned)blocks, 256, 0, st>>>(
      q, reinterpret_cast<const __half*>(planes), reinterpret_cast<const __half*>(spare), record,
      accept, chains, D);
  return zsb_check_launch("hmc_select_planes");
}
