// Replaces, for a dense-Gaussian log-joint, one iteration of the leapfrog `tf.while_loop` of
// zhusuan/hmc.py:347-372 (body = leapfrog_integrator, hmc.py:38-43: q += eps1 * p / mass;
// g = tf.gradients(log_posterior, q); p += eps2 * g) plus the log p / kinetic terms of
// hamiltonian(), hmc.py:30-35, which get_acceptance_rate (hmc.py:46-61) would otherwise
// recompute with two extra forward evaluations.
//
// Dense-Gaussian leapfrog pass on the Hopper tensor cores (wgmma, tc_pipeline_kernel of
// tc_common.cuh) with a three-product split so the fp32 gradient  g = b - P q  keeps ~fp32 accuracy:
//   impl 1  TF32 operands:  q = q_hi + q_lo,  P = P_hi + P_lo  (hi = top 19 bits, what the TF32
//           datapath reads);  P q ~= P_hi q_hi + P_hi q_lo + P_lo q_hi  (dropped term ~2^-22)
//   impl 2  fp16 operands:  hi / lo planes of P*sP and q*sq (powers of two), three fp16 products at
//           twice the TF32 rate; the pass writes the planes of q_next for the next pass
//   impl 3  as impl 2, but the MMA warpgroup builds the planes of q from the fp32 rows itself
//           (no plane buffers in HBM); sq comes from the running max|q| the previous pass left
// The GEMM is computed TRANSPOSED, G^T[n, c] = sum_k P[n, k] q[c, k]  (A = P rows, B = chain rows,
// both K-major), so an accumulator row is a dimension n and a column a chain c: an epilogue warp
// then touches 32 consecutive dimensions of ONE chain per instruction -- a full 128-byte line of
// p / q / q_next -- instead of 32 chains 4 KB apart.  Tiles (128 dims x 128 chains) are assigned
// round-robin with the dimension block fastest, so the CTAs running concurrently share their chain
// rows and P through the L2.
#include "hmc_dense_epilogue.cuh"

namespace {

// OP 0: TF32 (impl 1), 1: fp16 planes (impl 2).  H16: epilogue flavour (0 TF32 residual, 1 fp16
// planes, 2 in-kernel split: q_next fp32 + running max|q_next|).  RB_: smem row bytes.
template <int OP, int RB_, int MODE, int DC, int H16>
struct DenseW {
  static constexpr int KIND = OP, RB = RB_, MNA = 0, MNB = 0, CVT = (H16 == 2);
  static constexpr int KE = OP ? RB / 2 : RB / 4;          // contraction elements per k-block
  static constexpr uint32_t TX = CVT ? 2 * Cfg<RB>::A_TILE : Cfg<RB>::STAGE;
  CUtensorMap m_phi, m_plo, m_qhi, m_qlo;
  EpiArgs ea;
  const float* bvec; const float* mu; const float* mass; const float* state;
  float* scales;                                           // OP 1: {sq, 1/(sP sq), -, sP, slots}
  float p_scale;
  int n_blk, D_rt, pass_index;
  struct EpiState { float amax = 0.f; };

  __device__ __forceinline__ int D() const { return DC ? DC : D_rt; }
  __host__ __device__ __forceinline__ int64_t units() const {
    return ((ea.chains + BN - 1) / BN) * (int64_t)n_blk;
  }
  __device__ __forceinline__ void kb_range(int64_t, int& kb0, int& kb1) const {
    kb0 = 0;
    kb1 = D() / KE;
  }
  __device__ __forceinline__ void prefetch() const {
    tma_prefetch_desc(&m_phi);
    tma_prefetch_desc(&m_plo);
    if (!CVT) { tma_prefetch_desc(&m_qhi); tma_prefetch_desc(&m_qlo); }
  }
  __device__ __forceinline__ void load(int64_t u, int kb, uint32_t sa, uint32_t fb) const {
    using C = Cfg<RB>;
    const int n0 = (int)(u % n_blk) * BM;
    const int c0 = (int)(u / n_blk) * BN;
    tma_load_2d(sa, &m_phi, fb, kb * KE, n0);
    tma_load_2d(sa + C::A_TILE, &m_plo, fb, kb * KE, n0);
    if (!CVT) {
      tma_load_2d(sa + 2 * C::A_TILE, &m_qhi, fb, kb * KE, c0);
      tma_load_2d(sa + 2 * C::A_TILE + C::B_TILE, &m_qlo, fb, kb * KE, c0);
    }
  }
  // impl 3: scale of this pass's q from the running-max slot the previous pass (or prepare) filled
  __device__ __forceinline__ float sq3() const {
    const unsigned int* slots = reinterpret_cast<const unsigned int*>(scales) + 4;
    const float qmax = __uint_as_float(slots[pass_index % 3]);
    int qe = 0;
    if (qmax > 0.f) frexpf(qmax, &qe);
    return ldexpf(1.f, 12 - qe);                          // max|q| * sq in [2^11, 2^12)
  }
  // impl 3: thread `tid` converts chain c0 + tid, contraction kb*KE .. +KE, into the B planes in
  // the SWIZZLE_128B K-major layout (16-byte chunk index XOR row % 8)
  __device__ __forceinline__ void convert(int64_t u, int kb, uint8_t* stage, int tid) const {
    if (!CVT) return;
    using C = Cfg<RB>;
    static_assert(!CVT || RB == 128, "in-kernel split uses 128-byte rows");
    const float sq = sq3();
    const int64_t c = (u / n_blk) * BN + tid;
    const bool ok = c < ea.chains;
    const float4* src = reinterpret_cast<const float4*>(ea.q_cur + (ok ? c : 0) * (int64_t)D() +
                                                        (int64_t)kb * KE);
    uint8_t* hi = stage + 2 * C::A_TILE + tid * RB;
    uint8_t* lo = hi + C::B_TILE;
#pragma unroll
    for (int ch = 0; ch < RB / 16; ++ch) {                 // 8 halves per 16-byte chunk
      const float4 a = ok ? __ldg(src + 2 * ch) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float4 b = ok ? __ldg(src + 2 * ch + 1) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float x[8] = {a.x * sq, a.y * sq, a.z * sq, a.w * sq,
                          b.x * sq, b.y * sq, b.z * sq, b.w * sq};
      uint32_t h[4], l[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const __half2 h2 = __floats2half2_rn(x[2 * i], x[2 * i + 1]);
        const float2 hf = __half22float2(h2);
        const __half2 l2 = __floats2half2_rn(x[2 * i] - hf.x, x[2 * i + 1] - hf.y);
        h[i] = *reinterpret_cast<const uint32_t*>(&h2);
        l[i] = *reinterpret_cast<const uint32_t*>(&l2);
      }
      const int off = ((ch ^ (tid & 7)) << 4);
      *reinterpret_cast<uint4*>(hi + off) = make_uint4(h[0], h[1], h[2], h[3]);
      *reinterpret_cast<uint4*>(lo + off) = make_uint4(l[0], l[1], l[2], l[3]);
    }
  }
  __device__ __forceinline__ void epilogue(int64_t u, uint32_t trow, int quarter, int lane,
                                           EpiState& st) const {
    const int nb = (int)(u % n_blk);
    const int n = nb * BM + quarter * 32 + lane;          // this thread's dimension
    const int64_t c0 = (u / n_blk) * BN;
    const int Dv = D();
    const bool n_ok = n < Dv;
    const float eps = state[ZSB_ST_EPS_USED];
    const float s2 = mul(eps, p_scale);
    const float m_n = n_ok ? mass[n] : 1.f;
    const float eps_over_m = fdiv(eps, m_n);              // q += eps * (p / m) as p * (eps / m)
    const float inv_m = fdiv(1.f, m_n);
    const float b_n = (n_ok && bvec) ? bvec[n] : 0.f;
    const float mu_n = (n_ok && mu) ? mu[n] : 0.f;
    const int64_t part_row = (int64_t)(nb * 4 + quarter) * ea.chains;
    EpiArgs a = ea;
    if (H16 == 1) { a.q_scale = scales[0]; a.acc_scale = scales[1]; }
    if (H16 == 2) a.acc_scale = 1.f / (scales[3] * sq3());   // powers of two: exact
    epilogue_half_tile<MODE, -1, DC, H16>(a, trow, n, n_ok, true, c0, part_row, lane, s2,
                                          eps_over_m, inv_m, b_n, mu_n, false, st.amax);
  }
  __device__ __forceinline__ void epi_finish(EpiState& st, int quarter, int lane) const {
    if (H16 != 2) return;
    unsigned int* slots = reinterpret_cast<unsigned int*>(scales) + 4;
    if (ea.q_next) {
      const float m = warp_max(st.amax);
      if (lane == 0) atomicMax(slots + (pass_index + 1) % 3, __float_as_uint(m));
    }
    if (blockIdx.x == 0 && quarter == 0 && lane == 0) slots[(pass_index + 2) % 3] = 0u;
  }
};

// q_lo = q - (q with the low 13 mantissa bits cleared): the residual the TF32 datapath drops.
__global__ void __launch_bounds__(256) split_lo_kernel(const float* __restrict__ q,
                                                       float* __restrict__ lo, int64_t n4) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = reinterpret_cast<const float4*>(q)[i];
    float4 r;
    r.x = v.x - __uint_as_float(__float_as_uint(v.x) & 0xFFFFE000u);
    r.y = v.y - __uint_as_float(__float_as_uint(v.y) & 0xFFFFE000u);
    r.z = v.z - __uint_as_float(__float_as_uint(v.z) & 0xFFFFE000u);
    r.w = v.w - __uint_as_float(__float_as_uint(v.w) & 0xFFFFE000u);
    reinterpret_cast<float4*>(lo)[i] = r;
  }
}

// fp16-split support (impl 2).  scales[0] = sq (power of two putting max|q| near 2^12: three bits of
// head-room below fp16's 2^15 so q may grow 8x inside a trajectory), scales[1] = 1/(sP*sq),
// scales[2] = running max|q| bits (uint), scales[3] = sP.
__global__ void __launch_bounds__(256) absmax_kernel(const float* __restrict__ q, int64_t n,
                                                     float* __restrict__ scales) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float a = fabsf(q[i]);
    m = (a == a && a <= 3.0e38f) ? fmaxf(m, a) : m;       // ignore NaN / inf
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0)
    atomicMax(reinterpret_cast<unsigned int*>(scales) + 2, __float_as_uint(m));
}
__global__ void scale_kernel(float* __restrict__ scales) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const float m = __uint_as_float(reinterpret_cast<unsigned int*>(scales)[2]);
  int e = 0;
  if (m > 0.f) frexpf(m, &e);              // m = f * 2^e, f in [0.5, 1)  ->  m < 2^e
  const float sq = ldexpf(1.f, 12 - e);    // max|q| * sq in [2^11, 2^12)
  scales[0] = sq;
  scales[1] = 1.f / (scales[3] * sq);
  reinterpret_cast<unsigned int*>(scales)[2] = 0u;   // reset the running max for the next call
}
__global__ void __launch_bounds__(256) split16_kernel(const float* __restrict__ q,
                                                      __half* __restrict__ planes, int64_t n,
                                                      const float* __restrict__ scales) {
  const float sq = scales[0];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float x = q[i] * sq;
    const __half h = __float2half_rn(x);
    planes[i] = h;
    planes[n + i] = __float2half_rn(x - __half2float(h));
  }
}

// seeds running-max slot 0 with max|q| and clears slots 1, 2 (scales[4..6])
__global__ void __launch_bounds__(256) absmax_slot_kernel(const float* __restrict__ q, int64_t n,
                                                          float* __restrict__ scales) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float a = fabsf(q[i]);
    m = (a <= 3.0e38f) ? fmaxf(m, a) : m;
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0)
    atomicMax(reinterpret_cast<unsigned int*>(scales) + 4, __float_as_uint(m));
}
__global__ void clear_slots_kernel(float* __restrict__ scales) {
  if (threadIdx.x < 3 && blockIdx.x == 0) reinterpret_cast<unsigned int*>(scales)[4 + threadIdx.x] = 0u;
}


int g_tc_bk = 32;   // impl-1 pipeline shape: 32 -> 128-byte rows (2 stages), 16 -> 64-byte (4)

// one pass on the tensor cores; q_lo: impl 1 TF32 residual of q_cur / impl 2 its fp16 planes
template <int OP, int RB, int H16>
int launch_dense(const float* q_cur, const void* q_lo, float* q_next, void* q_next_lo,
                 const float* p_in, float* p_out, const void* P_hi, const void* P_lo,
                 const float* bvec, const float* mu, const float* mass, const float* state,
                 float p_scale, float* lp_part, float* k_part, int64_t chains, int D, float* scales,
                 int pass_index, cudaStream_t st, const char* what) {
  if (k_part && !lp_part) {
    zsb_set_error("%s: k_part requires lp_part", what);
    return ZSB_ERR_INVALID;
  }
  CUtensorMap m_phi, m_plo, m_qhi, m_qlo;
  int rc;
  if ((rc = make_map(&m_phi, P_hi, (uint64_t)D, (uint64_t)D, BM, RB, OP))) return rc;
  if ((rc = make_map(&m_plo, P_lo, (uint64_t)D, (uint64_t)D, BM, RB, OP))) return rc;
  m_qhi = m_phi;
  m_qlo = m_plo;
  if (H16 != 2) {
    const void* qh = OP ? q_lo : (const void*)q_cur;
    const void* ql = OP ? (const void*)(reinterpret_cast<const __half*>(q_lo) + chains * D) : q_lo;
    if ((rc = make_map(&m_qhi, qh, (uint64_t)chains, (uint64_t)D, BN, RB, OP))) return rc;
    if ((rc = make_map(&m_qlo, ql, (uint64_t)chains, (uint64_t)D, BN, RB, OP))) return rc;
  }
  const EpiArgs ea{q_cur, q_next, reinterpret_cast<float*>(q_next_lo), p_in, p_out, lp_part,
                   k_part, chains, D, H16, 1.f, 1.f};
  const int n_blk = (D + BM - 1) / BM;
#define ZSB_DENSE(MODE, DCV)                                                                   \
  do {                                                                                         \
    const DenseW<OP, RB, MODE, DCV, H16> w{m_phi, m_plo, m_qhi, m_qlo, ea, bvec, mu, mass,     \
                                           state, scales, p_scale, n_blk, D, pass_index};      \
    return tc_launch(w, st, what);                                                             \
  } while (0)
#define ZSB_DENSE_MODE(DCV)                                                                    \
  do {                                                                                         \
    if (k_part) ZSB_DENSE(2, DCV);                                                             \
    else if (lp_part) ZSB_DENSE(1, DCV);                                                       \
    else ZSB_DENSE(0, DCV);                                                                    \
  } while (0)
  // the benchmark's dimension count is also compiled as a constant: the epilogue's per-column
  // offsets become immediates
  if constexpr (OP == 1 && H16 == 1)
    if (D == 1024) ZSB_DENSE_MODE(1024);
  ZSB_DENSE_MODE(0);
#undef ZSB_DENSE_MODE
#undef ZSB_DENSE
}

}  // namespace

// rows of the [parts, chains] lp/K partial scratch: 4 warp-quarters per 128-dimension block
int zsb_dense_tc_ntiles(int D) { return 4 * ((D + BM - 1) / BM); }

int zsb_dense_tc_set_bk(int cfg) {
  const int bk = cfg & 0xFF;
  if (bk != 16 && bk != 32) return ZSB_ERR_INVALID;
  g_tc_bk = bk;
  return ZSB_OK;
}

// `q_cur_lo` must hold the TF32 residual of q_cur on entry; the kernel writes q_next's residual to
// `q_next_lo`.
int zsb_dense_leapfrog_tc_launch(const float* q_cur, const float* q_cur_lo, float* q_next,
                                 float* q_next_lo, const float* p_in, float* p_out,
                                 const float* P_hi, const float* P_lo, const float* bvec,
                                 const float* mu, const float* mass, const float* state,
                                 float p_scale, float* lp_part, float* k_part, int64_t chains,
                                 int D, cudaStream_t st) {
  if (D % 32 != 0 || D < 32) {
    zsb_set_error("dense_tc: D must be a multiple of 32");
    return ZSB_ERR_INVALID;
  }
  if (chains >= (1LL << 31) || (q_next && !q_next_lo) || !q_cur_lo) {
    zsb_set_error("dense_tc: bad arguments");
    return ZSB_ERR_INVALID;
  }
  if (g_tc_bk == 16)
    return launch_dense<0, 64, 0>(q_cur, q_cur_lo, q_next, q_next_lo, p_in, p_out, P_hi, P_lo,
                                  bvec, mu, mass, state, p_scale, lp_part, k_part, chains, D,
                                  nullptr, 0, st, "hmc_dense_leapfrog_tc");
  return launch_dense<0, 128, 0>(q_cur, q_cur_lo, q_next, q_next_lo, p_in, p_out, P_hi, P_lo,
                                 bvec, mu, mass, state, p_scale, lp_part, k_part, chains, D,
                                 nullptr, 0, st, "hmc_dense_leapfrog_tc");
}

int zsb_dense_split_lo_launch(const float* q, float* lo, int64_t n, cudaStream_t st) {
  if (n % 4 != 0) {
    zsb_set_error("dense split: element count must be a multiple of 4");
    return ZSB_ERR_INVALID;
  }
  const int64_t n4 = n / 4;
  int64_t blocks = zsb_ceil_div(n4, 256);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  if (blocks < 1) blocks = 1;
  split_lo_kernel<<<(unsigned)blocks, 256, 0, st>>>(q, lo, n4);
  return zsb_check_launch("hmc_dense_split_lo");
}

// ---- impl 2: fp16-split operands ----
int zsb_dense_leapfrog_h16_launch(const float* q_cur, const void* q_cur_planes, float* q_next,
                                  void* q_next_planes, const float* p_in, float* p_out,
                                  const void* P_h16, const void* P_l16, const float* scales,
                                  const float* bvec, const float* mu, const float* mass,
                                  const float* state, float p_scale, float* lp_part, float* k_part,
                                  int64_t chains, int D, cudaStream_t st) {
  if (D % 64 != 0 || D < 64) {
    zsb_set_error("dense_h16: D must be a multiple of 64");
    return ZSB_ERR_INVALID;
  }
  if (chains >= (1LL << 31) || (q_next && !q_next_planes) || !q_cur_planes || !scales) {
    zsb_set_error("dense_h16: bad arguments");
    return ZSB_ERR_INVALID;
  }
  return launch_dense<1, 128, 1>(q_cur, q_cur_planes, q_next, q_next_planes, p_in, p_out, P_h16,
                                 P_l16, bvec, mu, mass, state, p_scale, lp_part, k_part, chains, D,
                                 const_cast<float*>(scales), 0, st, "hmc_dense_leapfrog_h16");
}

// impl 3 (in-kernel split).  scales: float[8] device scratch with scales[3] = sP.
int zsb_dense_leapfrog_h16i_launch(const float* q_cur, float* q_next, const float* p_in,
                                   float* p_out, const void* P_h16, const void* P_l16,
                                   float* scales, int pass_index, const float* bvec,
                                   const float* mu, const float* mass, const float* state,
                                   float p_scale, float* lp_part, float* k_part, int64_t chains,
                                   int D, cudaStream_t st) {
  if (D % 64 != 0 || D < 64) {
    zsb_set_error("dense_h16i: D must be a multiple of 64");
    return ZSB_ERR_INVALID;
  }
  if (chains >= (1LL << 31) || !scales || pass_index < 0) {
    zsb_set_error("dense_h16i: bad arguments");
    return ZSB_ERR_INVALID;
  }
  return launch_dense<1, 128, 2>(q_cur, nullptr, q_next, nullptr, p_in, p_out, P_h16, P_l16, bvec,
                                 mu, mass, state, p_scale, lp_part, k_part, chains, D, scales,
                                 pass_index, st, "hmc_dense_leapfrog_h16i");
}
int zsb_dense_h16i_prepare_launch(const float* q, float* scales, int64_t n, cudaStream_t st) {
  int64_t blocks = zsb_ceil_div(n, 256 * 8);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  if (blocks < 1) blocks = 1;
  clear_slots_kernel<<<1, 32, 0, st>>>(scales);
  absmax_slot_kernel<<<(unsigned)blocks, 256, 0, st>>>(q, n, scales);
  return zsb_check_launch("hmc_dense_h16i_prepare");
}

// scales[3] must hold sP on entry; computes sq from max|q| and writes the fp16 hi/lo planes.
int zsb_dense_h16_prepare_launch(const float* q, void* planes, float* scales, int64_t n,
                                 cudaStream_t st) {
  int64_t blocks = zsb_ceil_div(n, 256 * 8);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  if (blocks < 1) blocks = 1;
  absmax_kernel<<<(unsigned)blocks, 256, 0, st>>>(q, n, scales);
  scale_kernel<<<1, 32, 0, st>>>(scales);
  split16_kernel<<<(unsigned)blocks, 256, 0, st>>>(q, reinterpret_cast<__half*>(planes), n, scales);
  return zsb_check_launch("hmc_dense_h16_prepare");
}
