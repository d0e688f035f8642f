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
//           twice the TF32 rate; the pass writes the planes of q_next for the next pass, at the
//           scale the a-priori bound on |q_next| gives (hmc_dense_epilogue.cuh)
// The GEMM is computed TRANSPOSED, G^T[n, c] = sum_k P[n, k] q[c, k]  (A = P rows, B = chain rows,
// both K-major), so an accumulator row is a dimension n and a column a chain c: an epilogue warp
// then touches 32 consecutive dimensions of ONE chain per instruction -- a full 128-byte line of
// p / q / q_next -- instead of 32 chains 4 KB apart.  Tiles (128 dims x 128 chains) are assigned
// round-robin with the dimension block fastest, so the CTAs running concurrently share their chain
// rows and P through the L2.
#include "hmc_dense_epilogue.cuh"

namespace {

// OP 0: TF32 (impl 1), 1: fp16 planes (impl 2).  Both run on 128-byte smem rows.
template <int OP, int MODE, int DC>
struct DenseW {
  static constexpr int KIND = OP, RB = 128, MNA = 0, MNB = 0;
  static constexpr int KE = OP ? RB / 2 : RB / 4;          // contraction elements per k-block
  static constexpr uint32_t TX = Cfg<RB>::STAGE;
  CUtensorMap m_phi, m_plo, m_qhi, m_qlo;
  EpiArgs ea;
  const float* bvec; const float* mu; const float* mass; const float* state;
  float* scales;             // OP 1: plane-scale records (hmc_dense_epilogue.cuh)
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
    tma_prefetch_desc(&m_qhi);
    tma_prefetch_desc(&m_qlo);
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
    if (OP == 1) {   // planes of q_cur at sq_i, those of q_next at sq_alt
      const float sq = scale_rec(scales, pass_index)[0];
      a.acc_scale = 1.f / (scales[3] * sq);                  // powers of two: exact
      a.q_scale = ea.q_next ? next_plane_scale(scales, pass_index, eps, s2, sq) : sq;
    }
    epilogue_half_tile<MODE, DC, OP>(a, trow, n, n_ok, c0, part_row, lane, s2, eps_over_m, inv_m,
                                     b_n, mu_n, st.amax);
  }
  __device__ __forceinline__ void epi_finish(EpiState& st, int quarter, int lane) const {
    if (OP == 1 && ea.q_next) {
      const float eps = state[ZSB_ST_EPS_USED];
      const float sq = next_plane_scale(scales, pass_index, eps, mul(eps, p_scale),
                                        scale_rec(scales, pass_index)[0]);
      publish_plane_scale(scales, pass_index, sq, sq, st.amax, false, quarter, lane);
    }
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

// fp16-split support (impl 2, 5).  sq_0 is the power of two putting max|q0| in [2^11, 2^12).
// max|q0| and max|p0/m| go to the scratch words 2 and 6 (NaN / inf ignored).
__global__ void __launch_bounds__(256) absmax_kernel(const float* __restrict__ q,
                                                     const float* __restrict__ p,
                                                     const float* __restrict__ mass, int64_t n,
                                                     int64_t D, float* __restrict__ scales) {
  float mq = 0.f, mv = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    mq = finite_absmax(mq, q[i]);
    mv = finite_absmax(mv, fdiv(p[i], mass[i % D]));
  }
  mq = warp_max(mq);
  mv = warp_max(mv);
  if ((threadIdx.x & 31) == 0) {
    atomicMax(reinterpret_cast<unsigned int*>(scales) + 2, __float_as_uint(mq));
    atomicMax(reinterpret_cast<unsigned int*>(scales) + 6, __float_as_uint(mv));
  }
}
// one warp: scales[0] = sq, scales[1] = 1/(sP*sq) from the scratch max, max(1/m) and record 0
// (the scratch words are reset for the next call), and clears record 1, which pass 0 fills.
__global__ void scale_kernel(float* __restrict__ scales, const float* __restrict__ mass,
                             int64_t D) {
  float w = 0.f;
  for (int64_t i = threadIdx.x; i < D; i += 32) w = finite_absmax(w, fdiv(1.f, mass[i]));
  w = warp_max(w);
  if (threadIdx.x != 0) return;
  unsigned int* u = reinterpret_cast<unsigned int*>(scales);
  const float mq = __uint_as_float(u[2]), mv = __uint_as_float(u[6]);
  const float sq = pow2_plane_scale(mq);
  scales[0] = sq;
  scales[1] = 1.f / (scales[3] * sq);
  u[2] = 0u;
  float* r0 = scales + kScaleHdr;
  r0[0] = sq;
  r0[1] = sq;
  r0[2] = mq;
  r0[3] = mv;
  u[kScaleHdr + kScaleRec + 2] = 0u;
  u[kScaleHdr + kScaleRec + 3] = 0u;
  scales[7] = w;
  u[6] = 0u;
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

// one pass on the tensor cores; q_lo: impl 1 TF32 residual of q_cur / impl 2 its fp16 planes
template <int OP>
int launch_dense(const float* q_cur, const void* q_lo, float* q_next, void* q_next_lo,
                 const float* p_in, float* p_out, const void* P_hi, const void* P_lo,
                 const float* bvec, const float* mu, const float* mass, const float* state,
                 float p_scale, float* lp_part, float* k_part, int64_t chains, int D, float* scales,
                 int pass_index, cudaStream_t st, const char* what) {
  if (k_part && !lp_part) {
    zsb_set_error("%s: k_part requires lp_part", what);
    return ZSB_ERR_INVALID;
  }
  constexpr int RB = DenseW<OP, 0, 0>::RB;
  CUtensorMap m_phi, m_plo, m_qhi, m_qlo;
  int rc;
  if ((rc = make_map(&m_phi, P_hi, (uint64_t)D, (uint64_t)D, BM, RB, OP))) return rc;
  if ((rc = make_map(&m_plo, P_lo, (uint64_t)D, (uint64_t)D, BM, RB, OP))) return rc;
  const void* qh = OP ? q_lo : (const void*)q_cur;
  const void* ql = OP ? (const void*)(reinterpret_cast<const __half*>(q_lo) + chains * D) : q_lo;
  if ((rc = make_map(&m_qhi, qh, (uint64_t)chains, (uint64_t)D, BN, RB, OP))) return rc;
  if ((rc = make_map(&m_qlo, ql, (uint64_t)chains, (uint64_t)D, BN, RB, OP))) return rc;
  const EpiArgs ea{q_cur, q_next, reinterpret_cast<float*>(q_next_lo), p_in, p_out, lp_part,
                   k_part, chains, D, 1.f, 1.f};
  const int n_blk = (D + BM - 1) / BM;
#define ZSB_DENSE(MODE, DCV)                                                                   \
  do {                                                                                         \
    const DenseW<OP, MODE, DCV> w{m_phi, m_plo, m_qhi, m_qlo, ea, bvec, mu, mass, state,       \
                                  scales, p_scale, n_blk, D, pass_index};                      \
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
  if constexpr (OP == 1)
    if (D == 1024) ZSB_DENSE_MODE(1024);
  ZSB_DENSE_MODE(0);
#undef ZSB_DENSE_MODE
#undef ZSB_DENSE
}

}  // namespace

// rows of the [parts, chains] lp/K partial scratch: 4 warp-quarters per 128-dimension block
int zsb_dense_tc_ntiles(int D) { return 4 * ((D + BM - 1) / BM); }

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
  return launch_dense<0>(q_cur, q_cur_lo, q_next, q_next_lo, p_in, p_out, P_hi, P_lo, bvec, mu,
                         mass, state, p_scale, lp_part, k_part, chains, D, nullptr, 0, st,
                         "hmc_dense_leapfrog_tc");
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

// ---- impl 2: fp16-split operands; pass `pass_index` reads plane-scale record pass_index ----
int zsb_dense_leapfrog_h16_launch(const float* q_cur, const void* q_cur_planes, float* q_next,
                                  void* q_next_planes, const float* p_in, float* p_out,
                                  const void* P_h16, const void* P_l16, float* scales,
                                  int pass_index, const float* bvec, const float* mu,
                                  const float* mass, const float* state, float p_scale,
                                  float* lp_part, float* k_part, int64_t chains, int D,
                                  cudaStream_t st) {
  if (D % 64 != 0 || D < 64) {
    zsb_set_error("dense_h16: D must be a multiple of 64");
    return ZSB_ERR_INVALID;
  }
  if (chains >= (1LL << 31) || (q_next && !q_next_planes) || !q_cur_planes || !scales ||
      pass_index < 0) {
    zsb_set_error("dense_h16: bad arguments");
    return ZSB_ERR_INVALID;
  }
  return launch_dense<1>(q_cur, q_cur_planes, q_next, q_next_planes, p_in, p_out, P_h16, P_l16,
                         bvec, mu, mass, state, p_scale, lp_part, k_part, chains, D, scales,
                         pass_index, st, "hmc_dense_leapfrog_h16");
}

// scales[3], [4], [5] must hold sP, ||P||_inf, max|b| on entry; writes sq_0, plane-scale record 0
// and q's fp16 hi/lo planes at sq_0.
int zsb_dense_h16_prepare_launch(const float* q, const float* p, const float* mass, void* planes,
                                 float* scales, int64_t chains, int64_t D, cudaStream_t st) {
  const int64_t n = chains * D;
  int64_t blocks = zsb_ceil_div(n, 256 * 8);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  if (blocks < 1) blocks = 1;
  absmax_kernel<<<(unsigned)blocks, 256, 0, st>>>(q, p, mass, n, D, scales);
  scale_kernel<<<1, 32, 0, st>>>(scales, mass, D);
  split16_kernel<<<(unsigned)blocks, 256, 0, st>>>(q, reinterpret_cast<__half*>(planes), n, scales);
  return zsb_check_launch("hmc_dense_h16_prepare");
}
