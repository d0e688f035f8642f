// K2 + K8 for the dense-covariance Gaussian target (BASELINE config 2):
//     log p(x) = -1/2 (x-mu)^T P (x-mu) + const,    grad = -P (x-mu) = b - P x,  b = P mu.
//
// One launch == one iteration of the reference's leapfrog while-loop body (hmc.py:352-364):
//     g      = b - q_i P                      (GEMM [chains, D] x [D, D], P symmetric)
//     p      = p + (scale * eps) * g          (hmc.py:42; scale = 1/2 on the first/last pass)
//     q_{i+1}= q_i + eps * (p / mass)         (hmc.py:39 of the NEXT pass, fused here)
//     lp(q_i)= 1/2 sum_n (q_i - mu)_n g_n + const     (free by-product: no extra forward pass,
//                                                      unlike the reference's 2 extra evals, :47-50)
//     K(p)   = 1/2 sum_n p_n^2 / mass_n        (last pass only)
// so per chain per leapfrog step the kernel reads q_i (GEMM operand + epilogue tile), reads and
// writes p, writes q_{i+1}: 20*D bytes, against the 16*D algorithmic minimum (SURVEY 8d).
//
// This file holds the SIMT fp32 implementation (impl 0): 128x128x16 tiles, 8x8 register micro-tile,
// register-prefetch double buffering.  It is the always-available, any-D%16 reference kernel; the
// wgmma 3xTF32 tensor-core implementation (impl 1) lives in hmc_dense_tc.cu.
#include "common.cuh"

namespace {

constexpr int BM = 128, BN = 128, BK = 16;
constexpr int APAD = 4;


__global__ void __launch_bounds__(256, 2)
dense_leapfrog_simt_kernel(const float* __restrict__ q_cur, float* __restrict__ q_next,
                           const float* __restrict__ p_in, float* __restrict__ p_out,
                           const float* __restrict__ P, const float* __restrict__ bvec,
                           const float* __restrict__ mu, const float* __restrict__ mass,
                           const float* __restrict__ state, float p_scale,
                           float* __restrict__ lp_part, float* __restrict__ k_part,
                           int64_t chains, int D) {
  __shared__ __align__(16) float As[2][BK][BM + APAD];
  __shared__ __align__(16) float Bs[2][BK][BN];

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = (int64_t)blockIdx.y * BM;
  const int n0 = blockIdx.x * BN;

  // global->smem load assignment
  const int a_row = tid >> 2;        // 0..63 (+64)
  const int a_k4 = (tid & 3) * 4;    // 0,4,8,12
  const int b_row = tid >> 5;        // 0..7 (+8)
  const int b_n4 = (tid & 31) * 4;   // 0..124

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  float4 a_reg[2], b_reg[2];
  auto load_tiles = [&](int k0) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t m = m0 + a_row + h * 64;
      a_reg[h] = (m < chains)
                     ? *reinterpret_cast<const float4*>(q_cur + m * D + k0 + a_k4)
                     : make_float4(0.f, 0.f, 0.f, 0.f);
      const int n = n0 + b_n4;
      b_reg[h] = (n < D) ? *reinterpret_cast<const float4*>(P + (int64_t)(k0 + b_row + h * 8) * D + n)
                         : make_float4(0.f, 0.f, 0.f, 0.f);
    }
  };
  auto store_tiles = [&](int buf) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int r = a_row + h * 64;
      As[buf][a_k4 + 0][r] = a_reg[h].x;
      As[buf][a_k4 + 1][r] = a_reg[h].y;
      As[buf][a_k4 + 2][r] = a_reg[h].z;
      As[buf][a_k4 + 3][r] = a_reg[h].w;
      *reinterpret_cast<float4*>(&Bs[buf][b_row + h * 8][b_n4]) = b_reg[h];
    }
  };

  const int nk = D / BK;
  load_tiles(0);
  store_tiles(0);
  __syncthreads();
  for (int kt = 0; kt < nk; ++kt) {
    const int buf = kt & 1;
    if (kt + 1 < nk) load_tiles((kt + 1) * BK);
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
      const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    if (kt + 1 < nk) store_tiles(buf ^ 1);
    __syncthreads();
  }

  // ---- fused leapfrog epilogue ----
  const float eps = state[ZSB_ST_EPS_USED];
  const float s2 = mul(eps, p_scale);
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + (i - 4));
    float lp_acc = 0.f, k_acc = 0.f;
    if (m < chains) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int n = n0 + h * 64 + tx * 4;
        if (n < D) {
          const float4 pv = *reinterpret_cast<const float4*>(p_in + m * D + n);
          const float4 qv = *reinterpret_cast<const float4*>(q_cur + m * D + n);
          const float4 ms = *reinterpret_cast<const float4*>(mass + n);
          float4 bv = make_float4(0.f, 0.f, 0.f, 0.f), mv = bv;
          if (bvec) bv = *reinterpret_cast<const float4*>(bvec + n);
          if (mu) mv = *reinterpret_cast<const float4*>(mu + n);
          const float pe[4] = {pv.x, pv.y, pv.z, pv.w}, qe[4] = {qv.x, qv.y, qv.z, qv.w};
          const float me[4] = {ms.x, ms.y, ms.z, ms.w}, be[4] = {bv.x, bv.y, bv.z, bv.w};
          const float ue[4] = {mv.x, mv.y, mv.z, mv.w};
          float pn[4], qn[4];
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const float g = sub(be[j], acc[i][h * 4 + j]);
            pn[j] = add(pe[j], mul(s2, g));
            qn[j] = add(qe[j], mul(eps, fdiv(pn[j], me[j])));
            lp_acc += (qe[j] - ue[j]) * g;
            k_acc += fdiv(mul(pn[j], pn[j]), me[j]);
          }
          *reinterpret_cast<float4*>(p_out + m * D + n) = make_float4(pn[0], pn[1], pn[2], pn[3]);
          if (q_next)
            *reinterpret_cast<float4*>(q_next + m * D + n) = make_float4(qn[0], qn[1], qn[2], qn[3]);
        }
      }
    }
    // reduce across the 16 tx-threads that share this row (half-warp)
    if (lp_part) {
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) lp_acc += __shfl_xor_sync(0xffffffffu, lp_acc, o);
      if (tx == 0 && m < chains) lp_part[(int64_t)blockIdx.x * chains + m] = lp_acc;
    }
    if (k_part) {
#pragma unroll
      for (int o = 8; o > 0; o >>= 1) k_acc += __shfl_xor_sync(0xffffffffu, k_acc, o);
      if (tx == 0 && m < chains) k_part[(int64_t)blockIdx.x * chains + m] = k_acc;
    }
  }
}

// lp[c] = 0.5 * sum_t lp_part[t][c] + const ;  k[c] = 0.5 * sum_t k_part[t][c]   (fixed order)
__global__ void __launch_bounds__(256) dense_finish_kernel(const float* __restrict__ lp_part,
                                                           const float* __restrict__ k_part,
                                                           int ntiles, int64_t chains,
                                                           float const_term,
                                                           float* __restrict__ lp_out,
                                                           float* __restrict__ k_out) {
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < chains;
       c += (int64_t)gridDim.x * blockDim.x) {
    if (lp_part && lp_out) {
      float s = 0.f;
      for (int t = 0; t < ntiles; ++t) s += lp_part[(int64_t)t * chains + c];
      lp_out[c] = add(mul(0.5f, s), const_term);
    }
    if (k_part && k_out) {
      float s = 0.f;
      for (int t = 0; t < ntiles; ++t) s += k_part[(int64_t)t * chains + c];
      k_out[c] = mul(0.5f, s);
    }
  }
}

}  // namespace

// implemented in hmc_dense_tc.cu
int zsb_dense_leapfrog_tc_launch(const float* q_cur, const float* q_cur_lo, float* q_next,
                                 float* q_next_lo, const float* p_in, float* p_out,
                                 const float* P_hi, const float* P_lo, const float* bvec,
                                 const float* mu, const float* mass, const float* state,
                                 float p_scale, float* lp_part, float* k_part, int64_t chains,
                                 int D, cudaStream_t st);
int zsb_dense_split_lo_launch(const float* q, float* lo, int64_t n, cudaStream_t st);
int zsb_dense_tc_ntiles(int D);
int zsb_dense_leapfrog_h16_launch(const float* q_cur, const void* q_cur_planes, float* q_next,
                                  void* q_next_planes, const float* p_in, float* p_out,
                                  const void* P_h16, const void* P_l16, float* scales,
                                  int pass_index, const float* bvec, const float* mu,
                                  const float* mass, const float* state, float p_scale,
                                  float* lp_part, float* k_part, int64_t chains, int D,
                                  cudaStream_t st);
int zsb_dense_h16_prepare_launch(const float* q, const float* p, const float* mass, void* planes,
                                 float* scales, int64_t chains, int64_t D, cudaStream_t st);
// implemented in hmc_dense_res.cu
int zsb_dense_res_h16_launch(void* planes0, void* planes1, void* spare0, void* spare1,
                             const float* p0, float* pw, const void* P_h16, const void* P_l16,
                             float* scales, const float* bvec, const float* mu, const float* mass,
                             const float* state, float* lp0_part, float* lp1_part, float* k_part,
                             int64_t chains, int D, int L, cudaStream_t st);
int zsb_dense_select_planes_launch(float* q, const void* planes, const void* spare,
                                   const float* record, const int32_t* accept, int64_t chains,
                                   int64_t D, cudaStream_t st);

extern "C" {

// Rows of the lp_part / k_part scratch ([ntiles, chains]) for dimension D and implementation impl.
int zsb_hmc_dense_ntiles(int64_t D, int impl) {
  if (impl == 1) return zsb_dense_tc_ntiles((int)D);
  return (int)zsb_ceil_div(D, BN);
}

// impl 0: SIMT fp32 (P = full fp32 matrix; P_lo / q_cur_lo / q_next_lo ignored).
// impl 1: wgmma 3xTF32 (P = hi part, P_lo = residual; q_cur_lo = TF32 residual of q_cur on entry,
//         q_next_lo receives q_next's residual; D % 32 == 0).
int zsb_hmc_dense_leapfrog_f32(const float* q_cur, const float* q_cur_lo, float* q_next,
                               float* q_next_lo, const float* p_in, float* p_out,
                               const float* P, const float* P_lo, const float* bvec,
                               const float* mu, const float* mass, const float* state,
                               float p_scale, float* lp_part, float* k_part, int64_t chains,
                               int64_t D, int impl, void* stream) {
  ZSB_REQUIRE(q_cur && p_in && p_out && P && mass && state, "zsb_hmc_dense_leapfrog_f32: null arg");
  ZSB_REQUIRE(chains > 0 && D > 0 && D % BK == 0 && D <= (1 << 20),
              "zsb_hmc_dense_leapfrog_f32: D must be a positive multiple of 16");
  ZSB_REQUIRE(q_next != q_cur, "zsb_hmc_dense_leapfrog_f32: q_next must not alias q_cur");
  cudaStream_t st = (cudaStream_t)stream;
  if (impl == 1) {
    ZSB_REQUIRE(P_lo && q_cur_lo, "zsb_hmc_dense_leapfrog_f32: impl 1 needs the P_lo / q_lo splits");
    return zsb_dense_leapfrog_tc_launch(q_cur, q_cur_lo, q_next, q_next_lo, p_in, p_out, P, P_lo,
                                        bvec, mu, mass, state, p_scale, lp_part, k_part, chains,
                                        (int)D, st);
  }
  ZSB_REQUIRE(impl == 0, "zsb_hmc_dense_leapfrog_f32: unknown impl %d", impl);
  dim3 grid((unsigned)zsb_ceil_div(D, BN), (unsigned)zsb_ceil_div(chains, BM));
  dense_leapfrog_simt_kernel<<<grid, 256, 0, st>>>(q_cur, q_next, p_in, p_out, P, bvec, mu, mass,
                                                   state, p_scale, lp_part, k_part, chains, (int)D);
  return zsb_check_launch("hmc_dense_leapfrog_simt");
}

// lo[i] = q[i] - tf32_trunc(q[i])  (the residual operand of the 3xTF32 split), n % 4 == 0
int zsb_hmc_dense_split_lo_f32(const float* q, float* lo, int64_t n, void* stream) {
  ZSB_REQUIRE(q && lo && n >= 0, "zsb_hmc_dense_split_lo_f32: bad args");
  if (n == 0) return ZSB_OK;
  return zsb_dense_split_lo_launch(q, lo, n, (cudaStream_t)stream);
}

// impl 2 (fp16-split tensor-core path, one launch per leapfrog pass).  Operands are fp16 hi/lo
// planes of P*sP and q*sq: P_h16, P_l16: [D, D] __half; q_*_planes: [2][chains][D] __half (hi
// plane, lo plane).  The plane scale follows the chains: scales is a device float[8 + 4 * (L + 2)]
// of plane-scale records (hmc_dense_epilogue.cuh) with [3] sP, [4] ||P||_inf, [5] max|b| set by
// the caller once.  zsb_hmc_dense_traj_prepare_f32 (before every
// trajectory, after the momentum p is drawn) writes record 0 and q's planes; pass `pass_index`
// (from 0) reads planes at the scale of record pass_index and writes q_next's planes, and record
// pass_index + 1, at a scale lowered whenever a bound on |q_next| could overflow fp16.
// D % 64 == 0.
int zsb_hmc_dense_traj_prepare_f32(const float* q, const float* p, const float* mass, void* planes,
                                   float* scales, int64_t chains, int64_t D, void* stream) {
  ZSB_REQUIRE(q && p && mass && planes && scales && chains > 0 && D > 0,
              "zsb_hmc_dense_traj_prepare_f32: bad args");
  return zsb_dense_h16_prepare_launch(q, p, mass, planes, scales, chains, D,
                                      (cudaStream_t)stream);
}
int zsb_hmc_dense_leapfrog_h16_pass_f32(const float* q_cur, const void* q_cur_planes,
                                        float* q_next, void* q_next_planes, const float* p_in,
                                        float* p_out, const void* P_h16, const void* P_l16,
                                        float* scales, int pass_index, const float* bvec,
                                        const float* mu, const float* mass, const float* state,
                                        float p_scale, float* lp_part, float* k_part,
                                        int64_t chains, int64_t D, void* stream) {
  ZSB_REQUIRE(q_cur && p_in && p_out && P_h16 && P_l16 && mass && state && scales,
              "zsb_hmc_dense_leapfrog_h16_pass_f32: null arg");
  ZSB_REQUIRE(q_next != q_cur, "zsb_hmc_dense_leapfrog_h16_pass_f32: q_next must not alias q_cur");
  ZSB_REQUIRE(pass_index >= 0, "zsb_hmc_dense_leapfrog_h16_pass_f32: pass_index < 0");
  return zsb_dense_leapfrog_h16_launch(q_cur, q_cur_planes, q_next, q_next_planes, p_in, p_out,
                                       P_h16, P_l16, scales, pass_index, bvec, mu, mass, state,
                                       p_scale, lp_part, k_part, chains, (int)D,
                                       (cudaStream_t)stream);
}

// impl 5: the whole leapfrog `while_loop` of hmc.py:347-372 (L+1 passes, one launch each,
// hmc_dense_res.cu).  The sampler state inside the trajectory is the fp16 hi/lo plane pair of
// q*sq_i (+ fp32 p), with the plane-scale records of impl 2's trajectory form; planes0 comes from
// zsb_hmc_dense_traj_prepare_f32, planes1, spare0 and spare1 are work buffers of the same size
// (spare copies of the planes when a pass's bound could overflow them).  On return the proposal's
// planes are in buffer (n_leapfrogs & 1) or its spare -- zsb_hmc_dense_select_traj_planes_f32,
// given both and record n_leapfrogs, assigns them to the accepted chains -- and pw holds the final
// momentum.
// D % 64 == 0, n_leapfrogs >= 1.
int zsb_hmc_dense_resident_h16_f32(void* planes0, void* planes1, void* spare0, void* spare1,
                                   const float* p0, float* pw, const void* P_h16,
                                   const void* P_l16, float* scales, const float* bvec,
                                   const float* mu, const float* mass, const float* state,
                                   float* lp0_part, float* lp1_part, float* k_part,
                                   int64_t chains, int64_t D, int n_leapfrogs, void* stream) {
  ZSB_REQUIRE(planes0 && planes1 && spare0 && spare1 && p0 && pw && P_h16 && P_l16 && scales &&
                  mass && state && lp0_part && lp1_part && k_part,
              "zsb_hmc_dense_resident_h16_f32: null arg");
  ZSB_REQUIRE(p0 != pw, "zsb_hmc_dense_resident_h16_f32: aliased buffers");
  return zsb_dense_res_h16_launch(planes0, planes1, spare0, spare1, p0, pw, P_h16, P_l16, scales,
                                  bvec, mu, mass, state, lp0_part, lp1_part, k_part, chains, (int)D,
                                  n_leapfrogs, (cudaStream_t)stream);
}
// q[c, :] <- (hi + lo) / sq of the proposal of an impl-5 trajectory for the chains with
// accept[c] != 0 (hmc.py:488-497): `record` is its plane-scale record
// (&scales[8 + 4 * n_leapfrogs]), which says whether `planes` or `spare` holds the proposal, and
// at which scale.
int zsb_hmc_dense_select_traj_planes_f32(float* q, const void* planes, const void* spare,
                                         const float* record, const int32_t* accept,
                                         int64_t chains, int64_t D, void* stream) {
  ZSB_REQUIRE(q && planes && spare && record && accept && chains > 0 && D > 0 && D % 2 == 0,
              "zsb_hmc_dense_select_traj_planes_f32: bad args");
  return zsb_dense_select_planes_launch(q, planes, spare, record, accept, chains, D,
                                        (cudaStream_t)stream);
}

int zsb_hmc_dense_finish_f32(const float* lp_part, const float* k_part, int ntiles, int64_t chains,
                             float const_term, float* lp_out, float* k_out, void* stream) {
  ZSB_REQUIRE(chains > 0 && ntiles > 0, "zsb_hmc_dense_finish_f32: bad sizes");
  int64_t blocks = zsb_ceil_div(chains, 256);
  if (blocks > ZSB_NUM_SMS * 8) blocks = ZSB_NUM_SMS * 8;
  dense_finish_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      lp_part, k_part, ntiles, chains, const_term, lp_out, k_out);
  return zsb_check_launch("hmc_dense_finish");
}

}  // extern "C"
