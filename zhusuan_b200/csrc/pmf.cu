// The chunked log-joint of Bayesian probabilistic matrix factorisation and its gradient w.r.t. the
// sampled factor, for HMC that updates every chunk of one factor in a single call.
//
// Reference (examples/probabilistic_matrix_factorization/pmf_hmc.py:19-31, log_joint override
// 136-144; Normal._log_prob, zhusuan/distributions/univariate.py):
//     u [K, n, D] ~ N(0, alpha_u),  v [K, m, D] ~ N(0, alpha_v),
//     r_ij ~ N(sigmoid(u_i . v_j), alpha_pred)              for every observed rating (i, j)
// The example samples one chunk of `chunk_size` latent rows at a time, with the other factor fixed
// and restricted to the chunk's neighbour set (the distinct columns its ratings touch).  The chunks
// are conditionally independent, so one HMC iteration with chain shape [K, n_chunks] does the whole
// sweep.  For chunk c and particle k:
//     lp[k, c] = sum_{rows i in c} sum_d N(lat[k,i,d]; 0, std_lat)
//              + sum_{cols j in nbr(c)} sum_d N(fixed[k,j,d]; 0, std_fixed)
//              + sum_{ratings (i, j), i in c} N(r_ij; s_ij, std_rating),   s_ij = sigmoid(lat_i . fixed_j)
//     grad[k, i] = -lat_i / std_lat^2 + sum_j (r_ij - s_ij) s_ij (1 - s_ij) / std_rating^2 fixed_j
//
// Mapping: lanes over D.  One block = one latent row x one particle, four warps; each warp takes
// 32-rating tiles of the row (CSR, stride four tiles), loads the tile's column indices and ratings
// with one coalesced load, then walks it four ratings at a time: four independent coalesced
// gathers of a fixed-factor row (D floats: rows of D = 30 are not 16-byte aligned, so scalar
// loads), one butterfly sum each for the dot product, and the axpy into a per-lane gradient slice.
// Lanes over ratings would need a D-wide cross-lane reduction of the gradient per row and an
// uncoalesced per-lane row read; here every row read is one contiguous segment and the gradient
// stays in registers.  A long row is spread over four warps with four gathers in flight per warp,
// so it does not serialise on one thread; padding rows with no ratings only pay their prior.
// The four warps' partial gradients and values are summed in shared memory in warp order, and a
// second kernel sums the per-row values of a chunk and the fixed factor's prior over the chunk's
// neighbours with a fixed-shape block reduction: no floating-point atomics anywhere, so two calls
// on the same inputs give bit-identical outputs.  The work is a gather of fixed-factor rows (L2
// resident at MovieLens sizes), so the kernel is bound by L2 / L1 gather bandwidth, not by FMAs.
#include "common.cuh"

namespace {

constexpr int PMF_WARPS = 4;           // warps per row block
constexpr int PMF_TILE = 32;           // ratings staged per warp tile (one per lane)
constexpr int PMF_INFLIGHT = 4;        // gathers issued before their reductions
constexpr int PMF_MAX_D = 128;
constexpr float PMF_LOG_SQRT_2PI = 0.9189385332046727f;

template <int NV>                      // NV = ceil(D / 32) elements of a row per lane
__global__ void __launch_bounds__(PMF_WARPS * 32, 8) pmf_row_kernel(
    const float* __restrict__ lat, const float* __restrict__ fixed,
    const int64_t* __restrict__ row_ptr, const int32_t* __restrict__ col_idx,
    const float* __restrict__ rating, float logstd_lat, float logstd_rating,
    float* __restrict__ row_lp, float* __restrict__ grad_out, int64_t n_rows, int64_t n_cols,
    int D) {
  __shared__ float sg[PMF_WARPS][PMF_MAX_D];
  __shared__ float slp[PMF_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t i = blockIdx.x, k = blockIdx.y;
  const float* __restrict__ u = lat + (k * n_rows + i) * D;
  const float* __restrict__ vk = fixed + k * n_cols * D;
  const float prec_r = expf(-2.f * logstd_rating);
  const float c_r = -PMF_LOG_SQRT_2PI - logstd_rating;
  const bool want_grad = grad_out != nullptr;

  float ur[NV], g[NV];
#pragma unroll
  for (int e = 0; e < NV; ++e) {
    const int d = lane + 32 * e;
    ur[e] = d < D ? u[d] : 0.f;
    g[e] = 0.f;
  }
  float lp = 0.f;                                   // warp-uniform (butterfly sums)
  const int64_t r0 = row_ptr[i], r1 = row_ptr[i + 1];
  for (int64_t t0 = r0 + (int64_t)warp * PMF_TILE; t0 < r1; t0 += PMF_WARPS * PMF_TILE) {
    const int n = (int)((r1 - t0 < PMF_TILE) ? (r1 - t0) : PMF_TILE);
    const int j_l = lane < n ? col_idx[t0 + lane] : 0;
    const float r_l = lane < n ? rating[t0 + lane] : 0.f;
    for (int t = 0; t < n; t += PMF_INFLIGHT) {
      float v[PMF_INFLIGHT][NV], rr[PMF_INFLIGHT];
#pragma unroll
      for (int q = 0; q < PMF_INFLIGHT; ++q) {
        const int j = __shfl_sync(0xffffffffu, j_l, t + q);
        rr[q] = __shfl_sync(0xffffffffu, r_l, t + q);
        const bool ok = t + q < n;
        const float* __restrict__ vj = vk + (int64_t)j * D;
#pragma unroll
        for (int e = 0; e < NV; ++e) {
          const int d = lane + 32 * e;
          v[q][e] = (ok && d < D) ? vj[d] : 0.f;
        }
      }
#pragma unroll
      for (int q = 0; q < PMF_INFLIGHT; ++q) {
        if (t + q >= n) continue;                   // warp-uniform
        float dot = 0.f;
#pragma unroll
        for (int e = 0; e < NV; ++e) dot = fmaf(ur[e], v[q][e], dot);
        dot = warp_sum(dot);
        const float s = 1.f / (1.f + expf(-dot));
        const float diff = rr[q] - s;
        lp += c_r - 0.5f * prec_r * diff * diff;
        if (want_grad) {
          const float coef = diff * s * (1.f - s) * prec_r;
#pragma unroll
          for (int e = 0; e < NV; ++e) g[e] = fmaf(coef, v[q][e], g[e]);
        }
      }
    }
  }
  if (want_grad) {
#pragma unroll
    for (int e = 0; e < NV; ++e) {
      const int d = lane + 32 * e;
      if (d < D) sg[warp][d] = g[e];
    }
  }
  if (lane == 0) slp[warp] = lp;
  __syncthreads();
  const float prec_u = expf(-2.f * logstd_lat);
  if (want_grad) {
    for (int d = threadIdx.x; d < D; d += blockDim.x) {
      float s = sg[0][d];
#pragma unroll
      for (int w = 1; w < PMF_WARPS; ++w) s += sg[w][d];
      grad_out[(k * n_rows + i) * D + d] = s - prec_u * u[d];
    }
  }
  if (row_lp != nullptr && warp == 0) {
    const float c_u = -PMF_LOG_SQRT_2PI - logstd_lat;
    float pr = 0.f;
#pragma unroll
    for (int e = 0; e < NV; ++e)
      if (lane + 32 * e < D) pr += c_u - 0.5f * prec_u * ur[e] * ur[e];
    pr = warp_sum(pr);
    if (lane == 0) {
      float s = slp[0];
#pragma unroll
      for (int w = 1; w < PMF_WARPS; ++w) s += slp[w];
      row_lp[k * n_rows + i] = s + pr;
    }
  }
}

// lp[k, c] = sum of the chunk's row values + prior of the fixed factor over the chunk's neighbours
__global__ void __launch_bounds__(256) pmf_chunk_kernel(
    const float* __restrict__ row_lp, const float* __restrict__ fixed,
    const int64_t* __restrict__ nbr_ptr, const int32_t* __restrict__ nbr_idx, float logstd_fixed,
    float* __restrict__ lp_out, int64_t n_rows, int64_t n_cols, int64_t n_chunks, int D,
    int64_t chunk_size) {
  __shared__ float red[32];
  const int64_t c = blockIdx.x, k = blockIdx.y;
  const float prec_v = expf(-2.f * logstd_fixed);
  const float c_v = -PMF_LOG_SQRT_2PI - logstd_fixed;
  float s = 0.f;
  const float* __restrict__ rl = row_lp + k * n_rows + c * chunk_size;
  for (int64_t t = threadIdx.x; t < chunk_size; t += blockDim.x) s += rl[t];
  const int64_t b0 = nbr_ptr[c], n = (nbr_ptr[c + 1] - b0) * D;
  const float* __restrict__ vk = fixed + k * n_cols * D;
  for (int64_t e = threadIdx.x; e < n; e += blockDim.x) {
    const int64_t j = nbr_idx[b0 + e / D];
    const float x = vk[j * D + e % D];
    s += c_v - 0.5f * prec_v * x * x;
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) lp_out[k * n_chunks + c] = s;
}

}  // namespace

extern "C" {

// Chunked PMF log-joint and / or its gradient w.r.t. the latent factor
// (pmf_hmc.py:19-31, 136-144).  See include/zsb200.h.
int zsb_pmf_logjoint_f32(const float* lat, const float* fixed, const int64_t* row_ptr,
                         const int32_t* col_idx, const float* rating, const int64_t* nbr_ptr,
                         const int32_t* nbr_idx, float logstd_lat, float logstd_fixed,
                         float logstd_rating, float* lp_out, float* grad_out, float* work,
                         int64_t K, int64_t n_rows, int64_t n_cols, int64_t D, int64_t chunk_size,
                         void* stream) {
  ZSB_REQUIRE(lat && fixed && row_ptr && col_idx && rating && (lp_out || grad_out),
              "zsb_pmf_logjoint_f32: null pointer");
  ZSB_REQUIRE(!lp_out || (nbr_ptr && nbr_idx && work),
              "zsb_pmf_logjoint_f32: values need nbr_ptr, nbr_idx and work");
  ZSB_REQUIRE(D >= 1 && D <= PMF_MAX_D, "zsb_pmf_logjoint_f32: D = %lld outside [1, %d]",
              (long long)D, PMF_MAX_D);
  ZSB_REQUIRE(K > 0 && n_rows > 0 && n_cols > 0 && chunk_size > 0 && n_rows % chunk_size == 0,
              "zsb_pmf_logjoint_f32: bad sizes (K %lld, n_rows %lld, n_cols %lld, chunk %lld)",
              (long long)K, (long long)n_rows, (long long)n_cols, (long long)chunk_size);
  ZSB_REQUIRE(n_rows < (1LL << 31) && n_cols < (1LL << 31) && K < 65536,
              "zsb_pmf_logjoint_f32: grid limits exceeded (n_rows, n_cols < 2^31, K < 65536)");
  cudaStream_t st = (cudaStream_t)stream;
  const dim3 grid((unsigned)n_rows, (unsigned)K);
  float* row_lp = lp_out ? work : nullptr;
#define ZSB_PMF(NV)                                                                              \
  pmf_row_kernel<NV><<<grid, PMF_WARPS * 32, 0, st>>>(lat, fixed, row_ptr, col_idx, rating,      \
                                                      logstd_lat, logstd_rating, row_lp,         \
                                                      grad_out, n_rows, n_cols, (int)D)
  switch ((D + 31) / 32) {
    case 1: ZSB_PMF(1); break;
    case 2: ZSB_PMF(2); break;
    case 3: ZSB_PMF(3); break;
    default: ZSB_PMF(4); break;
  }
#undef ZSB_PMF
  int rc = zsb_check_launch("pmf_row");
  if (rc != ZSB_OK || !lp_out) return rc;
  const int64_t n_chunks = n_rows / chunk_size;
  pmf_chunk_kernel<<<dim3((unsigned)n_chunks, (unsigned)K), 256, 0, st>>>(
      row_lp, fixed, nbr_ptr, nbr_idx, logstd_fixed, lp_out, n_rows, n_cols, n_chunks, (int)D,
      chunk_size);
  return zsb_check_launch("pmf_chunk");
}

}  // extern "C"
