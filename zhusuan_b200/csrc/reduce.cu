// K6: sample-axis reductions for the multi-sample objectives.
//
//   log_mean_exp   zhusuan/utils.py:177-196     (IWAE bound, monte_carlo.py:137-141)
//   mean           exclusive_kl.py:131-137      (ELBO)
//   log_sum_exp    zhusuan/utils.py:153-174
//   sum
// and their backward passes (what TF autodiff produces for `.sgvb()`:
//   d LME / dx = softmax over the axis,  d mean / dx = 1/K).
//
// Input is viewed as [outer, K, inner] (row-major) and reduced over K.  Two layouts:
//   inner >= 2: one thread per (outer, inner) column, loads coalesced across inner (the IWAE
//               case: log_w [K, N], outer = 1, inner = N);
//   inner == 1: one warp per row, warp-shuffle reduction across K.
// The column kernel makes ONE pass over x (online max with rescaled running sum).
#include "common.cuh"

namespace {

enum { OP_LME = 0, OP_MEAN = 1, OP_LSE = 2, OP_SUM = 3 };

template <int OP>
__global__ void __launch_bounds__(256) reduce_cols_kernel(const float* __restrict__ x,
                                                          float* __restrict__ out, int64_t outer,
                                                          int64_t K, int64_t inner) {
  const int64_t ncols = outer * inner;
  for (int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; c < ncols;
       c += (int64_t)gridDim.x * blockDim.x) {
    const int64_t o = c / inner, i = c % inner;
    const float* p = x + o * K * inner + i;
    float r;
    if (OP == OP_LME || OP == OP_LSE) {
      // single pass over HBM: online max / rescaled sum (one read of x instead of two)
      float m = -INFINITY, s = 0.f;
      int64_t k = 0;
      for (; k + 3 < K; k += 4) {                       // 4 independent loads in flight
        const float x0 = p[k * inner], x1 = p[(k + 1) * inner];
        const float x2 = p[(k + 2) * inner], x3 = p[(k + 3) * inner];
        const float mm = fmaxf(fmaxf(fmaxf(x0, x1), fmaxf(x2, x3)), m);
        if (mm == -INFINITY || mm == INFINITY) {
          // all -inf (or NaN: fmaxf drops it from mm) so far, the sum stays 0 -- unless a NaN was
          // among them -- or a +inf: (inf - inf) = nan as in the reference
          const bool nan_in = isnan(x0) || isnan(x1) || isnan(x2) || isnan(x3);
          s = (mm == INFINITY || nan_in) ? NAN : s;
        } else {
          s = s * expf(m - mm) + expf(x0 - mm) + expf(x1 - mm) + expf(x2 - mm) + expf(x3 - mm);
        }
        m = mm;
      }
      for (; k < K; ++k) {
        const float x = p[k * inner];
        const float mm = fmaxf(x, m);
        if (mm == -INFINITY || mm == INFINITY) s = (mm == INFINITY || isnan(x)) ? NAN : s;
        else s = s * expf(m - mm) + expf(x - mm);
        m = mm;
      }
      if (m == -INFINITY) s = NAN;                      // exp(x - max) = exp(nan), as the reference
      if (OP == OP_LME) s = s / (float)K;
      r = logf(s) + m;
    } else {
      float s = 0.f;
      for (int64_t k = 0; k < K; ++k) s += p[k * inner];
      r = (OP == OP_MEAN) ? s / (float)K : s;
    }
    out[c] = r;
  }
}

template <int OP>
__global__ void __launch_bounds__(256) reduce_rows_kernel(const float* __restrict__ x,
                                                          float* __restrict__ out, int64_t rows,
                                                          int64_t K) {
  const int lane = threadIdx.x & 31;
  for (int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); row < rows;
       row += (int64_t)gridDim.x * 8) {
    const float* p = x + row * K;
    float r;
    if (OP == OP_LME || OP == OP_LSE) {
      float m = -INFINITY;
      for (int64_t k = lane; k < K; k += 32) m = fmaxf(m, p[k]);
      m = warp_max(m);
      float s = 0.f;
      for (int64_t k = lane; k < K; k += 32) s += expf(p[k] - m);
      s = warp_sum(s);
      if (OP == OP_LME) s = s / (float)K;
      r = logf(s) + m;
    } else {
      float s = 0.f;
      for (int64_t k = lane; k < K; k += 32) s += p[k];
      s = warp_sum(s);
      r = (OP == OP_MEAN) ? s / (float)K : s;
    }
    if (lane == 0) out[row] = r;
  }
}

// dx[o,k,i] = gout[o,i] * w,  w = softmax_k(x) for LME/LSE, 1/K for mean, 1 for sum.
// `y` is the forward result (LME/LSE value) so the softmax needs no second reduction:
//   LME: exp(x - y)/K ; LSE: exp(x - y).
template <int OP>
__global__ void __launch_bounds__(256) reduce_bwd_kernel(const float* __restrict__ x,
                                                         const float* __restrict__ y,
                                                         const float* __restrict__ gout,
                                                         float* __restrict__ dx, int64_t outer,
                                                         int64_t K, int64_t inner) {
  const int64_t n = outer * K * inner;
  const float invK = 1.f / (float)K;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n;
       e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t i = e % inner, o = e / (K * inner);
    const int64_t c = o * inner + i;
    const float g = gout[c];
    float w;
    if (OP == OP_LME) w = expf(x[e] - y[c]) * invK;
    else if (OP == OP_LSE) w = expf(x[e] - y[c]);
    else if (OP == OP_MEAN) w = invK;
    else w = 1.f;
    dx[e] = g * w;
  }
}

template <int OP>
int launch_fwd(const float* x, float* out, int64_t outer, int64_t K, int64_t inner,
               cudaStream_t st) {
  if (outer * inner == 0) return ZSB_OK;
  if (inner == 1) {
    int64_t blocks = zsb_ceil_div(outer, 8);
    if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
    reduce_rows_kernel<OP><<<(unsigned)blocks, 256, 0, st>>>(x, out, outer, K);
  } else {
    int64_t blocks = zsb_ceil_div(outer * inner, 256);
    if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
    reduce_cols_kernel<OP><<<(unsigned)blocks, 256, 0, st>>>(x, out, outer, K, inner);
  }
  return zsb_check_launch("reduce_fwd");
}
template <int OP>
int launch_bwd(const float* x, const float* y, const float* gout, float* dx, int64_t outer,
               int64_t K, int64_t inner, cudaStream_t st) {
  const int64_t n = outer * K * inner;
  if (n == 0) return ZSB_OK;
  int64_t blocks = zsb_ceil_div(n, 256);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  reduce_bwd_kernel<OP><<<(unsigned)blocks, 256, 0, st>>>(x, y, gout, dx, outer, K, inner);
  return zsb_check_launch("reduce_bwd");
}

}  // namespace

extern "C" {

// op: 0 log_mean_exp, 1 mean, 2 log_sum_exp, 3 sum.  x: [outer, K, inner] -> out: [outer, inner].
int zsb_reduce_fwd_f32(int op, const float* x, float* out, int64_t outer, int64_t K, int64_t inner,
                       void* stream) {
  ZSB_REQUIRE(outer >= 0 && K > 0 && inner >= 0, "zsb_reduce_fwd_f32: bad sizes (K must be > 0)");
  cudaStream_t st = (cudaStream_t)stream;
  switch (op) {
    case OP_LME: return launch_fwd<OP_LME>(x, out, outer, K, inner, st);
    case OP_MEAN: return launch_fwd<OP_MEAN>(x, out, outer, K, inner, st);
    case OP_LSE: return launch_fwd<OP_LSE>(x, out, outer, K, inner, st);
    case OP_SUM: return launch_fwd<OP_SUM>(x, out, outer, K, inner, st);
  }
  zsb_set_error("zsb_reduce_fwd_f32: unknown op %d", op);
  return ZSB_ERR_INVALID;
}
// y: forward output (used by ops 0 and 2; may be NULL otherwise).
int zsb_reduce_bwd_f32(int op, const float* x, const float* y, const float* gout, float* dx,
                       int64_t outer, int64_t K, int64_t inner, void* stream) {
  ZSB_REQUIRE(outer >= 0 && K > 0 && inner >= 0, "zsb_reduce_bwd_f32: bad sizes");
  cudaStream_t st = (cudaStream_t)stream;
  switch (op) {
    case OP_LME: return launch_bwd<OP_LME>(x, y, gout, dx, outer, K, inner, st);
    case OP_MEAN: return launch_bwd<OP_MEAN>(x, y, gout, dx, outer, K, inner, st);
    case OP_LSE: return launch_bwd<OP_LSE>(x, y, gout, dx, outer, K, inner, st);
    case OP_SUM: return launch_bwd<OP_SUM>(x, y, gout, dx, outer, K, inner, st);
  }
  zsb_set_error("zsb_reduce_bwd_f32: unknown op %d", op);
  return ZSB_ERR_INVALID;
}

}  // extern "C"
