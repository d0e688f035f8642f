// K1 / K7: distribution log_prob (+ analytic backward) and sampling kernels.
//
// Semantics follow zhusuan/distributions (reference file:line cited per kernel).  Operands are
// broadcast by "modular" indexing: element i of the broadcast result reads operand[i % operand_n],
// which covers every case where the operand's shape is a suffix of the broadcast shape (scalars,
// params shared across the leading sample/chain axes, `given` shared across particles).  Other
// broadcast patterns are materialised by the host (that is what the reference's
// maybe_explicit_broadcast does for ALL patterns, distributions/utils.py:52-78).
//
// All kernels are HBM-bound elementwise/row-reduce kernels: coalesced loads, grid-stride over rows,
// warp-shuffle reductions over the event (`group`) axis, deterministic summation order.
#include "common.cuh"

namespace {

constexpr float kHalfLog2Pi = 0.9189385332046727f;

// Broadcast operands of a [n_out, group] problem.  Element (row, j) of operand o lives at
// (row*group + j) % n[o]; the modulo is taken ONCE per row (64-bit) and the inner loop only adds
// (suffix-broadcast operands never wrap inside a row unless they are smaller than the row).
struct Ops3 {
  const float* p[3];
  int64_t n[3];
};
__device__ __forceinline__ float op_at(const float* __restrict__ p, int64_t n, int64_t base,
                                       int64_t j) {
  if (n == 1) return p[0];
  int64_t idx = base + j;
  if (idx >= n) idx %= n;
  return p[idx];
}

// rows of `group` consecutive elements; LANES threads cooperate on one row, 4 elements in flight
// per lane.  F: float f(float v0, float v1, float v2, int64_t i, int64_t row) -> contribution of element i.
template <int LANES, int NOPS, class F>
__global__ void __launch_bounds__(256) row_reduce_kernel(float* __restrict__ out, int64_t n_out,
                                                         int64_t group, Ops3 ops, F f) {
  const int rows_per_block = 256 / LANES;
  const int lane = threadIdx.x % LANES;
  const int rib = threadIdx.x / LANES;
  for (int64_t row = (int64_t)blockIdx.x * rows_per_block + rib; row < n_out;
       row += (int64_t)gridDim.x * rows_per_block) {
    const int64_t i0 = row * group;
    int64_t base[3];
#pragma unroll
    for (int o = 0; o < NOPS; ++o) {
      const int64_t n = ops.n[o];       // common cases first: no 64-bit modulo at all
      base[o] = (n == 1 || n == group) ? 0 : (n == n_out * group ? i0 : i0 % n);
    }
    float acc = 0.f;
    int64_t j = lane;
    for (; j + 3 * LANES < group; j += 4 * LANES) {          // 4 independent loads per operand
      float v[4][3];
#pragma unroll
      for (int u = 0; u < 4; ++u)
#pragma unroll
        for (int o = 0; o < NOPS; ++o) v[u][o] = op_at(ops.p[o], ops.n[o], base[o], j + u * LANES);
#pragma unroll
      for (int u = 0; u < 4; ++u) acc += f(v[u][0], v[u][1], v[u][2], i0 + j + u * LANES, row);
    }
    for (; j < group; j += LANES) {
      float v[3];
#pragma unroll
      for (int o = 0; o < NOPS; ++o) v[o] = op_at(ops.p[o], ops.n[o], base[o], j);
      acc += f(v[0], v[1], v[2], i0 + j, row);
    }
    acc = sub_warp_sum<LANES>(acc);
    if (lane == 0 && out) out[row] = acc;
  }
}

template <int NOPS, class F>
int launch_row_reduce(float* out, int64_t n_out, int64_t group, Ops3 ops, F f, cudaStream_t st,
                      const char* what) {
  if (n_out == 0) return ZSB_OK;
  int lanes = 1;
  while (lanes < 32 && lanes * 4 <= group) lanes <<= 1;      // >= 4 elements per lane when possible
  const int rows_per_block = 256 / lanes;
  int64_t blocks = zsb_ceil_div(n_out, rows_per_block);
  const int64_t cap = (int64_t)ZSB_NUM_SMS * 16;
  if (blocks > cap) blocks = cap;
#define ZSB_RR(LN) row_reduce_kernel<LN, NOPS><<<(unsigned)blocks, 256, 0, st>>>(out, n_out, group, ops, f)
  switch (lanes) {
    case 1: ZSB_RR(1); break;
    case 2: ZSB_RR(2); break;
    case 4: ZSB_RR(4); break;
    case 8: ZSB_RR(8); break;
    case 16: ZSB_RR(16); break;
    default: ZSB_RR(32); break;
  }
#undef ZSB_RR
  return zsb_check_launch(what);
}

// ---- 128-bit variant of row_reduce_kernel ---------------------------------------------------------
// Same rows / lanes decomposition, but a lane owns 4 CONSECUTIVE elements per step: every operand
// is one float4 load, side outputs are float4 stores, a Philox block serves the 4 elements it was
// generated for.  F4: float f4(float4 v0, float4 v1, float4 v2, int64_t i, int64_t row) with i the
// flat index of the first of the 4 elements (i % 4 == 0); returns the sum of their contributions.
// Preconditions (checked by launch_row_reduce4): group % 4 == 0, every operand either a scalar or
// 16-byte aligned with operand_n % group == 0 (so a row never wraps inside an operand).
__device__ __forceinline__ float4 op_at4(const float* __restrict__ p, int64_t n, int64_t base,
                                         int64_t j) {
  if (n == 1) { const float v = p[0]; return make_float4(v, v, v, v); }
  return *reinterpret_cast<const float4*>(p + base + j);
}
template <int LANES, int NOPS, class F4>
__global__ void __launch_bounds__(256) row_reduce_vec4_kernel(float* __restrict__ out,
                                                              int64_t n_out, int64_t group,
                                                              Ops3 ops, F4 f4) {
  // independent (row, chunk) items a thread keeps in flight.  Long rows: 4 chunks (measured
  // 0.243 -> 0.230 ms on the [64, 4096, 784] Bernoulli log-prob).  Short rows are bound by
  // instruction issue, not by loads in flight: 4 rows at once cost 128 registers and ran SLOWER
  // (0.45 -> 0.55 ms on 16.7 M rows of 16), so they keep one row per thread.
  constexpr int U = LANES == 32 ? 4 : 1;
  const int rows_per_block = 256 / LANES;
  const int lane = threadIdx.x % LANES;
  const int rib = threadIdx.x / LANES;
  auto row_base = [&](int64_t i0, int64_t* base) {
#pragma unroll
    for (int o = 0; o < 3; ++o) {
      const int64_t n = o < NOPS ? ops.n[o] : 1;
      base[o] = (n == 1 || n == group) ? 0 : (n == n_out * group ? i0 : i0 % n);
    }
  };
  auto ld = [&](int o, const int64_t* base, int64_t j) -> float4 {
    return o < NOPS ? op_at4(ops.p[o], ops.n[o], base[o], j) : make_float4(0.f, 0.f, 0.f, 0.f);
  };
  if (LANES == 32) {
    // long rows: U chunks of the same row in flight
    for (int64_t row = (int64_t)blockIdx.x * rows_per_block + rib; row < n_out;
         row += (int64_t)gridDim.x * rows_per_block) {
      const int64_t i0 = row * group;
      int64_t base[3];
      row_base(i0, base);
      float acc = 0.f;
      for (int64_t j = 4 * lane; j < group; j += 4 * LANES * U) {
        float4 v[U][3];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int64_t jj = j + (int64_t)u * 4 * LANES;
          if (jj < group) { v[u][0] = ld(0, base, jj); v[u][1] = ld(1, base, jj); v[u][2] = ld(2, base, jj); }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int64_t jj = j + (int64_t)u * 4 * LANES;
          if (jj < group) acc += f4(v[u][0], v[u][1], v[u][2], i0 + jj, row);
        }
      }
      acc = sub_warp_sum<LANES>(acc);
      if (lane == 0 && out) out[row] = acc;
    }
  } else {
    // short rows (a lane sees one or two chunks of a row): U rows in flight
    const int64_t G = (int64_t)gridDim.x * rows_per_block;
    for (int64_t r0 = (int64_t)blockIdx.x * rows_per_block + rib; r0 < n_out; r0 += U * G) {
      int64_t base[U][3];
      float acc[U];
#pragma unroll
      for (int u = 0; u < U; ++u) {
        acc[u] = 0.f;
        const int64_t row = r0 + u * G;
        if (row < n_out) row_base(row * group, base[u]);
      }
      for (int64_t j = 4 * lane; j < group; j += 4 * LANES) {
        float4 v[U][3];
#pragma unroll
        for (int u = 0; u < U; ++u) {
          if (r0 + u * G < n_out) {
            v[u][0] = ld(0, base[u], j); v[u][1] = ld(1, base[u], j); v[u][2] = ld(2, base[u], j);
          }
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
          const int64_t row = r0 + u * G;
          if (row < n_out) acc[u] += f4(v[u][0], v[u][1], v[u][2], row * group + j, row);
        }
      }
#pragma unroll
      for (int u = 0; u < U; ++u) {
        const float t = sub_warp_sum<LANES>(acc[u]);
        const int64_t row = r0 + u * G;
        if (lane == 0 && out && row < n_out) out[row] = t;
      }
    }
  }
}

__host__ inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Picks the 128-bit kernel when the layout allows it (side_ok: every side-output pointer the
// functors write is 16-byte aligned), the scalar kernel otherwise.
template <int NOPS, class F, class F4>
int launch_row_reduce4(float* out, int64_t n_out, int64_t group, Ops3 ops, F f, F4 f4, bool side_ok,
                       cudaStream_t st, const char* what) {
  if (n_out == 0) return ZSB_OK;
  bool vec = side_ok && group % 4 == 0;
  for (int o = 0; o < NOPS && vec; ++o)
    vec = ops.n[o] == 1 || (ops.n[o] % group == 0 && aligned16(ops.p[o]));
  if (!vec) return launch_row_reduce<NOPS>(out, n_out, group, ops, f, st, what);
  int lanes = 1;
  while (lanes < 32 && lanes * 8 <= group) lanes <<= 1;      // >= 4 elements per lane
  const int rows_per_block = 256 / lanes;
  int64_t blocks = zsb_ceil_div(n_out, rows_per_block);
  const int64_t cap = (int64_t)ZSB_NUM_SMS * 16;
  if (blocks > cap) blocks = cap;
#define ZSB_RR4(LN) \
  row_reduce_vec4_kernel<LN, NOPS><<<(unsigned)blocks, 256, 0, st>>>(out, n_out, group, ops, f4)
  switch (lanes) {
    case 1: ZSB_RR4(1); break;
    case 2: ZSB_RR4(2); break;
    case 4: ZSB_RR4(4); break;
    case 8: ZSB_RR4(8); break;
    case 16: ZSB_RR4(16); break;
    default: ZSB_RR4(32); break;
  }
#undef ZSB_RR4
  return zsb_check_launch(what);
}

template <class F>
__global__ void __launch_bounds__(256) elementwise_kernel(int64_t n, F f) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    f(i);
}
template <class F>
int launch_elementwise(int64_t n, F f, cudaStream_t st, const char* what) {
  if (n == 0) return ZSB_OK;
  int64_t blocks = zsb_ceil_div(n, 256);
  const int64_t cap = (int64_t)ZSB_NUM_SMS * 16;
  if (blocks > cap) blocks = cap;
  elementwise_kernel<<<(unsigned)blocks, 256, 0, st>>>(n, f);
  return zsb_check_launch(what);
}

// TF's numerically stable sigmoid cross entropy: max(l,0) - l*x + log1p(exp(-|l|)).
// softplus(-|l|) = log(1 + e^{-|l|}) with e^{-|l|} in (0, 1]: the fast exp/log intrinsics are
// accurate to ~1e-7 ABSOLUTE here, far inside the 1e-5 relative bar on the grouped sums.
__device__ __forceinline__ float bernoulli_lp(float x, float l) {
  return -(fmaxf(l, 0.f) - l * x + __logf(1.f + __expf(-fabsf(l))));
}

// One warp per row of C categories: returns (max, log-sum-exp) over logits[row*C .. +C).
__device__ __forceinline__ float warp_row_lse(const float* __restrict__ l, int64_t C, int lane) {
  float m = -INFINITY;
  for (int64_t j = lane; j < C; j += 32) m = fmaxf(m, l[j]);
  m = warp_max(m);
  float s = 0.f;
  for (int64_t j = lane; j < C; j += 32) s += expf(l[j] - m);
  s = warp_sum(s);
  return logf(s) + m;
}

// Categorical._log_prob, univariate.py:496-548: log_softmax(logits)[given].
__global__ void __launch_bounds__(256) categorical_lp_kernel(const int32_t* __restrict__ given,
                                                             int64_t given_n,
                                                             const float* __restrict__ logits,
                                                             int64_t logits_rows, int64_t C,
                                                             float* __restrict__ out, int64_t rows) {
  const int lane = threadIdx.x & 31;
  for (int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); row < rows;
       row += (int64_t)gridDim.x * 8) {
    const float* l = logits + (row % logits_rows) * C;
    const float lse = warp_row_lse(l, C, lane);
    if (lane == 0) {
      const int32_t k = given[row % given_n];
      out[row] = (k >= 0 && k < C) ? (l[k] - lse) : NAN;
    }
  }
}
// d lp / d logits = gout * (onehot(given) - softmax(logits)); written at full (row, C) size.
// A class outside [0, C) gives a NaN row, like its NaN log-prob (and the reference's
// sparse_softmax_cross_entropy_with_logits on a GPU).
__global__ void __launch_bounds__(256) categorical_bwd_kernel(
    const int32_t* __restrict__ given, int64_t given_n, const float* __restrict__ logits,
    int64_t logits_rows, int64_t C, const float* __restrict__ gout, float* __restrict__ dlogits,
    int64_t rows) {
  const int lane = threadIdx.x & 31;
  for (int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); row < rows;
       row += (int64_t)gridDim.x * 8) {
    const float* l = logits + (row % logits_rows) * C;
    const float lse = warp_row_lse(l, C, lane);
    const int32_t k = given[row % given_n];
    const bool in = k >= 0 && k < C;
    const float g = gout[row];
    for (int64_t j = lane; j < C; j += 32)
      dlogits[row * C + j] = in ? g * ((j == k ? 1.f : 0.f) - expf(l[j] - lse)) : NAN;
  }
}

// Dirichlet._log_prob, multivariate.py:665-677.
__global__ void __launch_bounds__(256) dirichlet_lp_kernel(const float* __restrict__ given,
                                                           int64_t given_rows,
                                                           const float* __restrict__ alpha,
                                                           int64_t alpha_rows, int64_t C,
                                                           float* __restrict__ out, int64_t rows) {
  const int lane = threadIdx.x & 31;
  for (int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); row < rows;
       row += (int64_t)gridDim.x * 8) {
    const float* x = given + (row % given_rows) * C;
    const float* a = alpha + (row % alpha_rows) * C;
    float sa = 0.f, slg = 0.f, s = 0.f;
    for (int64_t j = lane; j < C; j += 32) {
      const float aj = a[j];
      sa += aj;
      slg += lgammaf(aj);
      s += (aj - 1.f) * logf(x[j]);
    }
    sa = warp_sum(sa); slg = warp_sum(slg); s = warp_sum(s);
    if (lane == 0) out[row] = -(slg - lgammaf(sa)) + s;
  }
}
// d lp / d given_j = gout * (alpha_j - 1) / x_j  (the HMC-relevant gradient), full size.
__global__ void __launch_bounds__(256) dirichlet_bwd_given_kernel(
    const float* __restrict__ given, int64_t given_rows, const float* __restrict__ alpha,
    int64_t alpha_rows, int64_t C, const float* __restrict__ gout, float* __restrict__ dgiven,
    int64_t rows) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < rows * C;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / C, j = i % C;
    const float x = given[(row % given_rows) * C + j];
    const float a = alpha[(row % alpha_rows) * C + j];
    dgiven[i] = gout[row] * (a - 1.f) / x;
  }
}

// UnnormalizedMultinomial._log_prob, multivariate.py:435-443: sum x * (logits - [LSE]).
__global__ void __launch_bounds__(256) unnorm_multinomial_lp_kernel(
    const float* __restrict__ given, int64_t given_rows, const float* __restrict__ logits,
    int64_t logits_rows, int64_t C, int normalize, float* __restrict__ out, int64_t rows) {
  const int lane = threadIdx.x & 31;
  for (int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); row < rows;
       row += (int64_t)gridDim.x * 8) {
    const float* x = given + (row % given_rows) * C;
    const float* l = logits + (row % logits_rows) * C;
    const float lse = normalize ? warp_row_lse(l, C, lane) : 0.f;
    float s = 0.f;
    for (int64_t j = lane; j < C; j += 32) s += x[j] * (l[j] - lse);
    s = warp_sum(s);
    if (lane == 0) out[row] = s;
  }
}
// d lp / d logits_j = gout * (x_j - [sum_x * softmax_j]), full size.
__global__ void __launch_bounds__(256) unnorm_multinomial_bwd_kernel(
    const float* __restrict__ given, int64_t given_rows, const float* __restrict__ logits,
    int64_t logits_rows, int64_t C, int normalize, const float* __restrict__ gout,
    float* __restrict__ dlogits, int64_t rows) {
  const int lane = threadIdx.x & 31;
  for (int64_t row = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5); row < rows;
       row += (int64_t)gridDim.x * 8) {
    const float* x = given + (row % given_rows) * C;
    const float* l = logits + (row % logits_rows) * C;
    float lse = 0.f, sx = 0.f;
    if (normalize) {
      lse = warp_row_lse(l, C, lane);
      for (int64_t j = lane; j < C; j += 32) sx += x[j];
      sx = warp_sum(sx);
    }
    const float g = gout[row];
    for (int64_t j = lane; j < C; j += 32) {
      const float sm = normalize ? sx * expf(l[j] - lse) : 0.f;
      dlogits[row * C + j] = g * (x[j] - sm);
    }
  }
}

// MultivariateNormalCholesky._log_prob, multivariate.py:169-189.  One block per row; forward
// substitution in shared memory (x = L^{-1}(given - mean)), L read through L2.
__global__ void __launch_bounds__(128) mvn_chol_lp_kernel(const float* __restrict__ given,
                                                          int64_t given_rows,
                                                          const float* __restrict__ mean,
                                                          int64_t mean_rows,
                                                          const float* __restrict__ L,
                                                          int64_t L_mats, int64_t D,
                                                          float* __restrict__ out, int64_t rows,
                                                          float* __restrict__ x_out) {
  extern __shared__ float sh[];  // D floats + 32
  float* y = sh;
  float* red = sh + D;
  for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
    const float* g = given + (row % given_rows) * D;
    const float* mu = mean + (row % mean_rows) * D;
    const float* Lm = L + (row % L_mats) * D * D;
    for (int64_t j = threadIdx.x; j < D; j += blockDim.x) y[j] = g[j] - mu[j];
    __syncthreads();
    float logdet_half = 0.f;
    for (int64_t j = threadIdx.x; j < D; j += blockDim.x) logdet_half += logf(Lm[j * D + j]);
    // column-oriented forward substitution
    for (int64_t k = 0; k < D; ++k) {
      if (threadIdx.x == 0) y[k] = y[k] / Lm[k * D + k];
      __syncthreads();
      const float xk = y[k];
      for (int64_t j = k + 1 + threadIdx.x; j < D; j += blockDim.x) y[j] -= Lm[j * D + k] * xk;
      __syncthreads();
    }
    float ss = 0.f;
    for (int64_t j = threadIdx.x; j < D; j += blockDim.x) {
      ss += y[j] * y[j];
      if (x_out) x_out[row * D + j] = y[j];
    }
    ss = block_sum(ss, red);
    logdet_half = block_sum(logdet_half, red);
    if (threadIdx.x == 0)
      out[row] = -(float)D * kHalfLog2Pi - logdet_half - 0.5f * ss;
    __syncthreads();
  }
}
// d lp / d given = -L^{-T} x, x = L^{-1}(given - mean): back substitution, one block per row.
__global__ void __launch_bounds__(128) mvn_chol_bwd_given_kernel(
    const float* __restrict__ x_in, const float* __restrict__ L, int64_t L_mats, int64_t D,
    const float* __restrict__ gout, float* __restrict__ dgiven, int64_t rows) {
  extern __shared__ float sh[];
  float* y = sh;
  for (int64_t row = blockIdx.x; row < rows; row += gridDim.x) {
    const float* Lm = L + (row % L_mats) * D * D;
    for (int64_t j = threadIdx.x; j < D; j += blockDim.x) y[j] = x_in[row * D + j];
    __syncthreads();
    for (int64_t k = D - 1; k >= 0; --k) {
      if (threadIdx.x == 0) y[k] = y[k] / Lm[k * D + k];
      __syncthreads();
      const float zk = y[k];
      // L^T[j][k] = L[k][j], j < k
      for (int64_t j = threadIdx.x; j < k; j += blockDim.x) y[j] -= Lm[k * D + j] * zk;
      __syncthreads();
    }
    const float g = gout[row];
    for (int64_t j = threadIdx.x; j < D; j += blockDim.x) dgiven[row * D + j] = -g * y[j];
    __syncthreads();
  }
}

}  // namespace

extern "C" {

// Normal._log_prob, univariate.py:174-181 + base.py:303-304 group sum.
int zsb_logprob_normal_f32(const float* given, int64_t given_n, const float* mean, int64_t mean_n,
                           const float* logstd, int64_t logstd_n, float* out, int64_t n_out,
                           int64_t group, void* stream) {
  ZSB_REQUIRE(given_n > 0 && mean_n > 0 && logstd_n > 0 && group > 0 && n_out >= 0,
              "zsb_logprob_normal_f32: bad sizes");
  Ops3 ops{{given, mean, logstd}, {given_n, mean_n, logstd_n}};
  auto f = [=] __device__(float x, float mu, float ls, int64_t, int64_t) -> float {
    const float d = x - mu;
    return -kHalfLog2Pi - ls - 0.5f * expf(-2.f * ls) * d * d;
  };
  auto f4 = [=] __device__(float4 x, float4 mu, float4 ls, int64_t, int64_t) -> float {
    return (f(x.x, mu.x, ls.x, 0, 0) + f(x.y, mu.y, ls.y, 0, 0)) +
           (f(x.z, mu.z, ls.z, 0, 0) + f(x.w, mu.w, ls.w, 0, 0));
  };
  return launch_row_reduce4<3>(out, n_out, group, ops, f, f4, true, (cudaStream_t)stream,
                               "logprob_normal");
}

// Elementwise analytic backward; each output (nullable) has n_out*group elements.
int zsb_logprob_normal_bwd_f32(const float* given, int64_t given_n, const float* mean,
                               int64_t mean_n, const float* logstd, int64_t logstd_n,
                               const float* gout, int64_t n_out, int64_t group, float* dgiven,
                               float* dmean, float* dlogstd, void* stream) {
  ZSB_REQUIRE(given_n > 0 && mean_n > 0 && logstd_n > 0 && group > 0 && n_out >= 0,
              "zsb_logprob_normal_bwd_f32: bad sizes");
  Ops3 ops{{given, mean, logstd}, {given_n, mean_n, logstd_n}};
  auto f = [=] __device__(float x, float mu, float ls, int64_t i, int64_t row) -> float {
    const float g = gout[row];
    const float prec = expf(-2.f * ls), d = x - mu;
    if (dgiven) dgiven[i] = -g * prec * d;
    if (dmean) dmean[i] = g * prec * d;
    if (dlogstd) dlogstd[i] = g * (prec * d * d - 1.f);
    return 0.f;
  };
  auto f4 = [=] __device__(float4 x, float4 mu, float4 ls, int64_t i, int64_t row) -> float {
    const float g = gout[row];
    const float xs[4] = {x.x, x.y, x.z, x.w}, ms[4] = {mu.x, mu.y, mu.z, mu.w},
                lss[4] = {ls.x, ls.y, ls.z, ls.w};
    float dg[4], dl[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float prec = expf(-2.f * lss[k]), d = xs[k] - ms[k];
      dg[k] = -g * prec * d;
      dl[k] = g * (prec * d * d - 1.f);
    }
    if (dgiven) *reinterpret_cast<float4*>(dgiven + i) = make_float4(dg[0], dg[1], dg[2], dg[3]);
    if (dmean) *reinterpret_cast<float4*>(dmean + i) = make_float4(-dg[0], -dg[1], -dg[2], -dg[3]);
    if (dlogstd) *reinterpret_cast<float4*>(dlogstd + i) = make_float4(dl[0], dl[1], dl[2], dl[3]);
    return 0.f;
  };
  const bool side_ok = aligned16(dgiven) && aligned16(dmean) && aligned16(dlogstd);
  return launch_row_reduce4<3>(nullptr, n_out, group, ops, f, f4, side_ok, (cudaStream_t)stream,
                               "logprob_normal_bwd");
}

// Bernoulli._log_prob, univariate.py:398-403 (given already cast to float by the host, :399).
int zsb_logprob_bernoulli_f32(const float* given, int64_t given_n, const float* logits,
                              int64_t logits_n, float* out, int64_t n_out, int64_t group,
                              void* stream) {
  ZSB_REQUIRE(given_n > 0 && logits_n > 0 && group > 0 && n_out >= 0,
              "zsb_logprob_bernoulli_f32: bad sizes");
  Ops3 ops{{given, logits, nullptr}, {given_n, logits_n, 1}};
  auto f = [=] __device__(float x, float l, float, int64_t, int64_t) -> float {
    return bernoulli_lp(x, l);
  };
  auto f4 = [=] __device__(float4 x, float4 l, float4, int64_t, int64_t) -> float {
    return (bernoulli_lp(x.x, l.x) + bernoulli_lp(x.y, l.y)) +
           (bernoulli_lp(x.z, l.z) + bernoulli_lp(x.w, l.w));
  };
  return launch_row_reduce4<2>(out, n_out, group, ops, f, f4, true, (cudaStream_t)stream,
                               "logprob_bernoulli");
}
int zsb_logprob_bernoulli_bwd_f32(const float* given, int64_t given_n, const float* logits,
                                  int64_t logits_n, const float* gout, int64_t n_out,
                                  int64_t group, float* dlogits, void* stream) {
  ZSB_REQUIRE(given_n > 0 && logits_n > 0 && group > 0 && n_out >= 0 && dlogits,
              "zsb_logprob_bernoulli_bwd_f32: bad sizes");
  Ops3 ops{{given, logits, gout}, {given_n, logits_n, 1}};
  auto f = [=] __device__(float x, float l, float, int64_t i, int64_t row) -> float {
    dlogits[i] = gout[row] * (x - sigmoidf_(l));
    return 0.f;
  };
  auto f4 = [=] __device__(float4 x, float4 l, float4, int64_t i, int64_t row) -> float {
    const float g = gout[row];
    *reinterpret_cast<float4*>(dlogits + i) =
        make_float4(g * (x.x - sigmoidf_(l.x)), g * (x.y - sigmoidf_(l.y)),
                    g * (x.z - sigmoidf_(l.z)), g * (x.w - sigmoidf_(l.w)));
    return 0.f;
  };
  return launch_row_reduce4<2>(nullptr, n_out, group, ops, f, f4, aligned16(dlogits),
                               (cudaStream_t)stream, "logprob_bernoulli_bwd");
}

int zsb_logprob_categorical_f32(const int32_t* given, int64_t given_n, const float* logits,
                                int64_t logits_rows, int64_t n_categories, float* out,
                                int64_t rows, void* stream) {
  ZSB_REQUIRE(given_n > 0 && logits_rows > 0 && n_categories > 0 && rows >= 0,
              "zsb_logprob_categorical_f32: bad sizes");
  if (rows == 0) return ZSB_OK;
  int64_t blocks = zsb_ceil_div(rows, 8);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  categorical_lp_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      given, given_n, logits, logits_rows, n_categories, out, rows);
  return zsb_check_launch("logprob_categorical");
}
int zsb_logprob_categorical_bwd_f32(const int32_t* given, int64_t given_n, const float* logits,
                                    int64_t logits_rows, int64_t n_categories, const float* gout,
                                    float* dlogits, int64_t rows, void* stream) {
  ZSB_REQUIRE(given_n > 0 && logits_rows > 0 && n_categories > 0 && rows >= 0,
              "zsb_logprob_categorical_bwd_f32: bad sizes");
  if (rows == 0) return ZSB_OK;
  int64_t blocks = zsb_ceil_div(rows, 8);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  categorical_bwd_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      given, given_n, logits, logits_rows, n_categories, gout, dlogits, rows);
  return zsb_check_launch("logprob_categorical_bwd");
}

int zsb_logprob_dirichlet_f32(const float* given, int64_t given_rows, const float* alpha,
                              int64_t alpha_rows, int64_t n_categories, float* out, int64_t rows,
                              void* stream) {
  ZSB_REQUIRE(given_rows > 0 && alpha_rows > 0 && n_categories >= 2 && rows >= 0,
              "zsb_logprob_dirichlet_f32: bad sizes (n_categories must be >= 2)");
  if (rows == 0) return ZSB_OK;
  int64_t blocks = zsb_ceil_div(rows, 8);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  dirichlet_lp_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      given, given_rows, alpha, alpha_rows, n_categories, out, rows);
  return zsb_check_launch("logprob_dirichlet");
}
int zsb_logprob_dirichlet_bwd_given_f32(const float* given, int64_t given_rows,
                                        const float* alpha, int64_t alpha_rows,
                                        int64_t n_categories, const float* gout, float* dgiven,
                                        int64_t rows, void* stream) {
  ZSB_REQUIRE(given_rows > 0 && alpha_rows > 0 && n_categories >= 2 && rows >= 0,
              "zsb_logprob_dirichlet_bwd_given_f32: bad sizes");
  if (rows == 0) return ZSB_OK;
  int64_t blocks = zsb_ceil_div(rows * n_categories, 256);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  dirichlet_bwd_given_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      given, given_rows, alpha, alpha_rows, n_categories, gout, dgiven, rows);
  return zsb_check_launch("logprob_dirichlet_bwd_given");
}

int zsb_logprob_unnorm_multinomial_f32(const float* given, int64_t given_rows,
                                       const float* logits, int64_t logits_rows,
                                       int64_t n_categories, int normalize_logits, float* out,
                                       int64_t rows, void* stream) {
  ZSB_REQUIRE(given_rows > 0 && logits_rows > 0 && n_categories > 0 && rows >= 0,
              "zsb_logprob_unnorm_multinomial_f32: bad sizes");
  if (rows == 0) return ZSB_OK;
  int64_t blocks = zsb_ceil_div(rows, 8);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  unnorm_multinomial_lp_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      given, given_rows, logits, logits_rows, n_categories, normalize_logits, out, rows);
  return zsb_check_launch("logprob_unnorm_multinomial");
}
int zsb_logprob_unnorm_multinomial_bwd_f32(const float* given, int64_t given_rows,
                                           const float* logits, int64_t logits_rows,
                                           int64_t n_categories, int normalize_logits,
                                           const float* gout, float* dlogits, int64_t rows,
                                           void* stream) {
  ZSB_REQUIRE(given_rows > 0 && logits_rows > 0 && n_categories > 0 && rows >= 0,
              "zsb_logprob_unnorm_multinomial_bwd_f32: bad sizes");
  if (rows == 0) return ZSB_OK;
  int64_t blocks = zsb_ceil_div(rows, 8);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  unnorm_multinomial_bwd_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      given, given_rows, logits, logits_rows, n_categories, normalize_logits, gout, dlogits, rows);
  return zsb_check_launch("logprob_unnorm_multinomial_bwd");
}

// x_out (nullable, rows*D) receives L^{-1}(given-mean) for the backward.
int zsb_logprob_mvn_chol_f32(const float* given, int64_t given_rows, const float* mean,
                             int64_t mean_rows, const float* cov_tril, int64_t tril_mats,
                             int64_t n_dim, float* out, float* x_out, int64_t rows,
                             void* stream) {
  ZSB_REQUIRE(given_rows > 0 && mean_rows > 0 && tril_mats > 0 && n_dim > 0 && rows >= 0,
              "zsb_logprob_mvn_chol_f32: bad sizes");
  ZSB_REQUIRE(n_dim <= 12000, "zsb_logprob_mvn_chol_f32: n_dim too large for shared memory");
  if (rows == 0) return ZSB_OK;
  int64_t blocks = rows < ZSB_NUM_SMS * 8 ? rows : ZSB_NUM_SMS * 8;
  const size_t smem = (size_t)(n_dim + 32) * sizeof(float);
  mvn_chol_lp_kernel<<<(unsigned)blocks, 128, smem, (cudaStream_t)stream>>>(
      given, given_rows, mean, mean_rows, cov_tril, tril_mats, n_dim, out, rows, x_out);
  return zsb_check_launch("logprob_mvn_chol");
}
int zsb_logprob_mvn_chol_bwd_given_f32(const float* x_in, const float* cov_tril,
                                       int64_t tril_mats, int64_t n_dim, const float* gout,
                                       float* dgiven, int64_t rows, void* stream) {
  ZSB_REQUIRE(tril_mats > 0 && n_dim > 0 && rows >= 0, "zsb_logprob_mvn_chol_bwd_given_f32: bad sizes");
  ZSB_REQUIRE(n_dim <= 12000, "zsb_logprob_mvn_chol_bwd_given_f32: n_dim too large");
  if (rows == 0) return ZSB_OK;
  int64_t blocks = rows < ZSB_NUM_SMS * 8 ? rows : ZSB_NUM_SMS * 8;
  const size_t smem = (size_t)(n_dim + 32) * sizeof(float);
  mvn_chol_bwd_given_kernel<<<(unsigned)blocks, 128, smem, (cudaStream_t)stream>>>(
      x_in, cov_tril, tril_mats, n_dim, gout, dgiven, rows);
  return zsb_check_launch("logprob_mvn_chol_bwd_given");
}

// out[r] = sum_{j<group} in[r*group + j]   (Distribution.log_prob's reduce_sum, base.py:303-304)
int zsb_group_sum_f32(const float* in, float* out, int64_t n_out, int64_t group, void* stream) {
  ZSB_REQUIRE(group > 0 && n_out >= 0, "zsb_group_sum_f32: bad sizes");
  Ops3 ops{{in, nullptr, nullptr}, {n_out * group > 0 ? n_out * group : 1, 1, 1}};
  auto f = [=] __device__(float v, float, float, int64_t, int64_t) -> float { return v; };
  auto f4 = [=] __device__(float4 v, float4, float4, int64_t, int64_t) -> float {
    return (v.x + v.y) + (v.z + v.w);
  };
  return launch_row_reduce4<1>(out, n_out, group, ops, f, f4, true, (cudaStream_t)stream,
                               "group_sum");
}

// K7: Normal._sample (univariate.py:161-172) fused with log q(z) of the drawn sample
// (StochasticTensor.cond_log_p, bn.py:194-204).  eps: injected standard normals [n_out*group] or
// NULL -> in-kernel Philox (stream SAMPLE, counter (i/4, 0, iter, stream)).
// z = eps * exp(logstd) + mean;   logq[r] = sum_j (-0.5 log 2pi - logstd - 0.5 eps^2)
// (identical to Normal._log_prob at z because (z - mean) * exp(-logstd) == eps up to rounding;
// the kernel evaluates the reference expression on z itself for parity).
int zsb_reparam_normal_f32(const float* mean, int64_t mean_n, const float* logstd,
                           int64_t logstd_n, const float* eps, uint64_t seed, uint32_t iter,
                           float* z_out, float* eps_out, float* logq_out, int64_t n_out,
                           int64_t group, void* stream) {
  ZSB_REQUIRE(mean_n > 0 && logstd_n > 0 && group > 0 && n_out >= 0 && z_out,
              "zsb_reparam_normal_f32: bad sizes");
  Ops3 ops{{mean, logstd, nullptr}, {mean_n, logstd_n, 1}};
  // no row sums requested and one element per row (the plain sample() call): regroup by four so
  // the 128-bit path applies -- element i still reads operand[i % operand_n]
  if (!logq_out && group == 1 && n_out % 4 == 0) { group = 4; n_out /= 4; }
  const uint32_t* ep = zsb_epoch_ptr();
  auto f = [=] __device__(float mu, float ls, float, int64_t i, int64_t) -> float {
    float e;
    if (eps) {
      e = eps[i];
    } else {
      float z4[4];
      philox_normal4(seed, ZSB_STREAM_SAMPLE, iter + (ep ? *ep : 0u),
                     (uint32_t)((uint64_t)i >> 34),
                     (uint32_t)(i >> 2), z4);
      e = z4[i & 3];
    }
    const float z = e * expf(ls) + mu;
    z_out[i] = z;
    if (eps_out) eps_out[i] = e;
    const float d = z - mu;
    return -kHalfLog2Pi - ls - 0.5f * expf(-2.f * ls) * d * d;
  };
  // 4 consecutive elements = exactly one Philox block (element i is component i & 3 of block
  // i >> 2): the 128-bit path generates it once instead of once per element
  auto f4 = [=] __device__(float4 mu, float4 ls, float4, int64_t i, int64_t) -> float {
    float e[4];
    if (eps) {
      const float4 t = *reinterpret_cast<const float4*>(eps + i);
      e[0] = t.x; e[1] = t.y; e[2] = t.z; e[3] = t.w;
    } else {
      philox_normal4(seed, ZSB_STREAM_SAMPLE, iter + (ep ? *ep : 0u),
                     (uint32_t)((uint64_t)i >> 34), (uint32_t)(i >> 2), e);
    }
    const float ms[4] = {mu.x, mu.y, mu.z, mu.w}, lss[4] = {ls.x, ls.y, ls.z, ls.w};
    float z[4], lq[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      z[k] = e[k] * expf(lss[k]) + ms[k];
      const float d = z[k] - ms[k];
      lq[k] = -kHalfLog2Pi - lss[k] - 0.5f * expf(-2.f * lss[k]) * d * d;
    }
    *reinterpret_cast<float4*>(z_out + i) = make_float4(z[0], z[1], z[2], z[3]);
    if (eps_out) *reinterpret_cast<float4*>(eps_out + i) = make_float4(e[0], e[1], e[2], e[3]);
    return (lq[0] + lq[1]) + (lq[2] + lq[3]);
  };
  const bool side_ok = aligned16(z_out) && aligned16(eps_out) && aligned16(eps);
  return launch_row_reduce4<2>(logq_out, n_out, group, ops, f, f4, side_ok, (cudaStream_t)stream,
                               "reparam_normal");
}

// Bernoulli._sample, univariate.py:386-396: (u < sigmoid(logits)) as int32; u injected or Philox.
int zsb_sample_bernoulli_i32(const float* logits, int64_t logits_n, const float* u, uint64_t seed,
                             uint32_t iter, int32_t* out, int64_t n, void* stream) {
  ZSB_REQUIRE(logits_n > 0 && n >= 0, "zsb_sample_bernoulli_i32: bad sizes");
  const uint32_t* ep = zsb_epoch_ptr();
  auto f = [=] __device__(int64_t i) {
    float uu;
    if (u) {
      uu = u[i];
    } else {
      const Philox4 r = philox4x32_10((uint32_t)(i >> 2), (uint32_t)((uint64_t)i >> 34),
                                      iter + (ep ? *ep : 0u),
                                      ZSB_STREAM_SAMPLE, (uint32_t)seed, (uint32_t)(seed >> 32));
      const uint32_t w = (i & 3) == 0 ? r.x : (i & 3) == 1 ? r.y : (i & 3) == 2 ? r.z : r.w;
      uu = u32_to_uniform(w);
    }
    out[i] = uu < sigmoidf_(logits[i % logits_n]) ? 1 : 0;
  };
  return launch_elementwise(n, f, (cudaStream_t)stream, "sample_bernoulli");
}

}  // extern "C"
