// K1 (widened, SURVEY 8f row 3): the remaining elementwise univariate densities of
// zhusuan/distributions/univariate.py behind ONE pair of entry points, on the same row-reduce
// template as Normal/Bernoulli (modular broadcast of every operand + sum over the last
// `group` elements, distributions/base.py:303-304):
//
//   id  distribution  params (a, b)            reference _log_prob
//   0   FoldNormal    mean, logstd             univariate.py:319-329
//   1   Uniform       minval, maxval           univariate.py:646-660
//   2   Gamma         alpha, beta              univariate.py:737-747
//   3   Beta          alpha, beta              univariate.py:833-851
//   4   Poisson       rate, -                  univariate.py:922-933
//   5   Binomial      logits, n_experiments    univariate.py:1047-1064
//   6   InverseGamma  alpha, beta              univariate.py:1146-1158
//   7   Laplace       loc, scale               univariate.py:1267-1273
//   8   BinConcrete   temperature, logits      univariate.py:1381-1400
//
// The backward entry point writes the full-size elementwise gradients wrt given / a / b (each
// nullable), i.e. what tf.gradients yields before the broadcast reduction (done by the host).
#include "common.cuh"

namespace {

constexpr float kHalfLog2Pi = 0.9189385332046727f;
constexpr float kLog2 = 0.6931471805599453f;

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

// LANES threads per row of `group` elements; F(x, a, b, element index, row) -> contribution.
template <int LANES, class F>
__global__ void __launch_bounds__(256) uni_row_kernel(float* __restrict__ out, int64_t n_out,
                                                      int64_t group, Ops3 ops, F f) {
  const int rows_per_block = 256 / LANES;
  const int lane = threadIdx.x % LANES;
  const int rib = threadIdx.x / LANES;
  for (int64_t row = (int64_t)blockIdx.x * rows_per_block + rib; row < n_out;
       row += (int64_t)gridDim.x * rows_per_block) {
    const int64_t i0 = row * group;
    int64_t base[3];
#pragma unroll
    for (int o = 0; o < 3; ++o) {
      const int64_t n = ops.n[o];
      base[o] = (n == 1 || n == group) ? 0 : (n == n_out * group ? i0 : i0 % n);
    }
    float acc = 0.f;
    for (int64_t j = lane; j < group; j += LANES) {
      const float x = op_at(ops.p[0], ops.n[0], base[0], j);
      const float a = op_at(ops.p[1], ops.n[1], base[1], j);
      const float b = ops.p[2] ? op_at(ops.p[2], ops.n[2], base[2], j) : 0.f;
      acc += f(x, a, b, i0 + j, row);
    }
    acc = sub_warp_sum<LANES>(acc);
    if (lane == 0 && out) out[row] = acc;
  }
}

template <class F>
int launch_uni(float* out, int64_t n_out, int64_t group, Ops3 ops, F f, cudaStream_t st,
               const char* what) {
  if (n_out == 0) return ZSB_OK;
  int lanes = 1;
  while (lanes < 32 && lanes * 2 <= group) lanes <<= 1;
  const int rows_per_block = 256 / lanes;
  int64_t blocks = zsb_ceil_div(n_out, rows_per_block);
  const int64_t cap = (int64_t)ZSB_NUM_SMS * 16;
  if (blocks > cap) blocks = cap;
#define ZSB_UR(LN) uni_row_kernel<LN><<<(unsigned)blocks, 256, 0, st>>>(out, n_out, group, ops, f)
  switch (lanes) {
    case 1: ZSB_UR(1); break;
    case 2: ZSB_UR(2); break;
    case 4: ZSB_UR(4); break;
    case 8: ZSB_UR(8); break;
    case 16: ZSB_UR(16); break;
    default: ZSB_UR(32); break;
  }
#undef ZSB_UR
  return zsb_check_launch(what);
}

__device__ __forceinline__ float softplusf_(float t) {       // tf.nn.softplus
  return fmaxf(t, 0.f) + log1pf(expf(-fabsf(t)));
}
// psi(x): for x <= 0 the reflection psi(x) = psi(1 - x) - pi cot(pi x) (as Eigen and torch do;
// infinite at 0 and the negative integers, NaN at -inf), then for x > 0 the recurrence up to
// x >= 6 -- at most 6 steps, so no argument can keep it looping -- and the asymptotic series.
// NaN and +inf pass straight through.
__device__ __forceinline__ float digammaf_(float x) {
  float r = 0.f;
  if (x <= 0.f) {
    float s, c;
    sincospif(x, &s, &c);
    r = -3.14159265358979f * c / s;
    x = 1.f - x;
  }
  for (int k = 0; k < 6 && x < 6.f; ++k) { r -= 1.f / x; x += 1.f; }
  const float i = 1.f / x, i2 = i * i;
  return r + logf(x) - 0.5f * i - i2 * (1.f / 12.f - i2 * (1.f / 120.f - i2 * (1.f / 252.f)));
}

enum { D_FOLDNORMAL = 0, D_UNIFORM, D_GAMMA, D_BETA, D_POISSON, D_BINOMIAL, D_INVGAMMA,
       D_LAPLACE, D_BINCONCRETE, D_COUNT };

template <int DIST>
__device__ __forceinline__ float uni_lp(float x, float a, float b) {
  switch (DIST) {
    case D_FOLDNORMAL: {                 // a = mean, b = logstd
      const float prec = expf(-2.f * b), d = x - a;
      const float mask = logf(x >= 0.f ? 1.f : 0.f);
      return (-kHalfLog2Pi - (b + 0.5f * prec * d * d) + softplusf_(-2.f * a * x * prec)) + mask;
    }
    case D_UNIFORM: {                    // a = minval, b = maxval
      const float mask = (a <= x && x < b) ? 1.f : 0.f;
      return logf((1.f / (b - a)) * mask);
    }
    case D_GAMMA:                        // a = alpha, b = beta
      return a * logf(b) - lgammaf(a) + (a - 1.f) * logf(x) - b * x;
    case D_BETA:
      return (a - 1.f) * logf(x) + (b - 1.f) * logf(1.f - x) -
             (lgammaf(a) + lgammaf(b) - lgammaf(a + b));
    case D_POISSON:                      // a = rate
      return x * logf(a) - a - lgammaf(x + 1.f);
    case D_BINOMIAL:                     // a = logits, b = n
      return lgammaf(b + 1.f) - lgammaf(b - x + 1.f) - lgammaf(x + 1.f) + x * a +
             b * (-softplusf_(a));
    case D_INVGAMMA:
      return a * logf(b) - lgammaf(a) - (a + 1.f) * logf(x) - b / x;
    case D_LAPLACE:                      // a = loc, b = scale
      return -kLog2 - logf(b) - fabsf(x - a) / b;
    case D_BINCONCRETE: {                // a = temperature, b = logits
      const float lx = logf(x), l1x = logf(1.f - x);
      const float t = a * (lx - l1x) - b;
      return logf(a) - lx - l1x + t - 2.f * softplusf_(t);
    }
  }
  return 0.f;
}

// gradients of the elementwise log density wrt (x, a, b)
template <int DIST>
__device__ __forceinline__ void uni_grad(float x, float a, float b, float& dx, float& da,
                                         float& db) {
  dx = da = db = 0.f;
  switch (DIST) {
    case D_FOLDNORMAL: {
      const float prec = expf(-2.f * b), d = x - a;
      const float t = -2.f * a * x * prec, s = sigmoidf_(t);
      dx = -prec * d + s * (-2.f * a * prec);
      da = prec * d + s * (-2.f * x * prec);
      db = -1.f + prec * d * d - 2.f * s * t;
      break;
    }
    case D_UNIFORM: {                    // d log(p * mask): 0/0 outside the support, as in TF
      const bool in = (a <= x && x < b);
      const float nan = __int_as_float(0x7fc00000);
      da = in ? 1.f / (b - a) : nan;
      db = in ? -1.f / (b - a) : nan;
      break;
    }
    case D_GAMMA:
      dx = (a - 1.f) / x - b;
      da = logf(b) - digammaf_(a) + logf(x);
      db = a / b - x;
      break;
    case D_BETA: {
      const float pab = digammaf_(a + b);
      dx = (a - 1.f) / x - (b - 1.f) / (1.f - x);
      da = logf(x) - digammaf_(a) + pab;
      db = logf(1.f - x) - digammaf_(b) + pab;
      break;
    }
    case D_POISSON:
      da = x / a - 1.f;
      break;
    case D_BINOMIAL:
      da = x - b * sigmoidf_(a);
      break;
    case D_INVGAMMA:
      dx = -(a + 1.f) / x + b / (x * x);
      da = logf(b) - digammaf_(a) - logf(x);
      db = a / b - 1.f / x;
      break;
    case D_LAPLACE: {
      const float d = x - a;
      const float sg = (d > 0.f) ? 1.f : (d < 0.f ? -1.f : 0.f);
      dx = -sg / b;
      da = sg / b;
      db = -1.f / b + fabsf(d) / (b * b);
      break;
    }
    case D_BINCONCRETE: {
      const float lg = logf(x) - logf(1.f - x);
      const float t = a * lg - b;
      const float u = 1.f - 2.f * sigmoidf_(t);
      dx = -1.f / x + 1.f / (1.f - x) + u * a * (1.f / x + 1.f / (1.f - x));
      da = 1.f / a + u * lg;
      db = -u;
      break;
    }
  }
}

template <int DIST>
int fwd(Ops3 ops, float* out, int64_t n_out, int64_t group, cudaStream_t st) {
  auto f = [=] __device__(float x, float a, float b, int64_t, int64_t) -> float {
    return uni_lp<DIST>(x, a, b);
  };
  return launch_uni(out, n_out, group, ops, f, st, "logprob_univariate");
}
template <int DIST>
int bwd(Ops3 ops, const float* gout, int64_t n_out, int64_t group, float* dgiven, float* da_out,
        float* db_out, cudaStream_t st) {
  auto f = [=] __device__(float x, float a, float b, int64_t i, int64_t row) -> float {
    float dx, da, db;
    uni_grad<DIST>(x, a, b, dx, da, db);
    const float g = gout[row];
    if (dgiven) dgiven[i] = g * dx;
    if (da_out) da_out[i] = g * da;
    if (db_out) db_out[i] = g * db;
    return 0.f;
  };
  return launch_uni(nullptr, n_out, group, ops, f, st, "logprob_univariate_bwd");
}

}  // namespace

extern "C" {

int zsb_logprob_univariate_f32(int dist, const float* given, int64_t given_n, const float* a,
                               int64_t a_n, const float* b, int64_t b_n, float* out,
                               int64_t n_out, int64_t group, void* stream) {
  ZSB_REQUIRE(dist >= 0 && dist < D_COUNT, "zsb_logprob_univariate_f32: unknown distribution id");
  ZSB_REQUIRE(given_n > 0 && a_n > 0 && group > 0 && n_out >= 0 && (!b || b_n > 0),
              "zsb_logprob_univariate_f32: bad sizes");
  ZSB_REQUIRE(b || dist == D_POISSON, "zsb_logprob_univariate_f32: second parameter missing");
  Ops3 ops{{given, a, b}, {given_n, a_n, b ? b_n : 1}};
  cudaStream_t st = (cudaStream_t)stream;
  switch (dist) {
    case D_FOLDNORMAL: return fwd<D_FOLDNORMAL>(ops, out, n_out, group, st);
    case D_UNIFORM: return fwd<D_UNIFORM>(ops, out, n_out, group, st);
    case D_GAMMA: return fwd<D_GAMMA>(ops, out, n_out, group, st);
    case D_BETA: return fwd<D_BETA>(ops, out, n_out, group, st);
    case D_POISSON: return fwd<D_POISSON>(ops, out, n_out, group, st);
    case D_BINOMIAL: return fwd<D_BINOMIAL>(ops, out, n_out, group, st);
    case D_INVGAMMA: return fwd<D_INVGAMMA>(ops, out, n_out, group, st);
    case D_LAPLACE: return fwd<D_LAPLACE>(ops, out, n_out, group, st);
    default: return fwd<D_BINCONCRETE>(ops, out, n_out, group, st);
  }
}

int zsb_logprob_univariate_bwd_f32(int dist, const float* given, int64_t given_n, const float* a,
                                   int64_t a_n, const float* b, int64_t b_n, const float* gout,
                                   int64_t n_out, int64_t group, float* dgiven, float* da,
                                   float* db, void* stream) {
  ZSB_REQUIRE(dist >= 0 && dist < D_COUNT,
              "zsb_logprob_univariate_bwd_f32: unknown distribution id");
  ZSB_REQUIRE(given_n > 0 && a_n > 0 && group > 0 && n_out >= 0 && gout && (!b || b_n > 0),
              "zsb_logprob_univariate_bwd_f32: bad sizes");
  ZSB_REQUIRE(b || dist == D_POISSON, "zsb_logprob_univariate_bwd_f32: second parameter missing");
  Ops3 ops{{given, a, b}, {given_n, a_n, b ? b_n : 1}};
  cudaStream_t st = (cudaStream_t)stream;
  switch (dist) {
    case D_FOLDNORMAL: return bwd<D_FOLDNORMAL>(ops, gout, n_out, group, dgiven, da, db, st);
    case D_UNIFORM: return bwd<D_UNIFORM>(ops, gout, n_out, group, dgiven, da, db, st);
    case D_GAMMA: return bwd<D_GAMMA>(ops, gout, n_out, group, dgiven, da, db, st);
    case D_BETA: return bwd<D_BETA>(ops, gout, n_out, group, dgiven, da, db, st);
    case D_POISSON: return bwd<D_POISSON>(ops, gout, n_out, group, dgiven, da, db, st);
    case D_BINOMIAL: return bwd<D_BINOMIAL>(ops, gout, n_out, group, dgiven, da, db, st);
    case D_INVGAMMA: return bwd<D_INVGAMMA>(ops, gout, n_out, group, dgiven, da, db, st);
    case D_LAPLACE: return bwd<D_LAPLACE>(ops, gout, n_out, group, dgiven, da, db, st);
    default: return bwd<D_BINCONCRETE>(ops, gout, n_out, group, dgiven, da, db, st);
  }
}

}  // extern "C"
