// The BNN regression log-joint of examples/bayesian_neural_nets/bnn_vi.py:18-35, 83-86 (and
// bnn_sgmcmc.py:19-35, 74-77) for K particles, its gradient w.r.t. both weight layers and
// y_logstd, and the per-point predictions, in ONE launch:
//   w0 [K, H, n_in+1] ~ N(0, exp(logstd0)),  w1 [K, 1, H+1] ~ N(0, exp(logstd1))
//   h0 = [x, 1];  a1 = h0 w0^T / sqrt(n_in+1);  r1 = relu(a1);  h1 = [r1, 1]
//   y_mean = h1 w1^T / sqrt(H+1);   y ~ N(y_mean, exp(y_logstd))
//   lp[k] = sum log p(w0[k]) + sum log p(w1[k]) + n_train * mean_b log p(y_b | x_b, w[k])
// This is what the variational objectives (elbo / iw_objective / klpq / is_loglikelihood), HMC
// and test-set evaluation need from the net: a value, a gradient to backpropagate through
// (y_logstd is learned by bnn_vi.py, so it is read from device memory, never synced to the host)
// and y_mean / log N(y_b; y_mean, exp(y_logstd)) per particle and point.
//
// Layout follows csrc/sgmcmc_bnn.cu: one warp per particle, lane l owns hidden units l and l+32
// (their w0 rows, gradient accumulators and w1 entries live in registers), rows are read from
// shared memory with 128-bit broadcast loads, and the forward pass of row block i+1 is issued
// between the butterfly rounds of block i (PB = 4 rows per block).  It differs where the callers
// differ: rows are staged in tiles of up to 512, so any number of rows works (full-batch HMC, the
// test set), and the particle loop is block-uniform because the tiles are separated by
// __syncthreads; the value is accumulated with lane b % 32 owning row b's squared residual (one
// warp reduction at the end, so the rounding error grows like sqrt(B / 32) rather than B); only
// the outputs asked for are written, and without g0 / g1 the backward pass is compiled out.  The
// SG-MCMC kernel is left alone: sharing its row loop would make a tuned, bit-pinned update step
// branch on which caller it serves (tiling, value accumulation and the output set all differ).
//
// No floating-point atomics: every sum has a fixed order, so repeated calls are bitwise equal.
#include <atomic>

#include "common.cuh"

namespace {

constexpr int MAX_IN1 = 16;   // n_in + 1 <= 16
constexpr int MAX_H = 64;     // two hidden units per lane
constexpr int TILE = 512;     // rows staged per tile (a multiple of 32: lane b % 32 owns row b)
constexpr int NW = 8;         // warps (particles in flight) per block
constexpr int PB = 4;         // rows processed together (independent FMA / shuffle chains)
constexpr float HALF_LOG_2PI = 0.918938533204672742f;

struct LjArgs {
  const float* w0; const float* w1; const float* x; const float* y;
  const float* logstd0; const float* logstd1; const float* y_logstd;
  float* lp; float* g0; float* g1; float* gys; float* ym; float* ll;
  int64_t K; int B, n_in, H, ls0_n, ls1_n, tile_rows;
  float n_train;
};

template <int IN1, bool GRAD>
__global__ void __launch_bounds__(32 * NW, 2) bnn_logjoint_kernel(LjArgs a) {
  extern __shared__ float4 sh4[];
  constexpr int X4 = (IN1 + 3) / 4;     // a staged row = X4 float4 (bias column, 0 pad)
  constexpr int XP = 4 * X4;
  const int H = a.H, H1 = H + 1, n0 = H * IN1;
  const int n0p = (n0 + 3) & ~3, n1p = (H1 + 3) & ~3;
  const int TR = a.tile_rows;                                // multiple of PB
  float* xs = reinterpret_cast<float*>(sh4);                 // [TR + PB][XP]
  float2* yc = reinterpret_cast<float2*>(xs + (TR + PB) * XP);   // [TR] {y, dout coefficient or 0}
  float* pr0 = reinterpret_cast<float*>(yc + TR);            // [n0p] prior precision exp(-2 ls)
  float* pr1 = pr0 + n0p;                                    // [n1p]
  float* stg = pr1 + n1p;                                    // [NW][n0p + n1p] weights / gradients
  __shared__ float red[32];
  const float inv_s0 = rsqrtf((float)IN1), inv_s1 = rsqrtf((float)H1);
  const float ys = *a.y_logstd;
  const float prec_y = expf(-2.f * ys);
  const float lik_scale = a.n_train / (float)a.B;
  // d lp / d (h1 . w1) = prec_y (y - y_mean) * (n_train / B) / sqrt(H + 1)
  const float cf = prec_y * lik_scale * inv_s1;
  const float c_ll = -HALF_LOG_2PI - ys;                     // log N(y; m, s) = c_ll - prec/2 r^2
  float lsum = 0.f;
  for (int i = threadIdx.x; i < n0p; i += blockDim.x) {
    float p = 0.f;
    if (i < n0) { const float l = a.logstd0[i % a.ls0_n]; p = expf(-2.f * l); lsum += l; }
    pr0[i] = p;
  }
  for (int i = threadIdx.x; i < n1p; i += blockDim.x) {
    float p = 0.f;
    if (i < H1) { const float l = a.logstd1[i % a.ls1_n]; p = expf(-2.f * l); lsum += l; }
    pr1[i] = p;
  }
  lsum = block_sum(lsum, red);
  // scalars the row loop needs only at its end or in the owning lane: read from shared memory
  // where used, so they hold no registers across the loop (IN1 = 16 with the gradient is at 128)
  __shared__ float cst[3];
  if (threadIdx.x == 0) {
    cst[0] = -(float)(n0 + H1) * HALF_LOG_2PI - lsum;   // weight-independent part of the prior
    cst[1] = c_ll;
    cst[2] = -0.5f * prec_y;
  }

  const int ntiles = (a.B + TR - 1) / TR;
  auto stage = [&](int t) {
    const int r0 = t * TR, nr = min(TR, a.B - r0);
    for (int i = threadIdx.x; i < (TR + PB) * XP; i += blockDim.x) {
      const int b = i / XP, k = i % XP;
      xs[i] = (b < nr) ? ((k < a.n_in) ? a.x[(int64_t)(r0 + b) * a.n_in + k]
                                       : (k == a.n_in ? 1.f : 0.f))
                       : 0.f;
    }
    for (int i = threadIdx.x; i < TR; i += blockDim.x)
      yc[i] = (i < nr) ? make_float2(a.y[r0 + i], cf) : make_float2(0.f, 0.f);
  };
  if (ntiles == 1) stage(0);              // one tile: staged once for every particle
  __syncthreads();

  // warp index through a shuffle: provably warp-uniform, so the shuffles below are plain SHFL
  const int lane = threadIdx.x & 31;
  const int wib = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  float* S0 = stg + wib * (n0p + n1p);
  float* S1 = S0 + n0p;

  // block-uniform particle loop: every warp of the block walks every tile, warps past K idle
  for (int64_t base = (int64_t)blockIdx.x * NW; base < a.K; base += (int64_t)gridDim.x * NW) {
    const int64_t c = base + wib;
    const bool act = c < a.K;
    float W[2][IN1], G[2][IN1];
    float w1r[2], w1s[2], g1r[2];
    float w1b = 0.f, g1b = 0.f, rsq = 0.f;
    if (act) {
      const float* w0c = a.w0 + c * n0;
      const float* w1c = a.w1 + c * H1;
      for (int i = lane; i < n0; i += 32) S0[i] = w0c[i];
      for (int i = lane; i < H1; i += 32) S1[i] = w1c[i];
      __syncwarp();
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int m = lane + 32 * u;
        const bool mv = m < H;
#pragma unroll
        for (int k = 0; k < IN1; ++k) {
          W[u][k] = mv ? S0[m * IN1 + k] : 0.f;
          G[u][k] = 0.f;
        }
        w1r[u] = mv ? S1[m] : 0.f;
        w1s[u] = w1r[u] * inv_s0;
        g1r[u] = 0.f;
      }
      if (lane == 0) w1b = S1[H];
      __syncwarp();                        // the staging buffer receives the gradient later
    }
    const float bias_l = w1b;              // bias unit of h1 (lane 0 only)
    auto load_row = [&](int b, float* xv) {
      const float4* xr = reinterpret_cast<const float4*>(xs + b * XP);
#pragma unroll
      for (int j = 0; j < X4; ++j) {
        const float4 t = xr[j];
        xv[4 * j] = t.x; xv[4 * j + 1] = t.y; xv[4 * j + 2] = t.z; xv[4 * j + 3] = t.w;
      }
    };
    auto forward1 = [&](int b, float& s0, float& s1, float& pt) {
      float xv[XP];
      load_row(b, xv);
      float sacc0 = 0.f, sacc1 = 0.f;
#pragma unroll
      for (int k = 0; k < IN1; ++k) {
        sacc0 = fmaf(W[0][k], xv[k], sacc0);
        sacc1 = fmaf(W[1][k], xv[k], sacc1);
      }
      s0 = sacc0; s1 = sacc1;
      pt = fmaf(w1s[1], fmaxf(sacc1, 0.f), fmaf(w1s[0], fmaxf(sacc0, 0.f), bias_l));
    };
    for (int t = 0; t < ntiles; ++t) {
      if (ntiles > 1) {
        __syncthreads();                   // every warp is done with the previous tile
        stage(t);
        __syncthreads();
      }
      if (!act) continue;
      const int r0 = t * TR, nr = min(TR, a.B - r0);
      const int Bp = (nr + PB - 1) / PB * PB;      // padded with zero-weight rows
      float sa[2][PB], part[PB];
#pragma unroll
      for (int p = 0; p < PB; ++p) forward1(p, sa[0][p], sa[1][p], part[p]);
      for (int b0 = 0; b0 < Bp; b0 += PB) {
        float sn[2][PB], pn[PB];
#define ZSB_BFLY(o)                                                                   \
  _Pragma("unroll") for (int p = 0; p < PB; ++p)                                      \
      part[p] += __shfl_xor_sync(0xffffffffu, part[p], o);
        ZSB_BFLY(16)
        forward1(b0 + PB + 0, sn[0][0], sn[1][0], pn[0]);
        ZSB_BFLY(8)
        forward1(b0 + PB + 1, sn[0][1], sn[1][1], pn[1]);
        ZSB_BFLY(4)
        forward1(b0 + PB + 2, sn[0][2], sn[1][2], pn[2]);
        ZSB_BFLY(2)
        forward1(b0 + PB + 3, sn[0][3], sn[1][3], pn[3]);
        ZSB_BFLY(1)
#undef ZSB_BFLY
#pragma unroll
        for (int p = 0; p < PB; ++p) {
          const int b = b0 + p;
          const float2 yw = yc[b];
          const float r = fmaf(-inv_s1, part[p], yw.x);           // y - y_mean
          if constexpr (GRAD) {
            float xv[XP];
            load_row(b, xv);
            const float dout = r * yw.y;                          // 0 for padding rows
#pragma unroll
            for (int u = 0; u < 2; ++u) {
              g1r[u] = fmaf(dout, fmaxf(sa[u][p], 0.f), g1r[u]);
              const float da = (sa[u][p] > 0.f) ? dout * w1s[u] : 0.f;
#pragma unroll
              for (int k = 0; k < IN1; ++k) G[u][k] = fmaf(da, xv[k], G[u][k]);
            }
            g1b += dout;                   // every lane accumulates; only lane 0's copy is used
          }
          if (lane == (b & 31) && b < nr) {   // this lane owns row b's likelihood term
            rsq = fmaf(r, r, rsq);
            const int64_t o = c * a.B + r0 + b;
            if (a.ym) a.ym[o] = part[p] * inv_s1;
            if (a.ll) a.ll[o] = fmaf(cst[2], r * r, cst[1]);
          }
        }
#pragma unroll
        for (int p = 0; p < PB; ++p) {
          part[p] = pn[p];
          sa[0][p] = sn[0][p]; sa[1][p] = sn[1][p];
        }
      }
    }
    if (!act) continue;
    // ---- value: prior quadratic form + likelihood, each reduced once over the warp
    float quad = 0.f;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int m = lane + 32 * u;
      if (m < H) {
#pragma unroll
        for (int k = 0; k < IN1; ++k) quad = fmaf(pr0[m * IN1 + k] * W[u][k], W[u][k], quad);
        quad = fmaf(pr1[m] * w1r[u], w1r[u], quad);
      }
    }
    if (lane == 0) quad = fmaf(pr1[H] * w1b, w1b, quad);
    quad = warp_sum(quad);
    const float rsum = warp_sum(rsq);
    if (lane == 0) {
      const float sq = -2.f * cst[2] * lik_scale * rsum;   // n_train * mean_b prec r_b^2
      if (a.lp) a.lp[c] = (cst[0] - 0.5f * quad) + (a.n_train * cst[1] - 0.5f * sq);
      if (a.gys) a.gys[c] = sq - a.n_train;
    }
    if constexpr (GRAD) {
      // ---- gradient: likelihood part minus the prior's precision * w, out through the staging
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int m = lane + 32 * u;
        if (m < H) {
#pragma unroll
          for (int k = 0; k < IN1; ++k) {
            const int idx = m * IN1 + k;
            S0[idx] = G[u][k] - pr0[idx] * W[u][k];
          }
          S1[m] = g1r[u] * inv_s0 - pr1[m] * w1r[u];
        }
      }
      if (lane == 0) S1[H] = g1b - pr1[H] * w1b;
      __syncwarp();
      if (a.g0) for (int i = lane; i < n0; i += 32) a.g0[c * n0 + i] = S0[i];
      if (a.g1) for (int i = lane; i < H1; i += 32) a.g1[c * H1 + i] = S1[i];
      __syncwarp();                        // the buffer is restaged for the next particle
    }
  }
}

// dynamic shared memory of one block: staged rows, {y, coefficient}, prior precisions, per-warp
// staging (at the maximum shape ~76 KB: two blocks, 16 particles in flight, per SM)
size_t lj_smem(int in1, int H, int tile_rows) {
  const int XP = (in1 + 3) / 4 * 4;
  const int n0p = (H * in1 + 3) & ~3, n1p = (H + 1 + 3) & ~3;
  return (size_t)((tile_rows + PB) * XP + 2 * tile_rows + (1 + NW) * (n0p + n1p)) * sizeof(float);
}

// Opt an instantiation in to the largest dynamic shared memory any shape asks of it, once per
// device.  Without the opt-in the limit is 48 KB MINUS the kernel's static shared memory, so
// comparing a launch's dynamic size with 48 KB alone is not enough.
template <int IN1, bool GRAD>
int lj_opt_in() {
  static std::atomic<uint64_t> done{0};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  const uint64_t bit = dev < 64 ? (1ull << dev) : 0;
  if (e == cudaSuccess && (done.load(std::memory_order_acquire) & bit)) return ZSB_OK;
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(bnn_logjoint_kernel<IN1, GRAD>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)lj_smem(IN1, MAX_H, TILE));
  if (e != cudaSuccess) {
    zsb_set_error("zsb_bnn_logjoint_f32: shared-memory opt-in failed: %s", cudaGetErrorString(e));
    return ZSB_ERR_CUDA;
  }
  done.fetch_or(bit, std::memory_order_release);
  return ZSB_OK;
}

template <bool GRAD>
int lj_launch(const LjArgs& a, void* stream) {
  const size_t smem = lj_smem(a.n_in + 1, a.H, a.tile_rows);
  int64_t blocks = zsb_ceil_div(a.K, NW);
  if (blocks > 2 * ZSB_NUM_SMS) blocks = 2 * ZSB_NUM_SMS;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ZSB_OK;
  switch (a.n_in + 1) {
#define ZSB_LJ_CASE(N)                                                                       \
  case N:                                                                                    \
    rc = lj_opt_in<N, GRAD>();                                                               \
    if (rc) return rc;                                                                       \
    bnn_logjoint_kernel<N, GRAD><<<(unsigned)blocks, 32 * NW, smem, st>>>(a);                \
    break;
    ZSB_LJ_CASE(2) ZSB_LJ_CASE(3) ZSB_LJ_CASE(4) ZSB_LJ_CASE(5) ZSB_LJ_CASE(6)
    ZSB_LJ_CASE(7) ZSB_LJ_CASE(8) ZSB_LJ_CASE(9) ZSB_LJ_CASE(10) ZSB_LJ_CASE(11)
    ZSB_LJ_CASE(12) ZSB_LJ_CASE(13) ZSB_LJ_CASE(14) ZSB_LJ_CASE(15) ZSB_LJ_CASE(16)
#undef ZSB_LJ_CASE
  }
  return zsb_check_launch("bnn_logjoint");
}

}  // namespace

extern "C" {

int zsb_bnn_logjoint_f32(const float* w0, const float* w1, const float* x, const float* y,
                         int64_t B, int n_in, int H, const float* logstd0, int64_t logstd0_n,
                         const float* logstd1, int64_t logstd1_n, const float* y_logstd,
                         float n_train, float* lp, float* g0, float* g1, float* g_ylogstd,
                         float* y_mean, float* log_lik, int64_t K, void* stream) {
  ZSB_REQUIRE(w0 && w1 && x && y && logstd0 && logstd1 && y_logstd,
              "zsb_bnn_logjoint_f32: null arg");
  ZSB_REQUIRE(K > 0 && B > 0 && B < (1LL << 31) && n_in > 0 && n_in + 1 <= MAX_IN1 && H > 0 &&
                  H <= MAX_H,
              "zsb_bnn_logjoint_f32: need K > 0, B > 0, 0 < n_in <= 15, 0 < H <= 64 "
              "(got K = %lld, B = %lld, n_in = %d, H = %d)",
              (long long)K, (long long)B, n_in, H);
  ZSB_REQUIRE(logstd0_n > 0 && logstd0_n <= (int64_t)H * (n_in + 1) && logstd1_n > 0 &&
                  logstd1_n <= H + 1,
              "zsb_bnn_logjoint_f32: logstd0_n / logstd1_n must be in [1, weights per particle]");
  LjArgs a;
  a.w0 = w0; a.w1 = w1; a.x = x; a.y = y;
  a.logstd0 = logstd0; a.logstd1 = logstd1; a.y_logstd = y_logstd;
  a.lp = lp; a.g0 = g0; a.g1 = g1; a.gys = g_ylogstd; a.ym = y_mean; a.ll = log_lik;
  a.K = K; a.B = (int)B; a.n_in = n_in; a.H = H;
  a.ls0_n = (int)logstd0_n; a.ls1_n = (int)logstd1_n;
  a.tile_rows = B > TILE ? TILE : (int)((B + PB - 1) / PB * PB);
  a.n_train = n_train;
  if (g0 || g1) return lj_launch<true>(a, stream);
  return lj_launch<false>(a, stream);
}

}  // extern "C"
