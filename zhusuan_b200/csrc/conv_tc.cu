// k x k convolutions over NHWC on the tensor-core dense products (gemm_logjoint_tc.cu): the two
// memory passes around the products of the batch-normalised convolutions of the GAN examples
// (examples/generative_adversarial_nets/dcgan.py, wasserstein_gan.py) and of the biased
// convolutions act(conv(x) + b + residual) (examples/utils/utils.py:74-113, with the residual added
// before the activation as in the resnet blocks of examples/variational_autoencoders/vae_conv.py).
//
// Geometry, on the convolution's side as in conv.cu: the "big" grid Hb x Wb is the input of the
// convolution (the output of the transposed one), the "small" grid Hs x Ws its output, and
//   big pixel (y, x) = (s i + kh - pt, s j + kw - pl)   for small pixel (i, j) and tap (kh, kw)
// with out-of-range big pixels counting as zero.  TF's SAME and VALID rules are expressed by the
// caller's choice of Hs, Ws, pt and pl.
//
//   gather-split: x [N, Hb, Wb, C] -> the fp16 hi/lo operand planes [2][N Hs Ws][kpad(k k C)] of
//                 the im2col matrix (column (kh k + kw) C + c), whose fp32 form is never written
//   col2im-sum:   cols [N Hs Ws, k k C] fp32 -> y [N, Hb, Wb, C], the sum over the (small pixel,
//                 tap) entries that land on each big pixel, gathered in a fixed tap order (kh, then
//                 kw, ascending): no atomics, deterministic.  Epilogues: none, act(sum + bias +
//                 residual), batch norm training (pre-activation + per-128-row moment partials for
//                 the merge of zsb_bn_finish_fused_f32) and batch norm evaluation.
//   act-grad:     gp = d/d(pre-activation) through the activation's output y, and the column sums
//                 of gp (the bias gradient), merged in a fixed order.
// Activation codes (act): 0 none, 1 ReLU, 2 sigmoid.
#include "tc_common.cuh"

namespace {

constexpr int TILE = 128;        // rows per moment / column-sum partial (the products' row tile)

struct Geo {
  int64_t N, Hb, Wb, Hs, Ws;
  int C, k, s, pt, pl;
};

inline unsigned blocks_for(int64_t n, int64_t per, int per_sm) {
  int64_t b = zsb_ceil_div(n, per);
  if (b > ZSB_NUM_SMS * per_sm) b = ZSB_NUM_SMS * per_sm;
  return (unsigned)(b < 1 ? 1 : b);
}

// y[n, y, x, c] = sum over the taps (kh, kw) with s i + kh - pt = y, s j + kw - pl = x of
// cols[(n Hs + i) Ws + j, (kh k + kw) C + c], kh then kw ascending
__device__ __forceinline__ float col2im_at(const float* __restrict__ cols, const Geo& g,
                                           int64_t r, int c) {
  const int64_t xo = r % g.Wb, t = r / g.Wb;
  const int64_t yo = t % g.Hb, n = t / g.Hb;
  const int64_t KK = (int64_t)g.k * g.k * g.C;
  const int64_t ny0 = yo + g.pt, nx0 = xo + g.pl;
  float acc = 0.f;
  for (int kh = (int)(ny0 % g.s); kh < g.k; kh += g.s) {
    const int64_t ny = ny0 - kh;
    if (ny < 0) break;
    const int64_t i = ny / g.s;
    if (i >= g.Hs) continue;
    for (int kw = (int)(nx0 % g.s); kw < g.k; kw += g.s) {
      const int64_t nx = nx0 - kw;
      if (nx < 0) break;
      const int64_t j = nx / g.s;
      if (j >= g.Ws) continue;
      acc += cols[((n * g.Hs + i) * g.Ws + j) * KK + (int64_t)(kh * g.k + kw) * g.C + c];
    }
  }
  return acc;
}

// scale[2] = running max |x| bits (NaN and inf skipped)
__global__ void __launch_bounds__(256) conv_absmax_kernel(const float* __restrict__ x, int64_t n,
                                                          float* __restrict__ scale) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    m = finite_absmax(m, x[i]);
  fold_amax(scale, m, threadIdx.x & 31);
}

// scale[0] = the plane scale of the max in scale[2], which is cleared for the next split
__global__ void conv_plane_scale_kernel(float* __restrict__ scale) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  scale[0] = pow2_plane_scale(__uint_as_float(reinterpret_cast<unsigned int*>(scale)[2]));
  reinterpret_cast<unsigned int*>(scale)[2] = 0u;
}

// One warp per im2col row (small pixel), its lanes along the columns: consecutive columns are
// consecutive channels of one tap, so the loads of x and the plane stores are coalesced.
__global__ void __launch_bounds__(256) gather_split_kernel(const float* __restrict__ x, Geo g,
                                                           int K, int Kp,
                                                           __half* __restrict__ planes,
                                                           const float* __restrict__ scale) {
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float sc = scale[0];
  const int64_t R = g.N * g.Hs * g.Ws;
  const int64_t n_pl = R * (int64_t)Kp;
  for (int64_t r = (int64_t)blockIdx.x * 8 + ty; r < R; r += (int64_t)gridDim.x * 8) {
    const int64_t j = r % g.Ws, t = r / g.Ws;
    const int64_t i = t % g.Hs, n = t / g.Hs;
    const int64_t y0 = i * g.s - g.pt, x0 = j * g.s - g.pl;
    const float* __restrict__ xn = x + n * g.Hb * g.Wb * g.C;
    for (int col = tx; col < Kp; col += 32) {
      float v = 0.f;
      if (col < K) {
        const int tap = col / g.C, c = col - tap * g.C;
        const int kh = tap / g.k, kw = tap - kh * g.k;
        const int64_t yy = y0 + kh, xx = x0 + kw;
        if (yy >= 0 && yy < g.Hb && xx >= 0 && xx < g.Wb) v = xn[(yy * g.Wb + xx) * g.C + c];
      }
      store_hilo(planes + r * Kp + col, n_pl, v * sc);
    }
  }
}

// Flat epilogues over the N Hb Wb x C outputs:
//   EPI 0  out = the sum                                    (the input gradient of a convolution)
//   EPI 1  out = act(sum + bias[c] + res), bias and res may be NULL    (biased transposed layers)
//   EPI 3  out = act(fmaf((sum - mean) rstd, gamma, beta)), act none or ReLU, mean / rstd of the
//          moving statistics (batch norm evaluation, EPI 11's rounding); pre (may be NULL) = sum;
//          stats = (mean, rstd)
// max |out| into amax_scale[2] (may be NULL).
template <int EPI>
__global__ void __launch_bounds__(256) col2im_flat_kernel(
    const float* __restrict__ cols, Geo g, const float* __restrict__ bias,
    const float* __restrict__ gamma, const float* __restrict__ beta,
    const float* __restrict__ mmean, const float* __restrict__ mvar, float eps, int act,
    float* __restrict__ stats, float* __restrict__ pre, float* __restrict__ out,
    float* __restrict__ amax_scale, const float* __restrict__ res) {
  const int64_t n = g.N * g.Hb * g.Wb * g.C;
  const int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (EPI == 3 && i0 < g.C) {
    stats[i0] = mmean[i0];
    stats[g.C + i0] = rsqrtf(mvar[i0] + eps);
  }
  float m = 0.f;
  for (int64_t e = i0; e < n; e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = e / g.C;
    const int c = (int)(e - r * g.C);
    const float l = col2im_at(cols, g, r, c);
    float y = l;
    if (EPI == 1) {
      if (bias) y += bias[c];
      if (res) y += res[e];
      if (act == 1) y = fmaxf(y, 0.f);
      else if (act == 2) y = sigmoidf_(y);
    } else if (EPI == 3) {
      y = fmaf((l - mmean[c]) * rsqrtf(mvar[c] + eps), gamma[c], beta[c]);
      if (act) y = fmaxf(y, 0.f);
      if (pre) pre[e] = l;
    }
    out[e] = y;
    m = finite_absmax(m, y);
  }
  if (amax_scale) fold_amax(amax_scale, m, threadIdx.x & 31);
}

// EPI 2 (batch norm training), per 128-row tile t of the N Hb Wb rows and 32 channels (8 warps of
// 16 rows each): pre = the sum, and the tile's moment partials of channel c, part[2 t C + c] = mean
// and part[(2 t + 1) C + c] = M2 about it -- the layout zsb_bn_finish_fused_f32 merges.
__global__ void __launch_bounds__(256) col2im_bn_train_kernel(const float* __restrict__ cols,
                                                              Geo g, float* pre,
                                                              float* __restrict__ part) {
  __shared__ float sh[8][32];
  __shared__ float tile_mean[32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int64_t R = g.N * g.Hb * g.Wb;
  const int64_t t = blockIdx.x;
  const int c = blockIdx.y * 32 + tx;
  const bool c_ok = c < g.C;
  float sum = 0.f;
#pragma unroll 1
  for (int i = 0; i < TILE / 8; ++i) {
    const int64_t r = t * TILE + ty + 8 * i;
    if (c_ok && r < R) {
      const float v = col2im_at(cols, g, r, c);
      pre[r * g.C + c] = v;
      sum += v;
    }
  }
  const int cnt = (int)min((int64_t)TILE, R - t * TILE);
  sh[ty][tx] = sum;
  __syncthreads();
  if (ty == 0) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += sh[i][tx];
    tile_mean[tx] = s / (float)cnt;
  }
  __syncthreads();
  const float mean = tile_mean[tx];
  float m2 = 0.f;               // about the tile mean, from this thread's own stores of pre
#pragma unroll 4
  for (int i = 0; i < TILE / 8; ++i) {
    const int64_t r = t * TILE + ty + 8 * i;
    if (c_ok && r < R) {
      const float d = pre[r * g.C + c] - mean;
      m2 = fmaf(d, d, m2);
    }
  }
  __syncthreads();
  sh[ty][tx] = m2;
  __syncthreads();
  if (ty == 0 && c_ok) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += sh[i][tx];
    part[2 * t * g.C + c] = mean;
    part[(2 * t + 1) * g.C + c] = s;
  }
}

// gp = the gradient through act's output y: g y (1 - y) (sigmoid), g (y > 0) (ReLU) or g (none, y
// not read); max |gp| into scale[2], and per 128-row tile t the column sums part[t C + c] (8 warps
// of 16 rows, met in a fixed order)
__global__ void __launch_bounds__(256) act_grad_kernel(const float* __restrict__ g,
                                                       const float* __restrict__ y, int act,
                                                       int64_t R, int C, float* __restrict__ gp,
                                                       float* __restrict__ part,
                                                       float* __restrict__ scale) {
  __shared__ float sh[8][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int64_t t = blockIdx.x;
  const int c = blockIdx.y * 32 + tx;
  float s1 = 0.f, m = 0.f;
  if (c < C) {
#pragma unroll 4
    for (int i = 0; i < TILE / 8; ++i) {
      const int64_t r = t * TILE + ty + 8 * i;
      if (r >= R) break;
      const float gv = g[r * C + c];
      float d = gv;
      if (act == 2) {
        const float yv = y[r * C + c];
        d = gv * (yv * (1.f - yv));
      } else if (act == 1) {
        d = y[r * C + c] > 0.f ? gv : 0.f;
      }
      gp[r * C + c] = d;
      s1 += d;
      m = finite_absmax(m, d);
    }
  }
  fold_amax(scale, m, tx);
  sh[ty][tx] = s1;
  __syncthreads();
  if (ty == 0 && c < C) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += sh[i][tx];
    part[t * C + c] = s;
  }
}

// One warp per channel: db[c] = the tile sums of act_grad_kernel in a fixed order (lane-strided
// runs, then a fixed shuffle tree)
__global__ void __launch_bounds__(256) col_sum_merge_kernel(const float* __restrict__ part,
                                                            int64_t n_t, int C,
                                                            float* __restrict__ db) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (c >= C) return;
  float s = 0.f;
  for (int64_t t = lane; t < n_t; t += 32) s += part[t * C + c];
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) s += __shfl_down_sync(0xffffffffu, s, off);
  if (lane == 0) db[c] = s;
}

int check_geo(const Geo& g, const char* what) {
  ZSB_REQUIRE(g.N > 0 && g.Hb > 0 && g.Wb > 0 && g.Hs > 0 && g.Ws > 0 && g.C > 0 && g.k >= 1 &&
                  g.k <= 7 && (g.s == 1 || g.s == 2) && g.pt >= 0 && g.pl >= 0 && g.pt < g.k &&
                  g.pl < g.k,
              "%s: bad geometry", what);
  ZSB_REQUIRE(g.N * g.Hb * g.Wb * g.C < (1LL << 31) &&
                  g.N * g.Hs * g.Ws * (int64_t)g.k * g.k * g.C < (1LL << 31),
              "%s: tensors too large", what);
  return ZSB_OK;
}

}  // namespace

extern "C" {

int zsb_conv_gather_split_f32(const float* x, int64_t N, int64_t Hb, int64_t Wb, int64_t C,
                              int64_t Hs, int64_t Ws, int k, int stride, int pt, int pl,
                              void* planes, float* scale, int have_amax, void* stream) {
  ZSB_REQUIRE(x && planes && scale, "zsb_conv_gather_split_f32: bad args");
  const Geo g{N, Hb, Wb, Hs, Ws, (int)C, k, stride, pt, pl};
  ZSB_REQUIRE(C > 0 && C < (1 << 20), "zsb_conv_gather_split_f32: bad channel count");
  int rc = check_geo(g, "zsb_conv_gather_split_f32");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int K = k * k * (int)C, Kp = ((K + 63) / 64) * 64;
  if (!have_amax) {
    const int64_t n = N * Hb * Wb * C;
    conv_absmax_kernel<<<blocks_for(n, 256 * 8, 16), 256, 0, st>>>(x, n, scale);
  }
  conv_plane_scale_kernel<<<1, 32, 0, st>>>(scale);
  gather_split_kernel<<<blocks_for(N * Hs * Ws, 8, 16), 256, 0, st>>>(
      x, g, K, Kp, reinterpret_cast<__half*>(planes), scale);
  return zsb_check_launch("conv_gather_split");
}

int zsb_conv_col2im_f32(int epi, const float* cols, int64_t N, int64_t Hb, int64_t Wb, int64_t C,
                        int64_t Hs, int64_t Ws, int k, int stride, int pt, int pl,
                        const float* bias, const float* residual, const float* gamma,
                        const float* beta, const float* moving_mean, const float* moving_var,
                        float eps, int act, float* stats, float* pre, float* part, float* out,
                        float* amax_scale, void* stream) {
  ZSB_REQUIRE(cols && epi >= 0 && epi <= 3 && act >= 0 && act <= 2,
              "zsb_conv_col2im_f32: bad args");
  ZSB_REQUIRE(act == 0 || epi == 1 || (epi == 3 && act == 1),
              "zsb_conv_col2im_f32: epi %d takes no act %d", epi, act);
  ZSB_REQUIRE(epi != 2 || (pre && part), "zsb_conv_col2im_f32: epi 2 needs pre and part");
  ZSB_REQUIRE(epi != 3 || (gamma && beta && moving_mean && moving_var && stats && out),
              "zsb_conv_col2im_f32: epi 3 needs gamma, beta, the moving statistics and stats");
  ZSB_REQUIRE(epi >= 2 || out, "zsb_conv_col2im_f32: out missing");
  ZSB_REQUIRE(C > 0 && C < (1 << 20), "zsb_conv_col2im_f32: bad channel count");
  const Geo g{N, Hb, Wb, Hs, Ws, (int)C, k, stride, pt, pl};
  int rc = check_geo(g, "zsb_conv_col2im_f32");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  if (epi == 2) {
    const int64_t n_t = zsb_ceil_div(N * Hb * Wb, TILE);
    col2im_bn_train_kernel<<<dim3((unsigned)n_t, (unsigned)((C + 31) / 32)), 256, 0, st>>>(
        cols, g, pre, part);
    return zsb_check_launch("conv_col2im_bn_train");
  }
  const int64_t n = N * Hb * Wb * C;
  int64_t blocks = blocks_for(n, 256, 16);
  if (epi == 3 && blocks * 256 < C) blocks = zsb_ceil_div(C, 256);     // every stats entry
  const unsigned nb = (unsigned)blocks;
  if (epi == 0)
    col2im_flat_kernel<0><<<nb, 256, 0, st>>>(cols, g, nullptr, nullptr, nullptr, nullptr,
                                              nullptr, 0.f, 0, nullptr, nullptr, out, amax_scale,
                                              nullptr);
  else if (epi == 1)
    col2im_flat_kernel<1><<<nb, 256, 0, st>>>(cols, g, bias, nullptr, nullptr, nullptr, nullptr,
                                              0.f, act, nullptr, nullptr, out, amax_scale,
                                              residual);
  else
    col2im_flat_kernel<3><<<nb, 256, 0, st>>>(cols, g, nullptr, gamma, beta, moving_mean,
                                              moving_var, eps, act, stats, pre, out, amax_scale,
                                              nullptr);
  return zsb_check_launch("conv_col2im");
}

int zsb_conv_act_grad_f32(const float* g, const float* y, int64_t R, int C, int act, float* gp,
                          float* part, float* db, float* scale, void* stream) {
  ZSB_REQUIRE(g && gp && part && scale && act >= 0 && act <= 2 && (y || act == 0) && R > 0 &&
                  C > 0 && C < (1 << 20) && R * C < (1LL << 31),
              "zsb_conv_act_grad_f32: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n_t = zsb_ceil_div(R, TILE);
  act_grad_kernel<<<dim3((unsigned)n_t, (unsigned)((C + 31) / 32)), 256, 0, st>>>(
      g, y, act, R, C, gp, part, scale);
  if (db) col_sum_merge_kernel<<<(unsigned)((C + 7) / 8), 256, 0, st>>>(part, n_t, C, db);
  return zsb_check_launch("conv_act_grad");
}

}  // extern "C"
