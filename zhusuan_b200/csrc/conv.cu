// 3x3 convolutions with TensorFlow "SAME" padding, NHWC, for the convolutional VAE
// (examples/variational_autoencoders/vae_conv.py:20-53, 80-87): tf.layers.conv2d(x, Cout, 3,
// strides=s, padding="same") and examples/utils/utils.py:74-113 (tf.nn.conv2d_transpose, SAME,
// plus bias_add), with their gradients.
//
// Geometry.  Every call is described on the convolution's side: the "big" grid [Hc, Wc] is the
// conv2d input, the "small" grid [Hs, Ws] its output, Hs = ceil(Hc / s).  The SAME pads are
//     pad_total = max((Hs - 1) s + 3 - Hc, 0),  pt = pad_total / 2  (likewise pl for columns)
// so stride 1 pads 1 and 1, and stride 2 pads 0 and 1 for an even Hc, 1 and 1 for an odd one.
//     conv:       y[n, i, j, co] = sum_{kh, kw, ci} x[n, s i + kh - pt, s j + kw - pl, ci] W[kh, kw, ci, co]
//     transpose:  its adjoint, big[n, h, w, co] = sum small[n, i, j, ci] W[kh, kw, co, ci] over
//                 h = s i + kh - pt, w = s j + kw - pl
// with out-of-range pixels counting as zero.  The input gradient of either is the other mode on
// the output gradient with the same W.
//
// Forward (conv3x3_fwd_kernel, one launch per layer).  A CTA of 256 threads stages a 32-channel
// slice of W in shared memory as [tap][ci][co] and takes a run of output pixels; lane l of a warp
// holds pixels l, l + 32, l + 64, l + 96 of the warp's run and 8 output channels, so the weights
// of a step are one broadcast shared load and the inputs one load per pixel.  For the stride-2
// transpose the output pixels are enumerated by row and column parity, so the pixels of a warp
// inside one parity class share their valid taps, and a tap no lane of the warp needs is skipped.
// The skip is per warp: warps that straddle a class or image boundary, or a border, still
// multiply zeros for some lanes.  The epilogue adds bias and residual and applies ReLU.  `gate` (the backward pass's saved ReLU output) masks the input
// where gate <= 0 as it is loaded, so the masked gradient is never written.  FP32 FFMA throughout.
//
// Weight gradient (conv3x3_wgrad_kernel + conv3x3_wgrad_merge_kernel).  With big and small as
// above (for conv2d big = x, small = g; for conv2d_transpose big = g, small = x)
//     dW[kh, kw, a, b] = sum_{n, i, j} big[n, s i + kh - pt, s j + kw - pl, a] small[n, i, j, b]
// which is conv2d's dW [3, 3, Cin, Cout] and conv2d_transpose's [3, 3, Cout, Cin] alike.  The
// grid has 10 slots of G CTAs: slots 0-8 are the taps, slot 9 sums the output gradient for db.
// CTA g of a slot takes pixel tiles g, g + G, ..., keeps its sums in registers and writes them to
// its own slice of `part` once; the merge sums the slices in CTA order.  No floating-point
// atomics: two identical calls give identical bits.
#include "common.cuh"

namespace {

constexpr int CV_THREADS = 256;
constexpr int CV_WARPS = CV_THREADS / 32;
constexpr int CV_PX = 4;                        // output pixels per thread
constexpr int CV_CO = 8;                        // output channels per thread
constexpr int CV_SLICE = 32;                    // output channels per CTA
constexpr int CV_MAX_C = 64;
constexpr int WG_TP = 64;                       // weight gradient: pixels per tile
constexpr int WG_SLOTS = 10;                    // 9 taps and the bias
constexpr int WG_TARGET_CTAS = 2 * ZSB_NUM_SMS;

struct CvGeom {
  int R, Hc, Wc, Hs, Ws, s, pt, pl;
};

__host__ __device__ inline int cv_pad_before(int big, int small, int s) {
  const int total = (small - 1) * s + 3 - big;
  return total > 0 ? total / 2 : 0;
}

// Output pixel p (flattened over the output tensor's [R, H, W]) -> (n, h, w).  The stride-2
// transpose enumerates each image's pixels by (row parity, column parity) class.
__device__ __forceinline__ void cv_decode(int p, const CvGeom& g, bool transpose, int& n, int& h,
                                          int& w) {
  const int Ho = transpose ? g.Hc : g.Hs, Wo = transpose ? g.Wc : g.Ws;
  const int hw = Ho * Wo;
  n = p / hw;
  int r = p - n * hw;
  if (transpose && g.s == 2) {
    const int h0 = (Ho + 1) >> 1, h1 = Ho >> 1, w0 = (Wo + 1) >> 1, w1 = Wo >> 1;
    int ph = 0, pw = 0, cw = w0;
    if (r < h0 * w0) {
    } else if ((r -= h0 * w0) < h0 * w1) {
      pw = 1; cw = w1;
    } else if ((r -= h0 * w1) < h1 * w0) {
      ph = 1;
    } else {
      r -= h1 * w0; ph = 1; pw = 1; cw = w1;
    }
    const int a = r / cw;
    h = 2 * a + ph;
    w = 2 * (r - a * cw) + pw;
  } else {
    h = r / Wo;
    w = r - h * Wo;
  }
}

// Source row (or column) of output coordinate o for tap k, or -1 when it is padding.
__device__ __forceinline__ int cv_src(int o, int k, int pad, int s, int n_in, bool transpose) {
  if (!transpose) {
    const int v = s * o + k - pad;
    return (v >= 0 && v < n_in) ? v : -1;
  }
  const int num = o + pad - k;
  if (num < 0) return -1;
  if (s == 2 && (num & 1)) return -1;
  const int v = s == 2 ? num >> 1 : num;
  return v < n_in ? v : -1;
}

// out = relu?(conv(x) + b + residual) for one 32-channel slice (blockIdx.y) of the output.
// `ngs` 8-channel groups per slice (1, 2 or 4); warp w takes group w % ngs.
template <bool GATE>
__global__ void __launch_bounds__(CV_THREADS) conv3x3_fwd_kernel(
    const float* __restrict__ x, const float* __restrict__ gate, const float* __restrict__ W,
    const float* __restrict__ b, const float* __restrict__ res, float* __restrict__ y, CvGeom g,
    int transpose, int Cin, int Cout, int relu, int ngs) {
  extern __shared__ float4 cv_smem[];
  float* __restrict__ ws = reinterpret_cast<float*>(cv_smem);
  const int cs = ngs * CV_CO;
  const int co0 = blockIdx.y * CV_SLICE;
  for (int t = threadIdx.x; t < 9 * Cin * cs; t += CV_THREADS) {
    const int row = t / cs, c = t - row * cs, co = co0 + c;        // row = tap * Cin + ci
    float v = 0.f;
    if (co < Cout) {
      if (!transpose) {
        v = __ldg(W + (int64_t)row * Cout + co);
      } else {
        const int tap = row / Cin, ci = row - tap * Cin;
        v = __ldg(W + ((int64_t)tap * Cout + co) * Cin + ci);
      }
    }
    ws[t] = v;
  }
  __syncthreads();

  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int cg = warp % ngs, pg = warp / ngs, pgs = CV_WARPS / ngs;
  const bool tr = transpose != 0;
  const int Hi = tr ? g.Hs : g.Hc, Wi = tr ? g.Ws : g.Wc;
  const int Ho = tr ? g.Hc : g.Hs, Wo = tr ? g.Wc : g.Ws;
  const int P = g.R * Ho * Wo;
  const int p0 = (blockIdx.x * pgs + pg) * 32 * CV_PX + lane;
  int pn[CV_PX], ph[CV_PX], pw[CV_PX];
#pragma unroll
  for (int k = 0; k < CV_PX; ++k) {
    const int p = p0 + 32 * k;
    if (p < P) {
      cv_decode(p, g, tr, pn[k], ph[k], pw[k]);
    } else {
      pn[k] = -1; ph[k] = pw[k] = 0;
    }
  }

  float acc[CV_PX][CV_CO];
#pragma unroll
  for (int k = 0; k < CV_PX; ++k)
#pragma unroll
    for (int c = 0; c < CV_CO; ++c) acc[k][c] = 0.f;

  const float* __restrict__ wg = ws + cg * CV_CO;
#pragma unroll 1
  for (int tap = 0; tap < 9; ++tap) {
    const int kh = tap / 3, kw = tap - 3 * kh;
    int off[CV_PX];
    bool any = false;
#pragma unroll
    for (int k = 0; k < CV_PX; ++k) {
      const int hi = pn[k] < 0 ? -1 : cv_src(ph[k], kh, g.pt, g.s, Hi, tr);
      const int wi = hi < 0 ? -1 : cv_src(pw[k], kw, g.pl, g.s, Wi, tr);
      off[k] = wi < 0 ? -1 : ((pn[k] * Hi + hi) * Wi + wi) * Cin;
      any |= wi >= 0;
    }
    if (!__any_sync(0xffffffffu, any)) continue;
    const float* __restrict__ wt = wg + tap * Cin * cs;
#pragma unroll 2
    for (int ci = 0; ci < Cin; ++ci) {
      float xv[CV_PX];
#pragma unroll
      for (int k = 0; k < CV_PX; ++k) {
        float v = 0.f;
        if (off[k] >= 0) {
          v = __ldg(x + off[k] + ci);
          if (GATE && !(__ldg(gate + off[k] + ci) > 0.f)) v = 0.f;
        }
        xv[k] = v;
      }
      const float4 w0 = *reinterpret_cast<const float4*>(wt + ci * cs);
      const float4 w1 = *reinterpret_cast<const float4*>(wt + ci * cs + 4);
      const float wv[CV_CO] = {w0.x, w0.y, w0.z, w0.w, w1.x, w1.y, w1.z, w1.w};
#pragma unroll
      for (int k = 0; k < CV_PX; ++k)
#pragma unroll
        for (int c = 0; c < CV_CO; ++c) acc[k][c] = fmaf(xv[k], wv[c], acc[k][c]);
    }
  }

  const int cb = co0 + cg * CV_CO;
  float bias[CV_CO];
#pragma unroll
  for (int c = 0; c < CV_CO; ++c)
    bias[c] = (b != nullptr && cb + c < Cout) ? __ldg(b + cb + c) : 0.f;
#pragma unroll
  for (int k = 0; k < CV_PX; ++k) {
    if (pn[k] < 0) continue;
    const int64_t o = ((int64_t)(pn[k] * Ho + ph[k]) * Wo + pw[k]) * Cout;
#pragma unroll
    for (int c = 0; c < CV_CO; ++c) {
      const int co = cb + c;
      if (co < Cout) {
        float v = acc[k][c] + bias[c];
        if (res != nullptr) v += __ldg(res + o + co);
        if (relu) v = fmaxf(v, 0.f);
        y[o + co] = v;
      }
    }
  }
}

// Slots 0-8: tap (kh, kw) = (slot / 3, slot % 3); each thread holds a 4 x 4 block of
// [Ca, Cb] for the pixels of its pixel group.  Slot 9: per-channel sums of the output gradient
// (small when grad_big = 0, big otherwise).  The grid covers slots slot0 .. 9 (slot0 = 9 when
// only db is wanted); slice slot * G + g of `part` has Ca * Cb floats.
template <bool GATE>
__global__ void __launch_bounds__(CV_THREADS) conv3x3_wgrad_kernel(
    const float* __restrict__ big, const float* __restrict__ small, const float* __restrict__ gate,
    int grad_big, float* __restrict__ part, CvGeom g, int Ca, int Cb, int G, int slot0) {
  __shared__ __align__(16) float bt[WG_TP * CV_MAX_C];
  __shared__ __align__(16) float st[WG_TP * CV_MAX_C];
  __shared__ float red[CV_THREADS * 16];
  const int gi = blockIdx.x % G, slot = slot0 + blockIdx.x / G;
  const int T = Ca * Cb;
  float* __restrict__ out = part + (int64_t)(blockIdx.x + slot0 * G) * T;
  const int tid = threadIdx.x;

  if (slot == 9) {
    const int C = grad_big ? Ca : Cb;
    const float* __restrict__ src = grad_big ? big : small;
    const int P = grad_big ? g.R * g.Hc * g.Wc : g.R * g.Hs * g.Ws;
    const int tiles = (P + WG_TP - 1) / WG_TP;
    const int c = tid & (CV_MAX_C - 1), rg = tid / CV_MAX_C;
    float acc = 0.f;
    if (c < C) {
      for (int t = gi; t < tiles; t += G) {
        for (int r = rg; r < WG_TP; r += CV_THREADS / CV_MAX_C) {
          const int p = t * WG_TP + r;
          if (p < P) {
            const int64_t o = (int64_t)p * C + c;
            float v = __ldg(src + o);
            if (GATE && !(__ldg(gate + o) > 0.f)) v = 0.f;
            acc += v;
          }
        }
      }
    }
    red[tid] = acc;
    __syncthreads();
    if (tid < C) {
      float v = 0.f;
#pragma unroll
      for (int q = 0; q < CV_THREADS / CV_MAX_C; ++q) v += red[q * CV_MAX_C + tid];
      out[tid] = v;
    }
    return;
  }

  const int kh = slot / 3, kw = slot - 3 * kh;
  const int as = (Ca + 3) & ~3, bs = (Cb + 3) & ~3;
  const int nA = as >> 2, nB = bs >> 2, nT = nA * nB;
  const int ngp = CV_THREADS / nT;                 // pixel groups, >= 1
  const int grp = tid / nT, loc = tid - grp * nT;
  const int ta = loc / nB, tb = loc - ta * nB;
  const bool active = grp < ngp;
  for (int t = tid; t < WG_TP * CV_MAX_C; t += CV_THREADS) bt[t] = st[t] = 0.f;

  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

  const int P = g.R * g.Hs * g.Ws, hw = g.Hs * g.Ws;
  const int tiles = (P + WG_TP - 1) / WG_TP;
  for (int t = gi; t < tiles; t += G) {
    __syncthreads();                               // the previous tile's reads are done
    for (int e = tid; e < WG_TP * Ca; e += CV_THREADS) {
      const int r = e / Ca, a = e - r * Ca, p = t * WG_TP + r;
      float v = 0.f;
      if (p < P) {
        const int n = p / hw, q = p - n * hw, i = q / g.Ws, j = q - i * g.Ws;
        const int hi = g.s * i + kh - g.pt, wi = g.s * j + kw - g.pl;
        if (hi >= 0 && hi < g.Hc && wi >= 0 && wi < g.Wc) {
          const int64_t o = ((int64_t)(n * g.Hc + hi) * g.Wc + wi) * Ca + a;
          v = __ldg(big + o);
          if (GATE && grad_big && !(__ldg(gate + o) > 0.f)) v = 0.f;
        }
      }
      bt[r * as + a] = v;
    }
    for (int e = tid; e < WG_TP * Cb; e += CV_THREADS) {
      const int r = e / Cb, bb = e - r * Cb, p = t * WG_TP + r;
      float v = 0.f;
      if (p < P) {
        const int64_t o = (int64_t)p * Cb + bb;
        v = __ldg(small + o);
        if (GATE && !grad_big && !(__ldg(gate + o) > 0.f)) v = 0.f;
      }
      st[r * bs + bb] = v;
    }
    __syncthreads();
    if (active) {
#pragma unroll 4
      for (int r = grp; r < WG_TP; r += ngp) {
        const float4 av = *reinterpret_cast<const float4*>(bt + r * as + 4 * ta);
        const float4 bv = *reinterpret_cast<const float4*>(st + r * bs + 4 * tb);
        const float a4[4] = {av.x, av.y, av.z, av.w}, b4[4] = {bv.x, bv.y, bv.z, bv.w};
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a4[i], b4[j], acc[i][j]);
      }
    }
  }

  // Sum the pixel groups in order and write the slice.
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) red[tid * 16 + i * 4 + j] = acc[i][j];
  __syncthreads();
  for (int e = tid; e < T; e += CV_THREADS) {
    const int a = e / Cb, bb = e - a * Cb;
    const int l = (a >> 2) * nB + (bb >> 2), k = (a & 3) * 4 + (bb & 3);
    float v = 0.f;
    for (int q = 0; q < ngp; ++q) v += red[(q * nT + l) * 16 + k];
    out[e] = v;
  }
}

// dW[e] = sum_g part[(tap G + g) T + e'] and db[c] = sum_g part[(9 G + g) T + c], g ascending.
// Either output may be NULL.
__global__ void __launch_bounds__(CV_THREADS) conv3x3_wgrad_merge_kernel(
    const float* __restrict__ part, int G, int T, int C, float* __restrict__ dW,
    float* __restrict__ db) {
  const int e0 = dW != nullptr ? 0 : 9 * T, n = 9 * T + (db != nullptr ? C : 0);
  for (int e = e0 + blockIdx.x * CV_THREADS + threadIdx.x; e < n;
       e += gridDim.x * CV_THREADS) {
    const int slot = e < 9 * T ? e / T : 9;
    const int k = e < 9 * T ? e - slot * T : e - 9 * T;
    const float* __restrict__ p = part + (int64_t)slot * G * T + k;
    float v = 0.f;
    for (int q = 0; q < G; ++q) v += p[(int64_t)q * T];
    if (e < 9 * T) dW[e] = v; else db[k] = v;
  }
}

int cv_ngs(int64_t Cout) {
  const int64_t groups = zsb_ceil_div(Cout < CV_SLICE ? Cout : CV_SLICE, CV_CO);
  return groups <= 1 ? 1 : (groups <= 2 ? 2 : 4);
}

int64_t cv_wgrad_ctas(int64_t R, int64_t Hc, int64_t Wc, int64_t Hs, int64_t Ws) {
  const int64_t Pb = R * Hc * Wc, Ps = R * Hs * Ws;
  const int64_t tiles = zsb_ceil_div(Pb > Ps ? Pb : Ps, WG_TP);
  const int64_t g = zsb_ceil_div(WG_TARGET_CTAS, WG_SLOTS);
  return tiles < g ? tiles : g;
}

// Sizes shared by the entry points: stride, grids and channel ranges.
bool cv_sizes_ok(int64_t R, int64_t Hc, int64_t Wc, int64_t Hs, int64_t Ws, int64_t Ca,
                 int64_t Cb, int s) {
  if (R < 0 || Hc < 1 || Wc < 1 || (s != 1 && s != 2)) return false;
  if (Hs != zsb_ceil_div(Hc, s) || Ws != zsb_ceil_div(Wc, s)) return false;
  return Ca >= 1 && Ca <= CV_MAX_C && Cb >= 1 && Cb <= CV_MAX_C;
}

}  // namespace

extern "C" {

// One 3x3 SAME convolution or transposed convolution with fused epilogue.  See include/zsb200.h.
int zsb_conv3x3_fwd_f32(const float* x, const float* gate, const float* W, const float* b,
                        const float* residual, float* y, int64_t R, int64_t Hc, int64_t Wc,
                        int64_t Cin, int64_t Cout, int stride, int transpose, int relu,
                        void* stream) {
  const int64_t Hs = zsb_ceil_div(Hc, stride > 0 ? stride : 1);
  const int64_t Ws = zsb_ceil_div(Wc, stride > 0 ? stride : 1);
  const int64_t Cbig = transpose ? Cout : Cin, Csmall = transpose ? Cin : Cout;
  ZSB_REQUIRE(cv_sizes_ok(R, Hc, Wc, Hs, Ws, Cbig, Csmall, stride),
              "zsb_conv3x3_fwd_f32: unsupported sizes (R %lld, H %lld, W %lld, Cin %lld, "
              "Cout %lld, stride %d)", (long long)R, (long long)Hc, (long long)Wc,
              (long long)Cin, (long long)Cout, stride);
  ZSB_REQUIRE(R * Hc * Wc * Cbig < (1LL << 31) && R * Hs * Ws * Csmall < (1LL << 31),
              "zsb_conv3x3_fwd_f32: R*H*W*C must be below 2^31");
  if (R == 0) return ZSB_OK;
  ZSB_REQUIRE(x && W && y, "zsb_conv3x3_fwd_f32: null pointer");
  CvGeom g;
  g.R = (int)R; g.Hc = (int)Hc; g.Wc = (int)Wc; g.Hs = (int)Hs; g.Ws = (int)Ws; g.s = stride;
  g.pt = cv_pad_before(g.Hc, g.Hs, stride);
  g.pl = cv_pad_before(g.Wc, g.Ws, stride);
  const int ngs = cv_ngs(Cout);
  const int64_t P = transpose ? R * Hc * Wc : R * Hs * Ws;
  const int64_t per_cta = (int64_t)(CV_WARPS / ngs) * 32 * CV_PX;
  const dim3 grid((unsigned)zsb_ceil_div(P, per_cta), (unsigned)zsb_ceil_div(Cout, CV_SLICE));
  const size_t smem = sizeof(float) * 9 * Cin * ngs * CV_CO;
  cudaStream_t st = (cudaStream_t)stream;
  cudaError_t e;
  if (gate != nullptr) {
    e = cudaFuncSetAttribute(conv3x3_fwd_kernel<true>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess)
      conv3x3_fwd_kernel<true><<<grid, CV_THREADS, smem, st>>>(
          x, gate, W, b, residual, y, g, transpose, (int)Cin, (int)Cout, relu, ngs);
  } else {
    e = cudaFuncSetAttribute(conv3x3_fwd_kernel<false>,
                             cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess)
      conv3x3_fwd_kernel<false><<<grid, CV_THREADS, smem, st>>>(
          x, nullptr, W, b, residual, y, g, transpose, (int)Cin, (int)Cout, relu, ngs);
  }
  if (e != cudaSuccess) {
    zsb_set_error("zsb_conv3x3_fwd_f32: %s", cudaGetErrorString(e));
    return ZSB_ERR_CUDA;
  }
  return zsb_check_launch("conv3x3_fwd");
}

// Slices of the weight-gradient sweep's `part` scratch; each is Ca * Cb floats.
int zsb_conv3x3_wgrad_parts(int64_t R, int64_t Hc, int64_t Wc, int stride) {
  if (R < 1 || Hc < 1 || Wc < 1 || (stride != 1 && stride != 2)) return 0;
  return (int)(WG_SLOTS * cv_wgrad_ctas(R, Hc, Wc, zsb_ceil_div(Hc, stride),
                                        zsb_ceil_div(Wc, stride)));
}

// Weight and bias gradient, one sweep plus one merge launch.  See include/zsb200.h.
int zsb_conv3x3_wgrad_f32(const float* big, const float* small, const float* gate, int grad_big,
                          float* part, float* dW, float* db, int64_t R, int64_t Hc, int64_t Wc,
                          int64_t Ca, int64_t Cb, int stride, void* stream) {
  const int64_t Hs = zsb_ceil_div(Hc, stride > 0 ? stride : 1);
  const int64_t Ws = zsb_ceil_div(Wc, stride > 0 ? stride : 1);
  ZSB_REQUIRE(cv_sizes_ok(R, Hc, Wc, Hs, Ws, Ca, Cb, stride),
              "zsb_conv3x3_wgrad_f32: unsupported sizes (R %lld, H %lld, W %lld, Ca %lld, "
              "Cb %lld, stride %d)", (long long)R, (long long)Hc, (long long)Wc, (long long)Ca,
              (long long)Cb, stride);
  ZSB_REQUIRE(R * Hc * Wc * Ca < (1LL << 31) && R * Hs * Ws * Cb < (1LL << 31),
              "zsb_conv3x3_wgrad_f32: R*H*W*C must be below 2^31");
  ZSB_REQUIRE(R >= 1, "zsb_conv3x3_wgrad_f32: R = 0 (nothing to sum; zero the outputs instead)");
  ZSB_REQUIRE(big && small && part && (dW || db), "zsb_conv3x3_wgrad_f32: null pointer");
  CvGeom g;
  g.R = (int)R; g.Hc = (int)Hc; g.Wc = (int)Wc; g.Hs = (int)Hs; g.Ws = (int)Ws; g.s = stride;
  g.pt = cv_pad_before(g.Hc, g.Hs, stride);
  g.pl = cv_pad_before(g.Wc, g.Ws, stride);
  const int G = (int)cv_wgrad_ctas(R, Hc, Wc, Hs, Ws);
  const int slot0 = dW != nullptr ? 0 : WG_SLOTS - 1;         // db only: the bias slot alone
  const unsigned grid = (unsigned)((WG_SLOTS - slot0) * G);
  cudaStream_t st = (cudaStream_t)stream;
  if (gate != nullptr)
    conv3x3_wgrad_kernel<true><<<grid, CV_THREADS, 0, st>>>(
        big, small, gate, grad_big, part, g, (int)Ca, (int)Cb, G, slot0);
  else
    conv3x3_wgrad_kernel<false><<<grid, CV_THREADS, 0, st>>>(
        big, small, nullptr, grad_big, part, g, (int)Ca, (int)Cb, G, slot0);
  int rc = zsb_check_launch("conv3x3_wgrad");
  if (rc != ZSB_OK) return rc;
  const int T = (int)(Ca * Cb);
  const int n = (dW != nullptr ? 9 * T : 0) + (db != nullptr ? (int)(grad_big ? Ca : Cb) : 0);
  conv3x3_wgrad_merge_kernel<<<(unsigned)zsb_ceil_div(n, CV_THREADS), CV_THREADS, 0, st>>>(
      part, G, T, (int)(grad_big ? Ca : Cb), dW, db);
  return zsb_check_launch("conv3x3_wgrad_merge");
}

}  // extern "C"
