// The geometry and the col2im gather shared by the k x k convolution passes around the tensor-core
// products: conv_tc.cu (the gather-split and col2im-sum every layer uses, and the passes of the
// batch-normalised and sigmoid layers) and conv_bias.cu (the passes of the biased layers with a
// residual and ReLU).  The geometry is described at the top of conv_tc.cu.
#pragma once
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

}  // namespace

// Host launchers one file gives the other; each kernel stays in the file that defines it.
// conv_tc.cu: db[c] = the column-sum partials part [n_t][C] merged in a fixed order
int conv_col_sum_merge_launch(const float* part, int64_t n_t, int C, float* db, cudaStream_t st);
// conv_bias.cu: epi 4 of zsb_conv_col2im_f32 on a checked geometry
int conv_col2im_bias_launch(const float* cols, int64_t N, int64_t Hb, int64_t Wb, int C,
                            int64_t Hs, int64_t Ws, int k, int stride, int pt, int pl,
                            const float* bias, const float* residual, int relu, float* out,
                            float* amax_scale, cudaStream_t st);
