// The passes of the biased k x k convolutions on the tensor-core products, relu?(conv(x) + b +
// residual): tf.layers.conv2d(..., activation=relu) and the conv2d_transpose of
// examples/utils/utils.py:74-113, with the residual added before the ReLU as in the resnet blocks
// of examples/variational_autoencoders/vae_conv.py:20-53.  Geometry as in conv_tc.cu.
//
// The convolution's forward needs no pass of its own: the gather-split of conv_tc.cu, then the
// dense product with its bias + residual + ReLU epilogue (EPI 16 of gemm_logjoint_tc.cu).  The
// transposed convolution's forward ends in
//   col2im-bias:  y = act(col2im-sum + bias[c] + res) and max |y|     (zsb_conv_col2im_f32 epi 4)
// and the backward of both starts with
//   relu-grad:    gp = g (y > 0), or g without ReLU, max |gp|, and per 128-row tile the column
//                 sums of gp, merged in a fixed order into db          (zsb_conv_relu_grad_f32)
#include "conv_tc.cuh"

namespace {

// out = act(sum + bias[c] + res) over the N Hb Wb x C outputs, bias and res may be NULL; max |out|
// into amax_scale[2] (may be NULL)
__global__ void __launch_bounds__(256) col2im_bias_kernel(const float* __restrict__ cols, Geo g,
                                                          const float* __restrict__ bias,
                                                          const float* __restrict__ res, int relu,
                                                          float* __restrict__ out,
                                                          float* __restrict__ amax_scale) {
  const int64_t n = g.N * g.Hb * g.Wb * g.C;
  float m = 0.f;
  for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < n;
       e += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = e / g.C;
    const int c = (int)(e - r * g.C);
    float y = col2im_at(cols, g, r, c);
    if (bias) y += bias[c];
    if (res) y += res[e];
    if (relu) y = fmaxf(y, 0.f);
    out[e] = y;
    m = finite_absmax(m, y);
  }
  if (amax_scale) fold_amax(amax_scale, m, threadIdx.x & 31);
}

// gp = g (y > 0) (relu) or g, max |gp| into scale[2], and per 128-row tile t the column sums
// part[t C + c] (8 warps of 16 rows, met in a fixed order): the ReLU counterpart of conv_tc.cu's
// sigmoid_grad_kernel.  y is not read without ReLU.
__global__ void __launch_bounds__(256) relu_grad_kernel(const float* __restrict__ g,
                                                        const float* __restrict__ y, int relu,
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
      const float d = (!relu || y[r * C + c] > 0.f) ? gv : 0.f;
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

}  // namespace

int conv_col2im_bias_launch(const float* cols, int64_t N, int64_t Hb, int64_t Wb, int C,
                            int64_t Hs, int64_t Ws, int k, int stride, int pt, int pl,
                            const float* bias, const float* residual, int relu, float* out,
                            float* amax_scale, cudaStream_t st) {
  const Geo g{N, Hb, Wb, Hs, Ws, C, k, stride, pt, pl};
  col2im_bias_kernel<<<blocks_for(N * Hb * Wb * C, 256, 16), 256, 0, st>>>(
      cols, g, bias, residual, relu, out, amax_scale);
  return zsb_check_launch("conv_col2im_bias");
}

extern "C" {

int zsb_conv_relu_grad_f32(const float* g, const float* y, int64_t R, int C, int relu, float* gp,
                           float* part, float* db, float* scale, void* stream) {
  ZSB_REQUIRE(g && gp && part && scale && (y || !relu) && R > 0 && C > 0 && C < (1 << 20) &&
                  R * C < (1LL << 31),
              "zsb_conv_relu_grad_f32: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t n_t = zsb_ceil_div(R, TILE);
  relu_grad_kernel<<<dim3((unsigned)n_t, (unsigned)((C + 31) / 32)), 256, 0, st>>>(
      g, y, relu, R, C, gp, part, scale);
  const int rc = zsb_check_launch("conv_relu_grad");
  if (rc || !db) return rc;
  return conv_col_sum_merge_launch(part, n_t, C, db, st);
}

}  // extern "C"
