// Backward pass of the Gaussian dense layer (zs.fused.LinearNormal, EPI 15 of gemm_logjoint_tc.cu)
// in one pass over the S draws: the gradient of the packed pre-activation [R, 2 Dp] (the mean and
// logstd heads in blocks of 64 columns, as the forward product packs them) from the upstream
// gradients of z and of log q(z), with eps recomputed from Philox (or read when it was injected).
// It is then split into operand planes and fed to the layer's input- and weight-gradient products,
// so nothing of size [S, R, D] is kept between the forward and the backward pass.
#include "tc_common.cuh"

namespace {

// One warp per row r, lane-strided over the Dp features (coalesced reads of gz); per (r, j) the S
// draws are summed in order (no atomics: bitwise repeatable).
//   reparameterised:      d mu = sum_s gz,                   d ls = sum_s (gz std eps - glq)
//   not reparameterised:  d mu = sum_s glq eps / std,        d ls = sum_s glq (eps^2 - 1)
// dpre[r, 128 (j / 64) + j % 64] = d mu, dpre[r, 128 (j / 64) + 64 + j % 64] = d ls; the padding
// columns j in [D, Dp) are written as zero.  max |dpre| into scale[2].
__global__ void __launch_bounds__(256) normal_grad_kernel(
    const float* __restrict__ logstd, const float* __restrict__ gz, const float* __restrict__ glq,
    const float* __restrict__ eps_in, uint64_t seed, uint32_t iter, const uint32_t* epoch,
    int reparam, int S, int64_t R, int D, int Dp, float* __restrict__ dpre,
    float* __restrict__ scale) {
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const uint32_t it = iter + (epoch ? *epoch : 0u);
  float m = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * 8 + ty; r < R; r += (int64_t)gridDim.x * 8) {
    for (int j = tx; j < Dp; j += 32) {
      float dmu = 0.f, dls = 0.f;
      if (j < D) {
        const float sd = expf(__ldg(logstd + r * D + j));
        for (int s = 0; s < S; ++s) {
          const int64_t srow = (int64_t)s * R + r;
          const int64_t i = srow * D + j;
          const float e = eps_in ? __ldg(eps_in + i) : philox_normal_at(seed, it, i);
          const float gl = glq ? __ldg(glq + srow) : 0.f;
          if (reparam) {
            const float g = gz ? __ldg(gz + i) : 0.f;
            dmu += g;
            dls += g * sd * e - gl;
          } else {
            dmu += gl * e / sd;
            dls += gl * (e * e - 1.f);
          }
        }
      }
      float* __restrict__ o = dpre + r * (2 * Dp) + (j / 64) * 128 + j % 64;
      o[0] = dmu;
      o[64] = dls;
      m = finite_absmax(finite_absmax(m, dmu), dls);
    }
  }
  fold_amax(scale, m, tx);
}

}  // namespace

extern "C" {

// Backward of zsb_linear_tc_normal_sample_f32 (see include/zsb200.h).
int zsb_linear_normal_grad_f32(const float* logstd, const float* gz, const float* glq,
                               const float* eps_in, uint64_t seed, uint32_t iter,
                               const uint32_t* epoch, int reparam, int S, int64_t R, int D,
                               float* dpre, float* amax_scale, void* stream) {
  ZSB_REQUIRE(logstd && dpre && amax_scale && R > 0 && S >= 1 && D >= 1 && D <= 256,
              "zsb_linear_normal_grad_f32: bad args");
  ZSB_REQUIRE((int64_t)S * R < (1LL << 31), "zsb_linear_normal_grad_f32: too many rows");
  const int Dp = ((D + 63) / 64) * 64;
  int64_t blocks = zsb_ceil_div(R, 8);
  if (blocks > ZSB_NUM_SMS * 8) blocks = ZSB_NUM_SMS * 8;
  normal_grad_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      logstd, gz, glq, eps_in, seed, iter, epoch, reparam, S, R, D, Dp, dpre,
      amax_scale);
  return zsb_check_launch("linear_normal_grad");
}

}  // extern "C"
