// K8: dense layer of a VAE / BNN log-joint on the tensor cores, with the likelihood fused into the
// GEMM epilogue so the [rows, features] logit matrix never reaches HBM (SURVEY 8a row a22: at
// config 3 the decoder output is 262 144 x 784 logits = 822 MB in fp32).
//
//   acc[j, r] = sum_k W[j, k] * h[r, k]          (A = weight rows j, B = activation rows r)
//   l[r, j]   = acc + bias[j]
//   EPI 0  out[r, j] = l  (optionally ReLU)                      plain dense layer
//   EPI 1  part[(j / 32), r] = sum_{j in 32-lane group} x[r % n_x, j] * l - softplus(l)
//          = Bernoulli(logits = l).log_prob(x) summed over the feature axis (univariate.py:398-403
//            + group_ndims = 1, base.py:303-304) once the partial rows are added up
//   EPI 2  out[r, j] = g[r] * (x - sigmoid(l))                   d(sum_r g[r] * log_prob[r]) / dl
//   EPI 3  the EPI 2 values, emitted directly as the fp16 hi/lo operand planes [2][R][Jp] of the
//          two backward products (dh = dl W, dW = dl^T h) plus their column sums (bias gradient):
//          the fp32 dl matrix (822 MB at config 3) is never written or re-read.  The planes' scale
//          is known BEFORE the GEMM: |dl| <= max|g| * (1 + max|x|)  (sigmoid in (0, 1)).
//
// fp32 accuracy on fp16 tensor cores: both operands are pre-split into scaled fp16 hi + lo planes
// (zsb_split16_pad_f32), three fp16 wgmma products per k-step accumulate hi*hi + hi*lo + lo*hi
// in fp32 (dropped term ~2^-22 relative) -- the scheme of the dense-Gaussian HMC kernel
// (hmc_dense_tc.cu), whose persistent pipeline (tc_pipeline_kernel: TMA producer warp, MMA
// warpgroup, 4 epilogue warps, 128 features x 128 rows per unit) this product shares.  As there,
// the product is computed transposed (accumulator row = feature j, column = row r) so an epilogue
// warp touches 32 consecutive features of one row per instruction: coalesced x loads and out stores.
#include "tc_common.cuh"

namespace {

__device__ __forceinline__ float bern_lp(float x, float l) {   // -sigmoid_cross_entropy(x, l)
  return -(fmaxf(l, 0.f) - l * x + __logf(1.f + __expf(-fabsf(l))));
}

// MN (bit 0: operand A, bit 1: operand B; EPI 0 only): the operand is read in a row-major plane
// layout [contraction rows, features] -- MN-major (transposed) wgmma operand.  MN = 3: weight
// gradient dW = g^T h from the row-major planes of g and h; MN = 1: input gradient dh = g W with
// A = the FORWARD planes of W [J, K] (no W^T copy): no product of a dense layer needs a transposed
// copy of anything.  A stage then holds, per plane, two TMA boxes of 64 contraction rows x 64
// features (128-byte rows, SWIZZLE_128B; see gmma_desc).  `Kp` is the padded contraction length.
// GL: the epi 2 / 3 epilogues load the upstream gradient per row instead of broadcasting it.
template <int EPI, int MN, int GL>
struct LinW {
  static constexpr int KIND = 1, RB = 128, MNA = MN & 1, MNB = (MN >> 1) & 1, CVT = 0;
  static constexpr uint32_t TX = Cfg<RB>::STAGE;
  CUtensorMap map_whi, map_wlo, map_hhi, map_hlo;
  const float* bias; const float* x_obs; int64_t n_x; const float* gout;
  float* out; float* part; int64_t R; int J; int Kp; int relu;
  const float* scale_w; const float* scale_h; int k_slices; float* amax_scale;
  int n_blk; int64_t n_tiles; int n_kb_all; int kb_per;
  struct EpiState { float amax = 0.f; };

  __host__ __device__ __forceinline__ int64_t units() const { return n_tiles * k_slices; }
  __device__ __forceinline__ void kb_range(int64_t uu, int& kb0, int& kb1) const {
    kb0 = (int)(uu / n_tiles) * kb_per;
    kb1 = min(kb0 + kb_per, n_kb_all);
  }
  __device__ __forceinline__ void prefetch() const {
    tma_prefetch_desc(&map_whi); tma_prefetch_desc(&map_wlo);
    tma_prefetch_desc(&map_hhi); tma_prefetch_desc(&map_hlo);
  }
  __device__ __forceinline__ void load(int64_t uu, int kb, uint32_t sa, uint32_t fb) const {
    using C = Cfg<RB>;
    const int64_t u = uu % n_tiles;
    const int j0 = (int)(u % n_blk) * BM;                  // feature block
    const int r0 = (int)((u / n_blk) * BN);                // row block
    if (MN & 1) {        // MN-major operand: two boxes of 64 features (c0) x 64 contraction rows
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const uint32_t o = (uint32_t)b * 8192u;
        tma_load_2d(sa + o, &map_whi, fb, j0 + 64 * b, kb * 64);
        tma_load_2d(sa + C::A_TILE + o, &map_wlo, fb, j0 + 64 * b, kb * 64);
      }
    } else {
      tma_load_2d(sa, &map_whi, fb, kb * 64, j0);
      tma_load_2d(sa + C::A_TILE, &map_wlo, fb, kb * 64, j0);
    }
    if (MN & 2) {
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const uint32_t o = (uint32_t)b * 8192u;
        tma_load_2d(sa + 2 * C::A_TILE + o, &map_hhi, fb, r0 + 64 * b, kb * 64);
        tma_load_2d(sa + 2 * C::A_TILE + C::B_TILE + o, &map_hlo, fb, r0 + 64 * b, kb * 64);
      }
    } else {
      tma_load_2d(sa + 2 * C::A_TILE, &map_hhi, fb, kb * 64, r0);
      tma_load_2d(sa + 2 * C::A_TILE + C::B_TILE, &map_hlo, fb, kb * 64, r0);
    }
  }
  __device__ __forceinline__ void convert(int64_t, int, uint8_t*, int) const {}
  __device__ __forceinline__ void epilogue(int64_t uu, uint32_t trow, int quarter, int lane,
                                           EpiState& st) const {
    float& amax = st.amax;   // max |stored output| (EPI 0 / 2): the consumer's fp16-split scale
    const float acc_scale = 1.f / (scale_w[0] * scale_h[0]);   // powers of two: exact
    // EPI 3: `out` = the fp16 plane pair [2][R][Jp_out], amax_scale[0] = their (a-priori) scale
    __half* __restrict__ pl_out = reinterpret_cast<__half*>(out);
    const int Jp_out = ((J + 63) / 64) * 64;
    const float s_out = (EPI == 3) ? amax_scale[0] : 1.f;
    const int64_t u = uu % n_tiles;
    const int slice = (int)(uu / n_tiles);
    const bool empty_slice = slice * kb_per >= n_kb_all;   // accumulator never written
    float* __restrict__ out_s = (EPI == 0 && out) ? out + (int64_t)slice * R * J : out;
    const int nb = (int)(u % n_blk);
    const int j = nb * BM + quarter * 32 + lane;
    const bool j_ok = j < J;
    const float b_j = (j_ok && bias) ? bias[j] : 0.f;
    const int64_t r0 = (u / n_blk) * BN;
    const int64_t part_row = (int64_t)(nb * 4 + quarter) * R;
    const float b_use = (slice == 0) ? b_j : 0.f;           // bias once across the slices
      const bool warp_j_ok = __all_sync(0xffffffffu, j_ok);
      float csum = 0.f;                                       // EPI 3: column sum of this lane's j
      // observations of one 16-column block (rows rbase .. rbase+15, this lane's feature j); all
      // 16 loads are issued back to back, one block AHEAD of their use (L2 latency ~1 us)
      auto load_x = [&](float* xe, float& ge, int c) {
        if (EPI == 0) return;
        const int64_t rbase = r0 + c;
        if (rbase >= R) return;                     // warp-uniform
        int64_t xr = rbase % n_x;
        const float* __restrict__ xp = x_obs + xr * J + j;
        const bool full = warp_j_ok && rbase + 16 <= R;
        if (full && xr + 16 <= n_x) {               // common case: no wrap, no predicates
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) xe[jj] = __ldg(xp + (uint32_t)jj * (uint32_t)J);
        } else {
#pragma unroll
          for (int jj = 0; jj < 16; ++jj) {
            xe[jj] = (j_ok && rbase + jj < R) ? __ldg(xp) : 0.f;
            if (++xr == n_x) { xr = 0; xp = x_obs + j; } else xp += J;
          }
        }
        // upstream gradient of the 16 rows: lane jj holds gout[rbase + jj] (GL = 0: broadcast by
        // shuffle in process(); GL = 1: process() loads it itself, warp-uniform addresses)
        if (EPI >= 2 && !GL) ge = (lane < 16 && rbase + lane < R) ? __ldg(gout + rbase + lane) : 0.f;
      };
      auto process = [&](const uint32_t* v, const float* xe, float ge, int c) {
        // NO early return for rbase >= R: every access below is predicated on the row anyway, and
        // a return here (uniform, but not provably so) makes the compiler wrap each warp shuffle of
        // the row sums in a WARPSYNC.COLLECTIVE sequence (125 SHFL + 70 WARPSYNC -> 63 SHFL)
        const int64_t rbase = r0 + c;
        float lpv[16];
        float* __restrict__ po = (EPI == 0 || EPI == 2) ? out_s + rbase * J + j : nullptr;
        const bool full = warp_j_ok && rbase + 16 <= R;   // no per-element predicates
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const bool ok = full || (j_ok && rbase + jj < R);
          const float l = empty_slice ? b_use : fmaf(__uint_as_float(v[jj]), acc_scale, b_use);
          if (EPI == 0) {
            const float y = relu ? fmaxf(l, 0.f) : l;
            if (ok) { *po = y; amax = fmaxf(amax, fabsf(y)); }
          } else if (EPI == 1) {
            lpv[jj] = ok ? bern_lp(xe[jj], l) : 0.f;
          } else if (EPI == 2) {
            const float g = GL ? ((full || rbase + jj < R) ? __ldg(gout + rbase + jj) : 0.f)
                               : __shfl_sync(0xffffffffu, ge, jj);
            const float y = g * (xe[jj] - __fdividef(1.f, 1.f + __expf(-l)));
            if (ok) { *po = y; amax = fmaxf(amax, fabsf(y)); }
          } else {
            const float g = GL ? ((full || rbase + jj < R) ? __ldg(gout + rbase + jj) : 0.f)
                               : __shfl_sync(0xffffffffu, ge, jj);
            const float y = ok ? g * (xe[jj] - __fdividef(1.f, 1.f + __expf(-l))) : 0.f;
            csum += y;
            lpv[jj] = y * s_out;
          }
          if (EPI == 0 || EPI == 2) po += J;
        }
        if (EPI == 3) {
          // fp16 hi/lo planes of this lane's feature column, two rows per packed conversion;
          // a warp instruction stores 64 contiguous bytes of one plane row
          __half* __restrict__ ph = pl_out + rbase * Jp_out + j;
          __half* __restrict__ pq = ph + R * (int64_t)Jp_out;
          const bool col_ok = j < Jp_out;
#pragma unroll
          for (int jj = 0; jj < 16; jj += 2) {
            const __half2 h2 = __floats2half2_rn(lpv[jj], lpv[jj + 1]);
            const float2 hf = __half22float2(h2);
            const __half2 l2 = __floats2half2_rn(lpv[jj] - hf.x, lpv[jj + 1] - hf.y);
            if (col_ok && (full || rbase + jj < R)) {
              ph[(size_t)jj * (size_t)Jp_out] = __low2half(h2);
              pq[(size_t)jj * (size_t)Jp_out] = __low2half(l2);
            }
            if (col_ok && (full || rbase + jj + 1 < R)) {
              ph[(size_t)(jj + 1) * (size_t)Jp_out] = __high2half(h2);
              pq[(size_t)(jj + 1) * (size_t)Jp_out] = __high2half(l2);
            }
          }
        }
        if (EPI == 1) {
          const float sum = warp_transpose_sum16(lpv, lane);
          if (lane < 16 && rbase + lane < R) part[part_row + rbase + lane] = sum;
        }
      };
      // the observation loads of block i+1 are in flight while block i is processed
      uint32_t va[16], vb[16];
      float xa[EPI ? 16 : 1], xb[EPI ? 16 : 1], ga = 0.f, gb = 0.f;
      load_x(xa, ga, 0);
#pragma unroll 1
      for (int c = 0; c < BN; c += 32) {
        load_x(xb, gb, c + 16);
        acc_ld16(trow + 4u * (uint32_t)c, va);
        process(va, xa, ga, c);
        if (c + 32 < BN) load_x(xa, ga, c + 32);
        acc_ld16(trow + 4u * (uint32_t)(c + 16), vb);
        process(vb, xb, gb, c + 16);
      }
      if (EPI == 3 && part && j_ok) atomicAdd(part + j, csum);   // bias gradient (part = col_sum)
  }
  __device__ __forceinline__ void epi_finish(EpiState& st, int, int lane) const {
    if ((EPI == 0 || EPI == 2) && amax_scale) {   // NaN / inf never win the max (fmaxf drops NaN)
      const float m = warp_max(st.amax <= 3.0e38f ? st.amax : 0.f);
      if (lane == 0 && m > 0.f)
        atomicMax(reinterpret_cast<unsigned int*>(amax_scale) + 2, __float_as_uint(m));
    }
  }
};

// one product on the tensor cores: A = w planes (J_ features), B = h planes (R rows)
template <int EPI, int MN, int GL>
int launch_linear(const CUtensorMap& whi, const CUtensorMap& wlo, const CUtensorMap& hhi,
                  const CUtensorMap& hlo, const float* bias, const float* x_obs, int64_t n_x,
                  const float* gout, float* out, float* part, int64_t R, int J_, int Kp, int relu,
                  const float* scale_w, const float* scale_h, int k_slices, float* amax_scale,
                  cudaStream_t st, const char* what) {
  const int n_blk = (J_ + BM - 1) / BM;
  const int64_t n_tiles = ((R + BN - 1) / BN) * n_blk;
  const int n_kb_all = Kp / 64;
  const int kb_per = (n_kb_all + k_slices - 1) / k_slices;
  const LinW<EPI, MN, GL> w{whi, wlo, hhi, hlo, bias, x_obs, n_x, gout, out, part, R, J_, Kp,
                            relu, scale_w, scale_h, k_slices, amax_scale, n_blk, n_tiles,
                            n_kb_all, kb_per};
  return tc_launch(w, st, what);
}

// One pass over an activation / gradient matrix that produces BOTH operand layouts of the dense
// layers: src [R, K] fp32 (optionally times the ReLU mask (mask_src > 0)) ->
//   planes   [2][R][Kp]  fp16 hi/lo of src * scale   (forward / input-gradient products)
//   planes_t [2][K][Rp]  fp16 hi/lo of (src * scale)^T (weight-gradient product, contraction over R)
//   col_sum  [K] += sum_r src[r, k] * mask           (the bias gradient; float atomics)
// 64 x 64 tiles through shared memory; float2 loads, half2 stores in both layouts.
__global__ void __launch_bounds__(256) split16_dual_kernel(
    const float* __restrict__ src, const float* __restrict__ mask_src, int64_t R, int K, int Kp,
    int64_t Rp, __half* __restrict__ planes, __half* __restrict__ planes_t,
    float* __restrict__ col_sum, const float* __restrict__ scale) {
  __shared__ float tile[64][65];
  __shared__ float csum[8][64];
  const float s = scale[0];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;        // 32 x 8
  const int64_t r_tiles = (Rp + 63) / 64;
  const int c_tiles = (Kp + 63) / 64;
  const int64_t n_pl = R * (int64_t)Kp, n_plt = (int64_t)K * Rp;
  for (int64_t t = blockIdx.x; t < r_tiles * c_tiles; t += gridDim.x) {
    const int64_t r0 = (t / c_tiles) * 64;
    const int c0 = (int)(t % c_tiles) * 64;
    const int c = c0 + 2 * tx;
    float cs0 = 0.f, cs1 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int rl = ty + 8 * i;
      const int64_t r = r0 + rl;
      float2 v = make_float2(0.f, 0.f);
      if (r < R && c < K) {                      // K is even: c + 1 < K as well
        v = *reinterpret_cast<const float2*>(src + r * K + c);
        if (mask_src) {
          const float2 m = *reinterpret_cast<const float2*>(mask_src + r * K + c);
          v.x = m.x > 0.f ? v.x : 0.f;
          v.y = m.y > 0.f ? v.y : 0.f;
        }
      }
      cs0 += v.x; cs1 += v.y;
      v.x *= s; v.y *= s;
      tile[rl][2 * tx] = v.x;
      tile[rl][2 * tx + 1] = v.y;
      if (planes && r < R && c < Kp) {
        const __half2 h = __floats2half2_rn(v.x, v.y);
        const float2 hf = __half22float2(h);
        *reinterpret_cast<__half2*>(planes + r * Kp + c) = h;
        *reinterpret_cast<__half2*>(planes + n_pl + r * Kp + c) =
            __floats2half2_rn(v.x - hf.x, v.y - hf.y);
      }
    }
    if (col_sum) { csum[ty][2 * tx] = cs0; csum[ty][2 * tx + 1] = cs1; }
    __syncthreads();
    if (col_sum && threadIdx.x < 64 && c0 + (int)threadIdx.x < K) {
      float a = 0.f;
#pragma unroll
      for (int i = 0; i < 8; ++i) a += csum[i][threadIdx.x];
      atomicAdd(col_sum + c0 + threadIdx.x, a);
    }
    if (planes_t) {
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int kl = ty + 8 * i;
        const int k = c0 + kl;
        const int64_t r = r0 + 2 * tx;
        if (k < K && r < Rp) {                   // Rp is a multiple of 64: r + 1 < Rp as well
          const float x0 = tile[2 * tx][kl], x1 = tile[2 * tx + 1][kl];
          const __half2 h = __floats2half2_rn(x0, x1);
          const float2 hf = __half22float2(h);
          *reinterpret_cast<__half2*>(planes_t + (int64_t)k * Rp + r) = h;
          *reinterpret_cast<__half2*>(planes_t + n_plt + (int64_t)k * Rp + r) =
              __floats2half2_rn(x0 - hf.x, x1 - hf.y);
        }
      }
    }
    __syncthreads();
  }
}

// scale[0] = power of two s with max|src| * s in [2^11, 2^12); scale[2] = running max bits
__global__ void __launch_bounds__(256) absmax2_kernel(const float* __restrict__ src, int64_t n,
                                                      float* __restrict__ scale) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float a = fabsf(src[i]);
    m = (a == a && a <= 3.0e38f) ? fmaxf(m, a) : m;
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0)
    atomicMax(reinterpret_cast<unsigned int*>(scale) + 2, __float_as_uint(m));
}
// Ticketed variant (ZSB_ABSMAX_TICKET=1):
// scale[0] = power of two s with max|src| * s in [2^11, 2^12); scale[2] = running max bits;
// scale[1] = block ticket.  The LAST block to finish turns the maximum into scale[0] and clears
// slots 1 and 2 again (no separate single-thread kernel; the slot must start zeroed).
__global__ void __launch_bounds__(256) absmax2_ticket_kernel(const float* __restrict__ src, int64_t n,
                                                      float* __restrict__ scale) {
  __shared__ float wm[8];
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float a = fabsf(src[i]);
    m = (a == a && a <= 3.0e38f) ? fmaxf(m, a) : m;
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) wm[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    float bm = wm[0];
#pragma unroll
    for (int w = 1; w < 8; ++w) bm = fmaxf(bm, wm[w]);
    unsigned int* u = reinterpret_cast<unsigned int*>(scale);
    atomicMax(u + 2, __float_as_uint(bm));
    __threadfence();
    if (atomicAdd(u + 1, 1u) == gridDim.x - 1) {
      const float mx = __uint_as_float(atomicAdd(u + 2, 0u));
      int e = 0;
      if (mx > 0.f) frexpf(mx, &e);
      scale[0] = ldexpf(1.f, 12 - e);
      u[2] = 0u;
      u[1] = 0u;
    }
  }
}
// EPI 3 scale, known before the GEMM runs: |g (x - sigmoid(l))| <= max|g| * (1 + max|x|).
// absmax_slot_kernel folds max|src| into scale[slot] (uint bits); bern_grad_scale_kernel turns
// slots 2 (g) and 3 (x) into scale[0] = power of two s with bound * s in [2^11, 2^12).
__global__ void __launch_bounds__(256) absmax_slot_kernel(const float* __restrict__ src, int64_t n,
                                                          float* __restrict__ scale, int slot) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const float a = fabsf(src[i]);
    m = (a == a && a <= 3.0e38f) ? fmaxf(m, a) : m;
  }
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0)
    atomicMax(reinterpret_cast<unsigned int*>(scale) + slot, __float_as_uint(m));
}
__global__ void bern_grad_scale_kernel(float* __restrict__ scale) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  unsigned int* u = reinterpret_cast<unsigned int*>(scale);
  const float m = __uint_as_float(u[2]) * (1.f + __uint_as_float(u[3]));
  int e = 0;
  if (m > 0.f && m <= 3.0e38f) frexpf(m, &e);
  scale[0] = ldexpf(1.f, 12 - e);
  u[2] = 0u;
  u[3] = 0u;
}
__global__ void pow2_scale_kernel(float* __restrict__ scale) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const float m = __uint_as_float(reinterpret_cast<unsigned int*>(scale)[2]);
  int e = 0;
  if (m > 0.f) frexpf(m, &e);
  scale[0] = ldexpf(1.f, 12 - e);
  reinterpret_cast<unsigned int*>(scale)[2] = 0u;
}
// max pass of an operand split: leaves scale[0].  Default: max kernel + single-thread power-of-two
// kernel; ZSB_ABSMAX_TICKET=1: one kernel whose last block converts the maximum.
inline bool absmax_ticket() {
  static const bool v = getenv("ZSB_ABSMAX_TICKET") && atoi(getenv("ZSB_ABSMAX_TICKET")) != 0;
  return v;
}
inline void launch_absmax_scale(const float* src, int64_t n, float* scale, unsigned blocks,
                                cudaStream_t st) {
  if (absmax_ticket()) {
    absmax2_ticket_kernel<<<blocks, 256, 0, st>>>(src, n, scale);
  } else {
    absmax2_kernel<<<blocks, 256, 0, st>>>(src, n, scale);
    pow2_scale_kernel<<<1, 32, 0, st>>>(scale);
  }
}
// src [rows, K] fp32 -> planes [2][rows][Kp] fp16 (hi, lo) of src * scale, zero padded to Kp
__global__ void __launch_bounds__(256) split16_pad_kernel(const float* __restrict__ src,
                                                          int64_t rows, int K, int Kp,
                                                          __half* __restrict__ planes,
                                                          const float* __restrict__ scale) {
  const float s = scale[0];
  const int64_t n = rows * Kp;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / Kp;
    const int k = (int)(i - r * Kp);
    const float x = (k < K) ? src[r * K + k] * s : 0.f;
    const __half h = __float2half_rn(x);
    planes[i] = h;
    planes[n + i] = __float2half_rn(x - __half2float(h));
  }
}
// src [R, C] fp32 -> planes [2][C][Rp] fp16 of (src * scale)^T, zero padded along R: the operand
// layout of the weight-gradient product dW = dl^T h, whose contraction runs over the rows.
__global__ void __launch_bounds__(256) split16_pad_t_kernel(const float* __restrict__ src,
                                                            int64_t R, int C, int64_t Rp,
                                                            __half* __restrict__ planes,
                                                            const float* __restrict__ scale) {
  __shared__ float tile[32][33];
  const float s = scale[0];
  const int64_t n = (int64_t)C * Rp;
  const int64_t r_tiles = (Rp + 31) / 32;
  const int c_tiles = (C + 31) / 32;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;      // 32 x 8
  for (int64_t t = blockIdx.x; t < r_tiles * c_tiles; t += gridDim.x) {
    const int64_t r0 = (t / c_tiles) * 32;
    const int c0 = (int)(t % c_tiles) * 32;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int64_t r = r0 + ty + 8 * i;
      const int c = c0 + tx;
      tile[ty + 8 * i][tx] = (r < R && c < C) ? src[r * C + c] * s : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int c = c0 + ty + 8 * i;
      const int64_t r = r0 + tx;
      if (c < C && r < Rp) {
        const float x = tile[tx][ty + 8 * i];
        const __half h = __float2half_rn(x);
        planes[(int64_t)c * Rp + r] = h;
        planes[n + (int64_t)c * Rp + r] = __float2half_rn(x - __half2float(h));
      }
    }
    __syncthreads();
  }
}
// out[i] = sum_s scratch[s][i]
__global__ void __launch_bounds__(256) slice_sum_kernel(const float* __restrict__ scratch,
                                                        int slices, int64_t n,
                                                        float* __restrict__ out) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int k = 0; k < slices; ++k) s += scratch[(int64_t)k * n + i];
    out[i] = s;
  }
}
__global__ void __launch_bounds__(256) part_sum_kernel(const float* __restrict__ part,
                                                       int n_parts, int64_t R,
                                                       float* __restrict__ out) {
  for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < R;
       r += (int64_t)gridDim.x * blockDim.x) {
    float s = 0.f;
    for (int p = 0; p < n_parts; ++p) s += part[(int64_t)p * R + r];
    out[r] = s;
  }
}

// ZSB_EPI_GLOAD=1: the epi 2 / 3 epilogues load the upstream gradient per row (warp-uniform loads)
// instead of broadcasting it by shuffle (A/B switch of an experiment; default = shuffle)
int epi_gload() {
  static const int v = getenv("ZSB_EPI_GLOAD") ? atoi(getenv("ZSB_EPI_GLOAD")) : 0;
  return v;
}

}  // namespace

extern "C" {

int zsb_linear_tc_kpad(int K) { return ((K + 63) / 64) * 64; }
// rows of the partial-sum scratch of epi 1 (each [R] floats)
int zsb_linear_tc_nparts(int J) { return 4 * ((J + BM - 1) / BM); }

// Operand preparation: src [rows, K] fp32 -> planes [2][rows][Kp] fp16 (Kp = zsb_linear_tc_kpad(K))
// and scale[0] (device float[4] scratch, zero-initialised once by the caller).
int zsb_split16_pad_f32(const float* src, int64_t rows, int K, void* planes, float* scale,
                        void* stream) {
  ZSB_REQUIRE(src && planes && scale && rows > 0 && K > 0, "zsb_split16_pad_f32: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  const int Kp = zsb_linear_tc_kpad(K);
  const int64_t n = rows * (int64_t)K;
  int64_t blocks = zsb_ceil_div(n, 256 * 8);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  if (blocks < 1) blocks = 1;
  launch_absmax_scale(src, n, scale, (unsigned)blocks, st);
  int64_t blocks2 = zsb_ceil_div(rows * (int64_t)Kp, 256 * 4);
  if (blocks2 > ZSB_NUM_SMS * 32) blocks2 = ZSB_NUM_SMS * 32;
  split16_pad_kernel<<<(unsigned)blocks2, 256, 0, st>>>(src, rows, K, Kp,
                                                        reinterpret_cast<__half*>(planes), scale);
  return zsb_check_launch("split16_pad");
}

// Transposed variant: src [R, C] -> planes [2][C][Rp] (Rp = zsb_linear_tc_kpad(R)) of src^T.
int zsb_split16_pad_t_f32(const float* src, int64_t R, int C, void* planes, float* scale,
                          void* stream) {
  ZSB_REQUIRE(src && planes && scale && R > 0 && C > 0, "zsb_split16_pad_t_f32: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t Rp = ((R + 63) / 64) * 64;
  const int64_t n = R * (int64_t)C;
  int64_t blocks = zsb_ceil_div(n, 256 * 8);
  if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
  launch_absmax_scale(src, n, scale, (unsigned)blocks, st);
  int64_t tiles = ((Rp + 31) / 32) * ((C + 31) / 32);
  if (tiles > ZSB_NUM_SMS * 32) tiles = ZSB_NUM_SMS * 32;
  split16_pad_t_kernel<<<(unsigned)tiles, 256, 0, st>>>(src, R, C, Rp,
                                                        reinterpret_cast<__half*>(planes), scale);
  return zsb_check_launch("split16_pad_t");
}

// Both operand layouts of one matrix in ONE pass (see split16_dual_kernel): planes [2][R][Kp]
// and / or planes_t [2][K][Rp] (either may be NULL), optional ReLU mask source, optional column
// sums (bias gradient; col_sum must be zeroed by the caller).  have_amax = 1: scale[2] already
// holds max |src| (written by zsb_linear_tc_amax_f32), so no max pass is run.  K must be even.
int zsb_split16_dual_f32(const float* src, const float* mask_src, int64_t R, int K, void* planes,
                         void* planes_t, float* col_sum, float* scale, int have_amax,
                         void* stream) {
  ZSB_REQUIRE(src && scale && R > 0 && K > 0 && K % 2 == 0 && (planes || planes_t),
              "zsb_split16_dual_f32: bad args (K must be even)");
  cudaStream_t st = (cudaStream_t)stream;
  const int Kp = zsb_linear_tc_kpad(K);
  const int64_t Rp = ((R + 63) / 64) * 64;
  if (!have_amax) {
    const int64_t n = R * (int64_t)K;
    int64_t blocks = zsb_ceil_div(n, 256 * 8);
    if (blocks > ZSB_NUM_SMS * 16) blocks = ZSB_NUM_SMS * 16;
    launch_absmax_scale(src, n, scale, (unsigned)blocks, st);
  } else {
    pow2_scale_kernel<<<1, 32, 0, st>>>(scale);    // max|src| left in scale[2] by a GEMM epilogue
  }
  int64_t tiles = ((Rp + 63) / 64) * ((Kp + 63) / 64);
  if (tiles > ZSB_NUM_SMS * 16) tiles = ZSB_NUM_SMS * 16;
  split16_dual_kernel<<<(unsigned)tiles, 256, 0, st>>>(
      src, mask_src, R, K, Kp, Rp, reinterpret_cast<__half*>(planes),
      reinterpret_cast<__half*>(planes_t), col_sum, scale);
  return zsb_check_launch("split16_dual");
}

// Fused dense layer on the tensor cores.  w_planes [2][J][Kp], h_planes [2][R][Kp] (fp16 planes
// from zsb_split16_pad_f32 with their scales); bias [J] or NULL.
//   epi 0: out [R, J] = h W^T + bias (ReLU if relu != 0)
//   epi 1: out [R] = sum_j Bernoulli(logits = h W^T + bias).log_prob(x[r % n_x, j]);
//          part = scratch of zsb_linear_tc_nparts(J) * R floats
//   epi 2: out [R, J] = gout[r] * (x - sigmoid(logits))
// Split-K (epi 0 only): when the output has fewer than one 128 x 128 tile per SM and `part` is
// given (zsb_linear_tc_slices(R, J, K) * R * J floats), the contraction is cut into slices that
// run on different SMs and are summed afterwards (the weight-gradient shape dW = dl^T h).
int zsb_linear_tc_slices(int64_t R, int J, int K) {
  const int n_blk = (J + BM - 1) / BM;
  const int64_t tiles = ((R + BN - 1) / BN) * n_blk;
  const int n_kb = zsb_linear_tc_kpad(K) / 64;
  int64_t want = ZSB_NUM_SMS / tiles;                       // CTAs per tile
  if (want < 1) want = 1;
  if (want > n_kb / 8) want = n_kb / 8;                      // >= 8 k-blocks per slice
  if (want < 1) want = 1;
  const int kb_per = (int)((n_kb + want - 1) / want);
  return (n_kb + kb_per - 1) / kb_per;                       // no empty slice
}
int zsb_linear_tc_amax_f32(int epi, const void* w_planes, const float* scale_w,
                           const void* h_planes, const float* scale_h, const float* bias,
                           const float* x_obs, int64_t n_x, const float* gout, float* out,
                           float* part, int64_t R, int J, int K, int relu, float* amax_scale,
                           void* stream);
int zsb_linear_tc_f32(int epi, const void* w_planes, const float* scale_w, const void* h_planes,
                      const float* scale_h, const float* bias, const float* x_obs, int64_t n_x,
                      const float* gout, float* out, float* part, int64_t R, int J, int K,
                      int relu, void* stream) {
  return zsb_linear_tc_amax_f32(epi, w_planes, scale_w, h_planes, scale_h, bias, x_obs, n_x, gout,
                                out, part, R, J, K, relu, nullptr, stream);
}
// As zsb_linear_tc_f32; additionally the running max |out| (epi 0 / 2, not with split-K) is
// folded into amax_scale[2] (uint bits, atomicMax): the scale slot zsb_split16_dual_f32 consumes
// with have_amax = 1, so the consumer's operand split needs no separate max pass over `out`.
int zsb_linear_tc_amax_f32(int epi, const void* w_planes, const float* scale_w,
                           const void* h_planes, const float* scale_h, const float* bias,
                           const float* x_obs, int64_t n_x, const float* gout, float* out,
                           float* part, int64_t R, int J, int K, int relu, float* amax_scale,
                           void* stream) {
  ZSB_REQUIRE(epi >= 0 && epi <= 2, "zsb_linear_tc_f32: unknown epilogue");
  ZSB_REQUIRE(w_planes && h_planes && scale_w && scale_h && out && R > 0 && J > 0 && K > 0,
              "zsb_linear_tc_f32: bad args");
  ZSB_REQUIRE(R < (1LL << 31), "zsb_linear_tc_f32: too many rows");
  ZSB_REQUIRE(epi == 0 || (x_obs && n_x > 0), "zsb_linear_tc_f32: observations missing");
  ZSB_REQUIRE(epi != 1 || part, "zsb_linear_tc_f32: partial-sum scratch missing");
  ZSB_REQUIRE(epi != 2 || gout, "zsb_linear_tc_f32: upstream gradient missing");
  cudaStream_t st = (cudaStream_t)stream;
  const int Kp = zsb_linear_tc_kpad(K);
  const __half* wp = reinterpret_cast<const __half*>(w_planes);
  const __half* hp = reinterpret_cast<const __half*>(h_planes);
  CUtensorMap m_whi, m_wlo, m_hhi, m_hlo;
  int rc;
  if ((rc = make_map(&m_whi, wp, (uint64_t)J, (uint64_t)Kp, BM, 128, 1))) return rc;
  if ((rc = make_map(&m_wlo, wp + (int64_t)J * Kp, (uint64_t)J, (uint64_t)Kp, BM, 128, 1)))
    return rc;
  if ((rc = make_map(&m_hhi, hp, (uint64_t)R, (uint64_t)Kp, BN, 128, 1))) return rc;
  if ((rc = make_map(&m_hlo, hp + R * Kp, (uint64_t)R, (uint64_t)Kp, BN, 128, 1))) return rc;
  const int n_blk = (J + BM - 1) / BM;
  int k_slices = 1;
  if (epi == 0 && part) {
    k_slices = zsb_linear_tc_slices(R, J, K);
    if (k_slices > 1 && relu) {
      zsb_set_error("zsb_linear_tc_f32: ReLU cannot be fused into a split-K launch");
      return ZSB_ERR_INVALID;
    }
  }
  float* out_k = (k_slices > 1) ? part : out;
  float* amax_k = k_slices > 1 ? nullptr : amax_scale;
  if (epi == 0)
    rc = launch_linear<0, 0, 0>(m_whi, m_wlo, m_hhi, m_hlo, bias, x_obs, n_x, gout, out_k, part,
                                R, J, Kp, relu, scale_w, scale_h, k_slices, amax_k, st,
                                "linear_tc");
  else if (epi == 1)
    rc = launch_linear<1, 0, 0>(m_whi, m_wlo, m_hhi, m_hlo, bias, x_obs, n_x, gout, nullptr,
                                part, R, J, Kp, relu, scale_w, scale_h, k_slices, amax_k, st,
                                "linear_tc");
  else if (!epi_gload())
    rc = launch_linear<2, 0, 0>(m_whi, m_wlo, m_hhi, m_hlo, bias, x_obs, n_x, gout, out_k, part,
                                R, J, Kp, relu, scale_w, scale_h, k_slices, amax_k, st,
                                "linear_tc");
  else
    rc = launch_linear<2, 0, 1>(m_whi, m_wlo, m_hhi, m_hlo, bias, x_obs, n_x, gout, out_k, part,
                                R, J, Kp, relu, scale_w, scale_h, k_slices, amax_k, st,
                                "linear_tc");

  if (rc == ZSB_OK && k_slices > 1) {
    const int64_t n = R * (int64_t)J;
    int64_t blocks = zsb_ceil_div(n, 256);
    if (blocks > ZSB_NUM_SMS * 8) blocks = ZSB_NUM_SMS * 8;
    slice_sum_kernel<<<(unsigned)blocks, 256, 0, st>>>(part, k_slices, n, out);
    return zsb_check_launch("linear_tc_slice_sum");
  }
  if (rc != ZSB_OK || epi != 1) return rc;
  int64_t blocks = zsb_ceil_div(R, 256);
  if (blocks > ZSB_NUM_SMS * 8) blocks = ZSB_NUM_SMS * 8;
  part_sum_kernel<<<(unsigned)blocks, 256, 0, st>>>(part, 4 * n_blk, R, out);
  return zsb_check_launch("linear_tc_part_sum");
}

// Backward of the Bernoulli likelihood layer with the operand split fused into the GEMM epilogue:
//   dl[r, j] = gout[r] * (x[r % n_x, j] - sigmoid(h W^T + bias))        (the epi-2 values)
// is written ONLY as its fp16 hi/lo planes dl_planes [2][R][kpad(J)] times scale_out[0] (the
// operands of dh = dl W and dW = dl^T h) and summed over the rows into col_sum [J] (+=, the bias
// gradient; may be NULL).  scale_out: device float[4], zeroed once by the caller; its power of two
// comes from the bound max|gout| * (1 + max|x_obs|) >= max|dl|, so no pass over dl is needed.
int zsb_linear_tc_bern_grad_planes_f32(const void* w_planes, const float* scale_w,
                                       const void* h_planes, const float* scale_h,
                                       const float* bias, const float* x_obs, int64_t n_x,
                                       const float* gout, void* dl_planes, float* col_sum,
                                       float* scale_out, int64_t R, int J, int K, void* stream) {
  ZSB_REQUIRE(w_planes && h_planes && scale_w && scale_h && x_obs && n_x > 0 && gout &&
                  dl_planes && scale_out && R > 0 && J > 0 && K > 0,
              "zsb_linear_tc_bern_grad_planes_f32: bad args");
  ZSB_REQUIRE(R < (1LL << 31), "zsb_linear_tc_bern_grad_planes_f32: too many rows");
  cudaStream_t st = (cudaStream_t)stream;
  {
    int64_t bg = zsb_ceil_div(R, 256 * 8), bx = zsb_ceil_div(n_x * (int64_t)J, 256 * 8);
    if (bg > ZSB_NUM_SMS * 16) bg = ZSB_NUM_SMS * 16;
    if (bx > ZSB_NUM_SMS * 16) bx = ZSB_NUM_SMS * 16;
    absmax_slot_kernel<<<(unsigned)bg, 256, 0, st>>>(gout, R, scale_out, 2);
    absmax_slot_kernel<<<(unsigned)bx, 256, 0, st>>>(x_obs, n_x * (int64_t)J, scale_out, 3);
    bern_grad_scale_kernel<<<1, 32, 0, st>>>(scale_out);
  }
  const int Kp = zsb_linear_tc_kpad(K);
  const __half* wp = reinterpret_cast<const __half*>(w_planes);
  const __half* hp = reinterpret_cast<const __half*>(h_planes);
  CUtensorMap m_whi, m_wlo, m_hhi, m_hlo;
  int rc;
  if ((rc = make_map(&m_whi, wp, (uint64_t)J, (uint64_t)Kp, BM, 128, 1))) return rc;
  if ((rc = make_map(&m_wlo, wp + (int64_t)J * Kp, (uint64_t)J, (uint64_t)Kp, BM, 128, 1)))
    return rc;
  if ((rc = make_map(&m_hhi, hp, (uint64_t)R, (uint64_t)Kp, BN, 128, 1))) return rc;
  if ((rc = make_map(&m_hlo, hp + R * Kp, (uint64_t)R, (uint64_t)Kp, BN, 128, 1))) return rc;
  if (epi_gload())
    return launch_linear<3, 0, 1>(m_whi, m_wlo, m_hhi, m_hlo, bias, x_obs, n_x, gout,
                                  reinterpret_cast<float*>(dl_planes), col_sum, R, J, Kp, 0,
                                  scale_w, scale_h, 1, scale_out, st,
                                  "linear_tc_bern_grad_planes");
  return launch_linear<3, 0, 0>(m_whi, m_wlo, m_hhi, m_hlo, bias, x_obs, n_x, gout,
                                reinterpret_cast<float*>(dl_planes), col_sum, R, J, Kp, 0,
                                scale_w, scale_h, 1, scale_out, st, "linear_tc_bern_grad_planes");

}

// Input gradient of a dense layer from the FORWARD weight planes:
//   out [R, K] = sum_j g[r, j] * W[j, k]            (dh = g W, tf.gradients of tf.layers.dense)
// w_planes [2][J][kpad(K)] = the planes of W [J, K] the forward product uses (operand A, read
// MN-major: the contraction runs over W's rows), g_planes [2][R][kpad(J)] (operand B, K-major).
// max |out| is folded into amax_scale[2] (may be NULL) as in zsb_linear_tc_amax_f32.
int zsb_linear_tc_dgrad_f32(const void* w_planes, const float* scale_w, const void* g_planes,
                            const float* scale_g, int64_t R, int J, int K, float* out,
                            float* amax_scale, void* stream) {
  ZSB_REQUIRE(w_planes && g_planes && scale_w && scale_g && out && R > 0 && J > 0 && K > 0,
              "zsb_linear_tc_dgrad_f32: bad args");
  ZSB_REQUIRE(R < (1LL << 31), "zsb_linear_tc_dgrad_f32: too many rows");
  cudaStream_t st = (cudaStream_t)stream;
  const int Kp_w = zsb_linear_tc_kpad(K), Jp = zsb_linear_tc_kpad(J);
  const __half* wp = reinterpret_cast<const __half*>(w_planes);
  const __half* gp = reinterpret_cast<const __half*>(g_planes);
  CUtensorMap m_whi, m_wlo, m_hhi, m_hlo;
  int rc;
  if ((rc = make_map(&m_whi, wp, (uint64_t)J, (uint64_t)Kp_w, 64, 128, 1))) return rc;
  if ((rc = make_map(&m_wlo, wp + (int64_t)J * Kp_w, (uint64_t)J, (uint64_t)Kp_w, 64, 128, 1)))
    return rc;
  if ((rc = make_map(&m_hhi, gp, (uint64_t)R, (uint64_t)Jp, BN, 128, 1))) return rc;
  if ((rc = make_map(&m_hlo, gp + R * Jp, (uint64_t)R, (uint64_t)Jp, BN, 128, 1))) return rc;
  return launch_linear<0, 1, 0>(m_whi, m_wlo, m_hhi, m_hlo, nullptr, nullptr, 0, nullptr, out,
                                nullptr, R, K, Jp, 0, scale_w, scale_g, 1, amax_scale, st,
                                "linear_tc_dgrad");

}

// Weight gradient of a dense layer WITHOUT transposed operands:
//   out [J, K] = sum_r g[r, j] * h[r, k]            (dW = g^T h, tf.gradients of tf.layers.dense)
// h_planes [2][R][Kp(K)], g_planes [2][R][Kp(J)]: the row-major fp16 hi/lo planes the forward /
// input-gradient products already use (zsb_split16_pad_f32 / zsb_split16_dual_f32).  The contraction
// runs over the rows, so both operands are MN-major wgmma operands (LinW<0, 3>);
// split-K over the SMs as in zsb_linear_tc_f32 (part = zsb_linear_tc_slices(J, K, R) * J * K
// floats, or NULL for a single slice).
int zsb_linear_tc_wgrad_f32(const void* h_planes, const float* scale_h, int K,
                            const void* g_planes, const float* scale_g, int J, int64_t R,
                            float* out, float* part, void* stream) {
  ZSB_REQUIRE(h_planes && g_planes && scale_h && scale_g && out && R > 0 && J > 0 && K > 0,
              "zsb_linear_tc_wgrad_f32: bad args");
  ZSB_REQUIRE(R < (1LL << 31) - 64, "zsb_linear_tc_wgrad_f32: too many rows");
  cudaStream_t st = (cudaStream_t)stream;
  const int Kp_h = zsb_linear_tc_kpad(K), Jp_g = zsb_linear_tc_kpad(J);
  const int Rp = zsb_linear_tc_kpad((int)R);                 // padded contraction length
  const __half* hp = reinterpret_cast<const __half*>(h_planes);
  const __half* gp = reinterpret_cast<const __half*>(g_planes);
  CUtensorMap m_whi, m_wlo, m_hhi, m_hlo;                    // "w" = h (rows = k), "h" = g
  int rc;
  if ((rc = make_map(&m_whi, hp, (uint64_t)R, (uint64_t)Kp_h, 64, 128, 1))) return rc;
  if ((rc = make_map(&m_wlo, hp + R * Kp_h, (uint64_t)R, (uint64_t)Kp_h, 64, 128, 1))) return rc;
  if ((rc = make_map(&m_hhi, gp, (uint64_t)R, (uint64_t)Jp_g, 64, 128, 1))) return rc;
  if ((rc = make_map(&m_hlo, gp + R * Jp_g, (uint64_t)R, (uint64_t)Jp_g, 64, 128, 1))) return rc;
  const int k_slices = part ? zsb_linear_tc_slices(J, K, (int)R) : 1;
  rc = launch_linear<0, 3, 0>(m_whi, m_wlo, m_hhi, m_hlo, nullptr, nullptr, 0, nullptr,
                              k_slices > 1 ? part : out, part, (int64_t)J, K, Rp, 0, scale_h,
                              scale_g, k_slices, nullptr, st, "linear_tc_wgrad");

  if (rc == ZSB_OK && k_slices > 1) {
    const int64_t n = (int64_t)J * K;
    int64_t blocks = zsb_ceil_div(n, 256);
    if (blocks > ZSB_NUM_SMS * 8) blocks = ZSB_NUM_SMS * 8;
    slice_sum_kernel<<<(unsigned)blocks, 256, 0, st>>>(part, k_slices, n, out);
    return zsb_check_launch("linear_tc_wgrad_slice_sum");
  }
  return rc;
}

}  // extern "C"
