// Shared device/host helpers for libzsb200 (sm_90a, H100).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <math.h>
#include <initializer_list>

#define ZSB_OK 0
#define ZSB_ERR_INVALID (-1)
#define ZSB_ERR_CUDA (-2)
#define ZSB_ERR_UNSUPPORTED (-3)

void zsb_set_error(const char* fmt, ...);
int zsb_check_launch(const char* what);
const uint32_t* zsb_epoch_ptr();   // device draw epoch (api.cu), NULL when not registered

#define ZSB_REQUIRE(cond, ...)                    \
  do {                                            \
    if (!(cond)) {                                \
      zsb_set_error(__VA_ARGS__);                 \
      return ZSB_ERR_INVALID;                     \
    }                                             \
  } while (0)

static inline int64_t zsb_ceil_div(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Number of SMs on H100 SXM; grids of grid-stride kernels are sized in multiples of this.
#define ZSB_NUM_SMS 132

// ---- device state of one HMC sampler (all float32, lives in HBM; hmc.py:258-264, 82-87, 118) ----
// Layout is part of the C ABI (include/zsb200.h: ZSB_HMC_STATE_*).
enum {
  ZSB_ST_T = 0,            // hmc.py:264   self.t
  ZSB_ST_STEP_SIZE = 1,    // hmc.py:258   self.step_size (persistent variable)
  ZSB_ST_TUNER_STEP = 2,   // hmc.py:82
  ZSB_ST_LOG_EPS_BAR = 3,  // hmc.py:84
  ZSB_ST_H_BAR = 4,        // hmc.py:86
  ZSB_ST_MU = 5,           // hmc.py:79    10 * initial step size
  ZSB_ST_EWMV_T = 6,       // hmc.py:118
  ZSB_ST_EPS_USED = 7,     // step size used by the current iteration's leapfrog
  ZSB_ST_ACC_MEAN = 8,     // global mean acceptance of the last MH test
  ZSB_ST_FLAGS = 9,        // bit 0: non-finite old log-prob (hmc.py:51-53), stored as uint32 bits
  ZSB_ST_SEARCH_LAST = 10, // _init_step_size loop: last acceptance (hmc.py:343)
  ZSB_ST_SEARCH_COND = 11, // _init_step_size loop: cond (1.0 = continue)
  ZSB_ST_SIZE = 16
};

#ifdef __CUDACC__

// Round-to-nearest mul/add/sub/div that the compiler may not contract into FMAs: the elementwise
// sampler arithmetic is written with these in the reference's operation order so the NumPy oracle
// reproduces it bit-for-bit (host versions are used for launch-time scalar constants).
__host__ __device__ __forceinline__ float mul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  volatile float r = a * b; return r;
#endif
}
__host__ __device__ __forceinline__ float add(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fadd_rn(a, b);
#else
  volatile float r = a + b; return r;
#endif
}
__host__ __device__ __forceinline__ float sub(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fsub_rn(a, b);
#else
  volatile float r = a - b; return r;
#endif
}
__host__ __device__ __forceinline__ float fdiv(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  volatile float r = a / b; return r;
#endif
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
// Reduce over groups of LANES consecutive lanes (LANES power of two <= 32).
template <int LANES>
__device__ __forceinline__ float sub_warp_sum(float v) {
#pragma unroll
  for (int o = LANES / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Block-wide sum for blockDim.x <= 1024 (result valid in all threads). smem: >= 32 floats.
__device__ __forceinline__ float block_sum(float v, float* smem) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) smem[wid] = v;
  __syncthreads();
  const int nw = (blockDim.x + 31) >> 5;
  float r = (lane < nw) ? smem[lane] : 0.f;
  r = warp_sum(r);
  return r;
}

// ---------------- Philox4x32-10 (Salmon et al. 2011); restated in oracle/philox.py ----------------
struct Philox4 {
  uint32_t x, y, z, w;
};
__device__ __forceinline__ Philox4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3,
                                                 uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(M0, c0), lo0 = M0 * c0;
    const uint32_t hi1 = __umulhi(M1, c2), lo1 = M1 * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0; c1 = lo1; c2 = n2; c3 = lo0;
    k0 += W0; k1 += W1;
  }
  Philox4 o; o.x = c0; o.y = c1; o.z = c2; o.w = c3;
  return o;
}
__device__ __forceinline__ float u32_to_uniform(uint32_t x) {        // [0, 1)
  return (float)(x >> 8) * (1.0f / 16777216.0f);
}
__device__ __forceinline__ float u32_to_uniform_open(uint32_t x) {   // (0, 1]
  return ((float)(x >> 8) + 1.0f) * (1.0f / 16777216.0f);
}
__device__ __forceinline__ void box_muller(uint32_t a, uint32_t b, float& z0, float& z1) {
  const float u1 = u32_to_uniform_open(a), u2 = u32_to_uniform(b);
  const float r = sqrtf(-2.0f * logf(u1));
  float s, c;
  sincospif(2.0f * u2, &s, &c);          // exact period reduction: cos(2 pi u2), sin(2 pi u2)
  z0 = r * c; z1 = r * s;
}
// Four standard normals for (row, 4-element block `blk`) of stream/iteration; counter layout
// (blk, row, iteration, stream) -- identical on every GPU count because `row` is the GLOBAL chain.
__device__ __forceinline__ void philox_normal4(uint64_t seed, uint32_t stream, uint32_t iter,
                                               uint32_t row, uint32_t blk, float z[4]) {
  const Philox4 r = philox4x32_10(blk, row, iter, stream, (uint32_t)seed, (uint32_t)(seed >> 32));
  box_muller(r.x, r.y, z[0], z[1]);
  box_muller(r.z, r.w, z[2], z[3]);
}
__device__ __forceinline__ float philox_uniform_row(uint64_t seed, uint32_t stream, uint32_t iter,
                                                    uint32_t row) {
  const Philox4 r = philox4x32_10(0u, row, iter, stream, (uint32_t)seed, (uint32_t)(seed >> 32));
  return u32_to_uniform(r.x);
}

// Vectorised elementwise launcher over a [rows, row_len] matrix with row_len % 4 == 0: one thread
// handles one float4 = one Philox block; f(i4, row, c4) with i4 the float4 index, c4 the float4
// column inside the row.  32-bit index math (n4 < 2^31).
template <class F>
__global__ void __launch_bounds__(256) ew4_kernel(uint32_t n4, uint32_t q4, F f) {
  for (uint32_t i4 = blockIdx.x * blockDim.x + threadIdx.x; i4 < n4; i4 += gridDim.x * blockDim.x) {
    const uint32_t row = i4 / q4;
    f(i4, row, i4 - row * q4);
  }
}
// same, additionally block-summing the returned value into part[blockIdx.x]
template <class F>
__global__ void __launch_bounds__(256) ew4_sum_kernel(uint32_t n4, uint32_t q4,
                                                      float* __restrict__ part, F f) {
  __shared__ float red4[32];
  float s = 0.f;
  for (uint32_t i4 = blockIdx.x * blockDim.x + threadIdx.x; i4 < n4; i4 += gridDim.x * blockDim.x) {
    const uint32_t row = i4 / q4;
    s += f(i4, row, i4 - row * q4);
  }
  s = block_sum(s, red4);
  if (threadIdx.x == 0) part[blockIdx.x] = s;
}
__device__ __forceinline__ float4 ld4(const float* p, uint32_t i4) {
  return reinterpret_cast<const float4*>(p)[i4];
}
__device__ __forceinline__ void st4(float* p, uint32_t i4, float4 v) {
  reinterpret_cast<float4*>(p)[i4] = v;
}
// vec4 path is legal when the row length is a multiple of 4, all pointers are 16-byte aligned and
// the element count fits 32-bit float4 indexing.
static inline bool zsb_vec4_ok(int64_t chains, int64_t row_len, std::initializer_list<const void*> ptrs) {
  if (row_len % 4 != 0 || chains * row_len / 4 >= (1LL << 31)) return false;
  for (const void* q : ptrs)
    if (q && (reinterpret_cast<uintptr_t>(q) & 15)) return false;
  return true;
}

// RNG stream ids (word 3 of the Philox counter)
#define ZSB_STREAM_MOMENTUM 1u
#define ZSB_STREAM_UNIFORM 2u
#define ZSB_STREAM_SGMCMC_NOISE 3u
#define ZSB_STREAM_SGMCMC_RESAMPLE 4u
#define ZSB_STREAM_SAMPLE 5u

#endif  // __CUDACC__
