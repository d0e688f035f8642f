// Shared Hopper (sm_90a) building blocks of the tensor-core kernels (hmc_dense_tc.cu,
// hmc_dense_res.cu, hmc_dense_traj.cu, gemm_logjoint_tc.cu): tile constants, mbarrier pipeline,
// TMA loads, wgmma descriptors and instructions, the shared-memory accumulator tile the epilogue
// warps read, the warp-transpose reduction of the epilogues, the host-side tensor-map encoder and
// one warp-specialised persistent kernel that every tensor-core product runs on.
// (No reference counterpart: ZhuSuan has no kernels; these serve the GEMMs inside the log-joints of
// zhusuan/hmc.py:347-372 and examples/variational_autoencoders/iwae.py:23-32.)
//
// Kernel shape (tc_pipeline_kernel, one persistent CTA per SM, 288 threads):
//   warps 0-3   MMA warpgroup: wgmma m64n128 (two per 128-row tile) accumulating in registers;
//               after the last k-block of a unit the accumulator is written to a padded fp32 tile
//               in shared memory, and the next unit's products start while the epilogue drains it
//   warp 4      TMA producer: cp.async.bulk.tensor swizzled operand tiles into a ring of stages
//   warps 5-8   epilogue: warp w owns accumulator rows 32*(w-5) .. +32, all 128 columns
// A unit is a 128 (rows of operand A) x 128 (rows of operand B) output tile; the three products of
// the fp32-accuracy split (lo*hi, hi*lo, hi*hi) accumulate into the same registers.
#pragma once
#include "common.cuh"
#include <cuda.h>
#include <cuda_fp16.h>

namespace {

constexpr int BM = 128;                                   // rows of operand A per tile (lanes)
constexpr int BN = 128;                                   // rows of operand B per tile (columns)
constexpr int NUM_EPI_WARPS = 4;                          // one per 32-row quarter
constexpr int PRODUCER_WARP = 4;
constexpr int EPI_WARP0 = 5;
constexpr int NUM_THREADS = 32 * (EPI_WARP0 + NUM_EPI_WARPS);   // 288
constexpr int ACC_LD = BN + 4;                            // padded row: conflict-free float4 reads
constexpr int ACC_BYTES = BM * ACC_LD * 4;                // 66 KB
constexpr int STAGE_BUDGET = 128 * 1024;                  // operand ring
constexpr long long WAIT_TIMEOUT_CYCLES = 4000000000LL;   // ~2 s: trap instead of hanging the box

// operand ring of a product whose smem rows are RB bytes (128: SWIZZLE_128B, 64: SWIZZLE_64B)
template <int RB>
struct Cfg {
  static constexpr int A_TILE = BM * RB;
  static constexpr int B_TILE = BN * RB;
  static constexpr int STAGE = 2 * A_TILE + 2 * B_TILE;      // hi + lo planes of A and B
  static constexpr int STAGES = STAGE_BUDGET / STAGE;        // 2 (RB 128) / 4 (RB 64)
  static constexpr int SMEM = STAGES * STAGE + ACC_BYTES + 128 + 1024;
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred P1;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 P1, [%1], %2;\n\t"
      "selp.b32 %0, 1, 0, P1;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
// no printf on timeout: a call anywhere in the kernel would serialise the wgmma pipeline
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity))
    if (clock64() - t0 > WAIT_TIMEOUT_CYCLES) __trap();
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}

// wgmma shared-memory descriptor.  K-major (MN = 0): rows of RB bytes, 8-row swizzle atoms (SBO =
// 8 rows); MN-major (MN = 1, fp16, SWIZZLE_128B): boxes of 64 elements x 64 contraction rows, LBO =
// 8 KB to the next 64 elements, SBO = 1 KB to the next 8 contraction rows.
template <int MN, int RB>
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
  uint64_t d = (uint64_t)((saddr & 0x3FFFF) >> 4);
  if (MN) {
    d |= (uint64_t)(8192 >> 4) << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;                                 // SWIZZLE_128B
  } else {
    d |= (uint64_t)1 << 16;                                 // unused for swizzled K-major
    d |= (uint64_t)((8 * RB) >> 4) << 32;
    d |= (uint64_t)(RB == 128 ? 1 : 2) << 62;               // SWIZZLE_128B / SWIZZLE_64B
  }
  return d;
}
__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void wgmma_tf32(float (&d)[64], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16(float (&d)[64], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, %66, %67;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "n"(TA), "n"(TB));
}

// 16 consecutive fp32 accumulator columns of this thread's row (`addr` = shared byte address)
__device__ __forceinline__ void acc_ld16(uint32_t addr, uint32_t v[16]) {
#pragma unroll
  for (int i = 0; i < 4; ++i)
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];"
                 : "=r"(v[4 * i]), "=r"(v[4 * i + 1]), "=r"(v[4 * i + 2]), "=r"(v[4 * i + 3])
                 : "r"(addr + 16u * i));
}

// In: every lane holds v[0..15] (value of "column" j at this lane's row).  Out: returns, on lanes
// l < 16 (and mirrored on l+16), the sum over the 32 lanes of column l & 15 (31 shuffles).
__device__ __forceinline__ float warp_transpose_sum16(float v[16], int lane) {
#pragma unroll
  for (int i = 0; i < 16; ++i) v[i] += __shfl_xor_sync(0xffffffffu, v[i], 16);
#pragma unroll
  for (int o = 8, cnt = 16; o >= 1; o >>= 1, cnt >>= 1) {
    const bool upper = (lane & o) != 0;
#pragma unroll
    for (int i = 0; i < cnt / 2; ++i) {
      const float keep = upper ? v[i + cnt / 2] : v[i];
      const float send = upper ? v[i] : v[i + cnt / 2];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, o);
    }
  }
  return v[0];
}

// One k-block (RB bytes of contraction per operand row) of the three split products for both
// 64-row halves of the tile.  KIND 0: TF32 operands, 1: fp16.  MNA / MNB: operand read MN-major.
template <int KIND, int RB, int MNA, int MNB>
__device__ __forceinline__ void mma_kblock(float (&d)[2][64], uint32_t sa) {
  using C = Cfg<RB>;
#pragma unroll
  for (int k = 0; k < RB / 32; ++k) {       // 32 B of contraction (8 TF32 / 16 fp16) per k-step
    const uint32_t bo = MNB ? (uint32_t)k * 2048u : (uint32_t)k * 32u;
    const uint64_t b_hi = gmma_desc<MNB, RB>(sa + 2 * C::A_TILE + bo);
    const uint64_t b_lo = gmma_desc<MNB, RB>(sa + 2 * C::A_TILE + C::B_TILE + bo);
#pragma unroll
    for (int mh = 0; mh < 2; ++mh) {
      const uint32_t ao = MNA ? (uint32_t)mh * 8192u + (uint32_t)k * 2048u
                              : (uint32_t)(mh * 64 * RB) + (uint32_t)k * 32u;
      const uint64_t a_hi = gmma_desc<MNA, RB>(sa + ao);
      const uint64_t a_lo = gmma_desc<MNA, RB>(sa + C::A_TILE + ao);
      // small cross terms first, hi*hi last
      if (KIND == 0) {
        wgmma_tf32(d[mh], a_lo, b_hi);
        wgmma_tf32(d[mh], a_hi, b_lo);
        wgmma_tf32(d[mh], a_hi, b_hi);
      } else {
        wgmma_f16<MNA, MNB>(d[mh], a_lo, b_hi);
        wgmma_f16<MNA, MNB>(d[mh], a_hi, b_lo);
        wgmma_f16<MNA, MNB>(d[mh], a_hi, b_hi);
      }
    }
  }
}

// The persistent warp-specialised kernel.  W describes one product:
//   KIND, RB, MNA, MNB, CVT       compile-time shape (CVT: the MMA warpgroup writes the B planes
//                                 itself through W::convert; the producer then loads A only)
//   units(), kb_range(u, kb0, kb1)
//   load(u, kb, stage_addr, bar)  the TMA loads of one stage (W::TX bytes)
//   EpiState, epilogue(u, acc_row_addr, quarter, lane, st), epi_finish(st, quarter, lane)
template <class W>
__global__ void __launch_bounds__(NUM_THREADS, 1) tc_pipeline_kernel(const __grid_constant__ W w) {
  using C = Cfg<W::RB>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t acc_base = smem_base + C::STAGES * C::STAGE;
  const uint32_t bars = acc_base + ACC_BYTES;
  const uint32_t full_bar = bars;                          // [STAGES]
  const uint32_t empty_bar = bars + 8 * C::STAGES;         // [STAGES]
  const uint32_t tfull_bar = bars + 16 * C::STAGES;        // accumulator tile written
  const uint32_t tempty_bar = tfull_bar + 8;               // accumulator tile drained

  // broadcast so the compiler knows the role branches are warp-uniform
  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int64_t n_units = w.units();

  if (threadIdx.x == 0) {
    for (int s = 0; s < C::STAGES; ++s) {
      mbar_init(full_bar + 8 * s, 1);
      mbar_init(empty_bar + 8 * s, 1);
    }
    mbar_init(tfull_bar, 128);
    mbar_init(tempty_bar, 32 * NUM_EPI_WARPS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // ===================== MMA warpgroup =====================
    const int tid = threadIdx.x;
    float d[2][64];
    int stage = 0;
    uint32_t phase = 0, acc_phase = 0;
    for (int64_t u = blockIdx.x; u < n_units; u += gridDim.x) {
      int kb0, kb1;
      w.kb_range(u, kb0, kb1);
#pragma unroll
      for (int mh = 0; mh < 2; ++mh)
#pragma unroll
        for (int i = 0; i < 64; ++i) d[mh][i] = 0.f;
      int prev = -1;
      for (int kb = kb0; kb < kb1; ++kb) {
        const uint32_t sa = smem_base + stage * C::STAGE;
        mbar_wait(full_bar + 8 * stage, phase);
        if (W::CVT) {
          w.convert(u, kb, smem_raw + (sa - smem_u32(smem_raw)), tid);
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // visible to wgmma
          asm volatile("bar.sync 1, 128;" ::: "memory");
        }
        wgmma_fence();
        mma_kblock<W::KIND, W::RB, W::MNA, W::MNB>(d, sa);
        wgmma_commit();
        wgmma_wait<1>();                                  // the previous stage has been read
        if (prev >= 0 && tid == 0) mbar_arrive(empty_bar + 8 * prev);
        prev = stage;
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
      }
      wgmma_wait<0>();
      if (prev >= 0 && tid == 0) mbar_arrive(empty_bar + 8 * prev);
      mbar_wait(tempty_bar, acc_phase ^ 1);           // epilogue drained the previous unit
      const int row = 16 * (tid >> 5) + ((tid & 31) >> 2);
      const int col = 2 * (tid & 3);
#pragma unroll
      for (int mh = 0; mh < 2; ++mh)
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const uint32_t a0 = acc_base + (uint32_t)(((64 * mh + row) * ACC_LD + 8 * j + col) * 4);
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a0), "f"(d[mh][4 * j]),
                       "f"(d[mh][4 * j + 1]) : "memory");
          asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a0 + 8u * ACC_LD * 4u),
                       "f"(d[mh][4 * j + 2]), "f"(d[mh][4 * j + 3]) : "memory");
        }
      mbar_arrive(tfull_bar);
      acc_phase ^= 1;
    }
  } else if (warp == PRODUCER_WARP) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      w.prefetch();
      int stage = 0;
      uint32_t phase = 0;
      for (int64_t u = blockIdx.x; u < n_units; u += gridDim.x) {
        int kb0, kb1;
        w.kb_range(u, kb0, kb1);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(empty_bar + 8 * stage, phase ^ 1);
          const uint32_t fb = full_bar + 8 * stage;
          mbar_expect_tx(fb, W::TX);
          w.load(u, kb, smem_base + stage * C::STAGE, fb);
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== epilogue =====================
    const int quarter = warp - EPI_WARP0;
    const uint32_t trow = acc_base + (uint32_t)((quarter * 32 + lane) * ACC_LD * 4);
    typename W::EpiState st;
    uint32_t acc_phase = 0;
    for (int64_t u = blockIdx.x; u < n_units; u += gridDim.x) {
      mbar_wait(tfull_bar, acc_phase);
      w.epilogue(u, trow, quarter, lane, st);
      __syncwarp();
      mbar_arrive(tempty_bar);
      acc_phase ^= 1;
    }
    w.epi_finish(st, quarter, lane);
  }
}

// one launch of tc_pipeline_kernel<W>: opt in to the dynamic shared memory once, one CTA per SM
template <class W>
int tc_launch(const W& w, cudaStream_t st, const char* what) {
  static const cudaError_t attr = cudaFuncSetAttribute(
      tc_pipeline_kernel<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<W::RB>::SMEM);
  if (attr != cudaSuccess) {
    zsb_set_error("%s: cudaFuncSetAttribute: %s", what, cudaGetErrorString(attr));
    return ZSB_ERR_CUDA;
  }
  int dev = 0, sms = ZSB_NUM_SMS;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  int64_t grid = w.units();
  if (grid > sms) grid = sms;
  if (grid < 1) grid = 1;
  tc_pipeline_kernel<W><<<(unsigned)grid, NUM_THREADS, Cfg<W::RB>::SMEM, st>>>(w);
  return zsb_check_launch(what);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) !=
            cudaSuccess || qres != cudaDriverEntryPointSuccess)
      return nullptr;
    fn = (EncodeTiledFn)p;
  }
  return fn;
}

// 2-D row-major [rows, cols] tensor (fp32, or fp16 when half_elems), box = [box_rows, rb bytes],
// swizzle = the row width (SWIZZLE_128B for rb = 128, SWIZZLE_64B for rb = 64).
int make_map(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows,
             int rb, int half_elems = 0) {
  EncodeTiledFn enc = get_encode_fn();
  if (!enc) {
    zsb_set_error("tc: cuTensorMapEncodeTiled unavailable");
    return ZSB_ERR_CUDA;
  }
  const int esz = half_elems ? 2 : 4;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * esz};
  cuuint32_t box[2] = {(cuuint32_t)(rb / esz), box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(map, half_elems ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32,
                   2, (void*)base, dims, strides, box, estr,
                   CU_TENSOR_MAP_INTERLEAVE_NONE,
                   rb == 128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    zsb_set_error("tc: cuTensorMapEncodeTiled failed (%d)", (int)r);
    return ZSB_ERR_CUDA;
  }
  return ZSB_OK;
}

}  // namespace
