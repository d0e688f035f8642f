// Shared Hopper (sm_90a) building blocks of the tensor-core kernels (hmc_dense_tc.cu,
// hmc_dense_res.cu, gemm_logjoint_tc.cu): tile constants, mbarrier pipeline,
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
//
// A work descriptor may declare CLUSTER > 1 (only the dense leapfrog pass, ResW, does): the CTAs
// then run as thread-block clusters of CLUSTER consecutive blocks, which take CLUSTER consecutive
// units per round and run the same k-block sequence.  Operand tiles two CTAs of a cluster share
// are fetched from L2 once: each CTA loads its slice of the tile and multicasts it into every
// CTA that uses it, so a stage of one CTA is written by several producers.  Every CTA still
// arms its own full barrier for the whole stage; its empty barrier counts one release from each
// CTA of the cluster, so no producer overwrites a stage that a peer has not finished reading.
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
constexpr unsigned long long WAIT_TIMEOUT_NS = 2000000000ULL;   // 2 s: trap instead of hanging

// Stall accounting of tc_pipeline_kernel (scripts/pass_stalls.py builds it; off in the shipped
// library, whose tensor-core kernels read no cycle counter).  Each CTA adds the clock64() cycles
// of its roles' waits into PASS_PROF_SLOTS counters of g_pass_prof[blockIdx.x], over every launch
// until zsb_pass_profile_read (hmc_dense_res.cu) copies them out and clears them.
enum PassProfSlot {
  PROF_MMA_TOTAL,        // MMA warpgroup: first unit to the last accumulator store
  PROF_MMA_FULL,         //   in mbar_spin(full) of the k-loop
  PROF_MMA_TEMPTY,       //   in mbar_wait(tempty): the epilogue has not drained the tile yet
  PROF_MMA_STORE,        //   storing the accumulator tile
  PROF_PROD_EMPTY,       // producer: in mbar_wait(empty)
  PROF_EPI_TFULL,        // epilogue warp 0: in mbar_wait(tfull)
  PROF_EPI_UNIT,         //   in the epilogue of its units
  PROF_UNITS,            // units of this CTA
  PASS_PROF_SLOTS
};
constexpr int PASS_PROF_CTAS = 1024;
#ifdef ZSB_PASS_PROFILE
constexpr bool kPassProfile = true;
__device__ unsigned long long g_pass_prof[PASS_PROF_CTAS * PASS_PROF_SLOTS];
#else
constexpr bool kPassProfile = false;
#endif
__device__ __forceinline__ long long prof_clock() {
  if constexpr (kPassProfile) return clock64();
  return 0;
}
__device__ __forceinline__ void prof_add(int slot, long long v) {
#ifdef ZSB_PASS_PROFILE
  if (blockIdx.x < PASS_PROF_CTAS)
    atomicAdd(&g_pass_prof[blockIdx.x * PASS_PROF_SLOTS + slot], (unsigned long long)v);
#endif
}

// operand ring of a product whose smem rows are RB bytes (128: SWIZZLE_128B, 64: SWIZZLE_64B).
// With 64-byte rows the ring takes five 32 KB stages: 160 KB beside the accumulator tile, the
// barriers and the 512 B that aligning a SWIZZLE_64B ring may cost, within the 227 KB of shared
// memory a CTA may have.  The stall accounting of the dense pass (scripts/pass_stalls.py) showed
// its MMA warpgroup waiting on full stages for over a third of its cycles with four.
template <int RB>
struct Cfg {
  static constexpr int A_TILE = BM * RB;
  static constexpr int B_TILE = BN * RB;
  static constexpr int STAGE = 2 * A_TILE + 2 * B_TILE;      // hi + lo planes of A and B
  static constexpr int STAGES = RB == 128 ? 2 : 5;
  static constexpr int ALIGN = RB == 128 ? 1024 : 512;       // the swizzle pattern's period
  static constexpr int SMEM = STAGES * STAGE + ACC_BYTES + 128 + ALIGN;
  static_assert(SMEM <= 227 * 1024, "operand ring exceeds shared memory");
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
__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}
// no printf on timeout: a call anywhere in the kernel would serialise the wgmma pipeline.  The
// timeout runs on the global timer, so that the cycle counter is read only by the stall accounting
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const unsigned long long t0 = global_ns();
  while (!mbar_try_wait(bar, parity))
    if (global_ns() - t0 > WAIT_TIMEOUT_NS) __trap();
}
// Wait without a timeout, for the MMA warpgroup's full-barrier wait inside the k-loop.  A trap
// path there, with wgmma accumulators in flight, makes ptxas wait for every wgmma before the next
// one issues (C7517 "warpgroup.wait is injected").  A stall of the MMA warpgroup still traps: the
// epilogue warps wait on tfull, with a timeout, for every unit the MMA warpgroup owes them.
__device__ __forceinline__ void mbar_spin(uint32_t bar, uint32_t parity) {
  while (!mbar_try_wait(bar, parity)) {
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      " [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
// tma_load_2d into the same shared offset of every CTA of the cluster in `mask`; each of them
// counts the box's bytes on its own barrier at offset `bar`
__device__ __forceinline__ void tma_load_2d_mc(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                               int c0, int c1, uint16_t mask) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes"
      ".multicast::cluster [%0], [%1, {%3, %4}], [%2], %5;"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c0), "r"(c1), "h"(mask)
      : "memory");
}
// arrive on the barrier at offset `bar` of cluster CTA `cta`.  Only for releasing a stage whose
// reads have completed (wgmma.wait_group): no memory operation is ordered by it, and a
// .release.cluster arrive would cost a MEMBAR.ALL.GPU before every call.
__device__ __forceinline__ void mbar_arrive_cluster(uint32_t bar, uint32_t cta) {
  asm volatile(
      "{\n\t.reg .b32 rb;\n\t"
      "mapa.shared::cluster.u32 rb, %0, %1;\n\t"
      "mbarrier.arrive.shared::cluster.b64 _, [rb];\n\t}"
      ::"r"(bar), "r"(cta)
      : "memory");
}
// every thread of every CTA of the cluster
__device__ __forceinline__ void cluster_sync() {
  asm volatile("barrier.cluster.arrive.release;\n\tbarrier.cluster.wait.acquire;" ::: "memory");
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

// The fp16 operand-plane format of every fp32 matrix the products read: planes [2][rows][cols] of
// x * s, hi = fp16(x s) and lo = fp16(x s - hi), for a power of two s that puts max |x| in
// [2^11, 2^12).  A split finds max |x| by folding it into word 2 of its scale slot.
__device__ __forceinline__ float pow2_plane_scale(float m) {
  int e = 0;
  if (m > 0.f) frexpf(m, &e);             // m = f * 2^e, f in [0.5, 1)  ->  m < 2^e
  return ldexpf(1.f, 12 - e);             // m * sq in [2^11, 2^12)
}
// max over finite |x| (NaN / inf are left to the chain that produced them)
__device__ __forceinline__ float finite_absmax(float m, float x) {
  const float a = fabsf(x);
  return (a <= 3.0e38f) ? fmaxf(m, a) : m;
}
// p[0] = hi, p[lo] = lo of the already scaled x (lo: offset of the lo plane)
__device__ __forceinline__ void store_hilo(__half* p, int64_t lo, float x) {
  const __half h = __float2half_rn(x);
  p[0] = h;
  p[lo] = __float2half_rn(x - __half2float(h));
}
// the warp's max of m (finite, >= 0) into scale[2] as uint bits, which order as the floats do
__device__ __forceinline__ void fold_amax(float* scale, float m, int lane) {
  m = warp_max(m);
  if (lane == 0 && m > 0.f) atomicMax(reinterpret_cast<unsigned int*>(scale) + 2, __float_as_uint(m));
}

// One k-block (RB bytes of contraction per operand row) of the three split products for both
// 64-row halves of the tile.  KIND 0: TF32 operands, 1: fp16.  MNA / MNB: operand read MN-major.
// ZLO (fp16 only): bit 0 / bit 1 = the lo plane of operand A / B is identically zero (a 0/1
// sample at an exact scale), so its product is skipped: two wgmma per half instead of three.  The
// skipped product adds exact zeros, so the result is bit-identical to the three-product order.
template <int KIND, int RB, int MNA, int MNB, int ZLO = 0>
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
        if (!(ZLO & 1)) wgmma_f16<MNA, MNB>(d[mh], a_lo, b_hi);
        if (!(ZLO & 2)) wgmma_f16<MNA, MNB>(d[mh], a_hi, b_lo);
        wgmma_f16<MNA, MNB>(d[mh], a_hi, b_hi);
      }
    }
  }
}

// The persistent warp-specialised kernel.  W describes one product:
//   KIND, RB, MNA, MNB            compile-time shape
//   units(), kb_range(u, kb0, kb1)
//   load(u, kb, stage_addr, bar)  the TMA loads of one stage (W::TX bytes)
//   EpiState, epilogue(u, acc_row_addr, quarter, lane, st), epi_finish(st, quarter, lane)
//   CLUSTER (optional, default 1)  CTAs per cluster; units() is then a multiple of it, and unit u
//                                 runs on cluster CTA u % CLUSTER
template <class W, class = void>
struct ClusterOf {
  static constexpr int value = 1;
};
template <class W>
struct ClusterOf<W, decltype((void)W::CLUSTER)> {
  static constexpr int value = W::CLUSTER;
};

// ZLO (optional, default 0)      operands whose lo plane is zero (mma_kblock); W::load then
//                                 skips those planes and W::TX counts only what it loads
template <class W, class = void>
struct ZloOf {
  static constexpr int value = 0;
};
template <class W>
struct ZloOf<W, decltype((void)W::ZLO)> {
  static constexpr int value = W::ZLO;
};

// The MMA warpgroup's accumulator d into the shared-memory tile the epilogue reads: stored, or
// (add) added to what the tile holds.  Each thread touches only its own elements.
__device__ __forceinline__ void acc_tile_write(uint32_t acc_base, int tid, const float (&d)[2][64],
                                               bool add) {
  const int row = 16 * (tid >> 5) + ((tid & 31) >> 2);
  const int col = 2 * (tid & 3);
#pragma unroll
  for (int mh = 0; mh < 2; ++mh)
#pragma unroll
    for (int j = 0; j < 16; ++j) {
      const uint32_t a0 = acc_base + (uint32_t)(((64 * mh + row) * ACC_LD + 8 * j + col) * 4);
      float v0 = d[mh][4 * j], v1 = d[mh][4 * j + 1], v2 = d[mh][4 * j + 2], v3 = d[mh][4 * j + 3];
      if (add) {
        float p0, p1, p2, p3;
        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(p0), "=f"(p1) : "r"(a0) : "memory");
        asm volatile("ld.shared.v2.f32 {%0, %1}, [%2];" : "=f"(p2), "=f"(p3)
                     : "r"(a0 + 8u * ACC_LD * 4u) : "memory");
        v0 += p0; v1 += p1; v2 += p2; v3 += p3;
      }
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a0), "f"(v0), "f"(v1) : "memory");
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(a0 + 8u * ACC_LD * 4u), "f"(v2),
                   "f"(v3) : "memory");
    }
}

// PROMOTE_KB (optional, default 0)  every PROMOTE_KB k-blocks of a unit the MMA warpgroup adds
//                                 its wgmma accumulator into the unit's tile in shared memory
//                                 (fp32 adds, rounded to nearest) and restarts it from zero.  The
//                                 tensor core's own fp32 accumulation does not round to nearest:
//                                 on partial sums of one sign it drifts toward zero by about 6 u
//                                 per k-block (H100), which over the hundreds of k-blocks of a
//                                 long contraction grows far past an fp32 sum's error.  The unit
//                                 then waits for the epilogue to drain the tile before its
//                                 mainloop instead of after it.
template <class W, class = void>
struct PromoteOf {
  static constexpr int value = 0;
};
template <class W>
struct PromoteOf<W, decltype((void)W::PROMOTE_KB)> {
  static constexpr int value = W::PROMOTE_KB;
};

template <class W>
__global__ void __launch_bounds__(NUM_THREADS, 1) tc_pipeline_kernel(const __grid_constant__ W w) {
  using C = Cfg<W::RB>;
  constexpr int CS = ClusterOf<W>::value;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t smem_base = (smem_u32(smem_raw) + (C::ALIGN - 1)) & ~(uint32_t)(C::ALIGN - 1);
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
      mbar_init(empty_bar + 8 * s, CS);
    }
    mbar_init(tfull_bar, 128);
    mbar_init(tempty_bar, 32 * NUM_EPI_WARPS);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  // peers multicast into this CTA's stages and arrive on its empty barriers: not before they exist
  if constexpr (CS > 1)
    cluster_sync();
  else
    __syncthreads();
  // the MMA warpgroup's release of a stage: one arrival on its empty barrier in every CTA of the
  // cluster (each of them may write into this CTA's copy of the stage)
  auto release = [&](int s) {
    if constexpr (CS > 1) {
#pragma unroll
      for (int r = 0; r < CS; ++r) mbar_arrive_cluster(empty_bar + 8 * s, (uint32_t)r);
    } else {
      mbar_arrive(empty_bar + 8 * s);
    }
  };

  if (warp < 4) {
    // ===================== MMA warpgroup =====================
    const int tid = threadIdx.x;
    float d[2][64];
    int stage = 0;
    uint32_t phase = 0, acc_phase = 0;
    const long long t_begin = prof_clock();
    long long t_full = 0, t_tempty = 0, t_store = 0, units = 0;
    for (int64_t u = blockIdx.x; u < n_units; u += gridDim.x) {
      int kb0, kb1;
      w.kb_range(u, kb0, kb1);
#pragma unroll
      for (int mh = 0; mh < 2; ++mh)
#pragma unroll
        for (int i = 0; i < 64; ++i) d[mh][i] = 0.f;
      int prev = -1;
      [[maybe_unused]] int since = 0;
      [[maybe_unused]] bool in_tile = false;            // the tile holds a promoted partial sum
      if constexpr (PromoteOf<W>::value > 0) {
        const long long t1 = prof_clock();
        mbar_wait(tempty_bar, acc_phase ^ 1);          // epilogue drained the previous unit
        t_tempty += prof_clock() - t1;
      }
      for (int kb = kb0; kb < kb1; ++kb) {
        const uint32_t sa = smem_base + stage * C::STAGE;
        const long long t0 = prof_clock();
        mbar_spin(full_bar + 8 * stage, phase);
        t_full += prof_clock() - t0;
        wgmma_fence();
        mma_kblock<W::KIND, W::RB, W::MNA, W::MNB, ZloOf<W>::value>(d, sa);
        wgmma_commit();
        wgmma_wait<1>();                                  // the previous stage has been read
        if (prev >= 0 && tid == 0) release(prev);
        prev = stage;
        if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        if constexpr (PromoteOf<W>::value > 0) {
          if (++since == PromoteOf<W>::value && kb + 1 < kb1) {
            wgmma_wait<0>();
            if (tid == 0) release(prev);
            prev = -1;
            acc_tile_write(acc_base, tid, d, in_tile);
            in_tile = true;
            since = 0;
#pragma unroll
            for (int mh = 0; mh < 2; ++mh)
#pragma unroll
              for (int i = 0; i < 64; ++i) d[mh][i] = 0.f;
          }
        }
      }
      wgmma_wait<0>();
      if (prev >= 0 && tid == 0) release(prev);
      const long long t1 = prof_clock();
      if constexpr (PromoteOf<W>::value == 0)
        mbar_wait(tempty_bar, acc_phase ^ 1);         // epilogue drained the previous unit
      const long long t2 = prof_clock();
      t_tempty += t2 - t1;
      acc_tile_write(acc_base, tid, d, in_tile);
      mbar_arrive(tfull_bar);
      acc_phase ^= 1;
      t_store += prof_clock() - t2;
      ++units;
    }
    if (kPassProfile && tid == 0) {
      prof_add(PROF_MMA_TOTAL, prof_clock() - t_begin);
      prof_add(PROF_MMA_FULL, t_full);
      prof_add(PROF_MMA_TEMPTY, t_tempty);
      prof_add(PROF_MMA_STORE, t_store);
      prof_add(PROF_UNITS, units);
    }
  } else if (warp == PRODUCER_WARP) {
    // ===================== TMA producer =====================
    if (lane == 0) {
      w.prefetch();
      int stage = 0;
      uint32_t phase = 0;
      long long t_empty = 0;
      for (int64_t u = blockIdx.x; u < n_units; u += gridDim.x) {
        int kb0, kb1;
        w.kb_range(u, kb0, kb1);
        for (int kb = kb0; kb < kb1; ++kb) {
          const long long t0 = prof_clock();
          mbar_wait(empty_bar + 8 * stage, phase ^ 1);
          t_empty += prof_clock() - t0;
          const uint32_t fb = full_bar + 8 * stage;
          mbar_expect_tx(fb, W::TX);
          w.load(u, kb, smem_base + stage * C::STAGE, fb);
          if (++stage == C::STAGES) { stage = 0; phase ^= 1; }
        }
      }
      if (kPassProfile) prof_add(PROF_PROD_EMPTY, t_empty);
    }
  } else {
    // ===================== epilogue =====================
    const int quarter = warp - EPI_WARP0;
    const uint32_t trow = acc_base + (uint32_t)((quarter * 32 + lane) * ACC_LD * 4);
    typename W::EpiState st;
    uint32_t acc_phase = 0;
    long long t_tfull = 0, t_unit = 0;
    for (int64_t u = blockIdx.x; u < n_units; u += gridDim.x) {
      const long long t0 = prof_clock();
      mbar_wait(tfull_bar, acc_phase);
      const long long t1 = prof_clock();
      w.epilogue(u, trow, quarter, lane, st);
      __syncwarp();
      mbar_arrive(tempty_bar);
      acc_phase ^= 1;
      t_tfull += t1 - t0;
      t_unit += prof_clock() - t1;
    }
    if (kPassProfile && quarter == 0 && lane == 0) {
      prof_add(PROF_EPI_TFULL, t_tfull);
      prof_add(PROF_EPI_UNIT, t_unit);
    }
    w.epi_finish(st, quarter, lane);
  }
  // no CTA leaves while a peer may still multicast into its shared memory or arrive on its barriers
  if constexpr (CS > 1) cluster_sync();
}

// one launch of tc_pipeline_kernel<W>: opt in to the dynamic shared memory once, one CTA per SM
// (with clusters: as many whole clusters as fit at once, which need not cover every SM)
template <class W>
int tc_launch(const W& w, cudaStream_t st, const char* what) {
  constexpr int CS = ClusterOf<W>::value;
  static const cudaError_t attr = cudaFuncSetAttribute(
      tc_pipeline_kernel<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg<W::RB>::SMEM);
  if (attr != cudaSuccess) {
    zsb_set_error("%s: cudaFuncSetAttribute: %s", what, cudaGetErrorString(attr));
    return ZSB_ERR_CUDA;
  }
  if constexpr (CS > 1) {
    const int64_t units = w.units();
    if (units < 1 || units % CS != 0) {
      zsb_set_error("%s: %lld units do not tile by clusters of %d", what, (long long)units, CS);
      return ZSB_ERR_INVALID;
    }
    cudaLaunchAttribute cl[1];
    cl[0].id = cudaLaunchAttributeClusterDimension;
    cl[0].val.clusterDim.x = CS;
    cl[0].val.clusterDim.y = 1;
    cl[0].val.clusterDim.z = 1;
    cudaLaunchConfig_t cfg = {};
    cfg.blockDim = dim3(NUM_THREADS);
    cfg.dynamicSmemBytes = Cfg<W::RB>::SMEM;
    cfg.stream = st;
    cfg.attrs = cl;
    cfg.numAttrs = 1;
    static int max_clusters = 0;
    if (max_clusters < 1) {
      cfg.gridDim = dim3(CS);
      const cudaError_t e =
          cudaOccupancyMaxActiveClusters(&max_clusters, tc_pipeline_kernel<W>, &cfg);
      if (e != cudaSuccess || max_clusters < 1) {
        zsb_set_error("%s: no cluster of %d CTAs fits (%s)", what, CS, cudaGetErrorString(e));
        max_clusters = 0;
        return ZSB_ERR_CUDA;
      }
    }
    int64_t grid = (int64_t)max_clusters * CS;
    if (grid > units) grid = units;
    cfg.gridDim = dim3((unsigned)grid);
    const cudaError_t e = cudaLaunchKernelEx(&cfg, tc_pipeline_kernel<W>, w);
    if (e != cudaSuccess) {
      zsb_set_error("%s: cudaLaunchKernelEx: %s", what, cudaGetErrorString(e));
      return ZSB_ERR_CUDA;
    }
    return zsb_check_launch(what);
  } else {
    int dev = 0, sms = ZSB_NUM_SMS;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int64_t grid = w.units();
    if (grid > sms) grid = sms;
    if (grid < 1) grid = 1;
    tc_pipeline_kernel<W><<<(unsigned)grid, NUM_THREADS, Cfg<W::RB>::SMEM, st>>>(w);
    return zsb_check_launch(what);
  }
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
