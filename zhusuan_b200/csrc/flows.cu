// Planar normalizing flows (zhusuan/transform.py:70-198): a stack of n flows applied along the last
// axis of [R, d] samples in one launch, and its gradient in one sweep plus one small merge.
//
// Flow k (transform.py:148-194), parameters b [n], aux_u [n, d], w [n, d]:
//     u_k   = aux_u_k + w_k / (w_k.w_k) * (softplus(w_k.aux_u_k) - 1 - w_k.aux_u_k)   (:161-164)
//     psi_k = u_k.w_k = softplus(w_k.aux_u_k) - 1 > -1                                 (:173)
//     a     = tanh(z.w_k + b_k),  log_q -= log(1 + psi_k (1 - a^2)),  z += a u_k       (:184-194)
// The softplus is the stable max(t, 0) + log1p(exp(-|t|)); the reference's log(exp(t) + 1) is inf
// for t > 88.  psi > -1 holds by construction, so there is no run-time invertibility assert.
//
// Mapping: a row is held by L lanes (1, 8 or 32 by d), each lane owning E elements j = l + L e, so
// z stays in registers across every flow and z.w is a sub-warp butterfly sum.  Each CTA first
// computes the per-flow scalars (the coefficient of w in u, psi and b) into shared memory, one warp
// per flow, for up to NF_CHUNK flows at a time; u_k is then formed on the fly from aux_u_k and w_k,
// which every row reads through L1.
//
// Backward: when a gradient is needed the forward pass also stores each flow's input z_{k-1}
// ([n, R, d]).  The reverse sweep recomputes a from it with the same instructions, so it sees
// exactly the forward's a, and no z_{k-1} is rebuilt as z_k - a u_k.  Per flow it gives
//     ga = u.gz + 2 g_lq psi a / det,  gs = ga (1 - a^2),  gz_{k-1} = gz_k + gs w
//     d u_k += a gz_k,  d w_k += gs z_{k-1},  d b_k += gs,  d psi_k += -g_lq (1 - a^2) / det
// summed over the rows of a warp with shuffles and accumulated into a slice of `part` that only
// that warp touches.  The merge sums the slices in warp order, adds psi's terms (d u += d psi w,
// d w += d psi u) and maps (d u, d w) through the reparameterisation to (d aux_u, d w).  No
// floating-point atomics: two identical calls give identical bits.
#include "common.cuh"

namespace {

constexpr int NF_THREADS = 256;
constexpr int NF_WARPS = NF_THREADS / 32;
constexpr int NF_CHUNK = 1024;                 // flows whose scalars sit in shared memory at once
constexpr int NF_MAX_D = 1024;
constexpr int NF_MAX_CTAS = 2 * ZSB_NUM_SMS;   // backward sweep: persistent CTAs
constexpr int64_t NF_PART_BUDGET = 1 << 23;    // floats of per-warp partials the sweep aims for

struct FlowScalars {
  float c[NF_CHUNK];     // coefficient of w_k in u_k
  float psi[NF_CHUNK];
  float b[NF_CHUNK];
};

__device__ __forceinline__ float softplus_(float t) {
  return fmaxf(t, 0.f) + log1pf(expf(-fabsf(t)));
}

// t = w.aux_u and ww = w.w of one flow, summed by one warp (valid in every lane)
__device__ __forceinline__ void flow_dots(const float* __restrict__ w,
                                          const float* __restrict__ aux, int d, float& t,
                                          float& ww) {
  float a = 0.f, q = 0.f;
  for (int j = threadIdx.x & 31; j < d; j += 32) {
    const float wj = w[j];
    a = fmaf(wj, aux[j], a);
    q = fmaf(wj, wj, q);
  }
  t = warp_sum(a);
  ww = warp_sum(q);
}

__device__ __forceinline__ void stage_scalars(FlowScalars& s, const float* __restrict__ b,
                                              const float* __restrict__ aux,
                                              const float* __restrict__ w, int d, int k0,
                                              int nk) {
  for (int i = threadIdx.x >> 5; i < nk; i += NF_WARPS) {
    const int64_t k = k0 + i;
    float t, ww;
    flow_dots(w + k * d, aux + k * d, d, t, ww);
    if ((threadIdx.x & 31) == 0) {
      const float sp = softplus_(t);
      s.c[i] = (sp - 1.f - t) / ww;
      s.psi[i] = sp - 1.f;
      s.b[i] = b[k];
    }
  }
}

// a = tanh(z.w + b) of one row held by L lanes; the forward and the backward sweep share it, so
// the backward pass sees the forward's a bit for bit.
template <int L, int E>
__device__ __forceinline__ float flow_act(const float (&z)[E], const float (&wv)[E], float b) {
  float dot = 0.f;
#pragma unroll
  for (int e = 0; e < E; ++e) dot = fmaf(z[e], wv[e], dot);
  return tanhf(sub_warp_sum<L>(dot) + b);
}

template <int L, int E>
__device__ __forceinline__ void load_w(float (&wv)[E], const float* __restrict__ wk, int l, int d) {
#pragma unroll
  for (int e = 0; e < E; ++e) {
    const int j = l + L * e;
    wv[e] = j < d ? __ldg(wk + j) : 0.f;
  }
}

template <int L, int E>
__global__ void __launch_bounds__(NF_THREADS) planar_flow_fwd_kernel(
    const float* __restrict__ z_in, const float* __restrict__ lq_in, const float* __restrict__ b,
    const float* __restrict__ aux, const float* __restrict__ w, float* __restrict__ z_out,
    float* __restrict__ lq_out, float* __restrict__ ck, int64_t R, int d, int n) {
  __shared__ FlowScalars s;
  const int g = threadIdx.x / L, l = threadIdx.x % L;
  const int64_t row = (int64_t)blockIdx.x * (NF_THREADS / L) + g;
  const bool ok = row < R;
  float z[E];
#pragma unroll
  for (int e = 0; e < E; ++e) {
    const int j = l + L * e;
    z[e] = (ok && j < d) ? z_in[row * d + j] : 0.f;
  }
  float lq = ok ? lq_in[row] : 0.f;
  for (int k0 = 0; k0 < n; k0 += NF_CHUNK) {
    const int nk = min(NF_CHUNK, n - k0);
    __syncthreads();
    stage_scalars(s, b, aux, w, d, k0, nk);
    __syncthreads();
    for (int i = 0; i < nk; ++i) {
      const int64_t k = k0 + i;
      const float* __restrict__ ak = aux + k * d;
      float wv[E];
      load_w<L, E>(wv, w + k * d, l, d);
      if (ck != nullptr && ok) {
#pragma unroll
        for (int e = 0; e < E; ++e)
          if (l + L * e < d) ck[(k * R + row) * d + l + L * e] = z[e];
      }
      const float a = flow_act<L, E>(z, wv, s.b[i]);
      lq -= log1pf(s.psi[i] * fmaf(-a, a, 1.f));
      const float c = s.c[i];
#pragma unroll
      for (int e = 0; e < E; ++e) {
        const int j = l + L * e;
        const float u = j < d ? fmaf(c, wv[e], __ldg(ak + j)) : 0.f;
        z[e] = fmaf(a, u, z[e]);
      }
    }
  }
  if (ok) {
#pragma unroll
    for (int e = 0; e < E; ++e)
      if (l + L * e < d) z_out[row * d + l + L * e] = z[e];
    if (l == 0) lq_out[row] = lq;
  }
}

// sum over the rows of a warp: lanes with the same position l inside their row
template <int L>
__device__ __forceinline__ float rows_sum(float v) {
#pragma unroll
  for (int o = L; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <int L, int E>
__global__ void __launch_bounds__(NF_THREADS) planar_flow_bwd_kernel(
    const float* __restrict__ ck, const float* __restrict__ gz_out,
    const float* __restrict__ glq, const float* __restrict__ b, const float* __restrict__ aux,
    const float* __restrict__ w, float* __restrict__ gz_in, float* __restrict__ part, int64_t R,
    int d, int n, int64_t n_tiles) {
  __shared__ FlowScalars s;
  const int g = threadIdx.x / L, l = threadIdx.x % L, lane = threadIdx.x & 31;
  const int64_t pstride = 2 * (int64_t)d + 2;
  float* __restrict__ pw =
      part + ((int64_t)blockIdx.x * NF_WARPS + (threadIdx.x >> 5)) * n * pstride;
  const bool one_chunk = n <= NF_CHUNK;
  if (one_chunk) {
    stage_scalars(s, b, aux, w, d, 0, n);
    __syncthreads();
  }
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const bool first = tile == blockIdx.x;
    const int64_t row = tile * (NF_THREADS / L) + g;
    const bool ok = row < R;
    float gz[E];
#pragma unroll
    for (int e = 0; e < E; ++e) {
      const int j = l + L * e;
      gz[e] = (ok && j < d) ? gz_out[row * d + j] : 0.f;
    }
    const float gl = ok ? glq[row] : 0.f;
    for (int k0 = ((n - 1) / NF_CHUNK) * NF_CHUNK; k0 >= 0; k0 -= NF_CHUNK) {
      const int nk = min(NF_CHUNK, n - k0);
      if (!one_chunk) {
        __syncthreads();
        stage_scalars(s, b, aux, w, d, k0, nk);
        __syncthreads();
      }
      for (int i = nk - 1; i >= 0; --i) {
        const int64_t k = k0 + i;
        const float* __restrict__ ak = aux + k * d;
        float zp[E], wv[E];
        load_w<L, E>(wv, w + k * d, l, d);
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int j = l + L * e;
          zp[e] = (ok && j < d) ? ck[(k * R + row) * d + j] : 0.f;
        }
        const float a = flow_act<L, E>(zp, wv, s.b[i]);
        const float om = fmaf(-a, a, 1.f);
        const float psi = s.psi[i], c = s.c[i];
        const float det = fmaf(psi, om, 1.f);
        float ug = 0.f;
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int j = l + L * e;
          const float u = j < d ? fmaf(c, wv[e], __ldg(ak + j)) : 0.f;
          ug = fmaf(u, gz[e], ug);
        }
        ug = sub_warp_sum<L>(ug);
        const float gs = ok ? (ug + 2.f * gl * psi * a / det) * om : 0.f;
        const float gpsi = ok ? -gl * om / det : 0.f;
        float* __restrict__ pk = pw + k * pstride;
#pragma unroll
        for (int e = 0; e < E; ++e) {
          const int j = l + L * e;
          const float du = rows_sum<L>(a * gz[e]);
          const float dw = rows_sum<L>(gs * zp[e]);
          if (lane < L && j < d) {
            pk[j] = first ? du : pk[j] + du;
            pk[d + j] = first ? dw : pk[d + j] + dw;
          }
          gz[e] = fmaf(gs, wv[e], gz[e]);
        }
        // gs and gpsi are equal in the L lanes of a row: sum one lane per row
        const float db = rows_sum<L>(l == 0 ? gs : 0.f);
        const float dpsi = rows_sum<L>(l == 0 ? gpsi : 0.f);
        if (lane == 0) {
          pk[2 * d] = first ? db : pk[2 * d] + db;
          pk[2 * d + 1] = first ? dpsi : pk[2 * d + 1] + dpsi;
        }
      }
    }
    if (ok) {
#pragma unroll
      for (int e = 0; e < E; ++e)
        if (l + L * e < d) gz_in[row * d + l + L * e] = gz[e];
    }
  }
}

// One CTA per flow: sum the warps' partials in order, then map (d u, d w) to (d aux_u, d w).
__global__ void __launch_bounds__(NF_THREADS) planar_flow_merge_kernel(
    const float* __restrict__ part, int64_t n_warps, const float* __restrict__ aux,
    const float* __restrict__ w, float* __restrict__ db, float* __restrict__ daux,
    float* __restrict__ dw, int d, int n) {
  __shared__ float sum[2 * NF_MAX_D + 2];
  __shared__ float red[32];
  __shared__ float sc[2];
  const int64_t k = blockIdx.x, pstride = 2 * (int64_t)d + 2;
  const float* __restrict__ wk = w + k * d;
  const float* __restrict__ ak = aux + k * d;
  if (threadIdx.x < 32) {
    float t, ww;
    flow_dots(wk, ak, d, t, ww);
    if (threadIdx.x == 0) { sc[0] = t; sc[1] = ww; }
  }
  // Column j of the warps' slices: with few columns the threads split the slices into `groups`
  // interleaved sets (loads coalesced over j), summed in set order afterwards.
  const int cols = (int)pstride;
  const int groups = cols >= NF_THREADS ? 1 : NF_THREADS / cols;
  for (int t = threadIdx.x; t < cols * groups; t += blockDim.x) {
    const int j = t % cols, s = t / cols;
    float v = 0.f;
#pragma unroll 8
    for (int64_t q = s; q < n_warps; q += groups) v += part[(q * n + k) * pstride + j];
    sum[t] = v;
  }
  __syncthreads();
  if (groups > 1) {
    const int j = threadIdx.x;          // cols < NF_THREADS here
    float v = 0.f;
    if (j < cols) {
      v = sum[j];
      for (int s = 1; s < groups; ++s) v += sum[s * cols + j];
    }
    __syncthreads();
    if (j < cols) sum[j] = v;
    __syncthreads();
  }
  const float t = sc[0], ww = sc[1];
  const float sp = softplus_(t);
  const float c = (sp - 1.f - t) / ww;
  const float sig1 = 1.f / (1.f + expf(-t)) - 1.f;       // d softplus / dt - 1
  const float dpsi = sum[2 * d + 1];
  float G = 0.f;
  for (int j = threadIdx.x; j < d; j += blockDim.x)
    G = fmaf(fmaf(dpsi, wk[j], sum[j]), wk[j], G);
  G = block_sum(G, red);                                  // (d u).w
  for (int j = threadIdx.x; j < d; j += blockDim.x) {
    const float wj = wk[j], aj = ak[j];
    const float u = fmaf(c, wj, aj);
    const float Du = fmaf(dpsi, wj, sum[j]);
    const float Dw = fmaf(dpsi, u, sum[d + j]);
    daux[k * d + j] = Du + G * sig1 / ww * wj;
    dw[k * d + j] = Dw + c * Du + G * (sig1 * aj - 2.f * c * wj) / ww;
  }
  if (threadIdx.x == 0) db[k] = sum[2 * d];
}

struct NfShape {
  int L, E;
};

NfShape nf_shape(int64_t d) {
  const int L = d <= 8 ? 1 : (d <= 64 ? 8 : 32);
  const int e = (int)((d + L - 1) / L);
  // E = 5 serves d = 33-40 (8 lanes) and 129-160 (32 lanes); with one lane per row (d <= 8) it
  // spilled a register, so those rows take E = 8.
  const int E = e <= 2 ? e
                       : (e <= 4 ? 4 : ((e <= 5 && L > 1) ? 5 : (e <= 8 ? 8 : (e <= 16 ? 16 : 32))));
  return {L, E};
}

int64_t nf_tiles(int64_t R, int64_t d) { return zsb_ceil_div(R, NF_THREADS / nf_shape(d).L); }

int64_t nf_bwd_ctas(int64_t R, int64_t d, int64_t n) {
  const int64_t per_cta = (int64_t)NF_WARPS * n * (2 * d + 2);
  int64_t g = NF_PART_BUDGET / (per_cta > 0 ? per_cta : 1);
  g = g < 1 ? 1 : (g > NF_MAX_CTAS ? NF_MAX_CTAS : g);
  const int64_t t = nf_tiles(R, d);
  return t < g ? t : g;
}

#define ZSB_NF_DISPATCH(KERNEL, SHAPE, GRID, ...)                                               \
  switch ((SHAPE).L * 100 + (SHAPE).E) {                                                         \
    case 101: KERNEL<1, 1><<<GRID, NF_THREADS, 0, st>>>(__VA_ARGS__); break;                     \
    case 102: KERNEL<1, 2><<<GRID, NF_THREADS, 0, st>>>(__VA_ARGS__); break;                     \
    case 104: KERNEL<1, 4><<<GRID, NF_THREADS, 0, st>>>(__VA_ARGS__); break;                     \
    case 108: KERNEL<1, 8><<<GRID, NF_THREADS, 0, st>>>(__VA_ARGS__); break;                     \
    case 802: KERNEL<8, 2><<<GRID, NF_THREADS, 0, st>>>(__VA_ARGS__); break;                     \
    case 804: KERNEL<8, 4><<<GRID, NF_THREADS, 0, st>>>(__VA_ARGS__); break;                     \
    case 805: KERNEL<8, 5><<<GRID, NF_THREADS, 0, st>>>(__VA_ARGS__); break;                     \
    case 808: KERNEL<8, 8><<<GRID, NF_THREADS, 0, st>>>(__VA_ARGS__); break;                     \
    case 3204: KERNEL<32, 4><<<GRID, NF_THREADS, 0, st>>>(__VA_ARGS__); break;                   \
    case 3205: KERNEL<32, 5><<<GRID, NF_THREADS, 0, st>>>(__VA_ARGS__); break;                   \
    case 3208: KERNEL<32, 8><<<GRID, NF_THREADS, 0, st>>>(__VA_ARGS__); break;                   \
    case 3216: KERNEL<32, 16><<<GRID, NF_THREADS, 0, st>>>(__VA_ARGS__); break;                  \
    default: KERNEL<32, 32><<<GRID, NF_THREADS, 0, st>>>(__VA_ARGS__); break;                    \
  }

}  // namespace

extern "C" {

// Warps of the backward sweep (transform.py:170-194): `part` holds warps * n_iters * (2 d + 2).
int zsb_planar_flow_warps(int64_t R, int64_t d, int64_t n_iters) {
  if (R < 1 || d < 1 || n_iters < 1) return 0;
  return (int)(nf_bwd_ctas(R, d, n_iters) * NF_WARPS);
}

// Forward pass of a planar flow stack (transform.py:148-194).  See include/zsb200.h.
int zsb_planar_flow_fwd_f32(const float* z_in, const float* lq_in, const float* b,
                            const float* aux_u, const float* w, float* z_out, float* lq_out,
                            float* ck, int64_t R, int64_t d, int64_t n_iters, void* stream) {
  ZSB_REQUIRE(b && aux_u && w, "zsb_planar_flow_fwd_f32: null pointer");
  ZSB_REQUIRE(d >= 1 && d <= NF_MAX_D, "zsb_planar_flow_fwd_f32: d = %lld outside [1, %d]",
              (long long)d, NF_MAX_D);
  ZSB_REQUIRE(R >= 0 && n_iters >= 1 && n_iters < (1LL << 31),
              "zsb_planar_flow_fwd_f32: bad sizes (R %lld, n_iters %lld)", (long long)R,
              (long long)n_iters);
  if (R == 0) return ZSB_OK;           // empty rows: the buffers may be NULL
  ZSB_REQUIRE(z_in && lq_in && z_out && lq_out, "zsb_planar_flow_fwd_f32: null pointer");
  const NfShape sh = nf_shape(d);
  const int64_t tiles = nf_tiles(R, d);
  ZSB_REQUIRE(tiles < (1LL << 31), "zsb_planar_flow_fwd_f32: R = %lld too large", (long long)R);
  cudaStream_t st = (cudaStream_t)stream;
  ZSB_NF_DISPATCH(planar_flow_fwd_kernel, sh, (unsigned)tiles, z_in, lq_in, b, aux_u, w, z_out,
                  lq_out, ck, R, (int)d, (int)n_iters);
  return zsb_check_launch("planar_flow_fwd");
}

// Backward pass of the stack (transform.py:170-194 differentiated).  See include/zsb200.h.
int zsb_planar_flow_bwd_f32(const float* ck, const float* gz_out, const float* glq,
                            const float* b, const float* aux_u, const float* w, float* gz_in,
                            float* part, float* db, float* daux_u, float* dw, int64_t R,
                            int64_t d, int64_t n_iters, void* stream) {
  ZSB_REQUIRE(b && aux_u && w && db && daux_u && dw, "zsb_planar_flow_bwd_f32: null pointer");
  ZSB_REQUIRE(R == 0 || (ck && gz_out && glq && gz_in && part),
              "zsb_planar_flow_bwd_f32: null pointer");
  ZSB_REQUIRE(d >= 1 && d <= NF_MAX_D, "zsb_planar_flow_bwd_f32: d = %lld outside [1, %d]",
              (long long)d, NF_MAX_D);
  ZSB_REQUIRE(R >= 0 && n_iters >= 1 && n_iters < (1LL << 31) && nf_tiles(R, d) < (1LL << 31),
              "zsb_planar_flow_bwd_f32: bad sizes (R %lld, n_iters %lld)", (long long)R,
              (long long)n_iters);
  cudaStream_t st = (cudaStream_t)stream;
  int64_t n_warps = 0;
  if (R > 0) {
    const NfShape sh = nf_shape(d);
    const int64_t ctas = nf_bwd_ctas(R, d, n_iters);
    n_warps = ctas * NF_WARPS;
    ZSB_NF_DISPATCH(planar_flow_bwd_kernel, sh, (unsigned)ctas, ck, gz_out, glq, b, aux_u, w,
                    gz_in, part, R, (int)d, (int)n_iters, nf_tiles(R, d));
    const int rc = zsb_check_launch("planar_flow_bwd");
    if (rc != ZSB_OK) return rc;
  }
  planar_flow_merge_kernel<<<(unsigned)n_iters, NF_THREADS, 0, st>>>(part, n_warps, aux_u, w, db,
                                                                     daux_u, dw, (int)d,
                                                                     (int)n_iters);
  return zsb_check_launch("planar_flow_merge");
}

}  // extern "C"
