// Sparse-GP conditional moments (examples/gaussian_process/utils.py:52-90, full_cov=False) for an
// RBF kernel (utils.py:18-49), and their gradient.  Only the work that grows with the number of
// rows B is here; the M x M algebra (Cholesky factor, Li = L^-1, V = fz Li^T) stays with the caller.
//
// With Kxz[b, m] = exp(-sum_j (x_bj - z_mj)^2 / s_j / 2) and A = Kxz Li^T ([B, M]):
//     mean = V A^T  [K, B],   var = 1 - rowsum(A^2),   std = sqrt(var)          (utils.py:69-87)
// The reference forms Kzz_inv = Li^T Li and Kxz Kzz_inv; mean = V A^T is the same product
// re-associated, so the two differ only by rounding.  var is not clamped, as in the reference.
//
// Mapping: a CTA of 256 threads takes a tile of 64 rows.  Lane l holds rows l and l + 32; warp w
// holds columns w + 8c, c < NC (8 NC >= M).  The tile's x, then its Kxz (from distances computed on
// the fly), then its A live in shared memory: neither Kxz nor the [B, M, d] differences reach HBM.
// A skips the zero upper triangle of Li.  All products are FP32 FFMA.
//
// Backward: per row, with c_b = -g_std_b / std_b (= -2 g_var_b),
//     dA_b = sum_k g_mean[k, b] V_k + c_b A_b,   dKxz_b = Li^T dA_b,   G = dKxz o Kxz
//     dV += g_mean A,   dLi += tril(dA^T Kxz),   dz[m, j] += sum_b G (x - z)_bj,
//     ds_j += sum_{b, m} G (x - z)_bj^2
// Kxz is recomputed with the forward's instructions; A comes from the forward pass.  Each CTA of
// a persistent sweep adds its tiles' B-sums to its own slice of `part`; the merge sums the slices
// in CTA order and applies 1 / s_j and 1 / (2 s_j^2).  No floating-point atomics: two identical
// calls give identical bits.
#include "common.cuh"

namespace {

constexpr int GP_THREADS = 256;
constexpr int GP_WARPS = GP_THREADS / 32;
constexpr int GP_ROWS = 64;                     // rows per tile: lanes l and l + 32
constexpr int GP_MAX_M = 256;
constexpr int GP_MAX_D = 64;
constexpr int GP_KC = 32;                       // backward: g_mean rows staged at once
constexpr int64_t GP_PART_BUDGET = 1 << 23;     // floats of per-CTA partials the sweep aims for

struct GpLayout {
  int ms, ds;                // odd row strides of the M- and d-wide tiles (no bank conflicts)
  int xs, ks, as, gs, rs, red;
  int floats;
};

// Shared-memory layout of a tile; `bwd` adds the A / dA / G tile and the g_mean chunk.
__host__ __device__ inline GpLayout gp_layout(int nc, int d, bool bwd) {
  GpLayout L;
  L.ms = 8 * nc + 1;
  L.ds = d | 1;
  L.xs = 0;
  L.ks = L.xs + GP_ROWS * L.ds;
  L.as = L.ks + GP_ROWS * L.ms;
  L.gs = L.as + (bwd ? GP_ROWS * L.ms : 0);
  L.rs = L.gs + (bwd ? GP_KC * (GP_ROWS + 1) : 0);
  L.red = L.rs + GP_MAX_D;
  L.floats = L.red + GP_WARPS * GP_ROWS;
  return L;
}

// x rows [b0, b0 + nb) into xs, zero rows after them.
__device__ __forceinline__ void gp_load_x(float* __restrict__ xs, const float* __restrict__ x,
                                          int64_t b0, int nb, int d, int ds) {
  for (int t = threadIdx.x; t < GP_ROWS * d; t += GP_THREADS) {
    const int r = t / d, j = t - r * d;
    xs[r * ds + j] = r < nb ? x[b0 * d + t] : 0.f;
  }
}

// Kxz of the tile into ks (columns M .. 8 NC - 1 zero).  The forward pass and the backward sweep
// share it, so the backward pass sees the forward's Kxz bit for bit.
template <int NC>
__device__ __forceinline__ void gp_kxz(float* __restrict__ ks, const float* __restrict__ xs,
                                       const float* __restrict__ z, const float* __restrict__ rs,
                                       int M, int d, int ms, int ds) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll 1
  for (int c = 0; c < NC; ++c) {
    const int m = warp + 8 * c;
    float q0 = 0.f, q1 = 0.f;
    if (m < M) {
      for (int j = 0; j < d; ++j) {
        const float zj = __ldg(z + (int64_t)m * d + j), r = rs[j];
        const float t0 = xs[lane * ds + j] - zj, t1 = xs[(lane + 32) * ds + j] - zj;
        q0 = fmaf(t0 * t0, r, q0);
        q1 = fmaf(t1 * t1, r, q1);
      }
    }
    ks[lane * ms + m] = m < M ? expf(-0.5f * q0) : 0.f;
    ks[(lane + 32) * ms + m] = m < M ? expf(-0.5f * q1) : 0.f;
  }
}

template <int NC>
__global__ void __launch_bounds__(GP_THREADS) gp_cond_fwd_kernel(
    const float* __restrict__ x, const float* __restrict__ z, const float* __restrict__ s,
    const float* __restrict__ Li, const float* __restrict__ V, float* __restrict__ mean,
    float* __restrict__ stdv, float* __restrict__ A_out, int64_t B, int M, int d, int K) {
  extern __shared__ float sm[];
  const GpLayout L = gp_layout(NC, d, false);
  float* __restrict__ xs = sm + L.xs;
  float* __restrict__ ks = sm + L.ks;
  float* __restrict__ rs = sm + L.rs;
  float* __restrict__ red = sm + L.red;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, ms = L.ms;
  const int64_t b0 = (int64_t)blockIdx.x * GP_ROWS;
  const int nb = (int)min((int64_t)GP_ROWS, B - b0);
  gp_load_x(xs, x, b0, nb, d, L.ds);
  if (threadIdx.x < d) rs[threadIdx.x] = 1.f / s[threadIdx.x];
  __syncthreads();
  gp_kxz<NC>(ks, xs, z, rs, M, d, ms, L.ds);
  __syncthreads();

  // A[b, i] = sum_{m <= i} Kxz[b, m] Li[i, m]
  float acc[2][NC];
#pragma unroll
  for (int c = 0; c < NC; ++c) acc[0][c] = acc[1][c] = 0.f;
  for (int m = 0; m < M; ++m) {
    const float k0 = ks[lane * ms + m], k1 = ks[(lane + 32) * ms + m];
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const int i = warp + 8 * c;
      if (i >= m && i < M) {
        const float l = __ldg(Li + (int64_t)i * M + m);
        acc[0][c] = fmaf(k0, l, acc[0][c]);
        acc[1][c] = fmaf(k1, l, acc[1][c]);
      }
    }
  }
  __syncthreads();                             // every read of Kxz is done: A replaces it
  float p0 = 0.f, p1 = 0.f;
#pragma unroll
  for (int c = 0; c < NC; ++c) {
    const int i = warp + 8 * c;
    ks[lane * ms + i] = acc[0][c];
    ks[(lane + 32) * ms + i] = acc[1][c];
    p0 = fmaf(acc[0][c], acc[0][c], p0);
    p1 = fmaf(acc[1][c], acc[1][c], p1);
  }
  red[warp * GP_ROWS + lane] = p0;
  red[warp * GP_ROWS + lane + 32] = p1;
  __syncthreads();
  if (threadIdx.x < nb) {
    float v = 0.f;
#pragma unroll
    for (int w = 0; w < GP_WARPS; ++w) v += red[w * GP_ROWS + threadIdx.x];
    stdv[b0 + threadIdx.x] = sqrtf(1.f - v);
  }
  if (A_out != nullptr) {
    for (int t = threadIdx.x; t < nb * M; t += GP_THREADS) {
      const int r = t / M;
      A_out[b0 * M + t] = ks[r * ms + t - r * M];
    }
  }

  // mean[k, b] = sum_i V[k, i] A[b, i]: each warp takes 4 consecutive k at a time
  for (int k0 = 4 * warp; k0 < K; k0 += 4 * GP_WARPS) {
    const float* __restrict__ v[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) v[q] = V + (int64_t)min(k0 + q, K - 1) * M;
    float s0[4] = {0.f, 0.f, 0.f, 0.f}, s1[4] = {0.f, 0.f, 0.f, 0.f};
    for (int i = 0; i < M; ++i) {
      const float a0 = ks[lane * ms + i], a1 = ks[(lane + 32) * ms + i];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float vq = __ldg(v[q] + i);
        s0[q] = fmaf(vq, a0, s0[q]);
        s1[q] = fmaf(vq, a1, s1[q]);
      }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      if (k0 + q < K) {
        float* __restrict__ mk = mean + (int64_t)(k0 + q) * B + b0;
        if (lane < nb) mk[lane] = s0[q];
        if (lane + 32 < nb) mk[lane + 32] = s1[q];
      }
    }
  }
}

// Persistent sweep: CTA c takes tiles c, c + P, ... and adds their B-sums to its slice of `part`
// ([dV K*M | dLi M*M | dz M*d | ds d]); its first tile writes the slice.
template <int NC>
__global__ void __launch_bounds__(GP_THREADS, 1) gp_cond_bwd_kernel(
    const float* __restrict__ x, const float* __restrict__ z, const float* __restrict__ s,
    const float* __restrict__ Li, const float* __restrict__ V, const float* __restrict__ A,
    const float* __restrict__ stdv, const float* __restrict__ g_mean,
    const float* __restrict__ g_std, float* __restrict__ part, int64_t B, int M, int d, int K,
    int64_t n_tiles) {
  extern __shared__ float sm[];
  const GpLayout L = gp_layout(NC, d, true);
  float* __restrict__ xs = sm + L.xs;
  float* __restrict__ ks = sm + L.ks;
  float* __restrict__ as = sm + L.as;
  float* __restrict__ gs = sm + L.gs;
  float* __restrict__ rs = sm + L.rs;
  float* __restrict__ red = sm + L.red;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, ms = L.ms;
  constexpr int GST = GP_ROWS + 1;
  const int64_t T = (int64_t)K * M + (int64_t)M * M + (int64_t)M * d + d;
  float* __restrict__ pV = part + (int64_t)blockIdx.x * T;
  float* __restrict__ pL = pV + (int64_t)K * M;
  float* __restrict__ pZ = pL + (int64_t)M * M;
  float* __restrict__ pS = pZ + (int64_t)M * d;
  if (threadIdx.x < d) rs[threadIdx.x] = 1.f / s[threadIdx.x];
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const bool first = tile == blockIdx.x;
    const int64_t b0 = tile * GP_ROWS;
    const int nb = (int)min((int64_t)GP_ROWS, B - b0);
    __syncthreads();                           // the previous tile's reads are done
    gp_load_x(xs, x, b0, nb, d, L.ds);
    for (int t = threadIdx.x; t < GP_ROWS * (ms - 1); t += GP_THREADS) {
      const int r = t / (ms - 1), i = t - r * (ms - 1);
      as[r * ms + i] = (r < nb && i < M) ? A[(b0 + r) * M + i] : 0.f;
    }
    // red[r] = c_b = -g_std / std for the tile's rows (0 without g_std)
    if (threadIdx.x < GP_ROWS) {
      const int r = threadIdx.x;
      red[r] = (g_std != nullptr && r < nb) ? -g_std[b0 + r] / stdv[b0 + r] : 0.f;
    }
    __syncthreads();
    gp_kxz<NC>(ks, xs, z, rs, M, d, ms, L.ds);

    // dA = g_mean^T V + c A (registers), and dV += g_mean A, over chunks of GP_KC particles
    float acc[2][NC];
#pragma unroll
    for (int c = 0; c < NC; ++c) acc[0][c] = acc[1][c] = 0.f;
    if (g_mean != nullptr) {
      for (int kc = 0; kc < K; kc += GP_KC) {
        const int nk = min(GP_KC, K - kc);
        __syncthreads();
        for (int t = threadIdx.x; t < GP_KC * GP_ROWS; t += GP_THREADS) {
          const int kk = t / GP_ROWS, r = t - kk * GP_ROWS;
          gs[kk * GST + r] = (kk < nk && r < nb) ? g_mean[(int64_t)(kc + kk) * B + b0 + r] : 0.f;
        }
        __syncthreads();
        for (int kk = 0; kk < nk; ++kk) {
          const float g0 = gs[kk * GST + lane], g1 = gs[kk * GST + lane + 32];
          const float* __restrict__ vk = V + (int64_t)(kc + kk) * M;
#pragma unroll
          for (int c = 0; c < NC; ++c) {
            const int i = warp + 8 * c;
            if (i < M) {
              const float v = __ldg(vk + i);
              acc[0][c] = fmaf(g0, v, acc[0][c]);
              acc[1][c] = fmaf(g1, v, acc[1][c]);
            }
          }
        }
        for (int kk = warp; kk < nk; kk += GP_WARPS) {
          for (int i = lane; i < M; i += 32) {
            float v = 0.f;
#pragma unroll 8
            for (int r = 0; r < GP_ROWS; ++r) v = fmaf(gs[kk * GST + r], as[r * ms + i], v);
            float* __restrict__ p = pV + (int64_t)(kc + kk) * M + i;
            *p = first ? v : *p + v;
          }
        }
      }
    }
    __syncthreads();                           // every read of A is done: dA replaces it
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const int i = warp + 8 * c;
      float* __restrict__ a0 = as + lane * ms + i;
      float* __restrict__ a1 = as + (lane + 32) * ms + i;
      *a0 = fmaf(red[lane], *a0, acc[0][c]);
      *a1 = fmaf(red[lane + 32], *a1, acc[1][c]);
    }
    __syncthreads();

    // dLi[i, m] += sum_b dA[b, i] Kxz[b, m], m <= i
    for (int i = warp; i < M; i += GP_WARPS) {
      for (int m = lane; m <= i; m += 32) {
        float v = 0.f;
#pragma unroll 8
        for (int r = 0; r < GP_ROWS; ++r) v = fmaf(as[r * ms + i], ks[r * ms + m], v);
        float* __restrict__ p = pL + (int64_t)i * M + m;
        *p = first ? v : *p + v;
      }
    }

    // dKxz[b, m] = sum_{i >= m} dA[b, i] Li[i, m], then G = dKxz o Kxz
#pragma unroll
    for (int c = 0; c < NC; ++c) acc[0][c] = acc[1][c] = 0.f;
    for (int i = 0; i < M; ++i) {
      const float a0 = as[lane * ms + i], a1 = as[(lane + 32) * ms + i];
      const float* __restrict__ li = Li + (int64_t)i * M;
#pragma unroll
      for (int c = 0; c < NC; ++c) {
        const int m = warp + 8 * c;
        if (m <= i) {
          const float l = __ldg(li + m);
          acc[0][c] = fmaf(a0, l, acc[0][c]);
          acc[1][c] = fmaf(a1, l, acc[1][c]);
        }
      }
    }
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const int m = warp + 8 * c;
      acc[0][c] *= ks[lane * ms + m];
      acc[1][c] *= ks[(lane + 32) * ms + m];
    }
    __syncthreads();                           // every read of dA is done: G replaces it
#pragma unroll
    for (int c = 0; c < NC; ++c) {
      const int m = warp + 8 * c;
      as[lane * ms + m] = acc[0][c];
      as[(lane + 32) * ms + m] = acc[1][c];
    }
    __syncthreads();

    // dz[m, j] += sum_b G[b, m] (x_bj - z_mj);  ds_j += sum_{b, m} G[b, m] (x_bj - z_mj)^2
    float ds0 = 0.f, ds1 = 0.f;
    for (int m = warp; m < M; m += GP_WARPS) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int j = lane + 32 * h;
        if (j < d) {
          const float zj = __ldg(z + (int64_t)m * d + j);
          float v = 0.f, w = 0.f;
#pragma unroll 8
          for (int r = 0; r < GP_ROWS; ++r) {
            const float t = xs[r * L.ds + j] - zj;
            const float gt = as[r * ms + m] * t;
            v += gt;
            w = fmaf(gt, t, w);
          }
          float* __restrict__ p = pZ + (int64_t)m * d + j;
          *p = first ? v : *p + v;
          if (h == 0) ds0 += w; else ds1 += w;
        }
      }
    }
    __syncthreads();                           // red (c_b) is read no more
    red[warp * GP_ROWS + lane] = ds0;
    red[warp * GP_ROWS + lane + 32] = ds1;
    __syncthreads();
    if (threadIdx.x < d) {
      float v = 0.f;
#pragma unroll
      for (int w = 0; w < GP_WARPS; ++w) v += red[w * GP_ROWS + threadIdx.x];
      pS[threadIdx.x] = first ? v : pS[threadIdx.x] + v;
    }
  }
}

// Sum the P slices in CTA order; dz and ds take the chain factors 1 / s_j and 1 / (2 s_j^2).
__global__ void __launch_bounds__(GP_THREADS) gp_cond_merge_kernel(
    const float* __restrict__ part, int64_t P, const float* __restrict__ s, int has_gm,
    float* __restrict__ dV, float* __restrict__ dLi, float* __restrict__ dz,
    float* __restrict__ ds, int M, int d, int K) {
  const int64_t oL = (int64_t)K * M, oZ = oL + (int64_t)M * M, oS = oZ + (int64_t)M * d;
  const int64_t T = oS + d;
  for (int64_t t = (int64_t)blockIdx.x * GP_THREADS + threadIdx.x; t < T;
       t += (int64_t)gridDim.x * GP_THREADS) {
    bool zero = false;
    if (t < oL) zero = !has_gm;
    else if (t < oZ) zero = (t - oL) % M > (t - oL) / M;       // upper triangle of dLi
    float v = 0.f;
    if (!zero) {
#pragma unroll 4
      for (int64_t p = 0; p < P; ++p) v += part[p * T + t];
    }
    if (t < oL) {
      dV[t] = v;
    } else if (t < oZ) {
      dLi[t - oL] = v;
    } else if (t < oS) {
      dz[t - oZ] = v / s[(t - oZ) % d];
    } else {
      const float sj = s[t - oS];
      ds[t - oS] = 0.5f * v / (sj * sj);
    }
  }
}

int gp_nc(int64_t M) { return M <= 64 ? 8 : (M <= 128 ? 16 : 32); }

int64_t gp_tiles(int64_t B) { return zsb_ceil_div(B, GP_ROWS); }

int64_t gp_slice(int64_t M, int64_t d, int64_t K) { return K * M + M * M + M * d + d; }

int64_t gp_bwd_ctas(int64_t B, int64_t M, int64_t d, int64_t K) {
  int64_t g = GP_PART_BUDGET / gp_slice(M, d, K);
  g = g < 1 ? 1 : (g > ZSB_NUM_SMS ? ZSB_NUM_SMS : g);
  const int64_t t = gp_tiles(B);
  return t < g ? t : g;
}

// The tiles need more than the default 48 KB of dynamic shared memory (up to 225 KB).
template <typename Kern>
int gp_allow_smem(Kern kernel, size_t smem, const char* what) {
  const cudaError_t e =
      cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (e != cudaSuccess) {
    zsb_set_error("%s: %s", what, cudaGetErrorString(e));
    return ZSB_ERR_CUDA;
  }
  return ZSB_OK;
}

#define ZSB_GP_LAUNCH(KERNEL, NC, GRID, SMEM, ...)                                               \
  do {                                                                                           \
    rc = gp_allow_smem(KERNEL<NC>, SMEM, #KERNEL);                                               \
    if (rc == ZSB_OK) KERNEL<NC><<<GRID, GP_THREADS, SMEM, st>>>(__VA_ARGS__);                   \
  } while (0)

#define ZSB_GP_DISPATCH(KERNEL, NC, GRID, SMEM, ...)                                             \
  switch (NC) {                                                                                  \
    case 8: ZSB_GP_LAUNCH(KERNEL, 8, GRID, SMEM, __VA_ARGS__); break;                            \
    case 16: ZSB_GP_LAUNCH(KERNEL, 16, GRID, SMEM, __VA_ARGS__); break;                          \
    default: ZSB_GP_LAUNCH(KERNEL, 32, GRID, SMEM, __VA_ARGS__); break;                          \
  }

}  // namespace

extern "C" {

// Slices of the backward sweep's `part` scratch (utils.py:52-90); each is K*M + M*M + M*d + d.
int zsb_gp_cond_parts(int64_t B, int64_t M, int64_t d, int64_t K) {
  if (B < 1 || M < 1 || M > GP_MAX_M || d < 1 || d > GP_MAX_D || K < 0) return 0;
  return (int)gp_bwd_ctas(B, M, d, K);
}

// Forward moments (utils.py:69-87, full_cov=False).  See include/zsb200.h.
int zsb_gp_cond_fwd_f32(const float* x, const float* z, const float* s, const float* Li,
                        const float* V, float* mean, float* stdv, float* A_out, int64_t B,
                        int64_t M, int64_t d, int64_t K, void* stream) {
  ZSB_REQUIRE(M >= 1 && M <= GP_MAX_M, "zsb_gp_cond_fwd_f32: M = %lld outside [1, %d]",
              (long long)M, GP_MAX_M);
  ZSB_REQUIRE(d >= 1 && d <= GP_MAX_D, "zsb_gp_cond_fwd_f32: d = %lld outside [1, %d]",
              (long long)d, GP_MAX_D);
  ZSB_REQUIRE(B >= 0 && K >= 0 && K < (1LL << 31) && gp_tiles(B) < (1LL << 31),
              "zsb_gp_cond_fwd_f32: bad sizes (B %lld, K %lld)", (long long)B, (long long)K);
  if (B == 0) return ZSB_OK;                   // empty rows: nothing to compute
  ZSB_REQUIRE(x && z && s && Li && stdv && (K == 0 || (V && mean)),
              "zsb_gp_cond_fwd_f32: null pointer");
  const int nc = gp_nc(M);
  const size_t smem = sizeof(float) * gp_layout(nc, (int)d, false).floats;
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ZSB_OK;
  ZSB_GP_DISPATCH(gp_cond_fwd_kernel, nc, (unsigned)gp_tiles(B), smem, x, z, s, Li, V, mean,
                  stdv, A_out, B, (int)M, (int)d, (int)K);
  if (rc != ZSB_OK) return rc;
  return zsb_check_launch("gp_cond_fwd");
}

// Backward of the moments, one sweep plus one merge launch.  See include/zsb200.h.
int zsb_gp_cond_bwd_f32(const float* x, const float* z, const float* s, const float* Li,
                        const float* V, const float* A, const float* stdv, const float* g_mean,
                        const float* g_std, float* part, float* dz, float* ds, float* dLi,
                        float* dV, int64_t B, int64_t M, int64_t d, int64_t K, void* stream) {
  ZSB_REQUIRE(M >= 1 && M <= GP_MAX_M, "zsb_gp_cond_bwd_f32: M = %lld outside [1, %d]",
              (long long)M, GP_MAX_M);
  ZSB_REQUIRE(d >= 1 && d <= GP_MAX_D, "zsb_gp_cond_bwd_f32: d = %lld outside [1, %d]",
              (long long)d, GP_MAX_D);
  ZSB_REQUIRE(B >= 0 && K >= 0 && K < (1LL << 31) && gp_tiles(B) < (1LL << 31),
              "zsb_gp_cond_bwd_f32: bad sizes (B %lld, K %lld)", (long long)B, (long long)K);
  if (B == 0) return ZSB_OK;                   // empty rows: the outputs are left untouched
  ZSB_REQUIRE(x && z && s && Li && A && stdv && part && dz && ds && dLi && (K == 0 || (V && dV)),
              "zsb_gp_cond_bwd_f32: null pointer");
  if (K == 0) g_mean = nullptr;
  const int nc = gp_nc(M);
  const size_t smem = sizeof(float) * gp_layout(nc, (int)d, true).floats;
  const int64_t ctas = gp_bwd_ctas(B, M, d, K);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = ZSB_OK;
  ZSB_GP_DISPATCH(gp_cond_bwd_kernel, nc, (unsigned)ctas, smem, x, z, s, Li, V, A, stdv, g_mean,
                  g_std, part, B, (int)M, (int)d, (int)K, gp_tiles(B));
  if (rc != ZSB_OK) return rc;
  rc = zsb_check_launch("gp_cond_bwd");
  if (rc != ZSB_OK) return rc;
  const int64_t T = gp_slice(M, d, K);
  const int64_t grid = zsb_ceil_div(T, GP_THREADS) < 4 * ZSB_NUM_SMS
                           ? zsb_ceil_div(T, GP_THREADS) : 4 * ZSB_NUM_SMS;
  gp_cond_merge_kernel<<<(unsigned)grid, GP_THREADS, 0, st>>>(
      part, ctas, s, g_mean != nullptr, dV, dLi, dz, ds, (int)M, (int)d, (int)K);
  return zsb_check_launch("gp_cond_merge");
}

}  // extern "C"
