// Inverse Autoregressive Flow with the linear autoregressive network (zhusuan/transform.py:17-67,
// :200-282): a stack of n flows applied along the last axis of [R, d] samples in one launch, and
// its gradient in one sweep plus one merge.
//
// Flow k, weights m_w [n, d, d], s_w [n, d, d], read only above the diagonal (mask[i][j] = i < j,
// transform.py:38-43, :55-56):
//     m_j = sum_{i<j} z_i m_w[k][i][j],  t_j = sum_{i<j} z_i s_w[k][i][j],  s = exp(t)   (:58-61)
//     normal: z = s z + m,                   log_q -= sum_j t_j                        (:271-273)
//     gru:    g = sigmoid(s), z = g z + (1 - g) m,  log_q -= sum_j log g_j            (:266-269)
//     z = reverse(z)                                                                    (:275)
// log s is t itself, not log(exp(t)), and log sigmoid(s) = -softplus(-s) = -log1p(exp(-s)) (s > 0),
// which stays finite where the reference's log(sigmoid(s)) would round sigmoid to 1 or 0.
//
// Mapping: a CTA holds a tile of TR rows in shared memory across every flow.  Per flow it walks
// the columns in blocks of CB, from the last block to the first, and streams the two weight
// triangles through shared memory in chunks of IC rows; chunks wholly below the diagonal are never
// loaded.  Each thread accumulates an RM x 4 tile of both m and t.  A column block only reads
// z_i for i < j, which the blocks still to come never change, so the update is written in place.
// The reversal is an index flip: after an odd number of flows logical element j of a row sits at
// physical position d-1-j.  The log-determinant terms stay in registers until the last flow.
//
// Backward: when a gradient is needed the forward pass stores each flow's input z ([n, R, d]).  The
// persistent sweep takes a tile of rows through the flows in reverse order: it recomputes m and t
// from the stored input with the same instructions (so it sees the forward's values exactly), forms
//     normal: g_m = gz,  g_t = gz z s - g_lq,                    direct = gz s
//     gru:    g_m = gz (1 - g),  g_t = (gz (z - m) g - g_lq)(1 - g) s,  direct = gz g
// and the input gradient gz_i = direct_i + sum_{j>i} (m_w[i][j] g_m_j + s_w[i][j] g_t_j).  The
// weight gradients Z^T g_m and Z^T g_t (upper triangles) of its tile are added into a slice of
// `part` that only this CTA touches.  The merge sums the slices in CTA order.  No floating-point
// atomics: two identical calls give identical bits.
#include "common.cuh"

namespace {

constexpr int IAF_THREADS = 256;
constexpr int IAF_IC = 16;                      // weight rows (or columns) per streamed chunk
constexpr int IAF_MAX_D = 256;
constexpr int IAF_MAX_CTAS = 2 * ZSB_NUM_SMS;   // backward sweep: persistent CTAs
constexpr int64_t IAF_PART_BUDGET = 1 << 27;    // floats of per-CTA weight-gradient slices

// Tile geometry for CGS column groups of 4 columns and RM rows per thread.
template <int CGS, int RM>
struct Geo {
  static constexpr int CB = 4 * CGS;                    // columns per block
  static constexpr int RG = IAF_THREADS / CGS;          // row groups
  static constexpr int TR = RG * RM;                    // rows per tile
  static constexpr int DMAX = CGS == 4 ? 16 : (CGS == 8 ? 64 : 256);
  static constexpr int LD = DMAX + 1;                   // odd row stride: rows fall in different banks
};

// m and t of column block [j0, j0 + CB) for the thread's RM rows and 4 columns, from a tile zs
// (row stride LD; logical element i at physical i, or d-1-i when `flip`).  Starts and ends with
// every thread past a barrier that follows its last read of the weight buffers.  The sum over i
// runs from 0 upwards with fmaf whatever the tile geometry, so the forward and the backward sweep
// compute the same m and t bit for bit.
template <int CGS, int RM>
__device__ __forceinline__ void mt_block(const float* __restrict__ zs, bool flip, int d, int j0,
                                         const float* __restrict__ mwk,
                                         const float* __restrict__ swk, float* __restrict__ wm,
                                         float* __restrict__ wt, int rg, int cg,
                                         float (&am)[RM][4], float (&at)[RM][4]) {
  using G = Geo<CGS, RM>;
#pragma unroll
  for (int q = 0; q < RM; ++q)
#pragma unroll
    for (int c = 0; c < 4; ++c) am[q][c] = at[q][c] = 0.f;
  const int iend = min(j0 + G::CB, d);                  // i < j <= j0 + CB - 1
  for (int i0 = 0; i0 < iend; i0 += IAF_IC) {
    __syncthreads();
    for (int e = threadIdx.x; e < IAF_IC * G::CB; e += IAF_THREADS) {
      const int i = i0 + e / G::CB, j = j0 + e % G::CB;
      const bool on = i < j && j < d;
      wm[e] = on ? __ldg(mwk + (int64_t)i * d + j) : 0.f;
      wt[e] = on ? __ldg(swk + (int64_t)i * d + j) : 0.f;
    }
    __syncthreads();
    const int ni = min(IAF_IC, iend - i0);
    for (int ii = 0; ii < ni; ++ii) {
      const int i = i0 + ii;
      const int p = flip ? d - 1 - i : i;
      const float4 a = reinterpret_cast<const float4*>(wm + ii * G::CB)[cg];
      const float4 b = reinterpret_cast<const float4*>(wt + ii * G::CB)[cg];
#pragma unroll
      for (int q = 0; q < RM; ++q) {
        const float z = zs[(rg * RM + q) * G::LD + p];
        am[q][0] = fmaf(z, a.x, am[q][0]);
        am[q][1] = fmaf(z, a.y, am[q][1]);
        am[q][2] = fmaf(z, a.z, am[q][2]);
        am[q][3] = fmaf(z, a.w, am[q][3]);
        at[q][0] = fmaf(z, b.x, at[q][0]);
        at[q][1] = fmaf(z, b.y, at[q][1]);
        at[q][2] = fmaf(z, b.z, at[q][2]);
        at[q][3] = fmaf(z, b.w, at[q][3]);
      }
    }
  }
  __syncthreads();
}

__device__ __forceinline__ float sigmoid_(float s) { return 1.f / (1.f + expf(-s)); }

template <int CGS>
__global__ void __launch_bounds__(IAF_THREADS, 1) iaf_fwd_kernel(
    const float* __restrict__ z_in, const float* __restrict__ lq_in,
    const float* __restrict__ m_w, const float* __restrict__ s_w, float* __restrict__ z_out,
    float* __restrict__ lq_out, float* __restrict__ ck, int64_t R, int d, int n, int gru) {
  constexpr int RM = 2;
  using G = Geo<CGS, RM>;
  __shared__ __align__(16) float zs[G::TR * G::LD];
  __shared__ __align__(16) float wm[IAF_IC * G::CB];
  __shared__ __align__(16) float wt[IAF_IC * G::CB];
  __shared__ float red[G::TR * CGS];
  const int cg = threadIdx.x % CGS, rg = threadIdx.x / CGS;
  const int64_t row0 = (int64_t)blockIdx.x * G::TR;
  const int rows = (int)(R - row0 < G::TR ? R - row0 : G::TR);
  for (int e = threadIdx.x; e < G::TR * d; e += IAF_THREADS) {
    const int r = e / d, j = e % d;
    zs[r * G::LD + j] = r < rows ? z_in[(row0 + r) * d + j] : 0.f;
  }
  float lsum[RM];
#pragma unroll
  for (int q = 0; q < RM; ++q) lsum[q] = 0.f;
  const int nb = (d + G::CB - 1) / G::CB;
  for (int k = 0; k < n; ++k) {
    const bool flip = k & 1;
    __syncthreads();
    if (ck != nullptr) {
      float* __restrict__ ckk = ck + ((int64_t)k * R + row0) * d;
      for (int e = threadIdx.x; e < rows * d; e += IAF_THREADS) {
        const int r = e / d, j = e % d;
        ckk[e] = zs[r * G::LD + (flip ? d - 1 - j : j)];
      }
    }
    const float* __restrict__ mwk = m_w + (int64_t)k * d * d;
    const float* __restrict__ swk = s_w + (int64_t)k * d * d;
    for (int b = nb - 1; b >= 0; --b) {
      const int j0 = b * G::CB;
      float am[RM][4], at[RM][4];
      mt_block<CGS, RM>(zs, flip, d, j0, mwk, swk, wm, wt, rg, cg, am, at);
#pragma unroll
      for (int c = 0; c < 4; ++c) {
        const int j = j0 + cg * 4 + c;
        if (j < d) {
          const int p = flip ? d - 1 - j : j;
#pragma unroll
          for (int q = 0; q < RM; ++q) {
            float* zp = zs + (rg * RM + q) * G::LD + p;
            const float x = *zp, m = am[q][c], t = at[q][c], s = expf(t);
            if (gru) {
              const float g = sigmoid_(s);
              *zp = fmaf(g, x, (1.f - g) * m);
              lsum[q] -= log1pf(expf(-s));
            } else {
              *zp = fmaf(s, x, m);
              lsum[q] += t;
            }
          }
        }
      }
    }
  }
  __syncthreads();
  const bool flip = n & 1;
  for (int e = threadIdx.x; e < rows * d; e += IAF_THREADS) {
    const int r = e / d, j = e % d;
    z_out[row0 * d + e] = zs[r * G::LD + (flip ? d - 1 - j : j)];
  }
  // the rows' log-determinants, summed over the column groups in order
#pragma unroll
  for (int q = 0; q < RM; ++q) red[(rg * RM + q) * CGS + cg] = lsum[q];
  __syncthreads();
  for (int r = threadIdx.x; r < rows; r += IAF_THREADS) {
    float s = 0.f;
    for (int c = 0; c < CGS; ++c) s += red[r * CGS + c];
    lq_out[row0 + r] = lq_in[row0 + r] - s;
  }
}

template <int CGS>
__global__ void __launch_bounds__(IAF_THREADS) iaf_bwd_kernel(
    const float* __restrict__ ck, const float* __restrict__ gz_out,
    const float* __restrict__ glq, const float* __restrict__ m_w, const float* __restrict__ s_w,
    float* __restrict__ gz_in, float* __restrict__ part, int64_t R, int d, int n, int gru,
    int64_t n_tiles) {
  constexpr int RM = 1;
  using G = Geo<CGS, RM>;
  extern __shared__ __align__(16) float smem[];
  float* __restrict__ wm = smem;                         // IC * CB
  float* __restrict__ wt = wm + IAF_IC * G::CB;          // IC * CB
  float* __restrict__ xs = wt + IAF_IC * G::CB;          // flow input, logical order
  float* __restrict__ gs = xs + G::TR * G::LD;           // gradient, physical order (flipped)
  float* __restrict__ gms = gs + G::TR * G::LD;          // g_m, logical order
  float* __restrict__ gts = gms + G::TR * G::LD;         // g_t, logical order
  const int cg = threadIdx.x % CGS, rg = threadIdx.x / CGS;
  const int nb = (d + G::CB - 1) / G::CB;
  const int64_t dd = (int64_t)d * d;
  float* __restrict__ pc = part + (int64_t)blockIdx.x * n * 2 * dd;
  const int nbq = (d + 3) / 4;                           // 4 x 4 blocks of the weight gradients
  for (int64_t tile = blockIdx.x; tile < n_tiles; tile += gridDim.x) {
    const bool first = tile == blockIdx.x;
    const int64_t row0 = tile * G::TR;
    const int rows = (int)(R - row0 < G::TR ? R - row0 : G::TR);
    __syncthreads();
    const bool flip_n = n & 1;
    for (int e = threadIdx.x; e < G::TR * d; e += IAF_THREADS) {
      const int r = e / d, j = e % d;
      gs[r * G::LD + (flip_n ? d - 1 - j : j)] = r < rows ? gz_out[(row0 + r) * d + j] : 0.f;
    }
    const int r_own = rg;                                // RM = 1: one row per thread
    const float gl = r_own < rows ? glq[row0 + r_own] : 0.f;
    for (int k = n - 1; k >= 0; --k) {
      const bool flip = k & 1;
      __syncthreads();
      const float* __restrict__ ckk = ck + ((int64_t)k * R + row0) * d;
      for (int e = threadIdx.x; e < G::TR * d; e += IAF_THREADS) {
        const int r = e / d, j = e % d;
        xs[r * G::LD + j] = r < rows ? ckk[e] : 0.f;
      }
      const float* __restrict__ mwk = m_w + (int64_t)k * dd;
      const float* __restrict__ swk = s_w + (int64_t)k * dd;
      // g_m, g_t and the direct term, block by block of columns
      for (int b = 0; b < nb; ++b) {
        const int j0 = b * G::CB;
        float am[RM][4], at[RM][4];
        mt_block<CGS, RM>(xs, false, d, j0, mwk, swk, wm, wt, rg, cg, am, at);
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int j = j0 + cg * 4 + c;
          if (j < d) {
            const int p = flip ? d - 1 - j : j;
            const float x = xs[r_own * G::LD + j], gy = gs[r_own * G::LD + p];
            const float m = am[0][c], s = expf(at[0][c]);
            float gm, gt, direct;
            if (gru) {
              const float g = sigmoid_(s), omg = 1.f - g;
              gm = gy * omg;
              gt = (gy * (x - m) * g - gl) * omg * s;
              direct = gy * g;
            } else {
              gm = gy;
              gt = gy * x * s - gl;
              direct = gy * s;
            }
            const bool ok = r_own < rows;
            gms[r_own * G::LD + j] = ok ? gm : 0.f;
            gts[r_own * G::LD + j] = ok ? gt : 0.f;
            gs[r_own * G::LD + p] = direct;
          }
        }
      }
      __syncthreads();
      // weight gradients of this tile: d m_w[i][j] += sum_r x_ri g_m_rj, i < j
      float* __restrict__ pk = pc + (int64_t)k * 2 * dd;
      for (int t = threadIdx.x; t < nbq * nbq; t += IAF_THREADS) {
        const int bi = t / nbq, bj = t % nbq;
        if (bi > bj) continue;
        float accm[4][4], acct[4][4];
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int c = 0; c < 4; ++c) accm[a][c] = acct[a][c] = 0.f;
        for (int r = 0; r < rows; ++r) {
          float xv[4], mv[4], tv[4];
#pragma unroll
          for (int a = 0; a < 4; ++a) {
            xv[a] = xs[r * G::LD + min(bi * 4 + a, d - 1)];
            mv[a] = gms[r * G::LD + min(bj * 4 + a, d - 1)];
            tv[a] = gts[r * G::LD + min(bj * 4 + a, d - 1)];
          }
#pragma unroll
          for (int a = 0; a < 4; ++a)
#pragma unroll
            for (int c = 0; c < 4; ++c) {
              accm[a][c] = fmaf(xv[a], mv[c], accm[a][c]);
              acct[a][c] = fmaf(xv[a], tv[c], acct[a][c]);
            }
        }
#pragma unroll
        for (int a = 0; a < 4; ++a)
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int i = bi * 4 + a, j = bj * 4 + c;
            if (i < j && j < d) {
              float* q0 = pk + (int64_t)i * d + j;
              float* q1 = q0 + dd;
              *q0 = first ? accm[a][c] : *q0 + accm[a][c];
              *q1 = first ? acct[a][c] : *q1 + acct[a][c];
            }
          }
      }
      // input gradient: gz_i = direct_i + sum_{j>i} (m_w[i][j] g_m_j + s_w[i][j] g_t_j), written
      // over the direct term at the same physical slot (the next flow down reads it flipped)
      for (int b = 0; b < nb; ++b) {
        const int i0 = b * G::CB;
        float acc[4] = {0.f, 0.f, 0.f, 0.f};
        for (int jc = i0; jc < d; jc += IAF_IC) {
          __syncthreads();
          for (int e = threadIdx.x; e < IAF_IC * G::CB; e += IAF_THREADS) {
            const int ii = e / IAF_IC, jj = e % IAF_IC;
            const int i = i0 + ii, j = jc + jj;
            const bool on = i < j && j < d;
            wm[jj * G::CB + ii] = on ? __ldg(mwk + (int64_t)i * d + j) : 0.f;
            wt[jj * G::CB + ii] = on ? __ldg(swk + (int64_t)i * d + j) : 0.f;
          }
          __syncthreads();
          const int nj = min(IAF_IC, d - jc);
          for (int jj = 0; jj < nj; ++jj) {
            const float4 a = reinterpret_cast<const float4*>(wm + jj * G::CB)[cg];
            const float4 c = reinterpret_cast<const float4*>(wt + jj * G::CB)[cg];
            const float m = gms[r_own * G::LD + jc + jj], t = gts[r_own * G::LD + jc + jj];
            acc[0] = fmaf(m, a.x, fmaf(t, c.x, acc[0]));
            acc[1] = fmaf(m, a.y, fmaf(t, c.y, acc[1]));
            acc[2] = fmaf(m, a.z, fmaf(t, c.z, acc[2]));
            acc[3] = fmaf(m, a.w, fmaf(t, c.w, acc[3]));
          }
        }
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int i = i0 + cg * 4 + c;
          if (i < d) {
            float* gp = gs + r_own * G::LD + (flip ? d - 1 - i : i);
            *gp += acc[c];
          }
        }
      }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < rows * d; e += IAF_THREADS) {
      const int r = e / d;
      gz_in[row0 * d + e] = gs[r * G::LD + e % d];      // flow 0 is unflipped
    }
  }
}

// d m_w and d s_w [n, d, d]: the CTAs' slices summed in CTA order; zero on and below the diagonal.
__global__ void __launch_bounds__(IAF_THREADS) iaf_merge_kernel(
    const float* __restrict__ part, int64_t n_slices, float* __restrict__ dm_w,
    float* __restrict__ ds_w, int d, int n) {
  const int64_t dd = (int64_t)d * d, total = 2 * (int64_t)n * dd;
  for (int64_t o = (int64_t)blockIdx.x * IAF_THREADS + threadIdx.x; o < total;
       o += (int64_t)gridDim.x * IAF_THREADS) {
    const int64_t e = o % dd;
    const int i = (int)(e / d), j = (int)(e % d);
    float v = 0.f;
    if (i < j)
      for (int64_t s = 0; s < n_slices; ++s) v += part[s * total + o];
    const int64_t k = o / (2 * dd), w = (o / dd) & 1;
    (w ? ds_w : dm_w)[k * dd + e] = v;
  }
}

int iaf_cgs(int64_t d) { return d <= 16 ? 4 : (d <= 64 ? 8 : 16); }

int64_t iaf_tiles(int64_t R, int64_t d, int rm) {
  return zsb_ceil_div(R, (int64_t)rm * IAF_THREADS / iaf_cgs(d));
}

int64_t iaf_bwd_ctas(int64_t R, int64_t d, int64_t n) {
  const int64_t per_cta = 2 * n * d * d;
  int64_t g = IAF_PART_BUDGET / (per_cta > 0 ? per_cta : 1);
  g = g < 1 ? 1 : (g > IAF_MAX_CTAS ? IAF_MAX_CTAS : g);
  const int64_t t = iaf_tiles(R, d, 1);
  return t < g ? t : g;
}

template <int CGS>
size_t iaf_bwd_smem() {
  using G = Geo<CGS, 1>;
  return sizeof(float) * (2 * IAF_IC * G::CB + 4 * G::TR * G::LD);
}

template <int CGS>
int iaf_bwd_launch(int64_t ctas, cudaStream_t st, const float* ck, const float* gz_out,
                   const float* glq, const float* m_w, const float* s_w, float* gz_in,
                   float* part, int64_t R, int d, int n, int gru, int64_t n_tiles) {
  const size_t smem = iaf_bwd_smem<CGS>();
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(
        iaf_bwd_kernel<CGS>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    ZSB_REQUIRE(e == cudaSuccess, "iaf_bwd: shared-memory opt-in failed: %s",
                cudaGetErrorString(e));
  }
  iaf_bwd_kernel<CGS><<<(unsigned)ctas, IAF_THREADS, smem, st>>>(
      ck, gz_out, glq, m_w, s_w, gz_in, part, R, d, n, gru, n_tiles);
  return zsb_check_launch("iaf_bwd");
}

}  // namespace

extern "C" {

// CTAs (weight-gradient slices) of the backward sweep (transform.py:17-67, :200-282): `part`
// holds slices * n_iters * 2 * d * d floats.
int zsb_iaf_slices(int64_t R, int64_t d, int64_t n_iters) {
  if (R < 1 || d < 1 || d > IAF_MAX_D || n_iters < 1) return 0;
  return (int)iaf_bwd_ctas(R, d, n_iters);
}

// Forward pass of a linear IAF stack (transform.py:17-67, :255-277).  See include/zsb200.h.
int zsb_iaf_fwd_f32(const float* z_in, const float* lq_in, const float* m_w, const float* s_w,
                    float* z_out, float* lq_out, float* ck, int64_t R, int64_t d,
                    int64_t n_iters, int update, void* stream) {
  ZSB_REQUIRE(m_w && s_w, "zsb_iaf_fwd_f32: null pointer");
  ZSB_REQUIRE(d >= 1 && d <= IAF_MAX_D, "zsb_iaf_fwd_f32: d = %lld outside [1, %d]",
              (long long)d, IAF_MAX_D);
  ZSB_REQUIRE(update == 0 || update == 1, "zsb_iaf_fwd_f32: update %d is neither 0 nor 1",
              update);
  ZSB_REQUIRE(R >= 0 && n_iters >= 1 && n_iters < (1LL << 31),
              "zsb_iaf_fwd_f32: bad sizes (R %lld, n_iters %lld)", (long long)R,
              (long long)n_iters);
  if (R == 0) return ZSB_OK;           // empty rows: the buffers may be NULL
  ZSB_REQUIRE(z_in && lq_in && z_out && lq_out, "zsb_iaf_fwd_f32: null pointer");
  const int64_t tiles = iaf_tiles(R, d, 2);
  ZSB_REQUIRE(tiles < (1LL << 31), "zsb_iaf_fwd_f32: R = %lld too large", (long long)R);
  cudaStream_t st = (cudaStream_t)stream;
  switch (iaf_cgs(d)) {
    case 4: iaf_fwd_kernel<4><<<(unsigned)tiles, IAF_THREADS, 0, st>>>(
        z_in, lq_in, m_w, s_w, z_out, lq_out, ck, R, (int)d, (int)n_iters, update); break;
    case 8: iaf_fwd_kernel<8><<<(unsigned)tiles, IAF_THREADS, 0, st>>>(
        z_in, lq_in, m_w, s_w, z_out, lq_out, ck, R, (int)d, (int)n_iters, update); break;
    default: iaf_fwd_kernel<16><<<(unsigned)tiles, IAF_THREADS, 0, st>>>(
        z_in, lq_in, m_w, s_w, z_out, lq_out, ck, R, (int)d, (int)n_iters, update); break;
  }
  return zsb_check_launch("iaf_fwd");
}

// Backward pass of the stack, one sweep plus one merge launch.  See include/zsb200.h.
int zsb_iaf_bwd_f32(const float* ck, const float* gz_out, const float* glq, const float* m_w,
                    const float* s_w, float* gz_in, float* part, float* dm_w, float* ds_w,
                    int64_t R, int64_t d, int64_t n_iters, int update, void* stream) {
  ZSB_REQUIRE(m_w && s_w && dm_w && ds_w, "zsb_iaf_bwd_f32: null pointer");
  ZSB_REQUIRE(R == 0 || (ck && gz_out && glq && gz_in && part),
              "zsb_iaf_bwd_f32: null pointer");
  ZSB_REQUIRE(d >= 1 && d <= IAF_MAX_D, "zsb_iaf_bwd_f32: d = %lld outside [1, %d]",
              (long long)d, IAF_MAX_D);
  ZSB_REQUIRE(update == 0 || update == 1, "zsb_iaf_bwd_f32: update %d is neither 0 nor 1",
              update);
  ZSB_REQUIRE(R >= 0 && n_iters >= 1 && n_iters < (1LL << 31) &&
                  iaf_tiles(R, d, 1) < (1LL << 31),
              "zsb_iaf_bwd_f32: bad sizes (R %lld, n_iters %lld)", (long long)R,
              (long long)n_iters);
  cudaStream_t st = (cudaStream_t)stream;
  int64_t slices = 0;
  if (R > 0) {
    slices = iaf_bwd_ctas(R, d, n_iters);
    const int64_t tiles = iaf_tiles(R, d, 1);
    int rc;
    switch (iaf_cgs(d)) {
      case 4: rc = iaf_bwd_launch<4>(slices, st, ck, gz_out, glq, m_w, s_w, gz_in, part, R,
                                     (int)d, (int)n_iters, update, tiles); break;
      case 8: rc = iaf_bwd_launch<8>(slices, st, ck, gz_out, glq, m_w, s_w, gz_in, part, R,
                                     (int)d, (int)n_iters, update, tiles); break;
      default: rc = iaf_bwd_launch<16>(slices, st, ck, gz_out, glq, m_w, s_w, gz_in, part, R,
                                       (int)d, (int)n_iters, update, tiles); break;
    }
    if (rc != ZSB_OK) return rc;
  }
  const int64_t total = 2 * n_iters * d * d;
  int64_t blocks = zsb_ceil_div(total, IAF_THREADS);
  blocks = blocks < 8 * ZSB_NUM_SMS ? blocks : 8 * ZSB_NUM_SMS;
  iaf_merge_kernel<<<(unsigned)blocks, IAF_THREADS, 0, st>>>(part, slices, dm_w, ds_w, (int)d,
                                                              (int)n_iters);
  return zsb_check_launch("iaf_merge");
}

}  // extern "C"
