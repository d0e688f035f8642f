// The BNN regression log-joint of examples/bayesian_neural_nets/bnn_vi.py:18-35, 83-86 and
// bnn_sgmcmc.py:19-35, 74-77 for L >= 3 weight layers, layer_sizes = [n_0, n_1, ..., n_{L-1}, 1]:
//   w_i [K, n_{i+1}, n_i + 1] ~ N(0, exp(logstd_i))
//   h_0 = x;  h_{i+1} = [h_i, 1] w_i^T / sqrt(n_i + 1), ReLU after every layer but the last
//   y_mean = h_L[..., 0];  y ~ N(y_mean, exp(y_logstd))
//   lp[k] = sum_i sum log p(w_i[k]) + n_train * mean_b log p(y_b | x_b, w[k])
// Two kernels share one particle pass (forward, backward into a per-particle gradient):
//   zsb_bnn_deep_logjoint_f32      value, gradient of every layer and y_logstd, y_mean and the
//                                  per-point log-likelihood (the two-layer zsb_bnn_logjoint_f32's
//                                  outputs), only those asked for; no backward pass without g
//   zsb_sgmcmc_bnn_deep_step_f32   gradient + the SGHMC / SGLD / PSGLD / SGNHT update of every
//                                  layer, in the update arithmetic of csrc/sgmcmc_bnn.cu
//
// Layout.  One particle's weights no longer fit a warp's registers ([10, 50, 50, 1]: 3151 floats),
// so a CTA of 256 threads works on one particle at a time, persistent over particles.  The
// particle's layers are staged in shared memory (rows padded to an odd stride: conflict-free
// column reads).  Rows are processed in tiles of TR <= 64 (any B); a tile's activations of every
// layer stay in shared memory for the backward pass, where the ReLU mask is read back as a > 0.
// Each layer is one product over the CTA; a thread owns RB = 4 rows of one output column (forward,
// d/d activations) or 4 output rows of one weight column (weight gradient), so every sum has one
// owner and a fixed order.  The weight gradient goes straight to global memory (the g outputs, or
// the step kernel's per-CTA workspace): the weights and their gradient do not both fit shared
// memory at [90, 100, 100, 100, 1] (29401 weights).  Its first tile starts from the prior term.
//
// Limits: 3 <= L <= 8, n_0 <= 128, hidden widths <= 128, at most 32768 weights per particle; any
// B >= 1 and K >= 1.  No floating-point atomics: two identical calls give identical bits.
#include <atomic>

#include "common.cuh"

namespace {

constexpr int MAX_L = 8;          // weight layers
constexpr int MAX_WIDTH = 128;    // n_0 and every hidden width
constexpr int MAX_P = 32768;      // weights per particle
constexpr int NT = 256;           // threads per CTA
constexpr int RB = 4;             // rows (or weight rows) per thread in a product
constexpr int TR_MAX = 64;        // rows per tile
constexpr float HALF_LOG_2PI = 0.918938533204672742f;
// dynamic shared memory available to one CTA on sm_90 (227 KB opt-in, minus the static part)
constexpr size_t SMEM_MAX = 227 * 1024 - 1024;

enum Method : int { SGHMC = 0, SGLD = 1, PSGLD = 2, SGNHT_VEC = 3, SGNHT_SCALAR = 4 };
__host__ __device__ constexpr bool has_momentum(int m) { return m == SGHMC || m == SGNHT_VEC || m == SGNHT_SCALAR; }
__host__ __device__ constexpr bool has_ksum(int m) { return m == SGHMC || m == SGNHT_SCALAR; }

// Shapes and per-layer pointers, passed by value (a __grid_constant__ parameter: indexed by the
// layer without a copy to local memory, and capturable in a CUDA graph).
struct Net {
  int L, B, TR;
  int n[MAX_L + 1];                 // layer widths, n[L] = 1
  int off[MAX_L];                   // offset of layer i in one particle's flat weights
  int soff[MAX_L], ldw[MAX_L];      // staged layer i: offset and (odd) row stride
  int aoff[MAX_L], lda[MAX_L];      // tile activations [h_i, 1]: offset and (odd) row stride
  int P, Wp, Asz, ldz;              // weights, staged floats, activation floats, dZ row stride
  const float* ls[MAX_L]; int ls_n[MAX_L];
  const float* x; const float* y;
  float n_train;
};

struct LjArgs {
  Net net;
  const float* w[MAX_L];
  float* g[MAX_L];
  const float* y_logstd;
  float* lp; float* gys; float* ym; float* ll;
  int64_t K;
};

struct StepArgs {
  Net net;
  float* w[MAX_L]; float* v[MAX_L]; float* al[MAX_L]; float* k[MAX_L];
  const float* aeff[MAX_L];
  const float* noise[MAX_L]; const float* rs[MAX_L];
  float* part; int part_cap;
  float* work;
  int64_t chains;
  float y_logstd, lr, alpha, beta, decay, epsilon, var_extra, tune_rate;
  float hl, omd, ht;
  int second_order, resample;
  uint64_t seed; uint32_t iter; int64_t row0;
};

__host__ __device__ inline int odd(int v) { return v | 1; }

// Shared memory: staged weights | activations | two dZ buffers | {y, dout coefficient} per row.
struct Smem {
  float* W; float* A; float* Z0; float* Z1; float2* yc;
};
__device__ inline Smem carve(const Net& t, float* sh) {
  Smem s;
  s.W = sh;
  s.A = s.W + t.Wp;
  s.Z0 = s.A + t.Asz;
  s.Z1 = s.Z0 + t.TR * t.ldz + RB;
  s.yc = reinterpret_cast<float2*>(s.Z1 + t.TR * t.ldz + RB);
  return s;
}
size_t smem_floats(const Net& t, int extra) {
  return (size_t)t.Wp + t.Asz + 2 * (t.TR * t.ldz + RB) + 2 * t.TR + extra;
}

// log-prior precision of weight idx of layer i
__device__ __forceinline__ float prior_prec(const Net& t, int i, int idx) {
  return expf(-2.f * t.ls[i][idx % t.ls_n[i]]);
}

// rows r0 .. r0 + nr of x into the tile's input activations, and {y, cf} per row
__device__ void stage_tile(const Net& t, const Smem& s, int r0, int nr, float cf) {
  const int n0 = t.n[0], ld = t.lda[0];
  for (int i = threadIdx.x; i < nr * n0; i += NT) {
    const int b = i / n0, k = i - b * n0;
    s.A[b * ld + k] = t.x[(int64_t)(r0 + b) * n0 + k];
  }
  for (int b = threadIdx.x; b < t.TR; b += NT) {
    s.A[b * ld + n0] = 1.f;
    s.yc[b] = b < nr ? make_float2(t.y[r0 + b], cf) : make_float2(0.f, 0.f);
  }
}

// The forward and (GRAD) backward pass of one particle staged in s.W over every row tile.
// Per row b the last layer's output z_b and the staged y_b go through `row(b_global, z_b, y_b)`,
// which returns the residual y_b - y_mean; the weight gradient of layer i is accumulated into gof(i) (flat, one
// particle; NULL: not needed), starting from -prec * w.  rsq receives this thread's sum of
// squared residuals.
template <bool GRAD, class Gof, class Row>
__device__ void particle_pass(const Net& t, const Smem& s, Gof gof, float cf, bool staged,
                              float& rsq, Row row) {
  const int L = t.L, TR = t.TR;
  const int ntiles = (t.B + TR - 1) / TR;
  for (int tile = 0; tile < ntiles; ++tile) {
    const int r0 = tile * TR, nr = min(TR, t.B - r0);
    if (!staged) {
      __syncthreads();
      stage_tile(t, s, r0, nr, cf);
    }
    __syncthreads();
    const int nrg = (nr + RB - 1) / RB;
    // ---- forward: layer i maps activations i ([h_i, 1]) to i + 1, the last one to s.Z1[b]
#pragma unroll 1
    for (int i = 0; i < L; ++i) {
      const int kin = t.n[i] + 1, nout = t.n[i + 1], la = t.lda[i], lw = t.ldw[i];
      const float* A = s.A + t.aoff[i];
      const float* W = s.W + t.soff[i];
      const float sc = rsqrtf((float)kin);
      const bool last = i == L - 1;
      float* O = last ? s.Z1 : s.A + t.aoff[i + 1];
      const int lo = last ? 1 : t.lda[i + 1];
      for (int it = threadIdx.x; it < nrg * nout; it += NT) {
        const int bg = it / nout, m = it - bg * nout, b0 = bg * RB;
        float acc[RB] = {0.f, 0.f, 0.f, 0.f};
        const float* wr = W + m * lw;
        const float* ar = A + b0 * la;
        for (int k = 0; k < kin; ++k) {
          const float wv = wr[k];
#pragma unroll
          for (int j = 0; j < RB; ++j) acc[j] = fmaf(ar[j * la + k], wv, acc[j]);
        }
#pragma unroll
        for (int j = 0; j < RB; ++j)
          if (b0 + j < nr) {
            const float z = acc[j] * sc;
            O[(b0 + j) * lo + m] = last ? z : fmaxf(z, 0.f);
          }
      }
      if (!last) {
        float* An = s.A + t.aoff[i + 1];
        for (int b = threadIdx.x; b < nr; b += NT) An[b * lo + nout] = 1.f;
      }
      __syncthreads();
    }
    // ---- output rows: residual, the caller's per-row outputs, and d lp / d z_b
    for (int b = threadIdx.x; b < nr; b += NT) {
      const float r = row(r0 + b, s.Z1[b], s.yc[b].x);
      rsq = fmaf(r, r, rsq);
      s.Z0[b * t.ldz] = r * s.yc[b].y;
    }
    if constexpr (GRAD) {
      __syncthreads();
      float* dZ = s.Z0;     // d lp / d (pre-activation of layer i + 1), [nr][ldz]
      float* dN = s.Z1;
#pragma unroll 1
      for (int i = L - 1; i >= 0; --i) {
        const int kin = t.n[i] + 1, nout = t.n[i + 1], la = t.lda[i], lw = t.ldw[i], lz = t.ldz;
        const float* A = s.A + t.aoff[i];
        const float* W = s.W + t.soff[i];
        const float sc = rsqrtf((float)kin);
        // weight gradient: g[m][k] += sc * sum_b dZ[b][m] A[b][k]
        float* G = gof(i);
        if (G) {
          const int nmg = (nout + RB - 1) / RB;
          for (int it = threadIdx.x; it < nmg * kin; it += NT) {
            const int mg = it / kin, k = it - mg * kin, m0 = mg * RB;
            float acc[RB] = {0.f, 0.f, 0.f, 0.f};
            for (int b = 0; b < nr; ++b) {
              const float av = A[b * la + k];
              const float* zr = dZ + b * lz + m0;
#pragma unroll
              for (int j = 0; j < RB; ++j) acc[j] = fmaf(zr[j], av, acc[j]);
            }
#pragma unroll
            for (int j = 0; j < RB; ++j) {
              const int m = m0 + j;
              if (m < nout) {
                const int idx = m * kin + k;
                const float base = tile == 0 ? -prior_prec(t, i, idx) * W[m * lw + k] : G[idx];
                G[idx] = fmaf(acc[j], sc, base);
              }
            }
          }
        }
        if (i == 0) break;
        // d/d activations of layer i, masked by its ReLU: dN[b][k] = [A[b][k] > 0] sc sum_m dZ W
        const int nin = t.n[i];
        for (int it = threadIdx.x; it < nrg * nin; it += NT) {
          const int bg = it / nin, k = it - bg * nin, b0 = bg * RB;
          float acc[RB] = {0.f, 0.f, 0.f, 0.f};
          for (int m = 0; m < nout; ++m) {
            const float wv = W[m * lw + k];
#pragma unroll
            for (int j = 0; j < RB; ++j) acc[j] = fmaf(dZ[(b0 + j) * lz + m], wv, acc[j]);
          }
#pragma unroll
          for (int j = 0; j < RB; ++j)
            if (b0 + j < nr) dN[(b0 + j) * lz + k] = A[(b0 + j) * la + k] > 0.f ? acc[j] * sc : 0.f;
        }
        __syncthreads();
        float* tmp = dZ; dZ = dN; dN = tmp;
      }
    }
  }
  __syncthreads();
}

// one-off: every hidden layer's bias column of the tile activations (the forward pass writes the
// rows it computes, and rows past nr are never read)
__device__ void init_bias_columns(const Net& t, const Smem& s) {
  for (int i = 1; i < t.L; ++i)
    for (int b = threadIdx.x; b < t.TR; b += NT) s.A[t.aoff[i] + b * t.lda[i] + t.n[i]] = 1.f;
}

// sum over every weight of logstd (the weight-independent part of the prior), block-reduced
__device__ float logstd_sum(const Net& t, float* red) {
  float l = 0.f;
  for (int i = 0; i < t.L; ++i) {
    const int nw = t.n[i + 1] * (t.n[i] + 1);
    for (int idx = threadIdx.x; idx < nw; idx += NT) l += t.ls[i][idx % t.ls_n[i]];
  }
  return block_sum(l, red);
}

template <bool GRAD>
__global__ void __launch_bounds__(NT) bnn_deep_logjoint_kernel(const __grid_constant__ LjArgs a) {
  extern __shared__ float4 sh4[];
  __shared__ float red[32];
  const Net& t = a.net;
  const Smem s = carve(t, reinterpret_cast<float*>(sh4));
  const float ys = *a.y_logstd;
  const float prec_y = expf(-2.f * ys);
  const float lik_scale = t.n_train / (float)t.B;
  const float cf = prec_y * lik_scale;              // d lp / d z_b = cf (y_b - z_b)
  const float c_ll = -HALF_LOG_2PI - ys;
  const float cst0 = -(float)t.P * HALF_LOG_2PI - logstd_sum(t, red);
  const bool one_tile = t.B <= t.TR;
  init_bias_columns(t, s);
  if (one_tile) stage_tile(t, s, 0, t.B, cf);
  for (int64_t c = blockIdx.x; c < a.K; c += gridDim.x) {
    for (int i = 0; i < t.L; ++i) {
      const int nw = t.n[i + 1] * (t.n[i] + 1), kin = t.n[i] + 1;
      const float* wc = a.w[i] + c * nw;
      float* W = s.W + t.soff[i];
      for (int idx = threadIdx.x; idx < nw; idx += NT) {
        const int m = idx / kin;
        W[m * t.ldw[i] + idx - m * kin] = wc[idx];
      }
    }
    auto gof = [&](int i) {
      return a.g[i] ? a.g[i] + c * (int64_t)(t.n[i + 1] * (t.n[i] + 1)) : nullptr;
    };
    float rsq = 0.f;
    particle_pass<GRAD>(t, s, gof, cf, one_tile, rsq, [&](int b, float z, float yb) {
      const float r = yb - z;
      const int64_t o = c * t.B + b;
      if (a.ym) a.ym[o] = z;
      if (a.ll) a.ll[o] = fmaf(-0.5f * prec_y, r * r, c_ll);
      return r;
    });
    const float rsum = block_sum(rsq, red);
    if (a.lp) {
      float quad = 0.f;
      for (int i = 0; i < t.L; ++i) {
        const int nw = t.n[i + 1] * (t.n[i] + 1), kin = t.n[i] + 1;
        const float* W = s.W + t.soff[i];
        for (int idx = threadIdx.x; idx < nw; idx += NT) {
          const int m = idx / kin;
          const float w = W[m * t.ldw[i] + idx - m * kin];
          quad = fmaf(prior_prec(t, i, idx) * w, w, quad);
        }
      }
      quad = block_sum(quad, red);
      if (threadIdx.x == 0) {
        const float sq = prec_y * lik_scale * rsum;
        a.lp[c] = (cst0 - 0.5f * quad) + (t.n_train * c_ll - 0.5f * sq);
      }
    }
    if (a.gys && threadIdx.x == 0) a.gys[c] = prec_y * lik_scale * rsum - t.n_train;
    __syncthreads();                       // s.W is restaged for the next particle
  }
}

// `n` standard normals of element block b (component e & 3 of block e >> 2) of a Philox row, or
// the injected ones: the numbers the element-wise zsb_sgmcmc_*_f32 kernels draw
__device__ __forceinline__ void normals4(float z[4], const float* injected, int64_t flat0, int blk,
                                         int n, uint64_t seed, uint32_t stream, uint32_t iter,
                                         int64_t row) {
  if (injected) {
#pragma unroll
    for (int j = 0; j < 4; ++j) z[j] = 4 * blk + j < n ? injected[flat0 + 4 * blk + j] : 0.f;
  } else {
    philox_normal4(seed, stream, iter, (uint32_t)row, (uint32_t)blk, z);
  }
}

template <int M>
__global__ void __launch_bounds__(NT) bnn_deep_step_kernel(const __grid_constant__ StepArgs a) {
  extern __shared__ float4 sh4[];
  __shared__ float red[32];
  constexpr bool HV = has_momentum(M);
  const Net& t = a.net;
  const Smem s = carve(t, reinterpret_cast<float*>(sh4));
  float* ks = reinterpret_cast<float*>(s.yc + t.TR);         // [L][NT] per-thread v^2 sums
  const float prec_y = expf(-2.f * a.y_logstd);
  const float cf = prec_y * (t.n_train / (float)t.B);
  const bool one_tile = t.B <= t.TR;
  init_bias_columns(t, s);
  if (one_tile) stage_tile(t, s, 0, t.B, cf);
  if constexpr (has_ksum(M))
    for (int i = 0; i < t.L; ++i) ks[i * NT + threadIdx.x] = 0.f;
  const float sd_xi = (M == SGNHT_VEC || M == SGNHT_SCALAR)
                          ? sqrtf(mul(mul(2.f, a.var_extra), a.lr))
                          : sqrtf(mul(mul(2.f, sub(a.alpha, a.beta)), a.lr));
  const float sd_v = sqrtf(a.lr);
  const bool resample = HV && a.resample;
  float* gw = a.work + (int64_t)blockIdx.x * t.P;

  for (int64_t c = blockIdx.x; c < a.chains; c += gridDim.x) {
    const int64_t grow = a.row0 + c;
    // ---- stage q1 = q (+ v / 2 in second order, v re-drawn first when due)
    for (int i = 0; i < t.L; ++i) {
      const int kin = t.n[i] + 1, nw = t.n[i + 1] * kin, nblk = (nw + 3) >> 2;
      const float* wc = a.w[i] + c * nw;
      float* W = s.W + t.soff[i];
      for (int blk = threadIdx.x; blk < nblk; blk += NT) {
        float z[4];
        if (resample && a.second_order)
          normals4(z, a.rs[i], c * nw, blk, nw, a.seed + i, ZSB_STREAM_SGMCMC_RESAMPLE, a.iter,
                   grow);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int idx = 4 * blk + j;
          if (idx >= nw) break;
          float w = wc[idx];
          if (HV && a.second_order) {
            const float v = resample ? mul(z[j], sd_v) : a.v[i][c * nw + idx];
            w = add(w, mul(0.5f, v));
          }
          const int m = idx / kin;
          W[m * t.ldw[i] + idx - m * kin] = w;
        }
      }
    }
    auto gof = [&](int i) { return gw + t.off[i]; };
    float rsq = 0.f;
    particle_pass<true>(t, s, gof, cf, one_tile, rsq,
                        [&](int, float z, float yb) { return yb - z; });
    // ---- the update, one Philox block (4 weights) per thread and step of the loop
#pragma unroll 1
    for (int i = 0; i < t.L; ++i) {
      const int kin = t.n[i] + 1, nw = t.n[i + 1] * kin, nblk = (nw + 3) >> 2;
      const int64_t base = c * nw;
      const float* W = s.W + t.soff[i];
      const float* G = gw + t.off[i];
      float fr = a.alpha;
      if constexpr (M == SGNHT_SCALAR) fr = *a.aeff[i];
      const float dh = expf(mul(-0.5f, fr)), oma = sub(1.f, fr);
      float ksum = 0.f;
      for (int blk = threadIdx.x; blk < nblk; blk += NT) {
        float z[4], zr[4];
        normals4(z, a.noise[i], base, blk, nw, a.seed + i, ZSB_STREAM_SGMCMC_NOISE, a.iter, grow);
        if (resample)
          normals4(zr, a.rs[i], base, blk, nw, a.seed + i, ZSB_STREAM_SGMCMC_RESAMPLE, a.iter,
                   grow);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int idx = 4 * blk + j;
          if (idx >= nw) break;
          const int m = idx / kin;
          const float q1 = W[m * t.ldw[i] + idx - m * kin], g = G[idx];
          const int64_t e = base + idx;
          if constexpr (M == SGHMC || M == SGNHT_SCALAR) {
            const float xi = mul(z[j], sd_xi);
            const float vold = resample ? mul(zr[j], sd_v) : a.v[i][e];
            float nv, nq;
            if (a.second_order) {
              nv = mul(dh, add(add(mul(dh, vold), mul(a.lr, g)), xi));
              nq = add(q1, mul(0.5f, nv));
            } else {
              nv = add(add(mul(oma, vold), mul(a.lr, g)), xi);
              nq = add(q1, nv);
            }
            a.w[i][e] = nq; a.v[i][e] = nv;
            ksum += nv * nv;
          } else if constexpr (M == SGLD) {
            a.w[i][e] = add(add(q1, mul(a.hl, g)), mul(z[j], sd_v));
          } else if constexpr (M == PSGLD) {
            const float aux = add(mul(a.decay, a.v[i][e]), mul(a.omd, mul(g, g)));
            const float Gp = fdiv(1.f, add(a.epsilon, sqrtf(aux)));
            a.w[i][e] = add(add(q1, mul(mul(a.hl, Gp), g)), mul(z[j], sqrtf(mul(a.lr, Gp))));
            a.v[i][e] = aux;
          } else {                         // SGNHT_VEC
            const float xi = mul(z[j], sd_xi);
            const float ov = resample ? mul(zr[j], sd_v) : a.v[i][e], al = a.al[i][e];
            float nv, nq, na;
            if (a.second_order) {
              const float a1 = add(al, mul(a.ht, sub(mul(ov, ov), a.lr)));
              const float dh1 = expf(mul(-0.5f, a1));
              nv = mul(dh1, add(add(mul(dh1, ov), mul(a.lr, g)), xi));
              nq = add(q1, mul(0.5f, nv));
              na = add(a1, mul(a.ht, sub(mul(nv, nv), a.lr)));
            } else {
              nv = add(add(mul(sub(1.f, al), ov), mul(a.lr, g)), xi);
              nq = add(q1, nv);
              na = add(al, mul(a.tune_rate, sub(mul(nv, nv), a.lr)));
            }
            a.w[i][e] = nq; a.v[i][e] = nv; a.al[i][e] = na; a.k[i][e] = mul(nv, nv);
          }
        }
      }
      if constexpr (has_ksum(M)) ks[i * NT + threadIdx.x] += ksum;
    }
    __syncthreads();                       // s.W and the workspace are reused by the next particle
  }
  if constexpr (has_ksum(M)) {
    for (int i = 0; i < t.L; ++i) {
      const float v = block_sum(ks[i * NT + threadIdx.x], red);
      if (threadIdx.x == 0) a.part[(int64_t)i * a.part_cap + blockIdx.x] = v;
    }
  }
}

struct MeanK {
  const float* part; int part_cap, n_part, L;
  float count[MAX_L];
  float* mean_k[MAX_L];
};

// mean(v_new^2) per latent from the step's per-CTA partials, each merged in CTA order
__global__ void bnn_deep_mean_k_kernel(const __grid_constant__ MeanK m) {
  __shared__ float red[32];
  for (int i = 0; i < m.L; ++i) {
    float s = 0.f;
    for (int j = threadIdx.x; j < m.n_part; j += blockDim.x) s += m.part[i * m.part_cap + j];
    s = block_sum(s, red);
    if (threadIdx.x == 0) m.mean_k[i][0] = s / m.count[i];
  }
}

// Fill the shapes of `t` from the widths; 0, or an error message.  TR is the largest tile of at
// most TR_MAX rows (a multiple of RB) whose shared memory, plus `extra` floats, fits one CTA.
const char* plan(Net& t, int L, const int* widths, int64_t B, int extra) {
  t.L = L;
  t.B = (int)B;
  int P = 0, Wp = 0, sumlda = 0, maxout = 1;
  for (int i = 0; i <= L; ++i) t.n[i] = widths[i];
  for (int i = 0; i < L; ++i) {
    const int kin = t.n[i] + 1;
    t.off[i] = P;
    t.soff[i] = Wp;
    t.ldw[i] = odd(kin);
    t.lda[i] = odd(kin);
    P += t.n[i + 1] * kin;
    Wp += t.n[i + 1] * t.ldw[i];
    if (t.n[i + 1] > maxout) maxout = t.n[i + 1];
    sumlda += t.lda[i];
  }
  t.P = P;
  t.Wp = (Wp + 3) & ~3;
  t.ldz = odd(maxout);
  int TR = (int)(B < TR_MAX ? (B + RB - 1) / RB * RB : TR_MAX);
  for (;;) {
    t.TR = TR;
    int a = 0;
    for (int i = 0; i < L; ++i) { t.aoff[i] = a; a += TR * t.lda[i]; }
    t.Asz = (a + 3) & ~3;
    if (smem_floats(t, extra) * sizeof(float) <= SMEM_MAX) return nullptr;
    if (TR <= RB) return "the weights of one particle do not fit shared memory";
    TR = (TR / 2 + RB - 1) / RB * RB;
  }
}

const char* check_widths(int L, const int* widths) {
  if (!widths) return "null widths";
  if (L < 3 || L > MAX_L) return "need 3 <= L <= 8";
  if (widths[L] != 1) return "the last layer must have width 1";
  int64_t P = 0;
  for (int i = 0; i < L; ++i) {
    if (widths[i] < 1 || widths[i] > MAX_WIDTH) return "need 1 <= n_i <= 128 for i < L";
    P += (int64_t)widths[i + 1] * (widths[i] + 1);
  }
  if (P > MAX_P) return "more than 32768 weights per particle";
  return nullptr;
}

template <class K>
int opt_in(K kernel, std::atomic<uint64_t>& done, const char* what) {
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  const uint64_t bit = dev < 64 ? (1ull << dev) : 0;
  if (e == cudaSuccess && (done.load(std::memory_order_acquire) & bit)) return ZSB_OK;
  if (e == cudaSuccess)
    e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)SMEM_MAX);
  if (e != cudaSuccess) {
    zsb_set_error("%s: shared-memory opt-in failed: %s", what, cudaGetErrorString(e));
    return ZSB_ERR_CUDA;
  }
  done.fetch_or(bit, std::memory_order_release);
  return ZSB_OK;
}

// persistent grid: every CTA the SMs hold at this shared-memory size, at most `cap` and n_items
template <class K>
int grid_of(K kernel, size_t smem, int64_t n_items, int64_t cap, int64_t* grid) {
  int per_sm = 0;
  cudaError_t e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, NT, smem);
  if (e != cudaSuccess || per_sm < 1) {
    zsb_set_error("bnn_deep: occupancy query failed: %s", cudaGetErrorString(e));
    return ZSB_ERR_CUDA;
  }
  int64_t g = (int64_t)per_sm * ZSB_NUM_SMS;
  if (g > cap) g = cap;
  *grid = g < n_items ? g : n_items;
  return ZSB_OK;
}

template <bool GRAD>
int lj_launch(const LjArgs& a, void* stream) {
  static std::atomic<uint64_t> done{0};
  auto kernel = bnn_deep_logjoint_kernel<GRAD>;
  int rc = opt_in(kernel, done, "zsb_bnn_deep_logjoint_f32");
  if (rc) return rc;
  const size_t smem = smem_floats(a.net, 0) * sizeof(float);
  int64_t grid = 0;
  rc = grid_of(kernel, smem, a.K, 1LL << 30, &grid);
  if (rc) return rc;
  kernel<<<(unsigned)grid, NT, smem, (cudaStream_t)stream>>>(a);
  return zsb_check_launch("bnn_deep_logjoint");
}

template <int M>
int step_launch(const StepArgs& a, float* const* mean_k, void* stream) {
  static std::atomic<uint64_t> done{0};
  auto kernel = bnn_deep_step_kernel<M>;
  int rc = opt_in(kernel, done, "zsb_sgmcmc_bnn_deep_step_f32");
  if (rc) return rc;
  const int extra = has_ksum(M) ? a.net.L * NT : 0;
  const size_t smem = smem_floats(a.net, extra) * sizeof(float);
  int64_t grid = 0;
  rc = grid_of(kernel, smem, a.chains, a.part_cap, &grid);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  kernel<<<(unsigned)grid, NT, smem, st>>>(a);
  rc = zsb_check_launch("sgmcmc_bnn_deep");
  if (rc || !has_ksum(M)) return rc;
  MeanK m;
  m.part = a.part; m.part_cap = a.part_cap; m.n_part = (int)grid; m.L = a.net.L;
  for (int i = 0; i < MAX_L; ++i) {
    m.count[i] = i < a.net.L ? (float)(a.chains * a.net.n[i + 1] * (a.net.n[i] + 1)) : 1.f;
    m.mean_k[i] = i < a.net.L ? mean_k[i] : nullptr;
  }
  bnn_deep_mean_k_kernel<<<1, 256, 0, st>>>(m);
  return zsb_check_launch("sgmcmc_bnn_deep_mean_k");
}

}  // namespace

extern "C" {

int zsb_bnn_deep_logjoint_f32(int L, const int* widths, const float* const* w, const float* x,
                              const float* y, int64_t B, const float* const* logstd,
                              const int* logstd_n, const float* y_logstd, float n_train,
                              float* lp, float* const* g, float* g_ylogstd, float* y_mean,
                              float* log_lik, int64_t K, void* stream) {
  const char* bad = check_widths(L, widths);
  ZSB_REQUIRE(!bad, "zsb_bnn_deep_logjoint_f32: %s", bad);
  ZSB_REQUIRE(w && x && y && logstd && logstd_n && y_logstd, "zsb_bnn_deep_logjoint_f32: null arg");
  ZSB_REQUIRE(K > 0 && B > 0 && B < (1LL << 31),
              "zsb_bnn_deep_logjoint_f32: need K > 0 and 0 < B < 2^31 (got K = %lld, B = %lld)",
              (long long)K, (long long)B);
  LjArgs a;
  bool grad = false;
  for (int i = 0; i < MAX_L; ++i) {
    a.w[i] = nullptr; a.g[i] = nullptr; a.net.ls[i] = nullptr; a.net.ls_n[i] = 1;
  }
  for (int i = 0; i < L; ++i) {
    const int64_t nw = (int64_t)widths[i + 1] * (widths[i] + 1);
    ZSB_REQUIRE(w[i] && logstd[i], "zsb_bnn_deep_logjoint_f32: null weights or logstd of layer %d",
                i);
    ZSB_REQUIRE(logstd_n[i] > 0 && logstd_n[i] <= nw,
                "zsb_bnn_deep_logjoint_f32: logstd_n[%d] must be in [1, %lld]", i, (long long)nw);
    a.w[i] = w[i];
    a.g[i] = g ? g[i] : nullptr;
    grad = grad || a.g[i];
    a.net.ls[i] = logstd[i]; a.net.ls_n[i] = logstd_n[i];
  }
  bad = plan(a.net, L, widths, B, 0);
  ZSB_REQUIRE(!bad, "zsb_bnn_deep_logjoint_f32: %s", bad);
  a.net.x = x; a.net.y = y; a.net.n_train = n_train;
  a.y_logstd = y_logstd;
  a.lp = lp; a.gys = g_ylogstd; a.ym = y_mean; a.ll = log_lik;
  a.K = K;
  return grad ? lj_launch<true>(a, stream) : lj_launch<false>(a, stream);
}

int zsb_sgmcmc_bnn_deep_step_f32(int method, int L, const int* widths, float* const* w,
                                 float* const* v, float* const* aux,
                                 const float* const* alpha_eff, const float* x, const float* y,
                                 int64_t B, const float* const* logstd, const int* logstd_n,
                                 float y_logstd, float n_train, float lr, float friction,
                                 float variance_estimate, float decay, float epsilon,
                                 float variance_extra, float tune_rate, int second_order,
                                 int resample, const float* const* noise,
                                 const float* const* resample_noise, uint64_t seed, uint32_t iter,
                                 int64_t row0, float* part, float* const* mean_k, float* work,
                                 int64_t work_n, int64_t chains, void* stream) {
  const char* bad = check_widths(L, widths);
  ZSB_REQUIRE(!bad, "zsb_sgmcmc_bnn_deep_step_f32: %s", bad);
  ZSB_REQUIRE(w && x && y && logstd && logstd_n && work, "zsb_sgmcmc_bnn_deep_step_f32: null arg");
  ZSB_REQUIRE(chains > 0 && B > 0 && B < (1LL << 31),
              "zsb_sgmcmc_bnn_deep_step_f32: need chains > 0 and 0 < B < 2^31");
  ZSB_REQUIRE(method >= SGHMC && method <= SGNHT_SCALAR, "zsb_sgmcmc_bnn_deep_step_f32: bad method");
  const bool mom = has_momentum(method);
  const int cap = ZSB_NUM_SMS * 8;           // zsb_sgmcmc_parts()
  int64_t P = 0;
  for (int i = 0; i < L; ++i) P += (int64_t)widths[i + 1] * (widths[i] + 1);
  ZSB_REQUIRE(work_n >= (chains < cap ? chains : cap) * P,
              "zsb_sgmcmc_bnn_deep_step_f32: work needs min(chains, zsb_sgmcmc_parts()) * "
              "(weights per chain) floats");
  ZSB_REQUIRE(!mom || v, "zsb_sgmcmc_bnn_deep_step_f32: this method needs v");
  ZSB_REQUIRE((method != PSGLD && method != SGNHT_VEC) || aux,
              "zsb_sgmcmc_bnn_deep_step_f32: this method needs aux");
  ZSB_REQUIRE(method != SGNHT_SCALAR || alpha_eff,
              "zsb_sgmcmc_bnn_deep_step_f32: scalar SGNHT needs alpha_eff");
  ZSB_REQUIRE((method != SGHMC && method != SGNHT_SCALAR && method != SGNHT_VEC) || mean_k,
              "zsb_sgmcmc_bnn_deep_step_f32: this method needs mean_k");
  ZSB_REQUIRE((method != SGHMC && method != SGNHT_SCALAR) || part,
              "zsb_sgmcmc_bnn_deep_step_f32: this method needs part");
  ZSB_REQUIRE(method != SGNHT_SCALAR || !resample,
              "zsb_sgmcmc_bnn_deep_step_f32: scalar SGNHT re-draws v before the step, not in it");
  StepArgs a;
  for (int i = 0; i < MAX_L; ++i) {
    a.w[i] = nullptr; a.v[i] = nullptr; a.al[i] = nullptr; a.k[i] = nullptr;
    a.aeff[i] = nullptr; a.noise[i] = nullptr; a.rs[i] = nullptr;
    a.net.ls[i] = nullptr; a.net.ls_n[i] = 1;
  }
  for (int i = 0; i < L; ++i) {
    const int64_t nw = (int64_t)widths[i + 1] * (widths[i] + 1);
    ZSB_REQUIRE(w[i] && logstd[i], "zsb_sgmcmc_bnn_deep_step_f32: null weights or logstd of "
                "layer %d", i);
    ZSB_REQUIRE(logstd_n[i] > 0 && logstd_n[i] <= nw,
                "zsb_sgmcmc_bnn_deep_step_f32: logstd_n[%d] must be in [1, %lld]", i,
                (long long)nw);
    ZSB_REQUIRE(!mom || v[i], "zsb_sgmcmc_bnn_deep_step_f32: null v of layer %d", i);
    ZSB_REQUIRE((method != PSGLD && method != SGNHT_VEC) || aux[i],
                "zsb_sgmcmc_bnn_deep_step_f32: null aux of layer %d", i);
    ZSB_REQUIRE(method != SGNHT_SCALAR || alpha_eff[i],
                "zsb_sgmcmc_bnn_deep_step_f32: null alpha_eff of layer %d", i);
    ZSB_REQUIRE(!(mom && mean_k) || mean_k[i],
                "zsb_sgmcmc_bnn_deep_step_f32: null mean_k of layer %d", i);
    a.w[i] = w[i];
    a.v[i] = method == PSGLD ? aux[i] : (mom ? v[i] : nullptr);
    a.al[i] = method == SGNHT_VEC ? aux[i] : nullptr;
    a.k[i] = method == SGNHT_VEC ? mean_k[i] : nullptr;
    a.aeff[i] = method == SGNHT_SCALAR ? alpha_eff[i] : nullptr;
    a.noise[i] = noise ? noise[i] : nullptr;
    a.rs[i] = resample_noise ? resample_noise[i] : nullptr;
    a.net.ls[i] = logstd[i]; a.net.ls_n[i] = logstd_n[i];
  }
  bad = plan(a.net, L, widths, B, has_ksum(method) ? L * NT : 0);
  ZSB_REQUIRE(!bad, "zsb_sgmcmc_bnn_deep_step_f32: %s", bad);
  a.net.x = x; a.net.y = y; a.net.n_train = n_train;
  a.part = part; a.part_cap = cap; a.work = work; a.chains = chains;
  a.y_logstd = y_logstd; a.lr = lr; a.alpha = friction; a.beta = variance_estimate;
  a.decay = decay; a.epsilon = epsilon; a.var_extra = variance_extra; a.tune_rate = tune_rate;
  a.hl = mul(0.5f, lr); a.omd = sub(1.f, decay); a.ht = mul(0.5f, tune_rate);
  a.second_order = mom ? second_order : 0; a.resample = mom ? resample : 0;
  a.seed = seed; a.iter = iter; a.row0 = row0;
  switch (method) {
    case SGHMC: return step_launch<SGHMC>(a, mean_k, stream);
    case SGLD: return step_launch<SGLD>(a, mean_k, stream);
    case PSGLD: return step_launch<PSGLD>(a, mean_k, stream);
    case SGNHT_VEC: return step_launch<SGNHT_VEC>(a, mean_k, stream);
    default: return step_launch<SGNHT_SCALAR>(a, mean_k, stream);
  }
}

}  // extern "C"
