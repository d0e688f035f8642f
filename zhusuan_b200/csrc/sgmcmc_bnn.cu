// K5 + K8 for BASELINE config 4: SG-MCMC over per-chain Bayesian-NN weights, ONE launch per step.
//
// Model (examples/bayesian_neural_nets/bnn_sgmcmc.py:19-35, 74-77), layer sizes [n_in, H, 1]:
//   w0 [chains, H, n_in+1] ~ N(0, exp(logstd0)),  w1 [chains, 1, H+1] ~ N(0, exp(logstd1))
//   h0 = [x, 1];  a1 = h0 w0^T / sqrt(n_in+1);  r1 = relu(a1);  h1 = [r1, 1]
//   y_mean = h1 w1^T / sqrt(H+1);   y ~ N(y_mean, exp(y_logstd))
//   log_joint = sum log p(w) + mean_b log p(y_b | x_b, w) * n_train
// Update rules, per chain, fused (each in the rounding and operation order of its element-wise
// kernel in sgmcmc.cu, so fused and generic differ only in the gradient's summation order):
//   SGHMC (zhusuan/sgmcmc.py:326-371)
//     [resample v ~ N(0, sqrt(lr))]                                    sgmcmc.py:327-336
//     2nd order: q1 = q + v/2;  g = grad log_joint(q1);  v = dh (dh v + lr g + xi);  q = q1 + v/2
//     1st order: g = grad log_joint(q);  v = (1-alpha) v + lr g + xi;  q += v
//     xi ~ N(0, sqrt(2 (alpha-beta) lr));  partial sums of v^2 for mean_k            sgmcmc.py:358
//   SGLD (sgmcmc.py:195-200):   q += 0.5 lr g + N(0, sqrt(lr))
//   PSGLD (sgmcmc.py:225-257):  aux = decay aux + (1-decay) g^2;  G = 1/(eps + sqrt(aux));
//                               q += 0.5 lr G g + N(0, sqrt(lr G))
//   SGNHT, vector alpha (sgmcmc.py:460-523): SGHMC's integrator with a per-weight thermostat;
//     2nd order takes a1 = alpha + tune/2 (v_old^2 - lr) and dh = exp(-a1/2); k = v_new^2 is
//     written out; xi ~ N(0, sqrt(2 a lr))
//   SGNHT, scalar alpha: the SGHMC integrator with alpha_eff read from a device scalar per latent
//     (alpha, or alpha1 from mean(v_old^2) in 2nd order) and v^2 block partials out; the
//     thermostat itself couples all chains, so the host updates it around the launch.
//
// One warp per chain (persistent grid).  Lane l owns hidden units l and l+32: their w0 rows, gradient accumulators
// and w1 entries stay in registers across the whole minibatch; the minibatch (x, y) is staged once
// per block in shared memory, rows padded to a multiple of 4 floats so a row is read with 128-bit
// broadcast loads.  Round 1 spent 17.6 k warp instructions per chain and step, half of them outside
// the minibatch loop: every lane regenerated (under divergence) each Philox block it touched, and
// each weight paid an integer modulo + expf for its prior precision.  Now the warp generates each
// noise block once into shared memory and the prior precisions are tabulated once per block.  The gradient (tf.gradients in the reference, sgmcmc.py:96-98) is the
// hand-derived backward of the two-layer net.  HBM traffic per weight and chain-step: 8 B (SGLD,
// q r+w), 16 B (PSGLD, SGHMC: q and aux / v), 20 B (SGNHT scalar), 28 B (SGNHT vector: q, v,
// alpha r+w, k written); 601 weights per chain at [10, 50, 1]; ~0.36 MFLOP per chain-step.
//
// Occupancy: 2 blocks of up to 8 warps per SM.  Each warp stages one chain's weights plus the
// method's state (SGLD none, SGHMC / PSGLD / scalar SGNHT one array, vector SGNHT two) in shared
// memory.  SGHMC at the maximum shape (n_in + 1 = 16, H = 64, B = 512) takes ~109 KB per block at
// 8 warps; vector SGNHT would take ~143 KB there, so the launcher drops to the most warps per block
// that keep two blocks resident (5 at the maximum shape, 40 warps per SM; 8 at [10, 50, 1]).
#include "common.cuh"

namespace {

constexpr int MAX_IN1 = 16;   // n_in + 1 <= 16
constexpr int MAX_B = 512;    // minibatch rows staged in shared memory
constexpr int MAX_NW = 8;     // warps per block
// dynamic shared memory per block that still leaves room for a second block on the SM
// (228 KB per SM, 1 KB of it reserved per block)
constexpr size_t SMEM_TWO_BLOCKS = 113 * 1024;

// the update rules (ZSB_SGMCMC_* in zsb200.h)
enum Method : int { SGHMC = 0, SGLD = 1, PSGLD = 2, SGNHT_VEC = 3, SGNHT_SCALAR = 4 };
// per-warp staging arrays: the weights (A), the momentum or PSGLD's aux (B), SGNHT's vector alpha (C)
__host__ __device__ constexpr int n_stage(int m) { return m == SGLD ? 1 : (m == SGNHT_VEC ? 3 : 2); }
__host__ __device__ constexpr bool has_momentum(int m) { return m == SGHMC || m == SGNHT_VEC || m == SGNHT_SCALAR; }
__host__ __device__ constexpr bool has_ksum(int m) { return m == SGHMC || m == SGNHT_SCALAR; }

struct BnnArgs {
  float* w0; float* w1;
  float* v0; float* v1;              // B state: momentum, or PSGLD's aux
  float* al0; float* al1;            // C state: SGNHT's vector alpha
  float* k0; float* k1;              // vector SGNHT: k = v_new^2 out
  const float* aeff0; const float* aeff1;   // scalar SGNHT: alpha_eff per latent (device)
  const float* x; const float* y;
  const float* logstd0; int64_t logstd0_n; const float* logstd1; int64_t logstd1_n;
  const float* noise0; const float* noise1; const float* rs0; const float* rs1;
  float* part0; float* part1;
  int64_t chains; int B, n_in, H;
  float y_logstd, n_train, lr, alpha, beta;
  float decay, epsilon, var_extra, tune_rate;
  float hl, omd, ht;                 // 0.5 lr, 1 - decay, 0.5 tune_rate (host-rounded: no registers)
  int second_order, resample;
  uint64_t seed; uint32_t iter; int64_t row0;
};

constexpr int PB = 4;   // data points processed together (independent FMA / shuffle chains)

// `n` standard normals of (row, elements 0..n-1) of a Philox stream into a per-warp shared buffer
// (n rounded up to 4 floats), or the injected ones.  Element e is component e & 3 of block e >> 2
// -- the same numbers the element-wise kernels draw (sgmcmc.cu), so the fused and the generic path
// agree draw for draw.  Each block is generated ONCE per warp (round 1 generated a block in every
// lane that touched it, under divergence: 22 Philox evaluations per lane and step instead of 5).
__device__ __forceinline__ void warp_fill_normals(float* buf, int n, const float* injected,
                                                  int64_t flat0, uint64_t seed, uint32_t stream,
                                                  uint32_t iter, int64_t row, int lane) {
  if (injected) {
    for (int i = lane; i < n; i += 32) buf[i] = injected[flat0 + i];
  } else {
    const int nblk = (n + 3) >> 2;
    for (int b = lane; b < nblk; b += 32) {
      float z[4];
      philox_normal4(seed, stream, iter, (uint32_t)row, (uint32_t)b, z);
      reinterpret_cast<float4*>(buf)[b] = make_float4(z[0], z[1], z[2], z[3]);
    }
  }
  __syncwarp();
}

template <int IN1, int M>
__global__ void __launch_bounds__(256, 2) sgmcmc_bnn_kernel(BnnArgs a) {
  extern __shared__ float4 sh4[];
  constexpr int in1 = IN1;
  constexpr int X4 = (IN1 + 3) / 4;     // a staged minibatch row = X4 float4 (bias column, 0 pad)
  constexpr int XP = 4 * X4;
  constexpr int NS = n_stage(M);
  constexpr bool HV = has_momentum(M);
  const int H1 = a.H + 1;
  const int n0 = a.H * in1;                       // weights of layer 0 per chain
  const int n0p = (n0 + 3) & ~3, n1p = (H1 + 3) & ~3;
  const int Bp = (a.B + PB - 1) / PB * PB;        // padded with zero-weight rows
  float* xs = reinterpret_cast<float*>(sh4);                 // [Bp + PB][XP]
  float2* yc = reinterpret_cast<float2*>(xs + (Bp + PB) * XP);      // [Bp] {y, dout coefficient or 0}
  float* pr0 = reinterpret_cast<float*>(yc + Bp);            // [n0p] prior precision exp(-2 ls)
  float* pr1 = pr0 + n0p;                                    // [n1p]
  float* nzb = pr1 + n1p;                                    // [warps][NS][n0p + n1p] staging
  __shared__ float red[32];
  const float inv_s0 = rsqrtf((float)in1), inv_s1 = rsqrtf((float)H1);
  {
    const float prec_y = expf(-2.f * a.y_logstd);
    const float lik_scale = a.n_train / (float)a.B;
    // d log_joint / d (h1 . w1) = prec_y (y - y_mean) * (n_train / B) / sqrt(H + 1)
    const float cf = prec_y * lik_scale * inv_s1;
    for (int i = threadIdx.x; i < (Bp + PB) * XP; i += blockDim.x) {
      const int b = i / XP, k = i % XP;
      xs[i] = (b < a.B) ? ((k < a.n_in) ? a.x[b * a.n_in + k] : (k == a.n_in ? 1.f : 0.f)) : 0.f;
    }
    for (int i = threadIdx.x; i < Bp; i += blockDim.x)
      yc[i] = (i < a.B) ? make_float2(a.y[i], cf) : make_float2(0.f, 0.f);
    const int ls0_n = (int)a.logstd0_n, ls1_n = (int)a.logstd1_n;
    for (int i = threadIdx.x; i < n0p; i += blockDim.x)
      pr0[i] = (i < n0) ? expf(-2.f * a.logstd0[i % ls0_n]) : 0.f;
    for (int i = threadIdx.x; i < n1p; i += blockDim.x)
      pr1[i] = (i < H1) ? expf(-2.f * a.logstd1[i % ls1_n]) : 0.f;
  }
  __syncthreads();

  // warp index through a shuffle: provably warp-uniform, so the chain loop's exit is uniform and the
  // shuffles inside it compile to plain SHFL instead of WARPSYNC.COLLECTIVE sequences
  const int lane = threadIdx.x & 31, nwb = blockDim.x >> 5;
  const int wib = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  // per-warp staging: A = weights in / noise / new weights out, B = momentum (or aux) in / out,
  // C = vector alpha in / out.  Every global access of a chain's state is a coalesced, independent
  // copy through these buffers (round 1 read v element by element between dependent stores: 22
  // exposed global latencies).
  float* A0 = nzb + wib * NS * (n0p + n1p);
  float* A1 = A0 + n0p;
  float* B0 = A1 + n1p;
  float* B1 = B0 + n0p;
  float* C0 = B1 + n1p;
  float* C1 = C0 + n0p;
  const float sd_xi = (M == SGNHT_VEC || M == SGNHT_SCALAR)
                          ? sqrtf(mul(mul(2.f, a.var_extra), a.lr))
                          : sqrtf(mul(mul(2.f, sub(a.alpha, a.beta)), a.lr));
  const float sd_v = sqrtf(a.lr);
  // friction per latent: SGHMC's alpha, or scalar SGNHT's alpha_eff
  float fr0 = a.alpha, fr1 = a.alpha;
  if constexpr (M == SGNHT_SCALAR) { fr0 = *a.aeff0; fr1 = *a.aeff1; }
  const float dh0 = expf(mul(-0.5f, fr0)), oma0 = sub(1.f, fr0);
  const float dh1 = expf(mul(-0.5f, fr1)), oma1 = sub(1.f, fr1);
  const float hl = a.hl, omd = a.omd, ht = a.ht;
  float ksum0 = 0.f, ksum1 = 0.f;

  for (int64_t c = (int64_t)blockIdx.x * nwb + wib; c < a.chains;
       c += (int64_t)gridDim.x * nwb) {
    float* w0c = a.w0 + c * n0;
    float* w1c = a.w1 + c * H1;
    const int64_t grow = a.row0 + c;
    for (int i = lane; i < n0; i += 32) A0[i] = w0c[i];
    for (int i = lane; i < H1; i += 32) A1[i] = w1c[i];
    if constexpr (NS >= 2) {
      const float* v0c = a.v0 + c * n0;
      const float* v1c = a.v1 + c * H1;
      if (HV && a.resample) {   // momentum resample v ~ N(0, sqrt(lr)) (sgmcmc.py:327-336)
        warp_fill_normals(B0, n0, a.rs0, c * n0, a.seed, ZSB_STREAM_SGMCMC_RESAMPLE, a.iter, grow,
                          lane);
        warp_fill_normals(B1, H1, a.rs1, c * H1, a.seed + 1, ZSB_STREAM_SGMCMC_RESAMPLE, a.iter,
                          grow, lane);
        for (int i = lane; i < n0; i += 32) B0[i] = mul(B0[i], sd_v);
        for (int i = lane; i < H1; i += 32) B1[i] = mul(B1[i], sd_v);
      } else {
        for (int i = lane; i < n0; i += 32) B0[i] = v0c[i];
        for (int i = lane; i < H1; i += 32) B1[i] = v1c[i];
      }
    }
    if constexpr (NS >= 3) {
      for (int i = lane; i < n0; i += 32) C0[i] = a.al0[c * n0 + i];
      for (int i = lane; i < H1; i += 32) C1[i] = a.al1[c * H1 + i];
    }
    __syncwarp();
    // ---- this lane's parameters (hidden units m = lane, lane + 32; lane 0 also the h1 bias)
    float W[2][IN1], G[2][IN1];
    float w1r[2], w1s[2], g1r[2];
    float w1b = 0.f, g1b = 0.f;
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int m = lane + 32 * u;
      const bool mv = m < a.H;
#pragma unroll
      for (int k = 0; k < in1; ++k) {
        const int idx = m * in1 + k;
        float w = mv ? A0[idx] : 0.f;
        if (HV && a.second_order && mv) w = add(w, mul(0.5f, B0[idx]));   // q1 = q + v/2
        W[u][k] = w; G[u][k] = 0.f;
      }
      float w = mv ? A1[m] : 0.f;
      if (HV && a.second_order && mv) w = add(w, mul(0.5f, B1[m]));
      w1r[u] = w; w1s[u] = w * inv_s0; g1r[u] = 0.f;
    }
    if (lane == 0) {
      w1b = A1[a.H];
      if (HV && a.second_order) w1b = add(w1b, mul(0.5f, B1[a.H]));
    }
    __syncwarp();                          // A is overwritten with the update noise below
    // ---- forward + backward over the minibatch, PB points at a time.  A staged row is read as
    // X4 128-bit shared loads (every lane the same address: broadcast).  With s = W x (the
    // pre-activation before the 1/sqrt(n_in+1) scale), r = max(s, 0):
    //   h1 . w1 = sum_m (w1_m / sqrt(n_in+1)) r_m + bias;   dout = cf_b (y_b - (h1 . w1)/sqrt(H+1))
    //   d/dw1_m += dout r_m / sqrt(n_in+1) (scale applied once after the loop)
    //   d/dW_mk += [s_m > 0] dout (w1_m / sqrt(n_in+1)) x_k
    const float bias_l = (lane == 0) ? w1b : 0.f;                        // bias unit of h1
    auto load_row = [&](int b, float* xv) {
      const float4* xr = reinterpret_cast<const float4*>(xs + b * XP);
#pragma unroll
      for (int j = 0; j < X4; ++j) {
        const float4 t = xr[j];
        xv[4 * j] = t.x; xv[4 * j + 1] = t.y; xv[4 * j + 2] = t.z; xv[4 * j + 3] = t.w;
      }
    };
    auto forward1 = [&](int b, float& s0, float& s1, float& pt) {
      float xv[XP];
      load_row(b, xv);
      float sacc0 = 0.f, sacc1 = 0.f;
#pragma unroll
      for (int k = 0; k < in1; ++k) {
        sacc0 = fmaf(W[0][k], xv[k], sacc0);
        sacc1 = fmaf(W[1][k], xv[k], sacc1);
      }
      s0 = sacc0; s1 = sacc1;
      pt = fmaf(w1s[1], fmaxf(sacc1, 0.f), fmaf(w1s[0], fmaxf(sacc0, 0.f), bias_l));
    };
    // software pipeline: the forward pass of block i+1 (one data point per slot) is issued between
    // the butterfly rounds of block i's h1 . w1 reduction -- five dependent shuffles on which the
    // warp would otherwise idle.  xs holds PB zero rows past Bp, so the look-ahead needs no branch.
    static_assert(PB == 4, "the interleave below is written for 4 points per block");
    float sa[2][PB], part[PB];
#pragma unroll
    for (int p = 0; p < PB; ++p) forward1(p, sa[0][p], sa[1][p], part[p]);
    for (int b0 = 0; b0 < Bp; b0 += PB) {
      float sn[2][PB], pn[PB];
#define ZSB_BFLY(o)                                                                   \
  _Pragma("unroll") for (int p = 0; p < PB; ++p)                                      \
      part[p] += __shfl_xor_sync(0xffffffffu, part[p], o);
      ZSB_BFLY(16)
      forward1(b0 + PB + 0, sn[0][0], sn[1][0], pn[0]);
      ZSB_BFLY(8)
      forward1(b0 + PB + 1, sn[0][1], sn[1][1], pn[1]);
      ZSB_BFLY(4)
      forward1(b0 + PB + 2, sn[0][2], sn[1][2], pn[2]);
      ZSB_BFLY(2)
      forward1(b0 + PB + 3, sn[0][3], sn[1][3], pn[3]);
      ZSB_BFLY(1)
#undef ZSB_BFLY
#pragma unroll
      for (int p = 0; p < PB; ++p) {
        float xv[XP];
        load_row(b0 + p, xv);
        const float2 yw = yc[b0 + p];
        const float dout = fmaf(-inv_s1, part[p], yw.x) * yw.y;    // 0 for padding rows
#pragma unroll
        for (int u = 0; u < 2; ++u) {
          g1r[u] = fmaf(dout, fmaxf(sa[u][p], 0.f), g1r[u]);
          const float da = (sa[u][p] > 0.f) ? dout * w1s[u] : 0.f;
#pragma unroll
          for (int k = 0; k < in1; ++k) G[u][k] = fmaf(da, xv[k], G[u][k]);
        }
        g1b += dout;                       // every lane accumulates; only lane 0's copy is used
      }
#pragma unroll
      for (int p = 0; p < PB; ++p) {
        part[p] = pn[p];
        sa[0][p] = sn[0][p]; sa[1][p] = sn[1][p];
      }
    }
    // ---- prior gradient and the update (noise in A, old state in B / C; results overwrite them)
    warp_fill_normals(A0, n0, a.noise0, c * n0, a.seed, ZSB_STREAM_SGMCMC_NOISE, a.iter, grow,
                      lane);
    warp_fill_normals(A1, H1, a.noise1, c * H1, a.seed + 1, ZSB_STREAM_SGMCMC_NOISE, a.iter, grow,
                      lane);
    // one weight: q1 = the weight the gradient was taken at, g = its gradient; A[i] holds its
    // standard normal on entry and the new weight on exit, B[i] / C[i] its state
    auto update = [&](int layer, float q1, float g, float* A, float* B, float* C, int i,
                      float& ks) {
      if constexpr (M == SGHMC || M == SGNHT_SCALAR) {
        const float dh = layer ? dh1 : dh0, oma = layer ? oma1 : oma0;
        const float xi = mul(A[i], sd_xi), vold = B[i];
        float nv, nq;
        if (a.second_order) {
          nv = mul(dh, add(add(mul(dh, vold), mul(a.lr, g)), xi));
          nq = add(q1, mul(0.5f, nv));
        } else {
          nv = add(add(mul(oma, vold), mul(a.lr, g)), xi);
          nq = add(q1, nv);
        }
        A[i] = nq; B[i] = nv;
        ks += nv * nv;
      } else if constexpr (M == SGLD) {
        A[i] = add(add(q1, mul(hl, g)), mul(A[i], sd_v));
      } else if constexpr (M == PSGLD) {
        const float aux = add(mul(a.decay, B[i]), mul(omd, mul(g, g)));
        const float Gp = fdiv(1.f, add(a.epsilon, sqrtf(aux)));
        A[i] = add(add(q1, mul(mul(hl, Gp), g)), mul(A[i], sqrtf(mul(a.lr, Gp))));
        B[i] = aux;
      } else {                             // SGNHT_VEC
        const float xi = mul(A[i], sd_xi), ov = B[i], al = C[i];
        float nv, nq, na;
        if (a.second_order) {
          const float a1 = add(al, mul(ht, sub(mul(ov, ov), a.lr)));
          const float dh = expf(mul(-0.5f, a1));
          nv = mul(dh, add(add(mul(dh, ov), mul(a.lr, g)), xi));
          nq = add(q1, mul(0.5f, nv));
          na = add(a1, mul(ht, sub(mul(nv, nv), a.lr)));
        } else {
          nv = add(add(mul(sub(1.f, al), ov), mul(a.lr, g)), xi);
          nq = add(q1, nv);
          na = add(al, mul(a.tune_rate, sub(mul(nv, nv), a.lr)));
        }
        A[i] = nq; B[i] = nv; C[i] = na;
      }
    };
#pragma unroll
    for (int u = 0; u < 2; ++u) {
      const int m = lane + 32 * u;
      if (m < a.H) {
#pragma unroll
        for (int k = 0; k < in1; ++k) {
          const int idx = m * in1 + k;
          const float g = G[u][k] - pr0[idx] * W[u][k];
          update(0, W[u][k], g, A0, B0, C0, idx, ksum0);
        }
        const float g = g1r[u] * inv_s0 - pr1[m] * w1r[u];
        update(1, w1r[u], g, A1, B1, C1, m, ksum1);
      }
    }
    if (lane == 0) {
      const float g = g1b - pr1[a.H] * w1b;
      update(1, w1b, g, A1, B1, C1, a.H, ksum1);
    }
    __syncwarp();
    for (int i = lane; i < n0; i += 32) {
      w0c[i] = A0[i];
      if constexpr (NS >= 2) a.v0[c * n0 + i] = B0[i];
      if constexpr (NS >= 3) { a.al0[c * n0 + i] = C0[i]; a.k0[c * n0 + i] = mul(B0[i], B0[i]); }
    }
    for (int i = lane; i < H1; i += 32) {
      w1c[i] = A1[i];
      if constexpr (NS >= 2) a.v1[c * H1 + i] = B1[i];
      if constexpr (NS >= 3) { a.al1[c * H1 + i] = C1[i]; a.k1[c * H1 + i] = mul(B1[i], B1[i]); }
    }
    __syncwarp();                          // the buffers are restaged for the next chain
  }
  if constexpr (has_ksum(M)) {
    ksum0 = block_sum(ksum0, red);
    if (threadIdx.x == 0) a.part0[blockIdx.x] = ksum0;
    ksum1 = block_sum(ksum1, red);
    if (threadIdx.x == 0) a.part1[blockIdx.x] = ksum1;
  }
}

__global__ void bnn_mean_k_kernel(const float* part0, const float* part1, int n_part, float n0,
                                  float n1, float* mean_k0, float* mean_k1) {
  __shared__ float red[32];
  float s0 = 0.f, s1 = 0.f;
  for (int i = threadIdx.x; i < n_part; i += blockDim.x) { s0 += part0[i]; s1 += part1[i]; }
  s0 = block_sum(s0, red);
  s1 = block_sum(s1, red);
  if (threadIdx.x == 0) { mean_k0[0] = s0 / n0; mean_k1[0] = s1 / n1; }
}

template <int M>
int bnn_launch(const BnnArgs& a, float* mean_k0, float* mean_k1, void* stream) {
  const int Bp = (a.B + PB - 1) / PB * PB;
  const int n0p = (a.H * (a.n_in + 1) + 3) & ~3, n1p = (a.H + 1 + 3) & ~3;
  auto smem_of = [&](int nw) {
    return (size_t)((Bp + PB) * ((a.n_in + 1 + 3) / 4 * 4) + 2 * Bp +
                    (1 + nw * n_stage(M)) * (n0p + n1p)) * sizeof(float);
  };
  // persistent grid: two resident blocks per SM, each warp walks its chains.  (7 warps per block
  // would fill the last round of 8192 chains better -- 3.95 instead of 3.46 rounds -- but measured
  // the same: the kernel is bound by per-warp latency x warps in flight, not by the tail.)  Shapes
  // whose per-warp staging does not fit two blocks of 8 warps run fewer warps per block.
  int nw = MAX_NW;
  while (nw > 1 && smem_of(nw) > SMEM_TWO_BLOCKS) --nw;
  const size_t smem = smem_of(nw);
  int64_t blocks = zsb_ceil_div(a.chains, nw);
  if (blocks > 2 * ZSB_NUM_SMS) blocks = 2 * ZSB_NUM_SMS;
  cudaStream_t st = (cudaStream_t)stream;
  switch (a.n_in + 1) {
#define ZSB_BNN_CASE(N)                                                                          \
  case N:                                                                                        \
    if (smem > 48 * 1024)                                                                        \
      cudaFuncSetAttribute(sgmcmc_bnn_kernel<N, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                           (int)smem);                                                           \
    sgmcmc_bnn_kernel<N, M><<<(unsigned)blocks, 32 * nw, smem, st>>>(a);                         \
    break;
    ZSB_BNN_CASE(2) ZSB_BNN_CASE(3) ZSB_BNN_CASE(4) ZSB_BNN_CASE(5) ZSB_BNN_CASE(6)
    ZSB_BNN_CASE(7) ZSB_BNN_CASE(8) ZSB_BNN_CASE(9) ZSB_BNN_CASE(10) ZSB_BNN_CASE(11)
    ZSB_BNN_CASE(12) ZSB_BNN_CASE(13) ZSB_BNN_CASE(14) ZSB_BNN_CASE(15) ZSB_BNN_CASE(16)
#undef ZSB_BNN_CASE
  }
  int rc = zsb_check_launch("sgmcmc_bnn");
  if (rc || !has_ksum(M)) return rc;
  bnn_mean_k_kernel<<<1, 256, 0, st>>>(
      a.part0, a.part1, (int)blocks, (float)(a.chains * a.H * (a.n_in + 1)),
      (float)(a.chains * (a.H + 1)), mean_k0, mean_k1);
  return zsb_check_launch("sgmcmc_bnn_mean_k");
}

}  // namespace

extern "C" {

// One fused SG-MCMC step for the two-layer BNN regression log-joint (bnn_sgmcmc.py:19-35, 74-91);
// see zsb200.h for which state each method reads and writes.
int zsb_sgmcmc_bnn_step_f32(int method, float* w0, float* w1, float* v0, float* v1, float* aux0,
                            float* aux1, const float* alpha_eff0, const float* alpha_eff1,
                            const float* x, const float* y, int B, int n_in, int H,
                            const float* logstd0, int64_t logstd0_n, const float* logstd1,
                            int64_t logstd1_n, float y_logstd, float n_train, float lr,
                            float friction, float variance_estimate, float decay, float epsilon,
                            float variance_extra, float tune_rate, int second_order, int resample,
                            const float* noise0, const float* noise1, const float* resample0,
                            const float* resample1, uint64_t seed, uint32_t iter, int64_t row0,
                            float* part, float* mean_k0, float* mean_k1, int64_t chains,
                            void* stream) {
  ZSB_REQUIRE(w0 && w1 && x && y && logstd0 && logstd1, "zsb_sgmcmc_bnn_step_f32: null arg");
  ZSB_REQUIRE(chains > 0 && B > 0 && B <= MAX_B && n_in > 0 && n_in + 1 <= MAX_IN1 && H > 0 &&
                  H <= 64 && logstd0_n > 0 && logstd1_n > 0,
              "zsb_sgmcmc_bnn_step_f32: need 0 < B <= 512, n_in <= 15, H <= 64");
  const bool mom = method == SGHMC || method == SGNHT_VEC || method == SGNHT_SCALAR;
  ZSB_REQUIRE(method >= SGHMC && method <= SGNHT_SCALAR, "zsb_sgmcmc_bnn_step_f32: bad method");
  ZSB_REQUIRE(!mom || (v0 && v1), "zsb_sgmcmc_bnn_step_f32: this method needs v0, v1");
  ZSB_REQUIRE((method != PSGLD && method != SGNHT_VEC) || (aux0 && aux1),
              "zsb_sgmcmc_bnn_step_f32: this method needs aux0, aux1");
  ZSB_REQUIRE(method != SGNHT_VEC || (mean_k0 && mean_k1),
              "zsb_sgmcmc_bnn_step_f32: vector SGNHT needs mean_k0, mean_k1");
  ZSB_REQUIRE(method != SGNHT_SCALAR || (alpha_eff0 && alpha_eff1),
              "zsb_sgmcmc_bnn_step_f32: scalar SGNHT needs alpha_eff0, alpha_eff1");
  ZSB_REQUIRE((method != SGHMC && method != SGNHT_SCALAR) || (part && mean_k0 && mean_k1),
              "zsb_sgmcmc_bnn_step_f32: this method needs part, mean_k0, mean_k1");
  ZSB_REQUIRE(method != SGNHT_SCALAR || !resample,
              "zsb_sgmcmc_bnn_step_f32: scalar SGNHT re-draws v before the step, not in it");
  BnnArgs a;
  a.w0 = w0; a.w1 = w1;
  a.v0 = method == PSGLD ? aux0 : v0; a.v1 = method == PSGLD ? aux1 : v1;
  a.al0 = method == SGNHT_VEC ? aux0 : nullptr; a.al1 = method == SGNHT_VEC ? aux1 : nullptr;
  a.k0 = method == SGNHT_VEC ? mean_k0 : nullptr; a.k1 = method == SGNHT_VEC ? mean_k1 : nullptr;
  a.aeff0 = alpha_eff0; a.aeff1 = alpha_eff1;
  a.x = x; a.y = y;
  a.logstd0 = logstd0; a.logstd0_n = logstd0_n; a.logstd1 = logstd1; a.logstd1_n = logstd1_n;
  a.noise0 = noise0; a.noise1 = noise1; a.rs0 = resample0; a.rs1 = resample1;
  const int cap = ZSB_NUM_SMS * 8;
  a.part0 = part; a.part1 = part ? part + cap : nullptr;
  a.chains = chains; a.B = B; a.n_in = n_in; a.H = H;
  a.y_logstd = y_logstd; a.n_train = n_train; a.lr = lr; a.alpha = friction;
  a.beta = variance_estimate;
  a.decay = decay; a.epsilon = epsilon; a.var_extra = variance_extra; a.tune_rate = tune_rate;
  a.hl = mul(0.5f, lr); a.omd = sub(1.f, decay); a.ht = mul(0.5f, tune_rate);
  a.second_order = mom ? second_order : 0; a.resample = mom ? resample : 0;
  a.seed = seed; a.iter = iter; a.row0 = row0;
  switch (method) {
    case SGHMC: return bnn_launch<SGHMC>(a, mean_k0, mean_k1, stream);
    case SGLD: return bnn_launch<SGLD>(a, mean_k0, mean_k1, stream);
    case PSGLD: return bnn_launch<PSGLD>(a, mean_k0, mean_k1, stream);
    case SGNHT_VEC: return bnn_launch<SGNHT_VEC>(a, mean_k0, mean_k1, stream);
    default: return bnn_launch<SGNHT_SCALAR>(a, mean_k0, mean_k1, stream);
  }
}

// One fused SGHMC step (sgmcmc.py:326-371); mean_k: 2 floats, one per latent.
int zsb_sgmcmc_sghmc_bnn_f32(float* w0, float* w1, float* v0, float* v1, const float* x,
                             const float* y, int B, int n_in, int H, const float* logstd0,
                             int64_t logstd0_n, const float* logstd1, int64_t logstd1_n,
                             float y_logstd, float n_train, float lr, float alpha, float beta,
                             int second_order, int resample, const float* noise0,
                             const float* noise1, const float* resample0, const float* resample1,
                             uint64_t seed, uint32_t iter, int64_t row0, float* part,
                             float* mean_k, int64_t chains, void* stream) {
  ZSB_REQUIRE(mean_k, "zsb_sgmcmc_sghmc_bnn_f32: null arg");
  return zsb_sgmcmc_bnn_step_f32(SGHMC, w0, w1, v0, v1, nullptr, nullptr, nullptr, nullptr, x, y,
                                 B, n_in, H, logstd0, logstd0_n, logstd1, logstd1_n, y_logstd,
                                 n_train, lr, alpha, beta, 0.f, 0.f, 0.f, 0.f, second_order,
                                 resample, noise0, noise1, resample0, resample1, seed, iter, row0,
                                 part, mean_k, mean_k + 1, chains, stream);
}

}  // extern "C"
