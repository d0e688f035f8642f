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
//   EPI 16 out[r, j] = act(l + res[r, j])                         biased layer with a residual added
//          before the ReLU (the resnet blocks of vae_conv.py:39-53); res [R, J] is read through the
//          observation loads of EPI 1 (x_obs = res, n_x = R)
//
// fp32 accuracy on fp16 tensor cores: both operands are pre-split into scaled fp16 hi + lo planes
// (zsb_split16_pad_f32), three fp16 wgmma products per k-step accumulate hi*hi + hi*lo + lo*hi
// in fp32 (dropped term ~2^-22 relative) -- the scheme of the dense-Gaussian HMC kernel
// (hmc_dense_tc.cu), whose persistent pipeline (tc_pipeline_kernel: TMA producer warp, MMA
// warpgroup, 4 epilogue warps, 128 features x 128 rows per unit) this product shares.  As there,
// the product is computed transposed (accumulator row = feature j, column = row r) so an epilogue
// warp touches 32 consecutive features of one row per instruction: coalesced x loads and out stores.
#include "tc_common.cuh"

#include <type_traits>

extern "C" int zsb_linear_tc_kpad(int K);
extern "C" int zsb_linear_tc_slices(int64_t R, int J, int K);
extern "C" int zsb_linear_tc_nparts(int J);

namespace {

__device__ __forceinline__ float bern_lp(float x, float l) {   // -sigmoid_cross_entropy(x, l)
  return -(fmaxf(l, 0.f) - l * x + __logf(1.f + __expf(-fabsf(l))));
}

// Scale of the fp16 operand plane of a 0/1 sample (EPI 4): the power of two zsb_split16_* picks
// for a matrix whose max |.| is 1, so the sample's plane is the hi plane the split would make, and
// its lo plane is exactly zero.
constexpr float BIN_SCALE = 2048.f;

// Epilogues with S >= 1 rows of samples per logit row r (sample row s * R + r):
//   EPI 4  Bernoulli sampling: h = (u < sigmoidf_(l)) with u injected or drawn from Philox keyed as
//          zsb_sample_bernoulli_i32 keys element (s R + r) J + j; writes h (float or int32), its fp16
//          operand plane h * BIN_SCALE [S R][kpad(J)] (pad columns zero) and the epi-1 partial rows
//          of log Bernoulli(l).log_prob(h) ([nparts][S R])
//   EPI 5  the epi-1 partial rows of the given samples x[s R + r] against logit row r
//   EPI 6  out[r, j] = sum_s g[s R + r] * (x[s R + r, j] - sigmoid(l))     (d/dl of EPI 5)
//
// Class-conditioned epilogues (a dense layer of [h, onehot(y)]: the one-hot block of the product is
// column y of the class weights, gathered from the class table ctab [C, J] instead of multiplied):
//   EPI 7  out[r, j] = act(l + ctab[y, j]) with y = cls[r % n_cls]; a row whose y is outside
//          [0, C) is written as NaN and ctab is not read for it
//   EPI 8  out[c R + r, j] = act(l + ctab[c, j]) for every class c (class-major), from one product
//          over the R rows.  The same additions in the same order as EPI 7, so the result equals
//          EPI 7 on the input tiled C times bit for bit.
//
// Batch-normalised epilogues (no bias; variational_dropout.py:26-37, tf.contrib.layers.batch_norm):
//   EPI 9  out[r, j] = a = l (the pre-activation), and per 128-row tile t the moment partials of
//          column j over the tile's rows, part[2 t J + j] = mean and part[(2 t + 1) J + j] = M2
//          (sum of squared deviations from the tile mean); the tile's count is min(128, R - 128 t)
//   EPI 10 out[r, j] = act((l - bn_stats[j]) * bn_stats[J + j] + bn_beta[j]), bn_stats = (mean,
//          rsqrt(var + eps)) of the moving statistics (evaluation mode)
//   EPI 11 EPI 10 with batch norm's learned scale gamma (tf.layers.batch_normalization,
//          bernoulli_latent_vae.py:26-43):
//          out[r, j] = act(xhat * bn_gamma[j] + bn_beta[j]), xhat = (l - mean) rstd, and, when pre
//          is not NULL, pre[r, j] = l: what the gradient of gamma needs (xhat is never rebuilt
//          from out, which the ReLU and gamma = 0 lose)
//
// Categorical epilogues (J = C classes, 1 <= C <= 128, so one feature block holds a whole logit
// row; S draws per logit row, draw d = s R + r; onehot_categorical of a dense layer,
// vae_ssl_adaptive_is.py:61-68):
//   EPI 12 one-hot sampling: cls[d] = the class drawn from softmax(l[r]), one uniform per draw
//          (u_in[d], or word 0 of the Philox block zsb_sample_categorical_i32 keys on d), onehot
//          [S R, C] (float or int32) and logq[d] = l[y] - logsumexp(l[r])
//   EPI 13 out[d] = sum_j given[d % n_g, j] (l[r, j] - logsumexp(l[r]))
//   EPI 14 out[r, j] = sum_s gout[d] (given_j - (sum_i given_i) softmax(l[r])_j), given = row
//          d % n_g (d/dl of EPI 13)
//
// Gaussian-sampling epilogue (D features, 1 <= D <= 256; the two heads packed in blocks of 64
// columns, [mean 0..63 | logstd 0..63 | mean 64..127 | ...], so one 128-feature tile holds mean_j
// and logstd_j of the same 64 features; bn.normal of two dense heads, vae_ssl_adaptive_is.py:53-68):
//   EPI 15 z[s R + r, j] = eps * expf(ls) + mu with eps the standard normal
//          zsb_reparam_normal_f32 draws for element (s R + r) D + j (or injected), and the partial
//          rows of log N(z; mu, exp(ls)) summed over the features
//
// The descriptor tc_pipeline_kernel runs, LinW<E, EPI, MN, Z>, is a LinCore (the product) plus the
// fields of one epilogue family E: RowsEpi (EPI 0 - 2, 16), SamplesEpi (4 - 6), ClassEpi (7, 8),
// BnEpi (9 - 11), CatEpi (12 - 14) or NormalEpi (15).

// What a product's units past its first n_tiles are (unit u runs output tile u % n_tiles), as each
// epilogue family declares it:
//   K_SLICES       slices of the contraction, kb_per k-blocks each, summed afterwards
//   SAMPLE_CHUNKS  chunks of s_per sample rows, each over the whole contraction
//   TILES          none: one unit per tile, over the whole contraction
enum Units { TILES, K_SLICES, SAMPLE_CHUNKS };

// A unit as one epilogue lane sees it: slice or chunk `sub`, feature block nb and this lane's
// feature j in it, row tile `tile` and its first row r0
struct Unit {
  int sub; int nb; int j; int64_t tile; int64_t r0;
};

// The product acc[j, r] = sum_k A[j, k] B[r, k] over J features j (operand A: the weight rows of
// the forward product) and R rows r (operand B), on fp16 hi/lo planes of A and B at the
// power-of-two scales scale_w[0] and scale_h[0].
// MN (bit 0: operand A, bit 1: operand B; EPI 0 only): the operand is read in a row-major plane
// layout [contraction rows, features] -- MN-major (transposed) wgmma operand.  MN = 3: weight
// gradient dW = g^T h from the row-major planes of g and h; MN = 1: input gradient dh = g W with
// A = the FORWARD planes of W [J, K] (no W^T copy): no product of a dense layer needs a transposed
// copy of anything.  A stage then holds, per plane, two TMA boxes of 64 contraction rows x 64
// features (128-byte rows, SWIZZLE_128B; see gmma_desc).
// Z: bit 0 / 1 = the lo plane of operand A / B is zero (a 0/1 sample, see mma_kblock): it is
// neither loaded nor multiplied.
template <int MN, int Z>
struct LinCore {
  static constexpr int KIND = 1, RB = 128, MNA = MN & 1, MNB = (MN >> 1) & 1, ZLO = Z;
  // the weight gradient (MN = 3) contracts over all the rows of a batch -- 4096 k-blocks in the
  // IWAE decoder at K = 64, N = 4096, up to 1024 in one split-K slice -- so its units add their
  // accumulator into the shared tile every 8 k-blocks (PromoteOf in tc_common.cuh); the other
  // products contract over a layer's width, a few dozen k-blocks at most
  static constexpr int PROMOTE_KB = MN == 3 ? 8 : 0;
  static constexpr uint32_t TX = Cfg<RB>::STAGE - ((Z & 1) ? Cfg<RB>::A_TILE : 0) -
                                 ((Z & 2) ? Cfg<RB>::B_TILE : 0);
  CUtensorMap map_whi, map_wlo, map_hhi, map_hlo;
  const float* scale_w; const float* scale_h;
  int64_t R; int J;
  int n_blk; int64_t n_tiles; int n_kb_all; int kb_per; int k_slices;

  __host__ __device__ __forceinline__ int64_t units() const { return n_tiles * k_slices; }
  template <Units U>
  __device__ __forceinline__ void kb_range(int64_t uu, int& kb0, int& kb1) const {
    if (U != K_SLICES) {
      kb0 = 0;
      kb1 = n_kb_all;
      return;
    }
    kb0 = (int)(uu / n_tiles) * kb_per;
    kb1 = min(kb0 + kb_per, n_kb_all);
  }
  template <Units U>
  __device__ __forceinline__ Unit unit(int64_t uu, int quarter, int lane) const {
    const int64_t u = U == TILES ? uu : uu % n_tiles;
    Unit t;
    t.sub = U == TILES ? 0 : (int)(uu / n_tiles);
    t.nb = (int)(u % n_blk);
    t.j = t.nb * BM + quarter * 32 + lane;
    t.tile = u / n_blk;
    t.r0 = t.tile * BN;
    return t;
  }
  __device__ __forceinline__ float acc_scale() const {   // powers of two: exact
    return 1.f / (scale_w[0] * scale_h[0]);
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
        if (!(Z & 1)) tma_load_2d(sa + C::A_TILE + o, &map_wlo, fb, j0 + 64 * b, kb * 64);
      }
    } else {
      tma_load_2d(sa, &map_whi, fb, kb * 64, j0);
      if (!(Z & 1)) tma_load_2d(sa + C::A_TILE, &map_wlo, fb, kb * 64, j0);
    }
    if (MN & 2) {
#pragma unroll
      for (int b = 0; b < 2; ++b) {
        const uint32_t o = (uint32_t)b * 8192u;
        tma_load_2d(sa + 2 * C::A_TILE + o, &map_hhi, fb, r0 + 64 * b, kb * 64);
        if (!(Z & 2))
          tma_load_2d(sa + 2 * C::A_TILE + C::B_TILE + o, &map_hlo, fb, r0 + 64 * b, kb * 64);
      }
    } else {
      tma_load_2d(sa + 2 * C::A_TILE, &map_hhi, fb, kb * 64, r0);
      if (!(Z & 2)) tma_load_2d(sa + 2 * C::A_TILE + C::B_TILE, &map_hlo, fb, kb * 64, r0);
    }
  }
};

template <class E, int EPI, int MN = 0, int Z = 0>
struct LinW : LinCore<MN, Z> {
  E e;
  struct EpiState { float amax = 0.f; };   // max |stored output|: the consumer's fp16-split scale
  __device__ __forceinline__ void kb_range(int64_t uu, int& kb0, int& kb1) const {
    LinCore<MN, Z>::template kb_range<E::UNITS>(uu, kb0, kb1);
  }
  __device__ __forceinline__ void epilogue(int64_t uu, uint32_t trow, int quarter, int lane,
                                           EpiState& st) const {
    e.template run<EPI>(*this, uu, trow, quarter, lane, st.amax);
  }
  __device__ __forceinline__ void epi_finish(EpiState& st, int, int lane) const {
    if (E::folds_amax(EPI) && e.amax_scale)   // NaN / inf never win (fmaxf drops NaN)
      fold_amax(e.amax_scale, st.amax <= 3.0e38f ? st.amax : 0.f, lane);
  }
};

// EPI 9 - 11: this lane's feature j over the tile's rows.  EPI 9 reads the accumulator twice:
// once for the tile mean, once for M2 about it (never a sum of squares, which cancels).
struct BnEpi {
  static constexpr Units UNITS = TILES;
  // EPI 9 is given no amax_scale
  __host__ __device__ static constexpr bool folds_amax(int) { return true; }
  const float* bn_stats; const float* bn_beta;
  float* out; float* part; int relu; float* amax_scale;
  const float* bn_gamma; float* pre;                          // EPI 11 only

  template <int EPI, class Core>
  __device__ __forceinline__ void run(const Core& core, int64_t u, uint32_t trow, int quarter,
                                      int lane, float& amax) const {
    const int64_t& R = core.R;
    const int& J = core.J;
    const float acc_scale = core.acc_scale();
    const Unit pos = core.template unit<UNITS>(u, quarter, lane);
    const int j = pos.j;
    const bool j_ok = j < J;
    const int64_t tile = pos.tile;
    const int64_t r0 = pos.r0;
    if (EPI == 9) {
      float sum = 0.f;
#pragma unroll 1
      for (int c = 0; c < BN; c += 16) {
        const int64_t rbase = r0 + c;
        if (rbase >= R) break;                                 // warp-uniform
        uint32_t v[16];
        acc_ld16(trow + 4u * (uint32_t)c, v);
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
          if (j_ok && rbase + jj < R) {
            const float l = __uint_as_float(v[jj]) * acc_scale;
            out[(rbase + jj) * J + j] = l;
            sum += l;
          }
      }
      const float mean = sum / (float)min((int64_t)BN, R - r0);
      float m2 = 0.f;
#pragma unroll 1
      for (int c = 0; c < BN; c += 16) {
        const int64_t rbase = r0 + c;
        if (rbase >= R) break;
        uint32_t v[16];
        acc_ld16(trow + 4u * (uint32_t)c, v);
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
          if (rbase + jj < R) {
            const float d = __uint_as_float(v[jj]) * acc_scale - mean;
            m2 = fmaf(d, d, m2);
          }
      }
      if (j_ok) {
        part[2 * tile * J + j] = mean;
        part[(2 * tile + 1) * J + j] = m2;
      }
    } else {
      const float mu = j_ok ? bn_stats[j] : 0.f, rs = j_ok ? bn_stats[J + j] : 0.f;
      const float bt = j_ok ? bn_beta[j] : 0.f;
      const float gm = (EPI == 11 && j_ok) ? bn_gamma[j] : 1.f;
#pragma unroll 1
      for (int c = 0; c < BN; c += 16) {
        const int64_t rbase = r0 + c;
        if (rbase >= R) break;
        uint32_t v[16];
        acc_ld16(trow + 4u * (uint32_t)c, v);
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
          if (j_ok && rbase + jj < R) {
            const float l = __uint_as_float(v[jj]) * acc_scale;
            float y;
            if (EPI == 11) {
              y = fmaf((l - mu) * rs, gm, bt);
              if (pre) pre[(rbase + jj) * J + j] = l;
            } else {
              y = (l - mu) * rs + bt;
            }
            if (relu) y = fmaxf(y, 0.f);
            out[(rbase + jj) * J + j] = y;
            amax = fmaxf(amax, fabsf(y));
          }
      }
    }
  }
};

// EPI 7 / 8, per 16-row block of this lane's feature j
struct ClassEpi {
  static constexpr Units UNITS = TILES;
  __host__ __device__ static constexpr bool folds_amax(int) { return true; }
  const float* bias; const float* ctab; int C; const int32_t* cls; int64_t n_cls;
  float* out; int relu; float* amax_scale;

  template <int EPI, class Core>
  __device__ __forceinline__ void run(const Core& core, int64_t u, uint32_t trow, int quarter,
                                      int lane, float& amax) const {
    const int64_t& R = core.R;
    const int& J = core.J;
    const float acc_scale = core.acc_scale();
    const Unit pos = core.template unit<UNITS>(u, quarter, lane);
    const int j = pos.j;
    const bool j_ok = j < J;
    const float b_j = (j_ok && bias) ? bias[j] : 0.f;
    const int64_t r0 = pos.r0;
    const float* __restrict__ tj = ctab + j;                 // ctab[c, j] = tj[c * J]
    // the one rounding order of both forms: (acc * scale + bias) + table entry, then ReLU
    auto act = [&](float l, float t) {
      const float y = l + t;
      return relu ? fmaxf(y, 0.f) : y;
    };
#pragma unroll 1
    for (int c = 0; c < BN; c += 16) {
      const int64_t rbase = r0 + c;
      if (rbase >= R) break;                                 // warp-uniform
      uint32_t v[16];
      acc_ld16(trow + 4u * (uint32_t)c, v);
      float l[16];
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) l[jj] = fmaf(__uint_as_float(v[jj]), acc_scale, b_j);
      if (EPI == 7) {
        int64_t yr = rbase % n_cls;
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const int64_t r = rbase + jj;
          if (j_ok && r < R) {
            const int k = __ldg(cls + yr);
            float y;
            if (k >= 0 && k < C) {
              y = act(l[jj], __ldg(tj + (int64_t)k * J));
              amax = fmaxf(amax, fabsf(y));
            } else {
              y = __int_as_float(0x7fffffff);               // NaN: the class is not in the table
            }
            out[r * J + j] = y;
          }
          if (++yr == n_cls) yr = 0;
        }
      } else {
#pragma unroll 1
        for (int k = 0; k < C; ++k) {
          if (!j_ok) break;
          const float t = __ldg(tj + (int64_t)k * J);
          float* __restrict__ po = out + ((int64_t)k * R + rbase) * J + j;
#pragma unroll
          for (int jj = 0; jj < 16; ++jj)
            if (rbase + jj < R) {
              const float y = act(l[jj], t);
              po[(int64_t)jj * J] = y;
              amax = fmaxf(amax, fabsf(y));
            }
        }
      }
    }
  }
};

// EPI 4 - 6: per 16-row block of this lane's feature j, the logits once, then each of the sample
// rows s0 .. s1 of the unit's chunk of those logit rows.  EPI 4 / 5 split the S sample rows of a
// tile into chunks of s_per rows, each its own unit, so a layer with few logit rows and many draws
// still fills every SM.  The price: each chunk recomputes the tile's whole product (about 125
// times for the proposal's first layer at 100 rows and K = 1000).  EPI 4 also runs one Philox-10
// per element, four times the work of the elementwise sampler, which shares one draw among four
// elements; it keeps the sampler's keying so the samples are bit-identical.  Neither cost is
// measured on its own; the layer as a whole is (scripts/bench_sbn.py).  EPI 6 sums over all S
// draws in one chunk.
struct SamplesEpi {
  static constexpr Units UNITS = SAMPLE_CHUNKS;
  __host__ __device__ static constexpr bool folds_amax(int epi) { return epi == 6; }
  const float* bias; const float* x_obs; const float* gout; float* out; float* part;
  int S; int s_per; const float* u_in; uint64_t seed; uint32_t iter; const uint32_t* epoch;
  int h_int; __half* pl_out; float* amax_scale;

  template <int EPI, class Core>
  __device__ __forceinline__ void run(const Core& core, int64_t uu, uint32_t trow, int quarter,
                                      int lane, float& amax) const {
    const int64_t& R = core.R;
    const int& J = core.J;
    const float acc_scale = core.acc_scale();
    const Unit pos = core.template unit<UNITS>(uu, quarter, lane);
    const int s0 = pos.sub * s_per, s1 = min(S, s0 + s_per);
    const int nb = pos.nb;
    const int j = pos.j;
    const bool j_ok = j < J;
    const int Jp = ((J + 63) / 64) * 64;
    const bool col_ok = j < Jp;                    // EPI 4 plane: real and zero-padding columns
    const float b_j = (j_ok && bias) ? bias[j] : 0.f;
    const int64_t r0 = pos.r0;
    const int64_t part_row = (int64_t)(nb * 4 + quarter) * ((int64_t)S * R);
    const uint32_t it = (EPI == 4) ? iter + (epoch ? *epoch : 0u) : 0u;
#pragma unroll 1
    for (int c = 0; c < BN; c += 16) {
      const int64_t rbase = r0 + c;
      uint32_t v[16];
      acc_ld16(trow + 4u * (uint32_t)c, v);
      float l[16], sg[16], dl[16];
#pragma unroll
      for (int jj = 0; jj < 16; ++jj) {
        l[jj] = fmaf(__uint_as_float(v[jj]), acc_scale, b_j);
        sg[jj] = sigmoidf_(l[jj]);
        dl[jj] = 0.f;
      }
#pragma unroll 1
      for (int s = s0; s < s1; ++s) {
        float lpv[16];
#pragma unroll
        for (int jj = 0; jj < 16; ++jj) {
          const int64_t r = rbase + jj;
          const bool ok = j_ok && r < R;
          const int64_t srow = (int64_t)s * R + r;
          const int64_t i = srow * J + j;           // element of the flattened [S, R, J] sample
          float x = 0.f;
          if (EPI == 4) {
            float uu;
            if (u_in) {
              uu = ok ? __ldg(u_in + i) : 1.f;
            } else {
              const Philox4 p = philox4x32_10((uint32_t)(i >> 2), (uint32_t)((uint64_t)i >> 34), it,
                                              ZSB_STREAM_SAMPLE, (uint32_t)seed,
                                              (uint32_t)(seed >> 32));
              const uint32_t w = (i & 3) == 0 ? p.x : (i & 3) == 1 ? p.y : (i & 3) == 2 ? p.z : p.w;
              uu = u32_to_uniform(w);
            }
            const int hb = (ok && uu < sg[jj]) ? 1 : 0;
            x = (float)hb;
            if (ok) {
              if (h_int) reinterpret_cast<int32_t*>(out)[i] = hb;
              else out[i] = x;
            }
            if (col_ok && r < R) pl_out[srow * Jp + j] = __float2half_rn(x * BIN_SCALE);
          } else if (ok) {
            x = __ldg(x_obs + i);
          }
          if (EPI == 6) {
            const float g = r < R ? __ldg(gout + srow) : 0.f;
            dl[jj] += g * (x - sg[jj]);
          } else {
            lpv[jj] = ok ? bern_lp(x, l[jj]) : 0.f;
          }
        }
        if (EPI != 6) {
          const float sum = warp_transpose_sum16(lpv, lane);
          if (lane < 16 && rbase + lane < R) part[part_row + (int64_t)s * R + rbase + lane] = sum;
        }
      }
      if (EPI == 6) {
#pragma unroll
        for (int jj = 0; jj < 16; ++jj)
          if (j_ok && rbase + jj < R) {
            out[(rbase + jj) * J + j] = dl[jj];
            amax = fmaxf(amax, fabsf(dl[jj]));
          }
      }
    }
  }
};

// ZSB_STREAM_CATEGORICAL of samplers.cu: EPI 12 draws what zsb_sample_categorical_i32 draws
constexpr uint32_t CAT_STREAM = 6u;
constexpr int CAT_MAX_C = 128;
constexpr int CAT_PER_LANE = CAT_MAX_C / 32;

// EPI 12 - 14.  The accumulator's natural layout gives a lane one class of 16 rows; a draw needs
// all C logits of one row, laid out as categorical_sample_kernel (samplers.cu) lays them out: one
// warp per draw, lane l holding the ceil(C / 32) contiguous classes from l * ceil(C / 32).  So each
// epilogue warp takes 32 of the tile's rows (the tile is complete once tfull has fired, and no warp
// overwrites it before all four have arrived on tempty) and reads each row's logits from the whole
// tile in the sampler's layout.  Per row the max, the sum of exps and its prefix scan are formed
// once, in the sampler's order; each draw of the unit's chunk then needs only its uniform.
// Cost (H100, 4e5 rows, 500 -> 10, scripts/bench_ssl_ais.py): the EPI 12 and EPI 13 launches
// take 0.83 ms where EPI 0 over the same operands takes 0.38 ms, and EPI 14 takes 0.90 ms.  Rows go
// one at a time, each a chain of dependent shuffles, and the reads of one row's classes are bank
// conflicts (class pitch ACC_LD = 132 words: 4-way for C <= 32, 16-way at C = 128).  Several rows
// in flight per warp would hide that latency; not done.
struct CatEpi {
  static constexpr Units UNITS = SAMPLE_CHUNKS;
  __host__ __device__ static constexpr bool folds_amax(int epi) { return epi == 14; }
  const float* bias; const float* given; int64_t n_g; const float* gout; float* out;
  int32_t* cls; void* onehot; int h_int; float* logq;
  int S; int s_per; const float* u_in; uint64_t seed; uint32_t iter; const uint32_t* epoch;
  float* amax_scale;

  template <int EPI, class Core>
  __device__ __forceinline__ void run(const Core& core, int64_t uu, uint32_t trow, int quarter,
                                      int lane, float& amax) const {
    const int64_t& R = core.R;
    const int& C = core.J;
    const float acc_scale = core.acc_scale();
    const Unit pos = core.template unit<UNITS>(uu, quarter, lane);
    const int s0 = pos.sub * s_per, s1 = min(S, s0 + s_per);
    const uint32_t acc0 = trow - (uint32_t)((quarter * 32 + lane) * ACC_LD * 4);
    const int chunk = (C + 31) / 32;
    const int c0 = lane * chunk, c1 = min(C, c0 + chunk);
    const uint32_t it = (EPI == 12) ? iter + (epoch ? *epoch : 0u) : 0u;
    float b[CAT_PER_LANE];
#pragma unroll
    for (int t = 0; t < CAT_PER_LANE; ++t)
      b[t] = (c0 + t < c1 && bias) ? __ldg(bias + c0 + t) : 0.f;
#pragma unroll 1
    for (int i = 0; i < 32; ++i) {
      const int rl = quarter * 32 + i;
      const int64_t r = pos.r0 + rl;
      if (r >= R) break;                                     // warp-uniform
      float l[CAT_PER_LANE], e[CAT_PER_LANE];
      float m = -INFINITY;
#pragma unroll
      for (int t = 0; t < CAT_PER_LANE; ++t) {
        l[t] = 0.f;
        if (c0 + t < c1) {
          float a;
          asm volatile("ld.shared.f32 %0, [%1];"
                       : "=f"(a) : "r"(acc0 + (uint32_t)(((c0 + t) * ACC_LD + rl) * 4)));
          l[t] = fmaf(a, acc_scale, b[t]);
          m = fmaxf(m, l[t]);
        }
      }
      m = warp_max(m);
      float s = 0.f;
#pragma unroll
      for (int t = 0; t < CAT_PER_LANE; ++t) {
        e[t] = 0.f;
        if (c0 + t < c1) {
          e[t] = expf(l[t] - m);
          s += e[t];
        }
      }
      float pre = s;                                         // inclusive prefix of the lane sums
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const float v = __shfl_up_sync(0xffffffffu, pre, o);
        if (lane >= o) pre += v;
      }
      const float total = __shfl_sync(0xffffffffu, pre, 31);
      const float log_total = logf(total);
      if (EPI == 12) {
        int last = -1;                                       // last class with non-zero mass
#pragma unroll
        for (int t = 0; t < CAT_PER_LANE; ++t)
          if (c0 + t < c1 && e[t] > 0.f) last = c0 + t;
#pragma unroll 1
        for (int sd = s0; sd < s1; ++sd) {
          const int64_t d = (int64_t)sd * R + r;
          float u;
          if (u_in) {
            u = __ldg(u_in + d);
          } else {
            const Philox4 p = philox4x32_10(0u, (uint32_t)d, it ^ (uint32_t)((uint64_t)d >> 32),
                                            CAT_STREAM, (uint32_t)seed, (uint32_t)(seed >> 32));
            u = u32_to_uniform(p.x);
          }
          const float target = u * total;
          // first lane whose inclusive prefix exceeds the target
          const unsigned hit = __ballot_sync(0xffffffffu, pre > target && s > 0.f);
          int pick;
          if (hit) {
            const int src = __ffs(hit) - 1;
            const float base = __shfl_sync(0xffffffffu, pre - s, src);
            pick = -1;
            if (lane == src) {
              float acc = base;
              int lst = c0;
#pragma unroll
              for (int t = 0; t < CAT_PER_LANE; ++t) {
                if (c0 + t < c1 && pick < 0) {
                  if (e[t] > 0.f) lst = c0 + t;
                  acc += e[t];
                  if (acc > target) pick = c0 + t;
                }
              }
              if (pick < 0) pick = lst;                      // round-off at the chunk's end
            }
            pick = __shfl_sync(0xffffffffu, pick, src);
          } else {
            // u * total rounded up to the total: last class with non-zero mass
            int lst = last;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) lst = max(lst, __shfl_xor_sync(0xffffffffu, lst, o));
            pick = lst < 0 ? 0 : lst;
          }
          // l[pick] - logsumexp(l) = (l[pick] - m) - log(total), from the lane that holds it
          float lp = 0.f;
#pragma unroll
          for (int t = 0; t < CAT_PER_LANE; ++t)
            if (c0 + t == pick) lp = (l[t] - m) - log_total;
          lp = __shfl_sync(0xffffffffu, lp, min(pick / chunk, 31));
          if (lane == 0) {
            cls[d] = pick;
            logq[d] = lp;
          }
#pragma unroll
          for (int t = 0; t < CAT_PER_LANE; ++t)
            if (c0 + t < c1) {
              const int64_t k = d * C + c0 + t;
              if (h_int) reinterpret_cast<int32_t*>(onehot)[k] = (c0 + t == pick) ? 1 : 0;
              else reinterpret_cast<float*>(onehot)[k] = (c0 + t == pick) ? 1.f : 0.f;
            }
        }
      } else if (EPI == 13) {
#pragma unroll 1
        for (int sd = s0; sd < s1; ++sd) {
          const int64_t d = (int64_t)sd * R + r;
          const float* __restrict__ gr = given + (d % n_g) * C;
          float lp = 0.f;
#pragma unroll
          for (int t = 0; t < CAT_PER_LANE; ++t)
            if (c0 + t < c1) lp = fmaf(__ldg(gr + c0 + t), (l[t] - m) - log_total, lp);
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) lp += __shfl_xor_sync(0xffffffffu, lp, o);
          if (lane == 0) out[d] = lp;
        }
      } else {
        const float inv_total = 1.f / total;
        float dl[CAT_PER_LANE];
#pragma unroll
        for (int t = 0; t < CAT_PER_LANE; ++t) dl[t] = 0.f;
#pragma unroll 1
        for (int sd = 0; sd < S; ++sd) {
          const int64_t d = (int64_t)sd * R + r;
          const float* __restrict__ gr = given + (d % n_g) * C;
          const float g = __ldg(gout + d);
          float x[CAT_PER_LANE], n = 0.f;
#pragma unroll
          for (int t = 0; t < CAT_PER_LANE; ++t) {
            x[t] = (c0 + t < c1) ? __ldg(gr + c0 + t) : 0.f;
            n += x[t];
          }
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(0xffffffffu, n, o);
#pragma unroll
          for (int t = 0; t < CAT_PER_LANE; ++t)
            dl[t] = fmaf(g, x[t] - n * (e[t] * inv_total), dl[t]);
        }
#pragma unroll
        for (int t = 0; t < CAT_PER_LANE; ++t)
          if (c0 + t < c1) {
            out[r * C + c0 + t] = dl[t];
            amax = fmaxf(amax, fabsf(dl[t]));
          }
      }
    }
  }
};

constexpr float NORMAL_HALF_LOG_2PI = 0.9189385332046727f;   // kHalfLog2Pi of distributions.cu
constexpr int NORMAL_MAX_D = 256;

// EPI 15.  The heads of feature j sit in accumulator rows f and 64 + f of the tile (f = j % 64), so
// a lane takes one feature over half of the tile's rows: warps 0 / 1 features 0 - 31 / 32 - 63 of
// rows 0 - 63, warps 2 / 3 the same features of rows 64 - 127 (every warp reads rows another warp
// was given; the tile is complete once tfull has fired, as for CatEpi).  Per 4-row block, mu, std
// and the log-density's constants once, then each sample row of the unit's chunk.  Each element
// runs its own Philox-10 and one Box-Muller pair, twice the transcendental work and four times the
// Philox work of zsb_reparam_normal_f32, which shares one block among four elements; the keying is
// the same, so z is that sampler's draw bit for bit.  The partial row of warp q for feature block nb
// is nb * 2 + (q & 1): Dp / 32 rows in all, summed in a fixed order.
struct NormalEpi {
  static constexpr Units UNITS = SAMPLE_CHUNKS;
  __host__ __device__ static constexpr bool folds_amax(int) { return true; }
  const float* bias; int D; float* z; float* part; float* mean_out; float* logstd_out;
  int S; int s_per; const float* eps_in; uint64_t seed; uint32_t iter; const uint32_t* epoch;
  float* amax_scale;

  template <int EPI, class Core>
  __device__ __forceinline__ void run(const Core& core, int64_t uu, uint32_t trow, int quarter,
                                      int lane, float& amax) const {
    const int64_t& R = core.R;
    const float acc_scale = core.acc_scale();
    const Unit pos = core.template unit<UNITS>(uu, quarter, lane);
    const int s0 = pos.sub * s_per, s1 = min(S, s0 + s_per);
    const int f = (quarter & 1) * 32 + lane;
    const int j = pos.nb * 64 + f;
    const bool j_ok = j < D;
    const int half = quarter >> 1;
    const uint32_t acc0 = trow - (uint32_t)((quarter * 32 + lane) * ACC_LD * 4);
    const uint32_t row_mu = acc0 + (uint32_t)((f * ACC_LD + 64 * half) * 4);
    const uint32_t row_ls = row_mu + (uint32_t)(64 * ACC_LD * 4);
    const float bm = (j_ok && bias) ? __ldg(bias + pos.nb * 128 + f) : 0.f;
    const float bl = (j_ok && bias) ? __ldg(bias + pos.nb * 128 + 64 + f) : 0.f;
    const int64_t SR = (int64_t)S * R;
    const int64_t part_row = (int64_t)(pos.nb * 2 + (quarter & 1)) * SR;
    const uint32_t it = iter + (epoch ? *epoch : 0u);
#pragma unroll 1
    for (int c = 0; c < 64; c += 4) {
      const int64_t rbase = pos.r0 + 64 * half + c;
      if (rbase >= R) break;                                 // warp-uniform
      float vm[4], vl[4], mu[4], sd[4], c1[4], hv[4];
      asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                   : "=f"(vm[0]), "=f"(vm[1]), "=f"(vm[2]), "=f"(vm[3])
                   : "r"(row_mu + 4u * (uint32_t)c));
      asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                   : "=f"(vl[0]), "=f"(vl[1]), "=f"(vl[2]), "=f"(vl[3])
                   : "r"(row_ls + 4u * (uint32_t)c));
#pragma unroll
      for (int jj = 0; jj < 4; ++jj) {
        mu[jj] = fmaf(vm[jj], acc_scale, bm);
        const float ls = fmaf(vl[jj], acc_scale, bl);
        const int64_t r = rbase + jj;
        if (pos.sub == 0 && j_ok && r < R) {
          if (mean_out) mean_out[r * D + j] = mu[jj];
          if (logstd_out) logstd_out[r * D + j] = ls;
        }
        sd[jj] = expf(ls);
        c1[jj] = -NORMAL_HALF_LOG_2PI - ls;
        hv[jj] = 0.5f * expf(-2.f * ls);
      }
#pragma unroll 1
      for (int s = s0; s < s1; ++s) {
        float lpv[4];
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) {
          const int64_t r = rbase + jj;
          const bool ok = j_ok && r < R;
          const int64_t i = ((int64_t)s * R + r) * D + j;      // element of the [S, R, D] sample
          const float e = !ok ? 0.f : eps_in ? __ldg(eps_in + i) : philox_normal_at(seed, it, i);
          const float zz = e * sd[jj] + mu[jj];                 // zsb_reparam_normal_f32's rounding
          const float d = zz - mu[jj];
          lpv[jj] = ok ? c1[jj] - hv[jj] * d * d : 0.f;
          if (ok) {
            z[i] = zz;
            amax = fmaxf(amax, fabsf(zz));
          }
        }
#pragma unroll
        for (int jj = 0; jj < 4; ++jj) lpv[jj] = warp_sum(lpv[jj]);
        const float sum = lane == 0 ? lpv[0] : lane == 1 ? lpv[1] : lane == 2 ? lpv[2] : lpv[3];
        if (lane < 4 && rbase + lane < R) part[part_row + (int64_t)s * R + rbase + lane] = sum;
      }
    }
  }
};

// EPI 0 - 2 and 16; EPI 0 with K-slices writes slice s of the product to out + s R J
struct RowsEpi {
  static constexpr Units UNITS = K_SLICES;
  __host__ __device__ static constexpr bool folds_amax(int epi) { return epi != 1; }
  const float* bias; const float* x_obs; int64_t n_x; const float* gout;
  float* out; float* part; int relu; float* amax_scale;

  template <int EPI, class Core>
  __device__ __forceinline__ void run(const Core& core, int64_t uu, uint32_t trow, int quarter,
                                      int lane, float& amax) const {
    const int64_t& R = core.R;
    const int& J = core.J;
    const float acc_scale = core.acc_scale();
    const Unit pos = core.template unit<UNITS>(uu, quarter, lane);
    const int slice = pos.sub;
    const bool empty_slice = slice * core.kb_per >= core.n_kb_all;   // accumulator never written
    float* __restrict__ out_s = (EPI == 0 && out) ? out + (int64_t)slice * R * J : out;
    const int nb = pos.nb;
    const int j = pos.j;
    const bool j_ok = j < J;
    const float b_j = (j_ok && bias) ? bias[j] : 0.f;
    const int64_t r0 = pos.r0;
    const int64_t part_row = (int64_t)(nb * 4 + quarter) * R;
    const float b_use = (slice == 0) ? b_j : 0.f;           // bias once across the slices
    const bool warp_j_ok = __all_sync(0xffffffffu, j_ok);
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
      // upstream gradient of the 16 rows: lane jj holds gout[rbase + jj], broadcast by shuffle
      // in process()
      if (EPI == 2) ge = (lane < 16 && rbase + lane < R) ? __ldg(gout + rbase + lane) : 0.f;
    };
    auto process = [&](const uint32_t* v, const float* xe, float ge, int c) {
      // NO early return for rbase >= R: every access below is predicated on the row anyway, and
      // a return here (uniform, but not provably so) makes the compiler wrap each warp shuffle of
      // the row sums in a WARPSYNC.COLLECTIVE sequence (125 SHFL + 70 WARPSYNC -> 63 SHFL)
      const int64_t rbase = r0 + c;
      float lpv[16];
      float* __restrict__ po =
          (EPI == 0 || EPI == 2 || EPI == 16) ? out_s + rbase * J + j : nullptr;
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
        } else if (EPI == 16) {
          const float a = l + xe[jj];
          const float y = relu ? fmaxf(a, 0.f) : a;
          if (ok) { *po = y; amax = fmaxf(amax, fabsf(y)); }
        } else {
          const float g = __shfl_sync(0xffffffffu, ge, jj);
          const float y = g * (xe[jj] - __fdividef(1.f, 1.f + __expf(-l)));
          if (ok) { *po = y; amax = fmaxf(amax, fabsf(y)); }
        }
        if (EPI == 0 || EPI == 2 || EPI == 16) po += J;
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
  }
};

// output tiles of a product over J features and R rows
inline int64_t lin_tiles(int64_t R, int J) { return ((R + BN - 1) / BN) * ((J + BM - 1) / BM); }

// Tensor maps of one operand's fp16 planes [2][rows][cols] (hi, then lo), in boxes of 64 rows
// (MN-major) or of the tile's 128 rows (K-major, BM = BN).  A binary operand has its hi plane only;
// its lo map, never loaded, points at that plane.
int plane_maps(CUtensorMap* hi, CUtensorMap* lo, const void* planes, int64_t rows, int cols,
               bool mn_major, bool binary) {
  const __half* p = reinterpret_cast<const __half*>(planes);
  const uint32_t box = mn_major ? 64 : BM;
  const int rc = make_map(hi, p, (uint64_t)rows, (uint64_t)cols, box, 128, 1);
  if (rc) return rc;
  return make_map(lo, binary ? p : p + rows * cols, (uint64_t)rows, (uint64_t)cols, box, 128, 1);
}

// The core of a product over J features, R rows and contraction length K, cut into k_slices
// units per tile, from the planes of A (w_planes, scale_w) and B (h_planes, scale_h).  A K-major
// operand's planes are [2][J or R][kpad(K)], an MN-major one's [2][K][kpad(J or R)]; an operand
// whose bit of Z is set has its hi plane only.
template <int MN, int Z>
int make_core(LinCore<MN, Z>& c, const void* w_planes, const float* scale_w, const void* h_planes,
              const float* scale_h, int J, int64_t R, int64_t K, int k_slices = 1) {
  const int Kp = zsb_linear_tc_kpad((int)K);
  int rc = (MN & 1) ? plane_maps(&c.map_whi, &c.map_wlo, w_planes, K, zsb_linear_tc_kpad(J), true,
                                 Z & 1)
                    : plane_maps(&c.map_whi, &c.map_wlo, w_planes, J, Kp, false, Z & 1);
  if (rc) return rc;
  rc = (MN & 2) ? plane_maps(&c.map_hhi, &c.map_hlo, h_planes, K, zsb_linear_tc_kpad((int)R), true,
                             Z & 2)
                : plane_maps(&c.map_hhi, &c.map_hlo, h_planes, R, Kp, false, Z & 2);
  if (rc) return rc;
  c.scale_w = scale_w;
  c.scale_h = scale_h;
  c.R = R;
  c.J = J;
  c.n_blk = (J + BM - 1) / BM;
  c.n_tiles = lin_tiles(R, J);
  c.n_kb_all = Kp / 64;
  c.kb_per = (c.n_kb_all + k_slices - 1) / k_slices;
  c.k_slices = k_slices;
  return ZSB_OK;
}

// EPI 4 / 5: the sample rows per chunk that give a launch about two units per SM
int sample_chunk(int64_t R, int J, int S) {
  const int64_t n_tiles = lin_tiles(R, J);
  int64_t want = (2 * ZSB_NUM_SMS + n_tiles - 1) / n_tiles;
  if (want > S) want = S;
  if (want < 1) want = 1;
  return (int)((S + want - 1) / want);
}

// f(std::integral_constant<int, Z>()) with Z = 2 when operand B is a 0/1 sample whose planes are
// its hi plane only (h_binary), else Z = 0
template <class F>
int with_h_binary(int h_binary, F f) {
  if (h_binary) return f(std::integral_constant<int, 2>());
  return f(std::integral_constant<int, 0>());
}

// One pass over an activation / gradient matrix that produces its operand planes:
// src [R, K] fp32 (optionally times the ReLU mask (mask_src > 0)) ->
//   planes   [2][R][Kp]  fp16 hi/lo of src * scale   (the operand of all three products of a layer)
//   col_sum  [K] += sum_r src[r, k] * mask           (the bias gradient; float atomics)
// 64 x 64 tiles, float2 loads, half2 stores; the column sums of a tile meet in shared memory.
// At most 32 registers, so that 8 blocks fill an SM: left free, ptxas takes 44 to hoist loads,
// 5 blocks fit, and this memory-bound pass ran 7-16% slower (H100 SXM, 700 W).
__global__ void __launch_bounds__(256, 8) split16_dual_kernel(
    const float* __restrict__ src, const float* __restrict__ mask_src, int64_t R, int K, int Kp,
    __half* __restrict__ planes, float* __restrict__ col_sum, const float* __restrict__ scale) {
  __shared__ float csum[8][64];
  const float s = scale[0];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;        // 32 x 8
  const int64_t r_tiles = (R + 63) / 64;
  const int c_tiles = (Kp + 63) / 64;
  const int64_t n_pl = R * (int64_t)Kp;
  for (int64_t t = blockIdx.x; t < r_tiles * c_tiles; t += gridDim.x) {
    const int64_t r0 = (t / c_tiles) * 64;
    const int c0 = (int)(t % c_tiles) * 64;
    const int c = c0 + 2 * tx;
    float cs0 = 0.f, cs1 = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int64_t r = r0 + ty + 8 * i;
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
      if (r < R && c < Kp) {
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
    __syncthreads();
  }
}

// Backward pass of the class-conditioned layer (EPI 7 / 8) in one pass over the upstream gradient
// src (optionally times the ReLU mask (mask_src > 0)):
//   planes  [2][R][Kp]  fp16 hi/lo of G * scale, where G = src [R, K] (per-row classes cls) or,
//                       with cls == NULL, G[r] = sum_c src[c R + r] (src [C R, K], class-major):
//                       the operand of the input- and weight-gradient products, over R rows
//   col_sum [K]    += sum_r G[r, k]                              (bias gradient)
//   dtab    [C, K] += sum of src over the rows of class c        (class-table gradient)
// A thread holds 8 consecutive rows of a 64 x 64 tile and the two columns tx and tx + 32.  The
// class-table sums of a tile whose rows all have one class are its column sums (met in shared
// memory); in any other tile each thread adds every run of equal classes with a float atomic.
// Rows whose class is outside [0, C) add nothing to dtab.
__global__ void __launch_bounds__(256) split16_class_kernel(
    const float* __restrict__ src, const float* __restrict__ mask_src, int64_t R, int K, int Kp,
    const int32_t* __restrict__ cls, int64_t n_cls, int C, __half* __restrict__ planes,
    float* __restrict__ col_sum, float* __restrict__ dtab, const float* __restrict__ scale) {
  __shared__ float csum[8][64];
  const float s = scale[0];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;        // 32 x 8
  const int64_t r_tiles = (R + 63) / 64;
  const int c_tiles = (Kp + 63) / 64;
  const int64_t n_pl = R * (int64_t)Kp;
  const int n_pass = cls ? 1 : C;
  for (int64_t t = blockIdx.x; t < r_tiles * c_tiles; t += gridDim.x) {
    const int64_t r0 = (t / c_tiles) * 64;
    const int c0 = (int)(t % c_tiles) * 64;
    const int64_t rt = r0 + 8 * ty;                              // this thread's first row
    const int col[2] = {c0 + tx, c0 + tx + 32};
    int k8[8];                                                   // class of each row (per-row form)
    int k0 = 0;
    bool uniform = true;
    if (cls) {
      k0 = __ldg(cls + r0 % n_cls);
      int64_t yr = rt % n_cls;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        k8[i] = rt + i < R ? __ldg(cls + yr) : k0;
        uniform = uniform && k8[i] == k0;
        if (++yr == n_cls) yr = 0;
      }
      uniform = __syncthreads_and(uniform && k0 >= 0 && k0 < C);
    }
    float g[8][2];
#pragma unroll
    for (int i = 0; i < 8; ++i) g[i][0] = g[i][1] = 0.f;
    float tsum = 0.f;                              // threads < 64: the tile's column sums of G
    for (int p = 0; p < n_pass; ++p) {
      float cs[2] = {0.f, 0.f}, run[2] = {0.f, 0.f};
      int run_k = -1;
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int64_t r = rt + i;
        float v[2];
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          v[h] = 0.f;
          if (r < R && col[h] < K) {
            const int64_t idx = ((int64_t)p * R + r) * K + col[h];
            v[h] = src[idx];
            if (mask_src && !(mask_src[idx] > 0.f)) v[h] = 0.f;
          }
          g[i][h] += v[h];
          cs[h] += v[h];
        }
        if (cls && !uniform && dtab) {
          if (k8[i] != run_k) {
            if (run_k >= 0 && run_k < C) {
#pragma unroll
              for (int h = 0; h < 2; ++h)
                if (col[h] < K) atomicAdd(dtab + (int64_t)run_k * K + col[h], run[h]);
            }
            run_k = k8[i];
            run[0] = run[1] = 0.f;
          }
          run[0] += v[0];
          run[1] += v[1];
        }
      }
      if (cls && !uniform && dtab && run_k >= 0 && run_k < C) {
#pragma unroll
        for (int h = 0; h < 2; ++h)
          if (col[h] < K) atomicAdd(dtab + (int64_t)run_k * K + col[h], run[h]);
      }
      csum[ty][tx] = cs[0];
      csum[ty][tx + 32] = cs[1];
      __syncthreads();
      if (threadIdx.x < 64 && c0 + (int)threadIdx.x < K) {
        float a = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) a += csum[i][threadIdx.x];
        tsum += a;
        if (dtab && uniform) atomicAdd(dtab + (int64_t)(cls ? k0 : p) * K + c0 + threadIdx.x, a);
      }
      __syncthreads();
    }
    if (col_sum && threadIdx.x < 64 && c0 + (int)threadIdx.x < K)
      atomicAdd(col_sum + c0 + threadIdx.x, tsum);
#pragma unroll
    for (int i = 0; i < 8; ++i) {
      const int64_t r = rt + i;
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (r < R && col[h] < Kp) store_hilo(planes + r * Kp + col[h], n_pl, g[i][h] * s);
    }
  }
}

// ---- The noisy, batch-normalised dense layer of variational_dropout.py:26-37 --------------------
// Elementwise passes over [rows, cols] matrices run on 32 x 8 thread blocks: a warp takes 32
// consecutive columns of one row (coalesced for any width, odd ones included), the 8 warps take
// 8 rows, and the blocks stride over the rows.
constexpr int BN_TILE = 128;     // rows per moment partial: the product's row tile (BN)

// x = h[r % n_h, k] * noise[r, k] for r < R, k < K: the layer's input, never stored in fp32.
// PLANES = false: its max |x| into scale[2] (atomicMax; NaN and inf skipped).  PLANES = true:
// planes [2][R][Kp] = fp16 hi/lo of x * scale[0], pad columns zero.
template <bool PLANES>
__global__ void __launch_bounds__(256) noisy_split_kernel(
    const float* __restrict__ h, int64_t n_h, const float* __restrict__ noise, int64_t R, int K,
    int Kp, __half* __restrict__ planes, float* __restrict__ scale) {
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float s = PLANES ? scale[0] : 0.f;
  const int64_t n_pl = R * (int64_t)Kp;
  float m = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * 8 + ty; r < R; r += (int64_t)gridDim.x * 8) {
    const float* __restrict__ hr = h + (r % n_h) * K;
    const float* __restrict__ nr = noise + r * K;
    for (int k = tx; k < (PLANES ? Kp : K); k += 32) {
      const float x = k < K ? __ldg(hr + k) * nr[k] : 0.f;
      if (PLANES) store_hilo(planes + r * Kp + k, n_pl, x * s);
      else m = finite_absmax(m, x);
    }
  }
  if (!PLANES) fold_amax(scale, m, tx);
}

// Chan's update of (count n, mean, M2) with a second set (nb, mb, qb)
__device__ __forceinline__ void chan_merge(double& n, double& mean, double& m2, double nb,
                                           double mb, double qb) {
  if (nb == 0.0) return;
  const double nn = n + nb, d = mb - mean;
  mean += d * (nb / nn);
  m2 += qb + d * d * (n * nb / nn);
  n = nn;
}

// One warp per column j.  training: the batch moments from the EPI 9 partials, merged in a fixed
// order (lane l folds tiles l, l + 32, ... in turn, then a fixed shuffle tree), so two identical
// calls give identical bits; stats = (mean, rsqrt(var + eps)) with the population variance, and
// the moving statistics move towards the batch's: m -= (m - batch) * rate (rate = 1 - decay).
// BESSEL (TF 1.x's fused batch norm, the path of 4-D inputs): the moving variance moves towards the
// Bessel-corrected batch variance M2 / (R - 1) instead, and towards M2 / R = 0 when R = 1.
// Evaluation: stats from the moving statistics, which stay as they are.
template <bool BESSEL>
__global__ void __launch_bounds__(256) bn_stats_kernel(const float* __restrict__ part, int64_t R,
                                                       int J, float* __restrict__ mmean,
                                                       float* __restrict__ mvar, float rate,
                                                       float eps, int training,
                                                       float* __restrict__ stats) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (j >= J) return;                                            // warp-uniform
  if (!training) {
    if (lane == 0) {
      stats[j] = mmean[j];
      stats[J + j] = rsqrtf(mvar[j] + eps);
    }
    return;
  }
  const int64_t n_t = (R + BN_TILE - 1) / BN_TILE;
  double n = 0.0, mean = 0.0, m2 = 0.0;
  for (int64_t t = lane; t < n_t; t += 32)
    chan_merge(n, mean, m2, (double)min((int64_t)BN_TILE, R - t * BN_TILE),
               part[2 * t * J + j], part[(2 * t + 1) * J + j]);
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    const double nb = __shfl_down_sync(0xffffffffu, n, off);
    const double mb = __shfl_down_sync(0xffffffffu, mean, off);
    const double qb = __shfl_down_sync(0xffffffffu, m2, off);
    chan_merge(n, mean, m2, nb, mb, qb);
  }
  if (lane == 0) {
    const float mu = (float)mean, var = (float)(m2 / n);
    const float var_mv = BESSEL ? (float)(m2 / (n > 1.0 ? n - 1.0 : n)) : var;
    stats[j] = mu;
    stats[J + j] = rsqrtf(var + eps);
    mmean[j] -= (mmean[j] - mu) * rate;
    mvar[j] -= (mvar[j] - var_mv) * rate;
  }
}

// Training forward after EPI 9, in the rounding order of EPI 10 / 11: out = act(fma(a - mean,
// rstd, beta)) without GAMMA (not the same bits as gamma = 1), act(fma(xhat, gamma, beta)), xhat =
// (a - mean) * rstd, with it; max |out| into amax_scale[2] (may be NULL).  GAMMA is a template
// argument rather than a NULL test, which took this pass from 40 to 48 registers.
template <bool GAMMA>
__global__ void __launch_bounds__(256) bn_apply_kernel(const float* __restrict__ a, int64_t R,
                                                       int J, const float* __restrict__ stats,
                                                       const float* __restrict__ gamma,
                                                       const float* __restrict__ beta, int relu,
                                                       float* __restrict__ out,
                                                       float* __restrict__ amax_scale) {
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  float m = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * 8 + ty; r < R; r += (int64_t)gridDim.x * 8)
    for (int j = tx; j < J; j += 32) {
      const float d = a[r * J + j] - __ldg(stats + j), rs = __ldg(stats + J + j);
      float y = GAMMA ? fmaf(d * rs, __ldg(gamma + j), __ldg(beta + j))
                      : fmaf(d, rs, __ldg(beta + j));
      if (relu) y = fmaxf(y, 0.f);
      out[r * J + j] = y;
      m = fmaxf(m, fabsf(y));
    }
  if (amax_scale) fold_amax(amax_scale, m <= 3.0e38f ? m : 0.f, tx);
}

// Backward, per 128-row tile t and column j (block: 32 columns x 8 warps, 16 rows per warp, then
// the 8 warps meet in shared memory in a fixed order):
//   part[2 t J + j] = sum_r g',  part[(2 t + 1) J + j] = sum_r g' xhat   (training only)
// with g' = g [y > 0] (relu) or g, xhat = (a - mean) * rstd.
__global__ void __launch_bounds__(256) bn_grad_sums_kernel(
    const float* __restrict__ g, const float* __restrict__ y, const float* __restrict__ a,
    const float* __restrict__ stats, int relu, int64_t R, int J, float* __restrict__ part) {
  __shared__ float sh[2][8][32];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int64_t t = blockIdx.x;
  const int j = blockIdx.y * 32 + tx;
  float s1 = 0.f, s2 = 0.f;
  if (j < J) {
    const float mu = a ? stats[j] : 0.f, rs = a ? stats[J + j] : 0.f;
#pragma unroll 4
    for (int i = 0; i < BN_TILE / 8; ++i) {
      const int64_t r = t * BN_TILE + ty + 8 * i;
      if (r >= R) break;
      float gg = g[r * J + j];
      if (relu && !(y[r * J + j] > 0.f)) gg = 0.f;
      s1 += gg;
      if (a) s2 = fmaf(gg, (a[r * J + j] - mu) * rs, s2);
    }
  }
  sh[0][ty][tx] = s1;
  sh[1][ty][tx] = s2;
  __syncthreads();
  if (ty < 2 && j < J) {
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < 8; ++i) s += sh[ty][i][tx];
    part[(2 * t + ty) * J + j] = s;
  }
}

// One warp per column: the tile sums of bn_grad_sums_kernel in a fixed order (lane-strided runs,
// then a fixed shuffle tree) -> dbeta[j] = sum g', dgamma[j] = sum g' xhat (either may be NULL),
// coef = (sum g' / R, sum g' xhat / R)
__global__ void __launch_bounds__(256) bn_grad_combine_kernel(const float* __restrict__ part,
                                                              int64_t R, int J,
                                                              float* __restrict__ dbeta,
                                                              float* __restrict__ dgamma,
                                                              float* __restrict__ coef) {
  const int lane = threadIdx.x & 31;
  const int j = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (j >= J) return;
  const int64_t n_t = (R + BN_TILE - 1) / BN_TILE;
  float s1 = 0.f, s2 = 0.f;
  for (int64_t t = lane; t < n_t; t += 32) {
    s1 += part[2 * t * J + j];
    s2 += part[(2 * t + 1) * J + j];
  }
#pragma unroll
  for (int off = 16; off > 0; off >>= 1) {
    s1 += __shfl_down_sync(0xffffffffu, s1, off);
    s2 += __shfl_down_sync(0xffffffffu, s2, off);
  }
  if (lane == 0) {
    if (dbeta) dbeta[j] = s1;
    if (dgamma) dgamma[j] = s2;
    coef[j] = s1 / (float)R;
    coef[J + j] = s2 / (float)R;
  }
}

// What bn_grad_apply_kernel writes of da
enum BnGradOut {
  BN_GRAD_AMAX,     // nothing: max |da| into scale[2]
  BN_GRAD_PLANES,   // planes [2][R][Jp] = fp16 hi/lo of da * scale[0], pad columns zero -- the
                    // operand zsb_linear_tc_dgrad_f32 / _wgrad_f32 read
  BN_GRAD_F32       // da [R, J] in fp32, and max |da| into scale[2]
};
// da = gamma rstd (g' - coef[0] - xhat coef[1]) in training, gamma rstd g' in evaluation, with
// rstd in place of gamma rstd when gamma is NULL
template <BnGradOut OUT>
__global__ void __launch_bounds__(256) bn_grad_apply_kernel(
    const float* __restrict__ g, const float* __restrict__ y, const float* __restrict__ a,
    int training, const float* __restrict__ stats, const float* __restrict__ gamma,
    const float* __restrict__ coef, int relu, int64_t R, int J, int Jp,
    __half* __restrict__ planes, float* __restrict__ da, float* __restrict__ scale) {
  constexpr bool PLANES = OUT == BN_GRAD_PLANES;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const float s = PLANES ? scale[0] : 0.f;
  const int64_t n_pl = R * (int64_t)Jp;
  float m = 0.f;
  for (int64_t r = (int64_t)blockIdx.x * 8 + ty; r < R; r += (int64_t)gridDim.x * 8)
    for (int j = tx; j < (PLANES ? Jp : J); j += 32) {
      float d = 0.f;
      if (j < J) {
        float gg = g[r * J + j];
        if (relu && !(y[r * J + j] > 0.f)) gg = 0.f;
        const float rs = __ldg(stats + J + j);
        if (training) {
          const float xh = (a[r * J + j] - __ldg(stats + j)) * rs;
          gg = gg - __ldg(coef + j) - xh * __ldg(coef + J + j);
        }
        d = (gamma ? __ldg(gamma + j) * rs : rs) * gg;
      }
      if (PLANES) {
        store_hilo(planes + r * Jp + j, n_pl, d * s);
      } else {
        if (OUT == BN_GRAD_F32) da[r * J + j] = d;
        m = finite_absmax(m, d);
      }
    }
  if (!PLANES) fold_amax(scale, m, tx);
}

// From d = d(h * noise) [R, K]: dnoise[r] = d[r] * h[r % n_h] and dh[i] = sum_s d[s n_h + i] *
// noise[s n_h + i] over the R / n_h particle rows that share row i of h, in order (either output
// may be NULL).
__global__ void __launch_bounds__(256) noisy_grad_kernel(
    const float* __restrict__ d, const float* __restrict__ h, int64_t n_h,
    const float* __restrict__ noise, int64_t R, int K, float* __restrict__ dnoise,
    float* __restrict__ dh) {
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int64_t S = R / n_h;
  for (int64_t i = (int64_t)blockIdx.x * 8 + ty; i < n_h; i += (int64_t)gridDim.x * 8)
    for (int k = tx; k < K; k += 32) {
      const float hv = h[i * K + k];
      float acc = 0.f;
      for (int64_t s = 0; s < S; ++s) {
        const int64_t e = (s * n_h + i) * K + k;
        const float dv = d[e];
        if (dnoise) dnoise[e] = dv * hv;
        if (dh) acc = fmaf(dv, noise[e], acc);
      }
      if (dh) dh[i * K + k] = acc;
    }
}

// blocks of a grid-stride pass over n items at `per` items per block, at most per_sm per SM
inline unsigned grid_blocks(int64_t n, int64_t per, int per_sm) {
  int64_t b = zsb_ceil_div(n, per);
  if (b > ZSB_NUM_SMS * per_sm) b = ZSB_NUM_SMS * per_sm;
  return (unsigned)(b < 1 ? 1 : b);
}

// scale[2] = running max |src| bits (atomicMax over the blocks; NaN and inf are skipped)
__global__ void __launch_bounds__(256) absmax2_kernel(const float* __restrict__ src, int64_t n,
                                                      float* __restrict__ scale) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n;
       i += (int64_t)gridDim.x * blockDim.x)
    m = finite_absmax(m, src[i]);
  fold_amax(scale, m, threadIdx.x & 31);
}
// scale[0] = the plane scale of the bound mult * max|src|, from the max in scale[2], which it
// clears again for the next split (mult > 1: the class fold of split16_class_kernel adds up to
// `mult` rows of src)
__global__ void pow2_scale_mult_kernel(float* __restrict__ scale, float mult) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  scale[0] = pow2_plane_scale(__uint_as_float(reinterpret_cast<unsigned int*>(scale)[2]) * mult);
  reinterpret_cast<unsigned int*>(scale)[2] = 0u;
}
// max pass of an operand split: leaves scale[0]
inline void launch_absmax_scale(const float* src, int64_t n, float* scale, cudaStream_t st) {
  absmax2_kernel<<<grid_blocks(n, 256 * 8, 16), 256, 0, st>>>(src, n, scale);
  pow2_scale_mult_kernel<<<1, 32, 0, st>>>(scale, 1.f);
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
    store_hilo(planes + i, n, (k < K) ? src[r * K + k] * s : 0.f);
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
// out[r] = the sum of the partial rows part [nparts(J)][rows] that EPI 1 / 4 / 5 write
int launch_part_sum(const float* part, int J, int64_t rows, float* out, cudaStream_t st,
                    const char* what) {
  part_sum_kernel<<<grid_blocks(rows, 256, 8), 256, 0, st>>>(part, zsb_linear_tc_nparts(J), rows,
                                                             out);
  return zsb_check_launch(what);
}

// zsb_linear_tc_amax_f32 (Z = 0) and zsb_linear_tc_bin_f32 (Z = 2: h is a 0/1 sample)
template <int Z>
int linear_tc_amax(int epi, const void* w_planes, const float* scale_w, const void* h_planes,
                   const float* scale_h, const float* bias, const float* x_obs, int64_t n_x,
                   const float* gout, float* out, float* part, int64_t R, int J, int K, int relu,
                   float* amax_scale, cudaStream_t st) {
  ZSB_REQUIRE((epi >= 0 && epi <= 2) || (epi == 16 && Z == 0),
              "zsb_linear_tc_f32: unknown epilogue");
  ZSB_REQUIRE(w_planes && h_planes && scale_w && scale_h && out && R > 0 && J > 0 && K > 0,
              "zsb_linear_tc_f32: bad args");
  ZSB_REQUIRE(R < (1LL << 31), "zsb_linear_tc_f32: too many rows");
  ZSB_REQUIRE(epi == 0 || (x_obs && n_x > 0), "zsb_linear_tc_f32: observations missing");
  ZSB_REQUIRE(epi != 16 || (n_x == R && R * J < (1LL << 31)),
              "zsb_linear_tc_f32: epi 16 needs a residual of R x J (n_x = R) below 2^31 entries");
  ZSB_REQUIRE(epi != 1 || part, "zsb_linear_tc_f32: partial-sum scratch missing");
  ZSB_REQUIRE(epi != 2 || gout, "zsb_linear_tc_f32: upstream gradient missing");
  LinCore<0, Z> c;
  int rc = make_core(c, w_planes, scale_w, h_planes, scale_h, J, R, K);
  if (rc) return rc;
  const RowsEpi e{.bias = bias, .x_obs = x_obs, .n_x = n_x, .gout = gout, .out = out,
                  .part = part, .relu = relu, .amax_scale = amax_scale};
  if (epi == 0) return tc_launch(LinW<RowsEpi, 0, 0, Z>{c, e}, st, "linear_tc");
  if (epi == 2) return tc_launch(LinW<RowsEpi, 2, 0, Z>{c, e}, st, "linear_tc");
  if constexpr (Z == 0)
    if (epi == 16) return tc_launch(LinW<RowsEpi, 16, 0, 0>{c, e}, st, "linear_tc_residual");
  rc = tc_launch(LinW<RowsEpi, 1, 0, Z>{c, e}, st, "linear_tc");
  return rc ? rc : launch_part_sum(part, J, R, out, st, "linear_tc_part_sum");
}

// zsb_linear_tc_wgrad_f32 (Z = 0) and zsb_linear_tc_wgrad_bin_f32 (Z = 1: h is a 0/1 sample)
template <int Z>
int linear_tc_wgrad(const void* h_planes, const float* scale_h, int K, const void* g_planes,
                    const float* scale_g, int J, int64_t R, float* out, float* part,
                    cudaStream_t st) {
  ZSB_REQUIRE(h_planes && g_planes && scale_h && scale_g && out && R > 0 && J > 0 && K > 0,
              "zsb_linear_tc_wgrad_f32: bad args");
  ZSB_REQUIRE(R < (1LL << 31) - 64, "zsb_linear_tc_wgrad_f32: too many rows");
  const int k_slices = part ? zsb_linear_tc_slices(J, K, (int)R) : 1;
  LinCore<3, Z> c;              // A = h (K features), B = g (J rows), contraction over the R rows
  int rc = make_core(c, h_planes, scale_h, g_planes, scale_g, K, J, R, k_slices);
  if (rc) return rc;
  rc = tc_launch(LinW<RowsEpi, 0, 3, Z>{c, {.out = k_slices > 1 ? part : out}}, st,
                 "linear_tc_wgrad");
  if (rc != ZSB_OK || k_slices == 1) return rc;
  const int64_t n = (int64_t)J * K;
  slice_sum_kernel<<<grid_blocks(n, 256, 8), 256, 0, st>>>(part, k_slices, n, out);
  return zsb_check_launch("linear_tc_wgrad_slice_sum");
}

// The training step of batch norm after a pass that left the pre-activation a [R, J] and its
// moment partials part (EPI 9's layout): the merge into stats and the moving statistics (bessel:
// the moving variance of TF's fused batch norm), then the affine step and ReLU
int bn_finish(const float* a, const float* part, int64_t R, int J, const float* gamma,
              const float* beta, float* moving_mean, float* moving_var, float rate, float eps,
              int bessel, float* stats, float* out, int relu, float* amax_scale, cudaStream_t st) {
  const unsigned col_blocks = (unsigned)((J + 7) / 8);
  if (bessel)
    bn_stats_kernel<true><<<col_blocks, 256, 0, st>>>(part, R, J, moving_mean, moving_var, rate,
                                                      eps, 1, stats);
  else
    bn_stats_kernel<false><<<col_blocks, 256, 0, st>>>(part, R, J, moving_mean, moving_var, rate,
                                                       eps, 1, stats);
  const unsigned blocks = grid_blocks(R, 8, 16);
  if (gamma)
    bn_apply_kernel<true><<<blocks, 256, 0, st>>>(a, R, J, stats, gamma, beta, relu, out,
                                                  amax_scale);
  else
    bn_apply_kernel<false><<<blocks, 256, 0, st>>>(a, R, J, stats, gamma, beta, relu, out,
                                                   amax_scale);
  return zsb_check_launch("bn_finish");
}

// The backward passes of zsb_bn_grad_f32 (OUT = BN_GRAD_PLANES) and zsb_bn_grad_f32out
// (BN_GRAD_F32): the per-tile column sums, their merge into dbeta, dgamma and coef, then da
template <BnGradOut OUT>
int bn_grad(int training, const float* g, const float* y, const float* a, const float* stats,
            const float* gamma, int relu, int64_t R, int J, float* part, float* dbeta,
            float* dgamma, void* planes, float* da, float* scale, cudaStream_t st) {
  const int64_t n_t = (R + BN_TILE - 1) / BN_TILE;
  float* coef = part + 2 * n_t * J;
  bn_grad_sums_kernel<<<dim3((unsigned)n_t, (unsigned)((J + 31) / 32)), 256, 0, st>>>(
      g, y, training || dgamma ? a : nullptr, stats, relu, R, J, part);
  bn_grad_combine_kernel<<<(unsigned)((J + 7) / 8), 256, 0, st>>>(part, R, J, dbeta, dgamma,
                                                                  coef);
  const unsigned blocks = grid_blocks(R, 8, 16);
  if constexpr (OUT == BN_GRAD_F32) {
    bn_grad_apply_kernel<BN_GRAD_F32><<<blocks, 256, 0, st>>>(
        g, y, a, training, stats, gamma, coef, relu, R, J, J, nullptr, da, scale);
  } else {
    const int Jp = zsb_linear_tc_kpad(J);
    __half* pl = reinterpret_cast<__half*>(planes);
    bn_grad_apply_kernel<BN_GRAD_AMAX><<<blocks, 256, 0, st>>>(
        g, y, a, training, stats, gamma, coef, relu, R, J, Jp, pl, nullptr, scale);
    pow2_scale_mult_kernel<<<1, 32, 0, st>>>(scale, 1.f);
    bn_grad_apply_kernel<BN_GRAD_PLANES><<<blocks, 256, 0, st>>>(
        g, y, a, training, stats, gamma, coef, relu, R, J, Jp, pl, nullptr, scale);
  }
  return zsb_check_launch("bn_grad");
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
  launch_absmax_scale(src, rows * (int64_t)K, scale, st);
  split16_pad_kernel<<<grid_blocks(rows * (int64_t)Kp, 256 * 4, 32), 256, 0, st>>>(
      src, rows, K, Kp, reinterpret_cast<__half*>(planes), scale);
  return zsb_check_launch("split16_pad");
}

// The operand planes of one matrix in ONE pass (see split16_dual_kernel): planes [2][R][Kp],
// optional ReLU mask source, optional column sums (bias gradient; col_sum must be zeroed by the
// caller).  have_amax = 1: scale[2] already holds max |src| (written by zsb_linear_tc_amax_f32),
// so no max pass is run.  K must be even.
int zsb_split16_dual_f32(const float* src, const float* mask_src, int64_t R, int K, void* planes,
                         float* col_sum, float* scale, int have_amax, void* stream) {
  ZSB_REQUIRE(src && planes && scale && R > 0 && K > 0 && K % 2 == 0,
              "zsb_split16_dual_f32: bad args (K must be even)");
  cudaStream_t st = (cudaStream_t)stream;
  const int Kp = zsb_linear_tc_kpad(K);
  if (!have_amax)
    launch_absmax_scale(src, R * (int64_t)K, scale, st);
  else
    pow2_scale_mult_kernel<<<1, 32, 0, st>>>(scale, 1.f);   // max|src| left by a GEMM epilogue
  split16_dual_kernel<<<grid_blocks(((R + 63) / 64) * (Kp / 64), 1, 16), 256, 0, st>>>(
      src, mask_src, R, K, Kp, reinterpret_cast<__half*>(planes), col_sum, scale);
  return zsb_check_launch("split16_dual");
}

// Fused dense layer on the tensor cores.  w_planes [2][J][Kp], h_planes [2][R][Kp] (fp16 planes
// from zsb_split16_pad_f32 with their scales); bias [J] or NULL.
//   epi 0: out [R, J] = h W^T + bias (ReLU if relu != 0)
//   epi 1: out [R] = sum_j Bernoulli(logits = h W^T + bias).log_prob(x[r % n_x, j]);
//          part = scratch of zsb_linear_tc_nparts(J) * R floats
//   epi 2: out [R, J] = gout[r] * (x - sigmoid(logits))
//   epi 16 (zsb_linear_tc_amax_f32 only): out [R, J] = act(h W^T + bias + x) with the residual
//          x [R, J] (n_x = R), added before the ReLU
// `part` is read by epi 1 only.
//
// Split-K slices of the weight-gradient product zsb_linear_tc_wgrad_f32 (R output rows, J
// features, contraction length K): when the output has fewer than one 128 x 128 tile per SM, the
// contraction is cut into slices that run on different SMs and are summed afterwards.
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
// As zsb_linear_tc_f32; additionally the running max |out| (epi 0 / 2) is
// folded into amax_scale[2] (uint bits, atomicMax): the scale slot zsb_split16_dual_f32 consumes
// with have_amax = 1, so the consumer's operand split needs no separate max pass over `out`.
int zsb_linear_tc_amax_f32(int epi, const void* w_planes, const float* scale_w,
                           const void* h_planes, const float* scale_h, const float* bias,
                           const float* x_obs, int64_t n_x, const float* gout, float* out,
                           float* part, int64_t R, int J, int K, int relu, float* amax_scale,
                           void* stream) {
  return linear_tc_amax<0>(epi, w_planes, scale_w, h_planes, scale_h, bias, x_obs, n_x, gout, out,
                           part, R, J, K, relu, amax_scale, (cudaStream_t)stream);
}
// As zsb_linear_tc_amax_f32 for a 0/1 activation h whose planes are its hi plane only, at scale
// 2048 (zsb_linear_tc_bern_sample_f32): two fp16 products per k-step instead of three, the same
// result bit for bit.
int zsb_linear_tc_bin_f32(int epi, const void* w_planes, const float* scale_w,
                          const void* h_planes, const float* scale_h, const float* bias,
                          const float* x_obs, int64_t n_x, const float* gout, float* out,
                          float* part, int64_t R, int J, int K, int relu, float* amax_scale,
                          void* stream) {
  return linear_tc_amax<2>(epi, w_planes, scale_w, h_planes, scale_h, bias, x_obs, n_x, gout, out,
                           part, R, J, K, relu, amax_scale, (cudaStream_t)stream);
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
  LinCore<1, 0> c;              // A = W (K features), B = g (R rows), contraction over J
  const int rc = make_core(c, w_planes, scale_w, g_planes, scale_g, K, R, J);
  if (rc) return rc;
  return tc_launch(LinW<RowsEpi, 0, 1>{c, {.out = out, .amax_scale = amax_scale}},
                   (cudaStream_t)stream, "linear_tc_dgrad");
}

// Weight gradient of a dense layer WITHOUT transposed operands:
//   out [J, K] = sum_r g[r, j] * h[r, k]            (dW = g^T h, tf.gradients of tf.layers.dense)
// h_planes [2][R][Kp(K)], g_planes [2][R][Kp(J)]: the row-major fp16 hi/lo planes the forward /
// input-gradient products already use (zsb_split16_pad_f32 / zsb_split16_dual_f32).  The contraction
// runs over the rows, so both operands are MN-major wgmma operands (MN = 3);
// split-K over the SMs (part = zsb_linear_tc_slices(J, K, R) * J * K floats, or NULL for a single
// slice).
int zsb_linear_tc_wgrad_f32(const void* h_planes, const float* scale_h, int K,
                            const void* g_planes, const float* scale_g, int J, int64_t R,
                            float* out, float* part, void* stream) {
  return linear_tc_wgrad<0>(h_planes, scale_h, K, g_planes, scale_g, J, R, out, part,
                            (cudaStream_t)stream);
}
// As zsb_linear_tc_wgrad_f32 for a 0/1 activation h whose planes are its hi plane only
// (zsb_linear_tc_bern_sample_f32): two products per k-step, the same result bit for bit.
int zsb_linear_tc_wgrad_bin_f32(const void* h_planes, const float* scale_h, int K,
                                const void* g_planes, const float* scale_g, int J, int64_t R,
                                float* out, float* part, void* stream) {
  return linear_tc_wgrad<1>(h_planes, scale_h, K, g_planes, scale_g, J, R, out, part,
                            (cudaStream_t)stream);
}

// Bernoulli layer with S draws per logit row, l = h W^T + bias never leaving the epilogue (EPI 4):
//   h_out [S R, J] = (u < sigmoid(l[r])), float (h_int = 0) or int32; u = u_in [S R J] or the
//                    Philox draw of zsb_sample_bernoulli_i32 for (seed, iter) at element (s R + r) J + j
//   h_planes_out [S R][kpad(J)] fp16 = h * 2048, zero padding: the operand of the next layer
//   logq [S R] = sum_j Bernoulli(l[r]).log_prob(h[s R + r]);  part = nparts(J) * S R floats
// h_binary: h_planes is itself such a sample plane (one plane, lo plane zero).
int zsb_linear_tc_bern_sample_f32(const void* w_planes, const float* scale_w, const void* h_planes,
                                  const float* scale_h, int h_binary, const float* bias,
                                  const float* u_in, uint64_t seed, uint32_t iter, int S,
                                  void* h_out, int h_int, void* h_planes_out, float* logq,
                                  float* part, int64_t R, int J, int K, void* stream) {
  ZSB_REQUIRE(w_planes && h_planes && scale_w && scale_h && h_out && h_planes_out && logq &&
                  part && R > 0 && J > 0 && K > 0 && S >= 1,
              "zsb_linear_tc_bern_sample_f32: bad args");
  ZSB_REQUIRE((int64_t)S * R < (1LL << 31), "zsb_linear_tc_bern_sample_f32: too many rows");
  cudaStream_t st = (cudaStream_t)stream;
  const int s_per = sample_chunk(R, J, S);
  const SamplesEpi e{.bias = bias, .out = reinterpret_cast<float*>(h_out), .part = part, .S = S,
                     .s_per = s_per, .u_in = u_in, .seed = seed, .iter = iter,
                     .epoch = zsb_epoch_ptr(), .h_int = h_int,
                     .pl_out = reinterpret_cast<__half*>(h_planes_out)};
  return with_h_binary(h_binary, [&](auto z) {
    LinCore<0, z> c;
    int rc = make_core(c, w_planes, scale_w, h_planes, scale_h, J, R, K, (S + s_per - 1) / s_per);
    if (rc) return rc;
    rc = tc_launch(LinW<SamplesEpi, 4, 0, z>{c, e}, st, "linear_tc_bern_sample");
    if (rc) return rc;
    return launch_part_sum(part, J, (int64_t)S * R, logq, st, "linear_tc_bern_sample_part_sum");
  });
}

// Bernoulli layer against S given rows per logit row, l[r] = (h W^T + bias)[r]:
//   epi 1: out [S R] = sum_j Bernoulli(l[r]).log_prob(given[s R + r, j]); part = nparts(J) * S R
//   epi 2: out [R, J] = sum_s gout[s R + r] * (given[s R + r, j] - sigmoid(l[r, j])), the gradient
//          of sum gout * (epi 1) wrt the logits; max |out| folded into amax_scale[2] (may be NULL)
// h_binary as in zsb_linear_tc_bern_sample_f32.
int zsb_linear_tc_bern_given_f32(int epi, const void* w_planes, const float* scale_w,
                                 const void* h_planes, const float* scale_h, int h_binary,
                                 const float* bias, const float* given, int S, const float* gout,
                                 float* out, float* part, int64_t R, int J, int K,
                                 float* amax_scale, void* stream) {
  ZSB_REQUIRE(epi == 1 || epi == 2, "zsb_linear_tc_bern_given_f32: epi must be 1 or 2");
  ZSB_REQUIRE(w_planes && h_planes && scale_w && scale_h && given && out && R > 0 && J > 0 &&
                  K > 0 && S >= 1 && (epi != 1 || part) && (epi != 2 || gout),
              "zsb_linear_tc_bern_given_f32: bad args");
  ZSB_REQUIRE((int64_t)S * R < (1LL << 31), "zsb_linear_tc_bern_given_f32: too many rows");
  cudaStream_t st = (cudaStream_t)stream;
  const int s_per = epi == 1 ? sample_chunk(R, J, S) : S;   // EPI 6 sums over the draws: one chunk
  const SamplesEpi e{.bias = bias, .x_obs = given, .gout = gout, .out = out, .part = part, .S = S,
                     .s_per = s_per, .amax_scale = amax_scale};
  return with_h_binary(h_binary, [&](auto z) {
    LinCore<0, z> c;
    int rc = make_core(c, w_planes, scale_w, h_planes, scale_h, J, R, K, (S + s_per - 1) / s_per);
    if (rc) return rc;
    if (epi == 2) return tc_launch(LinW<SamplesEpi, 6, 0, z>{c, e}, st, "linear_tc_bern_given");
    rc = tc_launch(LinW<SamplesEpi, 5, 0, z>{c, e}, st, "linear_tc_bern_given");
    if (rc) return rc;
    return launch_part_sum(part, J, (int64_t)S * R, out, st, "linear_tc_bern_given_part_sum");
  });
}

// One-hot categorical layer with S draws per logit row, l = h W^T + bias never leaving the epilogue
// (EPI 12; replaces dense + OnehotCategorical._sample + log_prob, vae_ssl_adaptive_is.py:61-68 and
// multivariate.py:522-562):
//   cls [S R] int32     the class of draw d = s R + r, drawn as zsb_sample_categorical_i32 draws it
//                       from the logits l[r] for (seed, iter), or from the uniform u_in[d]
//   onehot [S R, C]     its one-hot row, float (h_int = 0) or int32
//   logq [S R]          l[r, cls] - logsumexp(l[r])
// 1 <= C <= 128 classes; h_binary as in zsb_linear_tc_bern_sample_f32.
int zsb_linear_tc_cat_sample_f32(const void* w_planes, const float* scale_w, const void* h_planes,
                                 const float* scale_h, int h_binary, const float* bias,
                                 const float* u_in, uint64_t seed, uint32_t iter, int S,
                                 int32_t* cls, void* onehot, int h_int, float* logq, int64_t R,
                                 int C, int K, void* stream) {
  ZSB_REQUIRE(w_planes && h_planes && scale_w && scale_h && cls && onehot && logq && R > 0 &&
                  K > 0 && S >= 1,
              "zsb_linear_tc_cat_sample_f32: bad args");
  ZSB_REQUIRE(C >= 1 && C <= CAT_MAX_C, "zsb_linear_tc_cat_sample_f32: C must be in [1, 128]");
  ZSB_REQUIRE((int64_t)S * R < (1LL << 31), "zsb_linear_tc_cat_sample_f32: too many rows");
  cudaStream_t st = (cudaStream_t)stream;
  const int s_per = sample_chunk(R, C, S);
  const CatEpi e{.bias = bias, .cls = cls, .onehot = onehot, .h_int = h_int, .logq = logq, .S = S,
                 .s_per = s_per, .u_in = u_in, .seed = seed, .iter = iter,
                 .epoch = zsb_epoch_ptr()};
  return with_h_binary(h_binary, [&](auto z) {
    LinCore<0, z> c;
    const int rc = make_core(c, w_planes, scale_w, h_planes, scale_h, C, R, K, (S + s_per - 1) / s_per);
    if (rc) return rc;
    return tc_launch(LinW<CatEpi, 12, 0, z>{c, e}, st, "linear_tc_cat_sample");
  });
}

// One-hot categorical layer against S given rows per logit row, l[r] = (h W^T + bias)[r], given
// [n_g, C] float, draw d = s R + r scored against given row d % n_g (n_g divides S R)
// (OnehotCategorical._log_prob, multivariate.py:542-562 = unnormalized_multinomial_log_prob with
// normalize_logits, multivariate.py:435-443):
//   epi 1: out [S R] = sum_j given_j (l[r, j] - logsumexp(l[r]))
//   epi 2: out [R, C] = sum_s gout[d] (given_j - (sum_i given_i) softmax(l[r])_j), the gradient of
//          sum gout * (epi 1) wrt the logits; max |out| folded into amax_scale[2] (may be NULL)
// 1 <= C <= 128; h_binary as in zsb_linear_tc_bern_sample_f32.
int zsb_linear_tc_cat_given_f32(int epi, const void* w_planes, const float* scale_w,
                                const void* h_planes, const float* scale_h, int h_binary,
                                const float* bias, const float* given, int64_t n_g, int S,
                                const float* gout, float* out, int64_t R, int C, int K,
                                float* amax_scale, void* stream) {
  ZSB_REQUIRE(epi == 1 || epi == 2, "zsb_linear_tc_cat_given_f32: epi must be 1 or 2");
  ZSB_REQUIRE(w_planes && h_planes && scale_w && scale_h && given && out && R > 0 && K > 0 &&
                  S >= 1 && n_g > 0 && (epi != 2 || gout),
              "zsb_linear_tc_cat_given_f32: bad args");
  ZSB_REQUIRE(C >= 1 && C <= CAT_MAX_C, "zsb_linear_tc_cat_given_f32: C must be in [1, 128]");
  ZSB_REQUIRE((int64_t)S * R < (1LL << 31), "zsb_linear_tc_cat_given_f32: too many rows");
  ZSB_REQUIRE(((int64_t)S * R) % n_g == 0,
              "zsb_linear_tc_cat_given_f32: given rows must divide the draws");
  cudaStream_t st = (cudaStream_t)stream;
  const int s_per = epi == 1 ? sample_chunk(R, C, S) : S;   // EPI 14 sums over the draws: one chunk
  const CatEpi e{.bias = bias, .given = given, .n_g = n_g, .gout = gout, .out = out, .S = S,
                 .s_per = s_per, .amax_scale = amax_scale};
  return with_h_binary(h_binary, [&](auto z) {
    LinCore<0, z> c;
    const int rc = make_core(c, w_planes, scale_w, h_planes, scale_h, C, R, K, (S + s_per - 1) / s_per);
    if (rc) return rc;
    if (epi == 2) return tc_launch(LinW<CatEpi, 14, 0, z>{c, e}, st, "linear_tc_cat_given");
    return tc_launch(LinW<CatEpi, 13, 0, z>{c, e}, st, "linear_tc_cat_given");
  });
}

// Gaussian layer with S draws per row, the heads mu = h W_mean^T + b_mean and ls = h W_logstd^T +
// b_logstd never leaving the epilogue (EPI 15; replaces two dense layers + Normal._sample + log_prob,
// vae_ssl_adaptive_is.py:53-68 and univariate.py:161-181).  w_planes / bias: the packed heads
// [2 Dp, K] / [2 Dp], Dp = kpad(D), in blocks of 64 rows [mean | logstd | mean | ...], zero padded.
//   z [S R, D]       eps * exp(ls) + mu, eps = eps_in [S R D] or the Philox normal
//                    zsb_reparam_normal_f32 draws for (seed, iter) at element (s R + r) D + j
//   logq [S R]       sum_j log N(z; mu, exp(ls));  part = Dp / 32 * S R floats of scratch
//   mean_out, logstd_out [R, D] (either may be NULL)
// max |z| is folded into amax_scale[2] (may be NULL).  1 <= D <= 256; h_binary as in
// zsb_linear_tc_bern_sample_f32.
int zsb_linear_tc_normal_sample_f32(const void* w_planes, const float* scale_w,
                                    const void* h_planes, const float* scale_h, int h_binary,
                                    const float* bias, const float* eps_in, uint64_t seed,
                                    uint32_t iter, int S, float* z, float* logq, float* part,
                                    float* mean_out, float* logstd_out, int64_t R, int D, int K,
                                    float* amax_scale, void* stream) {
  ZSB_REQUIRE(w_planes && h_planes && scale_w && scale_h && z && logq && part && R > 0 && K > 0 &&
                  S >= 1,
              "zsb_linear_tc_normal_sample_f32: bad args");
  ZSB_REQUIRE(D >= 1 && D <= NORMAL_MAX_D, "zsb_linear_tc_normal_sample_f32: D must be in [1, 256]");
  ZSB_REQUIRE((int64_t)S * R < (1LL << 31),
              "zsb_linear_tc_normal_sample_f32: too many rows");
  cudaStream_t st = (cudaStream_t)stream;
  const int J = 2 * zsb_linear_tc_kpad(D);
  const int s_per = sample_chunk(R, J, S);
  const NormalEpi e{.bias = bias, .D = D, .z = z, .part = part, .mean_out = mean_out,
                    .logstd_out = logstd_out, .S = S, .s_per = s_per, .eps_in = eps_in,
                    .seed = seed, .iter = iter, .epoch = zsb_epoch_ptr(), .amax_scale = amax_scale};
  return with_h_binary(h_binary, [&](auto zb) {
    LinCore<0, zb> c;
    int rc = make_core(c, w_planes, scale_w, h_planes, scale_h, J, R, K, (S + s_per - 1) / s_per);
    if (rc) return rc;
    rc = tc_launch(LinW<NormalEpi, 15, 0, zb>{c, e}, st, "linear_tc_normal_sample");
    if (rc) return rc;
    const int64_t rows = (int64_t)S * R;                 // two partial rows per 64 features
    part_sum_kernel<<<grid_blocks(rows, 256, 8), 256, 0, st>>>(part, J / 64, rows, logq);
    return zsb_check_launch("linear_tc_normal_sample_part_sum");
  });
}

// Class-conditioned dense layer (EPI 7 / 8): l = h W^T + bias plus row y of the class table
// ctab [C, J] (the class weights transposed), ReLU if relu.
//   cls != NULL: out [R, J], y = cls[r % n_cls]; a row with y outside [0, C) is all NaN
//   cls == NULL: out [C R, J], row c R + r for class c (every class, one product over R rows)
// max |out| (NaN rows excluded) is folded into amax_scale[2] (may be NULL).  h_binary as in
// zsb_linear_tc_bern_sample_f32.
int zsb_linear_tc_class_f32(const void* w_planes, const float* scale_w, const void* h_planes,
                            const float* scale_h, int h_binary, const float* bias,
                            const float* ctab, int C, const int32_t* cls, int64_t n_cls,
                            float* out, int64_t R, int J, int K, int relu, float* amax_scale,
                            void* stream) {
  ZSB_REQUIRE(w_planes && h_planes && scale_w && scale_h && ctab && out && R > 0 && J > 0 &&
                  K > 0 && C > 0 && (!cls || n_cls > 0),
              "zsb_linear_tc_class_f32: bad args");
  ZSB_REQUIRE(R < (1LL << 31), "zsb_linear_tc_class_f32: too many rows");
  cudaStream_t st = (cudaStream_t)stream;
  const ClassEpi e{.bias = bias, .ctab = ctab, .C = C, .cls = cls, .n_cls = n_cls, .out = out,
                   .relu = relu, .amax_scale = amax_scale};
  return with_h_binary(h_binary, [&](auto z) {
    LinCore<0, z> c;
    const int rc = make_core(c, w_planes, scale_w, h_planes, scale_h, J, R, K);
    if (rc) return rc;
    if (cls) return tc_launch(LinW<ClassEpi, 7, 0, z>{c, e}, st, "linear_tc_class");
    return tc_launch(LinW<ClassEpi, 8, 0, z>{c, e}, st, "linear_tc_class");
  });
}

// The backward pass of zsb_linear_tc_class_f32 in one pass (split16_class_kernel) over the upstream
// gradient src (times the ReLU mask mask_src > 0, the layer's output, when not NULL):
//   cls != NULL: src [R, K], planes [2][R][kpad(K)] of src
//   cls == NULL: src [C R, K] class-major, planes of G[r] = sum_c src[c R + r]
//   col_sum [K] += column sums of G, dtab [C, K] += per-class column sums (both may be NULL and
//   must be zeroed by the caller).
// have_amax = 1: scale[2] already holds max |src| (written by the producing GEMM).  The planes'
// scale is that of C * max|src| in the enumerated form (a bound of max|G|), else of max|src|.
int zsb_split16_class_f32(const float* src, const float* mask_src, int64_t R, int K,
                          const int32_t* cls, int64_t n_cls, int C, void* planes, float* col_sum,
                          float* dtab, float* scale, int have_amax, void* stream) {
  ZSB_REQUIRE(src && planes && scale && R > 0 && K > 0 && C > 0 && (!cls || n_cls > 0),
              "zsb_split16_class_f32: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  const int Kp = zsb_linear_tc_kpad(K);
  const int64_t n = (cls ? 1 : C) * R * (int64_t)K;
  if (!have_amax) absmax2_kernel<<<grid_blocks(n, 256 * 8, 16), 256, 0, st>>>(src, n, scale);
  pow2_scale_mult_kernel<<<1, 32, 0, st>>>(scale, cls ? 1.f : (float)C);
  split16_class_kernel<<<grid_blocks(((R + 63) / 64) * (Kp / 64), 1, 16), 256, 0, st>>>(
      src, mask_src, R, K, Kp, cls, n_cls, C, reinterpret_cast<__half*>(planes), col_sum, dtab,
      scale);
  return zsb_check_launch("split16_class");
}

// Operand planes [2][R][kpad(K)] of x = h[r % n_h] * noise[r] (h [n_h, K], noise [R, K], n_h
// dividing R) with scale[0] chosen from max |x| as zsb_split16_dual_f32 chooses it: a max pass
// and a split pass, both reading h and noise; x is never stored in fp32.
int zsb_split16_noisy_f32(const float* h, int64_t n_h, const float* noise, int64_t R, int K,
                          void* planes, float* scale, void* stream) {
  ZSB_REQUIRE(h && noise && planes && scale && R > 0 && K > 0 && n_h > 0 && R % n_h == 0,
              "zsb_split16_noisy_f32: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  const int Kp = zsb_linear_tc_kpad(K);
  __half* pl = reinterpret_cast<__half*>(planes);
  const unsigned blocks = grid_blocks(R, 8, 16);
  noisy_split_kernel<false><<<blocks, 256, 0, st>>>(h, n_h, noise, R, K, Kp, pl, scale);
  pow2_scale_mult_kernel<<<1, 32, 0, st>>>(scale, 1.f);
  noisy_split_kernel<true><<<blocks, 256, 0, st>>>(h, n_h, noise, R, K, Kp, pl, scale);
  return zsb_check_launch("split16_noisy");
}

// Batch-normalised dense layer, no bias: a = h W^T from the planes of h (h_binary: the one plane
// of a 0/1 sample, as in zsb_linear_tc_bern_sample_f32), then out [R, J] = act(xhat * gamma +
// beta), xhat = (a - mean) rstd (act = ReLU if relu), stats [2][J] = (mean, rstd).  gamma = NULL:
// out = act((a - mean) rstd + beta), rounded as such, not as gamma = 1.
//   training != 0: mean and the population variance over the R rows (EPI 9 writes a [R, J] and
//     the moment partials part [ceil(R / 128) * 2 J], merged in a fixed order), rstd =
//     rsqrt(var + eps); moving_mean / moving_var -= (moving - batch) * rate, where with bessel
//     (TF 1.x's fused batch norm, 4-D inputs) the moving variance moves towards R / (R - 1) var
//     (towards var = 0 when R = 1); a pass applies the affine step and ReLU.
//   training == 0: mean / rstd of the moving statistics, which are not changed; the product's
//     epilogue writes out (EPI 10, or 11 with gamma) and, with gamma, the pre-activation into a
//     (may be NULL) for the gradient of gamma; part is not used.
// max |out| is folded into amax_scale[2] (may be NULL).
int zsb_linear_tc_bn_f32(int training, int bessel, const void* w_planes, const float* scale_w,
                         const void* h_planes, const float* scale_h, int h_binary,
                         const float* gamma, const float* beta, float* moving_mean,
                         float* moving_var, float rate, float eps, float* stats, float* a,
                         float* part, float* out, int64_t R, int J, int K, int relu,
                         float* amax_scale, void* stream) {
  ZSB_REQUIRE(w_planes && h_planes && scale_w && scale_h && beta && moving_mean && moving_var &&
                  stats && out && R > 0 && J > 0 && K > 0 && (!training || (a && part)),
              "zsb_linear_tc_bn_f32: bad args");
  ZSB_REQUIRE(R < (1LL << 31), "zsb_linear_tc_bn_f32: too many rows");
  // EPI 10 is built on the two-plane mainloop only
  ZSB_REQUIRE(gamma || !h_binary, "zsb_linear_tc_bn_f32: a 0/1 sample needs gamma");
  cudaStream_t st = (cudaStream_t)stream;
  return with_h_binary(h_binary, [&](auto z) {
    LinCore<0, z> c;
    int rc = make_core(c, w_planes, scale_w, h_planes, scale_h, J, R, K);
    if (rc) return rc;
    if (training) {
      rc = tc_launch(LinW<BnEpi, 9, 0, z>{c, {.out = a, .part = part}}, st, "linear_tc_bn_train");
      return rc ? rc : bn_finish(a, part, R, J, gamma, beta, moving_mean, moving_var, rate, eps,
                                 bessel, stats, out, relu, amax_scale, st);
    }
    bn_stats_kernel<false><<<(unsigned)((J + 7) / 8), 256, 0, st>>>(nullptr, R, J, moving_mean,
                                                                    moving_var, rate, eps, 0,
                                                                    stats);
    if ((rc = zsb_check_launch("linear_tc_bn_stats")) != ZSB_OK) return rc;
    const BnEpi e{.bn_stats = stats, .bn_beta = beta, .out = out, .relu = relu,
                  .amax_scale = amax_scale, .bn_gamma = gamma, .pre = a};
    if constexpr (decltype(z)::value == 0)
      if (!gamma) return tc_launch(LinW<BnEpi, 10>{c, e}, st, "linear_tc_bn_eval");
    return tc_launch(LinW<BnEpi, 11, 0, z>{c, e}, st, "linear_tc_bn_eval");
  });
}

// The training step of zsb_linear_tc_bn_f32 with bessel after a pass that left the pre-activation
// a [R, J] and its per-128-row-tile moment partials part (EPI 9's layout): the deterministic
// merge, stats = (mean, rstd), the moving statistics updated, then out = act(xhat * gamma + beta),
// max |out| into amax_scale[2] (may be NULL).
int zsb_bn_finish_fused_f32(const float* a, const float* part, int64_t R, int J,
                            const float* gamma, const float* beta, float* moving_mean,
                            float* moving_var, float rate, float eps, float* stats, float* out,
                            int relu, float* amax_scale, void* stream) {
  ZSB_REQUIRE(a && part && gamma && beta && moving_mean && moving_var && stats && out && R > 0 &&
                  J > 0,
              "zsb_bn_finish_fused_f32: bad args");
  return bn_finish(a, part, R, J, gamma, beta, moving_mean, moving_var, rate, eps, 1, stats, out,
                   relu, amax_scale, (cudaStream_t)stream);
}

// Backward of zsb_linear_tc_bn_f32 from the upstream gradient g [R, J], its output y (the ReLU
// mask, read when relu), the pre-activation a (training, or when dgamma is wanted) and stats:
//   g' = g [y > 0] (relu) or g;  dbeta [J] = sum_r g',  dgamma [J] = sum_r g' xhat (either may be
//   NULL), xhat = (a - mean) rstd
//   training: da = gamma rstd (g' - mean_r g' - xhat mean_r(g' xhat));  else: da = gamma rstd g'
//   (rstd in place of gamma rstd when gamma is NULL)
// The column sums run per 128-row tile and are merged in a fixed order (deterministic).
// planes [2][R][kpad(J)] = fp16 hi/lo of da times scale[0], a power of two picked from max |da|:
// the operand of zsb_linear_tc_dgrad_f32 / zsb_linear_tc_wgrad_f32.  part = (ceil(R / 128) + 1)
// * 2 J floats of scratch; scale = device float[4] with scale[2] zero.
int zsb_bn_grad_f32(int training, const float* g, const float* y, const float* a,
                    const float* stats, const float* gamma, int relu, int64_t R, int J,
                    float* part, float* dbeta, float* dgamma, void* planes, float* scale,
                    void* stream) {
  ZSB_REQUIRE(g && stats && part && planes && scale && R > 0 && J > 0 && (!relu || y) &&
                  (!(training || dgamma) || a),
              "zsb_bn_grad_f32: bad args");
  return bn_grad<BN_GRAD_PLANES>(training, g, y, a, stats, gamma, relu, R, J, part, dbeta, dgamma,
                                 planes, nullptr, scale, (cudaStream_t)stream);
}

// As zsb_bn_grad_f32, but da [R, J] is written in fp32 and max |da| folded into scale[2]
// (device float[4] with scale[2] zero), for a consumer that gathers da before splitting it.
int zsb_bn_grad_f32out(int training, const float* g, const float* y, const float* a,
                       const float* stats, const float* gamma, int relu, int64_t R, int J,
                       float* part, float* dbeta, float* dgamma, float* da, float* scale,
                       void* stream) {
  ZSB_REQUIRE(g && stats && part && da && scale && R > 0 && J > 0 && (!relu || y) &&
                  (!(training || dgamma) || a),
              "zsb_bn_grad_f32out: bad args");
  return bn_grad<BN_GRAD_F32>(training, g, y, a, stats, gamma, relu, R, J, part, dbeta, dgamma,
                              nullptr, da, scale, (cudaStream_t)stream);
}

// Gradients of x = h[r % n_h] * noise[r] from d = dL/dx [R, K]: dnoise [R, K] = d * h[r % n_h] and
// dh [n_h, K] = the sum of d * noise over the R / n_h rows that share each row of h, added in row
// order.  Either output may be NULL.
int zsb_noisy_grad_f32(const float* d, const float* h, int64_t n_h, const float* noise, int64_t R,
                       int K, float* dnoise, float* dh, void* stream) {
  ZSB_REQUIRE(d && h && noise && R > 0 && K > 0 && n_h > 0 && R % n_h == 0,
              "zsb_noisy_grad_f32: bad args");
  noisy_grad_kernel<<<grid_blocks(n_h, 8, 16), 256, 0, (cudaStream_t)stream>>>(d, h, n_h, noise, R,
                                                                             K, dnoise, dh);
  return zsb_check_launch("noisy_grad");
}

}  // extern "C"
