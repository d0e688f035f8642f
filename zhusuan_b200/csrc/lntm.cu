// K8 for config 5: the E-step log-joint of the Logistic-Normal Topic Model and its gradient in one
// fused, sparsity-aware kernel, and the M-step likelihood gradient w.r.t. beta.
//
// Reference (examples/topic_models/lntm_mcem.py:33-48, 97-99; UnnormalizedMultinomial._log_prob,
// zhusuan/distributions/multivariate.py:435-443 with normalize_logits=False):
//     theta = softmax(eta)                         eta  [chains, docs, K]
//     phi   = softmax(beta)                        beta [K, V]
//     log p = sum_k Normal(eta_k; mean_k, exp(logstd_k)).log_prob            (cond_log_prob('eta'))
//           + sum_v x[d, v] * log(theta @ phi)[v]                            (cond_log_prob('x'))
// TensorFlow materialises doc_word = theta @ phi as a [chains * docs, V] matrix (at config 5:
// 1024 x 10 000 x 8192 floats = 335 TB -- it cannot run) and differentiates through it.  x is a bag of
// words: a document touches a few hundred of the V columns, so here only those are ever formed:
//     S_j   = sum_k theta_k * phi[k, w_j]          for the document's words w_j (CSR)
//     log p += c_j * log S_j
//     dtheta_k += (c_j / S_j) * phi[k, w_j]
//     deta  = theta * (dtheta - <theta, dtheta>) - (eta - mean) * exp(-2 logstd)
// = 4 K flops per (chain, word occurrence) instead of 4 K V per chain-document; the [rows, V] matrix
// never exists anywhere.  phi is kept transposed ([V, Kp], 4 MB at config 5: L2 resident) so that a
// word's topic vector is one contiguous 512-byte row.
//
// Any 1 <= K <= 128: the topic axis of phi_t is padded to Kp = 16 ceil(K / 16) with zero
// columns, padded topics get theta = 0 exactly, the prior sums over the K real topics only and
// padded gradient entries are never written.  eta keeps its stride K.  For K % 16 == 0 the kernel
// is the unpadded instance, whose arithmetic does not depend on the padding code.
//
// Mapping: one block = one document x 64 chains; a quad of threads owns a chain (each thread Kp/4
// topics, as float4 groups interleaved across the quad: conflict-free LDS.128 of the phi tile, the
// 8 chains of a warp read the same words by broadcast); 32 words of the document at a time are
// staged in shared memory.  Bound by the fp32 FMA pipe (2 FMAs + 1/16 LDS.128 per topic-word).
#include "common.cuh"

namespace {

constexpr int LN_CHAINS = 64;        // chains per block
constexpr int LN_WORDS = 32;         // words staged per round
constexpr int LN_MAX_TOPICS = 128;
constexpr int LN_MS_WARPS = 8;       // M-step forward: warps sharing one (chain, document)

inline int lntm_padded_topics(int64_t K) { return (int)(16 * zsb_ceil_div(K, 16)); }

// phi_t[v, k] = softmax_v(beta[k, :])[v] for k < K and 0 for K <= k < Kp: one block per topic row,
// two passes
__global__ void __launch_bounds__(256) lntm_phi_t_kernel(const float* __restrict__ beta, int K,
                                                         int Kp, int64_t V,
                                                         float* __restrict__ phi_t) {
  __shared__ float red[32];
  const int k = blockIdx.x;
  if (k >= K) {
    for (int64_t v = threadIdx.x; v < V; v += blockDim.x) phi_t[v * Kp + k] = 0.f;
    return;
  }
  const float* __restrict__ b = beta + (int64_t)k * V;
  float m = -INFINITY;
  for (int64_t v = threadIdx.x; v < V; v += blockDim.x) m = fmaxf(m, b[v]);
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  m = red[0];
  for (int i = 1; i < (int)(blockDim.x >> 5); ++i) m = fmaxf(m, red[i]);
  __syncthreads();
  float s = 0.f;
  for (int64_t v = threadIdx.x; v < V; v += blockDim.x) s += expf(b[v] - m);
  s = block_sum(s, red);
  const float inv = 1.f / s;
  for (int64_t v = threadIdx.x; v < V; v += blockDim.x) phi_t[v * Kp + k] = expf(b[v] - m) * inv;
}

// Topics k0 .. k0 + 3 of a row of K floats, `pad` past the last topic.  The unpadded instance loads
// 16 bytes; the padded one loads scalars, since a row is not 16-byte aligned when K % 4 != 0.
template <bool PAD>
__device__ __forceinline__ float4 lntm_ld4(const float* __restrict__ p, int k0, int K, float pad) {
  if (!PAD) return *reinterpret_cast<const float4*>(p + k0);
  return make_float4(k0 < K ? p[k0] : pad, k0 + 1 < K ? p[k0 + 1] : pad,
                     k0 + 2 < K ? p[k0 + 2] : pad, k0 + 3 < K ? p[k0 + 3] : pad);
}

// The same, re-read from memory: an asm volatile load cannot be merged with an earlier load of the
// same address, so the compiler does not keep the prologue's eta / mean / logstd alive across the
// word loop (which at Kp >= 112 spills them to the stack).
__device__ __forceinline__ float lntm_reload(const float* p) {
  float v;
  asm volatile("ld.global.nc.f32 %0, [%1];" : "=f"(v) : "l"(p));
  return v;
}
template <bool PAD>
__device__ __forceinline__ float4 lntm_reload4(const float* __restrict__ p, int k0, int K) {
  if (!PAD) {
    float4 v;
    asm volatile("ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p + k0));
    return v;
  }
  return make_float4(k0 < K ? lntm_reload(p + k0) : 0.f, k0 + 1 < K ? lntm_reload(p + k0 + 1) : 0.f,
                     k0 + 2 < K ? lntm_reload(p + k0 + 2) : 0.f,
                     k0 + 3 < K ? lntm_reload(p + k0 + 3) : 0.f);
}

template <int G, bool PAD>           // G = float4 groups per thread = Kp / 16; PAD: K < Kp
__global__ void __launch_bounds__(256, 2) lntm_logjoint_kernel(
    const float* __restrict__ eta, const float* __restrict__ eta_mean,
    const float* __restrict__ eta_logstd, const float* __restrict__ phi_t,
    const int64_t* __restrict__ doc_ptr, const int32_t* __restrict__ word_idx,
    const float* __restrict__ word_cnt, const int64_t* __restrict__ doc_ids,
    const float* __restrict__ temperature, float* __restrict__ lp_out,
    float* __restrict__ grad_out, int64_t chains, int64_t docs, int n_topics) {
  constexpr int KP = 16 * G;
  const int K = PAD ? n_topics : KP;
  __shared__ float4 tile[LN_WORDS][KP / 4];      // phi_t rows of the staged words
  __shared__ float cnt[LN_WORDS];
  const int q = threadIdx.x & 3;                 // thread inside the chain's quad
  const int64_t d = blockIdx.x;                  // row of eta; corpus document doc_ids[d]
  const int64_t c = (int64_t)blockIdx.y * LN_CHAINS + (threadIdx.x >> 2);
  const bool live = c < chains;
  const int64_t row = (live ? c : 0) * docs + d;
  const float* __restrict__ e = eta + row * K;

  // this thread's topics: float4 groups g*4 + q, g < G; padded topics start at -inf: theta = 0
  float4 th[G], dth[G];
  float mx = -INFINITY;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    th[g] = lntm_ld4<PAD>(e, 4 * (g * 4 + q), K, -INFINITY);
    dth[g] = make_float4(0.f, 0.f, 0.f, 0.f);
    mx = fmaxf(mx, fmaxf(fmaxf(th[g].x, th[g].y), fmaxf(th[g].z, th[g].w)));
  }
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
  mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
  // prior (Normal, group_ndims = 1) on eta before it is overwritten by theta
  float lp = 0.f;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    const int k0 = 4 * (g * 4 + q);
    const float4 mu = PAD ? float4{} : lntm_ld4<false>(eta_mean, k0, K, 0.f);
    const float4 ls = PAD ? float4{} : lntm_ld4<false>(eta_logstd, k0, K, 0.f);
    const float ev[4] = {th[g].x, th[g].y, th[g].z, th[g].w};
    const float mv[4] = {mu.x, mu.y, mu.z, mu.w};
    const float lv[4] = {ls.x, ls.y, ls.z, ls.w};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      if (PAD && k0 + i >= K) continue;               // the prior is over the real topics only
      const float l = PAD ? eta_logstd[k0 + i] : lv[i];
      const float prec = expf(-2.f * l);
      const float dd = ev[i] - (PAD ? eta_mean[k0 + i] : mv[i]);
      lp += -0.9189385332046727f - l - 0.5f * prec * dd * dd;         // univariate.py:174-181
    }
  }
  float sum = 0.f;
#pragma unroll
  for (int g = 0; g < G; ++g) {
    th[g].x = expf(th[g].x - mx); th[g].y = expf(th[g].y - mx);
    th[g].z = expf(th[g].z - mx); th[g].w = expf(th[g].w - mx);
    sum += (th[g].x + th[g].y) + (th[g].z + th[g].w);
  }
  sum += __shfl_xor_sync(0xffffffffu, sum, 1);
  sum += __shfl_xor_sync(0xffffffffu, sum, 2);
  const float inv = 1.f / sum;
#pragma unroll
  for (int g = 0; g < G; ++g) { th[g].x *= inv; th[g].y *= inv; th[g].z *= inv; th[g].w *= inv; }

  const int64_t doc = doc_ids ? doc_ids[d] : d;
  const int64_t w0 = doc_ptr[doc], w1 = doc_ptr[doc + 1];
  for (int64_t wb = w0; wb < w1; wb += LN_WORDS) {
    const int nw = (int)((w1 - wb < LN_WORDS) ? (w1 - wb) : LN_WORDS);
    __syncthreads();                                   // previous round consumed
    for (int i = threadIdx.x; i < nw * (KP / 4); i += blockDim.x) {
      const int w = i / (KP / 4), kk = i % (KP / 4);
      tile[w][kk] = *reinterpret_cast<const float4*>(
          phi_t + (int64_t)word_idx[wb + w] * KP + 4 * kk);
    }
    if ((int)threadIdx.x < nw) {       // tempered: t c_j scales the likelihood and its gradient
      const float cw = word_cnt[wb + threadIdx.x];
      cnt[threadIdx.x] = temperature ? *temperature * cw : cw;
    }
    __syncthreads();
    for (int w = 0; w < nw; ++w) {
      float s = 0.f;
#pragma unroll
      for (int g = 0; g < G; ++g) {
        const float4 ph = tile[w][g * 4 + q];
        s = fmaf(th[g].x, ph.x, s); s = fmaf(th[g].y, ph.y, s);
        s = fmaf(th[g].z, ph.z, s); s = fmaf(th[g].w, ph.w, s);
      }
      s += __shfl_xor_sync(0xffffffffu, s, 1);
      s += __shfl_xor_sync(0xffffffffu, s, 2);
      const float cw = cnt[w];
      const float r = cw / s;                          // multivariate.py:435-443 differentiated
      if (q == 0) lp += cw * logf(s);
      if (grad_out == nullptr) continue;               // value only (MH test): skip the axpy
#pragma unroll
      for (int g = 0; g < G; ++g) {                    // (re-read: keeps the kernel at 2 blocks/SM)
        const float4 ph = tile[w][g * 4 + q];
        dth[g].x = fmaf(r, ph.x, dth[g].x); dth[g].y = fmaf(r, ph.y, dth[g].y);
        dth[g].z = fmaf(r, ph.z, dth[g].z); dth[g].w = fmaf(r, ph.w, dth[g].w);
      }
    }
  }
  // softmax backward + prior gradient
  float dot = 0.f;
#pragma unroll
  for (int g = 0; g < G; ++g)
    dot += (th[g].x * dth[g].x + th[g].y * dth[g].y) + (th[g].z * dth[g].z + th[g].w * dth[g].w);
  dot += __shfl_xor_sync(0xffffffffu, dot, 1);
  dot += __shfl_xor_sync(0xffffffffu, dot, 2);
  lp += __shfl_xor_sync(0xffffffffu, lp, 1);
  lp += __shfl_xor_sync(0xffffffffu, lp, 2);
  if (!live) return;
  if (lp_out && q == 0) lp_out[row] = lp;
  if (grad_out) {
    float* __restrict__ go = grad_out + row * K;
#pragma unroll
    for (int g = 0; g < G; ++g) {
      const int k0 = 4 * (g * 4 + q);
      const float4 ev = lntm_reload4<PAD>(e, k0, K);                   // prior gradient
      const float4 mu = lntm_reload4<PAD>(eta_mean, k0, K);
      const float4 ls = lntm_reload4<PAD>(eta_logstd, k0, K);
      float4 o;
      o.x = fmaf(th[g].x, dth[g].x - dot, -expf(-2.f * ls.x) * (ev.x - mu.x));
      o.y = fmaf(th[g].y, dth[g].y - dot, -expf(-2.f * ls.y) * (ev.y - mu.y));
      o.z = fmaf(th[g].z, dth[g].z - dot, -expf(-2.f * ls.z) * (ev.z - mu.z));
      o.w = fmaf(th[g].w, dth[g].w - dot, -expf(-2.f * ls.w) * (ev.w - mu.w));
      if (!PAD) {
        *reinterpret_cast<float4*>(go + k0) = o;
      } else {                                         // padded topics are never written
        if (k0 < K) go[k0] = o.x;
        if (k0 + 1 < K) go[k0 + 1] = o.y;
        if (k0 + 2 < K) go[k0 + 2] = o.z;
        if (k0 + 3 < K) go[k0 + 3] = o.w;
      }
    }
  }
}

// M-step forward: one block per (chain, row of eta), warp w takes the document's words
// w, w + 8, ...; lane l owns topics l + 32 i.  Writes theta [chains, docs, Kp] (0 on padded
// topics), ratio[c, j] = c_j / S_cj for the document's corpus entries j, and
// lp = sum_j c_j log S_cj, summed per warp and then over the warps in order.
__global__ void __launch_bounds__(32 * LN_MS_WARPS) lntm_mstep_fwd_kernel(
    const float* __restrict__ eta, const float* __restrict__ phi_t,
    const int64_t* __restrict__ doc_ptr, const int32_t* __restrict__ word_idx,
    const float* __restrict__ word_cnt, const int64_t* __restrict__ doc_ids,
    float* __restrict__ lp_out, float* __restrict__ ratio, float* __restrict__ theta,
    int64_t docs, int64_t nnz, int K, int Kp) {
  constexpr int NT = LN_MAX_TOPICS / 32;
  __shared__ float part[LN_MS_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t pair = blockIdx.x;
  const int64_t c = pair / docs, d = pair % docs;
  const float* __restrict__ e = eta + pair * K;
  float th[NT];
  float mx = -INFINITY;
#pragma unroll
  for (int i = 0; i < NT; ++i) {
    const int k = lane + 32 * i;
    th[i] = k < K ? e[k] : -INFINITY;
    mx = fmaxf(mx, th[i]);
  }
  mx = warp_max(mx);
  float sum = 0.f;
#pragma unroll
  for (int i = 0; i < NT; ++i) { th[i] = expf(th[i] - mx); sum += th[i]; }
  const float inv = 1.f / warp_sum(sum);
  float* __restrict__ tr = theta + pair * Kp;
#pragma unroll
  for (int i = 0; i < NT; ++i) {
    th[i] *= inv;
    if (warp == 0 && lane + 32 * i < Kp) tr[lane + 32 * i] = th[i];
  }
  const int64_t doc = doc_ids ? doc_ids[d] : d;
  float lp = 0.f;
  for (int64_t j = doc_ptr[doc] + warp; j < doc_ptr[doc + 1]; j += LN_MS_WARPS) {
    const float* __restrict__ ph = phi_t + (int64_t)word_idx[j] * Kp;
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < NT; ++i)
      if (lane + 32 * i < K) s = fmaf(th[i], ph[lane + 32 * i], s);
    s = warp_sum(s);
    const float cw = word_cnt[j];
    lp += cw * logf(s);
    if (lane == 0) ratio[c * nnz + j] = cw / s;
  }
  if (lane == 0) part[warp] = lp;
  __syncthreads();
  if (threadIdx.x == 0) {
    float t = 0.f;
    for (int w = 0; w < LN_MS_WARPS; ++w) t += part[w];
    lp_out[pair] = t;
  }
}

// M-step backward, one block per vocabulary word v, thread k per topic:
//   G[v, k] = sum_{entries j of word v} sum_c g[c, d_j] ratio[c, j] theta[c, d_j, k]
// over the word's corpus entries in CSC order, skipping documents outside the batch
// (doc_slot[doc] < 0).  The block reads the entries' indices blockDim.x at a time and keeps the
// batch's entries in order in shared memory, so that a word found in many documents costs one
// coalesced read per blockDim.x entries.  A fixed order and no atomics: the same inputs give the
// same bits.
__global__ void __launch_bounds__(LN_MAX_TOPICS) lntm_mstep_word_kernel(
    const float* __restrict__ g, const float* __restrict__ ratio,
    const float* __restrict__ theta, const int64_t* __restrict__ csc_ptr,
    const int32_t* __restrict__ csc_entry, const int32_t* __restrict__ entry_doc,
    const int32_t* __restrict__ doc_slot, float* __restrict__ G, int64_t chains, int64_t docs,
    int64_t nnz, int Kp) {
  __shared__ int32_t s_entry[LN_MAX_TOPICS], s_slot[LN_MAX_TOPICS];
  __shared__ int s_warp[LN_MAX_TOPICS / 32];
  const int64_t v = blockIdx.x;
  const int k = threadIdx.x, lane = k & 31, warp = k >> 5;
  const int64_t i1 = csc_ptr[v + 1];
  float acc = 0.f;
  for (int64_t i0 = csc_ptr[v]; i0 < i1; i0 += blockDim.x) {
    int32_t j = 0, slot = -1;
    if (i0 + k < i1) {
      j = csc_entry[i0 + k];
      slot = doc_slot ? doc_slot[entry_doc[i0 + k]] : entry_doc[i0 + k];
    }
    const unsigned keep = __ballot_sync(0xffffffffu, slot >= 0);
    if (lane == 0) s_warp[warp] = __popc(keep);
    __syncthreads();
    int pos = __popc(keep & ((1u << lane) - 1u)), n = 0;
    for (int w = 0; w < (int)(blockDim.x >> 5); ++w) {
      if (w < warp) pos += s_warp[w];
      n += s_warp[w];
    }
    if (slot >= 0) { s_entry[pos] = j; s_slot[pos] = slot; }
    __syncthreads();
    if (k < Kp) {
      for (int e = 0; e < n; ++e) {
        const int64_t je = s_entry[e], se = s_slot[e];
        for (int64_t c = 0; c < chains; ++c) {
          const float r = g[c * docs + se] * ratio[c * nnz + je];
          acc = fmaf(r, theta[(c * docs + se) * Kp + k], acc);
        }
      }
    }
    __syncthreads();                                   // the next round rewrites the lists
  }
  if (k < Kp) G[v * Kp + k] = acc;
}

// dbeta[k, v] = phi[k, v] (G[v, k] - sum_v' phi[k, v'] G[v', k]): the softmax over the vocabulary
// (lntm_mcem.py:42) differentiated, one block per topic, the sum over v in a fixed order.
__global__ void __launch_bounds__(256) lntm_mstep_topic_kernel(const float* __restrict__ phi_t,
                                                               const float* __restrict__ G,
                                                               int64_t V, int Kp,
                                                               float* __restrict__ dbeta) {
  __shared__ float red[32];
  const int k = blockIdx.x;
  float dot = 0.f;
  for (int64_t v = threadIdx.x; v < V; v += blockDim.x)
    dot = fmaf(phi_t[v * Kp + k], G[v * Kp + k], dot);
  dot = block_sum(dot, red);
  float* __restrict__ out = dbeta + (int64_t)k * V;
  for (int64_t v = threadIdx.x; v < V; v += blockDim.x)
    out[v] = phi_t[v * Kp + k] * (G[v * Kp + k] - dot);
}

}  // namespace

extern "C" {

// phi_t [V, Kp] = softmax(beta [K, V], axis = vocabulary) transposed (lntm_mcem.py:41), with
// Kp = 16 ceil(K / 16) and zero pad columns.
int zsb_lntm_phi_t_f32(const float* beta, int64_t n_topics, int64_t n_vocab, float* phi_t,
                       void* stream) {
  ZSB_REQUIRE(beta && phi_t && n_topics > 0 && n_vocab > 0, "zsb_lntm_phi_t_f32: bad args");
  const int Kp = lntm_padded_topics(n_topics);
  lntm_phi_t_kernel<<<(unsigned)Kp, 256, 0, (cudaStream_t)stream>>>(beta, (int)n_topics, Kp,
                                                                    n_vocab, phi_t);
  return zsb_check_launch("lntm_phi_t");
}

// E-step log-joint of the LNTM and its gradient w.r.t. eta (lntm_mcem.py:33-48, 97-99), tempered
// for AIS (evaluation.py:91-94).
//   eta [chains, docs, n_topics]; eta_mean / eta_logstd [n_topics]; phi_t [n_vocab, Kp];
//   corpus in CSR: doc_ptr [n_corpus_docs + 1] (int64), word_idx [nnz] (int32), word_cnt [nnz];
//   doc_ids [docs] (int64): row d of eta is corpus document doc_ids[d]; NULL = documents 0..docs-1;
//   temperature: a device scalar t; the result is prior + t * likelihood and its gradient, i.e.
//   log_prior * (1 - t) + log_joint * t when the proposal is the eta prior.  NULL = t of 1.
//   lp_out [chains, docs] and / or grad_out like eta.  1 <= n_topics <= 128.
int zsb_lntm_logjoint_f32(const float* eta, const float* eta_mean, const float* eta_logstd,
                          const float* phi_t, const int64_t* doc_ptr, const int32_t* word_idx,
                          const float* word_cnt, const int64_t* doc_ids, const float* temperature,
                          float* lp_out, float* grad_out, int64_t chains, int64_t docs,
                          int64_t n_topics, void* stream) {
  ZSB_REQUIRE(eta && eta_mean && eta_logstd && phi_t && doc_ptr && (lp_out || grad_out) &&
                  chains > 0 && docs > 0 && docs < (1LL << 31),
              "zsb_lntm_logjoint_f32: bad args");
  ZSB_REQUIRE(n_topics >= 1 && n_topics <= LN_MAX_TOPICS,
              "zsb_lntm_logjoint_f32: n_topics must be in [1, 128] (got %lld)",
              (long long)n_topics);
  const dim3 grid((unsigned)docs, (unsigned)zsb_ceil_div(chains, LN_CHAINS));
  ZSB_REQUIRE(grid.y < 65536, "zsb_lntm_logjoint_f32: too many chains");
  cudaStream_t st = (cudaStream_t)stream;
  const int K = (int)n_topics;
#define ZSB_LN(G, PAD)                                                                         \
  lntm_logjoint_kernel<G, PAD><<<grid, 256, 0, st>>>(eta, eta_mean, eta_logstd, phi_t, doc_ptr, \
                                                     word_idx, word_cnt, doc_ids, temperature, \
                                                     lp_out, grad_out, chains, docs, K)
#define ZSB_LN_G(G)                                                                            \
  case G:                                                                                      \
    if (K % 16 == 0) ZSB_LN(G, false); else ZSB_LN(G, true);                                   \
    break;
  switch (lntm_padded_topics(K) / 16) {
    ZSB_LN_G(1) ZSB_LN_G(2) ZSB_LN_G(3) ZSB_LN_G(4)
    ZSB_LN_G(5) ZSB_LN_G(6) ZSB_LN_G(7) ZSB_LN_G(8)
  }
#undef ZSB_LN_G
#undef ZSB_LN
  return zsb_check_launch("lntm_logjoint");
}

// M-step likelihood, forward (lntm_mcem.py:106-110, cond_log_prob('x')):
//   lp_out [chains, docs] = log p(x_d | eta_c, beta) = sum_j c_j log S_cj over the entries j of
//   corpus document doc_ids[d] (doc_ids NULL: document d), S_cj = (softmax(eta_cd) @ phi)[w_j].
//   Also writes what zsb_lntm_mstep_grad_f32 reads: theta [chains, docs, Kp] and
//   ratio [chains, nnz] (c_j / S_cj at the batch's corpus entries; other entries are not written).
int zsb_lntm_mstep_f32(const float* eta, const float* phi_t, const int64_t* doc_ptr,
                       const int32_t* word_idx, const float* word_cnt, const int64_t* doc_ids,
                       float* lp_out, float* ratio, float* theta, int64_t chains, int64_t docs,
                       int64_t nnz, int64_t n_topics, void* stream) {
  ZSB_REQUIRE(eta && phi_t && doc_ptr && word_idx && word_cnt && lp_out && ratio && theta &&
                  chains > 0 && docs > 0 && nnz >= 0 && n_topics >= 1 &&
                  n_topics <= LN_MAX_TOPICS,
              "zsb_lntm_mstep_f32: bad args");
  ZSB_REQUIRE(chains * docs < (1LL << 31), "zsb_lntm_mstep_f32: too many (chain, document) pairs");
  lntm_mstep_fwd_kernel<<<(unsigned)(chains * docs), 32 * LN_MS_WARPS, 0, (cudaStream_t)stream>>>(
      eta, phi_t, doc_ptr, word_idx, word_cnt, doc_ids, lp_out, ratio, theta, docs, nnz,
      (int)n_topics, lntm_padded_topics(n_topics));
  return zsb_check_launch("lntm_mstep");
}

// M-step likelihood, gradient (lntm_mcem.py:106-114, tf.gradients w.r.t. beta):
//   dbeta [n_topics, n_vocab] = d/d beta of sum_{c,d} g[c, d] lp[c, d], from the theta and ratio
//   that zsb_lntm_mstep_f32 wrote with the same eta, doc_ids and phi_t.
//   Corpus entries by word (CSC): csc_ptr [n_vocab + 1] (int64); csc_entry [nnz] the corpus entry
//   index j, ascending within a word; entry_doc [nnz] its corpus document.
//   doc_slot [n_corpus_docs]: the row d with doc_ids[d] == doc, -1 for documents outside the batch
//   (doc_ids must be distinct); NULL when doc_ids was NULL.
//   G [n_vocab, Kp] is scratch.  Deterministic: fixed summation orders, no atomics.
int zsb_lntm_mstep_grad_f32(const float* g, const float* ratio, const float* theta,
                            const float* phi_t, const int64_t* csc_ptr, const int32_t* csc_entry,
                            const int32_t* entry_doc, const int32_t* doc_slot, float* G,
                            float* dbeta, int64_t chains, int64_t docs, int64_t nnz,
                            int64_t n_topics, int64_t n_vocab, void* stream) {
  ZSB_REQUIRE(g && ratio && theta && phi_t && csc_ptr && csc_entry && entry_doc && G && dbeta &&
                  chains > 0 && docs > 0 && nnz >= 0 && n_topics >= 1 &&
                  n_topics <= LN_MAX_TOPICS && n_vocab > 0 && n_vocab < (1LL << 31),
              "zsb_lntm_mstep_grad_f32: bad args");
  cudaStream_t st = (cudaStream_t)stream;
  const int Kp = lntm_padded_topics(n_topics);
  lntm_mstep_word_kernel<<<(unsigned)n_vocab, (unsigned)(32 * zsb_ceil_div(Kp, 32)), 0, st>>>(
      g, ratio, theta, csc_ptr, csc_entry, entry_doc, doc_slot, G, chains, docs, nnz, Kp);
  int rc = zsb_check_launch("lntm_mstep_word");
  if (rc) return rc;
  lntm_mstep_topic_kernel<<<(unsigned)n_topics, 256, 0, st>>>(phi_t, G, n_vocab, Kp, dbeta);
  return zsb_check_launch("lntm_mstep_topic");
}

}  // extern "C"
