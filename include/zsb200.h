/* zsb200.h -- C ABI of libzsb200.so, the H100 (sm_90a) kernels behind zhusuan's
 * HMC / SG-MCMC / ELBO-IWAE hot path.
 *
 * The reference (thu-ml/zhusuan) has NO native boundary: its arithmetic is TensorFlow-1.x graph
 * ops.  Each entry point below therefore replaces a *set of TF ops inside one reference function*;
 * the function it replaces is cited as zhusuan/<file>:<lines>.  INTEGRATION.md shows the ctypes
 * binding a zhusuan maintainer would add at each of those sites.
 *
 * Conventions
 *   - every function returns int: 0 ok, <0 error (ZSB_ERR_*); zsb_last_error() gives the message
 *     of the calling thread's last failure.  No exceptions cross the ABI.
 *   - all data pointers are DEVICE pointers to float32 / int32 unless marked host; the caller
 *     owns every buffer.  `stream` is a cudaStream_t (NULL = legacy default stream); all work is
 *     enqueued asynchronously on it, nothing synchronises.
 *   - latents are row-major [chains, row_len]; per-dimension vectors are [row_len].
 *   - operands named (ptr, ptr_n) are broadcast by modular indexing: element i reads ptr[i % ptr_n]
 *     (covers every broadcast where the operand's shape is a suffix of the result's shape).
 *   - `noise`/`u`/`eps` pointers may be NULL: the kernel then draws Philox4x32-10 numbers keyed by
 *     (seed; stream id, iter, row0 + local chain, 4-element block), i.e. by GLOBAL chain index, so
 *     results do not depend on how chains are sharded over GPUs.
 *   - there is no CPU fallback: without a CUDA device every compute call fails with ZSB_ERR_CUDA.
 */
#ifndef ZSB200_H_
#define ZSB200_H_
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ZSB_OK 0
#define ZSB_ERR_INVALID (-1)
#define ZSB_ERR_CUDA (-2)
#define ZSB_ERR_UNSUPPORTED (-3)

int zsb_version(void);
int zsb_last_error(char* buf, size_t n);       /* host buffer */
int zsb_device_count(void);
int zsb_stream_sync(void* stream);
/* Device-resident draw epoch.  The reference's random ops (tf.random_normal hmc.py:22,
 * univariate.py:161-172; tf.random_uniform univariate.py:386-396; tf.random.categorical
 * univariate.py:478-494; tf.random_gamma multivariate.py:660-663) advance a per-op counter on every
 * sess.run.  Here every sampler call takes (seed, iter) by value; when a step is captured once into
 * a CUDA graph those values are frozen, so a registered device uint32 `epoch` is ADDED to `iter`
 * inside the kernels and zsb_random_bump_epoch (captured at the end of the step) advances it:
 * each replay draws fresh numbers.  NULL unregisters. */
int zsb_random_set_device_epoch(const uint32_t* epoch);
int zsb_random_bump_epoch(uint32_t* epoch, uint32_t by, void* stream);

/* ---- sampler state block: 16 float32 in device memory (tf.Variables of hmc.py:258-264,
 *      StepsizeTuner hmc.py:82-87, EWMV.t hmc.py:118) ------------------------------------- */
enum {
  ZSB_HMC_STATE_T = 0, ZSB_HMC_STATE_STEP_SIZE = 1, ZSB_HMC_STATE_TUNER_STEP = 2,
  ZSB_HMC_STATE_LOG_EPS_BAR = 3, ZSB_HMC_STATE_H_BAR = 4, ZSB_HMC_STATE_MU = 5,
  ZSB_HMC_STATE_EWMV_T = 6, ZSB_HMC_STATE_EPS_USED = 7, ZSB_HMC_STATE_ACC_MEAN = 8,
  ZSB_HMC_STATE_FLAGS = 9 /* uint32 bits; bit0 = non-finite old log-prob, hmc.py:51-53 */,
  ZSB_HMC_STATE_SEARCH_LAST = 10, ZSB_HMC_STATE_SEARCH_COND = 11, ZSB_HMC_STATE_SIZE = 16
};

/* ---- K1: Distribution.log_prob (zhusuan/distributions/base.py:290-304) --------------------- */
/* Normal._log_prob univariate.py:174-181; out[r] = sum over `group` consecutive elements. */
int zsb_logprob_normal_f32(const float* given, int64_t given_n, const float* mean, int64_t mean_n,
                           const float* logstd, int64_t logstd_n, float* out, int64_t n_out,
                           int64_t group, void* stream);
/* analytic backward (replaces tf.gradients through :174-181); outputs nullable, n_out*group each */
int zsb_logprob_normal_bwd_f32(const float* given, int64_t given_n, const float* mean,
                               int64_t mean_n, const float* logstd, int64_t logstd_n,
                               const float* gout, int64_t n_out, int64_t group, float* dgiven,
                               float* dmean, float* dlogstd, void* stream);
/* Bernoulli._log_prob univariate.py:398-403 (given pre-cast to float, :399) */
int zsb_logprob_bernoulli_f32(const float* given, int64_t given_n, const float* logits,
                              int64_t logits_n, float* out, int64_t n_out, int64_t group,
                              void* stream);
int zsb_logprob_bernoulli_bwd_f32(const float* given, int64_t given_n, const float* logits,
                                  int64_t logits_n, const float* gout, int64_t n_out,
                                  int64_t group, float* dlogits, void* stream);
/* Categorical._log_prob univariate.py:496-548; logits [logits_rows, C], out [rows] */
int zsb_logprob_categorical_f32(const int32_t* given, int64_t given_n, const float* logits,
                                int64_t logits_rows, int64_t n_categories, float* out,
                                int64_t rows, void* stream);
int zsb_logprob_categorical_bwd_f32(const int32_t* given, int64_t given_n, const float* logits,
                                    int64_t logits_rows, int64_t n_categories, const float* gout,
                                    float* dlogits, int64_t rows, void* stream);
/* Dirichlet._log_prob multivariate.py:665-677 */
int zsb_logprob_dirichlet_f32(const float* given, int64_t given_rows, const float* alpha,
                              int64_t alpha_rows, int64_t n_categories, float* out, int64_t rows,
                              void* stream);
int zsb_logprob_dirichlet_bwd_given_f32(const float* given, int64_t given_rows,
                                        const float* alpha, int64_t alpha_rows,
                                        int64_t n_categories, const float* gout, float* dgiven,
                                        int64_t rows, void* stream);
/* UnnormalizedMultinomial._log_prob multivariate.py:435-443 */
int zsb_logprob_unnorm_multinomial_f32(const float* given, int64_t given_rows,
                                       const float* logits, int64_t logits_rows,
                                       int64_t n_categories, int normalize_logits, float* out,
                                       int64_t rows, void* stream);
int zsb_logprob_unnorm_multinomial_bwd_f32(const float* given, int64_t given_rows,
                                           const float* logits, int64_t logits_rows,
                                           int64_t n_categories, int normalize_logits,
                                           const float* gout, float* dlogits, int64_t rows,
                                           void* stream);
/* MultivariateNormalCholesky._log_prob multivariate.py:169-189; x_out (nullable) = L^-1(x-mean) */
int zsb_logprob_mvn_chol_f32(const float* given, int64_t given_rows, const float* mean,
                             int64_t mean_rows, const float* cov_tril, int64_t tril_mats,
                             int64_t n_dim, float* out, float* x_out, int64_t rows, void* stream);
int zsb_logprob_mvn_chol_bwd_given_f32(const float* x_in, const float* cov_tril,
                                       int64_t tril_mats, int64_t n_dim, const float* gout,
                                       float* dgiven, int64_t rows, void* stream);
/* reduce_sum over the last group_ndims axes, base.py:303-304 */
int zsb_group_sum_f32(const float* in, float* out, int64_t n_out, int64_t group, void* stream);

/* ---- K7: Normal._sample (univariate.py:161-172) fused with cond_log_p (bn.py:194-204) ------- */
int zsb_reparam_normal_f32(const float* mean, int64_t mean_n, const float* logstd,
                           int64_t logstd_n, const float* eps, uint64_t seed, uint32_t iter,
                           float* z_out, float* eps_out, float* logq_out, int64_t n_out,
                           int64_t group, void* stream);
/* Bernoulli._sample univariate.py:386-396 */
int zsb_sample_bernoulli_i32(const float* logits, int64_t logits_n, const float* u, uint64_t seed,
                             uint32_t iter, int32_t* out, int64_t n, void* stream);

/* ---- K1 (widened): the other elementwise univariate densities behind one entry point.
 * dist: 0 FoldNormal(mean, logstd) univariate.py:319-329 | 1 Uniform(minval, maxval) :646-660
 *       2 Gamma(alpha, beta) :737-747 | 3 Beta(alpha, beta) :833-851 | 4 Poisson(rate, NULL) :922-933
 *       5 Binomial(logits, n) :1047-1064 | 6 InverseGamma(alpha, beta) :1146-1158
 *       7 Laplace(loc, scale) :1267-1273 | 8 BinConcrete(temperature, logits) :1381-1400
 * Operands broadcast modularly like zsb_logprob_normal_f32; out [n_out] = sum over `group`.
 * The backward writes full-size elementwise gradients (each output nullable). */
int zsb_logprob_univariate_f32(int dist, const float* given, int64_t given_n, const float* a,
                               int64_t a_n, const float* b, int64_t b_n, float* out,
                               int64_t n_out, int64_t group, void* stream);
int zsb_logprob_univariate_bwd_f32(int dist, const float* given, int64_t given_n, const float* a,
                                   int64_t a_n, const float* b, int64_t b_n, const float* gout,
                                   int64_t n_out, int64_t group, float* dgiven, float* da,
                                   float* db, void* stream);

/* ---- K6: sample-axis reductions; x viewed as [outer, K, inner], reduced over K --------------
 * op 0 log_mean_exp (zhusuan/utils.py:177-196; monte_carlo.py:137-141)
 *    1 mean         (exclusive_kl.py:131-137)   2 log_sum_exp (utils.py:153-174)   3 sum       */
int zsb_reduce_fwd_f32(int op, const float* x, float* out, int64_t outer, int64_t K, int64_t inner,
                       void* stream);
/* backward = what tf.gradients yields for .sgvb(): softmax weights (op 0/2), 1/K (op 1) */
int zsb_reduce_bwd_f32(int op, const float* x, const float* y, const float* gout, float* dx,
                       int64_t outer, int64_t K, int64_t inner, void* stream);

/* ---- K6b: score-function / self-normalised estimators on the same tile (no backward: the
 * reference wraps them in tf.stop_gradient) ------------------------------------------------------
 * VIMCO learning signal, monte_carlo.py:194-223: signal[k] = LME_j(x_j) - LME_j(x_j with entry k
 * replaced by the mean of the others); O(K) per column instead of the reference's [.., K, K] tile.
 * `lme` (optional, [outer, inner]) receives log_mean_exp(x).  K >= 2 (ValueError in the reference). */
int zsb_vimco_signal_f32(const float* x, float* signal, float* lme, int64_t outer, int64_t K,
                         int64_t inner, void* stream);
/* self-normalised importance weights, inclusive_kl.py:139-143: exp(x - max) / sum exp(x - max) */
int zsb_normalized_weights_f32(const float* x, float* w, int64_t outer, int64_t K, int64_t inner,
                               void* stream);

/* ---- K8: dense layer of a VAE/BNN log-joint on wgmma with the likelihood fused into the GEMM
 * epilogue (the model code of examples/variational_autoencoders/iwae.py:23-32: tf.layers.dense +
 * bn.bernoulli('x', logits, group_ndims=1)); fp32 accuracy from a 3-product fp16 hi/lo split.
 * Operands are fp16 plane pairs [2][rows][Kp], Kp = zsb_linear_tc_kpad(K), produced by
 * zsb_split16_pad_f32 together with their power-of-two scale (device float[4], zeroed once).
 *   epi 0: out [R, J] = h W^T + bias (ReLU if relu)
 *   epi 1: out [R]    = sum_j Bernoulli(logits).log_prob(x[r % n_x, j])   (univariate.py:398-403,
 *          base.py:303-304); part = scratch of zsb_linear_tc_nparts(J) * R floats
 *   epi 2: out [R, J] = gout[r] * (x - sigmoid(logits))   (gradient of epi 1 wrt the logits)   */
int zsb_linear_tc_kpad(int K);
int zsb_linear_tc_nparts(int J);
int zsb_split16_pad_f32(const float* src, int64_t rows, int K, void* planes, float* scale,
                        void* stream);
/* split-K slices of the weight-gradient product zsb_linear_tc_wgrad_f32 with R output rows, J
 * features and contraction length K (its `part` holds slices * R * J floats) */
int zsb_linear_tc_slices(int64_t R, int J, int K);
/* `part` is read by epi 1 only */
int zsb_linear_tc_f32(int epi, const void* w_planes, const float* scale_w, const void* h_planes,
                      const float* scale_h, const float* bias, const float* x_obs, int64_t n_x,
                      const float* gout, float* out, float* part, int64_t R, int J, int K,
                      int relu, void* stream);
/* As zsb_linear_tc_f32, additionally folding max |out| (epi 0 / 2 / 16) into amax_scale[2] so that
 * the consumer's operand split (zsb_split16_dual_f32, have_amax = 1) needs no pass over `out`.
 *   epi 16: out [R, J] = act(h W^T + bias + x) with the residual x [R, J] (n_x = R) added before
 *           the ReLU: tf.layers.conv2d(..., activation=relu) of a resnet block whose shortcut is
 *           added first (vae_conv.py:39-53), on the im2col planes of zsb_conv_gather_split_f32 */
int zsb_linear_tc_amax_f32(int epi, const void* w_planes, const float* scale_w,
                           const void* h_planes, const float* scale_h, const float* bias,
                           const float* x_obs, int64_t n_x, const float* gout, float* out,
                           float* part, int64_t R, int J, int K, int relu, float* amax_scale,
                           void* stream);
/* The operand planes of an activation / gradient matrix in one pass: planes [2][R][Kp] of
 * src * scale, optionally times the ReLU mask (mask_src > 0) -- the `g * (y > 0)` of the dense
 * layer's backward (tf.layers.dense + relu, iwae.py:23-44) -- and the column sums of the masked
 * matrix (bias gradient) into col_sum (may be NULL).  K must be even. */
int zsb_split16_dual_f32(const float* src, const float* mask_src, int64_t R, int K, void* planes,
                         float* col_sum, float* scale, int have_amax, void* stream);

/* Input gradient of the dense layer, dh [R, K] = g W = sum_j g[r, j] * W[j, k] (tf.gradients of
 * tf.layers.dense w.r.t. its input), with operand A = the FORWARD planes of W [J, K]
 * (w_planes [2][J][kpad(K)], read MN-major) and B = g_planes [2][R][kpad(J)]: no W^T copy.
 * max |dh| is folded into amax_scale[2] when amax_scale != NULL. */
int zsb_linear_tc_dgrad_f32(const void* w_planes, const float* scale_w, const void* g_planes,
                            const float* scale_g, int64_t R, int J, int K, float* out,
                            float* amax_scale, void* stream);
/* Weight gradient of the dense layer, dW [J, K] = g^T h = sum_r g[r, j] * h[r, k] (the
 * tf.gradients of tf.layers.dense w.r.t. its kernel, iwae.py:23-44), read straight from the
 * ROW-MAJOR planes h_planes [2][R][kpad(K)] and g_planes [2][R][kpad(J)]: the contraction runs
 * over the rows, so both operands are MN-major wgmma operands and no transposed copy of an
 * activation is ever written.  part = zsb_linear_tc_slices(J, K, R) * J * K floats of split-K
 * scratch (NULL: one slice). */
int zsb_linear_tc_wgrad_f32(const void* h_planes, const float* scale_h, int K,
                            const void* g_planes, const float* scale_g, int J, int64_t R,
                            float* out, float* part, void* stream);

/* ---- Sigmoid belief net layers: tf.layers.dense + bn.bernoulli(..., n_samples, dtype=tf.float32)
 * of examples/sigmoid_belief_nets/sbn_vimco.py:19-44 (and sbn_adaptive_is.py), with
 * Bernoulli._sample / _log_prob (univariate.py:386-403) in the GEMM epilogue.
 * A "binary" activation is a 0/1 sample whose operand is ONE fp16 plane h * 2048 (its lo plane is
 * identically zero and is neither stored nor loaded): its products issue two fp16 wgmma per k-step
 * instead of three and give the same result bit for bit as the split planes of the same matrix.
 *
 * One launch per sampled layer, l = h W^T + bias never written: h_out [S R, J] = (u < sigmoid(l))
 * (float, or int32 when h_int) with u = u_in [S R J] or the Philox draw of zsb_sample_bernoulli_i32
 * for (seed, iter) at element (s R + r) J + j (so the result equals sampling the fp32 logits of
 * zsb_linear_tc_f32); h_planes_out [S R][kpad(J)] = its binary operand plane; logq [S R] = the
 * grouped log-probability of each draw; part = zsb_linear_tc_nparts(J) * S R floats of scratch.
 * h_binary: h_planes is itself a binary plane. */
int zsb_linear_tc_bern_sample_f32(const void* w_planes, const float* scale_w, const void* h_planes,
                                  const float* scale_h, int h_binary, const float* bias,
                                  const float* u_in, uint64_t seed, uint32_t iter, int S,
                                  void* h_out, int h_int, void* h_planes_out, float* logq,
                                  float* part, int64_t R, int J, int K, void* stream);
/* S given rows per logit row (a [S, R, J] sample against [R, J] logits, univariate.py:398-403):
 *   epi 1: out [S R] = sum_j Bernoulli(l[r]).log_prob(given[s R + r, j]);  part as above
 *   epi 2: out [R, J] = sum_s gout[s R + r] * (given[s R + r, j] - sigmoid(l[r, j]))  (d/dl of the
 *          broadcast), max |out| folded into amax_scale[2] (may be NULL) */
int zsb_linear_tc_bern_given_f32(int epi, const void* w_planes, const float* scale_w,
                                 const void* h_planes, const float* scale_h, int h_binary,
                                 const float* bias, const float* given, int S, const float* gout,
                                 float* out, float* part, int64_t R, int J, int K,
                                 float* amax_scale, void* stream);
/* One-hot categorical layer over C classes (1 <= C <= 128), logits l = h W^T + bias never written
 * (replaces tf.layers.dense + bn.onehot_categorical, vae_ssl_adaptive_is.py:61-68, with
 * OnehotCategorical._sample / _log_prob, multivariate.py:522-562).  Draw d = s R + r of S per
 * logit row; S R < 2^31.
 *   cls [S R] int32: the class drawn from softmax(l[r]) exactly as zsb_sample_categorical_i32 draws
 *   it (u_in [S R], or word 0 of Philox block (0, d, iter, stream 6)); onehot [S R, C] its one-hot
 *   row, float (h_int = 0) or int32; logq [S R] = l[r, cls] - logsumexp(l[r]).
 * h_binary: h_planes is itself a binary plane. */
int zsb_linear_tc_cat_sample_f32(const void* w_planes, const float* scale_w, const void* h_planes,
                                 const float* scale_h, int h_binary, const float* bias,
                                 const float* u_in, uint64_t seed, uint32_t iter, int S,
                                 int32_t* cls, void* onehot, int h_int, float* logq, int64_t R,
                                 int C, int K, void* stream);
/* The same layer against given [n_g, C] float rows, draw d scored against row d % n_g (n_g divides
 * S R; OnehotCategorical._log_prob = unnormalized_multinomial_log_prob with normalized logits,
 * multivariate.py:435-443, 547-556):
 *   epi 1: out [S R] = sum_j given_j (l[r, j] - logsumexp(l[r]))
 *   epi 2: out [R, C] = sum_s gout[d] (given_j - (sum_i given_i) softmax(l[r])_j)  (d/dl of the
 *          sum), max |out| folded into amax_scale[2] (may be NULL) */
int zsb_linear_tc_cat_given_f32(int epi, const void* w_planes, const float* scale_w,
                                const void* h_planes, const float* scale_h, int h_binary,
                                const float* bias, const float* given, int64_t n_g, int S,
                                const float* gout, float* out, int64_t R, int C, int K,
                                float* amax_scale, void* stream);
/* Gaussian dense layer over D features (1 <= D <= 256), the heads mu = h W_mean^T + b_mean and
 * ls = h W_logstd^T + b_logstd never written unless asked for (replaces two tf.layers.dense +
 * bn.normal(..., logstd=..., n_samples=K), vae_ssl_adaptive_is.py:53-68, with Normal._sample /
 * _log_prob, univariate.py:161-181).  w_planes: the planes of the packed heads [2 Dp, K], Dp =
 * zsb_linear_tc_kpad(D), in blocks of 64 rows [mean 0..63 | logstd 0..63 | mean 64..127 | ...],
 * zero padded; bias: the packed biases [2 Dp] or NULL.  Draw s R + r of S per row; S R < 2^31.
 *   z [S R, D] = eps * exp(ls) + mu, eps = eps_in [S R D] or element (s R + r) D + j of the normals
 *   zsb_reparam_normal_f32 draws for (seed, iter): z is that sampler's draw bit for bit;
 *   logq [S R] = sum_j log N(z; mu, exp(ls)), summed in a fixed order from part (Dp / 32 * S R
 *   floats of scratch: two partial rows per 64 features);
 *   mean_out / logstd_out [R, D] (either may be NULL); max |z| folded into amax_scale[2] (may be
 *   NULL).  h_binary: h_planes is itself a binary plane. */
int zsb_linear_tc_normal_sample_f32(const void* w_planes, const float* scale_w,
                                    const void* h_planes, const float* scale_h, int h_binary,
                                    const float* bias, const float* eps_in, uint64_t seed,
                                    uint32_t iter, int S, float* z, float* logq, float* part,
                                    float* mean_out, float* logstd_out, int64_t R, int D, int K,
                                    float* amax_scale, void* stream);
/* Its backward pass in one launch, summed over the S draws in order (no float atomics), with eps
 * recomputed from (seed, iter + *epoch) or read from eps_in.  epoch (may be NULL): a copy of the
 * device epoch taken when the forward launch ran, so the draws are recomputed as they were drawn
 * even if the epoch has moved since:
 *   reparam:   d mu = sum_s gz_s,                d ls = sum_s (gz_s std eps_s - glq_s)
 *   otherwise: d mu = sum_s glq_s eps_s / std,   d ls = sum_s glq_s (eps_s^2 - 1)
 * (Normal._sample stop-gradients mean and std when not reparameterised, univariate.py:161-172;
 * log q keeps its partials).  gz [S R, D] and glq [S R] may each be NULL (zero); logstd [R, D].
 * dpre [R, 2 Dp]: the gradient of the packed pre-activation, padding columns zero, max |dpre|
 * folded into amax_scale[2] (must start at zero): the operand of zsb_split16_dual_f32 with
 * have_amax = 1. */
int zsb_linear_normal_grad_f32(const float* logstd, const float* gz, const float* glq,
                               const float* eps_in, uint64_t seed, uint32_t iter,
                               const uint32_t* epoch, int reparam, int S, int64_t R, int D,
                               float* dpre, float* amax_scale, void* stream);
/* zsb_linear_tc_amax_f32 / zsb_linear_tc_wgrad_f32 with a binary activation h (h_planes = its one
 * plane, scale_h[0] = 2048): the forward, epi 1 / 2 and weight-gradient products of a layer fed a
 * sample (sbn_vimco.py:25-30, 40-43). */
int zsb_linear_tc_bin_f32(int epi, const void* w_planes, const float* scale_w,
                          const void* h_planes, const float* scale_h, const float* bias,
                          const float* x_obs, int64_t n_x, const float* gout, float* out,
                          float* part, int64_t R, int J, int K, int relu, float* amax_scale,
                          void* stream);
int zsb_linear_tc_wgrad_bin_f32(const void* h_planes, const float* scale_h, int K,
                                const void* g_planes, const float* scale_g, int J, int64_t R,
                                float* out, float* part, void* stream);

/* ---- Class-conditioned dense layer: tf.layers.dense of a one-hot class y beside an activation h,
 * examples/semi_supervised_vae/vae_ssl.py:24-28 (relu(dense(z) + dense(onehot(y)))) and :38
 * (dense(concat([x, y]))).  onehot(y) W_y^T is row y of the class table ctab [C, J] = W_y^T, added
 * in the epilogue of the product h W^T instead of multiplied:
 *   cls != NULL: out [R, J] = act(h W^T + bias + ctab[cls[r % n_cls]]); a row whose class is
 *                outside [0, C) is written as NaN (ctab is not read for it)
 *   cls == NULL: out [C R, J], row c R + r = act(h W^T + bias + ctab[c])[r] for every class c
 *                (class-major), from ONE product over the R rows -- the unlabeled bound's class
 *                enumeration, vae_ssl.py:108-124, without tiling h C times.  Bit-identical to the
 *                cls form on h tiled C times with cls = c for the rows of block c.
 * act = ReLU if relu.  max |out| is folded into amax_scale[2] (may be NULL) as in
 * zsb_linear_tc_amax_f32; h_binary: h_planes is a binary plane (zsb_linear_tc_bern_sample_f32). */
int zsb_linear_tc_class_f32(const void* w_planes, const float* scale_w, const void* h_planes,
                            const float* scale_h, int h_binary, const float* bias,
                            const float* ctab, int C, const int32_t* cls, int64_t n_cls,
                            float* out, int64_t R, int J, int K, int relu, float* amax_scale,
                            void* stream);
/* Its backward pass over the upstream gradient src (times the ReLU mask mask_src > 0 when not
 * NULL) in one pass: planes [2][R][kpad(K)] of G for zsb_linear_tc_dgrad_f32 /
 * zsb_linear_tc_wgrad_f32, with G = src [R, K] (cls != NULL) or G[r] = sum_c src[c R + r]
 * (cls == NULL, src [C R, K] class-major: the products then run over R rows, not C R);
 * col_sum [K] += column sums of G (bias gradient) and dtab [C, K] += the column sums of src over
 * the rows of each class (class-table gradient); both may be NULL and are zeroed by the caller.
 * have_amax: scale[2] holds max |src| from the producing GEMM.  The planes' scale bounds
 * C max|src| in the cls == NULL form. */
int zsb_split16_class_f32(const float* src, const float* mask_src, int64_t R, int K,
                          const int32_t* cls, int64_t n_cls, int C, void* planes, float* col_sum,
                          float* dtab, float* scale, int have_amax, void* stream);

/* ---- Noisy, batch-normalised dense layer of examples/bayesian_neural_nets/variational_dropout.py:26-37:
 * relu(batch_norm(fully_connected(h * eps))), with tf.contrib.layers defaults (no bias, beta but no
 * gamma, population variance over all rows in training, moving averages updated in place with
 * m -= (m - batch) * (1 - decay), the moving statistics in evaluation).
 * Operand planes [2][R][kpad(K)] of x = h[r % n_h] * noise[r] (h [n_h, K] broadcast over the
 * particle rows of noise [R, K]; n_h divides R), scale[0] from a max pass over x; x is never
 * written in fp32.  scale = device float[4], zero-initialised. */
int zsb_split16_noisy_f32(const float* h, int64_t n_h, const float* noise, int64_t R, int K,
                          void* planes, float* scale, void* stream);
/* Dense layer without bias + batch norm (tf.layers.dense(use_bias=False) +
 * tf.layers.batch_normalization, bernoulli_latent_vae.py:25-30 and 39-44; the convolutions of the
 * GAN examples; with gamma = NULL, the layers of variational_dropout.py): a = h W^T from the planes
 * of h (those of zsb_split16_noisy_f32, or with h_binary the one plane of a 0/1 sample,
 * zsb_linear_tc_bern_sample_f32, which needs gamma), out [R, J] = act(xhat * gamma + beta), xhat =
 * (a - mean) rstd (act = ReLU if relu), stats [2][J] = (mean, rstd).  gamma = NULL: out = act((a -
 * mean) rstd + beta), rounded as such rather than as gamma = 1.
 *   training: mean and population variance of a over its R rows, rstd = rsqrt(var + eps); a [R, J]
 *     is written, part = ceil(R / 128) * 2 J floats of moment partials (per 128-row tile: mean and
 *     sum of squared deviations), merged in a fixed order (Chan); moving_mean / moving_var -=
 *     (moving - batch) * rate, rate = 1 - decay.  bessel (TF 1.x's fused_batch_norm, the path of
 *     4-D inputs): the moving variance moves towards the Bessel-corrected R / (R - 1) var (towards
 *     0 when R = 1); the output still normalises with var.
 *   else: mean / rstd of the moving statistics (unchanged), applied in the product's epilogue;
 *     part is not used, and with gamma a (may be NULL) receives the pre-activation, which the
 *     gradient of gamma reads.
 * max |out| is folded into amax_scale[2] (may be NULL) as in zsb_linear_tc_amax_f32. */
int zsb_linear_tc_bn_f32(int training, int bessel, const void* w_planes, const float* scale_w,
                         const void* h_planes, const float* scale_h, int h_binary,
                         const float* gamma, const float* beta, float* moving_mean,
                         float* moving_var, float rate, float eps, float* stats, float* a,
                         float* part, float* out, int64_t R, int J, int K, int relu,
                         float* amax_scale, void* stream);
/* The training step of zsb_linear_tc_bn_f32 with bessel after a pass that left the pre-activation
 * a [R, J] and its per-128-row-tile moment partials part [ceil(R / 128)][2][J] (mean, M2): the
 * deterministic merge, stats = (mean, rstd), the moving statistics updated, and out = act(xhat *
 * gamma + beta); max |out| into amax_scale[2] (may be NULL). */
int zsb_bn_finish_fused_f32(const float* a, const float* part, int64_t R, int J,
                            const float* gamma, const float* beta, float* moving_mean,
                            float* moving_var, float rate, float eps, float* stats, float* out,
                            int relu, float* amax_scale, void* stream);
/* The backward pass of zsb_linear_tc_bn_f32 from the upstream gradient g [R, J], the output y
 * (read when relu), a and stats: g' = g [y > 0] (relu) or g, dbeta [J] = sum_r g', dgamma [J] = sum_r g' xhat (either may
 * be NULL; a is needed in training and for dgamma), and the planes [2][R][kpad(J)] of da = gamma
 * rstd (g' - mean_r g' - xhat mean_r(g' xhat)) in training, of da = gamma rstd g' otherwise (rstd
 * alone when gamma is NULL) -- the operand of zsb_linear_tc_dgrad_f32 / zsb_linear_tc_wgrad_f32.
 * Column sums are deterministic.  part = (ceil(R / 128) + 1) * 2 J floats; scale = device float[4]
 * with scale[2] zero. */
int zsb_bn_grad_f32(int training, const float* g, const float* y, const float* a,
                    const float* stats, const float* gamma, int relu, int64_t R, int J,
                    float* part, float* dbeta, float* dgamma, void* planes, float* scale,
                    void* stream);
/* As zsb_bn_grad_f32, but da [R, J] is written in fp32 and max |da| is folded into scale[2]
 * (scale = device float[4] with scale[2] zero): for a consumer that gathers da (the transposed
 * convolution) before splitting it into planes. */
int zsb_bn_grad_f32out(int training, const float* g, const float* y, const float* a,
                       const float* stats, const float* gamma, int relu, int64_t R, int J,
                       float* part, float* dbeta, float* dgamma, float* da, float* scale,
                       void* stream);
/* From d = d(h * noise) [R, K]: dnoise [R, K] = d * h[r % n_h], dh [n_h, K] = sum over the R / n_h
 * particle rows of d * noise (either may be NULL). */
int zsb_noisy_grad_f32(const float* d, const float* h, int64_t n_h, const float* noise, int64_t R,
                       int K, float* dnoise, float* dh, void* stream);

/* ---- diagnostics: effective sample size (zhusuan/diagnostics.py:17-64, the Stan estimator) on the
 * device; samples [M, D] row-major with burn-in already dropped -> ess [D].  M >= 2. */
int zsb_effective_sample_size_f32(const float* samples, int64_t M, int64_t D, float* ess,
                                  void* stream);

/* ---- K2/K3/K4: HMC building blocks (zhusuan/hmc.py) ----------------------------------------- */
int zsb_hmc_acc_parts(void);   /* capacity (floats) callers must give every acc_part scratch */
int zsb_hmc_mass_parts(void);  /* mass_stats scratch = zsb_hmc_mass_parts()*2*D floats */
/* random_momentum hmc.py:21-23 (+ kinetic hmc.py:32-34 into k_out, optional) */
int zsb_hmc_momentum_f32(float* p, const float* noise, const float* mass, int64_t mass_n,
                         int64_t chains, int64_t row_len, uint64_t seed, uint32_t iter,
                         uint32_t stream_id, int64_t row0, float* k_out, int accumulate,
                         const float* iter_state, void* stream);
int zsb_hmc_kinetic_f32(const float* p, const float* mass, int64_t mass_n, int64_t chains,
                        int64_t row_len, float* k_out, int accumulate, void* stream);
/* leapfrog_integrator hmc.py:38-43: q += (eps*scale) * (p/mass);  p += (eps*scale) * grad.
 * eps_dev points at state[ZSB_HMC_STATE_EPS_USED]. */
int zsb_hmc_leapfrog_q_f32(float* q, const float* p, const float* mass, int64_t mass_n,
                           int64_t row_len, const float* eps_dev, float scale, int64_t n,
                           void* stream);
int zsb_hmc_leapfrog_p_f32(float* p, const float* g, const float* eps_dev, float scale, int64_t n,
                           void* stream);
/* get_acceptance_rate + MH decision hmc.py:46-61, 485-486, 498 */
int zsb_hmc_mh_f32(const float* lp0, const float* lp1, const float* k0, const float* k1,
                   const float* u, uint64_t seed, uint32_t iter, int64_t row0, int64_t chains,
                   float* h0, float* h1, float* acc, int32_t* accept, float* lp_sel,
                   float* acc_part, int* n_part_out /* host */, float* state, void* stream);
/* where(accept, q_new, q) hmc.py:488-497 */
int zsb_hmc_select_f32(float* q, const float* q_new, const int32_t* accept, int64_t chains,
                       int64_t row_len, void* stream);
/* stats[0] = sum(acc), stats[1] = local chain count; all-reduce(sum) stats across ranks, then tune */
int zsb_hmc_acc_sum_f32(const float* acc_part, int n_part, int64_t chains, float* stats,
                        void* stream);
/* Device-driven iterations (CUDA-graph replay): pass start_search = -1 to zsb_hmc_begin_f32 (the
 * kernel then advances state[T] itself), iter = 0xFFFFFFFF to the kernels that draw Philox numbers
 * (they read the iteration from the state block; zsb_hmc_momentum_f32 takes it via iter_state),
 * t_now = -1 to zsb_hmc_tune_f32, use_ones = -(mass_collect_iters + 1) to
 * zsb_hmc_mass_update_f32, and zsb_hmc_ewmv_bump_f32 after an adaptive mass update. */
int zsb_hmc_begin_f32(float* state, int start_search, void* stream);
int zsb_hmc_ewmv_bump_f32(float* state, void* stream);
/* one pass of _init_step_size's loop bookkeeping hmc.py:326-338 */
int zsb_hmc_search_update_f32(float* state, const float* stats, float target, void* stream);
/* StepsizeTuner.tune hmc.py:89-112 + step_size assign hmc.py:379 */
int zsb_hmc_tune_f32(float* state, const float* stats, int has_tuner, int adapt, float fresh_start,
                     float gamma, float t0, float kappa, float delta, float t_now, void* stream);
/* ExponentialWeightedMovingVariance hmc.py:115-159 + _adapt_mass hmc.py:283-305.
 * stats = [sum_c (q-mean) (D), sum_c (q-mean)^2 (D)]; all-reduce(sum) across ranks between calls */
int zsb_hmc_mass_stats_f32(const float* q, const float* ewmv_mean, int64_t chains, int64_t D,
                           float* part, float* stats, void* stream);
int zsb_hmc_mass_update_f32(float* ewmv_mean, float* ewmv_var, float* mass, const float* stats,
                            float n_chains_global, int64_t D, float decay, float ewmv_t_new,
                            int adapt, int use_ones, float* state, void* stream);

/* Fused whole iteration for a diagonal-Gaussian target (Normal node, group_ndims=1;
 * examples/toy_examples/gaussian.py:15-20): momentum, L+1 gradient passes, Hamiltonians, MH,
 * in-place select in ONE launch.  search_mode=1: the acceptance probe of hmc.py:314-326. */
int zsb_hmc_diag_normal_step_f32(float* q, const float* noise, const float* u, const float* mean,
                                 int64_t mean_n, const float* logstd, int64_t logstd_n,
                                 const float* mass, int64_t mass_n, float* state, int n_leapfrogs,
                                 int64_t chains, int64_t D, uint64_t seed, uint32_t iter,
                                 int64_t row0, int search_mode, float* p0_out, float* h0, float* h1,
                                 float* lp0, float* lp_sel, float* acc, int32_t* accept,
                                 float* acc_part, int* n_part_out /* host */, void* stream);

/* Dense-Gaussian target log p = -1/2 (x-mu)^T P (x-mu) + c: one launch per pass of the leapfrog
 * while-loop body (hmc.py:352-364): g = b - q_cur P; p_out = p_in + p_scale*eps*g;
 * q_next = q_cur + eps*p_out/mass (skipped if NULL); lp_part/k_part [ntiles, chains] partials.
 * impl 0 = SIMT fp32 (P full fp32; *_lo ignored).
 * impl 1 = wgmma TF32, 3xTF32 split: P = hi part (low 13 mantissa bits cleared),
 *          P_lo = P - hi; q_cur_lo = residual of q_cur (zsb_hmc_dense_split_lo_f32 for the first
 *          pass), q_next_lo receives the residual of q_next. */
int zsb_hmc_dense_ntiles(int64_t D, int impl);
int zsb_hmc_dense_leapfrog_f32(const float* q_cur, const float* q_cur_lo, float* q_next,
                               float* q_next_lo, const float* p_in, float* p_out,
                               const float* P, const float* P_lo, const float* bvec,
                               const float* mu, const float* mass, const float* state,
                               float p_scale, float* lp_part, float* k_part, int64_t chains,
                               int64_t D, int impl, void* stream);
int zsb_hmc_dense_split_lo_f32(const float* q, float* lo, int64_t n, void* stream);
/* impl 2: fp16-split tensor-core path (3 fp16 wgmma products per k-step at twice the TF32 rate).
 * P_h16/P_l16: [D,D] __half hi/lo of P*sP; q_*_planes: [2][chains][D] __half hi/lo of q*sq_i,
 * where the plane scale sq_i follows the chains through the trajectory.  scales: device
 * float[8 + 4*(L+2)] for trajectories of up to L+1 passes; the caller sets [3] = sP,
 * [4] = ||P||_inf (max row sum of |P|), [5] = max|b| once.  Record i at [8 + 4*i] =
 * {sq_i, sq_alt_i, max|q_i| bound, flag} describes the planes pass i reads.  traj_prepare (after
 * the momentum is drawn, p = p0; before every trajectory) writes record 0 and q's planes at sq_0
 * (max|q| * sq_0 in [2^11, 2^12)); pass `pass_index` (from 0) writes q_next's planes at sq_i, or
 * at a smaller power of two when an a-priori bound on |q_next| could overflow fp16 at sq_i.  A
 * chain may therefore move any distance from where the trajectory started.  D % 64 == 0. */
int zsb_hmc_dense_traj_prepare_f32(const float* q, const float* p, const float* mass, void* planes,
                                   float* scales, int64_t chains, int64_t D, void* stream);
int zsb_hmc_dense_leapfrog_h16_pass_f32(const float* q_cur, const void* q_cur_planes,
                                        float* q_next, void* q_next_planes, const float* p_in,
                                        float* p_out, const void* P_h16, const void* P_l16,
                                        float* scales, int pass_index, const float* bvec,
                                        const float* mu, const float* mass, const float* state,
                                        float p_scale, float* lp_part, float* k_part,
                                        int64_t chains, int64_t D, void* stream);
/* impl 5: the whole leapfrog `while_loop` of hmc.py:347-372 (L+1 passes, body = leapfrog_integrator
 * hmc.py:38-43, plus the log p / kinetic terms of hamiltonian() hmc.py:30-35) with the fp16 hi/lo
 * plane pair of q*sq_i as the state of q inside the trajectory (planes0 from
 * zsb_hmc_dense_traj_prepare_f32, scales as there; planes1, spare0, spare1 = work buffers of the
 * same size, all distinct).  A pass whose bound says its planes might overflow fp16 writes them at
 * sq_i, as any other pass, plus a spare copy at a smaller scale, which the next pass reads if they
 * did overflow; trajectories whose planes fit are unchanged by the bound.  The proposal's planes
 * end in buffer (n_leapfrogs & 1) or its spare, and zsb_hmc_dense_select_traj_planes_f32, given
 * both and &scales[8 + 4*n_leapfrogs], assigns them to the accepted chains (the `tf.where` +
 * assign of hmc.py:488-497).  D % 64 == 0, n_leapfrogs >= 1. */
int zsb_hmc_dense_resident_h16_f32(void* planes0, void* planes1, void* spare0, void* spare1,
                                   const float* p0, float* pw, const void* P_h16,
                                   const void* P_l16, float* scales, const float* bvec,
                                   const float* mu, const float* mass, const float* state,
                                   float* lp0_part, float* lp1_part, float* k_part,
                                   int64_t chains, int64_t D, int n_leapfrogs, void* stream);
int zsb_hmc_dense_select_traj_planes_f32(float* q, const void* planes, const void* spare,
                                         const float* record, const int32_t* accept,
                                         int64_t chains, int64_t D, void* stream);
int zsb_hmc_dense_finish_f32(const float* lp_part, const float* k_part, int ntiles, int64_t chains,
                             float const_term, float* lp_out, float* k_out, void* stream);

/* ---- device samplers of the discrete / gamma-family distributions (csrc/samplers.cu) ----------
 * Categorical._sample (univariate.py:478-494, tf.random.categorical): inverse CDF of
 * softmax(logits) with one uniform per draw (u injected [n_samples*rows] or Philox); out[s, r].
 * Dirichlet._sample (multivariate.py:660-663): Gamma(alpha, 1) by Marsaglia-Tsang on Philox
 * (or injected gamma variates) normalised by the row sum.  Gamma._sample: Gamma(alpha, 1) / beta. */
int zsb_sample_categorical_i32(const float* logits, int64_t logit_rows, int64_t rows,
                               int64_t n_categories, int64_t n_samples, const float* u,
                               uint64_t seed, uint32_t iter, int32_t* out, void* stream);
int zsb_sample_dirichlet_f32(const float* alpha, int64_t alpha_rows, int64_t n_rows,
                             int64_t n_categories, const float* gammas, uint64_t seed,
                             uint32_t iter, float* out, void* stream);
int zsb_sample_gamma_f32(const float* alpha, int64_t alpha_rows, const float* beta,
                         int64_t beta_rows, int64_t n_rows, int64_t row_len, uint64_t seed,
                         uint32_t iter, float* out, void* stream);
/* Base noise (kind 0: U[0,1), kind 1: N(0,1)) for the samplers whose transform is composed on the
 * host side (tf.random_uniform / tf.random_normal of univariate.py:306-317, 622-640, 1246-1265,
 * 1363-1379): Philox block (i / 4, 0, iter, 9), word i % 4. */
int zsb_sample_base_noise_f32(int kind, float* out, int64_t n, uint64_t seed, uint32_t iter,
                              void* stream);
/* ---- ExpConcrete / Concrete (multivariate.py:683-958; csrc/concrete.cu) -----------------------
 * Rows of C categories, 1 <= C <= 1024; value row r reads parameter row r % logits_rows (the
 * parameters broadcast as a suffix) and given row r % given_rows.  `temperature` is a device
 * pointer to one float, so no call synchronises with the host.  log_space = 1: ExpConcrete (values
 * are log-probabilities), 0: Concrete (values on the simplex).
 *
 * zsb_sample_concrete_f32 (ExpConcrete._sample multivariate.py:768-782, Concrete._sample
 * :905-919): out [rows, C] = log_softmax((l + g) / t) or softmax(...), g = -log(-log(u)), u
 * clamped to [1e-7, 1 - 1e-7].  u = injected uniforms [rows, C], or NULL: element e of the flat
 * output is word e % 4 of Philox block (e / 4, 0, iter, 9), the draw of zsb_sample_base_noise_f32
 * kind 0 for the same (seed, iter).
 * zsb_sample_concrete_bwd_f32: the reparameterisation gradient from the saved sample y [rows, C]
 * and its cotangent gy alone: dA = gy - exp(y) sum(gy) (log space) or y (gy - sum(y gy));
 * dlogits [logits_rows, C] = sum over the rows s * logits_rows + lr of dA / t, in a fixed order;
 * d t = -sum(dA y) / t (log space) or -sum(dA log y) / t, into dtemp [1].  rows must be a
 * multiple of logits_rows.  Either output may be NULL.
 * zsb_logprob_concrete_f32 (ExpConcrete._log_prob :800-812, Concrete._log_prob :938-955):
 * out [rows] = lgamma(C) + (C-1) log t + sum(temp) [- sum(log given)] - C LSE(temp), temp = l - t x,
 * x = given (log space) or log(given).
 * zsb_logprob_concrete_bwd_f32: with w = 1 - C softmax(temp) and gout [rows]: dgiven [rows, C] =
 * gout (-t w) or gout (-t w - 1) / given; dlogits [logits_rows, C] = sum of gout w over the rows
 * of each parameter row, in a fixed order; d t = sum gout ((C-1)/t - sum(w x)), into dtemp [1].
 * rows must be a multiple of logits_rows; every output may be NULL.
 * Both backward entries take `work`, zsb_concrete_bwd_work(logits_rows, C, rows) floats of
 * scratch: ZSB_CONCRETE_PARTS temperature partials, one per CTA, and, when the sample axis is split
 * across CTAs (few parameter rows, many samples), each chunk's logits-gradient partial.  A second
 * launch merges both in a fixed order.  No float atomics: identical calls give identical bits. */
#define ZSB_CONCRETE_PARTS 1024
int zsb_sample_concrete_f32(const float* logits, int64_t logits_rows, const float* temperature,
                            int64_t n_categories, int log_space, const float* u, uint64_t seed,
                            uint32_t iter, float* out, int64_t rows, void* stream);
int zsb_sample_concrete_bwd_f32(const float* y, const float* gy, int64_t logits_rows,
                                const float* temperature, int64_t n_categories, int log_space,
                                float* dlogits, float* dtemp, float* work, int64_t rows,
                                void* stream);
int zsb_logprob_concrete_f32(const float* given, int64_t given_rows, const float* logits,
                             int64_t logits_rows, const float* temperature, int64_t n_categories,
                             int log_space, float* out, int64_t rows, void* stream);
int zsb_logprob_concrete_bwd_f32(const float* given, int64_t given_rows, const float* logits,
                                 int64_t logits_rows, const float* temperature,
                                 int64_t n_categories, int log_space, const float* gout,
                                 float* dgiven, float* dlogits, float* dtemp, float* work,
                                 int64_t rows, void* stream);
int zsb_concrete_bwd_work(int64_t logits_rows, int64_t n_categories, int64_t rows);
/* Poisson._sample (univariate.py:915-920) / Binomial._sample (univariate.py:1025-1045): kind 0 =
 * Poisson(rate = param), 1 = Binomial(n_experiments, sigmoid(param)); one uniform per draw
 * (injected u [n] or Philox), inverse transform enumerating the support outwards from the mode. */
int zsb_sample_count_i32(int kind, const float* param, int64_t param_n, int64_t n_experiments,
                         const float* u, uint64_t seed, uint32_t iter, int32_t* out, int64_t n,
                         void* stream);

/* ---- K8, config 5: Logistic-Normal Topic Model E-step log-joint and M-step (csrc/lntm.cu) -------
 * log p = sum_k Normal(eta_k; mean_k, exp(logstd_k)).log_prob + sum_v x[d,v] log(softmax(eta) @ phi)[v]
 * (examples/topic_models/lntm_mcem.py:33-48, e_obj :97-99; UnnormalizedMultinomial._log_prob,
 * multivariate.py:435-443 with normalize_logits=False) and its gradient w.r.t. eta, fused and
 * sparsity-aware: the corpus is CSR, only the words a document contains are formed, the
 * [chains*docs, V] matrix of the reference never exists.  1 <= n_topics <= 128; the topic axis of
 * phi_t = softmax(beta)^T is padded to Kp = 16 ceil(n_topics / 16): phi_t [V, Kp], zero pad columns.
 *
 * zsb_lntm_logjoint_f32 (lntm_mcem.py:33-48, 97-99; tempered as evaluation.py:91-94):
 *   doc_ids [docs] (int64, nullable): row d of eta is corpus document doc_ids[d]; NULL = 0..docs-1.
 *   temperature (device scalar, nullable): returns prior + t * likelihood and its gradient, which is
 *   log_prior * (1 - t) + log_joint * t when the proposal is the eta prior; NULL = today's result.
 * zsb_lntm_mstep_f32 / zsb_lntm_mstep_grad_f32 (lntm_mcem.py:106-114, cond_log_prob('x') and
 * tf.gradients of -log_joint_beta w.r.t. beta): lp [chains, docs] = log p(x_d | eta_c, beta), then
 * dbeta [K, V] = d/d beta sum_{c,d} g[c,d] lp[c,d].  The forward writes theta [chains, docs, Kp]
 * and ratio [chains, nnz] for the gradient; the gradient groups the corpus entries by word (CSC:
 * csc_ptr [V+1], csc_entry [nnz] ascending within a word, entry_doc [nnz]) and sums in a fixed
 * order, with no atomics.  doc_slot [n_corpus_docs]: batch row of each corpus document, -1 outside
 * the batch (NULL when doc_ids is NULL).  G [V, Kp] is scratch. */
int zsb_lntm_phi_t_f32(const float* beta, int64_t n_topics, int64_t n_vocab, float* phi_t,
                       void* stream);
int zsb_lntm_logjoint_f32(const float* eta, const float* eta_mean, const float* eta_logstd,
                          const float* phi_t, const int64_t* doc_ptr, const int32_t* word_idx,
                          const float* word_cnt, const int64_t* doc_ids, const float* temperature,
                          float* lp_out, float* grad_out, int64_t chains, int64_t docs,
                          int64_t n_topics, void* stream);
int zsb_lntm_mstep_f32(const float* eta, const float* phi_t, const int64_t* doc_ptr,
                       const int32_t* word_idx, const float* word_cnt, const int64_t* doc_ids,
                       float* lp_out, float* ratio, float* theta, int64_t chains, int64_t docs,
                       int64_t nnz, int64_t n_topics, void* stream);
int zsb_lntm_mstep_grad_f32(const float* g, const float* ratio, const float* theta,
                            const float* phi_t, const int64_t* csc_ptr, const int32_t* csc_entry,
                            const int32_t* entry_doc, const int32_t* doc_slot, float* G,
                            float* dbeta, int64_t chains, int64_t docs, int64_t nnz,
                            int64_t n_topics, int64_t n_vocab, void* stream);

/* ---- Bayesian PMF, one HMC sweep over every chunk of one factor (csrc/pmf.cu) ------------------
 * The model of examples/probabilistic_matrix_factorization/pmf_hmc.py:19-31 with its log_joint
 * override (136-144), Normal._log_prob of zhusuan/distributions/univariate.py:
 *   lat [K, n_rows, D] ~ N(0, exp(logstd_lat)), fixed [K, n_cols, D] ~ N(0, exp(logstd_fixed)),
 *   r_ij ~ N(sigmoid(lat_i . fixed_j), exp(logstd_rating)).
 * Ratings in CSR by latent row: row_ptr [n_rows + 1], col_idx / rating [nnz].  nbr_ptr
 * [n_chunks + 1] / nbr_idx: the distinct columns rated inside each chunk of chunk_size rows.
 * lp_out [K, n_chunks] = prior of the chunk's latent rows + prior of the fixed factor over the
 * chunk's neighbours + the chunk's rating terms; grad_out (like lat) = d lp / d lat.  Either may be
 * NULL; values need work [K, n_rows].  1 <= D <= 128.  No floating-point atomics: deterministic. */
int zsb_pmf_logjoint_f32(const float* lat, const float* fixed, const int64_t* row_ptr,
                         const int32_t* col_idx, const float* rating, const int64_t* nbr_ptr,
                         const int32_t* nbr_idx, float logstd_lat, float logstd_fixed,
                         float logstd_rating, float* lp_out, float* grad_out, float* work,
                         int64_t K, int64_t n_rows, int64_t n_cols, int64_t D, int64_t chunk_size,
                         void* stream);

/* ---- Planar normalizing flows (csrc/flows.cu; zhusuan/transform.py:70-198) --------------------
 * A stack of n_iters planar flows along the last axis of z [R, d], parameters b [n_iters],
 * aux_u [n_iters, d], w [n_iters, d] (the reference's param_b_i, aux_u_i, para_w_i stacked,
 * transform.py:148-168).  Per flow (transform.py:161-194):
 *   u = aux_u + w / (w.w) * (softplus(w.aux_u) - 1 - w.aux_u),  psi = u.w = softplus(w.aux_u) - 1
 *   a = tanh(z.w + b),  log_q -= log(1 + psi (1 - a^2)),  z += a u
 * with a stable softplus and no invertibility assert (psi > -1 by construction).  1 <= d <= 1024,
 * n_iters >= 1, R >= 0.  No floating-point atomics: deterministic. */
/* Forward, one launch (transform.py:148-194): z_out [R, d], lq_out [R] from z_in, lq_in.  ck: NULL,
 * or [n_iters, R, d] receiving every flow's input z_{k-1}, which zsb_planar_flow_bwd_f32 reads. */
int zsb_planar_flow_fwd_f32(const float* z_in, const float* lq_in, const float* b,
                            const float* aux_u, const float* w, float* z_out, float* lq_out,
                            float* ck, int64_t R, int64_t d, int64_t n_iters, void* stream);
/* Warps of the backward sweep for these sizes; its `part` scratch is
 * warps * n_iters * (2 d + 2) floats. */
int zsb_planar_flow_warps(int64_t R, int64_t d, int64_t n_iters);
/* Backward of transform.py:170-194, one sweep plus one merge launch.  gz_out [R, d] and glq [R]:
 * upstream gradients of z_out and lq_out; gz_in [R, d] = d / d z_in (d / d lq_in is glq itself);
 * db [n_iters], daux_u and dw [n_iters, d]: the parameter gradients through the reparameterisation
 * of u (transform.py:161-164).  ck as written by the forward pass. */
int zsb_planar_flow_bwd_f32(const float* ck, const float* gz_out, const float* glq,
                            const float* b, const float* aux_u, const float* w, float* gz_in,
                            float* part, float* db, float* daux_u, float* dw, int64_t R,
                            int64_t d, int64_t n_iters, void* stream);

/* ---- Inverse autoregressive flows (csrc/iaf.cu; zhusuan/transform.py:17-67, :200-282) ---------
 * A stack of n_iters IAF flows with linear_ar's network along the last axis of z [R, d], weights
 * m_w and s_w [n_iters, d, d] (linear_ar's m_w and s_w of every flow, stacked; only the entries
 * i < j are read, transform.py:38-43, :55-56).  Per flow (transform.py:58-61, :263-275):
 *   m = z (mask * m_w),  t = z (mask * s_w),  s = exp(t)
 *   update 0 ('normal'): z = s z + m,                  log_q -= sum_j t_j
 *   update 1 ('gru'):    g = sigmoid(s), z = g z + (1 - g) m,  log_q += sum_j log1p(exp(-s_j))
 *   z = reverse(z)
 * 1 <= d <= 256, n_iters >= 1, R >= 0.  No floating-point atomics: deterministic. */
/* Forward, one launch: z_out [R, d], lq_out [R] from z_in, lq_in.  ck: NULL, or [n_iters, R, d]
 * receiving every flow's input z, which zsb_iaf_bwd_f32 reads. */
int zsb_iaf_fwd_f32(const float* z_in, const float* lq_in, const float* m_w, const float* s_w,
                    float* z_out, float* lq_out, float* ck, int64_t R, int64_t d,
                    int64_t n_iters, int update, void* stream);
/* Slices of the backward sweep for these sizes; its `part` scratch is
 * slices * n_iters * 2 * d * d floats.  0 when R = 0. */
int zsb_iaf_slices(int64_t R, int64_t d, int64_t n_iters);
/* Backward of the stack, one sweep plus one merge launch.  gz_out [R, d] and glq [R]: upstream
 * gradients of z_out and lq_out; gz_in [R, d] = d / d z_in (d / d lq_in is glq itself); dm_w and
 * ds_w [n_iters, d, d], zero at i >= j.  ck as written by the forward pass. */
int zsb_iaf_bwd_f32(const float* ck, const float* gz_out, const float* glq, const float* m_w,
                    const float* s_w, float* gz_in, float* part, float* dm_w, float* ds_w,
                    int64_t R, int64_t d, int64_t n_iters, int update, void* stream);

/* ---- Sparse-GP conditional moments (csrc/gp.cu; examples/gaussian_process/utils.py:52-90) -----
 * gp_conditional(z, fz, x, full_cov=False, RBFKernel) for x [B, d], inducing points z [M, d],
 * kernel scales s [d] (softplus(k_raw_scale), utils.py:16), Li = chol(Kzz)^-1 [M, M] (only its lower
 * triangle is read) and V = fz Li^T [K, M].  With Kxz[b, m] = exp(-sum_j (x_bj - z_mj)^2 / s_j / 2)
 * (utils.py:35-39) and A = Kxz Li^T:
 *   mean = V A^T [K, B]  (utils.py:69-73, re-associated: the same product up to rounding)
 *   std  = sqrt(1 - rowsum(A^2)) [B]  (utils.py:84-87, Kdiag = 1; no clamp)
 * Replaces the [B, M, d] broadcast of utils.py:35-39 and the products of utils.py:70-86.
 * 1 <= M <= 256, 1 <= d <= 64, B >= 0, K >= 0; B = 0 returns without a launch.  No floating-point
 * atomics: deterministic. */
/* Forward, one launch: mean (may be NULL when K = 0) and std.  A_out: NULL, or [B, M] receiving A,
 * which zsb_gp_cond_bwd_f32 reads. */
int zsb_gp_cond_fwd_f32(const float* x, const float* z, const float* s, const float* Li,
                        const float* V, float* mean, float* stdv, float* A_out, int64_t B,
                        int64_t M, int64_t d, int64_t K, void* stream);
/* Slices of the backward sweep for these sizes; its `part` scratch is
 * slices * (K*M + M*M + M*d + d) floats.  0 when B = 0. */
int zsb_gp_cond_parts(int64_t B, int64_t M, int64_t d, int64_t K);
/* Backward of the moments, one sweep plus one merge launch.  g_mean [K, B] and g_std [B]: upstream
 * gradients, either may be NULL (zero).  Outputs dz [M, d], ds [d], dLi [M, M] (zero above the
 * diagonal) and dV [K, M].  A and stdv as written by the forward pass.  B = 0 returns without a
 * launch and leaves the outputs untouched. */
int zsb_gp_cond_bwd_f32(const float* x, const float* z, const float* s, const float* Li,
                        const float* V, const float* A, const float* stdv, const float* g_mean,
                        const float* g_std, float* part, float* dz, float* ds, float* dLi,
                        float* dV, int64_t B, int64_t M, int64_t d, int64_t K, void* stream);

/* ---- 3x3 SAME convolutions, NHWC (csrc/conv.cu; examples/variational_autoencoders/vae_conv.py) --
 * conv: tf.layers.conv2d(x, Cout, 3, strides=stride, padding="same") (vae_conv.py:39-53, 80) with
 * W [3, 3, Cin, Cout]; transpose: tf.nn.conv2d_transpose(..., padding="SAME") + bias_add of
 * examples/utils/utils.py:74-113 (vae_conv.py:20-36, 63-68) with W [3, 3, Cout, Cin].  Geometry is
 * given on the convolution's side: Hc x Wc is the conv input grid ("big"), Hs = ceil(Hc / stride)
 * x Ws its output grid ("small"); pads before are max((Hs - 1) stride + 3 - Hc, 0) / 2.  R images;
 * stride 1 or 2; 1 <= Cin, Cout <= 64; R*H*W*C < 2^31 on both grids.  No floating-point atomics:
 * deterministic. */
/* One layer, one launch: y = relu?(conv(x) + b + residual), replacing conv + bias_add + add + relu
 * (vae_conv.py:40-53, utils.py:101-111).  transpose = 0: x [R, Hc, Wc, Cin] -> y [R, Hs, Ws, Cout];
 * transpose = 1: x [R, Hs, Ws, Cin] -> y [R, Hc, Wc, Cout] (stride 2 by output parity: a
 * warp skips the taps none of its pixels needs).  b, residual (y's shape) may be NULL.  gate: NULL, or x's shape, and x
 * counts as 0 where gate <= 0 (the ReLU mask of a backward pass).  The input gradient of either
 * mode is the other mode on the output gradient with the same W.  R = 0 returns without a launch. */
int zsb_conv3x3_fwd_f32(const float* x, const float* gate, const float* W, const float* b,
                        const float* residual, float* y, int64_t R, int64_t Hc, int64_t Wc,
                        int64_t Cin, int64_t Cout, int stride, int transpose, int relu,
                        void* stream);
/* Slices of the weight-gradient sweep for these sizes; its `part` scratch is slices * Ca * Cb
 * floats.  0 when R = 0. */
int zsb_conv3x3_wgrad_parts(int64_t R, int64_t Hc, int64_t Wc, int stride);
/* Weight and bias gradient, one persistent sweep plus one merge launch (the tf.gradients of
 * vae_conv.py's convolutions): dW[kh, kw, a, b] = sum big[n, s i + kh - pt, s j + kw - pl, a]
 * small[n, i, j, b] over the small grid, big [R, Hc, Wc, Ca], small [R, Hs, Ws, Cb].  conv2d:
 * big = x, small = g, grad_big = 0, dW [3, 3, Cin, Cout]; conv2d_transpose: big = g, small = x,
 * grad_big = 1, dW [3, 3, Cout, Cin].  db (may be NULL): the output gradient summed over pixels.
 * dW may be NULL when only db is wanted: then only the bias sums run.  Not both NULL.
 * gate: NULL, or the gradient's shape, masking it where gate <= 0.  R >= 1. */
int zsb_conv3x3_wgrad_f32(const float* big, const float* small, const float* gate, int grad_big,
                          float* part, float* dW, float* db, int64_t R, int64_t Hc, int64_t Wc,
                          int64_t Ca, int64_t Cb, int stride, void* stream);

/* ---- k x k convolutions on the tensor-core products, NHWC (csrc/conv_tc.cu; the GAN examples) --
 * The memory passes around the dense products that make a k x k convolution (1 <= k <= 7, stride 1
 * or 2).  Geometry on the convolution's side: the big grid Hb x Wb is its input (the transposed
 * convolution's output), the small grid Hs x Ws its output, N images, C channels of the tensor the
 * pass reads or writes, and big pixel (s i + kh - pt, s j + kw - pl) meets small pixel (i, j) at
 * tap (kh, kw); big pixels outside the grid count as zero.  TF's SAME and VALID are the caller's
 * choice of Hs, Ws and the pads (0 <= pt, pl < k).  N Hb Wb C and N Hs Ws k k C below 2^31.
 * Gather-split: x [N, Hb, Wb, C] -> planes [2][N Hs Ws][kpad(k k C)], the fp16 hi/lo operand
 * planes of the im2col matrix (column (kh k + kw) C + c) at the power-of-two scale of max |x|,
 * which is taken from scale[2] when have_amax (a producer's max |.| tag) or found by a max pass;
 * the fp32 matrix is never written.  scale = device float[4] with scale[2] zero or the tag. */
int zsb_conv_gather_split_f32(const float* x, int64_t N, int64_t Hb, int64_t Wb, int64_t C,
                              int64_t Hs, int64_t Ws, int k, int stride, int pt, int pl,
                              void* planes, float* scale, int have_amax, void* stream);
/* Col2im-sum: the big-grid tensor [N, Hb, Wb, C] whose entry is the sum, over the taps that land
 * on it (kh, then kw, ascending: deterministic, no atomics), of cols [N Hs Ws, k k C] fp32.
 *   epi 0: out = the sum (a convolution's input gradient)
 *   epi 1: out = act(sum + bias[c] + residual) with bias [C] and residual [N, Hb, Wb, C] (either
 *          may be NULL): the generators' sigmoid output layers, and the transposed convolution of
 *          examples/utils/utils.py:74-113 with the resnet blocks' residual added before the ReLU
 *          (vae_conv.py:20-36)
 *   epi 2: batch norm training: pre = the sum and part [ceil(N Hb Wb / 128)][2][C] its per-tile
 *          moments, for zsb_bn_finish_fused_f32 (out unused)
 *   epi 3: batch norm evaluation: out = act(xhat gamma + beta), xhat = (sum - moving_mean)
 *          rsqrt(moving_var + eps); stats [2][C] = (moving_mean, rstd); pre (may be NULL) = sum
 * act: 0 none, 1 ReLU, 2 sigmoid; epi 1 takes any, epi 3 none or ReLU, epi 0 and 2 none.  max |out|
 * into amax_scale[2] (may be NULL; epi 0, 1, 3). */
int zsb_conv_col2im_f32(int epi, const float* cols, int64_t N, int64_t Hb, int64_t Wb, int64_t C,
                        int64_t Hs, int64_t Ws, int k, int stride, int pt, int pl,
                        const float* bias, const float* residual, const float* gamma,
                        const float* beta, const float* moving_mean, const float* moving_var,
                        float eps, int act, float* stats, float* pre, float* part, float* out,
                        float* amax_scale, void* stream);
/* Backward through act(conv + b + residual) with output y [R, C] (the tf.gradients of the
 * activation, bias_add and residual add): gp = g y (1 - y) (act 2, sigmoid), g (y > 0) (act 1,
 * ReLU) or g (act 0; y may then be NULL), which is also the residual's gradient; max |gp| into
 * scale[2], and db [C] (may be NULL) = the column sums of gp, merged in a fixed order from
 * part [ceil(R / 128)][C].  C < 2^20, R C < 2^31. */
int zsb_conv_act_grad_f32(const float* g, const float* y, int64_t R, int C, int act, float* gp,
                          float* part, float* db, float* scale, void* stream);

/* ---- K5: SG-MCMC updates (zhusuan/sgmcmc.py) ------------------------------------------------ */
int zsb_sgmcmc_parts(void);   /* capacity (floats) of every `part` scratch */
int zsb_sgmcmc_sgld_f32(float* q, const float* g, const float* noise, float lr, int64_t chains,
                        int64_t row_len, uint64_t seed, uint32_t iter, int64_t row0,
                        void* stream);                                   /* sgmcmc.py:195-200 */
int zsb_sgmcmc_psgld_f32(float* q, float* aux, const float* g, const float* noise, float lr,
                         float decay, float epsilon, int64_t chains, int64_t row_len,
                         uint64_t seed, uint32_t iter, int64_t row0, void* stream); /* :225-257 */
int zsb_sgmcmc_resample_v_f32(float* v, const float* noise, float lr, int64_t chains,
                              int64_t row_len, uint64_t seed, uint32_t iter, int64_t row0,
                              void* stream);                             /* :320-336 */
int zsb_sgmcmc_half_q_f32(float* q, const float* v, int64_t n, void* stream);  /* :351, :493 */
int zsb_sgmcmc_sghmc_f32(float* q, float* v, const float* g, const float* noise, float lr,
                         float alpha, float beta, int second_order, int64_t chains,
                         int64_t row_len, uint64_t seed, uint32_t iter, int64_t row0,
                         float* part, float* mean_k, void* stream);      /* :338-358 */
int zsb_sgmcmc_sgnht_vec_f32(float* q, float* v, float* alpha, const float* g, const float* noise,
                             float lr, float a, float tune_rate, int second_order, int64_t chains,
                             int64_t row_len, uint64_t seed, uint32_t iter, int64_t row0,
                             float* mean_k_out, void* stream);           /* :460-523 vector alpha */
int zsb_sgmcmc_mean_sq_f32(const float* v, int64_t n, float* part, float* out, void* stream);
int zsb_sgmcmc_sgnht_scalar_f32(float* q, float* v, const float* alpha_eff, const float* g,
                                const float* noise, float lr, float a, int second_order,
                                int64_t chains, int64_t row_len, uint64_t seed, uint32_t iter,
                                int64_t row0, float* part, float* mean_k, void* stream);
int zsb_sgmcmc_sgnht_alpha_f32(float* out, const float* in, const float* mean_k, float coef,
                               float lr, void* stream);

/* Fused SGHMC step for the two-layer BNN regression log-joint of
 * examples/bayesian_neural_nets/bnn_sgmcmc.py:19-35, 74-91 (layer sizes [n_in, H, 1]; per-chain
 * weights w0 [chains,H,n_in+1], w1 [chains,1,H+1]): momentum resample, half step, hand-derived
 * forward/backward over the minibatch, prior gradient and the sgmcmc.py:338-358 update in ONE
 * launch.  part: 2*zsb_sgmcmc_parts() floats; mean_k: 2 floats (one per latent).
 * Same as zsb_sgmcmc_bnn_step_f32(ZSB_SGMCMC_SGHMC, ...). */
int zsb_sgmcmc_sghmc_bnn_f32(float* w0, float* w1, float* v0, float* v1, const float* x,
                             const float* y, int B, int n_in, int H, const float* logstd0,
                             int64_t logstd0_n, const float* logstd1, int64_t logstd1_n,
                             float y_logstd, float n_train, float lr, float alpha, float beta,
                             int second_order, int resample, const float* noise0,
                             const float* noise1, const float* resample0, const float* resample1,
                             uint64_t seed, uint32_t iter, int64_t row0, float* part,
                             float* mean_k, int64_t chains, void* stream);

/* Update rules of zsb_sgmcmc_bnn_step_f32. */
enum zsb_sgmcmc_method {
  ZSB_SGMCMC_SGHMC = 0,         /* sgmcmc.py:326-371 */
  ZSB_SGMCMC_SGLD = 1,          /* sgmcmc.py:195-200 */
  ZSB_SGMCMC_PSGLD = 2,         /* sgmcmc.py:225-257 */
  ZSB_SGMCMC_SGNHT_VEC = 3,     /* sgmcmc.py:460-523, use_vector_alpha=True */
  ZSB_SGMCMC_SGNHT_SCALAR = 4   /* sgmcmc.py:460-523, use_vector_alpha=False */
};

/* One fused SG-MCMC step of `method` for the same BNN log-joint and shape limits as
 * zsb_sgmcmc_sghmc_bnn_f32 (n_in + 1 <= 16, H <= 64, B <= 512), replacing the generic gradient plus
 * zsb_sgmcmc_{sgld,psgld,sghmc,sgnht_vec,sgnht_scalar}_f32 with ONE launch.  Each rule keeps the
 * rounding and operation order of its element-wise kernel.  State (NULL where unused):
 *   v0/v1        momenta (SGHMC, SGNHT), shaped like w0 / w1
 *   aux0/aux1    PSGLD's RMS accumulator (sgmcmc.py:225-230) or vector SGNHT's thermostat alpha
 *                (sgmcmc.py:454-458), shaped like w0 / w1
 *   alpha_eff0/1 scalar SGNHT: device scalar per latent, alpha (1st order) or alpha1 (2nd)
 *   mean_k0/1    SGHMC, scalar SGNHT: one float each, mean(v_new^2) of this call's chains;
 *                vector SGNHT: shaped like w0 / w1, receives k = v_new^2 (sgmcmc.py:497-505)
 *   part         2*zsb_sgmcmc_parts() floats (SGHMC, scalar SGNHT)
 * friction/variance_estimate: SGHMC; decay/epsilon: PSGLD; variance_extra/tune_rate: SGNHT.
 * second_order and resample apply to SGHMC and vector SGNHT; scalar SGNHT re-draws v with
 * zsb_sgmcmc_resample_v_f32 before the step and updates alpha from mean_k after it
 * (zsb_sgmcmc_mean_sq_f32 / zsb_sgmcmc_sgnht_alpha_f32), as the generic path does. */
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
                            void* stream);

/* ---- BNN regression log-joint, value / gradient / predictions (csrc/bnn_logjoint.cu) ----------
 * The model and log-joint of examples/bayesian_neural_nets/bnn_vi.py:18-35, 83-86 (the same as
 * bnn_sgmcmc.py:19-35, 74-77) for K particles, replacing the einsum / concat / relu / Normal
 * log_prob graph and its tf.gradients (bnn_vi.py:88-89) and the prediction fetches (:98-103):
 *   lp[k] = sum log N(w0[k]; 0, exp(ls0)) + sum log N(w1[k]; 0, exp(ls1))
 *           + n_train * mean_b log N(y_b; y_mean[k, b], exp(y_logstd))
 * w0 [K, H, n_in+1], w1 [K, 1, H+1], x [B, n_in], y [B]; logstd0 / logstd1 are read flat over one
 * particle's weights, index modulo logstd*_n.  y_logstd is a DEVICE scalar (learnable, no host
 * sync).  Outputs, each written only when non-NULL: lp [K]; g0 / g1 (shaped like w0 / w1) =
 * d lp / d w; g_ylogstd [K] = d lp[k] / d y_logstd; y_mean [K, B]; log_lik [K, B] =
 * log N(y_b; y_mean, exp(y_logstd)), unscaled.  n_in + 1 <= 16, H <= 64, any B >= 1.  No
 * floating-point atomics: deterministic. */
int zsb_bnn_logjoint_f32(const float* w0, const float* w1, const float* x, const float* y,
                         int64_t B, int n_in, int H, const float* logstd0, int64_t logstd0_n,
                         const float* logstd1, int64_t logstd1_n, const float* y_logstd,
                         float n_train, float* lp, float* g0, float* g1, float* g_ylogstd,
                         float* y_mean, float* log_lik, int64_t K, void* stream);

/* ---- BNN regression with L >= 3 weight layers (csrc/bnn_deep.cu) -------------------------------
 * build_bnn of examples/bayesian_neural_nets/bnn_vi.py:18-35 and bnn_sgmcmc.py:19-35 at
 * layer_sizes = [n_0, ..., n_{L-1}, 1] (widths[0..L], widths[L] = 1), with the log-joint override
 * of bnn_vi.py:83-86 / bnn_sgmcmc.py:74-77, replacing the per-layer einsum / concat / relu /
 * Normal log_prob graph, its tf.gradients (bnn_vi.py:88-89, sgmcmc.py:96-98) and the prediction
 * fetches (bnn_vi.py:98-103).  Layer i: w[i] [K, widths[i+1], widths[i] + 1], prior
 * N(0, exp(logstd[i])) read flat over one particle's layer, index modulo logstd_n[i].  The
 * per-layer arrays (w, g, logstd, logstd_n, ...) are HOST arrays of L entries.  Limits:
 * 3 <= L <= 8, widths[i] <= 128 for i < L, at most 32768 weights per particle; any B and K >= 1.
 * No floating-point atomics: deterministic.
 *
 * Value, gradients and predictions in one launch; outputs as zsb_bnn_logjoint_f32's, each
 * written only when non-NULL (g may be NULL, or hold NULL for a layer whose gradient is not
 * needed).  y_logstd is a DEVICE scalar. */
int zsb_bnn_deep_logjoint_f32(int L, const int* widths /* host */, const float* const* w /* host */,
                              const float* x, const float* y, int64_t B,
                              const float* const* logstd /* host */,
                              const int* logstd_n /* host */, const float* y_logstd,
                              float n_train, float* lp, float* const* g /* host */,
                              float* g_ylogstd, float* y_mean, float* log_lik, int64_t K,
                              void* stream);

/* One fused SG-MCMC step of `method` (enum zsb_sgmcmc_method) on the same log-joint, gradient and
 * update of every layer in one launch (sgmcmc.py:195-200, 225-257, 326-371, 460-523), with
 * zsb_sgmcmc_bnn_step_f32's state per layer (host arrays of L device pointers; NULL arrays where
 * the method has no such state): v, aux, alpha_eff, mean_k.  The noise of latent i is
 * (seed + i, iter, row0 + chain), as the element-wise zsb_sgmcmc_*_f32 kernels draw it, or
 * injected through noise / resample_noise (host arrays, or NULL).  part: L*zsb_sgmcmc_parts()
 * floats (SGHMC, scalar SGNHT); work: work_n >= min(chains, zsb_sgmcmc_parts()) * (weights per
 * chain) floats of scratch for the gradient. */
int zsb_sgmcmc_bnn_deep_step_f32(int method, int L, const int* widths /* host */,
                                 float* const* w /* host */, float* const* v /* host */,
                                 float* const* aux /* host */,
                                 const float* const* alpha_eff /* host */, const float* x,
                                 const float* y, int64_t B, const float* const* logstd /* host */,
                                 const int* logstd_n /* host */, float y_logstd, float n_train,
                                 float lr, float friction, float variance_estimate, float decay,
                                 float epsilon, float variance_extra, float tune_rate,
                                 int second_order, int resample,
                                 const float* const* noise /* host */,
                                 const float* const* resample_noise /* host */, uint64_t seed,
                                 uint32_t iter, int64_t row0, float* part,
                                 float* const* mean_k /* host */, float* work, int64_t work_n,
                                 int64_t chains, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ZSB200_H_ */
