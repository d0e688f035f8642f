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
/* src [R, C] -> planes [2][C][kpad(R)] of src^T (operands of the weight-gradient product) */
int zsb_split16_pad_t_f32(const float* src, int64_t R, int C, void* planes, float* scale,
                          void* stream);
/* split-K slices an epi-0 launch uses when `part` (slices * R * J floats) is supplied */
int zsb_linear_tc_slices(int64_t R, int J, int K);
int zsb_linear_tc_f32(int epi, const void* w_planes, const float* scale_w, const void* h_planes,
                      const float* scale_h, const float* bias, const float* x_obs, int64_t n_x,
                      const float* gout, float* out, float* part, int64_t R, int J, int K,
                      int relu, void* stream);
/* As zsb_linear_tc_f32, additionally folding max |out| (epi 0 / 2) into amax_scale[2] so that the
 * consumer's operand split (zsb_split16_dual_f32, have_amax = 1) needs no pass over `out`. */
int zsb_linear_tc_amax_f32(int epi, const void* w_planes, const float* scale_w,
                           const void* h_planes, const float* scale_h, const float* bias,
                           const float* x_obs, int64_t n_x, const float* gout, float* out,
                           float* part, int64_t R, int J, int K, int relu, float* amax_scale,
                           void* stream);
/* Both operand layouts of an activation / gradient matrix in one pass: planes [2][R][Kp] and
 * planes_t [2][K][Rp] (either may be NULL) of src * scale, optionally times the ReLU mask
 * (mask_src > 0) -- the `g * (y > 0)` of the dense layer's backward (tf.layers.dense + relu,
 * iwae.py:23-44) -- and the column sums of the masked matrix (bias gradient) into col_sum. */
int zsb_split16_dual_f32(const float* src, const float* mask_src, int64_t R, int K, void* planes,
                         void* planes_t, float* col_sum, float* scale, int have_amax,
                         void* stream);

/* Backward of the fused Bernoulli likelihood layer (gradient of epi 1 wrt the logits, epi 2)
 * emitted directly as the operand planes of the two backward products: dl_planes [2][R][kpad(J)]
 * = fp16 hi/lo of gout[r] * (x - sigmoid(logits)) * scale_out[0], col_sum [J] += its column sums
 * (bias gradient, may be NULL).  scale_out = device float[4], zeroed once by the caller; the power
 * of two follows from max|gout| * (1 + max|x_obs|) >= max|dl| BEFORE the GEMM, so the fp32
 * dl matrix (822 MB at config 3: univariate.py:398-403 differentiated) never exists. */
int zsb_linear_tc_bern_grad_planes_f32(const void* w_planes, const float* scale_w,
                                       const void* h_planes, const float* scale_h,
                                       const float* bias, const float* x_obs, int64_t n_x,
                                       const float* gout, void* dl_planes, float* col_sum,
                                       float* scale_out, int64_t R, int J, int K, void* stream);
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
int zsb_hmc_dense_tc_config(int bk);   /* impl-1 pipeline shape: 32 (2x64 KB) or 16 (4x32 KB) */
int zsb_hmc_dense_split_lo_f32(const float* q, float* lo, int64_t n, void* stream);
/* impl 2: fp16-split tensor-core path (3 fp16 wgmma products per k-step at twice the TF32 rate).
 * P_h16/P_l16: [D,D] __half hi/lo of P*sP; q_*_planes: [2][chains][D] __half hi/lo of q*sq;
 * scales: device float[4] = {sq, 1/(sP*sq), scratch, sP}.  D % 64 == 0. */
int zsb_hmc_dense_h16_prepare_f32(const float* q, void* planes, float* scales, int64_t n,
                                  void* stream);
int zsb_hmc_dense_leapfrog_h16_f32(const float* q_cur, const void* q_cur_planes, float* q_next,
                                   void* q_next_planes, const float* p_in, float* p_out,
                                   const void* P_h16, const void* P_l16, const float* scales,
                                   const float* bvec, const float* mu, const float* mass,
                                   const float* state, float p_scale, float* lp_part,
                                   float* k_part, int64_t chains, int64_t D, void* stream);
/* impl 3: impl 2 with the fp16 planes of q produced inside the kernel (by the MMA warpgroup from
 * the fp32 rows): HBM traffic per pass = the algorithmic 16*D bytes per chain.  scales: device
 * float[8], [3] = sP, [4..6] rotating max|q| slots; prepare before pass 0 of each trajectory. */
int zsb_hmc_dense_h16i_prepare_f32(const float* q, float* scales, int64_t n, void* stream);
int zsb_hmc_dense_leapfrog_h16i_f32(const float* q_cur, float* q_next, const float* p_in,
                                    float* p_out, const void* P_h16, const void* P_l16,
                                    float* scales, int pass_index, const float* bvec,
                                    const float* mu, const float* mass, const float* state,
                                    float p_scale, float* lp_part, float* k_part, int64_t chains,
                                    int64_t D, void* stream);
/* impl 4: the whole leapfrog `while_loop` of hmc.py:347-372 (L+1 passes) through one entry point
 * with impl 2's buffers and ping-pong schedule.  D == 1024, L >= 1.
 * Buffers as impl 2 (planes0 from zsb_hmc_dense_h16_prepare_f32); the proposal ends in qa when
 * L - 1 is even, else in qb; pw holds the final momentum. */
int zsb_hmc_dense_trajectory_h16_f32(const float* q0, const void* planes0, float* qa,
                                     void* planes_a, float* qb, void* planes_b, const float* p0,
                                     float* pw, const void* P_h16, const void* P_l16,
                                     const float* scales, const float* bvec, const float* mu,
                                     const float* mass, const float* state, float* lp0_part,
                                     float* lp1_part, float* k_part, int64_t chains, int64_t D,
                                     int n_leapfrogs, void* stream);
/* impl 5: the whole leapfrog `while_loop` of hmc.py:347-372 (L+1 passes, body = leapfrog_integrator
 * hmc.py:38-43, plus the log p / kinetic terms of hamiltonian() hmc.py:30-35) with the fp16 hi/lo
 * plane pair of q*sq as the state of q inside the trajectory (planes0 from
 * zsb_hmc_dense_h16_prepare_f32; planes1 = work buffer of the same size, distinct from planes0);
 * the proposal's planes end in buffer (n_leapfrogs & 1) and zsb_hmc_dense_select_planes_f32
 * assigns them to the accepted chains (the `tf.where` + assign of hmc.py:488-497).  `flags`
 * (zsb_hmc_dense_resident_flags(chains) int32 words) is reserved scratch.  D % 64 == 0,
 * n_leapfrogs >= 1. */
int zsb_hmc_dense_resident_flags(int64_t chains);
int zsb_hmc_dense_resident_group(int64_t D);
int zsb_hmc_dense_resident_h16_f32(void* planes0, void* planes1, const float* p0, float* pw,
                                   const void* P_h16, const void* P_l16, const float* scales,
                                   const float* bvec, const float* mu, const float* mass,
                                   const float* state, float* lp0_part, float* lp1_part,
                                   float* k_part, int32_t* flags, int64_t chains, int64_t D,
                                   int n_leapfrogs, void* stream);
int zsb_hmc_dense_select_planes_f32(float* q, const void* planes, const float* scales,
                                    const int32_t* accept, int64_t chains, int64_t D,
                                    void* stream);
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
/* Poisson._sample (univariate.py:915-920) / Binomial._sample (univariate.py:1025-1045): kind 0 =
 * Poisson(rate = param), 1 = Binomial(n_experiments, sigmoid(param)); one uniform per draw
 * (injected u [n] or Philox), inverse transform enumerating the support outwards from the mode. */
int zsb_sample_count_i32(int kind, const float* param, int64_t param_n, int64_t n_experiments,
                         const float* u, uint64_t seed, uint32_t iter, int32_t* out, int64_t n,
                         void* stream);

/* ---- K8, config 5: Logistic-Normal Topic Model E-step log-joint (csrc/lntm.cu) -----------------
 * log p = sum_k Normal(eta_k; mean_k, exp(logstd_k)).log_prob + sum_v x[d,v] log(softmax(eta) @ phi)[v]
 * (examples/topic_models/lntm_mcem.py:33-48, e_obj :97-99; UnnormalizedMultinomial._log_prob,
 * multivariate.py:435-443 with normalize_logits=False) and its gradient w.r.t. eta, fused and
 * sparsity-aware: the corpus is CSR, only the words a document contains are formed, the
 * [chains*docs, V] matrix of the reference never exists.  phi_t = softmax(beta)^T [V, K]. */
int zsb_lntm_phi_t_f32(const float* beta, int64_t n_topics, int64_t n_vocab, float* phi_t,
                       void* stream);
int zsb_lntm_logjoint_f32(const float* eta, const float* eta_mean, const float* eta_logstd,
                          const float* phi_t, const int64_t* doc_ptr, const int32_t* word_idx,
                          const float* word_cnt, float* lp_out, float* grad_out, int64_t chains,
                          int64_t docs, int64_t n_topics, void* stream);

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
 * launch.  part: 2*zsb_sgmcmc_parts() floats; mean_k: 2 floats (one per latent). */
int zsb_sgmcmc_sghmc_bnn_f32(float* w0, float* w1, float* v0, float* v1, const float* x,
                             const float* y, int B, int n_in, int H, const float* logstd0,
                             int64_t logstd0_n, const float* logstd1, int64_t logstd1_n,
                             float y_logstd, float n_train, float lr, float alpha, float beta,
                             int second_order, int resample, const float* noise0,
                             const float* noise1, const float* resample0, const float* resample1,
                             uint64_t seed, uint32_t iter, int64_t row0, float* part,
                             float* mean_k, int64_t chains, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* ZSB200_H_ */
