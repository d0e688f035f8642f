// Trajectory entry point of dense_impl = 4: the L+1 leapfrog passes of zhusuan/hmc.py:347-372
// (body = leapfrog_integrator, hmc.py:38-43, plus the log p / kinetic terms of hamiltonian(),
// hmc.py:30-35) for every chain, with the buffers and operand planes of the per-pass fp16-split
// kernel (impl 2, hmc_dense_tc.cu) and the ping-pong schedule of the per-pass host loop
// (zhusuan_b200/hmc.py: q0 -> qa -> qb -> qa ...).  Each pass is one launch of that kernel.
#include "common.cuh"

int zsb_dense_leapfrog_h16_launch(const float* q_cur, const void* q_cur_planes, float* q_next,
                                  void* q_next_planes, const float* p_in, float* p_out,
                                  const void* P_h16, const void* P_l16, float* scales,
                                  int pass_index, const float* bvec, const float* mu,
                                  const float* mass, const float* state, float p_scale,
                                  float* lp_part, float* k_part, int64_t chains, int D,
                                  cudaStream_t st);

//   q0 / planes0: current state and its fp16 planes (zsb_hmc_dense_h16_prepare_f32);
//   qa, qb, planes_a, planes_b: work buffers; on return the proposal is in (L-1 even ? qa : qb);
//   p0 -> pw (final momentum); lp0_part / lp1_part / k_part and the plane-scale records as the
//   per-pass kernel writes them (pass i = launch i).
int zsb_dense_traj_h16_launch(const float* q0, const void* planes0, float* qa, void* planes_a,
                              float* qb, void* planes_b, const float* p0, float* pw,
                              const void* P_h16, const void* P_l16, float* scales,
                              const float* bvec, const float* mu, const float* mass,
                              const float* state, float* lp0_part, float* lp1_part,
                              float* k_part, int64_t chains, int D, int L, cudaStream_t st) {
  if (D != 1024 || L < 1 || chains <= 0 || chains >= (1LL << 31)) {
    zsb_set_error("dense_traj: needs D == 1024, n_leapfrogs >= 1");
    return ZSB_ERR_INVALID;
  }
  const float* cur = q0;
  const void* cur_pl = planes0;
  float* nxt = qa;
  void* nxt_pl = planes_a;
  const float* p_in = p0;
  for (int i = 0; i <= L; ++i) {
    const bool last = i == L;
    const int rc = zsb_dense_leapfrog_h16_launch(
        cur, cur_pl, last ? nullptr : nxt, last ? nullptr : nxt_pl, p_in, pw, P_h16, P_l16,
        scales, i, bvec, mu, mass, state, (i > 0 && !last) ? 1.f : 0.5f,
        i == 0 ? lp0_part : (last ? lp1_part : nullptr), last ? k_part : nullptr, chains, D, st);
    if (rc != ZSB_OK) return rc;
    p_in = pw;
    if (!last) {
      cur = nxt;
      cur_pl = nxt_pl;
      nxt = (nxt == qa) ? qb : qa;
      nxt_pl = (nxt == qa) ? planes_a : planes_b;
    }
  }
  return ZSB_OK;
}
