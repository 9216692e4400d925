// inst.cu - compiled once per (INST_N, INST_M) pair (see Makefile): explicit launchers for
// the step and gradient kernels in float and double.
#include "lqr_grad.cuh"
#include "lqr_rollout.cuh"
#include "lqr_step.cuh"
#include "lqr_step2.cuh"

#ifndef INST_N
#error "compile with -DINST_N=<n_state> -DINST_M=<n_ctrl>"
#endif

#define MPCB_CAT_(a, b, c, d) a##b##_##c##_##d
#define MPCB_CAT(a, b, c, d) MPCB_CAT_(a, b, c, d)

namespace mpcb200 {

// a.impl: 0 = pick (the column-pair kernel where its shape constraints hold), 1 = generic kernel, 2 = pair kernel
template <typename R>
static int step_dispatch(const StepArgs& a, int max_smem, cudaStream_t s) {
  if (a.impl == 2 || (a.impl == 0 && Step2Cfg<R, INST_N, INST_M>::PAIR_DEFAULT)) {
    const int rc = launch_step2<R, INST_N, INST_M>(a, max_smem, s);
    if (rc != STEP2_DECLINED && !(rc == MPCB200_ERR_SMEM && a.impl == 0)) return rc;
    if (a.impl == 2 && rc == STEP2_DECLINED) return MPCB200_ERR_UNSUPPORTED_DIMS;
  }
  return launch_step<R, INST_N, INST_M>(a, max_smem, s);
}
int MPCB_CAT(step_f32_, , INST_N, INST_M)(const StepArgs& a, int max_smem, cudaStream_t s) {
  return step_dispatch<float>(a, max_smem, s);
}
int MPCB_CAT(step_f64_, , INST_N, INST_M)(const StepArgs& a, int max_smem, cudaStream_t s) {
  return step_dispatch<double>(a, max_smem, s);
}
int MPCB_CAT(grad_f32_, , INST_N, INST_M)(const GradArgs& a, cudaStream_t s) {
  return launch_grad<float, INST_N, INST_M>(a, s);
}
int MPCB_CAT(grad_f64_, , INST_N, INST_M)(const GradArgs& a, cudaStream_t s) {
  return launch_grad<double, INST_N, INST_M>(a, s);
}
int MPCB_CAT(roll_f32_, , INST_N, INST_M)(const RolloutArgs& a, cudaStream_t s) {
  return launch_rollout<float, INST_N, INST_M>(a, s);
}
int MPCB_CAT(roll_f64_, , INST_N, INST_M)(const RolloutArgs& a, cudaStream_t s) {
  return launch_rollout<double, INST_N, INST_M>(a, s);
}
int MPCB_CAT(pws_f32_, , INST_N, INST_M)(int T, int ms) { return step_prefers_workspace<float, INST_N, INST_M>(T, ms); }
int MPCB_CAT(pws_f64_, , INST_N, INST_M)(int T, int ms) { return step_prefers_workspace<double, INST_N, INST_M>(T, ms); }
size_t MPCB_CAT(smem_f32_, , INST_N, INST_M)(int T) { return step_smem_query<float, INST_N, INST_M>(T); }
size_t MPCB_CAT(smem_f64_, , INST_N, INST_M)(int T) { return step_smem_query<double, INST_N, INST_M>(T); }

}  // namespace mpcb200
