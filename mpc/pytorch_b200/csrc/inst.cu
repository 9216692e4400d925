// inst.cu - compiled once per (INST_N, INST_M) pair (see Makefile): the Instance record inst__<n>_<m> with the
// step, gradient and rollout launchers of that shape in float and double.
#include "instance.cuh"
#include "lqr_step2.cuh"

#ifndef INST_N
#error "compile with -DINST_N=<n_state> -DINST_M=<n_ctrl>"
#endif

#define MPCB_CAT_(a, b, c) a##b##_##c
#define MPCB_CAT(a, b, c) MPCB_CAT_(a, b, c)

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

template <typename R>
static constexpr InstanceOps kOps = {step_dispatch<R>, launch_grad<R, INST_N, INST_M>,
                                     launch_rollout<R, INST_N, INST_M>, step_prefers_workspace<R, INST_N, INST_M>,
                                     step_smem_query<R, INST_N, INST_M>};
extern const Instance MPCB_CAT(inst__, INST_N, INST_M);
constexpr Instance MPCB_CAT(inst__, INST_N, INST_M) = {DYN_LINEAR, INST_N, INST_M, {kOps<float>, kOps<double>}};

}  // namespace mpcb200
