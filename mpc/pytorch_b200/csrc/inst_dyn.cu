// inst_dyn.cu - compiled once per dynamics kind of dyn_instances.def (see Makefile): the generic step kernel with
// that kind's step function compiled into its line-search rollout, in float and double.
#include "lqr_step.cuh"

#ifndef INST_DYN
#error "compile with -DINST_DYN=<dynamics kind>"
#endif

#define MPCB_CAT_(a, b) a##b
#define MPCB_CAT(a, b) MPCB_CAT_(a, b)

namespace mpcb200 {

using DD = DynDims<INST_DYN>;

// a.impl (the MPCB200_KERNEL knob) 2 asks for the column-pair kernel, which has no in-kernel dynamics
template <typename R>
static int dyn_step_dispatch(const StepArgs& a, int max_smem, cudaStream_t s) {
  if (a.impl == 2 || a.dyn_kind != INST_DYN) return MPCB200_ERR_UNSUPPORTED_DIMS;
  return launch_step<R, DD::N, DD::M, INST_DYN>(a, max_smem, s);
}
int MPCB_CAT(dstep_f32__, INST_DYN)(const StepArgs& a, int max_smem, cudaStream_t s) {
  return dyn_step_dispatch<float>(a, max_smem, s);
}
int MPCB_CAT(dstep_f64__, INST_DYN)(const StepArgs& a, int max_smem, cudaStream_t s) {
  return dyn_step_dispatch<double>(a, max_smem, s);
}
int MPCB_CAT(dpws_f32__, INST_DYN)(int T, int ms) { return step_prefers_workspace<float, DD::N, DD::M>(T, ms); }
int MPCB_CAT(dpws_f64__, INST_DYN)(int T, int ms) { return step_prefers_workspace<double, DD::N, DD::M>(T, ms); }
size_t MPCB_CAT(dsmem_f32__, INST_DYN)(int T) { return step_smem_query<float, DD::N, DD::M>(T); }
size_t MPCB_CAT(dsmem_f64__, INST_DYN)(int T) { return step_smem_query<double, DD::N, DD::M>(T); }

}  // namespace mpcb200
