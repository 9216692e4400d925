// inst_dyn.cu - compiled once per dynamics kind of dyn_instances.def (see Makefile): the Instance record
// inst_dyn__<kind> with the generic step kernel that has that kind's step function compiled into its line-search
// rollout, in float and double.  No gradient or rollout launchers.
#include "instance.cuh"

#ifndef INST_DYN
#error "compile with -DINST_DYN=<dynamics kind>"
#endif

#define MPCB_CAT_(a, b) a##b
#define MPCB_CAT(a, b) MPCB_CAT_(a, b)

namespace mpcb200 {

using DD = DynDims<INST_DYN>;
#define MPCB200_DYN_INST(kind, n, m) \
  static_assert(kind != INST_DYN || (DD::N == n && DD::M == m), "dyn_instances.def disagrees with DynDims");
#include "dyn_instances.def"
#undef MPCB200_DYN_INST

// a.impl (the MPCB200_KERNEL knob) 2 asks for the column-pair kernel, which has no in-kernel dynamics
template <typename R>
static int dyn_step_dispatch(const StepArgs& a, int max_smem, cudaStream_t s) {
  if (a.impl == 2 || a.dyn_kind != INST_DYN) return MPCB200_ERR_UNSUPPORTED_DIMS;
  return launch_step<R, DD::N, DD::M, INST_DYN>(a, max_smem, s);
}

template <typename R>
static constexpr InstanceOps kOps = {dyn_step_dispatch<R>, nullptr, nullptr, step_prefers_workspace<R, DD::N, DD::M>,
                                     step_smem_query<R, DD::N, DD::M>};
extern const Instance MPCB_CAT(inst_dyn__, INST_DYN);
constexpr Instance MPCB_CAT(inst_dyn__, INST_DYN) = {INST_DYN, DD::N, DD::M, {kOps<float>, kOps<double>}};

}  // namespace mpcb200
