// instance.cuh - the record each compiled instance exports (inst.cu, inst_dyn.cu) and api.cu dispatches through.
#pragma once
#include "lqr_grad.cuh"
#include "lqr_rollout.cuh"
#include "lqr_step.cuh"

namespace mpcb200 {

struct InstanceOps {                  // one element type of one compiled shape
  int (*step)(const StepArgs&, int max_smem, cudaStream_t);
  int (*grad)(const GradArgs&, cudaStream_t);          // nullptr: dynamics-only instance
  int (*rollout)(const RolloutArgs&, cudaStream_t);    // nullptr: dynamics-only instance
  int (*prefers_workspace)(int T, int max_smem);
  size_t (*smem_bytes)(int T);
};
// kind: DYN_LINEAR for an (n, m) instance of instances.def, or the dynamics kind of a dynamics-only instance.
// Constant-initialised (addresses only), so the records and api.cu's table of them need no start-up code.
struct Instance {
  int kind, n, m;
  InstanceOps ops[2];                 // [0] float, [1] double
};

}  // namespace mpcb200
