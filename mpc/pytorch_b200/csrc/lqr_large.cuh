// lqr_large.cuh - entry points of the kernels for (n_state, n_ctrl) shapes without a compiled instance
// (lqr_large.cu): the LQR step, the gradient assembly of the KKT adjoint and the LinDx rollout, one thread block
// per problem with runtime n and m.  Same argument blocks and contracts as the instance kernels.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include "lqr_grad.cuh"
#include "lqr_rollout.cuh"
#include "lqr_step.cuh"

namespace mpcb200 {

// which per-problem spans of a time step the large step kernel streams with 1-D bulk copies (16-byte aligned
// start and length at every t); the others are copied by the block's threads
enum : unsigned { LB_C = 1u, LB_F = 2u, LB_c = 4u, LB_f = 8u, LB_x = 16u, LB_u = 32u, LB_BOX = 64u };

// dynamic shared memory (bytes) of the large step kernel with 1 or 2 stages of per-time-step tiles
size_t large_step_smem_bytes(int n, int m, int elem_size, int stages);
// whether the large step kernel runs (n, m) with max_smem bytes of shared memory per block
bool large_step_fits(int n, int m, int elem_size, int max_smem);

// Ks/ks are required (the gains always go through global memory); return MPCB200_* codes
template <typename R>
int large_step_launch(const StepArgs& a, int n, int m, unsigned bulk, int max_smem, cudaStream_t stream);
template <typename R>
int large_grad_launch(const GradArgs& a, int n, int m, cudaStream_t stream);
template <typename R>
int large_rollout_launch(const RolloutArgs& a, int n, int m, cudaStream_t stream);

}  // namespace mpcb200
