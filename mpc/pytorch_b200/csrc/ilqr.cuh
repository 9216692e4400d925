// ilqr.cuh - the bookkeeping kernels of the device-side iLQR loop (mpcb200_ilqr_*): start, best-iterate
// tracking and the stop test of MPC.forward's outer loop (reference mpc/mpc.py:244-301), so that the whole loop
// runs as one CUDA graph with a conditional `while` node and no host round trip per iteration.
//
// One iteration of the loop body: rollout -> [linearisation] -> step -> ilqr_track_kernel -> ilqr_stop_kernel.
// Every buffer a body kernel reads is rewritten by an earlier body kernel of the same iteration or reset by
// ilqr_init_kernel, so the body consists of kernel nodes only.
// The kernels are instantiated in ilqr.cu alone (api.cu calls the launchers declared at the end): the stop kernel
// calls the device runtime's cudaGraphSetConditional, which the driver resolves when it loads that module.
#pragma once
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../../include/mpcb200.h"

namespace mpcb200 {

struct IlqrState {        // device-resident loop state, reset by ilqr_init_kernel
  int32_t iter;           // iterations completed; 0 = the best buffers are still empty
  int32_t n_not_improved;
  int32_t n_unconverged;  // iterations in which some problem's pnqp hit its iteration cap
  int32_t reserved;
};

enum : uint8_t { ILQR_BETTER = 1u, ILQR_UNCONVERGED = 2u };

// u = u_init (or 0); loop state and info reset; the loop's handle set to 1.  The handle's launch default would do
// that only when the graph is launched: a loop nested in the body of another (mpcb200_episode_*) restarts here.
template <typename R>
__global__ void __launch_bounds__(256)
ilqr_init_kernel(size_t n_u, const R* __restrict__ u_init, R* __restrict__ u, IlqrState* __restrict__ st,
                 int32_t* __restrict__ info, cudaGraphConditionalHandle handle) {
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (size_t i = i0; i < n_u; i += (size_t)gridDim.x * blockDim.x) u[i] = u_init != nullptr ? u_init[i] : R(0);
  if (i0 == 0) {
    st->iter = 0; st->n_not_improved = 0; st->n_unconverged = 0; st->reserved = 0;
    info[0] = 0; info[1] = 0;
    cudaGraphSetConditional(handle, 1);
  }
}

// `costs[b] <= best_costs[b] + best_cost_eps` in R, as torch evaluates it (a NaN on either side compares false)
template <typename R>
__device__ __forceinline__ bool ilqr_better(const R* costs, const R* best_costs, R best_cost_eps, int b) {
  return costs[b] <= best_costs[b] + best_cost_eps;
}

// After each step, grid-wide.  Element-wise: best_x / best_u take new_x / new_u where the problem improved (or on
// the first iteration): the select torch.where makes, so the best buffers are bitwise what it would give.  u, the
// next iteration's nominal controls, becomes new_u (the latest iterate, not the best one); controls past m_ref
// (zero padding up to a compiled instance) restart at 0, as a freshly padded tensor would.
// Per problem b: the reference's batch-mixing full_du_norm (mpc/lqr_step.py:244-245): du_first[T,B,M] restricted
// to the caller's m_ref controls, transposed to [T,m,B], viewed as [B, T*m], row 2-norm; and the flags
// ILQR_BETTER (never on the first iteration) and ILQR_UNCONVERGED for ilqr_stop_kernel.  best_costs and
// best_full_du_norm are updated by ilqr_stop_kernel, after every thread here has read best_costs.
template <typename R>
__global__ void __launch_bounds__(256)
ilqr_track_kernel(int B, int T, int N, int M, int m_ref, R best_cost_eps, const R* __restrict__ new_x,
                  const R* __restrict__ new_u, const R* __restrict__ costs, const R* __restrict__ du_first,
                  const int32_t* __restrict__ status, const R* __restrict__ best_costs, R* __restrict__ best_x,
                  R* __restrict__ best_u, R* __restrict__ u, R* __restrict__ fdn, uint8_t* __restrict__ flags,
                  const IlqrState* __restrict__ st) {
  const bool first = st->iter == 0;
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  const size_t nx = (size_t)T * B * N, nu = (size_t)T * B * M;
  for (size_t i = i0; i < nx; i += step) {
    const int b = (int)((i / N) % B);
    if (first || ilqr_better(costs, best_costs, best_cost_eps, b)) best_x[i] = new_x[i];
  }
  for (size_t i = i0; i < nu; i += step) {
    const int j = (int)(i % M), b = (int)((i / M) % B);
    const R v = new_u[i];
    if (first || ilqr_better(costs, best_costs, best_cost_eps, b)) best_u[i] = v;
    u[i] = j < m_ref ? v : R(0);
  }
  const size_t row = (size_t)T * m_ref, mB = (size_t)m_ref * B;
  for (size_t b = i0; b < (size_t)B; b += step) {
    R ss = R(0);
    for (size_t k = b * row; k < (b + 1) * row; ++k) {      // flat index k of the [T, m, B] transpose
      const size_t t = k / mB, j = (k / B) % m_ref, bb = k % B;
      const R d = du_first[(t * B + bb) * M + j];
      ss += d * d;
    }
    fdn[b] = sqrt(ss);
    uint8_t fl = 0;
    if (!first && ilqr_better(costs, best_costs, best_cost_eps, (int)b)) fl |= ILQR_BETTER;
    if (status[b] & MPCB200_ST_PNQP_UNCONVERGED) fl |= ILQR_UNCONVERGED;
    flags[b] = fl;
  }
}

// One block of ILQR_STOP_THREADS threads, after ilqr_track_kernel.  Takes costs / full_du_norm into the best
// buffers where the problem improved (or on the first iteration), reduces max_b full_du_norm (a NaN propagates,
// as in torch.max), any(better) and any(unconverged), updates the counters as the host loop does (reference
// mpc/mpc.py:244-301) and ends the loop through the conditional handle when
//   (double)max_du < eps   (a NaN never stops it),  n_not_improved > not_improved_lim,  or iter == lqr_iter.
constexpr int ILQR_STOP_THREADS = 256;
template <typename R>
__global__ void __launch_bounds__(ILQR_STOP_THREADS)
ilqr_stop_kernel(int B, int lqr_iter, int not_improved_lim, double eps, const R* __restrict__ costs,
                 const R* __restrict__ fdn, const uint8_t* __restrict__ flags, R* __restrict__ best_costs,
                 R* __restrict__ best_fdn, IlqrState* __restrict__ st, int32_t* __restrict__ info,
                 cudaGraphConditionalHandle handle) {
  __shared__ R s_max[ILQR_STOP_THREADS];
  const bool first = st->iter == 0;
  R mx = R(-INFINITY);
  int nan = 0, better = 0, unconv = 0;
  for (int b = threadIdx.x; b < B; b += ILQR_STOP_THREADS) {
    const uint8_t fl = flags[b];
    const R v = fdn[b];
    if (first || (fl & ILQR_BETTER)) {
      best_costs[b] = costs[b];
      best_fdn[b] = v;
    }
    if (v != v) nan = 1;
    else if (v > mx) mx = v;
    better |= fl & ILQR_BETTER;
    unconv |= (fl & ILQR_UNCONVERGED) ? 1 : 0;
  }
  s_max[threadIdx.x] = mx;
  nan = __syncthreads_or(nan);
  better = __syncthreads_or(better);
  unconv = __syncthreads_or(unconv);
  for (int w = ILQR_STOP_THREADS / 2; w > 0; w >>= 1) {
    if (threadIdx.x < w && s_max[threadIdx.x + w] > s_max[threadIdx.x]) s_max[threadIdx.x] = s_max[threadIdx.x + w];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const int iter = st->iter + 1;
    const int nni = better ? 0 : st->n_not_improved + 1;
    const int nun = st->n_unconverged + (unconv ? 1 : 0);
    st->iter = iter; st->n_not_improved = nni; st->n_unconverged = nun;
    info[0] = iter; info[1] = nun;
    const bool converged = !nan && (double)s_max[0] < eps;
    if (converged || nni > not_improved_lim || iter >= lqr_iter) cudaGraphSetConditional(handle, 0);
  }
}

// ---------------------------------------------------------------------------------------------
// the receding-horizon episode (mpcb200_episode_*): an outer `while` node whose body is the iLQR loop above, the
// model step from its best controls, then episode_advance_kernel
// ---------------------------------------------------------------------------------------------
struct EpisodeState {     // device-resident episode state, reset by episode_init_kernel
  int32_t step;           // control steps completed
  uint32_t tickets;       // blocks of the current episode_advance_kernel that have finished
  int32_t reserved[2];
};

// state = xs[0] = x_init; warm = u_init (or 0); counters reset; the episode's handle set to 1.
template <typename R>
__global__ void __launch_bounds__(256)
episode_init_kernel(size_t n_x, size_t n_u, const R* __restrict__ x_init, const R* __restrict__ u_init,
                    R* __restrict__ state, R* __restrict__ xs0, R* __restrict__ warm, EpisodeState* __restrict__ ep,
                    cudaGraphConditionalHandle handle) {
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  for (size_t i = i0; i < n_x; i += step) {
    const R v = x_init[i];
    state[i] = v;
    xs0[i] = v;
  }
  for (size_t i = i0; i < n_u; i += step) warm[i] = u_init != nullptr ? u_init[i] : R(0);
  if (i0 == 0) {
    ep->step = 0; ep->tickets = 0u; ep->reserved[0] = ep->reserved[1] = 0;
    cudaGraphSetConditional(handle, 1);
  }
}

// After the model step of control step k = ep->step, grid-wide.  us[k] = best_u[0]; xs[k+1] and the next solve's
// x_init (state) = traj[1]; the next warm start warm[t] = best_u[t+1] for t < T-2, best_u[T-2] at t = T-2, 0 at
// t = T-1 (cat(u[1:], 0), then w[-2] = w[-3]), with controls past m_ref at 0 as a freshly padded u_init has them;
// costs[k] = best_costs, info_out[k] = info.  The last block to finish advances ep->step and ends the episode's
// loop after n_steps control steps: every block has read ep->step by then.  DISTURB (mpcb200_episode_plant_*):
// traj[1] + w[k] instead of traj[1], w [n_steps, B, N] staged at the problem's shape.
template <typename R, bool DISTURB>
__device__ __forceinline__ void
episode_advance_body(int B, int T, int N, int M, int m_ref, int n_steps, const R* __restrict__ traj,
                     const R* __restrict__ best_u, const R* __restrict__ best_costs, const int32_t* __restrict__ info,
                     const R* __restrict__ w, R* __restrict__ state, R* __restrict__ warm, R* __restrict__ xs,
                     R* __restrict__ us, R* __restrict__ costs, int32_t* __restrict__ info_out,
                     EpisodeState* __restrict__ ep, cudaGraphConditionalHandle handle) {
  const int k = ep->step;
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  const size_t BM = (size_t)B * M, BN = (size_t)B * N;
  for (size_t i = i0; i < (size_t)T * BM; i += step) {
    const int t = (int)(i / BM), j = (int)(i % M);
    R v = R(0);
    if (j < m_ref && t < T - 1) v = best_u[t < T - 2 ? i + BM : i];
    warm[i] = v;
  }
  for (size_t i = i0; i < BM; i += step) us[(size_t)k * BM + i] = best_u[i];
  for (size_t i = i0; i < BN; i += step) {
    const R v = DISTURB ? traj[BN + i] + w[(size_t)k * BN + i] : traj[BN + i];
    state[i] = v;
    xs[(size_t)(k + 1) * BN + i] = v;
  }
  for (size_t b = i0; b < (size_t)B; b += step) costs[(size_t)k * B + b] = best_costs[b];
  if (i0 == 0) {
    info_out[2 * k] = info[0];
    info_out[2 * k + 1] = info[1];
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&ep->tickets, 1u) == gridDim.x - 1) {
      ep->tickets = 0u;
      ep->step = k + 1;
      if (k + 1 >= n_steps) cudaGraphSetConditional(handle, 0);
    }
  }
}
template <typename R>
__global__ void __launch_bounds__(256)
episode_advance_kernel(int B, int T, int N, int M, int m_ref, int n_steps, const R* __restrict__ traj,
                       const R* __restrict__ best_u, const R* __restrict__ best_costs, const int32_t* __restrict__ info,
                       R* __restrict__ state, R* __restrict__ warm, R* __restrict__ xs, R* __restrict__ us,
                       R* __restrict__ costs, int32_t* __restrict__ info_out, EpisodeState* __restrict__ ep,
                       cudaGraphConditionalHandle handle) {
  episode_advance_body<R, false>(B, T, N, M, m_ref, n_steps, traj, best_u, best_costs, info, nullptr, state, warm, xs,
                                 us, costs, info_out, ep, handle);
}
template <typename R>
__global__ void __launch_bounds__(256)
episode_advance_disturbed_kernel(int B, int T, int N, int M, int m_ref, int n_steps, const R* __restrict__ traj,
                                 const R* __restrict__ best_u, const R* __restrict__ best_costs,
                                 const int32_t* __restrict__ info, const R* __restrict__ w, R* __restrict__ state,
                                 R* __restrict__ warm, R* __restrict__ xs, R* __restrict__ us, R* __restrict__ costs,
                                 int32_t* __restrict__ info_out, EpisodeState* __restrict__ ep,
                                 cudaGraphConditionalHandle handle) {
  episode_advance_body<R, true>(B, T, N, M, m_ref, n_steps, traj, best_u, best_costs, info, w, state, warm, xs, us,
                                costs, info_out, ep, handle);
}

// Launchers (ilqr.cu), instantiated for float and double; 0 or MPCB200_ERR_LAUNCH.
template <typename R>
int ilqr_launch_init(size_t n_u, const R* u_init, R* u, IlqrState* st, int32_t* info,
                     cudaGraphConditionalHandle handle, cudaStream_t stream);
template <typename R>
int episode_launch_init(size_t n_x, size_t n_u, const R* x_init, const R* u_init, R* state, R* xs0, R* warm,
                        EpisodeState* ep, cudaGraphConditionalHandle handle, cudaStream_t stream);
// w NULL: episode_advance_kernel; otherwise its disturbed form
template <typename R>
int episode_launch_advance(int B, int T, int N, int M, int m_ref, int n_steps, const R* traj, const R* best_u,
                           const R* best_costs, const int32_t* info, const R* w, R* state, R* warm, R* xs, R* us,
                           R* costs, int32_t* info_out, EpisodeState* ep, cudaGraphConditionalHandle handle,
                           cudaStream_t stream);
template <typename R>
int ilqr_launch_track(int B, int T, int N, int M, int m_ref, R best_cost_eps, const R* new_x, const R* new_u,
                      const R* costs, const R* du_first, const int32_t* status, const R* best_costs, R* best_x,
                      R* best_u, R* u, R* fdn, uint8_t* flags, const IlqrState* st, cudaStream_t stream);
template <typename R>
int ilqr_launch_stop(int B, int lqr_iter, int not_improved_lim, double eps, const R* costs, const R* fdn,
                     const uint8_t* flags, R* best_costs, R* best_fdn, IlqrState* st, int32_t* info,
                     cudaGraphConditionalHandle handle, cudaStream_t stream);

}  // namespace mpcb200
