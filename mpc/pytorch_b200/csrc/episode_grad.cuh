// episode_grad.cuh - the reverse sweep of a receding-horizon episode (mpcb200_episode_backward_*): the closed loop's
// chain rule over control steps k = n_steps-1 .. 0, as one CUDA graph with a conditional `while` node.
//
// Forward (mpcb200_episode_plans_*): episode_plans_kernel keeps each solve's best iterate, plan_x[k], plan_u[k].
// Backward, with g = dL/dx_{k+1} carried in dx_init:
//   a. epgrad_stage_*_kernel: plan_x[k], plan_u[k] into fixed buffers; the model step's VJP at (x_k, u_k):
//      gx = R^T g, dl_du[0] = dl_dus[k] + S^T g (rows t > 0 stay 0), and the parameter part (LinDx: dF[0] += g z^T,
//      df[0] += g; a known system: theta_step = g . dx'/dtheta with the Jacobian held constant, the VJP's `first`);
//   b. a known system's linearisation along the staged plan, c. the KKT adjoint on the staged plan, d. a known
//      system's linearisation VJP (first + second) - the library's own launchers, recorded on the body stream;
//   e. epgrad_accum_kernel: g = dl_dxs[k] + gx + dx_init_k, and the adjoint's dC, dc (dF, df; theta) summed in.
// Every buffer a body kernel reads is written by an earlier kernel of the same iteration or by epgrad_init_kernel,
// so the body holds kernel nodes only.
// A slew-rate episode (mpcb200_episode_backward_slew_*) runs the same sweep on its augmented problem over
// [u_{k-1}; x_k] (LinDx, or a known system's passthrough kind) with the previous control detached, as the reference
// detaches prev_ctrl: the *_detach_kernel forms of init and accumulate set g's first n_prev entries to 0, so no
// gradient flows into them and the passthrough row of the model step carries nothing back.
// An episode closed on a plant other than the model, x_{k+1} = plant(x_k, u_k) + w_k
// (mpcb200_episode_backward_plant_*): step a. runs on the plant (its kind, dp, F; its dF, df, theta_step), and the
// *_plant_kernel forms of init and accumulate zero and sum the plant's own accumulators, keep theta_step out of the
// model's dtheta, and write dw[k] = g.  They apply the detach rule too, with n_prev = 0 meaning none.
// A time-varying episode (mpcb200_episode_backward_window_*): window_stage_kernel stages step k's window first, and
// the *_window_kernel forms zero the full-length outputs and add each step's gradients at offset k (EpWindow).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "dynamics.cuh"
#include "ilqr.cuh"

namespace mpcb200 {

struct EpGradState {      // device-resident sweep state, reset by epgrad_init_kernel
  int32_t k;              // the control step the body works on
  uint32_t tickets;       // blocks of the current epgrad_accum_kernel that have finished
  int32_t reserved[2];
};

template <typename R>
struct EpGradArgs {
  int B, T, N, M, n_steps, F_T, has_f, kind, NP;
  DynParams dp;
  const R *xs, *us, *plan_x, *plan_u, *dl_dxs, *dl_dus;
  const R* F;             // LinDx: slice 0 of the staged F, [B, N, N+M]
  R *stage_x, *stage_u;   // [T, B, N], [T, B, M]: the plan of step k
  R *dl_dx, *dl_du;       // the adjoint's incoming gradients [T, B, N] (0), [T, B, M] (row 0 written per step)
  R *gx, *theta_step;     // R^T g [B, N]; the model step's parameter part [B, NP]
  R* g;                   // dL/dx_{k+1}; dL/dx_init after the loop (the caller's dx_init)
  const R *dx_k, *dC_k, *dc_k, *dF_k, *df_k, *first, *second;     // the adjoint's (and VJP's) outputs of step k
  R *dC, *dc, *dF, *df, *dtheta;
  EpGradState* st;
};

// The plant's side of a sweep (mpcb200_episode_backward_plant_*): the stage kernel runs on a copy of EpGradArgs with
// the plant's kind, dp, F, dF, df and theta_step, and the *_plant_kernel forms of init and accumulate read this.
template <typename R>
struct EpPlantArgs {
  int kind, has_f, NP;    // the plant's kind, whether its f is given, its parameter count (0 for LinDx)
  const R* theta_step;    // the stage's parameter part [B, NP] (the plant's)
  R *dF, *df;             // LinDx plant: slice 0 of its dF [B, N, N+M], df [B, N] (the stage adds g z^T, g)
  R* dtheta;              // known plant: [B, NP], sum over k of theta_step
  R* dw;                  // dL/dw [n_steps, B, N] (dw[k] = dL/dx_{k+1}), or NULL
};

// A time-varying episode (mpcb200_episode_window_*, mpcb200_episode_backward_window_*): window_stage_kernel, the
// first node of each control step's body (forward and sweep), copies slices k .. k+n-1 of each windowed input into
// the fixed buffers the body's nodes were recorded with, k read from the device-resident step counter (EpisodeState
// step, EpGradState k).  One grid-stride loop per input.  tstride: elements between the source's slices, < 0 for a
// time-invariant source (every slice reads its one slice).
constexpr int WINDOW_INPUTS = 8;      // C, c, F, f, u_lower, u_upper, F_plant, f_plant
template <typename R>
struct WindowCopy {
  const R* src[WINDOW_INPUTS];        // NULL: not windowed
  R* dst[WINDOW_INPUTS];
  long long tstride[WINDOW_INPUTS];
  long long slice[WINDOW_INPUTS];     // elements per slice
  int n[WINDOW_INPUTS];               // slices copied
  const int32_t* k;
};

// The sweep's window (the *_window_kernel forms of init, stage and accumulate): which outputs are full length, and
// their slice counts.  Solve k's dC_k, dc_k (cost) and dF_k, df_k (dyn) go in at offset k; the stage's g z^T and g
// go into slice k of the stepping LinDx's dF, df (step).
struct EpWindow {
  int cost, dyn, step;    // dC, dc on the axis; the model's dF, df; the stepping LinDx's dF, df (plant or model)
  int L, LF, Lf, Lp;      // slices of dC / dc, of the model's dF, of its df, of the plant's dF / df
};

// Launchers (episode_grad.cu), instantiated for float and double; 0 or MPCB200_ERR_LAUNCH.
template <typename R>
int window_launch_stage(const WindowCopy<R>& w, cudaStream_t stream);
// the *_window_kernel forms of init and accumulate (the plant forms when pl is non-NULL); n_prev as below
template <typename R>
int epgrad_launch_init_window(const EpGradArgs<R>& a, int n_prev, const EpPlantArgs<R>* pl, const EpWindow& wn,
                              cudaGraphConditionalHandle handle, cudaStream_t stream);
template <typename R>
int epgrad_launch_accum_window(const EpGradArgs<R>& a, int n_prev, const EpPlantArgs<R>* pl, const EpWindow& wn,
                               cudaGraphConditionalHandle handle, cudaStream_t stream);
// epgrad_launch_stage, with a LinDx step's parameter part added into slice k of its dF, df when wn.step
template <typename R>
int epgrad_launch_stage_window(const EpGradArgs<R>& a, const EpWindow& wn, cudaStream_t stream);
template <typename R>
int episode_launch_plans(int B, int T, int N, int M, const R* best_x, const R* best_u, R* plan_x, R* plan_u,
                         const EpisodeState* ep, cudaStream_t stream);
// n_prev > 0 (a slew-rate episode, mpcb200_episode_backward_slew_*): the detach rule, g[:, :n_prev] = 0.
// pl non-NULL (mpcb200_episode_backward_plant_*): the plant forms, which also take n_prev = 0
template <typename R>
int epgrad_launch_init(const EpGradArgs<R>& a, int n_prev, const EpPlantArgs<R>* pl, cudaGraphConditionalHandle handle,
                       cudaStream_t stream);
template <typename R>
int epgrad_launch_stage(const EpGradArgs<R>& a, cudaStream_t stream);
template <typename R>
int epgrad_launch_accum(const EpGradArgs<R>& a, int n_prev, const EpPlantArgs<R>* pl,
                        cudaGraphConditionalHandle handle, cudaStream_t stream);
template <typename R>
int epgrad_launch_vjp_passthrough(const DynVjpArgs& a, cudaStream_t stream);
template <typename R>
int launch_fill_zero(size_t n, R* p, cudaStream_t stream);

// An episode planned with a learned model (mpcb200_episode_backward_mlp_*).  Its parameters are the network's packed
// weights, shared by every problem, so the per-problem parameter part of init and accumulate does not apply: the
// sweep runs them with kind EPGRAD_KIND_NET and NP = 0 (and a plant record of that kind when the network itself
// steps a disturbed loop), and they do everything else (g, dC, dc, dw, the plant's accumulators, the loop counter).
// Body, no plant: plan -> the network's linearisation along the staged plan (Fk) -> stage_net (the model step's VJP
// in x_k, u_k from slice 0 of Fk) -> adjoint -> net_step_param (g z_0^T, g into the adjoint's dF_k[0], df_k[0]) ->
// the linearisation VJP into dtheta_k -> add (dtheta += dtheta_k) -> accumulate.  With a plant, the plant's stage
// replaces plan and stage_net, and net_step_param is not run.
constexpr int EPGRAD_KIND_NET = -1;
// stage_x, stage_u = plan_x[k], plan_u[k]
template <typename R>
int epgrad_launch_plan(const EpGradArgs<R>& a, cudaStream_t stream);
// gx = R^T g, dl_du[0] = dl_dus[k] + S^T g with [R S] = a.F, slice 0 of the network's linearisation
template <typename R>
int epgrad_launch_stage_net(const EpGradArgs<R>& a, cudaStream_t stream);
// dF_k[0] += g [x_k; u_k]^T, df_k[0] += g
template <typename R>
int epgrad_launch_net_step_param(const EpGradArgs<R>& a, R* dF_k, R* df_k, cudaStream_t stream);
// dst[i] += src[i], i < n
template <typename R>
int epgrad_launch_add(size_t n, const R* src, R* dst, cudaStream_t stream);

}  // namespace mpcb200
