// mlp.cuh - a learned model's network (mpc.dynamics.NNDynamics: x' = [x +] MLP([x; u])) in the kernels: the rollout,
// the exact Jacobians and the line search of the LQR step's split mode (mlp.cu).  The step kernels are not involved:
// the step runs with do_rollout = 0 and these kernels read its gains.
//
// Work split: one warp per problem (rollout, line search) or per (t, b) (linearisation); every CTA stages the packed
// weights and biases of the network (mpcb200_mlp.params) into shared memory once, then runs its warps' items
// grid-stride.  Each warp owns a slice of shared memory for its activations.  Every sum runs in an order fixed by
// the network's widths alone, so a problem's outputs do not depend on the batch size or its position in the batch,
// and nothing is accumulated with atomics.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "../../../include/mpcb200.h"

namespace mpcb200 {

// Sizes the three kernels agree on, derived from the record alone (host and device).  Elements, not bytes.
struct MlpShape {
  int L, act, passthrough, n_prev, ns, ms, maxw;
  int w[MPCB200_MLP_MAX_LAYERS + 1];
  long long W_off[MPCB200_MLP_MAX_LAYERS], b_off[MPCB200_MLP_MAX_LAYERS];
  long long n_params;     // elements of the parameter block the kernels stage: [0, n_params) of mlp.params
  int per_warp;           // elements of one warp's shared-memory slice (a multiple of 16 bytes for f32 and f64)
  int p_max;              // largest staged N + M the calls take
};

int max_smem_optin();    // api.cu

// false for a malformed record (layer count, widths, activation, n_prev, offsets)
bool mlp_shape(const mpcb200_mlp* rec, MlpShape& s);
// dynamic shared memory of a CTA of `warps` warps, in bytes
size_t mlp_smem_bytes(const MlpShape& s, int elem_size, int warps);

// the line search of the split-mode step (mpcb200_mlp_step_*): the arguments of mlp_linesearch_kernel
template <typename R>
struct MlpLsArgs {
  int B, T, N, M, bounds_kind, has_mask, has_delta, max_ls;
  long long C_ts, c_ts;
  R u_lo, u_hi, delta_u, decay;
  const R *C, *c, *x_init, *cur_x, *cur_u, *Ks, *ks, *u_lower, *u_upper;
  const uint8_t* zero_mask;
  R *new_x, *new_u, *costs, *alphas, *du_first;
};

// Launchers (mlp.cu), instantiated for float and double; 0 or an MPCB200_ERR_* code.  N, M: the staged sizes.
template <typename R>
int mlp_launch_rollout(const mpcb200_mlp* rec, int B, int T, int N, int M, const R* x_init, const R* u, R* x,
                       cudaStream_t stream);
template <typename R>
int mlp_launch_linearize(const mpcb200_mlp* rec, int B, int T, int N, int M, const R* x, const R* u, R* F, R* f,
                         cudaStream_t stream);
template <typename R>
int mlp_launch_linesearch(const mpcb200_mlp* rec, const MlpLsArgs<R>& a, cudaStream_t stream);

// The linearisation's VJP in the parameters (mpcb200_mlp_linearize_vjp_*): one warp per item (t, b) computes
// d/dtheta [<G^, J> + <df, y>], G^ = dJ - df z^T, by reverse over forward with matrix tangents T_i = dh_i/dz.  Its
// per-warp slice holds z, the hidden outputs, T_1 .. T_{L-1} [w_i, w_0], two adjoint buffers [maxw, w_0] and two
// [maxw] (mlp_vjp_shape).  The items are dealt to G slots (mlp_vjp_slots, a function of the item and parameter
// counts alone): slot g sums items g, g + G, ... in increasing order into row g of a [G, n_params] workspace, and a
// second kernel adds the G rows in slot order into dtheta, so dtheta is bitwise the same for any grid.
constexpr long long kMlpVjpSlotElems = 1ll << 23;   // G * n_params stays at or below this (or G = 1)
constexpr int kMlpVjpMaxSlots = 2048;
constexpr int kMlpVjpMaxCtas = 128;                 // CTAs of the VJP kernel; a warp serves every (warps)-th slot
// s with per_warp set to the VJP kernel's slice
MlpShape mlp_vjp_shape(const MlpShape& s);
// G = max(1, min(items, kMlpVjpMaxSlots, max(1, kMlpVjpSlotElems / n_params)))
int mlp_vjp_slots(long long items, long long n_params);
// ws: G * n_params elements
template <typename R>
int mlp_launch_linearize_vjp(const mpcb200_mlp* rec, int B, int T, int N, int M, const R* x, const R* u, const R* dF,
                             const R* df, R* dtheta, R* ws, cudaStream_t stream);

}  // namespace mpcb200
