/*
 * mpcb200.h - C ABI of the H100-native batched box-constrained LQR step.
 *
 * This is the drop-in boundary for ONE path of locuslab/mpc.pytorch: the body of
 * LQRStepFn.forward / LQRStepFn.backward (reference mpc/lqr_step.py:277-309 and
 * :312-407).  The reference has no FFI of its own (it is pure Python on top of
 * ATen); these entry points are what a binding for that path would call.  The
 * Python host side (mpc/pytorch_b200/) mirrors the reference's LQRStep / MPC
 * signatures on top of this ABI through ctypes; see INTEGRATION.md.
 *
 * Conventions
 *  - plain pointers and sizes only; no torch types, no exceptions, no prints.
 *  - every pointer is a DEVICE pointer on the current device; all tensors are
 *    dense, row-major, time-major / batch-second exactly like the reference:
 *      C[T,B,p,p]  c[T,B,p]  F[F_T,B,n,p] (F_T = T-1 or T)  f[T-1,B,n] or NULL
 *      x_init[B,n] cur_x[T,B,n] cur_u[T,B,m]  (p = n+m)
 *  - the caller owns every buffer; the library allocates nothing, frees nothing
 *    and never writes an input.  Calls are asynchronous on `stream`, re-entrant,
 *    and keep no global state besides a launch counter and, per host thread, the
 *    plan of the last step launch (mpcb200_last_step_plan).
 *  - return value: 0 on success, MPCB200_ERR_* otherwise (mpcb200_strerror()).
 *  - optional outputs may be NULL.
 */
#ifndef MPCB200_H_
#define MPCB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MPCB200_VERSION 2

enum {
  MPCB200_OK = 0,
  MPCB200_ERR_NULL_POINTER = 1,      /* a required pointer is NULL                          */
  MPCB200_ERR_BAD_DIMS = 2,          /* B,T,n,m <= 0, F_T not in {T-1,T}, bad option combo  */
  MPCB200_ERR_UNSUPPORTED_DIMS = 3,  /* (n,m) has no compiled kernel instance               */
  MPCB200_ERR_SMEM = 4,              /* problem does not fit shared memory and no workspace */
  MPCB200_ERR_LAUNCH = 5,            /* cudaGetLastError() after launch != cudaSuccess      */
  MPCB200_ERR_NO_DEVICE = 6,         /* no usable sm_90 device / wrong architecture         */
  MPCB200_ERR_NO_GRAPH_COND = 7      /* conditional graph nodes unavailable (driver < 12.3)  */
};

/* Problem sizes and options.  Mirrors the closure arguments of
 * LQRStep(...) (reference mpc/lqr_step.py:22-38). */
typedef struct mpcb200_dims {
  int32_t B;              /* n_batch                                                   */
  int32_t T;              /* horizon                                                   */
  int32_t n;              /* n_state                                                   */
  int32_t m;              /* n_ctrl                                                    */
  int32_t F_T;            /* time slices present in F: T-1 or T (only F[:T-1] is read) */
  int32_t has_f;          /* f given ([T-1,B,n]); 0 = reference's "empty tensor"       */
  int32_t bounds_kind;    /* 0 none, 1 scalar (params.u_lo/u_hi), 2 tensors [T,B,m]    */
  int32_t has_zero_mask;  /* u_zero_I given: uint8 [T,B,m], nonzero = forced-zero ctrl */
  int32_t has_delta_u;    /* trust region |du| <= params.delta_u (needs bounds)        */
  int32_t max_ls_iter;    /* max_linesearch_iter (>=1)                                 */
  int32_t pnqp_max_iter;  /* projected-Newton iteration cap (reference: 20)            */
  int32_t do_rollout;     /* 1: Riccati sweep + line-search rollout (LinDx/QuadCost)
                             0: Riccati sweep only; Ks/ks must be given                */
  int32_t dynamics_kind;  /* true dynamics of the rollout (reference lqr_step.py:217-225):
                             MPCB200_DYN_LINEAR = LinDx(F,f); MPCB200_DYN_CARTPOLE / _PENDULUM /
                             _PENDULUM_FULL = the step
                             function of that system evaluated inside the kernel (params.dyn); F,f are
                             then its linearisation and are used by the Riccati sweep only (ABI v2);
                             OR'd with MPCB200_DYN_CTRL_PASSTHROUGH: that system under a slew-rate penalty */
  int32_t reserved0;      /* 0 (keeps the 64-bit fields below naturally aligned)              */
  /* Elements between consecutive TIME slices of C, c, F, f (ABI v2).  0: dense ([T,B,...] contiguous; what a
   * zero-initialised struct means).  > 0: that many elements.  MPCB200_TIME_INVARIANT (-1): one [B,...] slice
   * reused for every t (a torch stride of 0), which is what the reference's
   * `C.unsqueeze(0).expand(T, ...)` hands over (mpc/mpc.py:205-226) and what an LTI system is; the slice is
   * read from HBM / copied from the host once instead of T times.  The batch dimension stays dense. */
  int64_t C_tstride, c_tstride, F_tstride, f_tstride;
} mpcb200_dims;

typedef struct mpcb200_params {
  double u_lo, u_hi;      /* scalar bounds (bounds_kind == 1)   */
  double delta_u;         /* has_delta_u                        */
  double ls_decay;        /* linesearch_decay                   */
  double dyn[8];          /* parameters of a known system (dims.dynamics_kind != 0), see mpcb200_dyn_* (ABI v2) */
} mpcb200_params;

/* Known nonlinear systems (reference mpc/env_dx/cartpole.py:63-96, mpc/env_dx/pendulum.py:49-84).
 * dyn[] = cartpole: gravity, masscart, masspole, length, force_mag, dt   (state x,dx,cos th,sin th,dth; n=5, m=1)
 *         pendulum: g, m, l, (unused), max_torque, dt                    (state cos th,sin th,dth; n=3, m=1)
 *         pendulum_full: g, m, l, d, b, max_torque, dt                   (state cos th,sin th,dth; n=3, m=1)
 * PENDULUM is the reference's PendulumDx(simple=True); PENDULUM_FULL is PendulumDx(simple=False), with damping d on
 * the wrapped angle atan2(sin th, cos th) and gravity bias b inside sin(th + b), as the reference writes them.  The
 * step of PENDULUM_FULL runs on a dynamics-only kernel instance at (3, 1).
 * MPCB200_DYN_CTRL_PASSTHROUGH, OR'd into any of the three: the slew-rate augmented system of the reference's
 * CtrlPassthroughDynamics (mpc/dynamics.py:133-156).  State [u_{t-1}; x] (n = n_system + 1, m = 1), step
 * [u; step(x, u)] with u the control before the system's own clamp; its linearisation is F = [[0, 0, I], [0, R, S]],
 * f = [0; f_system].  Same dyn[] as the system.  Accepted by every call that takes a kind, at exactly that (n, m);
 * the step runs a dynamics-only kernel instance, which mpcb200_supported / _supported_list do not list. */
enum {
  MPCB200_DYN_LINEAR = 0, MPCB200_DYN_CARTPOLE = 1, MPCB200_DYN_PENDULUM = 2, MPCB200_DYN_PENDULUM_FULL = 4,
  MPCB200_DYN_CTRL_PASSTHROUGH = 16
};
#define MPCB200_TIME_INVARIANT (-1)

/* Per-problem status bits written to `status[B]`. */
#define MPCB200_ST_PNQP_UNCONVERGED 1u /* some time step hit pnqp_max_iter (reference prints a warning, pnqp.py:81) */
#define MPCB200_ST_NONFINITE 2u        /* final cost is not finite                                              */
#define MPCB200_ST_BAD_PIVOT 4u        /* an LDL^T pivot of the free block was <= 0 (Quu not positive definite) */

/*
 * One LQR step: replaces LQRStepFn.forward (reference mpc/lqr_step.py:277-309):
 *   c_back = C*tau_bar + c; lqr_backward (:52-160) incl. pnqp (mpc/pnqp.py:5-82);
 *   lqr_forward rollout + line search (:164-261) with true model QuadCost(C,c)/LinDx(F,f).
 *
 * Outputs: new_x[T,B,n] new_u[T,B,m] costs[B] full_du_norm[B] alphas[B]
 *          (mean_alphas of the reference is mean(alphas); reduced by the caller)
 * Optional outputs (NULL to skip):
 *   du_first[T,B,m]  cur_u - new_u of the FIRST (alpha = 1) rollout pass, i.e. the vector whose
 *                  per-problem 2-norm is full_du_norm.  (The reference computes its
 *                  full_du_norm from a [T,m,B]-ordered buffer viewed as [B,T*m]
 *                  (lqr_step.py:244-245), which mixes batch elements when B > 1; the
 *                  Python host side reproduces that from du_first, this ABI returns the
 *                  per-problem norm.)
 *   qp_iters[T,B]  int32  pnqp iterations "i" per (t,b); the reference's
 *                  n_total_qp_iter is sum_t (1 + max_b qp_iters[t,b])   (lqr_step.py:140)
 *   free_mask[T,B,m] uint8  pnqp free set If (1 = free) / complement of u_zero_I
 *   status[B]      int32  MPCB200_ST_* bits
 *   Ks[T,B,m,n] ks[T,B,m]  feedback gains in FORWARD time order
 * pnqp semantics are per problem (what the reference computes for n_batch=1).
 */
int mpcb200_lqr_step_f32(const mpcb200_dims* dims, const mpcb200_params* params,
                         const float* C, const float* c, const float* F, const float* f,
                         const float* x_init, const float* cur_x, const float* cur_u,
                         const float* u_lower, const float* u_upper, const uint8_t* u_zero_I,
                         float* new_x, float* new_u, float* costs, float* full_du_norm,
                         float* alphas, float* du_first, int32_t* qp_iters, uint8_t* free_mask, int32_t* status,
                         float* Ks, float* ks, void* stream);

int mpcb200_lqr_step_f64(const mpcb200_dims* dims, const mpcb200_params* params,
                         const double* C, const double* c, const double* F, const double* f,
                         const double* x_init, const double* cur_x, const double* cur_u,
                         const double* u_lower, const double* u_upper, const uint8_t* u_zero_I,
                         double* new_x, double* new_u, double* costs, double* full_du_norm,
                         double* alphas, double* du_first, int32_t* qp_iters, uint8_t* free_mask, int32_t* status,
                         double* Ks, double* ks, void* stream);

/*
 * Gradient assembly of the KKT adjoint: replaces the second half of
 * LQRStepFn.backward (reference mpc/lqr_step.py:342-404).  The caller first runs
 * mpcb200_lqr_step_* with (c = -[dl_dx;dl_du], f = NULL, x_init = 0, cur_x = cur_u = 0,
 * u_zero_I = active set, no bounds) to obtain (dx,du) (reference :328-340), then:
 *   dC[t] = -0.5 (dtau tau' + tau dtau'), dc = -dtau,
 *   lambda / dlambda costate recursions, dF[t] = -(dlam_{t+1} tau_t' + lam_{t+1} dtau_t'),
 *   df = -dlam[1:], dx_init = -dlam[0].
 * r = [dl_dx; dl_du] enters only through r_x.  dF has F_T slices (slice T-1, if present, is zeroed).
 * df may be NULL (reference returns an empty tensor when f is empty).
 * workspace: required device buffer of 2*T*B*n elements (lambda_t, dlambda_t; MPCB200_ERR_NULL_POINTER
 * without it).  The call runs as two kernels: sequential costates, then fully parallel outer products.
 */
int mpcb200_lqr_grad_f32(const mpcb200_dims* dims,
                         const float* C, const float* c, const float* F,
                         const float* new_x, const float* new_u,
                         const float* dx, const float* du, const float* dl_dx,
                         float* dx_init, float* dC, float* dc, float* dF, float* df,
                         void* workspace, void* stream);

int mpcb200_lqr_grad_f64(const mpcb200_dims* dims,
                         const double* C, const double* c, const double* F,
                         const double* new_x, const double* new_u,
                         const double* dx, const double* du, const double* dl_dx,
                         double* dx_init, double* dC, double* dc, double* dF, double* df,
                         void* workspace, void* stream);

/*
 * The whole KKT-adjoint backward in ONE call: replaces LQRStepFn.backward (reference mpc/lqr_step.py:312-407).
 * Given the solution (new_x, new_u) of the forward solve and the upstream gradients dl_dx[T,B,n], dl_du[T,B,m]:
 *   1. prep kernel: r = -[dl_dx; dl_du]; active set I = (|u* - u_lower| <= 1e-8) | (|u* - u_upper| <= 1e-8)
 *      from the box (dims->bounds_kind / params->u_lo,u_hi / u_lower,u_upper), reference :316-326;
 *   2. the masked LQR step from the zero trajectory (c = r, x_init = 0, u_zero_I = I, default line search),
 *      i.e. the nested MPC(lqr_iter=1) of :328-340, with the step kernel;
 *   3. costates and outer products (mpcb200_lqr_grad_*, :342-404).
 * The library picks the kernels.  The nested step keeps its gains in the workspace at the horizons and shapes where
 * mpcb200_step_prefers_workspace says a step does, so every horizon a step with Ks/ks takes works here too.  Where it
 * does not, and the column-pair kernel takes the shape, alignment and horizon, steps 2 and 3 run as one fused kernel
 * (2 launches in all); otherwise the masked step kernel and the two gradient kernels run (4 launches).
 * Outputs dx_init[B,n] dC[T,B,p,p] dc[T,B,p] dF[F_T,B,n,p] df[T-1,B,n] (df only if dims->has_f; F and dF may be
 * NULL when T = 1 and F_T = 0).
 * workspace: device buffer of mpcb200_adjoint_workspace_bytes(dims, elem_size) bytes (scratch; contents
 * undefined on return).  The size includes the nested step's Ks/ks where that step keeps its gains in a buffer.
 * Only dims->{B,T,n,m,F_T,has_f,bounds_kind}, the time strides of C, c and F, and params->{u_lo,u_hi} are read.
 */
size_t mpcb200_adjoint_workspace_bytes(const mpcb200_dims* dims, int32_t elem_size);
int mpcb200_lqr_adjoint_f32(const mpcb200_dims* dims, const mpcb200_params* params,
                            const float* C, const float* c, const float* F,
                            const float* new_x, const float* new_u, const float* dl_dx, const float* dl_du,
                            const float* u_lower, const float* u_upper,
                            float* dx_init, float* dC, float* dc, float* dF, float* df,
                            void* workspace, size_t workspace_bytes, void* stream);
int mpcb200_lqr_adjoint_f64(const mpcb200_dims* dims, const mpcb200_params* params,
                            const double* C, const double* c, const double* F,
                            const double* new_x, const double* new_u, const double* dl_dx, const double* dl_du,
                            const double* u_lower, const double* u_upper,
                            double* dx_init, double* dC, double* dc, double* dF, double* df,
                            void* workspace, size_t workspace_bytes, void* stream);

/*
 * Nominal trajectory under LinDx dynamics: replaces util.get_traj for LinDx (reference
 * mpc/util.py:102-126, called once per iLQR iteration at mpc/mpc.py:251):
 *   x[0] = x_init;  x[t+1] = F[t] [x[t]; u[t]] + f[t]   (f may be NULL; dims->has_f)
 * x[T,B,n] is written; only dims->{B,T,n,m,F_T,has_f} are read.
 */
int mpcb200_rollout_f32(const mpcb200_dims* dims, const float* F, const float* f, const float* x_init,
                        const float* u, float* x, void* stream);
int mpcb200_rollout_f64(const mpcb200_dims* dims, const double* F, const double* f, const double* x_init,
                        const double* u, double* x, void* stream);

/*
 * Known nonlinear dynamics on the device (SURVEY.md section 8(f) rank 2).
 *   mpcb200_dyn_rollout_*:   x[0] = x_init, x[t+1] = step(x[t], u[t])  - util.get_traj for a Module
 *                            (reference mpc/util.py:102-126 with dynamics(x,u), one Python call per step).
 *   mpcb200_dyn_linearize_*: F[t,b] = [d step/dx, d step/du], f[t,b] = step(x,u) - F [x;u] at (x[t,b], u[t,b]),
 *                            t < T-1 - linearize_dynamics (reference mpc/mpc.py:490-601; its AUTO_DIFF mode does
 *                            (T-1)*n_state autograd passes).  Exact Jacobians by forward-mode dual numbers.
 * kind = MPCB200_DYN_CARTPOLE | MPCB200_DYN_PENDULUM | MPCB200_DYN_PENDULUM_FULL, optionally
 * | MPCB200_DYN_CTRL_PASSTHROUGH; dyn = HOST pointer
 * to 8 doubles (see mpcb200_params.dyn); x_init[B,n] u[T,B,m] x[T,B,n] F[T-1,B,n,n+m] f[T-1,B,n]; n, m are those of
 * the kind (n_system + 1 states with the passthrough).
 */
int mpcb200_dyn_rollout_f32(int32_t kind, const double* dyn, int32_t B, int32_t T, const float* x_init,
                            const float* u, float* x, void* stream);
int mpcb200_dyn_rollout_f64(int32_t kind, const double* dyn, int32_t B, int32_t T, const double* x_init,
                            const double* u, double* x, void* stream);
int mpcb200_dyn_linearize_f32(int32_t kind, const double* dyn, int32_t B, int32_t T, const float* x,
                              const float* u, float* F, float* f, void* stream);
int mpcb200_dyn_linearize_f64(int32_t kind, const double* dyn, int32_t B, int32_t T, const double* x,
                              const double* u, double* F, double* f, void* stream);

/*
 * Vector-Jacobian product of mpcb200_dyn_linearize_* in the system's learnable parameters theta: cartpole dyn[0..3]
 * (gravity, masscart, masspole, length), pendulum dyn[0..2] (g, m, l), pendulum_full dyn[0..4] (g, m, l, d, b);
 * force_mag / max_torque and dt are constants.
 * For t < T-1, with z = [x; u], J = [d step/dx, d step/du] and f = step(x, u) - J z at (x[t,b], u[t,b]):
 *   first[t,b,k]  = sum_r df[t,b,r] d step_r/dtheta_k
 *   second[t,b,k] = sum_{r,j} (dF[t,b,r,j] - df[t,b,r] z_j) dJ_rj/dtheta_k
 * so first + second, summed over (t, b), is the gradient of <dF, F> + <df, f> in theta; `first` alone is that gradient
 * with J held constant.  A control beyond the clamp contributes no u column (the clamp's derivative is 0 there).
 * kind = MPCB200_DYN_CARTPOLE, MPCB200_DYN_PENDULUM or MPCB200_DYN_PENDULUM_FULL (a passthrough kind is
 * MPCB200_ERR_BAD_DIMS); dyn = HOST pointer to 8 doubles; x[T,B,n] u[T,B,1] dF[T-1,B,n,n+1] df[T-1,B,n]; first,
 * second [T-1,B,NP] (NP = 4 cartpole, 3 pendulum, 5 pendulum_full), either may be NULL.  One kernel; nothing is
 * launched when T = 1 or both outputs are NULL.
 */
int mpcb200_dyn_linearize_vjp_f32(int32_t kind, const double* dyn, int32_t B, int32_t T, const float* x,
                                  const float* u, const float* dF, const float* df, float* first, float* second,
                                  void* stream);
int mpcb200_dyn_linearize_vjp_f64(int32_t kind, const double* dyn, int32_t B, int32_t T, const double* x,
                                  const double* u, const double* dF, const double* df, double* first, double* second,
                                  void* stream);

/*
 * Standalone projected-Newton box QP, n <= mpcb200_pnqp_max_n(elem_size): replaces
 * pnqp(H,q,lower,upper,x_init,n_iter) of the reference (mpc/pnqp.py:5-82) for batches of QPs
 * min 0.5 x'Hx + q'x, lower <= x <= upper.
 * H[B,n,n] q,lower,upper[B,n]; x_init[B,n] or NULL (cold start -H^{-1}q).  Outputs x[B,n],
 * H_free[B,n,n] (the masked matrix H_ of the returning iteration, whose LU the reference returns),
 * If[B,n] uint8 free set, iters[B] (the reference's `i`), status[B] optional (MPCB200_ST_* bits).
 * Per-problem control flow (what the reference computes for n_batch = 1).  H must be symmetric: the
 * Newton systems are solved by LDL^T of the lower triangle of H_.  n <= 8 runs one thread per QP,
 * larger n one thread block per QP with the QP in shared memory; n > mpcb200_pnqp_max_n returns
 * MPCB200_ERR_SMEM.
 */
int mpcb200_pnqp_f32(int32_t B, int32_t n, const float* H, const float* q, const float* lower,
                     const float* upper, const float* x_init, int32_t n_iter, float* x, float* H_free,
                     uint8_t* If, int32_t* iters, int32_t* status, void* stream);
int mpcb200_pnqp_f64(int32_t B, int32_t n, const double* H, const double* q, const double* lower,
                     const double* upper, const double* x_init, int32_t n_iter, double* x, double* H_free,
                     uint8_t* If, int32_t* iters, int32_t* status, void* stream);

/* Largest n mpcb200_pnqp_* solves for elem_size 4 (f32) or 8 (f64), from the current device's opt-in shared
 * memory per block (227 KB, the H100's, when no device is visible); 0 for any other elem_size. */
int32_t mpcb200_pnqp_max_n(int32_t elem_size);

/*
 * Implicit gradient of a standalone pnqp solution, for a loss L(x).  Inputs: H[B,n,n] and lower,upper[B,n] of the
 * solved QPs, the solution x[B,n] and free set If[B,n] (uint8, 1 = free) that mpcb200_pnqp_* returned, and
 * dl_dx[B,n].  With F the free set and A the rest (clamped, x_i exactly at lower_i or upper_i), v solves
 * (H_FF + 1e-11 I) v = dl_dx_F, the regularised block the forward factors; then
 *   dq[B,n]:     -v on F, 0 on A;
 *   dH[B,n,n]:   row i = -v_i x^T for i in F, 0 on the rows of A (unsymmetrised: autograd of g = Hx + q);
 *   dlower, dupper[B,n]: on i in A, dl_dx_i - sum_{k in F} H_ki v_k goes to dlower_i when x_i == lower_i, else to
 *                dupper_i; every other entry is 0.
 * This is the reference's unrolled autograd (mpc/pnqp.py:5-82) on a problem whose last accepted Newton step was a
 * full step with the final free set; on an unconverged problem it is the same formula at the returned point, not the
 * derivative of the iterations.  x_init gets no gradient.  status[B] optional: MPCB200_ST_BAD_PIVOT when a pivot of
 * the free block is <= 0 or not finite, else 0.  H must be symmetric (LDL^T of the lower triangle).  n <= 8 runs one
 * thread per QP, larger n one thread block per QP; n > mpcb200_pnqp_max_n returns MPCB200_ERR_SMEM before any device
 * is needed.  Every output element is written, without atomics: the result is the same bits on every call.
 */
int mpcb200_pnqp_backward_f32(int32_t B, int32_t n, const float* H, const float* x, const uint8_t* If,
                              const float* lower, const float* upper, const float* dl_dx, float* dH, float* dq,
                              float* dlower, float* dupper, int32_t* status, void* stream);
int mpcb200_pnqp_backward_f64(int32_t B, int32_t n, const double* H, const double* x, const uint8_t* If,
                              const double* lower, const double* upper, const double* dl_dx, double* dH, double* dq,
                              double* dlower, double* dupper, int32_t* status, void* stream);

/*
 * Shapes without a compiled instance.  The step, the gradient assembly, the rollout and the adjoint's nested solve
 * of an (n_state, n_ctrl) pair that no instance covers run the large-shape kernels: one thread block per problem,
 * runtime sizes, the per-time-step tiles of one problem in shared memory.  Their step needs Ks/ks (it returns
 * MPCB200_ERR_SMEM without them, or when the shape does not fit shared memory).  The one-call adjoint works too; its
 * workspace then includes the nested solve's gains.
 * mpcb200_step_large_fits: 1 if the large-shape step runs (n, m) with elem_size 4 (f32) or 8 (f64), assuming the
 * H100's 227 KB of opt-in shared memory per block (no device needed); 0 otherwise.  It does not look at whether an
 * instance exists.
 */
int mpcb200_step_large_fits(const mpcb200_dims* dims, int32_t elem_size);

/*
 * The whole iLQR loop of MPC.forward (reference mpc/mpc.py:244-301) on the device, with a QuadCost(C, c) and either
 * LinDx(F, f) dynamics or a known system (dims->dynamics_kind, params->dyn; F and f are then NULL and the
 * linearisation is recomputed on the device every iteration).  One CUDA graph: an init kernel, then a conditional
 * `while` node whose body is
 *   LinDx:        rollout -> step -> track -> stop
 *   known system: rollout -> linearisation (F, f into the workspace) -> step with in-kernel dynamics -> track -> stop
 * The step runs with dims/params exactly as mpcb200_lqr_step_* (do_rollout = 1; du_first and status are requested,
 * qp_iters and free_mask are not; Ks/ks go into the workspace when mpcb200_step_prefers_workspace asks for them), so
 * mpcb200_last_step_plan reports its plan.  The track kernel keeps, per problem, the iterate of the lowest cost so far
 * (`costs <= best_costs + best_cost_eps`, evaluated in the element type), carries the latest controls forward and forms
 * the reference's batch-mixing full_du_norm over the caller's m_ref controls; the stop kernel ends the loop when
 * max_b full_du_norm < eps (a NaN never does), when more than not_improved_lim iterations in a row improved no problem,
 * or after lqr_iter iterations.
 *
 * u_init[T,B,m] or NULL (zeros).  Outputs best_x[T,B,n] best_u[T,B,m] best_costs[B] best_full_du_norm[B] and
 * info[2] (int32, device): iterations run, iterations in which some problem's pnqp did not converge.
 * workspace: device buffer of mpcb200_ilqr_workspace_bytes() bytes, 256-byte aligned, contents undefined on return.
 * If `stream` is capturing (cudaStreamIsCapturing), nothing is launched: the init kernel and the conditional node
 * join the caller's capture graph, which makes the whole solve capturable.  Otherwise the graph is instantiated,
 * launched on `stream` and its executable destroyed; the call does not synchronise the host.
 * mpcb200_launch_count counts each kernel node of the graph once, when the node is added; the number of iterations
 * the loop ran is info[0].  Returns MPCB200_ERR_NO_GRAPH_COND (before launching anything) when the driver has no
 * conditional nodes.
 */
typedef struct mpcb200_ilqr_opts {
  int32_t lqr_iter;          /* >= 1                                                                          */
  int32_t not_improved_lim;
  int32_t m_ref;             /* the caller's n_ctrl (<= dims->m when zero padded): full_du_norm mixes over these */
  int32_t reserved0;
  double eps, best_cost_eps;
} mpcb200_ilqr_opts;

size_t mpcb200_ilqr_workspace_bytes(const mpcb200_dims* dims, const mpcb200_ilqr_opts* opts, int32_t elem_size);
int mpcb200_ilqr_f32(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                     const float* C, const float* c, const float* F, const float* f,
                     const float* x_init, const float* u_init,
                     const float* u_lower, const float* u_upper, const uint8_t* u_zero_I,
                     float* best_x, float* best_u, float* best_costs, float* best_full_du_norm,
                     int32_t* info, void* workspace, size_t workspace_bytes, void* stream);
int mpcb200_ilqr_f64(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                     const double* C, const double* c, const double* F, const double* f,
                     const double* x_init, const double* u_init,
                     const double* u_lower, const double* u_upper, const uint8_t* u_zero_I,
                     double* best_x, double* best_u, double* best_costs, double* best_full_du_norm,
                     int32_t* info, void* workspace, size_t workspace_bytes, void* stream);

/*
 * A receding-horizon MPC episode on the device: for k = 0 .. n_steps-1, solve the problem from state x_k with warm
 * start w_k exactly as mpcb200_ilqr_* does (same dims, params, opts and inputs), apply u_k = best_u[0], step the
 * model to x_{k+1}, and shift the warm start.
 *   x_0 = x_init;  w_0 = u_init[T,B,m] or zeros;
 *   x_{k+1} = the rollout of the problem's own dynamics over the two steps (x_k, best_u[0:2]), at t = 1: for LinDx
 *             F[0] [x_k; u_k] + f[0] (exact for a time-invariant system), for a known system one step of it
 *             (params->dyn).  For a slew-rate augmented problem the state is [u_{t-1}; x] and the passthrough makes
 *             it [u_k; x_{k+1}];
 *   w_{k+1} = cat(best_u[1:], 0) with then w_{k+1}[T-2] = w_{k+1}[T-3], controls past opts->m_ref at 0.
 * Outputs xs[n_steps+1,B,n] (xs[0] = x_init), us[n_steps,B,m], costs[n_steps,B] (best_costs of each solve),
 * info[n_steps,2] (int32, each solve's info) and u_next[T,B,m] = w_{n_steps}, which continues the episode as the
 * u_init of a later call.  Needs T >= 3 and n_steps >= 1 (else MPCB200_ERR_BAD_DIMS).
 * One CUDA graph: an init kernel, then a conditional `while` node over control steps whose body is the iLQR loop's
 * init kernel and `while` node, the model step (mpcb200_rollout_* or mpcb200_dyn_rollout_* at T = 2) and an advance
 * kernel that writes the outputs and ends the loop after n_steps steps.  Capture contract, launch counting and
 * MPCB200_ERR_NO_GRAPH_COND (also for a driver that refuses a conditional node inside a conditional body) as for
 * mpcb200_ilqr_*.  workspace: mpcb200_episode_workspace_bytes() bytes, 256-byte aligned, undefined on return.
 */
size_t mpcb200_episode_workspace_bytes(const mpcb200_dims* dims, const mpcb200_ilqr_opts* opts, int32_t elem_size);
int mpcb200_episode_f32(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                        int32_t n_steps, const float* C, const float* c, const float* F, const float* f,
                        const float* x_init, const float* u_init,
                        const float* u_lower, const float* u_upper, const uint8_t* u_zero_I,
                        float* xs, float* us, float* costs, int32_t* info, float* u_next,
                        void* workspace, size_t workspace_bytes, void* stream);
int mpcb200_episode_f64(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                        int32_t n_steps, const double* C, const double* c, const double* F, const double* f,
                        const double* x_init, const double* u_init,
                        const double* u_lower, const double* u_upper, const uint8_t* u_zero_I,
                        double* xs, double* us, double* costs, int32_t* info, double* u_next,
                        void* workspace, size_t workspace_bytes, void* stream);

/*
 * mpcb200_episode_* that also keeps each solve's best iterate: plan_x[n_steps,T,B,n] and plan_u[n_steps,T,B,m]
 * (plan_u[k][0] = us[k]), the linearisation points of mpcb200_episode_backward_*.  Same arguments, outputs and graph
 * as mpcb200_episode_*, plus one kernel node per control step (before the advance kernel) that copies the plan.
 * NULL plan_x or plan_u: MPCB200_ERR_NULL_POINTER.  Workspace: mpcb200_episode_workspace_bytes().
 */
int mpcb200_episode_plans_f32(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                              int32_t n_steps, const float* C, const float* c, const float* F, const float* f,
                              const float* x_init, const float* u_init,
                              const float* u_lower, const float* u_upper, const uint8_t* u_zero_I,
                              float* xs, float* us, float* costs, int32_t* info, float* u_next,
                              float* plan_x, float* plan_u, void* workspace, size_t workspace_bytes, void* stream);
int mpcb200_episode_plans_f64(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                              int32_t n_steps, const double* C, const double* c, const double* F, const double* f,
                              const double* x_init, const double* u_init,
                              const double* u_lower, const double* u_upper, const uint8_t* u_zero_I,
                              double* xs, double* us, double* costs, int32_t* info, double* u_next,
                              double* plan_x, double* plan_u, void* workspace, size_t workspace_bytes, void* stream);

/*
 * The reverse sweep of an episode of mpcb200_episode_plans_* (a slew-rate episode: mpcb200_episode_backward_slew_*,
 * below): given dl_dxs[n_steps+1,B,n]
 * and dl_dus[n_steps,B,m], the gradient of L(xs, us) for the closed loop
 *   plan_k = the solve from x_k (its KKT adjoint at the best iterate, as mpcb200_lqr_adjoint_* with u_lower/u_upper;
 *            a known system's F, f its linearisation along the plan, differentiable in theta),
 *   u_k = plan_u[k][0],  x_{k+1} = the model step (LinDx F[0] [x_k; u_k] + f[0]; a known system one step of it),
 * with the warm starts held constant.  dims, params, C, c, F, u_lower, u_upper: the staged problem of the forward
 * (f does not enter the gradient); xs, us, plan_x, plan_u: its outputs.
 * Outputs: dx_init[B,n], dC[T,B,p,p], dc[T,B,p] (dense, whatever C's and c's time strides); LinDx: dF[F_T,B,n,p]
 * (dense) and, with has_f, df[T-1,B,n] (the model step's f[0] and the adjoints' f[t < T-1]); a known system
 * (dims->dynamics_kind 1, 2 or 4): dtheta[B,NP], per problem b the gradient in the system's learnable parameters
 * params->dyn[0..NP), summed in a fixed order (NP = 4, 3, 5); dF, df unused.
 * One CUDA graph: an init kernel, then a conditional `while` node over k = n_steps-1 .. 0 whose body is a staging
 * kernel (the plan of step k into fixed buffers and the model step's VJP), [the linearisation,] the adjoint, [the
 * linearisation's VJP] and an accumulate kernel that counts k down.  Capture contract, launch counting and
 * MPCB200_ERR_NO_GRAPH_COND as for mpcb200_ilqr_*.  T >= 3 and n_steps >= 1, else MPCB200_ERR_BAD_DIMS.
 * workspace: mpcb200_episode_backward_workspace_bytes() bytes (0 for dims it does not take), 256-byte aligned.
 */
size_t mpcb200_episode_backward_workspace_bytes(const mpcb200_dims* dims, int32_t elem_size);
int mpcb200_episode_backward_f32(const mpcb200_dims* dims, const mpcb200_params* params, int32_t n_steps,
                                 const float* C, const float* c, const float* F,
                                 const float* u_lower, const float* u_upper,
                                 const float* xs, const float* us, const float* plan_x, const float* plan_u,
                                 const float* dl_dxs, const float* dl_dus,
                                 float* dx_init, float* dC, float* dc, float* dF, float* df, float* dtheta,
                                 void* workspace, size_t workspace_bytes, void* stream);
int mpcb200_episode_backward_f64(const mpcb200_dims* dims, const mpcb200_params* params, int32_t n_steps,
                                 const double* C, const double* c, const double* F,
                                 const double* u_lower, const double* u_upper,
                                 const double* xs, const double* us, const double* plan_x, const double* plan_u,
                                 const double* dl_dxs, const double* dl_dus,
                                 double* dx_init, double* dC, double* dc, double* dF, double* df, double* dtheta,
                                 void* workspace, size_t workspace_bytes, void* stream);

/*
 * The reverse sweep of a slew-rate episode: mpcb200_episode_backward_* on the augmented problem over
 * [u_{k-1}; x_k] that mpcb200_episode_plans_* staged and ran (C~ = slew_C + C, c~ = [0; c], LinDx F~ = [[0, 0, I],
 * [0, F]], f~ = [0; f]; a known system's passthrough kind), with the previous control held constant, as the
 * reference detaches prev_ctrl: the first n_prev entries of every augmented state get no gradient, so
 * dl_dxs[k][:, :n_prev] is ignored, dx_init[:, :n_prev] is returned 0, and the model step's passthrough row carries
 * nothing back.  Every argument after n_prev is that of mpcb200_episode_backward_*, in the augmented (padded) sizes;
 * the caller crops the gradients (dC[.., n_prev:, n_prev:], dc[.., n_prev:], dF[.., n_prev:, n_prev:],
 * df[.., n_prev:], dx_init[:, n_prev:]).  A known system's dtheta is its linearisation VJP applied to the
 * [n_prev:, n_prev:] block of each adjoint's dF~ and to df~[n_prev:], plus the model step's direct part.
 * n_prev: the system's n_ctrl, explicit because zero padding can make dims->m larger and an augmented LinDx
 * problem looks like a plain one; 1 <= n_prev <= dims->m and n_prev < dims->n, else MPCB200_ERR_BAD_DIMS.  A known
 * system: dims->dynamics_kind is its passthrough kind (17, 18, 20) at the dynamics-only shape (n_state + 1, 1) and
 * n_prev = 1; kinds 1, 2 and 4 take mpcb200_episode_backward_* instead (MPCB200_ERR_BAD_DIMS here).  Errors, capture
 * contract, launch counting and MPCB200_ERR_NO_GRAPH_COND as for mpcb200_episode_backward_*; every argument error
 * is reported before anything is captured.  workspace: mpcb200_episode_backward_slew_workspace_bytes() bytes (0 for
 * arguments it does not take), 256-byte aligned.
 */
size_t mpcb200_episode_backward_slew_workspace_bytes(const mpcb200_dims* dims, int32_t n_prev, int32_t elem_size);
int mpcb200_episode_backward_slew_f32(const mpcb200_dims* dims, const mpcb200_params* params, int32_t n_steps,
                                      int32_t n_prev, const float* C, const float* c, const float* F,
                                      const float* u_lower, const float* u_upper,
                                      const float* xs, const float* us, const float* plan_x, const float* plan_u,
                                      const float* dl_dxs, const float* dl_dus,
                                      float* dx_init, float* dC, float* dc, float* dF, float* df, float* dtheta,
                                      void* workspace, size_t workspace_bytes, void* stream);
int mpcb200_episode_backward_slew_f64(const mpcb200_dims* dims, const mpcb200_params* params, int32_t n_steps,
                                      int32_t n_prev, const double* C, const double* c, const double* F,
                                      const double* u_lower, const double* u_upper,
                                      const double* xs, const double* us, const double* plan_x, const double* plan_u,
                                      const double* dl_dxs, const double* dl_dus,
                                      double* dx_init, double* dC, double* dc, double* dF, double* df, double* dtheta,
                                      void* workspace, size_t workspace_bytes, void* stream);

/*
 * An episode closed on a plant other than the model the solves plan with, with additive process disturbances:
 *   x_{k+1} = plant(x_k, u_k) + w_k
 * where each solve still plans with the problem's own dynamics (dims, params, F, f).  The plant is
 *   kind MPCB200_DYN_LINEAR: F_plant[B,n,n+m] and, with has_f, f_plant[B,n] - the t = 0 slices of a LinDx, at the
 *        problem's (padded) sizes: x' = F_plant [x; u] + f_plant;
 *   a known kind (dyn[] as in mpcb200_params.dyn): its own step, with its own parameters.  Its (n, m) must be the
 *        problem's exactly, else MPCB200_ERR_BAD_DIMS; under a slew-rate penalty that is its passthrough kind, which
 *        steps [u_{k-1}; x_k] to [u_k; plant(x_k, u_k)].
 * mpcb200_episode_plant_* takes no n_prev, so it cannot tell a slew-rate augmented problem from a plain one of the
 * same (n, m): it accepts a passthrough plant wherever the shapes match, and a passthrough plant on a problem that is
 * not augmented would read x[0] as the previous control.  The caller pairs them; mpcb200_episode_backward_plant_*,
 * which takes n_prev, refuses the mismatch (MPCB200_ERR_BAD_DIMS).
 */
typedef struct mpcb200_plant {
  int32_t kind;           /* MPCB200_DYN_LINEAR or a known kind (| MPCB200_DYN_CTRL_PASSTHROUGH) */
  int32_t has_f;          /* LinDx: f_plant given                                                 */
  double dyn[8];          /* known kind: its parameters                                           */
} mpcb200_plant;

/*
 * mpcb200_episode_plans_* with the model step replaced by the plant's (mpcb200_plant above) plus w[n_steps,B,n]
 * (NULL: none), added before xs[k+1] and the next solve's state are written.  Under a slew-rate penalty w's first
 * n_ctrl entries (the previous control) are the caller's to keep at 0.  plan_x and plan_u may both be NULL (only one:
 * MPCB200_ERR_NULL_POINTER), which records mpcb200_episode_*'s graph.  Checks, capture contract, launch counting and
 * workspace (mpcb200_episode_workspace_bytes()) as for mpcb200_episode_*; every argument error is reported before
 * anything is captured.
 */
int mpcb200_episode_plant_f32(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                              const mpcb200_plant* plant, int32_t n_steps, const float* C, const float* c,
                              const float* F, const float* f, const float* F_plant, const float* f_plant,
                              const float* w, const float* x_init, const float* u_init, const float* u_lower,
                              const float* u_upper, const uint8_t* u_zero_I, float* xs, float* us, float* costs,
                              int32_t* info, float* u_next, float* plan_x, float* plan_u, void* workspace,
                              size_t workspace_bytes, void* stream);
int mpcb200_episode_plant_f64(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                              const mpcb200_plant* plant, int32_t n_steps, const double* C, const double* c,
                              const double* F, const double* f, const double* F_plant, const double* f_plant,
                              const double* w, const double* x_init, const double* u_init, const double* u_lower,
                              const double* u_upper, const uint8_t* u_zero_I, double* xs, double* us, double* costs,
                              int32_t* info, double* u_next, double* plan_x, double* plan_u, void* workspace,
                              size_t workspace_bytes, void* stream);

/*
 * The reverse sweep of an episode of mpcb200_episode_plant_* (run with plan_x, plan_u): mpcb200_episode_backward_*
 * (n_prev = 0) or mpcb200_episode_backward_slew_* (n_prev > 0, the same n_prev rules) with the model step's VJP taken
 * at the plant.  The model's outputs dF, df (LinDx) or dtheta (a known system) get the solves' part only: the
 * adjoints, and a known system's linearisation VJP.  The plant's own outputs get the plant steps' direct part:
 *   LinDx plant: dF_plant[B,n,n+m] = sum_k g_k [x_k; u_k]^T and, with has_f, df_plant[B,n] = sum_k g_k;
 *   a known plant: dtheta_plant[B,NP_plant] = sum_k the VJP's `first` (its Jacobian held constant);
 * with g_k = dL/dx_{k+1}.  dw[n_steps,B,n] (NULL: not written) = dL/dw_k = g_k.  A known plant must be a passthrough
 * kind exactly when n_prev > 0, with n_prev its n_ctrl, else MPCB200_ERR_BAD_DIMS.  Errors, capture contract and
 * launch counting as for mpcb200_episode_backward_*; every argument error is reported before anything is captured.
 * workspace: mpcb200_episode_backward_plant_workspace_bytes() bytes (0 for arguments it does not take).
 */
size_t mpcb200_episode_backward_plant_workspace_bytes(const mpcb200_dims* dims, int32_t n_prev,
                                                      const mpcb200_plant* plant, int32_t elem_size);
int mpcb200_episode_backward_plant_f32(const mpcb200_dims* dims, const mpcb200_params* params,
                                       const mpcb200_plant* plant, int32_t n_steps, int32_t n_prev, const float* C,
                                       const float* c, const float* F, const float* F_plant, const float* u_lower,
                                       const float* u_upper, const float* xs, const float* us, const float* plan_x,
                                       const float* plan_u, const float* dl_dxs, const float* dl_dus, float* dx_init,
                                       float* dC, float* dc, float* dF, float* df, float* dtheta, float* dF_plant,
                                       float* df_plant, float* dtheta_plant, float* dw, void* workspace,
                                       size_t workspace_bytes, void* stream);
int mpcb200_episode_backward_plant_f64(const mpcb200_dims* dims, const mpcb200_params* params,
                                       const mpcb200_plant* plant, int32_t n_steps, int32_t n_prev, const double* C,
                                       const double* c, const double* F, const double* F_plant,
                                       const double* u_lower, const double* u_upper, const double* xs,
                                       const double* us, const double* plan_x, const double* plan_u,
                                       const double* dl_dxs, const double* dl_dus, double* dx_init, double* dC,
                                       double* dc, double* dF, double* df, double* dtheta, double* dF_plant,
                                       double* df_plant, double* dtheta_plant, double* dw, void* workspace,
                                       size_t workspace_bytes, void* stream);

/*
 * Episodes on a time-varying problem: every time-indexed input lies on the EPISODE's time axis of L >= n_steps + T - 1
 * slices, and solve k plans on the window of slices k .. k+T-1 of it.  At the start of each control step (and of each
 * step of the reverse sweep) one kernel node copies that window into fixed workspace buffers, which the solve's nodes
 * were recorded with; the solve kernels are those of mpcb200_episode_*.  Per input, its bit in `on`:
 *   MPCB200_WIN_COST:   C[L,B,p,p], c[L,B,p]; solve k takes C[k .. k+T-1], c[k .. k+T-1];
 *   MPCB200_WIN_DYN:    a LinDx model's F[L-T+F_T,B,n,p] and f[L-1 or L,B,n]; solve k takes F[k .. k+F_T-1] and
 *                       f[k .. k+T-2], and the model steps control step k with F[k], f[k];
 *   MPCB200_WIN_BOUNDS: tensor bounds u_lower, u_upper [L,B,m] (dims->bounds_kind 2); solve k takes [k .. k+T-1];
 *   MPCB200_WIN_PLANT:  a LinDx plant's F_plant[L-1 or L,B,n,p] and f_plant[L-1 or L,B,n]; control step k steps
 *                       with slice k.
 * An input whose bit is clear is what mpcb200_episode_plant_* takes (the solve's own [T,...] with dims' time strides,
 * or a plant's slice [B,...]).  MPCB200_WIN_COST is required, MPCB200_WIN_DYN only with a LinDx model,
 * MPCB200_WIN_BOUNDS only with tensor bounds, MPCB200_WIN_PLANT only with a LinDx plant (else MPCB200_ERR_BAD_DIMS).
 * The *_tstride fields give the elements between consecutive slices of each windowed input, with dims' convention:
 * 0 dense, > 0 that many elements (each [B,...] slice contiguous), MPCB200_TIME_INVARIANT one slice for every time.
 */
#define MPCB200_WIN_COST 1
#define MPCB200_WIN_DYN 2
#define MPCB200_WIN_BOUNDS 4
#define MPCB200_WIN_PLANT 8
typedef struct mpcb200_window {
  int32_t L;              /* slices on the episode's axis; L < n_steps + T - 1 is MPCB200_ERR_BAD_DIMS          */
  int32_t on;             /* MPCB200_WIN_* bits                                                                 */
  int64_t C_tstride, c_tstride, F_tstride, f_tstride, lo_tstride, hi_tstride, Fp_tstride, fp_tstride;
} mpcb200_window;

/*
 * mpcb200_episode_plant_* on a time-varying problem (mpcb200_window above).  plant may be NULL: the model steps the
 * loop (its window's F[k], f[k] for a LinDx model), and w (NULL: none) is still added.  plan_x and plan_u may both be
 * NULL.  Checks, capture contract, launch counting and outputs as for mpcb200_episode_plant_*; every argument error is
 * reported before anything is captured.  workspace: mpcb200_episode_window_workspace_bytes() bytes (0 for arguments
 * it does not take), 256-byte aligned.
 */
size_t mpcb200_episode_window_workspace_bytes(const mpcb200_dims* dims, const mpcb200_ilqr_opts* opts,
                                              const mpcb200_window* window, int32_t elem_size);
int mpcb200_episode_window_f32(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                               const mpcb200_window* window, const mpcb200_plant* plant, int32_t n_steps,
                               const float* C, const float* c, const float* F, const float* f, const float* F_plant,
                               const float* f_plant, const float* w, const float* x_init, const float* u_init,
                               const float* u_lower, const float* u_upper, const uint8_t* u_zero_I, float* xs,
                               float* us, float* costs, int32_t* info, float* u_next, float* plan_x, float* plan_u,
                               void* workspace, size_t workspace_bytes, void* stream);
int mpcb200_episode_window_f64(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                               const mpcb200_window* window, const mpcb200_plant* plant, int32_t n_steps,
                               const double* C, const double* c, const double* F, const double* f,
                               const double* F_plant, const double* f_plant, const double* w, const double* x_init,
                               const double* u_init, const double* u_lower, const double* u_upper,
                               const uint8_t* u_zero_I, double* xs, double* us, double* costs, int32_t* info,
                               double* u_next, double* plan_x, double* plan_u, void* workspace, size_t workspace_bytes,
                               void* stream);

/*
 * The reverse sweep of an episode of mpcb200_episode_window_* (run with plan_x, plan_u), with the rules of
 * mpcb200_episode_backward_* (plant NULL, n_prev 0), _slew_* (plant NULL, n_prev > 0) or _plant_* (plant given).  The
 * inputs are the forward's, on the same window.  Each step's window is staged before its adjoint, and the outputs of
 * windowed inputs are full length, element t summing, in the order k = n_steps-1 .. 0, every solve whose window holds
 * t: dC[L,B,p,p] and dc[L,B,p] (MPCB200_WIN_COST); dF[L-T+F_T,B,n,p] and df[L-1,B,n] (MPCB200_WIN_DYN), with the
 * model step's g_k [x_k; u_k]^T and g_k in slice k; dF_plant[L-1,B,n,p] and df_plant[L-1,B,n] (MPCB200_WIN_PLANT),
 * the plant step's in slice k.  Outputs of inputs whose bit is clear are those of the entry named above.  Every output
 * is written in full.  workspace: mpcb200_episode_backward_window_workspace_bytes() bytes (0 for arguments it does
 * not take), 256-byte aligned.
 */
size_t mpcb200_episode_backward_window_workspace_bytes(const mpcb200_dims* dims, int32_t n_prev,
                                                       const mpcb200_window* window, const mpcb200_plant* plant,
                                                       int32_t elem_size);
int mpcb200_episode_backward_window_f32(const mpcb200_dims* dims, const mpcb200_params* params,
                                        const mpcb200_window* window, const mpcb200_plant* plant, int32_t n_steps,
                                        int32_t n_prev, const float* C, const float* c, const float* F,
                                        const float* F_plant, const float* u_lower, const float* u_upper,
                                        const float* xs, const float* us, const float* plan_x, const float* plan_u,
                                        const float* dl_dxs, const float* dl_dus, float* dx_init, float* dC, float* dc,
                                        float* dF, float* df, float* dtheta, float* dF_plant, float* df_plant,
                                        float* dtheta_plant, float* dw, void* workspace, size_t workspace_bytes,
                                        void* stream);
int mpcb200_episode_backward_window_f64(const mpcb200_dims* dims, const mpcb200_params* params,
                                        const mpcb200_window* window, const mpcb200_plant* plant, int32_t n_steps,
                                        int32_t n_prev, const double* C, const double* c, const double* F,
                                        const double* F_plant, const double* u_lower, const double* u_upper,
                                        const double* xs, const double* us, const double* plan_x,
                                        const double* plan_u, const double* dl_dxs, const double* dl_dus,
                                        double* dx_init, double* dC, double* dc, double* dF, double* df,
                                        double* dtheta, double* dF_plant, double* df_plant, double* dtheta_plant,
                                        double* dw, void* workspace, size_t workspace_bytes, void* stream);

/*
 * A learned model in the kernels: the network of the reference's NNDynamics (mpc/dynamics.py:15-131),
 * x' = [x +] MLP([x; u]), with n_layers Linear layers (1..4), an activation after every layer but the last, and the
 * last layer linear.  width[0] = n_s + m_s (the network's own state and control counts), width[n_layers] = n_s,
 * every width 1..MPCB200_MLP_MAX_WIDTH.  params: ONE device buffer of the element type holding every layer's weight
 * W_i [width[i+1], width[i]] (row-major, as nn.Linear stores it) at element offset W_off[i] and bias b_i
 * [width[i+1]] at b_off[i]; the kernels stage elements [0, max end) of it into shared memory per CTA.
 * n_prev: 0, or m_s for the slew-rate augmented state [u_{t-1}; x] of CtrlPassthroughDynamics, stepped as
 * [u; MLP(x, u)].  The calls work on a staged problem of N states and M controls (zero padded as the step is):
 * the network reads states n_prev .. n_prev+n_s-1 and controls 0 .. m_s-1, N >= n_prev + n_s, M >= m_s and
 * N + M <= n_prev + width[0] + MPCB200_MLP_PAD_SLACK (else MPCB200_ERR_BAD_DIMS); states past n_prev + n_s are
 * written as 0.
 */
#define MPCB200_MLP_MAX_LAYERS 4
#define MPCB200_MLP_MAX_WIDTH 256
#define MPCB200_MLP_PAD_SLACK 16
enum { MPCB200_ACT_SIGMOID = 0, MPCB200_ACT_RELU = 1, MPCB200_ACT_ELU = 2 };
typedef struct mpcb200_mlp {
  int32_t n_layers;
  int32_t width[MPCB200_MLP_MAX_LAYERS + 1];
  int32_t activation;     /* MPCB200_ACT_*; ELU with alpha = 1                                              */
  int32_t passthrough;    /* 1: x' = x + MLP(z)                                                             */
  int32_t n_prev;
  int32_t reserved0;
  const void* params;
  int64_t W_off[MPCB200_MLP_MAX_LAYERS];
  int64_t b_off[MPCB200_MLP_MAX_LAYERS];
} mpcb200_mlp;

/* 1 if the kernels below take the network in elem_size-byte elements: its parameters plus one warp's activation
 * buffers fit the opt-in shared memory of an H100 (227 KB); 0 otherwise or for a malformed record.  Needs no
 * device.  A caller keeps its own path for a network that does not fit. */
int mpcb200_mlp_fits(const mpcb200_mlp* mlp, int32_t elem_size);

/* x[T,B,N]: x[0] = x_init[B,N], x[t+1] = step(x[t], u[t]) for t < T-1 (reference mpc/util.py:102-126). */
int mpcb200_mlp_rollout_f32(const mpcb200_mlp* mlp, int32_t B, int32_t T, int32_t N, int32_t M,
                            const float* x_init, const float* u, float* x, void* stream);
int mpcb200_mlp_rollout_f64(const mpcb200_mlp* mlp, int32_t B, int32_t T, int32_t N, int32_t M,
                            const double* x_init, const double* u, double* x, void* stream);
/* The exact linearisation for t < T-1: F[T-1,B,N,N+M] = [R S] and f[T-1,B,N] = x' - R x - S u at (x[t], u[t]) of
 * x[T,B,N], u[T,B,M], with the Jacobian chain of NNDynamics.grad_input (the activation's slope taken from its
 * output, relu's 0 at 0) and I added to R with passthrough.  Under n_prev the rows of the previous control are
 * [0 0 I] and f 0.  Nothing is written or launched for T = 1. */
int mpcb200_mlp_linearize_f32(const mpcb200_mlp* mlp, int32_t B, int32_t T, int32_t N, int32_t M, const float* x,
                              const float* u, float* F, float* f, void* stream);
int mpcb200_mlp_linearize_f64(const mpcb200_mlp* mlp, int32_t B, int32_t T, int32_t N, int32_t M, const double* x,
                              const double* u, double* F, double* f, void* stream);
/* The VJP of mpcb200_mlp_linearize_* in the parameters: dtheta[n_params] (the record's packed layout, n_params the
 * largest end of a W_i or b_i; elements of no layer are 0) = d/dtheta of the sum over t < T-1 and b of
 * <dF[t,b], F[t,b]> + <df[t,b], f[t,b]>, with x, u, dF[T-1,B,N,N+M] and df[T-1,B,N] at the staged shapes of
 * mpcb200_mlp_linearize_*.  Only the network's block of dF and df enters (rows n_prev .. n_prev+n_s-1, columns of
 * its state and control); the passthrough identity, the rows of the previous control and the padding are constants.
 * The (t, b) items are summed in an order fixed by B, T and the record alone, with no atomics: dtheta is bitwise the
 * same for every call, stream and graph replay on one card type.  Two kernels; T = 1 writes dtheta = 0.
 * workspace: mpcb200_mlp_linearize_vjp_workspace_bytes() bytes, 256-byte aligned.  MPCB200_ERR_SMEM for a network
 * whose VJP does not fit (that function's 0). */
size_t mpcb200_mlp_linearize_vjp_workspace_bytes(const mpcb200_mlp* mlp, int32_t B, int32_t T, int32_t elem_size);
int mpcb200_mlp_linearize_vjp_f32(const mpcb200_mlp* mlp, int32_t B, int32_t T, int32_t N, int32_t M, const float* x,
                                  const float* u, const float* dF, const float* df, float* dtheta, void* workspace,
                                  size_t workspace_bytes, void* stream);
int mpcb200_mlp_linearize_vjp_f64(const mpcb200_mlp* mlp, int32_t B, int32_t T, int32_t N, int32_t M,
                                  const double* x, const double* u, const double* dF, const double* df,
                                  double* dtheta, void* workspace, size_t workspace_bytes, void* stream);
/* One LQR step whose true dynamics are the network and whose true cost is QuadCost(C, c): mpcb200_lqr_step_* with
 * do_rollout = 0 (dims->do_rollout is ignored, dims->dynamics_kind must be 0) writes the gains into the workspace,
 * then one kernel runs the line search of the reference's lqr_forward (mpc/lqr_step.py:164-261) per problem:
 * u = K (x - cur_x) + cur_u + alpha k, u_zero_I, then the box (with delta_u) clamped lower bound first, x stepped by
 * the network, the true cost summed; alpha *= ls_decay while the cost exceeds that of (cur_x, cur_u), for at most
 * max_ls_iter passes, and alpha /= ls_decay after a last pass that was still worse.  Outputs new_x, new_u, costs[B],
 * alphas[B] and optional du_first (cur_u - new_u of the first pass), qp_iters, free_mask, status (the step's).
 * workspace: mpcb200_mlp_step_workspace_bytes() bytes, 256-byte aligned. */
size_t mpcb200_mlp_step_workspace_bytes(const mpcb200_dims* dims, int32_t elem_size);
int mpcb200_mlp_step_f32(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_mlp* mlp,
                         const float* C, const float* c, const float* F, const float* f, const float* x_init,
                         const float* cur_x, const float* cur_u, const float* u_lower, const float* u_upper,
                         const uint8_t* u_zero_I, float* new_x, float* new_u, float* costs, float* alphas,
                         float* du_first, int32_t* qp_iters, uint8_t* free_mask, int32_t* status, void* workspace,
                         size_t workspace_bytes, void* stream);
int mpcb200_mlp_step_f64(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_mlp* mlp,
                         const double* C, const double* c, const double* F, const double* f, const double* x_init,
                         const double* cur_x, const double* cur_u, const double* u_lower, const double* u_upper,
                         const uint8_t* u_zero_I, double* new_x, double* new_u, double* costs, double* alphas,
                         double* du_first, int32_t* qp_iters, uint8_t* free_mask, int32_t* status, void* workspace,
                         size_t workspace_bytes, void* stream);
/* mpcb200_ilqr_* with the network as the dynamics (dims->dynamics_kind 0, no F or f): the loop body is
 *   mlp rollout -> mlp linearisation (F, f into the workspace) -> step (do_rollout = 0, gains into the workspace)
 *   -> mlp line search -> track -> stop
 * with the init, track and stop kernels, outputs, capture contract, launch counting and MPCB200_ERR_NO_GRAPH_COND of
 * mpcb200_ilqr_*.  Under a slew-rate penalty the caller passes the augmented problem and mlp->n_prev = m.
 * workspace: mpcb200_ilqr_mlp_workspace_bytes() bytes, 256-byte aligned. */
size_t mpcb200_ilqr_mlp_workspace_bytes(const mpcb200_dims* dims, const mpcb200_ilqr_opts* opts, int32_t elem_size);
int mpcb200_ilqr_mlp_f32(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                         const mpcb200_mlp* mlp, const float* C, const float* c, const float* x_init,
                         const float* u_init, const float* u_lower, const float* u_upper, const uint8_t* u_zero_I,
                         float* best_x, float* best_u, float* best_costs, float* best_full_du_norm, int32_t* info,
                         void* workspace, size_t workspace_bytes, void* stream);
int mpcb200_ilqr_mlp_f64(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                         const mpcb200_mlp* mlp, const double* C, const double* c, const double* x_init,
                         const double* u_init, const double* u_lower, const double* u_upper,
                         const uint8_t* u_zero_I, double* best_x, double* best_u, double* best_costs,
                         double* best_full_du_norm, int32_t* info, void* workspace, size_t workspace_bytes,
                         void* stream);
/* A receding-horizon episode planned with the network (mlp->n_prev 0; no slew-rate penalty): mpcb200_episode_plant_*
 * with every solve the loop of mpcb200_ilqr_mlp_* (dims->dynamics_kind 0, no F or f).  plant NULL: the network steps
 * the loop, x_{k+1} = net(x_k, u_k) (+ w_k), by mpcb200_mlp_rollout_* at T = 2 from x_k and the solve's best
 * controls.  Otherwise the plant steps it as in mpcb200_episode_plant_* (a LinDx or a known system's own kind, not a
 * passthrough kind).  w, plan_x and plan_u are optional (plan_x and plan_u together).  Checks, capture contract,
 * launch counting and MPCB200_ERR_NO_GRAPH_COND as for mpcb200_episode_*; every argument error is reported before
 * anything is captured: MPCB200_ERR_SMEM for a network that does not fit, MPCB200_ERR_BAD_DIMS for T < 3 or
 * n_steps < 1.  workspace: mpcb200_episode_mlp_workspace_bytes() bytes (0 for arguments it does not take),
 * 256-byte aligned. */
size_t mpcb200_episode_mlp_workspace_bytes(const mpcb200_dims* dims, const mpcb200_ilqr_opts* opts,
                                           const mpcb200_mlp* mlp, int32_t elem_size);
int mpcb200_episode_mlp_f32(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                            const mpcb200_mlp* mlp, const mpcb200_plant* plant, int32_t n_steps, const float* C,
                            const float* c, const float* F_plant, const float* f_plant, const float* w,
                            const float* x_init, const float* u_init, const float* u_lower, const float* u_upper,
                            const uint8_t* u_zero_I, float* xs, float* us, float* costs, int32_t* info, float* u_next,
                            float* plan_x, float* plan_u, void* workspace, size_t workspace_bytes, void* stream);
int mpcb200_episode_mlp_f64(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                            const mpcb200_mlp* mlp, const mpcb200_plant* plant, int32_t n_steps, const double* C,
                            const double* c, const double* F_plant, const double* f_plant, const double* w,
                            const double* x_init, const double* u_init, const double* u_lower, const double* u_upper,
                            const uint8_t* u_zero_I, double* xs, double* us, double* costs, int32_t* info,
                            double* u_next, double* plan_x, double* plan_u, void* workspace, size_t workspace_bytes,
                            void* stream);
/* The reverse sweep of an episode of mpcb200_episode_mlp_* (run with plan_x, plan_u): mpcb200_episode_backward_plant_*
 * with each solve's part taken through the network's linearisation along its plan, and dtheta[n_params] (the
 * record's packed layout) the gradient of the network's parameters: the sum over control steps of the VJP of that
 * linearisation (mpcb200_mlp_linearize_vjp_*) in the solve's adjoint, plus, with plant NULL, the network step's
 * d<g_k, x_{k+1}>/dtheta.  The plant's outputs (dF_plant, df_plant or dtheta_plant) are those of
 * mpcb200_episode_backward_plant_*; dw[n_steps,B,n] (NULL: not written) = g_k.  Every sum runs in a fixed order with
 * no float atomics: dtheta is bitwise the same for every call, stream and graph replay on one card type.  Checks,
 * capture contract, launch counting and MPCB200_ERR_NO_GRAPH_COND as for mpcb200_episode_backward_*; every argument
 * error is reported before anything is captured, MPCB200_ERR_SMEM for a network or network VJP that does not fit.
 * workspace: mpcb200_episode_backward_mlp_workspace_bytes() bytes (0 for arguments it does not take, among them a
 * network whose VJP does not fit), 256-byte aligned. */
size_t mpcb200_episode_backward_mlp_workspace_bytes(const mpcb200_dims* dims, const mpcb200_mlp* mlp,
                                                    const mpcb200_plant* plant, int32_t elem_size);
int mpcb200_episode_backward_mlp_f32(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_mlp* mlp,
                                     const mpcb200_plant* plant, int32_t n_steps, const float* C, const float* c,
                                     const float* F_plant, const float* u_lower, const float* u_upper,
                                     const float* xs, const float* us, const float* plan_x, const float* plan_u,
                                     const float* dl_dxs, const float* dl_dus, float* dx_init, float* dC, float* dc,
                                     float* dtheta, float* dF_plant, float* df_plant, float* dtheta_plant, float* dw,
                                     void* workspace, size_t workspace_bytes, void* stream);
int mpcb200_episode_backward_mlp_f64(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_mlp* mlp,
                                     const mpcb200_plant* plant, int32_t n_steps, const double* C, const double* c,
                                     const double* F_plant, const double* u_lower, const double* u_upper,
                                     const double* xs, const double* us, const double* plan_x, const double* plan_u,
                                     const double* dl_dxs, const double* dl_dus, double* dx_init, double* dC,
                                     double* dc, double* dtheta, double* dF_plant, double* df_plant,
                                     double* dtheta_plant, double* dw, void* workspace, size_t workspace_bytes,
                                     void* stream);

/* 1 if a kernel instance for (n_state, n_ctrl) is compiled in, else 0. */
int mpcb200_supported(int32_t n_state, int32_t n_ctrl);

/* Fills `out` with up to `cap` supported (n,m) pairs (n0,m0,n1,m1,...); returns the count of pairs. */
int mpcb200_supported_list(int32_t* out, int32_t cap);

/* Number of kernels this library has launched in this process (bench.py's gpu_launches). */
uint64_t mpcb200_launch_count(void);

/* Dynamic shared memory (bytes) the step kernel needs for these dims / element size (4 or 8); 0 if unsupported. */
size_t mpcb200_step_smem_bytes(const mpcb200_dims* dims, int32_t elem_size);

/* 1 if the step kernel wants caller-provided Ks/ks buffers for these dims: either the gain store of all
 * T steps does not fit shared memory, or (one-problem-per-warp shapes such as n=16) moving it out of shared
 * memory is what lets enough warps be resident, or the shape runs the large-shape kernel.  Pass Ks[T,B,m,n],
 * ks[T,B,m] then. */
int mpcb200_step_prefers_workspace(const mpcb200_dims* dims, int32_t elem_size);

/* Plan of the last step-kernel launch made by the calling thread (mpcb200_lqr_step_*, or the nested solve of
 * mpcb200_lqr_adjoint_*), as MPCB200_PLAN_* bits; 0 if that thread's last step call launched no step kernel.
 * The launchers record what they actually launched: the kernel, where the gains K_t, k_t of the T steps lived
 * between the Riccati sweep and the rollout, and whether the rollout read them column per lane. */
#define MPCB200_PLAN_GENERIC 1u    /* the generic kernel ran (one column per lane)                           */
#define MPCB200_PLAN_PAIR 2u       /* the column-pair kernel ran                                              */
#define MPCB200_PLAN_GAINS_SMEM 4u /* gains kept in shared memory; otherwise they went through Ks/ks          */
#define MPCB200_PLAN_KREDUCE 8u    /* generic kernel, gains in Ks/ks: lane i reads column i, butterfly K dx   */
#define MPCB200_PLAN_LARGE 16u     /* the large-shape kernel ran (one thread block per problem, gains in Ks/ks) */
int32_t mpcb200_last_step_plan(void);

int mpcb200_version(void);
const char* mpcb200_strerror(int code);

#ifdef __cplusplus
}
#endif
#endif /* MPCB200_H_ */
