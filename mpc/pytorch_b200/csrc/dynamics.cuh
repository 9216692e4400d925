// dynamics.cuh - known nonlinear dynamics evaluated inside the kernels (SURVEY.md section 8(f) rank 2).
//
// The reference linearises Module dynamics with autograd - (T-1)*n_state backward passes per iLQR iteration
// (mpc/mpc.py:490-601, AUTO_DIFF :538-550) - and rolls them out with one Python call per time step
// (mpc/util.py:102-126, mpc/lqr_step.py:224-225).  For the two systems its examples ship, the step functions
// are restated here (cartpole: mpc/env_dx/cartpole.py:63-96, pendulum: mpc/env_dx/pendulum.py:49-84) as ONE
// generic device function each, evaluated on plain numbers (rollouts, line search) or on forward-mode dual
// numbers (exact Jacobians R = dx'/dx, S = dx'/du in one pass; f = x' - R x - S u as the reference forms it).
#pragma once
#include "common.cuh"

namespace mpcb200 {

// DYN_CTRL_PASSTHROUGH is OR'd into a system's kind: the slew-rate augmented state [u_{t-1}; x] with dynamics
// [u; f(x, u)] (reference CtrlPassthroughDynamics, mpc/dynamics.py:133-156), n_state + n_ctrl states
enum { DYN_LINEAR = 0, DYN_CARTPOLE = 1, DYN_PENDULUM = 2, DYN_CTRL_PASSTHROUGH = 16 };

struct DynParams {
  // cartpole: p[0..3] = gravity, masscart, masspole, length; p[4] = force_mag; p[5] = dt
  // pendulum: p[0..2] = g, m, l;                              p[4] = max_torque; p[5] = dt
  double p[8];
};

// ------------------------------------------------------------------ forward-mode dual numbers
template <typename R, int NV>
struct Dual {
  R v;
  R d[NV];
};
template <typename R, int NV>
MPCB_DEV Dual<R, NV> dual_var(R v, int k) {
  Dual<R, NV> o;
  o.v = v;
#pragma unroll
  for (int i = 0; i < NV; ++i) o.d[i] = i == k ? R(1) : R(0);
  return o;
}
#define MPCB_DUAL_BIN(op, VAL, DER)                                                     \
  template <typename R, int NV>                                                          \
  MPCB_DEV Dual<R, NV> operator op(const Dual<R, NV>& a, const Dual<R, NV>& b) {        \
    Dual<R, NV> o;                                                                       \
    o.v = VAL;                                                                           \
    _Pragma("unroll") for (int i = 0; i < NV; ++i) o.d[i] = DER;                         \
    return o;                                                                            \
  }
MPCB_DUAL_BIN(+, a.v + b.v, a.d[i] + b.d[i])
MPCB_DUAL_BIN(-, a.v - b.v, a.d[i] - b.d[i])
MPCB_DUAL_BIN(*, a.v * b.v, a.d[i] * b.v + a.v * b.d[i])
MPCB_DUAL_BIN(/, a.v / b.v, (a.d[i] * b.v - a.v * b.d[i]) / (b.v * b.v))
#undef MPCB_DUAL_BIN
template <typename R, int NV>
MPCB_DEV Dual<R, NV> operator*(R s, const Dual<R, NV>& a) {
  Dual<R, NV> o;
  o.v = s * a.v;
#pragma unroll
  for (int i = 0; i < NV; ++i) o.d[i] = s * a.d[i];
  return o;
}
template <typename R, int NV>
MPCB_DEV Dual<R, NV> operator+(R s, const Dual<R, NV>& a) {
  Dual<R, NV> o = a;
  o.v = s + a.v;
  return o;
}
template <typename R, int NV>
MPCB_DEV Dual<R, NV> operator-(R s, const Dual<R, NV>& a) {
  Dual<R, NV> o;
  o.v = s - a.v;
#pragma unroll
  for (int i = 0; i < NV; ++i) o.d[i] = -a.d[i];
  return o;
}
template <typename R, int NV>
MPCB_DEV Dual<R, NV> dsin(const Dual<R, NV>& a) {
  Dual<R, NV> o;
  const R c = cos(a.v);
  o.v = sin(a.v);
#pragma unroll
  for (int i = 0; i < NV; ++i) o.d[i] = c * a.d[i];
  return o;
}
template <typename R, int NV>
MPCB_DEV Dual<R, NV> dcos(const Dual<R, NV>& a) {
  Dual<R, NV> o;
  const R s = -sin(a.v);
  o.v = cos(a.v);
#pragma unroll
  for (int i = 0; i < NV; ++i) o.d[i] = s * a.d[i];
  return o;
}
template <typename R, int NV>
MPCB_DEV Dual<R, NV> datan2(const Dual<R, NV>& y, const Dual<R, NV>& x) {
  Dual<R, NV> o;
  const R den = x.v * x.v + y.v * y.v;
  o.v = atan2(y.v, x.v);
#pragma unroll
  for (int i = 0; i < NV; ++i) o.d[i] = (x.v * y.d[i] - y.v * x.d[i]) / den;
  return o;
}
// torch.clamp: value clamped, gradient 1 inside [lo, hi] (inclusive), 0 outside
template <typename R, int NV>
MPCB_DEV Dual<R, NV> dclamp(const Dual<R, NV>& a, R lo, R hi) {
  Dual<R, NV> o;
  const bool in = a.v >= lo && a.v <= hi;
  o.v = a.v < lo ? lo : (a.v > hi ? hi : a.v);
#pragma unroll
  for (int i = 0; i < NV; ++i) o.d[i] = in ? a.d[i] : R(0);
  return o;
}
// the same vocabulary on plain numbers
MPCB_DEV float dsin(float a) { return sinf(a); }
MPCB_DEV double dsin(double a) { return sin(a); }
MPCB_DEV float dcos(float a) { return cosf(a); }
MPCB_DEV double dcos(double a) { return cos(a); }
MPCB_DEV float datan2(float y, float x) { return atan2f(y, x); }
MPCB_DEV double datan2(double y, double x) { return atan2(y, x); }
MPCB_DEV float dclamp(float a, float lo, float hi) { return a < lo ? lo : (a > hi ? hi : a); }
MPCB_DEV double dclamp(double a, double lo, double hi) { return a < lo ? lo : (a > hi ? hi : a); }

// ------------------------------------------------------------------ the two systems
// cartpole (mpc/env_dx/cartpole.py:63-96): state (x, dx, cos th, sin th, dth), one control (force)
template <typename R, typename T>
MPCB_DEV void cartpole_step(const DynParams& dp, const T (&s)[5], const T& u_in, T (&o)[5]) {
  const R gravity = (R)dp.p[0], masscart = (R)dp.p[1], masspole = (R)dp.p[2], length = (R)dp.p[3];
  const R force_mag = (R)dp.p[4], dt = (R)dp.p[5];
  const R total_mass = masspole + masscart, polemass_length = masspole * length;
  const T u = dclamp(u_in, -force_mag, force_mag);
  const T th = datan2(s[3], s[2]);
  const T cart_in = (R(1) / total_mass) * (u + polemass_length * (s[4] * s[4] * s[3]));
  const T th_acc = (gravity * s[3] - s[2] * cart_in) /
                   (length * (R(4.) / R(3.) - (masspole / total_mass) * (s[2] * s[2])));
  const T xacc = cart_in - (polemass_length / total_mass) * (th_acc * s[2]);
  const T th2 = th + dt * s[4];
  o[0] = s[0] + dt * s[1];
  o[1] = s[1] + dt * xacc;
  o[2] = dcos(th2);
  o[3] = dsin(th2);
  o[4] = s[4] + dt * th_acc;
}
// pendulum, `simple` parametrisation (mpc/env_dx/pendulum.py:49-84): state (cos th, sin th, dth), one control (torque)
template <typename R, typename T>
MPCB_DEV void pendulum_step(const DynParams& dp, const T (&s)[3], const T& u_in, T (&o)[3]) {
  const R g = (R)dp.p[0], m = (R)dp.p[1], l = (R)dp.p[2], max_torque = (R)dp.p[4], dt = (R)dp.p[5];
  const T u = dclamp(u_in, -max_torque, max_torque);
  const T th = datan2(s[1], s[0]);
  const T newdth = s[2] + dt * ((R(3.) * g / (R(2.) * l)) * s[1] + (R(3.) / (m * l * l)) * u);
  const T newth = th + dt * newdth;
  o[0] = dcos(newth);
  o[1] = dsin(newth);
  o[2] = newdth;
}

template <int KIND>
struct DynDims {        // a passthrough kind: [u_{t-1}; x]
  static_assert((KIND & DYN_CTRL_PASSTHROUGH) != 0, "unknown dynamics kind");
  using Inner = DynDims<KIND & ~DYN_CTRL_PASSTHROUGH>;
  static constexpr int N = Inner::N + Inner::M, M = Inner::M;
};
template <>
struct DynDims<DYN_CARTPOLE> { static constexpr int N = 5, M = 1; };
template <>
struct DynDims<DYN_PENDULUM> { static constexpr int N = 3, M = 1; };

// (n_state, n_ctrl) of a known kind, passthrough or not; false for DYN_LINEAR and anything unknown
inline bool dyn_kind_dims(int kind, int& n, int& m) {
  const int sys = kind & ~DYN_CTRL_PASSTHROUGH;
  if (sys == DYN_CARTPOLE) n = DynDims<DYN_CARTPOLE>::N, m = DynDims<DYN_CARTPOLE>::M;
  else if (sys == DYN_PENDULUM) n = DynDims<DYN_PENDULUM>::N, m = DynDims<DYN_PENDULUM>::M;
  else return false;
  if (kind & DYN_CTRL_PASSTHROUGH) n += m;
  return true;
}

// one step of a known kind; a passthrough kind copies u (before the system's own clamp) into the first M states
template <typename R, int KIND, typename T>
MPCB_DEV void dyn_step(const DynParams& dp, const T (&s)[DynDims<KIND>::N], const T& u, T (&o)[DynDims<KIND>::N]) {
  if constexpr ((KIND & DYN_CTRL_PASSTHROUGH) != 0) {
    constexpr int SYS = KIND & ~DYN_CTRL_PASSTHROUGH, NI = DynDims<SYS>::N;
    static_assert(DynDims<SYS>::M == 1, "the known systems have one control");
    T si[NI], oi[NI];
#pragma unroll
    for (int i = 0; i < NI; ++i) si[i] = s[1 + i];
    dyn_step<R, SYS, T>(dp, si, u, oi);
    o[0] = u;
#pragma unroll
    for (int i = 0; i < NI; ++i) o[1 + i] = oi[i];
  } else if constexpr (KIND == DYN_CARTPOLE) {
    cartpole_step<R, T>(dp, s, u, o);
  } else {
    pendulum_step<R, T>(dp, s, u, o);
  }
}

// ------------------------------------------------------------------ kernels
struct DynArgs {
  int B, T, kind;
  DynParams dp;
  const void *x_init, *x, *u;     // rollout reads x_init,u; linearize reads x,u
  void *x_out, *F, *f;
};

// x[0] = x_init, x[t+1] = dyn(x[t], u[t]): util.get_traj for a known Module (one thread per problem); for a
// passthrough kind x is [T, B, n+m] and x[t+1] = [u[t]; dyn(x[t][m:], u[t])]
template <typename R, int KIND>
__global__ void __launch_bounds__(128) dyn_rollout_kernel(const DynArgs a) {
  constexpr int N = DynDims<KIND>::N, M = DynDims<KIND>::M;
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.B) return;
  const R* gu = (const R*)a.u;
  R* gx = (R*)a.x_out;
  R s[N];
#pragma unroll
  for (int i = 0; i < N; ++i) {
    s[i] = ((const R*)a.x_init)[(size_t)b * N + i];
    gx[(size_t)b * N + i] = s[i];
  }
  for (int t = 0; t + 1 < a.T; ++t) {
    R o[N];
    const R u = gu[((size_t)t * a.B + b) * M];
    dyn_step<R, KIND, R>(a.dp, s, u, o);
#pragma unroll
    for (int i = 0; i < N; ++i) {
      s[i] = o[i];
      gx[((size_t)(t + 1) * a.B + b) * N + i] = o[i];
    }
  }
}

// F[t,b] = [dx'/dx  dx'/du], f[t,b] = x' - F [x;u] at (x[t,b], u[t,b]) for t < T-1 (one thread per (t, problem))
// A passthrough kind differentiates only the system itself (n + m dual variables, the system's own F and f) and
// writes F~ = [[0, 0, I], [0, R, S]], f~ = [0; f]: the blocks MPC assembles from the system's F and f.
template <typename R, int KIND>
__global__ void __launch_bounds__(128) dyn_linearize_kernel(const DynArgs a) {
  constexpr int N = DynDims<KIND>::N, M = DynDims<KIND>::M, P = N + M;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)(a.T - 1) * a.B) return;
  const R* gx = (const R*)a.x + i * N;
  const R* gu = (const R*)a.u + i * M;
  if constexpr ((KIND & DYN_CTRL_PASSTHROUGH) != 0) {
    constexpr int SYS = KIND & ~DYN_CTRL_PASSTHROUGH, NI = DynDims<SYS>::N, PI = NI + M;
    using D = Dual<R, PI>;
    D s[NI], o[NI];
    R xv[PI];
#pragma unroll
    for (int k = 0; k < NI; ++k) {
      xv[k] = gx[M + k];
      s[k] = dual_var<R, PI>(xv[k], k);
    }
    xv[NI] = gu[0];
    const D u = dual_var<R, PI>(xv[NI], NI);
    dyn_step<R, SYS, D>(a.dp, s, u, o);
    R* oF = (R*)a.F + i * N * P;
    R* of = (R*)a.f + i * N;
#pragma unroll
    for (int r = 0; r < M; ++r) {              // u_{t} -> the first M states
#pragma unroll
      for (int k = 0; k < P; ++k) oF[r * P + k] = k == N + r ? R(1) : R(0);
      of[r] = R(0);
    }
#pragma unroll
    for (int r = 0; r < NI; ++r) {
      R acc = o[r].v;
      R* row = oF + (M + r) * P;
#pragma unroll
      for (int k = 0; k < M; ++k) row[k] = R(0);
#pragma unroll
      for (int k = 0; k < PI; ++k) {
        row[M + k] = o[r].d[k];
        acc -= o[r].d[k] * xv[k];
      }
      of[M + r] = acc;
    }
  } else {
    using D = Dual<R, P>;
    D s[N], o[N];
    R xv[P];
#pragma unroll
    for (int k = 0; k < N; ++k) {
      xv[k] = gx[k];
      s[k] = dual_var<R, P>(xv[k], k);
    }
    xv[N] = gu[0];
    const D u = dual_var<R, P>(xv[N], N);
    dyn_step<R, KIND, D>(a.dp, s, u, o);
    R* oF = (R*)a.F + i * N * P;
    R* of = (R*)a.f + i * N;
#pragma unroll
    for (int r = 0; r < N; ++r) {
      R acc = o[r].v;
#pragma unroll
      for (int k = 0; k < P; ++k) {
        oF[r * P + k] = o[r].d[k];
        acc -= o[r].d[k] * xv[k];
      }
      of[r] = acc;
    }
  }
}

template <typename R>
int launch_dyn_rollout(const DynArgs& a, cudaStream_t stream) {
  const int grid = (a.B + 127) / 128;
  constexpr int CP = DYN_CARTPOLE | DYN_CTRL_PASSTHROUGH, PP = DYN_PENDULUM | DYN_CTRL_PASSTHROUGH;
  if (a.kind == DYN_CARTPOLE) dyn_rollout_kernel<R, DYN_CARTPOLE><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == DYN_PENDULUM) dyn_rollout_kernel<R, DYN_PENDULUM><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == CP) dyn_rollout_kernel<R, CP><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == PP) dyn_rollout_kernel<R, PP><<<grid, 128, 0, stream>>>(a);
  else return 2;
  return cudaGetLastError() == cudaSuccess ? 0 : 5;
}
template <typename R>
int launch_dyn_linearize(const DynArgs& a, cudaStream_t stream) {
  const size_t items = (size_t)(a.T - 1) * a.B;
  if (items == 0) return 0;
  const int grid = (int)((items + 127) / 128);
  constexpr int CP = DYN_CARTPOLE | DYN_CTRL_PASSTHROUGH, PP = DYN_PENDULUM | DYN_CTRL_PASSTHROUGH;
  if (a.kind == DYN_CARTPOLE) dyn_linearize_kernel<R, DYN_CARTPOLE><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == DYN_PENDULUM) dyn_linearize_kernel<R, DYN_PENDULUM><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == CP) dyn_linearize_kernel<R, CP><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == PP) dyn_linearize_kernel<R, PP><<<grid, 128, 0, stream>>>(a);
  else return 2;
  return cudaGetLastError() == cudaSuccess ? 0 : 5;
}

}  // namespace mpcb200
