// dynamics.cuh - known nonlinear dynamics evaluated inside the kernels (SURVEY.md section 8(f) rank 2).
//
// The reference linearises Module dynamics with autograd - (T-1)*n_state backward passes per iLQR iteration
// (mpc/mpc.py:490-601, AUTO_DIFF :538-550) - and rolls them out with one Python call per time step
// (mpc/util.py:102-126, mpc/lqr_step.py:224-225).  For the two systems its examples ship, the step functions
// are restated here (cartpole: mpc/env_dx/cartpole.py:63-96, pendulum: mpc/env_dx/pendulum.py:49-84, in its
// `simple` (g, m, l) and its five-parameter (g, m, l, d, b) form) as ONE generic device function each, evaluated on
// plain numbers (rollouts, line search) or on forward-mode dual numbers (exact Jacobians R = dx'/dx, S = dx'/du in
// one pass; f = x' - R x - S u as the reference forms it).
#pragma once
#include "common.cuh"

namespace mpcb200 {

// DYN_CTRL_PASSTHROUGH is OR'd into a system's kind: the slew-rate augmented state [u_{t-1}; x] with dynamics
// [u; f(x, u)] (reference CtrlPassthroughDynamics, mpc/dynamics.py:133-156), n_state + n_ctrl states
enum { DYN_LINEAR = 0, DYN_CARTPOLE = 1, DYN_PENDULUM = 2, DYN_PENDULUM_FULL = 4, DYN_CTRL_PASSTHROUGH = 16 };

struct DynParams {
  // cartpole: p[0..3] = gravity, masscart, masspole, length; p[4] = force_mag; p[5] = dt
  // pendulum: p[0..2] = g, m, l;                              p[4] = max_torque; p[5] = dt
  // pendulum_full: p[0..4] = g, m, l, d, b;                   p[5] = max_torque; p[6] = dt
  // The learnable parameters lead (DynLearnable<KIND>::NP of them): the VJP kernel seeds p[0..NP).
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
// ------------------------------------------------------------------ nested duals Dual<Dual<R, NV>, NW>
// Forward mode over forward mode: the inner dual carries d/dz, the outer one d/dtheta of a system parameter, so the
// outer derivative of an inner derivative is a mixed second derivative d2/(dtheta dz) (dyn_linearize_vjp_kernel).
// The generic operators above cover nested-with-nested; these are the scalar-on-the-left forms and the elementary
// functions, whose generic versions call cos / sin / atan2 on the value.
template <typename R, int NV>
MPCB_DEV Dual<R, NV> dual_const(R v) {
  Dual<R, NV> o;
  o.v = v;
#pragma unroll
  for (int i = 0; i < NV; ++i) o.d[i] = R(0);
  return o;
}
template <typename R, int NV, int NW>
MPCB_DEV Dual<Dual<R, NV>, NW> operator*(R s, const Dual<Dual<R, NV>, NW>& a) {
  Dual<Dual<R, NV>, NW> o;
  o.v = s * a.v;
#pragma unroll
  for (int i = 0; i < NW; ++i) o.d[i] = s * a.d[i];
  return o;
}
template <typename R, int NV, int NW>
MPCB_DEV Dual<Dual<R, NV>, NW> operator-(R s, const Dual<Dual<R, NV>, NW>& a) {
  Dual<Dual<R, NV>, NW> o;
  o.v = s - a.v;
#pragma unroll
  for (int i = 0; i < NW; ++i) o.d[i] = R(0) - a.d[i];
  return o;
}
template <typename R, int NV, int NW>
MPCB_DEV Dual<Dual<R, NV>, NW> operator/(R s, const Dual<Dual<R, NV>, NW>& a) {
  Dual<Dual<R, NV>, NW> c;
  c.v = dual_const<R, NV>(s);
#pragma unroll
  for (int i = 0; i < NW; ++i) c.d[i] = dual_const<R, NV>(R(0));
  return c / a;
}
template <typename R, int NV, int NW>
MPCB_DEV Dual<Dual<R, NV>, NW> dsin(const Dual<Dual<R, NV>, NW>& a) {
  Dual<Dual<R, NV>, NW> o;
  const Dual<R, NV> c = dcos(a.v);
  o.v = dsin(a.v);
#pragma unroll
  for (int i = 0; i < NW; ++i) o.d[i] = c * a.d[i];
  return o;
}
template <typename R, int NV, int NW>
MPCB_DEV Dual<Dual<R, NV>, NW> dcos(const Dual<Dual<R, NV>, NW>& a) {
  Dual<Dual<R, NV>, NW> o;
  const Dual<R, NV> s = R(0) - dsin(a.v);
  o.v = dcos(a.v);
#pragma unroll
  for (int i = 0; i < NW; ++i) o.d[i] = s * a.d[i];
  return o;
}
template <typename R, int NV, int NW>
MPCB_DEV Dual<Dual<R, NV>, NW> datan2(const Dual<Dual<R, NV>, NW>& y, const Dual<Dual<R, NV>, NW>& x) {
  Dual<Dual<R, NV>, NW> o;
  const Dual<R, NV> den = x.v * x.v + y.v * y.v;
  o.v = datan2(y.v, x.v);
#pragma unroll
  for (int i = 0; i < NW; ++i) o.d[i] = (x.v * y.d[i] - y.v * x.d[i]) / den;
  return o;
}
// dclamp's rule at every order: inside [lo, hi] (inclusive) the clamp is the identity, outside a constant
template <typename R, int NV, int NW>
MPCB_DEV Dual<Dual<R, NV>, NW> dclamp(const Dual<Dual<R, NV>, NW>& a, R lo, R hi) {
  Dual<Dual<R, NV>, NW> o;
  const bool in = a.v.v >= lo && a.v.v <= hi;
  o.v = dclamp(a.v, lo, hi);
#pragma unroll
  for (int i = 0; i < NW; ++i) o.d[i] = in ? a.d[i] : dual_const<R, NV>(R(0));
  return o;
}

// A system parameter p[i] as a number of type P: a plain constant, or (P a nested dual) the variable of the outer
// derivative when i == seed, else a constant.
template <typename R, typename P>
struct DynParam {
  static MPCB_DEV P get(const DynParams& dp, int i, int) { return (P)dp.p[i]; }
};
template <typename R, int NV>
struct DynParam<R, Dual<Dual<R, NV>, 1>> {
  static MPCB_DEV Dual<Dual<R, NV>, 1> get(const DynParams& dp, int i, int seed) {
    Dual<Dual<R, NV>, 1> o;
    o.v = dual_const<R, NV>((R)dp.p[i]);
    o.d[0] = dual_const<R, NV>(i == seed ? R(1) : R(0));
    return o;
  }
};

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
// The parameter number type P is R by default; a nested dual P differentiates in the learnable parameter `seed`
// (cartpole p[0..3], pendulum p[0..2], pendulum_full p[0..4]).  force_mag / max_torque and dt are constants of type R.
// cartpole (mpc/env_dx/cartpole.py:63-96): state (x, dx, cos th, sin th, dth), one control (force)
template <typename R, typename T, typename P = R>
MPCB_DEV void cartpole_step(const DynParams& dp, const T (&s)[5], const T& u_in, T (&o)[5], int seed = -1) {
  using DP = DynParam<R, P>;
  const P gravity = DP::get(dp, 0, seed), masscart = DP::get(dp, 1, seed), masspole = DP::get(dp, 2, seed),
          length = DP::get(dp, 3, seed);
  const R force_mag = (R)dp.p[4], dt = (R)dp.p[5];
  const P total_mass = masspole + masscart, polemass_length = masspole * length;
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
template <typename R, typename T, typename P = R>
MPCB_DEV void pendulum_step(const DynParams& dp, const T (&s)[3], const T& u_in, T (&o)[3], int seed = -1) {
  using DP = DynParam<R, P>;
  const P g = DP::get(dp, 0, seed), m = DP::get(dp, 1, seed), l = DP::get(dp, 2, seed);
  const R max_torque = (R)dp.p[4], dt = (R)dp.p[5];
  const T u = dclamp(u_in, -max_torque, max_torque);
  const T th = datan2(s[1], s[0]);
  const T newdth = s[2] + dt * ((R(3.) * g / (R(2.) * l)) * s[1] + (R(3.) / (m * l * l)) * u);
  const T newth = th + dt * newdth;
  o[0] = dcos(newth);
  o[1] = dsin(newth);
  o[2] = newdth;
}
// pendulum, five-parameter form (mpc/env_dx/pendulum.py:68-80, simple=False): damping d and gravity bias b.  As the
// reference writes it: the damping acts on the wrapped angle th = atan2(sin, cos), not on dth, and the gravity term
// is sin(th + b), not the state's sin th.
template <typename R, typename T, typename P = R>
MPCB_DEV void pendulum_full_step(const DynParams& dp, const T (&s)[3], const T& u_in, T (&o)[3], int seed = -1) {
  using DP = DynParam<R, P>;
  const P g = DP::get(dp, 0, seed), m = DP::get(dp, 1, seed), l = DP::get(dp, 2, seed), d = DP::get(dp, 3, seed),
          b = DP::get(dp, 4, seed);
  const R max_torque = (R)dp.p[5], dt = (R)dp.p[6];
  const T u = dclamp(u_in, -max_torque, max_torque);
  const T th = datan2(s[1], s[0]);
  const T newdth = s[2] + dt * ((R(3.) * g / (R(2.) * l)) * dsin(b + th) + (R(3.) / (m * l * l)) * u - d * th);
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
template <>
struct DynDims<DYN_PENDULUM_FULL> { static constexpr int N = 3, M = 1; };

// (n_state, n_ctrl) of a known kind, passthrough or not; false for DYN_LINEAR and anything unknown
inline bool dyn_kind_dims(int kind, int& n, int& m) {
  const int sys = kind & ~DYN_CTRL_PASSTHROUGH;
  if (sys == DYN_CARTPOLE) n = DynDims<DYN_CARTPOLE>::N, m = DynDims<DYN_CARTPOLE>::M;
  else if (sys == DYN_PENDULUM) n = DynDims<DYN_PENDULUM>::N, m = DynDims<DYN_PENDULUM>::M;
  else if (sys == DYN_PENDULUM_FULL) n = DynDims<DYN_PENDULUM_FULL>::N, m = DynDims<DYN_PENDULUM_FULL>::M;
  else return false;
  if (kind & DYN_CTRL_PASSTHROUGH) n += m;
  return true;
}

// one step of a known kind; a passthrough kind copies u (before the system's own clamp) into the first M states
template <typename R, int KIND, typename T, typename P = R>
MPCB_DEV void dyn_step(const DynParams& dp, const T (&s)[DynDims<KIND>::N], const T& u, T (&o)[DynDims<KIND>::N],
                       int seed = -1) {
  if constexpr ((KIND & DYN_CTRL_PASSTHROUGH) != 0) {
    constexpr int SYS = KIND & ~DYN_CTRL_PASSTHROUGH, NI = DynDims<SYS>::N;
    static_assert(DynDims<SYS>::M == 1, "the known systems have one control");
    T si[NI], oi[NI];
#pragma unroll
    for (int i = 0; i < NI; ++i) si[i] = s[1 + i];
    dyn_step<R, SYS, T, P>(dp, si, u, oi, seed);
    o[0] = u;
#pragma unroll
    for (int i = 0; i < NI; ++i) o[1 + i] = oi[i];
  } else if constexpr (KIND == DYN_CARTPOLE) {
    cartpole_step<R, T, P>(dp, s, u, o, seed);
  } else if constexpr (KIND == DYN_PENDULUM) {
    pendulum_step<R, T, P>(dp, s, u, o, seed);
  } else {
    static_assert(KIND == DYN_PENDULUM_FULL, "unknown dynamics kind");
    pendulum_full_step<R, T, P>(dp, s, u, o, seed);
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

// Learnable parameters theta of a system: its first NP entries of DynParams::p (cartpole gravity, masscart, masspole,
// length; pendulum g, m, l; pendulum_full g, m, l, d, b).  force_mag / max_torque and dt are constants.
template <int KIND>
struct DynLearnable {   // a passthrough kind: the system's own (its passthrough row has no parameter)
  static_assert((KIND & DYN_CTRL_PASSTHROUGH) != 0, "unknown dynamics kind");
  static constexpr int NP = DynLearnable<KIND & ~DYN_CTRL_PASSTHROUGH>::NP;
};
template <>
struct DynLearnable<DYN_CARTPOLE> { static constexpr int NP = 4; };
template <>
struct DynLearnable<DYN_PENDULUM> { static constexpr int NP = 3; };
template <>
struct DynLearnable<DYN_PENDULUM_FULL> { static constexpr int NP = 5; };

struct DynVjpArgs {
  int B, T, kind;
  DynParams dp;
  const void *x, *u, *dF, *df;
  void *first, *second;           // [T-1, B, NP] each; either may be NULL
};

// Vector-Jacobian product of dyn_linearize_kernel in theta, one thread per (t, problem), t < T-1.  With z = [x; u],
// J = dx'/dz and f = x' - J z at (x[t,b], u[t,b]):
//   first[t,b,k]  = sum_r df_r dx'_r/dtheta_k                        (J held constant: the reference's gradient)
//   second[t,b,k] = sum_{r,j} (dF_rj - df_r z_j) dJ_rj/dtheta_k      (what J's own dependence on theta adds)
// so first + second = d/dtheta_k (<dF, J> + <df, f>).  One pass per theta_k over the nested dual Dual<Dual<R, P>, 1>:
// the inner dual is the Jacobian dyn_linearize_kernel forms, the outer one carries d/dtheta_k, so its derivative part
// holds dx'/dtheta_k and dJ/dtheta_k.  The clamp follows dclamp: a saturated control has no u column at any order.
template <typename R, int KIND>
__global__ void __launch_bounds__(128) dyn_linearize_vjp_kernel(const DynVjpArgs a) {
  constexpr int N = DynDims<KIND>::N, M = DynDims<KIND>::M, P = N + M, NP = DynLearnable<KIND>::NP;
  static_assert(M == 1, "the known systems have one control");
  using D2 = Dual<Dual<R, P>, 1>;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)(a.T - 1) * a.B) return;
  const R* gdF = (const R*)a.dF + i * N * P;
  const R* gdf = (const R*)a.df + i * N;
  R z[P];
#pragma unroll
  for (int k = 0; k < N; ++k) z[k] = ((const R*)a.x)[i * N + k];
  z[N] = ((const R*)a.u)[i * M];
#pragma unroll 1
  for (int k = 0; k < NP; ++k) {
    D2 s[N], o[N], u;
#pragma unroll
    for (int j = 0; j < N; ++j) {
      s[j].v = dual_var<R, P>(z[j], j);
      s[j].d[0] = dual_const<R, P>(R(0));
    }
    u.v = dual_var<R, P>(z[N], N);
    u.d[0] = dual_const<R, P>(R(0));
    dyn_step<R, KIND, D2, D2>(a.dp, s, u, o, k);
    R first = R(0), second = R(0);
#pragma unroll
    for (int r = 0; r < N; ++r) {
      const R dfr = gdf[r];
      first += dfr * o[r].d[0].v;
#pragma unroll
      for (int j = 0; j < P; ++j) second += (gdF[r * P + j] - dfr * z[j]) * o[r].d[0].d[j];
    }
    if (a.first != nullptr) ((R*)a.first)[i * NP + k] = first;
    if (a.second != nullptr) ((R*)a.second)[i * NP + k] = second;
  }
}

template <typename R>
int launch_dyn_rollout(const DynArgs& a, cudaStream_t stream) {
  const int grid = (a.B + 127) / 128;
  constexpr int CP = DYN_CARTPOLE | DYN_CTRL_PASSTHROUGH, PP = DYN_PENDULUM | DYN_CTRL_PASSTHROUGH,
                FP = DYN_PENDULUM_FULL | DYN_CTRL_PASSTHROUGH;
  if (a.kind == DYN_CARTPOLE) dyn_rollout_kernel<R, DYN_CARTPOLE><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == DYN_PENDULUM) dyn_rollout_kernel<R, DYN_PENDULUM><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == DYN_PENDULUM_FULL) dyn_rollout_kernel<R, DYN_PENDULUM_FULL><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == CP) dyn_rollout_kernel<R, CP><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == PP) dyn_rollout_kernel<R, PP><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == FP) dyn_rollout_kernel<R, FP><<<grid, 128, 0, stream>>>(a);
  else return 2;
  return cudaGetLastError() == cudaSuccess ? 0 : 5;
}
template <typename R>
int launch_dyn_linearize(const DynArgs& a, cudaStream_t stream) {
  const size_t items = (size_t)(a.T - 1) * a.B;
  if (items == 0) return 0;
  const int grid = (int)((items + 127) / 128);
  constexpr int CP = DYN_CARTPOLE | DYN_CTRL_PASSTHROUGH, PP = DYN_PENDULUM | DYN_CTRL_PASSTHROUGH,
                FP = DYN_PENDULUM_FULL | DYN_CTRL_PASSTHROUGH;
  if (a.kind == DYN_CARTPOLE) dyn_linearize_kernel<R, DYN_CARTPOLE><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == DYN_PENDULUM) dyn_linearize_kernel<R, DYN_PENDULUM><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == DYN_PENDULUM_FULL) dyn_linearize_kernel<R, DYN_PENDULUM_FULL><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == CP) dyn_linearize_kernel<R, CP><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == PP) dyn_linearize_kernel<R, PP><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == FP) dyn_linearize_kernel<R, FP><<<grid, 128, 0, stream>>>(a);
  else return 2;
  return cudaGetLastError() == cudaSuccess ? 0 : 5;
}
// the VJP of the linearisation of a known system (no passthrough kinds: the slew-rate tail linearises the system;
// the reverse sweep of a slew-rate episode instantiates the kernel at a passthrough kind itself, episode_grad.cu)
template <typename R>
int launch_dyn_linearize_vjp(const DynVjpArgs& a, cudaStream_t stream) {
  const size_t items = (size_t)(a.T - 1) * a.B;
  if (a.kind != DYN_CARTPOLE && a.kind != DYN_PENDULUM && a.kind != DYN_PENDULUM_FULL) return 2;
  if (items == 0) return 0;
  const int grid = (int)((items + 127) / 128);
  if (a.kind == DYN_CARTPOLE) dyn_linearize_vjp_kernel<R, DYN_CARTPOLE><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == DYN_PENDULUM) dyn_linearize_vjp_kernel<R, DYN_PENDULUM><<<grid, 128, 0, stream>>>(a);
  else dyn_linearize_vjp_kernel<R, DYN_PENDULUM_FULL><<<grid, 128, 0, stream>>>(a);
  return cudaGetLastError() == cudaSuccess ? 0 : 5;
}

}  // namespace mpcb200
