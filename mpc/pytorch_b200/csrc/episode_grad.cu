// episode_grad.cu - the kernels of an episode's reverse sweep (episode_grad.cuh) and their launchers, in a module of
// their own: the init and accumulate kernels call the device runtime's cudaGraphSetConditional.
#include "episode_grad.cuh"

namespace mpcb200 {

static unsigned epgrad_grid(size_t items) {   // grid-stride kernels: enough blocks to cover `items`, at most 4096
  const size_t g = (items + 255) / 256;
  return (unsigned)(g < 1 ? 1 : (g > 4096 ? 4096 : g));
}
static int launched() { return cudaGetLastError() == cudaSuccess ? MPCB200_OK : MPCB200_ERR_LAUNCH; }

// plan_x[k] = best_x, plan_u[k] = best_u for the control step k = ep->step (before episode_advance_kernel moves it)
template <typename R>
__global__ void __launch_bounds__(256)
episode_plans_kernel(size_t n_x, size_t n_u, const R* __restrict__ best_x, const R* __restrict__ best_u,
                     R* __restrict__ plan_x, R* __restrict__ plan_u, const EpisodeState* __restrict__ ep) {
  const size_t k = (size_t)ep->step;
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  for (size_t i = i0; i < n_x; i += step) plan_x[k * n_x + i] = best_x[i];
  for (size_t i = i0; i < n_u; i += step) plan_u[k * n_u + i] = best_u[i];
}

template <typename R>
__global__ void __launch_bounds__(256) fill_zero_kernel(size_t n, R* __restrict__ p) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    p[i] = R(0);
}

// slices k .. k+n-1 of each windowed input into its fixed buffer (WindowCopy, episode_grad.cuh)
template <typename R>
__global__ void __launch_bounds__(256) window_stage_kernel(const WindowCopy<R> w) {
  const long long k = *w.k;
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
#pragma unroll 1
  for (int a = 0; a < WINDOW_INPUTS; ++a) {
    if (w.src[a] == nullptr) continue;
    const size_t slice = (size_t)w.slice[a], len = (size_t)w.n[a] * slice;
    const long long ts = w.tstride[a];
    const R* __restrict__ src = w.src[a] + (ts < 0 ? 0 : k * ts);
    R* __restrict__ dst = w.dst[a];
    for (size_t i = i0; i < len; i += step) {
      const size_t t = i / slice, j = i - t * slice;
      dst[i] = src[ts < 0 ? j : t * (size_t)ts + j];
    }
  }
}

// g = dl_dxs[n_steps]; the accumulators and the adjoint's incoming gradients zeroed; k = n_steps - 1; the loop's
// handle set to 1.  DETACH (a slew-rate episode): g's first n_prev entries, the previous control, are 0.  PLANT:
// the plant's accumulators zeroed too, and dw[n_steps-1] = g
// WINDOW: the full-length outputs of EpWindow are zeroed over their whole length.
template <typename R, bool DETACH, bool PLANT, bool WINDOW = false>
__device__ __forceinline__ void epgrad_init_body(const EpGradArgs<R>& a, int n_prev, const EpPlantArgs<R>& pl,
                                                 cudaGraphConditionalHandle handle, const EpWindow& wn = EpWindow{}) {
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  const size_t B = a.B, T = a.T, N = a.N, M = a.M, P = N + M;
  for (size_t i = i0; i < B * N; i += step) {
    const R v = DETACH && i % N < (size_t)n_prev ? R(0) : a.dl_dxs[(size_t)a.n_steps * B * N + i];
    a.g[i] = v;
    if (PLANT && pl.dw != nullptr) pl.dw[(size_t)(a.n_steps - 1) * B * N + i] = v;
  }
  if constexpr (WINDOW) {             // the full-length outputs over their whole length
    const size_t tC = wn.cost ? (size_t)wn.L : T, tp = PLANT && wn.step ? (size_t)wn.Lp : 1;
    const size_t tF = wn.dyn ? (size_t)wn.LF : (size_t)a.F_T, tf = wn.dyn ? (size_t)wn.Lf : T - 1;
    if (PLANT) {
      if (pl.kind == DYN_LINEAR) {
        for (size_t i = i0; i < tp * B * N * P; i += step) pl.dF[i] = R(0);
        if (pl.has_f)
          for (size_t i = i0; i < tp * B * N; i += step) pl.df[i] = R(0);
      } else {
        for (size_t i = i0; i < B * pl.NP; i += step) pl.dtheta[i] = R(0);
      }
    }
    for (size_t i = i0; i < tC * B * P * P; i += step) a.dC[i] = R(0);
    for (size_t i = i0; i < tC * B * P; i += step) a.dc[i] = R(0);
    for (size_t i = i0; i < T * B * N; i += step) a.dl_dx[i] = R(0);
    for (size_t i = i0; i < T * B * M; i += step) a.dl_du[i] = R(0);
    if (a.kind == DYN_LINEAR) {
      for (size_t i = i0; i < tF * B * N * P; i += step) a.dF[i] = R(0);
      if (a.has_f)
        for (size_t i = i0; i < tf * B * N; i += step) a.df[i] = R(0);
    } else {
      for (size_t i = i0; i < B * a.NP; i += step) a.dtheta[i] = R(0);
    }
  } else {
    if (PLANT) {
      if (pl.kind == DYN_LINEAR) {
        for (size_t i = i0; i < B * N * P; i += step) pl.dF[i] = R(0);
        if (pl.has_f)
          for (size_t i = i0; i < B * N; i += step) pl.df[i] = R(0);
      } else {
        for (size_t i = i0; i < B * pl.NP; i += step) pl.dtheta[i] = R(0);
      }
    }
    for (size_t i = i0; i < T * B * P * P; i += step) a.dC[i] = R(0);
    for (size_t i = i0; i < T * B * P; i += step) a.dc[i] = R(0);
    for (size_t i = i0; i < T * B * N; i += step) a.dl_dx[i] = R(0);
    for (size_t i = i0; i < T * B * M; i += step) a.dl_du[i] = R(0);
    if (a.kind == DYN_LINEAR) {
      for (size_t i = i0; i < (size_t)a.F_T * B * N * P; i += step) a.dF[i] = R(0);
      if (a.has_f)
        for (size_t i = i0; i < (T - 1) * B * N; i += step) a.df[i] = R(0);
    } else {
      for (size_t i = i0; i < B * a.NP; i += step) a.dtheta[i] = R(0);
    }
  }
  if (i0 == 0) {
    a.st->k = a.n_steps - 1; a.st->tickets = 0u; a.st->reserved[0] = a.st->reserved[1] = 0;
    cudaGraphSetConditional(handle, 1);
  }
}
template <typename R>
__global__ void __launch_bounds__(256) epgrad_init_kernel(const EpGradArgs<R> a, cudaGraphConditionalHandle handle) {
  epgrad_init_body<R, false, false>(a, 0, EpPlantArgs<R>{}, handle);
}
template <typename R>
__global__ void __launch_bounds__(256)
epgrad_init_detach_kernel(const EpGradArgs<R> a, int n_prev, cudaGraphConditionalHandle handle) {
  epgrad_init_body<R, true, false>(a, n_prev, EpPlantArgs<R>{}, handle);
}
template <typename R>
__global__ void __launch_bounds__(256)
epgrad_init_plant_kernel(const EpGradArgs<R> a, const EpPlantArgs<R> pl, int n_prev,
                         cudaGraphConditionalHandle handle) {
  epgrad_init_body<R, true, true>(a, n_prev, pl, handle);
}
template <typename R, bool PLANT>
__global__ void __launch_bounds__(256)
epgrad_init_window_kernel(const EpGradArgs<R> a, const EpPlantArgs<R> pl, const EpWindow wn, int n_prev,
                          cudaGraphConditionalHandle handle) {
  epgrad_init_body<R, true, PLANT, true>(a, n_prev, pl, handle, wn);
}

// the plan of step k into the fixed buffers the body's launchers read
template <typename R>
__device__ __forceinline__ void epgrad_stage_plan(const EpGradArgs<R>& a, size_t k, size_t i0, size_t step) {
  const size_t nx = (size_t)a.T * a.B * a.N, nu = (size_t)a.T * a.B * a.M;
  for (size_t i = i0; i < nx; i += step) a.stage_x[i] = a.plan_x[k * nx + i];
  for (size_t i = i0; i < nu; i += step) a.stage_u[i] = a.plan_u[k * nu + i];
}

// LinDx: x' = F[0] z + f[0] with z = [x_k; u_k].  One thread per (b, column j of F[0]): column j of F[0]^T g goes
// to gx (j < N) or into dl_du[0] (j >= N), and column j of dF[0] takes g z_j.  WINDOW: F[0] is the staged window's
// F[k], and g z^T, g go into slice k of the full-length dF, df.
template <typename R, bool WINDOW>
__device__ __forceinline__ void epgrad_stage_linear_body(const EpGradArgs<R>& a) {
  const size_t k = (size_t)a.st->k;
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  epgrad_stage_plan(a, k, i0, step);
  const int N = a.N, M = a.M, P = N + M;
  const size_t B = a.B;
  R* const dF = WINDOW ? a.dF + k * B * N * P : a.dF;
  R* const df = WINDOW && a.has_f ? a.df + k * B * N : a.df;
  for (size_t idx = i0; idx < B * P; idx += step) {
    const size_t b = idx / P;
    const int j = (int)(idx % P);
    const R* g = a.g + b * N;
    const R* Fb = a.F + b * N * P;
    R* dFb = dF + b * N * P;
    const R zj = j < N ? a.xs[(k * B + b) * N + j] : a.us[(k * B + b) * M + (j - N)];
    R v = R(0);
    for (int i = 0; i < N; ++i) {
      const R gi = g[i];
      v += Fb[(size_t)i * P + j] * gi;
      dFb[(size_t)i * P + j] += gi * zj;
    }
    if (j < N) a.gx[b * N + j] = v;
    else a.dl_du[b * M + (j - N)] = a.dl_dus[(k * B + b) * M + (j - N)] + v;
    if (a.has_f && j == 0)
      for (int i = 0; i < N; ++i) df[b * N + i] += g[i];
  }
}
template <typename R>
__global__ void __launch_bounds__(256) epgrad_stage_linear_kernel(const EpGradArgs<R> a) {
  epgrad_stage_linear_body<R, false>(a);
}
template <typename R>
__global__ void __launch_bounds__(256) epgrad_stage_linear_window_kernel(const EpGradArgs<R> a) {
  epgrad_stage_linear_body<R, true>(a);
}

// A known system: R, S by the forward-mode duals dyn_linearize_kernel uses, and theta_step = sum_r g_r dx'_r/dtheta
// by the nested duals of dyn_linearize_vjp_kernel (its `first`, with df = g).  One thread per problem.
template <typename R, int KIND>
__global__ void __launch_bounds__(256) epgrad_stage_known_kernel(const EpGradArgs<R> a) {
  constexpr int N = DynDims<KIND>::N, M = DynDims<KIND>::M, P = N + M, NP = DynLearnable<KIND>::NP;
  static_assert(M == 1, "the known systems have one control");
  const size_t k = (size_t)a.st->k;
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  epgrad_stage_plan(a, k, i0, step);
  for (size_t b = i0; b < (size_t)a.B; b += step) {
    R z[P], g[N];
#pragma unroll
    for (int j = 0; j < N; ++j) {
      z[j] = a.xs[(k * a.B + b) * N + j];
      g[j] = a.g[b * N + j];
    }
    z[N] = a.us[k * a.B + b];
    {
      using D = Dual<R, P>;
      D s[N], o[N];
#pragma unroll
      for (int j = 0; j < N; ++j) s[j] = dual_var<R, P>(z[j], j);
      const D u = dual_var<R, P>(z[N], N);
      dyn_step<R, KIND, D>(a.dp, s, u, o);
#pragma unroll
      for (int j = 0; j < P; ++j) {
        R v = R(0);
#pragma unroll
        for (int r = 0; r < N; ++r) v += o[r].d[j] * g[r];
        if (j < N) a.gx[b * N + j] = v;
        else a.dl_du[b] = a.dl_dus[k * a.B + b] + v;
      }
    }
    using D2 = Dual<Dual<R, P>, 1>;
#pragma unroll 1
    for (int p = 0; p < NP; ++p) {
      D2 s[N], o[N], u;
#pragma unroll
      for (int j = 0; j < N; ++j) {
        s[j].v = dual_var<R, P>(z[j], j);
        s[j].d[0] = dual_const<R, P>(R(0));
      }
      u.v = dual_var<R, P>(z[N], N);
      u.d[0] = dual_const<R, P>(R(0));
      dyn_step<R, KIND, D2, D2>(a.dp, s, u, o, p);
      R first = R(0);
#pragma unroll
      for (int r = 0; r < N; ++r) first += g[r] * o[r].d[0].v;
      a.theta_step[b * NP + p] = first;
    }
  }
}

// g = dl_dxs[k] + R^T g + dx_init_k; dC, dc (LinDx: dF, df) += the adjoint's; a known system: dtheta[b] +=
// theta_step[b] + sum_t (first + second)[t, b] in t order.  The last block to finish counts k down and ends the
// loop after k = 0: every block has read st->k by then.  DETACH: g's first n_prev entries are 0, as in init.
// PLANT: theta_step is the plant's and goes into the plant's dtheta, not into the model's; dw[k-1] = g (k > 0).
// WINDOW: step k's dC_k, dc_k (wn.cost) and dF_k, df_k (wn.dyn) go into the full-length outputs at offset k.
template <typename R, bool DETACH, bool PLANT, bool WINDOW = false>
__device__ __forceinline__ void epgrad_accum_body(const EpGradArgs<R>& a, int n_prev, const EpPlantArgs<R>& pl,
                                                  cudaGraphConditionalHandle handle, const EpWindow& wn = EpWindow{}) {
  const int k = a.st->k;
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  const size_t B = a.B, T = a.T, N = a.N, M = a.M, P = N + M;
  for (size_t i = i0; i < B * N; i += step) {
    const R v = DETACH && i % N < (size_t)n_prev ? R(0) : a.dl_dxs[(size_t)k * B * N + i] + a.gx[i] + a.dx_k[i];
    a.g[i] = v;
    if (PLANT && pl.dw != nullptr && k > 0) pl.dw[(size_t)(k - 1) * B * N + i] = v;
  }
  if (PLANT && pl.kind != DYN_LINEAR)
    for (size_t i = i0; i < B * pl.NP; i += step) pl.dtheta[i] += pl.theta_step[i];
  if constexpr (WINDOW) {             // at offset k in the full-length outputs
    const size_t kc = wn.cost ? (size_t)k : 0, kd = wn.dyn ? (size_t)k : 0;
    R* const dC = a.dC + kc * B * P * P;
    R* const dc = a.dc + kc * B * P;
    for (size_t i = i0; i < T * B * P * P; i += step) dC[i] += a.dC_k[i];
    for (size_t i = i0; i < T * B * P; i += step) dc[i] += a.dc_k[i];
    if (a.kind == DYN_LINEAR) {
      R* const dF = a.dF + kd * B * N * P;
      for (size_t i = i0; i < (size_t)a.F_T * B * N * P; i += step) dF[i] += a.dF_k[i];
      if (a.has_f) {
        R* const df = a.df + kd * B * N;
        for (size_t i = i0; i < (T - 1) * B * N; i += step) df[i] += a.df_k[i];
      }
    }
  } else {
    for (size_t i = i0; i < T * B * P * P; i += step) a.dC[i] += a.dC_k[i];
    for (size_t i = i0; i < T * B * P; i += step) a.dc[i] += a.dc_k[i];
  }
  if (a.kind == DYN_LINEAR) {
    if (!WINDOW) {
      for (size_t i = i0; i < (size_t)a.F_T * B * N * P; i += step) a.dF[i] += a.dF_k[i];
      if (a.has_f)
        for (size_t i = i0; i < (T - 1) * B * N; i += step) a.df[i] += a.df_k[i];
    }
  } else {
    const size_t NP = a.NP;
    for (size_t i = i0; i < B * NP; i += step) {
      const size_t b = i / NP, p = i % NP;
      R acc = PLANT ? a.dtheta[i] : a.dtheta[i] + a.theta_step[i];
      for (size_t t = 0; t + 1 < T; ++t) acc += a.first[(t * B + b) * NP + p] + a.second[(t * B + b) * NP + p];
      a.dtheta[i] = acc;
    }
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    __threadfence();
    if (atomicAdd(&a.st->tickets, 1u) == gridDim.x - 1) {
      a.st->tickets = 0u;
      a.st->k = k - 1;
      if (k == 0) cudaGraphSetConditional(handle, 0);
    }
  }
}
template <typename R>
__global__ void __launch_bounds__(256) epgrad_accum_kernel(const EpGradArgs<R> a, cudaGraphConditionalHandle handle) {
  epgrad_accum_body<R, false, false>(a, 0, EpPlantArgs<R>{}, handle);
}
template <typename R>
__global__ void __launch_bounds__(256)
epgrad_accum_detach_kernel(const EpGradArgs<R> a, int n_prev, cudaGraphConditionalHandle handle) {
  epgrad_accum_body<R, true, false>(a, n_prev, EpPlantArgs<R>{}, handle);
}
template <typename R>
__global__ void __launch_bounds__(256)
epgrad_accum_plant_kernel(const EpGradArgs<R> a, const EpPlantArgs<R> pl, int n_prev,
                          cudaGraphConditionalHandle handle) {
  epgrad_accum_body<R, true, true>(a, n_prev, pl, handle);
}
template <typename R, bool PLANT>
__global__ void __launch_bounds__(256)
epgrad_accum_window_kernel(const EpGradArgs<R> a, const EpPlantArgs<R> pl, const EpWindow wn, int n_prev,
                           cudaGraphConditionalHandle handle) {
  epgrad_accum_body<R, true, PLANT, true>(a, n_prev, pl, handle, wn);
}

template <typename R>
int episode_launch_plans(int B, int T, int N, int M, const R* best_x, const R* best_u, R* plan_x, R* plan_u,
                         const EpisodeState* ep, cudaStream_t stream) {
  const size_t nx = (size_t)T * B * N, nu = (size_t)T * B * M;
  episode_plans_kernel<R><<<epgrad_grid(nx > nu ? nx : nu), 256, 0, stream>>>(nx, nu, best_x, best_u, plan_x, plan_u,
                                                                              ep);
  return launched();
}

template <typename R>
int window_launch_stage(const WindowCopy<R>& w, cudaStream_t stream) {
  size_t items = 0;
  for (int a = 0; a < WINDOW_INPUTS; ++a) {
    const size_t len = w.src[a] != nullptr ? (size_t)w.n[a] * (size_t)w.slice[a] : 0;
    if (len > items) items = len;
  }
  window_stage_kernel<R><<<epgrad_grid(items), 256, 0, stream>>>(w);
  return launched();
}

template <typename R>
int launch_fill_zero(size_t n, R* p, cudaStream_t stream) {
  fill_zero_kernel<R><<<epgrad_grid(n), 256, 0, stream>>>(n, p);
  return launched();
}

// the largest grid-stride range of the init and accumulate kernels: dC
template <typename R>
static size_t epgrad_items(const EpGradArgs<R>& a) {
  const size_t P = (size_t)a.N + a.M;
  return (size_t)a.T * a.B * P * P;
}

template <typename R>
int epgrad_launch_init(const EpGradArgs<R>& a, int n_prev, const EpPlantArgs<R>* pl, cudaGraphConditionalHandle handle,
                       cudaStream_t stream) {
  if (pl != nullptr)
    epgrad_init_plant_kernel<R><<<epgrad_grid(epgrad_items(a)), 256, 0, stream>>>(a, *pl, n_prev, handle);
  else if (n_prev == 0) epgrad_init_kernel<R><<<epgrad_grid(epgrad_items(a)), 256, 0, stream>>>(a, handle);
  else epgrad_init_detach_kernel<R><<<epgrad_grid(epgrad_items(a)), 256, 0, stream>>>(a, n_prev, handle);
  return launched();
}

// the largest grid-stride range of the window forms of init and accumulate: dC over the axis
template <typename R>
static size_t epgrad_window_items(const EpGradArgs<R>& a, const EpWindow& wn) {
  const size_t P = (size_t)a.N + a.M;
  return (size_t)(wn.cost ? wn.L : a.T) * a.B * P * P;
}

template <typename R>
int epgrad_launch_init_window(const EpGradArgs<R>& a, int n_prev, const EpPlantArgs<R>* pl, const EpWindow& wn,
                              cudaGraphConditionalHandle handle, cudaStream_t stream) {
  const unsigned grid = epgrad_grid(epgrad_window_items(a, wn));
  if (pl != nullptr) epgrad_init_window_kernel<R, true><<<grid, 256, 0, stream>>>(a, *pl, wn, n_prev, handle);
  else epgrad_init_window_kernel<R, false><<<grid, 256, 0, stream>>>(a, EpPlantArgs<R>{}, wn, n_prev, handle);
  return launched();
}

template <typename R>
int epgrad_launch_accum_window(const EpGradArgs<R>& a, int n_prev, const EpPlantArgs<R>* pl, const EpWindow& wn,
                               cudaGraphConditionalHandle handle, cudaStream_t stream) {
  const unsigned grid = epgrad_grid(epgrad_items(a));
  if (pl != nullptr) epgrad_accum_window_kernel<R, true><<<grid, 256, 0, stream>>>(a, *pl, wn, n_prev, handle);
  else epgrad_accum_window_kernel<R, false><<<grid, 256, 0, stream>>>(a, EpPlantArgs<R>{}, wn, n_prev, handle);
  return launched();
}

template <typename R>
int epgrad_launch_stage_window(const EpGradArgs<R>& a, const EpWindow& wn, cudaStream_t stream) {
  if (a.kind != DYN_LINEAR || !wn.step) return epgrad_launch_stage<R>(a, stream);
  const size_t items = (size_t)a.T * a.B * (a.N > a.M ? a.N : a.M);
  epgrad_stage_linear_window_kernel<R><<<epgrad_grid(items), 256, 0, stream>>>(a);
  return launched();
}

// a passthrough kind runs the system's stage kernel code at its augmented shape: with g's first entry 0 (the detach
// rule), gx = [0; R^T g[1:]], dl_du[0] = dl_dus[k] + S^T g[1:] and theta_step the VJP's `first` with df = g[1:]
template <typename R>
int epgrad_launch_stage(const EpGradArgs<R>& a, cudaStream_t stream) {
  const size_t items = (size_t)a.T * a.B * (a.N > a.M ? a.N : a.M);
  const unsigned grid = epgrad_grid(items);
  constexpr int CP = DYN_CARTPOLE | DYN_CTRL_PASSTHROUGH, PP = DYN_PENDULUM | DYN_CTRL_PASSTHROUGH,
                FP = DYN_PENDULUM_FULL | DYN_CTRL_PASSTHROUGH;
  if (a.kind == DYN_LINEAR) epgrad_stage_linear_kernel<R><<<grid, 256, 0, stream>>>(a);
  else if (a.kind == DYN_CARTPOLE) epgrad_stage_known_kernel<R, DYN_CARTPOLE><<<grid, 256, 0, stream>>>(a);
  else if (a.kind == DYN_PENDULUM) epgrad_stage_known_kernel<R, DYN_PENDULUM><<<grid, 256, 0, stream>>>(a);
  else if (a.kind == DYN_PENDULUM_FULL) epgrad_stage_known_kernel<R, DYN_PENDULUM_FULL><<<grid, 256, 0, stream>>>(a);
  else if (a.kind == CP) epgrad_stage_known_kernel<R, CP><<<grid, 256, 0, stream>>>(a);
  else if (a.kind == PP) epgrad_stage_known_kernel<R, PP><<<grid, 256, 0, stream>>>(a);
  else if (a.kind == FP) epgrad_stage_known_kernel<R, FP><<<grid, 256, 0, stream>>>(a);
  else return MPCB200_ERR_BAD_DIMS;
  return launched();
}

template <typename R>
int epgrad_launch_accum(const EpGradArgs<R>& a, int n_prev, const EpPlantArgs<R>* pl,
                        cudaGraphConditionalHandle handle, cudaStream_t stream) {
  if (pl != nullptr)
    epgrad_accum_plant_kernel<R><<<epgrad_grid(epgrad_items(a)), 256, 0, stream>>>(a, *pl, n_prev, handle);
  else if (n_prev == 0) epgrad_accum_kernel<R><<<epgrad_grid(epgrad_items(a)), 256, 0, stream>>>(a, handle);
  else epgrad_accum_detach_kernel<R><<<epgrad_grid(epgrad_items(a)), 256, 0, stream>>>(a, n_prev, handle);
  return launched();
}

// The linearisation VJP of a passthrough kind, dyn_linearize_vjp_kernel at that kind: the augmented F~ = [[0, 0, I],
// [0, R, S]] depends on theta only through its [1:, 1:] block and f~ only through f~[1:], so the kernel applies the
// system's VJP to the [1:, 1:] block of dF~ and to df~[1:] at x~[1:] (the structural zeros add nothing).  The public
// mpcb200_dyn_linearize_vjp_* keeps taking the systems themselves only (launch_dyn_linearize_vjp).
template <typename R>
int epgrad_launch_vjp_passthrough(const DynVjpArgs& a, cudaStream_t stream) {
  constexpr int CP = DYN_CARTPOLE | DYN_CTRL_PASSTHROUGH, PP = DYN_PENDULUM | DYN_CTRL_PASSTHROUGH,
                FP = DYN_PENDULUM_FULL | DYN_CTRL_PASSTHROUGH;
  const size_t items = (size_t)(a.T - 1) * a.B;
  if (items == 0) return MPCB200_OK;
  const int grid = (int)((items + 127) / 128);
  if (a.kind == CP) dyn_linearize_vjp_kernel<R, CP><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == PP) dyn_linearize_vjp_kernel<R, PP><<<grid, 128, 0, stream>>>(a);
  else if (a.kind == FP) dyn_linearize_vjp_kernel<R, FP><<<grid, 128, 0, stream>>>(a);
  else return MPCB200_ERR_BAD_DIMS;
  return launched();
}

// ---- a learned model's sweep (episode_grad.cuh, EPGRAD_KIND_NET) ----
template <typename R>
__global__ void __launch_bounds__(256) epgrad_plan_kernel(const EpGradArgs<R> a) {
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  epgrad_stage_plan(a, (size_t)a.st->k, i0, step);
}

// One thread per (b, column j of F[0]), as epgrad_stage_linear_body, without the parameter part
template <typename R>
__global__ void __launch_bounds__(256) epgrad_stage_net_kernel(const EpGradArgs<R> a) {
  const size_t k = (size_t)a.st->k;
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  const int N = a.N, M = a.M, P = N + M;
  for (size_t idx = i0; idx < (size_t)a.B * P; idx += step) {
    const size_t b = idx / P;
    const int j = (int)(idx % P);
    const R* g = a.g + b * N;
    const R* Fb = a.F + b * N * P;
    R v = R(0);
    for (int i = 0; i < N; ++i) v += Fb[(size_t)i * P + j] * g[i];
    if (j < N) a.gx[b * N + j] = v;
    else a.dl_du[b * M + (j - N)] = a.dl_dus[(k * a.B + b) * M + (j - N)] + v;
  }
}

// One thread per (b, column j): column j of dF_k[0] += g z_j, and (j = 0) df_k[0] += g
template <typename R>
__global__ void __launch_bounds__(256)
epgrad_net_step_param_kernel(const EpGradArgs<R> a, R* __restrict__ dF_k, R* __restrict__ df_k) {
  const size_t k = (size_t)a.st->k;
  const size_t i0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, step = (size_t)gridDim.x * blockDim.x;
  const int N = a.N, M = a.M, P = N + M;
  for (size_t idx = i0; idx < (size_t)a.B * P; idx += step) {
    const size_t b = idx / P;
    const int j = (int)(idx % P);
    const R* g = a.g + b * N;
    const R zj = j < N ? a.xs[(k * a.B + b) * N + j] : a.us[(k * a.B + b) * M + (j - N)];
    R* dFb = dF_k + b * N * P;
    for (int i = 0; i < N; ++i) dFb[(size_t)i * P + j] += g[i] * zj;
    if (j == 0)
      for (int i = 0; i < N; ++i) df_k[b * N + i] += g[i];
  }
}

template <typename R>
__global__ void __launch_bounds__(256) epgrad_add_kernel(size_t n, const R* __restrict__ src, R* __restrict__ dst) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    dst[i] += src[i];
}

template <typename R>
int epgrad_launch_plan(const EpGradArgs<R>& a, cudaStream_t stream) {
  const size_t items = (size_t)a.T * a.B * (a.N > a.M ? a.N : a.M);
  epgrad_plan_kernel<R><<<epgrad_grid(items), 256, 0, stream>>>(a);
  return launched();
}

template <typename R>
int epgrad_launch_stage_net(const EpGradArgs<R>& a, cudaStream_t stream) {
  epgrad_stage_net_kernel<R><<<epgrad_grid((size_t)a.B * (a.N + a.M)), 256, 0, stream>>>(a);
  return launched();
}

template <typename R>
int epgrad_launch_net_step_param(const EpGradArgs<R>& a, R* dF_k, R* df_k, cudaStream_t stream) {
  epgrad_net_step_param_kernel<R><<<epgrad_grid((size_t)a.B * (a.N + a.M)), 256, 0, stream>>>(a, dF_k, df_k);
  return launched();
}

template <typename R>
int epgrad_launch_add(size_t n, const R* src, R* dst, cudaStream_t stream) {
  epgrad_add_kernel<R><<<epgrad_grid(n), 256, 0, stream>>>(n, src, dst);
  return launched();
}

#define MPCB200_EPGRAD_INST(R)                                                                                     \
  template int epgrad_launch_plan<R>(const EpGradArgs<R>&, cudaStream_t);                                          \
  template int epgrad_launch_stage_net<R>(const EpGradArgs<R>&, cudaStream_t);                                     \
  template int epgrad_launch_net_step_param<R>(const EpGradArgs<R>&, R*, R*, cudaStream_t);                        \
  template int epgrad_launch_add<R>(size_t, const R*, R*, cudaStream_t);                                           \
  template int episode_launch_plans<R>(int, int, int, int, const R*, const R*, R*, R*, const EpisodeState*,        \
                                       cudaStream_t);                                                              \
  template int launch_fill_zero<R>(size_t, R*, cudaStream_t);                                                      \
  template int epgrad_launch_init<R>(const EpGradArgs<R>&, int, const EpPlantArgs<R>*, cudaGraphConditionalHandle, \
                                     cudaStream_t);                                                                \
  template int epgrad_launch_stage<R>(const EpGradArgs<R>&, cudaStream_t);                                         \
  template int epgrad_launch_accum<R>(const EpGradArgs<R>&, int, const EpPlantArgs<R>*,                            \
                                      cudaGraphConditionalHandle, cudaStream_t);                                   \
  template int epgrad_launch_vjp_passthrough<R>(const DynVjpArgs&, cudaStream_t);                                  \
  template int window_launch_stage<R>(const WindowCopy<R>&, cudaStream_t);                                         \
  template int epgrad_launch_init_window<R>(const EpGradArgs<R>&, int, const EpPlantArgs<R>*, const EpWindow&,     \
                                            cudaGraphConditionalHandle, cudaStream_t);                             \
  template int epgrad_launch_accum_window<R>(const EpGradArgs<R>&, int, const EpPlantArgs<R>*, const EpWindow&,    \
                                             cudaGraphConditionalHandle, cudaStream_t);                            \
  template int epgrad_launch_stage_window<R>(const EpGradArgs<R>&, const EpWindow&, cudaStream_t);
MPCB200_EPGRAD_INST(float)
MPCB200_EPGRAD_INST(double)

}  // namespace mpcb200
