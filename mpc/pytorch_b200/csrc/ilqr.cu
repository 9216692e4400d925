// ilqr.cu - launchers of the bookkeeping kernels of the device-side iLQR loop and of the receding-horizon episode
// around it (ilqr.cuh), in a module of their own.
#include "ilqr.cuh"

namespace mpcb200 {

static unsigned ilqr_grid(size_t items) {   // grid-stride kernels: enough blocks to cover `items`, at most 4096
  const size_t g = (items + 255) / 256;
  return (unsigned)(g < 1 ? 1 : (g > 4096 ? 4096 : g));
}

static int launched() { return cudaGetLastError() == cudaSuccess ? MPCB200_OK : MPCB200_ERR_LAUNCH; }

template <typename R>
int ilqr_launch_init(size_t n_u, const R* u_init, R* u, IlqrState* st, int32_t* info,
                     cudaGraphConditionalHandle handle, cudaStream_t stream) {
  ilqr_init_kernel<R><<<ilqr_grid(n_u), 256, 0, stream>>>(n_u, u_init, u, st, info, handle);
  return launched();
}

template <typename R>
int episode_launch_init(size_t n_x, size_t n_u, const R* x_init, const R* u_init, R* state, R* xs0, R* warm,
                        EpisodeState* ep, cudaGraphConditionalHandle handle, cudaStream_t stream) {
  episode_init_kernel<R><<<ilqr_grid(n_x > n_u ? n_x : n_u), 256, 0, stream>>>(n_x, n_u, x_init, u_init, state, xs0,
                                                                               warm, ep, handle);
  return launched();
}

template <typename R>
int episode_launch_advance(int B, int T, int N, int M, int m_ref, int n_steps, const R* traj, const R* best_u,
                           const R* best_costs, const int32_t* info, const R* w, R* state, R* warm, R* xs, R* us,
                           R* costs, int32_t* info_out, EpisodeState* ep, cudaGraphConditionalHandle handle,
                           cudaStream_t stream) {
  const unsigned grid = ilqr_grid((size_t)T * B * (N > M ? N : M));
  if (w == nullptr)
    episode_advance_kernel<R><<<grid, 256, 0, stream>>>(B, T, N, M, m_ref, n_steps, traj, best_u, best_costs, info,
                                                        state, warm, xs, us, costs, info_out, ep, handle);
  else
    episode_advance_disturbed_kernel<R><<<grid, 256, 0, stream>>>(B, T, N, M, m_ref, n_steps, traj, best_u,
                                                                  best_costs, info, w, state, warm, xs, us, costs,
                                                                  info_out, ep, handle);
  return launched();
}

template <typename R>
int ilqr_launch_track(int B, int T, int N, int M, int m_ref, R best_cost_eps, const R* new_x, const R* new_u,
                      const R* costs, const R* du_first, const int32_t* status, const R* best_costs, R* best_x,
                      R* best_u, R* u, R* fdn, uint8_t* flags, const IlqrState* st, cudaStream_t stream) {
  ilqr_track_kernel<R><<<ilqr_grid((size_t)T * B * (N > M ? N : M)), 256, 0, stream>>>(
      B, T, N, M, m_ref, best_cost_eps, new_x, new_u, costs, du_first, status, best_costs, best_x, best_u, u, fdn,
      flags, st);
  return launched();
}

template <typename R>
int ilqr_launch_stop(int B, int lqr_iter, int not_improved_lim, double eps, const R* costs, const R* fdn,
                     const uint8_t* flags, R* best_costs, R* best_fdn, IlqrState* st, int32_t* info,
                     cudaGraphConditionalHandle handle, cudaStream_t stream) {
  ilqr_stop_kernel<R><<<1, ILQR_STOP_THREADS, 0, stream>>>(B, lqr_iter, not_improved_lim, eps, costs, fdn, flags,
                                                           best_costs, best_fdn, st, info, handle);
  return launched();
}

#define MPCB200_ILQR_INST(R)                                                                                       \
  template int ilqr_launch_init<R>(size_t, const R*, R*, IlqrState*, int32_t*, cudaGraphConditionalHandle,        \
                                   cudaStream_t);                                                                  \
  template int episode_launch_init<R>(size_t, size_t, const R*, const R*, R*, R*, R*, EpisodeState*,              \
                                      cudaGraphConditionalHandle, cudaStream_t);                                   \
  template int episode_launch_advance<R>(int, int, int, int, int, int, const R*, const R*, const R*,              \
                                         const int32_t*, const R*, R*, R*, R*, R*, R*, int32_t*, EpisodeState*,    \
                                         cudaGraphConditionalHandle, cudaStream_t);                                \
  template int ilqr_launch_track<R>(int, int, int, int, int, R, const R*, const R*, const R*, const R*,            \
                                    const int32_t*, const R*, R*, R*, R*, R*, uint8_t*, const IlqrState*,          \
                                    cudaStream_t);                                                                 \
  template int ilqr_launch_stop<R>(int, int, int, double, const R*, const R*, const uint8_t*, R*, R*, IlqrState*, \
                                   int32_t*, cudaGraphConditionalHandle, cudaStream_t);
MPCB200_ILQR_INST(float)
MPCB200_ILQR_INST(double)
#undef MPCB200_ILQR_INST

}  // namespace mpcb200
