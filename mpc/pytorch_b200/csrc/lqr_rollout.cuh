// lqr_rollout.cuh - nominal trajectory x[t+1] = F[t] [x[t]; u[t]] + f[t] for LinDx dynamics (sm_90a).
//
// Replaces util.get_traj for LinDx (reference mpc/util.py:102-126: T-1 bmm/cat/add launches per iLQR
// iteration) with ONE launch.  N lanes per problem (lane r owns state component r and row r of F),
// 32/N problems per warp; tau_t is replicated with shuffles; row r of F[t+1] is fetched while step t
// computes.  Streams F once: bytes/problem = 4[(T-1) n p + (T-1) n + n + T m] read + 4 T n written.
#pragma once
#include "common.cuh"

namespace mpcb200 {

struct RolloutArgs {
  int B, T, has_f;
  const void *F, *f, *x_init, *u;
  void* x;
  long long F_ts, f_ts;   // elements between consecutive time slices of F, f (0 = time invariant)
};

template <typename R, int N, int M>
struct RolloutCfg {
  static constexpr int P = N + M;
  static constexpr int LP = N;
  static constexpr int PPW = 32 / LP;
  static constexpr int NW = 4;
  static constexpr int W = NW * PPW;
  static constexpr int THREADS = NW * 32;
};

template <typename R, int N, int M>
__global__ void __launch_bounds__(RolloutCfg<R, N, M>::THREADS)
lqr_rollout_kernel(const RolloutArgs a) {
  using K = RolloutCfg<R, N, M>;
  constexpr int P = K::P, LP = K::LP, PPW = K::PPW;
  const int T = a.T, B = a.B;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool writer_lane = lane < PPW * LP;
  const int pi = writer_lane ? lane / LP : PPW - 1;
  const int base = pi * LP;
  const int r = writer_lane ? lane - base : LP - 1;
  const int b = (blockIdx.x * K::NW + warp) * PPW + pi;
  const bool valid = b < B;
  const bool wr = writer_lane && valid;
  const int bb = valid ? b : 0;
  const R* gF = (const R*)a.F;
  const R* gf = (const R*)a.f;
  const R* gu = (const R*)a.u;
  R* gx = (R*)a.x;

  struct Tile {
    R row[P], fr, uu[M];  // row r of F[t], f[t][r], u[t][:] (replicated)
  };
  auto fetch = [&](int t, Tile& o) {
    const size_t tb = (size_t)t * B + bb;
    const R* Fr = gF + (size_t)t * a.F_ts + ((size_t)bb * N + r) * P;
#pragma unroll
    for (int i = 0; i < P; ++i) o.row[i] = __ldg(Fr + i);
    o.fr = a.has_f ? __ldg(gf + (size_t)t * a.f_ts + (size_t)bb * N + r) : R(0);
#pragma unroll
    for (int q = 0; q < M; ++q) o.uu[q] = __ldg(gu + tb * M + q);
  };
  R xr = __ldg((const R*)a.x_init + (size_t)bb * N + r);
  if (wr) gx[(size_t)bb * N + r] = xr;
  Tile cur, nxt;
  if (T > 1) fetch(0, cur);
  for (int t = 0; t < T - 1; ++t) {
    if (t + 1 < T - 1) fetch(t + 1, nxt);
    R acc = cur.fr;
#pragma unroll
    for (int i = 0; i < N; ++i) acc += cur.row[i] * shfl(xr, base + i);
#pragma unroll
    for (int q = 0; q < M; ++q) acc += cur.row[N + q] * cur.uu[q];
    xr = acc;
    if (wr) gx[((size_t)(t + 1) * B + b) * N + r] = xr;
    if (t + 1 < T - 1) cur = nxt;
  }
}

template <typename R, int N, int M>
int launch_rollout(const RolloutArgs& a, cudaStream_t stream) {
  using K = RolloutCfg<R, N, M>;
  const int grid = (a.B + K::W - 1) / K::W;
  lqr_rollout_kernel<R, N, M><<<grid, K::THREADS, 0, stream>>>(a);
  return cudaGetLastError() == cudaSuccess ? 0 : 5;
}

}  // namespace mpcb200
