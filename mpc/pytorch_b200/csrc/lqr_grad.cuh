// lqr_grad.cuh - gradient assembly of the KKT adjoint (sm_90a).
//
// Replaces the second half of LQRStepFn.backward (reference mpc/lqr_step.py:342-404):
// costates lambda_t / dlambda_t (backward in t), then
//   dC_t = -1/2 (dtau tau' + tau dtau'), dc_t = -dtau_t,
//   dF_t = -(dlam_{t+1} tau_t' + lam_{t+1} dtau_t'), df_t = -dlam_{t+1}, dx_init = -dlam_0.
// The adjoint solve that produces (dx,du) is the step kernel in masked mode (lqr_step.cuh).
//
// Mapping: P = n+m lanes per problem (lane j holds tau_j, dtau_j; lanes j<n hold lambda_j,
// dlambda_j), 32/P problems per warp.  The outer products are store bound (dC,dF dominate), so
// they are written with a FLAT index over the warp's contiguous problems: every store
// instruction covers one fully used 128-byte line; operands come from warp shuffles.
#pragma once
#include "common.cuh"

namespace mpcb200 {

struct GradArgs {
  int B, T, F_T, has_df;
  const void *C, *c, *F, *new_x, *new_u, *dx, *du, *dl_dx;
  void *dx_init, *dC, *dc, *dF, *df;
  void* workspace;   // 2*T*B*n elements: lambda_t, dlambda_t
  long long C_ts, c_ts, F_ts;   // elements between consecutive time slices of C, c, F (0 = time invariant)
};

template <typename R, int N, int M>
struct GradCfg {
  static constexpr int P = N + M;
  static constexpr int LP = P;
  static constexpr int PPW = 32 / LP;
  static constexpr int NW = 4;
  static constexpr int W = NW * PPW;
  static constexpr int THREADS = NW * 32;
  static constexpr int TCHUNK = 4;        // time steps per warp in the outer-product kernel
};

// ---------------------------------------------------------------------------------------------
// Two kernels, through the caller's workspace of 2*T*B*n elements:
//   1. lqr_costate_kernel: the sequential part - lambda_t, dlambda_t backward in t (reference
//      :355-385), next step's operands prefetched into registers; writes the costates to the
//      workspace plus dx_init and df.
//   2. lqr_outer_kernel: dC, dc, dF for every (t, b) independently (reference :346-353,387-395) -
//      T x more parallelism than a loop over t, a pure streaming-store kernel.
// ---------------------------------------------------------------------------------------------
template <typename R, int N, int M>
__global__ void __launch_bounds__(GradCfg<R, N, M>::THREADS)
lqr_costate_kernel(const GradArgs a) {
  using K = GradCfg<R, N, M>;
  constexpr int P = K::P, LP = K::LP, PPW = K::PPW;
  const int T = a.T, B = a.B;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool writer_lane = lane < PPW * LP;
  const int pi = writer_lane ? lane / LP : PPW - 1;
  const int base = pi * LP;
  const int j = writer_lane ? lane - base : LP - 1;
  const int b = (blockIdx.x * K::NW + warp) * PPW + pi;
  const bool valid = b < B;
  const bool wr = writer_lane && valid;
  const int bb = valid ? b : 0;
  const bool is_x = j < N;
  const int jr = is_x ? j : N - 1;
  const R* gC = (const R*)a.C;
  const R* gc = (const R*)a.c;
  const R* gF = (const R*)a.F;
  const R* gx = (const R*)a.new_x;
  const R* gu = (const R*)a.new_u;
  const R* gdx = (const R*)a.dx;
  const R* gdu = (const R*)a.du;
  const R* grx = (const R*)a.dl_dx;
  R* wl = (R*)a.workspace;
  R* wd = wl + (size_t)T * B * N;
  R* of = (R*)a.df;

  struct Tile {
    R crow[P], fcol[N], tj, dj, cx, rx;
  };
  auto fetch = [&](int t, Tile& o) {
    const size_t tb = (size_t)t * B + bb;
    o.tj = is_x ? __ldg(gx + tb * N + j) : __ldg(gu + tb * M + (j - N));
    o.dj = is_x ? __ldg(gdx + tb * N + j) : __ldg(gdu + tb * M + (j - N));
    const R* Crow = gC + (size_t)t * a.C_ts + ((size_t)bb * P + jr) * P;
#pragma unroll
    for (int i = 0; i < P; ++i) o.crow[i] = __ldg(Crow + i);
    o.cx = __ldg(gc + (size_t)t * a.c_ts + (size_t)bb * P + jr);
    o.rx = __ldg(grx + tb * N + jr);
    if (t < T - 1) {
      const R* Fc = gF + (size_t)t * a.F_ts + (size_t)bb * N * P + jr;
#pragma unroll
      for (int k = 0; k < N; ++k) o.fcol[k] = __ldg(Fc + k * P);
    }
  };
  R lam = R(0), dlam = R(0);
  auto compute = [&](int t, const Tile& cur) {
    R nl = cur.cx, ndl = -cur.rx;
#pragma unroll
    for (int i = 0; i < P; ++i) {
      nl += cur.crow[i] * shfl(cur.tj, base + i);
      ndl += cur.crow[i] * shfl(cur.dj, base + i);
    }
    if (t < T - 1) {
#pragma unroll
      for (int k = 0; k < N; ++k) {
        nl += cur.fcol[k] * shfl(lam, base + k);
        ndl += cur.fcol[k] * shfl(dlam, base + k);
      }
      if (a.has_df && wr && is_x) of[((size_t)t * B + b) * N + j] = -dlam;   // df_t = -dlambda_{t+1}
    }
    lam = nl;
    dlam = ndl;
    if (wr && is_x) {
      wl[((size_t)t * B + b) * N + j] = lam;
      wd[((size_t)t * B + b) * N + j] = dlam;
    }
  };
  // register ring of three tiles: operands of steps t-1 and t-2 are in flight while step t computes
  Tile r0, r1, r2;
  fetch(T - 1, r0);
  if (T > 1) fetch(T - 2, r1);
  for (int t = T - 1; t >= 0; t -= 3) {
    if (t - 2 >= 0) fetch(t - 2, r2);
    compute(t, r0);
    if (t - 1 < 0) break;
    if (t - 3 >= 0) fetch(t - 3, r0);
    compute(t - 1, r1);
    if (t - 2 < 0) break;
    if (t - 4 >= 0) fetch(t - 4, r1);
    compute(t - 2, r2);
  }
  if (wr && is_x) ((R*)a.dx_init)[(size_t)b * N + j] = -dlam;
}

template <typename R, int N, int M>
__global__ void __launch_bounds__(GradCfg<R, N, M>::THREADS)
lqr_outer_kernel(const GradArgs a) {
  using K = GradCfg<R, N, M>;
  constexpr int P = K::P, LP = K::LP, PPW = K::PPW;
  constexpr int TC = K::TCHUNK;                           // time steps handled by one warp
  const int T = a.T, B = a.B;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int groups = (B + PPW - 1) / PPW;                // problem groups (one warp-load each)
  const int tchunks = (T + TC - 1) / TC;
  const long long item = (long long)blockIdx.x * K::NW + warp;
  if (item >= (long long)groups * tchunks) return;
  const int tch = (int)(item / groups);
  const int bw0 = (int)(item - (long long)tch * groups) * PPW;
  const bool writer_lane = lane < PPW * LP;
  const int pi = writer_lane ? lane / LP : PPW - 1;
  const int j = writer_lane ? lane - pi * LP : LP - 1;
  const int b = bw0 + pi;
  const bool valid = b < B;
  const int bb = valid ? b : 0;
  const bool is_x = j < N;
  const int jr = is_x ? j : N - 1;
  const int nprob = min(PPW, B - bw0);
  R* oC = (R*)a.dC;
  R* oF = (R*)a.dF;
  const R* wl = (const R*)a.workspace;
  const R* wd = wl + (size_t)T * B * N;

  // flat-index decode (loop invariant): source lanes of the two factors of every stored element
  constexpr int TOTC = PPW * P * P, RC = (TOTC + 31) / 32;
  constexpr int TOTF = PPW * N * P, RF = (TOTF + 31) / 32;
  int cI[RC], cJ[RC], fK[RF], fJ[RF];
  unsigned okC = 0u, okF = 0u;
#pragma unroll
  for (int rr = 0; rr < RC; ++rr) {
    const int e = rr * 32 + lane, ec = e < TOTC ? e : TOTC - 1;
    const int pe = ec / (P * P), r = ec - pe * (P * P);
    cI[rr] = pe * LP + r / P;
    cJ[rr] = pe * LP + r % P;
    if (e < TOTC && pe < nprob) okC |= 1u << rr;
  }
#pragma unroll
  for (int rr = 0; rr < RF; ++rr) {
    const int e = rr * 32 + lane, ec = e < TOTF ? e : TOTF - 1;
    const int pe = ec / (N * P), r = ec - pe * (N * P);
    fK[rr] = pe * LP + r / P;
    fJ[rr] = pe * LP + r % P;
    if (e < TOTF && pe < nprob) okF |= 1u << rr;
  }
  static_assert(RC <= 32 && RF <= 32, "decode masks are 32 bit");

  const int t_end = min(T, (tch + 1) * TC);
  for (int t = tch * TC; t < t_end; ++t) {
    const size_t tb = (size_t)t * B + bb;
    const R tj = is_x ? __ldg((const R*)a.new_x + tb * N + j) : __ldg((const R*)a.new_u + tb * M + (j - N));
    const R dj = is_x ? __ldg((const R*)a.dx + tb * N + j) : __ldg((const R*)a.du + tb * M + (j - N));
    R lam = R(0), dlam = R(0);
    if (t < T - 1) {
      const size_t t1 = (size_t)(t + 1) * B + bb;
      lam = __ldg(wl + t1 * N + jr);
      dlam = __ldg(wd + t1 * N + jr);
    }
    if (writer_lane && valid) ((R*)a.dc)[tb * P + j] = -dj;
    R* pC = oC + ((size_t)t * B + bw0) * P * P + lane;
#pragma unroll
    for (int rr = 0; rr < RC; ++rr) {
      const R ti = shfl(tj, cI[rr]), di = shfl(dj, cI[rr]);
      const R tc = shfl(tj, cJ[rr]), dcc = shfl(dj, cJ[rr]);
      if ((okC >> rr) & 1u) pC[rr * 32] = R(-0.5) * (di * tc + ti * dcc);
    }
    if (t < T - 1) {
      R* pF = oF + ((size_t)t * B + bw0) * N * P + lane;
#pragma unroll
      for (int rr = 0; rr < RF; ++rr) {
        const R dl = shfl(dlam, fK[rr]), l = shfl(lam, fK[rr]);
        const R tc = shfl(tj, fJ[rr]), dc_ = shfl(dj, fJ[rr]);
        if ((okF >> rr) & 1u) pF[rr * 32] = -(dl * tc + l * dc_);
      }
    } else if (a.F_T == T) {
      R* pF = oF + ((size_t)t * B + bw0) * N * P + lane;
#pragma unroll
      for (int rr = 0; rr < RF; ++rr)
        if ((okF >> rr) & 1u) pF[rr * 32] = R(0);
    }
  }
}

template <typename R, int N, int M>
int launch_grad(const GradArgs& a, cudaStream_t stream) {
  using K = GradCfg<R, N, M>;
  const int grid = (a.B + K::W - 1) / K::W;
  lqr_costate_kernel<R, N, M><<<grid, K::THREADS, 0, stream>>>(a);
  if (cudaGetLastError() != cudaSuccess) return MPCB200_ERR_LAUNCH;
  const long long items = (long long)((a.B + K::PPW - 1) / K::PPW) * ((a.T + K::TCHUNK - 1) / K::TCHUNK);
  const int grid2 = (int)((items + K::NW - 1) / K::NW);
  lqr_outer_kernel<R, N, M><<<grid2, K::THREADS, 0, stream>>>(a);
  return cudaGetLastError() == cudaSuccess ? MPCB200_OK : MPCB200_ERR_LAUNCH;
}

}  // namespace mpcb200
