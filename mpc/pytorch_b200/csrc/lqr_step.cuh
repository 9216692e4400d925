// lqr_step.cuh - one box-constrained LQR step as ONE persistent-per-CTA kernel (sm_90a).
//
// Replaces the body of LQRStepFn.forward (reference mpc/lqr_step.py:277-309):
//   c_back (:289-295), lqr_backward (:52-160) with pnqp (mpc/pnqp.py:5-82) or the
//   u_zero_I masked solve (:100-127), and lqr_forward's rollout + line search (:164-261).
//
// Mapping (designed for the GPU, not translated from the reference's per-op loop):
//  * LP lanes own one problem, and slot s of lane j owns COLUMN j + s*LP of every p-wide matrix of
//    that problem (Q_t, F_t, C_t) and, for a state column, that column of the value matrix V and of K_t.
//    Most instances have LP = P = n+m and one slot; (8, 2) fp32 has LP = 8 and a second slot on lanes 0, 1
//    for the control columns (StepCfg).  32/LP problems share a warp; NW consumer warps (the smallest
//    count whose spans stay 16-byte aligned: small CTAs = fine load-balance granularity, the batch is
//    < 1 wave; 2 for the (8, 2) layout) + 1 producer warp form a CTA.  The dense products run as pairs
//    of independent FMA chains (common.cuh P2).
//  * the producer warp streams the per-time-step tiles C[t],F[t],c[t],f[t],x_bar[t],u_bar[t]
//    (+ tensor bounds) of the CTA's W consecutive problems - contiguous in the reference's
//    time-major layout - into a 3-stage shared-memory ring with 1-D bulk TMA
//    (cp.async.bulk + mbarrier complete_tx); full/empty mbarriers pace it.  Shapes whose
//    spans are not 16-byte aligned take a plain-load path in the same warp.
//  * V (n x n, stored transposed), v, K_t and Q_xu live in a per-problem shared scratch and are re-read as
//    broadcast vector loads; the m x m solve / pnqp runs redundantly on every lane of the
//    problem from shuffled copies of Q_uu, q_u (registers only, no divergence inside a problem).
//  * K_t,k_t for all t stay in shared memory between the backward sweep and the rollout;
//    the rollout re-streams the tiles (L2 hits, read evict-first) and never round-trips gains through HBM
//    (unless T is too long for shared memory, then a caller-provided Ks/ks buffer is used).
//  * line search: per-problem alpha; a CTA repeats the rollout while any of its problems is
//    worse and iterations remain - per problem this is exactly the reference's batch loop.
//  * MODE (template): PLAIN / BOX (pnqp) / MASK (u_zero_I adjoint solve) - no mode branches at run time.
// This is the GENERIC kernel (any n, m <= 32 lanes, unaligned spans): shapes with even n, m and 16-byte
// aligned tensors run the column-pair kernel in lqr_step2.cuh.  The round-1 experiments that lived here as
// compile-time knobs (two columns per lane, V in registers, padded tiles, mma.sync products, phase timers)
// are listed in DESIGN.md section 7; their code was removed.
#pragma once
#include "../../../include/mpcb200.h"
#include "common.cuh"
#include "dynamics.cuh"

namespace mpcb200 {

struct StepArgs {
  int B, T, F_T;
  int has_f, bounds_kind, has_mask, has_delta, max_ls, pnqp_iters, do_rollout;
  double u_lo, u_hi, delta_u, ls_decay;
  const void *C, *c, *F, *f, *x_init, *cur_x, *cur_u, *u_lower, *u_upper;
  const unsigned char* zero_mask;
  void *new_x, *new_u, *costs, *full_du_norm, *alphas, *du_first;
  int* qp_iters;
  unsigned char* free_mask;
  int* status;
  void *Ks, *ks;
  int bulk_ok;    // host-verified: all tensor bases and per-time-step strides are 16-byte aligned
  int k_in_smem;  // gains of all T steps fit in shared memory
  int impl;       // 0 pick, 1 generic (column per lane), 2 column-pair kernel (lqr_step2.cuh)
  long long C_ts, c_ts, F_ts, f_ts;   // elements between consecutive time slices of C, c, F, f (0 = time invariant)
  // fused KKT adjoint (column-pair kernel only): after the masked solve, a third sweep computes the costates and
  // writes dC, dc, dF, df, dx_init; `c` carries -r, the x_bar/u_bar tile slots carry the forward solution tau*
  int adj, adj_has_df;
  const void *adj_c, *adj_x, *adj_u;
  void *adj_dC, *adj_dc, *adj_dF, *adj_df, *adj_dx_init;
  long long adj_c_ts;
  int dyn_kind;   // true dynamics of the rollout: DYN_LINEAR (F,f) or a known system evaluated in the kernel
  DynParams dp;
};

// the plan (MPCB200_PLAN_* bits) of the step kernel this thread has just launched; read by mpcb200_last_step_plan
void record_step_plan(int plan);

template <typename R, int N, int M>
struct StepCfg {
  static constexpr int P = N + M;
  static constexpr int EA = 16 / (int)sizeof(R);
  static_assert(P <= 32, "one problem must fit a warp");
  // Lane layout.  By default P lanes own one problem, one column each.  (8, 2) in fp32 uses n lanes: lane j
  // keeps state column j, and lanes 0, 1 also keep control columns 8, 9 in a second slot (in the Riccati sweep
  // the control columns are split by rows instead, XS).  A warp then holds
  // 4 problems instead of 3 for about the same broadcast loads of V and F, and shared memory charges for the
  // bytes delivered to lanes, which bound that kernel (DESIGN.md section 7).  fp64 keeps one column per lane:
  // with the second slot it spilled under the 128-register cap of one-warp CTAs (92 B in PLAIN, 184 B in BOX).
  static constexpr bool STATE_LANES = N == 8 && M == 2 && sizeof(R) == 4;
  static constexpr int LP = STATE_LANES ? N : P;    // lanes per problem
  static constexpr int CPL = (P + LP - 1) / LP;     // column slots per lane; slot s of lane j is column j + s*LP
  static constexpr int PPW = 32 / LP;               // problems per warp
  // Slots whose columns the Riccati sweep computes one per lane.  With STATE_LANES only slot 0 does: the control
  // columns are split by rows over the problem's lanes instead (lane j: row j of Q_xu, and row n+ua of Q_uu with q_u[ua]
  // for the control ua of its slot 1), so no lane runs a whole control column and lanes 2..7 no longer compute a dead
  // one.  Each element keeps the FMA chain, and the chain order, of the column it belongs to.
  static constexpr int XS = STATE_LANES ? 1 : CPL;
  static_assert(!STATE_LANES || M == 2, "the row split keeps the two control columns as one pair");
  // slot sl can hold a state column (compile time: the later slots of the (8, 2) layout hold controls only)
  static constexpr bool x_slot(int sl) { return sl * LP < N; }
  // consumer warps per CTA: the smallest count whose per-time-step spans stay 16-byte aligned for every
  // tensor (so the bulk-TMA path applies).  Small CTAs matter: 4096 problems are < 1 wave, and the
  // kernel time is set by the most loaded SM, so the CTA granularity is the load-balance granularity.
  static constexpr bool span_ok(int nw) {
    return (nw * PPW * M * (int)sizeof(R)) % 16 == 0 && (nw * PPW * N * (int)sizeof(R)) % 16 == 0;
  }
  // The (8, 2) layout takes 2 (8 problems): one-warp CTAs measured slower on the H100 (DESIGN.md section 7).
  static constexpr int NW = STATE_LANES ? 2 : span_ok(1) ? 1 : span_ok(2) ? 2 : 4;
  static constexpr int W = NW * PPW;      // problems per CTA
  static_assert(span_ok(NW), "CTA problem count must keep spans 16-byte aligned");
  static constexpr int THREADS = (NW + 1) * 32;
  // resident CTAs per SM that the register budget must allow: config 3 (B = 4096) puts 32 problems on the
  // busiest of 132 SMs, 4 CTAs of the (8, 2) layout
  static constexpr int MIN_CTAS = STATE_LANES ? 32 / W : 0;
  static constexpr int S = 3;             // ring stages
  static constexpr int VS = round_up(N, 4);
  static constexpr int CS = P * P, FS = N * P;     // per-problem strides of the C and F tiles inside a stage
  // stage tile offsets (elements); every sub-tile starts 16-byte aligned (span_ok / padded strides)
  static constexpr int OFF_C = 0;
  static constexpr int OFF_F = OFF_C + W * CS;
  static constexpr int OFF_c = OFF_F + W * FS;
  static constexpr int OFF_f = OFF_c + W * P;
  static constexpr int OFF_x = OFF_f + W * N;
  static constexpr int OFF_u = OFF_x + W * N;
  static constexpr int OFF_lo = OFF_u + W * M;
  static constexpr int OFF_hi = OFF_lo + W * M;
  static constexpr int OFF_END = OFF_hi + W * M;
  static constexpr int STAGE_BYTES = round_up(OFF_END * (int)sizeof(R) + round_up(W * M, 16), 128);
  // per-problem scratch (elements)
  static constexpr int SC_V = 0;                 // N x VS value matrix
  static constexpr int SC_v = SC_V + N * VS;     // VS      value vector
  static constexpr int SC_K = SC_v + VS;         // M x VS (+ M) K_t,k_t exchange when gains are not smem resident
  static constexpr int KT = M * VS + round_up(M, 4);  // elements per (problem, t) of the gain store
  static constexpr int SC_Q = SC_K + KT;         // M x VS  Q_xu exchange (row a = Q[:n, n+a])
  static constexpr int SC_R = SC_Q + M * VS;     // cost reduction
  static constexpr int SC_RAW = SC_R + round_up(P, 4);
  static constexpr int SCR = (SC_RAW % 32 == 0 || SC_RAW % 32 == 16) ? SC_RAW + 4 : SC_RAW;
  // KREDUCE: when the gains live in the caller's Ks/ks buffer (long horizons / large n), lane i reads only
  // column i of K_t and the products are butterfly-reduced over the n state lanes (needs one problem per
  // warp and n a power of two).  For such shapes the gain store is moved out of shared memory on purpose
  // (GAIN_SMEM_LIMIT bytes per problem): it is what limits the resident warps per SM.
  static constexpr bool KREDUCE = CPL == 1 && PPW == 1 && (N & (N - 1)) == 0;
  static constexpr int GAIN_SMEM_LIMIT = 6144;
  static bool prefers_workspace(int T, int max_smem_optin) {
    return smem_bytes(T, true) > (size_t)max_smem_optin ||
           (KREDUCE && (size_t)T * KT * sizeof(R) > (size_t)GAIN_SMEM_LIMIT);
  }
  static constexpr int HDR_BYTES = 256;          // 2*S mbarriers + 32 vote words
  static size_t smem_bytes(int T, bool k_in_smem) {
    size_t b = HDR_BYTES + (size_t)S * STAGE_BYTES + (size_t)W * SCR * sizeof(R);
    if (k_in_smem) b += (size_t)W * T * KT * sizeof(R);
    return b;
  }
};

// ---------------------------------------------------------------------------------------------
// pnqp for one problem, executed redundantly by every lane of the problem (registers only).
// Control flow is what the reference takes for n_batch == 1 (mpc/pnqp.py:5-82).
// ---------------------------------------------------------------------------------------------
template <typename R, int M>
MPCB_DEV void pnqp_lane(const R (&H)[M][M], const R (&q)[M], const R (&lo)[M], const R (&hi)[M],
                        bool warm, R (&x)[M], Ldl<R, M>& fac, unsigned& fmask, int& iters,
                        bool& conv, bool& badpiv, int max_iter) {
  const R GAMMA = R(0.1);
  auto obj = [&](const R(&z)[M]) {            // pnqp.py:11-12
    R s = R(0);
#pragma unroll
    for (int a = 0; a < M; ++a) {
      R hz = R(0);
#pragma unroll
      for (int b = 0; b < M; ++b) hz += H[a][b] * z[b];
      s += z[a] * (R(0.5) * hz + q[a]);
    }
    return s;
  };
  badpiv = false;
  if (!warm) {                                 // pnqp.py:14-19
    fac.factor(H);
    badpiv = fac.bad;
    R t[M];
    fac.solve(q, t);
#pragma unroll
    for (int a = 0; a < M; ++a) x[a] = -t[a];
  }
#pragma unroll
  for (int a = 0; a < M; ++a) {                // :23  util.eclamp: lower bound first, then upper
    x[a] = x[a] < lo[a] ? lo[a] : x[a];
    x[a] = x[a] > hi[a] ? hi[a] : x[a];
  }

  for (int i = 0; i < max_iter; ++i) {
    R g[M];
#pragma unroll
    for (int a = 0; a < M; ++a) {              // :29
      R s = q[a];
#pragma unroll
      for (int b = 0; b < M; ++b) s += H[a][b] * x[b];
      g[a] = s;
    }
    fmask = 0u;
#pragma unroll
    for (int a = 0; a < M; ++a) {              // :32 exact equality with the assigned bound
      const bool cl = ((x[a] == lo[a]) && (g[a] > R(0))) || ((x[a] == hi[a]) && (g[a] < R(0)));
      if (!cl) fmask |= (1u << a);
    }
    R A[M][M], gm[M], dx[M];
#pragma unroll
    for (int a = 0; a < M; ++a) {              // :44-48
      const bool fa = (fmask >> a) & 1u;
      gm[a] = fa ? g[a] : R(0);
#pragma unroll
      for (int b = 0; b < M; ++b) {
        const bool fb = (fmask >> b) & 1u;
        A[a][b] = (fa && fb) ? H[a][b] : R(0);
      }
      A[a][a] += R(1e-11);
    }
    fac.factor(A);
    badpiv = badpiv || fac.bad;
    fac.solve(gm, dx);                         // :53-54
    R nrm2 = R(0);
#pragma unroll
    for (int a = 0; a < M; ++a) {
      dx[a] = -dx[a];
      nrm2 += dx[a] * dx[a];
    }
    if (!(sqrt(nrm2) >= R(1e-4))) {            // :56-59
      iters = i;
      conv = true;
      return;
    }
    R alpha = R(1), mx[M];
    const R fx = obj(x);
    int count = 0;
    bool again;
    do {                                       // :65-76 with n_batch == 1
#pragma unroll
      for (int a = 0; a < M; ++a) {
        const R v = x[a] + alpha * dx[a];
        const R vl = v < lo[a] ? lo[a] : v;
        mx[a] = vl > hi[a] ? hi[a] : vl;
      }
      R den = R(0);
#pragma unroll
      for (int a = 0; a < M; ++a) den += g[a] * (x[a] - mx[a]);
      const R arm = (fx - obj(mx)) / den;
      again = arm <= GAMMA;                    // NaN compares false, like torch
      if (again) alpha *= R(0.1);
      ++count;
    } while (again && count < 10);
    // A step that does not move x (bitwise) is a fixed point of the whole iteration: g, the active set,
    // H_, dx and the Armijo trials of every later iteration are identical.  In fp32 this is how the
    // reference fails to converge (|dx| stays just above 1e-4 while x + alpha dx rounds back to x);
    // returning now with the outcome of iteration max_iter-1 is exactly what the remaining iterations
    // would produce, without ~18 x 10 wasted Armijo trials that made this warp the kernel's tail.
    bool moved = false;
#pragma unroll
    for (int a = 0; a < M; ++a) {
      moved = moved || !(mx[a] == x[a]);
      x[a] = mx[a];                            // :78
    }
    if (!moved) break;
  }
  iters = max_iter - 1;                        // :80-82
  conv = false;
}

// ---------------------------------------------------------------------------------------------
// Shared by the step kernels (this file, lqr_step2.cuh, lqr_large.cu).
// ---------------------------------------------------------------------------------------------
enum { MODE_PLAIN = 0, MODE_BOX = 1, MODE_MASK = 2 };

// Where the gains K_t, k_t of all T steps live between the Riccati sweep and the rollout: shared memory when
// they fit, unless the kernel's own criterion `prefers_ws` moves them to the caller's Ks/ks.  Sets a.k_in_smem
// and smem to the kernel's dynamic shared memory; MPCB200_ERR_SMEM when neither placement works.
template <typename SmemFn>
int plan_gain_store(StepArgs& a, bool prefers_ws, int max_smem_optin, SmemFn smem_bytes, size_t& smem) {
  const bool have_ws = a.Ks != nullptr && a.ks != nullptr;
  a.k_in_smem = 1;
  smem = smem_bytes(true);
  if (smem > (size_t)max_smem_optin || (prefers_ws && have_ws && a.do_rollout)) {
    a.k_in_smem = 0;
    smem = smem_bytes(false);
    if (smem > (size_t)max_smem_optin) return MPCB200_ERR_SMEM;
    if (a.do_rollout && !have_ws) return MPCB200_ERR_SMEM;
  }
  return MPCB200_OK;
}

// The QP box of one control relative to the nominal u_bar (lqr_step.py:129-148): [lo - u_bar, hi - u_bar],
// clipped to +-delta_u when a slew limit is set.
template <typename R>
MPCB_DEV void qp_box(R lo_abs, R hi_abs, R ubar, bool has_delta, R du, R& lb, R& ub) {
  lb = lo_abs - ubar;
  ub = hi_abs - ubar;
  if (has_delta) {
    if (lb < -du) lb = -du;
    if (ub > du) ub = du;
  }
}

// The control solve of one time step, run redundantly by every lane of a problem (registers only), in two forms.
// Both give the feedforward kk and the factor of the free block of Q_uu that the gains are solved with, and OR
// MPCB200_ST_* bits into status.
//
// BOX (:129-148): pnqp on the box, warm started from kprev (which it updates).  Gives the free set fm and the pnqp
// iterations it.  The tensor bounds and u_bar come as callables q -> R, so each kernel reads them where it keeps them.
template <typename R, int M, typename Lo, typename Hi, typename Ubar>
MPCB_DEV void box_control_solve(const StepArgs& a, R (&Quu)[M][M], R (&qu)[M], R (&kprev)[M], bool valid, bool warm,
                                Lo lo_t, Hi hi_t, Ubar ubar, R (&kk)[M], unsigned& fm, int& it, Ldl<R, M>& fac,
                                unsigned& status) {
  const R s_lo = (R)a.u_lo, s_hi = (R)a.u_hi, s_du = (R)a.delta_u;
  R lb[M], ub[M];
#pragma unroll
  for (int q = 0; q < M; ++q) {
    qp_box<R>(a.bounds_kind == 2 ? lo_t(q) : s_lo, a.bounds_kind == 2 ? hi_t(q) : s_hi, ubar(q), a.has_delta, s_du,
              lb[q], ub[q]);
    kk[q] = kprev[q];
  }
  if (!valid) {   // padding problems of a tail CTA or warp compute on stale shared memory: give their
                  // (data dependent) pnqp loop a trivial QP so they never become the slowest problem
#pragma unroll
    for (int p1 = 0; p1 < M; ++p1) {
#pragma unroll
      for (int p2 = 0; p2 < M; ++p2) Quu[p1][p2] = p1 == p2 ? R(1) : R(0);
      qu[p1] = R(0);
      lb[p1] = R(-1);
      ub[p1] = R(1);
      kk[p1] = R(0);
    }
  }
  bool conv, badpiv;
  pnqp_lane<R, M>(Quu, qu, lb, ub, warm, kk, fac, fm, it, conv, badpiv, a.pnqp_iters);
  if (!conv) status |= MPCB200_ST_PNQP_UNCONVERGED;
  if (badpiv) status |= MPCB200_ST_BAD_PIVOT;
#pragma unroll
  for (int q = 0; q < M; ++q) kprev[q] = kk[q];
}

// PLAIN (:84-94) and MASK (:100-127): the LDL^T solve on the free set fm (all controls, or those u_zero_I leaves free);
// the rows and columns of the other controls are zeroed, with 1e-8 on their diagonal.
template <typename R, int M>
MPCB_DEV void ldl_control_solve(const R (&Quu)[M][M], const R (&qu)[M], unsigned fm, R (&kk)[M], Ldl<R, M>& fac,
                                unsigned& status) {
  R A[M][M], rhs[M], sol[M];
#pragma unroll
  for (int p1 = 0; p1 < M; ++p1) {
    const bool f1 = (fm >> p1) & 1u;
    rhs[p1] = f1 ? qu[p1] : R(0);
#pragma unroll
    for (int p2 = 0; p2 < M; ++p2) A[p1][p2] = (f1 && ((fm >> p2) & 1u)) ? Quu[p1][p2] : R(0);
    if (!f1) A[p1][p1] += R(1e-8);
  }
  fac.factor(A);
  if (fac.bad) status |= MPCB200_ST_BAD_PIVOT;
  fac.solve(rhs, sol);
#pragma unroll
  for (int q = 0; q < M; ++q) kk[q] = -sol[q];
}

// One control of a rollout (lqr_step.py:197-213), given u = K dx + u_bar + alpha k: zeroed where u_zero_I is set,
// then (box) clamped to [lo, hi] intersected with u_bar +- delta_u, lower bound first like util.eclamp.
template <typename R>
MPCB_DEV R rollout_control(R u, R ubar, bool masked, bool box, R lo, R hi, bool has_delta, R du) {
  if (masked) u = R(0);
  if (box) {
    if (has_delta) {
      const R l2 = ubar - du, h2 = ubar + du;
      lo = l2 < lo ? lo : l2;
      hi = h2 > hi ? hi : h2;
    }
    u = u < lo ? lo : u;
    u = u > hi ? hi : u;
  }
  return u;
}

// The line search after a rollout pass (lqr_step.py:243-247): the first pass gives ||du||, a cost worse than the
// nominal one shrinks alpha.  Returns whether the pass was worse; the kernel decides whether another pass runs.
template <typename R>
MPCB_DEV bool line_search_update(int pass, R cost, R oldcost, R du2, R decay, R& fdn, R& alpha) {
  if (pass == 0) fdn = sqrt(du2);
  const bool worse = cost > oldcost;
  if (worse) alpha *= decay;
  return worse;
}

MPCB_DEV void write_step_status(const StepArgs& a, int b, unsigned status) {
  if (a.status != nullptr) a.status[b] = (int)status;
}

// The per-problem results of a step with a rollout.  The kernels undo the last shrink of a worse final pass
// (alpha /= decay, :252) themselves: done in here, ptxas schedules the PLAIN kernels differently (DESIGN.md
// section 7).
template <typename R>
MPCB_DEV void write_step_result(const StepArgs& a, int b, R alpha, R cost, R fdn, unsigned status) {
  ((R*)a.costs)[b] = cost;
  ((R*)a.full_du_norm)[b] = fdn;
  ((R*)a.alphas)[b] = alpha;
  if (!(cost - cost == R(0))) status |= MPCB200_ST_NONFINITE;
  write_step_status(a, b, status);
}

// ---------------------------------------------------------------------------------------------
// producer warp: stream one (t) tile set of the CTA's problems into ring stage `tile % S`
// ---------------------------------------------------------------------------------------------
template <typename R, int N, int M>
MPCB_DEV void step_producer(const StepArgs& a, unsigned char* stage_base, uint64_t* full,
                            uint64_t* empty, volatile int* votes, int b0, int cnt, int lane) {
  using K = StepCfg<R, N, M>;
  constexpr int P = K::P;
  constexpr uint32_t SZ = sizeof(R);
  const R* gC = (const R*)a.C;
  const R* gc = (const R*)a.c;
  const R* gF = (const R*)a.F;
  const R* gf = (const R*)a.f;
  const R* gx = (const R*)a.cur_x;
  const R* gu = (const R*)a.cur_u;
  const R* glo = (const R*)a.u_lower;
  const R* ghi = (const R*)a.u_upper;
  const bool tail_ok = (cnt == K::W) || (((cnt * M * SZ) % 16 == 0) && ((cnt * N * SZ) % 16 == 0));
  const bool bulk = a.bulk_ok && tail_ok;
  const int T = a.T;
  int s = 0;
  uint32_t ph = 0;
  // The rollout reads each tile for the last time (a line-search repeat re-reads them, rarely).  Marking those
  // reads evict-first keeps the tiles the rollout has not reached yet in L2: at config 3 the tiles of one launch
  // (59 MB) exceed L2, and plain LRU replacement evicts exactly the lines the rollout reads next.
  const uint64_t last_use = l2_evict_first_policy();
  auto g2s = [&](void* dst, const void* src, uint32_t bytes, uint64_t* bar, bool fwd) {
    if (fwd) bulk_g2s(dst, src, bytes, bar, last_use);
    else bulk_g2s(dst, src, bytes, bar);
  };

  auto issue = [&](int t, bool fwd) {
    mbar_wait(&empty[s], ph ^ 1u);
    R* st = (R*)(stage_base + (size_t)s * K::STAGE_BYTES);
    const size_t tb = (size_t)t * a.B + b0;
    const size_t tC = (size_t)t * a.C_ts + (size_t)b0 * P * P, tF = (size_t)t * a.F_ts + (size_t)b0 * N * P;
    const size_t tc = (size_t)t * a.c_ts + (size_t)b0 * P, tf_ = (size_t)t * a.f_ts + (size_t)b0 * N;
    const bool needF = t < T - 1;
    const bool needf = fwd && needF && a.has_f;
    if (a.has_mask) {
      unsigned char* mk = (unsigned char*)(st + K::OFF_END);
      for (int i = lane; i < cnt * M; i += 32) mk[i] = a.zero_mask[tb * M + i];
    }
    if (bulk) {
      __syncwarp();
      if (lane == 0) {
        uint32_t bytes = (uint32_t)cnt * (P * P + P + N + M) * SZ;
        if (needF) bytes += (uint32_t)cnt * N * P * SZ;
        if (needf) bytes += (uint32_t)cnt * N * SZ;
        if (a.bounds_kind == 2) bytes += 2u * cnt * M * SZ;
        mbar_arrive_expect_tx(&full[s], bytes);
        if constexpr (K::CS == P * P) {
          g2s(st + K::OFF_C, gC + tC, (uint32_t)cnt * P * P * SZ, &full[s], fwd);
        } else {
          for (int q = 0; q < cnt; ++q)
            g2s(st + K::OFF_C + q * K::CS, gC + tC + (size_t)q * P * P, (uint32_t)P * P * SZ, &full[s], fwd);
        }
        if (needF) {
          if constexpr (K::FS == N * P) {
            g2s(st + K::OFF_F, gF + tF, (uint32_t)cnt * N * P * SZ, &full[s], fwd);
          } else {
            for (int q = 0; q < cnt; ++q)
              g2s(st + K::OFF_F + q * K::FS, gF + tF + (size_t)q * N * P, (uint32_t)N * P * SZ, &full[s], fwd);
          }
        }
        g2s(st + K::OFF_c, gc + tc, (uint32_t)cnt * P * SZ, &full[s], fwd);
        if (needf) g2s(st + K::OFF_f, gf + tf_, (uint32_t)cnt * N * SZ, &full[s], fwd);
        g2s(st + K::OFF_x, gx + tb * N, (uint32_t)cnt * N * SZ, &full[s], fwd);
        g2s(st + K::OFF_u, gu + tb * M, (uint32_t)cnt * M * SZ, &full[s], fwd);
        if (a.bounds_kind == 2) {
          g2s(st + K::OFF_lo, glo + tb * M, (uint32_t)cnt * M * SZ, &full[s], fwd);
          g2s(st + K::OFF_hi, ghi + tb * M, (uint32_t)cnt * M * SZ, &full[s], fwd);
        }
      }
    } else {
      auto cp = [&](R* dst, const R* src, int nelem) {
        for (int i = lane; i < nelem; i += 32) dst[i] = __ldg(src + i);
      };
      for (int q = 0; q < cnt; ++q) cp(st + K::OFF_C + q * K::CS, gC + tC + (size_t)q * P * P, P * P);
      if (needF)
        for (int q = 0; q < cnt; ++q) cp(st + K::OFF_F + q * K::FS, gF + tF + (size_t)q * N * P, N * P);
      cp(st + K::OFF_c, gc + tc, cnt * P);
      if (needf) cp(st + K::OFF_f, gf + tf_, cnt * N);
      cp(st + K::OFF_x, gx + tb * N, cnt * N);
      cp(st + K::OFF_u, gu + tb * M, cnt * M);
      if (a.bounds_kind == 2) {
        cp(st + K::OFF_lo, glo + tb * M, cnt * M);
        cp(st + K::OFF_hi, ghi + tb * M, cnt * M);
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&full[s]);
    }
    if (++s == K::S) { s = 0; ph ^= 1u; }
  };

  for (int t = T - 1; t >= 0; --t) issue(t, false);
  if (a.do_rollout) {
    for (int pass = 0;; ++pass) {
      for (int t = 0; t < T; ++t) issue(t, true);
      named_bar_sync(1, K::THREADS);
      const int cont = votes[pass & 31];
      if (!cont || pass + 1 >= a.max_ls) break;
    }
  }
}


// ---------------------------------------------------------------------------------------------
// consumer warps.  MODE (compile time): 0 plain (no bounds, no mask), 1 box (pnqp; optional
// u_zero_I), 2 mask (u_zero_I only - the adjoint solve).
// DYN: DYN_LINEAR for the (n, m) instances, whose rollout takes the true dynamics from a.dyn_kind; the kind of a
// dynamics-only instance (dyn_instances.def), whose rollout always runs that kind's dyn_step.
// ---------------------------------------------------------------------------------------------

template <typename R, int N, int M, int MODE, int DYN = DYN_LINEAR>
MPCB_DEV void step_consumer(const StepArgs& a, unsigned char* stage_base, uint64_t* full,
                            uint64_t* empty, volatile int* votes, R* scratch_all, R* kstore_all,
                            int b0, int warp, int lane) {
  using K = StepCfg<R, N, M>;
  constexpr int P = K::P, LP = K::LP, PPW = K::PPW, CPL = K::CPL, VS = K::VS, EA = K::EA, KT = K::KT;
  constexpr unsigned FULLM = (1u << M) - 1u;
  constexpr bool BOX = MODE == MODE_BOX;
  constexpr int A_N = align_elems<R>(N), A_M = align_elems<R>(M);
  constexpr int A_ROW = (P % 2 == 0) ? 2 : 1;   // row r*P of a per-problem tile (pair aligned for even P)
  constexpr int A_2P = align_elems<R>(2 * P), A_NP = align_elems<R>(K::FS);
  const int T = a.T, B = a.B;
  const bool writer_lane = lane < PPW * LP;
  const int pi = writer_lane ? lane / LP : PPW - 1;
  const int base = pi * LP;
  const int j = writer_lane ? lane - base : LP - 1;
  const int pw = warp * PPW + pi;
  const int b = b0 + pw;
  const bool valid = b < B;
  const bool wr = writer_lane && valid;

  // the CPL columns this lane owns: col = j + s*LP (slot 0 is always a state column)
  int cc[CPL], ua[CPL], fr[CPL];
  bool isx[CPL], wsl[CPL];
#pragma unroll
  for (int sl = 0; sl < CPL; ++sl) {
    const int col = j + sl * LP;
    wsl[sl] = writer_lane && col < P;
    cc[sl] = col < P ? col : P - 1;
    isx[sl] = K::x_slot(sl) && cc[sl] < N;
    ua[sl] = isx[sl] ? 0 : cc[sl] - N;       // control index of a u column
    fr[sl] = isx[sl] ? cc[sl] : N - 1;       // a valid row of F / V for every slot
  }

  // per-problem element offsets inside a stage (loop invariant)
  const int oC = K::OFF_C + pw * K::CS, oF = K::OFF_F + pw * K::FS;
  const int oc = K::OFF_c + pw * P, of_ = K::OFF_f + pw * N, ox = K::OFF_x + pw * N, ou = K::OFF_u + pw * M;
  const int olo = K::OFF_lo + pw * M, ohi = K::OFF_hi + pw * M;

  R* scr = scratch_all + (size_t)pw * K::SCR;
  R* Vs = scr + K::SC_V;
  R* vs = scr + K::SC_v;
  R* Qx = scr + K::SC_Q;
  R* red = scr + K::SC_R;
  R* kst = a.k_in_smem ? kstore_all + (size_t)pw * T * KT : scr + K::SC_K;
  R* gKs = (R*)a.Ks;
  R* gks = (R*)a.ks;

  const R s_lo = (R)a.u_lo, s_hi = (R)a.u_hi, s_du = (R)a.delta_u;
  const R decay = (R)a.ls_decay;
  const bool has_mask = MODE == MODE_MASK || (BOX && a.has_mask);

  int stg = 0;
  uint32_t ph = 0;
  unsigned status = 0u;
  // cost partials of the nominal trajectory, one per owned column, summed in column order below.  One column per
  // lane keeps the scalar: an array there changes the code of every single-column instance.
  R oldcost_part = R(0), oldcost_slot[CPL] = {};
  R kprev[M];
#pragma unroll
  for (int q = 0; q < M; ++q) kprev[q] = R(0);

  // ======================= backward Riccati sweep (lqr_step.py:61-158) =======================
  for (int t = T - 1; t >= 0; --t) {
    mbar_wait(&full[stg], ph);
    const R* st = (const R*)(stage_base + (size_t)stg * K::STAGE_BYTES);
    const unsigned char* mk = (const unsigned char*)(st + K::OFF_END) + pw * M;

    // nominal point tau_bar = [x_bar; u_bar] replicated on every lane
    Vec<R, P> tb;
    {
      Vec<R, N> tx;
      Vec<R, M> tu;
      tx.template load<A_N>(st + ox);
      tu.template load<A_M>(st + ou);
#pragma unroll
      for (int i = 0; i < N; ++i) tb.set(i, tx.get(i));
#pragma unroll
      for (int q = 0; q < M; ++q) tb.set(N + q, tu.get(q));
      if constexpr (P & 1) tb.p[Vec<R, P>::NP - 1].y = R(0);
    }
    // owned columns of C_t; c_back = (C_t tau_bar) + c for the owned rows  (lqr_step.py:289-295)
    Vec<R, P> Qc[CPL];
    R qj[CPL];
    // STATE_LANES: Q[j, n:n+2] (row j of Q_xu) and Q[cc[1], n:n+2] (the row of Q_uu of the control slot)
    P2<R> Qxu{}, Quq{};
#pragma unroll
    for (int sl = 0; sl < CPL; ++sl) {
      if constexpr (!K::STATE_LANES) Qc[sl].gather(st + oC + cc[sl], P);
      else if (sl == 0) Qc[sl].gather(st + oC + cc[sl], P);
      Vec<R, P> Crow;
      Crow.template load<A_ROW>(st + oC + cc[sl] * P);
      if constexpr (K::STATE_LANES) {
        if (sl == 0) Qxu = Crow.p[N / 2];
        else Quq = Crow.p[N / 2];
      }
      const R Ct = Crow.dot(tb);
      const R cj = st[oc + cc[sl]];
      const R tbj = st[(isx[sl] ? ox : ou - N) + cc[sl]];
      if constexpr (CPL == 1) {
        if (wsl[sl]) oldcost_part += tbj * (R(0.5) * Ct + cj);       // util.get_cost of the nominal trajectory (:169)
      } else {
        if (wsl[sl]) oldcost_slot[sl] += tbj * (R(0.5) * Ct + cj);
      }
      qj[sl] = Ct + cj;
    }
    if (t < T - 1) {                            // Q = C + F'VF, q = c_back + F'v  (:66-70)
      Vec<R, N> Fcol[CPL], Wc[CPL];
#pragma unroll
      for (int sl = 0; sl < K::XS; ++sl) Fcol[sl].gather(st + oF + cc[sl], P);
      Vec<R, N> Fuc;                              // STATE_LANES: F[:, cc[1]], for F[:, cc[1]]' v
      {
#pragma unroll
        for (int sl = 0; sl < K::XS; ++sl) Wc[sl].zero();
        P2<R> Wu{R(0), R(0)};                     // STATE_LANES: W[j, n:n+2]
#pragma unroll
        for (int k = 0; k < N; ++k) {             // W[:, c] = V F[:, c]; each V column load feeds XS columns
          Vec<R, N> Vcol;                         // Vs holds V transposed: row k of Vs == column k of V
          Vcol.template load<EA>(Vs + k * VS);
#pragma unroll
          for (int sl = 0; sl < K::XS; ++sl) Wc[sl].axpy(Vcol, Fcol[sl].get(k));
          if constexpr (K::STATE_LANES) {         // W[j, n+a] += V[j, k] F[k, n+a]
            Vec<R, M> Fu;
            Fu.template load<A_ROW>(st + oF + k * P + N);
            const R vjk = Vs[k * VS + j];
            Wu = fma2(P2<R>{vjk, vjk}, Fu.p[0], Wu);
          }
        }
        P2<R> Wk[K::STATE_LANES ? N : 1];         // STATE_LANES: W[k, n:n+2] from lane k
        if constexpr (K::STATE_LANES) {
#pragma unroll
          for (int k = 0; k < N; ++k) Wk[k] = P2<R>{shfl(Wu.x, base + k), shfl(Wu.y, base + k)};
        }
        static_for<0, N>([&](auto kc) {           // Q[:, c] += F' W[:, c]; rows of F are contiguous
          constexpr int k = decltype(kc)::value;
          constexpr int AK = k % 2 == 0 ? A_2P : align_elems<R>(P);
          Vec<R, P> Frow;
          Frow.template load<(AK < A_NP ? AK : A_NP)>(st + oF + k * P);
#pragma unroll
          for (int sl = 0; sl < K::XS; ++sl) Qc[sl].axpy(Frow, Wc[sl].get(k));
          if constexpr (K::STATE_LANES) {         // Q[r, n+a] += F[k, r] W[k, n+a] for r = j and r = cc[1]
            const R fx = Fcol[0].get(k);
            const R fu = ua[1] == 0 ? Frow.get(N) : Frow.get(N + 1);
            Fuc.set(k, fu);
            Qxu = fma2(P2<R>{fx, fx}, Wk[k], Qxu);
            Quq = fma2(P2<R>{fu, fu}, Wk[k], Quq);
          }
        });
      }
      Vec<R, N> vv;
      vv.template load<EA>(vs);
#pragma unroll
      for (int sl = 0; sl < K::XS; ++sl) qj[sl] += Fcol[sl].dot(vv);
      if constexpr (K::STATE_LANES) qj[1] += Fuc.dot(vv);
    }
    // replicate Q_uu, q_u on every lane of the problem (column n+b2 lives in lane (n+b2)%LP, slot (n+b2)/LP;
    // STATE_LANES: row n+b1 of Q_uu and q_u[b1] live in lane b1)
    R Quu[M][M], qu[M];
    if constexpr (K::STATE_LANES) {
#pragma unroll
      for (int p1 = 0; p1 < M; ++p1) {
        Quu[p1][0] = shfl(Quq.x, base + p1);
        Quu[p1][1] = shfl(Quq.y, base + p1);
        qu[p1] = shfl(qj[1], base + p1);
      }
    } else {
#pragma unroll
      for (int p2 = 0; p2 < M; ++p2) {
        const int src = base + (N + p2) % LP;
#pragma unroll
        for (int p1 = 0; p1 < M; ++p1) Quu[p1][p2] = shfl(Qc[(N + p2) / LP].get(N + p1), src);
        qu[p2] = shfl(qj[(N + p2) / LP], src);
      }
    }
    // This kernel keeps its own copy of box_control_solve and ldl_control_solve: with the shared ones, ptxas contracts
    // the f64 (8, 2) BOX kernel's multiplies and adds differently, so its outputs are no longer bitwise the same, and
    // it compiles the PLAIN kernels, config 3's among them, differently (DESIGN.md section 7).
    R kk[M];
    unsigned fm = FULLM;
    int it = 0;
    Ldl<R, M> fac;
    if constexpr (BOX) {                         // (:129-148)
      R lb[M], ub[M];
#pragma unroll
      for (int q = 0; q < M; ++q) {
        const R lo_abs = a.bounds_kind == 2 ? st[olo + q] : s_lo;
        const R hi_abs = a.bounds_kind == 2 ? st[ohi + q] : s_hi;
        const R ubq = tb.get(N + q);
        lb[q] = lo_abs - ubq;
        ub[q] = hi_abs - ubq;
        if (a.has_delta) {
          if (lb[q] < -s_du) lb[q] = -s_du;
          if (ub[q] > s_du) ub[q] = s_du;
        }
        kk[q] = kprev[q];
      }
      if (!valid) {   // padding problems of a tail CTA compute on stale shared memory: give their
                      // (data dependent) pnqp loop a trivial QP so they never become the slowest warp
#pragma unroll
        for (int p1 = 0; p1 < M; ++p1) {
#pragma unroll
          for (int p2 = 0; p2 < M; ++p2) Quu[p1][p2] = p1 == p2 ? R(1) : R(0);
          qu[p1] = R(0);
          lb[p1] = R(-1);
          ub[p1] = R(1);
          kk[p1] = R(0);
        }
      }
      bool conv, badpiv;
      pnqp_lane<R, M>(Quu, qu, lb, ub, t < T - 1, kk, fac, fm, it, conv, badpiv, a.pnqp_iters);
      if (!conv) status |= MPCB200_ST_PNQP_UNCONVERGED;
      if (badpiv) status |= MPCB200_ST_BAD_PIVOT;
#pragma unroll
      for (int q = 0; q < M; ++q) kprev[q] = kk[q];
    } else {                                     // unconstrained (:84-94) or u_zero_I masked (:100-127)
      if constexpr (MODE == MODE_MASK) {
        unsigned zm = 0u;
#pragma unroll
        for (int q = 0; q < M; ++q) zm |= (mk[q] ? 1u : 0u) << q;
        fm = FULLM & ~zm;
      }
      R A[M][M], rhs[M], sol[M];
#pragma unroll
      for (int p1 = 0; p1 < M; ++p1) {
        const bool f1 = (fm >> p1) & 1u;
        rhs[p1] = f1 ? qu[p1] : R(0);
#pragma unroll
        for (int p2 = 0; p2 < M; ++p2) A[p1][p2] = (f1 && ((fm >> p2) & 1u)) ? Quu[p1][p2] : R(0);
        if (!f1) A[p1][p1] += R(1e-8);
      }
      fac.factor(A);
      if (fac.bad) status |= MPCB200_ST_BAD_PIVOT;
      fac.solve(rhs, sol);
#pragma unroll
      for (int q = 0; q < M; ++q) kk[q] = -sol[q];
    }
    // K[:, c] = -Hff^{-1} Qux_f[:, c] for the owned columns (rows of clamped / masked controls are zero)
    R Kc[CPL][M];
    R* Kt = a.k_in_smem ? kst + (size_t)t * KT : kst;
#pragma unroll
    for (int sl = 0; sl < K::XS; ++sl) {
      R rhs[M], sol[M];
#pragma unroll
      for (int q = 0; q < M; ++q) rhs[q] = ((fm >> q) & 1u) ? Qc[sl].get(N + q) : R(0);
      fac.solve(rhs, sol);
#pragma unroll
      for (int q = 0; q < M; ++q) Kc[sl][q] = -sol[q];
      if (wsl[sl]) {
        if (isx[sl]) {
#pragma unroll
          for (int q = 0; q < M; ++q) Kt[q * VS + cc[sl]] = Kc[sl][q];
        } else {                          // u column: publish Q[:n, n+ua] = Q_xu[:, ua]
          Vec<R, N> qxu;                    // rows < n of the control column
#pragma unroll
          for (int i = 0; i < N; ++i) qxu.set(i, Qc[sl].get(i));
          qxu.template store<EA>(Qx + ua[sl] * VS);
        }
      }
    }
    if constexpr (K::STATE_LANES) {       // every lane publishes its row of Q_xu
      if (wsl[0]) {
        Qx[j] = Qxu.x;
        Qx[VS + j] = Qxu.y;
      }
    }
    if (j == 0) {
#pragma unroll
      for (int q = 0; q < M; ++q) Kt[M * VS + q] = kk[q];
    }
    if (wr) {
      const size_t tbo = (size_t)t * B + b;
      if (gKs != nullptr) {
#pragma unroll
        for (int sl = 0; sl < K::XS; ++sl) {
          if (wsl[sl] && isx[sl]) {
#pragma unroll
            for (int q = 0; q < M; ++q) gKs[(tbo * M + q) * N + cc[sl]] = Kc[sl][q];
          }
        }
        if (j == 0) {
#pragma unroll
          for (int q = 0; q < M; ++q) gks[tbo * M + q] = kk[q];
        }
      }
      if (BOX && a.qp_iters != nullptr && j == 0) a.qp_iters[tbo] = it;
      if (a.free_mask != nullptr) {
#pragma unroll
        for (int sl = 0; sl < CPL; ++sl)
          if (wsl[sl] && !isx[sl]) a.free_mask[tbo * M + ua[sl]] = (fm >> ua[sl]) & 1u;
      }
    }
    __syncwarp();

    // V = Qxx + Qxu K + K'Qux + K'Quu K ; v = qx + Qxu k + K'qu + K'Quu k   (:155-158)
    Vec<R, N> Vn[CPL];
    R vn[CPL], G[CPL][M];
#pragma unroll
    for (int sl = 0; sl < K::XS; ++sl) {
#pragma unroll
      for (int p1 = 0; p1 < M; ++p1) {
        R sacc = Qc[sl].get(N + p1);
#pragma unroll
        for (int p2 = 0; p2 < M; ++p2) sacc += Quu[p1][p2] * Kc[sl][p2];
        G[sl][p1] = sacc;
      }
#pragma unroll
      for (int i = 0; i < N; ++i) Vn[sl].set(i, Qc[sl].get(i));
      if constexpr (N & 1) Vn[sl].p[Vec<R, N>::NP - 1].y = R(0);
      vn[sl] = qj[sl];
    }
#pragma unroll
    for (int q = 0; q < M; ++q) {
      Vec<R, N> Qrow, Krow;
      Qrow.template load<EA>(Qx + q * VS);
      Krow.template load<EA>(Kt + q * VS);
      R sacc = qu[q];
#pragma unroll
      for (int p2 = 0; p2 < M; ++p2) sacc += Quu[q][p2] * kk[p2];
#pragma unroll
      for (int sl = 0; sl < K::XS; ++sl) {
        Vn[sl].axpy(Qrow, Kc[sl][q]);
        Vn[sl].axpy(Krow, G[sl][q]);
        if constexpr (K::STATE_LANES)            // Q[j, n+q]: this lane's own row of Q_xu
          vn[sl] += (q == 0 ? Qxu.x : Qxu.y) * kk[q] + Kc[sl][q] * sacc;
        else
          vn[sl] += Qx[q * VS + fr[sl]] * kk[q] + Kc[sl][q] * sacc;
      }
    }
#pragma unroll
    for (int sl = 0; sl < K::XS; ++sl) {
      if (wsl[sl] && isx[sl]) {
        Vn[sl].template store<EA>(Vs + cc[sl] * VS);        // column c of V, stored as row c (vector stores)
        vs[cc[sl]] = vn[sl];
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&empty[stg]);
    if (++stg == K::S) { stg = 0; ph ^= 1u; }
  }

  // nominal cost  (sum of the columns' partial sums, in column order)
  if constexpr (CPL == 1) {
    if (writer_lane) red[j] = oldcost_part;
  } else {
#pragma unroll
    for (int sl = 0; sl < CPL; ++sl)
      if (wsl[sl]) red[cc[sl]] = oldcost_slot[sl];
  }
  __syncwarp();
  R oldcost = R(0);
#pragma unroll
  for (int i = 0; i < P; ++i) oldcost += red[i];
  __syncwarp();

  if (!a.do_rollout) {
    if (wr && j == 0) write_step_status(a, b, status);
    return;
  }

  // ======================= rollout + line search (lqr_step.py:164-261) =======================
  const R* gx0 = (const R*)a.x_init;
  R* gnx = (R*)a.new_x;
  R* gnu = (R*)a.new_u;
  R* gdu1 = (R*)a.du_first;
  R alpha = R(1), fdn = R(0), cost = R(0);
  bool worse = false;
  for (int pass = 0;; ++pass) {
    Vec<R, N> xr;
#pragma unroll
    for (int i = 0; i < N; ++i) xr.set(i, valid ? gx0[(size_t)b * N + i] : R(0));
    if constexpr (N & 1) xr.p[Vec<R, N>::NP - 1].y = R(0);
    R xown[CPL];
#pragma unroll
    for (int sl = 0; sl < CPL; ++sl) xown[sl] = valid ? gx0[(size_t)b * N + fr[sl]] : R(0);
    R cpart = R(0), cpart_slot[CPL] = {}, dun2 = R(0);   // cost partials, as oldcost_part / oldcost_slot
    R kcol[M], kff[M];                        // KREDUCE with gains in global memory: column of K_t, k_t
#pragma unroll
    for (int q = 0; q < M; ++q) {
      kcol[q] = R(0);
      kff[q] = R(0);
    }
    if constexpr (K::KREDUCE) {
      if (!a.k_in_smem) {
        const size_t kb = (size_t)(valid ? b : 0) * M;
#pragma unroll
        for (int q = 0; q < M; ++q) {
          kcol[q] = __ldcg(gKs + (kb + q) * N + fr[0]);
          kff[q] = __ldcg(gks + kb + q);
        }
      }
    }
    size_t orow = (size_t)b;                     // t*B + b
    for (int t = 0; t < T; ++t, orow += (size_t)B) {
      mbar_wait(&full[stg], ph);
      const R* st = (const R*)(stage_base + (size_t)stg * K::STAGE_BYTES);
      const unsigned char* mk = (const unsigned char*)(st + K::OFF_END) + pw * M;

      Vec<R, N> xb, dxv;
      Vec<R, M> ubar;
      xb.template load<A_N>(st + ox);
      ubar.template load<A_M>(st + ou);
#pragma unroll
      for (int k2 = 0; k2 < Vec<R, N>::NP; ++k2) dxv.p[k2] = fma2(xb.p[k2], P2<R>{R(-1), R(-1)}, xr.p[k2]);
      R u[M];
      if (a.k_in_smem) {
        const R* Kt = kst + (size_t)t * KT;
#pragma unroll
        for (int q = 0; q < M; ++q) {
          Vec<R, N> Krow;
          Krow.template load<EA>(Kt + q * VS);
          u[q] = (Krow.dot(dxv) + ubar.get(q)) + alpha * Kt[M * VS + q];      // (:192)
        }
      } else if constexpr (K::KREDUCE) {
        // gains in the caller's buffer: this lane holds column cc of K_t and k_t (prefetched one step
        // ahead); K dx is reduced over the n state lanes with a butterfly, then broadcast
        const R dxi = xown[0] - st[ox + fr[0]];
        R part[M];
#pragma unroll
        for (int q = 0; q < M; ++q) part[q] = isx[0] ? kcol[q] * dxi : R(0);
#pragma unroll
        for (int off = N / 2; off >= 1; off >>= 1) {
#pragma unroll
          for (int q = 0; q < M; ++q) part[q] += __shfl_xor_sync(0xffffffffu, part[q], off);
        }
#pragma unroll
        for (int q = 0; q < M; ++q) u[q] = (shfl(part[q], base) + ubar.get(q)) + alpha * kff[q];
        if (t + 1 < T) {                         // prefetch the next step's column (L2 hit) behind this step
          const size_t kb = ((size_t)(t + 1) * B + (valid ? b : 0)) * M;
#pragma unroll
          for (int q = 0; q < M; ++q) {
            kcol[q] = __ldcg(gKs + (kb + q) * N + fr[0]);
            kff[q] = __ldcg(gks + kb + q);
          }
        }
      } else {
        const R* Kg = gKs + ((size_t)t * B + (valid ? b : 0)) * M * N;
        const R* kg = gks + ((size_t)t * B + (valid ? b : 0)) * M;
#pragma unroll
        for (int q = 0; q < M; ++q) {
          R sacc = R(0);
#pragma unroll
          for (int i = 0; i < N; ++i) sacc += __ldcg(Kg + q * N + i) * dxv.get(i);
          u[q] = (sacc + ubar.get(q)) + alpha * __ldcg(kg + q);
        }
      }
#pragma unroll
      for (int q = 0; q < M; ++q) {               // own copy of rollout_control, for the same reason
        if constexpr (MODE != MODE_PLAIN) {
          if (has_mask && mk[q]) u[q] = R(0);                     // (:197-198)
        }
        if constexpr (BOX) {                                      // (:200-213)
          R lo = a.bounds_kind == 2 ? st[olo + q] : s_lo;
          R hi = a.bounds_kind == 2 ? st[ohi + q] : s_hi;
          if (a.has_delta) {
            const R l2 = ubar.get(q) - s_du, h2 = ubar.get(q) + s_du;
            lo = l2 < lo ? lo : l2;
            hi = h2 > hi ? hi : h2;
          }
          u[q] = u[q] < lo ? lo : u[q];                                   // util.eclamp order: lower, then upper
          u[q] = u[q] > hi ? hi : u[q];
        }
        const R d = ubar.get(q) - u[q];
        dun2 += d * d;
      }
      Vec<R, P> tau;
#pragma unroll
      for (int i = 0; i < N; ++i) tau.set(i, xr.get(i));
#pragma unroll
      for (int q = 0; q < M; ++q) tau.set(N + q, u[q]);
      if constexpr (P & 1) tau.p[Vec<R, P>::NP - 1].y = R(0);

      R xn[CPL];
#pragma unroll
      for (int sl = 0; sl < CPL; ++sl) {
        R tj = xown[sl];
        if (!isx[sl]) {
#pragma unroll
          for (int q = 0; q < M; ++q)
            if (q == ua[sl]) tj = u[q];
        }
        Vec<R, P> Crow;
        Crow.template load<A_ROW>(st + oC + cc[sl] * P);
        const R Ct = Crow.dot(tau);
        if constexpr (CPL == 1) {
          if (wsl[sl]) cpart += tj * (R(0.5) * Ct + st[oc + cc[sl]]);           // (:232)
        } else {
          if (wsl[sl]) cpart_slot[sl] += tj * (R(0.5) * Ct + st[oc + cc[sl]]);
        }
        if (wr && wsl[sl]) {
          if (isx[sl]) {
            gnx[orow * N + cc[sl]] = tj;
          } else {
            gnu[orow * M + ua[sl]] = tj;
            if (pass == 0 && gdu1 != nullptr) gdu1[orow * M + ua[sl]] = st[ou + ua[sl]] - tj;
          }
        }
        xn[sl] = R(0);
        if (K::x_slot(sl) && t < T - 1) {                         // (:217-222), or true_dynamics(x, u) (:224-225)
          bool known = false;
          if constexpr (DYN != DYN_LINEAR) {      // dyn_step of the instance's kind ([u; ...] for a passthrough)
            static_assert(N == DynDims<DYN>::N && M == DynDims<DYN>::M, "instance shape of the dynamics kind");
            known = true;
            R sv[N], ov[N];
#pragma unroll
            for (int i = 0; i < N; ++i) sv[i] = tau.get(i);
            dyn_step<R, DYN, R>(a.dp, sv, tau.get(N), ov);
            xn[sl] = ov[0];
#pragma unroll
            for (int i = 1; i < N; ++i)
              if (fr[sl] == i) xn[sl] = ov[i];
          } else if constexpr (M == 1 && (N == DynDims<DYN_CARTPOLE>::N || N == DynDims<DYN_PENDULUM>::N)) {
            if (a.dyn_kind != DYN_LINEAR) {       // every lane evaluates the step function and keeps its row
              known = true;
              R sv[N], ov[N];
#pragma unroll
              for (int i = 0; i < N; ++i) sv[i] = tau.get(i);
              dyn_step<R, N == DynDims<DYN_CARTPOLE>::N ? DYN_CARTPOLE : DYN_PENDULUM, R>(a.dp, sv, tau.get(N), ov);
              xn[sl] = ov[0];
#pragma unroll
              for (int i = 1; i < N; ++i)
                if (fr[sl] == i) xn[sl] = ov[i];
            }
          }
          if (!known) {
            Vec<R, P> Frow;
            Frow.template load<A_ROW>(st + oF + fr[sl] * P);
            xn[sl] = Frow.dot(tau);
            if (a.has_f) xn[sl] += st[of_ + fr[sl]];
          }
        }
      }
      if (t < T - 1) {                           // x_{t+1} to every lane of the problem: element i from its column's lane
#pragma unroll
        for (int i = 0; i < N; ++i) xr.set(i, shfl(xn[i / LP], base + i % LP));
#pragma unroll
        for (int sl = 0; sl < CPL; ++sl) xown[sl] = xn[sl];
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[stg]);
      if (++stg == K::S) { stg = 0; ph ^= 1u; }
    }
    if constexpr (CPL == 1) {
      if (writer_lane) red[j] = cpart;
    } else {
#pragma unroll
      for (int sl = 0; sl < CPL; ++sl)
        if (wsl[sl]) red[cc[sl]] = cpart_slot[sl];
    }
    __syncwarp();
    cost = R(0);
#pragma unroll
    for (int i = 0; i < P; ++i) cost += red[i];
    __syncwarp();
    worse = line_search_update<R>(pass, cost, oldcost, dun2, decay, fdn, alpha);
    const bool more = pass + 1 < a.max_ls;
    if (wr && j == 0 && worse && more) votes[pass & 31] = 1;
    if (warp == 0 && lane == 0) votes[(pass + 16) & 31] = 0;
    named_bar_sync(1, K::THREADS);
    const int cont = votes[pass & 31];
    if (!cont || !more) break;
  }
  if (worse) alpha /= decay;                                      // (:252)
  if (wr && j == 0) write_step_result<R>(a, b, alpha, cost, fdn, status);
}

template <typename R, int N, int M, int MODE, int DYN = DYN_LINEAR>
__global__ void __launch_bounds__(StepCfg<R, N, M>::THREADS, StepCfg<R, N, M>::MIN_CTAS)
lqr_step_kernel(const StepArgs a) {
  using K = StepCfg<R, N, M>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  uint64_t* full = reinterpret_cast<uint64_t*>(smem_raw);
  uint64_t* empty = full + K::S;
  volatile int* votes = reinterpret_cast<volatile int*>(smem_raw + 128);
  unsigned char* stage_base = smem_raw + K::HDR_BYTES;
  R* scratch = reinterpret_cast<R*>(stage_base + (size_t)K::S * K::STAGE_BYTES);
  R* kstore = scratch + (size_t)K::W * K::SCR;

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int b0 = blockIdx.x * K::W;
  const int cnt = min(K::W, a.B - b0);
  if (tid == 0) {
#pragma unroll
    for (int s = 0; s < K::S; ++s) {
      mbar_init(&full[s], 1);
      mbar_init(&empty[s], K::NW);
    }
    mbar_fence_init();
  }
  if (tid < 32) votes[tid] = 0;
  __syncthreads();
  if (warp == K::NW) {
    step_producer<R, N, M>(a, stage_base, full, empty, votes, b0, cnt, lane);
  } else {
    step_consumer<R, N, M, MODE, DYN>(a, stage_base, full, empty, votes, scratch, kstore, b0, warp, lane);
  }
}

template <typename R, int N, int M, int MODE, int DYN = DYN_LINEAR>
int launch_step_mode(const StepArgs& args, int max_smem_optin, cudaStream_t stream) {
  using K = StepCfg<R, N, M>;
  StepArgs a = args;
  size_t smem;
  int rc = plan_gain_store(a, K::prefers_workspace(a.T, max_smem_optin), max_smem_optin,
                           [&](bool k_in_smem) { return K::smem_bytes(a.T, k_in_smem); }, smem);
  if (rc == MPCB200_OK) rc = allow_smem_optin<lqr_step_kernel<R, N, M, MODE, DYN>>(max_smem_optin);
  if (rc != MPCB200_OK) return rc;
  const int grid = (a.B + K::W - 1) / K::W;
  lqr_step_kernel<R, N, M, MODE, DYN><<<grid, K::THREADS, smem, stream>>>(a);
  if (cudaGetLastError() != cudaSuccess) return MPCB200_ERR_LAUNCH;
  record_step_plan((int)(MPCB200_PLAN_GENERIC | (a.k_in_smem ? MPCB200_PLAN_GAINS_SMEM : 0u) |
                         (K::KREDUCE && !a.k_in_smem && a.do_rollout ? MPCB200_PLAN_KREDUCE : 0u)));
  return MPCB200_OK;
}

template <typename R, int N, int M, int DYN = DYN_LINEAR>
int launch_step(const StepArgs& a, int max_smem_optin, cudaStream_t stream) {
  if (a.bounds_kind != 0) return launch_step_mode<R, N, M, MODE_BOX, DYN>(a, max_smem_optin, stream);
  if (a.has_mask) return launch_step_mode<R, N, M, MODE_MASK, DYN>(a, max_smem_optin, stream);
  return launch_step_mode<R, N, M, MODE_PLAIN, DYN>(a, max_smem_optin, stream);
}

template <typename R, int N, int M>
int step_prefers_workspace(int T, int max_smem_optin) {
  return StepCfg<R, N, M>::prefers_workspace(T, max_smem_optin) ? 1 : 0;
}

template <typename R, int N, int M>
size_t step_smem_query(int T) {
  return StepCfg<R, N, M>::smem_bytes(T, true);
}

}  // namespace mpcb200
