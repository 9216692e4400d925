// lqr_large.cu - the LQR step, gradient assembly and LinDx rollout for (n_state, n_ctrl) shapes that no compiled
// instance covers (instances.def).  Same contracts as lqr_step.cuh, lqr_grad.cuh and lqr_rollout.cuh; compiled
// once per element type with runtime n, m.
//
// Mapping: one thread block of NT threads per problem (as pnqp_large.cu).  The dense products of a time step are
// spread over the block one output element per thread; every element is summed by one thread in a fixed order
// and the cost sums reduce in a fixed order (block_sum2), so a problem's result does not depend on the batch.
//
// Step kernel, shared memory (layout: large_layout):
//   stage s (1 or 2):  C_t (p x p, becomes Q_t in place), F_t (n x p), c_t, f_t, x_bar_t, u_bar_t, tensor bounds
//                      and the u_zero_I bytes of this problem.  Spans whose start and length are 16-byte aligned at
//                      every t are streamed with 1-D bulk copies (completion on an mbarrier); the others are copied
//                      by the block.  With two stages the tile of the next time step is in flight while this one
//                      computes.
//   V (n x n), v, W (n x p: V F_t, then K_t and Q_uu K_t), q_t, tau, two state vectors, and the operands of the
//   m x m box QP in the layout of pnqp_cta.cuh.
// The gains K_t, k_t always go to global memory (the caller's Ks/ks); the rollout reads them back from L2.
// Backward sweep (reference lqr_step.py:61-158): q = C tau_bar + c; Q = C + F'(V F), q += F'v; then
//   BOX   pnqp_cta_solve on Q_uu (warm start k_{t+1}); K = -H_^{-1} Q_ux on the free rows from the factor of the
//         free block the QP returns,
//   PLAIN / MASK  LDL^T of Q_uu (masked: u_zero_I rows and columns zeroed, +1e-8 on their diagonal),
// and V = Q_xx + Q_xu K + K'Q_ux + K'(Q_uu K), v = q_x + Q_xu k + K'(q_u + Q_uu k) with the true Q_xu.
// Rollout + line search (:164-261): per-problem alpha, passes repeat while the cost is worse than the nominal one.
#include "../../../include/mpcb200.h"
#include "common.cuh"
#include "lqr_large.cuh"
#include "pnqp_cta.cuh"

namespace mpcb200 {

constexpr int LNT = 128;   // threads per problem

struct LargeLayout {
  // byte offsets; stage pieces are relative to the stage, the rest to the start of shared memory
  unsigned sC, sF, sc, sf, sx, su, slo, shi, smk, stage;
  unsigned stage0, V, v, W, qv, tau, xa, xb, H, P, q, lo, hi, x, g, pv, mx, w, dinv, red, fr, total;
};

__host__ __device__ inline unsigned lput(unsigned& o, unsigned bytes) {
  const unsigned r = o;
  o += (bytes + 15u) & ~15u;
  return r;
}

__host__ __device__ inline LargeLayout large_layout(int n, int m, int es, int stages) {
  LargeLayout L;
  const unsigned p = n + m, e = es;
  unsigned o = 0;
  L.sC = lput(o, p * p * e);
  L.sF = lput(o, n * p * e);
  L.sc = lput(o, p * e);
  L.sf = lput(o, n * e);
  L.sx = lput(o, n * e);
  L.su = lput(o, m * e);
  L.slo = lput(o, m * e);
  L.shi = lput(o, m * e);
  L.smk = lput(o, m);
  L.stage = (o + 127u) & ~127u;
  o = 128;                                      // two mbarriers
  L.stage0 = o;
  o += stages * L.stage;
  const unsigned wk = n * p > 2 * m * n ? n * p : 2 * m * n;
  L.V = lput(o, n * n * e);
  L.v = lput(o, n * e);
  L.W = lput(o, wk * e);
  L.qv = lput(o, p * e);
  L.tau = lput(o, p * e);
  L.xa = lput(o, n * e);
  L.xb = lput(o, n * e);
  L.H = lput(o, m * (m | 1) * e);
  L.P = lput(o, tri(m) * e);
  L.q = lput(o, m * e);
  L.lo = lput(o, m * e);
  L.hi = lput(o, m * e);
  L.x = lput(o, m * e);
  L.g = lput(o, m * e);
  L.pv = lput(o, m * e);
  L.mx = lput(o, m * e);
  L.w = lput(o, m * e);
  L.dinv = lput(o, m * e);
  L.red = lput(o, RED * e);
  L.fr = lput(o, m * 4);
  L.total = o;
  return L;
}

size_t large_step_smem_bytes(int n, int m, int elem_size, int stages) {
  return large_layout(n, m, elem_size, stages).total;
}

bool large_step_fits(int n, int m, int elem_size, int max_smem) {
  if (n <= 0 || m <= 0 || n > 4096 || m > 4096) return false;
  return large_step_smem_bytes(n, m, elem_size, 1) <= (size_t)max_smem;
}

MPCB_DEV void proxy_fence_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

struct LargeStepArgs {
  StepArgs s;
  int n, m, stages;
  unsigned bulk;
};

template <typename R>
__global__ void __launch_bounds__(LNT) lqr_large_step_kernel(const __grid_constant__ LargeStepArgs la) {
  extern __shared__ __align__(128) unsigned char sm[];
  const StepArgs& a = la.s;
  const int n = la.n, m = la.m, p = n + m, tid = threadIdx.x;
  const int T = a.T, B = a.B, b = blockIdx.x;
  const unsigned bulk = la.bulk;
  const LargeLayout L = large_layout(n, m, (int)sizeof(R), la.stages);
  uint64_t* full = reinterpret_cast<uint64_t*>(sm);
  R* V = (R*)(sm + L.V);
  R* vv = (R*)(sm + L.v);
  R* W = (R*)(sm + L.W);
  R* qv = (R*)(sm + L.qv);
  R* tau = (R*)(sm + L.tau);
  R* H = (R*)(sm + L.H);
  R* P = (R*)(sm + L.P);
  R* qq = (R*)(sm + L.q);
  R* plo = (R*)(sm + L.lo);
  R* phi = (R*)(sm + L.hi);
  R* kx = (R*)(sm + L.x);       // k_t: the QP solution, the warm start of step t-1
  R* gq = (R*)(sm + L.g);
  R* pv = (R*)(sm + L.pv);
  R* mx = (R*)(sm + L.mx);
  R* pw = (R*)(sm + L.w);
  R* dinv = (R*)(sm + L.dinv);
  R* red = (R*)(sm + L.red);
  int* fr = (int*)(sm + L.fr);
  const int LD = m | 1;
  const int mode = a.bounds_kind != 0 ? MODE_BOX : (a.has_mask ? MODE_MASK : MODE_PLAIN);
  const bool box2 = a.bounds_kind == 2;
  const bool has_mask = mode == MODE_MASK || (mode == MODE_BOX && a.has_mask);
  const R s_lo = (R)a.u_lo, s_hi = (R)a.u_hi, s_du = (R)a.delta_u;
  R* gKs = (R*)a.Ks;
  R* gks = (R*)a.ks;

  if (tid == 0) {
    mbar_init(&full[0], 1);
    mbar_init(&full[1], 1);
    mbar_fence_init();
  }
  __syncthreads();

  // ---- tile loader: stage s <- the spans of time step t (fwd: the rollout also needs f)
  auto issue = [&](int t, bool fwd, int s) {
    unsigned char* st = sm + L.stage0 + (size_t)s * L.stage;
    const size_t tb = (size_t)t * B + b;
    const bool needF = t < T - 1, needf = fwd && needF && a.has_f;
    const R* sC = (const R*)a.C + (size_t)t * a.C_ts + (size_t)b * p * p;
    const R* sF = needF ? (const R*)a.F + (size_t)t * a.F_ts + (size_t)b * n * p : nullptr;
    const R* sc = (const R*)a.c + (size_t)t * a.c_ts + (size_t)b * p;
    const R* sf = needf ? (const R*)a.f + (size_t)t * a.f_ts + (size_t)b * n : nullptr;
    const R* sx = (const R*)a.cur_x + tb * n;
    const R* su = (const R*)a.cur_u + tb * m;
    const R* slo = box2 ? (const R*)a.u_lower + tb * m : nullptr;
    const R* shi = box2 ? (const R*)a.u_upper + tb * m : nullptr;
    const unsigned z = sizeof(R);
    if (tid == 0) {
      uint32_t bytes = 0;
      if (bulk & LB_C) bytes += p * p * z;
      if (needF && (bulk & LB_F)) bytes += n * p * z;
      if (bulk & LB_c) bytes += p * z;
      if (needf && (bulk & LB_f)) bytes += n * z;
      if (bulk & LB_x) bytes += n * z;
      if (bulk & LB_u) bytes += m * z;
      if (box2 && (bulk & LB_BOX)) bytes += 2 * m * z;
      mbar_arrive_expect_tx(&full[s], bytes);
      if (bulk & LB_C) bulk_g2s(st + L.sC, sC, p * p * z, &full[s]);
      if (needF && (bulk & LB_F)) bulk_g2s(st + L.sF, sF, n * p * z, &full[s]);
      if (bulk & LB_c) bulk_g2s(st + L.sc, sc, p * z, &full[s]);
      if (needf && (bulk & LB_f)) bulk_g2s(st + L.sf, sf, n * z, &full[s]);
      if (bulk & LB_x) bulk_g2s(st + L.sx, sx, n * z, &full[s]);
      if (bulk & LB_u) bulk_g2s(st + L.su, su, m * z, &full[s]);
      if (box2 && (bulk & LB_BOX)) {
        bulk_g2s(st + L.slo, slo, m * z, &full[s]);
        bulk_g2s(st + L.shi, shi, m * z, &full[s]);
      }
    }
    auto cp = [&](unsigned off, const R* src, int cnt) {
      R* dst = (R*)(st + off);
      for (int i = tid; i < cnt; i += LNT) dst[i] = __ldg(src + i);
    };
    if (!(bulk & LB_C)) cp(L.sC, sC, p * p);
    if (needF && !(bulk & LB_F)) cp(L.sF, sF, n * p);
    if (!(bulk & LB_c)) cp(L.sc, sc, p);
    if (needf && !(bulk & LB_f)) cp(L.sf, sf, n);
    if (!(bulk & LB_x)) cp(L.sx, sx, n);
    if (!(bulk & LB_u)) cp(L.su, su, m);
    if (box2 && !(bulk & LB_BOX)) {
      cp(L.slo, slo, m);
      cp(L.shi, shi, m);
    }
    if (has_mask) {
      unsigned char* mk = st + L.smk;
      for (int i = tid; i < m; i += LNT) mk[i] = a.zero_mask[tb * m + i];
    }
  };
  // acquire the tile of step t and, with two stages, start the one of (nt, nfwd) into the other stage.  Generic
  // writes into a stage (Q_t is formed in place of C_t) are ordered before the next bulk copy into it by the
  // proxy fence ahead of the barrier.
  int cur = 0;
  unsigned ph = 0u;
  bool issued = false;
  auto acquire = [&](int t, bool fwd, int nt, bool nfwd, bool has_next) -> unsigned char* {
    proxy_fence_async();
    if (!issued) {
      __syncthreads();
      issue(t, fwd, cur);
    }
    mbar_wait(&full[cur], (ph >> cur) & 1u);
    ph ^= 1u << cur;
    __syncthreads();
    unsigned char* st = sm + L.stage0 + (size_t)cur * L.stage;
    issued = la.stages == 2 && has_next;
    if (la.stages == 2) cur ^= 1;
    if (issued) issue(nt, nfwd, cur);
    return st;
  };

  unsigned status = 0u;
  R ocp = R(0);   // this thread's part of the nominal cost
  // ======================= backward Riccati sweep =======================
  for (int t = T - 1; t >= 0; --t) {
    unsigned char* st = acquire(t, false, t > 0 ? t - 1 : 0, t == 0, t > 0 || a.do_rollout);
    R* Q = (R*)(st + L.sC);
    const R* F = (const R*)(st + L.sF);
    const R* cc = (const R*)(st + L.sc);
    const R* xs = (const R*)(st + L.sx);
    const R* us = (const R*)(st + L.su);
    const R* lo_t = (const R*)(st + L.slo);
    const R* hi_t = (const R*)(st + L.shi);
    const unsigned char* mk = st + L.smk;
    const size_t tbo = (size_t)t * B + b;

    for (int i = tid; i < p; i += LNT) tau[i] = i < n ? xs[i] : us[i - n];
    __syncthreads();
    // q = C tau_bar + c (:289-295) and the nominal cost; W = V F
    const int nW = t < T - 1 ? n * p : 0;
    for (int e = tid; e < p + nW; e += LNT) {
      if (e < p) {
        const R* Cr = Q + e * p;
        R s = R(0);
        for (int k = 0; k < p; ++k) s += Cr[k] * tau[k];
        qv[e] = s + cc[e];
        ocp += tau[e] * (R(0.5) * s + cc[e]);
      } else {
        const int i = (e - p) / p, c = (e - p) - i * p;
        const R* Vi = V + i * n;
        R s = R(0);
        for (int k = 0; k < n; ++k) s += Vi[k] * F[k * p + c];
        W[i * p + c] = s;
      }
    }
    __syncthreads();
    if (t < T - 1) {              // Q = C + F'W, q += F'v  (:66-70)
      for (int e = tid; e < p * p + p; e += LNT) {
        if (e < p * p) {
          const int r = e / p, c = e - r * p;
          R s = R(0);
          for (int k = 0; k < n; ++k) s += F[k * p + r] * W[k * p + c];
          Q[e] += s;
        } else {
          const int r = e - p * p;
          R s = R(0);
          for (int k = 0; k < n; ++k) s += F[k * p + r] * vv[k];
          qv[r] += s;
        }
      }
      __syncthreads();
    }
    // the control solve: k in kx, the free set in fr, LDL^T of the free block in P / dinv
    int iters = 0;
    if (mode == MODE_BOX) {       // (:129-148)
      for (int e = tid; e < m * m; e += LNT) {
        const int i = e / m, k = e - i * m;
        H[i * LD + k] = Q[(n + i) * p + n + k];
      }
      for (int i = tid; i < m; i += LNT) {
        qq[i] = qv[n + i];
        qp_box<R>(box2 ? lo_t[i] : s_lo, box2 ? hi_t[i] : s_hi, us[i], a.has_delta, s_du, plo[i], phi[i]);
      }
      __syncthreads();
      bool conv, badpiv;
      iters = pnqp_cta_solve<R, LNT>(H, P, qq, plo, phi, kx, gq, pv, mx, pw, dinv, red, fr, m, a.pnqp_iters,
                                     t < T - 1, conv, badpiv);
      if (!conv) status |= MPCB200_ST_PNQP_UNCONVERGED;
      if (badpiv) status |= MPCB200_ST_BAD_PIVOT;
    } else {                      // unconstrained (:84-94) or u_zero_I masked (:100-127)
      for (int i = tid; i < m; i += LNT) {
        const int f1 = mode == MODE_MASK ? !mk[i] : 1;
        fr[i] = f1;
        pv[i] = f1 ? qv[n + i] : R(0);
      }
      __syncthreads();
      for (int i = 0; i < m; ++i) {
        const bool fi = fr[i] != 0;
        for (int k = tid; k <= i; k += LNT)
          P[tri(i) + k] = ((fi && fr[k]) ? Q[(n + i) * p + n + k] : R(0)) + (k == i && !fi ? R(1e-8) : R(0));
      }
      __syncthreads();
      if (ldl_solve<R, LNT>(P, pv, pw, dinv, m)) status |= MPCB200_ST_BAD_PIVOT;
      for (int i = tid; i < m; i += LNT) kx[i] = -pv[i];
    }
    // K = -H_^{-1} Q_ux on the free rows: thread j solves column j with the factor (same order as ldl_solve)
    R* K = W;
    R* G = W + m * n;
    for (int j = tid; j < n; j += LNT) {
      for (int i = 0; i < m; ++i) K[i * n + j] = fr[i] ? Q[(n + i) * p + j] : R(0);
      for (int jj = 0; jj < m; ++jj) {
        const R vj = K[jj * n + j];
        for (int k = jj + 1; k < m; ++k) K[k * n + j] -= P[tri(k) + jj] * vj;
      }
      for (int i = 0; i < m; ++i) K[i * n + j] *= dinv[i];
      for (int k = m - 1; k > 0; --k) {
        const R xk = K[k * n + j];
        for (int i = 0; i < k; ++i) K[i * n + j] -= P[tri(k) + i] * xk;
      }
      for (int i = 0; i < m; ++i) K[i * n + j] = -K[i * n + j];
    }
    __syncthreads();
    for (int e = tid; e < m * n; e += LNT) gKs[tbo * m * n + e] = K[e];
    for (int i = tid; i < m; i += LNT) {
      gks[tbo * m + i] = kx[i];
      if (a.free_mask != nullptr) a.free_mask[tbo * m + i] = (unsigned char)(fr[i] != 0);
    }
    if (tid == 0 && mode == MODE_BOX && a.qp_iters != nullptr) a.qp_iters[tbo] = iters;
    // G = Q_uu K, gq = q_u + Q_uu k
    for (int e = tid; e < m * n + m; e += LNT) {
      if (e < m * n) {
        const int i = e / n, j = e - i * n;
        const R* Qr = Q + (n + i) * p + n;
        R s = R(0);
        for (int k = 0; k < m; ++k) s += Qr[k] * K[k * n + j];
        G[e] = s;
      } else {
        const int i = e - m * n;
        const R* Qr = Q + (n + i) * p + n;
        R s = R(0);
        for (int k = 0; k < m; ++k) s += Qr[k] * kx[k];
        gq[i] = qv[n + i] + s;
      }
    }
    __syncthreads();
    // V = Qxx + Qxu K + K'Qux + K'Quu K ; v = qx + Qxu k + K'(qu + Quu k)   (:155-158)
    for (int e = tid; e < n * n + n; e += LNT) {
      if (e < n * n) {
        const int i = e / n, j = e - i * n;
        R s1 = R(0), s2 = R(0), s3 = R(0);
        for (int k = 0; k < m; ++k) {
          const R Kki = K[k * n + i];
          s1 += Q[i * p + n + k] * K[k * n + j];
          s2 += Kki * Q[(n + k) * p + j];
          s3 += Kki * G[k * n + j];
        }
        V[e] = Q[i * p + j] + s1 + s2 + s3;
      } else {
        const int i = e - n * n;
        R s1 = R(0), s2 = R(0);
        for (int k = 0; k < m; ++k) {
          s1 += Q[i * p + n + k] * kx[k];
          s2 += K[k * n + i] * gq[k];
        }
        vv[i] = qv[i] + s1 + s2;
      }
    }
  }
  R oldcost = ocp, dummy = R(0);
  block_sum2<R, LNT>(oldcost, dummy, red);

  if (!a.do_rollout) {
    if (tid == 0) write_step_status(a, b, status);
    return;
  }

  // ======================= rollout + line search =======================
  const R* gx0 = (const R*)a.x_init;
  R* gnx = (R*)a.new_x;
  R* gnu = (R*)a.new_u;
  R* gdu1 = (R*)a.du_first;
  const R decay = (R)a.ls_decay;
  R alpha = R(1), fdn = R(0), cost = R(0);
  bool worse = false;
  for (int pass = 0;; ++pass) {
    R* xr = (R*)(sm + L.xa);
    R* xn = (R*)(sm + L.xb);
    for (int i = tid; i < n; i += LNT) xr[i] = gx0[(size_t)b * n + i];
    R cpart = R(0), du2 = R(0);
    for (int t = 0; t < T; ++t) {
      unsigned char* st = acquire(t, true, t + 1, true, t + 1 < T);
      const R* C = (const R*)(st + L.sC);
      const R* F = (const R*)(st + L.sF);
      const R* cc = (const R*)(st + L.sc);
      const R* ff = (const R*)(st + L.sf);
      const R* xs = (const R*)(st + L.sx);
      const R* us = (const R*)(st + L.su);
      const R* lo_t = (const R*)(st + L.slo);
      const R* hi_t = (const R*)(st + L.shi);
      const unsigned char* mk = st + L.smk;
      const size_t tbo = (size_t)t * B + b;
      for (int e = tid; e < m * n + m + n; e += LNT) {      // K_t, k_t (L2) and x_t - x_bar_t
        if (e < m * n) W[e] = __ldcg(gKs + tbo * m * n + e);
        else if (e < m * n + m) gq[e - m * n] = __ldcg(gks + tbo * m + (e - m * n));
        else {
          const int i = e - m * n - m;
          tau[i] = xr[i];
          W[m * n + i] = xr[i] - xs[i];
        }
      }
      __syncthreads();
      for (int q = tid; q < m; q += LNT) {                   // (:192), mask (:197-198), clamp (:200-213)
        const R* Kq = W + q * n;
        const R* dx = W + m * n;
        R s = R(0);
        for (int i = 0; i < n; ++i) s += Kq[i] * dx[i];
        const R u = rollout_control<R>((s + us[q]) + alpha * gq[q], us[q], has_mask && mk[q], mode == MODE_BOX,
                                       box2 ? lo_t[q] : s_lo, box2 ? hi_t[q] : s_hi, a.has_delta, s_du);
        const R d = us[q] - u;
        du2 += d * d;
        tau[n + q] = u;
      }
      __syncthreads();
      const int nF = t < T - 1 ? n : 0;
      for (int e = tid; e < p + nF; e += LNT) {              // cost (:232), x_{t+1} = F tau + f (:217-222)
        if (e < p) {
          const R* Cr = C + e * p;
          R s = R(0);
          for (int k = 0; k < p; ++k) s += Cr[k] * tau[k];
          const R tj = tau[e];
          cpart += tj * (R(0.5) * s + cc[e]);
          if (e < n) {
            gnx[tbo * n + e] = tj;
          } else {
            gnu[tbo * m + (e - n)] = tj;
            if (pass == 0 && gdu1 != nullptr) gdu1[tbo * m + (e - n)] = us[e - n] - tj;
          }
        } else {
          const int i = e - p;
          const R* Fr = F + i * p;
          R s = R(0);
          for (int k = 0; k < p; ++k) s += Fr[k] * tau[k];
          if (a.has_f) s += ff[i];
          xn[i] = s;
        }
      }
      R* tmp = xr;
      xr = xn;
      xn = tmp;
    }
    block_sum2<R, LNT>(cpart, du2, red);
    cost = cpart;
    worse = line_search_update<R>(pass, cost, oldcost, du2, decay, fdn, alpha);
    const bool more = pass + 1 < a.max_ls;
    if (!worse || !more) break;
  }
  if (worse) alpha /= decay;                                 // (:252)
  if (tid == 0) write_step_result<R>(a, b, alpha, cost, fdn, status);
}

template <typename R>
int large_step_launch(const StepArgs& a, int n, int m, unsigned bulk, int max_smem, cudaStream_t stream) {
  const int es = (int)sizeof(R);
  if (!large_step_fits(n, m, es, max_smem)) return MPCB200_ERR_SMEM;
  LargeStepArgs la;
  la.s = a;
  la.n = n;
  la.m = m;
  la.bulk = bulk;
  la.stages = large_step_smem_bytes(n, m, es, 2) <= (size_t)max_smem ? 2 : 1;
  const size_t smem = large_step_smem_bytes(n, m, es, la.stages);
  const int rc = allow_smem_optin<lqr_large_step_kernel<R>>(max_smem);
  if (rc != MPCB200_OK) return rc;
  lqr_large_step_kernel<R><<<a.B, LNT, smem, stream>>>(la);
  if (cudaGetLastError() != cudaSuccess) return MPCB200_ERR_LAUNCH;
  record_step_plan((int)MPCB200_PLAN_LARGE);
  return MPCB200_OK;
}

// ---------------------------------------------------------------------------------------------
// gradient assembly (reference lqr_step.py:342-404), contract of lqr_grad.cuh
// ---------------------------------------------------------------------------------------------
// dC_t, dc_t, dF_t (from lambda_{t+1}, dlambda_{t+1}) of one (t, b); the block writes them together
template <typename R>
MPCB_DEV void large_outer(const GradArgs& a, int n, int m, int t, int b, const R* tau, const R* dtau, const R* lam,
                          const R* dlam) {
  const int p = n + m, tid = threadIdx.x;
  const size_t tb = (size_t)t * a.B + b;
  R* oC = (R*)a.dC + tb * p * p;
  for (int e = tid; e < p * p; e += LNT) {
    const int i = e / p, c = e - i * p;
    oC[e] = R(-0.5) * (dtau[i] * tau[c] + tau[i] * dtau[c]);
  }
  for (int i = tid; i < p; i += LNT) ((R*)a.dc)[tb * p + i] = -dtau[i];
  if (t < a.T - 1 || a.F_T == a.T) {
    R* oF = (R*)a.dF + tb * n * p;
    const bool zero = t == a.T - 1;
    for (int e = tid; e < n * p; e += LNT) {
      const int k = e / p, c = e - k * p;
      oF[e] = zero ? R(0) : -(dlam[k] * tau[c] + lam[k] * dtau[c]);
    }
  }
}

template <typename R>
MPCB_DEV void load_tau(const GradArgs& a, int n, int m, size_t tb, R* tau, R* dtau) {
  const int p = n + m;
  for (int i = threadIdx.x; i < p; i += LNT) {
    tau[i] = i < n ? ((const R*)a.new_x)[tb * n + i] : ((const R*)a.new_u)[tb * m + (i - n)];
    dtau[i] = i < n ? ((const R*)a.dx)[tb * n + i] : ((const R*)a.du)[tb * m + (i - n)];
  }
}

// costates lambda_t, dlambda_t backward in t (:355-385), df, dx_init; the costates go to the workspace for
// large_outer_kernel
template <typename R>
__global__ void __launch_bounds__(LNT) lqr_large_costate_kernel(const GradArgs a, int n, int m) {
  extern __shared__ __align__(16) unsigned char sm[];
  const int p = n + m, T = a.T, B = a.B, b = blockIdx.x, tid = threadIdx.x;
  R* tau = (R*)sm;
  R* dtau = tau + p;
  R* lam = dtau + p;          // lambda_{t+1}, dlambda_{t+1}
  R* dlam = lam + n;
  R* nlam = dlam + n;         // lambda_t, dlambda_t
  R* ndlam = nlam + n;
  R* wl = (R*)a.workspace;
  R* wd = wl + (size_t)T * B * n;
  for (int t = T - 1; t >= 0; --t) {
    const size_t tb = (size_t)t * B + b;
    load_tau<R>(a, n, m, tb, tau, dtau);
    __syncthreads();
    const R* Cb = (const R*)a.C + (size_t)t * a.C_ts + (size_t)b * p * p;
    const R* Fb = t < T - 1 ? (const R*)a.F + (size_t)t * a.F_ts + (size_t)b * n * p : nullptr;
    for (int j = tid; j < n; j += LNT) {
      if (t < T - 1 && a.has_df) ((R*)a.df)[tb * n + j] = -dlam[j];   // df_t = -dlambda_{t+1}
      const R* Cr = Cb + (size_t)j * p;
      R nl = R(0), ndl = R(0);
      for (int i = 0; i < p; ++i) {
        const R cv = Cr[i];
        nl += cv * tau[i];
        ndl += cv * dtau[i];
      }
      nl += ((const R*)a.c)[(size_t)t * a.c_ts + (size_t)b * p + j];
      ndl -= ((const R*)a.dl_dx)[tb * n + j];
      if (t < T - 1) {
        for (int k = 0; k < n; ++k) {
          const R fv = Fb[(size_t)k * p + j];
          nl += fv * lam[k];
          ndl += fv * dlam[k];
        }
      }
      nlam[j] = nl;
      ndlam[j] = ndl;
      wl[tb * n + j] = nl;
      wd[tb * n + j] = ndl;
    }
    __syncthreads();
    for (int j = tid; j < n; j += LNT) {
      lam[j] = nlam[j];
      dlam[j] = ndlam[j];
    }
  }
  __syncthreads();
  for (int j = tid; j < n; j += LNT) ((R*)a.dx_init)[(size_t)b * n + j] = -dlam[j];
}

// dC, dc, dF of one (t, b) per block, from the costates in the workspace
template <typename R>
__global__ void __launch_bounds__(LNT) lqr_large_outer_kernel(const GradArgs a, int n, int m) {
  extern __shared__ __align__(16) unsigned char sm[];
  const int p = n + m, T = a.T, B = a.B;
  const int t = (int)(blockIdx.x / (unsigned)B), b = (int)(blockIdx.x - (unsigned)t * B);
  R* tau = (R*)sm;
  R* dtau = tau + p;
  R* lam = dtau + p;
  R* dlam = lam + n;
  load_tau<R>(a, n, m, (size_t)t * B + b, tau, dtau);
  if (t < T - 1) {
    const R* wl = (const R*)a.workspace;
    const size_t t1 = ((size_t)(t + 1) * B + b) * n;
    for (int j = threadIdx.x; j < n; j += LNT) {
      lam[j] = wl[t1 + j];
      dlam[j] = wl[(size_t)T * B * n + t1 + j];
    }
  }
  __syncthreads();
  large_outer<R>(a, n, m, t, b, tau, dtau, lam, dlam);
}

template <typename R>
int large_grad_launch(const GradArgs& a, int n, int m, cudaStream_t stream) {
  const size_t smem = (size_t)(2 * (n + m) + 4 * n) * sizeof(R);
  if (smem > 48 * 1024) return MPCB200_ERR_SMEM;
  lqr_large_costate_kernel<R><<<a.B, LNT, smem, stream>>>(a, n, m);
  if (cudaGetLastError() != cudaSuccess) return MPCB200_ERR_LAUNCH;
  lqr_large_outer_kernel<R><<<(unsigned)((size_t)a.T * a.B), LNT, smem, stream>>>(a, n, m);
  return cudaGetLastError() == cudaSuccess ? MPCB200_OK : MPCB200_ERR_LAUNCH;
}

// ---------------------------------------------------------------------------------------------
// LinDx rollout x[t+1] = F[t] [x[t]; u[t]] + f[t] (reference util.py:102-126), one block per problem
// ---------------------------------------------------------------------------------------------
template <typename R>
__global__ void __launch_bounds__(LNT) lqr_large_rollout_kernel(const RolloutArgs a, int n, int m) {
  extern __shared__ __align__(16) unsigned char sm[];
  const int p = n + m, T = a.T, B = a.B, b = blockIdx.x, tid = threadIdx.x;
  R* tau = (R*)sm;
  R* xn = tau + p;
  R* gx = (R*)a.x;
  for (int i = tid; i < n; i += LNT) {
    const R x0 = ((const R*)a.x_init)[(size_t)b * n + i];
    tau[i] = x0;
    gx[(size_t)b * n + i] = x0;
  }
  for (int t = 0; t < T - 1; ++t) {
    const size_t tb = (size_t)t * B + b;
    for (int q = tid; q < m; q += LNT) tau[n + q] = ((const R*)a.u)[tb * m + q];
    __syncthreads();
    const R* Fb = (const R*)a.F + (size_t)t * a.F_ts + (size_t)b * n * p;
    for (int r = tid; r < n; r += LNT) {
      R acc = a.has_f ? ((const R*)a.f)[(size_t)t * a.f_ts + (size_t)b * n + r] : R(0);
      const R* Fr = Fb + (size_t)r * p;
      for (int k = 0; k < p; ++k) acc += Fr[k] * tau[k];
      xn[r] = acc;
      gx[((size_t)(t + 1) * B + b) * n + r] = acc;
    }
    __syncthreads();
    for (int r = tid; r < n; r += LNT) tau[r] = xn[r];
  }
}

template <typename R>
int large_rollout_launch(const RolloutArgs& a, int n, int m, cudaStream_t stream) {
  const size_t smem = (size_t)(2 * n + m) * sizeof(R);
  if (smem > 48 * 1024) return MPCB200_ERR_SMEM;
  lqr_large_rollout_kernel<R><<<a.B, LNT, smem, stream>>>(a, n, m);
  return cudaGetLastError() == cudaSuccess ? MPCB200_OK : MPCB200_ERR_LAUNCH;
}

template int large_step_launch<float>(const StepArgs&, int, int, unsigned, int, cudaStream_t);
template int large_step_launch<double>(const StepArgs&, int, int, unsigned, int, cudaStream_t);
template int large_grad_launch<float>(const GradArgs&, int, int, cudaStream_t);
template int large_grad_launch<double>(const GradArgs&, int, int, cudaStream_t);
template int large_rollout_launch<float>(const RolloutArgs&, int, int, cudaStream_t);
template int large_rollout_launch<double>(const RolloutArgs&, int, int, cudaStream_t);

}  // namespace mpcb200
