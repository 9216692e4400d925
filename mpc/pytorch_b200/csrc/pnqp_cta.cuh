// pnqp_cta.cuh - projected-Newton box QP (reference mpc/pnqp.py:5-82) solved by a whole thread block on a QP
// that is already in shared memory.  Used by the standalone CTA-per-QP kernel (pnqp_large.cu) and by the step
// kernel for shapes without a compiled instance (lqr_large.cu), so both run the same operations in the same order.
// The standalone kernel's implicit gradient (pnqp_large.cu) factors the same H_ with the same pack_free_block and
// ldl_solve.
// Shared-memory operands of one QP (n = its size):
//   H    n x LD, LD = n | 1.  Row i of every mat-vec belongs to thread i % NT, so a warp reads a column of H at
//        a stride of LD elements; an odd LD puts its 32 rows in 32 banks (16 bank pairs in fp64).
//   P    the masked matrix H_ of the current iteration, lower triangle packed by rows (row i at i(i+1)/2) and
//        factored in place into L (below the diagonal) and D (on it).  H plus a full square factor would not
//        fit in fp64 at n = 128 (2 * 8 * 128^2 B > 227 KB).
//   q lo hi x g v mx w dinv (n each), a reduction buffer of RED elements, and the free flags of the current
//   iteration.
// As in Ldl<R,M>, only the lower triangle of H_ is factored: H must be symmetric (the mat-vecs read all of H).
// Reductions run in a fixed order (xor butterfly inside a warp, then the warp partials in warp order) and
// every branch depends on values all threads hold with the same bits, so the result of a problem does not
// depend on the batch, its position in it, or the run.
#pragma once
#include "common.cuh"

namespace mpcb200 {

constexpr int RED = 64;   // reduction buffer: two sums of up to 32 warp partials

__host__ __device__ constexpr int tri(int i) { return i * (i + 1) / 2; }   // row i of a packed lower triangle

// (a, b) <- the block sums of (a, b), with the same bits in every thread.  Also a block barrier.
template <typename R, int NT>
MPCB_DEV void block_sum2(R& a, R& b, R* red) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {   // both lanes of a pair add the same two values: all lanes end equal
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  if (NT > 32) {
    const int w = threadIdx.x >> 5;
    if ((threadIdx.x & 31) == 0) {
      red[w] = a;
      red[32 + w] = b;
    }
    __syncthreads();
    a = red[0];
    b = red[32];
#pragma unroll
    for (int k = 1; k < NT / 32; ++k) {
      a += red[k];
      b += red[32 + k];
    }
  }
  __syncthreads();
}

// LDL^T of the packed matrix P in place, then v <- P^{-1} v.  Right-looking: step j turns column j into
// L_kj = U_kj / d_j and subtracts L_ij U_kj from the trailing block; the forward substitution rides along
// (v_k -= L_kj v_j, same order as Ldl::solve).  Column k of the trailing block belongs to thread k % NT and a
// warp walks the rows together, so its columns of one row are consecutive elements.  Returns whether a pivot
// was <= 0 or not finite (every thread returns the same).  The block is in sync on entry and on return.
template <typename R, int NT>
MPCB_DEV bool ldl_solve(R* P, R* v, R* w, R* dinv, int n) {
  const int t = threadIdx.x;
  bool bad = false;
  for (int j = 0; j < n; ++j) {
    const R dj = P[tri(j) + j];
    bad = bad || !(dj > R(0));
    const R di = recip(dj);
    const R vj = v[j];
    for (int k = j + 1 + t; k < n; k += NT) {
      const R u = P[tri(k) + j];
      const R l = u * di;
      w[k] = u;
      P[tri(k) + j] = l;
      v[k] -= l * vj;
    }
    if (t == 0) dinv[j] = di;
    __syncthreads();
    for (int kb = 0; kb < n; kb += NT) {
      const int k = kb + t, wk0 = kb + (t & ~31);   // this thread's column, the first column of its warp
      if (wk0 + 31 <= j || wk0 >= n) continue;      // warp-uniform: no column of the warp is in the trailing block
      const bool own = k > j && k < n;
      const R u = own ? w[k] : R(0);
      int i = max(j + 1, wk0), ri = tri(i);         // rows above wk0 hold no trailing element of this warp
      for (; i + 3 < n; i += 4) {                    // four rows per trip: all loads, then the stores
        const int r[4] = {ri, ri + i + 1, ri + 2 * i + 3, ri + 3 * i + 6};
        R l[4], p[4];
#pragma unroll
        for (int s = 0; s < 4; ++s) {
          l[s] = P[r[s] + j];
          p[s] = own && k <= i + s ? P[r[s] + k] : R(0);
        }
#pragma unroll
        for (int s = 0; s < 4; ++s)
          if (own && k <= i + s) P[r[s] + k] = p[s] - l[s] * u;
        ri = r[3] + i + 4;
      }
      for (; i < n; ++i) {
        if (own && k <= i) P[ri + k] -= P[ri + j] * u;
        ri += i + 1;
      }
    }
    __syncthreads();
  }
  if (t < 32) {   // back substitution x_i = v_i / d_i - sum_{k>i} L_ki x_k by rows k of L: one warp, in place
    for (int i = t; i < n; i += 32) v[i] *= dinv[i];
    __syncwarp();
    for (int k = n - 1; k > 0; --k) {
      const R xk = v[k];
      const int rk = tri(k);
      for (int i = t; i < k; i += 32) v[i] -= P[rk + i] * xk;
      __syncwarp();
    }
  }
  __syncthreads();
  return bad;
}

// P <- the masked matrix H_ (pnqp.py:46-48), lower triangle packed by rows: H on the rows and columns that fr marks
// free, 0 elsewhere, plus 1e-11 on the diagonal.  Row i of H starts at H + i * ld (shared or global memory).
template <typename R, int NT>
MPCB_DEV void pack_free_block(R* P, const R* H, int ld, const int* fr, int n) {
  for (int i = 0; i < n; ++i) {
    const bool fi = fr[i] != 0;
    for (int k = threadIdx.x; k <= i; k += NT)
      P[tri(i) + k] = ((fi && fr[k]) ? H[i * ld + k] : R(0)) + (k == i ? R(1e-11) : R(0));
  }
}

// The projected-Newton iteration (pnqp.py:14-82) on the QP (H, q, lo, hi) in shared memory, from x (read when
// has_init) or from the clamped -H^{-1} q.  On return x is the solution, fr the free set and P, dinv the LDL^T
// factor of the H_ of the returning iteration (what the reference returns the LU of); conv / badpiv as in
// pnqp_lane.  Returns the reference's `i`.  The block is in sync on entry and on return.
template <typename R, int NT>
MPCB_DEV int pnqp_cta_solve(const R* H, R* P, const R* q, const R* lo, const R* hi, R* x, R* g, R* v, R* mx, R* w,
                            R* dinv, R* red, int* fr, int n, int n_iter, bool has_init, bool& conv, bool& badpiv) {
  const int LD = n | 1, t = threadIdx.x;
  badpiv = false;
  if (!has_init) {                             // pnqp.py:14-19  x = -H^{-1} q
    for (int i = 0; i < n; ++i)
      for (int k = t; k <= i; k += NT) P[tri(i) + k] = H[i * LD + k];
    for (int i = t; i < n; i += NT) v[i] = q[i];
    __syncthreads();
    badpiv = ldl_solve<R, NT>(P, v, w, dinv, n);
    for (int i = t; i < n; i += NT) x[i] = -v[i];
  }
  for (int i = t; i < n; i += NT) {            // :23  util.eclamp: lower bound first, then upper
    const R xl = x[i] < lo[i] ? lo[i] : x[i];
    x[i] = xl > hi[i] ? hi[i] : xl;
  }
  __syncthreads();

  const R GAMMA = R(0.1);
  int iters = n_iter - 1;                      // :80-82, unless the loop returns earlier
  conv = false;
  for (int it = 0; it < n_iter; ++it) {
    R fx = R(0), nrm2 = R(0);
    for (int i = t; i < n; i += NT) {          // :29 g, :32 clamped set by exact equality, :44-45 g_
      const R* Hi = H + i * LD;
      R hx = R(0);
      for (int k = 0; k < n; ++k) hx += Hi[k] * x[k];
      const R gi = hx + q[i];
      const bool cl = ((x[i] == lo[i]) && (gi > R(0))) || ((x[i] == hi[i]) && (gi < R(0)));
      g[i] = gi;
      fr[i] = !cl;
      v[i] = cl ? R(0) : gi;
      fx += x[i] * (R(0.5) * hx + q[i]);       // objective at x (:11-12) for the Armijo ratio
    }
    __syncthreads();
    pack_free_block<R, NT>(P, H, LD, fr, n);   // :46-48
    __syncthreads();
    badpiv = ldl_solve<R, NT>(P, v, w, dinv, n) || badpiv;
    for (int i = t; i < n; i += NT) {          // :53-54  dx = -H_^{-1} g_
      const R d = -v[i];
      v[i] = d;
      nrm2 += d * d;
    }
    block_sum2<R, NT>(fx, nrm2, red);
    if (!(sqrt(nrm2) >= R(1e-4))) {            // :56-59
      iters = it;
      conv = true;
      break;
    }
    R alpha = R(1);
    int count = 0;
    bool again;
    do {                                       // :65-76 for one problem
      for (int i = t; i < n; i += NT) {
        const R s = x[i] + alpha * v[i];
        const R sl = s < lo[i] ? lo[i] : s;
        mx[i] = sl > hi[i] ? hi[i] : sl;
      }
      __syncthreads();
      R fm = R(0), den = R(0);
      for (int i = t; i < n; i += NT) {
        const R* Hi = H + i * LD;
        R hz = R(0);
        for (int k = 0; k < n; ++k) hz += Hi[k] * mx[k];
        fm += mx[i] * (R(0.5) * hz + q[i]);
        den += g[i] * (x[i] - mx[i]);
      }
      block_sum2<R, NT>(fm, den, red);
      const R arm = (fx - fm) / den;
      again = arm <= GAMMA;                    // NaN compares false, like torch
      if (again) alpha *= R(0.1);
      ++count;
    } while (again && count < 10);
    // a step that does not move x (bitwise) is a fixed point of the whole iteration (see pnqp_lane): the
    // remaining iterations would return this x, free set and H_ with iters = n_iter - 1
    bool moved = false;
    for (int i = t; i < n; i += NT) {
      moved = moved || !(mx[i] == x[i]);
      x[i] = mx[i];                            // :78
    }
    if (!__syncthreads_or(moved)) break;
  }
  return iters;
}

}  // namespace mpcb200
