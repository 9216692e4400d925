// pnqp_large.cu - standalone projected-Newton box QP (reference mpc/pnqp.py:5-82) for 8 < n <= pnqp_max_n.
// One CTA per QP, runtime n.  The control flow and arithmetic per problem are those of pnqp_lane
// (lqr_step.cuh), which keeps a whole QP in one thread's registers and therefore stops at n = 8.  Here the
// threads of a block share one QP in shared memory; the iteration and its layout are in pnqp_cta.cuh.  The implicit
// gradient of the solution runs one CTA per QP over the same range of n.
#include "../../../include/mpcb200.h"
#include "common.cuh"
#include "pnqp.cuh"
#include "pnqp_cta.cuh"

namespace mpcb200 {

template <typename R, int NT>
__global__ void __launch_bounds__(NT) pnqp_cta_kernel(const PnqpArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int n = a.n, LD = n | 1, t = threadIdx.x;
  const size_t b = blockIdx.x;
  R* H = reinterpret_cast<R*>(smem_raw);
  R* P = H + n * LD;
  R* q = P + tri(n);
  R* lo = q + n;
  R* hi = lo + n;
  R* x = hi + n;      // iterate
  R* g = x + n;       // gradient Hx + q
  R* v = g + n;       // right-hand side of the solve, then the Newton step dx
  R* mx = v + n;      // Armijo trial point
  R* w = mx + n;      // column j of the factorisation before it is scaled
  R* dinv = w + n;
  R* red = dinv + n;
  int* fr = reinterpret_cast<int*>(red + RED);   // free set of the current iteration

  const R* gH = (const R*)a.H + b * n * n;
  for (int e = t; e < n * n; e += NT) H[(e / n) * LD + e % n] = gH[e];
  for (int i = t; i < n; i += NT) {
    q[i] = ((const R*)a.q)[b * n + i];
    lo[i] = ((const R*)a.lo)[b * n + i];
    hi[i] = ((const R*)a.hi)[b * n + i];
    x[i] = a.has_init ? ((const R*)a.x_init)[b * n + i] : R(0);
  }
  __syncthreads();
  bool conv, badpiv;
  const int iters = pnqp_cta_solve<R, NT>(H, P, q, lo, hi, x, g, v, mx, w, dinv, red, fr, n, a.n_iter, a.has_init != 0,
                                          conv, badpiv);

  R* ox = (R*)a.x + b * n;
  R* oH = (R*)a.Hfree + b * n * n;
  for (int i = t; i < n; i += NT) {
    ox[i] = x[i];
    a.If[b * n + i] = (unsigned char)fr[i];
  }
  for (int e = t; e < n * n; e += NT) {        // H_ of the returning iteration
    const int i = e / n, k = e % n;
    oH[e] = ((fr[i] && fr[k]) ? H[i * LD + k] : R(0)) + (i == k ? R(1e-11) : R(0));
  }
  if (t == 0) {
    a.iters[b] = iters;
    if (a.status != nullptr)
      a.status[b] = (conv ? 0 : (int)MPCB200_ST_PNQP_UNCONVERGED) | (badpiv ? (int)MPCB200_ST_BAD_PIVOT : 0);
  }
}

// The implicit gradient of the solution x with free set F (If) for g = dL/dx (contract in include/mpcb200.h):
// v = (H_FF + 1e-11 I)^{-1} g_F by the forward's factorisation of H_ (v is exactly 0 off F), dq = -v, dH = -v x^T on
// the rows of F, and on a clamped coordinate i the bound x_i sits on gets g_i - sum_{k in F} H_ki v_k.  H stays in
// global memory: the factor is packed from it and the clamped coordinates read its columns (consecutive i per warp),
// so shared memory holds P, x, v, w, dinv and the free set, less than the forward at every n.
template <typename R, int NT>
__global__ void __launch_bounds__(NT) pnqp_cta_backward_kernel(const PnqpGradArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  const int n = a.n, t = threadIdx.x;
  const size_t b = blockIdx.x;
  R* P = reinterpret_cast<R*>(smem_raw);
  R* x = P + tri(n);
  R* v = x + n;       // g on F (0 elsewhere), then (H_FF + 1e-11 I)^{-1} g_F
  R* w = v + n;
  R* dinv = w + n;
  int* fr = reinterpret_cast<int*>(dinv + n);

  const R* gH = (const R*)a.H + b * n * n;
  const R* gg = (const R*)a.g + b * n;
  for (int i = t; i < n; i += NT) {
    const bool f = a.If[b * n + i] != 0;
    fr[i] = f;
    x[i] = ((const R*)a.x)[b * n + i];
    v[i] = f ? gg[i] : R(0);
  }
  __syncthreads();
  pack_free_block<R, NT>(P, gH, n, fr, n);
  __syncthreads();
  const bool bad = ldl_solve<R, NT>(P, v, w, dinv, n);

  R* dH = (R*)a.dH + b * n * n;
  for (int e = t; e < n * n; e += NT) {
    const int i = e / n, k = e % n;
    dH[e] = fr[i] ? -v[i] * x[k] : R(0);
  }
  for (int i = t; i < n; i += NT) {
    R dq = R(0), dlo = R(0), dhi = R(0);
    if (fr[i]) {
      dq = -v[i];
    } else {
      R s = R(0);
      for (int k = 0; k < n; ++k)
        if (fr[k]) s += gH[k * n + i] * v[k];
      const R r = gg[i] - s;
      if (x[i] == ((const R*)a.lo)[b * n + i]) dlo = r;
      else dhi = r;
    }
    ((R*)a.dq)[b * n + i] = dq;
    ((R*)a.dlo)[b * n + i] = dlo;
    ((R*)a.dhi)[b * n + i] = dhi;
  }
  if (t == 0 && a.status != nullptr) a.status[b] = bad ? (int)MPCB200_ST_BAD_PIVOT : 0;
}

template <typename R, int NT>
static int launch(const PnqpArgs& a, int max_smem, cudaStream_t stream) {
  const int rc = allow_smem_optin<pnqp_cta_kernel<R, NT>>(max_smem);
  if (rc != MPCB200_OK) return rc;
  pnqp_cta_kernel<R, NT><<<a.B, NT, pnqp_cta_smem_bytes(a.n, (int)sizeof(R)), stream>>>(a);
  return cudaGetLastError() == cudaSuccess ? MPCB200_OK : MPCB200_ERR_LAUNCH;
}

template <typename R, int NT>
static int launch_backward(const PnqpGradArgs& a, int max_smem, cudaStream_t stream) {
  const int rc = allow_smem_optin<pnqp_cta_backward_kernel<R, NT>>(max_smem);
  if (rc != MPCB200_OK) return rc;
  const size_t N = (size_t)a.n, smem = sizeof(R) * ((size_t)tri(a.n) + 4 * N) + sizeof(int) * N;
  pnqp_cta_backward_kernel<R, NT><<<a.B, NT, smem, stream>>>(a);
  return cudaGetLastError() == cudaSuccess ? MPCB200_OK : MPCB200_ERR_LAUNCH;
}

size_t pnqp_cta_smem_bytes(int n, int elem_size) {
  const size_t N = (size_t)n;
  return (size_t)elem_size * (N * (size_t)(n | 1) + (size_t)tri(n) + 9 * N + RED) + sizeof(int) * N;
}

int pnqp_max_n(int elem_size, int max_smem) {
  int n = 8;
  while (pnqp_cta_smem_bytes(n + 1, elem_size) <= (size_t)max_smem) ++n;
  return n;
}

// one warp per QP up to n = 32, so that several QPs share an SM; four warps above
template <typename R>
int pnqp_cta_launch(const PnqpArgs& a, int max_smem, cudaStream_t stream) {
  return a.n <= 32 ? launch<R, 32>(a, max_smem, stream) : launch<R, 128>(a, max_smem, stream);
}
template int pnqp_cta_launch<float>(const PnqpArgs&, int, cudaStream_t);
template int pnqp_cta_launch<double>(const PnqpArgs&, int, cudaStream_t);

// the forward's CTA shapes
template <typename R>
int pnqp_cta_backward_launch(const PnqpGradArgs& a, int max_smem, cudaStream_t stream) {
  return a.n <= 32 ? launch_backward<R, 32>(a, max_smem, stream) : launch_backward<R, 128>(a, max_smem, stream);
}
template int pnqp_cta_backward_launch<float>(const PnqpGradArgs&, int, cudaStream_t);
template int pnqp_cta_backward_launch<double>(const PnqpGradArgs&, int, cudaStream_t);

}  // namespace mpcb200
