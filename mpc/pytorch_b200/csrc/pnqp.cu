// pnqp.cu - standalone projected-Newton box QP (reference mpc/pnqp.py:5-82), C entry points and dispatch.
// n <= 8: one thread per QP; same per-problem control flow and arithmetic as inside the step kernel
// (pnqp_lane in lqr_step.cuh).  8 < n <= pnqp_max_n: one CTA per QP (pnqp_large.cu).
// min 0.5 x'Hx + q'x  s.t. lower <= x <= upper.  The implicit gradient of its solution (mpcb200_pnqp_backward_*)
// is split the same way.
#include "../../../include/mpcb200.h"
#include "lqr_step.cuh"
#include "pnqp.cuh"

namespace mpcb200 {

template <typename R, int M>
__global__ void __launch_bounds__(128) pnqp_kernel(const PnqpArgs a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.B) return;
  const R* gH = (const R*)a.H + (size_t)b * M * M;
  const R* gq = (const R*)a.q + (size_t)b * M;
  const R* glo = (const R*)a.lo + (size_t)b * M;
  const R* ghi = (const R*)a.hi + (size_t)b * M;
  R H[M][M], q[M], lo[M], hi[M], x[M];
#pragma unroll
  for (int i = 0; i < M; ++i) {
#pragma unroll
    for (int j = 0; j < M; ++j) H[i][j] = gH[i * M + j];
    q[i] = gq[i];
    lo[i] = glo[i];
    hi[i] = ghi[i];
    x[i] = a.has_init ? ((const R*)a.x_init)[(size_t)b * M + i] : R(0);
  }
  Ldl<R, M> fac;
  unsigned fm = 0u;
  int it = 0;
  bool conv = false, badpiv = false;
  pnqp_lane<R, M>(H, q, lo, hi, a.has_init != 0, x, fac, fm, it, conv, badpiv, a.n_iter);
  R* ox = (R*)a.x + (size_t)b * M;
  R* oH = (R*)a.Hfree + (size_t)b * M * M;
#pragma unroll
  for (int i = 0; i < M; ++i) {
    ox[i] = x[i];
    a.If[(size_t)b * M + i] = (fm >> i) & 1u;
#pragma unroll
    for (int j = 0; j < M; ++j) {   // H_ of the returning iteration (reference mpc/pnqp.py:46-48)
      const bool ff = ((fm >> i) & 1u) && ((fm >> j) & 1u);
      oH[i * M + j] = (ff ? H[i][j] : R(0)) + (i == j ? R(1e-11) : R(0));
    }
  }
  a.iters[b] = it;
  if (a.status != nullptr) a.status[b] = (conv ? 0 : 1) | (badpiv ? 4 : 0);
}

template <typename R>
static int pnqp_dispatch(const PnqpArgs& a, int n, cudaStream_t stream) {
  const int grid = (a.B + 127) / 128;
  switch (n) {
#define MPCB_PNQP_CASE(MM) \
  case MM: pnqp_kernel<R, MM><<<grid, 128, 0, stream>>>(a); break;
    MPCB_PNQP_CASE(1) MPCB_PNQP_CASE(2) MPCB_PNQP_CASE(3) MPCB_PNQP_CASE(4)
    MPCB_PNQP_CASE(5) MPCB_PNQP_CASE(6) MPCB_PNQP_CASE(7) MPCB_PNQP_CASE(8)
#undef MPCB_PNQP_CASE
    default: {
      const int ms = max_smem_optin();
      if (ms <= 0) return MPCB200_ERR_NO_DEVICE;
      if (n > pnqp_max_n((int)sizeof(R), ms)) return MPCB200_ERR_SMEM;
      return pnqp_cta_launch<R>(a, ms, stream);
    }
  }
  return cudaGetLastError() == cudaSuccess ? MPCB200_OK : MPCB200_ERR_LAUNCH;
}

// The implicit gradient (contract in include/mpcb200.h, CTA form in pnqp_large.cu) for n <= 8, one thread per QP:
// the free block H_ as pnqp_lane builds it, its LDL^T in registers, v = H_^{-1} g_F (exactly 0 off F).
template <typename R, int M>
__global__ void __launch_bounds__(128) pnqp_backward_kernel(const PnqpGradArgs a) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.B) return;
  const R* gH = (const R*)a.H + (size_t)b * M * M;
  const R* gg = (const R*)a.g + (size_t)b * M;
  unsigned fm = 0u;
#pragma unroll
  for (int i = 0; i < M; ++i) fm |= (a.If[(size_t)b * M + i] != 0 ? 1u : 0u) << i;
  R A[M][M], gm[M], v[M];
#pragma unroll
  for (int i = 0; i < M; ++i) {                // pnqp.py:44-48
    const bool fi = (fm >> i) & 1u;
    gm[i] = fi ? gg[i] : R(0);
#pragma unroll
    for (int j = 0; j < M; ++j) A[i][j] = (fi && ((fm >> j) & 1u)) ? gH[i * M + j] : R(0);
    A[i][i] += R(1e-11);
  }
  Ldl<R, M> fac;
  fac.factor(A);
  fac.solve(gm, v);
  R x[M];
#pragma unroll
  for (int i = 0; i < M; ++i) x[i] = ((const R*)a.x)[(size_t)b * M + i];
  R* dH = (R*)a.dH + (size_t)b * M * M;
#pragma unroll
  for (int i = 0; i < M; ++i) {
    const bool fi = (fm >> i) & 1u;
#pragma unroll
    for (int j = 0; j < M; ++j) dH[i * M + j] = fi ? -v[i] * x[j] : R(0);
    R dq = R(0), dlo = R(0), dhi = R(0);
    if (fi) {
      dq = -v[i];
    } else {
      R s = R(0);
#pragma unroll
      for (int k = 0; k < M; ++k)
        if ((fm >> k) & 1u) s += gH[k * M + i] * v[k];
      const R r = gg[i] - s;
      if (x[i] == ((const R*)a.lo)[(size_t)b * M + i]) dlo = r;
      else dhi = r;
    }
    ((R*)a.dq)[(size_t)b * M + i] = dq;
    ((R*)a.dlo)[(size_t)b * M + i] = dlo;
    ((R*)a.dhi)[(size_t)b * M + i] = dhi;
  }
  if (a.status != nullptr) a.status[b] = fac.bad ? (int)MPCB200_ST_BAD_PIVOT : 0;
}

template <typename R>
static int pnqp_backward_impl(int32_t B, int32_t n, const R* H, const R* x, const uint8_t* If, const R* lower,
                              const R* upper, const R* dl_dx, R* dH, R* dq, R* dlower, R* dupper, int32_t* status,
                              void* stream) {
  if (B <= 0 || n <= 0) return MPCB200_ERR_BAD_DIMS;
  if (!H || !x || !If || !lower || !upper || !dl_dx || !dH || !dq || !dlower || !dupper)
    return MPCB200_ERR_NULL_POINTER;
  if (n > pnqp_max_n((int)sizeof(R), smem_optin_or_h100())) return MPCB200_ERR_SMEM;   // the forward's limit
  const int ms = max_smem_optin();
  if (ms <= 0) return MPCB200_ERR_NO_DEVICE;
  PnqpGradArgs a;
  a.B = B; a.n = n;
  a.H = H; a.x = x; a.lo = lower; a.hi = upper; a.g = dl_dx; a.If = If;
  a.dH = dH; a.dq = dq; a.dlo = dlower; a.dhi = dupper; a.status = status;
  const cudaStream_t st = (cudaStream_t)stream;
  const int grid = (B + 127) / 128;
  switch (n) {
#define MPCB_PNQP_BWD_CASE(MM) \
  case MM: pnqp_backward_kernel<R, MM><<<grid, 128, 0, st>>>(a); break;
    MPCB_PNQP_BWD_CASE(1) MPCB_PNQP_BWD_CASE(2) MPCB_PNQP_BWD_CASE(3) MPCB_PNQP_BWD_CASE(4)
    MPCB_PNQP_BWD_CASE(5) MPCB_PNQP_BWD_CASE(6) MPCB_PNQP_BWD_CASE(7) MPCB_PNQP_BWD_CASE(8)
#undef MPCB_PNQP_BWD_CASE
    default: return pnqp_cta_backward_launch<R>(a, ms, st);
  }
  return cudaGetLastError() == cudaSuccess ? MPCB200_OK : MPCB200_ERR_LAUNCH;
}

template <typename R>
static int pnqp_impl(int32_t B, int32_t n, const R* H, const R* q, const R* lower, const R* upper,
                     const R* x_init, int32_t n_iter, R* x, R* H_free, uint8_t* If, int32_t* iters,
                     int32_t* status, void* stream) {
  if (B <= 0 || n <= 0 || n_iter < 1) return MPCB200_ERR_BAD_DIMS;
  if (!H || !q || !lower || !upper || !x || !H_free || !If || !iters) return MPCB200_ERR_NULL_POINTER;
  PnqpArgs a;
  a.B = B; a.n = n; a.n_iter = n_iter; a.has_init = x_init != nullptr;
  a.H = H; a.q = q; a.lo = lower; a.hi = upper; a.x_init = x_init;
  a.x = x; a.Hfree = H_free; a.If = If; a.iters = iters; a.status = status;
  return pnqp_dispatch<R>(a, n, (cudaStream_t)stream);
}
}  // namespace mpcb200

extern "C" {
int mpcb200_pnqp_f32(int32_t B, int32_t n, const float* H, const float* q, const float* lower,
                     const float* upper, const float* x_init, int32_t n_iter, float* x, float* H_free,
                     uint8_t* If, int32_t* iters, int32_t* status, void* stream) {
  return mpcb200::pnqp_impl<float>(B, n, H, q, lower, upper, x_init, n_iter, x, H_free, If, iters, status, stream);
}
int mpcb200_pnqp_f64(int32_t B, int32_t n, const double* H, const double* q, const double* lower,
                     const double* upper, const double* x_init, int32_t n_iter, double* x, double* H_free,
                     uint8_t* If, int32_t* iters, int32_t* status, void* stream) {
  return mpcb200::pnqp_impl<double>(B, n, H, q, lower, upper, x_init, n_iter, x, H_free, If, iters, status, stream);
}
int mpcb200_pnqp_backward_f32(int32_t B, int32_t n, const float* H, const float* x, const uint8_t* If,
                              const float* lower, const float* upper, const float* dl_dx, float* dH, float* dq,
                              float* dlower, float* dupper, int32_t* status, void* stream) {
  return mpcb200::pnqp_backward_impl<float>(B, n, H, x, If, lower, upper, dl_dx, dH, dq, dlower, dupper, status,
                                            stream);
}
int mpcb200_pnqp_backward_f64(int32_t B, int32_t n, const double* H, const double* x, const uint8_t* If,
                              const double* lower, const double* upper, const double* dl_dx, double* dH, double* dq,
                              double* dlower, double* dupper, int32_t* status, void* stream) {
  return mpcb200::pnqp_backward_impl<double>(B, n, H, x, If, lower, upper, dl_dx, dH, dq, dlower, dupper, status,
                                             stream);
}
int32_t mpcb200_pnqp_max_n(int32_t elem_size) {
  if (elem_size != 4 && elem_size != 8) return 0;
  return mpcb200::pnqp_max_n(elem_size, mpcb200::smem_optin_or_h100());
}
}
