// pnqp.cuh - what the two standalone pnqp launchers share: the argument block, and the entry points of the
// CTA-per-QP kernel (pnqp_large.cu) that pnqp.cu dispatches to for n > 8.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>

namespace mpcb200 {

struct PnqpArgs {
  int B, n, n_iter, has_init;
  const void *H, *q, *lo, *hi, *x_init;
  void *x, *Hfree;
  unsigned char* If;
  int* iters;
  int* status;
};

// the implicit gradient of one batch of solutions (mpcb200_pnqp_backward_*): inputs H, x, If, lo, hi, g = dL/dx;
// outputs dH, dq, dlo, dhi and status
struct PnqpGradArgs {
  int B, n;
  const void *H, *x, *lo, *hi, *g;
  const unsigned char* If;
  void *dH, *dq, *dlo, *dhi;
  int* status;
};

// opt-in dynamic shared memory per block of the current device (bytes); <= 0 if no usable sm_90 device (api.cu)
int max_smem_optin();
// the same for a query that must answer without a device: the H100's limit (kOptinAssumed) when none is usable
int smem_optin_or_h100();

// dynamic shared memory (bytes) of the CTA-per-QP kernel for an n x n QP of elem_size-byte elements
size_t pnqp_cta_smem_bytes(int n, int elem_size);
// the largest n the standalone pnqp solves with max_smem bytes of shared memory per block (at least 8: the
// thread-per-QP kernel holds n <= 8 in registers)
int pnqp_max_n(int elem_size, int max_smem);
// one CTA per QP, 8 < n <= pnqp_max_n; returns an MPCB200_* code
template <typename R>
int pnqp_cta_launch(const PnqpArgs& a, int max_smem, cudaStream_t stream);
// the implicit gradient with one CTA per QP, 8 < n <= pnqp_max_n (it needs less shared memory than the forward)
template <typename R>
int pnqp_cta_backward_launch(const PnqpGradArgs& a, int max_smem, cudaStream_t stream);

}  // namespace mpcb200
