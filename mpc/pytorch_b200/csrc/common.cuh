// common.cuh - PTX helpers (mbarrier, 1-D bulk TMA), the launchers' shared-memory opt-in and tiny per-lane
// linear algebra.
// sm_90a only.  No reference code: the algorithms these serve are cited in lqr_step.cuh.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <atomic>
#include "../../../include/mpcb200.h"

namespace mpcb200 {

#define MPCB_DEV __device__ __forceinline__

// ------------------------------------------------------------------ mbarrier / bulk copy
MPCB_DEV uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

MPCB_DEV void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
MPCB_DEV void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }

MPCB_DEV void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
MPCB_DEV void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
               : "memory");
}
MPCB_DEV bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(smem_u32(bar)), "r"(parity)
      : "memory");
  return ok != 0;
}
MPCB_DEV void mbar_wait(uint64_t* bar, uint32_t parity) {
  // plain try_wait blocks in hardware for a bounded time; the suspend-hint form compiles to a
  // NANOSLEEP polling loop whose wake-up granularity hurts a latency-bound consumer
  while (!mbar_try_wait(bar, parity)) {
  }
}
// 1-D bulk TMA: global -> shared, completion signalled on an mbarrier (UBLKCP in SASS).
// dst/src 16-byte aligned, bytes a multiple of 16.
MPCB_DEV void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// The same copy with an L2 cache policy (createpolicy) for the lines it reads.
MPCB_DEV void bulk_g2s(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar, uint64_t policy) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;" ::"r"(
          smem_u32(dst_smem)),
      "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)), "l"(policy)
      : "memory");
}
MPCB_DEV uint64_t l2_evict_first_policy() {
  uint64_t p;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
  return p;
}
// CTA-wide named barrier.  `bar.sync` is the .aligned form (the whole warp must execute it
// convergently); callers reach it right after lane-divergent code, so reconverge first and use the
// non-aligned `barrier.sync` (compute-sanitizer synccheck flagged the aligned form here).
MPCB_DEV void named_bar_sync(int id, int nthreads) {
  __syncwarp();
  asm volatile("barrier.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// H100 opt-in shared memory per block, what the device-free queries assume when no device is visible
constexpr int kOptinAssumed = 227 * 1024;

// Raise Kern's opt-in dynamic shared-memory limit to max_smem_optin, once per device (the attribute is per
// context).  Keyed on the kernel itself: instances of one template have the same type.  Atomic flags:
// concurrent callers (one host thread per GPU is the expected pattern) may both set the attribute, which is
// idempotent, but never read a torn value.
template <auto Kern>
int allow_smem_optin(int max_smem_optin) {
  static std::atomic<int> configured[64];
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return MPCB200_ERR_NO_DEVICE;
  if (configured[dev].load(std::memory_order_acquire) < max_smem_optin) {
    if (cudaFuncSetAttribute(Kern, cudaFuncAttributeMaxDynamicSharedMemorySize, max_smem_optin) != cudaSuccess)
      return MPCB200_ERR_LAUNCH;
    configured[dev].store(max_smem_optin, std::memory_order_release);
  }
  return MPCB200_OK;
}

// ------------------------------------------------------------------ compile-time helpers
__host__ __device__ constexpr int round_up(int v, int a) { return (v + a - 1) / a * a; }
template <typename R, int V>
struct VecLoad;
template <>
struct VecLoad<float, 4> {
  MPCB_DEV static void ld(const float* p, float* o) {
    float4 v = *reinterpret_cast<const float4*>(p);
    o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
  }
};
template <>
struct VecLoad<float, 2> {
  MPCB_DEV static void ld(const float* p, float* o) {
    float2 v = *reinterpret_cast<const float2*>(p);
    o[0] = v.x; o[1] = v.y;
  }
};
template <>
struct VecLoad<float, 1> {
  MPCB_DEV static void ld(const float* p, float* o) { o[0] = p[0]; }
};
template <>
struct VecLoad<double, 2> {
  MPCB_DEV static void ld(const double* p, double* o) {
    double2 v = *reinterpret_cast<const double2*>(p);
    o[0] = v.x; o[1] = v.y;
  }
};
template <>
struct VecLoad<double, 1> {
  MPCB_DEV static void ld(const double* p, double* o) { o[0] = p[0]; }
};

// Load CNT contiguous elements whose start is aligned to V elements.
template <typename R, int CNT, int V>
MPCB_DEV void load_vec(const R* p, R (&out)[CNT]) {
  static_assert(CNT % V == 0, "vector width must divide count");
#pragma unroll
  for (int e = 0; e < CNT; e += V) VecLoad<R, V>::ld(p + e, &out[e]);
}

template <typename R>
MPCB_DEV R shfl(R v, int src) { return __shfl_sync(0xffffffffu, v, src); }

// ------------------------------------------------------------------ pairs
// Two independent lanes of arithmetic.  Hopper has no packed fp32 FMA, so a pair is two scalar FFMAs;
// the pair layout still matters: every operand a lane loads from shared memory feeds both of them.
// fmaf / __fmul_rn keep each lane-op a single IEEE-rounded operation (no contraction across ops).
template <typename R>
struct P2 {
  R x, y;
};
MPCB_DEV P2<float> fma2(P2<float> a, P2<float> b, P2<float> c) {   // a*b + c
  return {fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y)};
}
MPCB_DEV P2<float> mul2(P2<float> a, P2<float> b) { return {__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)}; }
MPCB_DEV P2<double> fma2(P2<double> a, P2<double> b, P2<double> c) {
  return {a.x * b.x + c.x, a.y * b.y + c.y};
}
MPCB_DEV P2<double> mul2(P2<double> a, P2<double> b) { return {a.x * b.x, a.y * b.y}; }

// Fixed-length register vector stored as pairs (odd lengths carry one zero pad lane).
template <typename R, int L>
struct Vec {
  static constexpr int NP = (L + 1) / 2;
  P2<R> p[NP];
  MPCB_DEV R get(int i) const { return (i & 1) ? p[i >> 1].y : p[i >> 1].x; }     // i: compile-time after unrolling
  MPCB_DEV void set(int i, R v) {
    if (i & 1) p[i >> 1].y = v;
    else p[i >> 1].x = v;
  }
  MPCB_DEV void zero() {
#pragma unroll
    for (int k = 0; k < NP; ++k) p[k] = {R(0), R(0)};
  }
  // this += a * s
  MPCB_DEV void axpy(const Vec& a, R s) {
#pragma unroll
    for (int k = 0; k < NP; ++k) p[k] = fma2(a.p[k], P2<R>{s, s}, p[k]);
  }
  // sum_i this[i] * b[i]  (even/odd partial sums, then one add)
  MPCB_DEV R dot(const Vec& b) const {
    P2<R> acc = mul2(p[0], b.p[0]);
#pragma unroll
    for (int k = 1; k < NP; ++k) acc = fma2(p[k], b.p[k], acc);
    return acc.x + acc.y;
  }
  // load L contiguous elements; V = vector width (elements) the address is aligned to
  template <int V>
  MPCB_DEV void load(const R* ptr) {
    R tmp[NP * 2];
    constexpr int LV = (L / V) * V;
    if constexpr (LV > 0) {
      R t2[LV > 0 ? LV : 1];
      load_vec<R, (LV > 0 ? LV : V), V>(ptr, t2);
#pragma unroll
      for (int i = 0; i < LV; ++i) tmp[i] = t2[i];
    }
#pragma unroll
    for (int i = LV; i < L; ++i) tmp[i] = ptr[i];
    if constexpr (L & 1) tmp[L] = R(0);
#pragma unroll
    for (int k = 0; k < NP; ++k) p[k] = {tmp[2 * k], tmp[2 * k + 1]};
  }
  // store L contiguous elements; V = vector width (elements) the address is aligned to
  template <int V>
  MPCB_DEV void store(R* ptr) const {
    constexpr int LV = (L / V) * V;
    if constexpr (V == 4 && sizeof(R) == 4) {
#pragma unroll
      for (int e = 0; e < LV; e += 4)
        *reinterpret_cast<float4*>(ptr + e) = make_float4(get(e), get(e + 1), get(e + 2), get(e + 3));
    } else if constexpr (V == 2 && sizeof(R) == 4) {
#pragma unroll
      for (int e = 0; e < LV; e += 2) *reinterpret_cast<float2*>(ptr + e) = make_float2(get(e), get(e + 1));
    } else if constexpr (V == 2 && sizeof(R) == 8) {
#pragma unroll
      for (int e = 0; e < LV; e += 2) *reinterpret_cast<double2*>(ptr + e) = make_double2(get(e), get(e + 1));
    } else {
#pragma unroll
      for (int e = 0; e < LV; ++e) ptr[e] = get(e);
    }
#pragma unroll
    for (int e = LV; e < L; ++e) ptr[e] = get(e);
  }
  // strided gather: element i from ptr[i * stride]
  MPCB_DEV void gather(const R* ptr, int stride) {
#pragma unroll
    for (int i = 0; i < L; ++i) set(i, ptr[i * stride]);
    if constexpr (L & 1) p[NP - 1].y = R(0);
  }
};

// compile-time loop: f(std::integral_constant<int, I>) for I in [B, E)
template <int I>
struct IC {
  static constexpr int value = I;
  MPCB_DEV constexpr operator int() const { return I; }
};
template <int B, int E, typename Fn>
MPCB_DEV void static_for(Fn&& f) {
  if constexpr (B < E) {
    f(IC<B>{});
    static_for<B + 1, E>(f);
  }
}

// widest vector width (elements) guaranteed for an address `base + off` when base is 16-byte
// aligned and off is a multiple of `off_elems` elements
template <typename R>
__host__ __device__ constexpr int align_elems(int off_elems) {
  return (off_elems * (int)sizeof(R)) % 16 == 0 ? 16 / (int)sizeof(R)
         : (off_elems * (int)sizeof(R)) % 8 == 0 ? 8 / (int)sizeof(R)
                                                 : 1;
}

// ------------------------------------------------------------------ M x M LDL^T (per lane, registers)
// Factor a symmetric matrix A = L D L^T (unit lower L).  Only the lower triangle of A is read.
// Masked (clamped) indices are presented by the caller as zero rows/cols with a tiny diagonal,
// exactly how the reference builds H_ (mpc/pnqp.py:46-48) and Qt_uu_ (mpc/lqr_step.py:107-116):
// they decouple, and a zero right-hand side gives an exactly zero solution component.
// reciprocal: MUFU.RCP + one Newton step for float (<= 1 ulp, no slow-path call), IEEE for double
MPCB_DEV float recip(float d) {
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(d));
  return fmaf(r, fmaf(-d, r, 1.0f), r);
}
MPCB_DEV double recip(double d) { return 1.0 / d; }

template <typename R, int M>
struct Ldl {
  R L[M][M];
  R d[M];
  R dinv[M];
  bool bad;  // a pivot was <= 0 or not finite

  MPCB_DEV void factor(const R (&A)[M][M]) {
    bad = false;
#pragma unroll
    for (int j = 0; j < M; ++j) {
      R dj = A[j][j];
#pragma unroll
      for (int k = 0; k < j; ++k) dj -= L[j][k] * L[j][k] * d[k];
      bad = bad || !(dj > R(0));
      d[j] = dj;
      dinv[j] = recip(dj);
#pragma unroll
      for (int i = j + 1; i < M; ++i) {
        R s = A[i][j];
#pragma unroll
        for (int k = 0; k < j; ++k) s -= L[i][k] * L[j][k] * d[k];
        L[i][j] = s * dinv[j];
      }
    }
  }
  // x = A^{-1} b
  MPCB_DEV void solve(const R (&b)[M], R (&x)[M]) const {
    R y[M];
#pragma unroll
    for (int i = 0; i < M; ++i) {
      R s = b[i];
#pragma unroll
      for (int k = 0; k < i; ++k) s -= L[i][k] * y[k];
      y[i] = s;
    }
#pragma unroll
    for (int i = M - 1; i >= 0; --i) {
      R s = y[i] * dinv[i];
#pragma unroll
      for (int k = i + 1; k < M; ++k) s -= L[k][i] * x[k];
      x[i] = s;
    }
  }
};

}  // namespace mpcb200
