// api.cu - the C ABI declared in include/mpcb200.h: argument checks, (n,m) dispatch, launch.
#include <atomic>
#include <cstdlib>
#include <cstring>

#include "../../../include/mpcb200.h"
#include "ilqr.cuh"
#include "lqr_grad.cuh"
#include "lqr_large.cuh"
#include "lqr_rollout.cuh"
#include "lqr_step.cuh"
#include "pnqp.cuh"

namespace mpcb200 {
#define MPCB200_INST(n, m)                                                  \
  int step_f32__##n##_##m(const StepArgs&, int, cudaStream_t);              \
  int step_f64__##n##_##m(const StepArgs&, int, cudaStream_t);              \
  int grad_f32__##n##_##m(const GradArgs&, cudaStream_t);                   \
  int grad_f64__##n##_##m(const GradArgs&, cudaStream_t);                   \
  int pws_f32__##n##_##m(int, int);                                         \
  int pws_f64__##n##_##m(int, int);                                         \
  int roll_f32__##n##_##m(const RolloutArgs&, cudaStream_t);                \
  int roll_f64__##n##_##m(const RolloutArgs&, cudaStream_t);                \
  size_t smem_f32__##n##_##m(int);                                          \
  size_t smem_f64__##n##_##m(int);
#include "instances.def"
#undef MPCB200_INST

struct Entry {
  int n, m;
  int (*step32)(const StepArgs&, int, cudaStream_t);
  int (*step64)(const StepArgs&, int, cudaStream_t);
  int (*grad32)(const GradArgs&, cudaStream_t);
  int (*grad64)(const GradArgs&, cudaStream_t);
  size_t (*smem32)(int);
  size_t (*smem64)(int);
  int (*roll32)(const RolloutArgs&, cudaStream_t);
  int (*roll64)(const RolloutArgs&, cudaStream_t);
  int (*pws32)(int, int);
  int (*pws64)(int, int);
};
static const Entry kTable[] = {
#define MPCB200_INST(n, m)                                                                  \
  {n, m, step_f32__##n##_##m, step_f64__##n##_##m, grad_f32__##n##_##m, grad_f64__##n##_##m, \
   smem_f32__##n##_##m, smem_f64__##n##_##m, roll_f32__##n##_##m, roll_f64__##n##_##m,   \
   pws_f32__##n##_##m, pws_f64__##n##_##m},
#include "instances.def"
#undef MPCB200_INST
};
static const int kTableLen = (int)(sizeof(kTable) / sizeof(kTable[0]));

// dynamics-only step instances (inst_dyn.cu): no gradient or rollout kernels, and not listed by mpcb200_supported*
#define MPCB200_DYN_INST(kind, n, m)                                        \
  int dstep_f32__##kind(const StepArgs&, int, cudaStream_t);                \
  int dstep_f64__##kind(const StepArgs&, int, cudaStream_t);                \
  int dpws_f32__##kind(int, int);                                           \
  int dpws_f64__##kind(int, int);                                           \
  size_t dsmem_f32__##kind(int);                                            \
  size_t dsmem_f64__##kind(int);
#include "dyn_instances.def"
#undef MPCB200_DYN_INST
struct DynEntry {
  int kind;
  Entry e;
};
static const DynEntry kDynTable[] = {
#define MPCB200_DYN_INST(kind, n, m)                                                                        \
  {kind, {n, m, dstep_f32__##kind, dstep_f64__##kind, nullptr, nullptr, dsmem_f32__##kind, dsmem_f64__##kind, \
          nullptr, nullptr, dpws_f32__##kind, dpws_f64__##kind}},
#include "dyn_instances.def"
#undef MPCB200_DYN_INST
};

static const Entry* find(int n, int m) {
  for (int i = 0; i < kTableLen; ++i)
    if (kTable[i].n == n && kTable[i].m == m) return &kTable[i];
  return nullptr;
}
// the step instance of a call: the (n, m) instance, or for a passthrough kind its dynamics-only instance at exactly
// that kind's (n, m)
static const Entry* find_step(const mpcb200_dims* d) {
  if ((d->dynamics_kind & DYN_CTRL_PASSTHROUGH) == 0) return find(d->n, d->m);
  for (const DynEntry& de : kDynTable)
    if (de.kind == d->dynamics_kind && de.e.n == d->n && de.e.m == d->m) return &de.e;
  return nullptr;
}

// developer A/B knob MPCB200_KERNEL=3: the large-shape kernels (lqr_large.cu) also for shapes with an instance
static bool large_forced() {
  const char* k = std::getenv("MPCB200_KERNEL");
  return k != nullptr && std::atoi(k) == 3;
}
// the step, gradient and rollout of (n, m) run the large-shape kernels
static bool runs_large(int n, int m) { return find(n, m) == nullptr || large_forced(); }
static constexpr int kOptinAssumed = 227 * 1024;   // H100 opt-in shared memory per block, for device-free queries

static std::atomic<uint64_t> g_launches{0};
static thread_local int t_step_plan = 0;      // MPCB200_PLAN_* bits of this thread's last step launch

void record_step_plan(int plan) { t_step_plan = plan; }

// per-device opt-in shared memory limit (cached for up to 64 devices)
int max_smem_optin() {
  static std::atomic<int> cache[64];         // written once per device with the same value: safe from any thread
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return -1;
  if (dev < 0 || dev >= 64) return -1;
  if (cache[dev].load(std::memory_order_acquire) == 0) {
    int v = 0, major = 0;
    if (cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess) return -1;
    if (cudaDeviceGetAttribute(&major, cudaDevAttrComputeCapabilityMajor, dev) != cudaSuccess) return -1;
    if (major != 9) return -1;    // sm_90a cubin only
    cache[dev].store(v, std::memory_order_release);
  }
  return cache[dev].load(std::memory_order_acquire);
}

// element strides between the time slices of C, c, F and f.  Each *_tstride field of mpcb200_dims: 0 = dense (what a
// zero-initialised mpcb200_dims means), < 0 = time invariant (stride 0), > 0 = that many elements
struct TimeStrides { long long C, c, F, f; };
static TimeStrides time_strides(const mpcb200_dims* d) {
  auto ts = [](long long given, long long dense) { return given == 0 ? dense : (given < 0 ? 0 : given); };
  const long long B = d->B, n = d->n, p = d->n + d->m;
  return {ts(d->C_tstride, B * p * p), ts(d->c_tstride, B * p), ts(d->F_tstride, B * n * p), ts(d->f_tstride, B * n)};
}

static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

static int check_dims(const mpcb200_dims* d) {
  if (d == nullptr) return MPCB200_ERR_NULL_POINTER;
  if (d->B <= 0 || d->T <= 0 || d->n <= 0 || d->m <= 0) return MPCB200_ERR_BAD_DIMS;
  if (d->F_T != d->T - 1 && d->F_T != d->T) return MPCB200_ERR_BAD_DIMS;
  return MPCB200_OK;
}

// the step's option checks, one order for every entry point: an argument error gets the same code from each
static int check_bounds(const mpcb200_dims* d, const void* lo, const void* hi) {
  if (d->bounds_kind < 0 || d->bounds_kind > 2) return MPCB200_ERR_BAD_DIMS;
  if (d->bounds_kind == 2 && (lo == nullptr || hi == nullptr)) return MPCB200_ERR_NULL_POINTER;
  return MPCB200_OK;
}
static int check_step_options(const mpcb200_dims* d, const void* lo, const void* hi, const uint8_t* zero_mask) {
  if (const int rc = check_bounds(d, lo, hi)) return rc;
  if (d->has_zero_mask && zero_mask == nullptr) return MPCB200_ERR_NULL_POINTER;
  if (d->has_delta_u && d->bounds_kind == 0) return MPCB200_ERR_BAD_DIMS;   // reference lqr_step.py:195
  if (d->max_ls_iter < 1 || d->pnqp_max_iter < 1) return MPCB200_ERR_BAD_DIMS;
  return MPCB200_OK;
}

static bool known_shape_ok(const mpcb200_dims* d) {
  int n = 0, m = 0;
  return dyn_kind_dims(d->dynamics_kind, n, m) && d->n == n && d->m == m;
}

struct AdjExtra {      // fused-adjoint request riding on a step launch (api-internal)
  const void *c, *x, *u;
  void *dC, *dc, *dF, *df, *dx_init;
  int has_df, ok;
  long long c_ts;
};

template <typename R>
static int step_impl(const mpcb200_dims* d, const mpcb200_params* p, const R* C, const R* c, const R* F,
                     const R* f, const R* x_init, const R* cur_x, const R* cur_u, const R* u_lower,
                     const R* u_upper, const uint8_t* u_zero_I, R* new_x, R* new_u, R* costs,
                     R* full_du_norm, R* alphas, R* du_first, int32_t* qp_iters, uint8_t* free_mask, int32_t* status,
                     R* Ks, R* ks, void* stream, const AdjExtra* adj = nullptr) {
  int rc = check_dims(d);
  if (rc) return rc;
  if (p == nullptr || C == nullptr || c == nullptr || cur_x == nullptr || cur_u == nullptr)
    return MPCB200_ERR_NULL_POINTER;
  if (d->T > 1 && F == nullptr) return MPCB200_ERR_NULL_POINTER;
  if (d->has_f && f == nullptr) return MPCB200_ERR_NULL_POINTER;
  rc = check_step_options(d, u_lower, u_upper, u_zero_I);
  if (rc) return rc;
  if (d->do_rollout) {
    if (x_init == nullptr || new_x == nullptr || new_u == nullptr || costs == nullptr ||
        full_du_norm == nullptr || alphas == nullptr)
      return MPCB200_ERR_NULL_POINTER;
  } else if (Ks == nullptr || ks == nullptr) {
    return MPCB200_ERR_NULL_POINTER;
  }
  if ((Ks == nullptr) != (ks == nullptr)) return MPCB200_ERR_NULL_POINTER;
  const Entry* e = find_step(d);
  const bool large = d->dynamics_kind == DYN_LINEAR && runs_large(d->n, d->m);
  if (e == nullptr && !large) return MPCB200_ERR_UNSUPPORTED_DIMS;
  const int smem = max_smem_optin();
  if (smem <= 0) return MPCB200_ERR_NO_DEVICE;

  StepArgs a;
  std::memset(&a, 0, sizeof(a));
  a.B = d->B; a.T = d->T; a.F_T = d->F_T;
  a.has_f = d->has_f ? 1 : 0;
  a.bounds_kind = d->bounds_kind;
  a.has_mask = d->has_zero_mask ? 1 : 0;
  a.has_delta = d->has_delta_u ? 1 : 0;
  a.max_ls = d->max_ls_iter;
  a.pnqp_iters = d->pnqp_max_iter;
  a.do_rollout = d->do_rollout ? 1 : 0;
  a.u_lo = p->u_lo; a.u_hi = p->u_hi; a.delta_u = p->delta_u; a.ls_decay = p->ls_decay;
  a.C = C; a.c = c; a.F = F; a.f = f; a.x_init = x_init; a.cur_x = cur_x; a.cur_u = cur_u;
  a.u_lower = u_lower; a.u_upper = u_upper; a.zero_mask = u_zero_I;
  a.new_x = new_x; a.new_u = new_u; a.costs = costs; a.full_du_norm = full_du_norm; a.alphas = alphas;
  a.du_first = du_first; a.qp_iters = qp_iters; a.free_mask = free_mask; a.status = status; a.Ks = Ks; a.ks = ks;
  // bulk-TMA eligibility: every per-time-step span must start 16-byte aligned
  const size_t sz = sizeof(R);
  bool ok = aligned16(C) && aligned16(c) && aligned16(cur_x) && aligned16(cur_u) &&
            (F == nullptr || aligned16(F)) && (!d->has_f || aligned16(f)) &&
            (d->bounds_kind != 2 || (aligned16(u_lower) && aligned16(u_upper)));
  ok = ok && (x_init == nullptr || aligned16(x_init));
  ok = ok && ((size_t)d->B * d->m * sz) % 16 == 0 && ((size_t)d->B * d->n * sz) % 16 == 0;
  a.bulk_ok = ok ? 1 : 0;
  const TimeStrides ts = time_strides(d);
  a.C_ts = ts.C; a.c_ts = ts.c; a.F_ts = ts.F; a.f_ts = ts.f;
  ok = ok && (a.C_ts * sz) % 16 == 0 && (a.c_ts * sz) % 16 == 0 && (a.F_ts * sz) % 16 == 0 && (a.f_ts * sz) % 16 == 0;
  a.bulk_ok = ok ? 1 : 0;
  a.dyn_kind = d->dynamics_kind;
  if (a.dyn_kind != DYN_LINEAR) {
    if (!known_shape_ok(d)) return MPCB200_ERR_BAD_DIMS;
    for (int i = 0; i < 8; ++i) a.dp.p[i] = p->dyn[i];
  }
  if (large) {
    // the fused adjoint has no large-shape kernel: adjoint_impl then takes its three-launch route
    if (adj != nullptr) return MPCB200_ERR_UNSUPPORTED_DIMS;
    if (Ks == nullptr) return MPCB200_ERR_SMEM;      // the gains always go through the caller's Ks/ks
    const int n = d->n, m = d->m, p = n + m;
    auto spans = [&](const void* base, long long ts, long long span) {
      return base != nullptr && aligned16(base) && (ts * (long long)sz) % 16 == 0 && (span * (long long)sz) % 16 == 0;
    };
    unsigned bulk = 0u;
    if (spans(C, a.C_ts, (long long)p * p)) bulk |= LB_C;
    if (spans(F, a.F_ts, (long long)n * p)) bulk |= LB_F;
    if (spans(c, a.c_ts, p)) bulk |= LB_c;
    if (d->has_f && spans(f, a.f_ts, n)) bulk |= LB_f;
    if (spans(cur_x, (long long)d->B * n, n)) bulk |= LB_x;
    if (spans(cur_u, (long long)d->B * m, m)) bulk |= LB_u;
    if (d->bounds_kind == 2 && spans(u_lower, (long long)d->B * m, m) && spans(u_upper, (long long)d->B * m, m))
      bulk |= LB_BOX;
    t_step_plan = 0;
    rc = large_step_launch<R>(a, n, m, bulk, smem, (cudaStream_t)stream);
    if (rc == 0) g_launches.fetch_add(1);
    return rc;
  }
  if (const char* k = std::getenv("MPCB200_KERNEL")) a.impl = std::atoi(k);
  if (adj != nullptr) {          // fused KKT adjoint: column-pair kernel only
    if (!adj->ok || !a.bulk_ok || a.impl == 1) return MPCB200_ERR_UNSUPPORTED_DIMS;
    a.impl = 2;
    a.adj = 1; a.adj_has_df = adj->has_df; a.adj_c = adj->c; a.adj_x = adj->x; a.adj_u = adj->u;
    a.adj_dC = adj->dC; a.adj_dc = adj->dc; a.adj_dF = adj->dF; a.adj_df = adj->df; a.adj_dx_init = adj->dx_init;
    a.adj_c_ts = adj->c_ts;
  }   // developer A/B knob: 1 generic, 2 pair
  t_step_plan = 0;             // the launcher that launches records its plan
  rc =(sizeof(R) == 4 ? e->step32 : e->step64)(a, smem, (cudaStream_t)stream);
  if (rc == 0) g_launches.fetch_add(1);
  return rc;
}

template <typename R>
static int grad_impl(const mpcb200_dims* d, const R* C, const R* c, const R* F, const R* new_x,
                     const R* new_u, const R* dx, const R* du, const R* dl_dx, R* dx_init, R* dC, R* dc,
                     R* dF, R* df, void* workspace, void* stream) {
  int rc = check_dims(d);
  if (rc) return rc;
  if (C == nullptr || c == nullptr || new_x == nullptr || new_u == nullptr || dx == nullptr ||
      du == nullptr || dl_dx == nullptr || dx_init == nullptr || dC == nullptr || dc == nullptr)
    return MPCB200_ERR_NULL_POINTER;
  if (d->F_T > 0 && (F == nullptr || dF == nullptr)) return MPCB200_ERR_NULL_POINTER;
  const Entry* e = find(d->n, d->m);
  const bool large = runs_large(d->n, d->m);
  if (max_smem_optin() <= 0) return MPCB200_ERR_NO_DEVICE;
  GradArgs a;
  std::memset(&a, 0, sizeof(a));
  a.B = d->B; a.T = d->T; a.F_T = d->F_T; a.has_df = df != nullptr;
  a.C = C; a.c = c; a.F = F; a.new_x = new_x; a.new_u = new_u; a.dx = dx; a.du = du; a.dl_dx = dl_dx;
  a.dx_init = dx_init; a.dC = dC; a.dc = dc; a.dF = dF; a.df = df; a.workspace = workspace;
  const TimeStrides ts = time_strides(d);
  a.C_ts = ts.C; a.c_ts = ts.c; a.F_ts = ts.F;
  rc = large ? large_grad_launch<R>(a, d->n, d->m, (cudaStream_t)stream)
             : (sizeof(R) == 4 ? e->grad32 : e->grad64)(a, (cudaStream_t)stream);
  if (rc == 0) g_launches.fetch_add(workspace != nullptr ? 2 : 1);
  return rc;
}
// ---------------------------------------------------------------------------------------------
// KKT adjoint in one call (reference LQRStepFn.backward, mpc/lqr_step.py:312-407)
// ---------------------------------------------------------------------------------------------
struct AdjLayout {                    // workspace carve-up (byte offsets, every piece 256-byte aligned)
  size_t negr, zeros, dx, du, costate, scal, mask, maskf, Ks, ks, total;
  bool gains;                         // Ks/ks of the nested solve (the large-shape step keeps its gains there)
};
static size_t up256(size_t v) { return (v + 255) / 256 * 256; }
static AdjLayout adj_layout(int B, int T, int n, int m, size_t sz) {
  AdjLayout l;
  const size_t TB = (size_t)T * B;
  size_t o = 0;
  l.negr = o;    o += up256(TB * (n + m) * sz);
  l.zeros = o;   o += up256((TB * (n + m) + (size_t)B * n) * sz);     // cur_x, cur_u, x_init of the nested solve
  l.dx = o;      o += up256(TB * n * sz);
  l.du = o;      o += up256(TB * m * sz);
  l.costate = o; o += up256(2 * TB * n * sz);
  l.scal = o;    o += up256((size_t)3 * B * sz);
  l.mask = o;    o += up256(TB * m);
  l.maskf = o;   o += up256(TB * m * sz);                               // the same mask as element-typed 0/1 (rides on the TMA tile)
  l.gains = runs_large(n, m);
  l.Ks = l.ks = 0;
  if (l.gains) {
    l.Ks = o;    o += up256(TB * m * n * sz);
    l.ks = o;    o += up256(TB * m * sz);
  }
  l.total = o;
  return l;
}

template <typename R>
__global__ void __launch_bounds__(256)
adjoint_prep_kernel(int B, int T, int n, int m, int bounds_kind, R s_lo, R s_hi, const R* __restrict__ dl_dx,
                    const R* __restrict__ dl_du, const R* __restrict__ new_u, const R* __restrict__ u_lower,
                    const R* __restrict__ u_upper, R* __restrict__ negr, unsigned char* __restrict__ mask,
                    R* __restrict__ maskf, R* __restrict__ z0) {
  const size_t tb = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (tb >= (size_t)T * B) return;
  const int p = n + m;
  if (tb < (size_t)B)                              // x_init = 0 of the nested solve (saves a memset node)
    for (int i = 0; i < n; ++i) z0[tb * n + i] = R(0);
  for (int i = 0; i < n; ++i) negr[tb * p + i] = -dl_dx[tb * n + i];
  for (int q = 0; q < m; ++q) {
    negr[tb * p + n + q] = -dl_du[tb * m + q];
    unsigned char on = 0;
    if (bounds_kind != 0) {                       // reference :325-326
      const R u = new_u[tb * m + q];
      const R lo = bounds_kind == 2 ? u_lower[tb * m + q] : s_lo;
      const R hi = bounds_kind == 2 ? u_upper[tb * m + q] : s_hi;
      on = (fabs(u - lo) <= R(1e-8)) || (fabs(u - hi) <= R(1e-8));
    }
    mask[tb * m + q] = on;
    maskf[tb * m + q] = on ? R(1) : R(0);
  }
}

template <typename R>
static int adjoint_impl(const mpcb200_dims* d, const mpcb200_params* p, const R* C, const R* c, const R* F,
                        const R* new_x, const R* new_u, const R* dl_dx, const R* dl_du, const R* u_lower,
                        const R* u_upper, R* dx_init, R* dC, R* dc, R* dF, R* df, void* workspace,
                        size_t workspace_bytes, void* stream) {
  int rc = check_dims(d);
  if (rc) return rc;
  if (p == nullptr || C == nullptr || c == nullptr || new_x == nullptr || new_u == nullptr || dl_dx == nullptr ||
      dl_du == nullptr || dx_init == nullptr || dC == nullptr || dc == nullptr || workspace == nullptr)
    return MPCB200_ERR_NULL_POINTER;
  if (d->T > 1 && (F == nullptr || dF == nullptr)) return MPCB200_ERR_NULL_POINTER;
  rc = check_bounds(d, u_lower, u_upper);
  if (rc) return rc;
  if (d->has_f && df == nullptr) return MPCB200_ERR_NULL_POINTER;
  const AdjLayout l = adj_layout(d->B, d->T, d->n, d->m, sizeof(R));
  if (workspace_bytes < l.total || !aligned16(workspace)) return MPCB200_ERR_BAD_DIMS;
  cudaStream_t st = (cudaStream_t)stream;
  char* ws = (char*)workspace;
  R* negr = (R*)(ws + l.negr);
  R* zeros = (R*)(ws + l.zeros);
  R* dxs = (R*)(ws + l.dx);
  R* dus = (R*)(ws + l.du);
  R* scal = (R*)(ws + l.scal);
  unsigned char* mask = (unsigned char*)(ws + l.mask);
  const size_t TB = (size_t)d->T * d->B;
  R* zx = zeros;
  R* zu = zeros + TB * d->n;
  R* z0 = zu + TB * d->m;
  adjoint_prep_kernel<R><<<(unsigned)((TB + 255) / 256), 256, 0, st>>>(
      d->B, d->T, d->n, d->m, d->bounds_kind, (R)p->u_lo, (R)p->u_hi, dl_dx, dl_du, new_u, u_lower, u_upper, negr, mask,
      (R*)(ws + l.maskf), z0);
  if (cudaGetLastError() != cudaSuccess) return MPCB200_ERR_LAUNCH;
  g_launches.fetch_add(1);
  // nested masked LQR step from the zero trajectory (reference :328-340: MPC(lqr_iter=1, u_zero_I=I) with its defaults)
  mpcb200_dims ds = *d;
  ds.has_f = 0; ds.bounds_kind = 0; ds.has_zero_mask = 1; ds.has_delta_u = 0;
  ds.max_ls_iter = 10; ds.pnqp_max_iter = 20; ds.do_rollout = 1; ds.dynamics_kind = 0;
  ds.c_tstride = 0; ds.f_tstride = 0;         // c of the nested solve is the dense -r; C and F keep the caller's strides
  mpcb200_params ps;
  std::memset(&ps, 0, sizeof(ps));
  ps.ls_decay = 0.2;
  // Preferred: ONE launch of the column-pair kernel doing solve + costates + outer products (C, F read from HBM
  // once, d tau kept in shared memory).  Shapes / alignments it does not take fall through to the 3-launch path.
  {
    AdjExtra ax;
    ax.c = c; ax.x = new_x; ax.u = new_u; ax.dC = dC; ax.dc = dc; ax.dF = dF; ax.df = d->has_f ? df : nullptr;
    ax.dx_init = dx_init; ax.has_df = d->has_f ? 1 : 0;
    ax.c_ts = time_strides(d).c;
    ax.ok = aligned16(c) && aligned16(new_x) && aligned16(new_u) && (ax.c_ts * (long long)sizeof(R)) % 16 == 0;
    const R* maskf = (const R*)(ws + l.maskf);
    rc = step_impl<R>(&ds, &ps, C, negr, F, (const R*)nullptr, z0, zx, zu, maskf, maskf, mask,
                      dxs, dus, scal, scal + d->B, scal + 2 * d->B, (R*)nullptr, (int32_t*)nullptr,
                      (uint8_t*)nullptr, (int32_t*)nullptr, (R*)nullptr, (R*)nullptr, stream, &ax);
    if (rc == 0) return 0;
    if (rc != MPCB200_ERR_UNSUPPORTED_DIMS && rc != MPCB200_ERR_SMEM) return rc;
  }
  // 3-launch path: the nested solve really reads its (zero) nominal trajectory
  if (cudaMemsetAsync(zeros, 0, TB * (d->n + d->m) * sizeof(R), st) != cudaSuccess) return MPCB200_ERR_LAUNCH;
  R* Ks = l.gains ? (R*)(ws + l.Ks) : nullptr;
  R* ks = l.gains ? (R*)(ws + l.ks) : nullptr;
  rc = step_impl<R>(&ds, &ps, C, negr, F, (const R*)nullptr, z0, zx, zu, (const R*)nullptr, (const R*)nullptr, mask,
                    dxs, dus, scal, scal + d->B, scal + 2 * d->B, (R*)nullptr, (int32_t*)nullptr,
                    (uint8_t*)nullptr, (int32_t*)nullptr, Ks, ks, stream);
  if (rc == MPCB200_ERR_SMEM) return rc;     // long horizons: use the two-call path with Ks/ks buffers
  if (rc) return rc;
  mpcb200_dims dg = *d;
  return grad_impl<R>(&dg, C, c, F, new_x, new_u, dxs, dus, dl_dx, dx_init, dC, dc, dF, d->has_f ? df : (R*)nullptr,
                      ws + l.costate, stream);
}

template <typename R>
static int rollout_impl(const mpcb200_dims* d, const R* F, const R* f, const R* x_init, const R* u, R* x,
                        void* stream) {
  int rc = check_dims(d);
  if (rc) return rc;
  if (x_init == nullptr || u == nullptr || x == nullptr) return MPCB200_ERR_NULL_POINTER;
  if (d->T > 1 && F == nullptr) return MPCB200_ERR_NULL_POINTER;
  if (d->has_f && f == nullptr) return MPCB200_ERR_NULL_POINTER;
  const Entry* e = find(d->n, d->m);
  const bool large = runs_large(d->n, d->m);
  if (max_smem_optin() <= 0) return MPCB200_ERR_NO_DEVICE;
  RolloutArgs a;
  std::memset(&a, 0, sizeof(a));
  a.B = d->B; a.T = d->T; a.has_f = d->has_f ? 1 : 0;
  a.F = F; a.f = f; a.x_init = x_init; a.u = u; a.x = x;
  const TimeStrides ts = time_strides(d);
  a.F_ts = ts.F; a.f_ts = ts.f;
  rc = large ? large_rollout_launch<R>(a, d->n, d->m, (cudaStream_t)stream)
             : (sizeof(R) == 4 ? e->roll32 : e->roll64)(a, (cudaStream_t)stream);
  if (rc == 0) g_launches.fetch_add(1);
  return rc;
}
template <typename R>
static int dyn_impl(bool linearize, int kind, const double* dyn, int B, int T, const R* x_or_init, const R* u,
                    R* x_out, R* F, R* f, void* stream) {
  if (dyn == nullptr || x_or_init == nullptr || u == nullptr) return MPCB200_ERR_NULL_POINTER;
  int n = 0, m = 0;
  if (B <= 0 || T <= 0 || !dyn_kind_dims(kind, n, m)) return MPCB200_ERR_BAD_DIMS;
  if (max_smem_optin() <= 0) return MPCB200_ERR_NO_DEVICE;
  DynArgs a;
  std::memset(&a, 0, sizeof(a));
  a.B = B; a.T = T; a.kind = kind;
  for (int i = 0; i < 8; ++i) a.dp.p[i] = dyn[i];
  a.u = u;
  int rc;
  if (linearize) {
    if (T > 1 && (F == nullptr || f == nullptr)) return MPCB200_ERR_NULL_POINTER;
    a.x = x_or_init; a.F = F; a.f = f;
    rc = launch_dyn_linearize<R>(a, (cudaStream_t)stream);
  } else {
    if (x_out == nullptr) return MPCB200_ERR_NULL_POINTER;
    a.x_init = x_or_init; a.x_out = x_out;
    rc = launch_dyn_rollout<R>(a, (cudaStream_t)stream);
  }
  if (rc == 0 && !(linearize && T == 1)) g_launches.fetch_add(1);
  return rc;
}

// ---------------------------------------------------------------------------------------------
// the iLQR loop of MPC.forward as one CUDA graph (reference mpc/mpc.py:244-301)
// ---------------------------------------------------------------------------------------------
// dims of the step inside the loop: the caller's, with the rollout on and, for a known system, the workspace F, f
static mpcb200_dims ilqr_step_dims(const mpcb200_dims* d) {
  mpcb200_dims ds = *d;
  ds.do_rollout = 1;
  if (d->dynamics_kind != DYN_LINEAR) {
    ds.F_T = d->T - 1; ds.has_f = d->T > 1 ? 1 : 0; ds.F_tstride = 0; ds.f_tstride = 0;
  }
  return ds;
}

struct IlqrLayout {                   // workspace carve-up (byte offsets, every piece 256-byte aligned)
  size_t u, x, new_x, new_u, costs, fdn_step, alphas, du_first, status, fdn, flags, state, F, f, Ks, ks, total;
  bool gains;
};
static IlqrLayout ilqr_layout(const mpcb200_dims* d, size_t sz) {
  IlqrLayout l;
  const size_t TB = (size_t)d->T * d->B, B = d->B;
  const size_t n = d->n, m = d->m;
  size_t o = 0;
  l.u = o;        o += up256(TB * m * sz);
  l.x = o;        o += up256(TB * n * sz);
  l.new_x = o;    o += up256(TB * n * sz);
  l.new_u = o;    o += up256(TB * m * sz);
  l.costs = o;    o += up256(B * sz);
  l.fdn_step = o; o += up256(B * sz);
  l.alphas = o;   o += up256(B * sz);
  l.du_first = o; o += up256(TB * m * sz);
  l.status = o;   o += up256(B * sizeof(int32_t));
  l.fdn = o;      o += up256(B * sz);
  l.flags = o;    o += up256(B);
  l.state = o;    o += up256(sizeof(IlqrState));
  l.F = l.f = 0;
  if (d->dynamics_kind != DYN_LINEAR) {         // the linearisation of a known system, rewritten every iteration
    const size_t TB1 = (size_t)(d->T > 1 ? d->T - 1 : 0) * B;
    l.F = o;      o += up256(TB1 * n * (n + m) * sz);
    l.f = o;      o += up256(TB1 * n * sz);
  }
  const mpcb200_dims ds = ilqr_step_dims(d);
  l.gains = mpcb200_step_prefers_workspace(&ds, (int32_t)sz) != 0;
  l.Ks = l.ks = 0;
  if (l.gains) {
    l.Ks = o;     o += up256(TB * m * n * sz);
    l.ks = o;     o += up256(TB * m * sz);
  }
  l.total = o;
  return l;
}

// argument checks that need no device: every error is reported before anything is captured or launched
template <typename R>
static int ilqr_check(const mpcb200_dims* d, const mpcb200_params* p, const mpcb200_ilqr_opts* o, const R* C,
                      const R* c, const R* F, const R* f, const R* x_init, const R* u_lower, const R* u_upper,
                      const uint8_t* u_zero_I, const R* best_x, const R* best_u, const R* best_costs,
                      const R* best_fdn, const int32_t* info, const void* workspace, size_t workspace_bytes) {
  int rc = check_dims(d);
  if (rc) return rc;
  if (p == nullptr || o == nullptr || C == nullptr || c == nullptr || x_init == nullptr || best_x == nullptr ||
      best_u == nullptr || best_costs == nullptr || best_fdn == nullptr || info == nullptr || workspace == nullptr)
    return MPCB200_ERR_NULL_POINTER;
  if (o->lqr_iter < 1 || o->m_ref < 1 || o->m_ref > d->m) return MPCB200_ERR_BAD_DIMS;
  if (d->dynamics_kind != DYN_LINEAR) {
    if (!known_shape_ok(d)) return MPCB200_ERR_BAD_DIMS;
  } else {
    if (d->T > 1 && F == nullptr) return MPCB200_ERR_NULL_POINTER;
    if (d->has_f && f == nullptr) return MPCB200_ERR_NULL_POINTER;
  }
  rc = check_step_options(d, u_lower, u_upper, u_zero_I);
  if (rc) return rc;
  if (d->dynamics_kind != DYN_LINEAR && find_step(d) == nullptr) return MPCB200_ERR_UNSUPPORTED_DIMS;
  const IlqrLayout l = ilqr_layout(d, sizeof(R));
  if (workspace_bytes < l.total || (reinterpret_cast<uintptr_t>(workspace) & 255u) != 0) return MPCB200_ERR_BAD_DIMS;
  return MPCB200_OK;
}

// Library-owned streams of this thread on the current device: [0] records a graph the caller does not capture,
// [1] records the loop body.  Capture only records work on them; nothing ever executes on them.
static cudaStream_t ilqr_stream(int which) {
  static thread_local cudaStream_t streams[64][2] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  cudaStream_t& s = streams[dev][which];
  if (s == nullptr && cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) s = nullptr;
  return s;
}

// Adds the init kernel and the `while` node (body recorded on `bs`) to the graph `os` is capturing.
template <typename R>
static int ilqr_record(cudaStream_t os, cudaStream_t bs, const mpcb200_dims* d, const mpcb200_params* p,
                       const mpcb200_ilqr_opts* o, const R* C, const R* c, const R* F, const R* f, const R* x_init,
                       const R* u_init, const R* u_lower, const R* u_upper, const uint8_t* u_zero_I, R* best_x,
                       R* best_u, R* best_costs, R* best_fdn, int32_t* info, void* workspace) {
  const IlqrLayout l = ilqr_layout(d, sizeof(R));
  char* ws = (char*)workspace;
  R* u = (R*)(ws + l.u);
  R* x = (R*)(ws + l.x);
  R* new_x = (R*)(ws + l.new_x);
  R* new_u = (R*)(ws + l.new_u);
  R* costs = (R*)(ws + l.costs);
  R* du_first = (R*)(ws + l.du_first);
  int32_t* status = (int32_t*)(ws + l.status);
  R* fdn = (R*)(ws + l.fdn);
  uint8_t* flags = (uint8_t*)(ws + l.flags);
  IlqrState* st = (IlqrState*)(ws + l.state);
  const int B = d->B, T = d->T, N = d->n, M = d->m;
  const size_t TB = (size_t)T * B;
  if (ilqr_launch_init<R>(TB * M, u_init, u, st, info, os) != 0) return MPCB200_ERR_LAUNCH;
  g_launches.fetch_add(1);

  cudaStreamCaptureStatus cst = cudaStreamCaptureStatusNone;
  cudaGraph_t g = nullptr;
  const cudaGraphNode_t* deps = nullptr;
  size_t ndeps = 0;
  if (cudaStreamGetCaptureInfo(os, &cst, nullptr, &g, &deps, &ndeps) != cudaSuccess ||
      cst != cudaStreamCaptureStatusActive)
    return MPCB200_ERR_LAUNCH;
  cudaGraphConditionalHandle handle;
  if (cudaGraphConditionalHandleCreate(&handle, g, 1, cudaGraphCondAssignDefault) != cudaSuccess) {
    cudaGetLastError();
    return MPCB200_ERR_NO_GRAPH_COND;
  }
  cudaGraphNodeParams np = {cudaGraphNodeTypeConditional};
  np.conditional.handle = handle;
  np.conditional.type = cudaGraphCondTypeWhile;
  np.conditional.size = 1;
  cudaGraphNode_t loop;
  if (cudaGraphAddNode(&loop, g, deps, ndeps, &np) != cudaSuccess) {
    cudaGetLastError();
    return MPCB200_ERR_NO_GRAPH_COND;
  }
  if (cudaStreamUpdateCaptureDependencies(os, &loop, 1, cudaStreamSetCaptureDependencies) != cudaSuccess)
    return MPCB200_ERR_LAUNCH;

  // the body: the library's own launchers, recorded on bs (same plan selection as a direct call)
  if (cudaStreamBeginCaptureToGraph(bs, np.conditional.phGraph_out[0], nullptr, nullptr, 0,
                                    cudaStreamCaptureModeRelaxed) != cudaSuccess)
    return MPCB200_ERR_LAUNCH;
  const mpcb200_dims ds = ilqr_step_dims(d);
  const R* Fs = F;
  const R* fs = f;
  int rc;
  if (d->dynamics_kind == DYN_LINEAR) {
    rc = rollout_impl<R>(d, F, f, x_init, u, x, bs);
  } else {
    R* Fw = (R*)(ws + l.F);
    R* fw = (R*)(ws + l.f);
    rc = dyn_impl<R>(false, d->dynamics_kind, p->dyn, B, T, x_init, u, x, nullptr, nullptr, bs);
    if (rc == 0) rc = dyn_impl<R>(true, d->dynamics_kind, p->dyn, B, T, x, u, nullptr, Fw, fw, bs);
    Fs = T > 1 ? Fw : nullptr;
    fs = T > 1 ? fw : nullptr;
  }
  if (rc == 0)
    rc = step_impl<R>(&ds, p, C, c, Fs, fs, x_init, x, u, u_lower, u_upper, u_zero_I, new_x, new_u, costs,
                      (R*)(ws + l.fdn_step), (R*)(ws + l.alphas), du_first, (int32_t*)nullptr, (uint8_t*)nullptr,
                      status, l.gains ? (R*)(ws + l.Ks) : (R*)nullptr, l.gains ? (R*)(ws + l.ks) : (R*)nullptr, bs);
  if (rc == 0)
    rc = ilqr_launch_track<R>(B, T, N, M, o->m_ref, (R)o->best_cost_eps, new_x, new_u, costs, du_first, status,
                              best_costs, best_x, best_u, u, fdn, flags, st, bs);
  if (rc == 0) {
    g_launches.fetch_add(1);
    rc = ilqr_launch_stop<R>(B, o->lqr_iter, o->not_improved_lim, o->eps, costs, fdn, flags, best_costs, best_fdn, st,
                             info, handle, bs);
    if (rc == 0) g_launches.fetch_add(1);
  }
  cudaGraph_t body = nullptr;
  if (cudaStreamEndCapture(bs, &body) != cudaSuccess && rc == 0) rc = MPCB200_ERR_LAUNCH;
  return rc;
}

template <typename R>
static int ilqr_impl(const mpcb200_dims* d, const mpcb200_params* p, const mpcb200_ilqr_opts* o, const R* C,
                     const R* c, const R* F, const R* f, const R* x_init, const R* u_init, const R* u_lower,
                     const R* u_upper, const uint8_t* u_zero_I, R* best_x, R* best_u, R* best_costs, R* best_fdn,
                     int32_t* info, void* workspace, size_t workspace_bytes, void* stream) {
  int rc = ilqr_check<R>(d, p, o, C, c, F, f, x_init, u_lower, u_upper, u_zero_I, best_x, best_u, best_costs,
                         best_fdn, info, workspace, workspace_bytes);
  if (rc) return rc;
  if (max_smem_optin() <= 0) return MPCB200_ERR_NO_DEVICE;
  int driver = 0;
  if (cudaDriverGetVersion(&driver) != cudaSuccess || driver < 12030) return MPCB200_ERR_NO_GRAPH_COND;
  cudaStream_t st = (cudaStream_t)stream;
  cudaStreamCaptureStatus cap = cudaStreamCaptureStatusNone;
  if (cudaStreamIsCapturing(st, &cap) != cudaSuccess || cap == cudaStreamCaptureStatusInvalidated)
    return MPCB200_ERR_LAUNCH;
  const bool caller_captures = cap == cudaStreamCaptureStatusActive;
  // the library's own graph and stream calls must not invalidate a capture the caller runs in global mode
  cudaStreamCaptureMode mode = cudaStreamCaptureModeRelaxed;
  cudaThreadExchangeStreamCaptureMode(&mode);
  cudaStream_t os = caller_captures ? st : ilqr_stream(0);
  cudaStream_t bs = ilqr_stream(1);
  if (os == nullptr || bs == nullptr) {
    rc = MPCB200_ERR_LAUNCH;
  } else if (caller_captures) {
    rc = ilqr_record<R>(os, bs, d, p, o, C, c, F, f, x_init, u_init, u_lower, u_upper, u_zero_I, best_x, best_u,
                        best_costs, best_fdn, info, workspace);
  } else if (cudaStreamBeginCapture(os, cudaStreamCaptureModeRelaxed) != cudaSuccess) {
    rc = MPCB200_ERR_LAUNCH;
  } else {
    rc = ilqr_record<R>(os, bs, d, p, o, C, c, F, f, x_init, u_init, u_lower, u_upper, u_zero_I, best_x, best_u,
                        best_costs, best_fdn, info, workspace);
    cudaGraph_t g = nullptr;
    if (cudaStreamEndCapture(os, &g) != cudaSuccess && rc == 0) rc = MPCB200_ERR_LAUNCH;
    if (rc == 0) {
      cudaGraphExec_t exec = nullptr;
      if (cudaGraphInstantiate(&exec, g, 0) != cudaSuccess) {
        rc = MPCB200_ERR_LAUNCH;
      } else {
        if (cudaGraphLaunch(exec, st) != cudaSuccess) rc = MPCB200_ERR_LAUNCH;
        cudaGraphExecDestroy(exec);        // released once the launch completes
      }
    }
    if (g != nullptr) cudaGraphDestroy(g);
  }
  cudaThreadExchangeStreamCaptureMode(&mode);
  if (rc) cudaGetLastError();              // a failed build leaves no sticky launch error behind
  return rc;
}
}  // namespace mpcb200

using namespace mpcb200;

extern "C" {

int mpcb200_lqr_step_f32(const mpcb200_dims* dims, const mpcb200_params* params, const float* C,
                         const float* c, const float* F, const float* f, const float* x_init,
                         const float* cur_x, const float* cur_u, const float* u_lower,
                         const float* u_upper, const uint8_t* u_zero_I, float* new_x, float* new_u,
                         float* costs, float* full_du_norm, float* alphas, float* du_first, int32_t* qp_iters,
                         uint8_t* free_mask, int32_t* status, float* Ks, float* ks, void* stream) {
  return step_impl<float>(dims, params, C, c, F, f, x_init, cur_x, cur_u, u_lower, u_upper, u_zero_I,
                          new_x, new_u, costs, full_du_norm, alphas, du_first, qp_iters, free_mask, status, Ks, ks,
                          stream);
}
int mpcb200_lqr_step_f64(const mpcb200_dims* dims, const mpcb200_params* params, const double* C,
                         const double* c, const double* F, const double* f, const double* x_init,
                         const double* cur_x, const double* cur_u, const double* u_lower,
                         const double* u_upper, const uint8_t* u_zero_I, double* new_x, double* new_u,
                         double* costs, double* full_du_norm, double* alphas, double* du_first, int32_t* qp_iters,
                         uint8_t* free_mask, int32_t* status, double* Ks, double* ks, void* stream) {
  return step_impl<double>(dims, params, C, c, F, f, x_init, cur_x, cur_u, u_lower, u_upper, u_zero_I,
                           new_x, new_u, costs, full_du_norm, alphas, du_first, qp_iters, free_mask, status, Ks, ks,
                           stream);
}
int mpcb200_lqr_grad_f32(const mpcb200_dims* dims, const float* C, const float* c, const float* F,
                         const float* new_x, const float* new_u, const float* dx, const float* du,
                         const float* dl_dx, float* dx_init, float* dC, float* dc, float* dF, float* df,
                         void* workspace, void* stream) {
  return grad_impl<float>(dims, C, c, F, new_x, new_u, dx, du, dl_dx, dx_init, dC, dc, dF, df, workspace, stream);
}
int mpcb200_lqr_grad_f64(const mpcb200_dims* dims, const double* C, const double* c, const double* F,
                         const double* new_x, const double* new_u, const double* dx, const double* du,
                         const double* dl_dx, double* dx_init, double* dC, double* dc, double* dF,
                         double* df, void* workspace, void* stream) {
  return grad_impl<double>(dims, C, c, F, new_x, new_u, dx, du, dl_dx, dx_init, dC, dc, dF, df, workspace, stream);
}

size_t mpcb200_adjoint_workspace_bytes(const mpcb200_dims* dims, int32_t elem_size) {
  if (dims == nullptr || check_dims(dims) != 0 || (elem_size != 4 && elem_size != 8)) return 0;
  return adj_layout(dims->B, dims->T, dims->n, dims->m, (size_t)elem_size).total;
}
int mpcb200_lqr_adjoint_f32(const mpcb200_dims* dims, const mpcb200_params* params, const float* C, const float* c,
                            const float* F, const float* new_x, const float* new_u, const float* dl_dx,
                            const float* dl_du, const float* u_lower, const float* u_upper, float* dx_init,
                            float* dC, float* dc, float* dF, float* df, void* workspace, size_t workspace_bytes,
                            void* stream) {
  return adjoint_impl<float>(dims, params, C, c, F, new_x, new_u, dl_dx, dl_du, u_lower, u_upper, dx_init, dC, dc,
                             dF, df, workspace, workspace_bytes, stream);
}
int mpcb200_lqr_adjoint_f64(const mpcb200_dims* dims, const mpcb200_params* params, const double* C, const double* c,
                            const double* F, const double* new_x, const double* new_u, const double* dl_dx,
                            const double* dl_du, const double* u_lower, const double* u_upper, double* dx_init,
                            double* dC, double* dc, double* dF, double* df, void* workspace, size_t workspace_bytes,
                            void* stream) {
  return adjoint_impl<double>(dims, params, C, c, F, new_x, new_u, dl_dx, dl_du, u_lower, u_upper, dx_init, dC, dc,
                              dF, df, workspace, workspace_bytes, stream);
}

int mpcb200_rollout_f32(const mpcb200_dims* dims, const float* F, const float* f, const float* x_init,
                        const float* u, float* x, void* stream) {
  return rollout_impl<float>(dims, F, f, x_init, u, x, stream);
}
int mpcb200_rollout_f64(const mpcb200_dims* dims, const double* F, const double* f, const double* x_init,
                        const double* u, double* x, void* stream) {
  return rollout_impl<double>(dims, F, f, x_init, u, x, stream);
}

int mpcb200_dyn_rollout_f32(int32_t kind, const double* dyn, int32_t B, int32_t T, const float* x_init,
                            const float* u, float* x, void* stream) {
  return dyn_impl<float>(false, kind, dyn, B, T, x_init, u, x, nullptr, nullptr, stream);
}
int mpcb200_dyn_rollout_f64(int32_t kind, const double* dyn, int32_t B, int32_t T, const double* x_init,
                            const double* u, double* x, void* stream) {
  return dyn_impl<double>(false, kind, dyn, B, T, x_init, u, x, nullptr, nullptr, stream);
}
int mpcb200_dyn_linearize_f32(int32_t kind, const double* dyn, int32_t B, int32_t T, const float* x,
                              const float* u, float* F, float* f, void* stream) {
  return dyn_impl<float>(true, kind, dyn, B, T, x, u, nullptr, F, f, stream);
}
int mpcb200_dyn_linearize_f64(int32_t kind, const double* dyn, int32_t B, int32_t T, const double* x,
                              const double* u, double* F, double* f, void* stream) {
  return dyn_impl<double>(true, kind, dyn, B, T, x, u, nullptr, F, f, stream);
}

size_t mpcb200_ilqr_workspace_bytes(const mpcb200_dims* dims, const mpcb200_ilqr_opts* opts, int32_t elem_size) {
  if (dims == nullptr || opts == nullptr || check_dims(dims) != 0 || (elem_size != 4 && elem_size != 8)) return 0;
  if (dims->dynamics_kind != DYN_LINEAR && !known_shape_ok(dims)) return 0;
  return ilqr_layout(dims, (size_t)elem_size).total;
}
int mpcb200_ilqr_f32(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                     const float* C, const float* c, const float* F, const float* f, const float* x_init,
                     const float* u_init, const float* u_lower, const float* u_upper, const uint8_t* u_zero_I,
                     float* best_x, float* best_u, float* best_costs, float* best_full_du_norm, int32_t* info,
                     void* workspace, size_t workspace_bytes, void* stream) {
  return ilqr_impl<float>(dims, params, opts, C, c, F, f, x_init, u_init, u_lower, u_upper, u_zero_I, best_x, best_u,
                          best_costs, best_full_du_norm, info, workspace, workspace_bytes, stream);
}
int mpcb200_ilqr_f64(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                     const double* C, const double* c, const double* F, const double* f, const double* x_init,
                     const double* u_init, const double* u_lower, const double* u_upper, const uint8_t* u_zero_I,
                     double* best_x, double* best_u, double* best_costs, double* best_full_du_norm, int32_t* info,
                     void* workspace, size_t workspace_bytes, void* stream) {
  return ilqr_impl<double>(dims, params, opts, C, c, F, f, x_init, u_init, u_lower, u_upper, u_zero_I, best_x, best_u,
                           best_costs, best_full_du_norm, info, workspace, workspace_bytes, stream);
}

int mpcb200_supported(int32_t n_state, int32_t n_ctrl) { return find(n_state, n_ctrl) != nullptr; }

int mpcb200_supported_list(int32_t* out, int32_t cap) {
  for (int i = 0; i < kTableLen && i < cap; ++i) {
    out[2 * i] = kTable[i].n;
    out[2 * i + 1] = kTable[i].m;
  }
  return kTableLen;
}

uint64_t mpcb200_launch_count(void) { return g_launches.load(); }

size_t mpcb200_step_smem_bytes(const mpcb200_dims* dims, int32_t elem_size) {
  if (dims == nullptr) return 0;
  const Entry* e = find_step(dims);
  if (e == nullptr) return 0;
  return elem_size == 8 ? e->smem64(dims->T) : e->smem32(dims->T);
}

int mpcb200_step_prefers_workspace(const mpcb200_dims* dims, int32_t elem_size) {
  if (dims == nullptr) return 0;
  const bool passthrough = (dims->dynamics_kind & DYN_CTRL_PASSTHROUGH) != 0;
  if (!passthrough && runs_large(dims->n, dims->m)) return 1;   // the large-shape step keeps its gains in Ks/ks
  const Entry* e = find_step(dims);
  if (e == nullptr) return 1;                   // no instance: the step call itself reports it
  int ms = max_smem_optin();
  if (ms <= 0) ms = kOptinAssumed;    // no device visible (CPU-side query): assume H100's opt-in limit
  return elem_size == 8 ? e->pws64(dims->T, ms) : e->pws32(dims->T, ms);
}

int mpcb200_step_large_fits(const mpcb200_dims* dims, int32_t elem_size) {
  if (dims == nullptr || (elem_size != 4 && elem_size != 8)) return 0;
  return large_step_fits(dims->n, dims->m, elem_size, kOptinAssumed) ? 1 : 0;
}

int32_t mpcb200_last_step_plan(void) { return t_step_plan; }

int mpcb200_version(void) { return MPCB200_VERSION; }

const char* mpcb200_strerror(int code) {
  switch (code) {
    case MPCB200_OK: return "ok";
    case MPCB200_ERR_NULL_POINTER: return "a required pointer is NULL";
    case MPCB200_ERR_BAD_DIMS: return "bad dimensions or option combination";
    case MPCB200_ERR_UNSUPPORTED_DIMS: return "no kernel instance compiled for this (n_state, n_ctrl)";
    case MPCB200_ERR_SMEM: return "problem does not fit shared memory (pass Ks/ks buffers for long horizons)";
    case MPCB200_ERR_LAUNCH: return "CUDA launch failed";
    case MPCB200_ERR_NO_DEVICE: return "no usable sm_90 device";
    case MPCB200_ERR_NO_GRAPH_COND: return "conditional CUDA graph nodes are unavailable (driver older than 12.3)";
    default: return "unknown error";
  }
}
}  // extern "C"
