// api.cu - the C ABI declared in include/mpcb200.h: argument checks, the table of compiled instances, launch.
// Every entry point gathers its tensor pointers into one record (StepCall, IlqrCall), reads the developer knob once
// (kernel_knob) and checks its arguments in one fixed order, so a malformed call gets the same code from each.
#include <atomic>
#include <cstdlib>
#include <cstring>

#include "../../../include/mpcb200.h"
#include "episode_grad.cuh"
#include "ilqr.cuh"
#include "instance.cuh"
#include "lqr_large.cuh"
#include "mlp.cuh"
#include "pnqp.cuh"

namespace mpcb200 {
#define MPCB200_INST(n, m) extern const Instance inst__##n##_##m;
#define MPCB200_DYN_INST(kind, n, m) extern const Instance inst_dyn__##kind;
#include "instances.def"
#include "dyn_instances.def"
#undef MPCB200_INST
#undef MPCB200_DYN_INST
// every compiled instance: the (n, m) instances of instances.def in file order, then the dynamics-only step
// instances (no gradient or rollout kernels, and not listed by mpcb200_supported*)
static constexpr const Instance* kInstances[] = {
#define MPCB200_INST(n, m) &inst__##n##_##m,
#define MPCB200_DYN_INST(kind, n, m) &inst_dyn__##kind,
#include "instances.def"
#include "dyn_instances.def"
#undef MPCB200_INST
#undef MPCB200_DYN_INST
};

static const Instance* find(int n, int m, int kind = DYN_LINEAR) {
  for (const Instance* e : kInstances)
    if (e->kind == kind && e->n == n && e->m == m) return e;
  return nullptr;
}
// whether the step of `kind` runs on a dynamics-only instance (dyn_instances.def): every passthrough kind, and every
// kind with a record there
static bool own_instance(int kind) {
  if ((kind & DYN_CTRL_PASSTHROUGH) != 0) return true;
  for (const Instance* e : kInstances)
    if (kind != DYN_LINEAR && e->kind == kind) return true;
  return false;
}
// the step instance of a call: such a kind runs its dynamics-only instance, at exactly that kind's (n, m); every
// other call runs the (n, m) instance.  (An (n, m) instance's line search has no branch for a kind that has its own
// instance.)
static const Instance* find_step(const mpcb200_dims* d) {
  return find(d->n, d->m, own_instance(d->dynamics_kind) ? d->dynamics_kind : DYN_LINEAR);
}

// The developer A/B knob MPCB200_KERNEL, read once per entry-point call (the tests flip it inside one process):
// 0 or unset = the measured dispatch, 1 = the generic step kernel, 2 = the column-pair step kernel (StepArgs::impl),
// 3 = the large-shape kernels (lqr_large.cu) also for linear-dynamics shapes that have an instance.
static int kernel_knob() {
  const char* k = std::getenv("MPCB200_KERNEL");
  return k != nullptr ? std::atoi(k) : 0;
}
// the step, gradient and rollout of (n, m) run the large-shape kernels
static bool runs_large(int n, int m, int knob) { return find(n, m) == nullptr || knob == 3; }

static std::atomic<uint64_t> g_launches{0};
static thread_local int t_step_plan = 0;      // MPCB200_PLAN_* bits of this thread's last step launch

void record_step_plan(int plan) { t_step_plan = plan; }
// counts the kernels of a launcher that returned rc
static int counted(int rc, int kernels = 1) {
  if (rc == 0) g_launches.fetch_add(kernels);
  return rc;
}

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
int smem_optin_or_h100() {
  const int ms = max_smem_optin();
  return ms > 0 ? ms : kOptinAssumed;
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
template <typename R>
static bool span16(long long elems) { return (elems * (long long)sizeof(R)) % 16 == 0; }
// base (NULL counts as aligned) and time stride of one tensor of a step call are 16-byte aligned
template <typename R>
static bool tile_aligned(const R* base, long long tstride) { return aligned16(base) && span16<R>(tstride); }

static int check_dims(const mpcb200_dims* d) {
  if (d == nullptr) return MPCB200_ERR_NULL_POINTER;
  if (d->B <= 0 || d->T <= 0 || d->n <= 0 || d->m <= 0) return MPCB200_ERR_BAD_DIMS;
  if (d->F_T != d->T - 1 && d->F_T != d->T) return MPCB200_ERR_BAD_DIMS;
  return MPCB200_OK;
}
// a call whose network or window record is NULL: check_dims's error where there is one, as where the record is checked
static int null_record(const mpcb200_dims* d) {
  const int rc = check_dims(d);
  return rc ? rc : MPCB200_ERR_NULL_POINTER;
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

// the tensor arguments of mpcb200_lqr_step_*, in the header's order
template <typename R>
struct StepCall {
  const R *C, *c, *F, *f, *x_init, *cur_x, *cur_u, *u_lower, *u_upper;
  const uint8_t* u_zero_I;
  R *new_x, *new_u, *costs, *full_du_norm, *alphas, *du_first;
  int32_t* qp_iters;
  uint8_t* free_mask;
  int32_t* status;
  R *Ks, *ks;
};

template <typename R>
static int step_impl(const mpcb200_dims* d, const mpcb200_params* p, const StepCall<R>& s, int knob, void* stream,
                     const AdjExtra* adj = nullptr) {
  int rc = check_dims(d);
  if (rc) return rc;
  if (p == nullptr || s.C == nullptr || s.c == nullptr || s.cur_x == nullptr || s.cur_u == nullptr)
    return MPCB200_ERR_NULL_POINTER;
  if (d->T > 1 && s.F == nullptr) return MPCB200_ERR_NULL_POINTER;
  if (d->has_f && s.f == nullptr) return MPCB200_ERR_NULL_POINTER;
  rc = check_step_options(d, s.u_lower, s.u_upper, s.u_zero_I);
  if (rc) return rc;
  if (d->do_rollout) {
    if (s.x_init == nullptr || s.new_x == nullptr || s.new_u == nullptr || s.costs == nullptr ||
        s.full_du_norm == nullptr || s.alphas == nullptr)
      return MPCB200_ERR_NULL_POINTER;
  } else if (s.Ks == nullptr || s.ks == nullptr) {
    return MPCB200_ERR_NULL_POINTER;
  }
  if ((s.Ks == nullptr) != (s.ks == nullptr)) return MPCB200_ERR_NULL_POINTER;
  const Instance* e = find_step(d);
  const bool large = d->dynamics_kind == DYN_LINEAR && runs_large(d->n, d->m, knob);
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
  a.C = s.C; a.c = s.c; a.F = s.F; a.f = s.f; a.x_init = s.x_init; a.cur_x = s.cur_x; a.cur_u = s.cur_u;
  a.u_lower = s.u_lower; a.u_upper = s.u_upper; a.zero_mask = s.u_zero_I;
  a.new_x = s.new_x; a.new_u = s.new_u; a.costs = s.costs; a.full_du_norm = s.full_du_norm; a.alphas = s.alphas;
  a.du_first = s.du_first; a.qp_iters = s.qp_iters; a.free_mask = s.free_mask; a.status = s.status;
  a.Ks = s.Ks; a.ks = s.ks;
  const TimeStrides ts = time_strides(d);
  a.C_ts = ts.C; a.c_ts = ts.c; a.F_ts = ts.F; a.f_ts = ts.f;
  // Bulk-copy eligibility, per tensor: base and time stride 16-byte aligned (f, the tensor bounds: where the call
  // has them).  The time stride of the batch-dense cur_x, cur_u and bounds is B*n, B*m elements.
  const int n = d->n, m = d->m;
  const long long Bn = (long long)d->B * n, Bm = (long long)d->B * m;
  const bool al_C = tile_aligned(s.C, a.C_ts), al_c = tile_aligned(s.c, a.c_ts), al_F = tile_aligned(s.F, a.F_ts),
             al_f = tile_aligned(d->has_f ? s.f : nullptr, a.f_ts), al_x = tile_aligned(s.cur_x, Bn),
             al_u = tile_aligned(s.cur_u, Bm),
             al_box = d->bounds_kind != 2 || (tile_aligned(s.u_lower, Bm) && tile_aligned(s.u_upper, Bm));
  // the instance kernels copy batch-wide spans of every tensor, or none
  a.bulk_ok = al_C && al_c && al_F && al_f && al_x && al_u && al_box && aligned16(s.x_init);
  a.dyn_kind = d->dynamics_kind;
  if (a.dyn_kind != DYN_LINEAR) {
    if (!known_shape_ok(d)) return MPCB200_ERR_BAD_DIMS;
    for (int i = 0; i < 8; ++i) a.dp.p[i] = p->dyn[i];
  }
  if (large) {
    // the fused adjoint has no large-shape kernel: adjoint_impl then takes its three-launch route
    if (adj != nullptr) return MPCB200_ERR_UNSUPPORTED_DIMS;
    if (s.Ks == nullptr) return MPCB200_ERR_SMEM;      // the gains always go through the caller's Ks/ks
    // the large-shape kernel copies per-problem spans, tensor by tensor: their lengths must be 16-byte multiples too
    const long long pp = n + m;
    unsigned bulk = 0u;
    if (al_C && span16<R>(pp * pp)) bulk |= LB_C;
    if (s.F != nullptr && al_F && span16<R>(n * pp)) bulk |= LB_F;
    if (al_c && span16<R>(pp)) bulk |= LB_c;
    if (d->has_f && al_f && span16<R>(n)) bulk |= LB_f;
    if (al_x && span16<R>(n)) bulk |= LB_x;
    if (al_u && span16<R>(m)) bulk |= LB_u;
    if (d->bounds_kind == 2 && al_box && span16<R>(m)) bulk |= LB_BOX;
    t_step_plan = 0;
    return counted(large_step_launch<R>(a, n, m, bulk, smem, (cudaStream_t)stream));
  }
  a.impl = knob;
  if (adj != nullptr) {          // fused KKT adjoint: column-pair kernel only
    if (!adj->ok || !a.bulk_ok || a.impl == 1) return MPCB200_ERR_UNSUPPORTED_DIMS;
    a.impl = 2;
    a.adj = 1; a.adj_has_df = adj->has_df; a.adj_c = adj->c; a.adj_x = adj->x; a.adj_u = adj->u;
    a.adj_dC = adj->dC; a.adj_dc = adj->dc; a.adj_dF = adj->dF; a.adj_df = adj->df; a.adj_dx_init = adj->dx_init;
    a.adj_c_ts = adj->c_ts;
  }
  t_step_plan = 0;             // the launcher that launches records its plan
  return counted(e->ops[sizeof(R) == 8].step(a, smem, (cudaStream_t)stream));
}

// whether the step of `d` keeps its gains in the caller's Ks/ks (mpcb200_step_prefers_workspace)
static int gains_in_workspace(const mpcb200_dims* d, int elem_size, int knob) {
  // the large-shape step keeps its gains in Ks/ks
  if (!own_instance(d->dynamics_kind) && runs_large(d->n, d->m, knob)) return 1;
  const Instance* e = find_step(d);
  if (e == nullptr) return 1;                   // no instance: the step call itself reports it
  return e->ops[elem_size == 8].prefers_workspace(d->T, smem_optin_or_h100());
}

template <typename R>
static int grad_impl(const mpcb200_dims* d, const R* C, const R* c, const R* F, const R* new_x,
                     const R* new_u, const R* dx, const R* du, const R* dl_dx, R* dx_init, R* dC, R* dc,
                     R* dF, R* df, void* workspace, int knob, void* stream) {
  int rc = check_dims(d);
  if (rc) return rc;
  if (C == nullptr || c == nullptr || new_x == nullptr || new_u == nullptr || dx == nullptr ||
      du == nullptr || dl_dx == nullptr || dx_init == nullptr || dC == nullptr || dc == nullptr ||
      workspace == nullptr)
    return MPCB200_ERR_NULL_POINTER;
  if (d->F_T > 0 && (F == nullptr || dF == nullptr)) return MPCB200_ERR_NULL_POINTER;
  const Instance* e = find(d->n, d->m);
  const bool large = runs_large(d->n, d->m, knob);
  if (max_smem_optin() <= 0) return MPCB200_ERR_NO_DEVICE;
  GradArgs a;
  std::memset(&a, 0, sizeof(a));
  a.B = d->B; a.T = d->T; a.F_T = d->F_T; a.has_df = df != nullptr;
  a.C = C; a.c = c; a.F = F; a.new_x = new_x; a.new_u = new_u; a.dx = dx; a.du = du; a.dl_dx = dl_dx;
  a.dx_init = dx_init; a.dC = dC; a.dc = dc; a.dF = dF; a.df = df; a.workspace = workspace;
  const TimeStrides ts = time_strides(d);
  a.C_ts = ts.C; a.c_ts = ts.c; a.F_ts = ts.F;
  return counted(large ? large_grad_launch<R>(a, d->n, d->m, (cudaStream_t)stream)
                       : e->ops[sizeof(R) == 8].grad(a, (cudaStream_t)stream), 2);
}
// ---------------------------------------------------------------------------------------------
// KKT adjoint in one call (reference LQRStepFn.backward, mpc/lqr_step.py:312-407)
// ---------------------------------------------------------------------------------------------
// dims of the nested masked step (reference :328-340: MPC(lqr_iter=1, u_zero_I=I) with its defaults): the caller's,
// without f, bounds or delta_u; its c is the dense -r, C and F keep the caller's strides
static mpcb200_dims adjoint_step_dims(const mpcb200_dims* d) {
  mpcb200_dims ds = *d;
  ds.has_f = 0; ds.bounds_kind = 0; ds.has_zero_mask = 1; ds.has_delta_u = 0;
  ds.max_ls_iter = 10; ds.pnqp_max_iter = 20; ds.do_rollout = 1; ds.dynamics_kind = 0;
  ds.c_tstride = 0; ds.f_tstride = 0;
  return ds;
}

struct AdjLayout {                    // workspace carve-up (byte offsets, every piece 256-byte aligned)
  size_t negr, zeros, dx, du, costate, scal, mask, maskf, Ks, ks, total;
  bool gains;                         // Ks/ks of the nested step, where that step keeps its gains in a caller buffer
};
static size_t up256(size_t v) { return (v + 255) / 256 * 256; }
static AdjLayout adj_layout(const mpcb200_dims* d, size_t sz, int knob) {
  AdjLayout l;
  const int B = d->B, n = d->n, m = d->m;
  const size_t TB = (size_t)d->T * B;
  size_t o = 0;
  l.negr = o;    o += up256(TB * (n + m) * sz);
  l.zeros = o;   o += up256((TB * (n + m) + (size_t)B * n) * sz);     // cur_x, cur_u, x_init of the nested solve
  l.dx = o;      o += up256(TB * n * sz);
  l.du = o;      o += up256(TB * m * sz);
  l.costate = o; o += up256(2 * TB * n * sz);
  l.scal = o;    o += up256((size_t)3 * B * sz);
  l.mask = o;    o += up256(TB * m);
  l.maskf = o;   o += up256(TB * m * sz);                               // the same mask as element-typed 0/1 (rides on the TMA tile)
  const mpcb200_dims ds = adjoint_step_dims(d);
  l.gains = gains_in_workspace(&ds, (int)sz, knob) != 0;
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
                        size_t workspace_bytes, int knob, void* stream, bool zero_by_kernel = false) {
  int rc = check_dims(d);
  if (rc) return rc;
  if (p == nullptr || C == nullptr || c == nullptr || new_x == nullptr || new_u == nullptr || dl_dx == nullptr ||
      dl_du == nullptr || dx_init == nullptr || dC == nullptr || dc == nullptr || workspace == nullptr)
    return MPCB200_ERR_NULL_POINTER;
  if (d->T > 1 && (F == nullptr || dF == nullptr)) return MPCB200_ERR_NULL_POINTER;
  rc = check_bounds(d, u_lower, u_upper);
  if (rc) return rc;
  if (d->has_f && df == nullptr) return MPCB200_ERR_NULL_POINTER;
  const AdjLayout l = adj_layout(d, sizeof(R), knob);
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
  // nested masked LQR step from the zero trajectory
  const mpcb200_dims ds = adjoint_step_dims(d);
  mpcb200_params ps;
  std::memset(&ps, 0, sizeof(ps));
  ps.ls_decay = 0.2;
  StepCall<R> sc = {};
  sc.C = C; sc.c = negr; sc.F = F; sc.x_init = z0; sc.cur_x = zx; sc.cur_u = zu; sc.u_zero_I = mask;
  sc.new_x = dxs; sc.new_u = dus; sc.costs = scal; sc.full_du_norm = scal + d->B; sc.alphas = scal + 2 * d->B;
  // Preferred: ONE launch of the column-pair kernel doing solve + costates + outer products (C, F read from HBM
  // once, d tau kept in shared memory).  Shapes / alignments it does not take fall through to the 3-launch path, and
  // so do horizons where the nested step keeps its gains in Ks/ks: there the masked step + gradient kernels are the
  // faster ones.  Config 5 ((16,4) f32, B = 4096, T = 50, past the KREDUCE switch) through LQRStepFn.backward on an
  // H100 80GB HBM3 at 700 W: fused kernel 1.49 ms best / 1.96 ms median, masked step + gradient kernels 1.32 / 1.62 ms
  // (tools/exp_grad.py, DESIGN.md section 4).
  if (!l.gains) {
    AdjExtra ax;
    ax.c = c; ax.x = new_x; ax.u = new_u; ax.dC = dC; ax.dc = dc; ax.dF = dF; ax.df = d->has_f ? df : nullptr;
    ax.dx_init = dx_init; ax.has_df = d->has_f ? 1 : 0;
    ax.c_ts = time_strides(d).c;
    ax.ok = tile_aligned(c, ax.c_ts) && aligned16(new_x) && aligned16(new_u);
    sc.u_lower = sc.u_upper = (const R*)(ws + l.maskf);     // the mask rides in the bounds' tile slots
    rc = step_impl<R>(&ds, &ps, sc, knob, stream, &ax);
    if (rc == 0) return 0;
    if (rc != MPCB200_ERR_UNSUPPORTED_DIMS && rc != MPCB200_ERR_SMEM) return rc;
  }
  // 3-launch path: the nested solve really reads its (zero) nominal trajectory, and keeps its gains in the workspace
  // where a step call with Ks/ks would (gains_in_workspace).  `zero_by_kernel`: a kernel zeroes it, for a caller
  // that records the adjoint into a conditional body, which holds kernel nodes only (mpcb200_episode_backward_*).
  if (zero_by_kernel) {
    if (counted(launch_fill_zero<R>(TB * (d->n + d->m), zeros, st)) != 0) return MPCB200_ERR_LAUNCH;
  } else if (cudaMemsetAsync(zeros, 0, TB * (d->n + d->m) * sizeof(R), st) != cudaSuccess) {
    return MPCB200_ERR_LAUNCH;
  }
  sc.u_lower = sc.u_upper = nullptr;
  if (l.gains) {
    sc.Ks = (R*)(ws + l.Ks);
    sc.ks = (R*)(ws + l.ks);
  }
  rc = step_impl<R>(&ds, &ps, sc, knob, stream);
  if (rc) return rc;
  return grad_impl<R>(d, C, c, F, new_x, new_u, dxs, dus, dl_dx, dx_init, dC, dc, dF, d->has_f ? df : (R*)nullptr,
                      ws + l.costate, knob, stream);
}

template <typename R>
static int rollout_impl(const mpcb200_dims* d, const R* F, const R* f, const R* x_init, const R* u, R* x, int knob,
                        void* stream) {
  int rc = check_dims(d);
  if (rc) return rc;
  if (x_init == nullptr || u == nullptr || x == nullptr) return MPCB200_ERR_NULL_POINTER;
  if (d->T > 1 && F == nullptr) return MPCB200_ERR_NULL_POINTER;
  if (d->has_f && f == nullptr) return MPCB200_ERR_NULL_POINTER;
  const Instance* e = find(d->n, d->m);
  const bool large = runs_large(d->n, d->m, knob);
  if (max_smem_optin() <= 0) return MPCB200_ERR_NO_DEVICE;
  RolloutArgs a;
  std::memset(&a, 0, sizeof(a));
  a.B = d->B; a.T = d->T; a.has_f = d->has_f ? 1 : 0;
  a.F = F; a.f = f; a.x_init = x_init; a.u = u; a.x = x;
  const TimeStrides ts = time_strides(d);
  a.F_ts = ts.F; a.f_ts = ts.f;
  return counted(large ? large_rollout_launch<R>(a, d->n, d->m, (cudaStream_t)stream)
                       : e->ops[sizeof(R) == 8].rollout(a, (cudaStream_t)stream));
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
template <typename R>
static int dyn_vjp_impl(int kind, const double* dyn, int B, int T, const R* x, const R* u, const R* dF, const R* df,
                        R* first, R* second, void* stream) {
  if (dyn == nullptr || x == nullptr || u == nullptr) return MPCB200_ERR_NULL_POINTER;
  if (B <= 0 || T <= 0 || (kind != DYN_CARTPOLE && kind != DYN_PENDULUM && kind != DYN_PENDULUM_FULL))
    return MPCB200_ERR_BAD_DIMS;
  if (T > 1 && (dF == nullptr || df == nullptr)) return MPCB200_ERR_NULL_POINTER;
  if (max_smem_optin() <= 0) return MPCB200_ERR_NO_DEVICE;
  if (T == 1 || (first == nullptr && second == nullptr)) return 0;
  DynVjpArgs a;
  std::memset(&a, 0, sizeof(a));
  a.B = B; a.T = T; a.kind = kind;
  for (int i = 0; i < 8; ++i) a.dp.p[i] = dyn[i];
  a.x = x; a.u = u; a.dF = dF; a.df = df; a.first = first; a.second = second;
  return counted(launch_dyn_linearize_vjp<R>(a, (cudaStream_t)stream));
}

// ---------------------------------------------------------------------------------------------
// a learned model's network (mlp.cu): its rollout and linearisation, and the split-mode step (the step kernels with
// do_rollout = 0, then the network's line search)
// ---------------------------------------------------------------------------------------------
static int mlp_check(const mpcb200_mlp* mlp, int B, int T, int N, int M, MlpShape& s) {
  if (mlp == nullptr) return MPCB200_ERR_NULL_POINTER;
  if (!mlp_shape(mlp, s)) return MPCB200_ERR_BAD_DIMS;
  if (B <= 0 || T <= 0 || N < s.n_prev + s.ns || M < s.ms || N + M > s.p_max) return MPCB200_ERR_BAD_DIMS;
  return MPCB200_OK;
}

// A network an episode takes: mlp_check's, without the slew-rate state, with kernels that fit `smem` bytes of shared
// memory (an entry's device, or kOptinAssumed for a workspace size).
static int episode_net_check(const mpcb200_dims* d, const mpcb200_mlp* mlp, int elem_size, int smem, MlpShape& s) {
  if (const int rc = mlp_check(mlp, d->B, d->T, d->n, d->m, s)) return rc;
  if (s.n_prev != 0) return MPCB200_ERR_BAD_DIMS;
  return mlp_smem_bytes(s, elem_size, 1) > (size_t)smem ? MPCB200_ERR_SMEM : MPCB200_OK;
}

template <typename R>
static int mlp_rollout_impl(const mpcb200_mlp* mlp, int B, int T, int N, int M, const R* x_init, const R* u, R* x,
                            void* stream) {
  MlpShape s;
  if (const int rc = mlp_check(mlp, B, T, N, M, s)) return rc;
  if (x_init == nullptr || u == nullptr || x == nullptr) return MPCB200_ERR_NULL_POINTER;
  return counted(mlp_launch_rollout<R>(mlp, B, T, N, M, x_init, u, x, (cudaStream_t)stream));
}

template <typename R>
static int mlp_linearize_impl(const mpcb200_mlp* mlp, int B, int T, int N, int M, const R* x, const R* u, R* F, R* f,
                              void* stream) {
  MlpShape s;
  if (const int rc = mlp_check(mlp, B, T, N, M, s)) return rc;
  if (x == nullptr || u == nullptr) return MPCB200_ERR_NULL_POINTER;
  if (T == 1) return MPCB200_OK;
  if (F == nullptr || f == nullptr) return MPCB200_ERR_NULL_POINTER;
  return counted(mlp_launch_linearize<R>(mlp, B, T, N, M, x, u, F, f, (cudaStream_t)stream));
}

// the linearisation VJP's workspace ([G, n_params] slot rows), 0 where its per-warp slice does not fit
static size_t mlp_vjp_ws(const MlpShape& s, int B, int T, size_t sz) {
  if (mlp_smem_bytes(mlp_vjp_shape(s), (int)sz, 1) > (size_t)kOptinAssumed) return 0;
  return up256((size_t)mlp_vjp_slots((long long)(T - 1) * B, s.n_params) * (size_t)s.n_params * sz);
}

template <typename R>
static int mlp_linearize_vjp_impl(const mpcb200_mlp* mlp, int B, int T, int N, int M, const R* x, const R* u,
                                  const R* dF, const R* df, R* dtheta, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  MlpShape s;
  if (const int rc = mlp_check(mlp, B, T, N, M, s)) return rc;
  if (x == nullptr || u == nullptr || dF == nullptr || df == nullptr || dtheta == nullptr || workspace == nullptr)
    return MPCB200_ERR_NULL_POINTER;
  const size_t need = mlp_vjp_ws(s, B, T, sizeof(R));
  if (need == 0) return MPCB200_ERR_SMEM;
  if (workspace_bytes < need || (reinterpret_cast<uintptr_t>(workspace) & 255u) != 0) return MPCB200_ERR_BAD_DIMS;
  return counted(mlp_launch_linearize_vjp<R>(mlp, B, T, N, M, x, u, dF, df, dtheta, (R*)workspace,
                                             (cudaStream_t)stream), 2);
}

static size_t mlp_step_ws(const mpcb200_dims* d, size_t sz) {
  const size_t TBM = (size_t)d->T * d->B * d->m;
  return up256(TBM * d->n * sz) + up256(TBM * sz);
}

// The line search's arguments: the gains the step wrote into q.Ks, q.ks, the iterate it writes into q's new_x, new_u,
// costs, alphas and du_first.
template <typename R>
static MlpLsArgs<R> mlp_ls_args(const mpcb200_dims* d, const mpcb200_params* p, const StepCall<R>& q) {
  MlpLsArgs<R> a;
  std::memset(&a, 0, sizeof(a));
  a.B = d->B; a.T = d->T; a.N = d->n; a.M = d->m;
  a.bounds_kind = d->bounds_kind; a.has_mask = d->has_zero_mask ? 1 : 0; a.has_delta = d->has_delta_u ? 1 : 0;
  a.max_ls = d->max_ls_iter;
  const TimeStrides ts = time_strides(d);
  a.C_ts = ts.C; a.c_ts = ts.c;
  a.u_lo = (R)p->u_lo; a.u_hi = (R)p->u_hi; a.delta_u = (R)p->delta_u; a.decay = (R)p->ls_decay;
  a.C = q.C; a.c = q.c; a.x_init = q.x_init; a.cur_x = q.cur_x; a.cur_u = q.cur_u; a.Ks = q.Ks; a.ks = q.ks;
  a.u_lower = q.u_lower; a.u_upper = q.u_upper; a.zero_mask = q.u_zero_I;
  a.new_x = q.new_x; a.new_u = q.new_u; a.costs = q.costs; a.alphas = q.alphas; a.du_first = q.du_first;
  return a;
}

// the checks of a split-mode step that need no device, before anything is launched
template <typename R>
static int mlp_step_check(const mpcb200_dims* d, const mpcb200_params* p, const mpcb200_mlp* mlp,
                          const StepCall<R>& q) {
  int rc = check_dims(d);
  if (rc) return rc;
  MlpShape s;
  if ((rc = mlp_check(mlp, d->B, d->T, d->n, d->m, s))) return rc;
  if (p == nullptr || q.C == nullptr || q.c == nullptr || q.x_init == nullptr || q.cur_x == nullptr ||
      q.cur_u == nullptr || q.new_x == nullptr || q.new_u == nullptr || q.costs == nullptr || q.alphas == nullptr)
    return MPCB200_ERR_NULL_POINTER;
  if (d->T > 1 && q.F == nullptr) return MPCB200_ERR_NULL_POINTER;
  if (d->has_f && q.f == nullptr) return MPCB200_ERR_NULL_POINTER;
  if ((rc = check_step_options(d, q.u_lower, q.u_upper, q.u_zero_I))) return rc;
  if (d->dynamics_kind != DYN_LINEAR) return MPCB200_ERR_BAD_DIMS;
  if (mlp_smem_bytes(s, sizeof(R), 1) > (size_t)smem_optin_or_h100()) return MPCB200_ERR_SMEM;
  return MPCB200_OK;
}

// The split-mode step of q: the step kernels with do_rollout = 0 write the gains into q.Ks, q.ks (and qp_iters,
// free_mask, status), then the network's line search writes the iterate.
template <typename R>
static int mlp_split_step(const mpcb200_dims* d, const mpcb200_params* p, const mpcb200_mlp* mlp, const StepCall<R>& q,
                          int knob, void* stream) {
  mpcb200_dims ds = *d;
  ds.do_rollout = 0;
  StepCall<R> sc = q;
  sc.new_x = sc.new_u = sc.costs = sc.full_du_norm = sc.alphas = sc.du_first = nullptr;
  if (const int rc = step_impl<R>(&ds, p, sc, knob, stream)) return rc;
  return counted(mlp_launch_linesearch<R>(mlp, mlp_ls_args<R>(d, p, q), (cudaStream_t)stream));
}

// q: the arguments of mpcb200_mlp_step_* after dims, params and the record (no full_du_norm, Ks or ks)
template <typename R>
static int mlp_step_impl(const mpcb200_dims* d, const mpcb200_params* p, const mpcb200_mlp* mlp, StepCall<R> q,
                         void* workspace, size_t workspace_bytes, void* stream) {
  const int knob = kernel_knob();
  int rc = mlp_step_check<R>(d, p, mlp, q);
  if (rc) return rc;
  if (workspace == nullptr) return MPCB200_ERR_NULL_POINTER;
  if (workspace_bytes < mlp_step_ws(d, sizeof(R)) || (reinterpret_cast<uintptr_t>(workspace) & 255u) != 0)
    return MPCB200_ERR_BAD_DIMS;
  q.Ks = (R*)workspace;
  q.ks = (R*)((char*)workspace + up256((size_t)d->T * d->B * d->m * d->n * sizeof(R)));
  return mlp_split_step<R>(d, p, mlp, q, knob, stream);
}

// ---------------------------------------------------------------------------------------------
// the iLQR loop of MPC.forward as one CUDA graph (reference mpc/mpc.py:244-301), on LinDx, a known system or a
// learned model's network (mpcb200_ilqr_mlp_*)
// ---------------------------------------------------------------------------------------------
// dims of the step inside the loop: the caller's, with the rollout on and, for a known system or a network (net), the
// workspace F, f
static mpcb200_dims ilqr_step_dims(const mpcb200_dims* d, bool net) {
  mpcb200_dims ds = *d;
  ds.do_rollout = 1;
  if (net || d->dynamics_kind != DYN_LINEAR) {
    ds.F_T = d->T - 1; ds.has_f = d->T > 1 ? 1 : 0; ds.F_tstride = 0; ds.f_tstride = 0;
  }
  return ds;
}

struct IlqrLayout {                   // workspace carve-up (byte offsets, every piece 256-byte aligned)
  size_t u, x, new_x, new_u, costs, fdn_step, alphas, du_first, status, fdn, flags, state, F, f, Ks, ks, total;
  bool gains;
};
// net: the loop of mpcb200_ilqr_mlp_*, whose split-mode step always writes the gains
static IlqrLayout ilqr_layout(const mpcb200_dims* d, size_t sz, int knob, bool net) {
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
  // the linearisation of a known system or the network, rewritten every iteration.  The network's entries refuse a
  // known kind; their workspace sizes for one count both linearisations.
  const size_t TB1 = (size_t)(d->T > 1 ? d->T - 1 : 0) * B;
  l.F = l.f = 0;
  for (int k = (d->dynamics_kind != DYN_LINEAR) + (net ? 1 : 0); k > 0; --k) {
    l.F = o;      o += up256(TB1 * n * (n + m) * sz);
    l.f = o;      o += up256(TB1 * n * sz);
  }
  const mpcb200_dims ds = ilqr_step_dims(d, net);
  l.gains = net || gains_in_workspace(&ds, (int)sz, knob) != 0;
  l.Ks = l.ks = 0;
  if (l.gains) {
    l.Ks = o;     o += up256(TB * m * n * sz);
    l.ks = o;     o += up256(TB * m * sz);
  }
  l.total = o;
  return l;
}

// the arguments of mpcb200_ilqr_*, in the header's order
template <typename R>
struct IlqrCall {
  const mpcb200_dims* d;
  const mpcb200_params* p;
  const mpcb200_ilqr_opts* o;
  const R *C, *c, *F, *f, *x_init, *u_init, *u_lower, *u_upper;
  const uint8_t* u_zero_I;
  R *best_x, *best_u, *best_costs, *best_fdn;
  int32_t* info;
  void* workspace;
  size_t workspace_bytes;
};

// argument checks that need no device: every error is reported before anything is captured or launched.  mlp: the
// network the loop plans with (non-NULL from mpcb200_ilqr_mlp_*), or NULL.
template <typename R>
static int ilqr_check(const IlqrCall<R>& q, const mpcb200_mlp* mlp, int knob) {
  const mpcb200_dims* d = q.d;
  int rc = check_dims(d);
  if (rc) return rc;
  MlpShape s;
  if (mlp != nullptr && (rc = mlp_check(mlp, d->B, d->T, d->n, d->m, s))) return rc;
  if (q.p == nullptr || q.o == nullptr || q.C == nullptr || q.c == nullptr || q.x_init == nullptr ||
      q.best_x == nullptr || q.best_u == nullptr || q.best_costs == nullptr || q.best_fdn == nullptr ||
      q.info == nullptr || q.workspace == nullptr)
    return MPCB200_ERR_NULL_POINTER;
  if (q.o->lqr_iter < 1 || q.o->m_ref < 1 || q.o->m_ref > d->m) return MPCB200_ERR_BAD_DIMS;
  if (mlp != nullptr) {
    if (d->T < 2 || d->dynamics_kind != DYN_LINEAR) return MPCB200_ERR_BAD_DIMS;
  } else if (d->dynamics_kind != DYN_LINEAR) {
    if (!known_shape_ok(d)) return MPCB200_ERR_BAD_DIMS;
  } else {
    if (d->T > 1 && q.F == nullptr) return MPCB200_ERR_NULL_POINTER;
    if (d->has_f && q.f == nullptr) return MPCB200_ERR_NULL_POINTER;
  }
  rc = check_step_options(d, q.u_lower, q.u_upper, q.u_zero_I);
  if (rc) return rc;
  if (mlp != nullptr) {
    if (mlp_smem_bytes(s, sizeof(R), 1) > (size_t)smem_optin_or_h100()) return MPCB200_ERR_SMEM;
  } else if (d->dynamics_kind != DYN_LINEAR && find_step(d) == nullptr) {
    return MPCB200_ERR_UNSUPPORTED_DIMS;
  }
  const IlqrLayout l = ilqr_layout(d, sizeof(R), knob, mlp != nullptr);
  if (q.workspace_bytes < l.total || (reinterpret_cast<uintptr_t>(q.workspace) & 255u) != 0)
    return MPCB200_ERR_BAD_DIMS;
  return MPCB200_OK;
}

// Library-owned streams of this thread on the current device: [0] records a graph the caller does not capture,
// [1] records the iLQR loop body, [2] the body of an episode's loop over control steps.  Capture only records work
// on them; nothing ever executes on them.
static cudaStream_t ilqr_stream(int which) {
  static thread_local cudaStream_t streams[64][3] = {};
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return nullptr;
  cudaStream_t& s = streams[dev][which];
  if (s == nullptr && cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) s = nullptr;
  return s;
}

// A conditional handle in the graph `os` is capturing: the graph of a top-level capture, or the body of an enclosing
// loop.  MPCB200_ERR_NO_GRAPH_COND when the driver refuses it.
static int while_handle(cudaStream_t os, cudaGraphConditionalHandle* handle) {
  cudaStreamCaptureStatus cst = cudaStreamCaptureStatusNone;
  cudaGraph_t g = nullptr;
  if (cudaStreamGetCaptureInfo(os, &cst, nullptr, &g, nullptr, nullptr) != cudaSuccess ||
      cst != cudaStreamCaptureStatusActive)
    return MPCB200_ERR_LAUNCH;
  if (cudaGraphConditionalHandleCreate(handle, g, 1, cudaGraphCondAssignDefault) != cudaSuccess) {
    cudaGetLastError();
    return MPCB200_ERR_NO_GRAPH_COND;
  }
  return MPCB200_OK;
}

// Adds a `while` node on `handle` after the work captured on `os` so far and starts recording its body on `bs`
// (which the caller ends with cudaStreamEndCapture).  MPCB200_ERR_NO_GRAPH_COND when the driver refuses the node,
// e.g. a conditional node inside a conditional body.
static int open_while(cudaStream_t os, cudaStream_t bs, cudaGraphConditionalHandle handle) {
  cudaStreamCaptureStatus cst = cudaStreamCaptureStatusNone;
  cudaGraph_t g = nullptr;
  const cudaGraphNode_t* deps = nullptr;
  size_t ndeps = 0;
  if (cudaStreamGetCaptureInfo(os, &cst, nullptr, &g, &deps, &ndeps) != cudaSuccess ||
      cst != cudaStreamCaptureStatusActive)
    return MPCB200_ERR_LAUNCH;
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
  if (cudaStreamBeginCaptureToGraph(bs, np.conditional.phGraph_out[0], nullptr, nullptr, 0,
                                    cudaStreamCaptureModeRelaxed) != cudaSuccess)
    return MPCB200_ERR_LAUNCH;
  return MPCB200_OK;
}

// Adds the init kernel and the `while` node (body recorded on `bs`) to the graph `os` is capturing.  Body: the model
// part, then track -> stop.  The model part: LinDx: rollout -> step; a known system: rollout -> linearisation -> step;
// mlp (non-NULL): the network's rollout -> linearisation -> split-mode step (mlp_split_step: step, line search).
template <typename R>
static int ilqr_record(cudaStream_t os, cudaStream_t bs, const IlqrCall<R>& q, int knob, const mpcb200_mlp* mlp) {
  const mpcb200_dims* d = q.d;
  const mpcb200_ilqr_opts* o = q.o;
  const IlqrLayout l = ilqr_layout(d, sizeof(R), knob, mlp != nullptr);
  char* ws = (char*)q.workspace;
  R* u = (R*)(ws + l.u);
  R* x = (R*)(ws + l.x);
  R* fdn = (R*)(ws + l.fdn);
  uint8_t* flags = (uint8_t*)(ws + l.flags);
  IlqrState* st = (IlqrState*)(ws + l.state);
  const int B = d->B, T = d->T, N = d->n, M = d->m;
  const size_t TB = (size_t)T * B;
  cudaGraphConditionalHandle handle;
  int rc = while_handle(os, &handle);
  if (rc) return rc;
  if (counted(ilqr_launch_init<R>(TB * M, q.u_init, u, st, q.info, handle, os)) != 0) return MPCB200_ERR_LAUNCH;
  // the body: the library's own launchers, recorded on bs (same plan selection as a direct call)
  rc = open_while(os, bs, handle);
  if (rc) return rc;
  const mpcb200_dims ds = ilqr_step_dims(d, mlp != nullptr);
  StepCall<R> sc = {};
  sc.C = q.C; sc.c = q.c; sc.F = q.F; sc.f = q.f; sc.x_init = q.x_init; sc.cur_x = x; sc.cur_u = u;
  sc.u_lower = q.u_lower; sc.u_upper = q.u_upper; sc.u_zero_I = q.u_zero_I;
  sc.new_x = (R*)(ws + l.new_x); sc.new_u = (R*)(ws + l.new_u); sc.costs = (R*)(ws + l.costs);
  sc.full_du_norm = (R*)(ws + l.fdn_step); sc.alphas = (R*)(ws + l.alphas); sc.du_first = (R*)(ws + l.du_first);
  sc.status = (int32_t*)(ws + l.status);
  if (l.gains) {
    sc.Ks = (R*)(ws + l.Ks);
    sc.ks = (R*)(ws + l.ks);
  }
  R* F = (R*)(ws + l.F);              // a known system's or the network's linearisation: the step reads it
  R* f = (R*)(ws + l.f);
  if (mlp != nullptr || d->dynamics_kind != DYN_LINEAR) {
    sc.F = T > 1 ? F : nullptr;
    sc.f = T > 1 ? f : nullptr;
  }
  if (mlp != nullptr) {
    rc = mlp_rollout_impl<R>(mlp, B, T, N, M, q.x_init, u, x, bs);
    if (rc == 0) rc = mlp_linearize_impl<R>(mlp, B, T, N, M, x, u, F, f, bs);
    if (rc == 0) rc = mlp_split_step<R>(&ds, q.p, mlp, sc, knob, bs);
  } else {
    if (d->dynamics_kind == DYN_LINEAR) {
      rc = rollout_impl<R>(d, q.F, q.f, q.x_init, u, x, knob, bs);
    } else {
      rc = dyn_impl<R>(false, d->dynamics_kind, q.p->dyn, B, T, q.x_init, u, x, nullptr, nullptr, bs);
      if (rc == 0) rc = dyn_impl<R>(true, d->dynamics_kind, q.p->dyn, B, T, x, u, nullptr, F, f, bs);
    }
    if (rc == 0) rc = step_impl<R>(&ds, q.p, sc, knob, bs);
  }
  if (rc == 0)
    rc = counted(ilqr_launch_track<R>(B, T, N, M, o->m_ref, (R)o->best_cost_eps, sc.new_x, sc.new_u, sc.costs,
                                      sc.du_first, sc.status, q.best_costs, q.best_x, q.best_u, u, fdn, flags, st, bs));
  if (rc == 0)
    rc = counted(ilqr_launch_stop<R>(B, o->lqr_iter, o->not_improved_lim, o->eps, sc.costs, fdn, flags, q.best_costs,
                                     q.best_fdn, st, q.info, handle, bs));
  cudaGraph_t body = nullptr;
  if (cudaStreamEndCapture(bs, &body) != cudaSuccess && rc == 0) rc = MPCB200_ERR_LAUNCH;
  return rc;
}

// Runs `record(os)`, which adds a solve's nodes to the graph `os` is capturing, with the capture contract of
// mpcb200_ilqr_*: on a capturing `stream` the nodes join the caller's graph and nothing is launched; otherwise the
// graph is captured on a library stream, instantiated, launched on `stream` and destroyed.
template <typename Record>
static int run_graph(void* stream, Record&& record) {
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
  // a caller that is not capturing gets a graph of the library's own: captured, instantiated and launched here
  cudaStream_t os = caller_captures ? st : ilqr_stream(0);
  int rc;
  if (os == nullptr ||
      (!caller_captures && cudaStreamBeginCapture(os, cudaStreamCaptureModeRelaxed) != cudaSuccess)) {
    rc = MPCB200_ERR_LAUNCH;
  } else {
    rc = record(os);
    if (!caller_captures) {
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
  }
  cudaThreadExchangeStreamCaptureMode(&mode);
  if (rc) cudaGetLastError();              // a failed build leaves no sticky launch error behind
  return rc;
}

template <typename R>
static int ilqr_impl(const IlqrCall<R>& q, const mpcb200_mlp* mlp, void* stream) {
  const int knob = kernel_knob();
  int rc = ilqr_check<R>(q, mlp, knob);
  if (rc) return rc;
  if (max_smem_optin() <= 0) return MPCB200_ERR_NO_DEVICE;
  return run_graph(stream, [&](cudaStream_t os) {
    cudaStream_t bs = ilqr_stream(1);
    return bs == nullptr ? MPCB200_ERR_LAUNCH : ilqr_record<R>(os, bs, q, knob, mlp);
  });
}

// ---------------------------------------------------------------------------------------------
// time-varying episodes (mpcb200_episode_window_*, mpcb200_episode_backward_window_*): each control step's window of
// the full-length inputs is staged into fixed workspace buffers, which the episode's (or sweep's) nodes read
// ---------------------------------------------------------------------------------------------
struct WindowLayout {                 // byte offsets of the window buffers, after the episode's (sweep's) workspace
  size_t at[WINDOW_INPUTS], total;
};
// d: the solve's dims.  f's buffer holds T slices (the kernels read T-1); a plant's, one
static WindowLayout window_layout(const mpcb200_dims* d, const mpcb200_window* w, size_t base, size_t sz) {
  WindowLayout l;
  const size_t B = d->B, T = d->T, n = d->n, m = d->m, p = n + m;
  const size_t len[WINDOW_INPUTS] = {T * B * p * p, T * B * p, (size_t)d->F_T * B * n * p, T * B * n,
                                     T * B * m, T * B * m, B * n * p, B * n};
  const int bit[WINDOW_INPUTS] = {MPCB200_WIN_COST, MPCB200_WIN_COST, MPCB200_WIN_DYN, MPCB200_WIN_DYN,
                                  MPCB200_WIN_BOUNDS, MPCB200_WIN_BOUNDS, MPCB200_WIN_PLANT, MPCB200_WIN_PLANT};
  size_t o = base;
  for (int a = 0; a < WINDOW_INPUTS; ++a) {
    l.at[a] = 0;
    if (w->on & bit[a]) {
      l.at[a] = o;
      o += up256(len[a] * sz);
    }
  }
  l.total = o;
  return l;
}

// the window record against the caller's dims: MPCB200_WIN_COST set, each other bit only where its input can be
// windowed, an axis that covers n_steps + T - 1 slices, and time strides of the dims convention
static int window_check(const mpcb200_dims* d, const mpcb200_window* w, int n_steps, const mpcb200_plant* plant) {
  if (w == nullptr) return MPCB200_ERR_NULL_POINTER;
  const int all = MPCB200_WIN_COST | MPCB200_WIN_DYN | MPCB200_WIN_BOUNDS | MPCB200_WIN_PLANT;
  if (!(w->on & MPCB200_WIN_COST) || (w->on & ~all) != 0) return MPCB200_ERR_BAD_DIMS;
  if ((w->on & MPCB200_WIN_DYN) && d->dynamics_kind != DYN_LINEAR) return MPCB200_ERR_BAD_DIMS;
  if ((w->on & MPCB200_WIN_BOUNDS) && d->bounds_kind != 2) return MPCB200_ERR_BAD_DIMS;
  if ((w->on & MPCB200_WIN_PLANT) && (plant == nullptr || plant->kind != DYN_LINEAR)) return MPCB200_ERR_BAD_DIMS;
  if (n_steps < 1 || (long long)w->L < (long long)n_steps + d->T - 1) return MPCB200_ERR_BAD_DIMS;
  const int64_t ts[WINDOW_INPUTS] = {w->C_tstride, w->c_tstride, w->F_tstride, w->f_tstride,
                                     w->lo_tstride, w->hi_tstride, w->Fp_tstride, w->fp_tstride};
  for (int64_t t : ts)
    if (t < MPCB200_TIME_INVARIANT) return MPCB200_ERR_BAD_DIMS;
  return MPCB200_OK;
}

// the solve's dims: the caller's, with the windowed inputs read from dense buffers
static mpcb200_dims window_solve_dims(const mpcb200_dims* d, const mpcb200_window* w) {
  mpcb200_dims ds = *d;
  if (w->on & MPCB200_WIN_COST) ds.C_tstride = ds.c_tstride = 0;
  if (w->on & MPCB200_WIN_DYN) ds.F_tstride = ds.f_tstride = 0;
  return ds;
}

// The copy of each windowed input into its staging buffer, k read from `step`.  in[a]: the call's field of input a
// (NULL, or a NULL field: not windowed or not given), which is pointed at the buffer.  Slices: T of C, c and the
// bounds, F_T of F, T-1 of f, 1 of the plant's F, f.
template <typename R>
static WindowCopy<R> window_copy(const mpcb200_dims* d, const mpcb200_window* w, const WindowLayout& l, char* ws,
                                 const R** const in[WINDOW_INPUTS], const int32_t* step) {
  WindowCopy<R> c;
  std::memset(&c, 0, sizeof(c));
  const long long B = d->B, T = d->T, n = d->n, m = d->m, p = n + m;
  const long long slice[WINDOW_INPUTS] = {B * p * p, B * p, B * n * p, B * n, B * m, B * m, B * n * p, B * n};
  const int cnt[WINDOW_INPUTS] = {(int)T, (int)T, d->F_T, (int)T - 1, (int)T, (int)T, 1, 1};
  const int64_t ts[WINDOW_INPUTS] = {w->C_tstride, w->c_tstride, w->F_tstride, w->f_tstride,
                                     w->lo_tstride, w->hi_tstride, w->Fp_tstride, w->fp_tstride};
  for (int a = 0; a < WINDOW_INPUTS; ++a) {
    if (l.at[a] == 0 || in[a] == nullptr || *in[a] == nullptr) continue;
    c.src[a] = *in[a];
    c.dst[a] = (R*)(ws + l.at[a]);
    c.tstride[a] = ts[a] == 0 ? slice[a] : ts[a];
    c.slice[a] = slice[a];
    c.n[a] = cnt[a];
    *in[a] = c.dst[a];
  }
  c.k = step;
  return c;
}

// ---------------------------------------------------------------------------------------------
// a receding-horizon episode as one CUDA graph: solve, apply, shift and re-solve, n_steps times
// ---------------------------------------------------------------------------------------------
struct EpisodeLayout {                // workspace carve-up: the iLQR loop's workspace, then the episode's buffers
  IlqrLayout ilqr;
  size_t best_x, best_u, best_costs, best_fdn, info, state, warm, traj, ep, total;
};
// net: the solve is a learned model's
static EpisodeLayout episode_layout(const mpcb200_dims* d, size_t sz, int knob, bool net = false) {
  EpisodeLayout l;
  l.ilqr = ilqr_layout(d, sz, knob, net);
  const size_t TB = (size_t)d->T * d->B, B = d->B;
  const size_t n = d->n, m = d->m;
  size_t o = l.ilqr.total;
  l.best_x = o;     o += up256(TB * n * sz);
  l.best_u = o;     o += up256(TB * m * sz);
  l.best_costs = o; o += up256(B * sz);
  l.best_fdn = o;   o += up256(B * sz);
  l.info = o;       o += up256(2 * sizeof(int32_t));
  l.state = o;      o += up256(B * n * sz);             // x_k: the x_init of the solve of control step k
  l.warm = o;       o += up256(TB * m * sz);            // w_k: its u_init
  l.traj = o;       o += up256(2 * B * n * sz);         // the model step [x_k, x_{k+1}]
  l.ep = o;         o += up256(sizeof(EpisodeState));
  l.total = o;
  return l;
}

// the arguments of mpcb200_episode_*, in the header's order
template <typename R>
struct EpisodeCall {
  const mpcb200_dims* d;
  const mpcb200_params* p;
  const mpcb200_ilqr_opts* o;
  int n_steps;
  const R *C, *c, *F, *f, *x_init, *u_init, *u_lower, *u_upper;
  const uint8_t* u_zero_I;
  R *xs, *us, *costs;
  int32_t* info;
  R* u_next;
  void* workspace;
  size_t workspace_bytes;
  R *plan_x, *plan_u;          // mpcb200_episode_plans_*: each solve's best iterate; NULL for mpcb200_episode_*
  // mpcb200_episode_plant_*: the plant that steps the loop and the disturbances; otherwise the model steps it
  const mpcb200_plant* plant;
  const R *F_plant, *f_plant, *w;
  // mpcb200_episode_mlp_*: the learned model every solve plans with and, without a plant, that steps the loop
  const mpcb200_mlp* mlp = nullptr;
};

// the model step's kind, parameters, F, f and has_f: the plant's where the call names one, else the model's
template <typename R>
struct EpisodeStep {
  int kind, has_f;
  const double* dyn;
  const R *F, *f;
};
template <typename R>
static EpisodeStep<R> episode_step(const EpisodeCall<R>& e) {
  if (e.plant == nullptr) return {e.d->dynamics_kind, e.d->has_f, e.p->dyn, e.F, e.f};
  return {e.plant->kind, e.plant->has_f, e.plant->dyn, e.F_plant, e.f_plant};
}

// a plant record against the staged dims: LinDx at those dims, or a known kind (its passthrough kind too) whose own
// (n, m) are exactly dims' (n, m)
static int plant_check(const mpcb200_dims* d, const mpcb200_plant* pl) {
  if (pl->kind == DYN_LINEAR) return MPCB200_OK;
  int n = 0, m = 0;
  if (!dyn_kind_dims(pl->kind, n, m) || n != d->n || m != d->m) return MPCB200_ERR_BAD_DIMS;
  return MPCB200_OK;
}

// the solve of every control step: the caller's problem from the state and warm-start buffers, its best iterate in
// the workspace
template <typename R>
static IlqrCall<R> episode_solve(const EpisodeCall<R>& e, const EpisodeLayout& l) {
  char* ws = (char*)e.workspace;
  const bool have = ws != nullptr;
  return {e.d, e.p, e.o, e.C, e.c, e.F, e.f,
          have ? (const R*)(ws + l.state) : nullptr, have ? (const R*)(ws + l.warm) : nullptr,
          e.u_lower, e.u_upper, e.u_zero_I,
          have ? (R*)(ws + l.best_x) : nullptr, have ? (R*)(ws + l.best_u) : nullptr,
          have ? (R*)(ws + l.best_costs) : nullptr, have ? (R*)(ws + l.best_fdn) : nullptr,
          have ? (int32_t*)(ws + l.info) : nullptr, e.workspace, l.ilqr.total};
}

// ilqr_check of the solve, plus the episode's own: every error is reported before anything is captured or launched
template <typename R>
static int episode_check(const EpisodeCall<R>& e, int knob) {
  int rc = check_dims(e.d);
  if (rc) return rc;
  if (e.x_init == nullptr || e.xs == nullptr || e.us == nullptr || e.costs == nullptr || e.info == nullptr ||
      e.u_next == nullptr || e.workspace == nullptr)
    return MPCB200_ERR_NULL_POINTER;
  if (e.d->T < 3 || e.n_steps < 1) return MPCB200_ERR_BAD_DIMS;     // the warm-start shift reads u[T-3]
  MlpShape s;
  if (e.mlp != nullptr && (rc = episode_net_check(e.d, e.mlp, sizeof(R), smem_optin_or_h100(), s))) return rc;
  if ((e.plan_x == nullptr) != (e.plan_u == nullptr)) return MPCB200_ERR_NULL_POINTER;
  if (e.plant != nullptr) {
    rc = plant_check(e.d, e.plant);
    if (rc) return rc;
    if (e.plant->kind == DYN_LINEAR && (e.F_plant == nullptr || (e.plant->has_f && e.f_plant == nullptr)))
      return MPCB200_ERR_NULL_POINTER;
  }
  const EpisodeLayout l = episode_layout(e.d, sizeof(R), knob, e.mlp != nullptr);
  if (e.workspace_bytes < l.total || (reinterpret_cast<uintptr_t>(e.workspace) & 255u) != 0)
    return MPCB200_ERR_BAD_DIMS;
  const IlqrCall<R> q = episode_solve(e, l);
  return ilqr_check<R>(q, e.mlp, knob);
}

// Adds the episode's init kernel and its `while` node over control steps (body recorded on `es`) to the graph `os`
// is capturing.  Body: [window_stage_kernel, with wc] -> the iLQR loop (its own `while` node, body on `bs`) -> model
// step -> [episode_plans_kernel, with plan_x / plan_u] -> episode_advance_kernel.  With e.mlp the iLQR loop plans
// with the network, and without a plant the model step is the network's rollout at T = 2.
template <typename R>
static int episode_record(cudaStream_t os, cudaStream_t es, cudaStream_t bs, const EpisodeCall<R>& e, int knob,
                          const WindowCopy<R>* wc = nullptr) {
  const mpcb200_dims* d = e.d;
  const EpisodeLayout l = episode_layout(d, sizeof(R), knob, e.mlp != nullptr);
  const IlqrCall<R> q = episode_solve(e, l);
  char* ws = (char*)e.workspace;
  R* state = (R*)(ws + l.state);
  R* warm = (R*)(ws + l.warm);
  R* traj = (R*)(ws + l.traj);
  EpisodeState* ep = (EpisodeState*)(ws + l.ep);
  const int B = d->B, T = d->T, N = d->n, M = d->m;
  cudaGraphConditionalHandle handle;
  int rc = while_handle(os, &handle);
  if (rc) return rc;
  if (counted(episode_launch_init<R>((size_t)B * N, (size_t)T * B * M, e.x_init, e.u_init, state, e.xs, warm, ep,
                                     handle, os)) != 0)
    return MPCB200_ERR_LAUNCH;
  rc = open_while(os, es, handle);
  if (rc) return rc;
  if (wc != nullptr) rc = counted(window_launch_stage<R>(*wc, es));
  if (rc == 0) rc = ilqr_record<R>(es, bs, q, knob, e.mlp);
  // the model step (the plant's, where the call names one) from the solve's best controls, by the launchers the
  // solve's rollout uses, at T = 2
  const EpisodeStep<R> s = episode_step(e);
  if (rc == 0 && e.mlp != nullptr && e.plant == nullptr) {
    rc = mlp_rollout_impl<R>(e.mlp, B, 2, N, M, state, q.best_u, traj, es);
  } else if (rc == 0 && s.kind == DYN_LINEAR) {
    mpcb200_dims d2 = *d;
    d2.T = 2;
    d2.F_T = 1;
    if (e.plant != nullptr) {         // the plant's slice 0, dense
      d2.has_f = s.has_f;
      d2.F_tstride = d2.f_tstride = 0;
    }
    rc = rollout_impl<R>(&d2, s.F, s.f, state, q.best_u, traj, knob, es);
  } else if (rc == 0) {
    rc = dyn_impl<R>(false, s.kind, s.dyn, B, 2, state, q.best_u, traj, nullptr, nullptr, es);
  }
  if (rc == 0 && e.plan_x != nullptr)
    rc = counted(episode_launch_plans<R>(B, T, N, M, q.best_x, q.best_u, e.plan_x, e.plan_u, ep, es));
  if (rc == 0)
    rc = counted(episode_launch_advance<R>(B, T, N, M, e.o->m_ref, e.n_steps, traj, q.best_u, q.best_costs, q.info,
                                           e.w, state, warm, e.xs, e.us, e.costs, e.info, ep, handle, es));
  cudaGraph_t body = nullptr;
  if (cudaStreamEndCapture(es, &body) != cudaSuccess && rc == 0) rc = MPCB200_ERR_LAUNCH;
  if (rc == 0 && cudaMemcpyAsync(e.u_next, warm, (size_t)T * B * M * sizeof(R), cudaMemcpyDeviceToDevice, os) !=
                     cudaSuccess)
    rc = MPCB200_ERR_LAUNCH;
  return rc;
}

// The episode of `e`; w (mpcb200_episode_window_*, non-NULL): each control step's window of e's full-length inputs is
// staged into workspace buffers that the episode reads.  Every argument error is reported before anything is captured.
template <typename R>
static int episode_impl(EpisodeCall<R> e, const mpcb200_window* w, void* stream) {
  const int knob = kernel_knob();
  mpcb200_dims ds;
  WindowCopy<R> wc;
  if (w != nullptr) {
    int rc = check_dims(e.d);
    if (rc) return rc;
    rc = window_check(e.d, w, e.n_steps, e.plant);
    if (rc) return rc;
    const bool has_f = e.d->has_f != 0;
    if (e.C == nullptr || e.c == nullptr || ((w->on & MPCB200_WIN_DYN) && (e.F == nullptr || (has_f && !e.f))) ||
        ((w->on & MPCB200_WIN_BOUNDS) && (e.u_lower == nullptr || e.u_upper == nullptr)) ||
        ((w->on & MPCB200_WIN_PLANT) && (e.F_plant == nullptr || (e.plant->has_f && e.f_plant == nullptr))))
      return MPCB200_ERR_NULL_POINTER;
    ds = window_solve_dims(e.d, w);
    const EpisodeLayout el = episode_layout(&ds, sizeof(R), knob);
    const WindowLayout l = window_layout(&ds, w, el.total, sizeof(R));
    if (e.workspace == nullptr) return MPCB200_ERR_NULL_POINTER;
    if (e.workspace_bytes < l.total || (reinterpret_cast<uintptr_t>(e.workspace) & 255u) != 0)
      return MPCB200_ERR_BAD_DIMS;
    char* ws = (char*)e.workspace;
    const R** in[WINDOW_INPUTS] = {&e.C, &e.c, &e.F, has_f ? &e.f : nullptr, &e.u_lower, &e.u_upper, &e.F_plant,
                                   e.plant != nullptr && e.plant->has_f ? &e.f_plant : nullptr};
    wc = window_copy<R>(&ds, w, l, ws, in, (const int32_t*)(ws + el.ep));
    e.d = &ds;
    e.workspace_bytes = el.total;
  }
  int rc = episode_check<R>(e, knob);
  if (rc) return rc;
  if (max_smem_optin() <= 0) return MPCB200_ERR_NO_DEVICE;
  return run_graph(stream, [&](cudaStream_t os) {
    cudaStream_t es = ilqr_stream(2), bs = ilqr_stream(1);
    return es == nullptr || bs == nullptr ? MPCB200_ERR_LAUNCH
                                          : episode_record<R>(os, es, bs, e, knob, w != nullptr ? &wc : nullptr);
  });
}

// ---------------------------------------------------------------------------------------------
// the reverse sweep of an episode (episode_grad.cuh): for k = n_steps-1 .. 0, the model step's VJP, each solve's KKT
// adjoint at its best iterate (a known system or a network: through its linearisation and that linearisation's VJP),
// summed
// ---------------------------------------------------------------------------------------------
// learnable parameters of a known system (DynLearnable), 0 for anything else
static int dyn_nparams(int kind) {
  return kind == DYN_CARTPOLE ? DynLearnable<DYN_CARTPOLE>::NP
         : kind == DYN_PENDULUM ? DynLearnable<DYN_PENDULUM>::NP
         : kind == DYN_PENDULUM_FULL ? DynLearnable<DYN_PENDULUM_FULL>::NP : 0;
}
// a sweep's parameter count: the system's, for its passthrough kind too
static int epgrad_nparams(int kind) { return dyn_nparams(kind & ~DYN_CTRL_PASSTHROUGH); }
// dims of each step's adjoint: the episode's; a known system's or the network's (net) F, f are its dense
// linearisation [T-1, B, ...]
static mpcb200_dims epgrad_adjoint_dims(const mpcb200_dims* d, bool net) {
  mpcb200_dims da = *d;
  if (net || d->dynamics_kind != DYN_LINEAR) {
    da.F_T = d->T - 1; da.has_f = 1; da.F_tstride = 0; da.f_tstride = 0;
  }
  da.dynamics_kind = DYN_LINEAR;
  return da;
}

struct EpGradLayout {                 // workspace carve-up (byte offsets, every piece 256-byte aligned)
  mpcb200_dims da;
  size_t adj, adj_bytes, stage_x, stage_u, dl_dx, dl_du, gx, theta, dxk, dCk, dck, dFk, dfk, Fk, fk, first, second,
      dthk, vjp, vjp_bytes, state, total;
};
// step_kind: the kind of the step whose parameter part the stage writes (the plant's; -1: the model's).  net: the
// shape of the network the episode planned with (mpcb200_episode_backward_mlp_*), or NULL; vjp_bytes is 0 where its
// linearisation VJP does not fit.
static EpGradLayout epgrad_layout(const mpcb200_dims* d, size_t sz, int knob, int step_kind = -1,
                                  const MlpShape* net = nullptr) {
  EpGradLayout l;
  l.da = epgrad_adjoint_dims(d, net != nullptr);
  const size_t B = d->B, T = d->T, n = d->n, m = d->m, p = n + m, TB = T * B, T1B = (T - 1) * B;
  const size_t NP = epgrad_nparams(d->dynamics_kind);
  const size_t NP_step = step_kind < 0 ? NP : (size_t)epgrad_nparams(step_kind);
  const bool known = d->dynamics_kind != DYN_LINEAR;
  size_t o = 0;
  l.adj_bytes = adj_layout(&l.da, sz, knob).total;
  l.adj = o;      o += up256(l.adj_bytes);
  l.stage_x = o;  o += up256(TB * n * sz);
  l.stage_u = o;  o += up256(TB * m * sz);
  l.dl_dx = o;    o += up256(TB * n * sz);
  l.dl_du = o;    o += up256(TB * m * sz);
  l.gx = o;       o += up256(B * n * sz);
  l.theta = o;    o += up256(B * NP_step * sz);
  l.dxk = o;      o += up256(B * n * sz);
  l.dCk = o;      o += up256(TB * p * p * sz);
  l.dck = o;      o += up256(TB * p * sz);
  l.dFk = o;      o += up256((size_t)l.da.F_T * B * n * p * sz);
  l.dfk = o;      o += up256(l.da.has_f ? T1B * n * sz : 0);
  l.Fk = l.fk = l.first = l.second = l.dthk = l.vjp = l.vjp_bytes = 0;
  if (known || net != nullptr) {      // the linearisation along the staged plan
    l.Fk = o;     o += up256(T1B * n * p * sz);
    l.fk = o;     o += up256(T1B * n * sz);
  }
  if (known) {                        // a known system's linearisation VJP
    l.first = o;  o += up256(T1B * NP * sz);
    l.second = o; o += up256(T1B * NP * sz);
  }
  if (net != nullptr) {               // step k's weight gradient, and the network's linearisation VJP
    l.dthk = o;   o += up256((size_t)net->n_params * sz);
    l.vjp_bytes = mlp_vjp_ws(*net, d->B, d->T, sz);
    l.vjp = o;    o += l.vjp_bytes;
  }
  l.state = o;    o += up256(sizeof(EpGradState));
  l.total = o;
  return l;
}

// the arguments of mpcb200_episode_backward_*, in the header's order; mpcb200_episode_backward_slew_* adds n_prev
template <typename R>
struct EpGradCall {
  const mpcb200_dims* d;
  const mpcb200_params* p;
  int n_steps;
  const R *C, *c, *F, *u_lower, *u_upper, *xs, *us, *plan_x, *plan_u, *dl_dxs, *dl_dus;
  R *dx_init, *dC, *dc, *dF, *df, *dtheta;
  void* workspace;
  size_t workspace_bytes;
  bool slew = false;          // the slew entry: the augmented problem, with the first n_prev states detached
  int n_prev = 0;
  // mpcb200_episode_backward_plant_*: the plant that stepped the loop, and its own outputs (EpPlantArgs)
  const mpcb200_plant* plant = nullptr;
  const R* F_plant = nullptr;
  R *dF_plant = nullptr, *df_plant = nullptr, *dtheta_plant = nullptr, *dw = nullptr;
  // mpcb200_episode_backward_mlp_*: the learned model; dtheta is then its packed parameters' gradient [n_params]
  const mpcb200_mlp* mlp = nullptr;
};

// the plant entry's own checks: plant_check, a passthrough kind exactly under a slew-rate penalty (n_prev its
// n_ctrl), and the outputs its kind writes
template <typename R>
static int epgrad_plant_check(const EpGradCall<R>& q) {
  const mpcb200_plant* pl = q.plant;
  int rc = plant_check(q.d, pl);
  if (rc) return rc;
  if (pl->kind == DYN_LINEAR) {
    if (q.F_plant == nullptr || q.dF_plant == nullptr || (pl->has_f && q.df_plant == nullptr))
      return MPCB200_ERR_NULL_POINTER;
    return MPCB200_OK;
  }
  int n = 0, m = 0;
  dyn_kind_dims(pl->kind & ~DYN_CTRL_PASSTHROUGH, n, m);
  const bool through = (pl->kind & DYN_CTRL_PASSTHROUGH) != 0;
  if (through != (q.n_prev > 0) || (through && q.n_prev != m)) return MPCB200_ERR_BAD_DIMS;
  return q.dtheta_plant == nullptr ? MPCB200_ERR_NULL_POINTER : MPCB200_OK;
}

// the slew entry's own dims checks: 1 <= n_prev <= m and n_prev < n; a known system is its passthrough kind at its
// dynamics-only shape, with n_prev its n_ctrl (the systems themselves belong to mpcb200_episode_backward_*)
static bool slew_dims_ok(const mpcb200_dims* d, int n_prev) {
  if (n_prev < 1 || n_prev > d->m || n_prev >= d->n) return false;
  if (d->dynamics_kind == DYN_LINEAR) return true;
  int n = 0, m = 0;
  return (d->dynamics_kind & DYN_CTRL_PASSTHROUGH) != 0 && epgrad_nparams(d->dynamics_kind) != 0 &&
         known_shape_ok(d) && dyn_kind_dims(d->dynamics_kind & ~DYN_CTRL_PASSTHROUGH, n, m) && n_prev == m;
}

// the model a reverse sweep takes: under a slew-rate penalty slew_dims_ok's, otherwise LinDx or a known system with
// learnable parameters at its own shape (mpcb200_episode_backward_*)
static bool sweep_model_ok(const mpcb200_dims* d, bool slew, int n_prev) {
  if (slew) return slew_dims_ok(d, n_prev);
  return d->dynamics_kind == DYN_LINEAR || (dyn_nparams(d->dynamics_kind) != 0 && known_shape_ok(d));
}

// argument checks that need no device: every error is reported before anything is captured or launched.  s: the
// shape of q.mlp, where the call has one.
template <typename R>
static int epgrad_check(const EpGradCall<R>& q, int knob, MlpShape& s) {
  const mpcb200_dims* d = q.d;
  const bool net = q.mlp != nullptr;
  int rc = check_dims(d);
  if (rc) return rc;
  if (q.p == nullptr || q.C == nullptr || q.c == nullptr || q.xs == nullptr || q.us == nullptr ||
      q.plan_x == nullptr || q.plan_u == nullptr || q.dl_dxs == nullptr || q.dl_dus == nullptr ||
      q.dx_init == nullptr || q.dC == nullptr || q.dc == nullptr || q.workspace == nullptr ||
      (net && q.dtheta == nullptr))
    return MPCB200_ERR_NULL_POINTER;
  if (d->T < 3 || q.n_steps < 1 || (net && d->dynamics_kind != DYN_LINEAR)) return MPCB200_ERR_BAD_DIMS;
  if (net) {                          // a network that fits, and whose linearisation VJP fits
    rc = episode_net_check(d, q.mlp, sizeof(R), smem_optin_or_h100(), s);
    if (rc) return rc;
    if (mlp_vjp_ws(s, d->B, d->T, sizeof(R)) == 0) return MPCB200_ERR_SMEM;
  }
  if (q.slew && !slew_dims_ok(d, q.n_prev)) return MPCB200_ERR_BAD_DIMS;
  rc = check_bounds(d, q.u_lower, q.u_upper);
  if (rc) return rc;
  if (!net) {
    if (!sweep_model_ok(d, q.slew, q.n_prev)) return MPCB200_ERR_BAD_DIMS;
    if (d->dynamics_kind != DYN_LINEAR) {
      if (q.dtheta == nullptr) return MPCB200_ERR_NULL_POINTER;
    } else if (q.F == nullptr || q.dF == nullptr || (d->has_f && q.df == nullptr)) {
      return MPCB200_ERR_NULL_POINTER;
    }
  }
  if (q.plant != nullptr) {
    rc = epgrad_plant_check(q);
    if (rc) return rc;
  }
  const EpGradLayout l = epgrad_layout(d, sizeof(R), knob, q.plant != nullptr ? q.plant->kind : -1, net ? &s : nullptr);
  if (q.workspace_bytes < l.total || (reinterpret_cast<uintptr_t>(q.workspace) & 255u) != 0)
    return MPCB200_ERR_BAD_DIMS;
  return MPCB200_OK;
}

// Adds the init kernel and the `while` node over k = n_steps-1 .. 0 (body recorded on `bs`) to the graph `os` is
// capturing.  Body: stage -> [linearisation] -> adjoint -> [linearisation VJP] -> accumulate.
// wc, wn (mpcb200_episode_backward_window_*): window_stage_kernel first in the body, and the window forms of init,
// stage and accumulate.
// q.mlp, s its shape (episode_grad.cuh): dtheta's zeroing before the init kernel, and the body plan or the plant's
// stage -> the network's linearisation -> [stage_net] -> adjoint -> [net_step_param] -> linearisation VJP -> add ->
// accumulate.
template <typename R>
static int epgrad_record(cudaStream_t os, cudaStream_t bs, const EpGradCall<R>& q, const MlpShape& s, int knob,
                         const WindowCopy<R>* wc, const EpWindow* wn) {
  const mpcb200_dims* d = q.d;
  const bool net = q.mlp != nullptr;
  const EpGradLayout l = epgrad_layout(d, sizeof(R), knob, q.plant != nullptr ? q.plant->kind : -1, net ? &s : nullptr);
  char* ws = (char*)q.workspace;
  const bool known = d->dynamics_kind != DYN_LINEAR;
  const int B = d->B, T = d->T, N = d->n, M = d->m;
  R* Fk = (R*)(ws + l.Fk);
  R* fk = (R*)(ws + l.fk);
  EpGradArgs<R> a;
  std::memset(&a, 0, sizeof(a));
  a.B = B; a.T = T; a.N = N; a.M = M; a.n_steps = q.n_steps; a.F_T = l.da.F_T; a.has_f = l.da.has_f;
  a.kind = net ? EPGRAD_KIND_NET : d->dynamics_kind; a.NP = epgrad_nparams(d->dynamics_kind);
  for (int i = 0; i < 8; ++i) a.dp.p[i] = q.p->dyn[i];
  a.xs = q.xs; a.us = q.us; a.plan_x = q.plan_x; a.plan_u = q.plan_u; a.dl_dxs = q.dl_dxs; a.dl_dus = q.dl_dus;
  a.F = net ? Fk : known ? nullptr : q.F;         // the network's: slice 0 is the model step's Jacobian at (x_k, u_k)
  a.stage_x = (R*)(ws + l.stage_x); a.stage_u = (R*)(ws + l.stage_u);
  a.dl_dx = (R*)(ws + l.dl_dx); a.dl_du = (R*)(ws + l.dl_du);
  a.gx = (R*)(ws + l.gx); a.theta_step = known ? (R*)(ws + l.theta) : nullptr;
  a.g = q.dx_init;
  R* dxk = (R*)(ws + l.dxk);
  R* dCk = (R*)(ws + l.dCk);
  R* dck = (R*)(ws + l.dck);
  R* dFk = (R*)(ws + l.dFk);
  R* dfk = l.da.has_f ? (R*)(ws + l.dfk) : nullptr;
  R* first = known ? (R*)(ws + l.first) : nullptr;
  R* second = known ? (R*)(ws + l.second) : nullptr;
  a.dx_k = dxk; a.dC_k = dCk; a.dc_k = dck; a.dF_k = dFk; a.df_k = dfk; a.first = first; a.second = second;
  a.dC = q.dC; a.dc = q.dc;
  a.dF = known ? nullptr : q.dF; a.df = known || !d->has_f ? nullptr : q.df;
  a.dtheta = known ? q.dtheta : nullptr;
  a.st = (EpGradState*)(ws + l.state);
  // the stage runs on the plant: a copy of `a` with its kind, parameters, F and parameter-part outputs
  EpGradArgs<R> as = a;
  EpPlantArgs<R> pl;
  std::memset(&pl, 0, sizeof(pl));
  if (q.plant != nullptr) {
    const bool pknown = q.plant->kind != DYN_LINEAR;
    as.kind = q.plant->kind; as.has_f = q.plant->has_f; as.NP = epgrad_nparams(q.plant->kind);
    for (int i = 0; i < 8; ++i) as.dp.p[i] = q.plant->dyn[i];
    as.F = pknown ? nullptr : q.F_plant;
    as.dF = pknown ? nullptr : q.dF_plant;
    as.df = pknown || !q.plant->has_f ? nullptr : q.df_plant;
    as.theta_step = pknown ? (R*)(ws + l.theta) : nullptr;
    pl.kind = as.kind; pl.has_f = as.has_f; pl.NP = as.NP; pl.theta_step = as.theta_step;
    pl.dF = as.dF; pl.df = as.df; pl.dtheta = pknown ? q.dtheta_plant : nullptr; pl.dw = q.dw;
  } else if (net && q.dw != nullptr) {  // the network steps a disturbed loop: the plant forms write dw, nothing else
    pl.kind = EPGRAD_KIND_NET;
    pl.dw = q.dw;
  }
  const EpPlantArgs<R>* plp = q.plant != nullptr || (net && q.dw != nullptr) ? &pl : nullptr;
  cudaGraphConditionalHandle handle;
  int rc = while_handle(os, &handle);
  if (rc) return rc;
  if (net && counted(launch_fill_zero<R>((size_t)s.n_params, q.dtheta, os)) != 0) return MPCB200_ERR_LAUNCH;
  if (counted(wn != nullptr ? epgrad_launch_init_window<R>(a, q.n_prev, plp, *wn, handle, os)
                            : epgrad_launch_init<R>(a, q.n_prev, plp, handle, os)) != 0)
    return MPCB200_ERR_LAUNCH;
  rc = open_while(os, bs, handle);
  if (rc) return rc;
  if (wc != nullptr) rc = counted(window_launch_stage<R>(*wc, bs));
  if (rc == 0)
    rc = counted(net && q.plant == nullptr ? epgrad_launch_plan<R>(a, bs)
                 : wn != nullptr           ? epgrad_launch_stage_window<R>(as, *wn, bs)
                                           : epgrad_launch_stage<R>(as, bs));
  if (rc == 0 && net) {
    rc = mlp_linearize_impl<R>(q.mlp, B, T, N, M, a.stage_x, a.stage_u, Fk, fk, bs);
    if (rc == 0 && q.plant == nullptr) rc = counted(epgrad_launch_stage_net<R>(a, bs));
  } else if (rc == 0 && known) {
    rc = dyn_impl<R>(true, d->dynamics_kind, q.p->dyn, B, T, a.stage_x, a.stage_u, nullptr, Fk, fk, bs);
  }
  if (rc == 0)
    rc = adjoint_impl<R>(&l.da, q.p, q.C, q.c, net || known ? Fk : q.F, a.stage_x, a.stage_u, a.dl_dx, a.dl_du,
                         q.u_lower, q.u_upper, dxk, dCk, dck, dFk, dfk, ws + l.adj, l.adj_bytes, knob, bs, true);
  if (rc == 0 && net) {
    R* dthk = (R*)(ws + l.dthk);
    // the network's own step: with (dJ, df) = (g z^T, g) the VJP's G^ = dJ - df z^T is 0, so it returns d<g, x'>/dtheta
    if (q.plant == nullptr) rc = counted(epgrad_launch_net_step_param<R>(a, dFk, dfk, bs));
    if (rc == 0)
      rc = mlp_linearize_vjp_impl<R>(q.mlp, B, T, N, M, a.stage_x, a.stage_u, dFk, dfk, dthk, ws + l.vjp, l.vjp_bytes,
                                     bs);
    if (rc == 0) rc = counted(epgrad_launch_add<R>((size_t)s.n_params, dthk, q.dtheta, bs));
  } else if (rc == 0 && known && !q.slew) {
    rc = dyn_vjp_impl<R>(d->dynamics_kind, q.p->dyn, B, T, a.stage_x, a.stage_u, dFk, dfk, first, second, bs);
  } else if (rc == 0 && known) {
    DynVjpArgs v;
    std::memset(&v, 0, sizeof(v));
    v.B = B; v.T = T; v.kind = d->dynamics_kind; v.dp = a.dp;
    v.x = a.stage_x; v.u = a.stage_u; v.dF = dFk; v.df = dfk; v.first = first; v.second = second;
    rc = counted(epgrad_launch_vjp_passthrough<R>(v, bs));
  }
  if (rc == 0)
    rc = counted(wn != nullptr ? epgrad_launch_accum_window<R>(a, q.n_prev, plp, *wn, handle, bs)
                               : epgrad_launch_accum<R>(a, q.n_prev, plp, handle, bs));
  cudaGraph_t body = nullptr;
  if (cudaStreamEndCapture(bs, &body) != cudaSuccess && rc == 0) rc = MPCB200_ERR_LAUNCH;
  return rc;
}

// The sweep of `q`; w (mpcb200_episode_backward_window_*, non-NULL): each control step's window of q's full-length
// inputs is staged into workspace buffers that the sweep reads.  Every argument error is reported before anything is
// captured.
template <typename R>
static int epgrad_impl(EpGradCall<R> q, const mpcb200_window* w, void* stream) {
  const int knob = kernel_knob();
  mpcb200_dims ds;
  WindowCopy<R> wc;
  EpWindow wn;
  if (w != nullptr) {
    int rc = check_dims(q.d);
    if (rc) return rc;
    rc = window_check(q.d, w, q.n_steps, q.plant);
    if (rc) return rc;
    if (q.C == nullptr || q.c == nullptr || ((w->on & MPCB200_WIN_DYN) && q.F == nullptr) ||
        ((w->on & MPCB200_WIN_BOUNDS) && (q.u_lower == nullptr || q.u_upper == nullptr)) ||
        ((w->on & MPCB200_WIN_PLANT) && q.F_plant == nullptr))
      return MPCB200_ERR_NULL_POINTER;
    if (q.d->T < 3) return MPCB200_ERR_BAD_DIMS;
    ds = window_solve_dims(q.d, w);
    const EpGradLayout gl = epgrad_layout(&ds, sizeof(R), knob, q.plant != nullptr ? q.plant->kind : -1);
    const WindowLayout l = window_layout(&ds, w, gl.total, sizeof(R));
    if (q.workspace == nullptr) return MPCB200_ERR_NULL_POINTER;
    if (q.workspace_bytes < l.total || (reinterpret_cast<uintptr_t>(q.workspace) & 255u) != 0)
      return MPCB200_ERR_BAD_DIMS;
    char* ws = (char*)q.workspace;
    const R** in[WINDOW_INPUTS] = {&q.C, &q.c, &q.F, nullptr, &q.u_lower, &q.u_upper, &q.F_plant, nullptr};
    wc = window_copy<R>(&ds, w, l, ws, in, (const int32_t*)(ws + gl.state));
    q.d = &ds;
    q.workspace_bytes = gl.total;
    wn.cost = 1;
    wn.dyn = (w->on & MPCB200_WIN_DYN) != 0;
    wn.step = q.plant != nullptr ? (w->on & MPCB200_WIN_PLANT) != 0 : wn.dyn;
    wn.L = w->L;
    wn.LF = w->L - ds.T + ds.F_T;
    wn.Lf = w->L - 1;
    wn.Lp = w->L - 1;
  }
  MlpShape s;
  int rc = epgrad_check<R>(q, knob, s);
  if (rc) return rc;
  if (max_smem_optin() <= 0) return MPCB200_ERR_NO_DEVICE;
  return run_graph(stream, [&](cudaStream_t os) {
    cudaStream_t bs = ilqr_stream(2);
    return bs == nullptr ? MPCB200_ERR_LAUNCH
                         : epgrad_record<R>(os, bs, q, s, knob, w != nullptr ? &wc : nullptr,
                                            w != nullptr ? &wn : nullptr);
  });
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
  return step_impl<float>(dims, params,
                          {C, c, F, f, x_init, cur_x, cur_u, u_lower, u_upper, u_zero_I, new_x, new_u, costs,
                           full_du_norm, alphas, du_first, qp_iters, free_mask, status, Ks, ks},
                          kernel_knob(), stream);
}
int mpcb200_lqr_step_f64(const mpcb200_dims* dims, const mpcb200_params* params, const double* C,
                         const double* c, const double* F, const double* f, const double* x_init,
                         const double* cur_x, const double* cur_u, const double* u_lower,
                         const double* u_upper, const uint8_t* u_zero_I, double* new_x, double* new_u,
                         double* costs, double* full_du_norm, double* alphas, double* du_first, int32_t* qp_iters,
                         uint8_t* free_mask, int32_t* status, double* Ks, double* ks, void* stream) {
  return step_impl<double>(dims, params,
                           {C, c, F, f, x_init, cur_x, cur_u, u_lower, u_upper, u_zero_I, new_x, new_u, costs,
                            full_du_norm, alphas, du_first, qp_iters, free_mask, status, Ks, ks},
                           kernel_knob(), stream);
}
int mpcb200_lqr_grad_f32(const mpcb200_dims* dims, const float* C, const float* c, const float* F,
                         const float* new_x, const float* new_u, const float* dx, const float* du,
                         const float* dl_dx, float* dx_init, float* dC, float* dc, float* dF, float* df,
                         void* workspace, void* stream) {
  return grad_impl<float>(dims, C, c, F, new_x, new_u, dx, du, dl_dx, dx_init, dC, dc, dF, df, workspace,
                          kernel_knob(), stream);
}
int mpcb200_lqr_grad_f64(const mpcb200_dims* dims, const double* C, const double* c, const double* F,
                         const double* new_x, const double* new_u, const double* dx, const double* du,
                         const double* dl_dx, double* dx_init, double* dC, double* dc, double* dF,
                         double* df, void* workspace, void* stream) {
  return grad_impl<double>(dims, C, c, F, new_x, new_u, dx, du, dl_dx, dx_init, dC, dc, dF, df, workspace,
                           kernel_knob(), stream);
}

size_t mpcb200_adjoint_workspace_bytes(const mpcb200_dims* dims, int32_t elem_size) {
  if (dims == nullptr || check_dims(dims) != 0 || (elem_size != 4 && elem_size != 8)) return 0;
  return adj_layout(dims, (size_t)elem_size, kernel_knob()).total;
}
int mpcb200_lqr_adjoint_f32(const mpcb200_dims* dims, const mpcb200_params* params, const float* C, const float* c,
                            const float* F, const float* new_x, const float* new_u, const float* dl_dx,
                            const float* dl_du, const float* u_lower, const float* u_upper, float* dx_init,
                            float* dC, float* dc, float* dF, float* df, void* workspace, size_t workspace_bytes,
                            void* stream) {
  return adjoint_impl<float>(dims, params, C, c, F, new_x, new_u, dl_dx, dl_du, u_lower, u_upper, dx_init, dC, dc,
                             dF, df, workspace, workspace_bytes, kernel_knob(), stream);
}
int mpcb200_lqr_adjoint_f64(const mpcb200_dims* dims, const mpcb200_params* params, const double* C, const double* c,
                            const double* F, const double* new_x, const double* new_u, const double* dl_dx,
                            const double* dl_du, const double* u_lower, const double* u_upper, double* dx_init,
                            double* dC, double* dc, double* dF, double* df, void* workspace, size_t workspace_bytes,
                            void* stream) {
  return adjoint_impl<double>(dims, params, C, c, F, new_x, new_u, dl_dx, dl_du, u_lower, u_upper, dx_init, dC, dc,
                              dF, df, workspace, workspace_bytes, kernel_knob(), stream);
}

int mpcb200_rollout_f32(const mpcb200_dims* dims, const float* F, const float* f, const float* x_init,
                        const float* u, float* x, void* stream) {
  return rollout_impl<float>(dims, F, f, x_init, u, x, kernel_knob(), stream);
}
int mpcb200_rollout_f64(const mpcb200_dims* dims, const double* F, const double* f, const double* x_init,
                        const double* u, double* x, void* stream) {
  return rollout_impl<double>(dims, F, f, x_init, u, x, kernel_knob(), stream);
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
int mpcb200_dyn_linearize_vjp_f32(int32_t kind, const double* dyn, int32_t B, int32_t T, const float* x,
                                  const float* u, const float* dF, const float* df, float* first, float* second,
                                  void* stream) {
  return dyn_vjp_impl<float>(kind, dyn, B, T, x, u, dF, df, first, second, stream);
}
int mpcb200_dyn_linearize_vjp_f64(int32_t kind, const double* dyn, int32_t B, int32_t T, const double* x,
                                  const double* u, const double* dF, const double* df, double* first, double* second,
                                  void* stream) {
  return dyn_vjp_impl<double>(kind, dyn, B, T, x, u, dF, df, first, second, stream);
}

size_t mpcb200_ilqr_workspace_bytes(const mpcb200_dims* dims, const mpcb200_ilqr_opts* opts, int32_t elem_size) {
  if (dims == nullptr || opts == nullptr || check_dims(dims) != 0 || (elem_size != 4 && elem_size != 8)) return 0;
  if (dims->dynamics_kind != DYN_LINEAR && !known_shape_ok(dims)) return 0;
  return ilqr_layout(dims, (size_t)elem_size, kernel_knob(), false).total;
}
int mpcb200_ilqr_f32(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                     const float* C, const float* c, const float* F, const float* f, const float* x_init,
                     const float* u_init, const float* u_lower, const float* u_upper, const uint8_t* u_zero_I,
                     float* best_x, float* best_u, float* best_costs, float* best_full_du_norm, int32_t* info,
                     void* workspace, size_t workspace_bytes, void* stream) {
  return ilqr_impl<float>({dims, params, opts, C, c, F, f, x_init, u_init, u_lower, u_upper, u_zero_I, best_x, best_u,
                           best_costs, best_full_du_norm, info, workspace, workspace_bytes},
                          nullptr, stream);
}
int mpcb200_ilqr_f64(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                     const double* C, const double* c, const double* F, const double* f, const double* x_init,
                     const double* u_init, const double* u_lower, const double* u_upper, const uint8_t* u_zero_I,
                     double* best_x, double* best_u, double* best_costs, double* best_full_du_norm, int32_t* info,
                     void* workspace, size_t workspace_bytes, void* stream) {
  return ilqr_impl<double>({dims, params, opts, C, c, F, f, x_init, u_init, u_lower, u_upper, u_zero_I, best_x, best_u,
                            best_costs, best_full_du_norm, info, workspace, workspace_bytes},
                           nullptr, stream);
}

size_t mpcb200_episode_workspace_bytes(const mpcb200_dims* dims, const mpcb200_ilqr_opts* opts, int32_t elem_size) {
  if (mpcb200_ilqr_workspace_bytes(dims, opts, elem_size) == 0) return 0;
  return episode_layout(dims, (size_t)elem_size, kernel_knob()).total;
}
int mpcb200_episode_f32(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                        int32_t n_steps, const float* C, const float* c, const float* F, const float* f,
                        const float* x_init, const float* u_init, const float* u_lower, const float* u_upper,
                        const uint8_t* u_zero_I, float* xs, float* us, float* costs, int32_t* info, float* u_next,
                        void* workspace, size_t workspace_bytes, void* stream) {
  return episode_impl<float>({dims, params, opts, n_steps, C, c, F, f, x_init, u_init, u_lower, u_upper, u_zero_I, xs,
                              us, costs, info, u_next, workspace, workspace_bytes},
                             nullptr, stream);
}
int mpcb200_episode_f64(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                        int32_t n_steps, const double* C, const double* c, const double* F, const double* f,
                        const double* x_init, const double* u_init, const double* u_lower, const double* u_upper,
                        const uint8_t* u_zero_I, double* xs, double* us, double* costs, int32_t* info, double* u_next,
                        void* workspace, size_t workspace_bytes, void* stream) {
  return episode_impl<double>({dims, params, opts, n_steps, C, c, F, f, x_init, u_init, u_lower, u_upper, u_zero_I,
                               xs, us, costs, info, u_next, workspace, workspace_bytes},
                              nullptr, stream);
}

int mpcb200_episode_plans_f32(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                              int32_t n_steps, const float* C, const float* c, const float* F, const float* f,
                              const float* x_init, const float* u_init, const float* u_lower, const float* u_upper,
                              const uint8_t* u_zero_I, float* xs, float* us, float* costs, int32_t* info,
                              float* u_next, float* plan_x, float* plan_u, void* workspace, size_t workspace_bytes,
                              void* stream) {
  if (plan_x == nullptr || plan_u == nullptr) return MPCB200_ERR_NULL_POINTER;
  return episode_impl<float>({dims, params, opts, n_steps, C, c, F, f, x_init, u_init, u_lower, u_upper, u_zero_I, xs,
                              us, costs, info, u_next, workspace, workspace_bytes, plan_x, plan_u},
                             nullptr, stream);
}
int mpcb200_episode_plans_f64(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,
                              int32_t n_steps, const double* C, const double* c, const double* F, const double* f,
                              const double* x_init, const double* u_init, const double* u_lower,
                              const double* u_upper, const uint8_t* u_zero_I, double* xs, double* us, double* costs,
                              int32_t* info, double* u_next, double* plan_x, double* plan_u, void* workspace,
                              size_t workspace_bytes, void* stream) {
  if (plan_x == nullptr || plan_u == nullptr) return MPCB200_ERR_NULL_POINTER;
  return episode_impl<double>({dims, params, opts, n_steps, C, c, F, f, x_init, u_init, u_lower, u_upper, u_zero_I,
                               xs, us, costs, info, u_next, workspace, workspace_bytes, plan_x, plan_u},
                              nullptr, stream);
}

size_t mpcb200_episode_backward_workspace_bytes(const mpcb200_dims* dims, int32_t elem_size) {
  if (dims == nullptr || check_dims(dims) != 0 || dims->T < 3 || (elem_size != 4 && elem_size != 8)) return 0;
  if (!sweep_model_ok(dims, false, 0)) return 0;
  return epgrad_layout(dims, (size_t)elem_size, kernel_knob()).total;
}
int mpcb200_episode_backward_f32(const mpcb200_dims* dims, const mpcb200_params* params, int32_t n_steps,
                                 const float* C, const float* c, const float* F, const float* u_lower,
                                 const float* u_upper, const float* xs, const float* us, const float* plan_x,
                                 const float* plan_u, const float* dl_dxs, const float* dl_dus, float* dx_init,
                                 float* dC, float* dc, float* dF, float* df, float* dtheta, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  return epgrad_impl<float>({dims, params, n_steps, C, c, F, u_lower, u_upper, xs, us, plan_x, plan_u, dl_dxs, dl_dus,
                             dx_init, dC, dc, dF, df, dtheta, workspace, workspace_bytes},
                            nullptr, stream);
}
int mpcb200_episode_backward_f64(const mpcb200_dims* dims, const mpcb200_params* params, int32_t n_steps,
                                 const double* C, const double* c, const double* F, const double* u_lower,
                                 const double* u_upper, const double* xs, const double* us, const double* plan_x,
                                 const double* plan_u, const double* dl_dxs, const double* dl_dus, double* dx_init,
                                 double* dC, double* dc, double* dF, double* df, double* dtheta, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  return epgrad_impl<double>({dims, params, n_steps, C, c, F, u_lower, u_upper, xs, us, plan_x, plan_u, dl_dxs,
                              dl_dus, dx_init, dC, dc, dF, df, dtheta, workspace, workspace_bytes},
                             nullptr, stream);
}

size_t mpcb200_episode_backward_slew_workspace_bytes(const mpcb200_dims* dims, int32_t n_prev, int32_t elem_size) {
  if (dims == nullptr || check_dims(dims) != 0 || dims->T < 3 || (elem_size != 4 && elem_size != 8)) return 0;
  if (!sweep_model_ok(dims, true, n_prev)) return 0;
  return epgrad_layout(dims, (size_t)elem_size, kernel_knob()).total;
}
int mpcb200_episode_backward_slew_f32(const mpcb200_dims* dims, const mpcb200_params* params, int32_t n_steps,
                                      int32_t n_prev, const float* C, const float* c, const float* F,
                                      const float* u_lower, const float* u_upper, const float* xs, const float* us,
                                      const float* plan_x, const float* plan_u, const float* dl_dxs,
                                      const float* dl_dus, float* dx_init, float* dC, float* dc, float* dF, float* df,
                                      float* dtheta, void* workspace, size_t workspace_bytes, void* stream) {
  return epgrad_impl<float>({dims, params, n_steps, C, c, F, u_lower, u_upper, xs, us, plan_x, plan_u, dl_dxs, dl_dus,
                             dx_init, dC, dc, dF, df, dtheta, workspace, workspace_bytes, true, n_prev},
                            nullptr, stream);
}
int mpcb200_episode_backward_slew_f64(const mpcb200_dims* dims, const mpcb200_params* params, int32_t n_steps,
                                      int32_t n_prev, const double* C, const double* c, const double* F,
                                      const double* u_lower, const double* u_upper, const double* xs,
                                      const double* us, const double* plan_x, const double* plan_u,
                                      const double* dl_dxs, const double* dl_dus, double* dx_init, double* dC,
                                      double* dc, double* dF, double* df, double* dtheta, void* workspace,
                                      size_t workspace_bytes, void* stream) {
  return epgrad_impl<double>({dims, params, n_steps, C, c, F, u_lower, u_upper, xs, us, plan_x, plan_u, dl_dxs,
                              dl_dus, dx_init, dC, dc, dF, df, dtheta, workspace, workspace_bytes, true, n_prev},
                             nullptr, stream);
}

#define MPCB200_EPISODE_PLANT(SUF, R)                                                                              \
  int mpcb200_episode_plant_##SUF(const mpcb200_dims* dims, const mpcb200_params* params,                          \
                                  const mpcb200_ilqr_opts* opts, const mpcb200_plant* plant, int32_t n_steps,      \
                                  const R* C, const R* c, const R* F, const R* f, const R* F_plant,                \
                                  const R* f_plant, const R* w, const R* x_init, const R* u_init, const R* u_lower, \
                                  const R* u_upper, const uint8_t* u_zero_I, R* xs, R* us, R* costs,               \
                                  int32_t* info, R* u_next, R* plan_x, R* plan_u, void* workspace,                 \
                                  size_t workspace_bytes, void* stream) {                                          \
    if (plant == nullptr) return MPCB200_ERR_NULL_POINTER;                                                         \
    EpisodeCall<R> e = {dims, params, opts, n_steps, C, c, F, f, x_init, u_init, u_lower, u_upper, u_zero_I, xs, us, \
                        costs, info, u_next, workspace, workspace_bytes, plan_x, plan_u, plant, F_plant, f_plant, w}; \
    return episode_impl<R>(e, nullptr, stream);                                                                    \
  }
MPCB200_EPISODE_PLANT(f32, float)
MPCB200_EPISODE_PLANT(f64, double)
#undef MPCB200_EPISODE_PLANT

size_t mpcb200_episode_backward_plant_workspace_bytes(const mpcb200_dims* dims, int32_t n_prev,
                                                      const mpcb200_plant* plant, int32_t elem_size) {
  if (dims == nullptr || plant == nullptr || check_dims(dims) != 0 || dims->T < 3 || (elem_size != 4 && elem_size != 8))
    return 0;
  if (!sweep_model_ok(dims, n_prev != 0, n_prev)) return 0;
  if (plant_check(dims, plant) != 0) return 0;
  return epgrad_layout(dims, (size_t)elem_size, kernel_knob(), plant->kind).total;
}
#define MPCB200_EPISODE_BACKWARD_PLANT(SUF, R)                                                                     \
  int mpcb200_episode_backward_plant_##SUF(                                                                        \
      const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_plant* plant, int32_t n_steps,         \
      int32_t n_prev, const R* C, const R* c, const R* F, const R* F_plant, const R* u_lower, const R* u_upper,    \
      const R* xs, const R* us, const R* plan_x, const R* plan_u, const R* dl_dxs, const R* dl_dus, R* dx_init,    \
      R* dC, R* dc, R* dF, R* df, R* dtheta, R* dF_plant, R* df_plant, R* dtheta_plant, R* dw, void* workspace,    \
      size_t workspace_bytes, void* stream) {                                                                      \
    if (plant == nullptr) return MPCB200_ERR_NULL_POINTER;                                                         \
    if (n_prev < 0) return MPCB200_ERR_BAD_DIMS;                                                                   \
    EpGradCall<R> q = {dims, params, n_steps, C, c, F, u_lower, u_upper, xs, us, plan_x, plan_u, dl_dxs, dl_dus,   \
                       dx_init, dC, dc, dF, df, dtheta, workspace, workspace_bytes, n_prev > 0, n_prev, plant,     \
                       F_plant, dF_plant, df_plant, dtheta_plant, dw};                                             \
    return epgrad_impl<R>(q, nullptr, stream);                                                                     \
  }
MPCB200_EPISODE_BACKWARD_PLANT(f32, float)
MPCB200_EPISODE_BACKWARD_PLANT(f64, double)
#undef MPCB200_EPISODE_BACKWARD_PLANT

size_t mpcb200_episode_window_workspace_bytes(const mpcb200_dims* dims, const mpcb200_ilqr_opts* opts,
                                              const mpcb200_window* window, int32_t elem_size) {
  (void)opts;
  if (dims == nullptr || window == nullptr || check_dims(dims) != 0 || (elem_size != 4 && elem_size != 8)) return 0;
  const mpcb200_dims ds = window_solve_dims(dims, window);
  const int knob = kernel_knob();
  return window_layout(&ds, window, episode_layout(&ds, (size_t)elem_size, knob).total, (size_t)elem_size).total;
}
#define MPCB200_EPISODE_WINDOW(SUF, R)                                                                             \
  int mpcb200_episode_window_##SUF(const mpcb200_dims* dims, const mpcb200_params* params,                         \
                                   const mpcb200_ilqr_opts* opts, const mpcb200_window* window,                    \
                                   const mpcb200_plant* plant, int32_t n_steps, const R* C, const R* c, const R* F, \
                                   const R* f, const R* F_plant, const R* f_plant, const R* w, const R* x_init,    \
                                   const R* u_init, const R* u_lower, const R* u_upper, const uint8_t* u_zero_I,   \
                                   R* xs, R* us, R* costs, int32_t* info, R* u_next, R* plan_x, R* plan_u,         \
                                   void* workspace, size_t workspace_bytes, void* stream) {                        \
    EpisodeCall<R> e = {dims, params, opts, n_steps, C, c, F, f, x_init, u_init, u_lower, u_upper, u_zero_I, xs, us, \
                        costs, info, u_next, workspace, workspace_bytes, plan_x, plan_u, plant, F_plant, f_plant, w}; \
    if (window == nullptr) return null_record(dims);                                                               \
    return episode_impl<R>(e, window, stream);                                                                     \
  }
MPCB200_EPISODE_WINDOW(f32, float)
MPCB200_EPISODE_WINDOW(f64, double)
#undef MPCB200_EPISODE_WINDOW

size_t mpcb200_episode_backward_window_workspace_bytes(const mpcb200_dims* dims, int32_t n_prev,
                                                       const mpcb200_window* window, const mpcb200_plant* plant,
                                                       int32_t elem_size) {
  if (dims == nullptr || window == nullptr || check_dims(dims) != 0 || dims->T < 3 || n_prev < 0 ||
      (elem_size != 4 && elem_size != 8))
    return 0;
  if (!sweep_model_ok(dims, n_prev != 0, n_prev)) return 0;
  if (plant != nullptr && plant_check(dims, plant) != 0) return 0;
  const mpcb200_dims ds = window_solve_dims(dims, window);
  const int knob = kernel_knob();
  const size_t base = epgrad_layout(&ds, (size_t)elem_size, knob, plant != nullptr ? plant->kind : -1).total;
  return window_layout(&ds, window, base, (size_t)elem_size).total;
}
#define MPCB200_EPISODE_BACKWARD_WINDOW(SUF, R)                                                                    \
  int mpcb200_episode_backward_window_##SUF(                                                                       \
      const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_window* window,                         \
      const mpcb200_plant* plant, int32_t n_steps, int32_t n_prev, const R* C, const R* c, const R* F,             \
      const R* F_plant, const R* u_lower, const R* u_upper, const R* xs, const R* us, const R* plan_x,             \
      const R* plan_u, const R* dl_dxs, const R* dl_dus, R* dx_init, R* dC, R* dc, R* dF, R* df, R* dtheta,        \
      R* dF_plant, R* df_plant, R* dtheta_plant, R* dw, void* workspace, size_t workspace_bytes, void* stream) {    \
    if (n_prev < 0) return MPCB200_ERR_BAD_DIMS;                                                                   \
    EpGradCall<R> q = {dims, params, n_steps, C, c, F, u_lower, u_upper, xs, us, plan_x, plan_u, dl_dxs, dl_dus,   \
                       dx_init, dC, dc, dF, df, dtheta, workspace, workspace_bytes, n_prev > 0, n_prev, plant,     \
                       F_plant, dF_plant, df_plant, dtheta_plant, dw};                                             \
    if (window == nullptr) return null_record(dims);                                                               \
    return epgrad_impl<R>(q, window, stream);                                                                      \
  }
MPCB200_EPISODE_BACKWARD_WINDOW(f32, float)
MPCB200_EPISODE_BACKWARD_WINDOW(f64, double)
#undef MPCB200_EPISODE_BACKWARD_WINDOW

size_t mpcb200_episode_mlp_workspace_bytes(const mpcb200_dims* dims, const mpcb200_ilqr_opts* opts,
                                           const mpcb200_mlp* mlp, int32_t elem_size) {
  MlpShape s;
  if (dims == nullptr || opts == nullptr || check_dims(dims) != 0 || dims->T < 3 || (elem_size != 4 && elem_size != 8))
    return 0;
  if (episode_net_check(dims, mlp, elem_size, kOptinAssumed, s) != 0) return 0;
  return episode_layout(dims, (size_t)elem_size, kernel_knob(), true).total;
}
#define MPCB200_EPISODE_MLP(SUF, R)                                                                                \
  int mpcb200_episode_mlp_##SUF(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts, \
                                const mpcb200_mlp* mlp, const mpcb200_plant* plant, int32_t n_steps, const R* C,   \
                                const R* c, const R* F_plant, const R* f_plant, const R* w, const R* x_init,       \
                                const R* u_init, const R* u_lower, const R* u_upper, const uint8_t* u_zero_I,      \
                                R* xs, R* us, R* costs, int32_t* info, R* u_next, R* plan_x, R* plan_u,            \
                                void* workspace, size_t workspace_bytes, void* stream) {                           \
    if (mlp == nullptr) return MPCB200_ERR_NULL_POINTER;                                                           \
    EpisodeCall<R> e = {dims, params, opts, n_steps, C, c, nullptr, nullptr, x_init, u_init, u_lower, u_upper,     \
                        u_zero_I, xs, us, costs, info, u_next, workspace, workspace_bytes, plan_x, plan_u, plant,  \
                        F_plant, f_plant, w, mlp};                                                                 \
    return episode_impl<R>(e, nullptr, stream);                                                                    \
  }
MPCB200_EPISODE_MLP(f32, float)
MPCB200_EPISODE_MLP(f64, double)
#undef MPCB200_EPISODE_MLP

size_t mpcb200_episode_backward_mlp_workspace_bytes(const mpcb200_dims* dims, const mpcb200_mlp* mlp,
                                                    const mpcb200_plant* plant, int32_t elem_size) {
  MlpShape s;
  if (dims == nullptr || check_dims(dims) != 0 || dims->T < 3 || dims->dynamics_kind != DYN_LINEAR ||
      (elem_size != 4 && elem_size != 8))
    return 0;
  if (episode_net_check(dims, mlp, elem_size, kOptinAssumed, s) != 0) return 0;
  if (plant != nullptr && (plant_check(dims, plant) != 0 || (plant->kind & DYN_CTRL_PASSTHROUGH) != 0)) return 0;
  const EpGradLayout l = epgrad_layout(dims, (size_t)elem_size, kernel_knob(), plant != nullptr ? plant->kind : -1, &s);
  return l.vjp_bytes == 0 ? 0 : l.total;
}
#define MPCB200_EPISODE_BACKWARD_MLP(SUF, R)                                                                       \
  int mpcb200_episode_backward_mlp_##SUF(                                                                          \
      const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_mlp* mlp, const mpcb200_plant* plant,  \
      int32_t n_steps, const R* C, const R* c, const R* F_plant, const R* u_lower, const R* u_upper, const R* xs,  \
      const R* us, const R* plan_x, const R* plan_u, const R* dl_dxs, const R* dl_dus, R* dx_init, R* dC, R* dc,    \
      R* dtheta, R* dF_plant, R* df_plant, R* dtheta_plant, R* dw, void* workspace, size_t workspace_bytes,        \
      void* stream) {                                                                                              \
    if (mlp == nullptr) return null_record(dims);                                                                  \
    EpGradCall<R> q = {dims, params, n_steps, C, c, nullptr, u_lower, u_upper, xs, us, plan_x, plan_u, dl_dxs,     \
                       dl_dus, dx_init, dC, dc, nullptr, nullptr, dtheta, workspace, workspace_bytes, false, 0,    \
                       plant, F_plant, dF_plant, df_plant, dtheta_plant, dw, mlp};                                 \
    return epgrad_impl<R>(q, nullptr, stream);                                                                     \
  }
MPCB200_EPISODE_BACKWARD_MLP(f32, float)
MPCB200_EPISODE_BACKWARD_MLP(f64, double)
#undef MPCB200_EPISODE_BACKWARD_MLP

int mpcb200_mlp_fits(const mpcb200_mlp* mlp, int32_t elem_size) {
  MlpShape s;
  if ((elem_size != 4 && elem_size != 8) || !mlp_shape(mlp, s)) return 0;
  return mlp_smem_bytes(s, elem_size, 1) <= (size_t)kOptinAssumed ? 1 : 0;
}
size_t mpcb200_mlp_linearize_vjp_workspace_bytes(const mpcb200_mlp* mlp, int32_t B, int32_t T, int32_t elem_size) {
  MlpShape s;
  if ((elem_size != 4 && elem_size != 8) || B <= 0 || T <= 0 || !mlp_shape(mlp, s)) return 0;
  return mlp_vjp_ws(s, B, T, (size_t)elem_size);
}
size_t mpcb200_mlp_step_workspace_bytes(const mpcb200_dims* dims, int32_t elem_size) {
  if (check_dims(dims) != MPCB200_OK || (elem_size != 4 && elem_size != 8)) return 0;
  return mlp_step_ws(dims, (size_t)elem_size);
}
size_t mpcb200_ilqr_mlp_workspace_bytes(const mpcb200_dims* dims, const mpcb200_ilqr_opts* opts, int32_t elem_size) {
  if (check_dims(dims) != MPCB200_OK || opts == nullptr || dims->T < 2 || (elem_size != 4 && elem_size != 8))
    return 0;
  return ilqr_layout(dims, (size_t)elem_size, kernel_knob(), true).total;
}
#define MPCB200_MLP_ENTRIES(sfx, R)                                                                                    \
  int mpcb200_mlp_rollout_##sfx(const mpcb200_mlp* mlp, int32_t B, int32_t T, int32_t N, int32_t M, const R* x_init,  \
                                const R* u, R* x, void* stream) {                                                      \
    return mlp_rollout_impl<R>(mlp, B, T, N, M, x_init, u, x, stream);                                                \
  }                                                                                                                    \
  int mpcb200_mlp_linearize_##sfx(const mpcb200_mlp* mlp, int32_t B, int32_t T, int32_t N, int32_t M, const R* x,     \
                                  const R* u, R* F, R* f, void* stream) {                                              \
    return mlp_linearize_impl<R>(mlp, B, T, N, M, x, u, F, f, stream);                                                \
  }                                                                                                                    \
  int mpcb200_mlp_linearize_vjp_##sfx(const mpcb200_mlp* mlp, int32_t B, int32_t T, int32_t N, int32_t M, const R* x, \
                                      const R* u, const R* dF, const R* df, R* dtheta, void* workspace,                \
                                      size_t workspace_bytes, void* stream) {                                          \
    return mlp_linearize_vjp_impl<R>(mlp, B, T, N, M, x, u, dF, df, dtheta, workspace, workspace_bytes, stream);      \
  }                                                                                                                    \
  int mpcb200_mlp_step_##sfx(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_mlp* mlp,           \
                             const R* C, const R* c, const R* F, const R* f, const R* x_init, const R* cur_x,          \
                             const R* cur_u, const R* u_lower, const R* u_upper, const uint8_t* u_zero_I, R* new_x,    \
                             R* new_u, R* costs, R* alphas, R* du_first, int32_t* qp_iters, uint8_t* free_mask,        \
                             int32_t* status, void* workspace, size_t workspace_bytes, void* stream) {                 \
    return mlp_step_impl<R>(dims, params, mlp,                                                                         \
                            {C, c, F, f, x_init, cur_x, cur_u, u_lower, u_upper, u_zero_I, new_x, new_u, costs,        \
                             nullptr, alphas, du_first, qp_iters, free_mask, status},                                  \
                            workspace, workspace_bytes, stream);                                                       \
  }                                                                                                                    \
  int mpcb200_ilqr_mlp_##sfx(const mpcb200_dims* dims, const mpcb200_params* params, const mpcb200_ilqr_opts* opts,   \
                             const mpcb200_mlp* mlp, const R* C, const R* c, const R* x_init, const R* u_init,         \
                             const R* u_lower, const R* u_upper, const uint8_t* u_zero_I, R* best_x, R* best_u,        \
                             R* best_costs, R* best_full_du_norm, int32_t* info, void* workspace,                      \
                             size_t workspace_bytes, void* stream) {                                                   \
    if (mlp == nullptr) return null_record(dims);                                                                     \
    return ilqr_impl<R>({dims, params, opts, C, c, nullptr, nullptr, x_init, u_init, u_lower, u_upper, u_zero_I,       \
                         best_x, best_u, best_costs, best_full_du_norm, info, workspace, workspace_bytes},             \
                        mlp, stream);                                                                                  \
  }
MPCB200_MLP_ENTRIES(f32, float)
MPCB200_MLP_ENTRIES(f64, double)

int mpcb200_supported(int32_t n_state, int32_t n_ctrl) { return find(n_state, n_ctrl) != nullptr; }

int mpcb200_supported_list(int32_t* out, int32_t cap) {
  int count = 0;
  for (const Instance* e : kInstances) {
    if (e->kind != DYN_LINEAR) continue;
    if (count < cap) {
      out[2 * count] = e->n;
      out[2 * count + 1] = e->m;
    }
    ++count;
  }
  return count;
}

uint64_t mpcb200_launch_count(void) { return g_launches.load(); }

size_t mpcb200_step_smem_bytes(const mpcb200_dims* dims, int32_t elem_size) {
  if (dims == nullptr) return 0;
  const Instance* e = find_step(dims);
  return e == nullptr ? 0 : e->ops[elem_size == 8].smem_bytes(dims->T);
}

int mpcb200_step_prefers_workspace(const mpcb200_dims* dims, int32_t elem_size) {
  return dims == nullptr ? 0 : gains_in_workspace(dims, elem_size, kernel_knob());
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
