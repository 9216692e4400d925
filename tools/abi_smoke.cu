// abi_smoke.cu - plain C++/CUDA-runtime caller of the C ABI (no torch): exercises every entry point on
// small random problems, incl. shapes whose spans are not 16-byte aligned and tail CTAs.  Meant to
// run under `compute-sanitizer --tool memcheck` (fast: no Python start-up).
//   nvcc -O2 -o abi_smoke tools/abi_smoke.cu -Iinclude -Lmpc/pytorch_b200 -lmpcb200 -Xlinker -rpath=$PWD/mpc/pytorch_b200
#include <cuda_runtime.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "mpcb200.h"

template <typename R>
struct Dev {
  R* p = nullptr;
  size_t n = 0;
  explicit Dev(size_t n_) : n(n_) { cudaMalloc(&p, (n ? n : 1) * sizeof(R)); }
  ~Dev() { cudaFree(p); }
  void up(const std::vector<R>& h) { cudaMemcpy(p, h.data(), n * sizeof(R), cudaMemcpyHostToDevice); }
  std::vector<R> down() const {
    std::vector<R> h(n);
    cudaMemcpy(h.data(), p, n * sizeof(R), cudaMemcpyDeviceToHost);
    return h;
  }
};
static float rnd() { return (float)rand() / RAND_MAX * 2.f - 1.f; }

static int run_case(int B, int T, int n, int m, int bounds_kind, int with_mask) {
  const int p = n + m;
  std::vector<float> C((size_t)T * B * p * p), c((size_t)T * B * p), F((size_t)(T - 1) * B * n * p),
      f((size_t)(T - 1) * B * n), x0((size_t)B * n), cx((size_t)T * B * n, 0.f), cu((size_t)T * B * m, 0.f),
      lo((size_t)T * B * m, -0.25f), hi((size_t)T * B * m, 0.25f);
  std::vector<unsigned char> mask((size_t)T * B * m, 0);
  for (size_t tb = 0; tb < (size_t)T * B; ++tb) {          // C = L L' / p + I
    std::vector<float> L((size_t)p * p);
    for (auto& v : L) v = rnd();
    for (int i = 0; i < p; ++i)
      for (int j = 0; j < p; ++j) {
        float s = i == j ? 1.f : 0.f;
        for (int k = 0; k < p; ++k) s += L[i * p + k] * L[j * p + k] / p;
        C[(tb * p + i) * p + j] = s;
      }
  }
  for (auto& v : c) v = rnd();
  for (size_t i = 0; i < F.size(); ++i) F[i] = 0.3f * rnd();
  for (size_t tb = 0; tb < (size_t)(T - 1) * B; ++tb)
    for (int i = 0; i < n; ++i) F[(tb * n + i) * p + i] += 0.9f;
  for (auto& v : f) v = 0.1f * rnd();
  for (auto& v : x0) v = rnd();
  for (auto& v : mask) v = (rand() % 4) == 0;
  Dev<float> dC(C.size()), dc(c.size()), dF(F.size()), df(f.size()), dx0(x0.size()), dcx(cx.size()), dcu(cu.size()),
      dlo(lo.size()), dhi(hi.size()), nx(cx.size()), nu(cu.size()), costs(B), fdn(B), al(B), du1(cu.size()),
      Ks((size_t)T * B * m * n), ks((size_t)T * B * m);
  Dev<unsigned char> dmask(mask.size()), fmask(mask.size());
  Dev<int> qp((size_t)T * B), st(B);
  dC.up(C); dc.up(c); dF.up(F); df.up(f); dx0.up(x0); dcu.up(cu); dlo.up(lo); dhi.up(hi);
  cudaMemcpy(dmask.p, mask.data(), mask.size(), cudaMemcpyHostToDevice);
  mpcb200_dims d = {B, T, n, m, T - 1, 1, bounds_kind, with_mask, 0, 10, 20, 1};
  mpcb200_params prm = {-0.25, 0.25, 0.0, 0.2};
  int rc = mpcb200_rollout_f32(&d, dF.p, df.p, dx0.p, dcu.p, dcx.p, nullptr);
  if (rc) return printf("rollout rc=%d\n", rc), 1;
  rc = mpcb200_lqr_step_f32(&d, &prm, dC.p, dc.p, dF.p, df.p, dx0.p, dcx.p, dcu.p,
                            bounds_kind == 2 ? dlo.p : nullptr, bounds_kind == 2 ? dhi.p : nullptr,
                            with_mask ? dmask.p : nullptr, nx.p, nu.p, costs.p, fdn.p, al.p, du1.p, qp.p,
                            fmask.p, st.p, Ks.p, ks.p, nullptr);
  if (rc) return printf("step rc=%d (%s)\n", rc, mpcb200_strerror(rc)), 1;
  // adjoint: masked step on (C, -r) from zeros, then the gradient assembly
  Dev<float> r(c.size()), zx(cx.size()), zu(cu.size()), z0(x0.size()), ax(cx.size()), au(cu.size()), rx(cx.size()),
      gx0(x0.size()), gC(C.size()), gc(c.size()), gF(F.size()), gf(f.size()), ws((size_t)2 * T * B * n);
  std::vector<float> rr(c.size());
  for (auto& v : rr) v = rnd();
  r.up(rr);
  cudaMemset(zx.p, 0, cx.size() * 4); cudaMemset(zu.p, 0, cu.size() * 4); cudaMemset(z0.p, 0, x0.size() * 4);
  cudaMemset(rx.p, 0, cx.size() * 4);
  mpcb200_dims da = d;
  da.has_f = 0; da.bounds_kind = 0; da.has_zero_mask = 1;
  rc = mpcb200_lqr_step_f32(&da, &prm, dC.p, r.p, dF.p, nullptr, z0.p, zx.p, zu.p, nullptr, nullptr, dmask.p, ax.p,
                            au.p, costs.p, fdn.p, al.p, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
  if (rc) return printf("adjoint step rc=%d\n", rc), 1;
  rc = mpcb200_lqr_grad_f32(&d, dC.p, dc.p, dF.p, nx.p, nu.p, ax.p, au.p, rx.p, gx0.p, gC.p, gc.p, gF.p, gf.p, ws.p,
                            nullptr);
  if (rc) return printf("grad rc=%d\n", rc), 1;
  {  // the whole KKT adjoint in one call (prep + nested masked step + costates + outer products)
    const size_t wsb = mpcb200_adjoint_workspace_bytes(&d, 4);
    Dev<unsigned char> aws(wsb);
    Dev<float> wu(cu.size());
    std::vector<float> hw(cu.size());
    for (auto& v : hw) v = rnd();
    wu.up(hw);
    rc = mpcb200_lqr_adjoint_f32(&d, &prm, dC.p, dc.p, dF.p, nx.p, nu.p, r.p /* [T,B,p] >= [T,B,n] */, wu.p,
                                 bounds_kind == 2 ? dlo.p : nullptr, bounds_kind == 2 ? dhi.p : nullptr, gx0.p, gC.p,
                                 gc.p, gF.p, gf.p, aws.p, wsb, nullptr);
    if (rc) return printf("one-call adjoint rc=%d (%s)\n", rc, mpcb200_strerror(rc)), 1;
    // time-invariant dynamics / cost through the stride fields (one slice read for every t)
    mpcb200_dims ds = d;
    ds.F_tstride = MPCB200_TIME_INVARIANT;
    ds.C_tstride = MPCB200_TIME_INVARIANT;
    rc = mpcb200_lqr_step_f32(&ds, &prm, dC.p, dc.p, dF.p, df.p, dx0.p, dcx.p, dcu.p,
                              bounds_kind == 2 ? dlo.p : nullptr, bounds_kind == 2 ? dhi.p : nullptr,
                              with_mask ? dmask.p : nullptr, nx.p, nu.p, costs.p, fdn.p, al.p, nullptr, nullptr,
                              nullptr, st.p, Ks.p, ks.p, nullptr);
    if (rc) return printf("strided step rc=%d\n", rc), 1;
  }
  if (m <= 8) {   // standalone pnqp on the last step's C_uu blocks
    std::vector<float> H((size_t)B * m * m), q((size_t)B * m), l2((size_t)B * m, -0.25f), h2((size_t)B * m, 0.25f);
    for (int b = 0; b < B; ++b)
      for (int i = 0; i < m; ++i) {
        q[b * m + i] = rnd();
        for (int j = 0; j < m; ++j) H[(b * m + i) * m + j] = C[(((size_t)(T - 1) * B + b) * p + n + i) * p + n + j];
      }
    Dev<float> dH(H.size()), dq(q.size()), dl(l2.size()), dh(h2.size()), ox(q.size()), oH(H.size());
    Dev<unsigned char> oI(q.size());
    Dev<int> oit(B), ost(B);
    dH.up(H); dq.up(q); dl.up(l2); dh.up(h2);
    rc = mpcb200_pnqp_f32(B, m, dH.p, dq.p, dl.p, dh.p, nullptr, 20, ox.p, oH.p, oI.p, oit.p, ost.p, nullptr);
    if (rc) return printf("pnqp rc=%d\n", rc), 1;
    Dev<float> gH(H.size()), gq(q.size()), gl(q.size()), gh(q.size());   // its gradient for dL/dx = q
    rc = mpcb200_pnqp_backward_f32(B, m, dH.p, ox.p, oI.p, dl.p, dh.p, dq.p, gH.p, gq.p, gl.p, gh.p, ost.p, nullptr);
    if (rc) return printf("pnqp backward rc=%d\n", rc), 1;
  }
  if (cudaDeviceSynchronize() != cudaSuccess) return printf("CUDA error: %s\n", cudaGetErrorString(cudaGetLastError())), 1;
  double s = 0;
  int bad = 0;
  for (float v : nu.down()) { s += v; bad += !std::isfinite(v); }
  for (float v : gC.down()) { s += v; bad += !std::isfinite(v); }
  printf("B=%d T=%d n=%d m=%d bounds=%d mask=%d: checksum %.6f nonfinite %d\n", B, T, n, m, bounds_kind, with_mask, s, bad);
  return bad != 0;
}

// known systems: rollout, exact Jacobians, and the step kernel with the system inside its line search
static int run_dyn(int kind, int B, int T) {
  const int n = kind == MPCB200_DYN_CARTPOLE ? 5 : 3, m = 1, p = n + m;
  const double prm_c[8] = {9.8, 1.0, 0.1, 0.5, 100.0, 0.05, 0, 0}, prm_p[8] = {10.0, 1.0, 1.0, 0.0, 2.0, 0.05, 0, 0},
               prm_pf[8] = {10.0, 1.0, 1.0, 0.3, 0.2, 2.0, 0.05, 0};
  const double* dyn = kind == MPCB200_DYN_CARTPOLE ? prm_c : (kind == MPCB200_DYN_PENDULUM ? prm_p : prm_pf);
  std::vector<float> x0((size_t)B * n), u((size_t)T * B * m), C((size_t)T * B * p * p, 0.f), c((size_t)T * B * p);
  for (int b = 0; b < B; ++b) {
    const float th = 3.f * rnd();
    float* s = &x0[(size_t)b * n];
    if (n == 5) { s[0] = rnd(); s[1] = rnd(); s[2] = cosf(th); s[3] = sinf(th); s[4] = rnd(); }
    else { s[0] = cosf(th); s[1] = sinf(th); s[2] = rnd(); }
  }
  for (auto& v : u) v = 0.5f * rnd();
  for (auto& v : c) v = 0.1f * rnd();
  for (size_t tb = 0; tb < (size_t)T * B; ++tb)
    for (int i = 0; i < p; ++i) C[(tb * p + i) * p + i] = 1.f;
  Dev<float> dx0(x0.size()), du(u.size()), dx((size_t)T * B * n), dF((size_t)(T - 1) * B * n * p), df((size_t)(T - 1) * B * n),
      dC(C.size()), dc(c.size()), nx((size_t)T * B * n), nu(u.size()), costs(B), fdn(B), al(B);
  dx0.up(x0); du.up(u); dC.up(C); dc.up(c);
  int rc = mpcb200_dyn_rollout_f32(kind, dyn, B, T, dx0.p, du.p, dx.p, nullptr);
  if (rc) return printf("dyn rollout rc=%d\n", rc), 1;
  rc = mpcb200_dyn_linearize_f32(kind, dyn, B, T, dx.p, du.p, dF.p, df.p, nullptr);
  if (rc) return printf("dyn linearize rc=%d\n", rc), 1;
  {  // parameter VJP of the linearisation with (dF, df) = (F, f); second output omitted once
    const int np = kind == MPCB200_DYN_CARTPOLE ? 4 : (kind == MPCB200_DYN_PENDULUM ? 3 : 5);
    Dev<float> first((size_t)(T - 1) * B * np), second((size_t)(T - 1) * B * np);
    rc = mpcb200_dyn_linearize_vjp_f32(kind, dyn, B, T, dx.p, du.p, dF.p, df.p, first.p, second.p, nullptr);
    if (rc) return printf("dyn linearize vjp rc=%d\n", rc), 1;
    rc = mpcb200_dyn_linearize_vjp_f32(kind, dyn, B, T, dx.p, du.p, dF.p, df.p, first.p, nullptr, nullptr);
    if (rc) return printf("dyn linearize vjp (first only) rc=%d\n", rc), 1;
    rc = mpcb200_dyn_linearize_vjp_f32(kind | MPCB200_DYN_CTRL_PASSTHROUGH, dyn, B, T, dx.p, du.p, dF.p, df.p, first.p,
                                       second.p, nullptr);
    if (rc != MPCB200_ERR_BAD_DIMS) return printf("dyn linearize vjp (passthrough) rc=%d\n", rc), 1;
    if (cudaDeviceSynchronize() != cudaSuccess) return printf("CUDA error: %s\n", cudaGetErrorString(cudaGetLastError())), 1;
    int bad = 0;
    for (float v : first.down()) bad += !std::isfinite(v);
    for (float v : second.down()) bad += !std::isfinite(v);
    if (bad) return printf("dyn linearize vjp: nonfinite %d\n", bad), 1;
  }
  mpcb200_dims d = {B, T, n, m, T - 1, 1, 1, 0, 0, 3, 20, 1, kind};
  mpcb200_params prm = {-2.0, 2.0, 0.0, 0.5, {0}};
  for (int i = 0; i < 8; ++i) prm.dyn[i] = dyn[i];
  rc = mpcb200_lqr_step_f32(&d, &prm, dC.p, dc.p, dF.p, df.p, dx0.p, dx.p, du.p, nullptr, nullptr, nullptr, nx.p, nu.p,
                            costs.p, fdn.p, al.p, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr);
  if (rc) return printf("dyn step rc=%d (%s)\n", rc, mpcb200_strerror(rc)), 1;
  if (cudaDeviceSynchronize() != cudaSuccess) return printf("CUDA error: %s\n", cudaGetErrorString(cudaGetLastError())), 1;
  double s = 0;
  int bad = 0;
  for (float v : nx.down()) { s += v; bad += !std::isfinite(v); }
  for (float v : dF.down()) { s += v; bad += !std::isfinite(v); }
  printf("known system %d B=%d T=%d: checksum %.6f nonfinite %d\n", kind, B, T, s, bad);
  return bad != 0;
}

// standalone pnqp above n = 8 (one thread block per QP): f64 box QPs H = L L' / n + I
static int run_pnqp_large(int B, int n) {
  const int max_n = mpcb200_pnqp_max_n(8);
  if (max_n < n) return printf("pnqp max_n(8) = %d < %d\n", max_n, n), 1;
  std::vector<double> L((size_t)n * n), H((size_t)B * n * n), q((size_t)B * n), lo((size_t)B * n, -0.5),
      hi((size_t)B * n, 0.5);
  for (int b = 0; b < B; ++b) {
    for (auto& v : L) v = rnd();
    for (int i = 0; i < n; ++i)
      for (int j = 0; j < n; ++j) {
        double s = i == j ? 1.0 : 0.0;
        for (int k = 0; k < n; ++k) s += L[(size_t)i * n + k] * L[(size_t)j * n + k] / n;
        H[((size_t)b * n + i) * n + j] = s;
      }
  }
  for (auto& v : q) v = 2.0 * rnd();
  Dev<double> dH(H.size()), dq(q.size()), dl(lo.size()), dh(hi.size()), ox(q.size()), oH(H.size());
  Dev<unsigned char> oI(q.size());
  Dev<int> oit(B), ost(B);
  dH.up(H); dq.up(q); dl.up(lo); dh.up(hi);
  int rc = mpcb200_pnqp_f64(B, n, dH.p, dq.p, dl.p, dh.p, nullptr, 20, ox.p, oH.p, oI.p, oit.p, ost.p, nullptr);
  if (rc) return printf("pnqp n=%d rc=%d (%s)\n", n, rc, mpcb200_strerror(rc)), 1;
  rc = mpcb200_pnqp_f64(B, max_n + 1, dH.p, dq.p, dl.p, dh.p, nullptr, 20, ox.p, oH.p, oI.p, oit.p, ost.p, nullptr);
  if (rc != MPCB200_ERR_SMEM) return printf("pnqp n=max_n+1 rc=%d\n", rc), 1;
  Dev<double> gH(H.size()), gq(q.size()), gl(q.size()), gh(q.size());   // the gradient for dL/dx = q
  Dev<int> gst(B);
  rc = mpcb200_pnqp_backward_f64(B, n, dH.p, ox.p, oI.p, dl.p, dh.p, dq.p, gH.p, gq.p, gl.p, gh.p, gst.p, nullptr);
  if (rc) return printf("pnqp backward n=%d rc=%d (%s)\n", n, rc, mpcb200_strerror(rc)), 1;
  if (cudaDeviceSynchronize() != cudaSuccess) return printf("CUDA error: %s\n", cudaGetErrorString(cudaGetLastError())), 1;
  double s = 0;
  int bad = 0;
  for (double v : ox.down()) { s += v; bad += !std::isfinite(v); }
  for (double v : gH.down()) { s += v; bad += !std::isfinite(v); }
  for (int v : ost.down()) bad += v != 0;
  for (int v : gst.down()) bad += v != 0;
  printf("pnqp B=%d n=%d (max_n f32 %d, f64 %d): checksum %.6f bad %d\n", B, n, mpcb200_pnqp_max_n(4), max_n, s, bad);
  return bad != 0;
}

// the slew-rate episode backward's argument checks (they run before anything is launched): the pendulum's
// passthrough kind at its dynamics-only shape (4, 1) takes n_prev = 1 only, and its workspace follows
static int run_episode_backward_slew() {
  mpcb200_dims d = {4, 5, 4, 1, 4, 1, 0, 0, 0, 10, 20, 1, MPCB200_DYN_PENDULUM | MPCB200_DYN_CTRL_PASSTHROUGH};
  mpcb200_params prm = {0.0, 0.0, 0.0, 0.2, {10.0, 1.0, 1.0, 2.0, 0.05}};
  const size_t need = mpcb200_episode_backward_slew_workspace_bytes(&d, 1, 4);
  if (need == 0 || mpcb200_episode_backward_slew_workspace_bytes(&d, 2, 4) != 0)
    return printf("episode backward slew workspace %zu\n", need), 1;
  Dev<float> buf(1024), ws(need / sizeof(float) + 64);
  float* p = buf.p;
  const int rc = mpcb200_episode_backward_slew_f32(&d, &prm, 3, 0, p, p, p, p, p, p, p, p, p, p, p, p, p, p, p, p, p,
                                                   ws.p, need, nullptr);
  if (rc != MPCB200_ERR_BAD_DIMS) return printf("episode backward slew n_prev=0 rc=%d\n", rc), 1;
  printf("episode backward slew: workspace %zu bytes, n_prev=0 refused\n", need);
  return 0;
}

// the plant entries' argument checks (they run before anything is launched): a pendulum model on a cartpole plant is
// refused (the plant steps (5, 1)), and the backward sizes its stage buffer by the five-parameter pendulum plant
static int run_episode_plant() {
  mpcb200_dims d = {4, 5, 3, 1, 4, 1, 0, 0, 0, 10, 20, 1, MPCB200_DYN_PENDULUM};
  mpcb200_params prm = {0.0, 0.0, 0.0, 0.2, {10.0, 1.0, 1.0, 2.0, 0.05}};
  mpcb200_ilqr_opts opts = {5, 5, 1, 0, 1e-7, 1e-4};
  mpcb200_plant cart = {MPCB200_DYN_CARTPOLE, 0, {9.8, 1.0, 0.1, 0.5, 100.0, 0.05}};
  mpcb200_plant full = {MPCB200_DYN_PENDULUM_FULL, 0, {10.0, 1.0, 1.0, 0.3, 0.2, 2.0, 0.05}};
  const size_t need = mpcb200_episode_backward_plant_workspace_bytes(&d, 0, &full, 4);
  if (need == 0 || mpcb200_episode_backward_plant_workspace_bytes(&d, 0, &cart, 4) != 0)
    return printf("episode backward plant workspace %zu\n", need), 1;
  const size_t fw = mpcb200_episode_workspace_bytes(&d, &opts, 4);
  Dev<float> buf(1024), ws((need > fw ? need : fw) / sizeof(float) + 64);
  int32_t* info = (int32_t*)buf.p;
  float* p = buf.p;
  int rc = mpcb200_episode_plant_f32(&d, &prm, &opts, &cart, 3, p, p, p, p, p, p, p, p, p, p, p, nullptr, p, p, p, info,
                                     p, nullptr, nullptr, ws.p, fw, nullptr);
  if (rc != MPCB200_ERR_BAD_DIMS) return printf("episode plant (cartpole plant) rc=%d\n", rc), 1;
  full.kind |= MPCB200_DYN_CTRL_PASSTHROUGH;      // a passthrough plant without a slew-rate penalty
  rc = mpcb200_episode_backward_plant_f32(&d, &prm, &full, 3, 0, p, p, p, p, p, p, p, p, p, p, p, p, p, p, p, p, p, p,
                                          p, p, p, p, ws.p, need, nullptr);
  if (rc != MPCB200_ERR_BAD_DIMS) return printf("episode backward plant (passthrough) rc=%d\n", rc), 1;
  printf("episode plant: backward workspace %zu bytes, other-shape and passthrough plants refused\n", need);
  return 0;
}

// the window entries' argument checks (they run before anything is captured): an axis one slice short and a window
// on a known model's F are refused; the workspace is the episode's plus the window buffers
static int run_episode_window() {
  mpcb200_dims d = {4, 5, 3, 1, 4, 1, 0, 0, 0, 10, 20, 1, MPCB200_DYN_PENDULUM};
  mpcb200_params prm = {0.0, 0.0, 0.0, 0.2, {10.0, 1.0, 1.0, 2.0, 0.05}};
  mpcb200_ilqr_opts opts = {5, 5, 1, 0, 1e-7, 1e-4};
  mpcb200_window win = {};
  win.L = 3 + 5 - 1;
  win.on = MPCB200_WIN_COST;
  const size_t need = mpcb200_episode_window_workspace_bytes(&d, &opts, &win, 4);
  const size_t bw = mpcb200_episode_backward_window_workspace_bytes(&d, 0, &win, nullptr, 4);
  if (need <= mpcb200_episode_workspace_bytes(&d, &opts, 4) || bw == 0)
    return printf("episode window workspace %zu / %zu\n", need, bw), 1;
  Dev<float> buf(4096), ws((need > bw ? need : bw) / sizeof(float) + 64);
  int32_t* info = (int32_t*)buf.p;
  float* p = buf.p;
  win.L -= 1;
  int rc = mpcb200_episode_window_f32(&d, &prm, &opts, &win, nullptr, 3, p, p, nullptr, nullptr, nullptr, nullptr,
                                      nullptr, p, p, nullptr, nullptr, nullptr, p, p, p, info, p, nullptr, nullptr,
                                      ws.p, need, nullptr);
  if (rc != MPCB200_ERR_BAD_DIMS) return printf("episode window (short axis) rc=%d\n", rc), 1;
  win.L += 1;
  win.on |= MPCB200_WIN_DYN;
  rc = mpcb200_episode_backward_window_f32(&d, &prm, &win, nullptr, 3, 0, p, p, p, nullptr, nullptr, nullptr, p, p, p,
                                           p, p, p, p, p, p, nullptr, nullptr, p, nullptr, nullptr, nullptr, nullptr,
                                           ws.p, bw, nullptr);
  if (rc != MPCB200_ERR_BAD_DIMS) return printf("episode backward window (known F) rc=%d\n", rc), 1;
  printf("episode window: workspace %zu / %zu bytes, short axis and known-model F window refused\n", need, bw);
  return 0;
}

// the network entries: a passthrough network with zero weights steps x' = x, so the rollout repeats x_init and the
// linearisation is F = [I 0], f = 0; a network too large for shared memory is refused by mpcb200_mlp_fits
static int run_mlp() {
  const int B = 5, T = 4, n = 3, m = 2, h = 8, p = n + m;
  mpcb200_mlp net = {};
  net.n_layers = 2; net.width[0] = p; net.width[1] = h; net.width[2] = n;
  net.activation = MPCB200_ACT_SIGMOID; net.passthrough = 1;
  net.W_off[0] = 0; net.b_off[0] = h * p; net.W_off[1] = h * p + h; net.b_off[1] = h * p + h + n * h;
  Dev<float> prm(h * p + h + n * h + n), x0(B * n), u(T * B * m), x(T * B * n);
  Dev<float> F((T - 1) * B * n * p), f((T - 1) * B * n);
  prm.up(std::vector<float>(prm.n, 0.f));
  std::vector<float> hx(B * n);
  for (auto& v : hx) v = rnd();
  x0.up(hx);
  u.up(std::vector<float>(u.n, 0.5f));
  net.params = prm.p;
  if (!mpcb200_mlp_fits(&net, 4)) return printf("mlp: small network does not fit\n"), 1;
  int rc = mpcb200_mlp_rollout_f32(&net, B, T, n, m, x0.p, u.p, x.p, nullptr);
  if (rc == 0) rc = mpcb200_mlp_linearize_f32(&net, B, T, n, m, x.p, u.p, F.p, f.p, nullptr);
  if (rc != 0 || cudaDeviceSynchronize() != cudaSuccess) return printf("mlp rollout / linearize rc=%d\n", rc), 1;
  int bad = 0;
  const auto gx = x.down(), gF = F.down(), gf = f.down();
  for (int i = 0; i < T * B * n; ++i) bad += gx[i] != hx[i % (B * n)];
  for (int i = 0; i < (T - 1) * B * n * p; ++i) {
    const int c = i % p, r = (i / p) % n;
    bad += gF[i] != (c == r ? 1.f : 0.f);
  }
  for (float v : gf) bad += v != 0.f;
  // the VJP with dF = 0, df = 1: every hidden output is sigmoid(0) = 1/2 and every tangent 0, so only the last layer
  // has a gradient, db_1 = (T-1) B and dW_1 = (T-1) B / 2
  const size_t vws = mpcb200_mlp_linearize_vjp_workspace_bytes(&net, B, T, 4);
  Dev<float> dF((T - 1) * B * n * p), df((T - 1) * B * n), dth(prm.n), vw(vws / sizeof(float) + 64);
  dF.up(std::vector<float>(dF.n, 0.f));
  df.up(std::vector<float>(df.n, 1.f));
  rc = vws == 0 ? -1 : mpcb200_mlp_linearize_vjp_f32(&net, B, T, n, m, x.p, u.p, dF.p, df.p, dth.p, vw.p, vws, nullptr);
  if (rc != 0 || cudaDeviceSynchronize() != cudaSuccess) return printf("mlp linearize vjp rc=%d\n", rc), 1;
  const auto gth = dth.down();
  for (int i = 0; i < (int)prm.n; ++i)
    bad += gth[i] != (i >= net.b_off[1] ? (T - 1) * B : i >= net.W_off[1] ? 0.5f * (T - 1) * B : 0.f);
  mpcb200_mlp big = net;
  big.n_layers = 3; big.width[1] = big.width[2] = 256; big.width[3] = n;
  big.W_off[1] = 256 * p + 256; big.b_off[1] = big.W_off[1] + 256 * 256;
  big.W_off[2] = big.b_off[1] + 256; big.b_off[2] = big.W_off[2] + 256 * n;
  if (mpcb200_mlp_fits(&big, 4)) ++bad;
  printf("mlp: rollout, linearisation and its VJP of x' = x, %d bad; [256, 256] refused by mpcb200_mlp_fits\n", bad);
  return bad != 0;
}

// the network episode entries: the zero-weight passthrough network steps x' = x, so with C = I, c = 0 every plan is
// u = 0 and the episode holds x_init; its reverse sweep with dl_dx = 0, dl_du = 0 gives zero gradients.  T < 3 and a
// network too large for shared memory are refused before anything is captured.
static int run_episode_mlp() {
  const int B = 3, T = 4, n = 3, m = 2, h = 8, p = n + m, steps = 3;
  mpcb200_mlp net = {};
  net.n_layers = 2; net.width[0] = p; net.width[1] = h; net.width[2] = n;
  net.activation = MPCB200_ACT_SIGMOID; net.passthrough = 1;
  net.W_off[0] = 0; net.b_off[0] = h * p; net.W_off[1] = h * p + h; net.b_off[1] = h * p + h + n * h;
  const int np = h * p + h + n * h + n;
  Dev<float> prm(np), C(T * B * p * p), c(T * B * p), x0(B * n), u0(T * B * m), xs((steps + 1) * B * n),
      us(steps * B * m), costs(steps * B), info(2 * steps), un(T * B * m), px(steps * T * B * n), pu(steps * T * B * m);
  prm.up(std::vector<float>(np, 0.f));
  std::vector<float> hC(C.n, 0.f), hx(B * n);
  for (int i = 0; i < T * B; ++i)
    for (int j = 0; j < p; ++j) hC[(size_t)i * p * p + j * p + j] = 1.f;
  for (auto& v : hx) v = rnd();
  C.up(hC); c.up(std::vector<float>(c.n, 0.f)); x0.up(hx); u0.up(std::vector<float>(u0.n, 0.f));
  net.params = prm.p;
  mpcb200_dims d = {B, T, n, m, T - 1, 0, 0, 0, 0, 10, 20, 1, 0};
  mpcb200_params pr = {0.0, 0.0, 0.0, 0.2, {}};
  mpcb200_ilqr_opts opts = {5, 5, m, 0, 1e-7, 1e-4};
  const size_t fw = mpcb200_episode_mlp_workspace_bytes(&d, &opts, &net, 4);
  const size_t bw = mpcb200_episode_backward_mlp_workspace_bytes(&d, &net, nullptr, 4);
  if (fw == 0 || bw == 0) return printf("episode mlp workspace %zu / %zu\n", fw, bw), 1;
  Dev<float> ws((fw > bw ? fw : bw) / sizeof(float) + 64);
  int rc = mpcb200_episode_mlp_f32(&d, &pr, &opts, &net, nullptr, steps, C.p, c.p, nullptr, nullptr, nullptr, x0.p,
                                   u0.p, nullptr, nullptr, nullptr, xs.p, us.p, costs.p, (int32_t*)info.p, un.p, px.p,
                                   pu.p, ws.p, fw, nullptr);
  if (rc != 0 || cudaDeviceSynchronize() != cudaSuccess) return printf("episode mlp rc=%d\n", rc), 1;
  int bad = 0;
  const auto gx = xs.down(), gu = us.down();
  for (int i = 0; i < (steps + 1) * B * n; ++i) bad += gx[i] != hx[i % (B * n)];
  for (float v : gu) bad += v != 0.f;
  Dev<float> gxs((steps + 1) * B * n), gus(steps * B * m), dx(B * n), dC(T * B * p * p), dc(T * B * p), dth(np);
  gxs.up(std::vector<float>(gxs.n, 0.f)); gus.up(std::vector<float>(gus.n, 0.f));
  rc = mpcb200_episode_backward_mlp_f32(&d, &pr, &net, nullptr, steps, C.p, c.p, nullptr, nullptr, nullptr, xs.p, us.p,
                                        px.p, pu.p, gxs.p, gus.p, dx.p, dC.p, dc.p, dth.p, nullptr, nullptr, nullptr,
                                        nullptr, ws.p, bw, nullptr);
  if (rc != 0 || cudaDeviceSynchronize() != cudaSuccess) return printf("episode backward mlp rc=%d\n", rc), 1;
  for (float v : dth.down()) bad += v != 0.f;
  for (float v : dx.down()) bad += v != 0.f;
  mpcb200_dims d2 = d;
  d2.T = 2;
  rc = mpcb200_episode_mlp_f32(&d2, &pr, &opts, &net, nullptr, steps, C.p, c.p, nullptr, nullptr, nullptr, x0.p, u0.p,
                               nullptr, nullptr, nullptr, xs.p, us.p, costs.p, (int32_t*)info.p, un.p, nullptr,
                               nullptr, ws.p, fw, nullptr);
  bad += rc != MPCB200_ERR_BAD_DIMS;
  mpcb200_mlp big = net;
  big.n_layers = 3; big.width[1] = big.width[2] = 256; big.width[3] = n;
  big.W_off[1] = 256 * p + 256; big.b_off[1] = big.W_off[1] + 256 * 256;
  big.W_off[2] = big.b_off[1] + 256; big.b_off[2] = big.W_off[2] + 256 * n;
  rc = mpcb200_episode_backward_mlp_f32(&d, &pr, &big, nullptr, steps, C.p, c.p, nullptr, nullptr, nullptr, xs.p, us.p,
                                        px.p, pu.p, gxs.p, gus.p, dx.p, dC.p, dc.p, dth.p, nullptr, nullptr, nullptr,
                                        nullptr, ws.p, bw, nullptr);
  bad += rc != MPCB200_ERR_SMEM;
  printf("episode mlp: x' = x held, zero gradients, %d bad; T < 3 and [256, 256] refused\n", bad);
  return bad != 0;
}

int main() {
  int fails = 0;
  fails += run_mlp();
  fails += run_episode_mlp();
  fails += run_episode_backward_slew();
  fails += run_episode_plant();
  fails += run_episode_window();
  fails += run_pnqp_large(3, 100);
  fails += run_dyn(MPCB200_DYN_CARTPOLE, 37, 9);
  fails += run_dyn(MPCB200_DYN_PENDULUM, 20, 7);
  fails += run_dyn(MPCB200_DYN_PENDULUM_FULL, 20, 7);
  const int cases[][6] = {{13, 6, 8, 2, 0, 0}, {13, 6, 8, 2, 1, 0}, {12, 5, 8, 2, 2, 1}, {7, 4, 3, 1, 1, 0},
                          {5, 4, 16, 4, 2, 0}, {1, 3, 2, 2, 0, 0}, {33, 7, 5, 1, 1, 1}, {9, 3, 3, 4, 2, 0},
                          {64, 40, 8, 2, 1, 0}, {16, 6, 4, 2, 1, 0}, {12, 5, 16, 4, 0, 0}, {24, 6, 8, 2, 2, 1},
                          {20, 9, 8, 4, 1, 0}};
  for (auto& cs : cases) fails += run_case(cs[0], cs[1], cs[2], cs[3], cs[4], cs[5]);
  printf("launches: %llu, failures: %d\n", (unsigned long long)mpcb200_launch_count(), fails);
  return fails;
}
