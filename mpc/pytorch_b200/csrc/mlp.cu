// mlp.cu - the learned model's kernels (mlp.cuh): rollout, exact linearisation and the split-mode line search.
// The network and its Jacobian chain follow the reference's NNDynamics (mpc/dynamics.py:15-131) as models.py
// states them; the line search follows lqr_forward (mpc/lqr_step.py:164-261) as step.rollout_split runs it.
#include <math.h>

#include "common.cuh"
#include "mlp.cuh"

namespace mpcb200 {

bool mlp_shape(const mpcb200_mlp* rec, MlpShape& s) {
  if (rec == nullptr || rec->params == nullptr) return false;
  const int L = rec->n_layers;
  if (L < 1 || L > MPCB200_MLP_MAX_LAYERS) return false;
  if (rec->activation < MPCB200_ACT_SIGMOID || rec->activation > MPCB200_ACT_ELU) return false;
  s.L = L; s.act = rec->activation; s.passthrough = rec->passthrough ? 1 : 0; s.maxw = 0;
  for (int i = 0; i <= L; ++i) {
    const int w = rec->width[i];
    if (w < 1 || w > MPCB200_MLP_MAX_WIDTH) return false;
    s.w[i] = w;
    if (w > s.maxw) s.maxw = w;
  }
  s.ns = s.w[L];
  s.ms = s.w[0] - s.ns;
  if (s.ms < 1) return false;
  s.n_prev = rec->n_prev;
  if (s.n_prev != 0 && s.n_prev != s.ms) return false;
  s.n_params = 0;
  for (int i = 0; i < L; ++i) {
    if (rec->W_off[i] < 0 || rec->b_off[i] < 0) return false;
    s.W_off[i] = rec->W_off[i]; s.b_off[i] = rec->b_off[i];
    const long long we = s.W_off[i] + (long long)s.w[i + 1] * s.w[i], be = s.b_off[i] + s.w[i + 1];
    if (we > s.n_params) s.n_params = we;
    if (be > s.n_params) s.n_params = be;
  }
  if (s.n_params > (1ll << 24)) return false;
  // linearisation: input, hidden outputs and output of the forward pass, then two Jacobian blocks [n_s, maxw];
  // rollout / line search: two activation buffers and the staged state and control
  int hidden = 0;
  for (int i = 1; i < L; ++i) hidden += s.w[i];
  const int lin = s.w[0] + hidden + s.ns + (L > 1 ? 2 * s.ns * s.maxw : 0);
  s.p_max = s.n_prev + s.w[0] + MPCB200_MLP_PAD_SLACK;
  const int ls = 2 * s.maxw + s.p_max;
  s.per_warp = round_up(lin > ls ? lin : ls, 4);
  return true;
}

size_t mlp_smem_bytes(const MlpShape& s, int elem_size, int warps) {
  const size_t params = ((size_t)s.n_params * elem_size + 15) / 16 * 16;
  return 16 + params + (size_t)warps * s.per_warp * elem_size;
}

namespace {

MPCB_DEV float mlp_exp(float v) { return expf(v); }
MPCB_DEV double mlp_exp(double v) { return exp(v); }
MPCB_DEV float mlp_expm1(float v) { return expm1f(v); }
MPCB_DEV double mlp_expm1(double v) { return expm1(v); }

template <typename R>
MPCB_DEV R act_apply(int act, R z) {
  if (act == MPCB200_ACT_SIGMOID) return R(1) / (R(1) + mlp_exp(-z));
  if (act == MPCB200_ACT_RELU) return z > R(0) ? z : R(0);
  return z > R(0) ? z : mlp_expm1(z);
}
// d act / d pre-activation from the post-activation value a (models._act_slope)
template <typename R>
MPCB_DEV R act_slope(int act, R a) {
  if (act == MPCB200_ACT_SIGMOID) return a * (R(1) - a);
  if (act == MPCB200_ACT_RELU) return a > R(0) ? R(1) : R(0);
  return a > R(0) ? R(1) : a + R(1);
}

// d^2 act / d pre-activation^2 from the post-activation value a: the derivative of act_slope through a
template <typename R>
MPCB_DEV R act_curv(int act, R a) {
  if (act == MPCB200_ACT_SIGMOID) return a * (R(1) - a) * (R(1) - R(2) * a);
  if (act == MPCB200_ACT_RELU) return R(0);
  return a > R(0) ? R(0) : a + R(1);
}

template <typename R>
MPCB_DEV R warp_sum(R v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;    // the butterfly adds the same pairs in every lane: every lane holds the same value
}

// out[j] = act(sum_k W[j,k] in[k] + b[j]) for j < w_out (act < 0: linear), by one warp.  A layer with few outputs
// splits each dot product over the lanes (butterfly sum); otherwise each lane owns outputs.  The choice and the
// order of every sum depend on the widths alone.
template <typename R>
MPCB_DEV void mlp_layer(const R* W, const R* b, const R* in, R* out, int w_in, int w_out, int act, int lane) {
  const int per_lane = (w_out + 31) / 32 * w_in, split = w_out * ((w_in + 31) / 32 + 5);
  if (split < per_lane) {
    for (int j = 0; j < w_out; ++j) {
      R acc = R(0);
      for (int k = lane; k < w_in; k += 32) acc = fma(W[(size_t)j * w_in + k], in[k], acc);
      acc = warp_sum(acc) + b[j];
      if (lane == 0) out[j] = act >= 0 ? act_apply(act, acc) : acc;
    }
  } else {
    for (int j = lane; j < w_out; j += 32) {
      const R* row = W + (size_t)j * w_in;
      R acc = R(0);
      for (int k = 0; k < w_in; ++k) acc = fma(row[k], in[k], acc);
      acc += b[j];
      out[j] = act >= 0 ? act_apply(act, acc) : acc;
    }
  }
  __syncwarp();
}

// The network on z (w[0] values in `a`), ping-ponging between a and b2; returns the buffer holding its n_s outputs.
template <typename R>
MPCB_DEV R* mlp_forward(const MlpShape& s, const R* prm, R* a, R* b2, int lane) {
  R* in = a;
  R* out = b2;
  for (int i = 0; i < s.L; ++i) {
    mlp_layer(prm + s.W_off[i], prm + s.b_off[i], in, out, s.w[i], s.w[i + 1], i + 1 < s.L ? s.act : -1, lane);
    R* t = in; in = out; out = t;
  }
  return in;
}

// z = [x[n_prev : n_prev + n_s]; u[0 : m_s]] into `z`
template <typename R>
MPCB_DEV void mlp_input(const MlpShape& s, const R* x, const R* u, R* z, int lane) {
  for (int i = lane; i < s.w[0]; i += 32) z[i] = i < s.ns ? x[s.n_prev + i] : u[i - s.ns];
  __syncwarp();
}

// x <- step(x, u) in place: [u[0:n_prev]; MLP(z) (+ x with passthrough); 0 ...] over the N staged states
template <typename R>
MPCB_DEV void mlp_advance(const MlpShape& s, const R* out, const R* u, R* x, int N, int lane) {
  for (int i = lane; i < N; i += 32) {
    R v = R(0);
    if (i < s.n_prev) v = u[i];
    else if (i < s.n_prev + s.ns) v = s.passthrough ? x[i] + out[i - s.n_prev] : out[i - s.n_prev];
    x[i] = v;
  }
  __syncwarp();
}

// Stages elements [0, n_params) of the parameter block into `dst` (16-byte aligned): one 1-D bulk copy of the
// 16-byte multiple when the source is aligned, the block's threads for the rest.  Ends with the block synchronised.
template <typename R>
MPCB_DEV void stage_params(const MlpShape& s, const R* src, R* dst, uint64_t* bar) {
  const size_t bytes = (size_t)s.n_params * sizeof(R);
  const bool bulk = (reinterpret_cast<uintptr_t>(src) & 15u) == 0;
  const size_t head = bulk ? bytes / 16 * 16 : 0;
  if (threadIdx.x == 0 && head > 0) {
    mbar_init(bar, 1);
    mbar_fence_init();
    mbar_arrive_expect_tx(bar, (uint32_t)head);
    bulk_g2s(dst, src, (uint32_t)head, bar);
  }
  for (size_t i = head / sizeof(R) + threadIdx.x; i < (size_t)s.n_params; i += blockDim.x) dst[i] = src[i];
  __syncthreads();
  if (head > 0) mbar_wait(bar, 0);
}

// the CTA's shared memory: mbarrier, parameters, then one slice per warp
template <typename R>
struct MlpSmem {
  uint64_t* bar;
  R* prm;
  R* mine;
};
template <typename R>
MPCB_DEV MlpSmem<R> carve(const MlpShape& s, unsigned char* smem, int warp) {
  MlpSmem<R> m;
  m.bar = reinterpret_cast<uint64_t*>(smem);
  m.prm = reinterpret_cast<R*>(smem + 16);
  const size_t params = ((size_t)s.n_params * sizeof(R) + 15) / 16 * 16;
  m.mine = reinterpret_cast<R*>(smem + 16 + params) + (size_t)warp * s.per_warp;
  return m;
}

extern __shared__ __align__(16) unsigned char mlp_smem[];

template <typename R>
__global__ void __launch_bounds__(256, 1)
mlp_rollout_kernel(const __grid_constant__ MlpShape s, const R* __restrict__ params, int B, int T, int N, int M,
                   const R* __restrict__ x_init, const R* __restrict__ u, R* __restrict__ x) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const MlpSmem<R> sm = carve<R>(s, mlp_smem, warp);
  stage_params(s, params, sm.prm, sm.bar);
  R* a = sm.mine;
  R* b2 = a + s.maxw;
  R* X = b2 + s.maxw;
  for (int b = blockIdx.x * wpb + warp; b < B; b += gridDim.x * wpb) {
    for (int i = lane; i < N; i += 32) {
      const R v = x_init[(size_t)b * N + i];
      X[i] = v;
      x[(size_t)b * N + i] = v;
    }
    __syncwarp();
    for (int t = 0; t + 1 < T; ++t) {
      const R* ut = u + ((size_t)t * B + b) * M;
      mlp_input(s, X, ut, a, lane);
      const R* out = mlp_forward(s, sm.prm, a, b2, lane);
      for (int i = lane; i < N; i += 32) {
        R v = R(0);
        if (i < s.n_prev) v = ut[i];
        else if (i < s.n_prev + s.ns) v = s.passthrough ? X[i] + out[i - s.n_prev] : out[i - s.n_prev];
        X[i] = v;
        x[((size_t)(t + 1) * B + b) * N + i] = v;
      }
      __syncwarp();
    }
  }
}

template <typename R>
__global__ void __launch_bounds__(256, 1)
mlp_linearize_kernel(const __grid_constant__ MlpShape s, const R* __restrict__ params, int B, int T, int N, int M,
                     const R* __restrict__ x, const R* __restrict__ u, R* __restrict__ F, R* __restrict__ f) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const MlpSmem<R> sm = carve<R>(s, mlp_smem, warp);
  stage_params(s, params, sm.prm, sm.bar);
  const int L = s.L, ns = s.ns, P = N + M;
  // z | hidden outputs h_1 .. h_{L-1} | output | J ping | J pong
  R* z = sm.mine;
  R* hid = z + s.w[0];
  R* out = hid;
  for (int i = 1; i < L; ++i) out += s.w[i];
  R* J0 = out + ns;
  R* J1 = J0 + (size_t)ns * s.maxw;
  const int items = (T - 1) * B;
  for (int it = blockIdx.x * wpb + warp; it < items; it += gridDim.x * wpb) {
    const int t = it / B, b = it - t * B;
    const R* xt = x + ((size_t)t * B + b) * N;
    const R* ut = u + ((size_t)t * B + b) * M;
    mlp_input(s, xt, ut, z, lane);
    // forward pass keeping every hidden output
    const R* in = z;
    R* h = hid;
    for (int i = 0; i < L; ++i) {
      R* o = i + 1 < L ? h : out;
      mlp_layer(sm.prm + s.W_off[i], sm.prm + s.b_off[i], in, o, s.w[i], s.w[i + 1], i + 1 < L ? s.act : -1, lane);
      in = o;
      if (i + 1 < L) h += s.w[i + 1];
    }
    // J = W_{L-1}; J <- (J * act'(h_i)) @ W_{i-1} for i = L-1 .. 1 (models.NNDynamics.grad_input)
    const R* J = sm.prm + s.W_off[L - 1];
    int wj = s.w[L - 1];
    R* hi = out;
    R* dst = J0;
    for (int i = L - 1; i >= 1; --i) {
      hi -= s.w[i];
      const R* W = sm.prm + s.W_off[i - 1];
      const int wn = s.w[i - 1];
      for (int e = lane; e < ns * wn; e += 32) {
        const int r = e / wn, c = e % wn;
        R acc = R(0);
        for (int k = 0; k < wj; ++k)
          acc = fma(J[(size_t)r * wj + k] * act_slope(s.act, hi[k]), W[(size_t)k * wn + c], acc);
        dst[e] = acc;
      }
      __syncwarp();
      J = dst;
      wj = wn;
      dst = dst == J0 ? J1 : J0;
    }
    // F = [R S] at the staged shape, f = x' - R x - S u
    R* Ft = F + ((size_t)t * B + b) * N * P;
    for (int e = lane; e < N * P; e += 32) {
      const int i = e / P, c = e % P;
      R v = R(0);
      if (i < s.n_prev) {
        v = c == N + i ? R(1) : R(0);
      } else if (i < s.n_prev + ns) {
        const int r = i - s.n_prev;
        if (c >= s.n_prev && c < s.n_prev + ns)
          v = J[(size_t)r * wj + (c - s.n_prev)] + (s.passthrough && c == i ? R(1) : R(0));
        else if (c >= N && c < N + s.ms) v = J[(size_t)r * wj + ns + (c - N)];
      }
      Ft[e] = v;
    }
    R* ft = f + ((size_t)t * B + b) * N;
    for (int i = lane; i < N; i += 32) {
      R v = R(0);
      if (i >= s.n_prev && i < s.n_prev + ns) {
        const int r = i - s.n_prev;
        const R* Jr = J + (size_t)r * wj;
        R rx = R(0), su = R(0);
        for (int c = 0; c < ns; ++c) rx = fma(Jr[c] + (s.passthrough && c == r ? R(1) : R(0)), xt[s.n_prev + c], rx);
        for (int k = 0; k < s.ms; ++k) su = fma(Jr[ns + k], ut[k], su);
        const R xn = s.passthrough ? xt[i] + out[r] : out[r];
        v = xn - rx - su;
      }
      ft[i] = v;
    }
    __syncwarp();
  }
}

// 0.5 tau' C tau + c' tau of one time step, by one warp (rows over the lanes, butterfly sums); every lane returns it
template <typename R>
MPCB_DEV R stage_cost(const R* C, const R* c, const R* X, const R* U, int N, int P, int lane) {
  R quad = R(0), lin = R(0);
  for (int i = lane; i < P; i += 32) {
    const R* row = C + (size_t)i * P;
    R ci = R(0);
    for (int j = 0; j < P; ++j) ci = fma(row[j], j < N ? X[j] : U[j - N], ci);
    const R ti = i < N ? X[i] : U[i - N];
    quad = fma(ti, ci, quad);
    lin = fma(ti, c[i], lin);
  }
  return R(0.5) * warp_sum(quad) + warp_sum(lin);
}

template <typename R>
__global__ void __launch_bounds__(256, 1)
mlp_linesearch_kernel(const __grid_constant__ MlpShape s, const R* __restrict__ params,
                      const __grid_constant__ MlpLsArgs<R> a) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const MlpSmem<R> sm = carve<R>(s, mlp_smem, warp);
  stage_params(s, params, sm.prm, sm.bar);
  const int B = a.B, T = a.T, N = a.N, M = a.M, P = N + M;
  R* z = sm.mine;
  R* z2 = z + s.maxw;
  R* X = z2 + s.maxw;
  R* U = X + N;
  for (int b = blockIdx.x * wpb + warp; b < B; b += gridDim.x * wpb) {
    // the cost of the nominal trajectory
    R old = R(0);
    for (int t = 0; t < T; ++t) {
      const size_t tb = (size_t)t * B + b;
      for (int i = lane; i < N; i += 32) X[i] = a.cur_x[tb * N + i];
      for (int j = lane; j < M; j += 32) U[j] = a.cur_u[tb * M + j];
      __syncwarp();
      old += stage_cost(a.C + t * a.C_ts + (size_t)b * P * P, a.c + t * a.c_ts + (size_t)b * P, X, U, N, P, lane);
      __syncwarp();
    }
    R alpha = R(1), cost = R(0);
    for (int pass = 0; pass < a.max_ls; ++pass) {
      for (int i = lane; i < N; i += 32) X[i] = a.x_init[(size_t)b * N + i];
      __syncwarp();
      cost = R(0);
      for (int t = 0; t < T; ++t) {
        const size_t tb = (size_t)t * B + b;
        for (int j = lane; j < M; j += 32) {
          const R* K = a.Ks + (tb * M + j) * N;
          const R* xb = a.cur_x + tb * N;
          R kx = R(0);
          for (int i = 0; i < N; ++i) kx = fma(K[i], X[i] - xb[i], kx);
          const R cu = a.cur_u[tb * M + j];
          R v = kx + cu + alpha * a.ks[tb * M + j];
          if (a.has_mask && a.zero_mask[tb * M + j] != 0) v = R(0);
          if (a.bounds_kind != 0) {
            R lo = a.bounds_kind == 1 ? a.u_lo : a.u_lower[tb * M + j];
            R hi = a.bounds_kind == 1 ? a.u_hi : a.u_upper[tb * M + j];
            if (a.has_delta) {
              lo = fmax(cu - a.delta_u, lo);
              hi = fmin(cu + a.delta_u, hi);
            }
            if (v < lo) v = lo;              // util.eclamp order: lower, then upper
            if (v > hi) v = hi;
          }
          U[j] = v;
          a.new_u[tb * M + j] = v;
          if (pass == 0 && a.du_first != nullptr) a.du_first[tb * M + j] = cu - v;
        }
        __syncwarp();
        for (int i = lane; i < N; i += 32) a.new_x[tb * N + i] = X[i];
        cost += stage_cost(a.C + t * a.C_ts + (size_t)b * P * P, a.c + t * a.c_ts + (size_t)b * P, X, U, N, P, lane);
        if (t + 1 < T) {
          mlp_input(s, X, U, z, lane);
          const R* out = mlp_forward(s, sm.prm, z, z2, lane);
          mlp_advance(s, out, U, X, N, lane);
        } else {
          __syncwarp();
        }
      }
      if (!(cost > old)) break;            // not worse: another pass would repeat these numbers
      alpha = alpha * a.decay;
      if (pass + 1 == a.max_ls) alpha = alpha / a.decay;  // a last pass still worse: lqr_step.py:252
    }
    if (lane == 0) {
      a.costs[b] = cost;
      a.alphas[b] = alpha;
    }
  }
}

// The VJP of mlp_linearize_kernel's (F, f) in the parameters, per item reverse over forward with matrix tangents
// (mlp.cuh).  Warp w serves the slots w, w + warps, ...; slot g runs the items g, g + G, ... in increasing order and
// adds each item's gradient into its own workspace row ws[g], every element of it always by the same lane.  s is the
// shape of mlp_vjp_shape (its per_warp is this kernel's slice).
template <typename R>
__global__ void __launch_bounds__(256, 1)
mlp_linearize_vjp_kernel(const __grid_constant__ MlpShape s, const R* __restrict__ params, int B, int T, int N, int M,
                         const R* __restrict__ x, const R* __restrict__ u, const R* __restrict__ dF,
                         const R* __restrict__ df, int G, R* __restrict__ ws) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, wpb = blockDim.x >> 5;
  const MlpSmem<R> sm = carve<R>(s, mlp_smem, warp);
  stage_params(s, params, sm.prm, sm.bar);
  const int L = s.L, ns = s.ns, p = s.w[0], P = N + M;
  int hidden = 0;
  for (int i = 1; i < L; ++i) hidden += s.w[i];
  // z | hidden outputs h_1 .. h_{L-1} | tangents T_1 .. T_{L-1} [w_i, p] | adjoints X, Y [maxw, p] | hx, hy [maxw]
  R* z = sm.mine;
  R* hid = z + p;
  R* tan = hid + hidden;
  R* X = tan + (size_t)hidden * p;
  R* Y = X + (size_t)s.maxw * p;
  R* hx = Y + (size_t)s.maxw * p;
  R* hy = hx + s.maxw;
  const long long items = (long long)(T - 1) * B;
  for (int g = blockIdx.x * wpb + warp; g < G; g += gridDim.x * wpb) {
    R* row = ws + (size_t)g * s.n_params;
    for (long long e = lane; e < s.n_params; e += 32) row[e] = R(0);
    __syncwarp();
    for (long long it = g; it < items; it += G) {
      const int t = (int)(it / B), b = (int)(it - (long long)t * B);
      const size_t tb = (size_t)t * B + b;
      mlp_input(s, x + tb * N, u + tb * M, z, lane);
      // forward: h_{i+1} = act(W_i h_i + b_i), T_{i+1} = diag(act'(h_{i+1})) W_i T_i, T_0 = I (Ti == nullptr)
      const R* hin = z;
      const R* Tin = nullptr;
      R* ho = hid;
      R* To = tan;
      for (int i = 0; i + 1 < L; ++i) {
        const R* W = sm.prm + s.W_off[i];
        const int wi = s.w[i], wo = s.w[i + 1];
        mlp_layer(W, sm.prm + s.b_off[i], hin, ho, wi, wo, s.act, lane);
        for (int e = lane; e < wo * p; e += 32) {
          const int r = e / p, c = e - r * p;
          R acc = R(0);
          if (Tin == nullptr) acc = W[(size_t)r * wi + c];
          else
            for (int k = 0; k < wi; ++k) acc = fma(W[(size_t)r * wi + k], Tin[(size_t)k * p + c], acc);
          To[e] = act_slope(s.act, ho[r]) * acc;
        }
        __syncwarp();
        hin = ho; Tin = To;
        ho += wo; To += (size_t)wo * p;
      }
      // seeds: X = G^ = dJ - df z^T and hx = df, the network's rows and columns of dF and df
      const R* dFt = dF + tb * N * P;
      const R* dft = df + tb * N + s.n_prev;
      for (int e = lane; e < ns * p; e += 32) {
        const int r = e / p, c = e - r * p;
        const R* dr = dFt + (size_t)(s.n_prev + r) * P;
        X[e] = (c < ns ? dr[s.n_prev + c] : dr[N + c - ns]) - dft[r] * z[c];
      }
      for (int r = lane; r < ns; r += 32) hx[r] = dft[r];
      __syncwarp();
      // reverse: layer i with X = the adjoint of its output tangent, hx = that of its output
      const R* hout = nullptr;
      for (int i = L - 1; i >= 0; --i) {
        const R* W = sm.prm + s.W_off[i];
        const int wi = s.w[i], wo = s.w[i + 1];
        if (i + 1 < L) {
          // a hidden layer: s^bar = rowsum(X .* A_i) with A_i = W_i T_i (Y holds the products),
          // a^bar = h^bar .* act' + s^bar .* act'' into hx, A^bar = diag(act') X into X
          if (s.act != MPCB200_ACT_RELU) {
            for (int e = lane; e < wo * p; e += 32) {
              const int r = e / p, c = e - r * p;
              R acc = R(0);
              if (Tin == nullptr) acc = W[(size_t)r * wi + c];
              else
                for (int k = 0; k < wi; ++k) acc = fma(W[(size_t)r * wi + k], Tin[(size_t)k * p + c], acc);
              Y[e] = X[e] * acc;
            }
            __syncwarp();
          }
          for (int r = lane; r < wo; r += 32) {
            R sb = R(0);
            if (s.act != MPCB200_ACT_RELU)
              for (int c = 0; c < p; ++c) sb += Y[(size_t)r * p + c];
            hx[r] = hx[r] * act_slope(s.act, hout[r]) + sb * act_curv(s.act, hout[r]);
          }
          for (int e = lane; e < wo * p; e += 32) X[e] *= act_slope(s.act, hout[e / p]);
          __syncwarp();
        }
        // dW_i += X T_i^T + hx h_i^T, db_i += hx
        R* dW = row + s.W_off[i];
        for (int e = lane; e < wo * wi; e += 32) {
          const int r = e / wi, k = e - r * wi;
          R v = R(0);
          if (Tin == nullptr) v = X[(size_t)r * p + k];
          else
            for (int c = 0; c < p; ++c) v = fma(X[(size_t)r * p + c], Tin[(size_t)k * p + c], v);
          dW[e] += fma(hx[r], hin[k], v);
        }
        R* db = row + s.b_off[i];
        for (int r = lane; r < wo; r += 32) db[r] += hx[r];
        if (i > 0) {
          // the adjoints of layer i's input: Y = W_i^T X, hy = W_i^T hx
          for (int e = lane; e < wi * p; e += 32) {
            const int k = e / p, c = e - k * p;
            R acc = R(0);
            for (int r = 0; r < wo; ++r) acc = fma(W[(size_t)r * wi + k], X[(size_t)r * p + c], acc);
            Y[e] = acc;
          }
          for (int k = lane; k < wi; k += 32) {
            R acc = R(0);
            for (int r = 0; r < wo; ++r) acc = fma(W[(size_t)r * wi + k], hx[r], acc);
            hy[k] = acc;
          }
          __syncwarp();
          R* t = X; X = Y; Y = t;
          t = hx; hx = hy; hy = t;
          hout = hin;
          hin = i == 1 ? z : hin - s.w[i - 1];
          Tin = i == 1 ? nullptr : Tin - (size_t)s.w[i - 1] * p;
        }
      }
      __syncwarp();
    }
  }
}

// dtheta[e] = sum of ws[g][e] over the slots g = 0 .. G-1, in that order
template <typename R>
__global__ void __launch_bounds__(256)
mlp_vjp_reduce_kernel(const R* __restrict__ ws, int G, long long n_params, R* __restrict__ dtheta) {
  for (long long e = blockIdx.x * (long long)blockDim.x + threadIdx.x; e < n_params;
       e += (long long)gridDim.x * blockDim.x) {
    R acc = ws[e];
    for (int g = 1; g < G; ++g) acc += ws[(size_t)g * n_params + e];
    dtheta[e] = acc;
  }
}

// warps per CTA: up to 8, as many as the opt-in shared memory holds, no more than there are items
int mlp_warps(const MlpShape& s, int elem_size, long long items, int smem_optin) {
  int w = 8;
  while (w > 1 && ((long long)w > items || mlp_smem_bytes(s, elem_size, w) > (size_t)smem_optin)) --w;
  return w;
}

template <auto Kern>
int mlp_prepare(const MlpShape& s, int elem_size, long long items, int& warps, int& grid, size_t& smem) {
  const int optin = max_smem_optin();
  if (optin <= 0) return MPCB200_ERR_NO_DEVICE;
  warps = mlp_warps(s, elem_size, items, optin);
  smem = mlp_smem_bytes(s, elem_size, warps);
  if (smem > (size_t)optin) return MPCB200_ERR_SMEM;
  if (const int rc = allow_smem_optin<Kern>(optin)) return rc;
  const long long g = (items + warps - 1) / warps;
  grid = (int)(g < 1024 ? g : 1024);
  return MPCB200_OK;
}

int launched() { return cudaGetLastError() == cudaSuccess ? MPCB200_OK : MPCB200_ERR_LAUNCH; }

}  // namespace

template <typename R>
int mlp_launch_rollout(const mpcb200_mlp* rec, int B, int T, int N, int M, const R* x_init, const R* u, R* x,
                       cudaStream_t stream) {
  MlpShape s;
  if (!mlp_shape(rec, s)) return MPCB200_ERR_BAD_DIMS;
  int warps, grid;
  size_t smem;
  if (const int rc = mlp_prepare<mlp_rollout_kernel<R>>(s, sizeof(R), B, warps, grid, smem)) return rc;
  mlp_rollout_kernel<R><<<grid, 32 * warps, smem, stream>>>(s, (const R*)rec->params, B, T, N, M, x_init, u, x);
  return launched();
}

template <typename R>
int mlp_launch_linearize(const mpcb200_mlp* rec, int B, int T, int N, int M, const R* x, const R* u, R* F, R* f,
                         cudaStream_t stream) {
  MlpShape s;
  if (!mlp_shape(rec, s)) return MPCB200_ERR_BAD_DIMS;
  int warps, grid;
  size_t smem;
  const long long items = (long long)(T - 1) * B;
  if (const int rc = mlp_prepare<mlp_linearize_kernel<R>>(s, sizeof(R), items, warps, grid, smem)) return rc;
  mlp_linearize_kernel<R><<<grid, 32 * warps, smem, stream>>>(s, (const R*)rec->params, B, T, N, M, x, u, F, f);
  return launched();
}

template <typename R>
int mlp_launch_linesearch(const mpcb200_mlp* rec, const MlpLsArgs<R>& a, cudaStream_t stream) {
  MlpShape s;
  if (!mlp_shape(rec, s)) return MPCB200_ERR_BAD_DIMS;
  int warps, grid;
  size_t smem;
  if (const int rc = mlp_prepare<mlp_linesearch_kernel<R>>(s, sizeof(R), a.B, warps, grid, smem)) return rc;
  mlp_linesearch_kernel<R><<<grid, 32 * warps, smem, stream>>>(s, (const R*)rec->params, a);
  return launched();
}

MlpShape mlp_vjp_shape(const MlpShape& s) {
  MlpShape v = s;
  const int p = s.w[0];
  int hidden = 0;
  for (int i = 1; i < s.L; ++i) hidden += s.w[i];
  v.per_warp = round_up(p + hidden + hidden * p + 2 * s.maxw * p + 2 * s.maxw, 4);
  return v;
}

int mlp_vjp_slots(long long items, long long n_params) {
  long long g = kMlpVjpSlotElems / n_params;
  if (g < 1) g = 1;
  if (g > kMlpVjpMaxSlots) g = kMlpVjpMaxSlots;
  if (g > items) g = items;
  return g < 1 ? 1 : (int)g;
}

template <typename R>
int mlp_launch_linearize_vjp(const mpcb200_mlp* rec, int B, int T, int N, int M, const R* x, const R* u, const R* dF,
                             const R* df, R* dtheta, R* ws, cudaStream_t stream) {
  MlpShape s;
  if (!mlp_shape(rec, s)) return MPCB200_ERR_BAD_DIMS;
  const MlpShape v = mlp_vjp_shape(s);
  const int G = mlp_vjp_slots((long long)(T - 1) * B, s.n_params);
  int warps, grid;
  size_t smem;
  if (const int rc = mlp_prepare<mlp_linearize_vjp_kernel<R>>(v, sizeof(R), G, warps, grid, smem)) return rc;
  if (grid > kMlpVjpMaxCtas) grid = kMlpVjpMaxCtas;
  mlp_linearize_vjp_kernel<R><<<grid, 32 * warps, smem, stream>>>(v, (const R*)rec->params, B, T, N, M, x, u, dF, df,
                                                                   G, ws);
  if (const int rc = launched()) return rc;
  const long long blocks = (s.n_params + 255) / 256;
  mlp_vjp_reduce_kernel<R><<<(int)(blocks < 1024 ? blocks : 1024), 256, 0, stream>>>(ws, G, s.n_params, dtheta);
  return launched();
}

#define MPCB200_MLP_INSTANTIATE(R)                                                                                    \
  template int mlp_launch_rollout<R>(const mpcb200_mlp*, int, int, int, int, const R*, const R*, R*, cudaStream_t);    \
  template int mlp_launch_linearize<R>(const mpcb200_mlp*, int, int, int, int, const R*, const R*, R*, R*,             \
                                       cudaStream_t);                                                                  \
  template int mlp_launch_linesearch<R>(const mpcb200_mlp*, const MlpLsArgs<R>&, cudaStream_t);                        \
  template int mlp_launch_linearize_vjp<R>(const mpcb200_mlp*, int, int, int, int, const R*, const R*, const R*,       \
                                           const R*, R*, R*, cudaStream_t);
MPCB200_MLP_INSTANTIATE(float)
MPCB200_MLP_INSTANTIATE(double)

}  // namespace mpcb200
