// lqr_step2.cuh - the box-constrained LQR step, column-PAIR mapping with self-feeding warps (sm_90a).
//
// Same contract as lqr_step.cuh (reference LQRStepFn.forward, mpc/lqr_step.py:277-309: c_back :289-295,
// lqr_backward :52-160 incl. pnqp mpc/pnqp.py:5-82 and the u_zero_I solve :100-127, lqr_forward :164-261),
// different machine mapping.  Why a second mapping: the round-1 kernel (one column per lane) issues one
// shared-memory operand per FMA and spends part of its instructions polling mbarriers between a producer warp
// and its consumers.  Here
//  * L = (n+m)/2 lanes own one problem; a lane owns the column PAIR (c0, c0+1) of Q_t, F_t, C_t (x lanes also
//    the pair of V and K_t columns).  Every value a lane loads from shared memory feeds two FMAs (pair x
//    broadcast scalar), so operands per FMA halve and 32/L problems share a warp
//    (n=8, m=2: 6 problems / warp instead of 3).
//  * no producer warp and no empty barriers: every warp streams its OWN tiles.  After a warp has consumed
//    stage s, up to 8 of its lanes each issue one 1-D bulk TMA copy (C, F, c, x_bar, u_bar, f, bounds) of tile
//    seq+S into that stage in ONE instruction; completion is an mbarrier transaction count.  Warps are
//    independent, so a CTA is one warp.
//  * V is exchanged through a per-problem row-major buffer (a lane stores its column pair of every row with
//    8-byte stores, readers take whole rows as broadcast 128-bit loads) - exact V, no symmetry assumption.
//  * gains K_t, k_t of all T steps stay in shared memory (or the caller's Ks/ks for long horizons); the
//    rollout keeps the state replicated in every lane, lane pairs compute their two rows of F tau and C tau.
// Shapes: n and m even and the per-warp spans 16-byte aligned (Step2Cfg::OK); everything else runs the
// generic kernel in lqr_step.cuh.
#pragma once
#include "lqr_step.cuh"

namespace mpcb200 {

template <typename R>
MPCB_DEV P2<R> ld_pair(const R* p);
template <>
MPCB_DEV P2<float> ld_pair<float>(const float* p) {
  const float2 v = *reinterpret_cast<const float2*>(p);
  return {v.x, v.y};
}
template <>
MPCB_DEV P2<double> ld_pair<double>(const double* p) {
  const double2 v = *reinterpret_cast<const double2*>(p);
  return {v.x, v.y};
}
MPCB_DEV void st_pair(float* p, P2<float> v) { *reinterpret_cast<float2*>(p) = make_float2(v.x, v.y); }
MPCB_DEV void st_pair(double* p, P2<double> v) { *reinterpret_cast<double2*>(p) = make_double2(v.x, v.y); }
// a * (s, s) + c
template <typename R>
MPCB_DEV P2<R> fma2s(P2<R> a, R s, P2<R> c) { return fma2(a, P2<R>{s, s}, c); }

// Load CNT contiguous elements whose address is aligned to A elements (A a power of two): widest vector
// loads first (at most 16 bytes), narrower ones for the remainder.
template <typename R, int CNT, int A>
MPCB_DEV void load_span(const R* p, R (&out)[CNT]) {
  constexpr int EA = 16 / (int)sizeof(R);
  constexpr int W = A < EA ? A : EA;
  constexpr int NV = (CNT / W) * W;
  if constexpr (NV > 0) {
#pragma unroll
    for (int e = 0; e < NV; e += W) VecLoad<R, W>::ld(p + e, &out[e]);
  }
  if constexpr (NV < CNT) {
    if constexpr (W >= 2) {
      R rest[CNT - NV];
      load_span<R, CNT - NV, W / 2>(p + NV, rest);
#pragma unroll
      for (int e = 0; e < CNT - NV; ++e) out[NV + e] = rest[e];
    } else {
#pragma unroll
      for (int e = NV; e < CNT; ++e) out[e] = p[e];
    }
  }
}
// sum_i a[i] b[i] with packed pair FMAs (even/odd partial sums, one final add); CNT even
template <typename R, int CNT>
MPCB_DEV R dot_span(const R (&a)[CNT], const R (&b)[CNT]) {
  static_assert(CNT % 2 == 0, "pairs");
  P2<R> acc = mul2(P2<R>{a[0], a[1]}, P2<R>{b[0], b[1]});
#pragma unroll
  for (int k = 2; k < CNT; k += 2) acc = fma2(P2<R>{a[k], a[k + 1]}, P2<R>{b[k], b[k + 1]}, acc);
  return acc.x + acc.y;
}

// two dot products against the same vector, FMAs interleaved (two independent chains per pair slot)
template <typename R, int CNT>
MPCB_DEV void dot2_span(const R (&a0)[CNT], const R (&a1)[CNT], const R (&b)[CNT], R& r0, R& r1) {
  static_assert(CNT % 2 == 0, "pairs");
  P2<R> acc0 = mul2(P2<R>{a0[0], a0[1]}, P2<R>{b[0], b[1]});
  P2<R> acc1 = mul2(P2<R>{a1[0], a1[1]}, P2<R>{b[0], b[1]});
#pragma unroll
  for (int k = 2; k < CNT; k += 2) {
    acc0 = fma2(P2<R>{a0[k], a0[k + 1]}, P2<R>{b[k], b[k + 1]}, acc0);
    acc1 = fma2(P2<R>{a1[k], a1[k + 1]}, P2<R>{b[k], b[k + 1]}, acc1);
  }
  r0 = acc0.x + acc0.y;
  r1 = acc1.x + acc1.y;
}

template <typename R, int N, int M>
struct Step2Cfg {
  static constexpr int P = N + M;
  static constexpr int L = P / 2;            // lanes per problem
  static constexpr int NXL = N / 2;          // x lanes (own two state columns each)
  static constexpr int PPW = 32 / L;         // problems per warp
  static constexpr int EA = 16 / (int)sizeof(R);
  static constexpr int SZ = (int)sizeof(R);
  // shapes this mapping supports: even n, m; per-warp spans of C and F 16-byte multiples (always true for even
  // n, m) and per-problem vectors that the lanes read straight from global memory with vector loads
  static constexpr bool OK = (N % 2 == 0) && (M % 2 == 0) && L <= 16 && N >= 2 && M >= 2 && (PPW * M * SZ) % 16 == 0 &&
                             (PPW * N * SZ) % 16 == 0 && (PPW * P * SZ) % 16 == 0;
  // default choice between this mapping and the generic kernel, from tools/exp_step.py --preset shapes --kernel 1,2
  // on an H100 SXM (400 W power limit), fp32, us per launch generic / pair: the pair mapping wins where the dense products dominate
  // (n=16, m=4, T=50, B=4096: 935 / 653; n=8, m=4: 107 / 89) and is no slower for narrow problems (n+m <= 6);
  // in between the generic kernel stays (n=8, m=2, B=16384: 196 / 206; n=12, m=4: 230 / 240).
  static constexpr bool PAIR_DEFAULT = OK && (P >= 18 || P <= 6 || (N == 8 && M == 4));
  // stage layout (elements): dense spans of the warp's PPW problems, in the tensors' own layouts
  // Per-problem tiles are dense (stride p*p / n*p).  Padding them per problem dodges the bank conflicts of the
  // broadcast loads (n=16, m=4: F tiles 320 floats apart) but costs one bulk copy per problem instead of one per
  // warp span; it did not pay off in an earlier measurement and was removed.
  static constexpr int CS = P * P, FS = N * P;
  static constexpr int OFF_C = 0;
  static constexpr int OFF_F = OFF_C + PPW * CS;
  static constexpr int OFF_c = OFF_F + PPW * FS;
  static constexpr int OFF_x = OFF_c + PPW * P;
  static constexpr int OFF_u = OFF_x + PPW * N;
  static constexpr int OFF_f = OFF_u + PPW * M;
  static constexpr int OFF_lo = OFF_f + PPW * N;
  static constexpr int OFF_hi = OFF_lo + PPW * M;
  static constexpr int OFF_c2 = OFF_hi + PPW * M;        // fused adjoint: the true cost's c (the c slot carries -r)
  static constexpr int OFF_END = OFF_c2 + PPW * P;
  static constexpr int STAGE_BYTES = round_up(OFF_END * SZ, 128);
  // ring depth: 4 stages for small tiles, 3 for big ones (n=16, m=4: 9.4 KB tiles).  Fewer stages let more warps
  // reside per SM but hide less of the copy latency; 3 was the best trade-off for the big tiles.
  static constexpr int S = STAGE_BYTES > 6144 ? 3 : 4;
  static constexpr int MAX_REGS = 255;
  // per-problem scratch (elements)
  static constexpr int NV = round_up(N, 4);             // row stride of V / K rows (16-byte aligned rows)
  static constexpr int VSTR = NV;
  static constexpr int SC_V = 0;                         // N x NV value matrix, row-major
  static constexpr int SC_v = SC_V + N * VSTR;           // NV
  static constexpr int SC_Q = SC_v + NV;                 // N x M   Q_xu, row-major [i][a]
  static constexpr int SC_X = SC_Q + round_up(N * M, 4); // 2 x NV  rollout state exchange
  static constexpr int SC_R = SC_X + 2 * NV;             // L       cost reduction
  static constexpr int SC_K = SC_R + round_up(L, 4);     // M x NV + M gain exchange when gains are not smem resident
  static constexpr int KT = M * NV + round_up(M, 4);     // elements per (problem, t) of the gain store
  static constexpr int SC_RAW = SC_K + KT;
  // guaranteed alignment (elements) of per-problem vectors in global memory (bases are 16-byte aligned)
  static constexpr int A_N = align_elems<R>(N), A_M = align_elems<R>(M), A_P = align_elems<R>(P);
  static constexpr int pick_scr() {
    // smallest stride >= SC_RAW, multiple of 4, with stride % 8 == 4: consecutive problems then start an odd
    // number of 16-byte bank groups apart and broadcast 128-bit loads of up to 8 problems never collide
    int s = round_up(SC_RAW, 4);
    while (s % 8 != 4) s += 4;
    return s;
  }
  static constexpr int SCRS = pick_scr();
  static constexpr int HDR_BYTES = 128;                  // S mbarriers (per warp)
  __host__ __device__ static size_t smem_bytes(int T, bool k_in_smem, bool adj = false) {
    size_t b = HDR_BYTES + (size_t)S * STAGE_BYTES + (size_t)PPW * SCRS * SZ;
    if (k_in_smem) b += (size_t)PPW * T * KT * SZ;
    if (adj) b += (size_t)PPW * T * P * SZ;              // d tau of every step, kept for the costate sweep
    return round_up((int)b, 128);
  }
};

// One warp's tile stream: where its spans start in global memory and where its ring lives in shared memory.
struct TileSrc {
  const char *pC, *pF, *pc, *px, *pu, *pf, *plo, *phi, *pc2;
  uint32_t ucnt;      // bytes per element-of-a-problem over the warp's problems (cnt * sizeof(R))
  uint32_t stage0;    // shared address of stage 0
  uint32_t bar0;      // shared address of full[0]
};

// Start the bulk copies of tile (t, fwd) into ring stage `stage` of the warp described by `ts`.  Branch free:
// one elected lane of the CALLING warp arrives on the stage's mbarrier with the byte count and issues up to
// eight copies (predicated PTX; UBLKCP executes once per warp).
template <typename R, int N, int M>
MPCB_DEV void tile_issue(const TileSrc& ts, const StepArgs& a, int stage, int t, bool fwd, int has_tb) {
  using K = Step2Cfg<R, N, M>;
  constexpr int P = K::P, SZ = K::SZ;
  const uint32_t dst = ts.stage0 + (uint32_t)stage * K::STAGE_BYTES;
  const uint32_t bar = ts.bar0 + (uint32_t)stage * 8u;
  const int needF = t < a.T - 1 ? 1 : 0;
  const int needf = (fwd && needF && a.has_f) ? 1 : 0;
  const size_t tB = (size_t)t * a.B * SZ;
  const uint32_t total = ts.ucnt * (P * P + P + N + M + (has_tb ? 2 * M : 0) + (a.adj ? P : 0)) +
                         (needF ? ts.ucnt * (N * P) : 0u) + (needf ? ts.ucnt * N : 0u);
  asm volatile(
      "{\n\t.reg .pred P, PF, Pf, PB;\n\t.reg .b32 d, n;\n\t"
      "elect.sync _|P, 0xffffffff;\n\t"
      "setp.ne.and.b32 PF, %12, 0, P;\n\t"
      "setp.ne.and.b32 Pf, %13, 0, P;\n\t"
      "setp.ne.and.b32 PB, %14, 0, P;\n\t"
      "@P mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t"
      "mul.lo.u32 n, %3, %15;\n\t"
      "@P cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%2], [%4], n, [%0];\n\t"
      "mul.lo.u32 n, %3, %16;\n\tadd.u32 d, %2, %17;\n\t"
      "@PF cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [d], [%5], n, [%0];\n\t"
      "mul.lo.u32 n, %3, %18;\n\tadd.u32 d, %2, %19;\n\t"
      "@P cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [d], [%6], n, [%0];\n\t"
      "mul.lo.u32 n, %3, %20;\n\tadd.u32 d, %2, %21;\n\t"
      "@P cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [d], [%7], n, [%0];\n\t"
      "add.u32 d, %2, %23;\n\t"
      "@Pf cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [d], [%9], n, [%0];\n\t"
      "mul.lo.u32 n, %3, %22;\n\tadd.u32 d, %2, %24;\n\t"
      "@P cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [d], [%8], n, [%0];\n\t"
      "add.u32 d, %2, %25;\n\t"
      "@PB cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [d], [%10], n, [%0];\n\t"
      "add.u32 d, %2, %26;\n\t"
      "@PB cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [d], [%11], n, [%0];\n\t"
      "}" ::"r"(bar), "r"(total), "r"(dst), "r"(ts.ucnt),                                                      // 0..3
      "l"(ts.pC + (size_t)t * a.C_ts * SZ), "l"(ts.pF + (size_t)t * a.F_ts * SZ),                             // 4 5
      "l"(ts.pc + (size_t)t * a.c_ts * SZ), "l"(ts.px + tB * N),                                               // 6 7
      "l"(ts.pu + tB * M), "l"(ts.pf + (size_t)t * a.f_ts * SZ), "l"(ts.plo + tB * M), "l"(ts.phi + tB * M),  // 8..11
      "r"(needF), "r"(needf), "r"(has_tb),                                                                      // 12 13 14
      "n"(P * P), "n"(N * P), "n"(K::OFF_F * SZ), "n"(P), "n"(K::OFF_c * SZ), "n"(N), "n"(K::OFF_x * SZ),      // 15..21
      "n"(M), "n"(K::OFF_f * SZ), "n"(K::OFF_u * SZ), "n"(K::OFF_lo * SZ), "n"(K::OFF_hi * SZ)                 // 22..26
      : "memory");
  if (a.adj) {      // fused adjoint: the true cost's c rides on the same mbarrier (its bytes are in `total`)
    asm volatile(
        "{\n\t.reg .pred P;\n\t"
        "elect.sync _|P, 0xffffffff;\n\t"
        "@P cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%1], [%2], %3, [%0];\n\t"
        "}" ::"r"(bar), "r"(dst + (uint32_t)K::OFF_c2 * SZ), "l"(ts.pc2 + (size_t)t * a.adj_c_ts * SZ), "r"(ts.ucnt * P)
        : "memory");
  }
}

template <typename R, int N, int M>
MPCB_DEV TileSrc tile_src(const StepArgs& a, int b0, int cnt, unsigned char* wbase) {
  using K = Step2Cfg<R, N, M>;
  constexpr int P = K::P, SZ = K::SZ;
  const size_t eb = (size_t)b0 * SZ;
  TileSrc ts;
  ts.pC = (const char*)a.C + eb * (P * P);
  ts.pF = (const char*)a.F + eb * (N * P);
  ts.pc = (const char*)a.c + eb * P;
  ts.px = (const char*)(a.adj ? a.adj_x : a.cur_x) + eb * N;      // adjoint: the nominal point is zero, the slots carry tau*
  ts.pu = (const char*)(a.adj ? a.adj_u : a.cur_u) + eb * M;
  ts.pc2 = (const char*)a.adj_c + eb * P;
  ts.pf = (const char*)a.f + eb * N;
  ts.plo = (const char*)a.u_lower + eb * M;
  ts.phi = (const char*)a.u_upper + eb * M;
  ts.ucnt = (uint32_t)cnt * SZ;
  ts.stage0 = smem_u32(wbase + K::HDR_BYTES);
  ts.bar0 = smem_u32(wbase);
  return ts;
}

template <typename R, int N, int M, int MODE, bool KSM, bool ADJ = false>
__global__ void __launch_bounds__(32) __maxnreg__((Step2Cfg<R, N, M>::MAX_REGS))
lqr_step2_kernel(const StepArgs a) {
  using K = Step2Cfg<R, N, M>;
  constexpr int P = K::P, L = K::L, NXL = K::NXL, PPW = K::PPW, S = K::S, SZ = K::SZ, KT = K::KT, VSTR = K::VSTR, NV = K::NV;
  constexpr int EA = K::EA, A_N = K::A_N, A_M = K::A_M;
  constexpr unsigned FULLM = (1u << M) - 1u;
  constexpr bool BOX = MODE == MODE_BOX;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  const int lane = threadIdx.x & 31;                        // one warp per CTA
  const int T = a.T, B = a.B;
  // tensor bounds ride in the lo/hi slots; the fused adjoint uses the lo slot for its active-set mask (as R values)
  const int has_tb = (ADJ || (BOX && a.bounds_kind == 2)) ? 1 : 0;
  // global tile sequence of the sweep + first rollout pass: g < T -> t = T-1-g (backward), else t = g-T (forward)
  const int G = T + (a.do_rollout ? T : 0);

  const int b0 = blockIdx.x * PPW;
  if (b0 >= B) return;                                      // warps are independent: no CTA-wide barrier below
  const int cnt = min(PPW, B - b0);
  unsigned char* wbase = smem_raw;
  uint64_t* full = reinterpret_cast<uint64_t*>(wbase);
  unsigned char* stage_base = wbase + K::HDR_BYTES;
  R* scratch = reinterpret_cast<R*>(stage_base + (size_t)S * K::STAGE_BYTES);
  R* kstore = scratch + (size_t)PPW * K::SCRS;
  R* dts_all = kstore + (KSM ? (size_t)PPW * T * KT : 0);   // ADJ: d tau store, [problem][t][P]

  const bool writer_lane = lane < PPW * L;
  const int pi = writer_lane ? lane / L : PPW - 1;
  const int base = pi * L;
  const int lq = writer_lane ? lane - base : L - 1;
  const int b = b0 + pi;
  const bool valid = b < B;
  const bool wr = writer_lane && valid;
  const bool isx = lq < NXL;
  const int c0 = 2 * lq;                                    // first owned column (x then u columns)
  const int ua0 = isx ? 0 : c0 - N;                         // first owned control (u lanes)
  const int xr0 = isx ? c0 : 0;                             // a valid state row for every lane
  const int bsafe = valid ? b : B - 1;

  // ------------------------------------------------------------------ tile streaming (this warp's own ring)
  // One tile = the warp's spans of C[t], F[t], c[t], x_bar[t], u_bar[t] (+ f[t] in the rollout, + tensor
  // bounds): up to eight 1-D bulk copies onto ONE mbarrier (tile_issue).  Nothing on the data path goes through
  // the load/store scoreboards (global loads that are prefetched across loop iterations end up sharing a
  // scoreboard with the mbarrier probe and expose the full DRAM latency every step - measured).
  const TileSrc tsrc = tile_src<R, N, M>(a, b0, cnt, wbase);
  if (lane == 0) {
#pragma unroll
    for (int s2 = 0; s2 < S; ++s2) mbar_init(&full[s2], 1);
    mbar_fence_init();
  }
  __syncwarp();
  int iss_s = 0;                                            // stage of the next tile to issue
  auto issue = [&](int t, bool fwd) {
    tile_issue<R, N, M>(tsrc, a, iss_s, t, fwd, has_tb);
    iss_s = iss_s + 1 == S ? 0 : iss_s + 1;
  };
  // "done with the stage of tile g": refill it with tile g + S of the global sequence.  (A variant with a
  // dedicated producer warp per two consumer warps - the consumer only arrives on an `empty` mbarrier - was
  // slower at config 3 and was removed.)
  auto release = [&](int g) {
    const int gn = g + S;
    if (gn < G) {
      if (gn < T) issue(T - 1 - gn, false);
      else issue(gn - T, true);
    }
  };
  int con_s = 0;                                            // stage / phase parity of the next tile to consume
  uint32_t con_ph = 0;
  // split acquire: probe early (the probe's latency overlaps the math that follows), block only if needed
  auto probe = [&]() -> uint32_t { return mbar_try_wait(&full[con_s], con_ph) ? 1u : 0u; };
  auto acquire = [&](uint32_t ok) -> const R* {
    const R* st = (const R*)(stage_base + (size_t)con_s * K::STAGE_BYTES);
    if (!ok) mbar_wait(&full[con_s], con_ph);
    if (++con_s == S) { con_s = 0; con_ph ^= 1u; }
    return st;
  };
  for (int g = 0; g < S && g < G; ++g) release(g - S);       // prologue: tiles 0 .. S-1

  const bool has_mask = MODE == MODE_MASK || (BOX && a.has_mask);
  const int olo_ = K::OFF_lo + pi * M;
  auto mask_bits = [&](int t, const R* stt) -> unsigned {  // u_zero_I of (t, problem)
    unsigned z = 0u;
    if constexpr (ADJ) {                                   // fused adjoint: on the tile (no global load on the chain)
#pragma unroll
      for (int q = 0; q < M; ++q) z |= (stt[olo_ + q] != R(0) ? 1u : 0u) << q;
    } else if (has_mask) {                                 // M bytes straight from global
#pragma unroll
      for (int q = 0; q < M; ++q) z |= (a.zero_mask[((size_t)t * B + bsafe) * M + q] ? 1u : 0u) << q;
    }
    return z;
  };

  // per-problem element offsets inside a stage
  const int oC = K::OFF_C + pi * K::CS, oF = K::OFF_F + pi * K::FS;
  const int oc = K::OFF_c + pi * P, of_ = K::OFF_f + pi * N, ox = K::OFF_x + pi * N, ou = K::OFF_u + pi * M;
  const int olo = K::OFF_lo + pi * M, ohi = K::OFF_hi + pi * M;
  R* scr = scratch + (size_t)pi * K::SCRS;
  R* Vs = scr + K::SC_V;
  R* vs = scr + K::SC_v;
  R* Qx = scr + K::SC_Q;
  R* xs = scr + K::SC_X;
  R* red = scr + K::SC_R;
  R* kst = KSM ? kstore + (size_t)pi * T * KT : scr + K::SC_K;
  R* gKs = (R*)a.Ks;
  R* gks = (R*)a.ks;
  const R s_lo = (R)a.u_lo, s_hi = (R)a.u_hi, s_du = (R)a.delta_u, decay = (R)a.ls_decay;

  unsigned status = 0u;
  R oldcost_part = R(0);
  R kprev[M];
#pragma unroll
  for (int q = 0; q < M; ++q) kprev[q] = R(0);

  // ======================= backward Riccati sweep (lqr_step.py:61-158) =======================
  // Software pipelined by hand: everything of step t-1 that does not depend on the value matrix (tile probe,
  // its column pairs of C and F, c_back = C tau_bar + c, the nominal cost) is issued inside step t, where it
  // fills the latency of the scalar solve and of the shared-memory round trips.
  P2<R> Qp[P];                                     // (Q[i][c0], Q[i][c0+1]); starts as the column pair of C_t
  P2<R> qp;                                        // (q[c0], q[c0+1]);       starts as c_back
  P2<R> Fp[N];                                     // (F[k][c0], F[k][c0+1])
  R ubar[M], blo[M], bhi[M];                       // u_bar_t and tensor bounds of the step being solved
  unsigned zmk = 0u;
  // the V-independent part of step tt, from its tile `stt`
  auto pre = [&](int tt, const R* stt) {
#pragma unroll
    for (int i = 0; i < P; ++i) Qp[i] = ld_pair<R>(stt + oC + i * P + c0);
    const P2<R> cj = ld_pair<R>(stt + oc + c0);
    R tb[P];
    if constexpr (ADJ) {         // KKT adjoint: the nested solve starts from the zero trajectory (c_back = c, cost 0);
#pragma unroll                 // the x_bar / u_bar slots of the tile carry tau* for the costate sweep instead
      for (int i = 0; i < P; ++i) tb[i] = R(0);
      qp = cj;
    } else {
      R Cr0[P], Cr1[P];
      load_span<R, P, EA>(stt + oC + c0 * P, Cr0);            // c0 * P is a multiple of 4
      load_span<R, P, 2>(stt + oC + (c0 + 1) * P, Cr1);
      R tx[N], tu[M];
      load_span<R, N, A_N>(stt + ox, tx);
      load_span<R, M, A_M>(stt + ou, tu);
#pragma unroll
      for (int i = 0; i < N; ++i) tb[i] = tx[i];
#pragma unroll
      for (int q = 0; q < M; ++q) tb[N + q] = tu[q];
      const P2<R> tj = ld_pair<R>(stt + (isx ? ox + c0 : ou + ua0));   // tau_bar[c0], tau_bar[c0+1]
      R ct0, ct1;
      dot2_span<R, P>(Cr0, Cr1, tb, ct0, ct1);                 // rows c0, c0+1 of C tau_bar (lqr_step.py:289-295)
      if (writer_lane) oldcost_part += tj.x * (R(0.5) * ct0 + cj.x) + tj.y * (R(0.5) * ct1 + cj.y);   // util.get_cost (:169)
      qp = {ct0 + cj.x, ct1 + cj.y};
    }
#pragma unroll
    for (int q = 0; q < M; ++q) {
      ubar[q] = tb[N + q];
      if (BOX && a.bounds_kind == 2) {
        blo[q] = stt[olo + q];
        bhi[q] = stt[ohi + q];
      }
    }
    zmk = mask_bits(tt, stt);
  };
  const R* st = acquire(0u);
  pre(T - 1, st);
  for (int t = T - 1; t >= 0; --t) {
    uint32_t ok_next = 0u;
    if (t > 0) ok_next = probe();                  // tile t-1: checked after the products
    if (t < T - 1) {                               // Q = C + F'VF, q = c_back + F'v  (:66-70)
      R Vr[N][N];                                  // the whole value matrix (broadcast 128-bit loads)
#pragma unroll
      for (int i = 0; i < N; ++i) load_span<R, N, EA>(Vs + i * VSTR, Vr[i]);
      R vv[N];
      load_span<R, N, EA>(vs, vv);
      P2<R> Wp[N];                                 // (W[i][c0], W[i][c0+1]),  W = V F : N independent FMA chains
#pragma unroll
      for (int i = 0; i < N; ++i) Wp[i] = mul2(Fp[0], P2<R>{Vr[i][0], Vr[i][0]});
#pragma unroll
      for (int k = 1; k < N; ++k) {
#pragma unroll
        for (int i = 0; i < N; ++i) Wp[i] = fma2s(Fp[k], Vr[i][k], Wp[i]);
      }
      // Q[:, pair] += F' W[:, pair]: rows of F come as 2-row chunks of the flat tile; P independent chains
#pragma unroll
      for (int k = 0; k < N; k += 2) {
        R Fr[2 * P];
        load_span<R, 2 * P, EA>(st + oF + k * P, Fr);     // k even: k * P is a multiple of 4
#pragma unroll
        for (int i = 0; i < P; ++i) Qp[i] = fma2s(Wp[k], Fr[i], Qp[i]);
#pragma unroll
        for (int i = 0; i < P; ++i) Qp[i] = fma2s(Wp[k + 1], Fr[P + i], Qp[i]);
      }
#pragma unroll
      for (int k = 0; k < N; ++k) qp = fma2s(Fp[k], vv[k], qp);
    }
    // tile t is consumed (its C pair / rows / vectors were read by pre(t)): refill the stage with tile g + S
    __syncwarp();
    release(T - 1 - t);
    const R* st_next = st;
    if (t > 0) {                                   // F column pair of step t-1: lands while the solve runs
      st_next = acquire(ok_next);
#pragma unroll
      for (int k = 0; k < N; ++k) Fp[k] = ld_pair<R>(st_next + oF + k * P + c0);
    }
    // replicate Q_uu, q_u: control column a lives in lane base + NXL + a/2, component a%2
    R Quu[M][M], qu[M];
#pragma unroll
    for (int a2 = 0; a2 < M; ++a2) {
      const int src = base + NXL + a2 / 2;
#pragma unroll
      for (int p1 = 0; p1 < M; ++p1) Quu[p1][a2] = shfl((a2 & 1) ? Qp[N + p1].y : Qp[N + p1].x, src);
      qu[a2] = shfl((a2 & 1) ? qp.y : qp.x, src);
    }
    R kk[M];
    unsigned fm = FULLM;
    int it = 0;
    Ldl<R, M> fac;
    if constexpr (BOX) {
      box_control_solve<R, M>(a, Quu, qu, kprev, valid, t < T - 1, [&](int q) { return blo[q]; },
                              [&](int q) { return bhi[q]; }, [&](int q) { return ubar[q]; }, kk, fm, it, fac, status);
    } else {
      if constexpr (MODE == MODE_MASK) fm = FULLM & ~zmk;
      ldl_control_solve<R, M>(Quu, qu, fm, kk, fac, status);
    }
    // K[:, pair] = -Hff^{-1} Qux_f[:, pair] (rows of clamped / masked controls are zero)
    P2<R> Kp[M];
    R* Kt = KSM ? kst + (size_t)t * KT : kst;
    {
      R r0[M], r1[M], s0[M], s1[M];
#pragma unroll
      for (int q = 0; q < M; ++q) {
        const bool fq = (fm >> q) & 1u;
        r0[q] = fq ? Qp[N + q].x : R(0);
        r1[q] = fq ? Qp[N + q].y : R(0);
      }
      fac.solve(r0, s0);
      fac.solve(r1, s1);
#pragma unroll
      for (int q = 0; q < M; ++q) Kp[q] = {-s0[q], -s1[q]};
    }
    // publish: x lanes their K pair (rows of the gain store), u lanes their Q_xu pair as rows [i][a] -
    // one predicated store sequence for both kinds of lanes
    {
      R* sbase = isx ? Kt + c0 : Qx + ua0;
      const int sstr = isx ? NV : M;
#pragma unroll
      for (int i = 0; i < (N > M ? N : M); ++i) {
        const bool on = writer_lane && (isx ? i < M : i < N);
        const P2<R> v = (isx && i < M) ? Kp[i < M ? i : 0] : Qp[i < N ? i : 0];
        if (on) st_pair(sbase + i * sstr, v);
      }
      if (writer_lane && lq == 0) {
#pragma unroll
        for (int q = 0; q < M; ++q) Kt[M * NV + q] = kk[q];
      }
    }
    if (gKs != nullptr || a.free_mask != nullptr || (BOX && a.qp_iters != nullptr)) {   // optional outputs
      if (wr) {
        const size_t tbo = (size_t)t * B + b;
        if (gKs != nullptr && isx) {
#pragma unroll
          for (int q = 0; q < M; ++q) st_pair(gKs + (tbo * M + q) * N + c0, Kp[q]);
          if (lq == 0) {
#pragma unroll
            for (int q = 0; q < M; ++q) gks[tbo * M + q] = kk[q];
          }
        }
        if (lq == 0) {
          if (BOX && a.qp_iters != nullptr) a.qp_iters[tbo] = it;
          if (a.free_mask != nullptr) {
#pragma unroll
            for (int q = 0; q < M; ++q) a.free_mask[tbo * M + q] = (fm >> q) & 1u;
          }
        }
      }
    }
    __syncwarp();
    // V = Qxx + Qxu K + K'Qux + K'Quu K ; v = qx + Qxu k + K'qu + K'Quu k   (:155-158)
    {
      P2<R> Gp[M];                                 // (Qux + Quu K)[a][pair]
      R gq[M];                                     // qu + Quu k
#pragma unroll
      for (int p1 = 0; p1 < M; ++p1) {
        Gp[p1] = Qp[N + p1];
        gq[p1] = qu[p1];
#pragma unroll
        for (int p2 = 0; p2 < M; ++p2) {
          Gp[p1] = fma2s(Kp[p2], Quu[p1][p2], Gp[p1]);
          gq[p1] += Quu[p1][p2] * kk[p2];
        }
      }
      R Qf[N * M];                                 // Q_xu flat [i][a]
      load_span<R, N * M, EA>(Qx, Qf);
      R Kr[M][N];
#pragma unroll
      for (int q = 0; q < M; ++q) load_span<R, N, EA>(Kt + q * NV, Kr[q]);
      R qa[2 * M];                                 // Q_xu rows c0, c0+1 (x lanes; any valid rows otherwise)
      load_span<R, 2 * M, (2 * M) % 4 == 0 ? 4 : 2>(Qx + xr0 * M, qa);
      P2<R> Vp[N];
#pragma unroll
      for (int i = 0; i < N; ++i) Vp[i] = Qp[i];
#pragma unroll
      for (int q = 0; q < M; ++q) {
#pragma unroll
        for (int i = 0; i < N; ++i) Vp[i] = fma2s(Kp[q], Qf[i * M + q], Vp[i]);
#pragma unroll
        for (int i = 0; i < N; ++i) Vp[i] = fma2s(Gp[q], Kr[q][i], Vp[i]);
      }
      P2<R> vp = qp;
#pragma unroll
      for (int q = 0; q < M; ++q) {
        vp.x += qa[q] * kk[q];
        vp.y += qa[M + q] * kk[q];
        vp = fma2s(Kp[q], gq[q], vp);
      }
      if (writer_lane && isx) {
#pragma unroll
        for (int i = 0; i < N; ++i) st_pair(Vs + i * VSTR + c0, Vp[i]);
        st_pair(vs + c0, vp);
      }
    }
    // V-independent part of step t-1, in the shadow of the V round trip through shared memory
    if (t > 0) {
      pre(t - 1, st_next);
      st = st_next;
    }
    __syncwarp();
  }

  // nominal cost (sum of the lanes' partial sums, fixed order)
  if (writer_lane) red[lq] = oldcost_part;
  __syncwarp();
  R oldcost = R(0);
#pragma unroll
  for (int i = 0; i < L; ++i) oldcost += red[i];
  __syncwarp();

  if (!a.do_rollout) {
    if (wr && lq == 0) write_step_status(a, b, status);
    return;
  }

  // ======================= rollout + line search (lqr_step.py:164-261) =======================
  // Per step the dependent chain is x -> u = K dx + .. -> clamp -> x' = F tau + f -> exchange.  The operands
  // of step t+1 (gain rows, rows of C and F, the small vectors) are loaded into the registers of step t as
  // soon as those are dead, so they are in flight while the chain of step t runs.
  const R* gx0 = (const R*)a.x_init;
  R* gnx = (R*)a.new_x;
  R* gnu = (R*)a.new_u;
  R* gdu1 = (R*)a.du_first;
  R alpha = R(1), fdn = R(0), cost = R(0);
  bool worse = false;
  for (int pass = 0;; ++pass) {
    if (pass > 0) {                                // line-search repeat: restart this warp's tile stream
      for (int g = 0; g < S && g < T; ++g) issue(g, true);
    }
    R xr[N];                                       // state replicated on every lane
    load_span<R, N, A_N>(gx0 + (size_t)bsafe * N, xr);
    P2<R> xown = ld_pair<R>(gx0 + (size_t)bsafe * N + xr0);
    R Krow[M][N], kq[M], Cr0[P], Cr1[P], Fr0[P], Fr1[P], tbx[N], tbu[M], lo_t[M], hi_t[M];
    P2<R> cj, fj;
    unsigned zm = 0u;
    auto load_gain = [&](int tt) {
      if constexpr (KSM) {
        const R* Kt = kst + (size_t)tt * KT;
#pragma unroll
        for (int q = 0; q < M; ++q) {
          load_span<R, N, EA>(Kt + q * NV, Krow[q]);
          kq[q] = Kt[M * NV + q];
        }
      } else {
        const size_t row = (size_t)tt * B + bsafe;
#pragma unroll
        for (int q = 0; q < M; ++q) {
          load_span<R, N, A_N>(gKs + (row * M + q) * N, Krow[q]);
          kq[q] = gks[row * M + q];
        }
      }
    };
    auto load_tile = [&](int tt, const R* stt) {   // rows c0, c0+1 of C and F, nominal point, c, f, bounds
      load_span<R, P, EA>(stt + oC + c0 * P, Cr0);
      load_span<R, P, 2>(stt + oC + (c0 + 1) * P, Cr1);
      if (tt < T - 1) {
        load_span<R, P, EA>(stt + oF + xr0 * P, Fr0);
        load_span<R, P, 2>(stt + oF + (xr0 + 1) * P, Fr1);
      }
      if constexpr (ADJ) {
#pragma unroll
        for (int i = 0; i < N; ++i) tbx[i] = R(0);
#pragma unroll
        for (int q = 0; q < M; ++q) tbu[q] = R(0);
      } else {
        load_span<R, N, A_N>(stt + ox, tbx);
        load_span<R, M, A_M>(stt + ou, tbu);
      }
      cj = ld_pair<R>(stt + oc + c0);
      fj = {R(0), R(0)};
      if (a.has_f && tt < T - 1) fj = ld_pair<R>(stt + of_ + xr0);
      if (BOX && a.bounds_kind == 2) {
#pragma unroll
        for (int q = 0; q < M; ++q) {
          lo_t[q] = stt[olo + q];
          hi_t[q] = stt[ohi + q];
        }
      }
      zm = mask_bits(tt, stt);
    };
    st = acquire(0u);
    load_gain(0);
    load_tile(0, st);
    R cpart = R(0), dun2 = R(0);
    size_t orow = (size_t)bsafe;                   // t*B + b
    for (int t = 0; t < T; ++t, orow += (size_t)B) {
      uint32_t ok_next = 0u;
      if (t + 1 < T) ok_next = probe();            // tile t+1
      R dxv[N];
#pragma unroll
      for (int i = 0; i < N; ++i) dxv[i] = xr[i] - tbx[i];
      R u[M];
#pragma unroll
      for (int q = 0; q < M; ++q) u[q] = (dot_span<R, N>(Krow[q], dxv) + tbu[q]) + alpha * kq[q];   // (:192)
      if (t + 1 < T) load_gain(t + 1);             // gain registers are dead: fetch the next step's rows
      P2<R> ubj = {tbu[0], tbu[1]};
#pragma unroll
      for (int q = 0; q < M; ++q) {
        u[q] = rollout_control<R>(u[q], tbu[q], MODE != MODE_PLAIN && has_mask && ((zm >> q) & 1u), BOX,
                                  a.bounds_kind == 2 ? lo_t[q] : s_lo, a.bounds_kind == 2 ? hi_t[q] : s_hi,
                                  a.has_delta, s_du);
        const R d = tbu[q] - u[q];
        dun2 += d * d;
      }
      R tau[P];
#pragma unroll
      for (int i = 0; i < N; ++i) tau[i] = xr[i];
#pragma unroll
      for (int q = 0; q < M; ++q) tau[N + q] = u[q];
      // own pair of tau: x lanes carry it, u lanes pick their controls
      P2<R> tj = xown;
      if (!isx) {
#pragma unroll
        for (int q = 0; q < M; q += 2)
          if (q == ua0) {
            tj = {u[q], u[q + 1]};
            ubj = {tbu[q], tbu[q + 1]};
          }
      }
      P2<R> xn = {R(0), R(0)};
      if (t < T - 1) {                                                        // (:217-222) - the chain first
        dot2_span<R, P>(Fr0, Fr1, tau, xn.x, xn.y);
        xn.x += fj.x;
        xn.y += fj.y;
        if (writer_lane && isx) st_pair(xs + (t & 1) * NV + c0, xn);
      }
      R ct0, ct1;
      dot2_span<R, P>(Cr0, Cr1, tau, ct0, ct1);
      if (writer_lane) cpart += tj.x * (R(0.5) * ct0 + cj.x) + tj.y * (R(0.5) * ct1 + cj.y);   // (:232)
      if (wr) {
        if (isx) {
          st_pair(gnx + orow * N + c0, tj);
        } else {
          st_pair(gnu + orow * M + ua0, tj);
          if (pass == 0 && gdu1 != nullptr) st_pair(gdu1 + orow * M + ua0, P2<R>{ubj.x - tj.x, ubj.y - tj.y});
        }
      }
      if constexpr (ADJ) {                          // d tau_t of this pass, for the costate sweep
        if (writer_lane) st_pair(dts_all + ((size_t)pi * T + t) * P + c0, tj);
      }
      // operands of step t+1 into the (now dead) registers of step t
      const R* st_next = st;
      if (t + 1 < T) {
        st_next = acquire(ok_next);
        load_tile(t + 1, st_next);
      }
      xown = xn;
      __syncwarp();
      if (t < T - 1) load_span<R, N, EA>(xs + (t & 1) * NV, xr);
      // tile t is consumed (its operands were loaded one step ago): refill its stage
      if (pass == 0) release(T + t);
      else if (t + S < T) issue(t + S, true);
      st = st_next;
    }
    if (writer_lane) red[lq] = cpart;
    __syncwarp();
    cost = R(0);
#pragma unroll
    for (int i = 0; i < L; ++i) cost += red[i];
    __syncwarp();
    worse = line_search_update<R>(pass, cost, oldcost, dun2, decay, fdn, alpha);
    const bool more = pass + 1 < a.max_ls;
    const bool again = __any_sync(0xffffffffu, wr && worse) && more;          // per problem == the reference's batch loop
    if (!again) break;
  }
  if constexpr (ADJ) {
    // ======================= costates and outer products (lqr_step.py:342-404) =======================
    // Third sweep, t = T-1 .. 0, over the same tiles (C, F, -r in the c slot, the true c, tau* in the x_bar/u_bar
    // slots; L2 hits) with d tau of every step in shared memory:
    //   lambda_t  = C^x_t tau*_t + c^x_t + F^x_t' lambda_{t+1},   dlambda_t = C^x_t dtau_t - r^x_t + F^x_t' dlambda_{t+1}
    //   dC_t = -1/2 (dtau tau*' + tau* dtau'),  dc_t = -dtau_t,  dF_t = -(dlambda_{t+1} tau*' + lambda_{t+1} dtau'),
    //   df_t = -dlambda_{t+1},  dx_init = -dlambda_0.     A lane writes its column pair of every row (8-byte stores).
    __syncwarp();
    for (int g = 0; g < S && g < T; ++g) issue(T - 1 - g, false);
    R* gdC = (R*)a.adj_dC;
    R* gdc = (R*)a.adj_dc;
    R* gdF = (R*)a.adj_dF;
    R* gdf = (R*)a.adj_df;
    const R* dts = dts_all + (size_t)pi * T * P;
    const int oc2 = K::OFF_c2 + pi * P;
    R lam[N], dlam[N];                             // lambda_{t+1}, dlambda_{t+1} replicated on every lane
#pragma unroll
    for (int k = 0; k < N; ++k) lam[k] = dlam[k] = R(0);
    P2<R> dl_own = {R(0), R(0)};                   // dlambda_{t+1}[c0], [c0+1] (x lanes)
    for (int t = T - 1; t >= 0; --t) {
      const R* stt = acquire(0u);
      const size_t tbo = (size_t)t * B + bsafe;
      R ts_[P], dt_[P];                            // tau*_t, dtau_t replicated
      {
        R tx[N], tu[M];
        load_span<R, N, A_N>(stt + ox, tx);
        load_span<R, M, A_M>(stt + ou, tu);
#pragma unroll
        for (int i = 0; i < N; ++i) ts_[i] = tx[i];
#pragma unroll
        for (int q = 0; q < M; ++q) ts_[N + q] = tu[q];
        load_span<R, P, 2>(dts + (size_t)t * P, dt_);
      }
      const P2<R> tsj = ld_pair<R>(stt + (isx ? ox + c0 : ou + ua0));     // tau*[c0], tau*[c0+1]
      const P2<R> dtj = ld_pair<R>(dts + (size_t)t * P + c0);             // dtau[c0], dtau[c0+1]
      if (wr) {
#pragma unroll
        for (int i = 0; i < P; ++i) {              // dC_t[i][pair]
          P2<R> v = mul2(tsj, P2<R>{dt_[i], dt_[i]});
          v = fma2s(dtj, ts_[i], v);
          st_pair(gdC + (tbo * P + i) * P + c0, P2<R>{R(-0.5) * v.x, R(-0.5) * v.y});
        }
        st_pair(gdc + tbo * P + c0, P2<R>{-dtj.x, -dtj.y});
        if (t < T - 1) {
#pragma unroll
          for (int k = 0; k < N; ++k) {            // dF_t[k][pair]
            P2<R> v = mul2(tsj, P2<R>{dlam[k], dlam[k]});
            v = fma2s(dtj, lam[k], v);
            st_pair(gdF + (tbo * N + k) * P + c0, P2<R>{-v.x, -v.y});
          }
          if (a.adj_has_df && isx) st_pair(gdf + tbo * N + c0, P2<R>{-dl_own.x, -dl_own.y});
        } else if (a.F_T == T) {
#pragma unroll
          for (int k = 0; k < N; ++k) st_pair(gdF + (tbo * N + k) * P + c0, P2<R>{R(0), R(0)});
        }
      }
      // costates of step t: rows c0, c0+1 (x lanes)
      {
        R Cr0[P], Cr1[P];
        load_span<R, P, EA>(stt + oC + xr0 * P, Cr0);
        load_span<R, P, 2>(stt + oC + (xr0 + 1) * P, Cr1);
        P2<R> nl, ndl;
        dot2_span<R, P>(Cr0, Cr1, ts_, nl.x, nl.y);
        dot2_span<R, P>(Cr0, Cr1, dt_, ndl.x, ndl.y);
        const P2<R> c2j = ld_pair<R>(stt + oc2 + xr0);       // true c^x
        const P2<R> nrj = ld_pair<R>(stt + oc + xr0);        // -r^x (the c slot)
        nl.x += c2j.x; nl.y += c2j.y;
        ndl.x += nrj.x; ndl.y += nrj.y;
        if (t < T - 1) {
#pragma unroll
          for (int k = 0; k < N; ++k) {
            const P2<R> fp = ld_pair<R>(stt + oF + k * P + xr0);        // F[k][c0], F[k][c0+1]
            nl = fma2s(fp, lam[k], nl);
            ndl = fma2s(fp, dlam[k], ndl);
          }
        }
        dl_own = ndl;
        if (writer_lane && isx) {
          st_pair(xs + c0, nl);
          st_pair(xs + NV + c0, ndl);
        }
      }
      __syncwarp();
      load_span<R, N, EA>(xs, lam);
      load_span<R, N, EA>(xs + NV, dlam);
      __syncwarp();
      if (t - S >= 0) issue(t - S, false);
    }
    if (wr && isx) st_pair((R*)a.adj_dx_init + (size_t)b * N + c0, P2<R>{-dl_own.x, -dl_own.y});
  }
  if (worse) alpha /= decay;                                                  // (:252)
  if (wr && lq == 0) write_step_result<R>(a, b, alpha, cost, fdn, status);
}

// launch_step2's answer when the column-pair mapping does not take the shape or the tensors' layout (or the fused
// adjoint is asked of a mode other than MASK): the caller runs the generic kernel instead
constexpr int STEP2_DECLINED = -1;

template <auto Kern>
int launch_step2_kernel(const StepArgs& a, int grid, size_t smem, int max_smem_optin, cudaStream_t stream) {
  const int rc = allow_smem_optin<Kern>(max_smem_optin);
  if (rc != MPCB200_OK) return rc;
  Kern<<<grid, 32, smem, stream>>>(a);
  if (cudaGetLastError() != cudaSuccess) return MPCB200_ERR_LAUNCH;
  record_step_plan((int)(MPCB200_PLAN_PAIR | (a.k_in_smem ? MPCB200_PLAN_GAINS_SMEM : 0u)));
  return MPCB200_OK;
}

template <typename R, int N, int M, int MODE>
int launch_step2_mode(const StepArgs& args, int max_smem_optin, cudaStream_t stream) {
  using K = Step2Cfg<R, N, M>;
  StepArgs a = args;
  const bool adj = a.adj != 0;
  if (adj && MODE != MODE_MASK) return STEP2_DECLINED;
  // keep a few warps per SM resident: move the gain store to the caller's buffer when it is what limits them
  const bool crowded = K::smem_bytes(a.T, true, adj) > (size_t)max_smem_optin / 6;
  size_t smem;
  const int rc = plan_gain_store(a, crowded, max_smem_optin,
                                 [&](bool k_in_smem) { return K::smem_bytes(a.T, k_in_smem, adj); }, smem);
  if (rc != MPCB200_OK) return rc;
  const int grid = (a.B + K::PPW - 1) / K::PPW;   // one warp per CTA
  if constexpr (MODE == MODE_MASK) {
    if (adj)                     // fused KKT adjoint (+ the d tau store)
      return a.k_in_smem ? launch_step2_kernel<lqr_step2_kernel<R, N, M, MODE, true, true>>(a, grid, smem, max_smem_optin, stream)
                         : launch_step2_kernel<lqr_step2_kernel<R, N, M, MODE, false, true>>(a, grid, smem, max_smem_optin, stream);
  }
  return a.k_in_smem ? launch_step2_kernel<lqr_step2_kernel<R, N, M, MODE, true>>(a, grid, smem, max_smem_optin, stream)
                     : launch_step2_kernel<lqr_step2_kernel<R, N, M, MODE, false>>(a, grid, smem, max_smem_optin, stream);
}

template <typename R, int N, int M>
int launch_step2(const StepArgs& a, int max_smem_optin, cudaStream_t stream) {
  if constexpr (Step2Cfg<R, N, M>::OK) {
    if (!a.bulk_ok) return STEP2_DECLINED;   // spans / bases not 16-byte aligned (odd batch sizes, sliced views)
    if (a.bounds_kind != 0) return launch_step2_mode<R, N, M, MODE_BOX>(a, max_smem_optin, stream);
    if (a.has_mask) return launch_step2_mode<R, N, M, MODE_MASK>(a, max_smem_optin, stream);
    return launch_step2_mode<R, N, M, MODE_PLAIN>(a, max_smem_optin, stream);
  } else {
    return STEP2_DECLINED;
  }
}

}  // namespace mpcb200
