// mma16.cuh - the two dense products of one Riccati step for n_state = 16 on the tensor cores (sm_90a).
//
//   Q' = F' V F   (p x p, p = 16 + m <= 22)      q' = F' v   (p)
// (reference mpc/lqr_step.py:66-70: Q_t = C_t + F_t' V_{t+1} F_t, q_t = c_t + F_t' v_{t+1}; the caller adds C, c.)
//
// Why: in the SIMT column-pair mapping every lane of a problem loads all of V and every row of F from shared
// memory (~23 KB delivered to registers per problem-step); the shared-memory -> register path (128 B / clk / SM)
// is what bounds the n=16 kernel (ncu: 73 % LSU wavefront utilisation, 27 % FMA pipe).  As mma.sync fragments the
// operands are delivered ONCE per warp (~2.5 KB per problem-step).
//
// One warp computes one problem at a time with mma.sync.m16n8k8 TF32 in three passes per product
// (3xTF32: a_lo*b_hi + a_hi*b_lo + a_hi*b_hi, fp32 accumulate: error ~4e-6 on |Q| ~ 13, the plain fp32 loop 2e-6;
// measured with tools/mma_probe.cu).  Formulation (g = lane >> 2, tq = lane & 3):
//   A  = F' (rows a = F column, 32 = 2 m-tiles, rows >= p are zero; contraction k = F row).  The k slots of a
//        fragment are PERMUTED: slot tq holds k = 2 tq, slot tq + 4 holds k = 2 tq + 1.  A contraction index may
//        be permuted freely as long as A and B agree - and with this permutation the accumulator layout of the
//        first product IS the B-fragment layout of the second, so no shuffles are needed in between.
//   1) G' = F' V  : D1[mt][nt] (rows a, cols j)  = sum_k F[k][a] V[j][k]        = (V F)[j][a]
//   2) Q' = F' [G | v] : B fragment (k = j, n = b) = G[j][b] = D1 registers (b < p), v[j] for b == p
//      Only the tiles of the upper block triangle are computed: rows 0-15 x cols 0-23 and rows 16-31 x cols
//      16-23; Q'[16.., 0..15] is stored as the transpose of Q'[0..15, 16..] (Q' is symmetric, and this makes it
//      bitwise symmetric).  48 mma.sync per problem instead of the 60 of the straightforward tiling.
#pragma once
#include "common.cuh"

namespace mpcb200 {

MPCB_DEV void tf32_split(float x, unsigned& hi, unsigned& lo) {
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
  const float r = x - __uint_as_float(hi);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(r));
}
MPCB_DEV void mma_tf32(float (&d)[4], const unsigned (&a)[4], const unsigned (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
MPCB_DEV void mma_3xtf32(float (&d)[4], const unsigned (&ah)[4], const unsigned (&al)[4], const unsigned (&bh)[2],
                         const unsigned (&bl)[2]) {
  mma_tf32(d, al, bh);      // small terms first
  mma_tf32(d, ah, bl);
  mma_tf32(d, ah, bh);
}

// Ft: F tile, [16][P] row-major.  Vm: V, [16][VSTR] row-major.  vv: v[16].
// Qout: [P][P] row-major (stride P) receives Q'; qout[P] receives q'.  All pointers: shared memory, 8-byte aligned.
// Must be called by all 32 lanes; the caller synchronises the warp before reading the outputs.
template <int P, int VSTR>
MPCB_DEV void ftvf_16(const float* __restrict__ Ft, const float* __restrict__ Vm, const float* __restrict__ vv,
                      float* __restrict__ Qout, float* __restrict__ qout, int lane) {
  static_assert(P > 16 && P <= 22 && P % 2 == 0, "n_state = 16, even n_ctrl <= 6");
  constexpr int MU = P - 16;                       // rows of the second m-tile that exist
  const int g = lane >> 2, tq = lane & 3;
  // ---- A fragments of F' (shared by both products), split into tf32 hi / lo
  unsigned Ah[2][2][4], Al[2][2][4];
#pragma unroll
  for (int kt = 0; kt < 2; ++kt) {
    const float* r0 = Ft + (8 * kt + 2 * tq) * P;  // F rows k0 = 8 kt + 2 tq and k0 + 1
    const float* r1 = r0 + P;
    tf32_split(r0[g], Ah[0][kt][0], Al[0][kt][0]);           // (row g,     slot tq)
    tf32_split(r0[g + 8], Ah[0][kt][1], Al[0][kt][1]);       // (row g + 8, slot tq)
    tf32_split(r1[g], Ah[0][kt][2], Al[0][kt][2]);           // (row g,     slot tq + 4)
    tf32_split(r1[g + 8], Ah[0][kt][3], Al[0][kt][3]);       // (row g + 8, slot tq + 4)
    const bool on = g < MU;                                  // second m-tile: rows 16 + g exist for g < m
    tf32_split(on ? r0[16 + g] : 0.f, Ah[1][kt][0], Al[1][kt][0]);
    tf32_split(on ? r1[16 + g] : 0.f, Ah[1][kt][2], Al[1][kt][2]);
    Ah[1][kt][1] = Al[1][kt][1] = Ah[1][kt][3] = Al[1][kt][3] = 0u;   // rows 24 + g never exist
  }
  // ---- 1) D1[mt][nt] = (F' V) tile: rows a = 16 mt + g (+8), cols j = 8 nt + 2 tq (+1)
  float D1[2][2][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int r = 0; r < 4; ++r) D1[mt][nt][r] = 0.f;
#pragma unroll
  for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
    for (int kt = 0; kt < 2; ++kt) {
      // B fragment (k slot tq -> k0, slot tq + 4 -> k0 + 1; n = j = 8 nt + g): V[j][k0], V[j][k0 + 1]
      const float2 vb = *reinterpret_cast<const float2*>(Vm + (8 * nt + g) * VSTR + 8 * kt + 2 * tq);
      unsigned bh[2], bl[2];
      tf32_split(vb.x, bh[0], bl[0]);
      tf32_split(vb.y, bh[1], bl[1]);
      mma_3xtf32(D1[0][nt], Ah[0][kt], Al[0][kt], bh, bl);
      mma_3xtf32(D1[1][nt], Ah[1][kt], Al[1][kt], bh, bl);
    }
  }
  // ---- 2) D2 = F' [G | v]; tiles (mt2 = 0, nt2 = 0..2) and (mt2 = 1, nt2 = 2)
  float E0[3][4], E1[4];
#pragma unroll
  for (int r = 0; r < 4; ++r) E0[0][r] = E0[1][r] = E0[2][r] = E1[r] = 0.f;
#pragma unroll
  for (int kt = 0; kt < 2; ++kt) {                 // contraction tile: j = 8 kt + 2 tq (+1)
#pragma unroll
    for (int nt2 = 0; nt2 < 3; ++nt2) {
      // B fragment (k = j, n = b = 8 nt2 + g): G[j][b] = D1[b / 16][kt] rows b % 16
      float b0 = nt2 == 0 ? D1[0][kt][0] : nt2 == 1 ? D1[0][kt][2] : D1[1][kt][0];
      float b1 = nt2 == 0 ? D1[0][kt][1] : nt2 == 1 ? D1[0][kt][3] : D1[1][kt][1];
      if (nt2 == 2 && g == MU) {                   // column p of [G | v]: v itself
        const float2 t2 = *reinterpret_cast<const float2*>(vv + 8 * kt + 2 * tq);
        b0 = t2.x;
        b1 = t2.y;
      }
      unsigned bh[2], bl[2];
      tf32_split(b0, bh[0], bl[0]);
      tf32_split(b1, bh[1], bl[1]);
      mma_3xtf32(E0[nt2], Ah[0][kt], Al[0][kt], bh, bl);
      if (nt2 == 2) mma_3xtf32(E1, Ah[1][kt], Al[1][kt], bh, bl);
    }
  }
  // ---- store.  Accumulator layout: e0,e1 = (row g, cols 2 tq, 2 tq + 1), e2,e3 = (row g + 8, same cols)
#pragma unroll
  for (int nt2 = 0; nt2 < 2; ++nt2) {              // rows 0-15, cols 0-15
    const int cc = 8 * nt2 + 2 * tq;
    *reinterpret_cast<float2*>(Qout + g * P + cc) = make_float2(E0[nt2][0], E0[nt2][1]);
    *reinterpret_cast<float2*>(Qout + (g + 8) * P + cc) = make_float2(E0[nt2][2], E0[nt2][3]);
  }
  {
    const int cc = 16 + 2 * tq;                    // cols 16..23: Q_xu block (cc < p), q' (cc == p), padding
    if (cc < P) {                                  // rows 0-15 x cols 16.. and its transpose rows 16.. x cols 0-15
      *reinterpret_cast<float2*>(Qout + g * P + cc) = make_float2(E0[2][0], E0[2][1]);
      *reinterpret_cast<float2*>(Qout + (g + 8) * P + cc) = make_float2(E0[2][2], E0[2][3]);
      Qout[cc * P + g] = E0[2][0];
      Qout[(cc + 1) * P + g] = E0[2][1];
      Qout[cc * P + g + 8] = E0[2][2];
      Qout[(cc + 1) * P + g + 8] = E0[2][3];
      if (g < MU) *reinterpret_cast<float2*>(Qout + (16 + g) * P + cc) = make_float2(E1[0], E1[1]);   // Q_uu
    } else if (cc == P) {                          // q' = F' v
      qout[g] = E0[2][0];
      qout[g + 8] = E0[2][2];
      if (g < MU) qout[16 + g] = E1[0];
    }
  }
}

}  // namespace mpcb200
