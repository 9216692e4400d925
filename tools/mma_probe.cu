// mma_probe.cu - round-2 feasibility probe (not part of the product): the two dense products of one
// backward step, W' = F'V and Q = C + F'W, for n=16, m=4 (p=20) with mma.sync.m16n8k8 TF32 in three
// passes (3xTF32: hi*hi + hi*lo + lo*hi, fp32 accumulate), ONE problem per warp, operands loaded once
// per warp into fragments.  Checks accuracy against a double-precision host result and times the
// steady-state cost per problem-step.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -o tools/mma_probe tools/mma_probe.cu
#include <cuda_runtime.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>

constexpr int N = 16, M = 4, P = 20;

__device__ __forceinline__ void split(float x, unsigned& hi, unsigned& lo) {
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(hi) : "f"(x));
  const float r = x - __uint_as_float(hi);
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(lo) : "f"(r));
}
__device__ __forceinline__ void mma(float (&d)[4], const unsigned (&a)[4], const unsigned (&b)[2]) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
__device__ __forceinline__ void mma3(float (&d)[4], const unsigned (&ah)[4], const unsigned (&al)[4],
                                     const unsigned (&bh)[2], const unsigned (&bl)[2]) {
  mma(d, al, bh);
  mma(d, ah, bl);
  mma(d, ah, bh);
}

// one warp = one problem; `reps` repetitions of the two products (results summed into Q to keep them live)
__global__ void __launch_bounds__(128) probe(const float* __restrict__ gV, const float* __restrict__ gF,
                                             const float* __restrict__ gC, float* __restrict__ gQ, int B, int reps) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= B) return;
  const int g = lane >> 2, t = lane & 3;
  const float* V = gV + (size_t)warp * N * N;
  const float* F = gF + (size_t)warp * N * P;
  const float* C = gC + (size_t)warp * P * P;
  // A fragments of F' (rows a = mt*16 + g (+8), cols k = ks*8 + t (+4)):  F'[a][k] = F[k][a]
  unsigned Ah[2][2][4], Al[2][2][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int a = mt * 16 + g + (r & 1) * 8, k = ks * 8 + t + (r >> 1) * 4;
        split(a < P ? F[k * P + a] : 0.f, Ah[mt][ks][r], Al[mt][ks][r]);
      }
  // B fragments of V (k = ks*8 + t (+4), n = nt*8 + g)
  unsigned Vh[2][2][2], Vl[2][2][2];
#pragma unroll
  for (int ks = 0; ks < 2; ++ks)
#pragma unroll
    for (int nt = 0; nt < 2; ++nt)
#pragma unroll
      for (int r = 0; r < 2; ++r) split(V[(ks * 8 + t + r * 4) * N + nt * 8 + g], Vh[ks][nt][r], Vl[ks][nt][r]);
  float Qacc[2][3][4];
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 3; ++nt)
#pragma unroll
      for (int r = 0; r < 4; ++r) Qacc[mt][nt][r] = 0.f;

  for (int rep = 0; rep < reps; ++rep) {
    // ---- step 1: W'[a][i] = sum_k F'[a][k] V[k][i]
    float Wt[2][2][4];
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 2; ++nt) {
#pragma unroll
        for (int r = 0; r < 4; ++r) Wt[mt][nt][r] = 0.f;
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) mma3(Wt[mt][nt], Ah[mt][ks], Al[mt][ks], Vh[ks][nt], Vl[ks][nt]);
      }
    // ---- D -> B re-layout: B2[ks][nt] = { W[ks*8+t][nt*8+g], W[ks*8+t+4][nt*8+g] },  W[k][b] = W'[b][k]
    unsigned Wh[2][3][2], Wl[2][3][2];
#pragma unroll
    for (int ks = 0; ks < 2; ++ks)
#pragma unroll
      for (int nt = 0; nt < 3; ++nt) {
        const int mt = nt >> 1, hi8 = (nt & 1) * 2;      // rows nt*8+g of W' live in tile mt, regs c(hi8 + parity)
#pragma unroll
        for (int r = 0; r < 2; ++r) {
          const int src = (lane & ~3) | ((t + r * 4) >> 1);
          const float xe = __shfl_sync(0xffffffffu, Wt[mt][ks][hi8 + 0], src);
          const float xo = __shfl_sync(0xffffffffu, Wt[mt][ks][hi8 + 1], src);
          split((t & 1) ? xo : xe, Wh[ks][nt][r], Wl[ks][nt][r]);
        }
      }
    // ---- step 2: Q[a][b] = C[a][b] + sum_k F'[a][k] W[k][b]
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
      for (int nt = 0; nt < 3; ++nt) {
        float acc[4];
#pragma unroll
        for (int r = 0; r < 4; ++r) {
          const int a = mt * 16 + g + (r >> 1) * 8, b = nt * 8 + 2 * t + (r & 1);
          acc[r] = (a < P && b < P) ? C[a * P + b] : 0.f;
        }
#pragma unroll
        for (int ks = 0; ks < 2; ++ks) mma3(acc, Ah[mt][ks], Al[mt][ks], Wh[ks][nt], Wl[ks][nt]);
#pragma unroll
        for (int r = 0; r < 4; ++r) Qacc[mt][nt][r] += acc[r];
      }
  }
  float* Q = gQ + (size_t)warp * P * P;
#pragma unroll
  for (int mt = 0; mt < 2; ++mt)
#pragma unroll
    for (int nt = 0; nt < 3; ++nt)
#pragma unroll
      for (int r = 0; r < 4; ++r) {
        const int a = mt * 16 + g + (r >> 1) * 8, b = nt * 8 + 2 * t + (r & 1);
        if (a < P && b < P) Q[a * P + b] = Qacc[mt][nt][r] / reps;
      }
}

int main() {
  const int B = 4096;
  std::vector<float> V((size_t)B * N * N), F((size_t)B * N * P), C((size_t)B * P * P);
  srand(1);
  auto rnd = [] { return (float)rand() / RAND_MAX * 2.f - 1.f; };
  for (int b = 0; b < B; ++b) {
    std::vector<float> L(N * N);
    for (auto& v : L) v = rnd();
    for (int i = 0; i < N; ++i)
      for (int j = 0; j < N; ++j) {
        float s = i == j ? 1.f : 0.f;
        for (int k = 0; k < N; ++k) s += L[i * N + k] * L[j * N + k] / N;
        V[((size_t)b * N + i) * N + j] = s;
      }
  }
  for (auto& v : F) v = rnd();
  for (auto& v : C) v = rnd();
  float *dV, *dF, *dC, *dQ;
  cudaMalloc(&dV, V.size() * 4); cudaMalloc(&dF, F.size() * 4); cudaMalloc(&dC, C.size() * 4);
  cudaMalloc(&dQ, C.size() * 4);
  cudaMemcpy(dV, V.data(), V.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(dF, F.data(), F.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(dC, C.data(), C.size() * 4, cudaMemcpyHostToDevice);
  probe<<<B / 4, 128>>>(dV, dF, dC, dQ, B, 1);
  std::vector<float> Q(C.size());
  cudaMemcpy(Q.data(), dQ, Q.size() * 4, cudaMemcpyDeviceToHost);
  double maxerr = 0, maxref = 0, maxerr32 = 0;
  for (int b = 0; b < 64; ++b) {
    const float *v = &V[(size_t)b * N * N], *f = &F[(size_t)b * N * P], *c = &C[(size_t)b * P * P];
    for (int a = 0; a < P; ++a)
      for (int bb = 0; bb < P; ++bb) {
        double s = c[a * P + bb];
        float s32 = c[a * P + bb];
        for (int k = 0; k < N; ++k) {
          double w = 0;
          float w32 = 0;
          for (int i = 0; i < N; ++i) { w += (double)v[k * N + i] * f[i * P + bb]; w32 += v[k * N + i] * f[i * P + bb]; }
          s += (double)f[k * P + a] * w;
          s32 += f[k * P + a] * w32;
        }
        maxerr = fmax(maxerr, fabs(Q[((size_t)b * P + a) * P + bb] - s));
        maxerr32 = fmax(maxerr32, fabs((double)s32 - s));
        maxref = fmax(maxref, fabs(s));
      }
  }
  printf("accuracy: max|Q_mma3xtf32 - Q_f64| = %.3e  (plain fp32 loop: %.3e, max|Q| = %.2f)\n", maxerr, maxerr32, maxref);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int reps : {50, 200}) {
    probe<<<B / 4, 128>>>(dV, dF, dC, dQ, B, reps);
    cudaEventRecord(e0);
    probe<<<B / 4, 128>>>(dV, dF, dC, dQ, B, reps);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    printf("reps=%d: %.1f us total, %.3f us per step-round of %d problems (60 mma.sync + 24 shfl per problem-step)\n",
           reps, ms * 1e3, ms * 1e3 / reps, B);
  }
  printf("cuda status: %s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
