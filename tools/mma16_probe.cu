// mma16_probe.cu - checks tools/mma16.cuh (F'VF and F'v of an n=16 problem by mma.sync 3xTF32 with the permuted
// contraction slots) against a double-precision host loop, and times it.  Not part of the product.
//   nvcc -O3 -std=c++17 -gencode arch=compute_90a,code=sm_90a -I mpc/pytorch_b200/csrc -I tools -o tools/mma16_probe tools/mma16_probe.cu
#include <cuda_runtime.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "mma16.cuh"

constexpr int N = 16, P = 20;

__global__ void __launch_bounds__(32) probe(const float* gV, const float* gF, const float* gv, float* gQ, float* gq, int reps) {
  __shared__ __align__(16) float sF[N * P], sV[N * N], sv[N], sQ[P * P], sq[P];
  const int b = blockIdx.x, lane = threadIdx.x;
  for (int i = lane; i < N * P; i += 32) sF[i] = gF[(size_t)b * N * P + i];
  for (int i = lane; i < N * N; i += 32) sV[i] = gV[(size_t)b * N * N + i];
  if (lane < N) sv[lane] = gv[(size_t)b * N + lane];
  __syncwarp();
  for (int r = 0; r < reps; ++r) {
    mpcb200::ftvf_16<P, N>(sF, sV, sv, sQ, sq, lane);
    __syncwarp();
  }
  for (int i = lane; i < P * P; i += 32) gQ[(size_t)b * P * P + i] = sQ[i];
  if (lane < P) gq[(size_t)b * P + lane] = sq[lane];
}

int main() {
  const int B = 4096;
  std::vector<float> V((size_t)B * N * N), F((size_t)B * N * P), v((size_t)B * N);
  srand(1);
  auto rnd = [] { return (float)rand() / RAND_MAX * 2.f - 1.f; };
  for (auto& x : V) x = rnd();                     // V need not be symmetric for the check
  for (auto& x : F) x = rnd();
  for (auto& x : v) x = rnd();
  float *dV, *dF, *dv, *dQ, *dq;
  cudaMalloc(&dV, V.size() * 4); cudaMalloc(&dF, F.size() * 4); cudaMalloc(&dv, v.size() * 4);
  cudaMalloc(&dQ, (size_t)B * P * P * 4); cudaMalloc(&dq, (size_t)B * P * 4);
  cudaMemcpy(dV, V.data(), V.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(dF, F.data(), F.size() * 4, cudaMemcpyHostToDevice);
  cudaMemcpy(dv, v.data(), v.size() * 4, cudaMemcpyHostToDevice);
  probe<<<B, 32>>>(dV, dF, dv, dQ, dq, 1);
  std::vector<float> Q((size_t)B * P * P), q((size_t)B * P);
  cudaMemcpy(Q.data(), dQ, Q.size() * 4, cudaMemcpyDeviceToHost);
  cudaMemcpy(q.data(), dq, q.size() * 4, cudaMemcpyDeviceToHost);
  double eQ = 0, eq = 0, mQ = 0, asym = 0;
  for (int b = 0; b < 64; ++b) {
    const float *vm = &V[(size_t)b * N * N], *f = &F[(size_t)b * N * P], *vv = &v[(size_t)b * N];
    for (int a = 0; a < P; ++a) {
      double sq = 0;
      for (int k = 0; k < N; ++k) sq += (double)f[k * P + a] * vv[k];
      eq = fmax(eq, fabs(q[(size_t)b * P + a] - sq));
      for (int c = 0; c < P; ++c) {
        double s = 0;                              // upper block triangle is computed, the rest mirrored
        const int ra = (a >= 16 && c < 16) ? c : a, rc = (a >= 16 && c < 16) ? a : c;
        for (int j = 0; j < N; ++j) {
          double w = 0;
          for (int k = 0; k < N; ++k) w += (double)vm[j * N + k] * f[k * P + rc];
          s += (double)f[j * P + ra] * w;
        }
        eQ = fmax(eQ, fabs(Q[((size_t)b * P + a) * P + c] - s));
        mQ = fmax(mQ, fabs(s));
      }
    }
  }
  printf("accuracy: max|Q' - f64| = %.3e (max|Q'| = %.2f)   max|q' - f64| = %.3e\n", eQ, mQ, eq);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int reps : {50, 200}) {
    probe<<<B, 32>>>(dV, dF, dv, dQ, dq, reps);
    cudaEventRecord(e0);
    probe<<<B, 32>>>(dV, dF, dv, dQ, dq, reps);
    cudaEventRecord(e1);
    cudaEventSynchronize(e1);
    float ms;
    cudaEventElapsedTime(&ms, e0, e1);
    printf("reps=%d: %.3f us per round of %d problems (48 mma.sync per problem, fragments reloaded every round)\n", reps,
           ms * 1e3 / reps, B);
  }
  printf("cuda status: %s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
