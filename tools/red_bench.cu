// Microbenchmark: cost of fire-and-forget red.global.add.v4.f32 traffic (decides how the blend adjoint
// combines per-block partial sums).  nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o red_bench red_bench.cu
#include <cstdio>
#include <cuda_runtime.h>
__global__ void k(float* acc, int n_rec, long long total, unsigned seed) {
  long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  long long stride = (long long)gridDim.x * blockDim.x;
  for (; i < total; i += stride) {
    unsigned h = (unsigned)(i >> 2) * 2654435761u + seed;   // 4 consecutive quarters of one pseudo-random record
    unsigned rec = h % (unsigned)n_rec;
    float* p = acc + (size_t)rec * 16 + (i & 3) * 4;
    asm volatile("red.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(1.f), "f"(2.f), "f"(3.f), "f"(4.f) : "memory");
  }
}
int main() {
  const int n_rec = 360000;
  float* acc; cudaMalloc(&acc, (size_t)n_rec * 64); cudaMemset(acc, 0, (size_t)n_rec * 64);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  for (long long total : {9000000LL, 27000000LL, 54000000LL}) {
    k<<<132 * 8, 256>>>(acc, n_rec, total, 1u);
    cudaEventRecord(a);
    for (int r = 0; r < 5; r++) k<<<132 * 8, 256>>>(acc, n_rec, total, r);
    cudaEventRecord(b); cudaEventSynchronize(b);
    float ms; cudaEventElapsedTime(&ms, a, b);
    printf("vector REDs %lld: %.1f us per launch (%.2f G red/s)\n", total, ms / 5 * 1e3, total / (ms / 5 * 1e-3) / 1e9);
  }
  return 0;
}
