// What a CUDA-event pair around ONE launch costs on this box, as a function of grid size, dynamic shared memory and the state
// of L2 (flushed by a 512 MiB memset + read beforehand, as bench.py does, or left alone); and what back-to-back launches cost.
// nvcc -arch=sm_90a -O3 -o launch_floor launch_floor.cu && ./launch_floor
#include <cstdio>
#include <cuda_runtime.h>
#include <algorithm>
#include <vector>
__global__ void k_empty(int* p) { if (p && threadIdx.x == 12345) *p = 1; }
__global__ void k_touch(const int* __restrict__ src, int* dst, int n) {  // every CTA reads 512 B and writes 4
  extern __shared__ int sm[];
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int v = i < n ? src[i] : 0;
  if (v == 0x7fffffff) dst[i] = v;
}
__global__ void k_read(const long long* p, long long n, long long* out) {
  long long acc = 0;
  for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) acc += p[i];
  if (acc == 0x7fffffffffffffffll) *out = acc;
}
int main() {
  cudaStream_t s; cudaStreamCreate(&s);
  char *flush, *drain; int *src, *dst; long long* out;
  const size_t FL = 512u << 20;
  cudaMalloc(&flush, FL); cudaMalloc(&drain, FL); cudaMalloc(&src, 1 << 22); cudaMalloc(&dst, 1 << 22); cudaMalloc(&out, 8);
  cudaMemset(drain, 0, FL); cudaMemset(src, 0, 1 << 22);
  cudaEvent_t a, b; cudaEventCreate(&a); cudaEventCreate(&b);
  cudaFuncSetAttribute(k_empty, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 << 10);
  cudaFuncSetAttribute(k_touch, cudaFuncAttributeMaxDynamicSharedMemorySize, 64 << 10);
  for (int flushed = 0; flushed < 2; ++flushed)
    for (int smem : {0, 24 << 10, 34 << 10})
      for (int grid : {132, 396, 792, 1003, 2000}) {
        for (int kind = 0; kind < 2; ++kind) {
          std::vector<float> t;
          for (int it = 0; it < 30; ++it) {
            if (flushed) { cudaMemsetAsync(flush, it, FL, s); k_read<<<1184, 256, 0, s>>>((const long long*)drain, FL / 8, out); }
            cudaEventRecord(a, s);
            if (kind == 0) k_empty<<<grid, 128, smem, s>>>(nullptr);
            else k_touch<<<grid, 128, smem, s>>>(src, dst, 1 << 20);
            cudaEventRecord(b, s);
            cudaStreamSynchronize(s);
            float ms; cudaEventElapsedTime(&ms, a, b);
            if (it >= 5) t.push_back(ms * 1e3f);
          }
          std::sort(t.begin(), t.end());
          printf("%s L2  smem %5d  grid %4d  %s  median %.2f us  min %.2f\n", flushed ? "flushed" : "warm   ", smem, grid, kind ? "touch" : "empty", t[t.size() / 2], t[0]);
        }
      }
  // back to back: K launches between one event pair
  for (int grid : {132, 1003}) {
    cudaEventRecord(a, s);
    for (int i = 0; i < 200; ++i) k_touch<<<grid, 128, 24 << 10, s>>>(src, dst, 1 << 20);
    cudaEventRecord(b, s);
    cudaStreamSynchronize(s);
    float ms; cudaEventElapsedTime(&ms, a, b);
    printf("back-to-back grid %4d: %.2f us per launch\n", grid, ms * 1e3f / 200);
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
