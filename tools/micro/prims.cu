// Latency (SM cycles, %clock64) of the building blocks of the pass's hand-offs, one warp of one CTA on an otherwise idle GPU
// and again with every other SM streaming from HBM: relaxed / acquire loads from L2, fences, returning atomics, nanosleep,
// a CTA barrier, a 3 KB bulk copy (cp.async.bulk + mbarrier) against the same bytes fetched with LDG.128, LDS chains.
// nvcc -arch=sm_90a -O3 -o prims prims.cu && ./prims
#include <cstdio>
#include <cuda_runtime.h>
#include <stdint.h>
__device__ __forceinline__ long long clk() { long long t; asm volatile("mov.u64 %0, %%clock64;" : "=l"(t) :: "memory"); return t; }
__device__ __forceinline__ unsigned ld_relaxed(const unsigned* p) { unsigned v; asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ unsigned ld_acquire(const unsigned* p) { unsigned v; asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory"); return v; }
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
constexpr int NREP = 16, NOPS = 14;
__global__ void k_prims(unsigned* g, const uint4* blob, long long* out, int busy_other) {
  __shared__ __align__(128) unsigned char buf[4096];
  __shared__ __align__(8) unsigned long long bar;
  __shared__ long long res[NOPS];
  if (blockIdx.x != 0) {  // background traffic
    if (!busy_other) return;
    const uint4* p = blob + 1024;
    uint4 acc = make_uint4(0, 0, 0, 0);
    for (long long i = (blockIdx.x * 256ll + threadIdx.x); i < (1ll << 24); i += (long long)(gridDim.x - 1) * 256) { uint4 v = p[i]; acc.x ^= v.x; acc.y ^= v.y; }
    if (acc.x == 0x12345 && acc.y == 0x54321) g[100] = 1;
    return;
  }
  const int tid = threadIdx.x;
  if (tid == 0) { asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_addr(&bar)) : "memory"); asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
  __syncthreads();
  long long t0, t1; unsigned sink = 0;
  for (int op = 0; op < NOPS; ++op) {
    long long best = 1ll << 60;
    for (int rep = 0; rep < NREP; ++rep) {
      __syncthreads();
      t0 = clk();
      switch (op) {
        case 0: if (tid == 0) sink += ld_relaxed(g + 32 * rep); break;                                   // L2 trip
        case 1: if (tid == 0) sink += ld_acquire(g + 32 * rep); break;                                   // + CCTL.IVALL
        case 2: if (tid == 0) { sink += ld_relaxed(g + 32 * rep); asm volatile("fence.acq_rel.gpu;" ::: "memory"); } break;
        case 3: if (tid == 0) __threadfence(); break;
        case 4: if (tid == 0) sink += atomicAdd(g + 1024 + rep, 1u); break;                               // returning atomic
        case 5: if (tid == 0) __nanosleep(40); break;
        case 6: __syncthreads(); break;
        case 7: if (tid == 0) {                                                                          // 3 KB bulk copy
          asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_addr(&bar)), "r"(3072) : "memory");
          asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_addr(buf)), "l"(blob + 256 * rep), "r"(3072), "r"(smem_addr(&bar)) : "memory");
          unsigned done = 0;
          while (!done) asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }" : "=r"(done) : "r"(smem_addr(&bar)), "r"(rep & 1) : "memory");
          sink += buf[5];
        } break;
        case 8: if (tid < 32) { for (int q = 0; q < 6; ++q) { uint4 v = __ldcg(blob + 8192 + 256 * rep + q * 32 + tid); reinterpret_cast<uint4*>(buf)[q * 32 + tid] = v; } __syncwarp(); sink += buf[5]; } break;  // the same 3 KB per-lane
        case 9: if (tid == 0) { unsigned i = buf[0] & 63; for (int q = 0; q < 8; ++q) i = buf[64 + (i & 63) * 4] + q; sink += i; } break;  // 8 dependent LDS
        case 10: if (tid == 0) { sink += ld_relaxed(g + 32 * rep); sink += ld_relaxed(g + 32 * rep + 4096); } break;  // two independent trips
        case 11: if (tid == 0) { unsigned v = ld_relaxed(g + 32 * rep); sink += ld_relaxed(g + 8192 + (v & 1) * 32); } break;  // two dependent trips
        case 12: if (tid == 0) atomicAdd(g + 2048 + rep, 1u); break;                                        // RED (no return)
        case 13: if (tid == 0) { __threadfence(); atomicAdd(g + 3072, 1u); } break;                          // signal
      }
      // make the result a dependency of the clock read
      if (sink == 0xdeadbeef) g[200] = sink;
      t1 = clk();
      if (rep >= 4 && t1 - t0 < best) best = t1 - t0;
    }
    if (tid == 0) res[op] = best;
  }
  __syncthreads();
  if (tid == 0) for (int op = 0; op < NOPS; ++op) out[op] = res[op];
  if (sink == 0xdeadbeef) g[201] = sink;
}
int main() {
  unsigned* g; uint4* blob; long long* out;
  cudaMalloc(&g, 1 << 20); cudaMemset(g, 0, 1 << 20);
  cudaMalloc(&blob, (1ll << 28) + (1 << 20)); cudaMemset(blob, 1, (1ll << 28) + (1 << 20));
  cudaMalloc(&out, 8 * NOPS);
  const char* names[NOPS] = {"ld.relaxed.gpu (L2 trip)", "ld.acquire.gpu", "ld.relaxed + fence.acq_rel.gpu", "__threadfence", "atomicAdd returning", "__nanosleep(40)",
                             "__syncthreads (128 thr)", "bulk copy 3 KB + mbarrier wait", "3 KB by one warp, LDG.128 + STS", "8 dependent LDS", "2 independent L2 trips",
                             "2 dependent L2 trips", "RED.ADD", "__threadfence + RED (signal)"};
  for (int busy = 0; busy < 2; ++busy) {
    k_prims<<<busy ? 132 * 4 : 1, busy ? 256 : 128>>>(g, blob, out, busy);
    cudaError_t e = cudaDeviceSynchronize();
    if (e != cudaSuccess) { printf("error %s\n", cudaGetErrorString(e)); return 1; }
    long long h[NOPS]; cudaMemcpy(h, out, sizeof h, cudaMemcpyDeviceToHost);
    printf("--- %s (cycles, best of %d; clock overhead included) ---\n", busy ? "other SMs streaming from HBM" : "idle GPU", NREP - 4);
    for (int op = 0; op < NOPS; ++op) printf("%-36s %6lld\n", names[op], h[op]);
  }
  return 0;
}
