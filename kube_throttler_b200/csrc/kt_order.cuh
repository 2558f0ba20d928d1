// kt_order.cuh -- row order of a pod table: the rows clustered by namespace on the device (DESIGN.md "Row order").
//
// A warp of the pass costs far more when its 32 rows belong to many namespaces than when they share one (every namespace
// brings its own word list).  A caller that cannot keep its rows namespace-clustered uploads them in arrival order; the
// engine then stores them sorted by namespace -- a stable LSD radix sort of the keys
//   key(row) = ns(row)  if 0 <= ns(row) < n_ns,  else n_ns  (every row outside the namespaces forms one group at the end)
// over only the 8-bit digits the largest possible key has -- and keeps two maps per table: caller_of[device row] and
// dev_of[caller row].  Every row number that crosses the ABI is the caller's; the maps translate at the boundary.
#pragma once
#include "kt_kernels.cuh"

namespace kt {

constexpr int kOrderThreads = 256;                 // threads of a sort block (8 warps)
constexpr int kOrderItems = 8;                     // rows per thread: every warp sorts 8 runs of 32 consecutive rows
constexpr int kOrderTile = kOrderThreads * kOrderItems;  // rows per sort block
constexpr int kOrderDigits = 256;                  // 8-bit digits

__device__ __forceinline__ uint32_t order_key(int32_t ns, uint32_t n_ns) { return (uint32_t)ns < n_ns ? (uint32_t)ns : n_ns; }

// keys of the caller's rows and the identity permutation the passes start from
__global__ void __launch_bounds__(256) k_order_keys(int64_t n, const int32_t* __restrict__ ns, uint32_t n_ns, uint32_t* __restrict__ keys,
                                                    uint32_t* __restrict__ vals) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  keys[i] = order_key(__ldg(&ns[i]), n_ns);
  vals[i] = (uint32_t)i;
}

// per sort block: how many of its rows carry each digit -> hist[digit * nblk + block] (digit-major, so that one exclusive scan
// over the whole array gives every (digit, block) its first output position)
__global__ void __launch_bounds__(kOrderThreads) k_order_hist(int64_t n, const uint32_t* __restrict__ keys, int shift, uint32_t* __restrict__ hist, int nblk) {
  __shared__ uint32_t s_h[kOrderDigits];
  for (int d = threadIdx.x; d < kOrderDigits; d += blockDim.x) s_h[d] = 0u;
  __syncthreads();
  const int64_t lo = (int64_t)blockIdx.x * kOrderTile;
  const int64_t hi = lo + kOrderTile < n ? lo + kOrderTile : n;
  for (int64_t i = lo + threadIdx.x; i < hi; i += blockDim.x) atomicAdd(&s_h[(__ldg(&keys[i]) >> shift) & 255u], 1u);
  __syncthreads();
  for (int d = threadIdx.x; d < kOrderDigits; d += blockDim.x) hist[(size_t)d * nblk + blockIdx.x] = s_h[d];
}

// exclusive scan of hist[len], one CTA
__global__ void __launch_bounds__(1024) k_order_scan(uint32_t* __restrict__ hist, int64_t len) {
  __shared__ uint32_t s_part[1024];
  const int tid = threadIdx.x;
  const int64_t per = (len + 1023) / 1024;
  const int64_t lo = tid * per, hi = lo + per < len ? lo + per : len;
  uint32_t sum = 0;
  for (int64_t j = lo; j < hi; ++j) sum += hist[j];
  s_part[tid] = sum;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {
    const uint32_t x = tid >= d ? s_part[tid - d] : 0u;
    __syncthreads();
    s_part[tid] += x;
    __syncthreads();
  }
  uint32_t run = tid ? s_part[tid - 1] : 0u;
  for (int64_t j = lo; j < hi; ++j) {
    const uint32_t c = hist[j];
    hist[j] = run;
    run += c;
  }
}

// One stable counting pass over the digit at `shift`.  Warp w of a block owns the block's rows [w * 256, (w + 1) * 256) and
// walks them in 8 runs of 32, in order: lanes with the same digit rank themselves by lane (__match_any_sync), the run's leader
// advances the warp's count of that digit.  The warps' counts then become positions: the block's first position for the
// digit (the scanned histogram) plus the counts of the warps before.  Rows with equal digits keep their order.
__global__ void __launch_bounds__(kOrderThreads) k_order_scatter(int64_t n, const uint32_t* __restrict__ keys_in, const uint32_t* __restrict__ vals_in, int shift,
                                                                 const uint32_t* __restrict__ first, int nblk, uint32_t* __restrict__ keys_out,
                                                                 uint32_t* __restrict__ vals_out) {
  constexpr int kWarps = kOrderThreads / 32;
  __shared__ uint32_t s_cnt[kWarps][kOrderDigits];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int j = tid; j < kWarps * kOrderDigits; j += kOrderThreads) (&s_cnt[0][0])[j] = 0u;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * kOrderTile + (int64_t)warp * 32 * kOrderItems;
  const uint32_t below = (1u << lane) - 1u;
  uint32_t key[kOrderItems], val[kOrderItems], rank[kOrderItems];
  int dig[kOrderItems];
#pragma unroll
  for (int it = 0; it < kOrderItems; ++it) {
    const int64_t i = base + it * 32 + lane;
    const bool on = i < n;
    key[it] = on ? __ldg(&keys_in[i]) : 0u;
    val[it] = on ? __ldg(&vals_in[i]) : 0u;
    dig[it] = on ? (int)((key[it] >> shift) & 255u) : kOrderDigits;  // lanes past the end share a digit no row has
    const uint32_t same = __match_any_sync(kFull, dig[it]);
    const int leader = __ffs(same) - 1;
    uint32_t before = 0u;
    if (on && lane == leader) {
      before = s_cnt[warp][dig[it]];
      s_cnt[warp][dig[it]] = before + __popc(same);
    }
    before = __shfl_sync(kFull, before, leader);
    rank[it] = before + __popc(same & below);
    __syncwarp();
  }
  __syncthreads();
  for (int d = tid; d < kOrderDigits; d += kOrderThreads) {
    uint32_t run = first[(size_t)d * nblk + blockIdx.x];
#pragma unroll
    for (int w = 0; w < kWarps; ++w) {
      const uint32_t c = s_cnt[w][d];
      s_cnt[w][d] = run;
      run += c;
    }
  }
  __syncthreads();
#pragma unroll
  for (int it = 0; it < kOrderItems; ++it) {
    if (dig[it] == kOrderDigits) continue;
    const uint32_t pos = s_cnt[warp][dig[it]] + rank[it];
    keys_out[pos] = key[it];
    vals_out[pos] = val[it];
  }
}

// dev_of[caller_of[j]] = j
__global__ void __launch_bounds__(256) k_order_invert(int64_t n, const uint32_t* __restrict__ caller_of, uint32_t* __restrict__ dev_of) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j < n) dev_of[__ldg(&caller_of[j])] = (uint32_t)j;
}

// Column-major row columns into the clustered order: dst[c][j] = src[c][map[j]] for cols columns of n rows (one lane per
// element; the writes are coalesced).  With map = caller_of this lays the caller's rows out by namespace; with map = dev_of it
// brings per-row device results back into the caller's order.
template <class T>
__global__ void __launch_bounds__(256) k_order_gather_cols(int64_t n, int cols, const uint32_t* __restrict__ map, const T* __restrict__ src, T* __restrict__ dst) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n * cols) return;
  const int64_t c = e / n, j = e - c * n;
  dst[e] = src[c * n + __ldg(&map[j])];
}

// Row-major result rows (bitmaps, code rows) in the caller's order: dst[j][w] = src[map[j]][w] for rows of W words.
__global__ void __launch_bounds__(256) k_order_gather_rows(int64_t n, int W, const uint32_t* __restrict__ map, const uint32_t* __restrict__ src,
                                                           uint32_t* __restrict__ dst) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n * W) return;
  const int64_t j = e / W, w = e - j * W;
  dst[e] = src[(int64_t)__ldg(&map[j]) * W + w];
}

// k caller rows -> device rows, in place (the host has checked the range)
__global__ void __launch_bounds__(256) k_order_map_rows(int64_t k, const uint32_t* __restrict__ dev_of, int64_t* __restrict__ rows) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < k) rows[i] = __ldg(&dev_of[rows[i]]);
}

// The row field of the sparse check entries the pass appended -> caller rows, once per pass (the entries stay unordered).
__global__ void __launch_bounds__(256) k_order_sparse_rows(const uint32_t* __restrict__ count, uint32_t cap, uint32_t* __restrict__ ent,
                                                           const uint32_t* __restrict__ caller_of) {
  const uint32_t c = *count, have = c < cap ? c : cap;
  for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < have; i += gridDim.x * blockDim.x) ent[3 * (size_t)i] = __ldg(&caller_of[ent[3 * (size_t)i]]);
}

}  // namespace kt
