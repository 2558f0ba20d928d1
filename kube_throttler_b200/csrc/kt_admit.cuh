// kt_admit.cuh -- queue-ordered greedy admission on the device (SURVEY.md 8f.2).
//
// The scheduler admits one pod per cycle: PreFilter, and on Success Reserve, so every admitted pod raises the reserved
// amounts the NEXT pod is checked against (plugin.go:148-238; reservedResourceAmounts.addPod,
// reserved_resource_amounts.go:66-77,113-136).  For a SORTED queue of pending rows that sequence is reproduced exactly,
// without walking the queue pod by pod:
//
//   * a throttle's view of the queue is its TOUCHER LIST: the queue positions whose pod it affects, ascending (a CSR built
//     once from the pending match bitmap: ColumnView below);
//   * the load pod i sees on throttle t is the sum of the requests of the ADMITTED pods before i in t's list -- an exclusive
//     prefix sum along the list;
//   * which pods are admitted is the unknown.  Every pod is Undecided, Admitted or surely-reJected.  One round computes, for
//     every (pod, throttle) pair, the check under the smallest load it can still see and the largest: every earlier Admitted
//     pod adds its request to both, every earlier Undecided pod adds min(v, 0) to the smallest and max(v, 0) to the largest
//     (requests may be negative), its presence bits and its pod count to the largest only.  CheckThrottledFor is monotone
//     in each resource's load and presence separately (S3 / S4 only ever turn true as used + reserved grows; S1 / S2 do not
//     look at it), so a pod that passes all its pairs under the LARGEST load is admitted whatever the pods before it do, and
//     a pod that fails a pair under the SMALLEST load is rejected whatever they do.  Rounds repeat until nobody is
//     Undecided; the first undecided pod of the queue sees equal bounds, so every round decides somebody, and pods on
//     disjoint throttles are decided together.  A last round, with
//     every load exact, writes the 2-bit codes each rejected pod saw at its turn.
//
// Typical queues settle in 2-4 rounds (a throttle with room for 300 of 1000 queued pods: round 1 admits the 300, round 2
// rejects the rest); each round is two launches and costs the host one 4-byte read.
#pragma once
#include "kt_kernels.cuh"

namespace kt {

constexpr int kColBlock = 1024;  // rows per counting block of a row-list build
constexpr uint8_t kUndecided = 0, kAdmitted = 1, kRejected = 2;

// ---- per-throttle row lists: the match relation transposed ---------------------------------------------------------
// For k listed throttles (duplicates allowed; idx == nullptr lists 0..k-1), the rows i in [0, count) whose bit of
// bitmap row first + i is set, ascending, as one CSR: entry j's rows are rows[off[j] .. off[j+1]).  Four launches:
// per-(block, entry) counts, per-entry block offsets and lengths, an exclusive scan of the lengths, the fill.  A warp
// walks one block of kColBlock rows for 32 consecutive entries, 32 rows at a time (lane = row): the word of an entry's
// throttle is loaded once per run of entries that share it, and a ballot per entry counts (and in the fill places)
// the rows in lane order.  Only the words of the listed throttles are read.  kt_admit_queue builds its toucher lists
// with it (all throttles over the queue rows), kt_get_match_columns the columns it is asked for (all rows).
struct ColumnView {
  const uint32_t* bitmap;  // [n][Wp]
  int Wp;
  int64_t first, count;    // the rows walked: [first, first + count); list entries hold i = row - first
  const int32_t* idx;      // [k] or nullptr
  int64_t k;
  int nblk;                // ceil(count / kColBlock)
  int32_t* cnt;            // [nblk][k] set bits per (block, entry); after k_col_lengths: the block's offset in the entry's list
  int64_t* off;            // [k + 1]
  int64_t* rows;           // [off[k]]
  const uint32_t* codes;   // [n][2Wp] 2-bit codes to gather beside the rows, or nullptr
  uint8_t* codes_out;      // [off[k]]
  const uint32_t* rowmap;  // caller row -> bitmap row of a table laid out by namespace (kt_order.cuh), or nullptr: the same row
};

template <bool FILL>
__device__ __forceinline__ void col_walk(const ColumnView& v) {
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  const int64_t groups = (v.k + 31) >> 5;
  if (warp >= (int64_t)v.nblk * groups) return;
  const int blk = (int)(warp / groups);
  const int64_t e0 = (warp % groups) * 32;
  const int ne = v.k - e0 < 32 ? (int)(v.k - e0) : 32;
  const int my_t = lane < ne ? (v.idx ? v.idx[e0 + lane] : (int)(e0 + lane)) : 0;
  const int64_t lo = (int64_t)blk * kColBlock, hi = lo + kColBlock < v.count ? lo + kColBlock : v.count;
  // count: this lane's entry's set bits so far; fill: where its next row goes
  int64_t at = 0;
  if (FILL && lane < ne) at = v.off[e0 + lane] + v.cnt[(size_t)blk * v.k + e0 + lane];
  const uint32_t below = (1u << lane) - 1u;
  for (int64_t base = lo; base < hi; base += 32) {
    const int64_t i = base + lane;
    const bool on = i < hi;
    const int64_t p = !v.rowmap ? v.first + i : on ? (int64_t)__ldg(&v.rowmap[v.first + i]) : 0;
    int wcur = -1;
    uint32_t x = 0u;
    for (int e = 0; e < ne; ++e) {
      const int t = __shfl_sync(kFull, my_t, e);
      if ((t >> 5) != wcur) {  // uniform: every lane sees the same t
        wcur = t >> 5;
        x = on ? __ldg(&v.bitmap[p * v.Wp + wcur]) : 0u;
      }
      const bool bit = (x >> (t & 31)) & 1u;
      const uint32_t m = __ballot_sync(kFull, bit);
      if (FILL) {
        const int64_t pos = __shfl_sync(kFull, at, e) + __popc(m & below);
        if (bit) {
          v.rows[pos] = i;
          if (v.codes) v.codes_out[pos] = (uint8_t)((__ldg(&v.codes[p * 2 * v.Wp + (t >> 4)]) >> (2 * (t & 15))) & 3u);
        }
      }
      if (lane == e) at += __popc(m);
    }
  }
  if (!FILL && lane < ne) v.cnt[(size_t)blk * v.k + e0 + lane] = (int32_t)at;
}
__global__ void __launch_bounds__(128) k_col_count(ColumnView v) { col_walk<false>(v); }
// per entry: block counts -> block offsets inside the entry's list, and the list length
__global__ void __launch_bounds__(256) k_col_lengths(ColumnView v) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= v.k) return;
  int32_t run = 0;
  for (int b = 0; b < v.nblk; ++b) {
    const int32_t c = v.cnt[(size_t)b * v.k + j];
    v.cnt[(size_t)b * v.k + j] = run;
    run += c;
  }
  v.off[j + 1] = run;  // length for now
}
__global__ void __launch_bounds__(1024) k_col_starts(ColumnView v) {  // exclusive scan of the lengths, one CTA
  __shared__ long long s_part[1024];
  const int tid = threadIdx.x;
  const int64_t per = (v.k + 1023) / 1024;
  const int64_t lo = tid * per, hi = lo + per < v.k ? lo + per : v.k;
  long long sum = 0;
  for (int64_t j = lo; j < hi; ++j) sum += v.off[j + 1];
  s_part[tid] = sum;
  __syncthreads();
  for (int d = 1; d < 1024; d <<= 1) {
    const long long x = tid >= d ? s_part[tid - d] : 0;
    __syncthreads();
    s_part[tid] += x;
    __syncthreads();
  }
  long long run = tid ? s_part[tid - 1] : 0;
  if (tid == 0) v.off[0] = 0;
  for (int64_t j = lo; j < hi; ++j) {
    run += v.off[j + 1];
    v.off[j + 1] = run;
  }
}
// the lists themselves: the same walk as k_col_count, each set bit stored at its entry's next position
__global__ void __launch_bounds__(128) k_col_fill(ColumnView v) { col_walk<true>(v); }

// ---- queue-ordered greedy admission -----------------------------------------------------------------------------------
struct AdmitView {
  int64_t first, count;            // the queue: pending rows [first, first + count), in row order
  const int64_t* req;              // [R][n] pending request columns
  const uint32_t* present;         // [n]
  const uint32_t* bitmap;          // [n][Wp] affectedThrottles rows of the pending pods (a match pass ran)
  int64_t n;                       // rows of the pending table
  int Wp, W, M, R;
  const unsigned char* pre;        // [M] pre-records of a GIVEN_STATUS pass (thresholds, observed used + reserved, flags)
  const int64_t* tl_off;           // [M + 1] toucher lists (ColumnView over the queue, every throttle)
  const int64_t* tl_pod;           // [nnz] queue positions, ascending per throttle
  uint8_t* state;                  // [count]
  uint32_t* fail;                  // [count] bit 0: some pair fails under the largest load, bit 1: under the smallest
  uint32_t* codes;                 // [n][2Wp] (rows of the pending table)
  unsigned char* admit;            // [n]
  uint32_t* counters;              // [0] undecided pods after the last update, [1] admitted
  const uint32_t* rowmap;          // caller row -> row of the pending columns when they are laid out by namespace, or nullptr
};
// the pending row of queue position i: the queue is in caller rows
__device__ __forceinline__ int64_t admit_row(const AdmitView& a, int64_t i) { return a.rowmap ? (int64_t)a.rowmap[a.first + i] : a.first + i; }

// start of a round: every pod forgets last round's pair verdicts; the code words of its affected throttles are cleared (the
// pairs OR their codes back in)
__global__ void __launch_bounds__(256) k_admit_begin(AdmitView a) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.count) return;
  a.fail[i] = 0u;
  const int64_t p = admit_row(a, i);
  for (int w = 0; w < a.W; ++w)
    if (a.bitmap[p * a.Wp + w]) *reinterpret_cast<uint2*>(&a.codes[p * 2 * a.Wp + 2 * w]) = make_uint2(0u, 0u);
  if (i == 0) { a.counters[0] = 0u; a.counters[1] = 0u; }
}

__device__ __forceinline__ long long warp_excl_scan(long long v, int lane, long long* total) {
  long long x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const long long y = __shfl_up_sync(kFull, x, d);
    if (lane >= d) x += y;
  }
  *total = __shfl_sync(kFull, x, 31);
  return x - v;
}
__device__ __forceinline__ uint32_t warp_excl_or(uint32_t v, int lane, uint32_t* total) {
  uint32_t x = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t y = __shfl_up_sync(kFull, x, d);
    if (lane >= d) x |= y;
  }
  *total = __shfl_sync(kFull, x, 31);
  const uint32_t up = __shfl_up_sync(kFull, x, 1);
  return lane ? up : 0u;
}

// One round, one warp per throttle: walk the toucher list 32 positions at a time; exclusive prefix sums of the requests of the
// Admitted pods plus the negative (smallest load) or positive (largest load) requests of the Undecided ones give every pair
// its two loads; the pair is checked under both (the 4 steps of CheckThrottledFor, throttle_types.go:128-153 / clusterthrottle_types.go:30-55, GIVEN_STATUS
// constants from the pre-record).  RMAX bounds R at compile time for the register arrays.
template <int RMAX>
__global__ void __launch_bounds__(128) k_admit_round(AdmitView a) {
  const int t = (int)((blockIdx.x * (unsigned)blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (t >= a.M) return;
  const int64_t lo = a.tl_off[t], hi = a.tl_off[t + 1];
  if (lo == hi) return;
  const int R = a.R;
  const unsigned char* src = a.pre + (size_t)t * pre_record_bytes(R);
  const uint4 phq = *reinterpret_cast<const uint4*>(src);
  const long long* pv = reinterpret_cast<const long long*>(src + 16);  // thrv[R], base[R], thr_cnt, base_cnt
  PreHdr ph;
  ph.thr_has = phq.x; ph.base_has = phq.y; ph.st_thr = phq.z; ph.flags = phq.w;
  const bool live = ph.flags & kPreLive, e3 = ph.flags & kPreE3, on_equal = ph.flags & kPreOnEqual;
  long long thr[RMAX], base[RMAX];
#pragma unroll
  for (int r = 0; r < RMAX; ++r) {
    thr[r] = r < R ? pv[r] : 0;
    base[r] = r < R ? pv[R + r] : 0;
  }
  const long long thr_c = pv[2 * R], base_c = pv[2 * R + 1];
  // running loads of the positions already walked: [0] Admitted only, [1] Admitted + Undecided
  long long run[2][RMAX], run_c[2] = {0, 0};
  uint32_t run_pres[2] = {0u, 0u};
#pragma unroll
  for (int r = 0; r < RMAX; ++r) run[0][r] = run[1][r] = 0;

  for (int64_t at = lo; at < hi; at += 32) {
    const bool on = at + lane < hi;
    const int64_t i = on ? a.tl_pod[at + lane] : 0;
    const int64_t p = admit_row(a, i);
    const uint8_t st = on ? a.state[i] : kRejected;
    const uint32_t present = on ? a.present[p] : 0u;
    long long v[RMAX];
    uint32_t nz = 0;
#pragma unroll
    for (int r = 0; r < RMAX; ++r) {
      v[r] = (r < R && on && ((present >> r) & 1)) ? a.req[(int64_t)r * a.n + p] : 0;
      if (v[r] != 0) nz |= 1u << r;
    }
    const bool in0 = st == kAdmitted, in1 = st != kRejected, und = st == kUndecided;
    uint32_t code[2];
#pragma unroll
    for (int z = 0; z < 2; ++z) {
      const bool in = z ? in1 : in0;  // the pod's count and presence
      // what the pods before this position have reserved on the throttle (Reserve adds ResourceAmountOfPod: every request key
      // of the pod, zero or not, and Counts{Pod: 1})
      long long tot;
      uint32_t ptot;
      const long long e_c = run_c[z] + warp_excl_scan(in ? 1 : 0, lane, &tot);
      const long long tot_c = tot;
      const uint32_t e_pres = run_pres[z] | warp_excl_or(in ? present : 0u, lane, &ptot);
      bool s1, s2, s3, s4;
      {  // the pod count: the pending pod itself counts 1; reservations always carry counts
        const bool has = ph.thr_has & KT_COUNT_BIT;
        const long long au = base_c + e_c;
        const bool au_has = (ph.base_has & KT_COUNT_BIT) || e_c > 0;
        s1 = has && 1 > thr_c;
        s2 = ph.st_thr & KT_COUNT_BIT;
        s3 = has && au_has && (e3 ? au >= thr_c : au > thr_c);
        s4 = has && (on_equal ? au + 1 >= thr_c : au + 1 > thr_c);
      }
#pragma unroll
      for (int r = 0; r < RMAX; ++r) {
        if (r < R) {  // uniform
          long long rtot;
          // the pod's request: all of it if Admitted; if Undecided, only the part that moves this bound
          const long long vz = und ? (z ? (v[r] > 0 ? v[r] : 0) : (v[r] < 0 ? v[r] : 0)) : (in0 ? v[r] : 0);
          const long long e = run[z][r] + warp_excl_scan(vz, lane, &rtot);
          run[z][r] += rtot;
          if ((nz >> r) & 1) {  // IsThrottledFor only looks at the pod's non-zero requests (Q5)
            const bool has = (ph.thr_has >> r) & 1;
            const long long au = base[r] + e;
            const bool au_has = ((ph.base_has >> r) & 1) || ((e_pres >> r) & 1);
            s1 = s1 || (has && v[r] > thr[r]);
            s2 = s2 || ((ph.st_thr >> r) & 1);
            s3 = s3 || (has && au_has && (e3 ? au >= thr[r] : au > thr[r]));
            s4 = s4 || (has && (on_equal ? v[r] >= thr[r] - au : v[r] > thr[r] - au));
          }
        }
      }
      run_c[z] += tot_c;
      run_pres[z] |= ptot;
      code[z] = !live ? KT_CHECK_NOT_THROTTLED
                      : (s1 ? KT_CHECK_POD_REQUESTS_EXCEEDS_THRESHOLD : ((s2 || s3) ? KT_CHECK_ACTIVE : (s4 ? KT_CHECK_INSUFFICIENT : KT_CHECK_NOT_THROTTLED)));
    }
    if (on) {
      const uint32_t f = (code[1] ? 1u : 0u) | (code[0] ? 2u : 0u);
      if (f) atomicOr(&a.fail[i], f);
      // the codes under the smallest load: exact once nobody before the pod is Undecided (the last round)
      if (code[0]) atomicOr(&a.codes[p * 2 * a.Wp + (t >> 4)], code[0] << (2 * (t & 15)));
    }
  }
}

// end of a round: an Undecided pod that passed every pair under the largest load is admitted; one that failed a pair under
// the smallest is rejected; the others wait.  admit[] mirrors the state.
__global__ void __launch_bounds__(256) k_admit_update(AdmitView a) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= a.count) return;
  uint8_t st = a.state[i];
  if (st == kUndecided) {
    const uint32_t f = a.fail[i];
    if (!(f & 1u)) st = kAdmitted;
    else if (f & 2u) st = kRejected;
    a.state[i] = st;
  }
  if (st == kUndecided) atomicAdd(&a.counters[0], 1u);
  if (st == kAdmitted) atomicAdd(&a.counters[1], 1u);
  a.admit[admit_row(a, i)] = st == kAdmitted;
}

}  // namespace kt
