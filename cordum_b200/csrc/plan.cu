// plan.cu — sm_90a kernels of cordum_batch_plan: a dispatched batch's jobs grouped by destination worker and by outcome.
//
// They read the batch's decision records (d_out, caller order) and nothing else.  Each job has a bucket key
// (include/cordum_b200.h cordum_plan): its worker slot when it was routed, else n_slots + outcome.  The grouping is a
// stable LSD radix sort of (key, job index) pairs, 8 key bits per pass, as many passes as the bucket count needs bits:
//   plan_count_kernel    per tile of 2,048 jobs: how many of them carry each of the 256 digit values -> counts[digit][tile]
//   plan_scan_kernel     a CTA per digit value: exclusive scan of its row over the tiles, the row total -> totals[digit]
//   plan_scatter_kernel  per tile: base of the digit (scan of the 256 totals) + the row offset + the job's rank among the
//                        tile's earlier jobs with that digit -> the job's place in the pass's output
// and then plan_offsets_kernel: offsets[k] = first position whose key is >= k, one binary search per bucket.
// How the jobs spread over the buckets does not change the work: per-tile state is over the 256 digit values (never over
// the n_slots buckets), ranks come from warp matches, and the offsets cost one search per bucket.  Job index order inside
// a bucket follows from every pass being stable and pass 0 reading the jobs in index order.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cordum_b200.h"
#include "kernels.h"

#define FULL 0xFFFFFFFFu

namespace {

constexpr uint32_t kThreads = 256, kWarps = kThreads / 32, kItems = CORDUM_PLAN_TILE / kThreads, kBins = 256;
static_assert(kItems * kThreads == CORDUM_PLAN_TILE && kItems == 8, "a warp owns 8 rounds of 32 consecutive jobs");
constexpr uint32_t kNone = 0xFFFFFFFFu;   // a lane with no job in this round

// Bucket key of one decision record (the header's cordum_plan); a record that fits no bucket raises *bad and counts as 0.
__device__ __forceinline__ uint32_t plan_key(uint4 rec, uint32_t n_slots, uint32_t* bad) {
  const uint32_t o = plan_outcome(rec.x), slot = rec.w;   // worker_slot
  uint32_t k = kNone;
  if (o == CORDUM_COUNT_ROUTED) {
    if (slot < n_slots) k = slot;
  } else if (o != CORDUM_PLAN_NONE) {
    k = n_slots + o;
  }
  if (k == kNone) {   // e.g. a worker slot beyond the registry the batch was routed on: the host refuses the plan
    atomicOr(bad, 1u);
    k = 0;
  }
  return k;
}

// The tile's jobs as this lane holds them: round r = tile position warp * 256 + r * 32 + lane (index order = round-major,
// then lane).  Pass 0 derives keys from the records and takes the job index as the value.
__device__ __forceinline__ void load_tile(const PlanPass& P, uint32_t (&key)[kItems], uint32_t (&val)[kItems]) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t base = blockIdx.x * CORDUM_PLAN_TILE + warp * (32 * kItems) + lane;
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t i = base + r * 32;
    key[r] = kNone;
    val[r] = 0;
    if (i < P.n) {
      if (P.recs) {
        key[r] = plan_key(__ldg(P.recs + i), P.n_slots, P.bad);
        val[r] = i;
      } else {
        key[r] = __ldg(P.keys_in + i);
        val[r] = __ldg(P.vals_in + i);
      }
    }
  }
}

__device__ __forceinline__ uint32_t digit_of(uint32_t key, uint32_t shift) { return key == kNone ? kNone : (key >> shift) & (kBins - 1); }

// wcnt[warp][d] += jobs of this warp's part of the tile with digit d.  Inside a round the group leaders hold distinct
// digits, and each warp writes its own row.
__device__ __forceinline__ void count_warp(const uint32_t (&key)[kItems], uint32_t shift, uint32_t (*wcnt)[kBins]) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t d = digit_of(key[r], shift);
    const uint32_t peers = __match_any_sync(FULL, d);
    if (d != kNone && lane == (uint32_t)(__ffs(peers) - 1)) wcnt[warp][d] += __popc(peers);
    __syncwarp();
  }
}

__device__ __forceinline__ void zero_counts(uint32_t (*wcnt)[kBins]) {
  for (uint32_t x = threadIdx.x; x < kWarps * kBins; x += kThreads) (&wcnt[0][0])[x] = 0;
  __syncthreads();
}

// Exclusive scan over the CTA (kThreads values, one per thread); returns this thread's prefix and the total in *sum.
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* warp_sums, uint32_t* sum) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t x = v;
#pragma unroll
  for (uint32_t o = 1; o < 32; o <<= 1) {
    const uint32_t y = __shfl_up_sync(FULL, x, o);
    if (lane >= o) x += y;
  }
  if (lane == 31) warp_sums[warp] = x;
  __syncthreads();
  uint32_t before = 0, total = 0;
#pragma unroll
  for (uint32_t w = 0; w < kWarps; ++w) {
    const uint32_t s = warp_sums[w];
    before += w < warp ? s : 0u;
    total += s;
  }
  __syncthreads();   // warp_sums is reused by the next call
  *sum = total;
  return before + x - v;
}

__global__ void __launch_bounds__(kThreads) plan_count_kernel(PlanPass P) {
  __shared__ uint32_t wcnt[kWarps][kBins];
  uint32_t key[kItems], val[kItems];
  load_tile(P, key, val);
  zero_counts(wcnt);
  count_warp(key, P.shift, wcnt);
  __syncthreads();
  const uint32_t d = threadIdx.x;
  uint32_t c = 0;
#pragma unroll
  for (uint32_t w = 0; w < kWarps; ++w) c += wcnt[w][d];
  P.counts[(size_t)d * P.n_tiles + blockIdx.x] = c;
}

// counts[d][*] -> exclusive prefix over the tiles; totals[d] = the row's sum.
__global__ void __launch_bounds__(kThreads) plan_scan_kernel(PlanPass P) {
  __shared__ uint32_t warp_sums[kWarps];
  uint32_t* row = P.counts + (size_t)blockIdx.x * P.n_tiles;
  uint32_t carry = 0;
  for (uint32_t t0 = 0; t0 < P.n_tiles; t0 += kThreads) {
    const uint32_t t = t0 + threadIdx.x;
    const uint32_t v = t < P.n_tiles ? row[t] : 0u;
    uint32_t sum;
    const uint32_t pre = block_exclusive_scan(v, warp_sums, &sum);
    if (t < P.n_tiles) row[t] = carry + pre;
    carry += sum;
  }
  if (threadIdx.x == 0) P.totals[blockIdx.x] = carry;
}

__global__ void __launch_bounds__(kThreads) plan_scatter_kernel(PlanPass P) {
  __shared__ uint32_t wcnt[kWarps][kBins];
  __shared__ uint32_t warp_sums[kWarps];
  uint32_t key[kItems], val[kItems];
  load_tile(P, key, val);
  zero_counts(wcnt);
  count_warp(key, P.shift, wcnt);
  // digit d of this tile starts at: jobs with a smaller digit (all tiles) + jobs with digit d in earlier tiles
  const uint32_t d = threadIdx.x;
  uint32_t sum;
  uint32_t run = block_exclusive_scan(P.totals[d], warp_sums, &sum) + P.counts[(size_t)d * P.n_tiles + blockIdx.x];   // its syncs order count_warp
#pragma unroll
  for (uint32_t w = 0; w < kWarps; ++w) {
    const uint32_t c = wcnt[w][d];
    wcnt[w][d] = run;
    run += c;
  }
  __syncthreads();
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, below = (1u << lane) - 1u;
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t dg = digit_of(key[r], P.shift);
    const uint32_t peers = __match_any_sync(FULL, dg);
    if (dg != kNone) {
      const uint32_t dst = wcnt[warp][dg] + __popc(peers & below);
      P.keys_out[dst] = key[r];
      P.vals_out[dst] = val[r];
    }
    __syncwarp();
    if (dg != kNone && lane == (uint32_t)(__ffs(peers) - 1)) wcnt[warp][dg] += __popc(peers);
    __syncwarp();
  }
}

// offsets[k] = number of sorted keys below k, for k = 0 .. n_buckets (offsets[n_buckets] = n)
__global__ void __launch_bounds__(kThreads) plan_offsets_kernel(const uint32_t* __restrict__ keys, uint32_t n, uint32_t n_buckets,
                                                                uint32_t* __restrict__ offsets) {
  const uint32_t k = blockIdx.x * kThreads + threadIdx.x;
  if (k > n_buckets) return;
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    if (__ldg(keys + mid) < k) lo = mid + 1;
    else hi = mid;
  }
  offsets[k] = lo;
}

}  // namespace

uint32_t plan_passes(uint32_t n_buckets) {
  uint32_t bits = 0;
  while (bits < 32 && (uint64_t(1) << bits) < n_buckets) ++bits;   // keys 0 .. n_buckets - 1
  return bits <= 8 ? 1u : (bits + 7) / 8;
}

cudaError_t launch_plan(const PlanParams& L, cudaStream_t s) {
  if (L.n == 0) return cudaSuccess;
  const uint32_t n_tiles = (uint32_t)(((uint64_t)L.n + CORDUM_PLAN_TILE - 1) / CORDUM_PLAN_TILE), passes = plan_passes(L.n_buckets);
  cudaError_t e = cudaMemsetAsync(L.bad, 0, sizeof(uint32_t), s);
  for (uint32_t p = 0; p < passes && e == cudaSuccess; ++p) {
    PlanPass P{};
    P.recs = p == 0 ? reinterpret_cast<const uint4*>(L.recs) : nullptr;
    P.keys_in = L.keys[(p + 1) & 1];
    P.vals_in = L.vals[(p + 1) & 1];
    P.keys_out = L.keys[p & 1];
    P.vals_out = L.vals[p & 1];
    P.counts = L.counts;
    P.totals = L.totals;
    P.bad = L.bad;
    P.n = L.n;
    P.n_slots = L.n_slots;
    P.n_tiles = n_tiles;
    P.shift = 8 * p;
    plan_count_kernel<<<n_tiles, kThreads, 0, s>>>(P);
    plan_scan_kernel<<<kBins, kThreads, 0, s>>>(P);
    plan_scatter_kernel<<<n_tiles, kThreads, 0, s>>>(P);
    e = cudaGetLastError();
  }
  if (e != cudaSuccess) return e;
  plan_offsets_kernel<<<(L.n_buckets + kThreads) / kThreads, kThreads, 0, s>>>(L.keys[(passes - 1) & 1], L.n, L.n_buckets, L.offsets);
  return cudaGetLastError();
}
