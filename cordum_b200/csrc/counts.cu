// counts.cu — sm_90a kernels of cordum_batch_topic_counts: a dispatched batch's jobs counted per (topic id, outcome column).
//
// They read the batch's sorted records (JobRec.topic, JobRec.orig) and its decision records (d_out[orig]); nothing is
// copied in.  Column = plan_outcome of the record (kernels.h): the plan's outcome bucket, or CORDUM_COUNT_ROUTED.
//   topic_count_kernel  per tile of CORDUM_COUNT_TILE sorted records: lanes holding the same (topic, column) are merged by
//                       warp matches; topics within CORDUM_COUNT_WINDOW ids of the tile's first record are added up in
//                       shared memory and flushed with one global atomic per non-zero cell, any other topic goes to the
//                       global table directly.  Records are sorted by topic, so a tile usually spans few topics and a
//                       topic that holds most of a batch costs one atomic per tile, not one per job; the order only
//                       makes it fast, the counts do not depend on it.
//   topic_rows_kernel   a thread per topic id: a row with a non-zero count takes the next place of the compacted output
//                       (warp-aggregated atomic) -> {topic id, counts}.  The host copies only these rows and merges them
//                       by label, so the copy is O(distinct topic ids), not O(dictionary) or O(jobs).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cordum_b200.h"
#include "kernels.h"

#define FULL 0xFFFFFFFFu

namespace {

constexpr uint32_t kThreads = 256, kItems = CORDUM_COUNT_TILE / kThreads, kCols = CORDUM_COUNT_COLUMNS, kWin = CORDUM_COUNT_WINDOW;
static_assert(kItems * kThreads == CORDUM_COUNT_TILE && kItems == 8, "a warp owns 8 rounds of 32 consecutive records");
constexpr uint32_t kNone = 0xFFFFFFFFu;

__global__ void __launch_bounds__(kThreads) topic_count_kernel(CountParams P) {
  __shared__ uint32_t win[kWin * kCols];
  for (uint32_t x = threadIdx.x; x < kWin * kCols; x += kThreads) win[x] = 0;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t base = blockIdx.x * CORDUM_COUNT_TILE + (threadIdx.x >> 5) * (32 * kItems) + lane;
  const uint32_t t0 = __ldg(&P.job[blockIdx.x * CORDUM_COUNT_TILE].topic);
  uint32_t topic[kItems], col[kItems];
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t s = base + r * 32;
    topic[r] = kNone;
    col[r] = s < P.n ? __ldg(&P.job[s].orig) : kNone;   // the record's job index until the decision record is read
    if (s < P.n) topic[r] = __ldg(&P.job[s].topic);
  }
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    if (topic[r] == kNone) continue;
    const uint32_t o = col[r];
    uint32_t c = CORDUM_PLAN_NONE;
    if (o < P.n) {
      const uint4 rec = __ldg(P.out + o);
      c = plan_outcome(rec.x);
      if (c == CORDUM_COUNT_ROUTED && rec.w >= P.n_slots) c = CORDUM_PLAN_NONE;   // a slot beyond the batch's registry
    }
    if (c == CORDUM_PLAN_NONE || topic[r] >= P.n_topics) {   // the host refuses the counts, as it refuses the plan
      atomicOr(P.head + 1, 1u);
      topic[r] = kNone;
    }
    col[r] = c;
  }
  __syncthreads();
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t t = topic[r], c = col[r];
    const uint32_t peers = __match_any_sync(FULL, t) & __match_any_sync(FULL, c);
    if (t != kNone && lane == (uint32_t)(__ffs(peers) - 1)) {
      const uint32_t d = t - t0;
      if (d < kWin) atomicAdd(&win[d * kCols + c], __popc(peers));
      else atomicAdd(&P.table[(size_t)t * kCols + c], __popc(peers));
    }
  }
  __syncthreads();
  for (uint32_t x = threadIdx.x; x < kWin * kCols; x += kThreads) {
    const uint32_t v = win[x];
    if (v) atomicAdd(&P.table[(size_t)t0 * kCols + x], v);   // only ids below n_topics were added here
  }
}

__global__ void __launch_bounds__(kThreads) topic_rows_kernel(CountParams P) {
  const uint32_t t = blockIdx.x * kThreads + threadIdx.x, lane = threadIdx.x & 31;
  uint32_t v[kCols], any = 0;
#pragma unroll
  for (uint32_t c = 0; c < kCols; ++c) {
    v[c] = t < P.n_topics ? P.table[(size_t)t * kCols + c] : 0u;
    any |= v[c];
  }
  const uint32_t keep = __ballot_sync(FULL, any != 0);
  uint32_t at = 0;
  if (lane == 0 && keep) at = atomicAdd(P.head, __popc(keep));
  at = __shfl_sync(FULL, at, 0) + __popc(keep & ((1u << lane) - 1u));
  if (!any) return;
  uint32_t* row = P.rows + (size_t)at * (1 + kCols);
  row[0] = t;
#pragma unroll
  for (uint32_t c = 0; c < kCols; ++c) row[1 + c] = v[c];
}

}  // namespace

cudaError_t launch_counts(const CountParams& P, cudaStream_t s) {
  if (P.n == 0) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(P.table, 0, (size_t)P.n_topics * kCols * 4, s);
  if (e == cudaSuccess) e = cudaMemsetAsync(P.head, 0, 2 * sizeof(uint32_t), s);
  if (e != cudaSuccess) return e;
  const uint32_t tiles = (uint32_t)(((uint64_t)P.n + CORDUM_COUNT_TILE - 1) / CORDUM_COUNT_TILE);
  topic_count_kernel<<<tiles, kThreads, 0, s>>>(P);
  topic_rows_kernel<<<(P.n_topics + kThreads - 1) / kThreads + (P.n_topics == 0), kThreads, 0, s>>>(P);
  return cudaGetLastError();
}
