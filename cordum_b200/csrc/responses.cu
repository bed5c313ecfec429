// responses.cu — sm_90a kernels of cordum_batch_responses: a dispatched batch's jobs grouped by safety response class.
//
// They read the batch's sorted records (JobRec.orig, .topic, .mcp) and its decision records (d_out[orig]); nothing is
// copied in.  All tiles are tile2k's 2,048 items (kernels.h).
//   resp_key_kernel      per sorted record: the class key (kernels.h RespParams) of its job, stored at the job's index, so
//                        the sort's input is in job order
//   resp_count_kernel    \  one stable LSD radix pass over 8 key bits of (key, job) pairs, as plan.cu's passes: per-tile
//   resp_scan_kernel      | digit counts, a scan of each digit's row over the tiles, then each pair's place from the digit
//   resp_scatter_kernel  /  base, the row offset and its rank among the tile's earlier pairs of that digit (warp matches).
//                        The host runs ceil(key bits / 8) passes: digits above the key's width are 0 for every key.
//   resp_heads_kernel    per sorted position: does a class start here?  Marks the job there as its class's first job
//                        (jobs are ascending inside a class, the passes being stable over job-ordered input), and ranks
//                        the boundary among the tile's boundaries
//   resp_tile_scan_kernel  ranks of the first jobs in job order, tile by tile (the class order: by first job)
//   resp_tiles_kernel    one CTA: exclusive scans of the per-tile counts; the class count
//   resp_classes_kernel  per boundary: its class number, its extent (binary search for the key's last position), the
//                        class descriptor decoded from the key
//   resp_tile_scan_kernel + resp_tiles_kernel again: class sizes -> offsets, in class order
//   resp_gather_kernel   per sorted position: its job's place in the output list
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cordum_b200.h"
#include "kernels.h"

#define FULL 0xFFFFFFFFu

namespace {

using tile2k::item_index;
using tile2k::kItems;
using tile2k::kThreads;
using tile2k::kWarps;
typedef unsigned long long u64;
constexpr uint32_t kBins = 256, kTile = CORDUM_SUBSET_TILE, kNone = 0xFFFFFFFFu;

__device__ __forceinline__ u64 field(u64 key, uint32_t shift, uint32_t width) { return (key >> shift) & ((1ull << width) - 1ull); }

// arg of the class key: the job's topic id for the effective-config topic reasons, its MCP value id of the quoted field
// for the MCP reasons, 0 for every other code (engine.cu reason_arg is the host's copy)
__device__ __forceinline__ uint32_t reason_arg(uint32_t code, const JobRec* j) {
  if (code == CORDUM_REASON_EFF_DENIED_TOPIC || code == CORDUM_REASON_EFF_NOT_ALLOWED_TOPIC) return __ldg(&j->topic);
  if (code >= CORDUM_REASON_TENANT_MCP && code < CORDUM_REASON_TENANT_MCP + 8) return __ldg(&j->mcp[(code - CORDUM_REASON_TENANT_MCP) >> 1]);
  if (code >= CORDUM_REASON_EFF_MCP && code < CORDUM_REASON_EFF_MCP + 8) return __ldg(&j->mcp[(code - CORDUM_REASON_EFF_MCP) >> 1]);
  return 0;
}

// The class key of one job (include/cordum_b200.h cordum_batch_responses; layout in kernels.h).  A rule index or an id
// wider than its field would alias another class: it raises head[1] and the host refuses the call.
__device__ __forceinline__ u64 class_key(const RespParams& P, const JobRec* j, uint4 rec) {
  const uint32_t dec = rec.x & 7u, sched = (rec.x >> 8) & 7u, f = (rec.x >> 16) & 0xFFu, code = rec.y & 31u;
  const uint32_t fl = (f & (CORDUM_F_APPROVAL_REQUIRED | CORDUM_F_HAS_SNAPSHOT | CORDUM_F_CONSTRAINTS)) | ((f & CORDUM_F_APPROVED_BYPASS) ? 8u : 0u);
  const uint32_t arg = reason_arg(code, j), rule1 = (uint32_t)((int32_t)rec.z + 1);
  if ((u64)arg >> P.w_arg || (u64)rule1 >> P.w_rule || (rec.x & 0xF8F8u) || (rec.y & 0xE0u)) atomicOr(P.head + 1, 1u);
  const uint32_t s = P.w_arg + P.w_rule;
  return (u64)arg | (u64)rule1 << P.w_arg | (u64)code << s | (u64)fl << (s + 5) | (u64)sched << (s + 9) | (u64)dec << (s + 12);
}

__global__ void __launch_bounds__(kThreads) resp_key_kernel(RespParams P) {
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t s = item_index(blockIdx.x, r);
    if (s >= P.n) continue;
    const JobRec* j = P.job + s;
    const uint32_t o = __ldg(&j->orig);
    if (o >= P.n) continue;
    P.keys[0][o] = class_key(P, j, __ldg(P.out + o));
    P.vals[0][o] = o;
  }
}

__device__ __forceinline__ uint32_t digit(const u64* keys, uint32_t i, uint32_t n, uint32_t shift) {
  return i < n ? (uint32_t)(keys[i] >> shift) & (kBins - 1) : kNone;
}

// wcnt[warp][d] += pairs of this warp's part of the tile with digit d (group leaders of a round hold distinct digits)
__device__ __forceinline__ void count_warp(const uint32_t (&d)[kItems], uint32_t (*wcnt)[kBins]) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t peers = __match_any_sync(FULL, d[r]);
    if (d[r] != kNone && lane == (uint32_t)(__ffs(peers) - 1)) wcnt[warp][d[r]] += __popc(peers);
    __syncwarp();
  }
}

__device__ __forceinline__ void zero_counts(uint32_t (*wcnt)[kBins]) {
  for (uint32_t x = threadIdx.x; x < kWarps * kBins; x += kThreads) (&wcnt[0][0])[x] = 0;
  __syncthreads();
}

__global__ void __launch_bounds__(kThreads) resp_count_kernel(RespParams P, uint32_t pass) {
  __shared__ uint32_t wcnt[kWarps][kBins];
  const u64* keys = P.keys[pass & 1];
  uint32_t d[kItems];
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) d[r] = digit(keys, item_index(blockIdx.x, r), P.n, 8 * pass);
  zero_counts(wcnt);
  count_warp(d, wcnt);
  __syncthreads();
  uint32_t c = 0;
#pragma unroll
  for (uint32_t w = 0; w < kWarps; ++w) c += wcnt[w][threadIdx.x];
  P.counts[(size_t)threadIdx.x * P.n_tiles + blockIdx.x] = c;
}

// counts[d][*] -> exclusive prefix over the tiles; totals[d] = the row's sum
__global__ void __launch_bounds__(kThreads) resp_scan_kernel(RespParams P, uint32_t pass) {
  __shared__ uint32_t warp_sums[kWarps];
  const uint32_t sum = tile2k::tiles_scan(P.counts + (size_t)blockIdx.x * P.n_tiles, P.n_tiles, warp_sums);
  if (threadIdx.x == 0) P.totals[blockIdx.x] = sum;
}

__global__ void __launch_bounds__(kThreads) resp_scatter_kernel(RespParams P, uint32_t pass) {
  __shared__ uint32_t wcnt[kWarps][kBins];
  __shared__ uint32_t base[kBins];
  __shared__ uint32_t warp_sums[kWarps];
  const u64* keys = P.keys[pass & 1];
  const uint32_t* vals = P.vals[pass & 1];
  u64* keys_out = P.keys[(pass + 1) & 1];
  uint32_t* vals_out = P.vals[(pass + 1) & 1];
  u64 key[kItems];
  uint32_t val[kItems], d[kItems];
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t i = item_index(blockIdx.x, r);
    key[r] = i < P.n ? keys[i] : 0ull;
    val[r] = i < P.n ? vals[i] : 0u;
    d[r] = i < P.n ? (uint32_t)(key[r] >> (8 * pass)) & (kBins - 1) : kNone;
  }
  base[threadIdx.x] = P.totals[threadIdx.x];
  zero_counts(wcnt);
  count_warp(d, wcnt);
  tile2k::tiles_scan(base, kBins, warp_sums);   // its barriers also order count_warp; thread t rebases its own digit t
  // digit t of this tile starts at: pairs with a smaller digit (all tiles) + pairs with digit t in earlier tiles
  uint32_t run = base[threadIdx.x] + P.counts[(size_t)threadIdx.x * P.n_tiles + blockIdx.x];
#pragma unroll
  for (uint32_t w = 0; w < kWarps; ++w) {
    const uint32_t c = wcnt[w][threadIdx.x];
    wcnt[w][threadIdx.x] = run;
    run += c;
  }
  __syncthreads();
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31, below = (1u << lane) - 1u;
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t peers = __match_any_sync(FULL, d[r]);
    if (d[r] != kNone) {
      const uint32_t dst = wcnt[warp][d[r]] + __popc(peers & below);
      keys_out[dst] = key[r];
      vals_out[dst] = val[r];
    }
    __syncwarp();
    if (d[r] != kNone && lane == (uint32_t)(__ffs(peers) - 1)) wcnt[warp][d[r]] += __popc(peers);
    __syncwarp();
  }
}

__global__ void __launch_bounds__(kThreads) resp_heads_kernel(RespParams P) {
  __shared__ uint32_t warp_sums[kWarps];
  const u64* keys = P.keys[P.passes & 1];
  const uint32_t* vals = P.vals[P.passes & 1];
  uint32_t h[kItems], pre[kItems], total;
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t i = item_index(blockIdx.x, r);
    h[r] = 0;
    if (i < P.n) {
      h[r] = i == 0 || keys[i] != keys[i - 1];
      P.jflag[vals[i]] = h[r];
    }
  }
  tile2k::tile_scan(h, pre, warp_sums, &total);
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t i = item_index(blockIdx.x, r);
    if (i < P.n) P.sloc[i] = pre[r];
  }
  if (threadIdx.x == 0) P.hcnt[blockIdx.x] = total;
}

// v[0 .. n) -> exclusive prefix inside each tile; cnt[tile] = the tile's sum.  n_dev: read n there instead (class count).
__global__ void __launch_bounds__(kThreads) resp_tile_scan_kernel(uint32_t* v, uint32_t* cnt, uint32_t n, const uint32_t* n_dev) {
  __shared__ uint32_t warp_sums[kWarps];
  if (n_dev) n = *n_dev;
  uint32_t x[kItems], pre[kItems], total;
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t i = item_index(blockIdx.x, r);
    x[r] = i < n ? v[i] : 0u;
  }
  tile2k::tile_scan(x, pre, warp_sums, &total);
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t i = item_index(blockIdx.x, r);
    if (i < n) v[i] = pre[r];
  }
  if (threadIdx.x == 0) cnt[blockIdx.x] = total;
}

// One CTA: exclusive prefixes of a[0 .. n_tiles) (when given) and b[0 .. n_tiles); *b_total = b's sum (when given).
__global__ void __launch_bounds__(kThreads) resp_tiles_kernel(uint32_t* a, uint32_t* b, uint32_t n_tiles, uint32_t* b_total) {
  __shared__ uint32_t warp_sums[kWarps];
  if (a) tile2k::tiles_scan(a, n_tiles, warp_sums);
  const uint32_t sum = tile2k::tiles_scan(b, n_tiles, warp_sums);
  if (b_total && threadIdx.x == 0) *b_total = sum;
}

__global__ void __launch_bounds__(kThreads) resp_classes_kernel(RespParams P) {
  const u64* keys = P.keys[P.passes & 1];
  const uint32_t* vals = P.vals[P.passes & 1];
#pragma unroll 1
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t i = item_index(blockIdx.x, r);
    if (i >= P.n) continue;
    const u64 key = keys[i];
    if (i && keys[i - 1] == key) continue;
    const uint32_t j = vals[i];
    const uint32_t c = P.jcnt[j / kTile] + P.jflag[j];   // rank of its first job among all first jobs
    P.perm[P.hcnt[blockIdx.x] + P.sloc[i]] = c;
    uint32_t lo = i + 1, hi = P.n;                       // first position past the class: keys ascend
    while (lo < hi) {
      const uint32_t mid = lo + ((hi - lo) >> 1);
      if (keys[mid] == key) lo = mid + 1;
      else hi = mid;
    }
    P.start[c] = i;
    P.size[c] = lo - i;
    const uint32_t s = P.w_arg + P.w_rule, fl = (uint32_t)field(key, s + 5, 4);
    cordum_response_class k;
    k.decision = (uint8_t)field(key, s + 12, 3);
    k.sched_decision = (uint8_t)field(key, s + 9, 3);
    k.flags = (uint8_t)((fl & 7u) | ((fl & 8u) ? CORDUM_F_APPROVED_BYPASS : 0u));
    k.reason_code = (uint8_t)field(key, s, 5);
    k.rule_idx = (int32_t)field(key, P.w_arg, P.w_rule) - 1;
    k.arg = (uint32_t)field(key, 0, P.w_arg);
    k.first_job = j;
    P.cls[c] = k;
  }
}

__global__ void __launch_bounds__(kThreads) resp_gather_kernel(RespParams P) {
  const u64* keys = P.keys[P.passes & 1];
  const uint32_t* vals = P.vals[P.passes & 1];
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t i = item_index(blockIdx.x, r);
    if (i >= P.n) continue;
    const uint32_t h = i == 0 || keys[i] != keys[i - 1];
    const uint32_t c = P.perm[P.hcnt[blockIdx.x] + P.sloc[i] + h - 1];   // the class of the last boundary at or before i
    const uint32_t off = P.ccnt[c / kTile] + P.size[c];
    P.jobs[off + (i - P.start[c])] = vals[i];
    if (h) P.offsets[c] = off;
    if (i == P.n - 1) P.offsets[*P.head] = P.n;
  }
}

}  // namespace

cudaError_t launch_responses(const RespParams& P, cudaStream_t s) {
  if (P.n == 0) return cudaSuccess;
  const uint32_t g = P.n_tiles;
  resp_key_kernel<<<g, kThreads, 0, s>>>(P);
  for (uint32_t p = 0; p < P.passes; ++p) {
    resp_count_kernel<<<g, kThreads, 0, s>>>(P, p);
    resp_scan_kernel<<<kBins, kThreads, 0, s>>>(P, p);
    resp_scatter_kernel<<<g, kThreads, 0, s>>>(P, p);
  }
  resp_heads_kernel<<<g, kThreads, 0, s>>>(P);
  resp_tile_scan_kernel<<<g, kThreads, 0, s>>>(P.jflag, P.jcnt, P.n, nullptr);
  resp_tiles_kernel<<<1, kThreads, 0, s>>>(P.hcnt, P.jcnt, g, P.head);
  resp_classes_kernel<<<g, kThreads, 0, s>>>(P);
  resp_tile_scan_kernel<<<g, kThreads, 0, s>>>(P.size, P.ccnt, P.n, P.head);   // sizes -> offsets inside each tile of classes
  resp_tiles_kernel<<<1, kThreads, 0, s>>>(nullptr, P.ccnt, g, nullptr);
  resp_gather_kernel<<<g, kThreads, 0, s>>>(P);
  return cudaGetLastError();
}
