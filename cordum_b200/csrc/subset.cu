// subset.cu — sm_90a kernels of cordum_batch_subset: a new encoded batch from a chosen subset of an encoded one.
//
// The source's records are sorted by (topic, tenant class); the subset keeps that order, so nothing is sorted again.  A
// job is selected by its outcome bucket (decision record, caller order) or by a list of job indices.  Everything is
// derived from JobRec.orig and the decision records: a host-encoded source has no slot_of on the device.  Four launches,
// each over tiles of CORDUM_SUBSET_TILE items (256 threads x 8 items, item = warp * 256 + round * 32 + lane):
//   subset_mark_kernel    per job tile: selected or not -> jloc = the job's rank among the tile's selected jobs, jcnt[tile]
//   subset_keep_kernel    per slot tile: kept = jloc[orig] != NONE -> sloc, scnt[tile]; per selective-list tile: kept
//                         entries and the extra words they carry -> eloc, ecnt / wcnt[tile]
//   subset_scan_kernel    one CTA per count array: exclusive prefix over the tiles, the total -> totals[4]
//   (the host reads totals, refuses or sizes the destination)
//   subset_gather_kernel  per slot tile: JobRec (orig renumbered), RouteRec and wide row to the new slot, slot_of and the
//                         parent index; per selective-list tile: {new slot, new x} and the re-packed extra words
// New job index = jcnt[orig / tile] + jloc[orig]; new slot = scnt[slot / tile] + sloc[slot]: both are O(1) lookups once the
// tile prefixes exist, so the gather needs no per-item scan of its own.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cordum_b200.h"
#include "kernels.h"

#define FULL 0xFFFFFFFFu

namespace {

using tile2k::kThreads;
using tile2k::kWarps;
using tile2k::kItems;
using tile2k::item_index;
using tile2k::tile_scan;
constexpr uint32_t kNone = CORDUM_SUBSET_NONE;

// Outcome bucket of a decision record (include/cordum_b200.h CORDUM_PLAN_*), or NONE for a routed job.
__device__ __forceinline__ uint32_t outcome_of(uint4 rec) {
  const uint32_t k = plan_outcome(rec.x);
  return k < CORDUM_PLAN_OUTCOMES ? k : kNone;
}

__global__ void __launch_bounds__(kThreads) subset_mark_kernel(SubsetParams P) {
  __shared__ uint32_t warp_sums[kWarps];
  __shared__ uint32_t bits[CORDUM_SUBSET_TILE / 32];   // list form: the tile's selected jobs
  const uint32_t tile = blockIdx.x;
  if (P.list) {
    // the list is ascending: the tile's entries are one run of it, found by two binary searches
    __shared__ uint32_t range[2];
    for (uint32_t x = threadIdx.x; x < CORDUM_SUBSET_TILE / 32; x += kThreads) bits[x] = 0;
    if (threadIdx.x < 2) {
      const uint32_t key = (tile + threadIdx.x) * CORDUM_SUBSET_TILE;
      uint32_t lo = 0, hi = P.n_list;
      while (lo < hi) {
        const uint32_t mid = lo + ((hi - lo) >> 1);
        if (__ldg(P.list + mid) < key) lo = mid + 1;
        else hi = mid;
      }
      range[threadIdx.x] = lo;
    }
    __syncthreads();
    for (uint32_t k = range[0] + threadIdx.x; k < range[1]; k += kThreads) {
      const uint32_t p = __ldg(P.list + k) - tile * CORDUM_SUBSET_TILE;
      atomicOr(&bits[p >> 5], 1u << (p & 31));
    }
    __syncthreads();
  }
  uint32_t flag[kItems], pre[kItems], total;
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t i = item_index(tile, r);
    flag[r] = 0;
    if (i < P.n) {
      if (P.list) {
        const uint32_t p = i - tile * CORDUM_SUBSET_TILE;
        flag[r] = (bits[p >> 5] >> (p & 31)) & 1u;
      } else {
        const uint32_t k = outcome_of(__ldg(P.out + i));
        flag[r] = k != kNone ? (P.mask >> k) & 1u : 0u;
      }
    }
  }
  tile_scan(flag, pre, warp_sums, &total);
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t i = item_index(tile, r);
    if (i < P.n) P.jloc[i] = flag[r] ? pre[r] : kNone;
  }
  if (threadIdx.x == 0) P.jcnt[tile] = total;
}

__global__ void __launch_bounds__(kThreads) subset_keep_kernel(SubsetParams P) {
  __shared__ uint32_t warp_sums[kWarps];
  uint32_t keep[kItems], pre[kItems], total;
  if (blockIdx.x < P.n_tiles) {   // sorted slots
    const uint32_t tile = blockIdx.x;
#pragma unroll
    for (uint32_t r = 0; r < kItems; ++r) {
      const uint32_t s = item_index(tile, r);
      keep[r] = s < P.n && __ldg(P.jloc + __ldg(&P.job[s].orig)) != kNone ? 1u : 0u;
    }
    tile_scan(keep, pre, warp_sums, &total);
#pragma unroll
    for (uint32_t r = 0; r < kItems; ++r) {
      const uint32_t s = item_index(tile, r);
      if (s < P.n) P.sloc[s] = keep[r] ? pre[r] : kNone;
    }
    if (threadIdx.x == 0) P.scnt[tile] = total;
    return;
  }
  // selective-list entries: kept with their slot; an entry with x != 0 carries 1 + extra[x] extra words
  const uint32_t tile = blockIdx.x - P.n_tiles;
  uint32_t words[kItems], wpre[kItems], wtotal;
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t e = item_index(tile, r);
    keep[r] = 0;
    words[r] = 0;
    if (e < P.n_sel) {
      const uint2 ent = __ldg(P.sel_jobs + e);
      if (__ldg(P.jloc + __ldg(&P.job[ent.x].orig)) != kNone) {
        keep[r] = 1;
        words[r] = ent.y ? 1u + __ldg(P.sel_extra + ent.y) : 0u;
      }
    }
  }
  tile_scan(keep, pre, warp_sums, &total);
  tile_scan(words, wpre, warp_sums, &wtotal);
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t e = item_index(tile, r);
    if (e < P.n_sel) P.eloc[e] = make_uint2(keep[r] ? pre[r] : kNone, wpre[r]);
  }
  if (threadIdx.x == 0) { P.ecnt[tile] = total; P.wcnt[tile] = wtotal; }
}

// CTA b: the count array b (jcnt, scnt over the job tiles; ecnt, wcnt over the selective-list tiles) -> exclusive
// prefixes in place, its total -> totals[b]
__global__ void __launch_bounds__(kThreads) subset_scan_kernel(SubsetParams P) {
  __shared__ uint32_t warp_sums[kWarps];
  uint32_t* row = blockIdx.x == 0 ? P.jcnt : blockIdx.x == 1 ? P.scnt : blockIdx.x == 2 ? P.ecnt : P.wcnt;
  const uint32_t n = blockIdx.x < 2 ? P.n_tiles : P.n_sel_tiles;
  const uint32_t carry = tile2k::tiles_scan(row, n, warp_sums);
  if (threadIdx.x == 0) P.totals[blockIdx.x] = carry;
}

__global__ void __launch_bounds__(kThreads) subset_gather_kernel(SubsetParams P) {
  const uint32_t lane = threadIdx.x & 31;
  if (blockIdx.x < P.n_tiles) {   // sorted slots
    const uint32_t tile = blockIdx.x;
#pragma unroll 1
    for (uint32_t r = 0; r < kItems; ++r) {
      const uint32_t s = item_index(tile, r);
      const uint32_t loc = s < P.n ? __ldg(P.sloc + s) : kNone;
      uint32_t ns = kNone;
      if (loc != kNone) {
        ns = P.scnt[tile] + loc;
        const uint4* src = reinterpret_cast<const uint4*>(P.job + s);
        uint4 j0 = __ldg(src), j1 = __ldg(src + 1), j2 = __ldg(src + 2), j3 = __ldg(src + 3);
        const uint32_t o = j0.z;   // JobRec.orig
        const uint32_t no = P.jcnt[o / CORDUM_SUBSET_TILE] + __ldg(P.jloc + o);
        j0.z = no;
        uint4* dst = reinterpret_cast<uint4*>(P.djob + ns);
        dst[0] = j0; dst[1] = j1; dst[2] = j2; dst[3] = j3;
        const uint4* rs = reinterpret_cast<const uint4*>(P.route + s);
        uint4* rd = reinterpret_cast<uint4*>(P.droute + ns);
        rd[0] = __ldg(rs); rd[1] = __ldg(rs + 1);
        P.dslot_of[no] = ns;
        P.dparent[no] = o;
      }
      if (P.ww) {   // wide rows: the warp copies each kept row of this round together
        uint32_t todo = __ballot_sync(FULL, loc != kNone);
        while (todo) {
          const uint32_t src_lane = __ffs(todo) - 1;
          todo &= todo - 1;
          const uint32_t from = __shfl_sync(FULL, s, src_lane), to = __shfl_sync(FULL, ns, src_lane);
          const uint64_t* a = P.wide + (size_t)from * P.ww;
          uint64_t* b = P.dwide + (size_t)to * P.ww;
          for (uint32_t w = lane; w < P.ww; w += 32) b[w] = __ldg(a + w);
        }
      }
    }
    return;
  }
  // selective-list entries
  const uint32_t tile = blockIdx.x - P.n_tiles;
  uint32_t* const dextra = P.dsel + 2 * (size_t)P.m_sel;
  if (tile == 0 && threadIdx.x == 0 && P.m_sel) dextra[0] = 0;   // x = 0 never points at a list
#pragma unroll 1
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t e = item_index(tile, r);
    if (e >= P.n_sel) continue;
    const uint2 loc = __ldg(P.eloc + e);
    if (loc.x == kNone) continue;
    const uint2 ent = __ldg(P.sel_jobs + e);
    const uint32_t ne = P.ecnt[tile] + loc.x;
    const uint32_t nx = ent.y ? 1u + P.wcnt[tile] + loc.y : 0u;
    P.dsel[2 * (size_t)ne] = P.scnt[ent.x / CORDUM_SUBSET_TILE] + __ldg(P.sloc + ent.x);
    P.dsel[2 * (size_t)ne + 1] = nx;
    if (ent.y) {
      const uint32_t c = __ldg(P.sel_extra + ent.y);
      for (uint32_t k = 0; k <= c; ++k) dextra[nx + k] = __ldg(P.sel_extra + ent.y + k);
    }
  }
}

}  // namespace

cudaError_t launch_subset_count(const SubsetParams& P, cudaStream_t s) {
  if (P.n == 0) return cudaSuccess;
  subset_mark_kernel<<<P.n_tiles, kThreads, 0, s>>>(P);
  subset_keep_kernel<<<P.n_tiles + P.n_sel_tiles, kThreads, 0, s>>>(P);
  subset_scan_kernel<<<4, kThreads, 0, s>>>(P);
  return cudaGetLastError();
}

cudaError_t launch_subset_gather(const SubsetParams& P, cudaStream_t s) {
  if (P.n == 0) return cudaSuccess;
  subset_gather_kernel<<<P.n_tiles + P.n_sel_tiles, kThreads, 0, s>>>(P);
  return cudaGetLastError();
}
