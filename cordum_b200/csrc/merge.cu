// merge.cu — sm_90a kernels of cordum_batch_merge: one encoded batch from two encoded batches of the same table epoch.
//
// Each source's records are sorted by the encoders' key (topic id * tenant_classes + tenant_class[tenant id]), stable in
// the job index.  The records of a's envelopes followed by b's, encoded together, are therefore the stable two-way merge
// of the two sorted sequences with a first on equal keys: a's slot i goes to i + (b's keys < key), b's slot j to
// j + (a's keys <= key), each rank a binary search over the other source's compacted keys.  Nothing is sorted.  Everything
// is derived from the sorted records and JobRec.orig (a host-encoded source has no slot_of on the device).  Three
// launches over tiles of CORDUM_SUBSET_TILE items (kernels.h tile2k); source 0 = a, 1 = b, and a grid covers a's slot
// tiles, b's slot tiles, a's selective-list tiles, b's selective-list tiles in that order:
//   merge_key_kernel     per slot tile: the record's key -> key[]; per selective-list tile: the extra words each entry
//                        carries (x != 0: 1 + extra[x]) -> wloc = their exclusive prefix in the tile, wcnt[tile]
//   merge_scan_kernel    one CTA per source: exclusive prefix of wcnt over its tiles, the total -> totals[source]
//   merge_gather_kernel  per slot tile: JobRec (b's orig + n_a), RouteRec and wide row to the merged slot, slot_of; per
//                        selective-list tile: the entry's merged position e + (the other source's entries before it),
//                        {merged slot, x} and its extra words re-packed behind the other source's entries' words
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
constexpr uint32_t T = CORDUM_SUBSET_TILE;

// Which source and which kind of tile block b of a grid is: slots (false) or selective-list entries (true).
__device__ __forceinline__ void block_role(const MergeParams& P, uint32_t& src, bool& sel, uint32_t& tile) {
  uint32_t b = blockIdx.x;
  sel = false;
  if (b < P.s[0].n_tiles) { src = 0; tile = b; return; }
  b -= P.s[0].n_tiles;
  if (b < P.s[1].n_tiles) { src = 1; tile = b; return; }
  b -= P.s[1].n_tiles;
  sel = true;
  if (b < P.s[0].n_sel_tiles) { src = 0; tile = b; return; }
  src = 1;
  tile = b - P.s[0].n_sel_tiles;
}

// Keys before `key` in the sorted keys[0 .. n): strictly below (upper = false), or up to and including it (upper = true).
__device__ __forceinline__ uint32_t rank_in(const uint32_t* keys, uint32_t n, uint32_t key, bool upper) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = lo + ((hi - lo) >> 1);
    const uint32_t k = __ldg(keys + mid);
    if (k < key || (upper && k == key)) lo = mid + 1;
    else hi = mid;
  }
  return lo;
}

// Merged slot of source src's sorted slot i: ties go to a.
__device__ __forceinline__ uint32_t merged_slot(const MergeParams& P, uint32_t src, uint32_t i) {
  const MergeSource& o = P.s[src ^ 1];
  return i + rank_in(o.key, o.n, __ldg(P.s[src].key + i), src != 0);
}

// Extra words of source s's entries [0, e) (e <= n_sel), once merge_scan_kernel has run.
__device__ __forceinline__ uint32_t words_before(const MergeParams& P, uint32_t s, uint32_t e) {
  const MergeSource& S = P.s[s];
  return e < S.n_sel ? S.wcnt[e / T] + __ldg(S.wloc + e) : P.totals[s];
}

__global__ void __launch_bounds__(kThreads) merge_key_kernel(MergeParams P) {
  __shared__ uint32_t warp_sums[kWarps];
  uint32_t src, tile;
  bool sel;
  block_role(P, src, sel, tile);
  const MergeSource& S = P.s[src];
  if (!sel) {
#pragma unroll
    for (uint32_t r = 0; r < kItems; ++r) {
      const uint32_t i = item_index(tile, r);
      if (i < S.n) {
        const uint4 h = __ldg(reinterpret_cast<const uint4*>(S.job + i));   // topic, flags, orig, tenant | tenant_pol << 16
        S.key[i] = h.x * P.tenant_classes + __ldg(P.tenant_class + (h.w & 0xFFFFu));
      }
    }
    return;
  }
  uint32_t words[kItems], pre[kItems], total;
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t e = item_index(tile, r);
    words[r] = 0;
    if (e < S.n_sel) {
      const uint32_t x = __ldg(&S.sel_jobs[e].y);
      words[r] = x ? 1u + __ldg(S.sel_extra + x) : 0u;
    }
  }
  tile_scan(words, pre, warp_sums, &total);
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t e = item_index(tile, r);
    if (e < S.n_sel) S.wloc[e] = pre[r];
  }
  if (threadIdx.x == 0) S.wcnt[tile] = total;
}

// CTA s: source s's extra-word counts per selective-list tile -> exclusive prefixes in place, their total -> totals[s]
__global__ void __launch_bounds__(kThreads) merge_scan_kernel(MergeParams P) {
  __shared__ uint32_t warp_sums[kWarps];
  const MergeSource& S = P.s[blockIdx.x];
  const uint32_t total = tile2k::tiles_scan(S.wcnt, S.n_sel_tiles, warp_sums);
  if (threadIdx.x == 0) P.totals[blockIdx.x] = total;
}

__global__ void __launch_bounds__(kThreads) merge_gather_kernel(MergeParams P) {
  const uint32_t lane = threadIdx.x & 31;
  uint32_t src, tile;
  bool sel;
  block_role(P, src, sel, tile);
  const MergeSource& S = P.s[src];
  const uint32_t orig_base = src ? P.s[0].n : 0u;
  if (!sel) {   // sorted slots
#pragma unroll 1
    for (uint32_t r = 0; r < kItems; ++r) {
      const uint32_t i = item_index(tile, r);
      const bool live = i < S.n;
      uint32_t ns = 0;
      if (live) {
        ns = merged_slot(P, src, i);
        const uint4* js = reinterpret_cast<const uint4*>(S.job + i);
        uint4 j0 = __ldg(js), j1 = __ldg(js + 1), j2 = __ldg(js + 2), j3 = __ldg(js + 3);
        j0.z += orig_base;   // JobRec.orig: b's jobs follow a's
        uint4* jd = reinterpret_cast<uint4*>(P.djob + ns);
        jd[0] = j0; jd[1] = j1; jd[2] = j2; jd[3] = j3;
        const uint4* rs = reinterpret_cast<const uint4*>(S.route + i);
        uint4* rd = reinterpret_cast<uint4*>(P.droute + ns);
        rd[0] = __ldg(rs); rd[1] = __ldg(rs + 1);
        P.dslot_of[j0.z] = ns;
      }
      if (P.ww) {   // wide rows: the warp copies each row of this round together
        uint32_t todo = __ballot_sync(FULL, live);
        while (todo) {
          const uint32_t src_lane = __ffs(todo) - 1;
          todo &= todo - 1;
          const uint32_t from = __shfl_sync(FULL, i, src_lane), to = __shfl_sync(FULL, ns, src_lane);
          const uint64_t* a = S.wide + (size_t)from * P.ww;
          uint64_t* b = P.dwide + (size_t)to * P.ww;
          for (uint32_t w = lane; w < P.ww; w += 32) b[w] = __ldg(a + w);
        }
      }
    }
    return;
  }
  // selective-list entries
  const MergeSource& O = P.s[src ^ 1];
  uint32_t* const dextra = P.dsel + 2 * (size_t)P.m_sel;
  if (blockIdx.x == P.s[0].n_tiles + P.s[1].n_tiles && threadIdx.x == 0) dextra[0] = 0;   // x = 0 never points at a list
#pragma unroll 1
  for (uint32_t r = 0; r < kItems; ++r) {
    const uint32_t e = item_index(tile, r);
    if (e >= S.n_sel) continue;
    const uint2 ent = __ldg(S.sel_jobs + e);
    const uint32_t ns = merged_slot(P, src, ent.x);
    // the other source's records before ns are its slots [0, ns - ent.x): its entries among them come first
    const uint32_t before = ns - ent.x;
    uint32_t lo = 0, hi = O.n_sel;
    while (lo < hi) {
      const uint32_t mid = lo + ((hi - lo) >> 1);
      if (__ldg(&O.sel_jobs[mid].x) < before) lo = mid + 1;
      else hi = mid;
    }
    const uint32_t k = lo, p = e + k;
    const uint32_t nx = ent.y ? 1u + words_before(P, src, e) + words_before(P, src ^ 1, k) : 0u;
    P.dsel[2 * (size_t)p] = ns;
    P.dsel[2 * (size_t)p + 1] = nx;
    if (ent.y) {
      const uint32_t c = __ldg(S.sel_extra + ent.y);
      for (uint32_t q = 0; q <= c; ++q) dextra[nx + q] = __ldg(S.sel_extra + ent.y + q);
    }
  }
}

}  // namespace

cudaError_t launch_merge(const MergeParams& P, cudaStream_t s) {
  const uint32_t grid = P.s[0].n_tiles + P.s[1].n_tiles + P.s[0].n_sel_tiles + P.s[1].n_sel_tiles;
  if (grid == 0) return cudaSuccess;
  merge_key_kernel<<<grid, kThreads, 0, s>>>(P);
  merge_scan_kernel<<<2, kThreads, 0, s>>>(P);
  merge_gather_kernel<<<grid, kThreads, 0, s>>>(P);
  return cudaGetLastError();
}
