// kernels.cu — sm_90a (H100) kernels of the policy-gate + dispatch path.
//
//   worker_chunk_kernel + worker_merge_kernel   per heartbeat epoch: load score / overload per worker (strategy_least_loaded.go:157-159,
//                        :177-193), pool kept sorted by load, per-label bitmaps over that order, per-pool argmin
//   policy_kernel        per job batch: first-match over the rule set (safety_policy.go:187-206, 259-294), decision
//                        mapping + tenant MCP + effective-config overlay (kernel.go:187-248), scheduler post-step
//                        (engine.go:528-530)
//   route_kernel         per job batch: pool filter + least-loaded pick (strategy_least_loaded.go:40-136) for the
//                        jobs that may dispatch (engine.go:298-347)
//   route_select_kernel  per job batch, after route_kernel: the worker pick of jobs that name selective placement pairs
//                        (labels few workers carry, e.g. hostnames), from per-pair holder lists
//
// Integer / bit work only: no tensor cores (north star).  Mapping to the hardware:
//   * a batch is two record arrays sorted by topic (64 B policy record, 32 B routing record per job).  A warp owns a
//     tile of 32 consecutive records; its 2 KB of policy records arrive in shared memory by ONE bulk async copy
//     (cp.async.bulk, completion on an mbarrier), issued for the next tile as soon as the lanes hold the current one in
//     registers, so the copy of tile k+1 overlaps the evaluation of tile k; lane = job, four 128-bit shared loads
//   * rule predicates live in bit-rows ("pass-rows") over rule positions; per attribute value a 64-bit summary says
//     which 128-bit words of its row hold anything.  A lane ANDs the summaries of its job's values and visits only the
//     surviving words; the warp walks the union of its lanes' live words, and because the records are topic-sorted and
//     the tables are stored word-major (tab[word][value]), the lanes' 16 B gathers for one word fall into few cache
//     lines (the gather rate of L1 - one 128 B line per cycle - is what bounds this kernel, not HBM)
//   * the tables are a few MB: L2-resident, hot words L1-resident; DRAM traffic is the records and the results
//   * first match = lowest surviving bit per word -> pos2rule -> min over words, all in the lane's registers; argmin
//     over workers = per-pool sorted views + label bitmaps (bitonic sort in shared memory at refresh time)
//   * decision records are written to the job's original index, 16 B per lane
// IEEE float32 with explicit _rn intrinsics, no fast-math: scores compare exactly like Go's.
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../include/cordum_b200.h"
#include "kernels.h"

#define FULL 0xFFFFFFFFu
#define KEY_NONE 0xFFFFFFFFFFFFFFFFull

namespace {

__device__ __forceinline__ uint4 or4(uint4 a, uint4 b) { return make_uint4(a.x | b.x, a.y | b.y, a.z | b.z, a.w | b.w); }
__device__ __forceinline__ uint64_t shfl64(unsigned mask, uint64_t v, int src) {
  uint32_t lo = __shfl_sync(mask, (uint32_t)v, src), hi = __shfl_sync(mask, (uint32_t)(v >> 32), src);
  return ((uint64_t)hi << 32) | lo;
}
__device__ __forceinline__ uint64_t shfl64_xor(unsigned mask, uint64_t v, int lanemask) {
  uint32_t lo = __shfl_xor_sync(mask, (uint32_t)v, lanemask), hi = __shfl_xor_sync(mask, (uint32_t)(v >> 32), lanemask);
  return ((uint64_t)hi << 32) | lo;
}

// float32 -> uint32 whose unsigned order equals the float order (no NaN by construction)
__device__ __forceinline__ uint32_t orderable(float s) {
  if (s == 0.0f) s = 0.0f;   // -0 -> +0: Go's `<` treats them as equal
  uint32_t b = __float_as_uint(s);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}

// A worker's key: (orderable load score << 32) | rank.  Overloaded workers keep their rank but carry
// an all-ones score field, so they sort last and are never selected; KEY_NONE = no candidate / padding.
__device__ __forceinline__ bool key_over(uint64_t k) { return (uint32_t)(k >> 32) == 0xFFFFFFFFu; }

// (key, count-at-minimum-score) pairs form a commutative monoid under this merge
__device__ __forceinline__ void merge_best(uint64_t& key, uint32_t& cnt, uint64_t k2, uint32_t c2) {
  uint32_t s1 = (uint32_t)(key >> 32), s2 = (uint32_t)(k2 >> 32);
  if (key_over(k2)) return;
  if (key_over(key) || s2 < s1) { key = k2; cnt = c2; }
  else if (s2 == s1) { key = k2 < key ? k2 : key; cnt += c2; }
}

}  // namespace

// ------------------------------------------------------------------ K2: worker-table refresh, one CTA per pool chunk
// Per heartbeat epoch: load score + overload test per worker, then the pool's keys in ascending order (the
// load-sorted view lets label-constrained jobs find the least-loaded worker carrying their labels from per-label
// bitmaps).  A pool is cut into chunks of CORDUM_POOL_CHUNK workers so that the whole GPU takes part in the refresh
// instead of one SM per pool: worker_chunk_kernel sorts one chunk per CTA in shared memory (and finishes pools that
// have a single chunk); worker_merge_kernel places every worker of a multi-chunk pool at
//     its index in its own chunk + the number of smaller keys in each sibling chunk        (keys are unique: rank)
// Pools above CORDUM_POOL_SORT_MAX workers keep only min / count-at-min; their jobs scan (route_kernel S').
__device__ __forceinline__ uint64_t worker_key(const DeviceTables& T, uint32_t pos) {
  const Load16 L = T.loads[T.pos_slot[pos]];
  bool over = false;
  if (L.max_parallel > 0) over = __fdiv_rn(__int2float_rn(L.active), __int2float_rn(L.max_parallel)) >= 0.9f;   // :177-184
  over = over || L.cpu >= 90.0f || L.gpu >= 90.0f;                                                               // :185-191
  const float score = __fadd_rn(__fadd_rn(__int2float_rn(L.active), __fdiv_rn(L.cpu, 100.0f)), __fdiv_rn(L.gpu, 100.0f));   // :157-159
  return ((uint64_t)(over ? 0xFFFFFFFFu : orderable(score)) << 32) | T.pos_rank[pos];
}

// Per (pool, label bit): what a job that requires exactly that one placement label gets from the pool - first two matches in
// the non-overloaded prefix of the load-sorted view (argmin + tie flag) and the number of matching workers.  Run by the CTA
// that completes the pool's bitmaps (the single chunk's, or the last merge CTA to finish): a warp per bit, lane = one
// 32-worker word, so even an 8,192-worker pool is eight coalesced steps per bit.  COHERENT = the view was written by other
// CTAs (read it past L1).
template <bool COHERENT>
__device__ __forceinline__ void pool_label_best(const DeviceTables& T, uint32_t p, uint32_t a, uint32_t words, uint32_t nok,
                                                uint32_t warp, uint32_t n_warps, uint32_t lane) {
  if (!T.lbest) return;
  const uint32_t nbits = T.place_bits;
  const uint32_t* bm = T.lbm + T.lbm_off[p];
  for (uint32_t b = warp; b < nbits; b += n_warps) {
    const uint32_t* row = bm + (size_t)b * words;
    uint64_t kstar = KEY_NONE;
    uint32_t kc = 0, tot = 0;
    bool done = false;
    for (uint32_t w0 = 0; w0 < words; w0 += 32) {
      const uint32_t w = w0 + lane, lo = w * 32;
      const uint32_t v = w < words ? (COHERENT ? __ldcg(row + w) : row[w]) : 0u;
      tot += __popc(v);
      uint32_t okv = (done || lo >= nok) ? 0u : (nok - lo >= 32 ? v : v & ((1u << (nok - lo)) - 1u));
      while (!done) {   // at most two rounds over the whole row: the argmin, then the next match for the tie flag
        const unsigned hit = __ballot_sync(FULL, okv != 0);
        if (!hit) break;
        const int L = __ffs((int)hit) - 1;
        const uint32_t pos = __shfl_sync(FULL, lo + (uint32_t)(okv ? __ffs((int)okv) - 1 : 0), L);
        const uint64_t kk = COHERENT ? __ldcg(T.skey + a + pos) : T.skey[a + pos];
        if (kstar == KEY_NONE) { kstar = kk; kc = 1; }
        else { if ((uint32_t)(kk >> 32) == (uint32_t)(kstar >> 32)) kc = 2; done = true; }
        if ((int)lane == L) okv &= okv - 1;
      }
    }
    tot = __reduce_add_sync(FULL, tot);
    if (lane == 0) T.lbest[(size_t)p * nbits + b] = make_uint4((uint32_t)kstar, (uint32_t)(kstar >> 32), kc, tot);
  }
}

// One CTA of CORDUM_POOL_CHUNK (512) threads per chunk: thread i holds key i.  Bitonic network: exchanges inside a warp are
// register shuffles (35 of the 45 stages of a 512-key sort), only partner distances >= 32 go through shared memory.
template <uint32_t NT>
__global__ void __launch_bounds__(NT) worker_chunk_kernel(DeviceTables T) {
  constexpr uint32_t CH = CORDUM_POOL_CHUNK;
  static_assert(NT == CH, "one thread per key");
  __shared__ uint64_t sk[CH];
  __shared__ uint32_t s_cnt, s_nok;
  const uint32_t g = blockIdx.x, tid = threadIdx.x, lane = tid & 31;
  const uint32_t p = T.chunk_pool[g], c = g - T.pool_chunk0[p], m = T.pool_chunk0[p + 1] - T.pool_chunk0[p];
  const uint32_t a = T.pool_off[p], n = T.pool_off[p + 1] - a;
  const uint32_t cs = c * CH, len = n - cs < CH ? n - cs : CH;   // an empty pool has one empty chunk
  const bool sortable = n <= CORDUM_POOL_SORT_MAX;
  uint32_t n_pad = 32;   // at least a warp: the shuffle stages need full warps
  while (n_pad < len) n_pad <<= 1;
  if (tid == 0) { s_cnt = 0; s_nok = 0; }
  uint64_t key = KEY_NONE;
  if (tid < len) { key = worker_key(T, a + cs + tid); T.pos_key[a + cs + tid] = key; }
  if (!sortable) return;   // chunk 0 of the pool reduces min / count in worker_merge_kernel
  // bitonic sort of n_pad keys (ascending), thread i = position i; KEY_NONE pads sort to the end
  for (uint32_t k = 2; k <= n_pad; k <<= 1)
    for (uint32_t jj = k >> 1; jj > 0; jj >>= 1) {
      uint64_t other;
      if (jj >= 32) {
        __syncthreads();
        sk[tid] = key;
        __syncthreads();
        other = sk[tid ^ jj];
      } else other = shfl64_xor(FULL, key, (int)jj);
      const bool up = (tid & k) == 0, lower = (tid & jj) == 0;   // ascending block; this thread keeps the smaller one
      const bool take_min = up == lower;
      if (tid < n_pad) key = take_min ? (other < key ? other : key) : (other > key ? other : key);
    }
  __syncthreads();
  sk[tid] = key;
  __syncthreads();
  const uint32_t words = (n + 31) >> 5, nbits = T.place_bits;
  uint32_t* bm = T.lbm + T.lbm_off[p];
  if (m > 1) {
    // hand the sorted chunk to worker_merge_kernel; clear what it accumulates into
    if (tid < len) T.ckey[a + cs + tid] = key;
    const uint64_t total = (uint64_t)nbits * words;
    for (uint64_t i = total * c / m + tid; i < total * (c + 1) / m; i += NT) bm[i] = 0;
    if (c == 0 && tid == 0) { T.pool_mincnt[p] = 0; T.pool_nok[p] = 0; T.pool_done[p] = 0; }
    return;
  }
  // single chunk: sorted view + label bitmaps; warp w = the 32 sorted workers of bitmap word w
  const uint64_t k0 = n ? sk[0] : KEY_NONE;
  const bool none = n == 0 || key_over(k0);
  uint32_t cnt = 0, ok = 0;
  const uint32_t w = tid >> 5;
  if (w < words) {
    uint64_t llo = 0, lhi = 0;
    uint32_t src = 0;
    if (tid < n) {
      src = T.rank_pos[(uint32_t)(key & 0xFFFFFFFFu)];   // every key (overloaded ones too) carries its rank
      llo = T.pos_label_lo[src]; lhi = T.pos_label_hi[src];
      T.skey[a + tid] = key;
      cnt = (!none && (uint32_t)(key >> 32) == (uint32_t)(k0 >> 32)) ? 1u : 0u;
      ok = key_over(key) ? 0u : 1u;
    }
    for (uint32_t b0 = 0; b0 < nbits; b0 += 32) {   // lane t keeps the word of label bit b0+t, then one strided store each
      uint32_t mine = 0;
      const uint32_t lim = nbits - b0 < 32 ? nbits - b0 : 32;
      uint32_t part;   // b0 is a multiple of 32
      if (b0 < 64) part = (uint32_t)(llo >> b0);
      else if (b0 < 128) part = (uint32_t)(lhi >> (b0 - 64));
      else part = tid < n ? (uint32_t)(T.pos_label_x[(size_t)src * T.wide.xw_place + ((b0 - 128) >> 6)] >> (b0 & 32)) : 0u;   // bits 128...
      for (uint32_t t = 0; t < lim; ++t) {
        const unsigned bal = __ballot_sync(FULL, (part >> t) & 1u);
        if (lane == t) mine = bal;
      }
      if (lane < lim) bm[(size_t)(b0 + lane) * words + w] = mine;
    }
  }
  cnt = __reduce_add_sync(FULL, cnt); ok = __reduce_add_sync(FULL, ok);
  if (lane == 0 && cnt) atomicAdd(&s_cnt, cnt);
  if (lane == 0 && ok) atomicAdd(&s_nok, ok);
  __syncthreads();   // also: this CTA's skey / bitmap stores are visible to all of its threads from here on
  if (tid == 0) { T.pool_best[p] = none ? KEY_NONE : k0; T.pool_mincnt[p] = s_cnt; T.pool_sorted[p] = 1; T.pool_nok[p] = s_nok; }
  pool_label_best<false>(T, p, a, words, s_nok, tid >> 5, NT >> 5, lane);
}

__global__ void __launch_bounds__(512) worker_merge_kernel(DeviceTables T) {
  constexpr uint32_t CH = CORDUM_POOL_CHUNK, NT = 512;   // one thread per worker of the chunk
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ uint32_t s_cnt, s_nok;
  __shared__ uint64_t s_best;
  uint64_t* sp = reinterpret_cast<uint64_t*>(smem_raw);   // the pool's keys, chunk by chunk, each chunk ascending
  const uint32_t g = T.merge_list[blockIdx.x], tid = threadIdx.x, lane = tid & 31;
  const uint32_t p = T.chunk_pool[g], c = g - T.pool_chunk0[p], m = T.pool_chunk0[p + 1] - T.pool_chunk0[p];
  const uint32_t a = T.pool_off[p], n = T.pool_off[p + 1] - a;
  if (tid == 0) { s_cnt = 0; s_nok = 0; s_best = KEY_NONE; }
  __syncthreads();
  if (n > CORDUM_POOL_SORT_MAX) {   // unsorted pool: min / count-at-min by reduction (listed once, as chunk 0)
    uint64_t best = KEY_NONE;
    for (uint32_t i = tid; i < n; i += NT) { const uint64_t k = T.pos_key[a + i]; if (!key_over(k) && k < best) best = k; }
    for (int o = 16; o; o >>= 1) { const uint64_t v = shfl64_xor(FULL, best, o); best = v < best ? v : best; }
    if (lane == 0) atomicMin(reinterpret_cast<unsigned long long*>(&s_best), (unsigned long long)best);
    __syncthreads();
    best = s_best;
    uint32_t cnt = 0;
    for (uint32_t i = tid; i < n; i += NT) { const uint64_t k = T.pos_key[a + i]; cnt += (!key_over(k) && (uint32_t)(k >> 32) == (uint32_t)(best >> 32)) ? 1u : 0u; }
    cnt = __reduce_add_sync(FULL, cnt);
    if (lane == 0 && cnt) atomicAdd(&s_cnt, cnt);
    __syncthreads();
    if (tid == 0) { T.pool_best[p] = best; T.pool_mincnt[p] = best == KEY_NONE ? 0 : s_cnt; T.pool_sorted[p] = 0; }
    return;
  }
  for (uint32_t i = tid; i < n; i += NT) sp[i] = T.ckey[a + i];
  __syncthreads();
  uint64_t k0 = KEY_NONE;
  for (uint32_t cc = 0; cc < m; ++cc) { const uint64_t h = sp[cc * CH]; k0 = h < k0 ? h : k0; }
  const bool none = key_over(k0);
  const uint32_t cs = c * CH, len = n - cs < CH ? n - cs : CH;
  const uint32_t words = (n + 31) >> 5;
  uint32_t* bm = T.lbm + T.lbm_off[p];
  uint32_t cnt = 0, ok = 0;
  for (uint32_t i = tid; i < len; i += NT) {
    const uint64_t k = sp[cs + i];
    uint32_t idx = i;
    for (uint32_t cc = 0; cc < m; ++cc) {
      if (cc == c) continue;
      const uint64_t* q = sp + cc * CH;
      uint32_t lo = 0, hi = n - cc * CH < CH ? n - cc * CH : CH;   // lower bound of k in the sibling chunk
      while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (q[mid] < k) lo = mid + 1; else hi = mid; }
      idx += lo;
    }
    const uint32_t src = T.rank_pos[(uint32_t)(k & 0xFFFFFFFFu)];
    uint64_t llo = T.pos_label_lo[src], lhi = T.pos_label_hi[src];
    T.skey[a + idx] = k;
    const uint32_t w = idx >> 5, bitv = 1u << (idx & 31);
    while (llo) { const uint32_t b = __ffsll((long long)llo) - 1; llo &= llo - 1; atomicOr(&bm[(size_t)b * words + w], bitv); }
    while (lhi) { const uint32_t b = 64 + __ffsll((long long)lhi) - 1; lhi &= lhi - 1; atomicOr(&bm[(size_t)b * words + w], bitv); }
    for (uint32_t x = 0; x < T.wide.xw_place; ++x)   // label bits 128...
      for (uint64_t lx = T.pos_label_x[(size_t)src * T.wide.xw_place + x]; lx; lx &= lx - 1)
        atomicOr(&bm[(size_t)(128u + 64u * x + (uint32_t)__ffsll((long long)lx) - 1u) * words + w], bitv);
    cnt += (!none && (uint32_t)(k >> 32) == (uint32_t)(k0 >> 32)) ? 1u : 0u;
    ok += key_over(k) ? 0u : 1u;
  }
  __threadfence();   // every thread's stores into the pool's view / bitmaps are ordered before its CTA signs off below
  cnt = __reduce_add_sync(FULL, cnt); ok = __reduce_add_sync(FULL, ok);
  if (lane == 0 && cnt) atomicAdd(&s_cnt, cnt);
  if (lane == 0 && ok) atomicAdd(&s_nok, ok);
  __syncthreads();
  __shared__ uint32_t s_last;
  if (tid == 0) {
    if (s_cnt) atomicAdd(&T.pool_mincnt[p], s_cnt);
    if (s_nok) atomicAdd(&T.pool_nok[p], s_nok);
    if (c == 0) { T.pool_best[p] = none ? KEY_NONE : k0; T.pool_sorted[p] = 1; }
    __threadfence();   // this CTA's share of the view, bitmaps and counters, before it signs off
    s_last = atomicAdd(&T.pool_done[p], 1u) == m - 1 ? 1u : 0u;
  }
  __syncthreads();
  if (s_last) {   // every CTA of the pool has signed off: the view is complete
    __threadfence();
    const uint32_t nok = __ldcg(T.pool_nok + p);
    pool_label_best<true>(T, p, a, words, nok, tid >> 5, NT >> 5, lane);
  }
}

// ------------------------------------------------------------------ wide masks (tables.h WideLayout)
// Everything below is reached only when a dictionary outgrew the records' own mask fields (T.wide_words != 0).
__device__ __forceinline__ bool wide_need_ok(const DeviceTables& T, uint32_t r, const uint64_t* wrow, uint32_t flags) {
  const uint32_t xq = T.wide.xw_req, xl = T.wide.xw_lab;
  const uint64_t* nx = T.rule_need_x + (size_t)r * (xq + xl);
  for (uint32_t k = 0; k < xq; ++k) if (__ldg(nx + k) & ~__ldg(wrow + WIDE_O_REQ(T.wide) + k)) return false;   // containsAll (:320-330)
  uint64_t any = 0;
  bool sub = true;
  for (uint32_t k = 0; k < xl; ++k) { const uint64_t n = __ldg(nx + xq + k); any |= n; sub &= (n & ~__ldg(wrow + WIDE_O_LAB(T.wide) + k)) == 0; }
  return any == 0 || ((flags & JF_HAS_LABELS) && sub);                                                            // labelsMatch (:332-345)
}
// poolSatisfies' subset test (:255-262) over all words of the requires mask
__device__ __forceinline__ bool pool_req_subset(const DeviceTables& T, uint32_t pid, uint64_t need_req, const uint64_t* wrow) {
  if (need_req & ~__ldg(T.pool_req_mask + pid)) return false;
  if (wrow) {
    const uint32_t xq = T.wide.xw_req;
    for (uint32_t k = 0; k < xq; ++k)
      if ((__ldg(wrow + WIDE_O_REQP(T.wide) + k) & ~__ldg(T.req_blank_x + k)) & ~__ldg(T.pool_req_x + (size_t)pid * xq + k)) return false;
  }
  return true;
}
__device__ __forceinline__ bool place_x_any(const DeviceTables& T, const uint64_t* wrow) {
  uint64_t any = 0;
  if (wrow) for (uint32_t k = 0; k < T.wide.xw_place; ++k) any |= __ldg(wrow + WIDE_O_PLACE(T.wide) + k);
  return any != 0;
}
__device__ __forceinline__ bool place_x_ok(const DeviceTables& T, uint32_t pos, const uint64_t* wrow) {   // matchesLabels (:161-175), bits 128...
  if (wrow)
    for (uint32_t k = 0; k < T.wide.xw_place; ++k) {
      const uint64_t need = __ldg(wrow + WIDE_O_PLACE(T.wide) + k);
      if ((__ldg(T.pos_label_x + (size_t)pos * T.wide.xw_place + k) & need) != need) return false;
    }
  return true;
}

// ------------------------------------------------------------------ policy: first match + decision
// A warp owns a tile of 32 consecutive (topic-sorted) job records: lane = job.  Needs no worker state, so it runs
// concurrently with the heartbeat exchange and the worker-table refresh.
//   L  the tile's records arrive in shared memory through one bulk async copy per tile (prefetched one tile ahead)
//   P  live words = AND of the summaries of the job's attribute values; the warp walks the union of its lanes' live
//      words; in each, a lane ANDs the 128-bit cells of the 7-12 rows its job selects; the lowest surviving bit maps
//      back to an original rule index; first match = min over words
//   D  decision mapping, tenant MCP, effective-config overlay, approval flags, scheduler post-step
namespace {
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity)
      : "memory");
}
// global -> shared bulk copy (the TMA engine; no tensor map needed for a contiguous run), completion on the mbarrier
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ uint4 and3(uint4 a, uint4 b, uint4 c) { return make_uint4(a.x & b.x & c.x, a.y & b.y & c.y, a.z & b.z & c.z, a.w & b.w & c.w); }
}  // namespace

template <int MINB>
__global__ void __launch_bounds__(256, MINB) policy_kernel(KParams P) {
  const DeviceTables& T = P.t;
  const unsigned lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const uint32_t n_tiles = (P.n_jobs + 31u) >> 5;
  const uint32_t warps_total = (gridDim.x * blockDim.x) >> 5;
  const uint32_t warp_id = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  __shared__ __align__(128) JobRec s_tile[8][32];   // one tile per warp
  __shared__ __align__(8) uint64_t s_bar[8];
  JobRec* tile_buf = s_tile[wib];
  uint64_t* bar = &s_bar[wib];
  if (lane == 0) mbar_init(bar, 1);
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  __syncwarp();
  auto prefetch = [&](uint32_t tile) {   // lane 0: this warp's next tile, global -> shared
    if (lane == 0 && tile < n_tiles) {
      const uint32_t jobs = P.n_jobs - tile * 32u < 32u ? P.n_jobs - tile * 32u : 32u;
      const uint32_t bytes = jobs * (uint32_t)sizeof(JobRec);
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // the lanes' reads of the buffer precede the async write
      mbar_expect_tx(bar, bytes);
      bulk_g2s(tile_buf, P.recs.job + (size_t)tile * 32u, bytes, bar);
    }
  };
  prefetch(warp_id);
  uint32_t parity = 0;
  const uint32_t n_words = T.row_u4, G = T.sum_group, use = T.sum_use;

  for (uint32_t tile = warp_id; tile < n_tiles; tile += warps_total) {
    const uint32_t s = tile * 32 + lane;   // slot in the sorted order
    const bool valid = s < P.n_jobs;
    mbar_wait(bar, parity);
    parity ^= 1u;
    // ---- L: the lane's record, four 128-bit shared loads
    uint4 q0 = make_uint4(0, 0, 0, 0), q1 = q0, q2 = q0, q3 = q0;
    if (valid) {
      const uint4* rp = reinterpret_cast<const uint4*>(tile_buf + lane);
      q0 = rp[0]; q1 = rp[1]; q2 = rp[2]; q3 = rp[3];
    }
    __syncwarp();
    prefetch(tile + warps_total);
    const uint32_t c_topic = q0.x, c_flags = q0.y, c_orig = q0.z, c_tenant = q0.w & 0xFFFFu, c_tpol = q0.w >> 16;
    const uint32_t c_cap = q1.x & 0xFFFFu, c_pack = q1.x >> 16, c_actor = q1.y & 0xFFFFu, c_eff = q1.y >> 16;
    const uint32_t mid[4] = {q1.z & 0xFFFFu, q1.z >> 16, q1.w & 0xFFFFu, q1.w >> 16};
    const uint64_t c_risk = ((uint64_t)q2.y << 32) | q2.x, c_req = ((uint64_t)q2.w << 32) | q2.z, c_lab = ((uint64_t)q3.y << 32) | q3.x;

    // =================================================================== P: first matching rule
    const bool bypass = P.honor_approved && (c_flags & JF_APPROVED);                                    // engine.go:484-522
    const bool early = (c_flags & (JF_TOPIC_MISSING | JF_TOPIC_UNSUPPORTED)) != 0;                        // kernel.go:171-176
    const bool eval = valid && !bypass && !early;
    const bool mcp_used = (c_flags & JF_MCP_USED) != 0;
    const uint32_t combo = CORDUM_COMBO_INDEX(c_flags);
    const uint64_t* wrow = (T.wide_words && P.recs.wide && valid) ? P.recs.wide + (size_t)s * T.wide_words : nullptr;   // rare: masks beyond the record's
    uint64_t live = 0;
    if (eval) {
      live = __ldg(T.sum_topic + c_topic);
      if (use & SUM_TENANT) live &= __ldg(T.sum_tenant + c_tenant);
      if (use & SUM_CAP) live &= __ldg(T.sum_cap + c_cap);
      if (use & SUM_PACK) live &= __ldg(T.sum_pack + c_pack);
      if (use & SUM_ACTOR) live &= __ldg(T.sum_actor + c_actor);
      if (use & SUM_COMBO) live &= __ldg(T.sum_combo + combo);
      if (use & SUM_RISK) {
        uint64_t rs = c_risk ? 0ull : __ldg(T.sum_risk);
        for (uint64_t m = c_risk; m; m &= m - 1) rs |= __ldg(T.sum_risk + __ffsll((long long)m));
        if (wrow)
          for (uint32_t k = 0; k < T.wide.xw_risk; ++k)
            for (uint64_t m = __ldg(wrow + k); m; m &= m - 1) rs |= __ldg(T.sum_risk + 64u * (k + 1u) + (uint32_t)__ffsll((long long)m));
        live &= rs;
      }
    }
    // cell indices inside one word of the unified table: fixed for the tile
    const uint32_t i_topic = T.off_topic + c_topic, i_tenant = T.off_tenant + c_tenant, i_cap = T.off_cap + c_cap,
                   i_pack = T.off_pack + c_pack, i_actor = T.off_actor + c_actor, i_combo = T.off_combo + combo;
    // risk tags: containsAny = OR over the job's tags (:308-318); row 0 = "no referenced tag", row 1+b = tag b.  The first
    // three rows are loaded without branching (a job with fewer tags repeats its first row); a fourth tag onwards loops.
    uint64_t rm = c_risk;
    const uint32_t i_risk0 = T.off_risk + (uint32_t)__ffsll((long long)rm);
    rm &= rm - 1;
    const bool risk2 = rm != 0;
    const uint32_t i_risk1 = risk2 ? T.off_risk + (uint32_t)__ffsll((long long)rm) : i_risk0;
    rm &= rm - 1;
    const bool risk3 = rm != 0;
    const uint32_t i_risk2 = risk3 ? T.off_risk + (uint32_t)__ffsll((long long)rm) : i_risk0;
    rm &= rm - 1;   // tags beyond the third
    uint32_t best = 0xFFFFFFFFu;
    uint32_t u_lo = __reduce_or_sync(FULL, (uint32_t)live), u_hi = __reduce_or_sync(FULL, (uint32_t)(live >> 32));
    for (uint64_t un = ((uint64_t)u_hi << 32) | u_lo; un; un &= un - 1) {   // warp-uniform walk over the union
      const uint32_t g = (uint32_t)__ffsll((long long)un) - 1u;
      if (!((live >> g) & 1ull)) continue;
      for (uint32_t w = g * G; w < (g + 1) * G && w < n_words; ++w) {
        const uint4* bw = reinterpret_cast<const uint4*>(T.rows) + (size_t)w * T.n_cells;
        uint4 rk = __ldg(bw + i_risk0);
        if (risk2) rk = or4(rk, __ldg(bw + i_risk1));
        if (risk3) rk = or4(rk, __ldg(bw + i_risk2));
        for (uint64_t m = rm; m; m &= m - 1) rk = or4(rk, __ldg(bw + T.off_risk + (uint32_t)__ffsll((long long)m)));
        if (wrow)   // tags 64...: row 1 + tag
          for (uint32_t k = 0; k < T.wide.xw_risk; ++k)
            for (uint64_t m = __ldg(wrow + k); m; m &= m - 1) rk = or4(rk, __ldg(bw + T.off_risk + 64u * (k + 1u) + (uint32_t)__ffsll((long long)m)));
        uint4 acc = and3(__ldg(bw + i_topic), __ldg(bw + i_tenant), __ldg(bw + i_cap));
        acc = and3(acc, __ldg(bw + i_pack), __ldg(bw + i_actor));
        acc = and3(acc, __ldg(bw + i_combo), rk);
        if (mcp_used) {   // mcpMatch (:365-382)
          acc = and3(acc, __ldg(bw + T.off_mcp[0] + mid[0]), __ldg(bw + T.off_mcp[1] + mid[1]));
          acc = and3(acc, __ldg(bw + T.off_mcp[2] + mid[2]), __ldg(bw + T.off_mcp[3] + mid[3]));
        }
        // Surviving bits -> original rule index.  Inside a word the positions ascend with the rule index, so the lowest
        // surviving bit is the word's first match; a further bit is looked at only when that rule carries a requires /
        // labels subset test (containsAll :320-330, labelsMatch :332-345) and the test fails.
        uint32_t wv[4] = {acc.x, acc.y, acc.z, acc.w};
        while (wv[0] | wv[1] | wv[2] | wv[3]) {
          uint32_t sel = 0, base = 0;
#pragma unroll
          for (int k = 3; k >= 0; --k) if (wv[k]) { sel = wv[k]; base = 32u * (uint32_t)k; }
          const uint32_t pos = w * 128u + base + (uint32_t)__ffs((int)sel) - 1u;
          const uint32_t r = __ldg(T.pos2rule + pos);
          bool ok = true;
          if ((__ldg(T.chk_words + (pos >> 5)) >> (pos & 31)) & 1u) {
            const uint64_t need = __ldg(T.rule_req_need + r), ln = __ldg(T.rule_lab_need + r);
            ok = ((need & ~c_req) == 0) && (ln == 0 || ((c_flags & JF_HAS_LABELS) && (ln & ~c_lab) == 0));
            if (ok && wrow) ok = wide_need_ok(T, r, wrow, c_flags);
          }
          if (ok) { best = r < best ? r : best; break; }
          const uint32_t drop = sel & (sel - 1);
#pragma unroll
          for (int k = 0; k < 4; ++k) if (base == 32u * (uint32_t)k) wv[k] = drop;
        }
      }
    }
    const int first = (int)best;   // 0xFFFFFFFF -> -1: no rule matched

    // =================================================================== D: decision (thread per job)
    uint32_t dec = CORDUM_DEC_UNSPECIFIED, sched = CORDUM_DEC_UNSPECIFIED, rflags = 0, reason = 0;
    int rule = -1;
    if (valid) {
      if (bypass) { dec = sched = CORDUM_DEC_ALLOW; reason = CORDUM_REASON_APPROVAL_GRANTED; rflags = CORDUM_F_APPROVED_BYPASS; }
      else if (c_flags & JF_TOPIC_MISSING) { dec = sched = CORDUM_DEC_DENY; reason = CORDUM_REASON_MISSING_TOPIC; }
      else if (c_flags & JF_TOPIC_UNSUPPORTED) { dec = sched = CORDUM_DEC_DENY; reason = CORDUM_REASON_UNSUPPORTED_TOPIC; }
      else {
        rule = first;
        uint32_t code = CORDUM_DEC_ALLOW;
        bool hascons = false;
        if (first >= 0) { uint8_t rd = __ldg(T.rule_dec + first); code = rd & 0x7Fu; hascons = rd & 0x80u; }
        const bool rule_approval = code == CORDUM_DEC_REQUIRE_HUMAN;   // safety_policy.go:200
        uint32_t tm = 0;                                               // tenant MCP lists, kernel.go:190-195
        if (mcp_used && c_tpol) {
          const uint8_t* base = T.tenant_mcp + (size_t)(c_tpol - 1) * 4 * T.mcp_stride;
          for (int q = 0; q < 4 && !tm; ++q) { uint8_t v = __ldg(base + q * T.mcp_stride + mid[q]); if (v) tm = 1 + q * 2 + (v - 1); }
          if (tm) code = CORDUM_DEC_DENY;
        }
        dec = CORDUM_DEC_ALLOW;                                        // kernel.go:198-215
        if (code == CORDUM_DEC_DENY) { dec = CORDUM_DEC_DENY; reason = tm ? CORDUM_REASON_TENANT_MCP + (tm - 1) : CORDUM_REASON_RULE; }
        else if (code == CORDUM_DEC_REQUIRE_HUMAN) { dec = CORDUM_DEC_REQUIRE_HUMAN; reason = CORDUM_REASON_RULE; }
        else if (code == CORDUM_DEC_THROTTLE) { dec = CORDUM_DEC_THROTTLE; reason = CORDUM_REASON_RULE; }
        else if (code == CORDUM_DEC_ALLOW_WITH_CONSTRAINTS || hascons) dec = CORDUM_DEC_ALLOW_WITH_CONSTRAINTS;
        if (c_eff) {                                                   // kernel.go:218-231
          const uint8_t tb = __ldg(T.eff_topic + (size_t)c_eff * T.topic_stride + c_topic);
          if (tb & 1) { dec = CORDUM_DEC_DENY; reason = CORDUM_REASON_EFF_DENIED_TOPIC; }
          if (tb & 2) { dec = CORDUM_DEC_DENY; reason = CORDUM_REASON_EFF_NOT_ALLOWED_TOPIC; }
          if (mcp_used) {
            const uint8_t* base = T.eff_mcp + (size_t)c_eff * 4 * T.mcp_stride;
            uint32_t em = 0;
            for (int q = 0; q < 4 && !em; ++q) { uint8_t v = __ldg(base + q * T.mcp_stride + mid[q]); if (v) em = 1 + q * 2 + (v - 1); }
            if (em) { dec = CORDUM_DEC_DENY; reason = CORDUM_REASON_EFF_MCP + (em - 1); }
          }
        }
        const bool approval = rule_approval || dec == CORDUM_DEC_REQUIRE_HUMAN;   // kernel.go:233
        rflags = CORDUM_F_HAS_SNAPSHOT | (approval ? CORDUM_F_APPROVAL_REQUIRED : 0) | (hascons ? CORDUM_F_CONSTRAINTS : 0);
        sched = dec;                                                   // engine.go:528-530
        if (approval && (dec == CORDUM_DEC_ALLOW || dec == CORDUM_DEC_ALLOW_WITH_CONSTRAINTS)) sched = CORDUM_DEC_REQUIRE_HUMAN;
      }
    }

    const uint32_t head = dec | (sched << 8) | (rflags << 16);
    if (valid)   // 16 B store per lane at the job's original index; the route fields are filled by route_kernel
      reinterpret_cast<uint4*>(P.out)[c_orig] = make_uint4(head, reason & 0xFFu, (uint32_t)rule, 0xFFFFFFFFu);
    if (P.route_list) {   // compact the jobs that may dispatch (engine.go:298-347): one atomic per tile
      const bool dr = valid && (sched == CORDUM_DEC_ALLOW || sched == CORDUM_DEC_ALLOW_WITH_CONSTRAINTS);
      const unsigned m = __ballot_sync(FULL, dr);
      if (m) {
        uint32_t base = 0;
        if (lane == 0) base = atomicAdd(P.route_count, (uint32_t)__popc(m));
        base = __shfl_sync(FULL, base, 0);
        if (dr) P.route_list[base + __popc(m & ((1u << lane) - 1u))] = make_uint2(s, head);   // slot + what policy decided
      }
    }
  }
}


// ------------------------------------------------------------------ route: pool filter + least-loaded pick
// Works on the compacted list of jobs that may dispatch (written by policy_kernel; in ROUTE_ONLY mode: all jobs).
//   D  topic->pools, preferred_pool, requires filter, preferred_worker_id and, for label-free jobs, the
//      merge of per-pool best keys: thread per job.
//   S  jobs with placement labels: 4 jobs per warp step, 8 lanes each.  For every eligible pool the group ANDs the
//      pool's label bitmaps over its load-sorted view (lane = 32 workers); first set bit in the non-overloaded
//      prefix = argmin, the next match decides the tie flag, popcount = candidate total.
//   S' jobs that touch a pool larger than K2's sort buffer: warp per job, coalesced scan (rare).
template <bool ROUTE_ONLY, int MINB = 4>
__global__ void __launch_bounds__(256, MINB) route_kernel(KParams P) {
  const DeviceTables& T = P.t;
  const unsigned lane = threadIdx.x & 31, g = lane >> 3, sub = lane & 7;
  const uint32_t n_items = ROUTE_ONLY ? P.n_jobs : *P.route_count;
  const uint32_t n_tiles = (n_items + 31u) >> 5;
  const uint32_t warps_total = (gridDim.x * blockDim.x) >> 5;
  const uint32_t warp_id = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;

  for (uint32_t tile = warp_id; tile < n_tiles; tile += warps_total) {
    const uint32_t item = tile * 32 + lane;
    const bool valid = item < n_items;
    uint32_t j = 0, head = 0, c_orig = 0;   // j: slot in the sorted record arrays
    uint32_t c_flags = 0, c_topic = 0, c_ppool = 0, c_pwork = 0;
    uint64_t c_req = 0, c_plo = 0, c_phi = 0;
    if (valid) {
      if (ROUTE_ONLY) j = item;
      else { const uint2 e = P.route_list[item]; j = e.x; head = e.y; }
      const uint4 a = __ldg(reinterpret_cast<const uint4*>(P.recs.job + j));   // topic, flags, orig of the 64 B record
      const uint4 r0 = __ldg(reinterpret_cast<const uint4*>(P.recs.route + j)), r1 = __ldg(reinterpret_cast<const uint4*>(P.recs.route + j) + 1);
      c_topic = a.x; c_flags = a.y; c_orig = a.z;
      c_plo = ((uint64_t)r0.y << 32) | r0.x; c_phi = ((uint64_t)r0.w << 32) | r0.z;
      c_req = ((uint64_t)r1.y << 32) | r1.x; c_ppool = r1.z; c_pwork = r1.w;
    }
    const uint64_t* wrow = (T.wide_words && P.recs.wide && valid) ? P.recs.wide + (size_t)j * T.wide_words : nullptr;   // rare: masks beyond the record's
    uint32_t rflags = 0, route = CORDUM_ROUTE_NOT_ATTEMPTED;
    int slot = -1;

    // =================================================================== D: pool filter, thread per job
    bool need_scan = false, slow = false;
    uint32_t r_off = 0, r_cnt = 0;
    int r_single = -1;
    uint64_t best = KEY_NONE;
    uint32_t bcnt = 0, total = 0;
    if (valid) {
      if (c_flags & JF_TOPIC_RAW_EMPTY) route = CORDUM_ROUTE_MISSING_TOPIC;   // :41-43
      else {
        r_off = __ldg(T.topic_pool_off + c_topic);
        r_cnt = __ldg(T.topic_pool_cnt + c_topic);
        if (c_ppool) {                                                         // preferred_pool (:50-55)
          bool found = false;
          if (c_ppool != CORDUM_PREF_UNKNOWN)
            for (uint32_t k = 0; k < r_cnt; ++k) found |= __ldg(T.pool_list + r_off + k) == c_ppool - 1;
          if (!found) route = CORDUM_ROUTE_NO_POOL_PREFERRED;
          else { r_single = (int)(c_ppool - 1); r_cnt = 1; }
        }
        if (route == CORDUM_ROUTE_NOT_ATTEMPTED && r_cnt == 0) route = CORDUM_ROUTE_NO_POOL_TOPIC;   // :56-58
        if (route == CORDUM_ROUTE_NOT_ATTEMPTED) {
          const bool req_any = c_flags & JF_REQ_NONEMPTY, req_unknown = c_flags & JF_REQ_UNKNOWN;
          const uint64_t need_req = c_req & ~T.req_blank_mask;
          const bool unsat = c_flags & JF_PLACE_UNSAT;
          const bool wide_place = place_x_any(T, wrow);
          const bool labelled = (c_plo | c_phi) != 0 || unsat || wide_place;
          // exactly one required label: the per-(pool, bit) answers of the refresh (pool_label_best) settle it here
          int one_bit = -1;
          if (T.lbest && !unsat && !wide_place) {
            if (c_phi == 0 && c_plo && !(c_plo & (c_plo - 1))) one_bit = __ffsll((long long)c_plo) - 1;
            else if (c_plo == 0 && c_phi && !(c_phi & (c_phi - 1))) one_bit = 64 + __ffsll((long long)c_phi) - 1;
          }
          int pw_pos = -1;
          uint32_t pw_pool = 0xFFFFFFFFu;
          if (c_pwork && c_pwork != CORDUM_PREF_UNKNOWN) {
            uint32_t p1 = __ldg(T.slot_pos + (c_pwork - 1));
            if (p1) { pw_pos = (int)p1 - 1; pw_pool = __ldg(T.pos_pool + pw_pos); }
          }
          uint32_t n_elig = 0;
          bool pw_in_set = false;
          for (uint32_t k = 0; k < r_cnt; ++k) {
            const uint32_t pid = r_single >= 0 ? (uint32_t)r_single : __ldg(T.pool_list + r_off + k);
            // poolSatisfies (:241-265)
            if (req_any && !(__ldg(T.pool_req_nonempty + pid) && !req_unknown && pool_req_subset(T, pid, need_req, wrow))) continue;
            n_elig++;
            pw_in_set |= pid == pw_pool;
            if (!labelled) {
              total += __ldg(T.pool_off + pid + 1) - __ldg(T.pool_off + pid);
              merge_best(best, bcnt, T.pool_best[pid], T.pool_mincnt[pid]);
            } else {
              const bool sorted = T.pool_sorted[pid] != 0;
              slow |= !sorted;
              if (one_bit >= 0 && sorted) {
                const uint4 lb = __ldg(T.lbest + (size_t)pid * T.place_bits + (uint32_t)one_bit);
                total += lb.w;
                merge_best(best, bcnt, ((uint64_t)lb.y << 32) | lb.x, lb.z);
              }
            }
          }
          const bool settled = one_bit >= 0 && !slow;   // every eligible pool answered from the table
          if (n_elig == 0) route = CORDUM_ROUTE_NO_POOL_REQUIRES;              // :64-66
          else {
            bool took_pref = false;
            if (pw_pos >= 0 && pw_in_set && !unsat) {                           // :73-87
              uint64_t llo = __ldg(T.pos_label_lo + pw_pos), lhi = __ldg(T.pos_label_hi + pw_pos);
              if ((llo & c_plo) == c_plo && (lhi & c_phi) == c_phi && place_x_ok(T, (uint32_t)pw_pos, wrow) && !key_over(T.pos_key[pw_pos])) {
                took_pref = true; route = CORDUM_ROUTE_OK_PREFERRED; slot = (int)(c_pwork - 1);
              }
            }
            if (!took_pref) need_scan = labelled && !unsat && !settled;   // label-free, single-label and unsatisfiable jobs are final already
            if (!took_pref && !need_scan) {
              if (best != KEY_NONE) {
                route = CORDUM_ROUTE_OK;
                slot = (int)__ldg(T.rank_slot + (uint32_t)(best & 0xFFFFFFFFu));
                if (bcnt > 1) rflags |= CORDUM_F_TIE;
              } else route = total > 0 ? CORDUM_ROUTE_POOL_OVERLOADED : CORDUM_ROUTE_NO_WORKERS;   // :114-119
            }
          }
        }
      }
    }

    // =================================================================== S: label picks, 4 jobs x 8 lanes per step
    for (unsigned todo = __ballot_sync(FULL, need_scan && !slow); todo;) {
      int own[4];   // the (up to) four jobs of this step: group q serves lane own[q]
#pragma unroll
      for (int q = 0; q < 4; ++q) { own[q] = todo ? __ffs(todo) - 1 : -1; todo &= todo - 1; }
      const int src = g == 0 ? own[0] : g == 1 ? own[1] : g == 2 ? own[2] : own[3];
      const bool act = src >= 0;
      const int s_ = act ? src : 0;
      const uint32_t off = __shfl_sync(FULL, r_off, s_), fl = __shfl_sync(FULL, c_flags, s_);
      const uint32_t cnt_all = __shfl_sync(FULL, r_cnt, s_);   // every lane takes part in every shuffle
      const uint32_t cnt = act ? cnt_all : 0u;
      const int single = __shfl_sync(FULL, r_single, s_);
      const uint64_t need_req = shfl64(FULL, c_req, s_) & ~T.req_blank_mask;
      const uint64_t need_lo = shfl64(FULL, c_plo, s_), need_hi = shfl64(FULL, c_phi, s_);
      const bool req_any = fl & JF_REQ_NONEMPTY, req_unknown = fl & JF_REQ_UNKNOWN;
      const uint32_t jw = __shfl_sync(FULL, j, s_);
      const uint64_t* wr = (T.wide_words && P.recs.wide && act) ? P.recs.wide + (size_t)jw * T.wide_words : nullptr;
      // required label bits -> bitmap row numbers, once per job (not per pool and word): four 8-bit row numbers in lbp
      uint32_t lbp = 0, nlb = 0;
      bool more;
      {
        uint64_t rl = need_lo, rh = need_hi;
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          uint32_t bit = 0;
          bool got = false;
          if (rl) { bit = (uint32_t)__ffsll((long long)rl) - 1u; rl &= rl - 1; got = true; }
          else if (rh) { bit = 64u + (uint32_t)__ffsll((long long)rh) - 1u; rh &= rh - 1; got = true; }
          if (got) { nlb = (uint32_t)t + 1u; lbp |= bit << (8 * t); }
        }
        more = (rl | rh) != 0 || place_x_any(T, wr);
      }
      uint64_t b = KEY_NONE;
      uint32_t bc = 0, tot = 0;
      for (uint32_t k = 0; __any_sync(FULL, k < cnt); ++k) {
        const bool kin = k < cnt;
        const uint32_t pid = kin ? (single >= 0 ? (uint32_t)single : __ldg(T.pool_list + off + k)) : 0u;
        const bool elig = kin && (!req_any || (__ldg(T.pool_req_nonempty + pid) && !req_unknown && pool_req_subset(T, pid, need_req, wr)));
        const uint32_t a = __ldg(T.pool_off + pid), e = __ldg(T.pool_off + pid + 1);
        const uint32_t words = elig ? (e - a + 31) >> 5 : 0u, nok = T.pool_nok[pid];
        const uint32_t* bm = T.lbm + __ldg(T.lbm_off + pid);
        uint64_t kstar = KEY_NONE;
        uint32_t kc = 0;
        bool tie_done = false;
        for (uint32_t w0 = 0; __any_sync(FULL, w0 < words && !tie_done); w0 += CORDUM_GROUP) {
          const uint32_t w = w0 + sub;
          uint32_t v = 0;
          if (w < words && !tie_done) {   // matchesLabels (:161-175) for 32 load-sorted workers at once
            // the first four required label bits are independent predicated loads; more than four is rare
            const uint32_t x0 = nlb > 0 ? bm[(lbp & 0xFFu) * words + w] : 0xFFFFFFFFu;
            const uint32_t x1 = nlb > 1 ? bm[((lbp >> 8) & 0xFFu) * words + w] : 0xFFFFFFFFu;
            const uint32_t x2 = nlb > 2 ? bm[((lbp >> 16) & 0xFFu) * words + w] : 0xFFFFFFFFu;
            const uint32_t x3 = nlb > 3 ? bm[(lbp >> 24) * words + w] : 0xFFFFFFFFu;
            v = (x0 & x1) & (x2 & x3);
            if (more) {   // AND is idempotent: walk all required bits again
              for (uint64_t m = need_lo; m; m &= m - 1) v &= bm[(uint32_t)(__ffsll((long long)m) - 1) * words + w];
              for (uint64_t m = need_hi; m; m &= m - 1) v &= bm[(uint32_t)(64 + __ffsll((long long)m) - 1) * words + w];
              if (wr)
                for (uint32_t x = 0; x < T.wide.xw_place; ++x)
                  for (uint64_t m = __ldg(wr + WIDE_O_PLACE(T.wide) + x); m; m &= m - 1)
                    v &= bm[(size_t)(128u + 64u * x + (uint32_t)__ffsll((long long)m) - 1u) * words + w];
            }
          }
          tot += __popc(v);                                     // label-matching candidates, overloaded ones included
          const uint32_t lo = w * 32;
          uint32_t okv = lo >= nok ? 0u : (nok - lo >= 32 ? v : v & ((1u << (nok - lo)) - 1u));   // non-overloaded prefix
          while (true) {   // at most two rounds per group: the argmin, then the next match for the tie flag
            const unsigned hit = __ballot_sync(FULL, okv != 0 && !tie_done);
            if (!hit) break;
            const unsigned gb = (hit >> (g * 8)) & 0xFFu;
            const int L = (int)(g * 8) + (gb ? __ffs(gb) - 1 : 0);
            const uint32_t pos = __shfl_sync(FULL, lo + (uint32_t)(okv ? __ffs(okv) - 1 : 0), L);
            if (gb) {
              const uint64_t kk = T.skey[a + pos];
              if (kstar == KEY_NONE) { kstar = kk; kc = 1; }
              else { if ((uint32_t)(kk >> 32) == (uint32_t)(kstar >> 32)) kc = 2; tie_done = true; }
              if ((int)lane == L) okv &= okv - 1;
            }
          }
        }
        merge_best(b, bc, kstar, kc);
      }
      tot += __shfl_xor_sync(FULL, tot, 1);
      tot += __shfl_xor_sync(FULL, tot, 2);
      tot += __shfl_xor_sync(FULL, tot, 4);
#pragma unroll
      for (int q = 0; q < 4; ++q) {   // hand each job's result to its owner lane
        const uint64_t vb = shfl64(FULL, b, q * 8);
        const uint32_t vc = __shfl_sync(FULL, bc, q * 8), vt = __shfl_sync(FULL, tot, q * 8);
        if ((int)lane == own[q]) { best = vb; bcnt = vc; total = vt; }
      }
    }

    // =================================================================== S': pools beyond the sort buffer, warp per job
    for (unsigned todo = __ballot_sync(FULL, need_scan && slow); todo; todo &= todo - 1) {
      const int i = __ffs(todo) - 1;
      const uint32_t off = __shfl_sync(FULL, r_off, i), cnt = __shfl_sync(FULL, r_cnt, i), fl = __shfl_sync(FULL, c_flags, i);
      const int single = __shfl_sync(FULL, r_single, i);
      const uint64_t need_req = shfl64(FULL, c_req, i) & ~T.req_blank_mask;
      const uint64_t need_lo = shfl64(FULL, c_plo, i), need_hi = shfl64(FULL, c_phi, i);
      const bool req_any = fl & JF_REQ_NONEMPTY, req_unknown = fl & JF_REQ_UNKNOWN;
      const uint32_t jw = __shfl_sync(FULL, j, i);
      const uint64_t* wr = (T.wide_words && P.recs.wide) ? P.recs.wide + (size_t)jw * T.wide_words : nullptr;
      uint64_t b = KEY_NONE;
      uint32_t bc = 0, tot = 0;
      for (uint32_t k = 0; k < cnt; ++k) {
        const uint32_t pid = single >= 0 ? (uint32_t)single : __ldg(T.pool_list + off + k);
        if (req_any && !(__ldg(T.pool_req_nonempty + pid) && !req_unknown && pool_req_subset(T, pid, need_req, wr))) continue;
        const uint32_t a = __ldg(T.pool_off + pid), e = __ldg(T.pool_off + pid + 1);
        for (uint32_t pos = a + lane; pos < e; pos += 32) {   // matchesLabels (:161-175), coalesced
          const uint64_t llo = __ldg(T.pos_label_lo + pos), lhi = __ldg(T.pos_label_hi + pos);
          if ((llo & need_lo) != need_lo || (lhi & need_hi) != need_hi || !place_x_ok(T, pos, wr)) continue;
          tot++;
          merge_best(b, bc, T.pos_key[pos], 1);
        }
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        const uint64_t k2 = shfl64_xor(FULL, b, o);
        const uint32_t c2 = __shfl_xor_sync(FULL, bc, o);
        merge_best(b, bc, k2, c2);
        tot += __shfl_xor_sync(FULL, tot, o);
      }
      if ((int)lane == i) { best = b; bcnt = bc; total = tot; }
    }

    if (need_scan) {
      if (best != KEY_NONE) {
        route = CORDUM_ROUTE_OK;
        slot = (int)__ldg(T.rank_slot + (uint32_t)(best & 0xFFFFFFFFu));
        if (bcnt > 1) rflags |= CORDUM_F_TIE;
      } else route = total > 0 ? CORDUM_ROUTE_POOL_OVERLOADED : CORDUM_ROUTE_NO_WORKERS;
    }
    if (valid) {
      const uint32_t h = (head & 0x00FFFFFFu) | (rflags << 16) | (route << 24);   // rflags only adds CORDUM_F_TIE
      uint32_t* o = reinterpret_cast<uint32_t*>(P.out + c_orig);
      if (ROUTE_ONLY) *reinterpret_cast<uint4*>(o) = make_uint4(h, 0u, 0xFFFFFFFFu, (uint32_t)slot);
      else { o[0] = h; o[3] = (uint32_t)slot; }   // policy_kernel wrote the record; only these two words change
    }
  }
}

// ------------------------------------------------------------------ route: selective placement pairs
// Jobs that name selective pairs (tables.h JF_SELECTIVE, DeviceTables.sel_*) carry JF_PLACE_UNSAT too, so route_kernel has
// settled what the reference decides before its worker scan (:41-66) and left CORDUM_ROUTE_NO_WORKERS for the rest.  Runs
// after route_kernel on the same stream, one warp per job of the batch's selective list:
//   1  the eligible pools again (topic pool list or preferred pool, poolSatisfies)
//   2  the preferred_worker_id shortcut (:73-87)
//   3  the holders of the job's shortest selective list, one per lane; a holder is a candidate when its pool is eligible,
//      its dense mask covers the dense needs and its own selective list holds the job's other selective needs (:161-175)
//   4  candidate count and least-loaded pick over the non-overloaded ones, tie flag as route_kernel (:89-119, SURVEY A.4)
__global__ void __launch_bounds__(256) route_select_kernel(KParams P) {
  const DeviceTables& T = P.t;
  const uint32_t lane = threadIdx.x & 31;
  const uint32_t warps_total = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t item = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; item < P.recs.n_sel_jobs; item += warps_total) {
    const uint2 ent = P.recs.sel_jobs[item];
    const uint4* jr = reinterpret_cast<const uint4*>(P.recs.job + ent.x);
    const uint4 a = __ldg(jr), sv = __ldg(jr + 3);   // {topic, flags, orig, ..}, {lab, sel[0], sel[1]}
    const uint32_t flags = a.y;
    uint32_t* o = reinterpret_cast<uint32_t*>(P.out + a.z);
    const uint32_t h = o[0];   // written by route_kernel, earlier on this stream
    if ((h >> 24) != CORDUM_ROUTE_NO_WORKERS || !(flags & JF_SELECTIVE)) continue;   // settled before the worker scan
    const uint4 r0 = __ldg(reinterpret_cast<const uint4*>(P.recs.route + ent.x)), r1 = __ldg(reinterpret_cast<const uint4*>(P.recs.route + ent.x) + 1);
    const uint64_t need_lo = ((uint64_t)r0.y << 32) | r0.x, need_hi = ((uint64_t)r0.w << 32) | r0.z;
    const uint64_t need_req = (((uint64_t)r1.y << 32) | r1.x) & ~T.req_blank_mask;
    const uint32_t ppool = r1.z, pwork = r1.w;
    const uint64_t* wrow = (T.wide_words && P.recs.wide) ? P.recs.wide + (size_t)ent.x * T.wide_words : nullptr;
    // the job's selective pair ids: sel[0], sel[1], then its extra words
    const uint32_t n_ids = 1u + (sv.w ? 1u : 0u) + (ent.y ? __ldg(P.recs.sel_extra + ent.y) : 0u);
    auto id_at = [&](uint32_t k) -> uint32_t { return k == 0 ? sv.z - 1u : k == 1 ? sv.w - 1u : __ldg(P.recs.sel_extra + ent.y + k - 1); };
    // 1: pools.  A preferred pool passed route_kernel's check, so it is in the topic's list.
    const uint32_t r_off = __ldg(T.topic_pool_off + a.x), r_cnt = __ldg(T.topic_pool_cnt + a.x);
    const bool req_any = flags & JF_REQ_NONEMPTY, req_unknown = flags & JF_REQ_UNKNOWN;
    auto pool_ok = [&](uint32_t pid) -> bool {   // poolSatisfies (:241-265) of a pool the job may use
      bool listed = ppool ? pid == ppool - 1 : false;
      for (uint32_t k = 0; !ppool && !listed && k < r_cnt; ++k) listed = __ldg(T.pool_list + r_off + k) == pid;
      return listed && (!req_any || (__ldg(T.pool_req_nonempty + pid) && !req_unknown && pool_req_subset(T, pid, need_req, wrow)));
    };
    auto carries = [&](uint32_t pos, uint32_t skip) -> bool {   // matchesLabels (:161-175) but for selective need #skip
      if ((__ldg(T.pos_label_lo + pos) & need_lo) != need_lo || (__ldg(T.pos_label_hi + pos) & need_hi) != need_hi || !place_x_ok(T, pos, wrow))
        return false;
      const uint32_t s0 = __ldg(T.pos_sel_off + pos), s1 = __ldg(T.pos_sel_off + pos + 1);
      for (uint32_t k = 0; k < n_ids; ++k) {
        if (k == skip) continue;
        const uint32_t id = id_at(k);
        bool found = false;
        for (uint32_t q = s0; q < s1 && !found; ++q) found = __ldg(T.pos_sel + q) == id;
        if (!found) return false;
      }
      return true;
    };
    uint32_t route = CORDUM_ROUTE_NO_WORKERS, rflags = 0;
    int slot = -1;
    // 2: preferred worker (every lane decides the same)
    bool took_pref = false;
    if (pwork && pwork != CORDUM_PREF_UNKNOWN) {
      const uint32_t p1 = __ldg(T.slot_pos + (pwork - 1));
      if (p1) {
        const uint32_t pos = p1 - 1;
        took_pref = pool_ok(__ldg(T.pos_pool + pos)) && carries(pos, 0xFFFFFFFFu) && !key_over(T.pos_key[pos]);
      }
    }
    if (took_pref) { route = CORDUM_ROUTE_OK_PREFERRED; slot = (int)(pwork - 1); }
    else {
      // 3: the shortest holder list
      uint32_t kmin = 0, len = 0xFFFFFFFFu;
      for (uint32_t k = 0; k < n_ids; ++k) {
        const uint32_t id = id_at(k), l = __ldg(T.sel_off + id + 1) - __ldg(T.sel_off + id);
        if (l < len) { len = l; kmin = k; }
      }
      const uint32_t base = __ldg(T.sel_off + id_at(kmin));
      uint64_t b = KEY_NONE;
      uint32_t bc = 0, tot = 0;
      for (uint32_t i = lane; i < len; i += 32) {
        const uint32_t pos = __ldg(T.sel_pos + base + i);
        if (!pool_ok(__ldg(T.pos_pool + pos)) || !carries(pos, kmin)) continue;
        tot++;                                    // label-matching candidates, overloaded ones included
        merge_best(b, bc, T.pos_key[pos], 1);     // merge_best skips overloaded keys
      }
      // 4: across the warp
#pragma unroll
      for (int off = 16; off; off >>= 1) {
        const uint64_t k2 = shfl64_xor(FULL, b, off);
        const uint32_t c2 = __shfl_xor_sync(FULL, bc, off);
        merge_best(b, bc, k2, c2);
        tot += __shfl_xor_sync(FULL, tot, off);
      }
      if (b != KEY_NONE) {
        route = CORDUM_ROUTE_OK;
        slot = (int)__ldg(T.rank_slot + (uint32_t)(b & 0xFFFFFFFFu));
        if (bc > 1) rflags |= CORDUM_F_TIE;
      } else route = tot > 0 ? CORDUM_ROUTE_POOL_OVERLOADED : CORDUM_ROUTE_NO_WORKERS;   // :114-119
    }
    if (lane == 0) { o[0] = (h & 0x00FFFFFFu) | (rflags << 16) | (route << 24); o[3] = (uint32_t)slot; }
  }
}

// ------------------------------------------------------------------ heartbeat exchange over peer memory
// One process per GPU; every rank owns a full slot-ordered load table (two alternate) that the other ranks have mapped
// (CUDA IPC over NVLink / NVSwitch).  Per epoch a rank copies its own slice from the host into its table, PUSHES the slice
// into every peer's table with plain peer stores (posted writes: no round trip per access), fences, and raises its epoch
// in every peer's flag array; one CTA then waits until every peer's flag shows the epoch.  After the kernel the local
// table is complete and the refresh kernels read it where it lies: no host round trip, no library collective, no copy.
// Reuse of a table (two alternate) is safe without acknowledgements: a rank announces epoch e+1 only after its own
// refresh of epoch e has consumed its table (stream order), and nobody writes into a peer's table of epoch e+2 before
// it has seen that peer's announcement of e+1.
__global__ void __launch_bounds__(256) peer_push_kernel(PeerPush G) {
  const uint32_t tid = threadIdx.x;
  const uint32_t epoch = *G.epoch_ptr;
  __shared__ uint32_t s_last;
  // ---- push: CTA b serves peer (b mod (world-1)), the CTAs of one peer split the slice
  const uint32_t n_peers = G.world - 1, ctas_per_peer = gridDim.x / n_peers;
  if (blockIdx.x < ctas_per_peer * n_peers) {
    const uint32_t pi = blockIdx.x % n_peers, part = blockIdx.x / n_peers;
    const uint32_t q = pi < G.rank ? pi : pi + 1;
    const uint4* src = reinterpret_cast<const uint4*>(G.my_slice);
    uint4* dst = reinterpret_cast<uint4*>(G.peer_slices[q]);
    for (uint32_t i = part * blockDim.x + tid; i < G.per; i += ctas_per_peer * blockDim.x) dst[i] = src[i];
  }
  __threadfence_system();   // this thread's peer stores are visible system-wide before anything below
  __syncthreads();
  if (tid == 0) s_last = atomicAdd(G.done_ctr, 1u) == gridDim.x - 1 ? 1u : 0u;   // the last CTA to finish its part announces
  __syncthreads();
  if (!s_last) return;
  if (tid == 0) *G.done_ctr = 0;   // for the next launch (stream order)
  __threadfence_system();
  if (tid < G.world && tid != G.rank) *reinterpret_cast<volatile uint32_t*>(G.peer_flags[tid] + G.rank) = epoch;
  // ---- wait: every peer's slice of this epoch has landed in my table
  if (tid < G.world && tid != G.rank) {
    const volatile uint32_t* f = G.my_flags + tid;
    while (*f < epoch) __nanosleep(200);
  }
  __threadfence_system();
}

// ------------------------------------------------------------------ launchers (C++ linkage, called by engine.cu)
// An SM changes its L1 / shared-memory split only when it is idle, so kernels that ask for different splits cannot
// share an SM: a refresh CTA (5 KiB of shared memory) would wait for every route / policy CTA (1-2 KiB, i.e. the
// smallest split) on that SM to drain.  All kernels of the path therefore ask for the same carveout, large enough
// for their resident CTAs side by side; the rest (>= 128 KiB) stays L1 for the pass-row gathers.
static cudaError_t configure_kernels() {
  static bool done[64] = {};
  int dev = 0;
  cudaError_t e = cudaGetDevice(&dev);
  if (e != cudaSuccess) return e;
  if (dev >= 0 && dev < 64 && done[dev]) return cudaSuccess;
  static const int kb = []() { const char* v = getenv("CORDUM_SMEM_KB"); return v ? atoi(v) : 72; }();   // tuning knob (policy_kernel: 16 KB of record tiles per CTA)
  const int pct = (kb * 100 + 227) / 228;
  const void* fns[] = {(const void*)worker_chunk_kernel<CORDUM_POOL_CHUNK>, (const void*)worker_merge_kernel, (const void*)peer_push_kernel,
                       (const void*)policy_kernel<3>, (const void*)policy_kernel<4>, (const void*)policy_kernel<5>, (const void*)policy_kernel<6>,
                       (const void*)route_kernel<true>, (const void*)route_kernel<false>,
                       (const void*)route_kernel<false, 3>, (const void*)route_kernel<false, 5>, (const void*)route_select_kernel};
  for (const void* f : fns) {
    e = cudaFuncSetAttribute(f, cudaFuncAttributePreferredSharedMemoryCarveout, pct);
    if (e != cudaSuccess) return e;
  }
  e = cudaFuncSetAttribute(worker_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(CORDUM_POOL_SORT_MAX * 8u));
  if (e != cudaSuccess) return e;
  if (dev >= 0 && dev < 64) done[dev] = true;
  return cudaSuccess;
}

cudaError_t launch_configure() { return configure_kernels(); }   // before a stream capture: attribute calls are not capturable

cudaError_t launch_peer_push(const PeerPush& G, cudaStream_t s) {
  if (G.world < 2) return cudaSuccess;
  const uint32_t n_peers = G.world - 1;
  uint32_t per_peer = (G.per + 2047) / 2048;   // ~8 records per thread
  if (per_peer > 8) per_peer = 8;
  peer_push_kernel<<<n_peers * per_peer, 256, 0, s>>>(G);
  return cudaGetLastError();
}

cudaError_t launch_worker_pools(const DeviceTables& T, cudaStream_t s, cudaEvent_t loads_read) {
  if (T.n_pools == 0) return loads_read ? cudaEventRecord(loads_read, s) : cudaSuccess;
  if (cudaError_t c = configure_kernels(); c != cudaSuccess) return c;
  worker_chunk_kernel<CORDUM_POOL_CHUNK><<<T.n_chunks, CORDUM_POOL_CHUNK, 0, s>>>(T);
  cudaError_t e = cudaGetLastError();
  if (e == cudaSuccess && loads_read) e = cudaEventRecord(loads_read, s);   // the load table is not read past this point
  if (e != cudaSuccess || T.n_merge == 0) return e;
  worker_merge_kernel<<<T.n_merge, 512, T.merge_smem, s>>>(T);
  return cudaGetLastError();
}


static uint32_t grid_for(uint32_t n_jobs, int sm_count, int resident) {
  static const int waves = []() { const char* v = getenv("CORDUM_WAVES"); return v ? atoi(v) : 4; }();
  const uint32_t tiles = (n_jobs + 31u) / 32u;
  uint32_t blocks = (tiles + 7u) / 8u;                                               // 8 warps (tiles) per 256-thread CTA
  const uint32_t cap = (uint32_t)sm_count * (uint32_t)resident * (uint32_t)waves;   // multiple of SM count x resident CTAs
  return blocks > cap ? cap : blocks;
}

// share > 0: the kernel runs next to others inside one graph (a scheduler tick): its persistent grid is capped at `share`
// CTAs per SM so that all branches are resident from the start instead of queueing behind each other's CTAs.
cudaError_t launch_policy(const KParams& P, int sm_count, cudaStream_t s, int share) {
  if (P.n_jobs == 0) return cudaSuccess;
  if (cudaError_t c = configure_kernels(); c != cudaSuccess) return c;
  static const int minb = []() { const char* v = getenv("CORDUM_MINB"); return v ? atoi(v) : 4; }();   // tuning knob
  uint32_t blocks = grid_for(P.n_jobs, sm_count, minb);
  if (share > 0 && blocks > (uint32_t)(sm_count * share)) blocks = (uint32_t)(sm_count * share);
  if (minb <= 3) policy_kernel<3><<<blocks, 256, 0, s>>>(P);
  else if (minb == 4) policy_kernel<4><<<blocks, 256, 0, s>>>(P);
  else if (minb == 5) policy_kernel<5><<<blocks, 256, 0, s>>>(P);
  else policy_kernel<6><<<blocks, 256, 0, s>>>(P);
  return cudaGetLastError();
}

cudaError_t launch_route(const KParams& P, bool route_only, int sm_count, cudaStream_t s, int share) {
  if (P.n_jobs == 0) return cudaSuccess;
  if (cudaError_t c = configure_kernels(); c != cudaSuccess) return c;
  static const int minb = []() { const char* v = getenv("CORDUM_ROUTE_MINB"); return v ? atoi(v) : 4; }();   // tuning knob
  uint32_t blocks = grid_for(P.n_jobs, sm_count, route_only ? 4 : minb);
  if (share > 0 && blocks > (uint32_t)(sm_count * share)) blocks = (uint32_t)(sm_count * share);
  if (route_only) route_kernel<true><<<blocks, 256, 0, s>>>(P);
  else if (minb == 3) route_kernel<false, 3><<<blocks, 256, 0, s>>>(P);
  else if (minb == 5) route_kernel<false, 5><<<blocks, 256, 0, s>>>(P);
  else route_kernel<false><<<blocks, 256, 0, s>>>(P);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess || route_launches(P) == 1) return e;
  uint32_t sel_blocks = (P.recs.n_sel_jobs + 7u) / 8u;   // a warp per job
  const uint32_t cap = (uint32_t)sm_count * 8u;
  if (sel_blocks > cap) sel_blocks = cap;
  if (share > 0 && sel_blocks > (uint32_t)(sm_count * share)) sel_blocks = (uint32_t)(sm_count * share);
  route_select_kernel<<<sel_blocks, 256, 0, s>>>(P);
  return cudaGetLastError();
}
