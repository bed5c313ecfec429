// kernels.h — kernel parameter block and launchers (kernels.cu <-> engine.cu).
#pragma once
#include <cuda_runtime.h>

#include "../../include/cordum_b200.h"
#include "tables.h"

struct KParams {
  JobRecords recs;        // device pointers to the encoded (topic-sorted) records of this batch
  DeviceTables t;         // device pointers to the compiled tables
  cordum_decision* out;   // device, n_jobs records
  uint32_t n_jobs;
  uint32_t* route_count;     // device: number of jobs policy_kernel found dispatchable (null: no compaction)
  uint2* route_list;         // device: {slot in the sorted records, head word policy_kernel wrote} per dispatchable job
  uint32_t honor_approved;   // POLICY_AND_ROUTE: jobs flagged JF_APPROVED bypass the policy (engine.go:484-522)
};

// peer-memory heartbeat exchange (kernels.cu peer_push_kernel)
#define CORDUM_MAX_PEERS 16
struct PeerPush {
  uint32_t rank, world, per;                 // per = worker slots per rank
  const uint32_t* epoch_ptr;                 // device: the epoch this launch announces and waits for (copied in with the slice)
  const Load16* my_slice;                    // local: this rank's slice inside its own table of this epoch's parity
  Load16* peer_slices[CORDUM_MAX_PEERS];     // where this rank's slice goes in every peer's table of that parity
  uint32_t* peer_flags[CORDUM_MAX_PEERS];    // every rank's flag array [CORDUM_MAX_PEERS]: peer_flags[q][r] = last epoch rank r announced to q
  const uint32_t* my_flags;                  // = peer_flags[rank]
  uint32_t* done_ctr;                        // local scratch: CTAs that have finished pushing
};
cudaError_t launch_peer_push(const PeerPush& G, cudaStream_t s);
cudaError_t launch_configure();

// loads_read (optional) is recorded once T.loads has been consumed (between the chunk and the merge kernel)
cudaError_t launch_worker_pools(const DeviceTables& T, cudaStream_t s, cudaEvent_t loads_read);   // chunk sort, merge, label_best
cudaError_t launch_policy(const KParams& P, int sm_count, cudaStream_t s, int share = 0);
// route_kernel, then route_select_kernel when the tables hold selective pairs and the batch lists jobs that name them
cudaError_t launch_route(const KParams& P, bool route_only, int sm_count, cudaStream_t s, int share = 0);
inline uint32_t route_launches(const KParams& P) { return P.n_jobs ? 1u + (P.t.n_sel && P.recs.n_sel_jobs ? 1u : 0u) : 0u; }

// ---- batch dispatch plan (plan.cu): the jobs of a batch grouped by bucket key (include/cordum_b200.h cordum_plan)
#define CORDUM_PLAN_TILE 2048u   // jobs per CTA of the count / scatter kernels
#define CORDUM_PLAN_NONE 0xFFFFFFFFu
// Outcome of a decision record, head = its first word (cordum_decision bytes 0..3), as the plan (plan.cu), the subsets
// (subset.cu) and the topic counts (counts.cu) classify it: the outcome bucket k (CORDUM_PLAN_*, 0..11) of a job that was
// not routed, CORDUM_COUNT_ROUTED for a routed one (its worker slot names the plan's bucket), CORDUM_PLAN_NONE for a
// record that fits no bucket.
__device__ __forceinline__ uint32_t plan_outcome(uint32_t head) {
  const uint32_t sched = (head >> 8) & 0xFFu, status = head >> 24;   // sched_decision, route_status
  if (status == CORDUM_ROUTE_OK || status == CORDUM_ROUTE_OK_PREFERRED) return CORDUM_COUNT_ROUTED;
  if (status == CORDUM_ROUTE_NOT_ATTEMPTED) return sched <= CORDUM_DEC_ALLOW_WITH_CONSTRAINTS ? sched : CORDUM_PLAN_NONE;
  if (status <= CORDUM_ROUTE_POOL_OVERLOADED) return CORDUM_PLAN_MISSING_TOPIC + (status - CORDUM_ROUTE_MISSING_TOPIC);
  return CORDUM_PLAN_NONE;
}
struct PlanPass {                // one 8-bit radix pass
  const uint4* recs;             // pass 0: the decision records (keys are derived from them); later passes: null
  const uint32_t *keys_in, *vals_in;
  uint32_t *keys_out, *vals_out;
  uint32_t* counts;              // [256][n_tiles]
  uint32_t* totals;              // [256]
  uint32_t* bad;                 // raised when a record fits no bucket
  uint32_t n, n_slots, n_tiles, shift;
};
struct PlanParams {
  const cordum_decision* recs;   // device, n records in caller order
  uint32_t n, n_slots, n_buckets;
  uint32_t *keys[2], *vals[2];   // device scratch, n each: the passes alternate between them
  uint32_t *counts, *totals, *bad;
  uint32_t* offsets;             // device, n_buckets + 1
};
uint32_t plan_passes(uint32_t n_buckets);
// The sorted job indices end in vals[(plan_passes(n_buckets) - 1) & 1].
cudaError_t launch_plan(const PlanParams& P, cudaStream_t s);
inline uint32_t plan_launches(const PlanParams& P) { return P.n ? 3u * plan_passes(P.n_buckets) + 1u : 0u; }

// ---- batch subsets (subset.cu): a new encoded batch from a chosen subset of an encoded one (cordum_batch_subset)
#define CORDUM_SUBSET_TILE 2048u   // items (jobs, sorted slots or selective-list entries) per CTA
#define CORDUM_SUBSET_NONE 0xFFFFFFFFu
// Tiles of CORDUM_SUBSET_TILE items, shared by the subset (subset.cu) and merge (merge.cu) kernels: 256 threads x 8 items,
// item = warp * 256 + round * 32 + lane.
namespace tile2k {
constexpr uint32_t kThreads = 256, kWarps = kThreads / 32, kItems = CORDUM_SUBSET_TILE / kThreads;
static_assert(kItems * kThreads == CORDUM_SUBSET_TILE && kItems == 8, "a warp owns 8 rounds of 32 consecutive items");

__device__ __forceinline__ uint32_t item_index(uint32_t tile, uint32_t r) {
  return tile * CORDUM_SUBSET_TILE + (threadIdx.x >> 5) * (32 * kItems) + r * 32 + (threadIdx.x & 31);
}

// Exclusive prefix of v over the tile in item order; *total = the tile's sum.  Every thread of the CTA calls it.
__device__ __forceinline__ void tile_scan(const uint32_t (&v)[kItems], uint32_t (&pre)[kItems], uint32_t* warp_sums, uint32_t* total) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t run = 0;
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) {
    uint32_t x = v[r];
#pragma unroll
    for (uint32_t o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
      if (lane >= o) x += y;
    }
    pre[r] = run + x - v[r];
    run += __shfl_sync(0xFFFFFFFFu, x, 31);
  }
  if (lane == 0) warp_sums[warp] = run;
  __syncthreads();
  uint32_t before = 0, sum = 0;
#pragma unroll
  for (uint32_t w = 0; w < kWarps; ++w) {
    const uint32_t s = warp_sums[w];
    before += w < warp ? s : 0u;
    sum += s;
  }
  __syncthreads();   // warp_sums is reused by the next call
#pragma unroll
  for (uint32_t r = 0; r < kItems; ++r) pre[r] += before;
  *total = sum;
}

// Exclusive prefix of row[0 .. n) in place (one CTA, every thread calls it); returns the sum.
__device__ __forceinline__ uint32_t tiles_scan(uint32_t* row, uint32_t n, uint32_t* warp_sums) {
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  uint32_t carry = 0;
  for (uint32_t t0 = 0; t0 < n; t0 += kThreads) {
    const uint32_t t = t0 + threadIdx.x;
    const uint32_t v = t < n ? row[t] : 0u;
    uint32_t x = v;
#pragma unroll
    for (uint32_t o = 1; o < 32; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, x, o);
      if (lane >= o) x += y;
    }
    if (lane == 31) warp_sums[warp] = x;
    __syncthreads();
    uint32_t before = 0, sum = 0;
#pragma unroll
    for (uint32_t w = 0; w < kWarps; ++w) {
      const uint32_t s = warp_sums[w];
      before += w < warp ? s : 0u;
      sum += s;
    }
    __syncthreads();
    if (t < n) row[t] = carry + before + x - v;
    carry += sum;
  }
  return carry;
}
}  // namespace tile2k
struct SubsetParams {
  // source batch (device)
  uint32_t n;                      // jobs
  const uint4* out;                // selection by outcome: the decision records (caller order); null for a list
  uint32_t mask;                   // outcome buckets selected (bit k = CORDUM_PLAN_* k)
  const uint32_t* list;            // selection by list: ascending job indices; null for an outcome mask
  uint32_t n_list;
  const JobRec* job;
  const RouteRec* route;
  const uint64_t* wide;            // [n][ww] or null
  uint32_t ww;
  const uint2* sel_jobs;           // the selective list (tables.h JobRecords) or null
  const uint32_t* sel_extra;
  uint32_t n_sel;
  uint32_t n_tiles, n_sel_tiles;   // tiles of n jobs / slots, and of n_sel entries
  // scratch (device)
  uint32_t* jloc;                  // [n] per job: rank among the selected jobs of its tile, or NONE
  uint32_t* sloc;                  // [n] per sorted slot: rank among the kept slots of its tile, or NONE
  uint2* eloc;                     // [n_sel] per entry: {rank among the tile's kept entries or NONE, its extra words' offset}
  uint32_t *jcnt, *scnt, *ecnt, *wcnt;   // per tile counts; exclusive prefixes over the tiles after the scan
  uint32_t* totals;                // [4]: selected jobs, kept slots, kept entries, their extra words
  // destination batch (device)
  JobRec* djob;
  RouteRec* droute;
  uint64_t* dwide;                 // [m][ww]
  uint32_t* dsel;                  // [2 m_sel] {slot, x}, then the extra words
  uint32_t m_sel;
  uint32_t* dslot_of;              // [m]
  uint32_t* dparent;               // [m] source job index of each new job
};
// mark -> keep -> scan, then (after the host has read totals and sized the destination) gather
cudaError_t launch_subset_count(const SubsetParams& P, cudaStream_t s);
cudaError_t launch_subset_gather(const SubsetParams& P, cudaStream_t s);
inline uint32_t subset_count_launches(const SubsetParams& P) { return P.n ? 3u : 0u; }
inline uint32_t subset_launches(const SubsetParams& P) { return P.n ? 4u : 0u; }

// ---- batch merges (merge.cu): one encoded batch from two of the same table epoch (cordum_batch_merge)
struct MergeSource {               // a source batch (device)
  const JobRec* job;
  const RouteRec* route;
  const uint64_t* wide;            // [n][MergeParams.ww] or null
  const uint2* sel_jobs;           // the selective list (tables.h JobRecords) or null
  const uint32_t* sel_extra;
  uint32_t n, n_sel;
  uint32_t n_tiles, n_sel_tiles;   // tiles of its n sorted slots and of its n_sel entries
  // scratch (device)
  uint32_t* key;                   // [n] the encoders' sort key of each sorted record
  uint32_t* wloc;                  // [n_sel] per entry: extra words of the tile's entries before it
  uint32_t* wcnt;                  // [n_sel_tiles] per tile: its extra words; exclusive prefix over the tiles after the scan
};
struct MergeParams {
  MergeSource s[2];                // a, b: b's jobs follow a's
  const uint8_t* tenant_class;     // device, per tenant id (EncodeTables.tenant_class)
  uint32_t tenant_classes;
  uint32_t ww;                     // wide-row width of the non-empty sources
  uint32_t* totals;                // [2] extra words of a's and of b's entries
  // destination batch (device)
  JobRec* djob;
  RouteRec* droute;
  uint64_t* dwide;                 // [n_a + n_b][ww]
  uint32_t* dsel;                  // [2 m_sel] {slot, x}, then the extra words
  uint32_t m_sel;                  // = a's n_sel + b's n_sel
  uint32_t* dslot_of;              // [n_a + n_b]
};
// key -> scan -> gather, all on stream s
cudaError_t launch_merge(const MergeParams& P, cudaStream_t s);
inline uint32_t merge_launches(const MergeParams& P) { return P.s[0].n + P.s[1].n ? 3u : 0u; }

// ---- per-topic outcome counts (counts.cu): a dispatched batch's jobs counted per (topic id, outcome column)
#define CORDUM_COUNT_TILE 2048u     // sorted records per CTA of the count kernel
#define CORDUM_COUNT_WINDOW 64u     // topic ids, from the tile's first one on, that a CTA adds up in shared memory
struct CountParams {
  const JobRec* job;                // device: the batch's sorted records (topic, orig)
  const uint4* out;                 // device: its decision records, caller order
  uint32_t n, n_slots, n_topics;    // jobs; slots of the registry it was routed on; topic ids of its dictionary generation
  uint32_t* table;                  // [n_topics][CORDUM_COUNT_COLUMNS]
  uint32_t* head;                   // [2]: non-zero rows, record-check flag (raised when a record fits no bucket)
  uint32_t* rows;                   // [n_topics][1 + CORDUM_COUNT_COLUMNS]: {topic id, counts} of the non-zero rows, any order
};
// zeroes table and head, counts, compacts the non-zero rows (rows[0 .. head[0]))
cudaError_t launch_counts(const CountParams& P, cudaStream_t s);
inline uint32_t counts_launches(const CountParams& P) { return P.n ? 2u : 0u; }

// ---- batch responses (responses.cu): a dispatched batch's jobs grouped by safety response (cordum_batch_responses)
// 64-bit class key, from bit 0 up: arg [w_arg] | rule_idx + 1 [w_rule] | reason_code [5] | flags [4] | sched_decision [3] |
// decision [3].  flags packs APPROVAL_REQUIRED, HAS_SNAPSHOT, CONSTRAINTS into bits 0-2 and APPROVED_BYPASS into bit 3.
#define CORDUM_RESP_FIXED_BITS 15u
struct RespParams {
  const JobRec* job;               // device: the batch's sorted records (topic, orig, mcp)
  const uint4* out;                // device: its decision records, caller order
  uint32_t n, n_tiles;             // jobs; tiles of CORDUM_SUBSET_TILE over them
  uint32_t w_arg, w_rule, passes;  // key field widths; 8-bit radix passes = ceil(key bits / 8)
  // scratch (device)
  unsigned long long* keys[2];     // [n] each: pass p reads keys[p & 1], writes keys[(p + 1) & 1]
  uint32_t* vals[2];               // [n] each: job indices alongside
  uint32_t *counts, *totals;       // [256][n_tiles], [256]
  uint32_t* jflag;                 // [n] job space: 1 = first job of its class, then its rank among the tile's first jobs
  uint32_t* sloc;                  // [n] sorted space: class boundaries before the position within its tile
  uint32_t *hcnt, *jcnt, *ccnt;    // [n_tiles] each: boundaries, first jobs, class sizes per tile; prefixes after the scans
  uint32_t* head;                  // [2]: classes, record-check flag (a field wider than its key width); zeroed by the host
  uint32_t *perm, *start, *size;   // [n] each: sorted-order class -> class; per class: first sorted position, its jobs (then
                                   // its offset inside its tile of classes)
  // output (device)
  cordum_response_class* cls;      // [n] (classes in first_job order)
  uint32_t* offsets;               // [n + 1]
  uint32_t* jobs;                  // [n]
};
// key -> passes x (count, scan, scatter) -> heads -> ranks -> tile scan -> classes -> class scan -> tile scan -> gather
cudaError_t launch_responses(const RespParams& P, cudaStream_t s);
inline uint32_t responses_launches(const RespParams& P) { return P.n ? 8u + 3u * P.passes : 0u; }

// ---- device-side encoder (encode.cu)
struct EncodeParams {
  uint32_t n_jobs;
  EncodeTables et;                 // device pointers (the engine rebases Host::export_dicts' offsets)
  // the envelope arrays of include/cordum_b200.h cordum_envelopes, on the device
  const uint8_t* arena;
  const cordum_str *topic, *tenant, *principal_id, *effective_config, *meta_tenant_id, *actor_id, *capability, *pack_id;
  const uint8_t *has_meta, *actor_type, *approved;
  const uint32_t *risk_off, *requires_off, *label_off;
  const cordum_str *risk_tags, *requires_, *label_keys, *label_vals;
  // work arrays (device)
  uint32_t *tid, *ten, *key, *hist, *slot_of, *fallback;
  JobRec* out_job;
  RouteRec* out_route;
};
cudaError_t launch_encode(const EncodeParams& P, uint32_t n_keys, cudaStream_t s);
