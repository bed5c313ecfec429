// engine.cu — device memory, streams, dispatch and the extern "C" boundary
// (include/cordum_b200.h).  The product has NO CPU evaluation path: every decision
// record is produced by kernels.cu; without a CUDA device engine creation fails.
#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <memory>
#include <tuple>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/cordum_b200.h"
#include "host.hpp"
#include "../../common/nvtx_range.hpp"
#include "kernels.h"

using cordum::Host;
using cordum::HostRecords;
using cordum::HostTables;
using cordum::sv;

namespace {
thread_local std::string g_err;

struct DevBuf {   // a device allocation that grows on demand and is freed with its owner
  void* p = nullptr;
  size_t cap = 0;
  DevBuf() = default;
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t upload(const void* src, size_t bytes, cudaStream_t s) {
    if (bytes > cap) {
      if (p) cudaFree(p);
      p = nullptr;
      size_t want = bytes + bytes / 4 + 256;
      cudaError_t e = cudaMalloc(&p, want);
      if (e != cudaSuccess) { cap = 0; return e; }
      cap = want;
    }
    if (bytes == 0) return cudaSuccess;
    return cudaMemcpyAsync(p, src, bytes, cudaMemcpyHostToDevice, s);
  }
  cudaError_t reserve(size_t bytes) {
    if (bytes <= cap) return cudaSuccess;
    if (p) cudaFree(p);
    p = nullptr;
    cudaError_t e = cudaMalloc(&p, bytes);
    cap = e == cudaSuccess ? bytes : 0;
    return e;
  }
};

// record slab for n jobs: n JobRec (64 B), then n RouteRec (32 B) - one contiguous H2D copy of 96 B per job
inline size_t slab_bytes(uint32_t n) { return (size_t)n * (sizeof(JobRec) + sizeof(RouteRec)); }

}  // namespace

struct cordum_batch;
constexpr int kSets = 3;

struct cordum_engine {
  int device = 0;
  int sm_count = 132;            // H100 SXM; replaced by the device's count at engine creation
  std::unique_ptr<Host> host;
  std::mutex mu;                 // serialises table sync
  bool failed = false;           // sticky CUDA failure
  std::string fail_msg;
  cudaStream_t s_tables = nullptr, s_copy = nullptr, s_xchg = nullptr;
  // engine-owned heartbeat exchange (cordum_exchange_init / cordum_workers_ingest)
  void* nccl_comm = nullptr;
  int xrank = 0, xworld = 1;
  uint64_t xepoch = 0;
  DevBuf gather[2];                              // gathered load tables, alternating per epoch
  cudaEvent_t gather_free[2] = {nullptr, nullptr};   // recorded once the refresh has consumed the table
  cudaEvent_t ev_xchg = nullptr;
  cudaEvent_t ev_copy = nullptr, ev_prod = nullptr;
  DeviceTables dt{};             // device pointers + scalars, as passed to kernels
  // device copies, one DevBuf per host vector
  DevBuf b_rows, b_row_check;   // all pass-row tables, word-major, in one array (tables.h)
  DevBuf b_req_need, b_lab_need, b_rule_dec, b_tenant_mcp, b_eff_mcp, b_eff_topic, b_pos2rule;
  DevBuf b_sum_tenant, b_sum_topic, b_sum_cap, b_sum_pack, b_sum_actor, b_sum_combo, b_sum_risk;
  DevBuf b_topic_pool_off, b_topic_pool_cnt, b_pool_list, b_pool_req_mask, b_pool_req_nonempty;
  DevBuf b_rule_need_x, b_pool_req_x, b_req_blank_x, b_pos_label_x;   // wide masks (tables.h WideLayout)
  DevBuf b_pool_off, b_pos_pool, b_pos_slot, b_pos_rank, b_slot_pos, b_rank_slot, b_pos_label_lo, b_pos_label_hi;
  DevBuf b_flush, b_lbm_off, b_rank_pos, b_chunk_pool, b_pool_chunk0, b_merge_list;
  DevBuf b_sel_off, b_sel_pos, b_pos_sel_off, b_pos_sel;   // selective placement pairs (tables.h DeviceTables.sel_*)
  DevBuf b_dicts;                // device encoder: dictionary images + side arrays (Host::export_dicts)
  EncodeTables et{};             // rebased onto b_dicts
  uint64_t v_dict = ~0ull;
  std::vector<cordum_envelopes*> env_sets;   // pinned envelope staging sets handed out by cordum_envelopes_alloc
  uint64_t tables_gen = 0;       // bumps whenever a device table pointer or scalar may have changed (captured graphs bake them in)
  // Pinned staging of this rank's heartbeat slice (+ the epoch word behind it), one per gather-buffer parity.  The ingest
  // graphs and the ticks share it: leave_tick_mode drains the tick streams before any ingest, and cordum_tick_async
  // synchronises the device when it enters tick mode, so the two never have a copy out of it in flight at once.
  Load16* stage[2] = {nullptr, nullptr};
  size_t stage_cap = 0;
  // ---- cordum_workers_ingest as one graph launch (world = 1, or the peer exchange): H2D -> [peer gather] -> chunk -> merge
  std::map<std::tuple<int, int, uint64_t>, cudaGraphExec_t> ing_graphs;   // (target set, buffer parity, tables generation)
  // ---- scheduler ticks (cordum_tick_async): one CUDA graph launch per tick
  struct Tick {
    cudaStream_t s[2] = {nullptr, nullptr};                // tick k is launched on s[k & 1]: consecutive ticks overlap
    cudaStream_t sa = nullptr, sc = nullptr;               // fork streams used only while capturing
    cudaEvent_t ev_fork = nullptr, ev_a = nullptr, ev_c = nullptr;   // capture-internal fork / join
    cudaEvent_t done[2] = {nullptr, nullptr};              // recorded behind tick k on s[k & 1]: staging reuse (host), and the
                                                           // route branch of tick k+1 waits for it inside its graph
    cudaEvent_t refreshed[2] = {nullptr, nullptr};         // recorded inside graph k at the end of its heartbeat branch: the
                                                           // heartbeat branch of tick k+1 starts behind it (the epochs stay ordered)
    cudaEvent_t ev_join = nullptr;
    cordum_batch* prev = nullptr;                          // its policy ran in the previous tick; its route is due
    uint64_t n = 0;                                        // ticks so far
    bool active = false;                                   // ticks have been issued since the last plain dispatch / ingest
    std::map<std::tuple<cordum_batch*, cordum_batch*, int, uint32_t, uint32_t, uint32_t, uint64_t>, cudaGraphExec_t> graphs;
  } tick;
  // ---- peer-memory heartbeat exchange (cordum_peer_export / cordum_peer_import)
  struct Peers {
    int rank = 0, world = 1;
    uint32_t per = 0;                                      // worker slots per rank
    uint8_t* mine = nullptr;                               // [flags 128 B | push counter | epoch words][full table parity 0][full table parity 1]
    size_t bytes = 0;
    uint8_t* base[CORDUM_MAX_PEERS] = {};                  // every rank's buffer as mapped here (mine included)
    bool ready = false;
  } peers;
  // Everything the worker-table refresh kernels derive from the loads, in kSets copies used round-robin: the refresh
  // for heartbeat epoch k+1 (and k+2) writes one set while route kernels of epoch k still read another, so consecutive
  // steps pipeline instead of serialising (with two sets the refresh of epoch k+2 would wait for epoch k's route kernel).
  struct DerivedSet {
    DevBuf loads, pos_key, ckey, skey, pool_sorted, pool_nok, pool_done, lbm, lbest, pool_best, pool_mincnt;
    cudaEvent_t ready = nullptr, loads_read = nullptr;   // refresh complete / load table consumed by the refresh
  } ds[kSets];
  int cur = 0;                   // set holding the latest refresh
  uint64_t v_policy = ~0ull, v_topic = ~0ull, v_mcp = ~0ull, v_routing = ~0ull, v_workers = ~0ull, v_loads = ~0ull;
  std::vector<cordum_batch*> batches;   // live batches (guarded by mu): K2 must wait for their kernels
  bool pools_dirty = true;       // K2 must run before the next dispatch
  std::atomic<uint64_t> launches{0};
};

struct cordum_batch {
  cordum_engine* e = nullptr;
  uint32_t max_jobs = 0, n = 0;
  uint64_t epoch = 0;
  // what the records of the last dispatch index (read under the same lock as the epoch check): rule text + snapshot of
  // the policy, worker ids of the registry.  Kept by the batch so that a later reload cannot relabel its decisions.
  std::shared_ptr<const cordum::PolicyText> text;
  std::shared_ptr<const std::vector<std::string>> wtext;
  std::shared_ptr<const std::vector<std::string>> ttext;   // raw topics by id of the dictionary generation the batch was encoded under
  bool encoded = false, resident = false, pending = false, enc_inflight = false, launched = false, timed_in = false, timed_out = false;
  int table_set = 0;             // derived-table set the last route_kernel of this batch read
  uint8_t* h_cols = nullptr;     // pinned: the encoded records (slab_bytes layout)
  uint8_t* d_cols = nullptr;
  uint64_t *h_wide = nullptr, *d_wide = nullptr;   // wide-mask rows (tables.h WideLayout), allocated on first need
  uint64_t wide_cap = 0;         // 64-bit words allocated at each of the two
  uint32_t wide_words = 0;       // row width of the encoded batch
  uint32_t *h_sel = nullptr, *d_sel = nullptr;   // the selective list (tables.h JobRecords), allocated on first need
  size_t sel_cap = 0;            // 32-bit words allocated at each of the two
  uint32_t n_sel_jobs = 0, sel_words = 0;   // of the encoded batch: listed jobs, words in use
  uint32_t* slot_of = nullptr;   // host: position of caller job j in the sorted records
  // device-side encode (cordum_encode_device)
  bool device_encoded = false, host_records_valid = true;
  const cordum_envelopes* env = nullptr;   // the caller's envelopes, kept until the batch has been waited for (host fallback)
  DevBuf d_env, d_work;          // envelope arrays on the device; tid / ten / key / slot_of / hist / flag
  uint32_t* h_fallback = nullptr;   // pinned: 1 = the device encoder left something to the host
  const uint32_t* d_slot_of = nullptr;   // device slot_of of records produced on the device (encoder work array or d_sub_idx)
  // cordum_batch_subset, when this batch is the destination
  bool is_subset = false;        // the records are a subset of another batch's: h_parent is valid
  DevBuf d_sub_idx;              // [max_jobs] slot_of, then [max_jobs] parent index (allocated on first use; a merge uses the first half)
  DevBuf d_subset;               // scratch of the call (subset_batch, merge_batch), grown on first need
  uint32_t* h_parent = nullptr;  // pinned [max_jobs]: source job index of each job
  uint32_t last_mode = 0;
  bool last_copy_out = false, timed = true;
  bool tick_pending = false;     // dispatched through cordum_tick_async: results are on the device once the tick streams have drained
  uint64_t tick_no = 0;          // the tick it was handed in with (its route runs in tick_no + 1)
  cordum_decision* h_out = nullptr;   // pinned
  cordum_decision* d_out = nullptr;
  bool results_ready = false;    // d_out holds the complete records of the last dispatch (cordum_batch_plan reads them)
  DevBuf d_plan;                 // cordum_batch_plan scratch (plan_batch), grown on first need
  uint32_t* h_plan = nullptr;    // pinned: the plan's offsets, the record-check flag, then its jobs
  size_t h_plan_cap = 0;         // 32-bit words
  DevBuf d_counts;               // cordum_batch_topic_counts scratch (count_batch), grown on first need
  uint32_t* h_counts = nullptr;  // pinned: the copied topic rows, then the output (counts | label offsets | label bytes)
  size_t h_counts_cap = 0;       // 32-bit words
  DevBuf d_resp;                 // cordum_batch_responses scratch (responses_batch), grown on first need
  uint32_t* h_resp = nullptr;    // pinned: the class count, classes, offsets, jobs, then the two text offset arrays
  size_t h_resp_cap = 0;         // 32-bit words
  uint8_t* h_resp_text = nullptr;   // pinned: the reasons' and rule ids' bytes
  size_t h_resp_text_cap = 0;
  uint2* d_route = nullptr;           // [0].x = count, [2..] = compacted list of dispatchable jobs {slot, head}
  cudaStream_t stream = nullptr;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr, evm = nullptr, ev2 = nullptr, ev3 = nullptr;
  float total_ms = 0, kernel_ms = 0, policy_ms = 0, route_ms = 0;
  HostRecords hr{};
};

namespace {

int fail(cordum_engine* e, cudaError_t err, const char* what) {
  g_err = std::string(what) + ": " + cudaGetErrorString(err);
  if (e) { e->failed = true; e->fail_msg = g_err; }
  return CORDUM_E_CUDA;
}
#define CK(call, what) do { cudaError_t _e = (call); if (_e != cudaSuccess) return fail(e, _e, what); } while (0)

void host_records(cordum_batch* b) {
  b->hr.job = (JobRec*)b->h_cols;
  b->hr.route = (RouteRec*)(b->h_cols + (size_t)b->n * sizeof(JobRec));
  b->hr.slot_of = b->slot_of;
  b->hr.wide = b->h_wide;
  b->hr.wide_cap = b->wide_cap;
}
void device_records(const cordum_batch* b, JobRecords& r) {
  r.job = (const JobRec*)b->d_cols;
  r.route = (const RouteRec*)(b->d_cols + (size_t)b->n * sizeof(JobRec));
  r.wide = b->wide_words ? b->d_wide : nullptr;
  r.n_sel_jobs = b->n_sel_jobs;
  r.sel_jobs = b->n_sel_jobs ? reinterpret_cast<const uint2*>(b->d_sel) : nullptr;
  r.sel_extra = b->n_sel_jobs ? b->d_sel + 2 * (size_t)b->n_sel_jobs : nullptr;
}

// Uploads a host table into b and points the kernels' view (field) at it.
template <class T, class P>
cudaError_t put(DevBuf& b, const std::vector<T>& v, const P*& field, cudaStream_t s) {
  cudaError_t err = b.upload(v.data(), v.size() * sizeof(T), s);
  field = (const P*)b.p;
  return err;
}

// Bring the device tables up to date with the host tables.  Called with host mutex held.
int sync_tables(cordum_engine* e) {
  cordum::NvtxRange nvtx_("cordum:table_upload");
  const HostTables& t = e->host->tables();
  DeviceTables& d = e->dt;
  bool any = t.v_policy != e->v_policy || t.v_topic != e->v_topic || t.v_mcp != e->v_mcp || t.v_routing != e->v_routing ||
             t.v_workers != e->v_workers || (t.v_loads != e->v_loads);
  if (!any) return CORDUM_OK;
  // Tables may be reallocated: nothing may be in flight.  Table changes are rare (policy/routing
  // reload, first sight of a topic) so a full device sync here is acceptable.
  CK(cudaDeviceSynchronize(), "sync before table upload");
  cudaStream_t s = e->s_tables;
  if (t.v_policy != e->v_policy || t.v_topic != e->v_topic || t.v_mcp != e->v_mcp) {
    // the unified word-major pass-row array (rebuilt whole: a few MB, and only on a reload or a first-seen topic)
    const cordum::RowTable* tabs[11] = {&t.row_topic, &t.row_tenant, &t.row_cap, &t.row_pack, &t.row_actor, &t.row_combo, &t.row_risk,
                                       &t.row_mcp[0], &t.row_mcp[1], &t.row_mcp[2], &t.row_mcp[3]};
    uint32_t off[11], cells = 0;
    for (int k = 0; k < 11; ++k) { off[k] = cells; cells += tabs[k]->n_rows; }
    const size_t w4 = t.row_words / 4;
    std::vector<uint32_t> wm((size_t)cells * t.row_words, 0);
    for (int k = 0; k < 11; ++k)
      for (size_t v = 0; v < tabs[k]->n_rows; ++v) {
        const uint32_t* row = tabs[k]->row((uint32_t)v);
        for (size_t w = 0; w < w4; ++w) std::memcpy(&wm[(w * cells + off[k] + v) * 4], row + 4 * w, 16);
      }
    CK(put(e->b_rows, wm, d.rows, s), "upload");
    CK(cudaStreamSynchronize(s), "upload");   // wm is a local
    d.n_cells = cells;
    d.off_topic = off[0]; d.off_tenant = off[1]; d.off_cap = off[2]; d.off_pack = off[3]; d.off_actor = off[4];
    d.off_combo = off[5]; d.off_risk = off[6];
    for (int f = 0; f < 4; ++f) d.off_mcp[f] = off[7 + f];
    d.n_topic = t.row_topic.n_rows;
  }
  if (t.v_policy != e->v_policy) {
    CK(put(e->b_row_check, t.row_check.data, d.chk_words, s), "upload");
    CK(put(e->b_sum_tenant, t.sum_tenant, d.sum_tenant, s), "upload"); CK(put(e->b_sum_cap, t.sum_cap, d.sum_cap, s), "upload");
    CK(put(e->b_sum_pack, t.sum_pack, d.sum_pack, s), "upload"); CK(put(e->b_sum_actor, t.sum_actor, d.sum_actor, s), "upload");
    CK(put(e->b_sum_combo, t.sum_combo, d.sum_combo, s), "upload"); CK(put(e->b_sum_risk, t.sum_risk, d.sum_risk, s), "upload");
    CK(put(e->b_req_need, t.rule_req_need, d.rule_req_need, s), "upload");
    CK(put(e->b_lab_need, t.rule_lab_need, d.rule_lab_need, s), "upload");
    CK(put(e->b_rule_dec, t.rule_dec, d.rule_dec, s), "upload"); CK(put(e->b_pos2rule, t.pos2rule, d.pos2rule, s), "upload");
    d.n_rules = t.n_rules; d.n_seg = t.n_seg; d.row_u4 = t.n_seg * CORDUM_SEG_U4; d.sum_group = t.sum_group;
    CK(put(e->b_rule_need_x, t.rule_need_x, d.rule_need_x, s), "upload");
    e->v_policy = t.v_policy;
  }
  if (t.v_topic != e->v_topic) {
    CK(put(e->b_sum_topic, t.sum_topic, d.sum_topic, s), "upload");
    CK(put(e->b_eff_topic, t.eff_topic, d.eff_topic, s), "upload");
    CK(put(e->b_topic_pool_off, t.topic_pool_off, d.topic_pool_off, s), "upload");
    CK(put(e->b_topic_pool_cnt, t.topic_pool_cnt, d.topic_pool_cnt, s), "upload");
    CK(put(e->b_pool_list, t.pool_list, d.pool_list, s), "upload");
    d.sum_use = t.sum_use;   // chosen against the topic rows (Host::choose_summaries)
    d.topic_stride = t.topic_stride;
    e->v_topic = t.v_topic;
  }
  if (t.v_mcp != e->v_mcp) {
    CK(put(e->b_tenant_mcp, t.tenant_mcp, d.tenant_mcp, s), "upload"); CK(put(e->b_eff_mcp, t.eff_mcp, d.eff_mcp, s), "upload");
    d.mcp_stride = t.mcp_stride;
    e->v_mcp = t.v_mcp;
  }
  if (t.v_routing != e->v_routing) {
    CK(put(e->b_pool_req_mask, t.pool_req_mask, d.pool_req_mask, s), "upload");
    CK(put(e->b_pool_req_nonempty, t.pool_req_nonempty, d.pool_req_nonempty, s), "upload");
    d.req_blank_mask = t.req_blank_mask; d.n_pools = t.n_pools;
    CK(put(e->b_pool_req_x, t.pool_req_x, d.pool_req_x, s), "upload"); CK(put(e->b_req_blank_x, t.req_blank_x, d.req_blank_x, s), "upload");
    e->v_routing = t.v_routing;
  }
  if (t.v_workers != e->v_workers) {
    CK(put(e->b_pool_off, t.pool_off, d.pool_off, s), "upload"); CK(put(e->b_pos_pool, t.pos_pool, d.pos_pool, s), "upload");
    CK(put(e->b_pos_slot, t.pos_slot, d.pos_slot, s), "upload"); CK(put(e->b_pos_rank, t.pos_rank, d.pos_rank, s), "upload");
    CK(put(e->b_slot_pos, t.slot_pos, d.slot_pos, s), "upload"); CK(put(e->b_rank_slot, t.rank_slot, d.rank_slot, s), "upload");
    CK(put(e->b_rank_pos, t.rank_pos, d.rank_pos, s), "upload");
    CK(put(e->b_pos_label_lo, t.pos_label_lo, d.pos_label_lo, s), "upload");
    CK(put(e->b_pos_label_hi, t.pos_label_hi, d.pos_label_hi, s), "upload");
    // the derived tables of every set, sized for the new registry
    const size_t pos = std::max<uint32_t>(t.n_pos, 1), pools = std::max<uint32_t>(t.n_pools, 1);
    const size_t lbest = t.place_bits <= CORDUM_LBEST_MAX_BITS ? pools * t.place_bits * 16 : 0;   // 0: not built
    for (auto& D : e->ds) {
      const std::pair<DevBuf*, size_t> sizes[] = {
          {&D.pos_key, pos * 8}, {&D.pool_best, pools * 8}, {&D.pool_mincnt, pools * 4}, {&D.skey, pos * 8}, {&D.ckey, pos * 8},
          {&D.pool_sorted, pools}, {&D.pool_nok, pools * 4}, {&D.pool_done, pools * 4},
          {&D.lbm, (size_t)std::max<uint64_t>(t.lbm_words, 1) * 4}, {&D.lbest, lbest},
          {&D.loads, (size_t)std::max<uint32_t>(t.n_slots, 1) * sizeof(Load16)}};
      for (const auto& [buf, bytes] : sizes) CK(buf->reserve(bytes), "alloc");
    }
    CK(put(e->b_chunk_pool, t.chunk_pool, d.chunk_pool, s), "upload"); CK(put(e->b_pool_chunk0, t.pool_chunk0, d.pool_chunk0, s), "upload");
    CK(put(e->b_merge_list, t.merge_list, d.merge_list, s), "upload");
    d.n_chunks = t.n_chunks; d.n_merge = t.n_merge; d.merge_smem = t.merge_smem;
    CK(put(e->b_lbm_off, t.lbm_off, d.lbm_off, s), "upload");
    d.place_bits = t.place_bits;
    d.n_pos = t.n_pos; d.n_pools = t.n_pools;
    CK(put(e->b_pos_label_x, t.pos_label_x, d.pos_label_x, s), "upload");
    CK(put(e->b_sel_off, t.sel_off, d.sel_off, s), "upload"); CK(put(e->b_sel_pos, t.sel_pos, d.sel_pos, s), "upload");
    CK(put(e->b_pos_sel_off, t.pos_sel_off, d.pos_sel_off, s), "upload"); CK(put(e->b_pos_sel, t.pos_sel, d.pos_sel, s), "upload");
    d.n_sel = t.n_sel;
    e->v_workers = t.v_workers;
    e->pools_dirty = true;
  }
  if (t.v_loads != e->v_loads) {   // heartbeat deltas applied on the host (cordum_workers_update)
    e->v_loads = t.v_loads;
    e->pools_dirty = true;
  }
  d.wide = t.wide;
  d.wide_words = WIDE_WORDS(t.wide);
  CK(cudaStreamSynchronize(s), "table upload");
  e->tables_gen++;
  return CORDUM_OK;
}

// Device encoder: the dictionaries follow the host's (called with the host mutex held, nothing in flight on the blob:
// callers go through sync_tables first, and a dictionary change always comes with a table change or a reload).
int sync_dicts(cordum_engine* e) {
  if (e->v_dict == e->host->dict_version()) return CORDUM_OK;
  CK(cudaDeviceSynchronize(), "sync before dictionary upload");
  std::vector<uint8_t> blob;
  EncodeTables et;
  e->host->export_dicts(blob, et);
  CK(e->b_dicts.upload(blob.data(), blob.size(), e->s_tables), "upload dictionaries");
  CK(cudaStreamSynchronize(e->s_tables), "upload dictionaries");
  const uint8_t* base = (const uint8_t*)e->b_dicts.p;
  et.blob = base;
  et.topic_flags = (const uint32_t*)(base + (size_t)et.topic_flags);
  et.tenant_class = base + (size_t)et.tenant_class;
  et.label_keymask = (const uint64_t*)(base + (size_t)et.label_keymask);
  e->et = et;
  e->v_dict = e->host->dict_version();
  return CORDUM_OK;
}

// Parameters of the peer push for table parity p; returns this rank's full table of that parity (inside its IPC buffer).
uint8_t* peer_push_params(const cordum_engine* e, int p, PeerPush& G) {
  const auto& P = e->peers;
  const size_t tbytes = (size_t)P.per * (size_t)P.world * sizeof(Load16), soff = (size_t)P.rank * P.per * sizeof(Load16);
  G.rank = (uint32_t)P.rank; G.world = (uint32_t)P.world; G.per = P.per;
  for (int q = 0; q < P.world; ++q) {
    G.peer_slices[q] = (Load16*)(P.base[q] + 256 + (size_t)p * tbytes + soff);
    G.peer_flags[q] = (uint32_t*)P.base[q];
  }
  G.my_flags = (const uint32_t*)P.mine;
  G.done_ctr = (uint32_t*)(P.mine + 128);
  G.epoch_ptr = (const uint32_t*)(P.mine + 160 + (size_t)p * 16);
  uint8_t* table = P.mine + 256 + (size_t)p * tbytes;
  G.my_slice = (const Load16*)(table + soff);
  return table;
}

// Ticks keep their own order on their own stream; a plain dispatch / ingest after ticks first lets that stream drain.
int tick_flush_locked(cordum_engine* e);
int leave_tick_mode(cordum_engine* e) {
  if (!e->tick.active) return CORDUM_OK;
  std::lock_guard<std::mutex> g(e->mu);
  int rc = tick_flush_locked(e);
  if (rc) return rc;
  for (cudaStream_t st : e->tick.s) CK(cudaStreamSynchronize(st), "drain tick stream");
  e->tick.active = false;
  return CORDUM_OK;
}

// The kernels' view of the tables with the derived pointers of one set.
DeviceTables view(const cordum_engine* e, int set) {
  DeviceTables d = e->dt;
  const auto& D = e->ds[set];
  d.loads = (const Load16*)D.loads.p;
  d.pos_key = (uint64_t*)D.pos_key.p; d.ckey = (uint64_t*)D.ckey.p; d.skey = (uint64_t*)D.skey.p;
  d.pool_sorted = (uint8_t*)D.pool_sorted.p; d.pool_nok = (uint32_t*)D.pool_nok.p; d.pool_done = (uint32_t*)D.pool_done.p; d.lbm = (uint32_t*)D.lbm.p;
  // The per-(pool, label) answers take work out of route_kernel but lengthen the refresh chain.  With one or two ranks
  // the chain hides behind policy_kernel; from four ranks on the per-rank batch is small and the chain is the critical
  // path of a step, so the table is built only when it pays.  CORDUM_LBEST=1 / 0 forces it on / off (both paths are
  // exact and parity-tested).
  const char* lb = getenv("CORDUM_LBEST");
  const bool use_lbest = lb ? lb[0] == '1' : e->xworld <= 2;
  d.lbest = (d.place_bits <= CORDUM_LBEST_MAX_BITS && use_lbest) ? (uint4*)D.lbest.p : nullptr;
  d.pool_best = (uint64_t*)D.pool_best.p; d.pool_mincnt = (uint32_t*)D.pool_mincnt.p;
  return d;
}

// Kernels one refresh of the derived worker tables launches (worker_chunk, worker_merge).
uint32_t refresh_launches(const cordum_engine* e) { return (e->dt.n_chunks ? 1 : 0) + (e->dt.n_merge ? 1 : 0); }

// The set the next heartbeat epoch is refreshed into: the one after the latest, once the route kernels that still read it
// (launched kSets-1 epochs ago) have finished.  Returns the set, or an error code (< 0).
int claim_set(cordum_engine* e) {
  const int target = (e->cur + 1) % kSets;
  for (cordum_batch* b : e->batches)
    if (b->launched && b->table_set == target) { CK(cudaStreamWaitEvent(e->s_tables, b->ev2, 0), "wait route"); b->launched = false; }
  return target;
}

// The refresh of set `target` has been enqueued on the tables stream (`launches` kernels): dispatches route on it from here on.
int publish_set(cordum_engine* e, int target, uint32_t launches) {
  CK(cudaEventRecord(e->ds[target].ready, e->s_tables), "event record");
  e->launches += launches;
  e->cur = target;
  e->pools_dirty = false;
  return CORDUM_OK;
}

// Refresh kernels of a heartbeat epoch on the tables stream, into set `target`.  loads: the full slot-ordered load table
// they read (null: the set's own copy); loads_read (optional) is recorded once they have consumed it.
int refresh_on_tables_stream(cordum_engine* e, int target, const Load16* loads, cudaEvent_t loads_read) {
  DeviceTables tv = view(e, target);
  if (loads) tv.loads = loads;
  CK(launch_worker_pools(tv, e->s_tables, loads_read), "worker-table refresh kernels");
  return publish_set(e, target, refresh_launches(e));
}

// One heartbeat epoch as captured into a graph on stream s: the staged slice of parity p to the device - into this rank's
// slice of the peer table of that parity, then pushed to every peer, when the peers exchange it - then the refresh
// kernels of `set` on the full table.
cudaError_t enqueue_heartbeat(cordum_engine* e, cudaStream_t s, int p, int set, bool peers) {
  uint8_t* table = (uint8_t*)e->gather[p].p;
  DeviceTables tv = view(e, set);
  cudaError_t ce = cudaSuccess;
  if (peers) {
    // the staging buffer carries the epoch number behind the slice; the push kernel - whose parameters the graph bakes
    // in - reads the epoch it announces and waits for from device memory
    const size_t slice_bytes = (size_t)e->peers.per * sizeof(Load16);
    PeerPush G{};
    table = peer_push_params(e, p, G);
    ce = cudaMemcpyAsync((void*)G.my_slice, e->stage[p], slice_bytes, cudaMemcpyHostToDevice, s);
    if (ce == cudaSuccess) ce = cudaMemcpyAsync((void*)G.epoch_ptr, (const uint8_t*)e->stage[p] + slice_bytes, 4, cudaMemcpyHostToDevice, s);
    if (ce == cudaSuccess) ce = launch_peer_push(G, s);
  } else {
    ce = cudaMemcpyAsync(table, e->stage[p], (size_t)e->host->tables().n_slots * sizeof(Load16), cudaMemcpyHostToDevice, s);
  }
  tv.loads = (const Load16*)table;
  return ce != cudaSuccess ? ce : launch_worker_pools(tv, s, nullptr);
}

// The pinned heartbeat staging, large enough for a slice of `bytes`.  Both graph caches bake its pointers in.
int grow_staging(cordum_engine* e, size_t bytes) {
  if (e->stage[0] && e->stage_cap >= bytes) return CORDUM_OK;
  CK(cudaDeviceSynchronize(), "sync before staging growth");
  for (auto& p : e->stage) { if (p) cudaFreeHost(p); p = nullptr; }
  for (auto& p : e->stage) CK(cudaHostAlloc((void**)&p, bytes + 64, cudaHostAllocDefault), "pinned heartbeat staging");
  e->stage_cap = bytes;
  for (auto& kv : e->ing_graphs) cudaGraphExecDestroy(kv.second);
  e->ing_graphs.clear();
  for (auto& kv : e->tick.graphs) cudaGraphExecDestroy(kv.second);
  e->tick.graphs.clear();
  return CORDUM_OK;
}

// The gathered load tables of both parities, large enough for `bytes`: nothing may still read the old buffers, and the
// captured graphs that bake their pointers in are stale.
int grow_gather(cordum_engine* e, size_t bytes) {
  if (e->gather[0].cap >= bytes && e->gather[1].cap >= bytes) return CORDUM_OK;
  CK(cudaDeviceSynchronize(), "sync before gather buffer allocation");
  for (auto& b : e->gather) CK(b.reserve(bytes), "alloc gather buffer");
  e->tables_gen++;
  return CORDUM_OK;
}

// What policy_kernel and route_kernel of batch b read and write, on tables t.  policy_and_route (CORDUM_MODE_POLICY_AND_ROUTE):
// approvals are honoured, and policy_kernel compacts the dispatchable jobs into the batch's route list for route_kernel.
KParams batch_params(const cordum_batch* b, const DeviceTables& t, bool policy_and_route) {
  KParams P{};
  P.t = t;
  device_records(b, P.recs);
  P.out = b->d_out;
  P.n_jobs = b->n;
  P.honor_approved = policy_and_route ? 1u : 0u;
  if (policy_and_route) { P.route_count = reinterpret_cast<uint32_t*>(b->d_route); P.route_list = b->d_route + 2; }
  return P;
}

// worker-table refresh kernels for a new heartbeat epoch, into the set that is NOT being read.  dev_loads: the full slot-ordered
// load table already in HBM (produced on `producer`), or null to take the host tables' loads.  Called with both mutexes held.
int refresh_pools(cordum_engine* e, const void* dev_loads, cudaStream_t producer) {
  cordum::NvtxRange nvtx_("cordum:worker_refresh");
  if (!e->pools_dirty && !dev_loads) return CORDUM_OK;
  const int target = claim_set(e);
  if (target < 0) return target;
  auto& D = e->ds[target];
  const HostTables& t = e->host->tables();
  const size_t bytes = (size_t)t.n_slots * sizeof(Load16);
  if (dev_loads) {
    // The gathered table is copied on its own stream, ordered after the producer (e.g. the NCCL all-gather stream) and
    // after the last refresh that read this set's copy - NOT after the refresh in flight on the tables stream - so the
    // refresh kernels of epoch k+1 sit directly behind those of epoch k and start ahead of epoch k's route kernel.
    CK(cudaEventRecord(e->ev_prod, producer), "event record");
    CK(cudaStreamWaitEvent(e->s_copy, e->ev_prod, 0), "wait producer");
    CK(cudaStreamWaitEvent(e->s_copy, D.loads_read, 0), "wait previous readers");
    if (bytes) CK(cudaMemcpyAsync(D.loads.p, dev_loads, bytes, cudaMemcpyDeviceToDevice, e->s_copy), "D2D loads");
    // later work on the producer stream (e.g. the next all-gather into the same buffer) must not overtake the copy
    CK(cudaEventRecord(e->ev_copy, e->s_copy), "event record");
    CK(cudaStreamWaitEvent(producer, e->ev_copy, 0), "order producer after copy");
    CK(cudaStreamWaitEvent(e->s_tables, e->ev_copy, 0), "order refresh after copy");
  } else if (bytes) {
    CK(cudaMemcpyAsync(D.loads.p, t.loads.data(), bytes, cudaMemcpyHostToDevice, e->s_tables), "H2D loads");
  }
  return refresh_on_tables_stream(e, target, nullptr, D.loads_read);
}

int run(cordum_engine* e, cordum_batch* b, uint32_t mode, bool copy_in, bool copy_out) {
  cordum::NvtxRange nvtx_("cordum:dispatch");
  if (!e || !b) { g_err = "null handle"; return CORDUM_E_INVALID; }
  const bool flush_l2 = mode & CORDUM_FLAG_FLUSH_L2;
  const bool timed = !(mode & CORDUM_FLAG_NO_TIMING);   // per-kernel timing events cost two API calls per dispatch
  mode &= 0xFFu;
  if (e->failed) { g_err = "engine failed earlier: " + e->fail_msg; return CORDUM_E_CUDA; }
  if (mode < CORDUM_MODE_POLICY_ONLY || mode > CORDUM_MODE_ROUTE_ONLY) { g_err = "bad mode"; return CORDUM_E_INVALID; }
  if (!b->encoded) { g_err = "batch has not been encoded"; return CORDUM_E_STATE; }
  if (b->device_encoded) copy_in = false;   // the records were produced on the device
  if (!copy_in && !b->resident) { g_err = "batch columns are not resident on the device"; return CORDUM_E_STATE; }
  b->last_mode = mode | (flush_l2 ? CORDUM_FLAG_FLUSH_L2 : 0u) | (timed ? 0u : CORDUM_FLAG_NO_TIMING);
  b->results_ready = false;
  b->timed = timed;
  b->last_copy_out = copy_out;
  if (b->pending) { CK(cudaStreamSynchronize(b->stream), "wait previous"); b->pending = false; b->enc_inflight = false; }
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  DeviceTables tv;
  cudaEvent_t ev_ready = nullptr;
  if (int rc = leave_tick_mode(e)) return rc;
  // e->mu is held until every launch of this dispatch is enqueued: a table sync on another thread (first sight of a
  // topic, a reload) synchronizes the device and may then free and reallocate table buffers - it must not slip in
  // between view() and the launches that use those pointers.
  std::lock_guard<std::mutex> g(e->mu);
  {
    std::lock_guard<std::mutex> gh(e->host->mutex());
    if (b->epoch != e->host->epoch()) { g_err = "tables were reloaded after this batch was encoded: encode again"; return CORDUM_E_STALE; }
    b->text = e->host->policy_text(); b->wtext = e->host->worker_text(); b->ttext = e->host->topic_text();
    int rc = sync_tables(e);
    if (rc) return rc;
    rc = refresh_pools(e, nullptr, nullptr);
    if (rc) return rc;
    tv = view(e, e->cur);
    b->table_set = e->cur;
    ev_ready = e->ds[e->cur].ready;
  }
  cudaStream_t s = b->stream;
  if (flush_l2) {   // evict the job columns from L2 between timed iterations (outside the timed region)
    if (!e->b_flush.p) CK(e->b_flush.reserve(size_t(256) << 20), "alloc flush buffer");
    CK(cudaMemsetAsync(e->b_flush.p, 0, e->b_flush.cap, s), "flush");
  }
  // timing events: a resident run has no copies, so its span is [ev1, ev2] and ev0 / ev3 are not recorded
  b->timed_in = copy_in; b->timed_out = copy_out;
  if (copy_in) {
    CK(cudaEventRecord(b->ev0, s), "event");
    CK(cudaMemcpyAsync(b->d_cols, b->h_cols, slab_bytes(b->n), cudaMemcpyHostToDevice, s), "H2D columns");
    if (b->wide_words) CK(cudaMemcpyAsync(b->d_wide, b->h_wide, (size_t)b->n * b->wide_words * 8, cudaMemcpyHostToDevice, s), "H2D wide masks");
    if (b->sel_words) CK(cudaMemcpyAsync(b->d_sel, b->h_sel, (size_t)b->sel_words * 4, cudaMemcpyHostToDevice, s), "H2D selective list");
    b->resident = true;
  }
  if (timed) CK(cudaEventRecord(b->ev1, s), "event");
  const KParams P = batch_params(b, tv, mode == CORDUM_MODE_POLICY_AND_ROUTE);
  if (P.route_count) CK(cudaMemsetAsync(b->d_route, 0, sizeof(uint32_t), s), "reset route count");
  // policy_kernel needs no worker state: it is NOT ordered after the heartbeat exchange / worker-table refresh kernels
  if (mode != CORDUM_MODE_ROUTE_ONLY) {
    CK(launch_policy(P, e->sm_count, s), "policy_kernel");
    if (b->n) e->launches++;
  }
  if (timed) CK(cudaEventRecord(b->evm, s), "event");
  if (mode != CORDUM_MODE_POLICY_ONLY) {
    CK(cudaStreamWaitEvent(s, ev_ready, 0), "wait worker tables");
    CK(launch_route(P, mode == CORDUM_MODE_ROUTE_ONLY, e->sm_count, s), "route_kernel");
    e->launches += route_launches(P);
  }
  CK(cudaEventRecord(b->ev2, s), "event");
  b->launched = true;
  if (copy_out) {
    CK(cudaMemcpyAsync(b->h_out, b->d_out, (size_t)b->n * sizeof(cordum_decision), cudaMemcpyDeviceToHost, s), "D2H results");
    CK(cudaEventRecord(b->ev3, s), "event");
  }
  b->pending = true;
  return CORDUM_OK;
}

int host_encode_into(cordum_engine* e, cordum_batch* b, const cordum_envelopes* env);

int wait(cordum_batch* b) {
  cordum_engine* e = b->e;
  cordum::NvtxRange nvtx_("cordum:wait");
  if (b->tick_pending) {   // dispatched by a tick: its route runs in the tick after its policy (or in the flush)
    {
      std::lock_guard<std::mutex> g(e->mu);
      if (e->tick.prev == b) { int rc = tick_flush_locked(e); if (rc) return rc; }
    }
    for (cudaStream_t st : e->tick.s) CK(cudaStreamSynchronize(st), "tick wait");
    b->tick_pending = false;
    b->results_ready = true;
    b->total_ms = b->kernel_ms = b->policy_ms = b->route_ms = 0;
  }
  if (!b->pending && !b->enc_inflight) return CORDUM_OK;
  CK(cudaStreamSynchronize(b->stream), "batch wait");
  const bool dispatched = b->pending;
  b->pending = false;
  b->enc_inflight = false;
  if (b->device_encoded && b->h_fallback && *b->h_fallback) {
    // The device encoder met something it leaves to the host (first sight of a topic / effective config, non-ASCII
    // text, an oversized string): encode the batch on the host - which also registers what is new - and run it again.
    *b->h_fallback = 0;
    e->host->host_fallbacks++;
    int rc = host_encode_into(e, b, b->env);
    if (rc) return rc;
    if (!dispatched) return CORDUM_OK;
    rc = run(e, b, b->last_mode, true, b->last_copy_out);
    if (rc) return rc;
    CK(cudaStreamSynchronize(b->stream), "batch wait");
    b->pending = false;
  }
  if (!dispatched) return CORDUM_OK;
  b->results_ready = true;
  if (!b->timed) { b->total_ms = b->kernel_ms = b->policy_ms = b->route_ms = 0; return CORDUM_OK; }
  CK(cudaEventElapsedTime(&b->total_ms, b->timed_in ? b->ev0 : b->ev1, b->timed_out ? b->ev3 : b->ev2), "elapsed");
  CK(cudaEventElapsedTime(&b->kernel_ms, b->ev1, b->ev2), "elapsed");
  CK(cudaEventElapsedTime(&b->policy_ms, b->ev1, b->evm), "elapsed");
  CK(cudaEventElapsedTime(&b->route_ms, b->evm, b->ev2), "elapsed");
  return CORDUM_OK;
}

int64_t copy_out(const std::string& s, char* buf, uint64_t cap) {
  if (buf && cap) {
    size_t n = std::min<size_t>(s.size(), cap - 1);
    std::memcpy(buf, s.data(), n);
    buf[n] = 0;
  }
  return (int64_t)s.size();
}

}  // namespace

static void batch_release(cordum_batch* b) {   // frees the batch's CUDA resources; the registry is the caller's business
  if (b->stream) cudaStreamSynchronize(b->stream);
  if (b->h_cols) cudaFreeHost(b->h_cols);
  if (b->d_cols) cudaFree(b->d_cols);
  if (b->h_wide) cudaFreeHost(b->h_wide);
  if (b->d_wide) cudaFree(b->d_wide);
  if (b->h_sel) cudaFreeHost(b->h_sel);
  if (b->d_sel) cudaFree(b->d_sel);
  if (b->h_out) cudaFreeHost(b->h_out);
  if (b->h_plan) cudaFreeHost(b->h_plan);
  if (b->h_counts) cudaFreeHost(b->h_counts);
  if (b->h_resp) cudaFreeHost(b->h_resp);
  if (b->h_resp_text) cudaFreeHost(b->h_resp_text);
  if (b->h_parent) cudaFreeHost(b->h_parent);
  if (b->d_out) cudaFree(b->d_out);
  if (b->d_route) cudaFree(b->d_route);
  std::free(b->slot_of);
  if (b->h_fallback) cudaFreeHost(b->h_fallback);
  for (cudaEvent_t ev : {b->ev0, b->ev1, b->evm, b->ev2, b->ev3}) if (ev) cudaEventDestroy(ev);
  if (b->stream) cudaStreamDestroy(b->stream);
  delete b;
}


// ------------------------------------------------------------ NCCL, loaded at run time
// The library must not depend on libnccl at link time (single-GPU hosts do not need it), and inside a PyTorch process it
// has to use the copy PyTorch already loaded.  Prototypes restated from nccl.h (2.x ABI).
namespace {
struct NcclId { char internal[128]; };
struct NcclApi {
  void* lib = nullptr;
  int (*GetUniqueId)(NcclId*) = nullptr;
  int (*CommInitRank)(void**, int, NcclId, int) = nullptr;
  int (*AllGather)(const void*, void*, size_t, int, void*, cudaStream_t) = nullptr;
  int (*CommDestroy)(void*) = nullptr;
  const char* (*GetErrorString)(int) = nullptr;
};
constexpr int kNcclUint8 = 1;   // ncclDataType_t: ncclInt8 = 0, ncclUint8 = 1

NcclApi* nccl_api() {
  static NcclApi api;
  static std::once_flag once;
  std::call_once(once, [] {
    const char* names[3] = {getenv("CORDUM_NCCL_LIB"), "libnccl.so.2", "libnccl.so"};
    for (const char* n : names) {
      if (!n || !*n) continue;
      if (void* h = dlopen(n, RTLD_NOW | RTLD_GLOBAL)) { api.lib = h; break; }
    }
    if (!api.lib) return;
    api.GetUniqueId = (int (*)(NcclId*))dlsym(api.lib, "ncclGetUniqueId");
    api.CommInitRank = (int (*)(void**, int, NcclId, int))dlsym(api.lib, "ncclCommInitRank");
    api.AllGather = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(api.lib, "ncclAllGather");
    api.CommDestroy = (int (*)(void*))dlsym(api.lib, "ncclCommDestroy");
    api.GetErrorString = (const char* (*)(int))dlsym(api.lib, "ncclGetErrorString");
    if (!api.GetUniqueId || !api.CommInitRank || !api.AllGather || !api.CommDestroy) { dlclose(api.lib); api = NcclApi{}; }
  });
  return api.lib ? &api : nullptr;
}
int nccl_fail(cordum_engine* e, int rc, const char* what) {
  NcclApi* a = nccl_api();
  g_err = std::string(what) + ": NCCL error " + std::to_string(rc) + (a && a->GetErrorString ? std::string(" (") + a->GetErrorString(rc) + ")" : "");
  if (e) { e->failed = true; e->fail_msg = g_err; }
  return CORDUM_E_CUDA;
}

// One heartbeat epoch through the engine-owned exchange.  Called with both mutexes held.
int ingest(cordum_engine* e, const cordum_worker_load* slice, uint32_t first_slot, uint32_t n_slice) {
  const HostTables& t = e->host->tables();
  const uint32_t W = t.n_slots;
  if (W == 0) { g_err = "no workers loaded"; return CORDUM_E_STATE; }
  const uint32_t per = W / (uint32_t)e->xworld;
  if (W % (uint32_t)e->xworld) { g_err = "worker registry size is not a multiple of the exchange world size"; return CORDUM_E_INVALID; }
  if (first_slot != (uint32_t)e->xrank * per || n_slice != per) { g_err = "slice is not this rank's share of the worker registry"; return CORDUM_E_INVALID; }
  const int g = (int)(e->xepoch & 1);
  e->xepoch++;
  const size_t bytes = (size_t)W * sizeof(Load16), slice_bytes = (size_t)per * sizeof(Load16);
  const bool use_peers = e->peers.ready && e->peers.world > 1 && e->peers.world == e->xworld && e->peers.per == per;
  if (e->xworld == 1 || use_peers) {
    // One graph launch: H2D of the slice -> [gather of all ranks' slices over peer memory] -> worker_chunk -> worker_merge.
    if (int rc = grow_gather(e, bytes)) return rc;
    if (int rc = grow_staging(e, slice_bytes)) return rc;
    CK(cudaEventSynchronize(e->gather_free[g]), "wait staging");   // the epoch two back has consumed this staging / table buffer
    std::memcpy(e->stage[g], slice, slice_bytes);
    *reinterpret_cast<uint32_t*>((uint8_t*)e->stage[g] + slice_bytes) = (uint32_t)e->xepoch;   // the epoch, behind the slice
    const int target = claim_set(e);
    if (target < 0) return target;
    const auto key = std::make_tuple(target, g, e->tables_gen);
    cudaGraphExec_t ge = nullptr;
    auto it = e->ing_graphs.find(key);
    if (it != e->ing_graphs.end()) ge = it->second;
    else {
      if (e->ing_graphs.size() > 32) { for (auto& kv : e->ing_graphs) cudaGraphExecDestroy(kv.second); e->ing_graphs.clear(); }
      CK(launch_configure(), "kernel attributes");
      cudaStream_t S = e->s_tables;
      CK(cudaStreamBeginCapture(S, cudaStreamCaptureModeThreadLocal), "begin capture");
      const cudaError_t ce = enqueue_heartbeat(e, S, g, target, use_peers);
      cudaGraph_t gr = nullptr;
      cudaError_t ee = cudaStreamEndCapture(S, &gr);
      if (ce != cudaSuccess || ee != cudaSuccess) { if (gr) cudaGraphDestroy(gr); return fail(e, ce != cudaSuccess ? ce : ee, "capture of the ingest graph"); }
      cudaError_t ie = cudaGraphInstantiate(&ge, gr, 0);
      cudaGraphDestroy(gr);
      if (ie != cudaSuccess) return fail(e, ie, "graph instantiate");
      e->ing_graphs[key] = ge;
    }
    CK(cudaGraphLaunch(ge, e->s_tables), "graph launch");
    CK(cudaEventRecord(e->gather_free[g], e->s_tables), "event record");
    return publish_set(e, target, refresh_launches(e) + (use_peers ? 1 : 0));
  }
  if (int rc = grow_gather(e, bytes)) return rc;
  uint8_t* table = (uint8_t*)e->gather[g].p;
  // the refresh two epochs ago read this buffer
  CK(cudaStreamWaitEvent(e->s_xchg, e->gather_free[g], 0), "wait gather buffer");
  CK(cudaMemcpyAsync(table + (size_t)first_slot * sizeof(Load16), slice, slice_bytes, cudaMemcpyHostToDevice, e->s_xchg), "H2D heartbeat slice");
  if (e->xworld > 1) {   // in place: this rank's slice already sits at its offset of the receive buffer
    int rc = nccl_api()->AllGather(table + (size_t)first_slot * sizeof(Load16), table, slice_bytes, kNcclUint8, e->nccl_comm, e->s_xchg);
    if (rc) return nccl_fail(e, rc, "ncclAllGather");
  }
  CK(cudaEventRecord(e->ev_xchg, e->s_xchg), "event record");
  const int target = claim_set(e);
  if (target < 0) return target;
  CK(cudaStreamWaitEvent(e->s_tables, e->ev_xchg, 0), "order refresh after exchange");
  // the refresh reads the gathered table in place
  return refresh_on_tables_stream(e, target, (const Load16*)table, e->gather_free[g]);
}
}  // namespace

namespace {
// ------------------------------------------------------------ scheduler ticks
// One tick = one CUDA graph launch with three independent branches:
//     A  heartbeat epoch k: H2D of this rank's slice -> [peer gather over NVLink] -> worker_chunk -> worker_merge   (set k % 2)
//     B  policy_kernel of the batch handed in with this tick
//     C  route_kernel of the batch handed in with the PREVIOUS tick, on the worker tables of epoch k-1            (set (k-1) % 2)
// so a tick costs max(A, B, C) instead of their sum plus ~17 API calls, and consecutive ticks still overlap what the
// multi-stream path overlapped.  Graphs are cached per (new batch, previous batch, parity, sizes, table generation).
int tick_share() { static const int v = []() { const char* s = getenv("CORDUM_TICK_SHARE"); return s ? atoi(s) : 0; }(); return v; }   // > 0: cap each branch at that many CTAs per SM (measured: no gain, 0 = full grids)

int tick_graph(cordum_engine* e, cordum_batch* bn, cordum_batch* bp, int phase, bool bn_routed_last_tick, cudaGraphExec_t* out) {
  // phase = tick number mod 6: stream / staging / gather-buffer parity = phase & 1, derived-table set = phase % 3
  auto& T = e->tick;
  const uint32_t W = e->host->tables().n_slots;
  const auto key = std::make_tuple(bn, bp, phase + (bn_routed_last_tick ? 8 : 0), bn ? bn->n : 0u, bp ? bp->n : 0u,
                                   bp ? bp->n_sel_jobs : 0u, e->tables_gen);
  auto it = T.graphs.find(key);
  if (it != T.graphs.end()) { *out = it->second; return CORDUM_OK; }
  if (T.graphs.size() > 96) {   // stale generations / batches: start over
    for (auto& kv : T.graphs) cudaGraphExecDestroy(kv.second);
    T.graphs.clear();
  }
  CK(launch_configure(), "kernel attributes");
  const int parity = phase & 1, set_new = phase % 3, set_old = (phase + 2) % 3;
  cudaStream_t S = T.s[parity];
  CK(cudaStreamBeginCapture(S, cudaStreamCaptureModeThreadLocal), "begin capture");
  auto fail_capture = [&](cudaError_t err, const char* what) {
    cudaGraph_t g = nullptr;
    cudaStreamEndCapture(S, &g);
    if (g) cudaGraphDestroy(g);
    return fail(e, err, what);
  };
#define CKC(call, what) do { cudaError_t _e = (call); if (_e != cudaSuccess) return fail_capture(_e, what); } while (0)
  CKC(cudaEventRecord(T.ev_fork, S), "fork");
  // ---- A: heartbeat epoch, behind the heartbeat branch of the previous tick (a graph of its own, on the other stream)
  CKC(cudaStreamWaitEvent(T.sa, T.ev_fork, 0), "fork");
  CKC(cudaStreamWaitEvent(T.sa, T.refreshed[parity ^ 1], cudaEventWaitExternal), "order heartbeat epochs");
  if (W) CKC(enqueue_heartbeat(e, T.sa, parity, set_new, e->peers.ready && e->peers.world > 1), "heartbeat epoch");
  CKC(cudaEventRecordWithFlags(T.refreshed[parity], T.sa, cudaEventRecordExternal), "publish heartbeat epoch");
  CKC(cudaEventRecord(T.ev_a, T.sa), "join");
  // ---- C: route of the previous batch on the previous epoch's tables, once the previous tick (policy of that batch, refresh
  //         of that epoch) has finished
  if (bp && bp->n) {
    CKC(cudaStreamWaitEvent(T.sc, T.ev_fork, 0), "fork");
    CKC(cudaStreamWaitEvent(T.sc, T.done[parity ^ 1], cudaEventWaitExternal), "wait previous tick");
    CKC(launch_route(batch_params(bp, view(e, set_old), true), false, e->sm_count, T.sc, tick_share()), "route_kernel");
    CKC(cudaEventRecord(T.ev_c, T.sc), "join");
  }
  // ---- B: policy of the new batch
  if (bn && bn->n) {
    const KParams P = batch_params(bn, view(e, set_old), true);   // policy_kernel reads no worker state
    // this batch's previous use was routed by the tick before this one (only two batches alternate): that route still
    // reads what this policy run overwrites
    if (bn_routed_last_tick) CKC(cudaStreamWaitEvent(S, T.done[parity ^ 1], cudaEventWaitExternal), "wait previous route of this batch");
    CKC(cudaMemsetAsync(bn->d_route, 0, sizeof(uint32_t), S), "reset route count");
    CKC(launch_policy(P, e->sm_count, S, tick_share()), "policy_kernel");
  }
  CKC(cudaStreamWaitEvent(S, T.ev_a, 0), "join");
  if (bp && bp->n) CKC(cudaStreamWaitEvent(S, T.ev_c, 0), "join");
#undef CKC
  cudaGraph_t g = nullptr;
  CK(cudaStreamEndCapture(S, &g), "end capture");
  cudaGraphExec_t ge = nullptr;
  cudaError_t ie = cudaGraphInstantiate(&ge, g, 0);
  cudaGraphDestroy(g);
  if (ie != cudaSuccess) return fail(e, ie, "graph instantiate");
  T.graphs[key] = ge;
  *out = ge;
  return CORDUM_OK;
}

int tick_setup(cordum_engine* e) {
  auto& T = e->tick;
  if (T.s[0]) return CORDUM_OK;
  for (auto& st : T.s) CK(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking), "stream");
  {   // the heartbeat branch is the head of the next tick's dependency chain: its kernels are captured at high priority
    int lo = 0, hi = 0;
    CK(cudaDeviceGetStreamPriorityRange(&lo, &hi), "priority range");
    CK(cudaStreamCreateWithPriority(&T.sa, cudaStreamNonBlocking, hi), "stream");
  }
  CK(cudaStreamCreateWithFlags(&T.sc, cudaStreamNonBlocking), "stream");
  for (cudaEvent_t* ev : {&T.ev_fork, &T.ev_a, &T.ev_c, &T.ev_join}) CK(cudaEventCreateWithFlags(ev, cudaEventDisableTiming), "event");
  for (int i = 0; i < 2; ++i) {
    CK(cudaEventCreateWithFlags(&T.done[i], cudaEventDisableTiming), "event"); CK(cudaEventRecord(T.done[i], T.s[i]), "event");
    CK(cudaEventCreateWithFlags(&T.refreshed[i], cudaEventDisableTiming), "event"); CK(cudaEventRecord(T.refreshed[i], T.s[i]), "event");
  }
  return CORDUM_OK;
}

// one tick; e->mu and the host mutex held.  bn may be null (flush: only route the previous batch)
int tick_locked(cordum_engine* e, cordum_batch* bn, const cordum_worker_load* slice, uint32_t n_slice) {
  cordum::NvtxRange nvtx_("cordum:tick");
  auto& T = e->tick;
  const HostTables& t = e->host->tables();
  const uint32_t W = t.n_slots;
  const int phase = (int)(T.n % 6), parity = phase & 1;
  if (!bn) {
    // flush: the route of the previous batch alone, behind its tick (policy of that batch, refresh of that epoch); then both
    // tick streams are joined so that an event recorded on s[0] afterwards covers everything issued so far
    cordum_batch* bp = T.prev;
    if (bp) {
      const int pp = (int)((T.n + 5) % 6);   // phase of the previous tick
      cudaStream_t S = T.s[parity];
      CK(cudaStreamWaitEvent(S, T.done[pp & 1], 0), "wait previous tick");
      const KParams P = batch_params(bp, view(e, pp % 3), true);
      CK(launch_route(P, false, e->sm_count, S), "route_kernel");
      e->launches += route_launches(P);
      T.prev = nullptr;
    }
    CK(cudaEventRecord(T.ev_join, T.s[1]), "join"); CK(cudaStreamWaitEvent(T.s[0], T.ev_join, 0), "join");
    CK(cudaEventRecord(T.ev_join, T.s[0]), "join"); CK(cudaStreamWaitEvent(T.s[1], T.ev_join, 0), "join");
    return CORDUM_OK;
  }
  static const bool trace = getenv("CORDUM_TICK_TRACE") != nullptr;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto us = [](auto a, auto b) { return std::chrono::duration<double, std::micro>(b - a).count(); };
  const auto t0 = now();
  // staging of this parity was last read by the H2D of tick n-2
  CK(cudaEventSynchronize(T.done[parity]), "wait staging");
  const auto t1 = now();
  const size_t bytes = (size_t)n_slice * sizeof(Load16);
  if (int rc = grow_staging(e, bytes)) return rc;
  if (bytes) std::memcpy(e->stage[parity], slice, bytes);
  *reinterpret_cast<uint32_t*>((uint8_t*)e->stage[parity] + bytes) = (uint32_t)(++e->xepoch);   // the epoch (shared with cordum_workers_ingest), behind the slice
  if (int rc = grow_gather(e, (size_t)W * sizeof(Load16))) return rc;
  const auto t2 = now();
  cudaGraphExec_t ge = nullptr;
  // Ticks up to n-2 have finished when tick n starts (stream order + the route branch's wait); tick n-1 may still run.
  const bool routed_last = bn->tick_pending && T.n - bn->tick_no == 2;   // handed in with tick n-2, routed by tick n-1
  int rc = tick_graph(e, bn, T.prev, phase, routed_last, &ge);
  if (rc) return rc;
  const auto t3 = now();
  CK(cudaGraphLaunch(ge, T.s[parity]), "graph launch");
  CK(cudaEventRecord(T.done[parity], T.s[parity]), "event record");
  if (trace) {
    static double acc[4] = {0, 0, 0, 0};
    static uint64_t cnt = 0;
    const auto t4 = now();
    acc[0] += us(t0, t1); acc[1] += us(t1, t2); acc[2] += us(t2, t3); acc[3] += us(t3, t4);
    if (++cnt % 100 == 0) {
      fprintf(stderr, "tick host us (mean of 100): wait-staging %.1f  stage-slice %.1f  graph-lookup/capture %.1f  launch+record %.1f\n",
              acc[0] / 100, acc[1] / 100, acc[2] / 100, acc[3] / 100);
      acc[0] = acc[1] = acc[2] = acc[3] = 0;
    }
  }
  e->launches += (W ? refresh_launches(e) + (e->peers.ready && e->peers.world > 1 ? 1 : 0) : 0) + (bn->n ? 1 : 0) +
                 (T.prev ? route_launches(batch_params(T.prev, e->dt, true)) : 0);
  e->cur = phase % 3;   // the set this tick refreshed (a later plain dispatch continues from it)
  e->pools_dirty = false;
  bn->tick_no = T.n;
  T.prev = bn;
  T.n++;
  T.active = true;
  return CORDUM_OK;
}
int tick_flush_locked(cordum_engine* e) { return tick_locked(e, nullptr, nullptr, 0); }

// The host encoder's selective list into the batch's pinned staging (grown on first need), for the next H2D of the records.
int stage_selective(cordum_engine* e, cordum_batch* b) {
  const auto &jobs = b->hr.sel_jobs, &extra = b->hr.sel_extra;
  const size_t words = jobs.size() + extra.size();
  if (words > b->sel_cap) {
    std::lock_guard<std::mutex> g(e->mu);
    CK(cudaSetDevice(e->device), "cudaSetDevice");
    CK(cudaStreamSynchronize(b->stream), "wait before reallocating the selective list");
    if (b->h_sel) cudaFreeHost(b->h_sel);
    if (b->d_sel) cudaFree(b->d_sel);
    b->h_sel = b->d_sel = nullptr; b->sel_cap = 0;
    const size_t cap = std::max<size_t>(words + words / 4, 1024);
    CK(cudaHostAlloc((void**)&b->h_sel, cap * 4, cudaHostAllocDefault), "pinned selective list");
    CK(cudaMalloc((void**)&b->d_sel, cap * 4), "selective list");
    b->sel_cap = cap;
    e->tables_gen++;   // captured graphs bake the batch's pointers in
  }
  if (words) {
    std::memcpy(b->h_sel, jobs.data(), jobs.size() * 4);
    std::memcpy(b->h_sel + jobs.size(), extra.data(), extra.size() * 4);
  }
  b->n_sel_jobs = (uint32_t)(jobs.size() / 2);
  b->sel_words = (uint32_t)words;
  return CORDUM_OK;
}

int host_encode_into(cordum_engine* e, cordum_batch* b, const cordum_envelopes* env) {
  cordum::NvtxRange nvtx_("cordum:encode_host");
  if (!env) { g_err = "envelopes no longer available for the host encoder"; return CORDUM_E_STATE; }
  b->n = env->n_jobs;
  b->encoded = false;
  b->resident = false;
  b->device_encoded = false;
  b->results_ready = false;
  b->is_subset = false;
  uint64_t epoch_before = 0;
  int rc = CORDUM_OK;
  for (int attempt = 0; attempt < 3; ++attempt) {
    // a policy / registry whose dictionaries outgrow the records' mask fields needs a side row per job (WideLayout)
    // Sized by the jobs actually in the batch (rounded up), not by max_jobs: the rows are dense (a registry with 60k label
    // bits costs 7.5 KB per job), so a small batch must not pay for the largest one the handle could hold.
    const uint64_t ww = e->host->wide_words();
    const uint64_t jobs_cap = std::min<uint64_t>(b->max_jobs, std::max<uint64_t>(1024, (uint64_t)env->n_jobs + env->n_jobs / 4));
    const uint64_t need = ww * jobs_cap;
    if (ww * env->n_jobs > b->wide_cap) {
      if (need * 8 > (uint64_t(4) << 30)) {   // not a device failure: refuse this batch, keep the engine
        g_err = "wide-mask rows for this batch need " + std::to_string(need * 8 >> 20) + " MiB (" + std::to_string(ww * 8) +
                " B per job: the policy / registry label universe is very large); submit smaller batches";
        return CORDUM_E_CAPACITY;
      }
      std::lock_guard<std::mutex> g(e->mu);
      CK(cudaSetDevice(e->device), "cudaSetDevice");
      CK(cudaStreamSynchronize(b->stream), "wait before reallocating the wide rows");
      if (b->h_wide) cudaFreeHost(b->h_wide);
      if (b->d_wide) cudaFree(b->d_wide);
      b->h_wide = b->d_wide = nullptr; b->wide_cap = 0;
      if (cudaHostAlloc((void**)&b->h_wide, need * 8, cudaHostAllocDefault) != cudaSuccess || cudaMalloc((void**)&b->d_wide, need * 8) != cudaSuccess) {
        cudaGetLastError();   // an allocation that does not fit is this batch's problem, not a sticky engine failure
        if (b->h_wide) cudaFreeHost(b->h_wide);
        b->h_wide = b->d_wide = nullptr;
        g_err = "out of memory for " + std::to_string(need * 8 >> 20) + " MiB of wide-mask rows; submit smaller batches";
        return CORDUM_E_CAPACITY;
      }
      b->wide_cap = need;
      e->tables_gen++;   // captured graphs bake the batch's pointers in
    }
    host_records(b);
    rc = e->host->encode(env, b->hr, g_err);
    epoch_before = b->hr.epoch;   // the epoch the ids belong to, read under the encoder's lock (a dictionary reset inside the encode moves it)
    if (rc != cordum::kWideRetry) break;   // the tables changed between the look and the encode: size again
  }
  if (rc) return rc == cordum::kWideRetry ? CORDUM_E_STALE : rc;
  if (int rc2 = stage_selective(e, b)) return rc2;
  b->wide_words = b->hr.wide_words;
  b->epoch = epoch_before;
  b->encoded = true;
  b->host_records_valid = true;
  return CORDUM_OK;
}

// cordum_batch_plan on a batch whose records are complete in d_out.  Device scratch (32-bit words): keys / values x 2 (n
// each) | counts [256][tiles] | totals [256] | offsets [n_buckets + 1] | flag; pinned: offsets | flag | jobs [n].
int plan_batch(cordum_engine* e, cordum_batch* b, cordum_plan* out) {
  PlanParams P{};
  P.recs = b->d_out;
  P.n = b->n;
  P.n_slots = b->wtext ? (uint32_t)b->wtext->size() : 0u;   // the registry the batch was routed on
  P.n_buckets = P.n_slots + CORDUM_PLAN_OUTCOMES;
  const size_t n = P.n, nb = P.n_buckets, tiles = (n + CORDUM_PLAN_TILE - 1) / CORDUM_PLAN_TILE;
  const size_t dev_words = n ? 4 * n + 256 * tiles + 256 + nb + 2 : 0, host_words = nb + 2 + n;
  if (dev_words * 4 > b->d_plan.cap || host_words > b->h_plan_cap) {
    // an allocation that does not fit is this call's problem, not a sticky engine failure
    const size_t dev_bytes = dev_words * 4;
    const cudaError_t de = dev_bytes > b->d_plan.cap ? b->d_plan.reserve(dev_bytes + dev_bytes / 4) : cudaSuccess;
    cudaError_t he = cudaSuccess;
    if (de == cudaSuccess && host_words > b->h_plan_cap) {
      if (b->h_plan) cudaFreeHost(b->h_plan);
      b->h_plan = nullptr; b->h_plan_cap = 0;
      const size_t want = host_words + host_words / 4;
      he = cudaHostAlloc((void**)&b->h_plan, want * 4, cudaHostAllocDefault);
      if (he == cudaSuccess) b->h_plan_cap = want;
      else b->h_plan = nullptr;
    }
    if (de != cudaSuccess || he != cudaSuccess) {
      cudaGetLastError();
      g_err = "out of memory for the plan of " + std::to_string(n) + " jobs over " + std::to_string(nb) + " buckets";
      return CORDUM_E_CAPACITY;
    }
  }
  uint32_t* h = b->h_plan;
  out->n_slots = P.n_slots;
  out->n_jobs = P.n;
  out->offsets = h;
  out->jobs = h + nb + 2;
  if (n == 0) { std::memset(h, 0, (nb + 1) * 4); return CORDUM_OK; }
  uint32_t* w = (uint32_t*)b->d_plan.p;
  P.keys[0] = w; P.vals[0] = w + n; P.keys[1] = w + 2 * n; P.vals[1] = w + 3 * n;
  P.counts = w + 4 * n;
  P.totals = P.counts + 256 * tiles;
  P.offsets = P.totals + 256;
  P.bad = P.offsets + nb + 1;
  cudaStream_t s = b->stream;
  CK(launch_plan(P, s), "plan kernels");
  e->launches += plan_launches(P);
  CK(cudaMemcpyAsync(h, P.offsets, (nb + 2) * 4, cudaMemcpyDeviceToHost, s), "D2H plan offsets");
  CK(cudaMemcpyAsync(h + nb + 2, P.vals[(plan_passes(P.n_buckets) - 1) & 1], n * 4, cudaMemcpyDeviceToHost, s), "D2H plan jobs");
  CK(cudaStreamSynchronize(s), "plan");
  if (h[nb + 1]) {
    g_err = "a decision record of this batch names a worker slot outside the registry it was dispatched against (the registry "
            "was reloaded while the batch was in flight): encode and dispatch it again";
    return CORDUM_E_STALE;
  }
  return CORDUM_OK;
}

// The batch's pinned topic-count buffer, grown to at least `words` 32-bit words; false (buffer released) when it does not fit.
bool counts_host_reserve(cordum_batch* b, size_t words) {
  if (words <= b->h_counts_cap) return true;
  if (b->h_counts) cudaFreeHost(b->h_counts);
  b->h_counts = nullptr; b->h_counts_cap = 0;
  const size_t want = std::max<size_t>(words + words / 4, 64);
  if (cudaHostAlloc((void**)&b->h_counts, want * 4, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();   // an allocation that does not fit is this call's problem, not a sticky engine failure
    b->h_counts = nullptr;
    return false;
  }
  b->h_counts_cap = want;
  return true;
}

// cordum_batch_topic_counts on a batch whose records are complete in d_out.  Device scratch (32-bit words): table
// [n_topics][13] | head [2] | rows [n_topics][14].  Pinned: the copied non-zero rows; once they are merged by label, the
// output: counts [n_rows][13] | label offsets [n_rows + 1] | label bytes.
int count_batch(cordum_engine* e, cordum_batch* b, cordum_topic_counts* out) {
  constexpr uint32_t C = CORDUM_COUNT_COLUMNS;
  CountParams P{};
  JobRecords R;
  device_records(b, R);
  P.job = R.job;
  P.out = reinterpret_cast<const uint4*>(b->d_out);
  P.n = b->n;
  P.n_slots = b->wtext ? (uint32_t)b->wtext->size() : 0u;   // the registry the batch was routed on
  {
    std::lock_guard<std::mutex> g(e->host->mutex());        // a generation's topic store grows under this lock
    P.n_topics = b->ttext ? (uint32_t)b->ttext->size() : 0u;
  }
  const size_t nt = P.n_topics, dev_words = P.n ? nt * C + 2 + nt * (C + 1) : 0;
  const cudaError_t de = dev_words * 4 > b->d_counts.cap ? b->d_counts.reserve(dev_words * 5) : cudaSuccess;   // + 1/4
  if (de != cudaSuccess || !counts_host_reserve(b, 2)) {
    cudaGetLastError();
    g_err = "out of memory for the topic counts of " + std::to_string(P.n) + " jobs over " + std::to_string(nt) + " topic ids";
    return CORDUM_E_CAPACITY;
  }
  out->n_jobs = P.n;
  if (P.n == 0) {
    b->h_counts[0] = 0;
    out->n_rows = 0;
    out->counts = out->label_off = b->h_counts;
    out->label_bytes = reinterpret_cast<const uint8_t*>(b->h_counts + 1);
    return CORDUM_OK;
  }
  uint32_t* w = (uint32_t*)b->d_counts.p;
  P.table = w;
  P.head = w + nt * C;
  P.rows = P.head + 2;
  cudaStream_t s = b->stream;
  CK(launch_counts(P, s), "topic count kernels");
  e->launches += counts_launches(P);
  CK(cudaMemcpyAsync(b->h_counts, P.head, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s), "D2H topic count head");
  CK(cudaStreamSynchronize(s), "topic counts");
  if (b->h_counts[1]) {
    g_err = "a decision record of this batch names a worker slot outside the registry it was dispatched against (the registry "
            "was reloaded while the batch was in flight): encode and dispatch it again";
    return CORDUM_E_STALE;
  }
  const uint32_t m = b->h_counts[0];
  if (!counts_host_reserve(b, (size_t)m * (C + 1))) {
    g_err = "out of memory for the " + std::to_string(m) + " topic rows of a batch";
    return CORDUM_E_CAPACITY;
  }
  if (m) CK(cudaMemcpyAsync(b->h_counts, P.rows, (size_t)m * (C + 1) * 4, cudaMemcpyDeviceToHost, s), "D2H topic rows");
  CK(cudaStreamSynchronize(s), "topic rows");
  // merge by label, TrimSpace(raw topic) in the batch's dictionary generation, and order the rows by label bytes
  // (std::string compares as unsigned char)
  struct Row { std::string label; uint32_t cnt[C]; };
  std::vector<Row> rows(m);
  {
    std::lock_guard<std::mutex> g(e->host->mutex());
    for (uint32_t i = 0; i < m; ++i) {
      const uint32_t* r = b->h_counts + (size_t)i * (C + 1);
      rows[i].label = std::string(cordum::trim_space((*b->ttext)[r[0]]));   // r[0] < n_topics: the kernel checked it
      std::memcpy(rows[i].cnt, r + 1, sizeof rows[i].cnt);
    }
  }
  std::sort(rows.begin(), rows.end(), [](const Row& x, const Row& y) { return x.label < y.label; });
  std::vector<uint32_t> cnt, off{0};
  std::string bytes;
  for (uint32_t i = 0; i < m; ++i) {
    if (i == 0 || rows[i].label != rows[i - 1].label) {
      cnt.resize(cnt.size() + C, 0);
      bytes += rows[i].label;
      off.push_back((uint32_t)bytes.size());
    }
    for (uint32_t c = 0; c < C; ++c) cnt[cnt.size() - C + c] += rows[i].cnt[c];
  }
  const uint32_t n_rows = (uint32_t)off.size() - 1;
  if (!counts_host_reserve(b, cnt.size() + off.size() + (bytes.size() + 3) / 4)) {
    g_err = "out of memory for the topic counts of " + std::to_string(n_rows) + " labels";
    return CORDUM_E_CAPACITY;
  }
  uint32_t* h = b->h_counts;
  std::memcpy(h, cnt.data(), cnt.size() * 4);
  std::memcpy(h + cnt.size(), off.data(), off.size() * 4);
  std::memcpy(h + cnt.size() + off.size(), bytes.data(), bytes.size());
  out->n_rows = n_rows;
  out->counts = h;
  out->label_off = h + cnt.size();
  out->label_bytes = reinterpret_cast<const uint8_t*>(h + cnt.size() + off.size());
  return CORDUM_OK;
}

// arg of a record's reason code (the class key of include/cordum_b200.h; responses.cu reason_arg is the device's copy).
uint32_t reason_arg(uint32_t code, const JobRec& j) {
  if (code == CORDUM_REASON_EFF_DENIED_TOPIC || code == CORDUM_REASON_EFF_NOT_ALLOWED_TOPIC) return j.topic;
  if (code >= CORDUM_REASON_TENANT_MCP && code < CORDUM_REASON_TENANT_MCP + 8) return j.mcp[(code - CORDUM_REASON_TENANT_MCP) >> 1];
  if (code >= CORDUM_REASON_EFF_MCP && code < CORDUM_REASON_EFF_MCP + 8) return j.mcp[(code - CORDUM_REASON_EFF_MCP) >> 1];
  return 0;
}
bool mcp_reason(uint32_t code) {
  return (code >= CORDUM_REASON_TENANT_MCP && code < CORDUM_REASON_TENANT_MCP + 8) ||
         (code >= CORDUM_REASON_EFF_MCP && code < CORDUM_REASON_EFF_MCP + 8);
}

// The reason text of a record of batch b (kernel.go:172,175,221,225; safety_policy.go:410,413; engine.go:500), from its
// reason code, rule index and reason_arg.  With env, an MCP reason quotes the request's own spelling of job's value (%q of
// the trimmed label value, as the reference does); without it the canonical (trimmed, case-folded) form the dictionaries
// keep.  Called with the host mutex held.  False when that canonical form is gone (the value dictionaries were rebuilt
// since the batch was encoded).
bool render_reason(cordum_engine* e, const cordum_batch* b, uint32_t code, int32_t rule_idx, uint32_t arg, uint32_t flavor,
                   const cordum_envelopes* env, uint32_t job, std::string& s) {
  static const char* fields[4] = {"server", "tool", "resource", "action"};
  s.clear();
  if (code == CORDUM_REASON_RULE) {
    // the policy the batch was dispatched under, not whatever is in force by now
    if (b->text && rule_idx >= 0 && (size_t)rule_idx < b->text->rules.size()) s = b->text->rules[rule_idx].reason;
  } else if (code == CORDUM_REASON_MISSING_TOPIC) s = "missing topic";
  else if (code == CORDUM_REASON_UNSUPPORTED_TOPIC) s = "unsupported topic";
  else if (code == CORDUM_REASON_APPROVAL_GRANTED) s = "approval granted";
  else if (code == CORDUM_REASON_EFF_DENIED_TOPIC || code == CORDUM_REASON_EFF_NOT_ALLOWED_TOPIC) {
    std::string topic((b->ttext && arg < b->ttext->size()) ? cordum::trim_space((*b->ttext)[arg]) : sv());
    const char* tail = code == CORDUM_REASON_EFF_DENIED_TOPIC ? " denied by effective config" : " not allowed by effective config";
    // kernel.go:221,225 print '%s'; the gateway's copy of the evaluator prints %q (policy_bundles.go:1207,1211)
    s = "topic " + (flavor == CORDUM_REASON_FLAVOR_GATEWAY ? cordum::go_quote(topic) : "'" + topic + "'") + tail;
  } else if (mcp_reason(code)) {
    uint32_t k = code >= CORDUM_REASON_EFF_MCP ? code - CORDUM_REASON_EFF_MCP : code - CORDUM_REASON_TENANT_MCP;
    int f = (int)(k >> 1);
    if (!env && b->epoch != e->host->epoch()) return false;   // the value dictionaries were rebuilt since: only the envelopes still know
    std::string v = env ? cordum::mcp_request_value(env, job, f) : e->host->mcp_value_string(f, arg);
    s = std::string("mcp ") + fields[f] + " " + cordum::go_quote(v) + ((k & 1) ? " not allowed" : " denied");
  }
  return true;
}

// A pinned buffer of the batch grown to at least `count` elements; false (buffer released) when it does not fit.
template <class T>
bool pinned_reserve(T*& p, size_t& cap, size_t count) {
  if (count <= cap) return true;
  if (p) cudaFreeHost(p);
  p = nullptr;
  cap = 0;
  const size_t want = std::max<size_t>(count + count / 4, 64);
  if (cudaHostAlloc((void**)&p, want * sizeof(T), cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();   // an allocation that does not fit is this call's problem, not a sticky engine failure
    p = nullptr;
    return false;
  }
  cap = want;
  return true;
}

// cordum_batch_responses on a batch whose records are complete in d_out.  Device scratch (32-bit words): keys x 2 [2n
// each] | vals x 2 [n each] | jflag, sloc, perm, start, size [n each] | classes [4n] | offsets [n + 1] | jobs [n] | counts
// [256][tiles] | totals [256] | hcnt, jcnt, ccnt [tiles each] | head [2].  Pinned: head [2] | classes [4m] | offsets
// [m + 1] | jobs [n] | reason offsets [m + 1] | rule id offsets [m + 1]; the text bytes in an arena of their own.
int responses_batch(cordum_engine* e, cordum_batch* b, uint32_t flavor, cordum_responses* out) {
  constexpr uint32_t T = CORDUM_SUBSET_TILE;
  RespParams P{};
  JobRecords R;
  device_records(b, R);
  P.job = R.job;
  P.out = reinterpret_cast<const uint4*>(b->d_out);
  P.n = b->n;
  P.n_tiles = (uint32_t)(((uint64_t)P.n + T - 1) / T);
  size_t n_topics;
  {
    std::lock_guard<std::mutex> g(e->host->mutex());        // a generation's topic store grows under this lock
    n_topics = b->ttext ? b->ttext->size() : 0;
  }
  auto width = [](uint64_t v) { uint32_t k = 0; while (k < 64 && (v >> k)) ++k; return k; };   // bits that hold 0 .. v
  const uint64_t n_rules = b->text ? b->text->rules.size() : 0;
  P.w_rule = width(n_rules);                                   // rule_idx + 1 in 0 .. n_rules
  P.w_arg = std::max<uint32_t>(16, width(n_topics ? n_topics - 1 : 0));   // MCP value ids are 16-bit
  const uint32_t key_bits = CORDUM_RESP_FIXED_BITS + P.w_rule + P.w_arg;
  if (key_bits > 64) {
    g_err = "the response class key needs " + std::to_string(key_bits) + " bits (" + std::to_string(n_rules) + " rules, " +
            std::to_string(n_topics) + " topic ids), more than 64";
    return CORDUM_E_CAPACITY;
  }
  P.passes = (key_bits + 7) / 8;
  const size_t n = P.n, tiles = P.n_tiles, dev_words = n ? 6 * n + 5 * n + 4 * n + (n + 1) + n + 256 * tiles + 256 + 3 * tiles + 2 : 0;
  const cudaError_t de = dev_words * 4 > b->d_resp.cap ? b->d_resp.reserve(dev_words * 5) : cudaSuccess;   // + 1/4
  if (de != cudaSuccess || !pinned_reserve(b->h_resp, b->h_resp_cap, 2)) {
    cudaGetLastError();
    g_err = "out of memory for the responses of " + std::to_string(n) + " jobs";
    return CORDUM_E_CAPACITY;
  }
  out->n_jobs = P.n;
  out->policy_gen = b->text ? b->text->gen : 0;
  if (n == 0) {
    uint32_t* h = b->h_resp;
    h[0] = h[1] = 0;   // offsets, reason offsets and rule id offsets: [0]
    out->n_classes = 0;
    out->classes = reinterpret_cast<const cordum_response_class*>(h);
    out->offsets = out->jobs = out->reason_off = out->rule_id_off = h;
    out->reason_bytes = out->rule_id_bytes = reinterpret_cast<const uint8_t*>(h + 1);
    return CORDUM_OK;
  }
  uint32_t* w = (uint32_t*)b->d_resp.p;
  P.keys[0] = reinterpret_cast<unsigned long long*>(w);
  P.keys[1] = reinterpret_cast<unsigned long long*>(w + 2 * n);
  P.vals[0] = w + 4 * n;
  P.vals[1] = w + 5 * n;
  P.jflag = w + 6 * n;
  P.sloc = w + 7 * n;
  P.perm = w + 8 * n;
  P.start = w + 9 * n;
  P.size = w + 10 * n;
  P.cls = reinterpret_cast<cordum_response_class*>(w + 11 * n);
  P.offsets = w + 15 * n;
  P.jobs = w + 16 * n + 1;
  P.counts = w + 17 * n + 1;
  P.totals = P.counts + 256 * tiles;
  P.hcnt = P.totals + 256;
  P.jcnt = P.hcnt + tiles;
  P.ccnt = P.jcnt + tiles;
  P.head = P.ccnt + tiles;
  cudaStream_t s = b->stream;
  CK(cudaMemsetAsync(P.head, 0, 2 * sizeof(uint32_t), s), "responses head");
  CK(launch_responses(P, s), "response kernels");
  e->launches += responses_launches(P);
  CK(cudaMemcpyAsync(b->h_resp, P.head, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s), "D2H response head");
  CK(cudaStreamSynchronize(s), "responses");
  if (b->h_resp[1]) {
    g_err = "a decision record of this batch names a rule or a value outside the tables it was dispatched against: encode and "
            "dispatch it again";
    return CORDUM_E_STALE;
  }
  const size_t m = b->h_resp[0];
  const size_t at_cls = 2, at_off = at_cls + 4 * m, at_jobs = at_off + m + 1, at_roff = at_jobs + n, at_ioff = at_roff + m + 1;
  if (!pinned_reserve(b->h_resp, b->h_resp_cap, at_ioff + m + 1)) {
    g_err = "out of memory for the " + std::to_string(m) + " response classes of a batch";
    return CORDUM_E_CAPACITY;
  }
  uint32_t* h = b->h_resp;
  CK(cudaMemcpyAsync(h + at_cls, P.cls, m * sizeof(cordum_response_class), cudaMemcpyDeviceToHost, s), "D2H response classes");
  CK(cudaMemcpyAsync(h + at_off, P.offsets, (m + 1) * 4, cudaMemcpyDeviceToHost, s), "D2H response offsets");
  CK(cudaMemcpyAsync(h + at_jobs, P.jobs, n * 4, cudaMemcpyDeviceToHost, s), "D2H response jobs");
  CK(cudaStreamSynchronize(s), "response lists");
  // one reason and one rule id per class (frontend.cpp builds the same per job)
  auto* cls = reinterpret_cast<cordum_response_class*>(h + at_cls);
  uint32_t* roff = h + at_roff;
  uint32_t* ioff = h + at_ioff;
  std::string text, r;
  roff[0] = 0;
  {
    std::lock_guard<std::mutex> g(e->host->mutex());
    for (size_t c = 0; c < m; ++c) {
      cordum_response_class& k = cls[c];
      if (mcp_reason(k.reason_code) && b->epoch != e->host->epoch()) {
        g_err = "tables were reloaded after the batch was encoded, and a response quotes an MCP value of the dictionaries it "
                "was encoded against: encode and dispatch it again";
        return CORDUM_E_STALE;
      }
      // kernel.go:198-215: allow and allow_with_constraints drop the reason, except the approval bypass's (engine.go:500)
      const bool allow = k.decision == CORDUM_DEC_ALLOW || k.decision == CORDUM_DEC_ALLOW_WITH_CONSTRAINTS;
      if ((k.reason_code != CORDUM_REASON_NONE && !allow) || k.reason_code == CORDUM_REASON_APPROVAL_GRANTED) {
        render_reason(e, b, k.reason_code, k.rule_idx, k.arg, flavor, nullptr, k.first_job, r);
        if (mcp_reason(k.reason_code)) k.flags |= CORDUM_CLASS_QUOTES_VALUE;
        text += r;
      }
      roff[c + 1] = (uint32_t)text.size();
    }
    ioff[0] = (uint32_t)text.size();
    for (size_t c = 0; c < m; ++c) {
      const cordum_response_class& k = cls[c];
      if ((k.flags & CORDUM_F_HAS_SNAPSHOT) && b->text && k.rule_idx >= 0 && (size_t)k.rule_idx < b->text->rules.size())
        text += b->text->rules[k.rule_idx].id;
      ioff[c + 1] = (uint32_t)text.size();
    }
  }
  for (size_t c = 0; c <= m; ++c) ioff[c] -= roff[m];   // rule id offsets relative to their own arena
  if (!pinned_reserve(b->h_resp_text, b->h_resp_text_cap, text.size() + 1)) {
    g_err = "out of memory for the response text of " + std::to_string(m) + " classes";
    return CORDUM_E_CAPACITY;
  }
  std::memcpy(b->h_resp_text, text.data(), text.size());
  out->n_classes = (uint32_t)m;
  out->classes = cls;
  out->offsets = h + at_off;
  out->jobs = h + at_jobs;
  out->reason_off = roff;
  out->reason_bytes = b->h_resp_text;
  out->rule_id_off = ioff;
  out->rule_id_bytes = b->h_resp_text + roff[m];
  return CORDUM_OK;
}

// A new pinned + device pair of `bytes` each, for a subset's wide rows or selective list; both null when it does not fit.
struct NewPair {
  void *h = nullptr, *d = nullptr;
  bool alloc(size_t bytes) {
    if (cudaHostAlloc(&h, bytes, cudaHostAllocDefault) == cudaSuccess && cudaMalloc(&d, bytes) == cudaSuccess) return true;
    cudaGetLastError();   // an allocation that does not fit is this call's problem, not a sticky engine failure
    release();
    return false;
  }
  void release() {
    if (h) cudaFreeHost(h);
    if (d) cudaFree(d);
    h = d = nullptr;
  }
};

// cordum_batch_subset once the arguments and both batches' states have been checked.  Scratch of dst (32-bit words):
// jloc [n] | sloc [n] | eloc [2 n_sel] | jcnt, scnt [tiles] | ecnt, wcnt [sel tiles] | totals [4] | list [n_list].
int subset_batch(cordum_engine* e, cordum_batch* src, uint32_t mask, const uint32_t* jobs, uint32_t n_list, cordum_batch* dst, uint32_t* n_out) {
  SubsetParams P{};
  const uint32_t n = src->n, n_sel = src->n_sel_jobs, T = CORDUM_SUBSET_TILE;
  P.n = n;
  P.n_sel = n_sel;
  P.n_tiles = (uint32_t)(((uint64_t)n + T - 1) / T);
  P.n_sel_tiles = (uint32_t)(((uint64_t)n_sel + T - 1) / T);
  P.out = jobs ? nullptr : reinterpret_cast<const uint4*>(src->d_out);
  P.mask = mask;
  P.n_list = n_list;
  JobRecords R;
  device_records(src, R);
  P.job = R.job; P.route = R.route; P.wide = R.wide; P.ww = src->wide_words;
  P.sel_jobs = R.sel_jobs; P.sel_extra = R.sel_extra;
  const size_t words = 2 * (size_t)n + 2 * (size_t)n_sel + 2 * (size_t)P.n_tiles + 2 * (size_t)P.n_sel_tiles + 4 + n_list;
  const size_t idx_bytes = 2 * (size_t)dst->max_jobs * 4;
  cudaError_t ae = dst->d_subset.reserve((words + words / 4) * 4);
  if (ae == cudaSuccess) ae = dst->d_sub_idx.reserve(idx_bytes);
  if (ae == cudaSuccess && !dst->h_parent) {
    ae = cudaHostAlloc((void**)&dst->h_parent, (size_t)dst->max_jobs * 4, cudaHostAllocDefault);
    if (ae != cudaSuccess) dst->h_parent = nullptr;   // allocated here: nothing of an earlier subset is lost
  }
  if (ae != cudaSuccess) {
    cudaGetLastError();
    g_err = "out of memory for the scratch of a subset of " + std::to_string(n) + " jobs";
    return CORDUM_E_CAPACITY;
  }
  uint32_t* w = (uint32_t*)dst->d_subset.p;
  P.jloc = w; P.sloc = w + n;
  P.eloc = reinterpret_cast<uint2*>(w + 2 * (size_t)n);
  P.jcnt = w + 2 * (size_t)n + 2 * (size_t)n_sel; P.scnt = P.jcnt + P.n_tiles;
  P.ecnt = P.scnt + P.n_tiles; P.wcnt = P.ecnt + P.n_sel_tiles;
  P.totals = P.wcnt + P.n_sel_tiles;
  cudaStream_t s = dst->stream;
  if (jobs) {
    uint32_t* list = P.totals + 4;
    if (n_list) CK(cudaMemcpyAsync(list, jobs, (size_t)n_list * 4, cudaMemcpyHostToDevice, s), "H2D subset list");
    P.list = list;
  }
  // count: how many jobs, slots, selective entries and extra words the subset keeps
  uint32_t totals[4] = {0, 0, 0, 0};
  if (n) {
    CK(launch_subset_count(P, s), "subset count kernels");
    e->launches += subset_count_launches(P);
    CK(cudaMemcpyAsync(totals, P.totals, sizeof totals, cudaMemcpyDeviceToHost, s), "D2H subset totals");
  }
  CK(cudaStreamSynchronize(s), "subset count");
  const uint32_t m = totals[0];
  if (totals[1] != m) { g_err = "the source batch's records do not index its jobs one to one"; return CORDUM_E_STATE; }
  if (m > dst->max_jobs) {
    g_err = "the subset has " + std::to_string(m) + " jobs, more than the destination batch holds (" + std::to_string(dst->max_jobs) + ")";
    return CORDUM_E_CAPACITY;
  }
  // check capacity, then gather
  P.m_sel = totals[2];
  const uint64_t wide_need = (uint64_t)m * P.ww, sel_need = P.m_sel ? 2ull * P.m_sel + 1 + totals[3] : 0;
  if (wide_need > dst->wide_cap || sel_need > dst->sel_cap) {
    // Grown with the encoders' headroom (rows for m + m/4 jobs, at least 1,024; list words + words/4, at least 1,024).
    // Both new pairs are allocated before either old one is released, so a refusal leaves dst as it was.
    const uint64_t wide_want = wide_need > dst->wide_cap ? P.ww * std::min<uint64_t>(dst->max_jobs, std::max<uint64_t>(1024, (uint64_t)m + m / 4)) : 0;
    const uint64_t sel_want = sel_need > dst->sel_cap ? std::max<uint64_t>(sel_need + sel_need / 4, 1024) : 0;
    std::lock_guard<std::mutex> g(e->mu);
    NewPair nw, ns;
    if ((wide_want && !nw.alloc(wide_want * 8)) || (sel_want && !ns.alloc(sel_want * 4))) {
      nw.release();
      ns.release();
      g_err = "out of memory for the wide-mask rows or the selective list of a subset of " + std::to_string(m) + " jobs";
      return CORDUM_E_CAPACITY;
    }
    if (wide_want) {
      if (dst->h_wide) cudaFreeHost(dst->h_wide);
      if (dst->d_wide) cudaFree(dst->d_wide);
      dst->h_wide = (uint64_t*)nw.h; dst->d_wide = (uint64_t*)nw.d; dst->wide_cap = wide_want;
    }
    if (sel_want) {
      if (dst->h_sel) cudaFreeHost(dst->h_sel);
      if (dst->d_sel) cudaFree(dst->d_sel);
      dst->h_sel = (uint32_t*)ns.h; dst->d_sel = (uint32_t*)ns.d; dst->sel_cap = sel_want;
    }
    e->tables_gen++;   // captured tick graphs bake the batch's pointers in
  }
  P.djob = (JobRec*)dst->d_cols;
  P.droute = (RouteRec*)(dst->d_cols + (size_t)m * sizeof(JobRec));
  P.dwide = dst->d_wide;
  P.dsel = dst->d_sel;
  P.dslot_of = (uint32_t*)dst->d_sub_idx.p;
  P.dparent = P.dslot_of + dst->max_jobs;
  CK(launch_subset_gather(P, s), "subset gather kernel");
  e->launches += subset_launches(P) - subset_count_launches(P);
  if (m) CK(cudaMemcpyAsync(dst->h_parent, P.dparent, (size_t)m * 4, cudaMemcpyDeviceToHost, s), "D2H parent index");
  CK(cudaStreamSynchronize(s), "subset gather");
  dst->n = m;
  dst->epoch = src->epoch;
  dst->wide_words = P.ww;
  dst->n_sel_jobs = P.m_sel;
  dst->sel_words = (uint32_t)sel_need;
  dst->d_slot_of = P.dslot_of;
  dst->env = nullptr;
  if (dst->h_fallback) *dst->h_fallback = 0;   // records produced here never go back to the host encoder
  dst->encoded = dst->resident = dst->device_encoded = true;
  dst->host_records_valid = false;
  dst->results_ready = false;
  dst->is_subset = true;
  *n_out = m;
  return CORDUM_OK;
}

// cordum_batch_merge once the arguments, the three batches' states and dst's job capacity have been checked.  Scratch of
// dst (32-bit words): key a [n_a] | key b [n_b] | wloc a [n_sel_a] | wloc b [n_sel_b] | wcnt a, wcnt b [sel tiles] | totals [2].
int merge_batch(cordum_engine* e, cordum_batch* a, cordum_batch* b, cordum_batch* dst) {
  MergeParams P{};
  const uint32_t T = CORDUM_SUBSET_TILE, m = a->n + b->n;
  if (a->n && b->n && a->wide_words != b->wide_words) {
    g_err = "the two batches' records have different wide-mask widths: encode them again";
    return CORDUM_E_STALE;
  }
  P.ww = a->n ? a->wide_words : b->n ? b->wide_words : 0u;   // an empty source imposes no width
  size_t words = 2, extra = 0;
  cordum_batch* src[2] = {a, b};
  for (int k = 0; k < 2; ++k) {
    MergeSource& S = P.s[k];
    JobRecords R;
    device_records(src[k], R);
    S.job = R.job; S.route = R.route; S.wide = R.wide; S.sel_jobs = R.sel_jobs; S.sel_extra = R.sel_extra;
    S.n = src[k]->n;
    S.n_sel = R.n_sel_jobs;
    S.n_tiles = (uint32_t)(((uint64_t)S.n + T - 1) / T);
    S.n_sel_tiles = (uint32_t)(((uint64_t)S.n_sel + T - 1) / T);
    words += (size_t)S.n + S.n_sel + S.n_sel_tiles;
    // the source's extra words, without its leading 0 word (host encoder layout: sel_words = 2 n_sel + 1 + extra)
    if (S.n_sel) extra += src[k]->sel_words - 2 * (size_t)S.n_sel - 1;
  }
  P.m_sel = P.s[0].n_sel + P.s[1].n_sel;
  const uint64_t wide_need = (uint64_t)m * P.ww, sel_need = P.m_sel ? 2ull * P.m_sel + 1 + extra : 0;
  cudaError_t ae = dst->d_subset.reserve((words + words / 4) * 4);
  if (ae == cudaSuccess) ae = dst->d_sub_idx.reserve(2 * (size_t)dst->max_jobs * 4);   // the subset's size: neither call reallocates it
  if (ae != cudaSuccess) {
    cudaGetLastError();
    g_err = "out of memory for the scratch of a merge of " + std::to_string(m) + " jobs";
    return CORDUM_E_CAPACITY;
  }
  uint32_t* w = (uint32_t*)dst->d_subset.p;
  P.s[0].key = w; P.s[1].key = w + P.s[0].n;
  P.s[0].wloc = P.s[1].key + P.s[1].n; P.s[1].wloc = P.s[0].wloc + P.s[0].n_sel;
  P.s[0].wcnt = P.s[1].wloc + P.s[1].n_sel; P.s[1].wcnt = P.s[0].wcnt + P.s[0].n_sel_tiles;
  P.totals = P.s[1].wcnt + P.s[1].n_sel_tiles;
  cudaStream_t s = dst->stream;
  {
    // e->mu: a dictionary upload on another thread must not replace the tenant-class table between here and the launch
    std::lock_guard<std::mutex> g(e->mu);
    std::lock_guard<std::mutex> gh(e->host->mutex());
    if (a->epoch != e->host->epoch() || b->epoch != e->host->epoch()) {
      g_err = "tables were reloaded after a source batch was encoded: encode again";
      return CORDUM_E_STALE;
    }
    if (m) {
      int rc = sync_dicts(e);   // the tenant classes of the sources' epoch, also on an engine that never encoded on the device
      if (rc) return rc;
      P.tenant_class = e->et.tenant_class;
      P.tenant_classes = e->et.tenant_classes;
    }
    if (wide_need > dst->wide_cap || sel_need > dst->sel_cap) {
      // Grown with the encoders' headroom, as for a subset; both new pairs are allocated before either old one is released,
      // so a refusal leaves dst as it was.
      const uint64_t wide_want = wide_need > dst->wide_cap ? P.ww * std::min<uint64_t>(dst->max_jobs, std::max<uint64_t>(1024, (uint64_t)m + m / 4)) : 0;
      const uint64_t sel_want = sel_need > dst->sel_cap ? std::max<uint64_t>(sel_need + sel_need / 4, 1024) : 0;
      NewPair nw, ns;
      if ((wide_want && !nw.alloc(wide_want * 8)) || (sel_want && !ns.alloc(sel_want * 4))) {
        nw.release();
        ns.release();
        g_err = "out of memory for the wide-mask rows or the selective list of a merge of " + std::to_string(m) + " jobs";
        return CORDUM_E_CAPACITY;
      }
      if (wide_want) {
        if (dst->h_wide) cudaFreeHost(dst->h_wide);
        if (dst->d_wide) cudaFree(dst->d_wide);
        dst->h_wide = (uint64_t*)nw.h; dst->d_wide = (uint64_t*)nw.d; dst->wide_cap = wide_want;
      }
      if (sel_want) {
        if (dst->h_sel) cudaFreeHost(dst->h_sel);
        if (dst->d_sel) cudaFree(dst->d_sel);
        dst->h_sel = (uint32_t*)ns.h; dst->d_sel = (uint32_t*)ns.d; dst->sel_cap = sel_want;
      }
      e->tables_gen++;   // captured tick graphs bake the batch's pointers in
    }
    P.djob = (JobRec*)dst->d_cols;
    P.droute = (RouteRec*)(dst->d_cols + (size_t)m * sizeof(JobRec));
    P.dwide = dst->d_wide;
    P.dsel = dst->d_sel;
    P.dslot_of = (uint32_t*)dst->d_sub_idx.p;
    CK(launch_merge(P, s), "merge kernels");
    e->launches += merge_launches(P);
  }
  CK(cudaStreamSynchronize(s), "merge");
  dst->n = m;
  dst->epoch = a->epoch;
  dst->wide_words = P.ww;
  dst->n_sel_jobs = P.m_sel;
  dst->sel_words = (uint32_t)sel_need;
  dst->d_slot_of = P.dslot_of;
  dst->env = nullptr;
  if (dst->h_fallback) *dst->h_fallback = 0;   // records produced here never go back to the host encoder
  dst->encoded = dst->resident = dst->device_encoded = true;
  dst->host_records_valid = false;
  dst->results_ready = false;
  dst->is_subset = false;
  return CORDUM_OK;
}
}  // namespace

// ============================================================ C ABI
extern "C" {

const char* cordum_last_error(void) { return g_err.c_str(); }
const char* cordum_version(void) { return "cordum-b200 0.1 (sm_90a)"; }

int32_t cordum_engine_create(const cordum_engine_opts* opts, cordum_engine** out) {
  if (!out) { g_err = "null out"; return CORDUM_E_INVALID; }
  *out = nullptr;
  int count = 0;
  cudaError_t ce = cudaGetDeviceCount(&count);
  if (ce != cudaSuccess || count == 0) {
    g_err = std::string("no CUDA device (") + (ce == cudaSuccess ? "count 0" : cudaGetErrorString(ce)) +
            "): cordum-b200 has no CPU evaluation path";
    return CORDUM_E_NODEVICE;
  }
  auto e = std::make_unique<cordum_engine>();
  e->device = opts ? opts->device : 0;
  if (e->device < 0 || e->device >= count) { g_err = "bad device ordinal"; return CORDUM_E_INVALID; }
  cordum_engine* ep = e.get();
  {
    cordum_engine* e = ep;
    CK(cudaSetDevice(e->device), "cudaSetDevice");
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, e->device), "device properties");
    e->sm_count = prop.multiProcessorCount;
    {
      // the worker-table refresh is the head of every step's dependency chain (route kernels wait for it): its CTAs go
      // ahead of queued policy / route CTAs
      int lo = 0, hi = 0;
      CK(cudaDeviceGetStreamPriorityRange(&lo, &hi), "priority range");
      CK(cudaStreamCreateWithPriority(&e->s_tables, cudaStreamNonBlocking, hi), "stream");
      CK(cudaStreamCreateWithPriority(&e->s_copy, cudaStreamNonBlocking, hi), "stream");
      CK(cudaStreamCreateWithPriority(&e->s_xchg, cudaStreamNonBlocking, hi), "stream");
      for (auto& ev : e->gather_free) {
        CK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming), "event");
        CK(cudaEventRecord(ev, e->s_xchg), "event");
      }
      CK(cudaEventCreateWithFlags(&e->ev_xchg, cudaEventDisableTiming), "event");
    }
    for (auto& D : e->ds) {
      CK(cudaEventCreateWithFlags(&D.ready, cudaEventDisableTiming), "event");
      CK(cudaEventRecord(D.ready, e->s_tables), "event");
      CK(cudaEventCreateWithFlags(&D.loads_read, cudaEventDisableTiming), "event");
      CK(cudaEventRecord(D.loads_read, e->s_tables), "event");
    }
    CK(cudaEventCreateWithFlags(&e->ev_copy, cudaEventDisableTiming), "event");
    CK(cudaEventCreateWithFlags(&e->ev_prod, cudaEventDisableTiming), "event");
  }
  e->host = std::make_unique<Host>(opts ? opts->max_topics : 0, opts ? opts->max_effcfgs : 0, opts ? opts->encode_threads : 0);
  *out = e.release();
  return CORDUM_OK;
}

void cordum_engine_destroy(cordum_engine* e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  {
    std::vector<cordum_batch*> live;
    { std::lock_guard<std::mutex> g(e->mu); live.swap(e->batches); }
    for (cordum_batch* b : live) batch_release(b);
  }
  for (auto& kv : e->ing_graphs) cudaGraphExecDestroy(kv.second);
  for (auto& p : e->stage) if (p) cudaFreeHost(p);
  for (auto& kv : e->tick.graphs) cudaGraphExecDestroy(kv.second);
  for (cudaStream_t st : {e->tick.s[0], e->tick.s[1], e->tick.sa, e->tick.sc}) if (st) cudaStreamDestroy(st);
  for (cudaEvent_t ev : {e->tick.ev_fork, e->tick.ev_a, e->tick.ev_c, e->tick.ev_join, e->tick.done[0], e->tick.done[1], e->tick.refreshed[0], e->tick.refreshed[1]}) if (ev) cudaEventDestroy(ev);
  for (int q = 0; q < e->peers.world && e->peers.ready; ++q) if (q != e->peers.rank && e->peers.base[q]) cudaIpcCloseMemHandle(e->peers.base[q]);
  if (e->peers.mine) cudaFree(e->peers.mine);
  for (cordum_envelopes* env : e->env_sets) cudaFreeHost(env);
  e->env_sets.clear();
  for (auto& D : e->ds) {
    if (D.ready) cudaEventDestroy(D.ready);
    if (D.loads_read) cudaEventDestroy(D.loads_read);
  }
  if (e->ev_copy) cudaEventDestroy(e->ev_copy);
  if (e->ev_prod) cudaEventDestroy(e->ev_prod);
  if (e->s_tables) cudaStreamDestroy(e->s_tables);
  if (e->s_copy) cudaStreamDestroy(e->s_copy);
  if (e->nccl_comm && nccl_api()) nccl_api()->CommDestroy(e->nccl_comm);
  for (auto& ev : e->gather_free) if (ev) cudaEventDestroy(ev);
  if (e->ev_xchg) cudaEventDestroy(e->ev_xchg);
  if (e->s_xchg) cudaStreamDestroy(e->s_xchg);
  delete e;
}

int32_t cordum_policy_load(cordum_engine* e, const char* json, uint64_t len, const char* snapshot, uint64_t slen) {
  cordum::NvtxRange nvtx_("cordum:policy_load");
  if (!e) { g_err = "null engine"; return CORDUM_E_INVALID; }
  return e->host->load_policy(sv(json ? json : "", json ? len : 0), sv(snapshot ? snapshot : "", snapshot ? slen : 0), g_err);
}

int32_t cordum_policy_snapshots(cordum_engine* e, char* buf, uint64_t cap, uint32_t* n_out) {
  if (!e) { g_err = "null engine"; return CORDUM_E_INVALID; }
  std::lock_guard<std::mutex> g(e->host->mutex());
  uint64_t off = 0;
  uint32_t n = 0;
  for (auto& s : e->host->snapshots()) {
    if (off + s.size() + 1 > cap) break;
    std::memcpy(buf + off, s.data(), s.size());
    buf[off + s.size()] = 0;
    off += s.size() + 1;
    ++n;
  }
  if (n_out) *n_out = n;
  return CORDUM_OK;
}

/* PolicyCheckResponse.PolicySnapshot = the snapshot of the policy in force (kernel.go:243), which is "" when that policy
 * was loaded without one - not the newest entry of the history */
int64_t cordum_policy_snapshot(cordum_engine* e, char* buf, uint64_t cap) {
  if (!e) return -1;
  std::lock_guard<std::mutex> g(e->host->mutex());
  return copy_out(e->host->current_snapshot(), buf, cap);
}

/* ...and the one a given batch was dispatched under: a reload that lands after the dispatch does not relabel decisions
 * that were taken under the previous policy (kernel.go:140-147 reads policy and snapshot under one lock) */
int64_t cordum_batch_snapshot(const cordum_batch* b, char* buf, uint64_t cap) {
  if (!b) return -1;
  return copy_out(b->text ? b->text->snapshot : std::string(), buf, cap);
}
uint64_t cordum_batch_policy_gen(const cordum_batch* b) { return (b && b->text) ? b->text->gen : 0; }
uint64_t cordum_policy_generation(cordum_engine* e) { return e ? e->host->policy_generation() : 0; }

int32_t cordum_routing_load(cordum_engine* e, const char* json, uint64_t len) {
  if (!e) { g_err = "null engine"; return CORDUM_E_INVALID; }
  return e->host->load_routing(sv(json ? json : "", json ? len : 0), g_err);
}

int32_t cordum_workers_load(cordum_engine* e, const cordum_workers* w) {
  cordum::NvtxRange nvtx_("cordum:workers_load");
  if (!e) { g_err = "null engine"; return CORDUM_E_INVALID; }
  return e->host->load_workers(w, g_err);
}

int32_t cordum_workers_update(cordum_engine* e, uint32_t n, const uint32_t* slots, const cordum_worker_load* loads) {
  if (!e || (n && (!slots || !loads))) { g_err = "null argument"; return CORDUM_E_INVALID; }
  int rc = e->host->update_loads(n, slots, loads, g_err);
  return rc;
}

int32_t cordum_workers_set_loads_device(cordum_engine* e, const void* dptr, uint32_t n_workers, void* stream) {
  if (!e || !dptr) { g_err = "null argument"; return CORDUM_E_INVALID; }
  if (e->failed) { g_err = "engine failed earlier: " + e->fail_msg; return CORDUM_E_CUDA; }
  if (int rc = leave_tick_mode(e)) return rc;
  std::lock_guard<std::mutex> g(e->mu);
  std::lock_guard<std::mutex> gh(e->host->mutex());
  if (n_workers != e->host->tables().n_slots) { g_err = "load table size does not match the worker registry"; return CORDUM_E_INVALID; }
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  int rc = sync_tables(e);
  if (rc) return rc;
  return refresh_pools(e, dptr, (cudaStream_t)stream);
}

int32_t cordum_exchange_unique_id(char id[CORDUM_EXCHANGE_ID_BYTES]) {
  if (!id) { g_err = "null argument"; return CORDUM_E_INVALID; }
  NcclApi* a = nccl_api();
  if (!a) { g_err = "libnccl not found (set CORDUM_NCCL_LIB)"; return CORDUM_E_STATE; }
  NcclId u;
  int rc = a->GetUniqueId(&u);
  if (rc) return nccl_fail(nullptr, rc, "ncclGetUniqueId");
  std::memcpy(id, u.internal, CORDUM_EXCHANGE_ID_BYTES);
  return CORDUM_OK;
}

int32_t cordum_exchange_init(cordum_engine* e, const char id[CORDUM_EXCHANGE_ID_BYTES], int32_t rank, int32_t world) {
  if (!e || !id || world < 1 || rank < 0 || rank >= world) { g_err = "bad argument"; return CORDUM_E_INVALID; }
  if (e->failed) { g_err = "engine failed earlier: " + e->fail_msg; return CORDUM_E_CUDA; }
  std::lock_guard<std::mutex> g(e->mu);
  if (e->nccl_comm) { g_err = "exchange already initialised"; return CORDUM_E_STATE; }
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  if (world > 1) {
    NcclApi* a = nccl_api();
    if (!a) { g_err = "libnccl not found (set CORDUM_NCCL_LIB)"; return CORDUM_E_STATE; }
    NcclId u;
    std::memcpy(u.internal, id, CORDUM_EXCHANGE_ID_BYTES);
    void* comm = nullptr;
    int rc = a->CommInitRank(&comm, world, u, rank);
    if (rc) return nccl_fail(e, rc, "ncclCommInitRank");
    e->nccl_comm = comm;
  }
  e->xrank = rank; e->xworld = world;
  e->tables_gen++;   // view() depends on the world size (label-best table on / off): captured graphs are stale
  return CORDUM_OK;
}

int32_t cordum_workers_ingest(cordum_engine* e, const cordum_worker_load* slice, uint32_t first_slot, uint32_t n_slice) {
  cordum::NvtxRange nvtx_("cordum:heartbeat_ingest");
  if (!e || !slice) { g_err = "null argument"; return CORDUM_E_INVALID; }
  if (e->failed) { g_err = "engine failed earlier: " + e->fail_msg; return CORDUM_E_CUDA; }
  if (int rc = leave_tick_mode(e)) return rc;
  std::lock_guard<std::mutex> g(e->mu);
  std::lock_guard<std::mutex> gh(e->host->mutex());
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  int rc = sync_tables(e);
  if (rc) return rc;
  return ingest(e, slice, first_slot, n_slice);
}

int32_t cordum_peer_export(cordum_engine* e, int32_t rank, int32_t world, char handle[CORDUM_PEER_HANDLE_BYTES]) {
  if (!e || !handle || world < 1 || world > CORDUM_MAX_PEERS || rank < 0 || rank >= world) { g_err = "bad argument"; return CORDUM_E_INVALID; }
  std::lock_guard<std::mutex> g(e->mu);
  std::lock_guard<std::mutex> gh(e->host->mutex());
  const uint32_t W = e->host->tables().n_slots;
  if (W == 0 || W % (uint32_t)world) { g_err = "worker registry size is not a multiple of the world size"; return CORDUM_E_INVALID; }
  if (e->peers.mine) { g_err = "peer exchange already exported"; return CORDUM_E_STATE; }
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  auto& P = e->peers;
  P.rank = rank; P.world = world; P.per = W / (uint32_t)world;
  P.bytes = 256 + 2 * (size_t)W * sizeof(Load16);
  CK(cudaMalloc((void**)&P.mine, P.bytes), "peer exchange buffer");
  CK(cudaMemset(P.mine, 0, P.bytes), "peer exchange buffer");
  cudaIpcMemHandle_t h;
  CK(cudaIpcGetMemHandle(&h, P.mine), "cudaIpcGetMemHandle");
  static_assert(sizeof h <= CORDUM_PEER_HANDLE_BYTES, "handle size");
  std::memset(handle, 0, CORDUM_PEER_HANDLE_BYTES);
  std::memcpy(handle, &h, sizeof h);
  return CORDUM_OK;
}

int32_t cordum_peer_import(cordum_engine* e, const char* handles) {
  if (!e || !handles) { g_err = "null argument"; return CORDUM_E_INVALID; }
  std::lock_guard<std::mutex> g(e->mu);
  auto& P = e->peers;
  if (!P.mine) { g_err = "cordum_peer_export first"; return CORDUM_E_STATE; }
  if (P.ready) { g_err = "peers already imported"; return CORDUM_E_STATE; }
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  for (int q = 0; q < P.world; ++q) {
    if (q == P.rank) { P.base[q] = P.mine; continue; }
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handles + (size_t)q * CORDUM_PEER_HANDLE_BYTES, sizeof h);
    void* p = nullptr;
    CK(cudaIpcOpenMemHandle(&p, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle");
    P.base[q] = (uint8_t*)p;
  }
  P.ready = true;
  if (!e->nccl_comm) { e->xrank = P.rank; e->xworld = P.world; }   // cordum_workers_ingest uses the peer exchange too
  e->tables_gen++;
  return CORDUM_OK;
}

int32_t cordum_tick_async(cordum_engine* e, cordum_batch* b, uint32_t mode, const cordum_worker_load* slice, uint32_t first_slot,
                          uint32_t n_slice) {
  if (!e || !b || !slice) { g_err = "null argument"; return CORDUM_E_INVALID; }
  if (e->failed) { g_err = "engine failed earlier: " + e->fail_msg; return CORDUM_E_CUDA; }
  if ((mode & 0xFFu) != CORDUM_MODE_POLICY_AND_ROUTE) { g_err = "a tick evaluates policy and routes (CORDUM_MODE_POLICY_AND_ROUTE)"; return CORDUM_E_INVALID; }
  if (!b->encoded || !b->resident) { g_err = "the batch must be encoded and resident on the device (dispatch it once, or cordum_encode_device)"; return CORDUM_E_STATE; }
  // Work of this batch on its own stream (an encode, a plain dispatch) is waited for on the host.  An earlier TICK of the
  // same batch needs no host wait unless it was the previous tick (its route and this policy would share a graph): the
  // device-side order covers every older tick (tick_locked).
  if (b->pending || b->enc_inflight || (b->tick_pending && e->tick.n - b->tick_no < 2)) { int rc = wait(b); if (rc) return rc; }
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  std::lock_guard<std::mutex> g(e->mu);
  std::lock_guard<std::mutex> gh(e->host->mutex());
  if (b->epoch != e->host->epoch()) { g_err = "tables were reloaded after this batch was encoded: encode again"; return CORDUM_E_STALE; }
  b->text = e->host->policy_text(); b->wtext = e->host->worker_text(); b->ttext = e->host->topic_text();
  b->results_ready = false;
  const uint32_t W = e->host->tables().n_slots;
  if (e->peers.ready && e->peers.world > 1) {
    if (first_slot != (uint32_t)e->peers.rank * e->peers.per || n_slice != e->peers.per || e->peers.per * (uint32_t)e->peers.world != W) {
      g_err = "slice is not this rank's share of the worker registry"; return CORDUM_E_INVALID;
    }
  } else if (first_slot != 0 || n_slice != W) { g_err = "without a peer exchange the slice must be the whole worker table"; return CORDUM_E_INVALID; }
  if (!e->tick.active) CK(cudaDeviceSynchronize(), "enter tick mode");   // plain dispatches in flight read / write the same table sets
  int rc = sync_tables(e);
  if (rc) return rc;
  rc = tick_setup(e);
  if (rc) return rc;
  rc = tick_locked(e, b, slice, n_slice);
  if (rc) return rc;
  b->tick_pending = true;
  b->last_mode = CORDUM_MODE_POLICY_AND_ROUTE;
  return CORDUM_OK;
}

/* The cudaStream_t all ticks are launched on, so a harness can bracket them with its own CUDA events. */
void* cordum_tick_stream(cordum_engine* e) {
  if (!e) return nullptr;
  std::lock_guard<std::mutex> g(e->mu);
  if (cudaSetDevice(e->device) != cudaSuccess || tick_setup(e) != CORDUM_OK) return nullptr;
  return (void*)e->tick.s[0];
}

int32_t cordum_tick_flush(cordum_engine* e) {
  if (!e) { g_err = "null engine"; return CORDUM_E_INVALID; }
  if (!e->tick.s[0]) return CORDUM_OK;
  std::lock_guard<std::mutex> g(e->mu);
  std::lock_guard<std::mutex> gh(e->host->mutex());
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  return tick_flush_locked(e);
}

int32_t cordum_batch_alloc(cordum_engine* e, uint32_t max_jobs, cordum_batch** out) {
  if (!e || !out || max_jobs == 0) { g_err = "bad argument"; return CORDUM_E_INVALID; }
  *out = nullptr;
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  auto b = std::make_unique<cordum_batch>();
  b->e = e;
  b->max_jobs = max_jobs;
  size_t bytes = slab_bytes(max_jobs);
  CK(cudaHostAlloc((void**)&b->h_cols, bytes, cudaHostAllocDefault), "pinned columns");
  CK(cudaMalloc((void**)&b->d_cols, bytes), "device columns");
  CK(cudaHostAlloc((void**)&b->h_out, (size_t)max_jobs * sizeof(cordum_decision), cudaHostAllocDefault), "pinned results");
  CK(cudaMalloc((void**)&b->d_out, (size_t)max_jobs * sizeof(cordum_decision)), "device results");
  CK(cudaMalloc((void**)&b->d_route, ((size_t)max_jobs + 2) * sizeof(uint2)), "device route list");
  b->slot_of = (uint32_t*)std::malloc((size_t)max_jobs * sizeof(uint32_t));
  if (!b->slot_of) { g_err = "out of host memory"; return CORDUM_E_INVALID; }
  CK(cudaStreamCreateWithFlags(&b->stream, cudaStreamNonBlocking), "stream");
  CK(cudaEventCreate(&b->ev0), "event"); CK(cudaEventCreate(&b->ev1), "event"); CK(cudaEventCreate(&b->evm), "event");
  CK(cudaEventCreate(&b->ev2), "event"); CK(cudaEventCreate(&b->ev3), "event");
  { std::lock_guard<std::mutex> g(e->mu); e->batches.push_back(b.get()); }
  *out = b.release();
  return CORDUM_OK;
}

/* A batch must be freed BEFORE its engine is destroyed; cordum_engine_destroy releases any batch
 * that is still alive, after which those handles are invalid. */
void cordum_batch_free(cordum_batch* b) {
  if (!b) return;
  cudaSetDevice(b->e->device);
  {
    std::lock_guard<std::mutex> g(b->e->mu);
    auto& v = b->e->batches;
    for (size_t i = 0; i < v.size(); ++i) if (v[i] == b) { v.erase(v.begin() + i); break; }
  }
  batch_release(b);
}

int32_t cordum_encode(cordum_engine* e, cordum_batch* b, const cordum_envelopes* env) {
  if (!e || !b || !env) { g_err = "null argument"; return CORDUM_E_INVALID; }
  if (env->n_jobs > b->max_jobs) { g_err = "batch too small for these envelopes"; return CORDUM_E_INVALID; }
  if (b->pending || b->enc_inflight || b->tick_pending) { int rc = wait(b); if (rc) return rc; }
  return host_encode_into(e, b, env);
}

/* ---- device-side encode ---------------------------------------------------------------------------------------- */
namespace {
struct EnvLayout { size_t off[15]; size_t total; };   // arena + the 14 arrays, 256 B aligned, in cordum_envelopes order
EnvLayout env_layout(uint32_t n, uint64_t arena, uint32_t n_risk, uint32_t n_req, uint32_t n_lab) {
  const size_t sz[15] = {(size_t)arena + 16, (size_t)n * 8, (size_t)n * 8, (size_t)n * 8, (size_t)n * 8, (size_t)n, (size_t)n * 8, (size_t)n * 8,
                         (size_t)n, (size_t)n * 8, (size_t)n * 8, ((size_t)n + 1) * 4 + 16 + (size_t)n_risk * 8, ((size_t)n + 1) * 4 + 16 + (size_t)n_req * 8,
                         ((size_t)n + 1) * 4 + 16 + (size_t)n_lab * 16, (size_t)n};
  EnvLayout L{};
  size_t at = 0;
  for (int i = 0; i < 15; ++i) { L.off[i] = at; at += (sz[i] + 255) & ~size_t(255); }
  L.total = at;
  return L;
}
}  // namespace

int32_t cordum_envelopes_alloc(cordum_engine* e, const cordum_envelope_caps* caps, cordum_envelopes** out) {
  if (!e || !caps || !out || caps->max_jobs == 0) { g_err = "bad argument"; return CORDUM_E_INVALID; }
  *out = nullptr;
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  const uint32_t n = caps->max_jobs;
  const size_t sz[14] = {(size_t)caps->arena_bytes + 16, (size_t)n * 8, (size_t)n * 8, (size_t)n * 8, (size_t)n * 8, (size_t)n, (size_t)n * 8,
                         (size_t)n * 8, (size_t)n, (size_t)n * 8, (size_t)n * 8, ((size_t)n + 1) * 4, ((size_t)n + 1) * 4, ((size_t)n + 1) * 4};
  const size_t lists[4] = {(size_t)std::max<uint32_t>(caps->max_risk_tags, 1) * 8, (size_t)std::max<uint32_t>(caps->max_requires, 1) * 8,
                           (size_t)std::max<uint32_t>(caps->max_labels, 1) * 8, (size_t)std::max<uint32_t>(caps->max_labels, 1) * 8};
  size_t total = sizeof(cordum_envelopes) + 256 + n;
  for (size_t x : sz) total += (x + 255) & ~size_t(255);
  for (size_t x : lists) total += (x + 255) & ~size_t(255);
  uint8_t* base = nullptr;
  CK(cudaHostAlloc((void**)&base, total, cudaHostAllocDefault), "pinned envelope buffers");
  std::memset(base, 0, total);
  auto* env = reinterpret_cast<cordum_envelopes*>(base);
  size_t at = (sizeof(cordum_envelopes) + 255) & ~size_t(255);
  auto take = [&](size_t bytes) { uint8_t* p = base + at; at += (bytes + 255) & ~size_t(255); return p; };
  env->n_jobs = 0;
  env->arena = take(sz[0]); env->arena_len = 0;
  env->topic = (const cordum_str*)take(sz[1]); env->tenant = (const cordum_str*)take(sz[2]);
  env->principal_id = (const cordum_str*)take(sz[3]); env->effective_config = (const cordum_str*)take(sz[4]);
  env->has_meta = take(sz[5]); env->meta_tenant_id = (const cordum_str*)take(sz[6]); env->actor_id = (const cordum_str*)take(sz[7]);
  env->actor_type = take(sz[8]); env->capability = (const cordum_str*)take(sz[9]); env->pack_id = (const cordum_str*)take(sz[10]);
  env->risk_off = (const uint32_t*)take(sz[11]); env->risk_tags = (const cordum_str*)take(lists[0]);
  env->requires_off = (const uint32_t*)take(sz[12]); env->requires_ = (const cordum_str*)take(lists[1]);
  env->label_off = (const uint32_t*)take(sz[13]); env->label_keys = (const cordum_str*)take(lists[2]);
  env->label_vals = (const cordum_str*)take(lists[3]);
  env->approved = take(n);
  { std::lock_guard<std::mutex> g(e->mu); e->env_sets.push_back(env); }
  *out = env;
  return CORDUM_OK;
}

void cordum_envelopes_free(cordum_engine* e, cordum_envelopes* env) {
  if (!e || !env) return;
  cudaSetDevice(e->device);
  {
    std::lock_guard<std::mutex> g(e->mu);
    auto& v = e->env_sets;
    for (size_t i = 0; i < v.size(); ++i) if (v[i] == env) { v.erase(v.begin() + i); break; }
  }
  cudaFreeHost(env);
}

int32_t cordum_encode_device(cordum_engine* e, cordum_batch* b, const cordum_envelopes* env) {
  cordum::NvtxRange nvtx_("cordum:encode_device");
  if (!e || !b || !env) { g_err = "null argument"; return CORDUM_E_INVALID; }
  if (env->n_jobs > b->max_jobs) { g_err = "batch too small for these envelopes"; return CORDUM_E_INVALID; }
  if (e->failed) { g_err = "engine failed earlier: " + e->fail_msg; return CORDUM_E_CUDA; }
  if (b->pending || b->enc_inflight || b->tick_pending) { int rc = wait(b); if (rc) return rc; }
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  const uint32_t n = env->n_jobs;
  b->n = n;
  b->encoded = false; b->resident = false; b->device_encoded = false; b->results_ready = false; b->is_subset = false;
  b->wide_words = 0;   // a batch the device encoder completes has none (wide tables raise the fallback flag)
  b->n_sel_jobs = b->sel_words = 0;   // nor a selective list (a selective pair raises it too)
  if (n == 0) { b->encoded = true; b->resident = true; b->device_encoded = true; b->host_records_valid = true; b->epoch = e->host->epoch(); return CORDUM_OK; }
  if (!b->h_fallback) { CK(cudaHostAlloc((void**)&b->h_fallback, 64, cudaHostAllocDefault), "pinned flag"); *b->h_fallback = 0; }
  const uint32_t n_risk = env->risk_off ? env->risk_off[n] : 0, n_req = env->requires_off ? env->requires_off[n] : 0,
                 n_lab = env->label_off ? env->label_off[n] : 0;
  const EnvLayout L = env_layout(n, env->arena_len, n_risk, n_req, n_lab);
  EncodeParams P{};
  uint32_t n_keys = 0;
  {
    std::lock_guard<std::mutex> g(e->mu);
    std::lock_guard<std::mutex> gh(e->host->mutex());
    int rc = sync_tables(e);
    if (rc) return rc;
    rc = sync_dicts(e);
    if (rc) return rc;
    P.et = e->et;
    n_keys = P.et.n_topics * P.et.tenant_classes;
    b->epoch = e->host->epoch();
    // device buffers of this batch (grown on demand; nothing of this batch is in flight: it was waited for above)
    if (b->d_env.cap < L.total) CK(b->d_env.reserve(L.total + L.total / 8), "device envelope buffers");
    const size_t work = ((size_t)n * 4 + 255) / 256 * 256 * 4 + ((size_t)n_keys * 4 + 255) / 256 * 256 + 256;
    if (b->d_work.cap < work) CK(b->d_work.reserve(work + work / 8), "device encode work arrays");
  }
  cudaStream_t s = b->stream;
  uint8_t* d = (uint8_t*)b->d_env.p;
  auto h2d = [&](int i, const void* src, size_t bytes, size_t extra_off = 0) -> cudaError_t {
    if (!src || !bytes) return cudaSuccess;
    return cudaMemcpyAsync(d + L.off[i] + extra_off, src, bytes, cudaMemcpyHostToDevice, s);
  };
  CK(h2d(0, env->arena, env->arena_len), "H2D arena");
  CK(h2d(1, env->topic, (size_t)n * 8), "H2D"); CK(h2d(2, env->tenant, (size_t)n * 8), "H2D");
  CK(h2d(3, env->principal_id, (size_t)n * 8), "H2D"); CK(h2d(4, env->effective_config, (size_t)n * 8), "H2D");
  CK(h2d(5, env->has_meta, n), "H2D"); CK(h2d(6, env->meta_tenant_id, (size_t)n * 8), "H2D");
  CK(h2d(7, env->actor_id, (size_t)n * 8), "H2D"); CK(h2d(8, env->actor_type, n), "H2D");
  CK(h2d(9, env->capability, (size_t)n * 8), "H2D"); CK(h2d(10, env->pack_id, (size_t)n * 8), "H2D");
  const size_t offs_bytes = ((size_t)n + 1) * 4, offs = (offs_bytes + 15) & ~size_t(15);   // the span lists follow their offset arrays, 16 B aligned
  CK(h2d(11, env->risk_off, offs_bytes), "H2D"); CK(h2d(11, env->risk_tags, (size_t)n_risk * 8, offs), "H2D");
  CK(h2d(12, env->requires_off, offs_bytes), "H2D"); CK(h2d(12, env->requires_, (size_t)n_req * 8, offs), "H2D");
  CK(h2d(13, env->label_off, offs_bytes), "H2D"); CK(h2d(13, env->label_keys, (size_t)n_lab * 8, offs), "H2D");
  CK(h2d(13, env->label_vals, (size_t)n_lab * 8, offs + (size_t)n_lab * 8), "H2D");
  CK(h2d(14, env->approved, n), "H2D");
  P.n_jobs = n;
  P.arena = d + L.off[0];
  auto col = [&](int i, const void* src) { return src ? (const cordum_str*)(d + L.off[i]) : nullptr; };
  P.topic = col(1, env->topic); P.tenant = col(2, env->tenant); P.principal_id = col(3, env->principal_id);
  P.effective_config = col(4, env->effective_config); P.has_meta = env->has_meta ? d + L.off[5] : nullptr;
  P.meta_tenant_id = col(6, env->meta_tenant_id); P.actor_id = col(7, env->actor_id);
  P.actor_type = env->actor_type ? d + L.off[8] : nullptr; P.capability = col(9, env->capability); P.pack_id = col(10, env->pack_id);
  P.risk_off = env->risk_off ? (const uint32_t*)(d + L.off[11]) : nullptr; P.risk_tags = (const cordum_str*)(d + L.off[11] + offs);
  P.requires_off = env->requires_off ? (const uint32_t*)(d + L.off[12]) : nullptr; P.requires_ = (const cordum_str*)(d + L.off[12] + offs);
  P.label_off = env->label_off ? (const uint32_t*)(d + L.off[13]) : nullptr;
  P.label_keys = (const cordum_str*)(d + L.off[13] + offs); P.label_vals = (const cordum_str*)(d + L.off[13] + offs + (size_t)n_lab * 8);
  P.approved = env->approved ? d + L.off[14] : nullptr;
  uint8_t* w = (uint8_t*)b->d_work.p;
  const size_t arr = ((size_t)n * 4 + 255) / 256 * 256;
  P.tid = (uint32_t*)w; P.ten = (uint32_t*)(w + arr); P.key = (uint32_t*)(w + 2 * arr); P.slot_of = (uint32_t*)(w + 3 * arr);
  P.hist = (uint32_t*)(w + 4 * arr);
  P.fallback = (uint32_t*)(w + 4 * arr + ((size_t)n_keys * 4 + 255) / 256 * 256);
  P.out_job = (JobRec*)b->d_cols;
  P.out_route = (RouteRec*)(b->d_cols + (size_t)n * sizeof(JobRec));
  b->d_slot_of = P.slot_of;
  CK(launch_encode(P, n_keys, s), "encode kernels");
  e->launches += 3;
  CK(cudaMemcpyAsync(b->h_fallback, P.fallback, sizeof(uint32_t), cudaMemcpyDeviceToHost, s), "D2H fallback flag");
  b->env = env;
  b->encoded = true; b->resident = true; b->device_encoded = true; b->host_records_valid = false;
  b->enc_inflight = true;   // work is in flight on the batch stream; a dispatch simply queues behind it
  return CORDUM_OK;
}

/* host copies of the records of a device-encoded batch (cordum_reason / cordum_subject read topic and MCP ids) */
static int ensure_host_records(cordum_batch* b) {
  cordum_engine* e = b->e;
  if (b->host_records_valid) return CORDUM_OK;
  if (b->pending || b->enc_inflight || b->tick_pending) { int rc = wait(b); if (rc) return rc; }
  if (b->host_records_valid) return CORDUM_OK;   // the wait fell back to the host encoder
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  host_records(b);
  CK(cudaMemcpy(b->h_cols, b->d_cols, slab_bytes(b->n), cudaMemcpyDeviceToHost), "D2H records");
  CK(cudaMemcpy(b->slot_of, b->d_slot_of, (size_t)b->n * 4, cudaMemcpyDeviceToHost), "D2H slot_of");
  b->host_records_valid = true;
  return CORDUM_OK;
}

/* test / diagnostics: the encoded records of a batch, as (JobRec[n], RouteRec[n], slot_of[n]) in host memory */
int32_t cordum_batch_records(cordum_batch* b, void* job_out, void* route_out, uint32_t* slot_of_out) {
  if (!b) { g_err = "null batch"; return CORDUM_E_INVALID; }
  int rc = ensure_host_records(b);
  if (rc) return rc;
  if (job_out) std::memcpy(job_out, b->hr.job, (size_t)b->n * sizeof(JobRec));
  if (route_out) std::memcpy(route_out, b->hr.route, (size_t)b->n * sizeof(RouteRec));
  if (slot_of_out) std::memcpy(slot_of_out, b->slot_of, (size_t)b->n * sizeof(uint32_t));
  return CORDUM_OK;
}
uint64_t cordum_host_fallbacks(cordum_engine* e) { return e ? e->host->host_fallbacks : 0; }

int32_t cordum_dispatch_async(cordum_engine* e, cordum_batch* b, uint32_t mode) { return run(e, b, mode, true, true); }
int32_t cordum_batch_wait(cordum_batch* b) {
  if (!b) { g_err = "null batch"; return CORDUM_E_INVALID; }
  return wait(b);
}
int32_t cordum_dispatch(cordum_engine* e, cordum_batch* b, uint32_t mode) {
  int rc = run(e, b, mode, true, true);
  return rc ? rc : wait(b);
}
int32_t cordum_dispatch_resident(cordum_engine* e, cordum_batch* b, uint32_t mode) {
  int rc = run(e, b, mode, false, false);
  return rc ? rc : wait(b);
}
int32_t cordum_dispatch_resident_async(cordum_engine* e, cordum_batch* b, uint32_t mode) { return run(e, b, mode, false, false); }

uint32_t cordum_batch_size(const cordum_batch* b) { return b ? b->n : 0; }
const cordum_decision* cordum_batch_results(const cordum_batch* b) { return b ? b->h_out : nullptr; }
int32_t cordum_batch_timing(const cordum_batch* b, float* total_ms, float* kernel_ms) {
  if (!b) { g_err = "null batch"; return CORDUM_E_INVALID; }
  if (total_ms) *total_ms = b->total_ms;
  if (kernel_ms) *kernel_ms = b->kernel_ms;
  return CORDUM_OK;
}
int32_t cordum_batch_kernel_times(const cordum_batch* b, float* policy_ms, float* route_ms) {
  if (!b) { g_err = "null batch"; return CORDUM_E_INVALID; }
  if (policy_ms) *policy_ms = b->policy_ms;
  if (route_ms) *route_ms = b->route_ms;
  return CORDUM_OK;
}
int32_t cordum_batch_plan(cordum_batch* b, cordum_plan* out) {
  cordum::NvtxRange nvtx_("cordum:plan");
  if (!b || !out) { g_err = "null argument"; return CORDUM_E_INVALID; }
  cordum_engine* e = b->e;
  if (e->failed) { g_err = "engine failed earlier: " + e->fail_msg; return CORDUM_E_CUDA; }
  if (!b->results_ready) { g_err = "the batch has no completed dispatch: dispatch it, and wait for an asynchronous one, first"; return CORDUM_E_STATE; }
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  return plan_batch(e, b, out);
}
int32_t cordum_batch_topic_counts(cordum_batch* b, cordum_topic_counts* out) {
  cordum::NvtxRange nvtx_("cordum:topic_counts");
  if (!b || !out) { g_err = "null argument"; return CORDUM_E_INVALID; }
  cordum_engine* e = b->e;
  if (e->failed) { g_err = "engine failed earlier: " + e->fail_msg; return CORDUM_E_CUDA; }
  if (!b->results_ready) { g_err = "the batch has no completed dispatch: dispatch it, and wait for an asynchronous one, first"; return CORDUM_E_STATE; }
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  return count_batch(e, b, out);
}
int32_t cordum_batch_responses(cordum_batch* b, uint32_t flavor, cordum_responses* out) {
  cordum::NvtxRange nvtx_("cordum:responses");
  if (!b || !out) { g_err = "null argument"; return CORDUM_E_INVALID; }
  if (flavor > CORDUM_REASON_FLAVOR_GATEWAY) { g_err = "unknown reason flavor " + std::to_string(flavor); return CORDUM_E_INVALID; }
  cordum_engine* e = b->e;
  if (e->failed) { g_err = "engine failed earlier: " + e->fail_msg; return CORDUM_E_CUDA; }
  if (!b->results_ready) { g_err = "the batch has no completed dispatch: dispatch it, and wait for an asynchronous one, first"; return CORDUM_E_STATE; }
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  return responses_batch(e, b, flavor, out);
}
int32_t cordum_batch_subset(cordum_batch* src, uint32_t outcome_mask, const uint32_t* jobs, uint32_t n_list, cordum_batch* dst, uint32_t* n_out) {
  cordum::NvtxRange nvtx_("cordum:subset");
  if (!src || !dst || !n_out) { g_err = "null argument"; return CORDUM_E_INVALID; }
  if (src == dst) { g_err = "the subset must go to another batch than its source"; return CORDUM_E_INVALID; }
  if (src->e != dst->e) { g_err = "the two batches belong to different engines"; return CORDUM_E_INVALID; }
  if ((outcome_mask != 0) == (jobs != nullptr)) { g_err = "select by an outcome mask or by a job list, exactly one of the two"; return CORDUM_E_INVALID; }
  if (outcome_mask >> CORDUM_PLAN_OUTCOMES) { g_err = "outcome mask names a bucket beyond CORDUM_PLAN_OUTCOMES"; return CORDUM_E_INVALID; }
  for (uint32_t k = 0; jobs && k < n_list; ++k)
    if (jobs[k] >= src->n || (k && jobs[k] <= jobs[k - 1])) {
      g_err = "job list entry " + std::to_string(k) + " is out of range or not strictly ascending";
      return CORDUM_E_INVALID;
    }
  cordum_engine* e = src->e;
  if (e->failed) { g_err = "engine failed earlier: " + e->fail_msg; return CORDUM_E_CUDA; }
  if (!jobs && !src->results_ready) {
    g_err = "the source batch has no completed dispatch: dispatch it, and wait for an asynchronous one, first";
    return CORDUM_E_STATE;
  }
  if (jobs && (!src->encoded || !src->resident || src->pending || src->enc_inflight)) {
    g_err = "the source batch's records are not complete on the device: wait for its encode or dispatch, or dispatch it once";
    return CORDUM_E_STATE;
  }
  {
    std::lock_guard<std::mutex> gh(e->host->mutex());
    if (src->epoch != e->host->epoch()) { g_err = "tables were reloaded after the source batch was encoded: encode again"; return CORDUM_E_STALE; }
  }
  if (jobs && n_list > dst->max_jobs) { g_err = "the job list is longer than the destination batch holds"; return CORDUM_E_CAPACITY; }
  if (dst->pending || dst->enc_inflight || dst->tick_pending) { int rc = wait(dst); if (rc) return rc; }
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  return subset_batch(e, src, outcome_mask, jobs, n_list, dst, n_out);
}
const uint32_t* cordum_batch_parent_index(const cordum_batch* dst, uint32_t* n) {
  const bool ok = dst && dst->is_subset;
  if (n) *n = ok ? dst->n : 0;
  return ok ? dst->h_parent : nullptr;
}
int32_t cordum_batch_merge(cordum_batch* a, cordum_batch* b, cordum_batch* dst) {
  cordum::NvtxRange nvtx_("cordum:merge");
  if (!a || !b || !dst) { g_err = "null argument"; return CORDUM_E_INVALID; }
  if (dst == a || dst == b) { g_err = "the merge must go to another batch than its sources"; return CORDUM_E_INVALID; }
  if (a->e != b->e || a->e != dst->e) { g_err = "the batches belong to different engines"; return CORDUM_E_INVALID; }
  cordum_engine* e = a->e;
  if (e->failed) { g_err = "engine failed earlier: " + e->fail_msg; return CORDUM_E_CUDA; }
  for (const cordum_batch* x : {a, b})
    if (!x->encoded || !x->resident || x->pending || x->enc_inflight || x->tick_pending) {
      g_err = "a source batch's records are not complete on the device: wait for its encode, dispatch or tick, or dispatch it once";
      return CORDUM_E_STATE;
    }
  {
    std::lock_guard<std::mutex> gh(e->host->mutex());
    if (a->epoch != e->host->epoch() || b->epoch != e->host->epoch()) {
      g_err = "tables were reloaded after a source batch was encoded: encode again";
      return CORDUM_E_STALE;
    }
  }
  if ((uint64_t)a->n + b->n > dst->max_jobs) {
    g_err = "the merge has " + std::to_string((uint64_t)a->n + b->n) + " jobs, more than the destination batch holds (" +
            std::to_string(dst->max_jobs) + ")";
    return CORDUM_E_CAPACITY;
  }
  if (dst->pending || dst->enc_inflight || dst->tick_pending) { int rc = wait(dst); if (rc) return rc; }
  CK(cudaSetDevice(e->device), "cudaSetDevice");
  return merge_batch(e, a, b, dst);
}
/* copies the decision records still on the device into the pinned result buffer (after a resident run) */
int32_t cordum_batch_fetch(cordum_batch* b) {
  if (!b) { g_err = "null batch"; return CORDUM_E_INVALID; }
  cordum_engine* e = b->e;
  CK(cudaMemcpyAsync(b->h_out, b->d_out, (size_t)b->n * sizeof(cordum_decision), cudaMemcpyDeviceToHost, b->stream), "D2H results");
  CK(cudaStreamSynchronize(b->stream), "fetch");
  return CORDUM_OK;
}
/* raw CUDA stream of a batch (cudaStream_t) so a harness can bracket launches with its own events */
void* cordum_batch_stream(cordum_batch* b) { return b ? (void*)b->stream : nullptr; }

namespace {
// rule text of policy generation `gen` (0 = the policy in force); null when that generation is no longer kept
const cordum::PolicyText::Rule* rule_text(cordum_engine* e, uint64_t gen, int32_t rule_idx, std::shared_ptr<const cordum::PolicyText>& keep) {
  std::lock_guard<std::mutex> g(e->host->mutex());
  keep = e->host->policy_text(gen);
  if (!keep || rule_idx < 0 || (size_t)rule_idx >= keep->rules.size()) return nullptr;
  return &keep->rules[rule_idx];
}
}  // namespace

int64_t cordum_rule_id_at(cordum_engine* e, uint64_t gen, int32_t rule_idx, char* buf, uint64_t cap) {
  if (!e) return -1;
  std::shared_ptr<const cordum::PolicyText> keep;
  const auto* r = rule_text(e, gen, rule_idx, keep);
  return copy_out(r ? r->id : std::string(), buf, cap);
}
int64_t cordum_rule_constraints_json_at(cordum_engine* e, uint64_t gen, int32_t rule_idx, char* buf, uint64_t cap) {
  if (!e) return -1;
  std::shared_ptr<const cordum::PolicyText> keep;
  const auto* r = rule_text(e, gen, rule_idx, keep);
  return copy_out((r && r->has_constraints) ? r->constraints_json : std::string(), buf, cap);
}
int64_t cordum_rule_remediations_json_at(cordum_engine* e, uint64_t gen, int32_t rule_idx, char* buf, uint64_t cap) {
  if (!e) return -1;
  std::shared_ptr<const cordum::PolicyText> keep;
  const auto* r = rule_text(e, gen, rule_idx, keep);
  return copy_out(r ? r->remediations_json : std::string(), buf, cap);
}
int64_t cordum_rule_id(cordum_engine* e, int32_t rule_idx, char* buf, uint64_t cap) { return cordum_rule_id_at(e, 0, rule_idx, buf, cap); }
int64_t cordum_rule_constraints_json(cordum_engine* e, int32_t rule_idx, char* buf, uint64_t cap) {
  return cordum_rule_constraints_json_at(e, 0, rule_idx, buf, cap);
}
int64_t cordum_rule_remediations_json(cordum_engine* e, int32_t rule_idx, char* buf, uint64_t cap) {
  return cordum_rule_remediations_json_at(e, 0, rule_idx, buf, cap);
}

int64_t cordum_reason(cordum_engine* e, const cordum_batch* b, uint32_t job, char* buf, uint64_t cap) {
  return cordum_reason_flavor(e, b, job, CORDUM_REASON_FLAVOR_KERNEL, nullptr, buf, cap);
}

int64_t cordum_reason_flavor(cordum_engine* e, const cordum_batch* b, uint32_t job, uint32_t flavor,
                             const cordum_envelopes* env, char* buf, uint64_t cap) {
  if (!e || !b || job >= b->n || flavor > CORDUM_REASON_FLAVOR_GATEWAY || (env && env->n_jobs != b->n)) return -1;
  if (ensure_host_records(const_cast<cordum_batch*>(b))) return -1;
  std::lock_guard<std::mutex> g(e->host->mutex());
  const cordum_decision& r = b->h_out[job];
  std::string s;
  if (!render_reason(e, b, r.reason_code, r.rule_idx, reason_arg(r.reason_code, b->hr.job[b->hr.slot_of[job]]), flavor, env, job, s))
    return -1;
  return copy_out(s, buf, cap);
}

int64_t cordum_subject(cordum_engine* e, const cordum_batch* b, uint32_t job, char* buf, uint64_t cap) {
  if (!e || !b || job >= b->n) return -1;
  if (ensure_host_records(const_cast<cordum_batch*>(b))) return -1;
  std::lock_guard<std::mutex> g(e->host->mutex());
  const cordum_decision& r = b->h_out[job];
  std::string s;
  if ((r.route_status == CORDUM_ROUTE_OK || r.route_status == CORDUM_ROUTE_OK_PREFERRED) && r.worker_slot >= 0 && b->wtext &&
      (size_t)r.worker_slot < b->wtext->size()) {
    const std::string& id = (*b->wtext)[(size_t)r.worker_slot];   // the registry the batch was dispatched against
    const uint32_t tid = b->hr.job[b->hr.slot_of[job]].topic;
    s = !id.empty() ? "worker." + id + ".jobs" : (b->ttext && tid < b->ttext->size()) ? (*b->ttext)[tid] : std::string();   // bus/nats.go:94-99; :131-135
  }
  return copy_out(s, buf, cap);
}

int32_t cordum_stats(cordum_engine* e, cordum_table_stats* out) {
  if (!e || !out) { g_err = "null argument"; return CORDUM_E_INVALID; }
  std::lock_guard<std::mutex> g(e->host->mutex());
  const HostTables& t = e->host->tables();
  std::memset(out, 0, sizeof *out);
  out->n_rules = t.n_rules; out->n_rules_padded = t.n_seg * CORDUM_SEG_RULES; out->n_segments = t.n_seg;
  out->n_topics = t.row_topic.n_rows; out->n_tenants = t.row_tenant.n_rows; out->n_pools = t.n_pools;
  out->n_workers = t.n_slots; out->n_workers_routable = t.n_pos;
  size_t rows = t.row_tenant.data.size() + t.row_topic.data.size() + t.row_cap.data.size() + t.row_pack.data.size() +
                t.row_actor.data.size() + t.row_combo.data.size() + t.row_risk.data.size() + t.row_check.data.size();
  for (int f = 0; f < 4; ++f) rows += t.row_mcp[f].data.size();
  out->passrow_bytes = rows * 4;
  out->rulecol_bytes = (uint64_t)t.n_rules * (8 + 8 + 1) + t.tenant_mcp.size() + t.eff_mcp.size() + t.eff_topic.size();
  out->routing_bytes = (t.topic_pool_off.size() + t.topic_pool_cnt.size() + t.pool_list.size()) * 4 + (uint64_t)t.n_pools * 9;
  out->worker_bytes = (uint64_t)t.n_pos * (4 * 3 + 16 + 8) + (uint64_t)t.n_slots * (16 + 8) + (uint64_t)t.n_pools * 16;
  out->job_in_bytes = CORDUM_JOB_IN_BYTES;
  out->job_out_bytes = CORDUM_JOB_OUT_BYTES;
  return CORDUM_OK;
}

uint64_t cordum_launch_count(cordum_engine* e) { return e ? e->launches.load() : 0; }

/* ---- test hooks: the product's own string primitives, for differential tests against the oracle */
int32_t cordum_test_glob(const char* pat, uint64_t plen, const char* name, uint64_t nlen) {
  return cordum::test_glob(sv(pat, plen), sv(name, nlen));
}
void cordum_test_trim(const char* s, uint64_t n, uint64_t* off, uint64_t* len) {
  sv t = cordum::trim_space(sv(s, n));
  *off = t.empty() ? 0 : (uint64_t)(t.data() - s);
  *len = t.size();
}
/* canonical forms the table compiler uses: kind 0 = strings.EqualFold class of the string (no trim), 1 = strings.ToLower, 2 = strconv.Quote */
int64_t cordum_test_canon(int32_t kind, const char* s, uint64_t n, char* buf, uint64_t cap) {
  std::string o = kind == 0 ? cordum::fold_str(sv(s, n)) : kind == 1 ? cordum::lower_copy(sv(s, n)) : cordum::go_quote(sv(s, n));
  if (buf && cap) std::memcpy(buf, o.data(), std::min<size_t>(o.size(), cap));
  return (int64_t)o.size();
}
int32_t cordum_test_normalize_decision(const char* s, uint64_t n) { return cordum::normalize_decision_code(sv(s, n)); }
/* a batch's side records as the kernels read them: which = 0 its selective list (32-bit words, tables.h JobRecords), 1 its
 * wide-mask rows (64-bit words, [n][wide_words]).  Copies up to cap bytes into out; returns the full byte length, or -1 */
int64_t cordum_test_batch_side(cordum_batch* b, int32_t which, void* out, uint64_t cap) {
  if (!b || which < 0 || which > 1) return -1;
  if ((b->pending || b->enc_inflight || b->tick_pending) && wait(b)) return -1;
  const uint64_t bytes = which == 0 ? (uint64_t)b->sel_words * 4 : (uint64_t)b->n * b->wide_words * 8;
  const void* dev = which == 0 ? (const void*)b->d_sel : (const void*)b->d_wide;
  const void* host = which == 0 ? (const void*)b->h_sel : (const void*)b->h_wide;
  const size_t take = (size_t)std::min<uint64_t>(bytes, cap);
  if (take && b->resident) {   // what the last H2D put there, or what the device wrote
    cordum_engine* e = b->e;
    if (cudaSetDevice(e->device) != cudaSuccess || cudaMemcpy(out, dev, take, cudaMemcpyDeviceToHost) != cudaSuccess) return -1;
  } else if (take) {
    std::memcpy(out, host, take);
  }
  return (int64_t)bytes;
}
int32_t cordum_test_parse_effective(const char* s, uint64_t n, uint32_t* n_allowed, uint32_t* n_denied) {
  cordum::EffSafety cfg;
  bool ok = cordum::parse_effective_safety(sv(s, n), cfg);
  if (n_allowed) *n_allowed = (uint32_t)cfg.allowed_topics.size();
  if (n_denied) *n_denied = (uint32_t)cfg.denied_topics.size();
  return ok ? 1 : 0;
}

}  // extern "C"
