// test_hooks.cpp — host-only access to the table compiler and encoder, for CPU tests.
//
// These entry points create a Host (no CUDA involved), load documents, encode envelopes
// into a caller-provided slab and expose the compiled tables by name, so tests can check
// the tables + encoding against the oracle without a GPU (tests/table_walk.py re-walks
// the tables in Python the way kernels.cu does).  They evaluate nothing themselves.
#include <cstring>
#include <string>
#include <vector>

#include "host.hpp"

using cordum::Host;
using cordum::HostRecords;
using cordum::HostTables;
using cordum::sv;

namespace {
thread_local std::string t_err;
thread_local std::vector<uint32_t> t_sel_jobs, t_sel_extra;   // the selective list of the last cordum_test_host_encode
}  // namespace

extern "C" {

const char* cordum_test_last_error(void) { return t_err.c_str(); }
void* cordum_test_host_new(uint32_t max_topics, uint32_t max_effcfgs, uint32_t threads) {
  return new Host(max_topics, max_effcfgs, threads);
}
void cordum_test_host_free(void* h) { delete (Host*)h; }
int32_t cordum_test_host_policy(void* h, const char* json, uint64_t len) {
  return ((Host*)h)->load_policy(sv(json ? json : "", json ? len : 0), sv("test"), t_err);
}
int32_t cordum_test_host_routing(void* h, const char* json, uint64_t len) {
  return ((Host*)h)->load_routing(sv(json ? json : "", json ? len : 0), t_err);
}
int32_t cordum_test_host_workers(void* h, const cordum_workers* w) { return ((Host*)h)->load_workers(w, t_err); }
int32_t cordum_test_host_update(void* h, uint32_t n, const uint32_t* slots, const cordum_worker_load* loads) {
  return ((Host*)h)->update_loads(n, slots, loads, t_err);
}
uint64_t cordum_test_slab_bytes(uint32_t n) { return (uint64_t)n * (sizeof(JobRec) + sizeof(RouteRec) + sizeof(uint32_t)); }
uint32_t cordum_test_host_wide_words(void* h) { return ((Host*)h)->wide_words(); }

// encode into `slab` (cordum_test_slab_bytes(n) bytes, 16 B aligned): n JobRec, then n RouteRec (both in topic-sorted
// order, as a batch's pinned buffers hold them), then slot_of[n]
// `wide`: n * cordum_test_host_wide_words(h) 64-bit words (may be NULL when that is 0)
int32_t cordum_test_host_encode(void* h, const cordum_envelopes* env, uint8_t* slab, uint64_t* wide) {
  uint32_t n = env->n_jobs;
  HostRecords r;
  r.wide = wide;
  r.wide_cap = (uint64_t)n * ((Host*)h)->wide_words();
  r.job = (JobRec*)slab;
  r.route = (RouteRec*)(slab + (size_t)n * sizeof(JobRec));
  r.slot_of = (uint32_t*)(slab + (size_t)n * (sizeof(JobRec) + sizeof(RouteRec)));
  const int32_t rc = ((Host*)h)->encode(env, r, t_err);
  t_sel_jobs = std::move(r.sel_jobs);
  t_sel_extra = std::move(r.sel_extra);
  return rc;
}
// the selective list (tables.h JobRecords) of the last cordum_test_host_encode on this thread: which = 0 the {slot, x}
// pairs, 1 the extra words
int32_t cordum_test_host_sel(int32_t which, const void** ptr, uint64_t* bytes) {
  const std::vector<uint32_t>& v = which ? t_sel_extra : t_sel_jobs;
  *ptr = v.data();
  *bytes = v.size() * sizeof(uint32_t);
  return 0;
}
// selective placement pairs in registries above min_bits placement bits, for pairs with at most max_holders routable
// holders (defaults CORDUM_SEL_MIN_BITS, CORDUM_SEL_MAX_HOLDERS); process-wide, from the next worker / routing load on
void cordum_test_set_selective(uint32_t min_bits, uint32_t max_holders) { cordum::set_selective_limits(min_bits, max_holders); }

// common/mini_json.hpp (shared by the product and the oracle) differentially against an independent parser:
// returns -1 when the document is rejected, else the length of the re-dumped tree (written to buf up to cap)
int64_t cordum_test_json_canon(const char* text, uint64_t n, char* buf, uint64_t cap) {
  std::string out;
  if (!cordum::json_canon(sv(text, n), out)) return -1;
  if (buf && cap) std::memcpy(buf, out.data(), out.size() < cap ? out.size() : cap);
  return (int64_t)out.size();
}

// table access by name: returns pointer + byte length (valid until the next load/encode)
int32_t cordum_test_host_table(void* h, const char* name, const void** ptr, uint64_t* bytes) {
  const HostTables& t = ((Host*)h)->tables();
  std::string n(name);
#define VEC(nm, v) if (n == nm) { *ptr = (v).data(); *bytes = (v).size() * sizeof((v)[0]); return 0; }
  VEC("row_tenant", t.row_tenant.data) VEC("row_topic", t.row_topic.data) VEC("row_cap", t.row_cap.data)
  VEC("row_pack", t.row_pack.data) VEC("row_actor", t.row_actor.data) VEC("row_combo", t.row_combo.data)
  VEC("row_risk", t.row_risk.data) VEC("row_check", t.row_check.data)
  VEC("row_mcp0", t.row_mcp[0].data) VEC("row_mcp1", t.row_mcp[1].data) VEC("row_mcp2", t.row_mcp[2].data)
  VEC("row_mcp3", t.row_mcp[3].data)
  VEC("pos2rule", t.pos2rule)
  VEC("sum_tenant", t.sum_tenant) VEC("sum_topic", t.sum_topic) VEC("sum_cap", t.sum_cap) VEC("sum_pack", t.sum_pack)
  VEC("sum_actor", t.sum_actor) VEC("sum_combo", t.sum_combo) VEC("sum_risk", t.sum_risk)
  VEC("rule_req_need", t.rule_req_need) VEC("rule_lab_need", t.rule_lab_need) VEC("rule_dec", t.rule_dec)
  VEC("rule_need_x", t.rule_need_x) VEC("pool_req_x", t.pool_req_x) VEC("req_blank_x", t.req_blank_x) VEC("pos_label_x", t.pos_label_x)
  VEC("tenant_mcp", t.tenant_mcp) VEC("eff_mcp", t.eff_mcp) VEC("eff_topic", t.eff_topic)
  VEC("topic_pool_off", t.topic_pool_off) VEC("topic_pool_cnt", t.topic_pool_cnt) VEC("pool_list", t.pool_list)
  VEC("pool_req_mask", t.pool_req_mask) VEC("pool_req_nonempty", t.pool_req_nonempty)
  VEC("pool_off", t.pool_off) VEC("pos_pool", t.pos_pool) VEC("pos_slot", t.pos_slot) VEC("pos_rank", t.pos_rank)
  VEC("slot_pos", t.slot_pos) VEC("rank_slot", t.rank_slot) VEC("pos_label_lo", t.pos_label_lo)
  VEC("pos_label_hi", t.pos_label_hi) VEC("loads", t.loads)
  VEC("sel_off", t.sel_off) VEC("sel_pos", t.sel_pos) VEC("pos_sel_off", t.pos_sel_off) VEC("pos_sel", t.pos_sel)
  VEC("chunk_pool", t.chunk_pool) VEC("pool_chunk0", t.pool_chunk0) VEC("merge_list", t.merge_list)
  VEC("tenant_class", ((Host*)h)->tenant_class())
#undef VEC
  t_err = "unknown table " + n;
  return -1;
}
uint64_t cordum_test_host_scalar(void* h, const char* name) {
  const HostTables& t = ((Host*)h)->tables();
  std::string n(name);
  if (n == "n_rules") return t.n_rules;
  if (n == "n_seg") return t.n_seg;
  if (n == "sum_group") return t.sum_group;
  if (n == "sum_use") return t.sum_use;
  if (n == "n_chunks") return t.n_chunks;
  if (n == "n_merge") return t.n_merge;
  if (n == "merge_smem") return t.merge_smem;
  if (n == "row_words") return t.row_words;
  if (n == "mcp_stride") return t.mcp_stride;
  if (n == "topic_stride") return t.topic_stride;
  if (n == "n_effcfg") return t.n_effcfg;
  if (n == "req_blank_mask") return t.req_blank_mask;
  if (n == "n_pools") return t.n_pools;
  if (n == "n_pos") return t.n_pos;
  if (n == "n_slots") return t.n_slots;
  if (n == "n_topics") return t.row_topic.n_rows;
  if (n == "dict_resets") return ((Host*)h)->dict_resets();
  if (n == "tenant_classes") return ((Host*)h)->tenant_classes();
  if (n == "xw_risk") return t.wide.xw_risk;
  if (n == "xw_req") return t.wide.xw_req;
  if (n == "xw_lab") return t.wide.xw_lab;
  if (n == "xw_place") return t.wide.xw_place;
  if (n == "place_bits") return t.place_bits;
  if (n == "n_sel") return t.n_sel;
  if (n == "lbm_words") return t.lbm_words;
  return ~0ull;
}

}  // extern "C"
