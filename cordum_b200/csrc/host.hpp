// host.hpp — host side of the engine: policy/routing/worker models, the table compiler
// (strings -> dictionary-coded pass-rows and columns) and the job encoder.
// No CUDA in here: engine.cu owns device memory and uploads what this produces.
//
// Reference semantics compiled into tables (nothing here runs per job on the GPU path
// except encode(), which is pure dictionary lookup):
//   matchRule predicates            core/infra/config/safety_policy.go:259-294
//   legacyRules                     :225-257          normalizeDecision :208-223
//   MCPAllowed / matchMCPField      :385-416
//   request normalisation           core/controlplane/safetykernel/kernel.go:133-185, 348-414
//   ParseEffectiveSafety            core/infra/config/effective.go:12-39
//   pool / label filtering          core/controlplane/scheduler/strategy_least_loaded.go:161-265
#pragma once
#include <cstdint>
#include <cstring>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <memory>
#include <mutex>
#include <thread>
#include <deque>
#include <memory>
#include <string>
#include <string_view>
#include <unordered_map>
#include <vector>

#include "../../include/cordum_b200.h"
#include "gostr.hpp"
#include "tables.h"

namespace cordum {

struct EncodeCaches;

// ------------------------------------------------------------------ string-keyed hash table
// Open addressing, keyed by bytes, lookups take a string_view (no allocation on the encode path).
// The hash reads 8 bytes per step (two multiplies per 16 bytes).  hash_fold() lower-cases ASCII letters on the fly
// (SWAR), so that an ASCII value can be looked up under strings.EqualFold semantics without first being copied into
// its canonical form: canonical strings hold no upper-case ASCII, hence hash_fold(raw) == hash(fold_str(raw)).
class StrTable {
 public:
  StrTable() { slots_.assign(16, Slot{}); }
  static uint64_t rd8(const char* p) { uint64_t v; std::memcpy(&v, p, 8); return v; }
  static uint64_t rd4(const char* p) { uint32_t v; std::memcpy(&v, p, 4); return v; }
  static uint64_t mix(uint64_t a, uint64_t b) { __uint128_t r = (__uint128_t)a * b; return (uint64_t)r ^ (uint64_t)(r >> 64); }
  static uint64_t lower8(uint64_t v) {   // ASCII 'A'..'Z' -> 'a'..'z' in each byte, other bytes untouched
    const uint64_t v7 = v & 0x7F7F7F7F7F7F7F7Full;
    const uint64_t up = (v7 + 0x3F3F3F3F3F3F3F3Full) & ~(v7 + 0x2525252525252525ull) & ~v & 0x8080808080808080ull;
    return v | (up >> 2);
  }
  template <bool FOLD>
  static uint64_t hash_impl(sv s) {
    const char* p = s.data();
    size_t n = s.size();
    uint64_t h = 0x9E3779B97F4A7C15ull ^ (n * 0xA0761D6478BD642Full);
    auto L = [](uint64_t v) { return FOLD ? lower8(v) : v; };
    while (n > 16) {
      h = mix(L(rd8(p)) ^ 0xE7037ED1A0B428DBull, L(rd8(p + 8)) ^ h);
      p += 16; n -= 16;
    }
    uint64_t a = 0, b = 0;
    if (n >= 8) { a = L(rd8(p)); b = L(rd8(p + n - 8)); }
    else if (n >= 4) { a = L(rd4(p)); b = L(rd4(p + n - 4)); }
    else if (n > 0) { a = L(((uint64_t)(unsigned char)p[0] << 16) | ((uint64_t)(unsigned char)p[n >> 1] << 8) | (unsigned char)p[n - 1]); }
    h = mix(a ^ 0x8EBC6AF09C88C6E3ull, b ^ h);
    return h | 1;
  }
  static uint64_t hash(sv s) { return hash_impl<false>(s); }
  static uint64_t hash_fold(sv s) { return hash_impl<true>(s); }
  // returns value or `miss`
  uint32_t find(sv key, uint32_t miss) const {
    uint64_t h = hash(key);
    size_t m = slots_.size() - 1;
    for (size_t i = h & m;; i = (i + 1) & m) {
      const Slot& s = slots_[i];
      if (s.hash == 0) return miss;
      if (s.hash == h && s.len == key.size() && std::memcmp(pool_.data() + s.off, key.data(), s.len) == 0) return s.val;
    }
  }
  // key: an ASCII string; matches the stored canonical (ASCII-lowered) string it folds to
  uint32_t find_fold_ascii(sv key, uint32_t miss) const {
    uint64_t h = hash_fold(key);
    size_t m = slots_.size() - 1;
    for (size_t i = h & m;; i = (i + 1) & m) {
      const Slot& s = slots_[i];
      if (s.hash == 0) return miss;
      if (s.hash == h && s.len == key.size()) {
        const char* c = pool_.data() + s.off;
        size_t k = 0;
        for (; k < key.size(); ++k) {
          char x = key[k];
          if (x >= 'A' && x <= 'Z') x = char(x + 32);
          if (x != c[k]) break;
        }
        if (k == key.size()) return s.val;
      }
    }
  }
  // a label pair as one key: len(a) as 4 little-endian bytes, a, b.  A separator byte would not do: keys and values may
  // hold any byte, NUL included, and "a\0b" = "c" must not meet "a" = "b\0c".  encode.cu hash_pair builds the same bytes.
  static void put_pair(char* out, sv a, sv b) {
    const uint32_t n = (uint32_t)a.size();
    const char len[4] = {char(n), char(n >> 8), char(n >> 16), char(n >> 24)};
    std::memcpy(out, len, 4); std::memcpy(out + 4, a.data(), a.size()); std::memcpy(out + 4 + a.size(), b.data(), b.size());
  }
  static std::string pair_key(sv a, sv b) {
    std::string k(4 + a.size() + b.size(), '\0');
    put_pair(k.data(), a, b);
    return k;
  }
  // find(pair_key(a, b)), without building it on the heap
  uint32_t find_pair(sv a, sv b, uint32_t miss) const {
    char small[260];
    const size_t n = 4 + a.size() + b.size();
    if (n > sizeof small) return find(pair_key(a, b), miss);
    put_pair(small, a, b);
    return find(sv(small, n), miss);
  }
  bool contains(sv key) const { return find(key, 0xFFFFFFFEu) != 0xFFFFFFFEu; }
  void put(sv key, uint32_t val) {
    if ((count_ + 1) * 2 > slots_.size()) grow();
    uint64_t h = hash(key);
    size_t m = slots_.size() - 1;
    for (size_t i = h & m;; i = (i + 1) & m) {
      Slot& s = slots_[i];
      if (s.hash == 0) {
        s.hash = h; s.off = (uint32_t)pool_.size(); s.len = (uint32_t)key.size(); s.val = val;
        pool_.append(key.data(), key.size());
        ++count_;
        return;
      }
      if (s.hash == h && s.len == key.size() && std::memcmp(pool_.data() + s.off, key.data(), s.len) == 0) {
        s.val = val;
        return;
      }
    }
  }
  size_t size() const { return count_; }
  void clear() { slots_.assign(16, Slot{}); pool_.clear(); count_ = 0; }
  // Device image (tables.h DevDict): 32 B slots {hash, off, len, val} + the key bytes, appended to `blob`; the device
  // probes it with the same hash and the same linear probing, so host and device lookups agree by construction.
  void export_to(std::vector<uint8_t>& blob, DevDict& ref) const {
    auto align = [&](size_t a) { blob.resize((blob.size() + a - 1) / a * a); };
    align(32);
    ref.slots_off = (uint32_t)blob.size();
    ref.mask = (uint32_t)slots_.size() - 1;
    blob.resize(blob.size() + slots_.size() * 32);
    uint8_t* p = blob.data() + ref.slots_off;
    for (size_t i = 0; i < slots_.size(); ++i) {
      const Slot& s = slots_[i];
      uint32_t rec[8] = {(uint32_t)s.hash, (uint32_t)(s.hash >> 32), s.off, s.len, s.val, 0, 0, 0};
      std::memcpy(p + i * 32, rec, 32);
    }
    align(16);
    ref.pool_off = (uint32_t)blob.size();
    blob.insert(blob.end(), pool_.begin(), pool_.end());
    blob.resize(blob.size() + 16);   // slack: the device may read up to 8 bytes past a key
  }

 private:
  struct Slot { uint64_t hash = 0; uint32_t off = 0, len = 0, val = 0; };
  std::vector<Slot> slots_;
  std::string pool_;
  size_t count_ = 0;
  void grow() {
    std::vector<Slot> old;
    old.swap(slots_);
    slots_.assign(old.size() * 2, Slot{});
    size_t m = slots_.size() - 1;
    for (auto& s : old) {
      if (!s.hash) continue;
      size_t i = s.hash & m;
      while (slots_[i].hash) i = (i + 1) & m;
      slots_[i] = s;
    }
  }
};

// Dictionary of canonical strings: id 0 = raw-empty, 1 = other, >=2 referenced values.
struct Dict {
  StrTable table;
  std::vector<std::string> keys;   // keys[id-2]
  uint32_t intern(sv canon) {
    uint32_t id = table.find(canon, 0);
    if (id) return id;
    id = (uint32_t)keys.size() + 2;
    keys.emplace_back(canon);
    table.put(canon, id);
    return id;
  }
  uint32_t size() const { return (uint32_t)keys.size() + 2; }
  void clear() { table.clear(); keys.clear(); }
};

// ------------------------------------------------------------------ models
struct McpLists { std::vector<std::string> allow[4], deny[4]; };   // server, tool, resource, action

struct RuleModel {
  std::string id, decision, reason;
  std::vector<std::string> tenants, topics, capabilities, risk_tags, requires_, pack_ids, actor_ids, actor_types;
  std::vector<std::pair<std::string, std::string>> labels;
  int secrets_present = -1;
  McpLists mcp;
  bool has_constraints = false;
  std::string constraints_json, remediations_json;
};
// What the decision records of one dispatch index, as text.  Immutable once published: a batch keeps the one it was
// dispatched under, so a policy / registry reload after the dispatch cannot relabel its decisions (the reference's
// evaluate reads policy and snapshot under one lock and builds the whole response from them, kernel.go:140-147,239-248).
struct PolicyText {
  uint64_t gen = 0;   // 1, 2, ...: counts successful policy loads
  std::string snapshot;
  struct Rule { std::string id, reason, constraints_json, remediations_json; bool has_constraints = false; };
  std::vector<Rule> rules;
};
struct TenantModel { std::string name; std::vector<std::string> allow_topics, deny_topics; McpLists mcp; };
struct PolicyModel {
  bool nil = true;
  std::string default_tenant;
  std::vector<RuleModel> rules;       // effective rule list (legacy expansion applied)
  std::vector<TenantModel> tenants;   // sorted by name bytes
};
struct RoutingModel {
  std::vector<std::pair<std::string, std::vector<std::string>>> topics;
  std::vector<std::pair<std::string, std::vector<std::string>>> pools;   // name -> requires
};
struct EffSafety { std::vector<std::string> allowed_topics, denied_topics; McpLists mcp; };
// Worker snapshot kept as strings so that routing changes can recompile the worker tables.
struct WorkerRaw { std::string id, pool; std::vector<std::pair<std::string, std::string>> labels; };

bool parse_policy_json(sv text, PolicyModel& out, std::string& err);
bool parse_routing_json(sv text, RoutingModel& out, std::string& err);
bool parse_effective_safety(sv payload, EffSafety& out);
uint8_t normalize_decision_code(sv raw);   // CORDUM_DEC_*

// ------------------------------------------------------------------ compiled host tables
using Bits = std::vector<uint32_t>;   // one pass-row: n_seg*32 words

struct RowTable {                      // rows for one attribute, row-major
  uint32_t n_rows = 0, row_words = 0;
  std::vector<uint32_t> data;
  void init(uint32_t rows, uint32_t words) { n_rows = rows; row_words = words; data.assign((size_t)rows * words, 0); }
  uint32_t* row(uint32_t r) { return data.data() + (size_t)r * row_words; }
  const uint32_t* row(uint32_t r) const { return data.data() + (size_t)r * row_words; }
  void append(const Bits& b) { data.insert(data.end(), b.begin(), b.end()); ++n_rows; }
};

struct TopicEntry { uint32_t flags; uint32_t pool_off, pool_cnt; };

struct HostTables {
  // policy (pass-rows are kept row-major here; the engine uploads them word-major, tables.h)
  uint32_t n_rules = 0, n_seg = 1, row_words = 32;
  RowTable row_tenant, row_topic, row_cap, row_pack, row_actor, row_combo, row_risk, row_check, row_mcp[4];
  // per row: which 128-bit word groups hold any bit (bit g = words [g*sum_group, (g+1)*sum_group))
  std::vector<uint64_t> sum_tenant, sum_topic, sum_cap, sum_pack, sum_actor, sum_combo, sum_risk;
  uint32_t sum_group = 1, sum_use = 0;
  std::vector<uint64_t> rule_req_need, rule_lab_need;
  // wide masks (tables.h WideLayout): all empty / zero unless a dictionary outgrew the record's mask fields
  WideLayout wide{0, 0, 0, 0};
  std::vector<uint64_t> rule_need_x, pool_req_x, req_blank_x, pos_label_x;
  std::vector<uint8_t> rule_dec;
  std::vector<uint32_t> pos2rule;                 // bit position -> original rule index (0xFFFFFFFF = padding)
  uint32_t mcp_stride = 2;
  std::vector<uint8_t> tenant_mcp, eff_mcp, eff_topic;
  uint32_t topic_stride = 0, n_effcfg = 0;
  // routing
  std::vector<uint32_t> topic_pool_off, topic_pool_cnt, pool_list;
  std::vector<uint64_t> pool_req_mask;
  std::vector<uint8_t> pool_req_nonempty;
  uint64_t req_blank_mask = 0;
  uint32_t n_pools = 0;
  // workers
  uint32_t n_slots = 0, n_pos = 0;
  std::vector<uint32_t> pool_off, pos_pool, pos_slot, pos_rank, slot_pos, rank_slot, rank_pos, lbm_off;
  uint32_t place_bits = 1;
  uint64_t lbm_words = 0;
  uint32_t n_sel = 0;                                          // selective placement pairs (tables.h DeviceTables.sel_*)
  std::vector<uint32_t> sel_off, sel_pos, pos_sel_off, pos_sel;
  std::vector<uint32_t> chunk_pool, pool_chunk0, merge_list;   // worker-table refresh work list (tables.h)
  uint32_t n_chunks = 0, n_merge = 0, merge_smem = 0;
  std::vector<uint64_t> pos_label_lo, pos_label_hi;
  std::vector<Load16> loads;
  // change counters (engine re-uploads a group when its version moved)
  uint64_t v_policy = 0, v_topic = 0, v_mcp = 0, v_routing = 0, v_workers = 0, v_loads = 0;
};

// Encoded batch on the host (engine allocates the record arrays pinned and hands pointers in).  Records are in
// topic-sorted order; slot_of[j] is the position of caller job j (pageable host memory, host-side use only).
constexpr int kWideRetry = -100;   // Host::encode: HostRecords.wide is too small for the tables as they are now
struct HostRecords {
  JobRec* job = nullptr;
  RouteRec* route = nullptr;
  uint32_t* slot_of = nullptr;
  uint64_t* wide = nullptr;      // [n][wide_words] when the tables carry wide masks (Host::wide_words() at encode time)
  uint64_t wide_cap = 0;         // 64-bit words available at `wide`
  uint32_t wide_words = 0;       // out: the row width the encode used
  uint64_t epoch = 0;            // out: the table epoch the ids belong to (read under the encoder's lock)
  // out: the selective list (tables.h JobRecords): {slot, x} per JF_SELECTIVE job, then the extra words; both empty
  // when no job of the batch names a selective pair
  std::vector<uint32_t> sel_jobs, sel_extra;
};

// Which placement pairs are selective: registries with more than min_bits placement bits, pairs carried by at most
// max_holders routable workers (CORDUM_SEL_MIN_BITS / CORDUM_SEL_MAX_HOLDERS).  Tests move both to run the dense and the
// selective path on the same inputs; takes effect at the next worker / routing load.
void set_selective_limits(uint32_t min_bits, uint32_t max_holders);

// Persistent worker pool for the encoder: parallel_for over [0,n) in dynamically claimed chunks.  Completion
// is "every item processed", not "every worker checked in": a worker the OS has descheduled (busy or
// quota-throttled host) costs nothing once the others have drained the queue.
class WorkPool {
 public:
  explicit WorkPool(uint32_t threads);
  ~WorkPool();
  using Fn = std::function<void(uint32_t, uint32_t, uint32_t)>;   // fn(begin, end, worker)
  void parallel_for(uint32_t n, uint32_t grain, const Fn& fn);
  uint32_t size() const { return (uint32_t)threads_.size() + 1; }

 private:
  struct Job {
    const Fn* fn;
    uint32_t n, grain;
    std::atomic<uint32_t> next{0}, done{0};
  };
  void worker(uint32_t id);
  static void drain(Job& j, uint32_t id);
  std::vector<std::thread> threads_;
  std::mutex mu_;
  std::condition_variable cv_;
  std::shared_ptr<Job> current_;
  uint64_t epoch_ = 0;
  bool stop_ = false;
};

// extractMCPRequest's value of one field (0 server, 1 tool, 2 resource, 3 action) as the request spells it (kernel.go:395-414)
std::string mcp_request_value(const cordum_envelopes* env, uint32_t job, int field);

class Host {
 public:
  Host(uint32_t max_topics, uint32_t max_effcfgs, uint32_t encode_threads);
  ~Host();

  // documents
  int load_policy(sv json, sv snapshot, std::string& err);
  int load_routing(sv json, std::string& err);
  int load_workers(const cordum_workers* w, std::string& err);
  int update_loads(uint32_t n, const uint32_t* slots, const cordum_worker_load* loads, std::string& err);

  // encode a batch (thread-safe against itself via mu_)
  int encode(const cordum_envelopes* env, HostRecords& out, std::string& err);

  // bumps whenever dictionary ids may have been reassigned (policy / routing / worker reload):
  // batches encoded under an older epoch must be re-encoded before dispatch
  uint64_t epoch() const { return epoch_; }
  const HostTables& tables() const { return t_; }
  HostTables& tables_mut() { return t_; }
  std::mutex& mutex() { return mu_; }

  // Everything the device-side encoder needs besides the compiled tables: the dictionaries as probe-able images, the
  // per-id side arrays and a few scalars (tables.h EncodeTables).  Rebuilt when dict_version() moves.  Under mutex().
  uint64_t dict_version() const { return v_dict_; }
  void export_dicts(std::vector<uint8_t>& blob, EncodeTables& et) const;
  // the device encoder met something it leaves to the host (first sight of a topic / effective config, non-ASCII text):
  // same contract as encode(); kept separate so that callers can count how often it happens
  uint64_t host_fallbacks = 0;

  // string materialisation
  const PolicyModel& policy() const { return policy_; }
  const std::vector<std::string>& snapshots() const { return snapshots_; }
  const std::string& current_snapshot() const { return snapshot_; }
  const std::string& worker_id(uint32_t slot) const { return (*worker_ids_)[slot]; }
  uint32_t n_worker_slots() const { return (uint32_t)worker_ids_->size(); }
  std::shared_ptr<const std::vector<std::string>> worker_text() const { return worker_ids_; }
  std::shared_ptr<const PolicyText> policy_text(uint64_t gen = 0) const {   // 0 = the policy in force; else one of the last 8
    if (gen == 0) return text_.empty() ? nullptr : text_.back();
    for (auto& t : text_) if (t->gen == gen) return t;
    return nullptr;
  }
  const std::string& topic_raw(uint32_t topic_id) const { return (*topic_store_)[topic_id]; }
  std::shared_ptr<const std::vector<std::string>> topic_text() const { return topic_store_; }
  uint64_t dict_resets() const { return dict_resets_; }
  // the encoders' sort key of a job: topic id * tenant_classes() + tenant_class()[tenant dictionary id]
  uint32_t tenant_classes() const { return std::max<uint32_t>(1, tenant_classes_); }
  const std::vector<uint8_t>& tenant_class() const { return tenant_class_; }
  uint32_t wide_words() const { return WIDE_WORDS(t_.wide); }
  uint64_t policy_generation() const { return text_gen_.load(std::memory_order_acquire); }
  std::string mcp_value_string(int field, uint32_t id) const;
  const std::vector<std::string>& topic_pool_names(uint32_t topic_id) const;
  uint32_t n_topics() const { return (uint32_t)topic_store_->size(); }

 private:
  std::mutex mu_;
  uint64_t epoch_ = 1;
  uint64_t v_dict_ = 1;   // bumps whenever any dictionary changes (loads, first sight of a topic / effective config)
  uint32_t max_topics_, max_effcfgs_, threads_;
  std::string policy_capacity_error_, routing_capacity_error_;
  std::vector<WorkerRaw> workers_raw_;
  std::unique_ptr<WorkPool> pool_;   // created on first large encode
  std::vector<std::unique_ptr<EncodeCaches>> caches_;   // one per encoder thread, generation-tagged
  uint32_t encode_gen_ = 0;
  std::vector<uint32_t> scratch_tid_, scratch_ten_, scratch_hist_;   // encode() temporaries, kept between calls
  // sort key of the encoded records: (topic id, tenant class); class = which word group holds the tenant's per-tenant rule copies
  static constexpr uint32_t kMaxTenantClasses = 16;
  uint32_t tenant_classes_ = 1;
  std::vector<uint8_t> tenant_class_;   // per tenant dictionary id
  PolicyModel policy_;
  RoutingModel routing_;
  std::string snapshot_;
  std::vector<std::string> snapshots_;
  HostTables t_;

  // policy dictionaries
  Dict d_tenant_, d_cap_, d_pack_, d_actor_, d_risk_, d_req_, d_mcp_[4];
  StrTable tenant_pol_;   // exact tenant string -> 1 + index in policy_.tenants
  StrTable label_key_;    // rule label key -> index into label_key_pairs_
  std::vector<std::vector<std::pair<std::string, uint32_t>>> label_key_pairs_;   // per key: (value, bit)
  uint64_t label_empty_mask_ = 0;   // bits of pairs whose value is ""
  std::vector<uint64_t> label_empty_x_;   // ... beyond bit 63
  uint32_t n_label_pairs_ = 0;
  std::vector<std::vector<uint32_t>> rule_req_ids_, rule_lab_bits_;   // per rule: bit numbers of what it needs
  std::vector<std::vector<uint32_t>> pool_req_ids_;                   // per pool: bit numbers of what it declares
  void finalize_wide();
  std::string default_tenant_trim_;
  std::vector<std::vector<uint32_t>> rule_pos_;   // rule index -> its bit positions (see compile_policy)
  std::vector<std::vector<std::string>> rule_pos_tenant_;   // parallel: "" = the copy stands for every tenant the rule lists,
                                                            // else the one (folded) tenant this copy stands for
  // topic patterns (distinct trimmed pattern -> rules)
  struct Pattern { Glob glob; std::vector<uint32_t> rules; };
  std::vector<Pattern> patterns_;
  std::unordered_map<std::string, std::vector<uint32_t>> pat_by_prefix_;   // literal prefix -> patterns
  uint32_t eff_topic_n_ = 0;   // topics whose effective-config verdicts are filled in (for every config known)
  Bits vac_topic_;
  // topics (dynamic)
  StrTable topic_ids_;
  // raw topic per id (id 0 = ""); append-only within a dictionary generation, replaced whole by a reset, shared with
  // the batches dispatched under it (their strings must outlive a reset)
  std::shared_ptr<std::vector<std::string>> topic_store_ = std::make_shared<std::vector<std::string>>();
  uint64_t dict_resets_ = 0;
  static constexpr int kDictFull = -101;
  int encode_locked(const cordum_envelopes* env, HostRecords& out, std::string& err);
  void reset_dynamic_dictionaries();
  std::vector<TopicEntry> topic_entries_;
  std::vector<std::vector<std::string>> topic_pools_;   // original (not deduplicated) lists for messages
  // effective configs (dynamic)
  StrTable effcfg_ids_;
  std::vector<EffSafety> effcfgs_;               // index = id (0 unused)
  std::vector<uint8_t> effcfg_ok_;
  struct EffGlobs { std::vector<Glob> denied, allowed; bool has_allowed = false; };
  std::vector<EffGlobs> eff_globs_;
  // routing dictionaries
  Dict d_pool_;
  StrTable routing_topics_;   // raw topic -> index in routing_.topics
  // workers
  std::shared_ptr<const std::vector<std::string>> worker_ids_ = std::make_shared<std::vector<std::string>>();   // replaced, never edited
  std::deque<std::shared_ptr<const PolicyText>> text_;   // the last 8 policies' text, oldest first
  std::atomic<uint64_t> text_gen_{0};                   // generation of text_.back(), readable without the lock
  void publish_text();
  StrTable worker_slot_;      // worker_id -> slot (last wins)
  StrTable place_pair_;       // StrTable::pair_key(key, value) -> bit, or kSelTag | selective pair id   (value non-empty)
  StrTable place_key_;        // key -> bit E_k ("labels non-empty and k absent-or-empty")
  uint32_t place_any_bit_ = 0; // bit "worker has >= 1 label"
  uint32_t place_bits_ = 0;

  void compile_policy();
  void compile_routing();
  void compile_mcp_tables();
  int compile_workers(std::string& err, const std::vector<Load16>* new_loads = nullptr);   // checks capacity before mutating
  void rebuild_topics();
  uint32_t add_topic(sv raw);          // under mu_
  uint32_t add_effcfg(sv payload);     // under mu_
  void topic_row(sv trimmed, Bits& out) const;
  void eff_topic_fill(uint32_t cfg, uint32_t topic_id);
  uint64_t row_summary(const uint32_t* row) const;
  void choose_summaries();
  void summarize(const RowTable& rt, std::vector<uint64_t>& out) const;
  uint32_t resolve_topic(const cordum_envelopes* env, uint32_t j, struct EncodeCaches& cc) const;   // kMiss = not in the dictionary
  uint32_t resolve_tenant(const cordum_envelopes* env, uint32_t j, struct EncodeCaches& cc) const;   // id | exact-policy index << 16
  void encode_job(const cordum_envelopes* env, uint32_t j, uint32_t tid, uint32_t ten, JobRec& jr, RouteRec& rr, uint64_t* wx, bool& miss, struct EncodeCaches& cc) const;
  void gather_selective(HostRecords& out, uint32_t nthreads) const;
};

// test hooks (also exported through the C ABI as cordum_test_*)
int test_glob(sv pattern, sv name);   // 1 match, 0 no, -1 malformed
bool json_canon(sv text, std::string& out);   // parse + re-dump (differential test of common/mini_json.hpp)

}  // namespace cordum
