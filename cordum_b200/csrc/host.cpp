// host.cpp — models, table compiler and job encoder (see host.hpp).
#include "host.hpp"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <set>
#include <thread>

#include "../../common/mini_json.hpp"

namespace cordum {

// ============================================================ small helpers
namespace {

constexpr uint32_t kMiss = 0xFFFFFFFFu;
std::atomic<uint32_t> g_sel_min_bits{CORDUM_SEL_MIN_BITS}, g_sel_max_holders{CORDUM_SEL_MAX_HOLDERS};

// fold_key without heap allocation for ordinary-sized ASCII values (anything else takes the general path)
struct FoldBuf {
  char small[160];
  std::string big;
  sv view;
  explicit FoldBuf(sv raw) {
    sv t = trim_space(raw);
    if (t.size() <= sizeof small && is_ascii(t)) {
      for (size_t i = 0; i < t.size(); ++i) small[i] = lower_ascii(t[i]);
      view = sv(small, t.size());
    } else {
      big = fold_str(t);
      view = big;
    }
  }
};

bool fold_eq(sv a, sv b) {   // strings.EqualFold
  if (is_ascii(a) && is_ascii(b)) {
    if (a.size() != b.size()) return false;
    for (size_t i = 0; i < a.size(); ++i)
      if (lower_ascii(a[i]) != lower_ascii(b[i])) return false;
    return true;
  }
  return fold_str(a) == fold_str(b);
}

// No TrimSpace needed: the string starts and ends with an ASCII byte that is not white space (every Unicode space is
// either <= 0x20 or starts with a byte >= 0x80 in UTF-8).
inline bool untrimmed_ok(sv s) {
  const unsigned char a = (unsigned char)s.front(), b = (unsigned char)s.back();
  return a > 0x20 && a < 0x80 && b > 0x20 && b < 0x80;
}
// dictionary lookup of a job value under containsString semantics (safety_policy.go:296-306): EqualFold(Trim(v), Trim(x))
inline uint32_t lookup_value(const Dict& d, sv raw) {
  if (raw.empty()) return CORDUM_ID_EMPTY;
  if (untrimmed_ok(raw) && is_ascii(raw)) return d.table.find_fold_ascii(raw, CORDUM_ID_OTHER);   // the common case: one pass, no copy
  FoldBuf f(raw);
  return d.table.find(f.view, CORDUM_ID_OTHER);
}

inline void set_bit(Bits& b, uint32_t r) { b[r >> 5] |= 1u << (r & 31); }
inline void or_bits(uint32_t* dst, const Bits& src) { for (size_t i = 0; i < src.size(); ++i) dst[i] |= src[i]; }

std::string json_quote(sv s) {
  std::string o = "\"";
  for (unsigned char c : s) {
    if (c == '"' || c == '\\') { o.push_back('\\'); o.push_back((char)c); }
    else if (c < 0x20) { char b[8]; snprintf(b, sizeof b, "\\u%04x", c); o += b; }
    else o.push_back((char)c);
  }
  o.push_back('"');
  return o;
}

void json_dump(const mjson::Value& v, std::string& o) {
  switch (v.kind) {
    case mjson::Kind::Null: o += "null"; break;
    case mjson::Kind::Bool: o += v.b ? "true" : "false"; break;
    case mjson::Kind::Number:
      if (v.is_int) o += std::to_string(v.i);
      else if (!std::isfinite(v.d)) o += v.d < 0 ? "-1e999" : "1e999";   // beyond double: still a JSON number
      else { char b[40]; snprintf(b, sizeof b, "%.17g", v.d); o += b; }
      break;
    case mjson::Kind::String: o += json_quote(v.s); break;
    case mjson::Kind::Array:
      o.push_back('[');
      for (size_t i = 0; i < v.arr.size(); ++i) { if (i) o.push_back(','); json_dump(v.arr[i], o); }
      o.push_back(']');
      break;
    case mjson::Kind::Object:
      o.push_back('{');
      for (size_t i = 0; i < v.obj.size(); ++i) {
        if (i) o.push_back(',');
        o += json_quote(v.obj[i].first);
        o.push_back(':');
        json_dump(v.obj[i].second, o);
      }
      o.push_back('}');
      break;
  }
}

bool get_strings(const mjson::Value* v, std::vector<std::string>& out, const char* what, std::string& err) {
  out.clear();
  if (!v || v->is_null()) return true;
  if (!v->is_arr()) { err = std::string(what) + " must be a list of strings"; return false; }
  for (auto& e : v->arr) {
    if (e.is_null()) out.emplace_back();
    else if (e.is_str()) out.push_back(e.s);
    else { err = std::string(what) + " must be a list of strings"; return false; }
  }
  return true;
}

const char* kMcpAllow[4] = {"allow_servers", "allow_tools", "allow_resources", "allow_actions"};
const char* kMcpDeny[4] = {"deny_servers", "deny_tools", "deny_resources", "deny_actions"};

bool get_mcp(const mjson::Value* v, McpLists& m, std::string& err) {
  if (!v || v->is_null()) return true;
  if (!v->is_obj()) { err = "mcp must be a mapping"; return false; }
  for (int f = 0; f < 4; ++f)
    if (!get_strings(v->get(kMcpAllow[f]), m.allow[f], kMcpAllow[f], err) ||
        !get_strings(v->get(kMcpDeny[f]), m.deny[f], kMcpDeny[f], err))
      return false;
  return true;
}

int64_t num_i(const mjson::Value* v) { return (v && v->is_num()) ? (v->is_int ? v->i : (int64_t)v->d) : 0; }
size_t arr_n(const mjson::Value* v) { return (v && v->is_arr()) ? v->arr.size() : 0; }
bool is_true(const mjson::Value* v) { return v && v->is_bool() && v->b; }

// isConstraintsEmpty, kernel.go:447-453
bool constraints_nonempty(const mjson::Value* c) {
  if (!c || !c->is_obj()) return false;
  const mjson::Value* b = c->get("budgets");
  if (b && b->is_obj() && (num_i(b->get("max_runtime_ms")) || num_i(b->get("max_retries")) ||
                           num_i(b->get("max_artifact_bytes")) || num_i(b->get("max_concurrent_jobs"))))
    return true;
  const mjson::Value* s = c->get("sandbox");
  if (s && s->is_obj() && (is_true(s->get("isolated")) || arr_n(s->get("network_allowlist")) ||
                           arr_n(s->get("fs_read_only")) || arr_n(s->get("fs_read_write"))))
    return true;
  const mjson::Value* t = c->get("toolchain");
  if (t && t->is_obj() && (arr_n(t->get("allowed_tools")) || arr_n(t->get("allowed_commands")))) return true;
  const mjson::Value* d = c->get("diff");
  if (d && d->is_obj() && (num_i(d->get("max_files")) || num_i(d->get("max_lines")) || arr_n(d->get("deny_path_globs"))))
    return true;
  const mjson::Value* r = c->get("redaction_level");
  if (r && r->is_str() && !trim_space(r->s).empty()) return true;
  return false;
}

}  // namespace

// ============================================================ document parsing
uint8_t normalize_decision_code(sv raw) {   // safety_policy.go:208-223
  std::string s = lower_key(raw);   // strings.ToLower(strings.TrimSpace(raw))
  if (s == "deny" || s == "block") return CORDUM_DEC_DENY;
  if (s == "require_approval" || s == "require-approval" || s == "require_human") return CORDUM_DEC_REQUIRE_HUMAN;
  if (s == "allow_with_constraints" || s == "allow-with-constraints") return CORDUM_DEC_ALLOW_WITH_CONSTRAINTS;
  if (s == "throttle") return CORDUM_DEC_THROTTLE;
  return CORDUM_DEC_ALLOW;   // allow | permit | anything else
}

bool parse_policy_json(sv text, PolicyModel& out, std::string& err) {
  out = PolicyModel{};
  if (text.empty()) return true;   // nil policy: allow-all (kernel.go:187)
  mjson::Value root;
  if (!mjson::parse(text, root, &err)) { err = "policy: " + err; return false; }
  if (root.is_null()) return true;
  if (!root.is_obj()) { err = "policy: expected a mapping"; return false; }
  out.nil = false;
  if (const mjson::Value* v = root.get("default_tenant"); v && v->is_str()) out.default_tenant = v->s;
  std::map<std::string, TenantModel> tenants;
  if (const mjson::Value* tv = root.get("tenants"); tv && tv->is_obj()) {
    for (auto& kv : tv->obj) {
      TenantModel t;
      t.name = kv.first;
      if (kv.second.is_obj()) {
        if (!get_strings(kv.second.get("allow_topics"), t.allow_topics, "allow_topics", err) ||
            !get_strings(kv.second.get("deny_topics"), t.deny_topics, "deny_topics", err) ||
            !get_mcp(kv.second.get("mcp"), t.mcp, err))
          return false;
      }
      tenants[kv.first] = std::move(t);
    }
  }
  for (auto& kv : tenants) out.tenants.push_back(std::move(kv.second));
  if (const mjson::Value* rv = root.get("rules"); rv && !rv->is_null()) {
    if (!rv->is_arr()) { err = "policy: rules must be a list"; return false; }
    for (auto& r : rv->arr) {
      if (!r.is_obj()) { err = "policy: rule must be a mapping"; return false; }
      RuleModel m;
      if (auto* v = r.get("id"); v && v->is_str()) m.id = v->s;
      if (auto* v = r.get("decision"); v && v->is_str()) m.decision = v->s;
      if (auto* v = r.get("reason"); v && v->is_str()) m.reason = v->s;
      if (const mjson::Value* mv = r.get("match"); mv && mv->is_obj()) {
        if (!get_strings(mv->get("tenants"), m.tenants, "tenants", err) ||
            !get_strings(mv->get("topics"), m.topics, "topics", err) ||
            !get_strings(mv->get("capabilities"), m.capabilities, "capabilities", err) ||
            !get_strings(mv->get("risk_tags"), m.risk_tags, "risk_tags", err) ||
            !get_strings(mv->get("requires"), m.requires_, "requires", err) ||
            !get_strings(mv->get("pack_ids"), m.pack_ids, "pack_ids", err) ||
            !get_strings(mv->get("actor_ids"), m.actor_ids, "actor_ids", err) ||
            !get_strings(mv->get("actor_types"), m.actor_types, "actor_types", err) ||
            !get_mcp(mv->get("mcp"), m.mcp, err))
          return false;
        if (auto* l = mv->get("labels"); l && l->is_obj()) {
          std::map<std::string, std::string> uniq;
          for (auto& kv : l->obj) uniq[kv.first] = kv.second.is_str() ? kv.second.s : std::string();
          m.labels.assign(uniq.begin(), uniq.end());
        }
        if (auto* s = mv->get("secrets_present"); s && s->is_bool()) m.secrets_present = s->b ? 1 : 0;
      }
      if (const mjson::Value* c = r.get("constraints")) {
        m.has_constraints = constraints_nonempty(c);
        if (!c->is_null()) json_dump(*c, m.constraints_json);
      }
      if (const mjson::Value* rm = r.get("remediations"); rm && rm->is_arr() && !rm->arr.empty())
        json_dump(*rm, m.remediations_json);
      out.rules.push_back(std::move(m));
    }
  }
  if (out.rules.empty()) {   // legacyRules, safety_policy.go:225-257 (tenants in sorted order)
    for (auto& t : out.tenants) {
      for (size_t i = 0; i < t.deny_topics.size(); ++i) {
        RuleModel m;
        m.id = "legacy:" + t.name + ":deny:" + std::to_string(i + 1);
        m.decision = "deny";
        m.reason = "topic " + go_quote(t.deny_topics[i]) + " denied by tenant policy";
        m.tenants = {t.name};
        m.topics = {t.deny_topics[i]};
        m.mcp = t.mcp;
        out.rules.push_back(std::move(m));
      }
      for (size_t i = 0; i < t.allow_topics.size(); ++i) {
        RuleModel m;
        m.id = "legacy:" + t.name + ":allow:" + std::to_string(i + 1);
        m.decision = "allow";
        m.tenants = {t.name};
        m.topics = {t.allow_topics[i]};
        m.mcp = t.mcp;
        out.rules.push_back(std::move(m));
      }
    }
  }
  return true;
}

bool parse_routing_json(sv text, RoutingModel& out, std::string& err) {
  out = RoutingModel{};
  if (text.empty()) return true;
  mjson::Value root;
  if (!mjson::parse(text, root, &err)) { err = "routing: " + err; return false; }
  if (root.is_null()) return true;
  if (!root.is_obj()) { err = "routing: expected a mapping"; return false; }
  if (const mjson::Value* t = root.get("topics"); t && t->is_obj()) {
    std::map<std::string, std::vector<std::string>> uniq;
    for (auto& kv : t->obj) {
      std::vector<std::string> pools;
      if (kv.second.is_str()) pools.push_back(kv.second.s);   // pools.go:107-111 single-pool form
      else if (!get_strings(&kv.second, pools, "topic pools", err)) return false;
      uniq[kv.first] = std::move(pools);
    }
    out.topics.assign(uniq.begin(), uniq.end());
  }
  if (const mjson::Value* p = root.get("pools"); p && p->is_obj()) {
    std::map<std::string, std::vector<std::string>> uniq;
    for (auto& kv : p->obj) {
      std::vector<std::string> req;
      if (kv.second.is_obj() && !get_strings(kv.second.get("requires"), req, "requires", err)) return false;
      uniq[kv.first] = std::move(req);
    }
    out.pools.assign(uniq.begin(), uniq.end());
  }
  return true;
}

// ---- effective.go:12-39 with encoding/json typing (field names match case-insensitively;
//      any field of the wrong JSON type makes that Unmarshal fail)
namespace {
bool eff_list(const mjson::Value& v, std::vector<std::string>* dst) {
  if (v.is_null()) { if (dst) dst->clear(); return true; }
  if (!v.is_arr()) return false;
  bool ok = true;
  std::vector<std::string> tmp;
  for (auto& e : v.arr) {
    if (e.is_str()) tmp.push_back(e.s);
    else { tmp.emplace_back(); if (!e.is_null()) ok = false; }
  }
  if (dst) *dst = std::move(tmp);
  return ok;
}
int name_index(sv key, const char* const* names, int n) {
  for (int i = 0; i < n; ++i) if (key == names[i]) return i;
  for (int i = 0; i < n; ++i) if (fold_eq(key, names[i])) return i;
  return -1;
}
bool eff_mcp(const mjson::Value& v, McpLists& m) {
  if (v.is_null()) return true;
  if (!v.is_obj()) return false;
  static const char* names[8] = {"allow_servers", "deny_servers", "allow_tools", "deny_tools",
                                 "allow_resources", "deny_resources", "allow_actions", "deny_actions"};
  bool ok = true;
  for (auto& kv : v.obj) {
    int f = name_index(kv.first, names, 8);
    if (f < 0) continue;
    std::vector<std::string>* dst = (f & 1) ? &m.deny[f >> 1] : &m.allow[f >> 1];
    if (!eff_list(kv.second, dst)) ok = false;
  }
  return ok;
}
bool eff_struct(const mjson::Value& v, EffSafety& cfg) {
  cfg = EffSafety{};
  if (v.is_null()) return true;
  if (!v.is_obj()) return false;
  // categories.go:6-35 — kinds: b bool, s string, l []string, m map[string]float64, p MCPPolicy
  static const char* names[16] = {"pii_detection_enabled", "pii_action", "pii_types", "allowed_email_domains",
                                  "injection_detection", "injection_action", "injection_sensitivity",
                                  "content_filter_enabled", "blocked_categories", "anomaly_detection",
                                  "anomaly_thresholds", "allowed_topics", "denied_topics", "allowed_repo_hosts",
                                  "denied_repo_hosts", "mcp"};
  static const char kinds[17] = "bsllbssblbmllllp";
  bool ok = true;
  for (auto& kv : v.obj) {
    int f = name_index(kv.first, names, 16);
    if (f < 0) continue;
    const mjson::Value& x = kv.second;
    switch (kinds[f]) {
      case 'b': if (!x.is_null() && !x.is_bool()) ok = false; break;
      case 's': if (!x.is_null() && !x.is_str()) ok = false; break;
      case 'l':
        if (!eff_list(x, f == 11 ? &cfg.allowed_topics : f == 12 ? &cfg.denied_topics : nullptr)) ok = false;
        break;
      case 'm':
        if (x.is_null()) break;
        if (!x.is_obj()) { ok = false; break; }
        for (auto& e : x.obj) if (!e.second.is_null() && !(e.second.is_num() && std::isfinite(e.second.d))) ok = false;   // float64 out of range: the Unmarshal fails
        break;
      case 'p': if (!eff_mcp(x, cfg.mcp)) ok = false; break;
    }
  }
  return ok;
}
}  // namespace

bool parse_effective_safety(sv payload, EffSafety& out) {
  out = EffSafety{};
  if (payload.empty()) return false;
  mjson::Value top;
  if (!mjson::parse(payload, top) || !top.is_obj()) return false;
  if (const mjson::Value* raw = top.get("safety"))
    if (eff_struct(*raw, out)) return true;
  if (const mjson::Value* data = top.get("data"); data && data->is_obj())
    if (const mjson::Value* raw = data->get("safety"))
      if (eff_struct(*raw, out)) return true;
  out = EffSafety{};
  return false;
}

bool json_canon(sv text, std::string& out) {   // test hook: parse with the product's JSON reader, dump the tree
  mjson::Value v;
  if (!mjson::parse(text, v)) return false;
  out.clear();
  json_dump(v, out);
  return true;
}

int test_glob(sv pattern, sv name) {
  Glob g(pattern);
  if (!g.valid()) return -1;
  return g.match(name) ? 1 : 0;
}

// ============================================================ WorkPool
WorkPool::WorkPool(uint32_t threads) {
  for (uint32_t i = 1; i < threads; ++i) threads_.emplace_back([this, i]() { worker(i); });
}
WorkPool::~WorkPool() {
  { std::lock_guard<std::mutex> g(mu_); stop_ = true; }
  cv_.notify_all();
  for (auto& t : threads_) t.join();
}
void WorkPool::drain(Job& j, uint32_t id) {
  while (true) {
    uint32_t b = j.next.fetch_add(j.grain, std::memory_order_relaxed);
    if (b >= j.n) break;
    uint32_t e = std::min(j.n, b + j.grain);
    (*j.fn)(b, e, id);
    j.done.fetch_add(e - b, std::memory_order_release);
  }
}
void WorkPool::worker(uint32_t id) {
  uint64_t seen = 0;
  while (true) {
    std::shared_ptr<Job> job;
    {
      std::unique_lock<std::mutex> g(mu_);
      cv_.wait(g, [&]() { return stop_ || epoch_ != seen; });
      if (stop_) return;
      seen = epoch_;
      job = current_;
    }
    if (job) drain(*job, id);   // a late waker finds the queue empty and goes back to sleep
  }
}
void WorkPool::parallel_for(uint32_t n, uint32_t grain, const Fn& fn) {
  auto job = std::make_shared<Job>();
  job->fn = &fn; job->n = n; job->grain = grain ? grain : 1;
  { std::lock_guard<std::mutex> g(mu_); current_ = job; ++epoch_; }
  cv_.notify_all();
  drain(*job, 0);   // the caller works too
  while (job->done.load(std::memory_order_acquire) < n) std::this_thread::yield();   // only chunks still in flight
}

// ============================================================ Host
Host::Host(uint32_t max_topics, uint32_t max_effcfgs, uint32_t encode_threads)
    : max_topics_(max_topics ? max_topics : 65536), max_effcfgs_(std::min<uint32_t>(max_effcfgs ? max_effcfgs : 4096, CORDUM_ID16_MAX)) {
  unsigned hw = std::thread::hardware_concurrency();
  threads_ = encode_threads ? encode_threads : (hw ? hw : 4);
  if (!encode_threads) {
    // Containers: more busy threads than the CPU quota only buys CFS throttling stalls.
    double quota = 0;
    if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {                       // cgroup v2: "<quota|max> <period>"
      char q[32]; long per = 0;
      if (fscanf(f, "%31s %ld", q, &per) == 2 && per > 0 && q[0] != 'm') quota = atof(q) / (double)per;
      fclose(f);
    } else {
      long q = -1, per = 0;                                                      // cgroup v1
      if (FILE* a = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) { if (fscanf(a, "%ld", &q) != 1) q = -1; fclose(a); }
      if (FILE* b = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) { if (fscanf(b, "%ld", &per) != 1) per = 0; fclose(b); }
      if (q > 0 && per > 0) quota = (double)q / (double)per;
    }
    if (quota >= 1.0 && quota < threads_) threads_ = (uint32_t)(quota + 0.5);
  }
  if (threads_ > 64) threads_ = 64;
  std::string err;
  compile_policy();
  compile_routing();
  compile_mcp_tables();
  rebuild_topics();
  load_workers(nullptr, err);
}

// ------------------------------------------------------------ policy compile
void Host::compile_policy() {
  HostTables& t = t_;
  const auto& rules = policy_.rules;
  const uint32_t R = (uint32_t)rules.size();
  t.n_rules = R;
  // ---- bit positions.  A rule's bit does not sit at its index.  Each rule gets one position per distinct topic
  // pattern it lists (one position if it has none): the copy for pattern p carries the rule's other predicates
  // unchanged but only p's topic bits.  Positions are then ordered so that the rules a given job can match share
  // few 128-bit words: rules without a topic predicate first, the rest clustered by the literal "job.<pack>" prefix
  // of the pattern.  A cluster larger than one word (typically the rules without a topic predicate) is clustered a
  // second time by tenant: a rule that lists 1..kTenantSplit tenants gets one copy per tenant there, carrying only
  // that tenant's bit, so a tenant's row is sparse inside the cluster too.  First-match is recovered as the minimum
  // ORIGINAL rule index over the surviving bits (pos2rule), so duplicates and any ordering are harmless; a good
  // ordering makes the rows sparse at word granularity, which the per-row summaries (sum_*) expose to the kernel.
  constexpr size_t kTenantSplit = 8;
  struct Entry { uint32_t rule; int32_t pat; std::string key, tsub, tenant; };   // pat = index into rules[rule].topics, -1 = none
  std::vector<Entry> entries;
  for (uint32_t r = 0; r < R; ++r) {
    if (rules[r].topics.empty()) { entries.push_back({r, -1, std::string(), {}, {}}); continue; }
    std::vector<std::string> seen;
    for (size_t k = 0; k < rules[r].topics.size(); ++k) {
      sv pt = trim_space(rules[r].topics[k]);
      if (pt.empty()) continue;   // matchTopic: an empty pattern never matches
      if (std::find(seen.begin(), seen.end(), std::string(pt)) != seen.end()) continue;
      seen.emplace_back(pt);
      size_t cut = pt.find_first_of("*?[\\");
      sv lit = pt.substr(0, cut == sv::npos ? pt.size() : cut);
      size_t d1 = lit.find('.'), d2 = d1 == sv::npos ? sv::npos : lit.find('.', d1 + 1);
      std::string key(d2 == sv::npos ? lit : lit.substr(0, d2));
      entries.push_back({r, (int32_t)k, "\x02" + key, {}, {}});
    }
    if (seen.empty()) entries.push_back({r, -2, "\x01", {}, {}});   // only blank patterns: the rule can never match a topic
  }
  std::stable_sort(entries.begin(), entries.end(), [](const Entry& x, const Entry& y) { return x.key < y.key; });
  {   // second-level clustering by tenant inside clusters that span more than one word
    std::vector<Entry> out;
    out.reserve(entries.size());
    for (size_t g0 = 0; g0 < entries.size();) {
      size_t g1 = g0;
      while (g1 < entries.size() && entries[g1].key == entries[g0].key) ++g1;
      const size_t first = out.size();
      for (size_t i = g0; i < g1; ++i) {
        const Entry& e = entries[i];
        std::vector<std::string> ten;
        for (auto& v : rules[e.rule].tenants) {
          std::string f = fold_key(v);
          if (std::find(ten.begin(), ten.end(), f) == ten.end()) ten.push_back(std::move(f));
        }
        if (g1 - g0 <= 128 || ten.empty()) out.push_back({e.rule, e.pat, e.key, ten.empty() ? "" : "\x02", {}});
        else if (ten.size() > kTenantSplit) out.push_back({e.rule, e.pat, e.key, "\x02", {}});
        else for (auto& f : ten) out.push_back({e.rule, e.pat, e.key, "\x01" + f, f});
      }
      std::stable_sort(out.begin() + first, out.end(), [](const Entry& x, const Entry& y) { return x.tsub < y.tsub; });
      g0 = g1;
    }
    entries.swap(out);
  }
  // Word alignment: a cluster (or, inside a tenant-split cluster, one tenant's sub-cluster) that fits into one 128-bit
  // word is never laid across a word boundary - padding positions (no rule) fill the gap - so a job touches ONE word per
  // cluster it can match in.  Padding costs a few per cent of row length and saves a word per straddle.
  constexpr uint32_t kPad = 0xFFFFFFFFu;
  {
    std::vector<Entry> out;
    out.reserve(entries.size() + entries.size() / 8);
    for (size_t g0 = 0; g0 < entries.size();) {
      size_t g1 = g0;
      while (g1 < entries.size() && entries[g1].key == entries[g0].key) ++g1;
      auto place = [&](size_t a, size_t b) {   // unit [a, b): keep inside one word if it fits
        const size_t n = b - a, at = out.size() % 128;
        if (n <= 128 && at + n > 128) out.resize(out.size() + (128 - at), Entry{kPad, -3, {}, {}, {}});
        out.insert(out.end(), entries.begin() + (long)a, entries.begin() + (long)b);
      };
      if (g1 - g0 <= 128) place(g0, g1);
      else
        for (size_t u0 = g0; u0 < g1;) {
          size_t u1 = u0;
          while (u1 < g1 && entries[u1].tsub == entries[u0].tsub) ++u1;
          place(u0, u1);
          u0 = u1;
        }
      g0 = g1;
    }
    entries.swap(out);
  }
  const uint32_t NP = (uint32_t)entries.size();
  // Inside one 128-bit word the positions are put in ascending rule order (which words a job touches does not depend
  // on the order inside a word): the lowest surviving bit of a word is then that word's first match, and the kernel
  // looks at further bits only when a requires / labels subset test fails.  Padding sorts to the end of its word.
  for (uint32_t w0 = 0; w0 < NP; w0 += 128u)
    std::stable_sort(entries.begin() + w0, entries.begin() + std::min<uint32_t>(NP, w0 + 128u),
                     [](const Entry& x, const Entry& y) { return x.rule < y.rule; });
  t.n_seg = std::max<uint32_t>(1, (NP + CORDUM_SEG_RULES - 1) / CORDUM_SEG_RULES);
  t.row_words = t.n_seg * 32;
  t.sum_group = (t.n_seg * CORDUM_SEG_U4 + 63) / 64;
  const uint32_t W = t.row_words;
  rule_pos_.assign(R, {});
  rule_pos_tenant_.assign(R, {});
  t.pos2rule.assign((size_t)t.n_seg * CORDUM_SEG_RULES, 0xFFFFFFFFu);
  for (uint32_t p = 0; p < NP; ++p) {
    if (entries[p].rule == kPad) continue;
    rule_pos_[entries[p].rule].push_back(p);
    rule_pos_tenant_[entries[p].rule].push_back(entries[p].tenant);
    t.pos2rule[p] = entries[p].rule;
  }
  auto set_rule = [&](uint32_t* row, uint32_t r) { for (uint32_t p : rule_pos_[r]) row[p >> 5] |= 1u << (p & 31); };
  d_tenant_.clear(); d_cap_.clear(); d_pack_.clear(); d_actor_.clear(); d_risk_.clear();
  for (auto& d : d_mcp_) d.clear();
  d_req_.clear();
  tenant_pol_.clear(); label_key_.clear(); label_key_pairs_.clear(); label_empty_mask_ = 0;
  patterns_.clear();
  pat_by_prefix_.clear();
  default_tenant_trim_ = std::string(trim_space(policy_.default_tenant));
  for (size_t i = 0; i < policy_.tenants.size(); ++i) tenant_pol_.put(policy_.tenants[i].name, (uint32_t)i + 1);

  // requires dictionary is shared with the pools: rule tokens first, then pool tokens
  auto scalar_rows = [&](Dict& d, RowTable& rt, auto list_of) {
    Bits vac(W, 0);
    std::vector<std::vector<uint32_t>> hits;   // hits[id-2] = rules
    for (uint32_t r = 0; r < R; ++r) {
      const std::vector<std::string>& lst = list_of(rules[r]);
      if (lst.empty()) { set_rule(vac.data(), r); continue; }
      for (auto& e : lst) {
        uint32_t id = d.intern(fold_key(e));
        if (hits.size() < id - 1) hits.resize(id - 1);
        hits[id - 2].push_back(r);
      }
    }
    rt.init(d.size(), W);
    for (uint32_t id = 0; id < d.size(); ++id) {
      uint32_t* row = rt.row(id);
      or_bits(row, vac);
      if (id >= 2 && id - 2 < hits.size())
        for (uint32_t r : hits[id - 2]) set_rule(row, r);
    }
  };
  {   // tenants: like scalar_rows, except that a position may stand for ONE of the rule's tenants (see above)
    Dict& d = d_tenant_;
    Bits vac(W, 0);
    std::vector<std::vector<uint32_t>> hits;   // hits[id-2] = bit positions
    for (uint32_t r = 0; r < R; ++r) {
      if (rules[r].tenants.empty()) { set_rule(vac.data(), r); continue; }
      for (auto& e : rules[r].tenants) {
        std::string f = fold_key(e);
        uint32_t id = d.intern(f);
        if (hits.size() < id - 1) hits.resize(id - 1);
        for (size_t k = 0; k < rule_pos_[r].size(); ++k)
          if (rule_pos_tenant_[r][k].empty() || rule_pos_tenant_[r][k] == f) hits[id - 2].push_back(rule_pos_[r][k]);
      }
    }
    t.row_tenant.init(d.size(), W);
    for (uint32_t id = 0; id < d.size(); ++id) {
      uint32_t* row = t.row_tenant.row(id);
      or_bits(row, vac);
      if (id >= 2 && id - 2 < hits.size())
        for (uint32_t p : hits[id - 2]) row[p >> 5] |= 1u << (p & 31);
    }
    // Tenant class = which word group holds the tenant's first per-tenant copy.  The encoder sorts jobs by (topic,
    // class), so the lanes of a warp agree not only on their topic's words but also on their tenants' word.
    std::vector<uint32_t> first_group(d.size(), 0xFFFFFFFFu);
    std::vector<uint32_t> groups;   // distinct word groups that hold per-tenant copies, ascending
    for (uint32_t p = 0; p < NP; ++p) {
      if (entries[p].rule == kPad || entries[p].tenant.empty()) continue;
      const uint32_t id = d.table.find(entries[p].tenant, 0), g = (p / 128u) / t.sum_group;
      if (id < first_group.size()) first_group[id] = std::min(first_group[id], g);
      if (groups.empty() || groups.back() != g) groups.push_back(g);
    }
    std::sort(groups.begin(), groups.end());
    groups.erase(std::unique(groups.begin(), groups.end()), groups.end());
    tenant_classes_ = std::min<uint32_t>(kMaxTenantClasses, (uint32_t)groups.size() + 1);
    tenant_class_.assign(d.size(), 0);
    for (uint32_t id = 0; id < d.size(); ++id)
      if (first_group[id] != 0xFFFFFFFFu) {
        const uint32_t rank = (uint32_t)(std::lower_bound(groups.begin(), groups.end(), first_group[id]) - groups.begin());
        tenant_class_[id] = (uint8_t)std::min<uint32_t>(1 + rank, tenant_classes_ - 1);
      }
  }
  scalar_rows(d_cap_, t.row_cap, [](const RuleModel& m) -> const std::vector<std::string>& { return m.capabilities; });
  scalar_rows(d_pack_, t.row_pack, [](const RuleModel& m) -> const std::vector<std::string>& { return m.pack_ids; });
  scalar_rows(d_actor_, t.row_actor, [](const RuleModel& m) -> const std::vector<std::string>& { return m.actor_ids; });

  // risk tags: containsAny (safety_policy.go:308-318) -> OR of per-tag rows
  {
    Bits vac(W, 0);
    std::vector<std::vector<uint32_t>> hits;
    for (uint32_t r = 0; r < R; ++r) {
      if (rules[r].risk_tags.empty()) { set_rule(vac.data(), r); continue; }
      for (auto& e : rules[r].risk_tags) {
        uint32_t id = d_risk_.intern(fold_key(e));
        if (hits.size() < id - 1) hits.resize(id - 1);
        hits[id - 2].push_back(r);
      }
    }
    uint32_t nb = d_risk_.size() - 2;
    t.row_risk.init(1 + nb, W);
    or_bits(t.row_risk.row(0), vac);
    for (uint32_t b = 0; b < nb; ++b) {
      uint32_t* row = t.row_risk.row(1 + b);
      or_bits(row, vac);
      if (b < hits.size()) for (uint32_t r : hits[b]) set_rule(row, r);
    }
  }

  // topics: distinct trimmed patterns
  vac_topic_.assign(W, 0);
  {
    std::unordered_map<std::string, uint32_t> idx;
    for (uint32_t p = 0; p < NP; ++p) {
      const Entry& e = entries[p];
      if (e.pat == -1) { set_bit(vac_topic_, p); continue; }   // no topic predicate
      if (e.pat < 0) continue;                                 // only blank patterns
      sv pt = trim_space(rules[e.rule].topics[(size_t)e.pat]);
      auto it = idx.find(std::string(pt));
      if (it == idx.end()) {
        it = idx.emplace(std::string(pt), (uint32_t)patterns_.size()).first;
        // index by literal prefix (the bytes before the first metacharacter): a topic can only match patterns whose
        // literal prefix is a prefix of it, which turns 4k patterns x 2k topics of glob matching into a few per topic
        size_t lit = 0;
        while (lit < pt.size() && pt[lit] != '*' && pt[lit] != '?' && pt[lit] != '[' && pt[lit] != '\\') ++lit;
        pat_by_prefix_[std::string(pt.substr(0, lit))].push_back((uint32_t)patterns_.size());
        patterns_.push_back(Pattern{Glob(pt), {}});
      }
      patterns_[it->second].rules.push_back(p);   // bit positions
    }
  }

  // per-rule columns: decision, requires / labels need-masks, alive
  t.rule_dec.assign((size_t)t.n_seg * CORDUM_SEG_RULES, 0);
  t.rule_req_need.assign((size_t)t.n_seg * CORDUM_SEG_RULES, 0);
  t.rule_lab_need.assign((size_t)t.n_seg * CORDUM_SEG_RULES, 0);
  Bits alive(W, 0), check(W, 0);
  uint32_t n_pairs = 0;
  rule_req_ids_.assign(R, {});
  rule_lab_bits_.assign(R, {});
  label_empty_x_.clear();
  for (uint32_t r = 0; r < R; ++r) {
    const RuleModel& m = rules[r];
    t.rule_dec[r] = normalize_decision_code(m.decision) | (m.has_constraints ? 0x80 : 0);
    bool dead = false;
    uint64_t need = 0;
    for (auto& q : m.requires_) {
      if (q.empty()) { dead = true; continue; }   // containsString(values, "") is always false (:297)
      uint32_t id = d_req_.intern(fold_key(q));
      need |= (id - 2 < 64) ? (1ull << (id - 2)) : 0;
      rule_req_ids_[r].push_back(id - 2);          // bits beyond 63 go to rule_need_x (finalize_wide)
    }
    t.rule_req_need[r] = need;
    uint64_t lneed = 0;
    for (auto& kv : m.labels) {
      uint32_t ki = label_key_.find(kv.first, kMiss);
      if (ki == kMiss) { ki = (uint32_t)label_key_pairs_.size(); label_key_.put(kv.first, ki); label_key_pairs_.emplace_back(); }
      auto& pairs = label_key_pairs_[ki];
      uint32_t bit = kMiss;
      for (auto& pv : pairs) if (pv.first == kv.second) bit = pv.second;
      if (bit == kMiss) {
        bit = n_pairs++;
        pairs.emplace_back(kv.second, bit);
        if (kv.second.empty()) {
          if (bit < 64) label_empty_mask_ |= 1ull << bit;
          else { if (label_empty_x_.size() < (bit >> 6)) label_empty_x_.resize(bit >> 6, 0); label_empty_x_[(bit >> 6) - 1] |= 1ull << (bit & 63); }
        }
      }
      if (bit < 64) lneed |= 1ull << bit;
      rule_lab_bits_[r].push_back(bit);
    }
    t.rule_lab_need[r] = lneed;
    if (!dead) set_rule(alive.data(), r);
    if (!rule_req_ids_[r].empty() || !rule_lab_bits_[r].empty()) set_rule(check.data(), r);
  }
  n_label_pairs_ = n_pairs;
  policy_capacity_error_.clear();
  if (std::max({d_tenant_.size(), d_cap_.size(), d_pack_.size(), d_actor_.size()}) > CORDUM_ID16_MAX ||
      policy_.tenants.size() >= CORDUM_ID16_MAX)
    policy_capacity_error_ = "more than 65535 distinct values referenced by one predicate (tenants / capabilities / pack_ids / actor_ids)";
  t.row_check.init(1, W);
  or_bits(t.row_check.row(0), check);

  // combo rows: (actor_type in {"", human, service}) x secrets_present x "job has none of the requires tokens rules
  // list" x "job has none of the label pairs rules list", ANDed with the alive mask.  The last two settle the subset
  // tests of most jobs inside the row AND; what they leave is verified per surviving bit (row_check).
  t.row_combo.init(CORDUM_COMBO_ROWS, W);
  static const char* at_names[3] = {"", "human", "service"};
  for (uint32_t c = 0; c < CORDUM_COMBO_ROWS; ++c) {
    const int at = (int)(c % 6) / 2, s = (int)(c % 2);
    const bool no_req = (c / 6) & 1, no_lab = (c / 12) & 1;
    uint32_t* row = t.row_combo.row(c);
    for (uint32_t r = 0; r < R; ++r) {
      const RuleModel& m = rules[r];
      bool ok = true;
      if (!m.actor_types.empty()) {
        ok = false;
        if (at != 0)
          for (auto& e : m.actor_types) if (fold_key(e) == at_names[at]) ok = true;
      }
      if (m.secrets_present >= 0 && (m.secrets_present == 1) != (s == 1)) ok = false;
      if ((no_req && !rule_req_ids_[r].empty()) || (no_lab && !rule_lab_bits_[r].empty())) ok = false;
      if (ok) for (uint32_t p : rule_pos_[r]) if (alive[p >> 5] >> (p & 31) & 1) row[p >> 5] |= 1u << (p & 31);
    }
  }
  // summaries: which word groups of a row hold any bit.  An attribute's summaries are worth a gather per job only if
  // its rows are sparse at that granularity (topic always is; tenant once the topic-free rules are clustered by it).
  summarize(t.row_tenant, t.sum_tenant); summarize(t.row_cap, t.sum_cap); summarize(t.row_pack, t.sum_pack);
  summarize(t.row_actor, t.sum_actor); summarize(t.row_combo, t.sum_combo); summarize(t.row_risk, t.sum_risk);
  t.sum_use = 0;   // chosen by choose_summaries() once the topic rows exist (rebuild_topics)
  t.v_policy++;
}

// Which attributes' summaries are worth a gather per job: those that remove live words from what the topic's summary
// leaves.  Estimated on a sample of (topic, value) pairs: expected popcount(sum_topic & sum_attr) against
// popcount(sum_topic).  The topic summary is always used; tenant pays once the topic-free rules are clustered by tenant.
void Host::choose_summaries() {
  HostTables& t = t_;
  t.sum_use = 0;
  const size_t nt = t.sum_topic.size();
  if (nt == 0) return;
  const size_t tstep = std::max<size_t>(1, nt / 256);
  auto gain = [&](const std::vector<uint64_t>& sums) {
    if (sums.empty()) return false;
    const size_t vstep = std::max<size_t>(1, sums.size() / 512);
    uint64_t base = 0, with = 0;
    for (size_t i = 0; i < nt; i += tstep)
      for (size_t v = 0; v < sums.size(); v += vstep) {
        base += (uint64_t)__builtin_popcountll(t.sum_topic[i]);
        with += (uint64_t)__builtin_popcountll(t.sum_topic[i] & sums[v]);
      }
    return base > 0 && (double)with < 0.85 * (double)base;
  };
  if (gain(t.sum_tenant)) t.sum_use |= SUM_TENANT;
  if (gain(t.sum_cap)) t.sum_use |= SUM_CAP;
  if (gain(t.sum_pack)) t.sum_use |= SUM_PACK;
  if (gain(t.sum_actor)) t.sum_use |= SUM_ACTOR;
  if (gain(t.sum_combo)) t.sum_use |= SUM_COMBO;
  if (gain(t.sum_risk)) t.sum_use |= SUM_RISK;
  if (const char* v = getenv("CORDUM_SUM_USE")) t.sum_use = (uint32_t)atoi(v);   // tuning / test knob
}

uint64_t Host::row_summary(const uint32_t* row) const {
  const uint32_t gw = t_.sum_group * 4, n = t_.row_words / gw + (t_.row_words % gw ? 1 : 0);
  uint64_t m = 0;
  for (uint32_t g = 0; g < n; ++g) {
    uint32_t any = 0;
    for (uint32_t k = g * gw; k < std::min(t_.row_words, (g + 1) * gw); ++k) any |= row[k];
    if (any) m |= 1ull << g;
  }
  return m;
}
void Host::summarize(const RowTable& rt, std::vector<uint64_t>& out) const {
  out.assign(std::max<uint32_t>(rt.n_rows, 1), 0);
  for (uint32_t r = 0; r < rt.n_rows; ++r) out[r] = row_summary(rt.row(r));
}

// ------------------------------------------------------------ routing compile
void Host::compile_routing() {
  HostTables& t = t_;
  d_pool_.clear();
  routing_topics_.clear();
  for (auto& p : routing_.pools) d_pool_.intern(p.first);
  for (size_t i = 0; i < routing_.topics.size(); ++i) {
    routing_topics_.put(routing_.topics[i].first, (uint32_t)i);
    for (auto& p : routing_.topics[i].second) d_pool_.intern(p);
  }
  t.n_pools = d_pool_.size() - 2;
  t.pool_req_mask.assign(std::max<uint32_t>(t.n_pools, 1), 0);
  t.pool_req_nonempty.assign(std::max<uint32_t>(t.n_pools, 1), 0);
  pool_req_ids_.assign(std::max<uint32_t>(t.n_pools, 1), {});
  for (auto& p : routing_.pools) {
    uint32_t pid = d_pool_.table.find(p.first, 0) - 2;
    t.pool_req_nonempty[pid] = p.second.empty() ? 0 : 1;   // poolSatisfies: len(poolRequires)==0 -> false (:245)
    uint64_t mask = 0;
    for (auto& q : p.second) {
      std::string k = lower_key(q);   // ToLower(TrimSpace(req)) (:250); blank tokens are dropped (:251)
      if (k.empty()) continue;
      uint32_t id = d_req_.intern(k);
      if (id - 2 < 64) mask |= 1ull << (id - 2);
      pool_req_ids_[pid].push_back(id - 2);
    }
    t.pool_req_mask[pid] = mask;
  }
  routing_capacity_error_.clear();
  uint32_t blank = d_req_.table.find(sv(), 0);
  t.req_blank_mask = (blank >= 2 && blank - 2 < 64) ? (1ull << (blank - 2)) : 0;
  finalize_wide();
  t.v_routing++;
}

// The dictionaries are final here (compile_policy, then compile_routing): how many mask words beyond the records' own does
// a job need, and the rules' / pools' bits that live there.  Placement width belongs to the registry (compile_workers).
void Host::finalize_wide() {
  HostTables& t = t_;
  auto extra = [](uint32_t nbits, uint32_t base) { const uint32_t w = (nbits + 63) / 64; return w > base ? w - base : 0u; };
  t.wide.xw_risk = extra(d_risk_.size() - 2, 1);
  t.wide.xw_req = extra(d_req_.size() - 2, 1);
  t.wide.xw_lab = extra(n_label_pairs_, 1);
  const uint32_t xq = t.wide.xw_req, xl = t.wide.xw_lab, R = (uint32_t)policy_.rules.size();
  t.rule_need_x.assign((size_t)std::max<uint32_t>(R, 1) * (xq + xl) + 1, 0);
  for (uint32_t r = 0; r < R && r < rule_req_ids_.size(); ++r) {
    uint64_t* row = t.rule_need_x.data() + (size_t)r * (xq + xl);
    for (uint32_t b : rule_req_ids_[r]) if (b >= 64) row[(b >> 6) - 1] |= 1ull << (b & 63);
    for (uint32_t b : rule_lab_bits_[r]) if (b >= 64) row[xq + (b >> 6) - 1] |= 1ull << (b & 63);
  }
  t.pool_req_x.assign((size_t)std::max<uint32_t>(t.n_pools, 1) * xq + 1, 0);
  for (uint32_t p = 0; p < pool_req_ids_.size(); ++p)
    for (uint32_t b : pool_req_ids_[p]) if (b >= 64) t.pool_req_x[(size_t)p * xq + (b >> 6) - 1] |= 1ull << (b & 63);
  t.req_blank_x.assign(xq + 1, 0);
  const uint32_t blank = d_req_.table.find(sv(), 0);
  if (blank >= 2 && blank - 2 >= 64) t.req_blank_x[((blank - 2) >> 6) - 1] |= 1ull << ((blank - 2) & 63);
  label_empty_x_.resize(xl, 0);
  t.v_policy++;   // rule_need_x travels with the policy group
}

// ------------------------------------------------------------ MCP tables (rule rows, tenant + effective-config verdicts)
void Host::compile_mcp_tables() {
  HostTables& t = t_;
  const auto& rules = policy_.rules;
  const uint32_t R = (uint32_t)rules.size(), W = t.row_words;
  // intern every referenced value first so ids are final
  auto intern_lists = [&](const McpLists& m) {
    for (int f = 0; f < 4; ++f) {
      for (auto& e : m.allow[f]) d_mcp_[f].intern(fold_key(e));
      for (auto& e : m.deny[f]) d_mcp_[f].intern(fold_key(e));
    }
  };
  for (auto& r : rules) intern_lists(r.mcp);
  for (auto& tn : policy_.tenants) intern_lists(tn.mcp);
  for (size_t i = 1; i < effcfgs_.size(); ++i) intern_lists(effcfgs_[i].mcp);
  uint32_t stride = 2;
  for (int f = 0; f < 4; ++f) stride = std::max(stride, d_mcp_[f].size());
  t.mcp_stride = stride;
  // rule rows: bit r = value not denied by r and (r has no allow list or value in it)  (:408-416)
  for (int f = 0; f < 4; ++f) {
    Dict& d = d_mcp_[f];
    Bits base(W, 0);
    std::vector<std::vector<uint32_t>> allow_hits(d.size()), deny_hits(d.size());
    for (uint32_t r = 0; r < R; ++r) {
      const McpLists& m = rules[r].mcp;
      if (m.allow[f].empty()) for (uint32_t p : rule_pos_[r]) set_bit(base, p);
      for (auto& e : m.allow[f]) allow_hits[d.table.find(fold_key(e), 0)].push_back(r);
      for (auto& e : m.deny[f]) deny_hits[d.table.find(fold_key(e), 0)].push_back(r);
    }
    t.row_mcp[f].init(d.size(), W);
    for (uint32_t id = 0; id < d.size(); ++id) {
      uint32_t* row = t.row_mcp[f].row(id);
      or_bits(row, base);
      if (id >= 2) {
        for (uint32_t r : allow_hits[id]) for (uint32_t p : rule_pos_[r]) row[p >> 5] |= 1u << (p & 31);
        for (uint32_t r : deny_hits[id]) for (uint32_t p : rule_pos_[r]) row[p >> 5] &= ~(1u << (p & 31));
      }
    }
  }
  auto verdicts = [&](const McpLists& m, uint8_t* dst) {   // dst[4][stride]
    for (int f = 0; f < 4; ++f) {
      std::set<uint32_t> allow, deny;
      for (auto& e : m.allow[f]) allow.insert(d_mcp_[f].table.find(fold_key(e), 0));
      for (auto& e : m.deny[f]) deny.insert(d_mcp_[f].table.find(fold_key(e), 0));
      for (uint32_t id = 0; id < stride; ++id) {
        uint8_t v = 0;
        bool named = id >= 2;
        if (named && deny.count(id)) v = 1;
        else if (!m.allow[f].empty() && !(named && allow.count(id))) v = 2;
        dst[(size_t)f * stride + id] = v;
      }
    }
  };
  size_t nt = std::max<size_t>(policy_.tenants.size(), 1);
  t.tenant_mcp.assign(nt * 4 * stride, 0);
  for (size_t i = 0; i < policy_.tenants.size(); ++i) verdicts(policy_.tenants[i].mcp, &t.tenant_mcp[i * 4 * stride]);
  t.n_effcfg = (uint32_t)effcfgs_.size() ? (uint32_t)effcfgs_.size() - 1 : 0;
  t.eff_mcp.assign((size_t)(t.n_effcfg + 1) * 4 * stride, 0);
  for (size_t i = 1; i < effcfgs_.size(); ++i)
    if (effcfg_ok_[i]) verdicts(effcfgs_[i].mcp, &t.eff_mcp[i * 4 * stride]);
  t.v_mcp++;
}

// ------------------------------------------------------------ topics
void Host::topic_row(sv trimmed, Bits& out) const {
  out = vac_topic_;
  std::string key;
  for (size_t len = 0; len <= trimmed.size(); ++len) {
    key.assign(trimmed.data(), len);
    auto it = pat_by_prefix_.find(key);
    if (it == pat_by_prefix_.end()) continue;
    for (uint32_t pi : it->second) {
      const Pattern& p = patterns_[pi];
      if (p.glob.match(trimmed))
        for (uint32_t r : p.rules) out[r >> 5] |= 1u << (r & 31);
    }
  }
}

void Host::eff_topic_fill(uint32_t cfg, uint32_t topic_id) {
  uint8_t v = 0;
  if (effcfg_ok_[cfg]) {
    sv topic = trim_space((*topic_store_)[topic_id]);
    if (!topic.empty()) {   // matchAny: value == "" -> false (kernel.go:456)
      const EffGlobs& g = eff_globs_[cfg];
      for (auto& gl : g.denied) if (gl.match(topic)) { v |= 1; break; }
      if (g.has_allowed) {
        bool any = false;
        for (auto& gl : g.allowed) if (gl.match(topic)) { any = true; break; }
        if (!any) v |= 2;
      }
    } else if (eff_globs_[cfg].has_allowed) v |= 2;
  }
  t_.eff_topic[(size_t)cfg * t_.topic_stride + topic_id] = v;
}

// Recompute every per-topic table for the topics known so far (ids are stable).
void Host::rebuild_topics() {
  HostTables& t = t_;
  if ((*topic_store_).empty()) {   // id 0 = the empty raw topic
    (*topic_store_).emplace_back();
    topic_ids_.put(sv(), 0);
  }
  for (auto& tp : routing_.topics)   // pre-seed so steady state has no dictionary misses
    if (!topic_ids_.contains(tp.first) && (*topic_store_).size() < max_topics_) {
      topic_ids_.put(tp.first, (uint32_t)(*topic_store_).size());
      (*topic_store_).push_back(tp.first);
    }
  const uint32_t n = (uint32_t)(*topic_store_).size(), W = t.row_words;
  t.row_topic.init(n, W);
  topic_entries_.assign(n, TopicEntry{0, 0, 0});
  topic_pools_.assign(n, {});
  t.pool_list.clear();
  // rows in parallel (glob matching dominates at 4k rules x 2k topics)
  std::atomic<uint32_t> next{0};
  auto work = [&]() {
    Bits row;
    for (uint32_t i; (i = next.fetch_add(1)) < n;) {
      sv trimmed = trim_space((*topic_store_)[i]);
      uint32_t fl = 0;
      if ((*topic_store_)[i].empty()) fl |= JF_TOPIC_RAW_EMPTY;
      if (trimmed.empty()) fl |= JF_TOPIC_MISSING;
      else if (!starts_with(trimmed, "job.")) fl |= JF_TOPIC_UNSUPPORTED;
      topic_entries_[i].flags = fl;
      if (!(fl & (JF_TOPIC_MISSING | JF_TOPIC_UNSUPPORTED))) {
        topic_row(trimmed, row);
        std::memcpy(t.row_topic.row(i), row.data(), W * 4);
      }
    }
  };
  uint32_t nth = std::min<uint32_t>(threads_, std::max<uint32_t>(1, n / 16));
  if (nth <= 1) work();
  else {
    std::vector<std::thread> ts;
    for (uint32_t k = 0; k < nth; ++k) ts.emplace_back(work);
    for (auto& th : ts) th.join();
  }
  static const bool trace = getenv("CORDUM_LOAD_TRACE") != nullptr;
  const auto tt0 = std::chrono::steady_clock::now();
  summarize(t.row_topic, t.sum_topic);
  const auto tt1 = std::chrono::steady_clock::now();
  choose_summaries();
  const auto tt2 = std::chrono::steady_clock::now();
  if (trace) fprintf(stderr, "[rebuild_topics] n=%u threads=%u summarize %.2f choose %.2f ms\n", n, nth,
                     std::chrono::duration<double, std::milli>(tt1 - tt0).count(), std::chrono::duration<double, std::milli>(tt2 - tt1).count());
  for (uint32_t i = 0; i < n; ++i) {
    uint32_t ri = routing_topics_.find((*topic_store_)[i], kMiss);
    topic_entries_[i].pool_off = (uint32_t)t.pool_list.size();
    if (ri != kMiss) {
      topic_pools_[i] = routing_.topics[ri].second;
      for (auto& p : routing_.topics[ri].second) {
        uint32_t pid = d_pool_.table.find(p, 0) - 2;
        bool dup = false;
        for (uint32_t k = topic_entries_[i].pool_off; k < t.pool_list.size(); ++k) dup |= t.pool_list[k] == pid;
        if (!dup) t.pool_list.push_back(pid);
      }
    }
    topic_entries_[i].pool_cnt = (uint32_t)t.pool_list.size() - topic_entries_[i].pool_off;
  }
  t.topic_pool_off.resize(n);
  t.topic_pool_cnt.resize(n);
  for (uint32_t i = 0; i < n; ++i) { t.topic_pool_off[i] = topic_entries_[i].pool_off; t.topic_pool_cnt[i] = topic_entries_[i].pool_cnt; }
  if (t.pool_list.empty()) t.pool_list.push_back(0);
  // effective-config topic verdicts
  uint32_t stride = 1024;
  while (stride < n) stride *= 2;
  // The verdict of an effective config on a topic depends on neither the policy nor the routing: topic ids and config
  // ids are stable for the life of the engine, so a reload recomputes only what it added (with a few hundred configs
  // seen, recomputing all of them was most of a policy reload: 100 of 140 ms at config 3).
  const bool keep = t.topic_stride == stride && t.eff_topic.size() == (size_t)(t.n_effcfg + 1) * stride && eff_topic_n_ <= n;
  if (!keep) { t.eff_topic.assign((size_t)(t.n_effcfg + 1) * stride, 0); eff_topic_n_ = 0; }
  t.topic_stride = stride;
  for (uint32_t c = 1; c <= t.n_effcfg; ++c)
    for (uint32_t i = eff_topic_n_; i < n; ++i) eff_topic_fill(c, i);
  eff_topic_n_ = n;
  if (trace) fprintf(stderr, "[rebuild_topics] pools+eff (%u effcfgs) %.2f ms\n", t.n_effcfg,
                     std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - tt2).count());
  t.v_topic++;
}

uint32_t Host::add_topic(sv raw) {
  uint32_t id = topic_ids_.find(raw, kMiss);
  if (id != kMiss) return id;
  if ((*topic_store_).size() >= max_topics_) return kMiss;
  HostTables& t = t_;
  id = (uint32_t)(*topic_store_).size();
  topic_ids_.put(raw, id);
  (*topic_store_).emplace_back(raw);
  sv trimmed = trim_space((*topic_store_).back());
  TopicEntry e{0, (uint32_t)t.pool_list.size(), 0};
  if (trimmed.empty()) e.flags |= JF_TOPIC_MISSING;
  else if (!starts_with(trimmed, "job.")) e.flags |= JF_TOPIC_UNSUPPORTED;
  Bits row(t.row_words, 0);
  if (!e.flags) topic_row(trimmed, row);
  t.row_topic.append(row);
  if (t.sum_topic.size() < t.row_topic.n_rows) t.sum_topic.resize(t.row_topic.n_rows, 0);
  t.sum_topic[id] = row_summary(row.data());
  topic_pools_.emplace_back();
  uint32_t ri = routing_topics_.find(raw, kMiss);
  if (t.topic_pool_off.empty() && t.pool_list.size() == 1) {}   // keep placeholder entry
  if (ri != kMiss) {
    topic_pools_.back() = routing_.topics[ri].second;
    for (auto& p : routing_.topics[ri].second) {
      uint32_t pid = d_pool_.table.find(p, 0) - 2;
      bool dup = false;
      for (uint32_t k = e.pool_off; k < t.pool_list.size(); ++k) dup |= t.pool_list[k] == pid;
      if (!dup) t.pool_list.push_back(pid);
    }
  }
  e.pool_cnt = (uint32_t)t.pool_list.size() - e.pool_off;
  topic_entries_.push_back(e);
  t.topic_pool_off.push_back(e.pool_off);
  t.topic_pool_cnt.push_back(e.pool_cnt);
  if (id >= t.topic_stride) {   // grow the effective-config x topic table
    uint32_t stride = t.topic_stride;
    while (stride <= id) stride *= 2;
    std::vector<uint8_t> grown((size_t)(t.n_effcfg + 1) * stride, 0);
    for (uint32_t c = 0; c <= t.n_effcfg; ++c)
      std::memcpy(&grown[(size_t)c * stride], &t.eff_topic[(size_t)c * t.topic_stride], t.topic_stride);
    t.eff_topic.swap(grown);
    t.topic_stride = stride;
  }
  for (uint32_t c = 1; c <= t.n_effcfg; ++c) eff_topic_fill(c, id);
  if (eff_topic_n_ == id) eff_topic_n_ = id + 1;   // rows of topics [0, eff_topic_n_) are complete for every config
  t.v_topic++;
  v_dict_++;
  return id;
}

uint32_t Host::add_effcfg(sv payload) {
  uint32_t id = effcfg_ids_.find(payload, kMiss);
  if (id != kMiss) return id;
  if (effcfg_ids_.size() >= max_effcfgs_) return kMiss;
  EffSafety cfg;
  bool ok = parse_effective_safety(payload, cfg);
  if (!ok) { effcfg_ids_.put(payload, 0); v_dict_++; return 0; }   // unparsable: the overlay is skipped (kernel.go:218)
  if (effcfgs_.empty()) { effcfgs_.emplace_back(); effcfg_ok_.push_back(0); eff_globs_.emplace_back(); }
  id = (uint32_t)effcfgs_.size();
  effcfg_ids_.put(payload, id);
  EffGlobs g;
  g.has_allowed = !cfg.allowed_topics.empty();
  for (auto& p : cfg.denied_topics) { sv tp = trim_space(p); if (!tp.empty()) g.denied.emplace_back(tp); }
  for (auto& p : cfg.allowed_topics) { sv tp = trim_space(p); if (!tp.empty()) g.allowed.emplace_back(tp); }
  effcfgs_.push_back(std::move(cfg));
  effcfg_ok_.push_back(1);
  eff_globs_.push_back(std::move(g));
  HostTables& t = t_;
  compile_mcp_tables();   // dictionaries may have grown; sets n_effcfg
  if (t.mcp_stride > CORDUM_ID16_MAX) return kMiss;   // ids no longer fit the job record: the encode fails closed
  t.eff_topic.resize((size_t)(t.n_effcfg + 1) * t.topic_stride, 0);
  for (uint32_t i = 0; i < (*topic_store_).size(); ++i) eff_topic_fill(id, i);
  t.v_topic++;
  v_dict_++;
  return id;
}

// ------------------------------------------------------------ documents
int Host::load_policy(sv json, sv snapshot, std::string& err) {
  static const bool trace = getenv("CORDUM_LOAD_TRACE") != nullptr;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto ms = [](auto a, auto b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
  const auto t0 = now();
  PolicyModel m;
  if (!parse_policy_json(json, m, err)) return CORDUM_E_INVALID;   // outside the lock: dispatches go on meanwhile
  const auto t1 = now();
  std::lock_guard<std::mutex> g(mu_);
  PolicyModel old = std::move(policy_);
  policy_ = std::move(m);
  const auto t2 = now();
  compile_policy();
  const auto t3 = now();
  compile_routing();
  compile_mcp_tables();
  const auto t4 = now();
  struct Tr { bool on; decltype(t0) a, b, c, d, e; decltype(ms)& f; ~Tr() { if (on) fprintf(stderr, "[load_policy] parse %.2f  lock %.2f  compile_policy %.2f  routing+mcp %.2f  rest(topics) %.2f ms\n", f(a, b), f(b, c), f(c, d), f(d, e), f(e, std::chrono::steady_clock::now())); } } tr{trace, t0, t1, t2, t3, t4, ms};
  if (t_.mcp_stride > CORDUM_ID16_MAX) policy_capacity_error_ = "more than 65535 distinct MCP values referenced by allow / deny lists";
  if (!policy_capacity_error_.empty() || !routing_capacity_error_.empty()) {
    err = policy_capacity_error_.empty() ? routing_capacity_error_ : policy_capacity_error_;
    policy_ = std::move(old);   // keep serving the previous policy (watchPolicy keeps the old one on failure, kernel.go:495-499)
    compile_policy();
    compile_routing();
    compile_mcp_tables();
    rebuild_topics();
    return CORDUM_E_CAPACITY;
  }
  rebuild_topics();
  epoch_++;
  v_dict_++;
  snapshot_ = std::string(snapshot);
  if (!snapshot.empty()) {   // setPolicy, kernel.go:510-521
    snapshots_.insert(snapshots_.begin(), snapshot_);
    if (snapshots_.size() > 10) snapshots_.resize(10);
  }
  publish_text();
  return CORDUM_OK;
}

void Host::publish_text() {
  auto t = std::make_shared<PolicyText>();
  t->gen = text_.empty() ? 1 : text_.back()->gen + 1;
  t->snapshot = snapshot_;
  t->rules.reserve(policy_.rules.size());
  for (const RuleModel& r : policy_.rules)
    t->rules.push_back(PolicyText::Rule{r.id, r.reason, r.constraints_json, r.remediations_json, r.has_constraints});
  text_gen_.store(t->gen, std::memory_order_release);
  text_.push_back(std::move(t));
  if (text_.size() > 8) text_.pop_front();
}

int Host::load_routing(sv json, std::string& err) {
  RoutingModel m;
  if (!parse_routing_json(json, m, err)) return CORDUM_E_INVALID;
  std::lock_guard<std::mutex> g(mu_);
  RoutingModel old = std::move(routing_);
  routing_ = std::move(m);
  compile_policy();   // the requires dictionary is shared: rebuild both sides
  compile_routing();
  if (!routing_capacity_error_.empty()) {
    err = routing_capacity_error_;
    routing_ = std::move(old);
    compile_policy();
    compile_routing();
    compile_mcp_tables();
    rebuild_topics();
    return CORDUM_E_CAPACITY;
  }
  compile_mcp_tables();
  rebuild_topics();
  std::string e2;
  if (compile_workers(e2) != CORDUM_OK) {   // the new pool set makes more labelled workers routable than the label
    err = e2;                               // dictionary holds: keep the previous routing (nothing was committed for
    routing_ = std::move(old);              // the workers: compile_workers checks capacity before it mutates)
    compile_policy();
    compile_routing();
    compile_mcp_tables();
    rebuild_topics();
    std::string e3;
    compile_workers(e3);
    return CORDUM_E_CAPACITY;
  }
  epoch_++;
  v_dict_++;
  return CORDUM_OK;
}

int Host::load_workers(const cordum_workers* w, std::string& err) {
  std::lock_guard<std::mutex> g(mu_);
  // Everything is built in temporaries and committed only when the new registry compiles: a rejected load (NaN load,
  // label dictionary overflow) leaves the previous registry, its tables and every encoded batch untouched.
  std::vector<WorkerRaw> store;
  std::vector<Load16> loads;
  std::vector<std::string> ids;
  if (w) {
    auto sp = [&](const cordum_str* col, uint32_t i) { return sv((const char*)w->arena + col[i].off, col[i].len); };
    store.resize(w->n_workers);
    loads.resize(w->n_workers);
    ids.resize(w->n_workers);
    for (uint32_t i = 0; i < w->n_workers; ++i) {
      float cpu = w->cpu_load[i], gpu = w->gpu_utilization[i];
      if (cpu != cpu || gpu != gpu) { err = "worker load is NaN (ordering undefined in the reference)"; return CORDUM_E_INVALID; }
      store[i].id = std::string(sp(w->worker_id, i));
      store[i].pool = std::string(sp(w->pool, i));
      ids[i] = store[i].id;
      if (w->label_off)
        for (uint32_t k = w->label_off[i]; k < w->label_off[i + 1]; ++k) {
          std::string key(sp(w->label_keys, k));
          bool found = false;
          for (auto& kv : store[i].labels) if (kv.first == key) { kv.second = std::string(sp(w->label_vals, k)); found = true; }
          if (!found) store[i].labels.emplace_back(key, std::string(sp(w->label_vals, k)));
        }
      loads[i] = Load16{w->active_jobs[i], w->max_parallel_jobs[i], cpu, gpu};
    }
  }
  std::vector<WorkerRaw> old_store = std::move(workers_raw_);
  workers_raw_ = std::move(store);
  int rc = compile_workers(err, &loads);
  if (rc != CORDUM_OK) { workers_raw_ = std::move(old_store); return rc; }   // compile_workers mutated nothing
  worker_ids_ = std::make_shared<const std::vector<std::string>>(std::move(ids));
  epoch_++;
  v_dict_++;
  return CORDUM_OK;
}

void set_selective_limits(uint32_t min_bits, uint32_t max_holders) {
  g_sel_min_bits = min_bits;
  g_sel_max_holders = max_holders;
}

int Host::compile_workers(std::string& err, const std::vector<Load16>* new_loads) {
  HostTables& t = t_;
  auto& store = workers_raw_;
  const uint32_t n = (uint32_t)store.size();
  // ---- phase 1: everything that can fail, into locals (no member is written before the capacity check)
  StrTable worker_slot, place_pair, place_key;
  for (uint32_t s = 0; s < n; ++s) worker_slot.put(store[s].id, s);   // map semantics: last wins
  std::vector<uint32_t> live;
  for (uint32_t s = 0; s < n; ++s) if (worker_slot.find(store[s].id, kMiss) == s) live.push_back(s);
  std::sort(live.begin(), live.end(), [&](uint32_t a, uint32_t b) { return store[a].id < store[b].id; });
  std::vector<uint32_t> rank_of(n, 0);
  for (uint32_t r = 0; r < live.size(); ++r) rank_of[live[r]] = r;
  // routable = live and in a pool the routing table knows
  struct Pos { uint32_t pool, rank, slot; };
  std::vector<Pos> pos;
  for (uint32_t s : live) {
    uint32_t pid = d_pool_.table.find(store[s].pool, 0);
    if (pid >= 2) pos.push_back({pid - 2, rank_of[s], s});
  }
  std::sort(pos.begin(), pos.end(), [](const Pos& a, const Pos& b) { return a.pool != b.pool ? a.pool < b.pool : a.rank < b.rank; });
  // placement-label dictionary: pairs (k,v!=""), per-key "absent or empty" bits, "has any label" bit
  uint32_t nbits = 0;
  const uint32_t any_bit = nbits++;
  std::vector<uint32_t> pair_bits;   // the bits that stand for pairs, ascending
  std::vector<uint32_t> holders;     // per bit: routable workers carrying the pair
  for (auto& p : pos)
    for (auto& kv : store[p.slot].labels) {
      if (place_key.find(kv.first, kMiss) == kMiss) { place_key.put(kv.first, nbits++); holders.push_back(0); }
      if (!kv.second.empty()) {
        const std::string pk = StrTable::pair_key(kv.first, kv.second);
        uint32_t b = place_pair.find(pk, kMiss);
        if (b == kMiss) { b = nbits++; place_pair.put(pk, b); pair_bits.push_back(b); holders.push_back(0); }
        holders[b - 1]++;   // holders[0] is bit 1: the "has any label" bit is no pair
      }
    }
  // Selective pairs (tables.h DeviceTables.sel_*): once the registry needs more placement bits than the limit, a pair
  // carried by few routable workers (hostname-style labels) gets a holder list instead of a dense bit, a bitmap row per
  // pool and a side-row bit per job.  The remaining bits keep their order and are renumbered densely.
  const uint32_t sel_min_bits = g_sel_min_bits.load(), sel_max_holders = g_sel_max_holders.load();
  std::vector<uint32_t> remap;   // old bit -> dense bit, or CORDUM_SEL_TAG | selective pair id (empty: nothing moves)
  uint32_t dense_bits = nbits, n_sel = 0;
  if (nbits > sel_min_bits) {
    std::vector<uint8_t> sel(nbits, 0);
    for (uint32_t b : pair_bits) sel[b] = holders[b - 1] <= sel_max_holders;
    remap.resize(nbits);
    dense_bits = 0;
    for (uint32_t b = 0; b < nbits; ++b) remap[b] = sel[b] ? (CORDUM_SEL_TAG | n_sel++) : dense_bits++;
    if (n_sel == 0) { remap.clear(); dense_bits = nbits; }
  }
  {   // label bits beyond 128 spill into pos_label_x; what bounds them is the per-pool bitmaps (dense bits x workers / 8 bytes)
    std::vector<uint32_t> per_pool(std::max<uint32_t>(t.n_pools, 1), 0);
    for (auto& p : pos) per_pool[p.pool]++;
    uint64_t words = 0;
    for (uint32_t c : per_pool) words += (uint64_t)dense_bits * ((c + 31) / 32);
    if (nbits > 65536 || words > (1ull << 31)) {
      err = "placement labels on routable workers need " + std::to_string(nbits) + " label bits and " + std::to_string(words * 4 >> 20) +
            " MiB of per-pool label bitmaps (limits: 65536 bits, 8 GiB)";
      return CORDUM_E_CAPACITY;
    }
  }
  if (!remap.empty()) {   // the dictionaries with the new numbering
    StrTable pp, pk;
    for (auto& p : pos)
      for (auto& kv : store[p.slot].labels) {
        if (!pk.contains(kv.first)) pk.put(kv.first, remap[place_key.find(kv.first, 0)]);
        if (!kv.second.empty()) {
          const std::string k = StrTable::pair_key(kv.first, kv.second);
          if (!pp.contains(k)) pp.put(k, remap[place_pair.find(k, 0)]);
        }
      }
    place_pair = std::move(pp);
    place_key = std::move(pk);
  }
  // ---- phase 2: commit (cannot fail)
  t.n_slots = n;
  if (new_loads) t.loads = *new_loads;
  worker_slot_ = std::move(worker_slot);
  place_pair_ = std::move(place_pair);
  place_key_ = std::move(place_key);
  place_any_bit_ = any_bit;
  place_bits_ = dense_bits;
  t.rank_slot.assign(std::max<uint32_t>(n, 1), 0);
  for (uint32_t r = 0; r < live.size(); ++r) t.rank_slot[r] = live[r];
  const uint32_t np = (uint32_t)pos.size();
  t.n_pos = np;
  uint32_t cap = std::max<uint32_t>(np, 1);
  t.pos_pool.assign(cap, 0); t.pos_slot.assign(cap, 0); t.pos_rank.assign(cap, 0);
  t.pos_label_lo.assign(cap, 0); t.pos_label_hi.assign(cap, 0);
  const uint32_t xp = dense_bits > 128 ? (dense_bits - 128 + 63) / 64 : 0;
  t.wide.xw_place = xp;
  t.pos_label_x.assign((size_t)cap * xp + 1, 0);
  t.slot_pos.assign(std::max<uint32_t>(n, 1), 0);
  t.rank_pos.assign(std::max<uint32_t>(n, 1), 0);
  t.pool_off.assign(t.n_pools + 1, 0);
  // all keys, to set the "absent or empty" bits
  std::vector<std::pair<std::string, uint32_t>> keys;
  {
    std::set<std::string> seen;
    for (auto& p : pos) for (auto& kv : store[p.slot].labels) if (seen.insert(kv.first).second)
      keys.emplace_back(kv.first, place_key_.find(kv.first, 0));
  }
  // selective pairs: each worker's ids (pos_sel, CSR by pos) and each pair's holders (sel_pos, CSR by pair id)
  t.n_sel = n_sel;
  t.pos_sel_off.assign(cap + 1, 0);
  t.pos_sel.clear();
  t.sel_off.assign(n_sel + 1, 0);
  for (uint32_t i = 0; i < np; ++i) {
    const Pos& p = pos[i];
    t.pos_pool[i] = p.pool; t.pos_slot[i] = p.slot; t.pos_rank[i] = p.rank;
    t.slot_pos[p.slot] = i + 1;
    t.rank_pos[p.rank] = i;
    t.pool_off[p.pool + 1]++;
    uint64_t m[2] = {0, 0};
    uint64_t* mx = t.pos_label_x.data() + (size_t)i * xp;
    auto setb = [&](uint32_t b) { if (b < 128) m[b >> 6] |= 1ull << (b & 63); else mx[(b >> 6) - 2] |= 1ull << (b & 63); };
    const auto& labels = store[p.slot].labels;
    const size_t s0 = t.pos_sel.size();
    if (!labels.empty()) {
      setb(place_any_bit_);
      for (auto& k : keys) {
        const std::string* val = nullptr;
        for (auto& kv : labels) if (kv.first == k.first) val = &kv.second;
        if (!val || val->empty()) { setb(k.second); continue; }   // labels[k] == "" (matchesLabels, :169-171)
        const uint32_t b = place_pair_.find_pair(k.first, *val, 0);
        if (b & CORDUM_SEL_TAG) { t.pos_sel.push_back(b & ~CORDUM_SEL_TAG); t.sel_off[(b & ~CORDUM_SEL_TAG) + 1]++; }
        else setb(b);
      }
    }
    std::sort(t.pos_sel.begin() + s0, t.pos_sel.end());
    t.pos_sel_off[i + 1] = (uint32_t)t.pos_sel.size();
    t.pos_label_lo[i] = m[0]; t.pos_label_hi[i] = m[1];
  }
  for (uint32_t s = 0; s < n_sel; ++s) t.sel_off[s + 1] += t.sel_off[s];
  t.sel_pos.assign(std::max<size_t>(t.pos_sel.size(), 1), 0);
  {
    std::vector<uint32_t> fill(t.sel_off.begin(), t.sel_off.end() - 1);
    for (uint32_t i = 0; i < np; ++i)   // ascending pos: each pair's holders come out in pos order
      for (uint32_t k = t.pos_sel_off[i]; k < t.pos_sel_off[i + 1]; ++k) t.sel_pos[fill[t.pos_sel[k]]++] = i;
  }
  if (t.pos_sel.empty()) t.pos_sel.push_back(0);
  for (uint32_t p = 0; p < t.n_pools; ++p) t.pool_off[p + 1] += t.pool_off[p];
  // per-pool label bitmaps (filled on the device by worker-table refresh kernels): place_bits rows of ceil(n/32) words
  t.place_bits = std::max<uint32_t>(place_bits_, 1);
  t.lbm_off.assign(std::max<uint32_t>(t.n_pools, 1), 0);
  t.lbm_words = 0;
  for (uint32_t p = 0; p < t.n_pools; ++p) {
    t.lbm_off[p] = (uint32_t)t.lbm_words;
    t.lbm_words += (uint64_t)t.place_bits * ((t.pool_off[p + 1] - t.pool_off[p] + 31) / 32);
  }
  // refresh work list: chunks of CORDUM_POOL_CHUNK workers (an empty pool still owns one, empty, chunk)
  t.chunk_pool.clear(); t.merge_list.clear();
  t.pool_chunk0.assign(t.n_pools + 1, 0);
  t.merge_smem = 0;
  for (uint32_t p = 0; p < t.n_pools; ++p) {
    const uint32_t n = t.pool_off[p + 1] - t.pool_off[p];
    const uint32_t m = std::max<uint32_t>(1, (n + CORDUM_POOL_CHUNK - 1) / CORDUM_POOL_CHUNK);
    const uint32_t g0 = (uint32_t)t.chunk_pool.size();
    t.pool_chunk0[p] = g0;
    for (uint32_t c = 0; c < m; ++c) t.chunk_pool.push_back(p);
    if (n > CORDUM_POOL_SORT_MAX) t.merge_list.push_back(g0);
    else if (m > 1) {
      for (uint32_t c = 0; c < m; ++c) t.merge_list.push_back(g0 + c);
      t.merge_smem = std::max<uint32_t>(t.merge_smem, n * 8u);
    }
  }
  t.pool_chunk0[t.n_pools] = (uint32_t)t.chunk_pool.size();
  t.n_chunks = (uint32_t)t.chunk_pool.size();
  t.n_merge = (uint32_t)t.merge_list.size();
  if (t.chunk_pool.empty()) t.chunk_pool.push_back(0);
  if (t.merge_list.empty()) t.merge_list.push_back(0);
  if (t.loads.empty()) t.loads.push_back(Load16{0, 0, 0.f, 0.f});
  t.v_workers++;
  t.v_loads++;
  return CORDUM_OK;
}

int Host::update_loads(uint32_t n, const uint32_t* slots, const cordum_worker_load* loads, std::string& err) {
  std::lock_guard<std::mutex> g(mu_);
  // all or nothing: a refused call must not leave some of its rows in the table, where the next accepted call would
  // upload them along with its own
  for (uint32_t i = 0; i < n; ++i) {
    if (slots[i] >= t_.n_slots) { err = "worker slot out of range"; return CORDUM_E_INVALID; }
    if (loads[i].cpu_load != loads[i].cpu_load || loads[i].gpu_utilization != loads[i].gpu_utilization) {
      err = "worker load is NaN"; return CORDUM_E_INVALID;
    }
  }
  for (uint32_t i = 0; i < n; ++i)
    t_.loads[slots[i]] = Load16{loads[i].active_jobs, loads[i].max_parallel_jobs, loads[i].cpu_load, loads[i].gpu_utilization};
  t_.v_loads++;
  return CORDUM_OK;
}

std::string Host::mcp_value_string(int field, uint32_t id) const {
  if (id >= 2 && id - 2 < d_mcp_[field].keys.size()) return d_mcp_[field].keys[id - 2];
  return std::string();
}
const std::vector<std::string>& Host::topic_pool_names(uint32_t topic_id) const {
  static const std::vector<std::string> none;
  return topic_id < topic_pools_.size() ? topic_pools_[topic_id] : none;
}

// ============================================================ encoder
// Span-identity caches.  Envelope strings are (offset,len) spans into one arena and equal strings usually share
// one span (the arena packers intern), so within a call most lookups repeat an address already resolved.  A small
// direct-mapped cache keyed by (pointer, length) skips the byte hash + fold for those; it lives on the worker's
// stack for the duration of one encode call, while the arena is immutable.
struct EncodeCaches {
  // entries carry the generation (encode call) that wrote them: a cache object lives as long as the Host, and an
  // entry from an earlier call - whose arena is gone - simply does not match
  uint32_t gen = 1;
  struct Entry { const char* p = nullptr; uint32_t len = 0, val = 0, aux = 0, gen = 0; };
  template <uint32_t BITS>
  struct Tab {
    Entry e[1u << BITS];
    static uint32_t slot(sv s) { return (uint32_t)((((uintptr_t)s.data() >> 1) ^ s.size()) * 0x9E3779B1u) >> (32 - BITS); }
    bool get(sv s, uint32_t& val, uint32_t& aux, uint32_t gen) const {
      const Entry& x = e[slot(s)];
      if (x.p == s.data() && x.len == s.size() && x.gen == gen) { val = x.val; aux = x.aux; return true; }
      return false;
    }
    void put(sv s, uint32_t val, uint32_t aux, uint32_t gen) { e[slot(s)] = Entry{s.data(), (uint32_t)s.size(), val, aux, gen}; }
  };
  // sized for the cardinalities a batch typically shows (thousands of topics / capabilities, many principals)
  Tab<12> topic;
  Tab<11> cap, actor;
  Tab<9> tenant, pack, risk, req;
  // (label key, label value) pairs: what the pair does to the rule label mask and to the placement mask.  Keys that
  // carry per-job values (MCP aliases, secrets_present, preferred_pool, preferred_worker_id) are never cached.
  struct LabelEntry {
    const char* kp = nullptr; const char* vp = nullptr;
    uint32_t klen = 0, vlen = 0;
    uint64_t set = 0, clear = 0;   // rule label pairs: lab = (lab | set) & ~clear
    uint32_t place = 0;            // placement bit, or kPlaceNone / kPlaceUnsat
    uint32_t gen = 0;
  };
  static constexpr uint32_t kPlaceNone = 0xFFFFFFFFu, kPlaceUnsat = 0xFFFFFFFEu;
  LabelEntry label[1024];
  static uint32_t lslot(sv k, sv v) {
    return (uint32_t)(((((uintptr_t)k.data() >> 1) ^ k.size()) * 0x9E3779B1u) ^ ((((uintptr_t)v.data() >> 1) ^ v.size()) * 0x85EBCA6Bu)) >> 22;
  }
  // selective placement pairs: the ids of the job being encoded, and {slot, count, ids...} of this thread's JF_SELECTIVE jobs
  std::vector<uint32_t> sel_ids, sel_rec;
};

namespace {
inline sv span(const cordum_envelopes* e, const cordum_str* col, uint32_t j) {
  return col ? sv((const char*)e->arena + col[j].off, col[j].len) : sv();
}
// labels that never constrain placement (filterPlacementLabels, strategy_least_loaded.go:195-222)
inline bool placement_skips(sv k) {
  switch (k.size()) {
    case 6: return k == "run_id";
    case 7: return k == "step_id" || k == "node_id";
    case 9: return k == "worker_id";
    case 11: return k == "workflow_id";
    case 14: return k == "preferred_pool";
    case 15: return k == "secrets_present";
    case 16: return k == "approval_granted";
    case 19: return k == "preferred_worker_id";
    default: return false;
  }
}
// mcp label aliases (kernel.go:400-403): field*3 + variant, or -1
inline int mcp_key(sv k) {
  if (k.size() < 7 || k[0] != 'm' || k[1] != 'c' || k[2] != 'p') return -1;   // shortest alias: "mcpTool"
  static const char* names[12] = {"mcp.server", "mcp_server", "mcpServer", "mcp.tool", "mcp_tool", "mcpTool",
                                  "mcp.resource", "mcp_resource", "mcpResource", "mcp.action", "mcp_action", "mcpAction"};
  for (int i = 0; i < 12; ++i) if (k == names[i]) return i;
  return -1;
}

}  // namespace

// extractMCPRequest's value of one field for one envelope, spelled as the request spells it (kernel.go:395-414):
// the first alias whose value is non-blank, trimmed; the action lower-cased.  What the %q of an MCP reason prints.
std::string mcp_request_value(const cordum_envelopes* env, uint32_t j, int field) {
  if (!env || j >= env->n_jobs || !env->label_off) return std::string();
  sv pick[3];
  for (uint32_t k = env->label_off[j]; k < env->label_off[j + 1]; ++k) {
    const cordum_str &ks = env->label_keys[k], &vs = env->label_vals[k];
    int mk = mcp_key(sv((const char*)env->arena + ks.off, ks.len));
    if (mk >= 0 && mk / 3 == field) pick[mk % 3] = trim_space(sv((const char*)env->arena + vs.off, vs.len));   // later entry wins
  }
  for (const sv& v : pick)
    if (!v.empty()) return field == 3 ? lower_copy(v) : std::string(v);
  return std::string();
}


uint32_t Host::resolve_topic(const cordum_envelopes* env, uint32_t j, EncodeCaches& cc) const {
  // dictionary keyed by the RAW string: policy sees TrimSpace(topic), routing the raw one
  sv topic_raw = span(env, env->topic, j);
  uint32_t cv = 0, ca = 0;
  if (!topic_raw.empty() && cc.topic.get(topic_raw, cv, ca, cc.gen)) return cv;
  uint32_t tid = topic_ids_.find(topic_raw, kMiss);
  if (tid != kMiss && !topic_raw.empty()) cc.topic.put(topic_raw, tid, 0, cc.gen);
  return tid;
}

// tenant (kernel.go:134-169): dictionary id | exact-tenant policy index << 16
uint32_t Host::resolve_tenant(const cordum_envelopes* env, uint32_t j, EncodeCaches& cc) const {
  const bool has_meta = env->has_meta && env->has_meta[j];
  sv tenant = trim_space(span(env, env->tenant, j));
  if (tenant.empty() && has_meta) tenant = trim_space(span(env, env->meta_tenant_id, j));
  if (tenant.empty()) tenant = default_tenant_trim_;
  if (tenant.empty()) tenant = "default";
  uint32_t cv = 0, ca = 0;
  if (cc.tenant.get(tenant, cv, ca, cc.gen)) return cv | (ca << 16);
  cv = lookup_value(d_tenant_, tenant);
  ca = tenant_pol_.find(tenant, 0);   // exact-string map lookup (kernel.go:190)
  cc.tenant.put(tenant, cv, ca, cc.gen);
  return cv | (ca << 16);
}

void Host::encode_job(const cordum_envelopes* env, uint32_t j, uint32_t tid, uint32_t ten, JobRec& jr, RouteRec& rr, uint64_t* wx, bool& miss, EncodeCaches& cc) const {
  // wx: the job's row of extra mask words (tables.h WideLayout), zeroed here; null when the tables have none
  const WideLayout WL = t_.wide;
  const uint32_t o_req = WIDE_O_REQ(WL), o_lab = WIDE_O_LAB(WL), o_reqp = WIDE_O_REQP(WL), o_place = WIDE_O_PLACE(WL);
  if (wx) {
    std::memset(wx, 0, sizeof(uint64_t) * WIDE_WORDS(WL));
    for (uint32_t k = 0; k < WL.xw_lab; ++k) wx[o_lab + k] = label_empty_x_[k];
  }
  auto setx = [&](uint32_t off, uint32_t bit) { wx[off + (bit >> 6) - 1] |= 1ull << (bit & 63); };   // bit >= 64
  bool risk_any = false, req_any = false;
  uint32_t flags = 0;
  jr.topic = tid;
  jr.orig = j;
  jr.sel[0] = jr.sel[1] = 0;
  cc.sel_ids.clear();
  flags |= topic_entries_[tid].flags;
  const bool has_meta = env->has_meta && env->has_meta[j];
  jr.tenant = (uint16_t)(ten & 0xFFFFu);   // resolved in pass 1 (resolve_tenant)
  jr.tenant_pol = (uint16_t)(ten >> 16);
  // ---- meta (policyMetaFromRequest, kernel.go:348-368)
  sv principal = span(env, env->principal_id, j);
  sv cap, pack, actor = principal;
  int at = 0;
  if (has_meta) {
    cap = span(env, env->capability, j);
    pack = span(env, env->pack_id, j);
    sv a = span(env, env->actor_id, j);
    if (!a.empty()) actor = a;
    int raw_at = env->actor_type ? env->actor_type[j] : 0;
    at = (raw_at == 1 || raw_at == 2) ? raw_at : 0;
  }
  auto cached = [&](auto& tab, const Dict& d, sv v) -> uint16_t {
    if (v.empty()) return CORDUM_ID_EMPTY;
    uint32_t val, aux;
    if (tab.get(v, val, aux, cc.gen)) return (uint16_t)val;
    val = lookup_value(d, v);
    tab.put(v, val, 0, cc.gen);
    return (uint16_t)val;
  };
  jr.cap = cached(cc.cap, d_cap_, cap);
  jr.pack = cached(cc.pack, d_pack_, pack);
  jr.actor = cached(cc.actor, d_actor_, actor);
  // ---- risk tags / requires
  uint64_t risk = 0, req = 0, req_pool = 0;
  bool secrets_tag = false;
  if (has_meta && env->risk_off)
    for (uint32_t k = env->risk_off[j]; k < env->risk_off[j + 1]; ++k) {
      sv tag = span(env, env->risk_tags, k);
      uint32_t id, is_secrets;
      if (tag.empty()) continue;
      if (!cc.risk.get(tag, id, is_secrets, cc.gen)) {
        is_secrets = fold_eq(tag, "secrets") ? 1u : 0u;   // kernel.go:387-391 (no trim)
        id = lookup_value(d_risk_, tag);
        cc.risk.put(tag, id, is_secrets, cc.gen);
      }
      if (is_secrets) secrets_tag = true;
      if (id >= 2) {
        if (id - 2 < 64) risk |= 1ull << (id - 2); else setx(0, id - 2);
        risk_any = true;
      }
    }
  if (has_meta && env->requires_off) {
    uint32_t a = env->requires_off[j], b = env->requires_off[j + 1];
    if (b > a) flags |= JF_REQ_NONEMPTY;
    for (uint32_t k = a; k < b; ++k) {
      sv tok = span(env, env->requires_, k);
      // Two canonical forms over one dictionary of strings: rules compare with EqualFold (safety_policy.go:301),
      // pools with ToLower (strategy_least_loaded.go:250,256).  They differ only for non-ASCII tokens.
      uint32_t id, idp;   // idp: low bit = blank, rest = pool-side id + 1 (0 = same as the rule-side id)
      if (tok.empty() || !cc.req.get(tok, id, idp, cc.gen)) {
        FoldBuf f(tok);
        id = d_req_.table.find(f.view, 0);
        uint32_t pid = id;
        bool blank = f.view.empty();
        if (!is_ascii(tok)) {
          std::string lk = lower_key(tok);
          pid = d_req_.table.find(lk, 0);
          blank = lk.empty();
        }
        idp = (blank ? 1u : 0u) | ((pid + 1) << 1);
        if (!tok.empty()) cc.req.put(tok, id, idp, cc.gen);
      }
      const uint32_t pid = (idp >> 1) - 1;
      if (id >= 2) {
        if (id - 2 < 64) req |= 1ull << (id - 2); else setx(o_req, id - 2);
        req_any = true;
      }
      if (pid >= 2) { if (pid - 2 < 64) req_pool |= 1ull << (pid - 2); else setx(o_reqp, pid - 2); }
      else if (!(idp & 1)) flags |= JF_REQ_UNKNOWN;   // no pool declares it -> no pool satisfies (:255-262)
    }
  }
  jr.risk = risk;
  jr.req = req;
  rr.req_pool = req_pool;
  // ---- labels: one pass
  uint64_t lab = label_empty_mask_, place[2] = {0, 0};
  auto set_place = [&](uint32_t bit) {
    if (bit & CORDUM_SEL_TAG) cc.sel_ids.push_back(bit & ~CORDUM_SEL_TAG);   // a selective pair: no dense bit
    else if (bit < 128) place[bit >> 6] |= 1ull << (bit & 63);
    else wx[o_place + (bit >> 6) - 2] |= 1ull << (bit & 63);
  };
  sv mcpv[12];
  sv secrets_label, pref_pool, pref_worker;
  bool have_secrets_label = false;
  uint32_t la = env->label_off ? env->label_off[j] : 0, lb = env->label_off ? env->label_off[j + 1] : 0;
  if (lb > la) flags |= JF_HAS_LABELS;
  for (uint32_t k = la; k < lb; ++k) {
    sv key = span(env, env->label_keys, k), val = span(env, env->label_vals, k);
    bool shadowed = false;   // map semantics: a later entry with the same key wins
    for (uint32_t k2 = k + 1; k2 < lb && !shadowed; ++k2) shadowed = span(env, env->label_keys, k2) == key;
    if (shadowed) continue;
    EncodeCaches::LabelEntry& ce = cc.label[EncodeCaches::lslot(key, val)];
    if (ce.gen == cc.gen && ce.kp == key.data() && ce.klen == key.size() && ce.vp == val.data() && ce.vlen == val.size()) {
      lab = (lab | ce.set) & ~ce.clear;
      if (ce.place == EncodeCaches::kPlaceUnsat) flags |= JF_PLACE_UNSAT;
      else if (ce.place != EncodeCaches::kPlaceNone) set_place(ce.place);
      continue;
    }
    // rule label pairs: labels.get(k,"") == v
    uint64_t lset = 0, lclear = 0;
    bool special = false;   // the value matters per job: not cacheable
    uint32_t ki = label_key_.find(key, kMiss);
    if (ki != kMiss)
      for (auto& pv : label_key_pairs_[ki]) {
        if (pv.second >= 64) {   // a pair bit in the wide words: set / clear it there; the cache entry has no room for it
          uint64_t& w = wx[o_lab + (pv.second >> 6) - 1];
          const uint64_t b = 1ull << (pv.second & 63);
          if (sv(pv.first) == val) w |= b; else w &= ~b;
          special = true;
          continue;
        }
        if (sv(pv.first) == val) lset |= 1ull << pv.second; else lclear |= 1ull << pv.second;
      }
    lab = (lab | lset) & ~lclear;
    int mk = mcp_key(key);
    if (mk >= 0) { mcpv[mk] = trim_space(val); special = true; }
    if (key == "secrets_present") { secrets_label = trim_space(val); have_secrets_label = true; special = true; }
    else if (key == "preferred_pool") { pref_pool = val; special = true; }
    else if (key == "preferred_worker_id") { pref_worker = val; special = true; }
    // placement constraint?
    uint32_t bit = EncodeCaches::kPlaceNone;
    if (!(placement_skips(key) || starts_with(key, "cordum."))) {
      if (!val.empty()) {
        bit = place_pair_.find_pair(key, val, kMiss);
        if (bit == kMiss) bit = EncodeCaches::kPlaceUnsat;
      } else {
        bit = place_key_.find(key, kMiss);
        if (bit == kMiss) bit = place_any_bit_;   // no worker carries this key: any labelled worker passes
      }
      if (bit == EncodeCaches::kPlaceUnsat) flags |= JF_PLACE_UNSAT;
      else set_place(bit);
    }
    if (!special) ce = EncodeCaches::LabelEntry{key.data(), val.data(), (uint32_t)key.size(), (uint32_t)val.size(), lset, lclear, bit, cc.gen};
  }
  jr.lab = lab;
  rr.place_lo = place[0];
  rr.place_hi = place[1];
  if (!cc.sel_ids.empty()) {
    // route_kernel settles everything before the worker scan and leaves NO_WORKERS; route_select_kernel takes it from there.
    // A pair nobody carries (JF_PLACE_UNSAT already) makes the job NO_WORKERS whatever else it names.
    if (flags & JF_PLACE_UNSAT) cc.sel_ids.clear();
    else {
      flags |= JF_PLACE_UNSAT | JF_SELECTIVE;
      jr.sel[0] = cc.sel_ids[0] + 1;
      jr.sel[1] = cc.sel_ids.size() > 1 ? cc.sel_ids[1] + 1 : 0;
    }
  }
  // ---- MCP request (extractMCPRequest, kernel.go:395-414) and secrets (kernel.go:381-393)
  bool used = false;
  for (int f = 0; f < 4; ++f) {
    sv v;
    for (int a = 0; a < 3 && v.empty(); ++a) v = mcpv[f * 3 + a];
    if (f == 3 && !is_ascii(v)) {   // Action: strings.ToLower(pickLabel(...)) (kernel.go:403), then EqualFold against the lists
      std::string lv = lower_copy(v);
      jr.mcp[f] = (uint16_t)lookup_value(d_mcp_[f], lv);
    } else jr.mcp[f] = (uint16_t)lookup_value(d_mcp_[f], v);
    used |= !v.empty();
  }
  if (used) flags |= JF_MCP_USED;
  bool secrets = secrets_tag;
  if (have_secrets_label && !secrets_label.empty())
    secrets = secrets_label == "true" || secrets_label == "1" || fold_eq(secrets_label, "yes");
  flags |= (uint32_t)(at * 2 + (secrets ? 1 : 0));
  (void)risk_any;
  if (!req_any) flags |= JF_NO_REQ;
  bool lab_any = lab != 0;
  for (uint32_t k = 0; wx && k < WL.xw_lab; ++k) lab_any |= wx[o_lab + k] != 0;
  if (!(flags & JF_HAS_LABELS) || !lab_any) flags |= JF_NO_LAB;
  // ---- routing hints
  uint32_t pp = 0, pw = 0;
  if (!pref_pool.empty()) { uint32_t id = d_pool_.table.find(pref_pool, 0); pp = id >= 2 ? id - 1 : CORDUM_PREF_UNKNOWN; }
  if (!pref_worker.empty()) { uint32_t s = worker_slot_.find(pref_worker, kMiss); pw = s != kMiss ? s + 1 : CORDUM_PREF_UNKNOWN; }
  rr.pref_pool = pp;
  rr.pref_worker = pw;
  // ---- effective config
  sv eff = span(env, env->effective_config, j);
  uint32_t eid = 0;
  if (!eff.empty()) {
    eid = effcfg_ids_.find(eff, kMiss);
    if (eid == kMiss) { miss = true; eid = 0; }
  }
  jr.effcfg = (uint16_t)eid;
  if (env->approved && env->approved[j]) flags |= JF_APPROVED;
  jr.flags = flags;
}

// Encode = two passes over the envelopes.  Pass 1 resolves every job's topic and tenant and counts jobs per (part, key),
// key = (topic id, tenant class); a prefix sum turns the counts into each part's first slot per key; pass 2 encodes job j
// straight into its slot of the sorted record arrays (one sequential 64 B + 32 B write stream per (part, key), no
// scatter of columns).  The order is a stable counting sort, so it is a pure function of the batch.
int Host::encode(const cordum_envelopes* env, HostRecords& out, std::string& err) {
  if (!env) { err = "null envelopes"; return CORDUM_E_INVALID; }
  std::lock_guard<std::mutex> g(mu_);
  int rc = encode_locked(env, out, err);
  if (rc == kDictFull) {
    // A dictionary that grows with the traffic (raw topics, effective configs) is full: start a new generation of both -
    // keep only what the routing table pre-seeds, bump the epoch (batches encoded under the old ids are refused as stale
    // and get encoded again) - and encode this batch again; it registers what it needs.
    reset_dynamic_dictionaries();
    rc = encode_locked(env, out, err);
    if (rc == kDictFull) { err = "one batch references more distinct topics / effective configs than the dictionaries hold (max_topics / max_effcfgs)"; rc = CORDUM_E_CAPACITY; }
  }
  out.epoch = epoch_;
  return rc;
}

void Host::reset_dynamic_dictionaries() {
  topic_ids_.clear();
  topic_store_ = std::make_shared<std::vector<std::string>>();   // batches dispatched earlier keep the old names alive
  topic_entries_.clear();
  topic_pools_.clear();
  effcfg_ids_.clear();
  effcfgs_.clear(); effcfg_ok_.clear(); eff_globs_.clear();
  eff_topic_n_ = 0;
  t_.eff_topic.clear();
  compile_mcp_tables();   // no effective configs any more
  rebuild_topics();       // the routing table's topics, their rows, pools and (empty) effective-config verdicts
  epoch_++;
  v_dict_++;
  dict_resets_++;
}

int Host::encode_locked(const cordum_envelopes* env, HostRecords& out, std::string& err) {
  const uint32_t n = env->n_jobs;
  const uint32_t ww = WIDE_WORDS(t_.wide);
  out.wide_words = ww;
  out.sel_jobs.clear();
  out.sel_extra.clear();
  if (n == 0) return CORDUM_OK;
  if (ww && (!out.wide || (uint64_t)n * ww > out.wide_cap)) { err = "wide-mask buffer missing or too small for this policy"; return kWideRetry; }
  const uint32_t nthreads = (n < 8192 || threads_ <= 1) ? 1u : threads_;
  auto& caches = caches_;   // span-identity caches: entries are only valid within this call (generation tag)
  if (caches.size() < nthreads) caches.resize(nthreads);
  if (++encode_gen_ == 0) { for (auto& c : caches) c.reset(); encode_gen_ = 1; }
  for (uint32_t i = 0; i < nthreads; ++i) {
    if (!caches[i]) caches[i] = std::make_unique<EncodeCaches>();
    caches[i]->gen = encode_gen_;
    caches[i]->sel_rec.clear();
  }
  if (nthreads > 1 && !pool_) pool_ = std::make_unique<WorkPool>(threads_);
  static const bool trace = getenv("CORDUM_ENCODE_TRACE") != nullptr;
  auto now = [] { return std::chrono::steady_clock::now(); };
  auto t_start = now();
  // parts: contiguous job ranges, more of them than threads so that a descheduled thread costs little
  uint32_t parts = nthreads == 1 ? 1u : std::min<uint32_t>(4 * nthreads, (n + 4095) / 4096);
  auto part_range = [&](uint32_t p, uint32_t np, uint32_t& a, uint32_t& b) { a = (uint32_t)((uint64_t)n * p / np); b = (uint32_t)((uint64_t)n * (p + 1) / np); };
  std::vector<uint32_t>& tid = scratch_tid_;
  std::vector<uint32_t>& ten = scratch_ten_;
  if (tid.size() < n) { tid.resize(n); ten.resize(n); }
  // ---- pass 1: topic ids, tenants
  std::vector<std::vector<uint32_t>> misses(nthreads);
  const uint32_t p1parts = parts;
  auto pass1 = [&](uint32_t p0, uint32_t p1, uint32_t w) {
    for (uint32_t p = p0; p < p1; ++p) {
      uint32_t a, b;
      part_range(p, p1parts, a, b);
      for (uint32_t j = a; j < b; ++j) {
        tid[j] = resolve_topic(env, j, *caches[w]);
        ten[j] = resolve_tenant(env, j, *caches[w]);
        if (tid[j] == kMiss) misses[w].push_back(j);
      }
    }
  };
  if (nthreads == 1) pass1(0, parts, 0);
  else pool_->parallel_for(parts, 1, pass1);
  for (auto& lst : misses)   // first sight of a topic: register it (computes its pass-row), then the id is known
    for (uint32_t j : lst) {
      uint32_t id = add_topic(span(env, env->topic, j));
      if (id == kMiss) return kDictFull;
      tid[j] = id;
    }
  auto t_pass1 = now();
  // ---- slots: hist[p][key] -> first slot of (part p, key); key = topic * classes + tenant class
  const uint32_t ncls = std::max<uint32_t>(1, tenant_classes_);
  const uint32_t nk = (uint32_t)(*topic_store_).size() * ncls;
  while (parts > 1 && (uint64_t)parts * nk > (2u << 20)) parts = (parts + 1) / 2;   // bound the counter table (8 MB)
  auto key_of = [&](uint32_t j) { return tid[j] * ncls + tenant_class_[ten[j] & 0xFFFFu]; };
  std::vector<uint32_t>& hist = scratch_hist_;
  hist.assign((size_t)parts * nk, 0);
  const uint32_t p2parts = parts;
  auto count = [&](uint32_t p0, uint32_t p1, uint32_t) {
    for (uint32_t p = p0; p < p1; ++p) {
      uint32_t a, b;
      part_range(p, p2parts, a, b);
      uint32_t* h = hist.data() + (size_t)p * nk;
      for (uint32_t j = a; j < b; ++j) h[key_of(j)]++;
    }
  };
  if (nthreads == 1) count(0, parts, 0);
  else pool_->parallel_for(parts, 1, count);
  {
    uint32_t run = 0;
    for (uint32_t k = 0; k < nk; ++k)
      for (uint32_t p = 0; p < parts; ++p) { uint32_t c = hist[(size_t)p * nk + k]; hist[(size_t)p * nk + k] = run; run += c; }
  }
  auto t_slots = now();
  // ---- pass 2: encode every job into its slot
  for (auto& m : misses) m.clear();
  auto pass2 = [&](uint32_t p0, uint32_t p1, uint32_t w) {
    for (uint32_t p = p0; p < p1; ++p) {
      uint32_t a, b;
      part_range(p, p2parts, a, b);
      uint32_t* cur = hist.data() + (size_t)p * nk;
      for (uint32_t j = a; j < b; ++j) {
        const uint32_t slot = cur[key_of(j)]++;
        out.slot_of[j] = slot;
        bool miss = false;
        encode_job(env, j, tid[j], ten[j], out.job[slot], out.route[slot], ww ? out.wide + (size_t)slot * ww : nullptr, miss, *caches[w]);
        if (miss) misses[w].push_back(j);
        if (out.job[slot].flags & JF_SELECTIVE) {
          auto& rec = caches[w]->sel_rec;
          rec.push_back(slot);
          rec.push_back((uint32_t)caches[w]->sel_ids.size());
          rec.insert(rec.end(), caches[w]->sel_ids.begin(), caches[w]->sel_ids.end());
        }
      }
    }
  };
  if (nthreads == 1) pass2(0, parts, 0);
  else pool_->parallel_for(parts, 1, pass2);
  if (trace) {
    auto ms = [](auto a, auto b) { return std::chrono::duration<double, std::milli>(b - a).count(); };
    fprintf(stderr, "encode %u jobs, %u threads, %u parts: pass1 %.2f ms, slots %.2f ms, pass2 %.2f ms\n", n, nthreads, parts,
            ms(t_start, t_pass1), ms(t_pass1, t_slots), ms(t_slots, now()));
  }
  // effective configs seen for the first time: register them, then re-encode just those jobs in place
  for (auto& lst : misses)
    for (uint32_t j : lst) {
      sv eff = span(env, env->effective_config, j);
      if (!eff.empty() && add_effcfg(eff) == kMiss) {
        if (t_.mcp_stride > CORDUM_ID16_MAX) { err = "more than 65535 distinct MCP values referenced by allow / deny lists"; return CORDUM_E_CAPACITY; }
        return kDictFull;
      }
      bool miss = false;
      const uint32_t slot = out.slot_of[j];
      encode_job(env, j, tid[j], ten[j], out.job[slot], out.route[slot], ww ? out.wide + (size_t)slot * ww : nullptr, miss, *caches[0]);
    }
  gather_selective(out, nthreads);
  return CORDUM_OK;
}

// The batch's selective list (tables.h JobRecords) from the threads' records, in ascending slot order.
void Host::gather_selective(HostRecords& out, uint32_t nthreads) const {
  std::vector<std::pair<uint32_t, const uint32_t*>> jobs;   // slot, {slot, count, ids...}
  for (uint32_t w = 0; w < nthreads; ++w) {
    const auto& rec = caches_[w]->sel_rec;
    for (size_t i = 0; i < rec.size(); i += 2 + rec[i + 1]) jobs.emplace_back(rec[i], rec.data() + i);
  }
  if (jobs.empty()) return;
  std::sort(jobs.begin(), jobs.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
  out.sel_jobs.reserve(2 * jobs.size());
  out.sel_extra.assign(1, 0u);
  for (const auto& [slot, r] : jobs) {
    uint32_t x = 0;
    if (r[1] > 2) {
      x = (uint32_t)out.sel_extra.size();
      out.sel_extra.push_back(r[1] - 2);
      out.sel_extra.insert(out.sel_extra.end(), r + 4, r + 2 + r[1]);
    }
    out.sel_jobs.push_back(slot);
    out.sel_jobs.push_back(x);
  }
}

void Host::export_dicts(std::vector<uint8_t>& blob, EncodeTables& et) const {
  blob.clear();
  et = EncodeTables{};
  const StrTable* tabs[DD_COUNT] = {&topic_ids_, &d_tenant_.table, &tenant_pol_, &d_cap_.table, &d_pack_.table, &d_actor_.table,
                                    &d_risk_.table, &d_req_.table, &d_mcp_[0].table, &d_mcp_[1].table, &d_mcp_[2].table,
                                    &d_mcp_[3].table, &label_key_, nullptr, &place_pair_, &place_key_, &d_pool_.table,
                                    &worker_slot_, &effcfg_ids_};
  StrTable label_pair;   // StrTable::pair_key(key, value) -> bit, for the rule label pairs (host keeps them as per-key lists)
  std::vector<uint64_t> keymask(std::max<size_t>(label_key_pairs_.size(), 1), 0);
  for (size_t ki = 0; ki < label_key_pairs_.size(); ++ki)
    for (auto& pv : label_key_pairs_[ki])
      if (pv.second < 64) keymask[ki] |= 1ull << pv.second;
  // label_key_ stores key -> index; the pair table needs the key string: recover it by walking the rules
  for (auto& r : policy_.rules)
    for (auto& kv : r.labels) {
      uint32_t ki = label_key_.find(kv.first, kMiss);
      if (ki == kMiss) continue;
      for (auto& pv : label_key_pairs_[ki])
        if (pv.first == kv.second && pv.second < 64) label_pair.put(StrTable::pair_key(kv.first, kv.second), pv.second);
    }
  tabs[DD_LABEL_PAIR] = &label_pair;
  for (int i = 0; i < DD_COUNT; ++i) tabs[i]->export_to(blob, et.dict[i]);
  auto append = [&](const void* p, size_t n, size_t align) {
    blob.resize((blob.size() + align - 1) / align * align);
    size_t off = blob.size();
    blob.insert(blob.end(), (const uint8_t*)p, (const uint8_t*)p + n);
    return off;
  };
  std::vector<uint32_t> tflags(topic_entries_.size());
  for (size_t i = 0; i < topic_entries_.size(); ++i) tflags[i] = topic_entries_[i].flags;
  // offsets are smuggled through the pointer fields; the engine rebases them onto the device copy of the blob
  et.topic_flags = (const uint32_t*)append(tflags.data(), tflags.size() * 4, 16);
  std::vector<uint8_t> cls = tenant_class_;
  cls.resize(std::max<size_t>(cls.size(), d_tenant_.size()), 0);
  et.tenant_class = (const uint8_t*)append(cls.data(), cls.size(), 16);
  et.label_keymask = (const uint64_t*)append(keymask.data(), keymask.size() * 8, 16);
  et.n_topics = (uint32_t)topic_entries_.size();
  et.tenant_classes = std::max<uint32_t>(1, tenant_classes_);
  sv dt = default_tenant_trim_.empty() ? sv("default") : sv(default_tenant_trim_);
  et.default_tenant = lookup_value(d_tenant_, dt) | (tenant_pol_.find(dt, 0) << 16);
  et.place_any_bit = place_any_bit_;
  et.label_empty_mask = label_empty_mask_;
  et.wide_words = WIDE_WORDS(t_.wide);
  blob.resize(blob.size() + 64);
}

Host::~Host() = default;   // here, where EncodeCaches is complete

}  // namespace cordum
