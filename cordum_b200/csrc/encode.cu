// encode.cu — the job encoder on the device.
//
// Request normalisation + dictionary coding of string-level envelopes (kernel.go:133-185, 348-414;
// strategy_least_loaded.go:46-62,195-222) is the host-side cost that bounds the end-to-end rate: ~30 ms of lookups per
// million envelopes on 16 cores, against 0.2 ms of kernels.  This file does the same work on the GPU: the raw envelope
// bytes (string arena + span columns, ~250 B per job) cross PCIe once, and three kernels turn them into the
// topic-sorted job records policy_kernel / route_kernel read:
//     encode_key_kernel     thread per job: topic + tenant lookups -> sort key (topic id, tenant class); histogram
//     encode_scan_kernel    one CTA: exclusive prefix sum of the histogram -> first slot of every key
//     encode_job_kernel     thread per job: every other lookup, flags and masks; claims a slot of its key; writes
//                           the 64 B + 32 B records there and slot_of[job]
// The dictionaries are the host's own hash tables, uploaded as they are (tables.h DevDict): the device hashes with the
// same function and probes the same way, so a lookup gives the same id on both sides by construction.  The host encoder
// (host.cpp Host::encode_job) is the specification of this file; tests compare the two record for record.
//
// What stays on the host: anything that needs Unicode tables (TrimSpace / EqualFold / ToLower on non-ASCII text), the
// first sight of a topic or of an effective config (the host has to compute pass-rows / parse JSON), and strings longer
// than kMaxStr, and a selective placement pair (tables.h DeviceTables.sel_*).  A job that meets one of these raises the
// batch's fallback flag and the host encodes the batch instead.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/cordum_b200.h"
#include "kernels.h"

namespace {

constexpr uint32_t kMiss = 0xFFFFFFFFu;
constexpr uint32_t kMaxStr = 4096;   // longer strings (only effective-config payloads come close) go to the host

struct Str { const uint8_t* p; uint32_t n; };

__device__ __forceinline__ Str span_of(const uint8_t* arena, const cordum_str* col, uint32_t i) {
  if (!col) return Str{arena, 0};
  const uint2 s = __ldg(reinterpret_cast<const uint2*>(col) + i);
  return Str{arena + s.x, s.y};
}
// byte-addressed little-endian reads (the arena has no alignment)
__device__ __forceinline__ uint64_t rd8(const uint8_t* p) {
  uint64_t v = 0;
#pragma unroll
  for (int k = 0; k < 8; ++k) v |= (uint64_t)p[k] << (8 * k);
  return v;
}
__device__ __forceinline__ uint64_t rd4(const uint8_t* p) {
  return (uint64_t)p[0] | ((uint64_t)p[1] << 8) | ((uint64_t)p[2] << 16) | ((uint64_t)p[3] << 24);
}
__device__ __forceinline__ uint64_t mix(uint64_t a, uint64_t b) { return (a * b) ^ __umul64hi(a, b); }
__device__ __forceinline__ uint64_t lower8(uint64_t v) {
  const uint64_t v7 = v & 0x7F7F7F7F7F7F7F7Full;
  const uint64_t up = (v7 + 0x3F3F3F3F3F3F3F3Full) & ~(v7 + 0x2525252525252525ull) & ~v & 0x8080808080808080ull;
  return v | (up >> 2);
}
// host.hpp StrTable::hash_impl, bit for bit
template <bool FOLD>
__device__ uint64_t hash_str(Str s) {
  const uint8_t* p = s.p;
  uint32_t n = s.n;
  uint64_t h = 0x9E3779B97F4A7C15ull ^ ((uint64_t)n * 0xA0761D6478BD642Full);
  while (n > 16) {
    uint64_t a = rd8(p), b = rd8(p + 8);
    if (FOLD) { a = lower8(a); b = lower8(b); }
    h = mix(a ^ 0xE7037ED1A0B428DBull, b ^ h);
    p += 16; n -= 16;
  }
  uint64_t a = 0, b = 0;
  if (n >= 8) { a = rd8(p); b = rd8(p + n - 8); }
  else if (n >= 4) { a = rd4(p); b = rd4(p + n - 4); }
  else if (n > 0) { a = ((uint64_t)p[0] << 16) | ((uint64_t)p[n >> 1] << 8) | p[n - 1]; }
  if (FOLD) { a = lower8(a); b = lower8(b); }
  h = mix(a ^ 0x8EBC6AF09C88C6E3ull, b ^ h);
  return h | 1;
}
// the pair key of host.hpp StrTable::pair_key (len(a) as 4 little-endian bytes, a, b), built in `scratch`; returns its
// hash, and the key is Str{scratch, 4 + a.n + b.n}
__device__ uint64_t hash_pair(Str a, Str b, uint8_t* scratch) {
#pragma unroll
  for (int i = 0; i < 4; ++i) scratch[i] = (uint8_t)(a.n >> (8 * i));
  for (uint32_t i = 0; i < a.n; ++i) scratch[4 + i] = a.p[i];
  for (uint32_t i = 0; i < b.n; ++i) scratch[4 + a.n + i] = b.p[i];
  return hash_str<false>(Str{scratch, 4 + a.n + b.n});
}

__device__ __forceinline__ uint8_t lower1(uint8_t c) { return (c >= 'A' && c <= 'Z') ? (uint8_t)(c + 32) : c; }

// probe: exact (FOLD = false) or "key is ASCII, stored string is its lower-cased form" (FOLD = true)
template <bool FOLD>
__device__ uint32_t dict_find(const EncodeTables& E, int which, Str key, uint64_t h, uint32_t miss) {
  const DevDict d = E.dict[which];
  const uint8_t* slots = E.blob + d.slots_off;
  const uint8_t* pool = E.blob + d.pool_off;
  for (uint32_t i = (uint32_t)h & d.mask;; i = (i + 1) & d.mask) {
    const uint4 s = __ldg(reinterpret_cast<const uint4*>(slots + (size_t)i * 32));
    const uint64_t sh = ((uint64_t)s.y << 32) | s.x;
    if (sh == 0) return miss;
    if (sh == h && s.w == key.n) {
      const uint8_t* c = pool + s.z;
      uint32_t k = 0;
      for (; k < key.n; ++k) if ((FOLD ? lower1(key.p[k]) : key.p[k]) != c[k]) break;
      if (k == key.n) return __ldg(reinterpret_cast<const uint32_t*>(slots + (size_t)i * 32 + 16));
    }
  }
}
__device__ __forceinline__ uint32_t find_exact(const EncodeTables& E, int which, Str key, uint32_t miss) {
  return dict_find<false>(E, which, key, hash_str<false>(key), miss);
}

__device__ __forceinline__ bool is_ascii(Str s) {
  uint8_t acc = 0;
  for (uint32_t i = 0; i < s.n; ++i) acc |= s.p[i];
  return acc < 0x80;
}
__device__ __forceinline__ bool ascii_space(uint8_t c) { return c == ' ' || (c >= 0x09 && c <= 0x0D); }
// strings.TrimSpace for ASCII text (the caller has ruled out bytes >= 0x80)
__device__ __forceinline__ Str trim_ascii(Str s) {
  while (s.n && ascii_space(s.p[0])) { ++s.p; --s.n; }
  while (s.n && ascii_space(s.p[s.n - 1])) --s.n;
  return s;
}
__device__ __forceinline__ bool str_eq(Str a, const char* lit, uint32_t n) {
  if (a.n != n) return false;
  for (uint32_t i = 0; i < n; ++i) if (a.p[i] != (uint8_t)lit[i]) return false;
  return true;
}
__device__ __forceinline__ bool str_eq(Str a, Str b) {
  if (a.n != b.n) return false;
  for (uint32_t i = 0; i < a.n; ++i) if (a.p[i] != b.p[i]) return false;
  return true;
}
__device__ __forceinline__ bool fold_eq_lit(Str a, const char* lit, uint32_t n) {   // ASCII a, lower-case literal
  if (a.n != n) return false;
  for (uint32_t i = 0; i < n; ++i) if (lower1(a.p[i]) != (uint8_t)lit[i]) return false;
  return true;
}
#define LIT(s) s, (uint32_t)(sizeof(s) - 1)

// containsString semantics (safety_policy.go:296-306): id of EqualFold(TrimSpace(raw)); `bad` = needs the host
__device__ uint32_t lookup_value(const EncodeTables& E, int which, Str raw, bool& bad) {
  if (raw.n == 0) return CORDUM_ID_EMPTY;
  if (raw.n > kMaxStr || !is_ascii(raw)) { bad = true; return CORDUM_ID_OTHER; }
  const Str t = trim_ascii(raw);
  return dict_find<true>(E, which, t, hash_str<true>(t), CORDUM_ID_OTHER);
}

// tenant (kernel.go:134-169): dictionary id | exact-tenant policy index << 16
__device__ uint32_t resolve_tenant(const EncodeParams& P, uint32_t j, bool& bad) {
  const EncodeTables& E = P.et;
  const bool has_meta = P.has_meta && P.has_meta[j];
  Str t = span_of(P.arena, P.tenant, j);
  if (t.n > kMaxStr || !is_ascii(t)) { bad = true; return E.default_tenant; }
  t = trim_ascii(t);
  if (t.n == 0 && has_meta) {
    t = span_of(P.arena, P.meta_tenant_id, j);
    if (t.n > kMaxStr || !is_ascii(t)) { bad = true; return E.default_tenant; }
    t = trim_ascii(t);
  }
  if (t.n == 0) return E.default_tenant;
  const uint32_t id = dict_find<true>(E, DD_TENANT, t, hash_str<true>(t), CORDUM_ID_OTHER);
  const uint32_t tp = find_exact(E, DD_TENANT_POL, t, 0);
  return id | (tp << 16);
}

// labels that never constrain placement (filterPlacementLabels, strategy_least_loaded.go:195-222)
__device__ bool placement_skips(Str k) {
  switch (k.n) {
    case 6: return str_eq(k, LIT("run_id"));
    case 7: return str_eq(k, LIT("step_id")) || str_eq(k, LIT("node_id"));
    case 9: return str_eq(k, LIT("worker_id"));
    case 11: return str_eq(k, LIT("workflow_id"));
    case 14: return str_eq(k, LIT("preferred_pool"));
    case 15: return str_eq(k, LIT("secrets_present"));
    case 16: return str_eq(k, LIT("approval_granted"));
    case 19: return str_eq(k, LIT("preferred_worker_id"));
    default: return false;
  }
}
// mcp label aliases (kernel.go:400-403): field*3 + variant, or -1
__device__ int mcp_key(Str k) {
  if (k.n < 7 || k.p[0] != 'm' || k.p[1] != 'c' || k.p[2] != 'p') return -1;
  if (str_eq(k, LIT("mcp.server"))) return 0;
  if (str_eq(k, LIT("mcp_server"))) return 1;
  if (str_eq(k, LIT("mcpServer"))) return 2;
  if (str_eq(k, LIT("mcp.tool"))) return 3;
  if (str_eq(k, LIT("mcp_tool"))) return 4;
  if (str_eq(k, LIT("mcpTool"))) return 5;
  if (str_eq(k, LIT("mcp.resource"))) return 6;
  if (str_eq(k, LIT("mcp_resource"))) return 7;
  if (str_eq(k, LIT("mcpResource"))) return 8;
  if (str_eq(k, LIT("mcp.action"))) return 9;
  if (str_eq(k, LIT("mcp_action"))) return 10;
  if (str_eq(k, LIT("mcpAction"))) return 11;
  return -1;
}

}  // namespace

// ------------------------------------------------------------------ pass 1: sort keys
__global__ void __launch_bounds__(256) encode_key_kernel(EncodeParams P) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P.n_jobs) return;
  const EncodeTables& E = P.et;
  bool bad = E.wide_words != 0;   // masks wider than the records' fields (tables.h WideLayout): the host encoder writes those
  const Str topic = span_of(P.arena, P.topic, j);
  uint32_t tid = topic.n > kMaxStr ? kMiss : find_exact(E, DD_TOPIC, topic, kMiss);   // keyed by the RAW string
  if (tid == kMiss) { bad = true; tid = 0; }
  const uint32_t ten = resolve_tenant(P, j, bad);
  if (bad) atomicOr(P.fallback, 1u);
  const uint32_t key = tid * E.tenant_classes + __ldg(E.tenant_class + (ten & 0xFFFFu));
  P.tid[j] = tid;
  P.ten[j] = ten;
  P.key[j] = key;
  atomicAdd(P.hist + key, 1u);
}

// ------------------------------------------------------------------ pass 1b: exclusive scan of the histogram (one CTA)
__global__ void __launch_bounds__(1024) encode_scan_kernel(uint32_t* hist, uint32_t n_keys) {
  __shared__ uint32_t s_part[1024];
  const uint32_t tid = threadIdx.x, per = (n_keys + 1023u) / 1024u;
  const uint32_t a = tid * per, b = a + per < n_keys ? a + per : n_keys;
  uint32_t sum = 0;
  for (uint32_t i = a; i < b; ++i) sum += hist[i];
  s_part[tid] = sum;
  __syncthreads();
  for (uint32_t off = 1; off < 1024; off <<= 1) {   // inclusive scan of the per-thread sums
    uint32_t v = tid >= off ? s_part[tid - off] : 0;
    __syncthreads();
    s_part[tid] += v;
    __syncthreads();
  }
  uint32_t run = tid ? s_part[tid - 1] : 0;
  for (uint32_t i = a; i < b; ++i) { const uint32_t c = hist[i]; hist[i] = run; run += c; }
}

// ------------------------------------------------------------------ pass 2: the records
__global__ void __launch_bounds__(128) encode_job_kernel(EncodeParams P) {
  const uint32_t j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= P.n_jobs) return;
  const EncodeTables& E = P.et;
  const uint8_t* A = P.arena;
  bool bad = false;
  const uint32_t tid = P.tid[j], ten = P.ten[j];
  uint32_t flags = __ldg(E.topic_flags + tid);
  const bool has_meta = P.has_meta && P.has_meta[j];
  // ---- meta (policyMetaFromRequest, kernel.go:348-368)
  Str cap{A, 0}, pack{A, 0}, actor = span_of(A, P.principal_id, j);
  int at = 0;
  if (has_meta) {
    cap = span_of(A, P.capability, j);
    pack = span_of(A, P.pack_id, j);
    const Str a = span_of(A, P.actor_id, j);
    if (a.n) actor = a;
    const int raw_at = P.actor_type ? P.actor_type[j] : 0;
    at = (raw_at == 1 || raw_at == 2) ? raw_at : 0;
  }
  const uint32_t id_cap = lookup_value(E, DD_CAP, cap, bad), id_pack = lookup_value(E, DD_PACK, pack, bad),
                 id_actor = lookup_value(E, DD_ACTOR, actor, bad);
  // ---- risk tags / requires
  uint64_t risk = 0, req = 0, req_pool = 0;
  bool secrets_tag = false;
  if (has_meta && P.risk_off)
    for (uint32_t k = P.risk_off[j]; k < P.risk_off[j + 1]; ++k) {
      const Str tag = span_of(A, P.risk_tags, k);
      if (tag.n == 0) continue;
      if (tag.n > kMaxStr || !is_ascii(tag)) { bad = true; continue; }
      if (fold_eq_lit(tag, LIT("secrets"))) secrets_tag = true;   // kernel.go:387-391 (no trim)
      const uint32_t id = lookup_value(E, DD_RISK, tag, bad);
      if (id >= 2 && id - 2 < 64) risk |= 1ull << (id - 2);
    }
  if (has_meta && P.requires_off) {
    const uint32_t a = P.requires_off[j], b = P.requires_off[j + 1];
    if (b > a) flags |= JF_REQ_NONEMPTY;
    for (uint32_t k = a; k < b; ++k) {
      const Str tok = span_of(A, P.requires_, k);
      if (tok.n > kMaxStr || !is_ascii(tok)) { bad = true; continue; }
      // ASCII token: the EqualFold and the ToLower canonical forms coincide (host.cpp encode_job)
      const Str t = trim_ascii(tok);
      const uint32_t id = dict_find<true>(E, DD_REQ, t, hash_str<true>(t), 0);
      if (id >= 2 && id - 2 < 64) { req |= 1ull << (id - 2); req_pool |= 1ull << (id - 2); }
      else if (t.n != 0) flags |= JF_REQ_UNKNOWN;   // no pool declares it -> no pool satisfies (:255-262)
    }
  }
  // ---- labels: one pass
  uint64_t lab = E.label_empty_mask, place[2] = {0, 0};
  Str mcpv[12];
#pragma unroll
  for (int i = 0; i < 12; ++i) mcpv[i] = Str{A, 0};
  Str secrets_label{A, 0}, pref_pool{A, 0}, pref_worker{A, 0};
  bool have_secrets_label = false;
  const uint32_t la = P.label_off ? P.label_off[j] : 0, lb = P.label_off ? P.label_off[j + 1] : 0;
  if (lb > la) flags |= JF_HAS_LABELS;
  uint8_t scratch[520];
  for (uint32_t k = la; k < lb; ++k) {
    const Str key = span_of(A, P.label_keys, k), val = span_of(A, P.label_vals, k);
    bool shadowed = false;   // map semantics: a later entry with the same key wins
    for (uint32_t k2 = k + 1; k2 < lb && !shadowed; ++k2) shadowed = str_eq(span_of(A, P.label_keys, k2), key);
    if (shadowed) continue;
    if (key.n + val.n > 512) { bad = true; continue; }   // the pair probes build the 4 + key + value byte pair key in scratch
    // rule label pairs: labels.get(k,"") == v
    const uint32_t ki = find_exact(E, DD_LABEL_KEY, key, kMiss);
    if (ki != kMiss) {
      const uint64_t keymask = __ldg(E.label_keymask + ki);
      const uint32_t bit = dict_find<false>(E, DD_LABEL_PAIR, Str{scratch, 4 + key.n + val.n}, hash_pair(key, val, scratch), kMiss);
      lab = (lab & ~keymask) | (bit < 64 ? 1ull << bit : 0ull);
    }
    const int mk = mcp_key(key);
    if (mk >= 0) {
      if (val.n > kMaxStr || !is_ascii(val)) bad = true; else mcpv[mk] = trim_ascii(val);
    }
    if (str_eq(key, LIT("secrets_present"))) {
      if (val.n > kMaxStr || !is_ascii(val)) bad = true; else { secrets_label = trim_ascii(val); have_secrets_label = true; }
    } else if (str_eq(key, LIT("preferred_pool"))) pref_pool = val;
    else if (str_eq(key, LIT("preferred_worker_id"))) pref_worker = val;
    // placement constraint?
    const bool cordum_prefix = key.n >= 7 && str_eq(Str{key.p, 7}, LIT("cordum."));
    if (!(placement_skips(key) || cordum_prefix)) {
      uint32_t bit;
      if (val.n) {
        bit = dict_find<false>(E, DD_PLACE_PAIR, Str{scratch, 4 + key.n + val.n}, hash_pair(key, val, scratch), kMiss);
        if (bit == kMiss) flags |= JF_PLACE_UNSAT;
        else if (bit & CORDUM_SEL_TAG) bad = true;   // a selective pair: the host encoder writes the batch's selective list
      } else {
        bit = find_exact(E, DD_PLACE_KEY, key, kMiss);
        if (bit == kMiss) bit = E.place_any_bit;   // no worker carries this key: any labelled worker passes
      }
      if (bit != kMiss && bit < 128) place[bit >> 6] |= 1ull << (bit & 63);   // bits beyond 128: wide tables, the batch goes to the host encoder
    }
  }
  // ---- MCP request (extractMCPRequest, kernel.go:395-414) and secrets (kernel.go:381-393)
  uint32_t mid[4];
  bool used = false;
#pragma unroll
  for (int f = 0; f < 4; ++f) {
    Str v = mcpv[f * 3];
    if (v.n == 0) v = mcpv[f * 3 + 1];
    if (v.n == 0) v = mcpv[f * 3 + 2];
    mid[f] = v.n ? dict_find<true>(E, DD_MCP0 + f, v, hash_str<true>(v), CORDUM_ID_OTHER) : CORDUM_ID_EMPTY;   // already trimmed, ASCII
    used |= v.n != 0;
  }
  if (used) flags |= JF_MCP_USED;
  bool secrets = secrets_tag;
  if (have_secrets_label && secrets_label.n)
    secrets = str_eq(secrets_label, LIT("true")) || str_eq(secrets_label, LIT("1")) || fold_eq_lit(secrets_label, LIT("yes"));
  flags |= (uint32_t)(at * 2 + (secrets ? 1 : 0));
  if (req == 0) flags |= JF_NO_REQ;
  if (!(flags & JF_HAS_LABELS) || lab == 0) flags |= JF_NO_LAB;
  // ---- routing hints
  uint32_t pp = 0, pw = 0;
  if (pref_pool.n) {
    const uint32_t id = pref_pool.n > kMaxStr ? 0 : find_exact(E, DD_POOL, pref_pool, 0);
    pp = id >= 2 ? id - 1 : CORDUM_PREF_UNKNOWN;
  }
  if (pref_worker.n) {
    const uint32_t s = pref_worker.n > kMaxStr ? kMiss : find_exact(E, DD_WORKER, pref_worker, kMiss);
    pw = s != kMiss ? s + 1 : CORDUM_PREF_UNKNOWN;
  }
  // ---- effective config
  const Str eff = span_of(A, P.effective_config, j);
  uint32_t eid = 0;
  if (eff.n) {
    eid = eff.n > kMaxStr ? kMiss : find_exact(E, DD_EFFCFG, eff, kMiss);
    if (eid == kMiss) { bad = true; eid = 0; }   // first sight: the host parses and registers it
  }
  if (P.approved && P.approved[j]) flags |= JF_APPROVED;
  if (bad) atomicOr(P.fallback, 1u);

  // ---- claim a slot of this job's key and write the records there
  const uint32_t slot = atomicAdd(P.hist + P.key[j], 1u);
  P.slot_of[j] = slot;
  uint4* jo = reinterpret_cast<uint4*>(P.out_job + slot);
  jo[0] = make_uint4(tid, flags, j, ten);
  jo[1] = make_uint4(id_cap | (id_pack << 16), id_actor | (eid << 16), mid[0] | (mid[1] << 16), mid[2] | (mid[3] << 16));
  jo[2] = make_uint4((uint32_t)risk, (uint32_t)(risk >> 32), (uint32_t)req, (uint32_t)(req >> 32));
  jo[3] = make_uint4((uint32_t)lab, (uint32_t)(lab >> 32), 0u, 0u);
  uint4* ro = reinterpret_cast<uint4*>(P.out_route + slot);
  ro[0] = make_uint4((uint32_t)place[0], (uint32_t)(place[0] >> 32), (uint32_t)place[1], (uint32_t)(place[1] >> 32));
  ro[1] = make_uint4((uint32_t)req_pool, (uint32_t)(req_pool >> 32), pp, pw);
}

// ------------------------------------------------------------------ launcher
cudaError_t launch_encode(const EncodeParams& P, uint32_t n_keys, cudaStream_t s) {
  if (P.n_jobs == 0) return cudaSuccess;
  cudaError_t e = cudaMemsetAsync(P.hist, 0, (size_t)n_keys * sizeof(uint32_t), s);
  if (e != cudaSuccess) return e;
  e = cudaMemsetAsync(P.fallback, 0, sizeof(uint32_t), s);
  if (e != cudaSuccess) return e;
  encode_key_kernel<<<(P.n_jobs + 255) / 256, 256, 0, s>>>(P);
  encode_scan_kernel<<<1, 1024, 0, s>>>(P.hist, n_keys);
  encode_job_kernel<<<(P.n_jobs + 127) / 128, 128, 0, s>>>(P);
  return cudaGetLastError();
}
