// tables.h — layout of the compiled tables and encoded job records, shared by the
// host compiler/encoder (C++) and the CUDA kernels.  Plain C structs only.
//
// Bit-parallel first-match (SURVEY.md §7 K1): for every dictionary value v of every scalar
// attribute a there is a PASS-ROW: a bit vector over rule POSITIONS whose bit p says "the rule at
// position p passes its predicate on a for v" (vacuous predicates -> 1).  A job's candidate rules =
// AND of the rows its attribute values select; the first match is the minimum original rule index
// over the surviving bits (safety_policy.go:192-204).  Positions are laid out by the compiler so
// that a job's AND is non-zero in few 128-bit words (host.cpp compile_policy):
//   * per attribute value a 64-bit SUMMARY says which words of its row hold any bit; a job ANDs the
//     summaries first and only visits the words that survive;
//   * on the device a table is stored WORD-MAJOR, tab[word][value] (16 B cells): jobs are sorted by
//     topic, so the lanes of a warp visit the same word and their gathers fall into few cache lines.
#pragma once
#include <stdint.h>
#ifdef __CUDACC__
#include <vector_types.h>
#else
typedef struct __attribute__((aligned(16))) uint4 { unsigned int x, y, z, w; } uint4;
typedef struct __attribute__((aligned(8))) uint2 { unsigned int x, y; } uint2;
#endif

/* 16-byte units (the kernels reinterpret these as uint4 / int4) */
typedef struct __attribute__((aligned(16))) Row16 { uint32_t w[4]; } Row16;
typedef struct __attribute__((aligned(16))) Load16 { int32_t active, max_parallel; float cpu, gpu; } Load16;

#define CORDUM_SEG_RULES 1024u          /* rule positions per segment (rows are padded to whole segments) */
#define CORDUM_SEG_U4 8u                /* 128-bit words per row per segment                              */
#define CORDUM_GROUP 8u                 /* lanes cooperating on one job                       */

/* dictionary ids common to every attribute */
#define CORDUM_ID_EMPTY 0u              /* raw value == ""  (never matches a non-vacuous list, safety_policy.go:297) */
#define CORDUM_ID_OTHER 1u              /* non-empty but referenced by no list                                         */

/* job flag word */
#define JF_COMBO_MASK 0x7u              /* actor_type id (0 "",1 human,2 service) * 2 + secrets_present */
#define JF_MCP_USED 0x8u
#define JF_HAS_LABELS 0x10u
#define JF_APPROVED 0x20u
#define JF_REQ_NONEMPTY 0x40u           /* len(meta.requires) > 0 (strategy_least_loaded.go:228,242)   */
#define JF_REQ_UNKNOWN 0x80u            /* a non-blank requires token no pool declares                 */
#define JF_PLACE_UNSAT 0x100u           /* a placement label no worker can satisfy                     */
#define JF_TOPIC_MISSING 0x200u         /* TrimSpace(topic) == ""   (kernel.go:171)                    */
#define JF_TOPIC_UNSUPPORTED 0x400u     /* !HasPrefix(topic,"job.") (kernel.go:174)                    */
#define JF_TOPIC_RAW_EMPTY 0x800u       /* req.Topic == ""          (strategy_least_loaded.go:41)      */
#define JF_EFF_DENIED 0x1000u           /* effective config: topic matches denied_topics (kernel.go:219)*/
#define JF_EFF_NOT_ALLOWED 0x2000u      /* allowed_topics set and topic not in it (kernel.go:223)       */
#define JF_NO_REQ 0x4000u               /* the job carries no requires token any rule lists: every rule with a
                                           requires list fails containsAll (safety_policy.go:320-330)            */
#define JF_NO_LAB 0x8000u               /* no labels, or none of the label pairs any rule lists: every rule with a
                                           labels map fails labelsMatch (safety_policy.go:332-345)               */
#define JF_SELECTIVE 0x10000u           /* the job needs selective placement pairs (DeviceTables.sel_*): JobRec.sel holds the
                                           first two (id + 1), the batch's selective list the rest; JF_PLACE_UNSAT is set
                                           too, so route_kernel leaves CORDUM_ROUTE_NO_WORKERS for route_select_kernel     */
/* row_combo index: actor_type / secrets_present combination + 6 * NO_REQ + 12 * NO_LAB (24 rows) */
#define CORDUM_COMBO_ROWS 24u
#define CORDUM_COMBO_INDEX(flags) (((flags) & JF_COMBO_MASK) + (((flags) >> 14) & 3u) * 6u)

#define CORDUM_PREF_UNKNOWN 0xFFFFFFFFu /* preferred_pool / preferred_worker_id names nothing known    */

/* DeviceTables.sum_use */
#define SUM_TENANT 1u
#define SUM_CAP 2u
#define SUM_PACK 4u
#define SUM_ACTOR 8u
#define SUM_COMBO 16u
#define SUM_RISK 32u

/* Encoded jobs: two record arrays in the SAME order - sorted by topic id (stable), so that a warp's 32
   consecutive jobs share their topic's rows.  `orig` is the job's index in the caller's batch; results are written
   there.  Dictionary ids are 16-bit (a dictionary holds only values some rule / pool / tenant policy references). */
typedef struct __attribute__((aligned(16))) JobRec {   /* 64 B: everything policy_kernel reads */
  uint32_t topic;        /* topic dictionary id (keyed by the raw topic string)                        */
  uint32_t flags;        /* JF_*                                                                       */
  uint32_t orig;         /* index of the job in the caller's batch                                     */
  uint16_t tenant;       /* tenant dictionary id (fold+trim canonical)                                 */
  uint16_t tenant_pol;   /* 1 + index into policy.Tenants by EXACT string, 0 = none                    */
  uint16_t cap, pack, actor;
  uint16_t effcfg;       /* 0 none/unparsable, else effective-config id                                */
  uint16_t mcp[4];       /* server, tool, resource, action                                             */
  uint64_t risk;         /* bit per referenced risk tag                                                */
  uint64_t req;          /* bit per referenced requires token, EqualFold canonical (rules' containsAll) */
  uint64_t lab;          /* bit per rule label pair (k,v): labels.get(k,"") == v                       */
  uint32_t sel[2];       /* JF_SELECTIVE: the job's first two selective pair ids + 1 (0 = none)        */
} JobRec;
typedef struct __attribute__((aligned(16))) RouteRec {   /* 32 B: what only route_kernel reads */
  uint64_t place_lo, place_hi;   /* placement need mask                                                */
  uint64_t req_pool;     /* bit per requires token, ToLower canonical (poolSatisfies)                  */
  uint32_t pref_pool;    /* 0 none, else 1 + pool id, or CORDUM_PREF_UNKNOWN                           */
  uint32_t pref_worker;  /* 0 none, else 1 + worker slot, or CORDUM_PREF_UNKNOWN                       */
} RouteRec;
#define CORDUM_JOB_IN_BYTES 96u
#define CORDUM_JOB_OUT_BYTES 16u
#define CORDUM_ID16_MAX 65535u

/* ---- device-side encoder (encode.cu): the host's dictionaries as probe-able images.
   A DevDict is an open-addressing table inside one byte blob: 32 B slots {u64 hash (0 = empty), u32 key offset into
   the dict's key bytes, u32 key length, u32 value, pad}, linear probing, hash = host.hpp StrTable::hash. */
typedef struct DevDict { uint32_t slots_off, mask, pool_off, pad; } DevDict;
enum {
  DD_TOPIC = 0, DD_TENANT, DD_TENANT_POL, DD_CAP, DD_PACK, DD_ACTOR, DD_RISK, DD_REQ, DD_MCP0, DD_MCP1, DD_MCP2, DD_MCP3,
  DD_LABEL_KEY, DD_LABEL_PAIR, DD_PLACE_PAIR, DD_PLACE_KEY, DD_POOL, DD_WORKER, DD_EFFCFG, DD_COUNT
};
#define CORDUM_SEL_TAG 0x80000000u      /* DD_PLACE_PAIR value of a selective pair: CORDUM_SEL_TAG | pair id (else: dense bit) */
typedef struct EncodeTables {
  const uint8_t* blob;            /* device: all dictionaries                                             */
  DevDict dict[DD_COUNT];
  const uint32_t* topic_flags;    /* device, per topic id: JF_TOPIC_* of the topic                        */
  const uint8_t* tenant_class;    /* device, per tenant id: sort class (host.hpp tenant_class_)           */
  const uint64_t* label_keymask;  /* device, per rule label key: bits of all pairs of that key            */
  uint32_t n_topics, tenant_classes;
  uint32_t default_tenant;        /* tenant id | exact-policy index << 16 of the fallback tenant          */
  uint32_t place_any_bit;
  uint64_t label_empty_mask;
  uint32_t wide_words;            /* != 0: the device encoder hands the whole batch to the host encoder            */
} EncodeTables;

/* A batch's selective list (jobs flagged JF_SELECTIVE), one array of 32-bit words:
     [n_sel_jobs x {slot j in the sorted records, x}] [extra words]
   x = 0: the job names at most two selective pairs (JobRec.sel); else extra[x] = c, extra[x+1 .. x+c] = its further pair
   ids (extra[0] is a 0 word, so x = 0 never points at a list).  Entries are in ascending j. */
typedef struct JobRecords {
  const JobRec* job;
  const RouteRec* route;
  const uint64_t* wide;   /* [n_jobs][DeviceTables.wide_words], same (sorted) order; NULL when wide_words == 0 */
  const uint2* sel_jobs;  /* the selective list (NULL when n_sel_jobs == 0)                                   */
  const uint32_t* sel_extra;
  uint32_t n_sel_jobs;
} JobRecords;

/* Wide masks.  The records hold 64 bits per mask (placement: 128).  A policy that references more than 64 distinct risk
   tags / requires tokens / label pairs, or a registry with more than 128 dense placement-label bits, spills the further
   bits into a side row of 64-bit words per job: [risk xw_risk][requires, EqualFold form xw_req][label pairs xw_lab]
   [requires, ToLower form xw_req][placement xw_place].  All xw_* are 0 in the common case and nothing of this is read.
   Selective placement pairs (DeviceTables.sel_*) take no bit here. */
typedef struct WideLayout {
  uint32_t xw_risk, xw_req, xw_lab, xw_place;
} WideLayout;
#define WIDE_WORDS(L) ((L).xw_risk + 2u * (L).xw_req + (L).xw_lab + (L).xw_place)
#define WIDE_O_REQ(L) ((L).xw_risk)
#define WIDE_O_LAB(L) ((L).xw_risk + (L).xw_req)
#define WIDE_O_REQP(L) ((L).xw_risk + (L).xw_req + (L).xw_lab)
#define WIDE_O_PLACE(L) ((L).xw_risk + 2u * (L).xw_req + (L).xw_lab)

/* Everything the kernels read besides the job columns.  Pointers are device pointers. */
#define CORDUM_POOL_CHUNK 512u
#define CORDUM_POOL_SORT_MAX 8192u
#define CORDUM_LBEST_MAX_BITS 1024u
#define CORDUM_SEL_MIN_BITS CORDUM_LBEST_MAX_BITS   /* selective pairs only in registries with more placement bits than this */
#define CORDUM_SEL_MAX_HOLDERS 32u                  /* a selective pair is carried by at most this many routable workers     */

typedef struct DeviceTables {
  /* ---- policy.  All pass-row tables live in ONE word-major array on the device: the 16 B cell of word w for value v of
     table X is rows[w * n_cells + off_X + v] (n_cells = rows of all tables together), so a lane keeps one 32-bit cell
     index per attribute for the whole tile and a word costs one base computation.
     sum_X[v] bit g = "row v has a bit in word group g" (group g = words [g*sum_group, (g+1)*sum_group)). */
  uint32_t n_rules, n_seg, row_u4;            /* row_u4 = n_seg * 8 128-bit words per pass-row                       */
  uint32_t sum_group;                         /* words per summary bit = ceil(row_u4 / 64)                            */
  uint32_t sum_use;                           /* SUM_* bits: attributes whose summaries are worth ANDing              */
  const Row16* rows;  uint32_t n_cells;
  uint32_t off_topic, off_tenant, off_cap, off_pack, off_actor, off_combo, off_risk, off_mcp[4];
  uint32_t n_topic;                           /* topic rows (the dictionary grows on first sight of a topic)          */
  const uint64_t *sum_topic, *sum_tenant, *sum_cap, *sum_pack, *sum_actor, *sum_combo, *sum_risk;
  const uint32_t* chk_words;                  /* bit per position: the rule carries a requires/labels need-mask       */
  const uint64_t* rule_req_need;              /* per rule: requires tokens it needs (subset test)       */
  const uint64_t* rule_lab_need;              /* per rule: label pairs it needs                          */
  WideLayout wide;  uint32_t wide_words;      /* extra mask words (see WideLayout); wide_words = WIDE_WORDS(wide)           */
  const uint64_t* rule_need_x;                /* [n_rules][xw_req + xw_lab]: the rules' needs beyond bit 63               */
  const uint64_t* pool_req_x;                 /* [n_pools][xw_req]                                                        */
  const uint64_t* req_blank_x;                /* [xw_req]                                                                  */
  const uint64_t* pos_label_x;                /* [n_pos][xw_place]: placement label bits 128...                           */
  const uint8_t* rule_dec;                    /* per rule: CORDUM_DEC_* | 0x80 if constraints non-empty */
  const uint32_t* pos2rule;                   /* bit position -> rule index                              */
  /* tenant-level MCP lists (kernel.go:190-195) and effective-config overlay (kernel.go:218-231):
     verdict per (entry, field, value id): 0 ok, 1 denied, 2 not allowed */
  const uint8_t* tenant_mcp; uint32_t mcp_stride;   /* [n_tenant_pol][4][mcp_stride]                    */
  const uint8_t* eff_mcp;                           /* [n_effcfg+1][4][mcp_stride]                      */
  const uint8_t* eff_topic; uint32_t topic_stride;  /* [n_effcfg+1][topic_stride] bit0 denied, bit1 not-allowed */
  /* ---- routing */
  const uint32_t* topic_pool_off;             /* per topic id: start in pool_list                       */
  const uint32_t* topic_pool_cnt;             /* per topic id: number of (deduplicated) pools           */
  const uint32_t* pool_list;
  const uint64_t* pool_req_mask;              /* per pool: declared requires tokens                     */
  const uint8_t* pool_req_nonempty;           /* per pool: len(pool.requires) > 0                       */
  uint64_t req_blank_mask;                    /* bit of the token that trims to "" (ignored by pools)   */
  uint32_t n_pools;
  /* ---- workers (pool-sorted order = "pos") */
  uint32_t n_pos;                             /* routable workers                                       */
  const uint32_t* pool_off;                   /* [n_pools+1] pos ranges                                 */
  const uint32_t* pos_pool;                   /* pool id of pos                                         */
  const uint32_t* pos_slot;                   /* caller slot of pos                                     */
  const uint32_t* pos_rank;                   /* rank of pos in ascending worker_id byte order          */
  const uint32_t* slot_pos;                   /* [n_slots] 1 + pos, 0 = not routable                    */
  const uint32_t* rank_slot;                  /* [n_slots] slot of rank                                 */
  const uint32_t* rank_pos;                   /* [n_slots] pos of rank (routable workers only)          */
  const uint64_t* pos_label_lo;               /* placement label mask                                   */
  const uint64_t* pos_label_hi;
  const Load16* loads;                          /* [n_slots] {active, max_parallel, cpu(f32), gpu(f32)}   */
  uint64_t* pos_key;                          /* derived: (orderable score << 32) | rank; score field all-ones = overloaded */
  uint64_t* skey;                             /* derived: per pool, keys in ascending order (load-sorted view of the pool)  */
  uint8_t* pool_sorted;                       /* derived: 1 if the pool's sorted view is valid (pool fits the sort buffer)  */
  uint32_t* pool_done;                        /* derived scratch: merge CTAs of the pool that have signed off this epoch   */
  uint32_t* pool_nok;                         /* derived: workers of the pool that are NOT overloaded (= prefix of the sorted view) */
  uint32_t* lbm;                              /* derived: label bitmaps over the sorted view: lbm[lbm_off[p] + bit*words(p) + w],
                                                 bit i of word w = "sorted worker 32w+i carries label bit"               */
  const uint32_t* lbm_off;                    /* [n_pools] word offset of the pool's bitmaps                               */
  uint4* lbest;                               /* derived, or NULL (place_bits > CORDUM_LBEST_MAX_BITS): per (pool, label bit) what a
                                                 job that requires exactly that one label gets from the pool's sorted view -
                                                 {key lo, key hi (KEY_NONE: nobody), 1 | 2 = tie inside the pool, matching workers}  */
  uint32_t place_bits;                        /* dense label bits in use (beyond 128: pos_label_x)                         */
  /* selective placement pairs: pairs (k, v != "") carried by at most CORDUM_SEL_MAX_HOLDERS routable workers, in a registry
     whose placement labels need more than CORDUM_SEL_MIN_BITS bits.  They have no dense bit, bitmap row or lbest row:
     route_select_kernel finds a job's candidates through the holder lists instead.                                    */
  uint32_t n_sel;                             /* selective pairs (0: none, route_select_kernel is never launched)          */
  const uint32_t* sel_off;                    /* [n_sel+1] range of the pair in sel_pos                                    */
  const uint32_t* sel_pos;                    /* pos of every routable worker carrying the pair, ascending per pair         */
  const uint32_t* pos_sel_off;                /* [n_pos+1] range of the worker in pos_sel                                  */
  const uint32_t* pos_sel;                    /* selective pair ids the worker carries, ascending per worker                */
  /* worker-table refresh: a pool is cut into chunks of CORDUM_POOL_CHUNK workers, one CTA sorts one chunk, a second
     kernel merges the chunks of pools that have more than one (pools above CORDUM_POOL_SORT_MAX stay unsorted)       */
  const uint32_t* chunk_pool;                 /* [n_chunks] pool of the chunk                                              */
  const uint32_t* pool_chunk0;                /* [n_pools+1] first chunk of the pool                                       */
  const uint32_t* merge_list;                 /* [n_merge] chunks worker_merge_kernel runs (all chunks of a multi-chunk
                                                 sortable pool; chunk 0 only of an unsortable pool)                       */
  uint32_t n_chunks, n_merge;
  uint32_t merge_smem;                        /* bytes of shared memory worker_merge_kernel needs (largest merged pool)    */
  uint64_t* ckey;                             /* derived scratch: per chunk, its keys in ascending order                   */
  uint64_t* pool_best;                        /* derived: min key per pool (~0 = none)                  */
  uint32_t* pool_mincnt;                      /* derived: workers in the pool sharing the min score     */
} DeviceTables;
