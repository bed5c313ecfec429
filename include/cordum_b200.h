/* cordum_b200.h — C ABI of the H100-native (sm_90a) policy-gate + dispatch engine.
 *
 * This is the drop-in boundary for ONE path of cordum-io/cordum: the batched
 * form of
 *   safetykernel.(*server).evaluate        core/controlplane/safetykernel/kernel.go:129-257
 *   config.(*SafetyPolicy).Evaluate        core/infra/config/safety_policy.go:187-206
 *   scheduler.(*Engine).checkSafetyDecision post-step   core/controlplane/scheduler/engine.go:524-531
 *   scheduler.(*LeastLoadedStrategy).PickSubject        core/controlplane/scheduler/strategy_least_loaded.go:40-136
 *
 * The reference has no FFI; its seams are Go interfaces and one gRPC service
 * (SURVEY.md §8b).  Each entry point below names the reference call it stands
 * behind; INTEGRATION.md shows the cgo adapters a maintainer would add.
 *
 * Conventions
 *   - plain pointers + sizes only; no C++/torch types cross this boundary
 *   - every function returns int32 status: 0 = OK, <0 = error (CORDUM_E_*);
 *     cordum_last_error() returns a thread-local message owned by the library
 *   - strings are (offset,len) spans into a caller-owned byte arena; the
 *     library never keeps a caller pointer after the call returns (cgo rule)
 *   - the library owns every buffer it allocates (pinned host + device)
 *   - any CUDA failure makes the handle sticky-failed: callers must then fail
 *     closed (DENY / retryable routing error), never fall back to a CPU path
 */
#ifndef CORDUM_B200_H
#define CORDUM_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* ---------------------------------------------------------------- status */
#define CORDUM_OK 0
#define CORDUM_E_INVALID (-1)   /* bad argument / malformed input document        */
#define CORDUM_E_CAPACITY (-2)  /* a table outgrew its bound: 65,535 values per dictionary, 65,536 placement-label keys +
                                   pairs per registry, 8 GiB of label bitmaps (dense bits only: pairs carried by <= 32
                                   workers in registries above 1,024 label bits have none), 4 GiB of wide-mask rows per
                                   batch; the previous tables stay in force */
#define CORDUM_E_CUDA (-3)      /* CUDA runtime / kernel failure (sticky)         */
#define CORDUM_E_STATE (-4)     /* call order violated (e.g. dispatch before load)*/
#define CORDUM_E_NODEVICE (-5)  /* no CUDA device: the product has NO CPU path    */
#define CORDUM_E_STALE (-6)     /* tables were reloaded after the batch was encoded: encode it again and retry */

/* ------------------------------------------------------ wire: string spans */
typedef struct cordum_str {
  uint32_t off; /* byte offset into the arena   */
  uint32_t len; /* byte length; 0 = empty string */
} cordum_str;

/* Columnar batch of string-level job envelopes.
 *
 * Field set = what evaluate()/PickSubject() read from CAP v2
 * PolicyCheckRequest / JobRequest (SURVEY.md App. B):
 *   kernel.go:133-138 (topic, tenant, meta.tenant_id), :348-368 (meta),
 *   :381-414 (labels: secrets_present, mcp.*), :218 (effective_config),
 *   strategy_least_loaded.go:46-62 (labels, meta.requires, raw topic).
 * List-valued fields are CSR: entries [off[j], off[j+1]) belong to job j.
 * Labels are a map: keys unique per job (if repeated, the last one wins).
 */
typedef struct cordum_envelopes {
  uint32_t n_jobs;
  const uint8_t* arena;
  uint64_t arena_len;
  const cordum_str* topic;            /* req.Topic, raw (untrimmed)                         */
  const cordum_str* tenant;           /* PolicyCheckRequest.Tenant (scheduler route: ExtractTenant, tenant.go:8-21) */
  const cordum_str* principal_id;     /* PrincipalId (actor-id fallback, kernel.go:352,364)  */
  const cordum_str* effective_config; /* raw JSON bytes, len 0 = absent (safety_client.go:91-95) */
  const uint8_t* has_meta;            /* req.Meta != nil                                    */
  const cordum_str* meta_tenant_id;   /* Meta.TenantId                                      */
  const cordum_str* actor_id;         /* Meta.ActorId                                       */
  const uint8_t* actor_type;          /* 0 unspecified, 1 human, 2 service (kernel.go:370)  */
  const cordum_str* capability;       /* Meta.Capability                                    */
  const cordum_str* pack_id;          /* Meta.PackId                                        */
  const uint32_t* risk_off;           /* n_jobs+1 */
  const cordum_str* risk_tags;        /* Meta.RiskTags                                      */
  const uint32_t* requires_off;       /* n_jobs+1 */
  const cordum_str* requires_;        /* Meta.Requires                                      */
  const uint32_t* label_off;          /* n_jobs+1 */
  const cordum_str* label_keys;       /* req.Labels                                         */
  const cordum_str* label_vals;
  const uint8_t* approved;            /* may be NULL. 1 = host verified the approval record and
                                         job hash (engine.go:484-522): policy is bypassed     */
} cordum_envelopes;

/* Worker registry snapshot = map[worker_id]*Heartbeat (registry_memory.go:71-84),
 * columnar.  Index in these arrays is the worker "slot" reported in results. */
typedef struct cordum_workers {
  uint32_t n_workers;
  const uint8_t* arena;
  uint64_t arena_len;
  const cordum_str* worker_id;
  const cordum_str* pool;
  const int32_t* active_jobs;
  const int32_t* max_parallel_jobs;
  const float* cpu_load;
  const float* gpu_utilization;
  const uint32_t* label_off; /* n_workers+1 */
  const cordum_str* label_keys;
  const cordum_str* label_vals;
} cordum_workers;

/* Per-worker load record: the only heartbeat fields that change between
 * heartbeats of a live worker.  16 B; the multi-GPU exchange all-gathers these. */
typedef struct cordum_worker_load {
  int32_t active_jobs;
  int32_t max_parallel_jobs;
  float cpu_load;
  float gpu_utilization;
} cordum_worker_load;

/* ------------------------------------------------------- result record */
/* decision codes (DecisionType, core/protocol/pb/v1/pb.go:61-66; numeric values are
 * this ABI's own, the Go adapter maps them) */
#define CORDUM_DEC_UNSPECIFIED 0
#define CORDUM_DEC_ALLOW 1
#define CORDUM_DEC_DENY 2
#define CORDUM_DEC_REQUIRE_HUMAN 3
#define CORDUM_DEC_THROTTLE 4
#define CORDUM_DEC_ALLOW_WITH_CONSTRAINTS 5

/* reason codes: host formats the exact strings (kernel.go:172,175,221,225;
 * safety_policy.go:410,413; engine.go:500) */
#define CORDUM_REASON_NONE 0
#define CORDUM_REASON_RULE 1            /* rules[rule_idx].reason                   */
#define CORDUM_REASON_MISSING_TOPIC 2   /* "missing topic"                          */
#define CORDUM_REASON_UNSUPPORTED_TOPIC 3 /* "unsupported topic"                    */
#define CORDUM_REASON_TENANT_MCP 4      /* 4..11: field*2 + (0 denied | 1 not allowed), field = server,tool,resource,action */
#define CORDUM_REASON_EFF_DENIED_TOPIC 12
#define CORDUM_REASON_EFF_NOT_ALLOWED_TOPIC 13
#define CORDUM_REASON_EFF_MCP 14        /* 14..21, same sub-layout as TENANT_MCP    */
#define CORDUM_REASON_APPROVAL_GRANTED 22 /* "approval granted" (engine.go:500)     */

/* route status (strategy_least_loaded.go:40-136; errors.go:5-14) */
#define CORDUM_ROUTE_NOT_ATTEMPTED 0    /* decision did not allow dispatch (engine.go:298-347) */
#define CORDUM_ROUTE_OK 1               /* worker_slot valid: subject "worker.<id>.jobs"       */
#define CORDUM_ROUTE_OK_PREFERRED 2     /* preferred_worker_id shortcut (:73-87)               */
#define CORDUM_ROUTE_MISSING_TOPIC 3    /* :41-43                                              */
#define CORDUM_ROUTE_NO_POOL_PREFERRED 4 /* ErrNoPoolMapping, preferred pool not mapped (:52)  */
#define CORDUM_ROUTE_NO_POOL_TOPIC 5    /* ErrNoPoolMapping, topic has no pools (:57)          */
#define CORDUM_ROUTE_NO_POOL_REQUIRES 6 /* ErrNoPoolMapping, no pool satisfies requires (:65)  */
#define CORDUM_ROUTE_NO_WORKERS 7       /* ErrNoWorkers (:118)                                 */
#define CORDUM_ROUTE_POOL_OVERLOADED 8  /* ErrPoolOverloaded (:116)                            */

/* flags */
#define CORDUM_F_APPROVAL_REQUIRED 0x01 /* kernel.go:233                                        */
#define CORDUM_F_HAS_SNAPSHOT 0x02      /* response carries policy_snapshot/rule_id (not the early DENY returns, kernel.go:171-176) */
#define CORDUM_F_CONSTRAINTS 0x04       /* response carries rules[rule_idx].constraints (kernel.go:198,244) */
#define CORDUM_F_TIE 0x08               /* the minimum load score was shared by >1 candidate; the lowest
                                           worker_id (bytewise) was chosen (SURVEY.md A.4)      */
#define CORDUM_F_APPROVED_BYPASS 0x10   /* engine.go:484-522 path                                */

typedef struct cordum_decision {
  uint8_t decision;       /* CORDUM_DEC_*: the safety kernel's PolicyCheckResponse.Decision   */
  uint8_t sched_decision; /* CORDUM_DEC_* after engine.go:528-530 (approval_required & ALLOW* ->
                             REQUIRE_HUMAN i.e. SafetyRequireApproval); what engine.go:298 switches on */
  uint8_t flags;          /* CORDUM_F_*                                                        */
  uint8_t route_status;   /* CORDUM_ROUTE_*                                                    */
  uint8_t reason_code;    /* CORDUM_REASON_*                                                   */
  uint8_t reserved[3];
  int32_t rule_idx;       /* first matching rule, -1 = none (default allow)                    */
  int32_t worker_slot;    /* routed worker slot, -1 = none                                     */
} cordum_decision;        /* 16 bytes */

/* dispatch modes */
#define CORDUM_MODE_POLICY_ONLY 1      /* SafetyKernel Check/Evaluate/Explain/Simulate (kernel.go:106-120) */
#define CORDUM_MODE_POLICY_AND_ROUTE 2 /* processJob: checkSafetyDecision + PickSubject (engine.go:294,393) */
#define CORDUM_MODE_ROUTE_ONLY 3       /* SchedulingStrategy.PickSubject alone (types.go:40-42)            */
/* may be OR-ed into the mode of the *_resident calls (benchmarks): write a 256 MiB scratch buffer
 * first so the batch's columns are not served from L2 */
#define CORDUM_FLAG_FLUSH_L2 0x100
/* may be OR-ed into any dispatch mode: do not record the per-kernel timing events (cordum_batch_timing / _kernel_times
 * then report 0): two API calls less per dispatch, for callers that issue many small dispatches */
#define CORDUM_FLAG_NO_TIMING 0x200

/* ------------------------------------------------------------- engine */
typedef struct cordum_engine cordum_engine;
typedef struct cordum_batch cordum_batch;

typedef struct cordum_engine_opts {
  int32_t device;          /* CUDA device ordinal                                   */
  uint32_t max_topics;     /* capacity of the topic dictionary (0 = default 65536)   */
  uint32_t max_effcfgs;    /* capacity of distinct effective configs (0 = 4096)      */
  uint32_t encode_threads; /* host threads for cordum_encode (0 = hardware threads)  */
} cordum_engine_opts;

const char* cordum_last_error(void);
const char* cordum_version(void);

/* Replaces nothing in the reference: process-level setup.  Fails with
 * CORDUM_E_NODEVICE when no GPU is present — there is no CPU fallback. */
int32_t cordum_engine_create(const cordum_engine_opts* opts, cordum_engine** out);
void cordum_engine_destroy(cordum_engine* e);

/* safetykernel.(*server).setPolicy (kernel.go:510-521): swap the rule set.
 * policy_json = the merged config.SafetyPolicy (safety_policy.go:13-107) marshalled
 * with its yaml tag names as JSON keys; len 0 = nil policy (allow-all, kernel.go:187).
 * snapshot is kept (newest first, 10 deep) for ListSnapshots (kernel.go:122-127). */
int32_t cordum_policy_load(cordum_engine* e, const char* policy_json, uint64_t len,
                           const char* snapshot, uint64_t snapshot_len);
/* ListSnapshots: writes up to cap NUL-separated snapshot ids, newest first. */
int32_t cordum_policy_snapshots(cordum_engine* e, char* buf, uint64_t cap, uint32_t* n_out);
/* The snapshot of the policy in force = PolicyCheckResponse.PolicySnapshot (kernel.go:243): "" when the current policy
 * was loaded without one.  NUL-terminated into buf, returns the full length. */
int64_t cordum_policy_snapshot(cordum_engine* e, char* buf, uint64_t cap);
/* The snapshot the batch's last dispatch ran under (read under the same lock as the tables it used), and the generation
 * (1, 2, ...: successful cordum_policy_load calls) of that policy.  The engine keeps the rule text of the last 8
 * generations: cordum_rule_*_at(e, gen, rule_idx) resolve a record's rule_idx against the policy its batch ran under even
 * if a reload has landed since (the reference builds the whole response from the policy pointer it read under the lock,
 * kernel.go:140-147,239-248).  gen 0 = the policy in force now. */
int64_t cordum_batch_snapshot(const cordum_batch* b, char* buf, uint64_t cap);
uint64_t cordum_batch_policy_gen(const cordum_batch* b);
uint64_t cordum_policy_generation(cordum_engine* e);   /* of the policy in force; lock-free */
int64_t cordum_rule_id_at(cordum_engine* e, uint64_t gen, int32_t rule_idx, char* buf, uint64_t cap);
int64_t cordum_rule_constraints_json_at(cordum_engine* e, uint64_t gen, int32_t rule_idx, char* buf, uint64_t cap);
int64_t cordum_rule_remediations_json_at(cordum_engine* e, uint64_t gen, int32_t rule_idx, char* buf, uint64_t cap);

/* (*LeastLoadedStrategy).UpdateRouting (strategy_least_loaded.go:28-30).
 * routing_json = {"topics": {topic: [pool,...]}, "pools": {pool: {"requires": [...]}}}
 * i.e. scheduler.PoolRouting (routing.go:4-12) as built by buildRouting
 * (cmd/cordum-scheduler/config_overlay.go:155-174). */
int32_t cordum_routing_load(cordum_engine* e, const char* routing_json, uint64_t len);

/* WorkerRegistry snapshot (types.go:34-37; registry_memory.go:71-84): replace the table. */
int32_t cordum_workers_load(cordum_engine* e, const cordum_workers* w);
/* Heartbeat deltas for live workers (registry_memory.go:43-51): host-side loads by slot. */
int32_t cordum_workers_update(cordum_engine* e, uint32_t n, const uint32_t* slots,
                              const cordum_worker_load* loads);
/* Same, but the full slot-ordered load table is already on the device (e.g. the
 * receive buffer of a host-side all-gather of per-rank slices, SURVEY.md §8e).
 * dptr: n_workers x cordum_worker_load on this engine's device; stream: cudaStream_t
 * the data was produced on (0 = legacy default).  The engine copies the table on a
 * stream of its own, ordered after `stream`; work submitted to `stream` after this
 * call returns is ordered after that copy, so the buffer may be refilled there.
 * Asynchronous: returns once the copy and the table refresh are enqueued. */
int32_t cordum_workers_set_loads_device(cordum_engine* e, const void* dptr, uint32_t n_workers,
                                        void* stream);

/* ---- multi-GPU heartbeat exchange owned by the engine (SURVEY.md §8e; BASELINE config 4).
 * One process per GPU; jobs are sharded by the caller, the worker registry is replicated, and each
 * rank ingests the heartbeats of its own contiguous slice of worker slots.  The engine keeps the
 * NCCL communicator (libnccl is loaded at run time: $CORDUM_NCCL_LIB, else libnccl.so.2), so a host
 * that is not a PyTorch process (the Go scheduler) gets the same path.
 *   rank 0: cordum_exchange_unique_id(id)   -> ship the 128 bytes to the other ranks (any transport)
 *   all   : cordum_exchange_init(e, id, rank, world)        collective, blocks until all ranks joined
 *   per heartbeat epoch, all ranks: cordum_workers_ingest(e, loads_of_my_slice, first_slot, n)
 * cordum_workers_ingest copies the slice to the device (pinned host memory makes the copy
 * asynchronous), all-gathers the 16 B/worker records of all ranks in place, and refreshes the worker
 * tables from the gathered table; it returns once the work is enqueued.  The registry must divide
 * evenly: slice of rank r = slots [r * n_slots/world, (r+1) * n_slots/world).  Without
 * cordum_exchange_init (world = 1) the slice must be the whole table.
 * Buffer contract: with world = 1 and on the peer-memory path the slice is copied into library-owned staging before the
 * call returns.  On the NCCL path (world > 1) a page-locked slice is read by an asynchronous copy: leave it unchanged
 * until a batch dispatched after this call has been waited for (cordum_batch_wait), or alternate between two buffers and
 * synchronise once per epoch; a pageable slice is staged by the CUDA runtime before the call returns. */
#define CORDUM_EXCHANGE_ID_BYTES 128
int32_t cordum_exchange_unique_id(char id[CORDUM_EXCHANGE_ID_BYTES]);
int32_t cordum_exchange_init(cordum_engine* e, const char id[CORDUM_EXCHANGE_ID_BYTES], int32_t rank, int32_t world);
int32_t cordum_workers_ingest(cordum_engine* e, const cordum_worker_load* slice, uint32_t first_slot, uint32_t n_slice);

/* ---- scheduler ticks: one CUDA graph launch per tick.
 * A tick = one heartbeat epoch + one batch, pipelined across ticks: it refreshes the worker tables from this rank's
 * heartbeat slice (exchanged with the other ranks over peer memory when cordum_peer_import was called), evaluates the
 * policy for `b`, and routes the batch of the PREVIOUS tick on the tables of the previous epoch - three independent
 * branches of one captured graph, so a tick costs the longest of them and one launch instead of ~17 API calls.
 * `b` must be encoded and resident (cordum_encode_device, or one cordum_dispatch); results stay on the device:
 * cordum_batch_wait (which flushes the pipeline if `b` was the last batch) then cordum_batch_fetch.  The slice is copied
 * into library-owned staging before the call returns.  All ranks of a peer exchange must tick the same number of times. */
int32_t cordum_tick_async(cordum_engine* e, cordum_batch* b, uint32_t mode, const cordum_worker_load* slice,
                          uint32_t first_slot, uint32_t n_slice);
/* Routes the batch of the last tick (otherwise done by the next tick). */
int32_t cordum_tick_flush(cordum_engine* e);
/* The cudaStream_t ticks are launched on (for harnesses that bracket them with their own CUDA events). */
void* cordum_tick_stream(cordum_engine* e);
/* Peer-memory heartbeat exchange for ticks (replaces the NCCL all-gather of cordum_workers_ingest): each rank exports a
 * CUDA IPC handle of its exchange buffer, ships the 64 bytes to every other rank by any transport, and imports the
 * world x 64 bytes of all ranks (rank order).  Ranks then read each other's heartbeat slices over NVLink inside the
 * tick's gather kernel, with flag words for the epoch barrier - no collective library, no host round trip.
 * One process per GPU on one node; the worker registry (loaded before the export) must divide evenly. */
#define CORDUM_PEER_HANDLE_BYTES 64
int32_t cordum_peer_export(cordum_engine* e, int32_t rank, int32_t world, char handle[CORDUM_PEER_HANDLE_BYTES]);
int32_t cordum_peer_import(cordum_engine* e, const char* handles /* world x CORDUM_PEER_HANDLE_BYTES */);

/* Library-owned pinned SoA slabs for up to max_jobs jobs. */
int32_t cordum_batch_alloc(cordum_engine* e, uint32_t max_jobs, cordum_batch** out);
void cordum_batch_free(cordum_batch* b);

/* Request normalisation + dictionary coding of a batch of envelopes into the
 * batch's column-major attribute arrays (kernel.go:133-185, 348-414;
 * strategy_least_loaded.go:46-62,195-222).  Host work, multi-threaded. */
int32_t cordum_encode(cordum_engine* e, cordum_batch* b, const cordum_envelopes* env);

/* ---- encoding on the device.
 * cordum_encode is host work (hash lookups per string): ~30 ms per million envelopes on 16 cores, against 0.2 ms of
 * kernels.  cordum_encode_device does the same normalisation + dictionary coding in CUDA kernels: the envelope arrays
 * (string arena + span columns, ~250 B per job) are copied to the device as they are and encoded there, with the
 * host's own dictionaries uploaded as probe-able hash tables.  Asynchronous: returns once the copies and kernels are
 * enqueued on the batch's stream; a dispatch on the same batch queues behind them.  The envelope buffers must stay
 * unchanged until cordum_batch_wait returns.  Page-locked buffers (cordum_envelopes_alloc) are copied by DMA at full
 * PCIe rate; pageable memory works too, slower.
 * What the device leaves to the host - first sight of a topic or of an effective config (pass-rows have to be
 * computed / JSON parsed), non-ASCII text (Unicode TrimSpace / EqualFold), strings over 4 KiB, masks wider than the
 * records (more than 64 referenced risk tags / requires tokens / rule label pairs, more than 128 dense placement-label
 * bits), a placement label few workers carry (a selective pair, e.g. a hostname, in a registry above 1,024 label bits) - raises a per-batch
 * flag; cordum_batch_wait then encodes that batch with cordum_encode's code path and runs it again, so results are
 * the same either way (tests compare the two encoders record for record). */
typedef struct cordum_envelope_caps {
  uint32_t max_jobs;
  uint32_t max_risk_tags, max_requires, max_labels; /* total entries of the three list columns */
  uint64_t arena_bytes;
} cordum_envelope_caps;
/* A cordum_envelopes whose arrays are writable page-locked memory owned by the library (cast away the const to fill
 * them; set n_jobs and arena_len).  Freed by cordum_envelopes_free or with the engine. */
int32_t cordum_envelopes_alloc(cordum_engine* e, const cordum_envelope_caps* caps, cordum_envelopes** out);
void cordum_envelopes_free(cordum_engine* e, cordum_envelopes* env);
int32_t cordum_encode_device(cordum_engine* e, cordum_batch* b, const cordum_envelopes* env);
/* How many batches the device encoder handed back to the host encoder since the engine was created. */
uint64_t cordum_host_fallbacks(cordum_engine* e);
/* The encoded records of a batch (tests / diagnostics): n JobRec (64 B), n RouteRec (32 B) and slot_of[n], copied
 * into caller memory (any may be NULL).  Layouts: cordum_b200/csrc/tables.h. */
int32_t cordum_batch_records(cordum_batch* b, void* job_out, void* route_out, uint32_t* slot_of_out);

/* Batched evaluate() [+ post-step + PickSubject()].  Blocking:
 * H2D of the encoded columns, kernels, D2H of the decision records. */
int32_t cordum_dispatch(cordum_engine* e, cordum_batch* b, uint32_t mode);
/* Pipelined form: enqueue on the batch's stream / wait for it. */
int32_t cordum_dispatch_async(cordum_engine* e, cordum_batch* b, uint32_t mode);
int32_t cordum_batch_wait(cordum_batch* b);
/* Device-resident form used for kernel-only timing: assumes the columns of the
 * last dispatch on this batch are still in HBM; runs the kernels only, no copies. */
int32_t cordum_dispatch_resident(cordum_engine* e, cordum_batch* b, uint32_t mode);
int32_t cordum_dispatch_resident_async(cordum_engine* e, cordum_batch* b, uint32_t mode); /* then cordum_batch_wait */

/* After a resident run: copy the decision records from HBM into the pinned result buffer. */
int32_t cordum_batch_fetch(cordum_batch* b);
/* The batch's cudaStream_t, so a harness can bracket launches with its own CUDA events. */
void* cordum_batch_stream(cordum_batch* b);

uint32_t cordum_batch_size(const cordum_batch* b);
/* Decision records of the last completed dispatch (pinned host memory, n = batch size). */
const cordum_decision* cordum_batch_results(const cordum_batch* b);
/* Device time of the last completed dispatch on this batch (CUDA events on the
 * batch stream): total (copies included), and the kernels alone.  Milliseconds. */
int32_t cordum_batch_timing(const cordum_batch* b, float* total_ms, float* kernel_ms);
/* The two kernels of a dispatch separately: policy_kernel and route_kernel (CUDA events). */
int32_t cordum_batch_kernel_times(const cordum_batch* b, float* policy_ms, float* route_ms);

/* Host-side materialisation of what the record indexes (pure functions of rule_idx /
 * reason_code / worker_slot; SURVEY.md A.5).  Each writes a NUL-terminated string
 * into buf (truncating to cap) and returns the full length. */
int64_t cordum_rule_id(cordum_engine* e, int32_t rule_idx, char* buf, uint64_t cap);
int64_t cordum_reason(cordum_engine* e, const cordum_batch* b, uint32_t job, char* buf, uint64_t cap);
/* The reference evaluates a policy check in two places with the same code but one differing format verb in the
 * effective-config reasons: the safety kernel prints the topic as '%s' (kernel.go:221,225), the gateway's
 * evaluatePolicyCheck — used by bundle / pack policy simulation against a draft policy — as %q
 * (gateway/policy_bundles.go:1207,1211; strconv.Quote semantics).  cordum_reason == flavor KERNEL, env NULL.
 * env: the envelopes the batch was encoded from, or NULL.  The job record keeps an MCP value as the id of its
 * case-folded form, so without the envelopes an MCP reason quotes that canonical spelling ("evil"); with them it
 * quotes the request's own, as the reference does (safety_policy.go:410,413: %q of the trimmed label value). */
#define CORDUM_REASON_FLAVOR_KERNEL 0
#define CORDUM_REASON_FLAVOR_GATEWAY 1
int64_t cordum_reason_flavor(cordum_engine* e, const cordum_batch* b, uint32_t job, uint32_t flavor,
                             const cordum_envelopes* env, char* buf, uint64_t cap);
int64_t cordum_subject(cordum_engine* e, const cordum_batch* b, uint32_t job, char* buf, uint64_t cap);
/* JSON of rules[rule_idx].constraints / .remediations as loaded (kernel.go:244,247). */
int64_t cordum_rule_constraints_json(cordum_engine* e, int32_t rule_idx, char* buf, uint64_t cap);
int64_t cordum_rule_remediations_json(cordum_engine* e, int32_t rule_idx, char* buf, uint64_t cap);

/* ---- micro-batching front-end (cordum_b200/csrc/frontend.cpp).
 * The seams it stands behind handle ONE request per call: scheduler.SafetyChecker.Check (types.go:29-31),
 * scheduler.SchedulingStrategy.PickSubject (types.go:40-42), the four SafetyKernel RPCs (kernel.go:106-127, each on its
 * own goroutine), and processJob (engine.go:203-443) which calls the first two per job.  cordum_frontend_submit is that
 * call shape - blocking, thread-safe, one request in, one decision out - and batches concurrent callers behind it: a
 * batch is flushed when it holds max_batch requests or max_wait_us after its first request, whichever comes first, with
 * ONE encode + dispatch for all of them.  Strings need not be NUL-terminated. */
typedef struct cordum_sv { const char* p; uint32_t n; } cordum_sv;
typedef struct cordum_kv { cordum_sv key, val; } cordum_kv;
typedef struct cordum_request {      /* PolicyCheckRequest / JobRequest fields the path reads (SURVEY.md App. B) */
  cordum_sv topic, tenant, principal_id, effective_config;
  uint8_t has_meta, actor_type /* 0 unspecified, 1 human, 2 service */, approved, pad;
  cordum_sv meta_tenant_id, actor_id, capability, pack_id;
  const cordum_sv* risk_tags; uint32_t n_risk_tags;
  const cordum_sv* requires_; uint32_t n_requires;
  const cordum_kv* labels; uint32_t n_labels;
} cordum_request;
typedef struct cordum_response {     /* PolicyCheckResponse (kernel.go:239-248) + the routed subject (PickSubject) */
  cordum_decision rec;
  int32_t status;                    /* CORDUM_OK, or why the request failed closed (rec then says DENY)            */
  uint32_t reserved;
  uint64_t policy_gen;               /* generation of the policy the request was evaluated under: cordum_rule_*_at  */
  char rule_id[128];                 /* "" when the response carries none (kernel.go:171-176)                       */
  char reason[256];
  char subject[192];                 /* "worker.<id>.jobs" when routed (bus/nats.go:94-99)                          */
  char snapshot[96];                 /* PolicySnapshot                                                              */
} cordum_response;
typedef struct cordum_frontend_opts {
  uint32_t max_batch;                /* flush at this many requests (default 1024)                                  */
  uint32_t max_wait_us;              /* ... or this long after the first request of the batch (default 200; 0 = never wait) */
  uint32_t mode;                     /* CORDUM_MODE_* of every batch (default POLICY_AND_ROUTE)                     */
  uint32_t lanes;                    /* batches in flight (default 2: packing overlaps the GPU round trip)          */
  uint32_t arena_bytes_per_request;  /* string budget per request in the page-locked staging (default 1024)         */
  uint32_t reserved;
  uint64_t cache_ttl_us;             /* SAFETY_DECISION_CACHE_TTL (kernel.go:40,87,149-162,250-254): > 0 and mode POLICY_ONLY
                                        = answer a request identical to one evaluated under the same policy within the TTL
                                        from memory.  0 (the reference's default) = off                              */
} cordum_frontend_opts;
typedef struct cordum_frontend cordum_frontend;
int32_t cordum_frontend_create(cordum_engine* e, const cordum_frontend_opts* opts, cordum_frontend** out);
void cordum_frontend_destroy(cordum_frontend* f);
/* Blocking; any number of threads.  Returns resp->status. */
int32_t cordum_frontend_submit(cordum_frontend* f, const cordum_request* req, cordum_response* resp);
/* n requests of one caller at once (a Go adapter that drained a channel): returns the worst status. */
int32_t cordum_frontend_submit_many(cordum_frontend* f, const cordum_request* reqs, uint32_t n, cordum_response* resps);
int32_t cordum_frontend_stats(cordum_frontend* f, uint64_t* batches, uint64_t* requests, uint64_t* full_batches);
int32_t cordum_frontend_cache_stats(cordum_frontend* f, uint64_t* hits, uint64_t* misses, uint64_t* entries);
/* Diagnostics: native client threads submitting round-robin for `seconds`; latencies (us) into lat_us[cap]. */
uint64_t cordum_frontend_loadgen(cordum_frontend* f, const cordum_request* reqs, uint32_t n_reqs, uint32_t threads, double seconds,
                                 float* lat_us, uint64_t cap);

/* Introspection for tests/bench: table sizes and algorithmic byte counts. */
typedef struct cordum_table_stats {
  uint32_t n_rules, n_rules_padded, n_segments;
  uint32_t n_topics, n_tenants, n_pools, n_workers, n_workers_routable;
  uint64_t passrow_bytes;  /* all pass-row tables                         */
  uint64_t rulecol_bytes;  /* per-rule columns                            */
  uint64_t routing_bytes;  /* topic->pool CSR + pool columns              */
  uint64_t worker_bytes;   /* worker columns                              */
  uint32_t job_in_bytes;   /* bytes of encoded columns per job            */
  uint32_t job_out_bytes;  /* bytes of decision record per job            */
} cordum_table_stats;
int32_t cordum_stats(cordum_engine* e, cordum_table_stats* out);

/* Number of kernels this library has launched on the handle since creation. */
uint64_t cordum_launch_count(cordum_engine* e);

/* Test hooks: the library's own string primitives (table-compile time semantics), exported so
 * the test-suite can run them differentially against the oracle.  Not part of the drop-in surface. */
int32_t cordum_test_glob(const char* pat, uint64_t plen, const char* name, uint64_t nlen); /* 1, 0, -1 malformed */
void cordum_test_trim(const char* s, uint64_t n, uint64_t* off, uint64_t* len);
int32_t cordum_test_normalize_decision(const char* s, uint64_t n);
int64_t cordum_test_canon(int32_t kind, const char* s, uint64_t n, char* buf, uint64_t cap); /* 0: EqualFold class form, 1: strings.ToLower, 2: strconv.Quote */
int32_t cordum_test_parse_effective(const char* s, uint64_t n, uint32_t* n_allowed, uint32_t* n_denied);

#ifdef __cplusplus
}
#endif
#endif /* CORDUM_B200_H */
