"""Host-side mirror of the reference's seams for this path, over the CUDA engine.

Same names, argument meaning and error behaviour as the Go interfaces (SURVEY.md §8b), so
tests read like the reference's own:

  SafetyKernelServer.{check,evaluate,explain,simulate,list_snapshots}
        safetykernel.(*server).{Check,Evaluate,Explain,Simulate,ListSnapshots}  kernel.go:106-127
  GatewayPolicyEvaluator.evaluate_policy_check(policy, snapshot, req)
        gateway.evaluatePolicyCheck (draft-bundle / pack policy simulation)        gateway/policy_bundles.go:1132-1231
  SafetyClient.check(job_request)            scheduler.(*SafetyClient).Check       safety_client.go:68-115
  extract_tenant(job_request)                scheduler.ExtractTenant               tenant.go:8-21
  LeastLoadedStrategy.{pick_subject,update_routing,current_routing}                strategy_least_loaded.go:21-136
  MemoryRegistry.{update_heartbeat,snapshot} scheduler.MemoryRegistry              registry_memory.go:11-84
  Scheduler.process_jobs                     Engine.processJob's decision switch   engine.go:294-347,393
  topic_metrics(labels, counts)              the four topic-labelled counters      metrics/metrics.go:48-70
  decision_records(batch, engine)            checkSafetyDecision's stored records  engine.go:524-545, emitDLQ :325-346

Requests are plain dicts shaped like the CAP v2 messages (SURVEY App. B).  Every decision and
every routed subject comes from the GPU (cordum_dispatch); this module only maps fields,
formats the strings the records index, and keeps the registry's timestamps.  The Go adapters in
go/ do the same work in the reference's own language (INTEGRATION.md).
"""
from __future__ import annotations

import json as _json
import time

import numpy as np

from . import wire
from .engine import Engine

EFFECTIVE_CONFIG_ENV = "CORDUM_EFFECTIVE_CONFIG"   # config.EffectiveConfigEnvVar, effective.go:9
DEFAULT_TENANT = "default"                          # scheduler.DefaultTenant, tenant.go:5
DECISION_NAMES = {wire.DEC_ALLOW: "ALLOW", wire.DEC_DENY: "DENY", wire.DEC_REQUIRE_HUMAN: "REQUIRE_HUMAN",
                  wire.DEC_THROTTLE: "THROTTLE", wire.DEC_ALLOW_WITH_CONSTRAINTS: "ALLOW_WITH_CONSTRAINTS"}
# scheduler.SafetyDecision values (types.go:18-26) as decisionFromProto maps them (safety_client.go:117-132)
SAFETY_DECISION = {wire.DEC_ALLOW: "ALLOW", wire.DEC_DENY: "DENY", wire.DEC_REQUIRE_HUMAN: "REQUIRE_APPROVAL",
                   wire.DEC_THROTTLE: "THROTTLE", wire.DEC_ALLOW_WITH_CONSTRAINTS: "ALLOW_WITH_CONSTRAINTS",
                   wire.DEC_UNSPECIFIED: "DENY"}   # default branch: unknown enum -> deny (safety_client.go:129-131)


def decision_from_proto(code: int) -> str:
    """decisionFromProto (safety_client.go:117-132)."""
    return SAFETY_DECISION.get(code, "DENY")


class ErrNoPoolMapping(Exception):   # errors.go:7
    sentinel = "no_pool_mapping"


class ErrNoWorkers(Exception):       # errors.go:9
    sentinel = "no_workers"


class ErrPoolOverloaded(Exception):  # errors.go:11
    sentinel = "pool_overloaded"


def extract_tenant(req: dict) -> str:
    """ExtractTenant (tenant.go:8-21): TenantId, then env["tenant_id"], then "default"."""
    if req is None:
        return DEFAULT_TENANT
    if req.get("tenant_id"):
        return req["tenant_id"]
    env = req.get("env") or {}
    if env.get("tenant_id"):
        return env["tenant_id"]
    return DEFAULT_TENANT


def policy_check_request(job_request: dict) -> dict:
    """JobRequest -> PolicyCheckRequest exactly as SafetyClient.Check builds it (safety_client.go:80-95)."""
    out = {"job_id": job_request.get("job_id", ""), "topic": job_request.get("topic", ""),
           "tenant": extract_tenant(job_request), "principal_id": job_request.get("principal_id", ""),
           "labels": job_request.get("labels") or {}, "meta": job_request.get("meta")}
    env = job_request.get("env") or {}
    if env.get(EFFECTIVE_CONFIG_ENV):
        out["effective_config"] = env[EFFECTIVE_CONFIG_ENV].encode() if isinstance(env[EFFECTIVE_CONFIG_ENV], str) else env[EFFECTIVE_CONFIG_ENV]
    return out


def _envelope(req: dict) -> dict:
    """PolicyCheckRequest / JobRequest dict -> wire job (cordum_b200/wire.py)."""
    return {"topic": req.get("topic", ""), "tenant": req.get("tenant", ""), "principal_id": req.get("principal_id", ""),
            "labels": req.get("labels") or {}, "meta": req.get("meta"), "effective_config": req.get("effective_config"),
            "approved": bool(req.get("approved"))}


class SafetyKernelServer:
    """The gRPC surface of cmd/cordum-safety-kernel, batched.  All four modes are the same function
    (kernel.go:129: the mode string is ignored)."""

    def __init__(self, engine: Engine | None = None, device: int = 0):
        self.engine = engine or Engine(device=device)
        self._batch = None

    def set_policy(self, policy, snapshot: str = ""):
        """server.setPolicy (kernel.go:510-521)."""
        self.engine.load_policy(policy, snapshot)

    def list_snapshots(self) -> list[str]:
        return self.engine.snapshots()

    def evaluate_batch(self, requests: list[dict], *, flavor: int = wire.REASON_FLAVOR_KERNEL, snapshot: str | None = None) -> list[dict]:
        n = len(requests)
        if n == 0:
            return []
        if self._batch is None or self._batch.max_jobs < n:
            if self._batch is not None:
                self._batch.free()
            self._batch = self.engine.batch(max(n, 256))
        b = self._batch
        recs = b.encode([_envelope(r) for r in requests]).dispatch(wire.MODE_POLICY_ONLY)
        gen = b.policy_gen()          # rule text of the policy this batch ran under, whatever has been loaded since
        if snapshot is None:
            snapshot = b.snapshot()   # s.snapshot as read with the policy (kernel.go:141,243): "" when that policy has none
        out = []
        for j, (req, rec) in enumerate(zip(requests, recs)):
            flags = int(rec["flags"])
            rule_idx = int(rec["rule_idx"])
            has_snapshot = bool(flags & wire.F_HAS_SNAPSHOT)
            approval = bool(flags & wire.F_APPROVAL_REQUIRED)
            out.append({
                "decision": DECISION_NAMES[int(rec["decision"])],
                "reason": b.reason(j, flavor),
                "reason_code": int(rec["reason_code"]),                         # not a proto field: the record's own code
                "policy_snapshot": snapshot if has_snapshot else "",
                "rule_id": self.engine.rule_id(rule_idx, gen) if rule_idx >= 0 else "",
                "constraints": self.engine.rule_constraints(rule_idx, gen) if flags & wire.F_CONSTRAINTS else None,
                "approval_required": approval,
                "approval_ref": req.get("job_id", "") if approval else "",     # kernel.go:234-237
                "remediations": self.engine.rule_remediations(rule_idx, gen) if rule_idx >= 0 else [],
            })
        return out

    def check(self, req: dict) -> dict:
        return self.evaluate_batch([req])[0]

    evaluate = explain = simulate = check


class GatewayPolicyEvaluator:
    """gateway.evaluatePolicyCheck (gateway/policy_bundles.go:1132-1231): the gateway's own copy of the evaluator, which
    it runs against a policy that is NOT the one in force - the published bundles with one bundle swapped for a draft
    (handleSimulatePolicyBundle, :322-368).  Decisions are those of the safety kernel; the effective-config reasons
    print the topic with %q instead of '%s' (:1207,:1211), and the early topic denials carry no snapshot (:1154-1159).

    A draft policy is compiled into a scratch engine of its own (a table compile + upload, milliseconds), so simulating
    never touches the tables the live SafetyKernelServer dispatches from."""

    def __init__(self, device: int = 0):
        self._server = SafetyKernelServer(device=device)
        self._loaded = None

    def _load(self, policy):
        doc = policy if policy is not None else {}      # nil policy: every job allowed unless the topic is bad
        key = doc if isinstance(doc, (str, bytes)) else _json.dumps(doc, sort_keys=True)
        if key != self._loaded:
            self._server.set_policy(doc, "")
            self._loaded = key

    def evaluate_batch(self, policy, snapshot: str, requests: list[dict]) -> list[dict]:
        self._load(policy)
        out = self._server.evaluate_batch(requests, flavor=wire.REASON_FLAVOR_GATEWAY, snapshot=snapshot)
        for r in out:
            if r["reason_code"] in (wire.REASON_MISSING_TOPIC, wire.REASON_UNSUPPORTED_TOPIC):
                r["policy_snapshot"] = ""           # returned before the snapshot is attached (:1154-1159)
            else:
                r["policy_snapshot"] = snapshot     # :1221, unconditional
        return out

    def evaluate_policy_check(self, policy, snapshot: str, req: dict) -> dict:
        return self.evaluate_batch(policy, snapshot, [req])[0]


def pack_simulation_request(test_request: dict, pack_id: str, default_tenant: str = DEFAULT_TENANT, auth: dict | None = None) -> dict:
    """The PolicyCheckRequest runPolicySimulation builds from a pack's policy-simulation test (gateway/packs.go:1725-1760)
    before it calls safetyClient.Simulate: tenant / actor come from the caller's auth when present, pack_id and tenant
    default to the pack's and the gateway's."""
    if not test_request.get("topic"):
        raise ValueError("policy simulation missing topic")                      # :1726-1728
    tenant = test_request.get("tenant_id", "")
    meta = {"tenant_id": tenant, "capability": test_request.get("capability", ""),
            "risk_tags": list(test_request.get("risk_tags") or []), "requires": list(test_request.get("requires") or []),
            "pack_id": test_request.get("pack_id", ""), "actor_id": test_request.get("actor_id", ""),
            "actor_type": test_request.get("actor_type", "")}
    if auth:
        if auth.get("tenant"):
            tenant = meta["tenant_id"] = auth["tenant"]
        if auth.get("principal_id") and not meta["actor_id"]:
            meta["actor_id"] = auth["principal_id"]
    meta["pack_id"] = meta["pack_id"] or pack_id
    meta["tenant_id"] = meta["tenant_id"] or default_tenant
    return {"topic": test_request["topic"], "tenant": tenant, "meta": meta}


class SafetyClient:
    """scheduler.SafetyChecker over an in-process SafetyKernelServer (no gRPC hop).  Any engine error
    is mapped to a DENY record, as the reference does for transport errors (safety_client.go:98-101)."""

    def __init__(self, server: SafetyKernelServer):
        self.server = server

    def check_batch(self, job_requests: list[dict]) -> list[dict]:
        try:
            resps = self.server.evaluate_batch([policy_check_request(r) for r in job_requests])
        except Exception as exc:   # fail closed
            return [{"decision": "DENY", "reason": "safety kernel error: %s" % exc} for _ in job_requests]
        out = []
        for r in resps:
            code = {v: k for k, v in DECISION_NAMES.items()}[r["decision"]]
            out.append({"decision": SAFETY_DECISION[code], "reason": r["reason"], "rule_id": r["rule_id"],
                        "policy_snapshot": r["policy_snapshot"], "constraints": r["constraints"],
                        "approval_required": r["approval_required"], "approval_ref": r["approval_ref"],
                        "remediations": r["remediations"]})
        return out

    def check(self, job_request: dict) -> dict:
        return self.check_batch([job_request])[0]


class MemoryRegistry:
    """WorkerRegistry (types.go:34-37) with the reference's TTL semantics (registry_memory.go:23,43-84)."""

    def __init__(self, ttl_s: float = 30.0, clock=time.monotonic):
        self.ttl = ttl_s
        self.clock = clock
        self._hb: dict[str, tuple[dict, float]] = {}

    def update_heartbeat(self, hb: dict):
        if hb is None or not hb.get("worker_id"):
            return
        self._hb[hb["worker_id"]] = (hb, self.clock())

    def snapshot(self) -> dict[str, dict]:
        now = self.clock()
        return {wid: hb for wid, (hb, ts) in self._hb.items() if now - ts <= self.ttl}

    def workers_for_pool(self, pool: str) -> list[dict]:
        return [hb for hb in self.snapshot().values() if hb.get("pool", "") == pool]

    def expire(self):
        now = self.clock()
        for wid in [w for w, (_, ts) in self._hb.items() if now - ts > self.ttl]:
            del self._hb[wid]


class LeastLoadedStrategy:
    """SchedulingStrategy.PickSubject (types.go:40-42) on the GPU.  `workers` is the registry snapshot
    map[worker_id]*Heartbeat; it is uploaded when it changes (identity / pool / labels) or as load
    deltas when only the loads moved."""

    def __init__(self, routing: dict, engine: Engine | None = None, device: int = 0):
        self.engine = engine or Engine(device=device)
        self._routing = {"topics": {}, "pools": {}}
        self._shape = None
        self._ids: list[str] = []
        self._batch = None
        self.update_routing(routing)

    def update_routing(self, routing: dict):
        """UpdateRouting (strategy_least_loaded.go:28-30); cloneRouting semantics: a private copy is kept."""
        topics = {t: list(p) if not isinstance(p, str) else [p] for t, p in (routing.get("topics") or {}).items()}
        pools = {n: {"requires": list((c or {}).get("requires") or [])} for n, c in (routing.get("pools") or {}).items()}
        self._routing = {"topics": topics, "pools": pools}
        self.engine.load_routing(self._routing)
        self._shape = None

    def current_routing(self) -> dict:
        return {"topics": {t: list(p) for t, p in self._routing["topics"].items()},
                "pools": {n: {"requires": list(c["requires"])} for n, c in self._routing["pools"].items()}}

    def _sync_workers(self, workers: dict[str, dict]):
        ids = sorted(w for w, hb in workers.items() if hb is not None)
        shape = tuple((w, workers[w].get("pool", ""), tuple(sorted((workers[w].get("labels") or {}).items()))) for w in ids)
        if shape != self._shape:
            self.engine.load_workers([dict(workers[w], worker_id=w) for w in ids])
            self._shape, self._ids = shape, ids
            return
        loads = np.zeros(len(ids), dtype=wire.LOAD_DTYPE)
        for i, w in enumerate(ids):
            hb = workers[w]
            loads[i] = (hb.get("active_jobs", 0), hb.get("max_parallel_jobs", 0), hb.get("cpu_load", 0.0), hb.get("gpu_utilization", 0.0))
        if len(ids):
            self.engine.update_workers(np.arange(len(ids), dtype=np.uint32), loads)

    def pick_subjects(self, reqs: list[dict], workers: dict[str, dict]) -> list[tuple[str, Exception | None]]:
        self._sync_workers(workers)
        n = len(reqs)
        if n == 0:
            return []
        if self._batch is None or self._batch.max_jobs < n:
            if self._batch is not None:
                self._batch.free()
            self._batch = self.engine.batch(max(n, 256))
        b = self._batch
        jobs = []
        for r in reqs:
            j = _envelope(r or {})
            j["tenant"] = ""
            jobs.append(j)
        recs = b.encode(jobs).dispatch(wire.MODE_ROUTE_ONLY)
        out = []
        for j, (req, rec) in enumerate(zip(reqs, recs)):
            out.append(self._result(req or {}, int(rec["route_status"]), b.subject(j)))
        return out

    def _result(self, req: dict, status: int, subject: str):
        topic = req.get("topic", "")
        labels = req.get("labels") or {}
        if status in (wire.ROUTE_OK, wire.ROUTE_OK_PREFERRED):
            return subject, None
        if status == wire.ROUTE_MISSING_TOPIC:
            return "", ValueError("missing topic")
        if status == wire.ROUTE_NO_POOL_PREFERRED:
            return "", ErrNoPoolMapping('no_pool_mapping: preferred pool "%s" not mapped for topic "%s"' % (labels.get("preferred_pool", ""), topic))
        if status == wire.ROUTE_NO_POOL_TOPIC:
            return "", ErrNoPoolMapping('no_pool_mapping: topic "%s"' % topic)
        if status == wire.ROUTE_NO_POOL_REQUIRES:
            return "", ErrNoPoolMapping("no_pool_mapping: no pool satisfies requires")
        if status == wire.ROUTE_POOL_OVERLOADED:
            return "", ErrPoolOverloaded("pool_overloaded")
        return "", ErrNoWorkers("no_workers")

    def pick_subject(self, req: dict, workers: dict[str, dict]) -> str:
        """Returns "worker.<id>.jobs"; raises ValueError("missing topic") / ErrNoPoolMapping / ErrNoWorkers /
        ErrPoolOverloaded, which engine.go:445-472 classifies with errors.Is."""
        if req is None or req.get("topic", "") == "":
            raise ValueError("missing topic")
        subject, err = self.pick_subjects([req], workers)[0]
        if err is not None:
            raise err
        return subject


class Scheduler:
    """The decision switch of Engine.processJob (engine.go:294-347, 393) over one engine: safety check,
    approval post-step, and routing of the jobs that may dispatch, in ONE GPU pass per batch."""

    def __init__(self, engine: Engine | None = None, device: int = 0):
        self.engine = engine or Engine(device=device)
        self.strategy = LeastLoadedStrategy({"topics": {}, "pools": {}}, engine=self.engine)
        self.kernel = SafetyKernelServer(engine=self.engine)
        self._batch = None

    def process_jobs(self, job_requests: list[dict], workers: dict[str, dict], approved: list[bool] | None = None) -> list[dict]:
        self.strategy._sync_workers(workers)
        n = len(job_requests)
        if n == 0:
            return []
        if self._batch is None or self._batch.max_jobs < n:
            if self._batch is not None:
                self._batch.free()
            self._batch = self.engine.batch(max(n, 256))
        b = self._batch
        jobs = []
        for i, r in enumerate(job_requests):
            j = _envelope(policy_check_request(r))
            j["approved"] = bool(approved[i]) if approved else False
            jobs.append(j)
        recs = b.encode(jobs).dispatch(wire.MODE_POLICY_AND_ROUTE)
        out = []
        for j, (req, rec) in enumerate(zip(job_requests, recs)):
            subject, err = ("", None)
            if int(rec["route_status"]) != wire.ROUTE_NOT_ATTEMPTED:
                subject, err = self.strategy._result(req, int(rec["route_status"]), b.subject(j))
            out.append({"decision": SAFETY_DECISION[int(rec["sched_decision"])], "reason": b.reason(j),
                        "rule_id": self.engine.rule_id(int(rec["rule_idx"])) if rec["rule_idx"] >= 0 else "",
                        "approval_required": bool(rec["flags"] & wire.F_APPROVAL_REQUIRED), "subject": subject, "error": err})
        return out


def decision_records(batch, engine: Engine, flavor: int = wire.REASON_FLAVOR_KERNEL) -> list[dict]:
    """What checkSafetyDecision stores for the jobs of each response class of Batch.responses() (engine.go:524-545), and
    the reason code emitDLQ files a dead-lettered job under (engine.go:325-346): one dict per class, in the classes'
    first_job order, with "jobs" (its job indices), "record" (the SafetyDecisionRecord fields SafetyClient.Check fills,
    safety_client.go:104-113, as the job store keeps them, job_store.go:1036-1093) and "dlq_reason_code" (None for a job
    that is not dead-lettered).  Constraints and remediations are looked up once per class, from the policy generation
    the batch ran under."""
    resp = batch.responses(flavor)
    snapshot = batch.snapshot()
    gen = resp["policy_gen"]
    offsets, jobs = resp["offsets"], resp["jobs"]
    out = []
    for c, k in enumerate(resp["classes"]):
        flags, rule_idx, sched = int(k["flags"]), int(k["rule_idx"]), int(k["sched_decision"])
        record = {
            # decisionFromProto (safety_client.go:105, :117-132), then the approval post-step (engine.go:527-529)
            "decision": SAFETY_DECISION.get(sched, "DENY"),
            "reason": resp["reasons"][c],                                                                  # safety_client.go:106
            "rule_id": resp["rule_ids"][c],                                                                # safety_client.go:107
            "policy_snapshot": snapshot if flags & wire.F_HAS_SNAPSHOT else "",                            # safety_client.go:108
            "constraints": engine.rule_constraints(rule_idx, gen) if flags & wire.F_CONSTRAINTS else None,  # safety_client.go:109
            "approval_required": bool(flags & wire.F_APPROVAL_REQUIRED),                                   # safety_client.go:110
            "remediations": engine.rule_remediations(rule_idx, gen) if rule_idx >= 0 else [],             # safety_client.go:112
        }
        # emitDLQ: DENY -> "safety_denied" (engine.go:335), the default branch (an unknown decision) -> "safety_unknown"
        # (engine.go:345); every other decision is not dead-lettered here
        dlq = "safety_denied" if sched == wire.DEC_DENY else "safety_unknown" if sched == wire.DEC_UNSPECIFIED else None
        out.append({"jobs": jobs[offsets[c]:offsets[c + 1]].copy(), "record": record, "dlq_reason_code": dlq})
    return out


JOB_STATUS_FAILED = "JOB_STATUS_FAILED"   # pb.JobStatus_JOB_STATUS_FAILED.String()


def topic_metrics(labels: list[bytes], counts: np.ndarray) -> dict:
    """What handleJobRequest / processJob add to the four counter vectors of metrics.Prom (metrics/metrics.go:48-70) for
    the jobs of one table of Batch.topic_counts(): {"jobs_received_total": {topic: n}, "safety_denied_total": {topic: n},
    "jobs_completed_total": {(topic, status): n}, "jobs_dispatched_total": {topic: n}}, topics as the label bytes, zero
    increments left out (a counter child exists once it has been incremented).

    - The "" row is an invalid request (engine.go:209-218): the whole row goes to completed{"", FAILED} and nothing else.
    - received = the row's total (engine.go:239).
    - safety_denied = DENY + UNSPECIFIED (engine.go:333, :344).
    - completed{FAILED} = MISSING_TOPIC + the three NO_POOL columns: PickSubject errors that are not retryable
      (engine.go:404).
    - dispatched = the routed column (engine.go:435).  The reference increments it only after bus.Publish succeeded, so a
      caller subtracts the jobs of the worker buckets whose publish failed (those are retried, engine.go:426-433).
    - THROTTLE, NO_WORKERS, POOL_OVERLOADED (retried) and REQUIRE_HUMAN (awaits approval) increment nothing; ALLOW and
      ALLOW_WITH_CONSTRAINTS without routing (POLICY_ONLY) neither.
    The store gates before engine.go:239 (job lock, terminal or dispatched state) are the caller's: they keep a job from
    reaching any of these lines."""
    counts = np.asarray(counts, dtype=np.int64).reshape(len(labels), wire.COUNT_COLUMNS)
    received, denied, completed, dispatched = {}, {}, {}, {}

    def add(d, key, v):
        if v:
            d[key] = d.get(key, 0) + int(v)

    for label, row in zip(labels, counts):
        label = bytes(label)
        if label == b"":
            add(completed, (label, JOB_STATUS_FAILED), row.sum())
            continue
        add(received, label, row.sum())
        add(denied, label, row[wire.DEC_DENY] + row[wire.DEC_UNSPECIFIED])
        add(completed, (label, JOB_STATUS_FAILED), row[6:wire.PLAN_NO_WORKERS].sum())   # MISSING_TOPIC, NO_POOL_*
        add(dispatched, label, row[wire.COUNT_ROUTED])
    return {"jobs_received_total": received, "safety_denied_total": denied, "jobs_completed_total": completed,
            "jobs_dispatched_total": dispatched}
