"""Wire formats of the C ABI (include/cordum_b200.h) as ctypes structures, plus
packers from Python-level objects.

Python-level shapes mirror the CAP v2 messages the reference reads on this path
(SURVEY.md App. B):

  job (PolicyCheckRequest / JobRequest fields):
    {"topic": str, "tenant": str, "principal_id": str, "labels": {str: str},
     "meta": None | {"tenant_id": str, "actor_id": str, "actor_type": 0|1|2,
                     "capability": str, "risk_tags": [str], "requires": [str],
                     "pack_id": str},
     "effective_config": bytes|str, "approved": bool}
    "labels" may also be a list of (key, value) pairs, laid out in that order, repeated keys
    included (the encoders give a repeated key its last value, as a map decoded from the
    wire would hold it)
  worker (Heartbeat fields, snapshot.go:20-28):
    {"worker_id": str, "pool": str, "active_jobs": int, "max_parallel_jobs": int,
     "cpu_load": float, "gpu_utilization": float, "labels": {str: str}}

This module holds no policy logic; it only lays bytes out.
"""
from __future__ import annotations

import ctypes as C
from typing import Iterable, Sequence

import numpy as np

ACTOR_UNSPECIFIED, ACTOR_HUMAN, ACTOR_SERVICE = 0, 1, 2

STR_DTYPE = np.dtype([("off", "<u4"), ("len", "<u4")])


class CordumStr(C.Structure):
    _fields_ = [("off", C.c_uint32), ("len", C.c_uint32)]


_P = C.c_void_p


class CordumEnvelopes(C.Structure):
    _fields_ = [
        ("n_jobs", C.c_uint32),
        ("arena", _P),
        ("arena_len", C.c_uint64),
        ("topic", _P),
        ("tenant", _P),
        ("principal_id", _P),
        ("effective_config", _P),
        ("has_meta", _P),
        ("meta_tenant_id", _P),
        ("actor_id", _P),
        ("actor_type", _P),
        ("capability", _P),
        ("pack_id", _P),
        ("risk_off", _P),
        ("risk_tags", _P),
        ("requires_off", _P),
        ("requires_", _P),
        ("label_off", _P),
        ("label_keys", _P),
        ("label_vals", _P),
        ("approved", _P),
    ]


class CordumWorkers(C.Structure):
    _fields_ = [
        ("n_workers", C.c_uint32),
        ("arena", _P),
        ("arena_len", C.c_uint64),
        ("worker_id", _P),
        ("pool", _P),
        ("active_jobs", _P),
        ("max_parallel_jobs", _P),
        ("cpu_load", _P),
        ("gpu_utilization", _P),
        ("label_off", _P),
        ("label_keys", _P),
        ("label_vals", _P),
    ]


class CordumWorkerLoad(C.Structure):
    _fields_ = [
        ("active_jobs", C.c_int32),
        ("max_parallel_jobs", C.c_int32),
        ("cpu_load", C.c_float),
        ("gpu_utilization", C.c_float),
    ]


LOAD_DTYPE = np.dtype([("active_jobs", "<i4"), ("max_parallel_jobs", "<i4"), ("cpu_load", "<f4"), ("gpu_utilization", "<f4")])

DECISION_DTYPE = np.dtype(
    [
        ("decision", "u1"),
        ("sched_decision", "u1"),
        ("flags", "u1"),
        ("route_status", "u1"),
        ("reason_code", "u1"),
        ("reserved", "u1", (3,)),
        ("rule_idx", "<i4"),
        ("worker_slot", "<i4"),
    ]
)
assert DECISION_DTYPE.itemsize == 16


class CordumTableStats(C.Structure):
    _fields_ = [
        ("n_rules", C.c_uint32), ("n_rules_padded", C.c_uint32), ("n_segments", C.c_uint32),
        ("n_topics", C.c_uint32), ("n_tenants", C.c_uint32), ("n_pools", C.c_uint32),
        ("n_workers", C.c_uint32), ("n_workers_routable", C.c_uint32),
        ("passrow_bytes", C.c_uint64), ("rulecol_bytes", C.c_uint64),
        ("routing_bytes", C.c_uint64), ("worker_bytes", C.c_uint64),
        ("job_in_bytes", C.c_uint32), ("job_out_bytes", C.c_uint32),
    ]


class CordumEnvelopeCaps(C.Structure):
    _fields_ = [("max_jobs", C.c_uint32), ("max_risk_tags", C.c_uint32), ("max_requires", C.c_uint32), ("max_labels", C.c_uint32),
                ("arena_bytes", C.c_uint64)]


JOB_REC_DTYPE = np.dtype([("topic", "<u4"), ("flags", "<u4"), ("orig", "<u4"), ("tenant", "<u2"), ("tenant_pol", "<u2"),
                          ("capability", "<u2"), ("pack", "<u2"), ("actor", "<u2"), ("effcfg", "<u2"), ("mcp", "<u2", (4,)),
                          ("risk_mask", "<u8"), ("req_mask", "<u8"), ("lab_mask", "<u8"), ("spare", "<u4", (2,))])
ROUTE_REC_DTYPE = np.dtype([("place_lo", "<u8"), ("place_hi", "<u8"), ("req_pool", "<u8"), ("pref_pool", "<u4"), ("pref_worker", "<u4")])
assert JOB_REC_DTYPE.itemsize == 64 and ROUTE_REC_DTYPE.itemsize == 32


class CordumEngineOpts(C.Structure):
    _fields_ = [("device", C.c_int32), ("max_topics", C.c_uint32), ("max_effcfgs", C.c_uint32), ("encode_threads", C.c_uint32)]


# decision / status codes (mirror the header)
DEC_UNSPECIFIED, DEC_ALLOW, DEC_DENY, DEC_REQUIRE_HUMAN, DEC_THROTTLE, DEC_ALLOW_WITH_CONSTRAINTS = range(6)
DEC_NAMES = ["UNSPECIFIED", "ALLOW", "DENY", "REQUIRE_HUMAN", "THROTTLE", "ALLOW_WITH_CONSTRAINTS"]
F_APPROVAL_REQUIRED, F_HAS_SNAPSHOT, F_CONSTRAINTS, F_TIE, F_APPROVED_BYPASS = 0x01, 0x02, 0x04, 0x08, 0x10
(ROUTE_NOT_ATTEMPTED, ROUTE_OK, ROUTE_OK_PREFERRED, ROUTE_MISSING_TOPIC, ROUTE_NO_POOL_PREFERRED,
 ROUTE_NO_POOL_TOPIC, ROUTE_NO_POOL_REQUIRES, ROUTE_NO_WORKERS, ROUTE_POOL_OVERLOADED) = range(9)
MODE_POLICY_ONLY, MODE_POLICY_AND_ROUTE, MODE_ROUTE_ONLY = 1, 2, 3
FLAG_FLUSH_L2 = 0x100
REASON_FLAVOR_KERNEL, REASON_FLAVOR_GATEWAY = 0, 1   # cordum_reason_flavor
FLAG_NO_TIMING = 0x200
REASON_NONE, REASON_RULE, REASON_MISSING_TOPIC, REASON_UNSUPPORTED_TOPIC, REASON_TENANT_MCP = 0, 1, 2, 3, 4
REASON_EFF_DENIED_TOPIC, REASON_EFF_NOT_ALLOWED_TOPIC, REASON_EFF_MCP, REASON_APPROVAL_GRANTED = 12, 13, 14, 22


def _ptr(a: np.ndarray | None):
    return None if a is None else a.ctypes.data


class _Arena:
    """Append-only byte arena with interning (equal strings share one span)."""

    def __init__(self):
        self.buf = bytearray()
        self.seen: dict[bytes, tuple[int, int]] = {}

    def add(self, s) -> tuple[int, int]:
        if s is None:
            return (0, 0)
        b = s if isinstance(s, (bytes, bytearray)) else str(s).encode("utf-8", "surrogatepass")
        b = bytes(b)
        if not b:
            return (0, 0)
        hit = self.seen.get(b)
        if hit is None:
            hit = (len(self.buf), len(b))
            self.buf += b
            self.seen[b] = hit
        return hit

    def array(self) -> np.ndarray:
        return np.frombuffer(bytes(self.buf) or b"\0", dtype=np.uint8).copy()


class EnvelopeBatch:
    """Owns the numpy buffers behind one cordum_envelopes struct."""

    SCALARS = ("topic", "tenant", "principal_id", "effective_config", "meta_tenant_id", "actor_id", "capability", "pack_id")

    def __init__(self, n_jobs: int, arena: np.ndarray, cols: dict[str, np.ndarray]):
        self.n_jobs = int(n_jobs)
        self.arena = np.ascontiguousarray(arena, dtype=np.uint8)
        self.cols = {k: np.ascontiguousarray(v) for k, v in cols.items()}
        for k in self.SCALARS + ("risk_tags", "requires_", "label_keys", "label_vals"):
            assert self.cols[k].dtype == STR_DTYPE, k
        for k in ("risk_off", "requires_off", "label_off"):
            assert self.cols[k].dtype == np.uint32 and len(self.cols[k]) == self.n_jobs + 1, k
        for k in ("has_meta", "actor_type", "approved"):
            assert self.cols[k].dtype == np.uint8 and len(self.cols[k]) == self.n_jobs, k
        s = CordumEnvelopes()
        s.n_jobs = self.n_jobs
        s.arena = _ptr(self.arena)
        s.arena_len = len(self.arena)
        for name, _ in CordumEnvelopes._fields_[3:]:
            setattr(s, name, _ptr(self.cols[name]))
        self.struct = s

    def byref(self):
        return C.byref(self.struct)

    @property
    def address(self) -> int:
        return C.addressof(self.struct)

    @staticmethod
    def from_jobs(jobs: Sequence[dict]) -> "EnvelopeBatch":
        n = len(jobs)
        ar = _Arena()
        cols = {k: np.zeros(n, dtype=STR_DTYPE) for k in EnvelopeBatch.SCALARS}
        has_meta = np.zeros(n, np.uint8)
        actor_type = np.zeros(n, np.uint8)
        approved = np.zeros(n, np.uint8)
        risk_off = np.zeros(n + 1, np.uint32)
        req_off = np.zeros(n + 1, np.uint32)
        lab_off = np.zeros(n + 1, np.uint32)
        risk, req, lk, lv = [], [], [], []
        for j, job in enumerate(jobs):
            cols["topic"][j] = ar.add(job.get("topic", ""))
            cols["tenant"][j] = ar.add(job.get("tenant", ""))
            cols["principal_id"][j] = ar.add(job.get("principal_id", ""))
            cols["effective_config"][j] = ar.add(job.get("effective_config") or b"")
            meta = job.get("meta")
            if meta is not None:
                has_meta[j] = 1
                cols["meta_tenant_id"][j] = ar.add(meta.get("tenant_id", ""))
                cols["actor_id"][j] = ar.add(meta.get("actor_id", ""))
                at = meta.get("actor_type", 0)
                if isinstance(at, str):
                    at = {"human": ACTOR_HUMAN, "service": ACTOR_SERVICE}.get(at.lower(), ACTOR_UNSPECIFIED)
                actor_type[j] = at
                cols["capability"][j] = ar.add(meta.get("capability", ""))
                cols["pack_id"][j] = ar.add(meta.get("pack_id", ""))
                for t in meta.get("risk_tags") or []:
                    risk.append(ar.add(t))
                for t in meta.get("requires") or []:
                    req.append(ar.add(t))
            labels = job.get("labels") or {}
            for k, v in (labels.items() if isinstance(labels, dict) else labels):
                lk.append(ar.add(k))
                lv.append(ar.add(v))
            approved[j] = 1 if job.get("approved") else 0
            risk_off[j + 1] = len(risk)
            req_off[j + 1] = len(req)
            lab_off[j + 1] = len(lk)

        def strs(lst):
            a = np.zeros(max(len(lst), 1), dtype=STR_DTYPE)
            for i, t in enumerate(lst):
                a[i] = t
            return a

        cols.update(
            has_meta=has_meta, actor_type=actor_type, approved=approved,
            risk_off=risk_off, risk_tags=strs(risk), requires_off=req_off, requires_=strs(req),
            label_off=lab_off, label_keys=strs(lk), label_vals=strs(lv),
        )
        return EnvelopeBatch(n, ar.array(), cols)

    def _s(self, span) -> str:
        o, n = int(span["off"]), int(span["len"])
        return bytes(self.arena[o:o + n]).decode("utf-8", "surrogateescape")

    def to_jobs(self, first: int = 0, count: int | None = None) -> list[dict]:
        """Decode back to Python-level jobs (for the dict-level oracle and debugging)."""
        c = self.cols
        count = self.n_jobs - first if count is None else count
        out = []
        for j in range(first, first + count):
            job = {"topic": self._s(c["topic"][j]), "tenant": self._s(c["tenant"][j]),
                   "principal_id": self._s(c["principal_id"][j]), "labels": {}, "meta": None,
                   "approved": bool(c["approved"][j])}
            ec = c["effective_config"][j]
            if ec["len"]:
                job["effective_config"] = bytes(self.arena[int(ec["off"]): int(ec["off"]) + int(ec["len"])])
            if c["has_meta"][j]:
                job["meta"] = {
                    "tenant_id": self._s(c["meta_tenant_id"][j]), "actor_id": self._s(c["actor_id"][j]),
                    "actor_type": int(c["actor_type"][j]), "capability": self._s(c["capability"][j]),
                    "pack_id": self._s(c["pack_id"][j]),
                    "risk_tags": [self._s(c["risk_tags"][k]) for k in range(c["risk_off"][j], c["risk_off"][j + 1])],
                    "requires": [self._s(c["requires_"][k]) for k in range(c["requires_off"][j], c["requires_off"][j + 1])],
                }
            for k in range(c["label_off"][j], c["label_off"][j + 1]):
                job["labels"][self._s(c["label_keys"][k])] = self._s(c["label_vals"][k])
            out.append(job)
        return out

    def deinterned(self) -> "EnvelopeBatch":
        """The same jobs with NOTHING shared between them: every job's strings are laid out contiguously, job after job
        (topic, tenant, principal, meta fields, risk tags, requires, label key/value pairs, effective config), the way
        a shim unpacking one protobuf JobRequest after another would produce them.  Equal strings of different jobs
        are different byte ranges, so nothing downstream can resolve a value by its address."""
        c = self.cols
        n = self.n_jobs
        order = ["topic", "tenant", "principal_id", "meta_tenant_id", "actor_id", "capability", "pack_id"]
        lens = {k: c[k]["len"].astype(np.int64) for k in order + ["effective_config"]}

        def run_sums(off, ln):   # per-job sum of a CSR column's entry lengths, and each entry's prefix inside its run
            cs = np.concatenate([[0], np.cumsum(ln)])
            o = off.astype(np.int64)
            per_job = cs[o[1:]] - cs[o[:-1]]
            counts = np.diff(o)
            start_of_entry = np.repeat(cs[o[:-1]], counts)
            return per_job, cs[:len(ln)][: int(o[-1])] - start_of_entry

        nr, nq, nl = int(c["risk_off"][-1]), int(c["requires_off"][-1]), int(c["label_off"][-1])
        rl = c["risk_tags"]["len"][:nr].astype(np.int64)
        ql = c["requires_"]["len"][:nq].astype(np.int64)
        kl = c["label_keys"]["len"][:nl].astype(np.int64)
        vl = c["label_vals"]["len"][:nl].astype(np.int64)
        risk_job, risk_pre = run_sums(c["risk_off"], rl)
        req_job, req_pre = run_sums(c["requires_off"], ql)
        lab_job, lab_pre = run_sums(c["label_off"], kl + vl)
        total_job = sum(lens[k] for k in order) + risk_job + req_job + lab_job + lens["effective_config"]
        base = np.concatenate([[1], 1 + np.cumsum(total_job)])   # byte 0 stays reserved: (0, 0) is the empty string
        arena = np.zeros(int(base[-1]), dtype=np.uint8)
        new_cols = dict(c)

        def place(name, src_spans, dst_off, ln):
            ln = np.asarray(ln, dtype=np.int64)
            out = np.zeros(len(src_spans), dtype=STR_DTYPE)
            nz = ln > 0
            out["off"][: len(ln)][nz] = dst_off[nz]
            out["len"][: len(ln)] = ln
            tot = int(ln.sum())
            if tot:
                ramp = np.arange(tot, dtype=np.int64) - np.repeat(np.cumsum(ln) - ln, ln)
                arena[np.repeat(dst_off, ln) + ramp] = self.arena[np.repeat(src_spans["off"][: len(ln)].astype(np.int64), ln) + ramp]
            new_cols[name] = out

        cur = base[:-1].copy()
        for k in order:
            place(k, c[k], cur, lens[k])
            cur = cur + lens[k]
        jr = np.repeat(np.arange(n), np.diff(c["risk_off"].astype(np.int64)))
        place("risk_tags", c["risk_tags"], cur[jr] + risk_pre, rl)
        cur = cur + risk_job
        jq = np.repeat(np.arange(n), np.diff(c["requires_off"].astype(np.int64)))
        place("requires_", c["requires_"], cur[jq] + req_pre, ql)
        cur = cur + req_job
        jl = np.repeat(np.arange(n), np.diff(c["label_off"].astype(np.int64)))
        place("label_keys", c["label_keys"], cur[jl] + lab_pre, kl)
        place("label_vals", c["label_vals"], cur[jl] + lab_pre + kl, vl)
        cur = cur + lab_job
        place("effective_config", c["effective_config"], cur, lens["effective_config"])
        return EnvelopeBatch(n, arena, new_cols)

    def with_approved(self, mask) -> "EnvelopeBatch":
        cols = dict(self.cols)
        cols["approved"] = np.ascontiguousarray(mask, dtype=np.uint8)
        return EnvelopeBatch(self.n_jobs, self.arena, cols)

    def slice(self, first: int, count: int) -> "EnvelopeBatch":
        """A view-free copy of jobs [first, first+count) (CSR columns re-based)."""
        cols = {}
        sl = slice(first, first + count)
        for k in self.SCALARS + ("has_meta", "actor_type", "approved"):
            cols[k] = self.cols[k][sl].copy()
        for off, vals in (("risk_off", ("risk_tags",)), ("requires_off", ("requires_",)), ("label_off", ("label_keys", "label_vals"))):
            o = self.cols[off]
            a, b = int(o[first]), int(o[first + count])
            cols[off] = (o[first:first + count + 1] - o[first]).astype(np.uint32)
            for v in vals:
                part = self.cols[v][a:b].copy()
                cols[v] = part if len(part) else np.zeros(1, dtype=STR_DTYPE)
        return EnvelopeBatch(count, self.arena, cols)


class WorkerTable:
    """Owns the numpy buffers behind one cordum_workers struct."""

    def __init__(self, n: int, arena: np.ndarray, cols: dict[str, np.ndarray]):
        self.n_workers = int(n)
        self.arena = np.ascontiguousarray(arena, dtype=np.uint8)
        self.cols = {k: np.ascontiguousarray(v) for k, v in cols.items()}
        assert self.cols["active_jobs"].dtype == np.int32 and self.cols["max_parallel_jobs"].dtype == np.int32
        assert self.cols["cpu_load"].dtype == np.float32 and self.cols["gpu_utilization"].dtype == np.float32
        s = CordumWorkers()
        s.n_workers = self.n_workers
        s.arena = _ptr(self.arena)
        s.arena_len = len(self.arena)
        for name, _ in CordumWorkers._fields_[3:]:
            setattr(s, name, _ptr(self.cols[name]))
        self.struct = s

    def byref(self):
        return C.byref(self.struct)

    def loads(self) -> np.ndarray:
        out = np.zeros(self.n_workers, dtype=LOAD_DTYPE)
        for k in ("active_jobs", "max_parallel_jobs", "cpu_load", "gpu_utilization"):
            out[k] = self.cols[k][: self.n_workers]
        return out

    def worker_id(self, slot: int) -> str:
        s = self.cols["worker_id"][slot]
        return bytes(self.arena[int(s["off"]): int(s["off"]) + int(s["len"])]).decode("utf-8", "replace")

    def to_workers(self) -> list[dict]:
        c = self.cols

        def st(span):
            o, n = int(span["off"]), int(span["len"])
            return bytes(self.arena[o:o + n]).decode("utf-8", "surrogateescape")

        out = []
        for i in range(self.n_workers):
            out.append({"worker_id": st(c["worker_id"][i]), "pool": st(c["pool"][i]),
                        "active_jobs": int(c["active_jobs"][i]), "max_parallel_jobs": int(c["max_parallel_jobs"][i]),
                        "cpu_load": float(c["cpu_load"][i]), "gpu_utilization": float(c["gpu_utilization"][i]),
                        "labels": {st(c["label_keys"][k]): st(c["label_vals"][k])
                                   for k in range(c["label_off"][i], c["label_off"][i + 1])}})
        return out

    @staticmethod
    def from_workers(workers: Iterable[dict]) -> "WorkerTable":
        workers = list(workers)
        n = len(workers)
        ar = _Arena()
        m = max(n, 1)
        wid = np.zeros(m, dtype=STR_DTYPE)
        pool = np.zeros(m, dtype=STR_DTYPE)
        active = np.zeros(m, np.int32)
        maxp = np.zeros(m, np.int32)
        cpu = np.zeros(m, np.float32)
        gpu = np.zeros(m, np.float32)
        off = np.zeros(n + 1, np.uint32)
        lk, lv = [], []
        for i, w in enumerate(workers):
            wid[i] = ar.add(w.get("worker_id", ""))
            pool[i] = ar.add(w.get("pool", ""))
            active[i] = w.get("active_jobs", 0)
            maxp[i] = w.get("max_parallel_jobs", 0)
            cpu[i] = np.float32(w.get("cpu_load", 0.0))
            gpu[i] = np.float32(w.get("gpu_utilization", 0.0))
            for k, v in (w.get("labels") or {}).items():
                lk.append(ar.add(k))
                lv.append(ar.add(v))
            off[i + 1] = len(lk)

        def strs(lst):
            a = np.zeros(max(len(lst), 1), dtype=STR_DTYPE)
            for i, t in enumerate(lst):
                a[i] = t
            return a

        return WorkerTable(n, ar.array(), dict(
            worker_id=wid, pool=pool, active_jobs=active, max_parallel_jobs=maxp, cpu_load=cpu,
            gpu_utilization=gpu, label_off=off, label_keys=strs(lk), label_vals=strs(lv)))
