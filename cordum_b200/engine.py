"""Engine: thin Python handle over the C ABI (no logic of its own)."""
from __future__ import annotations

import ctypes as C
import json

import numpy as np

from . import _lib, policy_io, wire


class CordumError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__("cordum_b200 error %d: %s" % (code, msg))
        self.code = code


class Batch:
    def __init__(self, eng: "Engine", max_jobs: int):
        self.eng = eng
        self.L = eng.L
        h = C.c_void_p()
        eng._ck(self.L.cordum_batch_alloc(eng.h, max_jobs, C.byref(h)))
        self.h = h
        self.max_jobs = max_jobs
        eng._batches.append(self)

    def free(self):
        """Safe to call any number of times, and after the engine was closed (which already released the batch)."""
        if self.h and self.eng.h:
            self.L.cordum_batch_free(self.h)
        self.h = None
        if self in self.eng._batches:
            self.eng._batches.remove(self)

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass

    @property
    def size(self) -> int:
        return self.L.cordum_batch_size(self.h)

    default_device_encode = False   # tests flip this to run whole suites through cordum_encode_device

    def encode(self, env):
        if self.default_device_encode:
            return self.encode_device(env)
        if not isinstance(env, wire.EnvelopeBatch):
            env = wire.EnvelopeBatch.from_jobs(env)
        self._env = env   # keep the buffers alive for the duration of the call chain
        self.eng._ck(self.L.cordum_encode(self.eng.h, self.h, env.address))
        return self

    def encode_device(self, env):
        """Encode on the GPU (cordum_encode_device).  `env`: a PinnedEnvelopes (DMA at PCIe rate) or an EnvelopeBatch
        (pageable memory).  Asynchronous; the envelope buffers must stay unchanged until wait()."""
        if not isinstance(env, (wire.EnvelopeBatch, PinnedEnvelopes)):
            env = wire.EnvelopeBatch.from_jobs(env)
        self._env = env
        self.eng._ck(self.L.cordum_encode_device(self.eng.h, self.h, env.address))
        return self

    def records(self):
        """(JobRec[n], RouteRec[n], slot_of[n]) of the encoded batch, whichever encoder produced them."""
        n = self.size
        job = np.zeros(max(n, 1), dtype=wire.JOB_REC_DTYPE)
        route = np.zeros(max(n, 1), dtype=wire.ROUTE_REC_DTYPE)
        slot = np.zeros(max(n, 1), dtype=np.uint32)
        self.eng._ck(self.L.cordum_batch_records(self.h, job.ctypes.data, route.ctypes.data, slot.ctypes.data))
        return job[:n], route[:n], slot[:n]

    def dispatch(self, mode=wire.MODE_POLICY_AND_ROUTE) -> np.ndarray:
        self.eng._ck(self.L.cordum_dispatch(self.eng.h, self.h, mode))
        return self.results()

    def dispatch_async(self, mode=wire.MODE_POLICY_AND_ROUTE):
        self.eng._ck(self.L.cordum_dispatch_async(self.eng.h, self.h, mode))

    def wait(self) -> np.ndarray:
        self.eng._ck(self.L.cordum_batch_wait(self.h))
        return self.results()

    def dispatch_resident(self, mode=wire.MODE_POLICY_AND_ROUTE, flush_l2=False):
        self.eng._ck(self.L.cordum_dispatch_resident(self.eng.h, self.h, mode | (wire.FLAG_FLUSH_L2 if flush_l2 else 0)))

    def dispatch_resident_async(self, mode=wire.MODE_POLICY_AND_ROUTE, flush_l2=False):
        self.eng._ck(self.L.cordum_dispatch_resident_async(self.eng.h, self.h, mode | (wire.FLAG_FLUSH_L2 if flush_l2 else 0)))

    def tick(self, slice_ptr: int, first_slot: int, n_slice: int):
        """One scheduler tick (cordum_tick_async): heartbeat epoch + policy of this batch + route of the previous tick's batch,
        one graph launch.  Results: wait() then fetch()."""
        self.eng._ck(self.L.cordum_tick_async(self.eng.h, self.h, wire.MODE_POLICY_AND_ROUTE, C.c_void_p(slice_ptr), first_slot, n_slice))

    def fetch(self) -> np.ndarray:
        self.eng._ck(self.L.cordum_batch_fetch(self.h))
        return self.results()

    def results(self) -> np.ndarray:
        n = self.size
        ptr = self.L.cordum_batch_results(self.h)
        buf = (C.c_uint8 * (n * wire.DECISION_DTYPE.itemsize)).from_address(ptr)
        return np.frombuffer(buf, dtype=wire.DECISION_DTYPE, count=n)

    def timing(self):
        t, k = C.c_float(), C.c_float()
        self.eng._ck(self.L.cordum_batch_timing(self.h, C.byref(t), C.byref(k)))
        return t.value, k.value

    @property
    def stream(self) -> int:
        """The batch's cudaStream_t (as an integer), for harnesses that bracket launches with their own CUDA events."""
        return int(self.L.cordum_batch_stream(self.h) or 0)

    def kernel_times(self):
        p, r = C.c_float(), C.c_float()
        self.eng._ck(self.L.cordum_batch_kernel_times(self.h, C.byref(p), C.byref(r)))
        return p.value, r.value

    def plan(self):
        """(offsets, jobs, n_slots) of the last completed dispatch (cordum_batch_plan): jobs grouped by destination worker
        slot (buckets 0 .. n_slots-1), then by outcome (bucket n_slots + k, wire.PLAN_OUTCOME_NAMES[k]); bucket b holds
        jobs[offsets[b]:offsets[b+1]], ascending.  Views of library memory, valid until this batch's next encode,
        dispatch, plan or free."""
        p = wire.CordumPlan()
        self.eng._ck(self.L.cordum_batch_plan(self.h, C.byref(p)))
        nb = p.n_slots + wire.PLAN_OUTCOMES

        def view(ptr, count):
            return np.frombuffer((C.c_uint32 * count).from_address(ptr), dtype=np.uint32, count=count) if count else np.zeros(0, np.uint32)

        return view(p.offsets, nb + 1), view(p.jobs, p.n_jobs), int(p.n_slots)

    @staticmethod
    def plan_buckets(offsets, jobs):
        """The non-empty buckets of a plan: (bucket, job indices) pairs in bucket order."""
        for b in np.flatnonzero(np.diff(offsets)):
            yield int(b), jobs[offsets[b]:offsets[b + 1]]

    def topic_counts(self):
        """(labels, counts) of the last completed dispatch (cordum_batch_topic_counts): labels = the distinct
        TrimSpace(topic) of its jobs as bytes, ascending; counts = uint32 [len(labels), wire.COUNT_COLUMNS], column k <
        wire.PLAN_OUTCOMES the jobs of plan outcome k, column wire.COUNT_ROUTED the routed jobs.  The counts are a view of
        library memory, valid until this batch's next encode, dispatch, topic_counts or free."""
        t = wire.CordumTopicCounts()
        self.eng._ck(self.L.cordum_batch_topic_counts(self.h, C.byref(t)))
        n = t.n_rows
        if not n:
            return [], np.zeros((0, wire.COUNT_COLUMNS), np.uint32)
        off = np.frombuffer((C.c_uint32 * (n + 1)).from_address(t.label_off), dtype=np.uint32, count=n + 1)
        raw = C.string_at(t.label_bytes, int(off[n])) if off[n] else b""
        labels = [raw[off[r]:off[r + 1]] for r in range(n)]
        counts = np.frombuffer((C.c_uint32 * (n * wire.COUNT_COLUMNS)).from_address(t.counts), dtype=np.uint32,
                               count=n * wire.COUNT_COLUMNS).reshape(n, wire.COUNT_COLUMNS)
        return labels, counts

    def responses(self, flavor: int = wire.REASON_FLAVOR_KERNEL) -> dict:
        """The last completed dispatch's jobs grouped by safety response class (cordum_batch_responses): {"classes":
        wire.RESPONSE_CLASS_DTYPE [m] in first_job order, "reasons": [str] and "rule_ids": [str] per class, "offsets":
        uint32 [m + 1], "jobs": uint32 [n] (class c holds jobs[offsets[c]:offsets[c+1]], ascending), "policy_gen": int}.
        The arrays are views of library memory, valid until this batch's next encode, dispatch, responses call or free."""
        r = wire.CordumResponses()
        self.eng._ck(self.L.cordum_batch_responses(self.h, flavor, C.byref(r)))
        m, n = r.n_classes, r.n_jobs

        def view(ptr, count, dtype=np.uint32):
            if not count:
                return np.zeros(0, dtype)
            return np.frombuffer((C.c_uint8 * (count * np.dtype(dtype).itemsize)).from_address(ptr), dtype=dtype, count=count)

        def texts(off_ptr, bytes_ptr):
            off = view(off_ptr, m + 1)
            raw = C.string_at(bytes_ptr, int(off[m])) if off[m] else b""
            return [raw[off[c]:off[c + 1]].decode("utf-8", "replace") for c in range(m)]

        return {"classes": view(r.classes, m, wire.RESPONSE_CLASS_DTYPE), "reasons": texts(r.reason_off, r.reason_bytes),
                "rule_ids": texts(r.rule_id_off, r.rule_id_bytes), "offsets": view(r.offsets, m + 1), "jobs": view(r.jobs, n),
                "policy_gen": int(r.policy_gen)}

    def subset(self, dst: "Batch", outcomes: int = None, jobs=None) -> int:
        """Make `dst` the encoded batch of a subset of this one (cordum_batch_subset), on the device: the jobs whose plan
        outcome bucket k has bit k set in `outcomes` (e.g. wire.SUBSET_RETRYABLE), or the strictly ascending job indices
        `jobs`.  Returns dst's job count; dst.parent_index() maps its jobs back to this batch's."""
        m = C.c_uint32()
        if jobs is None:
            self.eng._ck(self.L.cordum_batch_subset(self.h, outcomes or 0, None, 0, dst.h, C.byref(m)))
        else:
            lst = np.ascontiguousarray(jobs, dtype=np.uint32)
            buf = lst if len(lst) else np.zeros(1, np.uint32)   # the empty list is a list: a non-null pointer
            self.eng._ck(self.L.cordum_batch_subset(self.h, outcomes or 0, C.c_void_p(buf.ctypes.data), len(lst), dst.h, C.byref(m)))
        dst._env = None   # dst holds no envelopes: MCP reasons quote the canonical spelling
        return m.value

    def merge(self, other: "Batch", dst: "Batch") -> int:
        """Make `dst` the encoded batch of this batch's jobs followed by `other`'s (cordum_batch_merge), on the device: its
        records are those a host encode of both batches' envelopes, this one's first, would give.  `other` may be this
        batch.  Returns dst's job count."""
        self.eng._ck(self.L.cordum_batch_merge(self.h, other.h, dst.h))
        dst._env = None   # dst holds no envelopes: MCP reasons quote the canonical spelling
        return dst.size

    def parent_index(self) -> np.ndarray:
        """This batch's job i -> the source batch's job index, when its records came from Batch.subset (else empty).  A
        view of library memory, valid until this batch's next encode, subset or free."""
        n = C.c_uint32()
        ptr = self.L.cordum_batch_parent_index(self.h, C.byref(n))
        if not ptr or not n.value:
            return np.zeros(0, np.uint32)
        return np.frombuffer((C.c_uint32 * n.value).from_address(ptr), dtype=np.uint32, count=n.value)

    def _text(self, fn, job: int, *extra) -> str:
        buf = C.create_string_buffer(4096)
        n = fn(self.eng.h, self.h, job, *extra, buf, len(buf))
        if n >= len(buf):
            buf = C.create_string_buffer(n + 1)
            fn(self.eng.h, self.h, job, *extra, buf, len(buf))
        return buf.value.decode("utf-8", "replace")

    def reason(self, job: int, flavor: int = wire.REASON_FLAVOR_KERNEL) -> str:
        """The reason string of the reference for this job's record, byte for byte.  flavor REASON_FLAVOR_GATEWAY: as the gateway's evaluatePolicyCheck words it (policy_bundles.go:1207,1211)."""
        env = getattr(self, "_env", None)   # the request's own spelling of an MCP value needs the envelopes
        addr = env.address if env is not None and getattr(env, "n_jobs", self.size) == self.size else None
        return self._text(self.L.cordum_reason_flavor, job, flavor, addr)

    def snapshot(self) -> str:
        """The policy snapshot the last dispatch of this batch ran under."""
        buf = C.create_string_buffer(1024)
        self.L.cordum_batch_snapshot(self.h, buf, len(buf))
        return buf.value.decode("utf-8", "replace")

    def policy_gen(self) -> int:
        """Generation of the policy the last dispatch ran under (Engine.rule_id(idx, gen) etc.)."""
        return int(self.L.cordum_batch_policy_gen(self.h))

    def subject(self, job: int) -> str:
        return self._text(self.L.cordum_subject, job)


class PinnedEnvelopes:
    """A cordum_envelopes whose arrays live in page-locked memory owned by the library (cordum_envelopes_alloc): the
    host writes strings and spans straight into what the GPU will DMA.  fill() copies an EnvelopeBatch in - standing
    in for a shim that unpacks its requests directly into these buffers."""

    LISTS = (("risk_off", ("risk_tags",)), ("requires_off", ("requires_",)), ("label_off", ("label_keys", "label_vals")))

    def __init__(self, eng: "Engine", max_jobs: int, arena_bytes: int, max_risk: int, max_requires: int, max_labels: int):
        self.eng = eng
        self.caps = wire.CordumEnvelopeCaps(max_jobs, max_risk, max_requires, max_labels, arena_bytes)
        h = C.c_void_p()
        eng._ck(eng.L.cordum_envelopes_alloc(eng.h, C.byref(self.caps), C.byref(h)))
        self.h = h
        self.struct = wire.CordumEnvelopes.from_address(h.value)
        self.address = h.value

    def _view(self, name, dtype, count):
        ptr = getattr(self.struct, name)
        buf = (C.c_uint8 * (count * np.dtype(dtype).itemsize)).from_address(ptr)
        return np.frombuffer(buf, dtype=dtype, count=count)

    def fill(self, env: "wire.EnvelopeBatch"):
        n = env.n_jobs
        c = env.cols
        assert n <= self.caps.max_jobs and len(env.arena) <= self.caps.arena_bytes
        self._view("arena", np.uint8, len(env.arena))[:] = env.arena
        for k in wire.EnvelopeBatch.SCALARS:
            self._view(k, wire.STR_DTYPE, n)[:] = c[k][:n]
        for k in ("has_meta", "actor_type", "approved"):
            self._view(k, np.uint8, n)[:] = c[k][:n]
        for off, vals in self.LISTS:
            self._view(off, np.uint32, n + 1)[:] = c[off]
            m = int(c[off][n])
            cap = {"risk_off": self.caps.max_risk_tags, "requires_off": self.caps.max_requires, "label_off": self.caps.max_labels}[off]
            assert m <= max(cap, 1)
            for v in vals:
                self._view(v, wire.STR_DTYPE, max(m, 1))[:m] = c[v][:m]
        self.struct.n_jobs = n
        self.struct.arena_len = len(env.arena)
        self.n_jobs = n
        return self

    def free(self):
        if self.h and self.eng.h:
            self.eng.L.cordum_envelopes_free(self.eng.h, self.h)
        self.h = None


class Engine:
    def __init__(self, device: int = 0, max_topics: int = 0, max_effcfgs: int = 0, encode_threads: int = 0):
        self.L = _lib.load()
        opts = wire.CordumEngineOpts(device, max_topics, max_effcfgs, encode_threads)
        h = C.c_void_p()
        rc = self.L.cordum_engine_create(C.byref(opts), C.byref(h))
        if rc:
            raise CordumError(rc, self.L.cordum_last_error().decode())
        self.h = h
        self._batches: list = []

    def _ck(self, rc: int):
        if rc:
            raise CordumError(rc, self.L.cordum_last_error().decode())

    def close(self):
        """Frees every live batch first: a batch must never outlive its engine."""
        if self.h:
            for b in list(self._batches):
                b.free()
            self.L.cordum_engine_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def load_policy(self, policy, snapshot: str = ""):
        doc = policy if isinstance(policy, (bytes, bytearray)) else policy_io.to_json(policy)
        snap = snapshot.encode()
        self._ck(self.L.cordum_policy_load(self.h, bytes(doc), len(doc), snap, len(snap)))

    def load_routing(self, routing):
        doc = routing if isinstance(routing, (bytes, bytearray)) else policy_io.to_json(routing)
        self._ck(self.L.cordum_routing_load(self.h, bytes(doc), len(doc)))

    def load_workers(self, workers):
        wt = workers if isinstance(workers, wire.WorkerTable) else wire.WorkerTable.from_workers(workers)
        self._workers = wt
        self._ck(self.L.cordum_workers_load(self.h, C.addressof(wt.struct)))

    def update_workers(self, slots, loads):
        slots = np.ascontiguousarray(slots, dtype=np.uint32)
        loads = np.ascontiguousarray(loads, dtype=wire.LOAD_DTYPE)
        self._ck(self.L.cordum_workers_update(self.h, len(slots), slots.ctypes.data, loads.ctypes.data))

    def set_loads_device(self, dptr: int, n_workers: int, stream: int = 0):
        self._ck(self.L.cordum_workers_set_loads_device(self.h, C.c_void_p(dptr), n_workers, C.c_void_p(stream)))

    # ---- engine-owned multi-GPU heartbeat exchange (include/cordum_b200.h: cordum_exchange_*)
    @staticmethod
    def exchange_unique_id() -> bytes:
        """Rank 0 creates the id and ships the 128 bytes to the other ranks (any transport)."""
        L = _lib.load()
        buf = C.create_string_buffer(128)
        rc = L.cordum_exchange_unique_id(buf)
        if rc:
            raise CordumError(rc, L.cordum_last_error().decode("utf-8", "replace"))
        return buf.raw

    def exchange_init(self, unique_id: bytes, rank: int, world: int):
        """Collective: every rank calls it with the same id; blocks until all have joined."""
        assert len(unique_id) == 128
        buf = C.create_string_buffer(unique_id, 128)
        self._ck(self.L.cordum_exchange_init(self.h, buf, rank, world))

    def tick_flush(self):
        self._ck(self.L.cordum_tick_flush(self.h))

    @property
    def tick_stream(self) -> int:
        return int(self.L.cordum_tick_stream(self.h) or 0)

    def peer_export(self, rank: int, world: int) -> bytes:
        buf = C.create_string_buffer(64)
        self._ck(self.L.cordum_peer_export(self.h, rank, world, buf))
        return buf.raw

    def peer_import(self, handles: list):
        blob = b"".join(handles)
        buf = C.create_string_buffer(blob, len(blob))
        self._ck(self.L.cordum_peer_import(self.h, buf))

    def ingest(self, slice_ptr: int, first_slot: int, n_slice: int):
        """One heartbeat epoch: this rank's slice of 16 B load records (host pointer, pinned for an asynchronous
        copy) -> device, all-gather across ranks, worker-table refresh.  Returns once enqueued."""
        self._ck(self.L.cordum_workers_ingest(self.h, C.c_void_p(slice_ptr), first_slot, n_slice))

    def snapshots(self) -> list[str]:
        buf = C.create_string_buffer(1 << 16)
        n = C.c_uint32()
        self._ck(self.L.cordum_policy_snapshots(self.h, buf, len(buf), C.byref(n)))
        return [s.decode() for s in buf.raw.split(b"\0")[: n.value]]

    def pinned_envelopes(self, like: "wire.EnvelopeBatch" = None, max_jobs=0, arena_bytes=0, max_risk=0, max_requires=0, max_labels=0) -> PinnedEnvelopes:
        """Page-locked envelope staging (cordum_envelopes_alloc), sized for `like` if given, and filled from it."""
        if like is not None:
            n = like.n_jobs
            p = PinnedEnvelopes(self, max(max_jobs, n), max(arena_bytes, len(like.arena)), max(max_risk, int(like.cols["risk_off"][n])),
                                max(max_requires, int(like.cols["requires_off"][n])), max(max_labels, int(like.cols["label_off"][n])))
            return p.fill(like)
        return PinnedEnvelopes(self, max_jobs, arena_bytes, max_risk, max_requires, max_labels)

    def host_fallbacks(self) -> int:
        return int(self.L.cordum_host_fallbacks(self.h))

    def current_snapshot(self) -> str:
        buf = C.create_string_buffer(4096)
        self.L.cordum_policy_snapshot(self.h, buf, len(buf))
        return buf.value.decode("utf-8", "replace")

    def batch(self, max_jobs: int) -> Batch:
        return Batch(self, max_jobs)

    # gen: policy generation the rule index belongs to (Batch.policy_gen()); 0 = the policy in force
    def _rule_text(self, fn, gen: int, idx: int) -> str:
        buf = C.create_string_buffer(1 << 12)
        n = fn(self.h, gen, idx, buf, len(buf))
        if n >= len(buf):
            buf = C.create_string_buffer(n + 1)
            fn(self.h, gen, idx, buf, len(buf))
        return buf.value.decode("utf-8", "replace") if n > 0 else ""

    def rule_id(self, idx: int, gen: int = 0) -> str:
        return self._rule_text(self.L.cordum_rule_id_at, gen, idx)

    def rule_constraints(self, idx: int, gen: int = 0):
        s = self._rule_text(self.L.cordum_rule_constraints_json_at, gen, idx)
        return json.loads(s) if s else None

    def rule_remediations(self, idx: int, gen: int = 0):
        s = self._rule_text(self.L.cordum_rule_remediations_json_at, gen, idx)
        return json.loads(s) if s else []

    def stats(self) -> wire.CordumTableStats:
        st = wire.CordumTableStats()
        self._ck(self.L.cordum_stats(self.h, C.byref(st)))
        return st

    def launch_count(self) -> int:
        return int(self.L.cordum_launch_count(self.h))
