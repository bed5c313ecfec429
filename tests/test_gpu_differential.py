"""Differential tests of the kernels (policy_kernel, route_kernel, worker_chunk_kernel, worker_merge_kernel) against the C++
oracle, bit-exact on every field of the decision record, where the kernels have machinery of their own:

  * the adversarial configurations of test_fuzz_three_way.py (awkward strings, legacy policies, MCP lists, effective
    configs, wide universes, reload / heartbeat life cycles), run through the engine instead of a re-walk of its tables
  * forced policy summaries (CORDUM_SUM_USE): every attribute's summary alone, none and all, so the word-group skipping
    of policy_kernel runs with summaries the table compiler would not pick on its own
  * refresh and route boundaries: pool sizes around the 32-worker bitmap word, the 512-worker chunk and the 8,192-worker
    sort limit, topics with more than four pools, pools above the sort limit next to sorted ones, non-overloaded
    prefixes ending on and next to a word boundary, label scans whose matches lie far apart, preference hints
  * edge load values (subnormal, signed zero, negative, infinite, the 90 / 0.9 thresholds, active_jobs beyond 2^24)
    delivered through every load path: cordum_workers_load, cordum_workers_update, cordum_workers_ingest,
    cordum_workers_set_loads_device and cordum_tick_async
  * grid shapes where a warp loops over several tiles, and the other template instances of the kernels (slow)

NaN loads stay out of the device paths: cordum_workers_ingest, cordum_workers_set_loads_device and cordum_tick_async do not
refuse them while the two host paths do, and in the reference the pick among NaN loads depends on map iteration order, so
there is no one answer to compare with yet.  Run on an H100: pytest -m gpu tests/test_gpu_differential.py."""
import functools
import json
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import kats
import oracle_lib
import table_walk
import test_fuzz_three_way as fuzz
from cordum_b200 import synth, wire

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIELDS = ("decision", "sched_decision", "flags", "route_status", "reason_code", "rule_idx", "worker_slot")
MODES = (wire.MODE_POLICY_AND_ROUTE, wire.MODE_POLICY_ONLY, wire.MODE_ROUTE_ONLY)
MODE_NAMES = {wire.MODE_POLICY_AND_ROUTE: "policy+route", wire.MODE_POLICY_ONLY: "policy", wire.MODE_ROUTE_ONLY: "route"}


def usable_cores() -> int:
    try:
        return max(1, len(os.sched_getaffinity(0)))
    except AttributeError:
        return os.cpu_count() or 1


@pytest.fixture(scope="module", params=["host-encode", "device-encode"])
def eng(request):
    """One engine for the module, run once with the host encoder and once with the device encoder."""
    from cordum_b200 import engine

    engine.Batch.default_device_encode = request.param == "device-encode"
    e = engine.Engine(device=0)
    # batches the device encoder was given / completed without handing them to the host (test_device_encoder_kept_batches)
    e.device_encodes = {"tried": 0, "kept": 0} if request.param == "device-encode" else None
    yield e
    e.close()
    engine.Batch.default_device_encode = False


def load(e, policy, routing, workers):
    e.load_policy(policy, "differential")
    e.load_routing(routing)
    e.load_workers(workers)


def job_json(job) -> str:
    return json.dumps(job, default=lambda x: x.decode("utf-8", "replace") if isinstance(x, bytes) else str(x))


def assert_same(got, want, what, jobs=None):
    assert len(got) == len(want), what
    for f in FIELDS:
        bad = np.nonzero(got[f] != want[f])[0]
        if len(bad):
            first = int(bad[0])
            pytest.fail("%s: field %s differs at %d jobs, first %s: kernels %s oracle %s\njob %d: %s" % (
                what, f, len(bad), bad[:8].tolist(), got[f][bad[:8]].tolist(), want[f][bad[:8]].tolist(), first,
                job_json(jobs[first]) if jobs is not None else "(synthetic batch)"))


def compare(e, o, jobs, what, modes=MODES):
    """Encode `jobs`, dispatch them in every mode and compare each record with the oracle.  Returns {mode: records}."""
    env = jobs if isinstance(jobs, wire.EnvelopeBatch) else wire.EnvelopeBatch.from_jobs(jobs)
    listed = None if isinstance(jobs, wire.EnvelopeBatch) else jobs
    b = e.batch(max(env.n_jobs, 1))
    out = {}
    try:
        for mode in modes:
            f0 = e.host_fallbacks()
            got = b.encode(env).dispatch(mode).copy()
            if getattr(e, "device_encodes", None) is not None:
                e.device_encodes["tried"] += 1
                e.device_encodes["kept"] += e.host_fallbacks() == f0
            assert_same(got, o.eval(env, mode, threads=usable_cores()), "%s, %s" % (what, MODE_NAMES[mode]), listed)
            out[mode] = got
    finally:
        b.free()
    return out


def assert_sum_use(policy, routing, workers, sum_use):
    """The knob is read where the engine's table compiler reads it (Host::choose_summaries): a host-only compile of the
    same configuration in this process shows what the engine's tables carry."""
    if sum_use is None:
        return
    h = table_walk.HostHarness(policy, routing, workers)
    assert h.tables()["sum_use"] == sum_use
    h.close()


# ------------------------------------------------------------------ the three-way fuzz, through the kernels
@pytest.mark.parametrize("seed,max_rules,sum_use", fuzz.with_sum_use([(s, 12, None) for s in range(60)] +
                                                                     [(100 + s, 400, u) for s in range(12) for u in [None] + fuzz.SUM_USE_FORCED]))
def test_fuzz_configs_through_the_kernels(eng, seed, max_rules, sum_use, monkeypatch):
    fuzz.force_sum_use(monkeypatch, sum_use)
    policy, routing, workers, jobs = fuzz.fuzz_case(seed, max_rules)
    load(eng, policy, routing, workers)
    assert_sum_use(policy, routing, workers, sum_use)
    o = oracle_lib.Oracle(policy, routing, workers)
    compare(eng, o, jobs, "seed %d (%d rules, sum_use %s)" % (seed, max_rules, sum_use))
    o.close()


@pytest.mark.parametrize("seed,sum_use", fuzz.with_sum_use([(s, u) for s in range(16) for u in [None] + fuzz.SUM_USE_FORCED]))
def test_wide_universes_through_the_kernels(eng, seed, sum_use, monkeypatch):
    fuzz.force_sum_use(monkeypatch, sum_use)
    fuzz.widen(monkeypatch)
    policy, routing, workers, jobs = fuzz.wide_case(seed)
    load(eng, policy, routing, workers)
    assert_sum_use(policy, routing, workers, sum_use)
    o = oracle_lib.Oracle(policy, routing, workers)
    compare(eng, o, jobs, "wide seed %d (sum_use %s)" % (seed, sum_use))
    o.close()


@functools.lru_cache(maxsize=None)
def c2_config():
    return synth.make_config("c2")


@pytest.mark.parametrize("sum_use", [None] + fuzz.SUM_USE_FORCED)
def test_c2_with_forced_summaries(eng, sum_use, monkeypatch):
    fuzz.force_sum_use(monkeypatch, sum_use)
    cfg = c2_config()
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    assert_sum_use(cfg.policy, cfg.routing, cfg.workers, sum_use)
    o = oracle_lib.Oracle(cfg.policy, cfg.routing, cfg.workers)
    compare(eng, o, cfg.jobs, "c2 (sum_use %s)" % sum_use)
    o.close()


@pytest.mark.parametrize("sum_use", [None] + fuzz.SUM_USE_FORCED)
def test_sparse_summaries_through_the_kernels(eng, sum_use, monkeypatch):
    """Risk, capability and pack summaries that prune word groups (one 128-bit word per risk tag, tags 64... in the wide
    row): a summary read from the wrong row skips the word of the first match."""
    fuzz.force_sum_use(monkeypatch, sum_use)
    policy, routing, workers, jobs = fuzz.sparse_summary_case()
    load(eng, policy, routing, workers)
    assert_sum_use(policy, routing, workers, sum_use)
    o = oracle_lib.Oracle(policy, routing, workers)
    got = compare(eng, o, jobs, "sparse summaries (sum_use %s)" % sum_use)
    assert len(set(got[wire.MODE_POLICY_ONLY]["rule_idx"].tolist())) > 100
    o.close()


# ------------------------------------------------------------------ load paths
LOAD_PATHS = ("update_workers", "ingest", "set_loads_device", "tick")


def deliver(e, path, table, host, keep, batch=None):
    """Put the full slot-ordered load `table` in force through one load path of the engine.

    `host` is the engine's host-side table (cordum_workers_load, then cordum_workers_update deltas): update_workers sends
    only the rows in which it differs from `table`, and keeps it current.  The three device paths replace the table the
    kernels read and leave the host's alone.  tick runs one tick of `batch` (encoded and resident) and waits for it; its
    records are then batch.fetch().  `keep` holds the buffers until the caller is done with the engine's results."""
    n = len(table)
    if path == "update_workers":
        rows = np.nonzero((host.view(np.uint8).reshape(n, 16) != table.view(np.uint8).reshape(n, 16)).any(axis=1))[0]
        e.update_workers(rows.astype(np.uint32), table[rows])
        host[rows] = table[rows]
    elif path == "ingest":
        buf = table.copy()
        keep.append(buf)
        e.ingest(buf.ctypes.data, 0, n)
    elif path == "set_loads_device":
        import torch

        dev = torch.from_numpy(table.view(np.uint8).reshape(n, 16).copy()).cuda()
        torch.cuda.synchronize()
        keep.append(dev)
        e.set_loads_device(dev.data_ptr(), n, torch.cuda.current_stream().cuda_stream)
    elif path == "tick":
        buf = table.copy()
        keep.append(buf)
        batch.tick(buf.ctypes.data, 0, n)
        batch.wait()
    else:
        raise ValueError(path)


@pytest.mark.parametrize("seed", range(30))
def test_life_cycle_through_the_kernels(eng, seed):
    """The reload / heartbeat life cycle of the CPU fuzz.  Heartbeat steps rotate through cordum_workers_update (the
    delta itself), cordum_workers_ingest and cordum_workers_set_loads_device (the whole table with the delta applied).
    A registry or routing reload rebuilds the worker tables from the host's loads, so from there the kernels route on
    those again."""
    o = None
    host = live = None
    keep, beats = [], 0
    for step, (kind, payload, jobs) in enumerate(fuzz.life_cycle(seed)):
        what = "load" if kind == "load" else "%s (step %d)" % (kind, step - 1)
        if kind == "load":
            policy, routing, workers = payload
            load(eng, policy, routing, workers)
            o = oracle_lib.Oracle(policy, routing, workers)
            host = wire.WorkerTable.from_workers(workers).loads()
            live = host.copy()
        elif kind == "heartbeat" and payload is not None:
            slots, loads = payload
            path = LOAD_PATHS[(seed + beats) % 3]
            beats += 1
            what += " via " + path
            if path == "update_workers":
                eng.update_workers(slots, loads)
                host[slots] = loads
                live = host.copy()
            else:
                live = live.copy()
                live[slots] = loads
                deliver(eng, path, live, host, keep)
            o.update_workers(np.arange(len(live), dtype=np.uint32), live)
        elif kind == "workers":
            eng.load_workers(payload)
            o.load_workers(payload)
            host = wire.WorkerTable.from_workers(payload).loads()
            live = host.copy()
        elif kind == "routing":
            eng.load_routing(payload)
            o.load_routing(payload)
            live = host.copy()
            o.update_workers(np.arange(len(live), dtype=np.uint32), live)
        elif kind == "policy":
            eng.load_policy(payload, "differential")
            o.load_policy(payload)
        compare(eng, o, jobs, "seed %d after %s" % (seed, what))
    o.close()


# ------------------------------------------------------------------ refresh and route boundaries
POOL_SIZES = (1, 31, 32, 33, 511, 512, 513, 1024, 1025, 4097, 8191, 8192, 8193)
LABELS = {"zone": ("a", "b"), "tier": ("x", "y"), "arch": ("arm", "x86"), "disk": ("ssd", "hdd"), "os": ("linux",),
          "gpu": ("true",), "net": ("fast", "slow")}
LABEL_COUNTS = (0, 1, 1, 2, 4, 5, 7)
NOK_TARGETS = lambda n: (0, 31, 32, 33, n // 2, n)   # noqa: E731  non-overloaded prefix of a pool's load-sorted view


@functools.lru_cache(maxsize=None)
def boundary_registry():
    """Pools of every size in POOL_SIZES (workers shuffled, so slot order, worker_id order and pool order all differ);
    topics with one pool, with more than four, and with the unsorted 8,193-worker pool next to sorted ones; a small label
    vocabulary carried by most workers, plus one label ("rack": "r7") so rare that its holders lie many bitmap words
    apart; two pools that declare a requires token."""
    rng = random.Random(31)
    pools = ["p%d" % n for n in POOL_SIZES]
    workers = []
    for n, p in zip(POOL_SIZES, pools):
        for i in range(n):
            labels = {k: rng.choice(v) for k, v in LABELS.items() if rng.random() < 0.9}
            if rng.random() < 1 / 300:
                labels["rack"] = "r7"
            workers.append(kats.hb("w-%s-%05d" % (p, i), p, 0, 0.0, 0.0, 0, labels))
    rng.shuffle(workers)
    topics = {"job.many": ["p1", "p31", "p32", "p33", "p511", "p512"], "job.chunks": ["p513", "p1024", "p1025", "p4097", "p8192"],
              "job.mix": ["p8193", "p33", "p8191", "p1"], "job.all": pools, "job.huge": ["p8193"]}
    topics.update({"job.one.%s" % p: [p] for p in pools})
    routing = {"topics": topics, "pools": {p: ({"requires": ["gpu"]} if p in ("p33", "p4097") else {}) for p in pools}}
    slots = {p: np.array([i for i, w in enumerate(workers) if w["pool"] == p]) for p in pools}
    by_pool = {p: [w["worker_id"] for w in workers if w["pool"] == p] for p in pools}
    jobs = []
    for _ in range(3000):
        topic = rng.choice(sorted(topics))
        labels = {k: rng.choice(LABELS[k]) for k in rng.sample(sorted(LABELS), rng.choice(LABEL_COUNTS))}
        r = rng.random()
        if r < 0.15:
            labels["rack"] = "r7"
        elif r < 0.18:
            labels["zone"] = "nowhere"                   # a label no worker carries
        r = rng.random()
        if r < 0.1:
            labels["preferred_pool"] = rng.choice(topics[topic] + ["p8193", "p1", "nope"])
        elif r < 0.25:
            pool = rng.choice(topics[topic] + ["p8193", "p32"])
            labels["preferred_worker_id"] = rng.choice(by_pool[pool])
        job = {"topic": topic, "labels": labels}
        if rng.random() < 0.1:
            job["meta"] = {"requires": ["gpu"]}
        jobs.append(job)
    return workers, routing, slots, jobs


def boundary_loads(slots, n, epoch):
    """Coarse loads (few distinct scores: equal minima span chunks and bitmap words) and, per pool, exactly as many
    overloaded workers as leave a non-overloaded prefix of 0, 31, 32, 33, half or all of the pool - rotated by epoch."""
    rng = np.random.default_rng(100 + epoch)
    t = np.zeros(n, dtype=wire.LOAD_DTYPE)
    t["active_jobs"] = rng.integers(0, 2, n)
    t["max_parallel_jobs"] = rng.choice([0, 4], n)
    t["cpu_load"] = rng.choice(np.array([0.0, 25.0, 50.0], np.float32), n)
    for k, s in enumerate(slots.values()):
        nok = min(NOK_TARGETS(len(s))[(epoch + k) % 6], len(s))
        over = rng.permutation(s)[: len(s) - nok]
        how = rng.integers(0, 3, len(over))
        t["cpu_load"][over[how == 0]] = 95.0
        t["active_jobs"][over[how == 1]] = 9
        t["max_parallel_jobs"][over[how == 1]] = 10
        t["gpu_utilization"][over[how == 2]] = 90.0
    return t


@pytest.mark.parametrize("lbest", ["0", "1"])
def test_refresh_and_route_boundaries(eng, lbest, monkeypatch):
    """Single-label jobs are answered from the per-(pool, label) table (pool_label_best) with CORDUM_LBEST=1 and by the
    label scan of route_kernel with 0; everything else takes the same path either way.  Epoch 0 comes with the registry,
    the next ones through each load path, the last one a scheduler tick."""
    monkeypatch.setenv("CORDUM_LBEST", lbest)
    workers, routing, slots, jobs = boundary_registry()
    n = len(workers)
    # what the configuration exercises
    h = table_walk.HostHarness(None, routing, workers)
    T = h.tables()
    sizes = np.diff(T["pool_off"][: T["n_pools"] + 1].astype(np.int64))
    assert T["n_merge"] > 0 and sizes.max() > 8192 and (sizes <= 8192).sum() >= 10
    h.close()
    counts = [len([k for k in j["labels"] if not k.startswith("preferred_")]) for j in jobs]
    assert {0, 1, 2, 4, 5, 7} <= set(counts) and max(len(t) for t in routing["topics"].values()) > 4

    table = boundary_loads(slots, n, 0)
    for w, row in zip(workers, table):
        w.update(active_jobs=int(row["active_jobs"]), max_parallel_jobs=int(row["max_parallel_jobs"]),
                 cpu_load=float(row["cpu_load"]), gpu_utilization=float(row["gpu_utilization"]))
    load(eng, None, routing, workers)
    o = oracle_lib.Oracle(None, routing, workers)
    host, keep, seen, ties = table.copy(), [], set(), 0
    got = compare(eng, o, jobs, "lbest %s, epoch 0 (registry)" % lbest, (wire.MODE_POLICY_AND_ROUTE, wire.MODE_ROUTE_ONLY))
    for r in got.values():
        seen |= set(r["route_status"].tolist())
        ties += int((r["flags"] & wire.F_TIE).astype(bool).sum())
    b = eng.batch(len(jobs))
    b.encode(jobs).dispatch()                            # resident, for the tick
    for epoch, path in enumerate(LOAD_PATHS, start=1):
        table = boundary_loads(slots, n, epoch)
        o.update_workers(np.arange(n, dtype=np.uint32), table)
        what = "lbest %s, epoch %d via %s" % (lbest, epoch, path)
        if path == "tick":
            deliver(eng, path, table, host, keep, batch=b)
            got = {wire.MODE_POLICY_AND_ROUTE: b.fetch().copy()}
            assert_same(got[wire.MODE_POLICY_AND_ROUTE], o.eval(jobs, threads=usable_cores()), what, jobs)
            # a plain dispatch after the tick continues from the tick's tables
            assert_same(b.dispatch(wire.MODE_ROUTE_ONLY), o.eval(jobs, wire.MODE_ROUTE_ONLY, threads=usable_cores()),
                        what + ", then a plain dispatch", jobs)
        else:
            deliver(eng, path, table, host, keep)
            got = compare(eng, o, jobs, what, (wire.MODE_POLICY_AND_ROUTE, wire.MODE_ROUTE_ONLY))
        for r in got.values():
            seen |= set(r["route_status"].tolist())
            ties += int((r["flags"] & wire.F_TIE).astype(bool).sum())
    b.free()
    o.close()
    # what the outputs show: every outcome of a pick, and ties
    assert {wire.ROUTE_OK, wire.ROUTE_OK_PREFERRED, wire.ROUTE_POOL_OVERLOADED, wire.ROUTE_NO_WORKERS} <= seen, seen
    assert ties > 0


# ------------------------------------------------------------------ edge load values
F32 = np.float32
SUB_KEPT, SUB_LOST = 1e-40, 1e-45   # a subnormal whose /100 is still subnormal, and one whose /100 rounds to 0
RATIO_ROUNDS_UP = (1_799_999, 1_999_999)   # below 0.9, but the float32 quotient is 0.9f: overloaded
RATIO_BELOW = (899_999, 999_999)           # below 0.9 and so is its float32 quotient: not overloaded


def test_edge_ratios_are_what_the_edge_cases_say():
    """The float32 facts the edge-value registry is built on."""
    q = lambda a, b: F32(F32(a) / F32(b))   # noqa: E731  __fdiv_rn(__int2float_rn(a), __int2float_rn(b))
    assert q(9, 10) == q(90, 100) == F32(0.9)
    assert RATIO_ROUNDS_UP[0] / RATIO_ROUNDS_UP[1] < 0.9 and q(*RATIO_ROUNDS_UP) == F32(0.9)
    assert RATIO_BELOW[0] / RATIO_BELOW[1] < 0.9 and q(*RATIO_BELOW) < F32(0.9)
    assert F32(SUB_KEPT) / F32(100) > 0 and F32(SUB_LOST) / F32(100) == 0
    assert F32(2**31 - 1) == F32(2**31 - 2) and F32(2**24 + 1) == F32(2**24)
    assert F32(89.99999) < F32(90.0)


EDGE_F = (SUB_LOST, SUB_KEPT, -0.0, 0.0, -5.0, -np.inf, np.inf, 89.99999, 90.0, 50.0)
EDGE_ACTIVE = (0, 1, 2**31 - 1, 2**31 - 2, 2**24, 2**24 + 1, -3, -2**31)
EDGE_MAX = (0, -5, 4, 10, 100)


def edge_registry():
    """Small pools whose pick is decided by one edge each (each row: worker loads as (active, max, cpu, gpu)), and a pool
    of every combination of edge values.  Pool order and worker_id order agree, so the first worker of a pool has the
    lowest rank and wins ties."""
    pools = {
        "sub-kept": [(0, 0, SUB_KEPT, 0.0), (0, 0, 0.0, 0.0)],            # 1e-42 > 0: decided by a subnormal
        "sub-lost": [(0, 0, SUB_LOST, 0.0), (0, 0, 0.0, 0.0)],            # 1e-45 / 100 == 0: a tie
        "sub-gpu": [(0, 0, 0.0, SUB_KEPT), (0, 0, 0.0, -0.0)],
        "signed-zero": [(0, 0, 0.0, -0.0), (0, 0, -0.0, 0.0)],
        "negative": [(0, 0, -5.0, 0.0), (0, 0, 0.0, -5.0), (0, 0, 0.0, 0.0)],
        "infinite": [(0, 0, -np.inf, 0.0), (0, 0, 0.0, np.inf), (0, 0, np.inf, -np.inf), (-2**31, 0, 0.0, 0.0)],
        "cpu-cut": [(0, 0, 90.0, 0.0), (0, 0, 89.99999, 0.0), (0, 0, 0.0, 90.0)],
        "ratio-9-10": [(9, 10, 0.0, 0.0)],
        "ratio-90-100": [(90, 100, 0.0, 0.0)],
        "ratio-up": [(RATIO_ROUNDS_UP[0], RATIO_ROUNDS_UP[1], 0.0, 0.0)],
        "ratio-below": [(RATIO_BELOW[0], RATIO_BELOW[1], 0.0, 0.0)],
        "ratio-mix": [(9, 10, 0.0, 0.0), (90, 100, 0.0, 0.0), (RATIO_ROUNDS_UP[0], RATIO_ROUNDS_UP[1], 0.0, 0.0),
                      (RATIO_BELOW[0], RATIO_BELOW[1], 0.0, 0.0), (RATIO_BELOW[0] + 1, RATIO_BELOW[1], 0.0, 0.0)],
        "big-active": [(2**31 - 1, 0, 0.0, 0.0), (2**31 - 2, 0, 0.0, 0.0)],   # equal as float32: a tie
        "above-2^24": [(2**24 + 1, 0, 0.0, 0.0), (2**24, 0, 0.0, 0.0), (2**24 + 2, 0, 0.0, 0.0)],
        "negative-active": [(-3, 4, 0.0, 0.0), (-3, -5, 0.0, 0.0), (0, -5, 0.0, 0.0), (-2**31, 10, 0.0, 0.0)],
        "max-not-positive": [(5, 0, 0.0, 0.0), (5, -5, 0.0, 0.0), (1, 0, 10.0, 0.0)],
    }
    rng = random.Random(5)
    pools["every-edge"] = [(rng.choice(EDGE_ACTIVE), rng.choice(EDGE_MAX), rng.choice(EDGE_F), rng.choice(EDGE_F)) for _ in range(200)]
    rows, workers = [], []
    for p, ws in pools.items():
        for i, r in enumerate(ws):
            workers.append(kats.hb("%s-%03d" % (p, i), p, labels={"zone": "a", "tier": "x"}))
            rows.append(r)
    routing = {"topics": {"job.%s" % p: [p] for p in pools}, "pools": {p: {} for p in pools}}
    routing["topics"]["job.all"] = list(pools)
    jobs = []
    for p, ws in pools.items():
        for labels in ({}, {"zone": "a"}, {"zone": "a", "tier": "x"}):
            jobs.append({"topic": "job.%s" % p, "labels": labels})
        for i in range(min(len(ws), 6)):
            jobs.append({"topic": "job.%s" % p, "labels": {"preferred_worker_id": "%s-%03d" % (p, i)}})
    jobs += [{"topic": "job.all", "labels": lab} for lab in ({}, {"zone": "a"}, {"zone": "a", "tier": "x"})]
    return list(pools), workers, routing, np.array(rows, dtype=wire.LOAD_DTYPE), jobs


def edge_loads(base, pool_of, epoch):
    """Epoch 0 is `base`; later epochs reverse the order of the workers' rows inside every pool on odd epochs (so a pick
    moves to the other worker) and re-draw the every-edge pool."""
    t = base.copy()
    if epoch % 2:
        for p in set(pool_of):
            idx = np.nonzero(pool_of == p)[0]
            t[idx] = base[idx[::-1]]
    rng = random.Random(epoch)
    for i in np.nonzero(pool_of == "every-edge")[0]:
        t[i] = (rng.choice(EDGE_ACTIVE), rng.choice(EDGE_MAX), rng.choice(EDGE_F), rng.choice(EDGE_F))
    return t


@pytest.mark.parametrize("lbest", ["0", "1"])
def test_edge_load_values_through_every_load_path(eng, lbest, monkeypatch):
    monkeypatch.setenv("CORDUM_LBEST", lbest)
    pools, workers, routing, base, jobs = edge_registry()
    n = len(workers)
    pool_of = np.array([w["pool"] for w in workers])
    table = edge_loads(base, pool_of, 0)
    for w, row in zip(workers, table):
        w.update(active_jobs=int(row["active_jobs"]), max_parallel_jobs=int(row["max_parallel_jobs"]),
                 cpu_load=float(row["cpu_load"]), gpu_utilization=float(row["gpu_utilization"]))
    load(eng, None, routing, workers)
    o = oracle_lib.Oracle(None, routing, workers)
    assert np.array_equal(wire.WorkerTable.from_workers(workers).loads().view(np.uint8), table.view(np.uint8))
    label_free = np.array(["labels" not in j or not j["labels"] for j in jobs])
    topic_of = np.array([j["topic"] for j in jobs])
    host, keep = table.copy(), []
    b = eng.batch(len(jobs))
    b.encode(jobs).dispatch()                            # resident, for the tick
    decided_by_subnormal = 0
    for epoch, path in enumerate(("load_workers",) + LOAD_PATHS):
        table = edge_loads(base, pool_of, epoch)
        o.update_workers(np.arange(n, dtype=np.uint32), table)
        what = "lbest %s, epoch %d via %s" % (lbest, epoch, path)
        if path == "tick":
            deliver(eng, path, table, host, keep, batch=b)
            got = b.fetch().copy()
            assert_same(got, o.eval(jobs), what, jobs)
            assert_same(b.dispatch(wire.MODE_ROUTE_ONLY), o.eval(jobs, wire.MODE_ROUTE_ONLY), what + ", then a plain dispatch", jobs)
        else:
            if path != "load_workers":
                deliver(eng, path, table, host, keep)
            got = compare(eng, o, jobs, what, (wire.MODE_POLICY_AND_ROUTE, wire.MODE_ROUTE_ONLY))[wire.MODE_POLICY_AND_ROUTE]
        # the pool whose two workers differ only by 1e-42: the pick is the one without it, and it is no tie
        sub = np.nonzero((topic_of == "job.sub-kept") & label_free)[0][0]
        zero = int(np.nonzero((pool_of == "sub-kept") & (table["cpu_load"] == 0))[0][0])
        if got["route_status"][sub] == wire.ROUTE_OK and got["worker_slot"][sub] == zero and not got["flags"][sub] & wire.F_TIE:
            decided_by_subnormal += 1
        lost = np.nonzero((topic_of == "job.sub-lost") & label_free)[0][0]
        assert got["flags"][lost] & wire.F_TIE, what
        for p in ("ratio-9-10", "ratio-90-100", "ratio-up"):
            assert got["route_status"][np.nonzero(topic_of == "job.%s" % p)[0][0]] == wire.ROUTE_POOL_OVERLOADED, (what, p)
        assert got["route_status"][np.nonzero(topic_of == "job.ratio-below")[0][0]] == wire.ROUTE_OK, what
        assert got["flags"][np.nonzero((topic_of == "job.big-active") & label_free)[0][0]] & wire.F_TIE, what
    b.free()
    o.close()
    assert decided_by_subnormal == len(LOAD_PATHS) + 1


# ------------------------------------------------------------------ refused heartbeat deltas
def test_refused_delta_applies_nothing(eng):
    """A refused cordum_workers_update leaves no row behind: the next accepted delta uploads its own rows only, and the
    kernels route as an oracle that never saw the refused call."""
    from cordum_b200.engine import CordumError

    routing = {"topics": {"job.a": ["p"]}, "pools": {"p": {}}}
    workers = [kats.hb("w0", "p", 2, 10.0, 0.0, 4), kats.hb("w1", "p", 2, 20.0, 0.0, 4), kats.hb("w2", "p", 3, 30.0, 0.0, 4)]
    jobs = [{"topic": "job.a"}, {"topic": "job.a", "labels": {"preferred_worker_id": "w1"}},
            {"topic": "job.a", "labels": {"zone": ""}}]
    load(eng, None, routing, workers)
    o = oracle_lib.Oracle(None, routing, workers)
    compare(eng, o, jobs, "before")
    # had they been applied, w0 would be the least loaded and w1 overloaded
    refused = np.array([(0, 4, 0.0, 0.0), (0, 0, 95.0, float("nan"))], dtype=wire.LOAD_DTYPE)
    with pytest.raises(CordumError, match="NaN"):
        eng.update_workers(np.array([0, 1], np.uint32), refused)
    with pytest.raises(CordumError, match="out of range"):
        eng.update_workers(np.array([0, 1, 3], np.uint32), np.array([(0, 4, 0.0, 0.0), (0, 0, 95.0, 0.0), (0, 0, 0.0, 0.0)], wire.LOAD_DTYPE))
    accepted = np.array([(0, 4, 5.0, 0.0)], dtype=wire.LOAD_DTYPE)
    eng.update_workers(np.array([2], np.uint32), accepted)
    o.update_workers(np.array([2], np.uint32), accepted)
    got = compare(eng, o, jobs, "after the refused and the accepted delta")
    assert got[wire.MODE_POLICY_AND_ROUTE]["worker_slot"][0] == 2
    assert got[wire.MODE_POLICY_AND_ROUTE]["route_status"][1] == wire.ROUTE_OK_PREFERRED
    o.close()


# ------------------------------------------------------------------ grid shapes and template instances
GRID_CHILD = r"""
import os, sys
import numpy as np
import oracle_lib
from cordum_b200 import engine, synth, wire

FIELDS = ("decision", "sched_decision", "flags", "route_status", "reason_code", "rule_idx", "worker_slot")
cfg = synth.make_config("c2", 300_000)
e = engine.Engine(device=0)
e.load_policy(cfg.policy, "grid")
e.load_routing(cfg.routing)
e.load_workers(cfg.workers)
o = oracle_lib.Oracle(cfg.policy, cfg.routing, cfg.workers)
b = e.batch(cfg.jobs.n_jobs)
b.encode(cfg.jobs)
bad = 0
for mode in (wire.MODE_POLICY_AND_ROUTE, wire.MODE_POLICY_ONLY, wire.MODE_ROUTE_ONLY):
    got = b.dispatch(mode).copy()
    want = o.eval(cfg.jobs, mode, threads=max(1, len(os.sched_getaffinity(0))))
    for f in FIELDS:
        d = np.nonzero(got[f] != want[f])[0]
        if len(d):
            bad += 1
            print("mode %d field %s differs at %d jobs, first %s: kernels %s oracle %s" % (
                mode, f, len(d), d[:8].tolist(), got[f][d[:8]].tolist(), want[f][d[:8]].tolist()))
    print("mode %d: %d records compared" % (mode, len(got)))
b.free()
e.close()
sys.exit(1 if bad else 0)
"""


@pytest.mark.slow
@pytest.mark.parametrize("minb,route_minb", [(3, 5), (5, 3), (6, 5)])
def test_multi_tile_grids_and_kernel_instances(minb, route_minb):
    """CORDUM_WAVES=1 caps the persistent grids at one wave of resident CTAs: c2 at 300,000 jobs is 9,375 tiles, so on an
    H100's 132 SMs every warp of policy_kernel<3|5|6> / route_kernel<false, 3|5> loops over two or three tiles (mbarrier
    parity flips, prefetch of the partial last tile).  The knobs are read once per process: one child process each."""
    env = dict(os.environ, CORDUM_WAVES="1", CORDUM_MINB=str(minb), CORDUM_ROUTE_MINB=str(route_minb),
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests")] + ([os.environ["PYTHONPATH"]] if os.environ.get("PYTHONPATH") else [])))
    r = subprocess.run([sys.executable, "-c", GRID_CHILD], cwd=ROOT, env=env, capture_output=True, text=True, timeout=900)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, "MINB=%d ROUTE_MINB=%d: exit %d\n%s\n%s" % (minb, route_minb, r.returncode, r.stdout, r.stderr)
    assert r.stdout.count("records compared") == 3


def test_device_encoder_kept_batches(eng):
    """The device-encode half of this module means something only if batches completed on the device: a batch that falls
    back is re-encoded by the host encoder, and its records then say nothing about encode.cu.  Runs after the other tests
    of its encoder (the module fixture groups them)."""
    if eng.device_encodes is None:
        pytest.skip("host encoder")
    if eng.device_encodes["tried"] == 0:
        pytest.skip("no device-encoded batch ran in this session")
    print("device-encoded batches: %d of %d completed on the device" % (eng.device_encodes["kept"], eng.device_encodes["tried"]))
    assert eng.device_encodes["kept"] > 0
