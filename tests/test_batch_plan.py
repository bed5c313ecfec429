"""cordum_batch_plan against a numpy grouping of the batch's own decision records: the jobs of a dispatched batch grouped by
destination worker slot (buckets 0 .. n_slots-1) and then by outcome (bucket n_slots + k), stable inside a bucket.  Every
dispatch path (blocking, async, resident, ticks), a device encode that fell back to the host encoder, tile and pass
boundaries, one bucket and all-distinct buckets, a 1-slot, a 60,000-hostname and a 70,000-worker registry, a reload between
the dispatch and the plan, the call order and the exact launch count."""
import numpy as np
import pytest

import kats
from cordum_b200 import synth, wire

pytestmark = pytest.mark.gpu

MODES = (wire.MODE_POLICY_ONLY, wire.MODE_POLICY_AND_ROUTE, wire.MODE_ROUTE_ONLY)
TILE = 2048           # jobs per CTA of the plan's count / scatter kernels (csrc/kernels.h CORDUM_PLAN_TILE)
E_STATE = -4


def expected(rec, n_slots):
    """numpy reference: bucket key per job, then a stable sort and per-bucket counts."""
    st = rec["route_status"].astype(np.int64)
    routed = (st == wire.ROUTE_OK) | (st == wire.ROUTE_OK_PREFERRED)
    key = np.where(routed, rec["worker_slot"].astype(np.int64),
                   np.where(st == wire.ROUTE_NOT_ATTEMPTED, n_slots + rec["sched_decision"].astype(np.int64),
                            n_slots + 6 + st - wire.ROUTE_MISSING_TOPIC))
    nb = n_slots + wire.PLAN_OUTCOMES
    assert len(key) == 0 or (key.min() >= 0 and key.max() < nb)
    offsets = np.zeros(nb + 1, np.int64)
    offsets[1:] = np.cumsum(np.bincount(key, minlength=nb))
    return offsets, np.argsort(key, kind="stable"), key


def launches_of_one_plan(n, n_slots):
    bits = (n_slots + wire.PLAN_OUTCOMES - 1).bit_length()
    return 0 if n == 0 else 3 * max(1, -(-bits // 8)) + 1


def check_plan(eng, b, rec, n_slots, what):
    before = eng.launch_count()
    offsets, jobs, ns = b.plan()
    assert eng.launch_count() - before == launches_of_one_plan(len(rec), n_slots), what
    assert ns == n_slots, (what, ns, n_slots)
    want_off, want_jobs, key = expected(rec, n_slots)
    assert np.array_equal(offsets, want_off), what
    assert np.array_equal(jobs, want_jobs), what
    # the iterator visits exactly the non-empty buckets
    seen = 0
    for bucket, members in b.plan_buckets(offsets, jobs):
        assert len(members) and (key[members] == bucket).all(), (what, bucket)
        seen += len(members)
    assert seen == len(rec)
    return offsets, jobs


def refused_before_wait(b):
    from cordum_b200 import engine

    with pytest.raises(engine.CordumError) as ei:
        b.plan()
    assert ei.value.code == E_STATE


@pytest.fixture(scope="module")
def eng():
    from cordum_b200 import engine

    e = engine.Engine(device=0)
    yield e
    e.close()


def load(eng, policy, routing, workers):
    eng.load_policy(policy, "plan")
    eng.load_routing(routing)
    eng.load_workers(workers)


def config(name):
    if name == "c5":
        c5 = kats.golden("c5_demo_guardrails.json")
        jobs, workers, _ = synth.make_c5(20_000)
        return c5["policy"], c5["routing"], workers, jobs
    cfg = synth.make_config(name)
    return cfg.policy, cfg.routing, cfg.workers, cfg.jobs


@pytest.mark.parametrize("name", ["tiny", "c2", "c5"])
def test_every_dispatch_path(eng, name):
    policy, routing, workers, jobs = config(name)
    load(eng, policy, routing, workers)
    W = workers.n_workers
    b = eng.batch(jobs.n_jobs)
    b.encode(jobs)
    refused_before_wait(b)                               # encoded, never dispatched
    outcomes = set()
    for mode in MODES:
        rec = b.dispatch(mode).copy()
        check_plan(eng, b, rec, W, "%s blocking mode %d" % (name, mode))
        b.dispatch_async(mode)
        refused_before_wait(b)
        check_plan(eng, b, b.wait().copy(), W, "%s async mode %d" % (name, mode))
        b.dispatch_resident_async(mode)
        refused_before_wait(b)
        b.wait()
        check_plan(eng, b, b.fetch().copy(), W, "%s resident mode %d" % (name, mode))
        outcomes |= set(expected(rec, W)[2][rec["route_status"] != wire.ROUTE_OK].tolist())
    assert len(outcomes) >= 3, outcomes
    # ticks: the first batch is routed by the second tick, the second by the flush
    c = eng.batch(jobs.n_jobs)
    c.encode(jobs).dispatch()
    loads = workers.loads()
    b.tick(loads.ctypes.data, 0, W)
    refused_before_wait(b)
    c.tick(loads.ctypes.data, 0, W)
    b.wait()
    check_plan(eng, b, b.fetch().copy(), W, "%s tick" % name)
    refused_before_wait(c)
    eng.tick_flush()
    c.wait()
    check_plan(eng, c, c.fetch().copy(), W, "%s tick flush" % name)
    # a new encode invalidates the plan until the batch is dispatched again
    b.encode(jobs)
    refused_before_wait(b)
    b.free()
    c.free()


def test_device_encode_that_falls_back_to_the_host(eng):
    cfg = synth.make_config("tiny")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    jobs = [{"topic": "job.first.sight.%d" % (i % 3)} if i % 5 == 0 else {"topic": "job.pack000.read", "labels": {"zone": "z%d" % (i % 4)}}
            for i in range(3000)]
    b = eng.batch(len(jobs))
    before = eng.host_fallbacks()
    b.encode_device(jobs)
    b.dispatch_async()
    refused_before_wait(b)
    rec = b.wait().copy()
    assert eng.host_fallbacks() == before + 1
    check_plan(eng, b, rec, cfg.workers.n_workers, "fallback")
    b.free()


@pytest.mark.parametrize("n", [0, 1, TILE - 1, TILE, TILE + 1, 3 * TILE + 17])
def test_batch_sizes(eng, n):
    cfg = synth.make_config("c2")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    b = eng.batch(max(n, 1))
    rec = b.encode(cfg.jobs.slice(0, n)).dispatch().copy()
    offsets, jobs = check_plan(eng, b, rec, cfg.workers.n_workers, "n=%d" % n)
    assert len(jobs) == n and offsets[-1] == n
    b.free()


def test_one_slot_registry_every_job_on_one_worker(eng):
    policy = {"default_tenant": "default", "rules": [{"id": "deny-x", "decision": "deny", "match": {"topics": ["job.x"]}}]}
    routing = {"topics": {"job.a": ["p"], "job.x": ["p"]}, "pools": {"p": {}}}
    load(eng, policy, routing, [kats.hb("solo", "p")])
    n = 3 * TILE + 5
    b = eng.batch(n)
    rec = b.encode([{"topic": "job.a"}] * n).dispatch().copy()
    offsets, jobs = check_plan(eng, b, rec, 1, "one worker")
    assert offsets[1] == n and np.array_equal(jobs, np.arange(n))
    assert b.subject(int(jobs[0])) == "worker.solo.jobs"
    mixed = [[{"topic": "job.a"}, {"topic": "job.x"}, {"topic": ""}, {"topic": "job.unmapped"},
              {"topic": "job.a", "labels": {"preferred_pool": "nope"}}, {"topic": "job.a", "meta": {"requires": ["gpu"]}}][i % 6]
             for i in range(n)]
    for mode in MODES:
        rec = b.encode(mixed).dispatch(mode).copy()
        check_plan(eng, b, rec, 1, "one slot, mixed outcomes, mode %d" % mode)
    b.free()


def test_every_job_on_a_distinct_worker_three_passes(eng):
    """70,000 slots: 17-bit keys, three radix passes.  30,000 jobs, each preferring a different worker (scattered order)."""
    W, n = 70_000, 30_000
    workers = wire.WorkerTable.from_workers([kats.hb("w%06d" % i, "p", i % 3, float(i % 50), 0.0, 8) for i in range(W)])
    load(eng, None, {"topics": {"job.a": ["p"]}, "pools": {"p": {}}}, workers)
    pick = (np.arange(n) * 7919) % W
    jobs = [{"topic": "job.a", "labels": {"preferred_worker_id": "w%06d" % s}} for s in pick]
    b = eng.batch(n)
    rec = b.encode(jobs).dispatch(wire.MODE_ROUTE_ONLY).copy()
    assert (rec["route_status"] == wire.ROUTE_OK_PREFERRED).all() and np.array_equal(rec["worker_slot"], pick)
    offsets, order = check_plan(eng, b, rec, W, "distinct workers")
    assert (np.diff(offsets)[:W] <= 1).all() and np.array_equal(order, np.argsort(pick))
    b.free()


def test_hostname_registry(eng):
    import test_selective_labels as tsl

    policy, routing, workers = tsl.registry(tsl.GPU_WORKERS, tsl.GPU_POOLS, seed=5, n_second=tsl.GPU_SECOND)
    table = wire.WorkerTable.from_workers(workers)
    load(eng, policy, routing, table)
    jobs = tsl.jobs_for(workers, tsl.GPU_POOLS, 6000, seed=6, n_second=tsl.GPU_SECOND)
    b = eng.batch(len(jobs))
    for mode in MODES:
        rec = b.encode(jobs).dispatch(mode).copy()
        check_plan(eng, b, rec, tsl.GPU_WORKERS, "hostnames mode %d" % mode)
    b.free()


def test_reload_after_the_dispatch_keeps_the_batch_registry(eng):
    cfg = synth.make_config("tiny")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    b = eng.batch(cfg.jobs.n_jobs)
    rec = b.encode(cfg.jobs).dispatch().copy()
    W = cfg.workers.n_workers
    eng.load_workers([kats.hb("other-%d" % i, "pool-000") for i in range(3)])
    offsets, jobs = check_plan(eng, b, rec, W, "after a workers reload")
    slot = int(np.flatnonzero(np.diff(offsets)[:W])[0])
    job = int(jobs[offsets[slot]])
    assert b.subject(job) == "worker.%s.jobs" % cfg.workers.worker_id(slot)
    b.free()


@pytest.mark.slow
def test_config3_million_jobs(eng):
    cfg = synth.make_config("c3")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    b = eng.batch(cfg.jobs.n_jobs)
    rec = b.encode(cfg.jobs).dispatch().copy()
    check_plan(eng, b, rec, cfg.workers.n_workers, "config 3")
    b.free()
