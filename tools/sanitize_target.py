"""Small end-to-end run of every kernel for compute-sanitizer (tools/sanitize.sh): policy_kernel, route_kernel (label
picks, multi-chunk and unsorted pools), worker_chunk / worker_merge, the device encoder, heartbeat ingest, scheduler ticks,
the wide-mask path, the dispatch plan kernels, the batch subset and merge kernels, the topic count kernels and the response kernels.  Checks the
results against the oracle (the plan against a numpy grouping of the records, a subset against its source's records, a
merge against a host encode of both sources' envelopes and their records, the topic counts against the records grouped
by trimmed topic), so a sanitizer-clean run is also a correct one."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import kats  # noqa: E402
import oracle_lib  # noqa: E402
from cordum_b200 import engine, synth, wire  # noqa: E402

FIELDS = ("decision", "sched_decision", "flags", "route_status", "reason_code", "rule_idx", "worker_slot")


def same(got, want, what):
    for f in FIELDS:
        assert np.array_equal(got[f], want[f]), (what, f)
    print("ok:", what, flush=True)


def plan_same(b, rec, n_slots, what):
    st = rec["route_status"].astype(np.int64)
    routed = (st == wire.ROUTE_OK) | (st == wire.ROUTE_OK_PREFERRED)
    key = np.where(routed, rec["worker_slot"].astype(np.int64),
                   np.where(st == wire.ROUTE_NOT_ATTEMPTED, n_slots + rec["sched_decision"].astype(np.int64),
                            n_slots + 6 + st - wire.ROUTE_MISSING_TOPIC))
    offsets, jobs, ns = b.plan()
    want = np.concatenate([[0], np.cumsum(np.bincount(key, minlength=n_slots + wire.PLAN_OUTCOMES))])
    assert ns == n_slots and np.array_equal(offsets, want) and np.array_equal(jobs, np.argsort(key, kind="stable")), what
    print("ok: plan,", what, flush=True)


def counts_same(b, rec, topics, what):
    """Batch.topic_counts() against the records' plan outcome columns grouped by TrimSpace(raw topic)."""
    st = rec["route_status"].astype(np.int64)
    col = np.where((st == wire.ROUTE_OK) | (st == wire.ROUTE_OK_PREFERRED), wire.COUNT_ROUTED,
                   np.where(st == wire.ROUTE_NOT_ATTEMPTED, rec["sched_decision"].astype(np.int64), 6 + st - wire.ROUTE_MISSING_TOPIC))
    lab = [oracle_lib.trim_space(t) for t in topics]
    names = sorted(set(lab))
    row = {x: i for i, x in enumerate(names)}
    want = np.zeros((len(names), wire.COUNT_COLUMNS), np.uint32)
    np.add.at(want, (np.array([row[x] for x in lab], np.int64), col), 1)
    labels, counts = b.topic_counts()
    assert labels == names and np.array_equal(counts, want), what
    print("ok: topic counts,", what, flush=True)


def topics_of(env):
    t = env.cols["topic"][:env.n_jobs]
    return [bytes(env.arena[int(o):int(o) + int(n)]) for o, n in zip(t["off"], t["len"])]


def responses_same(b, rec, what):
    """Batch.responses(): every job once, jobs ascending inside a class, classes by first job, each class one key of the
    records (masked flags, reason code, rule index) and each job's reason the library's per-job one."""
    resp = b.responses()
    off, jobs, cls = resp["offsets"].astype(np.int64), resp["jobs"].astype(np.int64), resp["classes"]
    assert off[-1] == len(rec) and np.array_equal(np.sort(jobs), np.arange(len(rec))), what
    assert (np.diff(cls["first_job"].astype(np.int64)) > 0).all(), what
    for c in range(len(cls)):
        m = jobs[off[c]:off[c + 1]]
        assert m[0] == cls["first_job"][c] and (np.diff(m) > 0).all(), what
        r = rec[m]
        assert (r["reason_code"] == cls["reason_code"][c]).all() and (r["rule_idx"] == cls["rule_idx"][c]).all(), what
        assert ((r["flags"] & wire.CLASS_FLAG_MASK) == (cls["flags"][c] & wire.CLASS_FLAG_MASK)).all(), what
    print("ok: responses,", what, len(cls), "classes", flush=True)


def subset_same(b, dst, rec, what):
    """A subset by outcome and one by list (across a tile edge), dispatched: each job decides as its source job did."""
    st = rec["route_status"]
    for kw in ({"outcomes": (1 << wire.PLAN_OUTCOMES) - 1}, {"jobs": np.arange(1, len(rec), 3)}):
        m = b.subset(dst, **kw)
        parent = dst.parent_index().copy()
        if "jobs" in kw:
            assert np.array_equal(parent, kw["jobs"]), what
        else:
            assert np.array_equal(parent, np.flatnonzero((st != wire.ROUTE_OK) & (st != wire.ROUTE_OK_PREFERRED))), what
        same(dst.dispatch().copy()[:m], rec[parent], "subset (%s), %s" % (sorted(kw)[0], what))


def merge_same(e, b, env, what):
    """b merged with a host encode of its first third, then with itself: records, selective list and wide rows equal a host
    encode of both envelope lists, and each job decides as it did in its source."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_batch_subset as tbs

    env = env if isinstance(env, wire.EnvelopeBatch) else wire.EnvelopeBatch.from_jobs(env)
    n = env.n_jobs
    k = max(1, n // 3)
    part, dst = e.batch(k), e.batch(2 * n)
    part.encode(env.slice(0, k)).dispatch()
    for other, idx in ((part, np.arange(k)), (b, np.arange(n))):
        assert b.merge(other, dst) == n + len(idx), what
        job, route, slot = dst.records()
        hjob, hroute, hslot, hsel, hwide = tbs.host_records_of(e, tbs.take(env, np.concatenate([np.arange(n), idx])))
        assert job.tobytes() == hjob.tobytes() and route.tobytes() == hroute.tobytes() and np.array_equal(slot, hslot), what
        assert np.array_equal(tbs.side(dst, 0), hsel) and np.array_equal(tbs.side(dst, 1), hwide), what
        same(dst.dispatch().copy(), np.concatenate([b.results().copy(), other.results().copy()]), "merge, %s" % what)
    part.free()
    dst.free()


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 3000
    light = len(sys.argv) > 2 and sys.argv[2] == "light"   # racecheck serialises everything: smaller pools, fewer phases
    cfg = synth.make_config("c2", n)                      # 256 rules, 1k workers
    e = engine.Engine(device=0)
    e.load_policy(cfg.policy, "san")
    e.load_routing(cfg.routing)
    e.load_workers(cfg.workers)
    o = oracle_lib.Oracle(cfg.policy, cfg.routing, cfg.workers)
    b = e.batch(n)
    for mode in (wire.MODE_POLICY_AND_ROUTE, wire.MODE_POLICY_ONLY, wire.MODE_ROUTE_ONLY):
        rec = b.encode(cfg.jobs).dispatch(mode)
        same(rec, o.eval(cfg.jobs, mode), "c2 host-encode mode %d" % mode)
        plan_same(b, rec, cfg.workers.n_workers, "c2 mode %d" % mode)   # 1,012 buckets: two radix passes
        counts_same(b, rec, topics_of(cfg.jobs), "c2 mode %d" % mode)
    same(b.encode_device(cfg.jobs).dispatch(), o.eval(cfg.jobs), "c2 device-encode")
    # heartbeat deltas + refresh
    rng = np.random.default_rng(3)
    slots = rng.choice(cfg.workers.n_workers, 200, replace=False).astype(np.uint32)
    loads = np.zeros(200, wire.LOAD_DTYPE)
    loads["active_jobs"] = rng.integers(0, 4, 200)
    loads["max_parallel_jobs"] = 4
    loads["cpu_load"] = rng.integers(0, 95, 200)
    e.update_workers(slots, loads)
    o.update_workers(slots, loads)
    same(b.encode(cfg.jobs).dispatch(), o.eval(cfg.jobs), "after heartbeat deltas")
    dst = e.batch(n)
    subset_same(b, dst, b.results().copy(), "c2")
    merge_same(e, b, cfg.jobs, "c2")
    # one big pool: multi-chunk merge (1300) and beyond the sort buffer (9000)
    for size in ((1300,) if light else (1300, 9000)):
        routing = {"topics": {"job.w.go": ["big"]}, "pools": {"big": {}}}
        workers = [kats.hb("m%05d" % i, "big", i % 3, float(i % 40), float(i % 7), 4, {"zone": "z%d" % (i % 4), "host": "m%05d" % (i % 97)}) for i in range(size)]
        e.load_routing(routing)
        e.load_workers(workers)
        o2 = oracle_lib.Oracle(cfg.policy, routing, workers)
        jobs = [{"topic": "job.w.go", "labels": {"zone": "z%d" % (i % 4)}} for i in range(64)] + \
               [{"topic": "job.w.go", "labels": {"host": "m%05d" % (i % 97), "zone": "z%d" % (i % 4)}} for i in range(64)] + [{"topic": "job.w.go"}] * 8
        same(b.encode(jobs).dispatch(wire.MODE_ROUTE_ONLY), o2.eval(jobs, wire.MODE_ROUTE_ONLY), "pool of %d workers" % size)
        plan_same(b, b.results(), size, "pool of %d workers" % size)
        responses_same(b, b.results(), "pool of %d workers" % size)
        o2.close()
    # wide masks
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import test_wide_masks as tw

    policy, routing, workers, jobs = tw.build(70 if light else 130)
    e.load_policy(policy, "wide")
    e.load_routing(routing)
    e.load_workers(workers)
    o3 = oracle_lib.Oracle(policy, routing, workers)
    bw = e.batch(len(jobs))
    same(bw.encode(jobs).dispatch(), o3.eval(jobs), "wide masks")
    responses_same(bw, bw.results(), "wide masks")
    subset_same(bw, e.batch(len(jobs)), bw.results().copy(), "wide masks")
    merge_same(e, bw, jobs, "wide masks")
    o3.close()
    # selective placement pairs: the subset re-packs the selective list and its extra words
    import test_selective_differential as tsd

    policy, routing, workers = tsd.pins_registry()
    jobs = tsd.pins_jobs(workers)[: 300 if light else None]
    e.load_policy(policy, "pins")
    e.load_routing(routing)
    e.load_workers(workers)
    bs = e.batch(len(jobs))
    subset_same(bs, e.batch(len(jobs)), bs.encode(jobs).dispatch().copy(), "selective pairs")
    merge_same(e, bs, jobs, "selective pairs")
    # scheduler ticks on the c2 tables
    e.load_policy(cfg.policy, "san2")
    e.load_routing(cfg.routing)
    e.load_workers(cfg.workers)
    o4 = oracle_lib.Oracle(cfg.policy, cfg.routing, cfg.workers)
    b1, b2 = e.batch(n), e.batch(n)
    b1.encode(cfg.jobs).dispatch()
    b2.encode_device(cfg.jobs).dispatch()
    W = cfg.workers.n_workers
    keep = []
    for t in range(4):
        loads = cfg.workers.loads()
        loads["active_jobs"] = rng.integers(0, 9, W)
        loads["cpu_load"] = (rng.random(W) * 100).astype(np.float32)
        keep.append(loads)
        (b1 if t % 2 == 0 else b2).tick(loads.ctypes.data, 0, W)
    b2.wait()                                  # routed by the flush, on the loads of the last tick
    o4.update_workers(np.arange(W, dtype=np.uint32), keep[3])
    same(b2.fetch(), o4.eval(cfg.jobs), "ticks")
    plan_same(b2, b2.results(), W, "ticks")
    responses_same(b2, b2.results(), "ticks")
    o4.close()
    o.close()
    print("sanitize target done", flush=True)


if __name__ == "__main__":
    main()
