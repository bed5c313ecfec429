"""cordum_batch_subset: a new encoded batch built on the device from part of an encoded one, selected by plan outcome or by
a job list, and dispatched without encoding again.  Against the source's own records (no load change: job i of the subset
decides exactly as source job parent[i] did), against the host encoder run on the selected envelopes (records, selective
list and wide rows bit for bit), against the C++ oracle after a heartbeat (every load source), and the refusals, tile
boundaries and launch counts."""
import numpy as np
import pytest

import kats
import oracle_lib
import test_batch_plan as tbp
import test_fuzz_three_way as f3
import test_selective_differential as tsd
import test_selective_labels as sl
from cordum_b200 import synth, wire

pytestmark = pytest.mark.gpu

FIELDS = sl.FIELDS
MODES = (wire.MODE_POLICY_ONLY, wire.MODE_POLICY_AND_ROUTE, wire.MODE_ROUTE_ONLY)
PATHS = ("blocking", "async", "resident", "tick")
TILE = 2048                  # items per CTA of the subset kernels (csrc/kernels.h CORDUM_SUBSET_TILE)
GRID_JOBS = tsd.GRID_JOBS    # listed jobs one grid of route_select_kernel covers on a 132-SM H100
E_INVALID, E_CAPACITY, E_STATE, E_STALE = -1, -2, -4, -6
SUBSET_LAUNCHES = 4


@pytest.fixture(scope="module")
def eng():
    from cordum_b200 import engine

    e = engine.Engine(device=0)
    yield e
    e.close()


@pytest.fixture(autouse=True)
def default_limits():
    sl.set_selective(sl.MIN_BITS, sl.MAX_HOLDERS)
    yield
    sl.set_selective(sl.MIN_BITS, sl.MAX_HOLDERS)


def load(eng, policy, routing, workers):
    eng.load_policy(policy, "subset")
    eng.load_routing(routing)
    eng.load_workers(workers)


def take(env, idx):
    """The envelopes of jobs idx (ascending) as a batch of their own (CSR columns re-based)."""
    idx = np.asarray(idx, dtype=np.int64)
    cols = {k: env.cols[k][idx].copy() for k in env.SCALARS + ("has_meta", "actor_type", "approved")}
    for off, vals in (("risk_off", ("risk_tags",)), ("requires_off", ("requires_",)), ("label_off", ("label_keys", "label_vals"))):
        o = env.cols[off].astype(np.int64)
        lens = o[idx + 1] - o[idx]
        new = np.zeros(len(idx) + 1, np.int64)
        np.cumsum(lens, out=new[1:])
        pick = np.repeat(o[idx] - new[:-1], lens) + np.arange(new[-1])
        cols[off] = new.astype(np.uint32)
        for v in vals:
            part = env.cols[v][pick].copy()
            cols[v] = part if len(part) else np.zeros(1, dtype=wire.STR_DTYPE)
    return wire.EnvelopeBatch(len(idx), env.arena, cols)


def outcome(rec):
    """Plan outcome bucket per job (-1: routed)."""
    st = rec["route_status"].astype(np.int64)
    return np.where((st == wire.ROUTE_OK) | (st == wire.ROUTE_OK_PREFERRED), -1,
                    np.where(st == wire.ROUTE_NOT_ATTEMPTED, rec["sched_decision"].astype(np.int64), 6 + st - wire.ROUTE_MISSING_TOPIC))


def selected_by(rec, mask):
    k = outcome(rec)
    return np.flatnonzero((k >= 0) & ((mask >> np.maximum(k, 0)) & 1).astype(bool))


def same(got, want, what):
    assert len(got) == len(want), (what, len(got), len(want))
    for f in FIELDS:
        bad = np.flatnonzero(got[f] != want[f])
        assert len(bad) == 0, (what, f, bad[:5], got[f][bad[:5]], want[f][bad[:5]])


def run(eng, b, mode, path, loads=None):
    """Dispatch b by one of the four paths; returns its records."""
    if path == "blocking":
        return b.dispatch(mode).copy()
    if path == "async":
        b.dispatch_async(mode)
        return b.wait().copy()
    if path == "resident":
        b.dispatch_resident_async(mode)
        b.wait()
        return b.fetch().copy()
    assert mode == wire.MODE_POLICY_AND_ROUTE
    b.tick(loads.ctypes.data, 0, len(loads))
    eng.tick_flush()
    b.wait()
    return b.fetch().copy()


def side(b, which):
    """The batch's selective list (which = 0, uint32 words) or wide rows (1, uint64 words) as the kernels read them."""
    L = b.L
    n = L.cordum_test_batch_side(b.h, which, None, 0)
    assert n >= 0
    out = np.zeros(max(n, 8), np.uint8)
    assert L.cordum_test_batch_side(b.h, which, out.ctypes.data, n) == n
    return out[:n].view(np.uint32 if which == 0 else np.uint64)


def subset_checked(eng, src, dst, src_rec, outcomes=None, jobs=None):
    """src.subset(...) with its launch count and parent index checked; returns the parent index (a copy)."""
    before = eng.launch_count()
    m = src.subset(dst, outcomes=outcomes, jobs=jobs)
    assert eng.launch_count() - before == (SUBSET_LAUNCHES if src.size else 0)
    want = selected_by(src_rec, outcomes) if jobs is None else np.asarray(jobs, np.int64)
    parent = dst.parent_index().copy()
    assert m == len(want) == dst.size and np.array_equal(parent, want), (m, len(want))
    return parent


def config(name):
    if name == "c5":
        c5 = kats.golden("c5_demo_guardrails.json")
        jobs, workers, _ = synth.make_c5(20_000)
        return c5["policy"], c5["routing"], workers, jobs
    if name == "fuzz":
        policy, routing, workers, jobs = f3.fuzz_case(3, 40)
        return policy, routing, wire.WorkerTable.from_workers(workers), wire.EnvelopeBatch.from_jobs(jobs * 20)
    cfg = synth.make_config(name)
    return cfg.policy, cfg.routing, cfg.workers, cfg.jobs


# ------------------------------------------------------------------ 1. identity without new loads
@pytest.mark.parametrize("encoder", ["host", "device"])
@pytest.mark.parametrize("name", ["tiny", "c2", "c5", "fuzz"])
def test_subset_decides_as_its_parent(eng, name, encoder):
    policy, routing, workers, env = config(name)
    load(eng, policy, routing, workers)
    n = env.n_jobs
    loads = workers.loads()
    src, dst = eng.batch(n), eng.batch(n)
    rng = np.random.default_rng(17)
    before = eng.host_fallbacks()
    src.encode_device(env.deinterned()) if encoder == "device" else src.encode(env)
    step = 0
    seen = set()
    for mode in MODES:
        rec = src.dispatch(mode).copy()
        if encoder == "device":
            src.wait()
        masks = [1 << k for k in sorted(set(outcome(rec).tolist()) - {-1})] + [wire.SUBSET_RETRYABLE]
        lists = [np.sort(rng.choice(n, size=int(rng.integers(1, n)), replace=False)), [int(rng.integers(n))], np.arange(n), []]
        for sel in [("mask", m) for m in masks] + [("list", x) for x in lists]:
            paths = [p for p in PATHS if p != "tick" or mode == wire.MODE_POLICY_AND_ROUTE]
            path = paths[step % len(paths)]
            step += 1
            parent = subset_checked(eng, src, dst, rec, **({"outcomes": sel[1]} if sel[0] == "mask" else {"jobs": sel[1]}))
            got = run(eng, dst, mode, path, loads)
            same(got, rec[parent], "%s %s mode %d %s %s" % (name, encoder, mode, sel[0], path))
            seen.add(path)
    assert seen == set(PATHS)
    if encoder == "device" and name != "fuzz":
        assert eng.host_fallbacks() == before
    src.free()
    dst.free()


# ------------------------------------------------------------------ 2. records against the host encoder
def host_records_of(eng, env):
    b = eng.batch(max(env.n_jobs, 1))
    b.encode(env)
    out = b.records() + (side(b, 0), side(b, 1))
    b.free()
    return out


def check_records_against_host_encode(eng, src, dst, env, parent, what):
    job, route, slot = dst.records()
    hjob, hroute, hslot, hsel, hwide = host_records_of(eng, take(env, parent))
    assert job.tobytes() == hjob.tobytes(), what
    assert route.tobytes() == hroute.tobytes(), what
    assert np.array_equal(slot, hslot), what
    assert np.array_equal(side(dst, 0), hsel), what
    assert np.array_equal(side(dst, 1), hwide), what


@pytest.mark.parametrize("registry", ["pins", "wide"])
def test_records_equal_a_host_encode_of_the_selection(eng, registry):
    if registry == "pins":
        policy, routing, workers = tsd.pins_registry()
        jobs = tsd.pins_jobs(workers)
    else:
        policy, routing, workers = tsd.wide_registry()
        jobs = tsd.wide_jobs(workers, 3000, 5)
    table = wire.WorkerTable.from_workers(workers)
    load(eng, policy, routing, table)
    env = wire.EnvelopeBatch.from_jobs(jobs)
    n = env.n_jobs
    src, dst = eng.batch(n), eng.batch(n)
    rec = src.encode(env).dispatch().copy()
    flagged = int(((src.records()[0]["flags"] & sl.JF_SELECTIVE) != 0).sum())
    assert flagged
    if registry == "pins":
        assert len(side(src, 0)) > 2 * flagged + 1       # extra words: jobs with three or more pins
    else:
        assert len(side(src, 1)) > 0                     # wide rows (xw_place > 0)
    rng = np.random.default_rng(3)
    o = oracle_lib.Oracle(policy, routing, table)
    for sel in (np.sort(rng.choice(n, n // 3, replace=False)), np.arange(0, n, 2), np.arange(n)):
        parent = subset_checked(eng, src, dst, rec, jobs=sel)
        check_records_against_host_encode(eng, src, dst, env, parent, "%s list of %d" % (registry, len(sel)))
        same(dst.dispatch().copy(), o.eval(take(env, parent)), registry)
    for mask in (wire.SUBSET_RETRYABLE, 1 << wire.PLAN_NO_WORKERS):
        parent = subset_checked(eng, src, dst, rec, outcomes=mask)
        assert len(parent)
        check_records_against_host_encode(eng, src, dst, env, parent, "%s mask %x" % (registry, mask))
        same(dst.dispatch().copy(), rec[parent], registry)
    o.close()
    src.free()
    dst.free()


def test_device_encoded_parent_records_per_job(eng):
    cfg = synth.make_config("c2")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    n = cfg.jobs.n_jobs
    src, dst = eng.batch(n), eng.batch(n)
    src.encode_device(cfg.jobs.deinterned()).wait()
    sjob, sroute, sslot = src.records()
    parent = subset_checked(eng, src, dst, None, jobs=np.arange(1, n, 3))
    job, route, slot = dst.records()
    for i in range(len(parent)):
        a, b = job[slot[i]].copy(), sjob[sslot[parent[i]]].copy()
        assert a["orig"] == i
        b["orig"] = i
        assert a.tobytes() == b.tobytes() and route[slot[i]].tobytes() == sroute[sslot[parent[i]]].tobytes(), i
    # the subset keeps the source's sorted order
    assert np.array_equal(parent[job["orig"]], sjob["orig"][np.isin(sjob["orig"], parent)])
    src.free()
    dst.free()


# ------------------------------------------------------------------ 3. retry after a heartbeat
def overloaded(workers, frac_pools):
    """Loads with the workers of some pools all overloaded (cpu 95)."""
    loads = workers.loads().copy()
    pools = np.array([w["pool"] for w in workers.to_workers()])
    hot = sorted(set(pools.tolist()))[::frac_pools]
    loads["cpu_load"][np.isin(pools, hot)] = 95.0
    return loads


@pytest.mark.parametrize("source", ["update_workers", "ingest", "set_loads_device", "tick"])
def test_retry_after_a_heartbeat(eng, source):
    cfg = synth.make_config("c2")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    W = cfg.workers.n_workers
    slots = np.arange(W, dtype=np.uint32)
    hot, cool = overloaded(cfg.workers, 2), cfg.workers.loads()
    eng.update_workers(slots, hot)
    n = cfg.jobs.n_jobs
    src, dst, dst2 = eng.batch(n), eng.batch(n), eng.batch(n)
    rec = src.encode(cfg.jobs).dispatch().copy()
    o = oracle_lib.Oracle(cfg.policy, cfg.routing, cfg.workers)
    o.update_workers(slots, hot)
    same(rec, o.eval(cfg.jobs), "hot loads")
    parent = subset_checked(eng, src, dst, rec, outcomes=wire.SUBSET_RETRYABLE)
    assert (rec["route_status"][parent] == wire.ROUTE_POOL_OVERLOADED).sum() > 0
    # a heartbeat delta does not make the source stale
    eng.update_workers(slots[:3], hot[:3])
    assert src.subset(dst, outcomes=wire.SUBSET_RETRYABLE) == len(parent)
    # the next heartbeat epoch
    if source == "update_workers":
        eng.update_workers(slots, cool)
        got = dst.dispatch().copy()
    elif source == "ingest":
        eng.ingest(cool.ctypes.data, 0, W)
        got = dst.dispatch().copy()
    elif source == "set_loads_device":
        import torch

        dev = torch.from_numpy(cool.view(np.uint8).reshape(W, 16).copy()).cuda()
        torch.cuda.synchronize()
        eng.set_loads_device(dev.data_ptr(), W, torch.cuda.current_stream().cuda_stream)
        got = dst.dispatch().copy()
    else:
        got = run(eng, dst, wire.MODE_POLICY_AND_ROUTE, "tick", cool)
    o.update_workers(slots, cool)
    sub_env = take(cfg.jobs, parent)
    want = o.eval(sub_env)
    same(got, want, "retry after %s" % source)
    assert (got["route_status"] == wire.ROUTE_OK).sum() > (rec["route_status"][parent] == wire.ROUTE_OK).sum()
    offsets, jobs, ns = dst.plan()
    want_off, want_jobs, _ = tbp.expected(got, W)
    assert ns == W and np.array_equal(offsets, want_off) and np.array_equal(jobs, want_jobs)
    # a subset of the subset composes through both parent maps
    pick = np.arange(0, len(parent), 3)
    p2 = subset_checked(eng, dst, dst2, got, jobs=pick)
    same(dst2.dispatch().copy(), want[p2], "subset of a subset")
    check_records_against_host_encode(eng, src, dst2, cfg.jobs, parent[p2], "subset of a subset, records")
    same(o.eval(take(cfg.jobs, parent[p2])), dst2.results(), "composed parents")
    o.close()
    for b in (src, dst, dst2):
        b.free()


@pytest.mark.parametrize("then", ["re-encode", "free"])
def test_subset_outlives_its_source(eng, then):
    """dst keeps no pointer to src: after src is encoded with other jobs, or freed, dst dispatches as before, on every path,
    and its selective list and wide rows are its own."""
    policy, routing, workers = tsd.wide_registry()
    table = wire.WorkerTable.from_workers(workers)
    load(eng, policy, routing, table)
    env = wire.EnvelopeBatch.from_jobs(tsd.wide_jobs(workers, 3000, 7))
    other = wire.EnvelopeBatch.from_jobs(tsd.wide_jobs(workers, 3000, 8))
    n = env.n_jobs
    src, dst = eng.batch(n), eng.batch(n)
    rec = src.encode(env).dispatch().copy()
    parent = subset_checked(eng, src, dst, rec, jobs=np.arange(0, n, 2))
    sel, wide = side(dst, 0), side(dst, 1)
    assert len(sel) and len(wide)
    if then == "re-encode":
        src.encode(other).dispatch()
    else:
        src.free()
    for path in PATHS:
        same(run(eng, dst, wire.MODE_POLICY_AND_ROUTE, path, table.loads()), rec[parent], "after src %s, %s" % (then, path))
    assert np.array_equal(side(dst, 0), sel) and np.array_equal(side(dst, 1), wide)
    assert np.array_equal(dst.parent_index(), parent)
    check_records_against_host_encode(eng, None, dst, env, parent, "after src %s" % then)
    if then == "re-encode":
        src.free()
    dst.free()


# ------------------------------------------------------------------ 4. boundaries
@pytest.mark.parametrize("n", [1, TILE - 1, TILE, TILE + 1, 3 * TILE + 17])
def test_tile_boundaries(eng, n):
    cfg = synth.make_config("c2")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    env = cfg.jobs.slice(0, n)
    src, dst = eng.batch(n), eng.batch(n)
    rec = src.encode(env).dispatch().copy()
    rng = np.random.default_rng(n)
    sizes = sorted({s for s in (0, 1, TILE - 1, TILE, TILE + 1, 2 * TILE, n - 1, n) if 0 <= s <= n})
    for m in sizes:
        sel = np.sort(rng.choice(n, m, replace=False))
        parent = subset_checked(eng, src, dst, rec, jobs=sel)
        same(dst.dispatch().copy(), rec[parent], "n=%d m=%d" % (n, m))
    # a run that ends exactly at a tile edge, and one that starts there
    for sel in (np.arange(max(0, TILE - 5), min(n, TILE)), np.arange(min(n, TILE), min(n, TILE + 5))):
        parent = subset_checked(eng, src, dst, rec, jobs=sel)
        same(dst.dispatch().copy(), rec[parent], "edge run")
    src.free()
    dst.free()


def test_selective_list_around_one_route_select_grid(eng):
    policy, routing, workers = tsd.pins_registry()
    table = wire.WorkerTable.from_workers(workers)
    load(eng, policy, routing, table)
    rng = np.random.default_rng(9)
    W = len(workers)
    jobs = []
    for t in range(GRID_JOBS + 3000):
        i = int(rng.integers(W))
        c = (1, 2, 3, 5)[t % 4]
        jobs.append({"topic": "job.any", "labels": {k: workers[i]["labels"][k] for k in sl.UNIQUE[:c]}})
    env = wire.EnvelopeBatch.from_jobs(jobs)
    n = env.n_jobs
    src, dst = eng.batch(n), eng.batch(n)
    rec = src.encode(env).dispatch().copy()
    o = oracle_lib.Oracle(policy, routing, table)
    for m in (GRID_JOBS - 1, GRID_JOBS, GRID_JOBS + 1):
        sel = np.sort(rng.choice(n, m, replace=False))
        parent = subset_checked(eng, src, dst, rec, jobs=sel)
        assert len(side(dst, 0)) > 2 * m     # every job is listed, and extra words follow
        before = eng.launch_count()
        got = dst.dispatch().copy()
        assert eng.launch_count() - before == 3
        same(got, rec[parent], "grid m=%d" % m)
    same(got, o.eval(take(env, parent)), "grid against the oracle")
    o.close()
    src.free()
    dst.free()


@pytest.mark.slow
def test_config3_million_jobs(eng):
    cfg = synth.make_config("c3")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    W = cfg.workers.n_workers
    eng.update_workers(np.arange(W, dtype=np.uint32), overloaded(cfg.workers, 3))
    n = cfg.jobs.n_jobs
    src, dst = eng.batch(n), eng.batch(n)
    rec = src.encode(cfg.jobs).dispatch().copy()
    parent = subset_checked(eng, src, dst, rec, outcomes=wire.SUBSET_RETRYABLE)
    assert len(parent) > n // 10
    dst.dispatch_resident()
    same(dst.fetch().copy(), rec[parent], "config 3")
    src.free()
    dst.free()


# ------------------------------------------------------------------ 5. refusals
def refused(code, fn):
    from cordum_b200 import engine

    with pytest.raises(engine.CordumError) as ei:
        fn()
    assert ei.value.code == code, (ei.value.code, str(ei.value))


def test_refusals(eng):
    cfg = synth.make_config("tiny")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    n = cfg.jobs.n_jobs
    src, dst, small = eng.batch(n), eng.batch(n), eng.batch(4)
    # E_STATE: a host-encoded batch never dispatched; the outcome form before the wait
    src.encode(cfg.jobs)
    refused(E_STATE, lambda: src.subset(dst, jobs=[0, 1]))
    refused(E_STATE, lambda: src.subset(dst, outcomes=wire.SUBSET_RETRYABLE))
    src.dispatch_async()
    refused(E_STATE, lambda: src.subset(dst, outcomes=wire.SUBSET_RETRYABLE))
    refused(E_STATE, lambda: src.subset(dst, jobs=[0, 1]))
    rec = src.wait().copy()
    # E_INVALID: bad arguments
    refused(E_INVALID, lambda: src.subset(src, jobs=[0]))
    refused(E_INVALID, lambda: src.subset(dst))
    refused(E_INVALID, lambda: src.subset(dst, outcomes=1, jobs=[0]))
    refused(E_INVALID, lambda: src.subset(dst, outcomes=1 << 12))
    refused(E_INVALID, lambda: src.subset(dst, jobs=[2, 1]))
    refused(E_INVALID, lambda: src.subset(dst, jobs=[1, 1]))
    refused(E_INVALID, lambda: src.subset(dst, jobs=[n]))
    from cordum_b200 import engine

    other = engine.Engine(device=0)
    load(other, cfg.policy, cfg.routing, cfg.workers)
    foreign = other.batch(n)
    refused(E_INVALID, lambda: src.subset(foreign, jobs=[0]))
    other.close()
    # E_CAPACITY: too small a destination; its previous records still dispatch as before
    small_rec = small.encode(cfg.jobs.slice(0, 4)).dispatch().copy()
    before = eng.launch_count()
    refused(E_CAPACITY, lambda: src.subset(small, jobs=np.arange(5)))
    assert eng.launch_count() == before            # a list is measured before any device work
    every = (1 << wire.PLAN_OUTCOMES) - 1
    assert len(selected_by(rec, every)) > 4
    refused(E_CAPACITY, lambda: src.subset(small, outcomes=every))
    assert eng.launch_count() - before == 3        # counted on the device, refused before the gather
    small.dispatch_resident()
    same(small.fetch().copy(), small_rec, "after a capacity refusal")
    # E_STALE: each reload, and a new dictionary generation; a heartbeat delta keeps the epoch
    eng.update_workers(np.arange(3, dtype=np.uint32), cfg.workers.loads()[:3])
    assert src.subset(dst, jobs=[0, 2]) == 2
    for reload in (lambda: eng.load_policy(cfg.policy, "again"), lambda: eng.load_routing(cfg.routing),
                   lambda: eng.load_workers(cfg.workers)):
        rec = src.encode(cfg.jobs).dispatch().copy()
        reload()
        refused(E_STALE, lambda: src.subset(dst, jobs=[0]))
        refused(E_STALE, lambda: src.subset(dst, outcomes=wire.SUBSET_RETRYABLE))
    for b in (src, dst, small):
        b.free()


def test_stale_after_a_dictionary_generation(eng):
    """A topic dictionary that fills up starts a new generation (new epoch): records of the old ids are refused."""
    from cordum_b200 import engine

    e2 = engine.Engine(device=0, max_topics=24, max_effcfgs=8)
    load(e2, {"rules": [{"id": "d", "decision": "deny", "match": {"topics": ["job.bad.*"]}}]},
         {"topics": {"job.keep.a": ["p"]}, "pools": {"p": {}}}, [kats.hb("w0", "p")])
    src, dst, b = e2.batch(32), e2.batch(32), e2.batch(32)
    rec = src.encode([{"topic": "job.keep.a"}, {"topic": "job.bad.x"}]).dispatch().copy()
    assert src.subset(dst, jobs=[1]) == 1
    for rnd in range(8):
        b.encode([{"topic": "job.ok.r%d-%d" % (rnd, i)} for i in range(9)]).dispatch()
    refused(E_STALE, lambda: src.subset(dst, jobs=[1]))
    refused(E_STALE, lambda: src.subset(dst, outcomes=1 << 2))   # DENY
    rec = src.encode([{"topic": "job.keep.a"}, {"topic": "job.bad.x"}]).dispatch().copy()
    assert src.subset(dst, outcomes=1 << 2) == 1
    same(dst.dispatch().copy(), rec[1:], "after the new generation")
    e2.close()


# ------------------------------------------------------------------ 6. launch counts, 7. strings
def test_launch_counts(eng):
    cfg = synth.make_config("c2")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    n = cfg.jobs.n_jobs
    src, dst = eng.batch(n), eng.batch(n)
    rec = src.encode(cfg.jobs).dispatch().copy()
    subset_checked(eng, src, dst, rec, jobs=np.arange(0, n, 2))
    before = eng.launch_count()
    dst.dispatch()
    assert eng.launch_count() - before == 2
    # with a selective list
    policy, routing, workers = tsd.pins_registry()
    load(eng, policy, routing, wire.WorkerTable.from_workers(workers))
    env = wire.EnvelopeBatch.from_jobs(tsd.pins_jobs(workers))
    src2, dst2 = eng.batch(env.n_jobs), eng.batch(env.n_jobs)
    rec2 = src2.encode(env).dispatch().copy()
    subset_checked(eng, src2, dst2, rec2, jobs=np.arange(0, env.n_jobs, 2))
    assert len(side(dst2, 0))
    before = eng.launch_count()
    dst2.dispatch()
    assert eng.launch_count() - before == 3
    # an empty source launches nothing
    e0, d0 = eng.batch(1), eng.batch(1)
    e0.encode(env.slice(0, 0)).dispatch()
    before = eng.launch_count()
    assert e0.subset(d0, jobs=[]) == 0 and eng.launch_count() == before
    for b in (src, dst, src2, dst2, e0, d0):
        b.free()


def test_strings_follow_the_parent(eng):
    c5 = kats.golden("c5_demo_guardrails.json")
    jobs, workers, _ = synth.make_c5(4000)
    load(eng, c5["policy"], c5["routing"], workers)
    src, dst = eng.batch(jobs.n_jobs), eng.batch(jobs.n_jobs)
    rec = src.encode(jobs).dispatch().copy()
    parent = subset_checked(eng, src, dst, rec, jobs=np.arange(0, jobs.n_jobs, 3))
    got = dst.dispatch().copy()
    same(got, rec[parent], "c5 strings")
    src._env = None   # both sides without envelopes: canonical MCP spelling
    gen = dst.policy_gen()
    for i in range(len(parent)):
        p = int(parent[i])
        assert dst.reason(i) == src.reason(p), i
        assert dst.subject(i) == src.subject(p), i
        assert eng.rule_id(int(got["rule_idx"][i]), gen) == eng.rule_id(int(rec["rule_idx"][p]), src.policy_gen())
    assert any(dst.reason(i) for i in range(len(parent))) and any(dst.subject(i) for i in range(len(parent)))
    src.free()
    dst.free()
