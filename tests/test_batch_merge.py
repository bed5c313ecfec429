"""cordum_batch_merge: one encoded batch built on the device from two encoded batches of the same table epoch.  Its records
must equal, bit for bit, a host encode of a's envelopes followed by b's (JobRec, RouteRec, slot_of, selective list, wide
rows); it must decide as a and b each dispatched on their own, and as the C++ oracle on the concatenated jobs, on every
dispatch path; and the retry loop (subset the retries -> merge with the new arrivals -> one tick) must give the plan and
topic counts of the two batches dispatched separately.  Also key interleavings and tile edges, lifetimes, refusals,
launch counts and buffer growth under captured tick graphs."""

import numpy as np
import pytest

import kats
import oracle_lib
import test_batch_subset as tbs
import test_selective_differential as tsd
import test_selective_labels as sl
from test_batch_subset import config, run, same, side, take
from cordum_b200 import synth, wire

pytestmark = pytest.mark.gpu

MODES = tbs.MODES
PATHS = tbs.PATHS
TILE = 2048                  # items per CTA of the merge kernels (csrc/kernels.h CORDUM_SUBSET_TILE)
GRID_JOBS = tsd.GRID_JOBS
E_INVALID, E_CAPACITY, E_STATE, E_STALE = -1, -2, -4, -6
MERGE_LAUNCHES = 3


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
    eng.load_policy(policy, "merge")
    eng.load_routing(routing)
    eng.load_workers(workers)


def ready(eng, b, env, encoder):
    """b encoded from env by one encoder, with its records complete on the device: a host encode is dispatched once; a
    device encode is waited for, and dispatched once only when it fell back to the host encoder."""
    b.device_order = False
    if encoder == "host":
        b.encode(env).dispatch()
    else:
        before = eng.host_fallbacks()
        b.encode_device(env.deinterned()).wait()
        b.device_order = eng.host_fallbacks() == before
        if not b.device_order:
            b.dispatch()
    return b


def merged(eng, a, b, dst):
    """a.merge(b, dst) with its launch count, job count and (empty) parent index checked."""
    before = eng.launch_count()
    m = a.merge(b, dst)
    assert m == a.size + b.size == dst.size
    assert eng.launch_count() - before == (MERGE_LAUNCHES if m else 0)
    assert len(dst.parent_index()) == 0
    return m


def by_job(b):
    """b's records in job order: JobRec, RouteRec, wide row and selective-list pairs (by job index) of each job."""
    job, route, slot = (x.copy() for x in b.records())
    sel, wide = side(b, 0), side(b, 1)
    n, k = len(job), int(((job["flags"] & sl.JF_SELECTIVE) != 0).sum())
    extra = sel[2 * k:]
    lists = {}
    for e in range(k):
        s, x = int(sel[2 * e]), int(sel[2 * e + 1])
        lists[int(job["orig"][s])] = tuple(extra[x + 1:x + 1 + int(extra[x])].tolist()) if x else ()
    rows = wide.reshape(n, len(wide) // n)[slot] if n and len(wide) else wide
    return job[slot], route[slot], lists, rows, job


def check_records(eng, dst, env, what, srcs=None):
    """dst's records, selective list and wide rows against a host encode of env, bit for bit.  The device encoder orders
    the jobs of one key as its threads claim slots (encode.cu), so with a device-ordered source (srcs = (a, b)) the sorted
    order is checked as the stable merge of a's and b's orders instead, and the records job by job."""
    job, route, slot = dst.records()
    hjob, hroute, hslot, hsel, hwide = tbs.host_records_of(eng, env)
    if srcs is None:
        assert job.tobytes() == hjob.tobytes(), what
        assert route.tobytes() == hroute.tobytes(), what
        assert np.array_equal(slot, hslot), what
        assert np.array_equal(side(dst, 0), hsel), what
        assert np.array_equal(side(dst, 1), hwide), what
        return
    hb = eng.batch(max(env.n_jobs, 1))
    hb.encode(env)
    want, got = by_job(hb), by_job(dst)
    hb.free()
    assert got[0].tobytes() == want[0].tobytes() and got[1].tobytes() == want[1].tobytes(), what
    assert got[2] == want[2] and np.array_equal(got[3], want[3]), what
    assert np.array_equal(got[4]["topic"], want[4]["topic"]), what      # the key's major part, slot by slot
    a, b = srcs
    orig, na = got[4]["orig"].astype(np.int64), a.size
    assert np.array_equal(orig[orig < na], a.records()[0]["orig"]), what
    assert np.array_equal(orig[orig >= na] - na, b.records()[0]["orig"]), what


def pair(eng, env, ia, ib, enc=("host", "host")):
    """a and b from env's jobs ia and ib.  env is host-encoded once first: the dictionaries assign ids on first sight (a
    new effective config brings its MCP values), and records of one vocabulary are what a merge keeps bit for bit."""
    tbs.host_records_of(eng, env)
    a, b = eng.batch(max(len(ia), 1)), eng.batch(max(len(ib), 1))
    ready(eng, a, take(env, ia), enc[0])
    ready(eng, b, take(env, ib), enc[1])
    return a, b


def free(*bs):
    for b in bs:
        b.free()


def split(n, seed):
    rng = np.random.default_rng(seed)
    ia = np.sort(rng.choice(n, size=int(n * 0.6), replace=False))
    ib = rng.choice(n, size=n - len(ia), replace=False)   # any order, and jobs of a again
    return ia, ib


# ------------------------------------------------------------------ 1. records against a host encode of a ++ b
@pytest.mark.parametrize("enc", [("host", "host"), ("host", "device"), ("device", "host"), ("device", "device")],
                         ids=["hh", "hd", "dh", "dd"])
@pytest.mark.parametrize("name", ["tiny", "c2", "c5", "fuzz"])
def test_records_equal_a_host_encode_of_both(eng, name, enc):
    policy, routing, workers, env = config(name)
    load(eng, policy, routing, workers)
    ia, ib = split(env.n_jobs, 5)
    a, b = pair(eng, env, ia, ib, enc)
    dst = eng.batch(env.n_jobs)
    merged(eng, a, b, dst)
    device = a.device_order or b.device_order   # a source stayed in the device encoder's order
    check_records(eng, dst, take(env, np.concatenate([ia, ib])), "%s %s" % (name, enc), (a, b) if device else None)
    free(a, b, dst)


@pytest.fixture(scope="module")
def hostnames():
    policy, routing, workers = sl.registry(sl.GPU_WORKERS, sl.GPU_POOLS, seed=5, n_second=sl.GPU_SECOND)
    jobs = sl.jobs_for(workers, sl.GPU_POOLS, 2000, seed=6, n_second=sl.GPU_SECOND) + sl.multi_jobs(workers[:sl.GPU_SECOND], (1, 2))
    for i in range(0, sl.GPU_SECOND, 40):   # three selective pairs: a hostname, an instance and a small svc group
        lab = workers[i]["labels"]
        jobs.append({"topic": "job.any", "labels": {"hostname": lab["hostname"], "instance": lab["instance"], "svc": "s%02d" % (i % 4)}})
    return policy, routing, wire.WorkerTable.from_workers(workers), wire.EnvelopeBatch.from_jobs(jobs)


def registry_case(kind, hostnames):
    if kind == "hostname":
        return hostnames
    if kind == "pins":
        policy, routing, workers = tsd.pins_registry()
        jobs = tsd.pins_jobs(workers)
    else:
        policy, routing, workers = tsd.wide_registry()
        jobs = tsd.wide_jobs(workers, 3000, 5)
    return policy, routing, wire.WorkerTable.from_workers(workers), wire.EnvelopeBatch.from_jobs(jobs)


@pytest.mark.parametrize("kind", ["hostname", "pins", "wide"])
def test_selective_lists_and_wide_rows(eng, kind, hostnames):
    policy, routing, table, env = registry_case(kind, hostnames)
    load(eng, policy, routing, table)
    n = env.n_jobs
    rng = np.random.default_rng(7)
    ia, ib = split(n, 8)
    a, b = pair(eng, env, ia, ib, ("host", "device"))
    jobs = a.records()[0]
    sel = side(a, 0)
    if kind == "wide":
        assert len(side(a, 1))
    else:
        # jobs naming no selective pair (no entry), and entries of 1, 2, 3 and (pins) 5 pairs
        flagged = (jobs["flags"] & sl.JF_SELECTIVE) != 0
        assert flagged.any() and (~flagged).any() and len(sel) > 2 * flagged.sum() + 1   # extra words: three or more pairs
    dst, dst2 = eng.batch(2 * n), eng.batch(2 * n)
    o = oracle_lib.Oracle(policy, routing, table)
    for x, y, what in ((ia, ib, "a, b"), (ib, ia, "b, a"), (ia, ia, "a, a")):
        s, t = (a, b) if what == "a, b" else (b, a) if what == "b, a" else (a, a)
        merged(eng, s, t, dst)
        both = take(env, np.concatenate([x, y]))
        check_records(eng, dst, both, "%s %s" % (kind, what))
        same(dst.dispatch().copy(), o.eval(both), "%s %s against the oracle" % (kind, what))
    # a subset of a merge, merged again: the selective list is re-packed each time
    pick = np.sort(rng.choice(dst.size, dst.size // 2, replace=False))
    dst.subset(dst2, jobs=pick)
    merged(eng, dst2, b, dst)
    check_records(eng, dst, take(env, np.concatenate([np.concatenate([ia, ia])[pick], ib])), "%s merge of a subset" % kind)
    o.close()
    free(a, b, dst, dst2)


# ------------------------------------------------------------------ 2. decisions on every path
@pytest.mark.parametrize("name", ["tiny", "c2", "c5", "fuzz"])
def test_merge_decides_as_its_sources(eng, name):
    policy, routing, workers, env = config(name)
    load(eng, policy, routing, workers)
    loads = workers.loads()
    ia, ib = split(env.n_jobs, 11)
    a, b = pair(eng, env, ia, ib, ("device", "host"))
    dst = eng.batch(env.n_jobs)
    merged(eng, a, b, dst)
    o = oracle_lib.Oracle(policy, routing, workers)
    seen = set()
    for mode in MODES:
        want = np.concatenate([a.dispatch(mode).copy(), b.dispatch(mode).copy()])
        same(want, o.eval(take(env, np.concatenate([ia, ib])), mode), "%s mode %d: oracle" % (name, mode))
        for path in PATHS:
            if path == "tick" and mode != wire.MODE_POLICY_AND_ROUTE:
                continue
            same(run(eng, dst, mode, path, loads), want, "%s mode %d %s" % (name, mode, path))
            seen.add(path)
    assert seen == set(PATHS)
    o.close()
    free(a, b, dst)


# ------------------------------------------------------------------ 3. key interleavings and tile edges
def by_key(eng, env):
    """Job indices of env in the encoders' sorted order, and each sorted slot's topic id."""
    b = eng.batch(env.n_jobs)
    job = b.encode(env).records()[0].copy()
    b.free()
    return job["orig"].astype(np.int64), job["topic"].astype(np.int64)


def interleavings(eng, env):
    order, topic = by_key(eng, env)
    cut = int(np.flatnonzero(np.diff(topic))[len(np.unique(topic)) // 2 - 1]) + 1   # a topic boundary near the middle
    low, high = np.sort(order[:cut]), np.sort(order[cut:])
    rng = np.random.default_rng(2)
    some = np.sort(rng.choice(env.n_jobs, env.n_jobs // 3, replace=False))
    return {"a below b": (low, high), "a above b": (high, low), "same keys": (some, rng.permutation(some)),
            "interleaved": (order[0::2], order[1::2])}


def test_key_interleavings(eng):
    cfg = synth.make_config("c2")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    env = cfg.jobs.slice(0, 3 * TILE + 100)
    dst = eng.batch(2 * env.n_jobs)
    for what, (ia, ib) in interleavings(eng, env).items():
        a, b = pair(eng, env, ia, ib)
        merged(eng, a, b, dst)
        check_records(eng, dst, take(env, np.concatenate([ia, ib])), what)
        same(dst.dispatch().copy(), np.concatenate([a.results().copy(), b.results().copy()]), what)
        free(a, b)
    # a == b: every key ties, a's copy first
    a = ready(eng, eng.batch(env.n_jobs), env, "host")
    merged(eng, a, a, dst)
    check_records(eng, dst, take(env, np.concatenate([np.arange(env.n_jobs)] * 2)), "a == b")
    orig, own = dst.records()[0]["orig"].astype(np.int64), a.records()[0]["orig"]
    assert np.array_equal(orig[orig < env.n_jobs], own) and np.array_equal(orig[orig >= env.n_jobs] - env.n_jobs, own)
    free(a, dst)


SIZES = [(0, 0), (0, 5), (5, 0), (1, 1), (TILE - 1, 3), (3, TILE - 1), (TILE, TILE), (TILE + 1, 1), (1, TILE + 1),
         (2 * TILE + 1, 7), (7, 2 * TILE + 1), (TILE - 1, TILE + 1)]


@pytest.mark.parametrize("na,nb", SIZES)
def test_tile_edges(eng, na, nb):
    cfg = synth.make_config("c2")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    rng = np.random.default_rng(na * 7 + nb)
    n = cfg.jobs.n_jobs
    ia, ib = np.sort(rng.choice(n, na, replace=False)), np.sort(rng.choice(n, nb, replace=False))
    a, b = pair(eng, cfg.jobs, ia, ib)
    dst = eng.batch(max(na + nb, 1))
    merged(eng, a, b, dst)
    both = take(cfg.jobs, np.concatenate([ia, ib]).astype(np.int64))
    check_records(eng, dst, both, "%d + %d" % (na, nb))
    want = np.concatenate([a.dispatch().copy(), b.dispatch().copy()])
    same(dst.dispatch().copy(), want, "%d + %d" % (na, nb))
    free(a, b, dst)


def test_one_topic_one_tenant_class(eng):
    policy, routing, workers = sl.registry(200, 8)
    table = wire.WorkerTable.from_workers(workers)
    load(eng, policy, routing, table)
    env = wire.EnvelopeBatch.from_jobs([{"topic": "job.any", "labels": {"zone": "z%d" % (i % 4)}} for i in range(TILE + 300)])
    ia, ib = np.arange(0, env.n_jobs, 3), np.arange(1, env.n_jobs, 2)
    a, b = pair(eng, env, ia, ib)
    dst = eng.batch(env.n_jobs * 2)
    merged(eng, a, b, dst)
    both = take(env, np.concatenate([ia, ib]))
    check_records(eng, dst, both, "one key")
    assert np.array_equal(dst.records()[0]["orig"], np.arange(dst.size))   # one key: job order
    o = oracle_lib.Oracle(policy, routing, table)
    same(dst.dispatch().copy(), o.eval(both), "one key")
    o.close()
    free(a, b, dst)


def test_tenant_classes_order_a_topic(eng):
    """Seven tenant classes (test_device_encode_differential's shape policy) on ten topics: inside a topic the key still
    orders the jobs by class, and a merge must interleave a's and b's jobs class by class."""
    import test_device_encode_differential as tde

    policy, routing, workers = tde.shape_config()
    load(eng, policy, routing, workers)
    tens = ("ten0", "TEN1", "ten2 ", "ten3", "ten4", "\tTen5", "other", "")
    env = wire.EnvelopeBatch.from_jobs([{"topic": "job.t.%d" % (i % 10), "tenant": tens[(i * 7 // 10) % 8]} for i in range(2 * TILE + 333)])
    i = np.arange(env.n_jobs)
    ia, ib = i[i % 3 != 0], i[i % 3 == 0]   # every topic has jobs of several classes in both sources
    a, b = pair(eng, env, ia, ib)
    dst = eng.batch(env.n_jobs)
    merged(eng, a, b, dst)
    both = take(env, np.concatenate([ia, ib]))
    check_records(eng, dst, both, "tenant classes")
    o = oracle_lib.Oracle(policy, routing, workers)
    same(dst.dispatch().copy(), o.eval(both), "tenant classes")
    o.close()
    free(a, b, dst)


def test_selective_list_beyond_one_route_select_grid(eng):
    policy, routing, workers = tsd.pins_registry()
    table = wire.WorkerTable.from_workers(workers)
    load(eng, policy, routing, table)
    rng = np.random.default_rng(9)
    W = len(workers)
    jobs = []
    for t in range(GRID_JOBS + 3000):
        i = int(rng.integers(W))
        jobs.append({"topic": "job.any", "labels": {k: workers[i]["labels"][k] for k in sl.UNIQUE[:(1, 2, 3, 5)[t % 4]]}})
    env = wire.EnvelopeBatch.from_jobs(jobs)
    n = env.n_jobs
    ia, ib = np.arange(0, n // 2 + 700), np.arange(n // 2 + 700, n)
    a, b = pair(eng, env, ia, ib)
    dst = eng.batch(n)
    merged(eng, a, b, dst)
    assert len(side(dst, 0)) > 2 * GRID_JOBS
    check_records(eng, dst, env, "one grid and more")
    before = eng.launch_count()
    got = dst.dispatch().copy()
    assert eng.launch_count() - before == 3
    o = oracle_lib.Oracle(policy, routing, table)
    same(got, o.eval(env), "one grid and more")
    o.close()
    free(a, b, dst)


# ------------------------------------------------------------------ 4. the retry loop
def topic_table(labels, counts):
    return {l: counts[i].astype(np.int64) for i, l in enumerate(labels)}


@pytest.mark.parametrize("name", ["c2", "c5"])
def test_retry_loop_in_one_tick(eng, name):
    policy, routing, workers, env = config(name)
    load(eng, policy, routing, workers)
    W = workers.n_workers
    slots = np.arange(W, dtype=np.uint32)
    hot, cool = tbs.overloaded(workers, 2), workers.loads()
    eng.update_workers(slots, hot)
    n = env.n_jobs
    first, second = np.arange(n // 2), np.arange(n // 2, n)
    src, retry, new, dst, d2, d3 = (eng.batch(n) for _ in range(6))
    rec = src.encode(take(env, first)).dispatch().copy()
    eng.update_workers(slots, cool)                                  # one heartbeat
    parent = tbs.subset_checked(eng, src, retry, rec, outcomes=wire.SUBSET_RETRYABLE)
    assert len(parent)
    ready(eng, new, take(env, second), "device")
    merged(eng, retry, new, dst)
    got = run(eng, dst, wire.MODE_POLICY_AND_ROUTE, "tick", cool)    # one tick
    rr, rn = retry.dispatch().copy(), new.dispatch().copy()
    same(got, np.concatenate([rr, rn]), "%s merged tick" % name)
    o = oracle_lib.Oracle(policy, routing, workers)
    o.update_workers(slots, cool)
    jobs_of_dst = np.concatenate([first[parent], second])
    same(got, o.eval(take(env, jobs_of_dst)), "%s against the oracle" % name)
    # the plan: bucket by bucket, retry's jobs then the new arrivals'
    off, jobs, ns = dst.plan()
    off, jobs = off.copy(), jobs.copy()
    offr, jobsr, _ = retry.plan()
    offr, jobsr = offr.copy(), jobsr.copy()
    offn, jobsn, _ = new.plan()
    assert ns == W and np.array_equal(off, offr + offn)
    for k in range(len(off) - 1):
        want = np.concatenate([jobsr[offr[k]:offr[k + 1]], jobsn[offn[k]:offn[k + 1]] + len(parent)])
        assert np.array_equal(jobs[off[k]:off[k + 1]], want), k
    # the topic counts: the two tables added label by label
    lab, cnt = dst.topic_counts()
    td = topic_table(lab, cnt.copy())
    tr = topic_table(*retry.topic_counts())
    tn = topic_table(*new.topic_counts())
    for l in set(tr) | set(tn):
        assert np.array_equal(td[l], tr.get(l, 0) + tn.get(l, 0)), l
    assert set(td) == set(tr) | set(tn)
    # chained: a subset of the merge, and a merge of the merge
    pick = np.arange(0, dst.size, 3)
    tbs.subset_checked(eng, dst, d2, got, jobs=pick)
    same(d2.dispatch().copy(), got[pick], "subset of a merge")
    merged(eng, dst, retry, d3)
    same(d3.dispatch().copy(), np.concatenate([got, rr]), "merge of a merge")
    check_records(eng, d3, take(env, np.concatenate([jobs_of_dst, first[parent]])), "merge of a merge, records", (dst, retry))
    o.close()
    free(src, retry, new, dst, d2, d3)


# ------------------------------------------------------------------ 5. lifetime
@pytest.mark.parametrize("then", ["re-encode", "free"])
def test_merge_outlives_its_sources(eng, then):
    policy, routing, workers = tsd.wide_registry()
    table = wire.WorkerTable.from_workers(workers)
    load(eng, policy, routing, table)
    env = wire.EnvelopeBatch.from_jobs(tsd.wide_jobs(workers, 3000, 7))
    other = wire.EnvelopeBatch.from_jobs(tsd.wide_jobs(workers, 3000, 8))
    n = env.n_jobs
    ia, ib = split(n, 3)
    a, b = pair(eng, env, ia, ib)
    want = np.concatenate([a.results().copy(), b.results().copy()])
    dst, helper = eng.batch(n), eng.batch(n)
    tbs.subset_checked(eng, a, dst, a.results().copy(), jobs=np.arange(0, len(ia), 2))
    assert len(dst.parent_index())
    merged(eng, a, b, dst)                                           # the parent index of the earlier subset is gone
    sel, wide = side(dst, 0), side(dst, 1)
    assert len(sel) and len(wide)
    if then == "re-encode":
        a.encode(other.slice(0, 100)).dispatch()
        b.encode(other.slice(100, 200)).dispatch()
    else:
        free(a, b)
    for path in PATHS:
        same(run(eng, dst, wire.MODE_POLICY_AND_ROUTE, path, table.loads()), want, "after the sources %s, %s" % (then, path))
    assert np.array_equal(side(dst, 0), sel) and np.array_equal(side(dst, 1), wide)
    assert len(dst.parent_index()) == 0
    check_records(eng, dst, take(env, np.concatenate([ia, ib])), "after the sources %s" % then)
    if then == "re-encode":
        free(a, b)
    free(dst, helper)


def test_strings_of_a_merge(eng):
    c5 = kats.golden("c5_demo_guardrails.json")
    jobs, workers, _ = synth.make_c5(4000)
    load(eng, c5["policy"], c5["routing"], workers)
    ia, ib = split(jobs.n_jobs, 4)
    a, b = pair(eng, jobs, ia, ib)
    dst = eng.batch(jobs.n_jobs)
    merged(eng, a, b, dst)
    got = dst.dispatch().copy()
    a._env = b._env = None   # the sources without envelopes too: canonical MCP spelling on both sides
    for i in range(dst.size):
        s, j = (a, i) if i < a.size else (b, i - a.size)
        assert dst.reason(i) == s.reason(j), i
        assert dst.subject(i) == s.subject(j), i
    assert any(dst.reason(i) for i in range(dst.size)) and any(dst.subject(i) for i in range(dst.size))
    free(a, b, dst)


# ------------------------------------------------------------------ 6. refusals
def refused(code, fn, text):
    from cordum_b200 import engine

    with pytest.raises(engine.CordumError) as ei:
        fn()
    assert ei.value.code == code, (ei.value.code, str(ei.value))
    assert text in str(ei.value), str(ei.value)


def test_refusals(eng):
    from cordum_b200 import engine

    cfg = synth.make_config("tiny")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    env = cfg.jobs
    n = env.n_jobs
    a, b, dst, small = eng.batch(n), eng.batch(n), eng.batch(2 * n), eng.batch(4)
    L = eng.L

    def usable():
        ready(eng, a, env, "host")
        ready(eng, b, env.slice(0, 50), "host")
        merged(eng, a, b, dst)
        same(dst.dispatch().copy(), np.concatenate([a.results().copy(), b.results().copy()]), "usable")

    usable()
    # E_INVALID
    refused(E_INVALID, lambda: eng._ck(L.cordum_batch_merge(None, b.h, dst.h)), "null argument")
    refused(E_INVALID, lambda: eng._ck(L.cordum_batch_merge(a.h, None, dst.h)), "null argument")
    refused(E_INVALID, lambda: eng._ck(L.cordum_batch_merge(a.h, b.h, None)), "null argument")
    refused(E_INVALID, lambda: a.merge(b, a), "another batch than its sources")
    refused(E_INVALID, lambda: a.merge(b, b), "another batch than its sources")
    other = engine.Engine(device=0)
    load(other, cfg.policy, cfg.routing, cfg.workers)
    foreign = other.batch(2 * n)
    ready(other, foreign, env, "host")
    refused(E_INVALID, lambda: a.merge(b, foreign), "different engines")
    refused(E_INVALID, lambda: a.merge(foreign, dst), "different engines")
    other.close()
    usable()
    # E_STATE: a host encode never dispatched; a device encode, an async dispatch and a tick not waited for
    text = "not complete on the device"
    a.encode(env)
    refused(E_STATE, lambda: a.merge(b, dst), text)
    refused(E_STATE, lambda: b.merge(a, dst), text)
    a.encode_device(env.deinterned())
    refused(E_STATE, lambda: a.merge(b, dst), text)
    a.wait()
    merged(eng, a, b, dst)
    a.dispatch_async()
    refused(E_STATE, lambda: a.merge(b, dst), text)
    a.wait()
    a.tick(cfg.workers.loads().ctypes.data, 0, cfg.workers.n_workers)
    refused(E_STATE, lambda: b.merge(a, dst), text)
    eng.tick_flush()
    a.wait()
    merged(eng, b, a, dst)
    usable()
    # E_CAPACITY: dst untouched, nothing launched
    small_rec = ready(eng, small, env.slice(0, 4), "host").results().copy()
    job, route, slot = (x.copy() for x in small.records())
    s0, s1 = side(small, 0), side(small, 1)
    before = eng.launch_count()
    refused(E_CAPACITY, lambda: a.merge(b, small), "more than the destination batch holds")
    assert eng.launch_count() == before
    assert small.size == 4
    j2, r2, sl2 = small.records()
    assert j2.tobytes() == job.tobytes() and r2.tobytes() == route.tobytes() and np.array_equal(sl2, slot)
    assert np.array_equal(side(small, 0), s0) and np.array_equal(side(small, 1), s1)
    small.dispatch_resident()
    same(small.fetch().copy(), small_rec, "after a capacity refusal")
    # a heartbeat delta keeps the epoch
    eng.update_workers(np.arange(3, dtype=np.uint32), cfg.workers.loads()[:3])
    merged(eng, a, b, dst)
    # E_STALE: each reload, for either source
    for reload in (lambda: eng.load_policy(cfg.policy, "again"), lambda: eng.load_routing(cfg.routing),
                   lambda: eng.load_workers(cfg.workers)):
        ready(eng, a, env, "host")
        ready(eng, b, env.slice(0, 50), "device")
        reload()
        refused(E_STALE, lambda: a.merge(b, dst), "reloaded")
        ready(eng, a, env, "host")
        refused(E_STALE, lambda: a.merge(b, dst), "reloaded")            # sources of two epochs
        refused(E_STALE, lambda: b.merge(a, dst), "reloaded")
        usable()
    free(a, b, dst, small)


def test_stale_after_a_dictionary_generation(eng):
    from cordum_b200 import engine

    e2 = engine.Engine(device=0, max_topics=24, max_effcfgs=8)
    load(e2, {"rules": [{"id": "d", "decision": "deny", "match": {"topics": ["job.bad.*"]}}]},
         {"topics": {"job.keep.a": ["p"]}, "pools": {"p": {}}}, [kats.hb("w0", "p")])
    a, b, dst, x = e2.batch(32), e2.batch(32), e2.batch(64), e2.batch(32)
    jobs = [{"topic": "job.keep.a"}, {"topic": "job.bad.x"}]
    a.encode(jobs).dispatch()
    b.encode(jobs[::-1]).dispatch()
    assert a.merge(b, dst) == 4
    for rnd in range(8):
        x.encode([{"topic": "job.ok.r%d-%d" % (rnd, i)} for i in range(9)]).dispatch()
    refused(E_STALE, lambda: a.merge(b, dst), "reloaded")
    rec = a.encode(jobs).dispatch().copy()
    refused(E_STALE, lambda: a.merge(b, dst), "reloaded")
    rb = b.encode(jobs[::-1]).dispatch().copy()
    assert a.merge(b, dst) == 4
    same(dst.dispatch().copy(), np.concatenate([rec, rb]), "after the new generation")
    e2.close()


# ------------------------------------------------------------------ 7. launch counts, growth under tick graphs
def test_launch_counts_and_empty_sources(eng):
    cfg = synth.make_config("c2")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    e0, e1, dst = eng.batch(1), eng.batch(1), eng.batch(cfg.jobs.n_jobs)
    ready(eng, e0, cfg.jobs.slice(0, 0), "host")
    ready(eng, e1, cfg.jobs.slice(0, 0), "device")
    before = eng.launch_count()
    assert e0.merge(e1, dst) == 0 and eng.launch_count() == before
    a = ready(eng, eng.batch(cfg.jobs.n_jobs), cfg.jobs, "host")
    merged(eng, a, e0, dst)                                          # 3 launches (checked inside)
    before = eng.launch_count()
    dst.dispatch()
    assert eng.launch_count() - before == 2
    free(e0, e1, a, dst)


def test_tick_graphs_follow_growth(eng):
    """A merge that grows dst's selective list or wide rows moves their pointers: tick graphs captured before must not be
    replayed with the old ones."""
    for registry in ("pins", "wide"):
        policy, routing, table, env = registry_case(registry, None)
        load(eng, policy, routing, table)
        loads = table.loads()
        n = env.n_jobs
        o = oracle_lib.Oracle(policy, routing, table)
        small_a, small_b = pair(eng, env, np.arange(3), np.arange(3, 5))
        big_a, big_b = pair(eng, env, np.arange(0, n, 2), np.arange(1, n, 2))
        dst, other = eng.batch(n), eng.batch(n)
        ready(eng, other, env.slice(0, 64), "host")
        for s, t, idx in ((small_a, small_b, np.arange(5)), (big_a, big_b, np.concatenate([np.arange(0, n, 2), np.arange(1, n, 2)])),
                          (small_a, small_b, np.arange(5))):
            merged(eng, s, t, dst)
            want = o.eval(take(env, idx))
            for _ in range(2):   # alternate with another batch, so both tick graphs are captured and replayed
                dst.tick(loads.ctypes.data, 0, len(loads))
                other.tick(loads.ctypes.data, 0, len(loads))
            eng.tick_flush()
            dst.wait()
            same(dst.fetch().copy(), want, "%s tick after a merge of %d" % (registry, len(idx)))
        o.close()
        free(small_a, small_b, big_a, big_b, dst, other)


# ------------------------------------------------------------------ 8. config 3 at a million jobs
@pytest.mark.slow
def test_config3_million_jobs_and_retries(eng):
    cfg = synth.make_config("c3")
    load(eng, cfg.policy, cfg.routing, cfg.workers)
    W = cfg.workers.n_workers
    eng.update_workers(np.arange(W, dtype=np.uint32), tbs.overloaded(cfg.workers, 3))
    n = cfg.jobs.n_jobs
    src, retry = eng.batch(n), eng.batch(n)
    rec = src.encode(cfg.jobs).dispatch().copy()
    parent = tbs.subset_checked(eng, src, retry, rec, outcomes=wire.SUBSET_RETRYABLE)
    assert len(parent) > n // 10
    dst = eng.batch(n + len(parent))
    merged(eng, src, retry, dst)
    want = np.concatenate([src.dispatch().copy(), retry.dispatch().copy()])
    dst.dispatch_resident()
    same(dst.fetch().copy(), want, "config 3")
    check_records(eng, dst, take(cfg.jobs, np.concatenate([np.arange(n), parent])), "config 3 records")
    free(src, retry, dst)
