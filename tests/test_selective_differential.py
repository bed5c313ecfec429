"""Selective placement pairs (test_selective_labels.py) at the shapes the 60,000-hostname registry never reaches:
- dense placement bits beyond 128 (pos_label_x) next to selective pairs;
- jobs naming three or more selective pairs, so that the ids in the batch's selective list decide;
- holder lists longer than one warp, with ties, the least loaded holder in the last 32-chunk, every holder overloaded,
  holders in pools the topic does not list, and a short list that is not the job's first;
- the 32/33-holder and 1,024/1,025-bit boundaries, forced limits and the fuzz;
- more listed jobs than one grid of route_select_kernel covers;
- routing and registry reloads that move a pair across the selective / dense line.

CPU: the Python walk of the host tables (SelHarness) against the C++ oracle, and against the Python oracle on a sample.
GPU: every registry through blocking (all three modes), async, resident and tick dispatch against the C++ oracle, bit for
bit on all seven record fields, and against the same inputs compiled with the dense encoding where that fits.  Each case
asserts that its inputs reach the shape it stands for, so that a change of the generators cannot hollow it out."""
import random

import numpy as np
import pytest

import kats
import oracle_lib
import table_walk
import test_fuzz_three_way as fuzz
import test_selective_labels as sl
from cordum_b200 import wire

MIN_BITS, MAX_HOLDERS, DENSE, MODES = sl.MIN_BITS, sl.MAX_HOLDERS, sl.DENSE, sl.MODES
PR = wire.MODE_POLICY_AND_ROUTE
GRID_JOBS = 132 * 8 * 8   # route_select_kernel's grid on a 132-SM H100: sm_count * 8 CTAs of 8 warps, a warp per listed job
E_STALE = -6
STATUSES = (wire.ROUTE_OK, wire.ROUTE_OK_PREFERRED, wire.ROUTE_NO_WORKERS, wire.ROUTE_POOL_OVERLOADED, wire.ROUTE_NO_POOL_REQUIRES)
POLICY = {"default_tenant": "default", "rules": [{"id": "deny-x", "decision": "deny", "match": {"topics": ["job.x"]}}]}


@pytest.fixture(autouse=True)
def default_limits():
    sl.set_selective(MIN_BITS, MAX_HOLDERS)
    yield
    sl.set_selective(MIN_BITS, MAX_HOLDERS)


# ------------------------------------------------------------------ registries and jobs
FEATURES, N_WIDE, WIDE_POOLS = 150, 1300, 24


def wide_registry():
    """Registry 1: every worker has a hostname and a serial of its own, 6 of 150 shared features (fNNN: "on", 52 workers
    each: dense) and a zone.  About 2,900 placement bits: the unique pairs become selective and the 308 dense bits that
    remain need side words (xw_place = 3)."""
    rng = random.Random(11)
    pools = ["p%03d" % p for p in range(WIDE_POOLS)]
    routing = {"topics": {"job.any": pools, "job.half": pools[: WIDE_POOLS // 2], "job.one": pools[1:2]},
               "pools": {p: ({"requires": ["gpu"]} if i % 4 == 0 else {}) for i, p in enumerate(pools)}}
    workers = []
    for i in range(N_WIDE):
        labels = {"hostname": "host-%05d" % i, "serial": "sn-%05d" % i}
        labels.update({"f%03d" % ((i + 25 * k) % FEATURES): "on" for k in range(6)})
        labels["zone"] = "z%d" % (i % 4)
        pool = pools[(i * 7) % WIDE_POOLS] if i % 97 != 5 else "ghost"
        workers.append(kats.hb("w%05d" % i, pool, rng.randrange(3), float(rng.choice([0, 10, 20, 95])), 0.0, 8, labels))
    return POLICY, routing, workers


def features(w):
    return sorted(k for k in w["labels"] if k[0] == "f")


def wide_jobs(workers, n, seed):
    rng = random.Random(seed)
    W = len(workers)
    over = [i for i, w in enumerate(workers) if w["cpu_load"] >= 90]
    jobs = []
    for t in range(n):
        i = rng.randrange(W)
        w = workers[i]
        own = features(w)
        lacks = "f%03d" % rng.choice([f for f in range(FEATURES) if "f%03d" % f not in w["labels"]])
        lab = {"hostname": w["labels"]["hostname"]}
        topic = rng.choice(["job.any", "job.any", "job.half", "job.one"])
        kind = t % 17
        if kind in (1, 2, 3):
            lab.update({f: "on" for f in rng.sample(own, 2 * kind)})        # wide dense bits the holder has
        elif kind == 4:
            lab.update({f: "on" for f in own[:2]})
            lab[lacks] = "on"                                          # ... and one it lacks
        elif kind == 5:
            lab[lacks] = ""                                            # k: "" on a key the holder lacks
        elif kind == 6:
            lab[rng.choice(own)] = ""                                  # ... on a key it has
        elif kind == 7:
            lab["serial"] = w["labels"]["serial"]                      # two pins of one worker
        elif kind == 8:
            lab["serial"] = workers[rng.randrange(W)]["labels"]["serial"]   # two pins, mostly of two workers
        elif kind == 9:
            lab.update({f: "on" for f in own[:2]})
            lab["preferred_worker_id"] = w["worker_id"]                # the holder
            topic = "job.any"
        elif kind == 10:
            o = workers[rng.choice(over)]                              # an overloaded holder
            lab = {"hostname": o["labels"]["hostname"], "preferred_worker_id": o["worker_id"]}
            topic = "job.any"
        elif kind == 11:
            lab["preferred_worker_id"] = workers[rng.randrange(W)]["worker_id"]   # mostly a non-holder
        elif kind == 12:
            lab[lacks] = "on"                                          # the holder, but it lacks a wide bit
            lab["preferred_worker_id"] = w["worker_id"]
            topic = "job.any"
        elif kind == 13:
            lab = {"hostname": w["labels"]["hostname"], "zone": w["labels"]["zone"]}
        elif kind == 14:
            topic = "job.x"                                            # denied: the route is not attempted
        elif kind == 15:
            lab = {f: "on" for f in own[:2]}                           # dense only
        j = {"topic": topic, "labels": lab}
        if kind == 13 or (kind == 0 and t % 3 == 0):
            j["meta"] = {"requires": ["gpu"]}                          # behind requires
        jobs.append(j)
    return jobs


def pins_registry():
    """Registry 2: five labels of its own per worker (hostname, instance, serial, uuid, mac)."""
    return sl.registry(1200, 16, n_unique=5)


def pins_jobs(workers):
    """Jobs naming 1, 2, 3 and 5 pins; jobs whose third, fourth or fifth pin (in label order, which is the order of the
    ids in the record and the selective list) belongs to another worker; a preferred worker with the first two pins only."""
    U = sl.UNIQUE
    jobs = sl.multi_jobs(workers, (1, 2, 3, 5))
    for i in range(3, len(workers), 61):
        w, x = workers[i]["labels"], workers[(i * 7 + 1) % len(workers)]["labels"]
        for c, foreign in ((3, 2), (4, 3), (5, 2), (5, 3), (5, 4)):
            jobs.append({"topic": "job.any", "labels": {k: (x if u == foreign else w)[k] for u, k in enumerate(U[:c])}})
        lab = {k: w[k] for k in U[:2]}
        lab[U[2]] = x[U[2]]
        lab["preferred_worker_id"] = workers[i]["worker_id"]
        jobs.append({"topic": "job.any", "labels": lab})
        jobs.append({"topic": "job.any", "labels": dict({k: w[k] for k in U[:5]}, preferred_worker_id=workers[i]["worker_id"])})
    return jobs + sl.jobs_for(workers, 16, 400, seed=4)


SIZES = (31, 32, 33, 63, 64, 65, 200)
VARIANTS = ("tie", "last", "over", "split")
LONG_POOLS = ["q%d" % p for p in range(8)]


def long_registry():
    """Registry 3: one group per (size, variant), its members sharing grp=<group>; run with set_selective(0, 200).
    tie    equal loads across eight pools: ties across lanes and across one lane's loop iterations
    last   one pool, loads falling with the worker id: the least loaded holder is the last of the list
    over   every member overloaded
    split  the least loaded members sit in pools q4-q7, which topic job.half does not list
    Every group also has two members in a pool the routing table does not know: no holders."""
    routing = {"topics": {"job.any": LONG_POOLS, "job.half": LONG_POOLS[:4]}, "pools": {p: {} for p in LONG_POOLS}}
    workers = []
    for size in SIZES:
        for v in VARIANTS:
            g = "%s%03d" % (v, size)
            for m in range(size + 2):
                pool = "ghost" if m >= size else LONG_POOLS[0] if v == "last" else LONG_POOLS[m % 8]
                act, cpu = {"tie": (1, 10.0), "last": (size - m, 0.0), "over": (0, 95.0),
                            "split": (0 if m % 8 >= 4 else 1 + m % 3, 0.0)}[v]
                if m >= size:
                    act, cpu = 0, 0.0                                  # the least loaded of all, but not routable
                labels = {"grp": g, "hostname": "%s-%03d" % (g, m), "rack": "r%d" % (len(workers) % 2)}
                workers.append(kats.hb("%s-%03d" % (g, m), pool, act, cpu, 0.0, 0, labels))
    return POLICY, routing, workers


def long_jobs(workers):
    rng = random.Random(3)
    groups = {}
    for w in workers:
        if w["pool"] != "ghost":
            groups.setdefault(w["labels"]["grp"], []).append(w)
    jobs = []
    for g, ms in groups.items():
        for topic in ("job.any", "job.half"):
            jobs.append({"topic": topic, "labels": {"grp": g}})
            jobs.append({"topic": topic, "labels": {"grp": g, "rack": "r1"}})
        for _ in range(3):
            m = ms[rng.randrange(1, len(ms) - 1)]   # neither the lowest rank nor the least loaded
            # the long list first, the member's own one-holder list second: the shortest list is not sel[0]
            jobs.append({"topic": "job.any", "labels": {"grp": g, "hostname": m["labels"]["hostname"]}})
            jobs.append({"topic": "job.any", "labels": {"hostname": m["labels"]["hostname"], "grp": g}})
            o = rng.choice(workers)["labels"]["hostname"]
            jobs.append({"topic": "job.any", "labels": {"grp": g, "hostname": o}})   # mostly another group's member
            jobs.append({"topic": "job.any", "labels": {"grp": g, "preferred_worker_id": m["worker_id"]}})
    return jobs


def boundary_registry():
    """1,100 one-worker hosts (so the registry has more than 1,024 bits) and three groups: k with 32 routable holders
    (selective), l with 33 (dense), m with 32 routable holders plus five in a pool the routing table does not know
    (selective).  The pool c is known to the routing table but listed by no topic."""
    routing = {"topics": {"job.any": ["a", "b"]}, "pools": {"a": {}, "b": {}, "c": {}}}
    workers = [kats.hb("u%04d" % i, "ab"[i % 2], i % 3, 0.0, 0.0, 4, {"host": "h%04d" % i}) for i in range(1100)]
    workers += [kats.hb("k%02d" % i, "a", i % 2, 0.0, 0.0, 4, {"grp": "k"}) for i in range(MAX_HOLDERS)]
    workers += [kats.hb("l%02d" % i, "b", 0, 0.0, 0.0, 4, {"grp": "l"}) for i in range(MAX_HOLDERS + 1)]
    workers += [kats.hb("m%02d" % i, "a" if i < MAX_HOLDERS else "ghost", 1, 0.0, 0.0, 4, {"grp": "m"}) for i in range(MAX_HOLDERS + 5)]
    # n: 20 holders in a, 20 in c: 40 routable holders, 20 once c leaves the routing table
    workers += [kats.hb("n%02d" % i, "ac"[i % 2], i % 3, 0.0, 0.0, 4, {"grp": "n"}) for i in range(40)]
    return None, routing, workers


def boundary_jobs(workers):
    jobs = [{"topic": "job.any", "labels": {"grp": g}} for g in "klmn" for _ in range(3)]
    jobs += [{"topic": "job.any", "labels": {"grp": g, "host": "h%04d" % i}} for g in "klmn" for i in (0, 1)]
    jobs += [{"topic": "job.any", "labels": {"host": "h%04d" % i}} for i in range(0, 1100, 37)]
    jobs += [{"topic": "job.any", "labels": {"grp": g, "preferred_worker_id": "%s%02d" % (g, i)}} for g in "klmn" for i in (3, 33, 36)]
    return jobs


def threshold_registry(bits):
    """bits = the any bit + the host key + one pair per worker."""
    routing = {"topics": {"job.any": ["a", "b"]}, "pools": {"a": {}, "b": {}}}
    workers = [kats.hb("w%04d" % i, "ab"[i % 2], i % 3, 0.0, 0.0, 4, {"host": "h%04d" % i}) for i in range(bits - 2)]
    return None, routing, workers


def threshold_jobs(n_hosts):
    return [{"topic": "job.any", "labels": {"host": "h%04d" % i}} for i in range(0, n_hosts, 7)] + [{"topic": "job.any"}]


# ------------------------------------------------------------------ what a case reaches
def sel_list(T, s):
    return T["sel_pos"][T["sel_off"][s]:T["sel_off"][s + 1]]


def own_ids(T, pos):
    return set(T["pos_sel"][T["pos_sel_off"][pos]:T["pos_sel_off"][pos + 1]].tolist())


def shapes(T, cols, rec):
    """The selective shapes a batch reaches, from the host tables, its records and the reference's decisions `rec`
    (POLICY_AND_ROUTE)."""
    key, _, _ = table_walk._worker_pools(T)
    low = (1 << 128) - 1
    got = set()
    for j, ids in cols["sel_ids"].items():
        lens = [len(sel_list(T, s)) for s in ids]
        kmin = lens.index(min(lens))
        need = cols["place"][j]
        st = int(rec["route_status"][j])
        got.add("status %d" % st)
        if rec["flags"][j] & wire.F_TIE:
            got.add("tie")
        if len(ids) >= 3:
            got.add("three or more ids")
        if max(lens) > 32:
            got.add("list longer than a warp")
        if lens[0] > lens[kmin]:
            got.add("shortest list is not the first")
        if need >> 128:
            got.add("wide dense need")
        for pos in sel_list(T, ids[kmin]):
            mine = own_ids(T, pos)
            lab = T["pos_label"][pos]
            if set(ids) <= mine and (lab & need & low) == (need & low) and (lab & need) != need:
                got.add("holder rejected by a wide bit alone")
            if set(ids[:2]) <= mine and not set(ids) <= mine:
                got.add("holder rejected by the selective list alone")
        for pos in sel_list(T, ids[0]):
            if lens[0] > lens[kmin] and ids[kmin] not in own_ids(T, pos) and key[pos] != table_walk.KEY_NONE:
                got.add("first list has holders the shortest lacks")
        if st == wire.ROUTE_OK:
            pos = int(T["slot_pos"][rec["worker_slot"][j]]) - 1
            if list(sel_list(T, ids[kmin])).index(pos) >= 32:
                got.add("winner past the first 32 holders")
        pw = int(cols["pref_worker"][j])
        if pw and pw != table_walk.PREF_UNKNOWN and T["slot_pos"][pw - 1]:
            p1 = int(T["slot_pos"][pw - 1]) - 1
            if set(ids) <= own_ids(T, p1) and key[p1] == table_walk.KEY_NONE:
                got.add("preferred holder overloaded")
            if set(ids) <= own_ids(T, p1) and (T["pos_label"][p1] & need & low) == (need & low) and (T["pos_label"][p1] & need) != need:
                got.add("preferred holder lacks a wide bit")
            if set(ids[:2]) <= own_ids(T, p1) and not set(ids) <= own_ids(T, p1):
                got.add("preferred holder lacks an extra pin")
        if st == wire.ROUTE_NOT_ATTEMPTED:
            got.add("listed, route not attempted")
    return got


def analyse(policy, routing, workers, jobs, rec):
    h = sl.SelHarness(policy, routing, workers)
    T = h.tables()
    cols = h.encode(jobs)
    h.close()
    return T, cols, shapes(T, cols, rec)


WIDE_SHAPES = {"wide dense need", "holder rejected by a wide bit alone", "preferred holder overloaded",
               "preferred holder lacks a wide bit", "listed, route not attempted"} | {"status %d" % s for s in STATUSES}
PIN_SHAPES = {"three or more ids", "holder rejected by the selective list alone", "preferred holder lacks an extra pin"}
LONG_SHAPES = {"list longer than a warp", "shortest list is not the first", "first list has holders the shortest lacks",
               "winner past the first 32 holders", "tie", "preferred holder overloaded",
               "status %d" % wire.ROUTE_POOL_OVERLOADED, "status %d" % wire.ROUTE_OK, "status %d" % wire.ROUTE_OK_PREFERRED}


def check_wide_tables(T):
    assert T["n_sel"] >= 2 * N_WIDE - 100 and T["place_bits"] > 256 and T["xw_place"] >= 2, (T["n_sel"], T["place_bits"], T["xw_place"])


def check_long_tables(T):
    lens = np.diff(T["sel_off"])
    for size in SIZES:
        assert (lens == size).sum() == len(VARIANTS), size


# ------------------------------------------------------------------ CPU: the walk against the oracles
def walk_against_oracles(policy, routing, workers, jobs, n_py=0):
    h = sl.SelHarness(policy, routing, workers)
    o = oracle_lib.Oracle(policy, routing, workers)
    env = wire.EnvelopeBatch.from_jobs(jobs)
    for mode in MODES:
        want = o.eval(env, mode, threads=8)
        sl.assert_same(h.evaluate(env, mode), want, "mode %d" % mode)
    want = o.eval(env, PR, threads=8)
    if n_py:
        sample = jobs[:n_py]
        assert fuzz.rec_tuples(want[:n_py]) == fuzz.py_records(policy, routing, workers, sample)
    o.close()
    h.close()
    return want


def test_wide_dense_bits_next_to_selective_pairs():
    policy, routing, workers = wide_registry()
    jobs = wide_jobs(workers, 1200, seed=5)
    want = walk_against_oracles(policy, routing, workers, jobs, n_py=120)
    T, cols, got = analyse(policy, routing, workers, jobs, want)
    check_wide_tables(T)
    assert WIDE_SHAPES <= got, WIDE_SHAPES - got


def test_three_to_five_pins():
    policy, routing, workers = pins_registry()
    jobs = pins_jobs(workers)
    want = walk_against_oracles(policy, routing, workers, jobs, n_py=80)
    _, _, got = analyse(policy, routing, workers, jobs, want)
    assert PIN_SHAPES <= got, PIN_SHAPES - got


def test_holder_lists_longer_than_a_warp():
    sl.set_selective(0, max(SIZES))
    policy, routing, workers = long_registry()
    jobs = long_jobs(workers)
    want = walk_against_oracles(policy, routing, workers, jobs, n_py=100)
    T, cols, got = analyse(policy, routing, workers, jobs, want)
    check_long_tables(T)
    assert LONG_SHAPES <= got, LONG_SHAPES - got


# ------------------------------------------------------------------ GPU
def new_engine(policy, routing, workers):
    """An engine loaded under the limits in force now."""
    from cordum_b200 import engine

    e = engine.Engine(device=0)
    e.load_policy(policy, "seldiff")
    e.load_routing(routing)
    e.load_workers(workers)
    return e


def dense_records(policy, routing, workers, jobs):
    """The same inputs compiled with every pair dense: records of all three modes."""
    sl.set_selective(*DENSE)
    h = sl.SelHarness(policy, routing, workers)
    assert h.tables()["n_sel"] == 0
    h.close()
    e = new_engine(policy, routing, workers)
    b = e.batch(len(jobs))
    out = {m: b.encode(jobs).dispatch(m).copy() for m in MODES}
    e.close()
    sl.set_selective(MIN_BITS, MAX_HOLDERS)
    return out


def every_path(eng, o, jobs, loads, what, listed, plan=False):
    """Blocking dispatch in all three modes, async, resident, and two batches alternating ticks (the second routed by the
    flush), against the oracle.  `listed`: whether the batch lists selective jobs (route_select_kernel runs).  Returns
    the records of each mode."""
    import test_batch_plan

    env = wire.EnvelopeBatch.from_jobs(jobs)
    want = {m: o.eval(env, m, threads=8) for m in MODES}
    b = eng.batch(len(jobs))
    b.encode(env).dispatch()   # the first dispatch after a load also refreshes the worker tables
    for m in MODES:
        before = eng.launch_count()
        got = b.dispatch(m).copy()
        if m == PR:
            assert eng.launch_count() - before == (3 if listed else 2), what   # policy, route[, route_select]
            if plan:
                test_batch_plan.check_plan(eng, b, got, len(loads), what)
        sl.assert_same(got, want[m], "%s blocking mode %d" % (what, m))
    b.dispatch_async()
    sl.assert_same(b.wait().copy(), want[PR], what + " async")
    b.dispatch_resident()
    sl.assert_same(b.fetch().copy(), want[PR], what + " resident")
    rev = wire.EnvelopeBatch.from_jobs(jobs[::-1])
    c = eng.batch(len(jobs))
    sl.assert_same(c.encode(rev).dispatch().copy(), want[PR][::-1], what + " reversed")
    W = len(loads)
    b.tick(loads.ctypes.data, 0, W)
    c.tick(loads.ctypes.data, 0, W)
    b.wait()
    sl.assert_same(b.fetch().copy(), want[PR], what + " tick")
    eng.tick_flush()
    c.wait()
    sl.assert_same(c.fetch().copy(), want[PR][::-1], what + " tick flush")
    b.free()
    c.free()
    return want


def listed(policy, routing, workers, jobs):
    h = sl.SelHarness(policy, routing, workers)
    n = len(h.encode(jobs)["sel_ids"])
    h.close()
    return n


@pytest.mark.gpu
def test_wide_registry_through_the_kernels():
    policy, routing, workers = wide_registry()
    table = wire.WorkerTable.from_workers(workers)
    jobs = wide_jobs(workers, 2400, seed=7)
    o = oracle_lib.Oracle(policy, routing, table)
    T, cols, got = analyse(policy, routing, workers, jobs, o.eval(jobs, threads=8))
    check_wide_tables(T)
    assert WIDE_SHAPES <= got, WIDE_SHAPES - got
    eng = new_engine(policy, routing, table)
    want = every_path(eng, o, jobs, table.loads(), "wide", True, plan=True)
    # the device encoder hands a batch that names selective pairs to the host encoder, once per encode
    b = eng.batch(len(jobs))
    for m in MODES:
        before = eng.host_fallbacks()
        sl.assert_same(b.encode_device(jobs).dispatch(m).copy(), want[m], "device encode mode %d" % m)
        assert eng.host_fallbacks() - before == 1
    eng.close()
    dense = dense_records(policy, routing, table, jobs)
    for m in MODES:
        sl.assert_same(dense[m], want[m], "dense path mode %d" % m)
    o.close()


@pytest.mark.gpu
def test_pins_registry_through_the_kernels():
    policy, routing, workers = pins_registry()
    table = wire.WorkerTable.from_workers(workers)
    jobs = pins_jobs(workers)
    o = oracle_lib.Oracle(policy, routing, table)
    _, _, got = analyse(policy, routing, workers, jobs, o.eval(jobs, threads=8))
    assert PIN_SHAPES <= got, PIN_SHAPES - got
    eng = new_engine(policy, routing, table)
    want = every_path(eng, o, jobs, table.loads(), "pins", True, plan=True)
    b = eng.batch(len(jobs))
    before = eng.host_fallbacks()
    sl.assert_same(b.encode_device(jobs).dispatch().copy(), want[PR], "device encode")
    assert eng.host_fallbacks() - before == 1
    eng.close()
    dense = dense_records(policy, routing, table, jobs)
    for m in MODES:
        sl.assert_same(dense[m], want[m], "dense path mode %d" % m)
    o.close()


@pytest.mark.gpu
def test_long_holder_lists_through_the_kernels():
    sl.set_selective(0, max(SIZES))
    policy, routing, workers = long_registry()
    table = wire.WorkerTable.from_workers(workers)
    jobs = long_jobs(workers)
    o = oracle_lib.Oracle(policy, routing, table)
    T, _, got = analyse(policy, routing, workers, jobs, o.eval(jobs, threads=8))
    check_long_tables(T)
    assert LONG_SHAPES <= got, LONG_SHAPES - got
    eng = new_engine(policy, routing, table)
    loads = table.loads()
    every_path(eng, o, jobs, loads, "long lists", True, plan=True)
    # heartbeats move the least loaded holder of each "last" list from its end to its front, then to the middle
    probe = [{"topic": "job.any", "labels": {"grp": "last%03d" % s}} for s in SIZES]
    p = eng.batch(len(probe))
    p.encode(probe)
    for where in (0, 0.5):
        slots = []
        for size in SIZES:
            members = [i for i, w in enumerate(workers) if w["labels"]["grp"] == "last%03d" % size and w["pool"] != "ghost"]
            m = members[int(where * (len(members) - 1))]
            loads["active_jobs"][members] = size + 1
            loads["active_jobs"][m] = 0
            slots += members
        slots = np.array(slots, np.uint32)
        eng.update_workers(slots, loads[slots])
        o.update_workers(slots, loads[slots])
        got = p.dispatch().copy()
        want = o.eval(probe)
        sl.assert_same(got, want, "heartbeat to %s" % where)
        assert (want["route_status"] == wire.ROUTE_OK).all()
        assert [workers[s]["labels"]["hostname"][-3:] for s in want["worker_slot"]] == ["%03d" % int(where * (s - 1)) for s in SIZES]
    every_path(eng, o, jobs, loads, "long lists after heartbeats", True)
    eng.close()
    dense = dense_records(policy, routing, table, jobs)   # the registry's own loads, before the heartbeats
    o.close()
    o = oracle_lib.Oracle(policy, routing, table)
    for m in MODES:
        sl.assert_same(dense[m], o.eval(jobs, m, threads=8), "dense path mode %d" % m)
    o.close()


@pytest.mark.gpu
def test_holder_boundary_and_unrouted_pools_through_the_kernels():
    policy, routing, workers = boundary_registry()
    table = wire.WorkerTable.from_workers(workers)
    T = sl.SelHarness(policy, routing, workers).tables()
    lens = sorted(np.diff(T["sel_off"]).tolist())
    assert lens.count(MAX_HOLDERS) == 2 and lens.count(1) == 1100 and len(lens) == 1102   # k and m selective; l and n dense
    jobs = boundary_jobs(workers)
    o = oracle_lib.Oracle(policy, routing, table)
    eng = new_engine(policy, routing, table)
    want = every_path(eng, o, jobs, table.loads(), "32/33 holders", True)
    assert (want[PR]["route_status"] == wire.ROUTE_OK_PREFERRED).any() and (want[PR]["flags"] & wire.F_TIE).any()
    eng.close()
    o.close()


@pytest.mark.gpu
@pytest.mark.parametrize("bits", [1024, 1025])
def test_threshold_through_the_kernels(bits):
    policy, routing, workers = threshold_registry(bits)
    table = wire.WorkerTable.from_workers(workers)
    assert sl.SelHarness(policy, routing, workers).tables()["n_sel"] == (0 if bits == 1024 else bits - 2)
    jobs = threshold_jobs(bits - 2)
    o = oracle_lib.Oracle(policy, routing, table)
    eng = new_engine(policy, routing, table)
    want = every_path(eng, o, jobs, table.loads(), "%d bits" % bits, bits > 1024)   # at 1,024: no route_select launch
    eng.close()
    dense = dense_records(policy, routing, table, jobs)
    for m in MODES:
        sl.assert_same(dense[m], want[m], "dense path mode %d" % m)
    o.close()


@pytest.mark.gpu
def test_forced_limits_through_the_kernels():
    sl.set_selective(0, 3)
    policy, routing, workers = sl.registry(1300, 24, n_unique=3)
    table = wire.WorkerTable.from_workers(workers)
    jobs = sl.jobs_for(workers, 24, 600) + sl.multi_jobs(workers, (1, 2, 3))
    assert listed(policy, routing, workers, jobs) > 300
    o = oracle_lib.Oracle(policy, routing, table)
    eng = new_engine(policy, routing, table)
    want = every_path(eng, o, jobs, table.loads(), "(0, 3)", True)
    st = want[PR]["route_status"]
    assert all((st == s).any() for s in STATUSES) and (want[PR]["flags"] & wire.F_TIE).any()
    eng.close()
    o.close()


@pytest.mark.gpu
def test_fuzz_with_selective_pairs_through_the_kernels():
    """fuzz_case and life_cycle seeds with every pair of at most two routable holders selective."""
    sl.set_selective(0, 2)
    n_listed = 0
    for seed in range(8):
        policy, routing, workers, jobs = fuzz.fuzz_case(seed, 12)
        if not workers:
            continue
        table = wire.WorkerTable.from_workers(workers)
        n = listed(policy, routing, workers, jobs)
        n_listed += n
        o = oracle_lib.Oracle(policy, routing, table)
        eng = new_engine(policy, routing, table)
        every_path(eng, o, jobs, table.loads(), "fuzz seed %d" % seed, n > 0)
        eng.close()
        o.close()
    for seed in range(4):
        eng = o = None
        for step, (kind, payload, jobs) in enumerate(fuzz.life_cycle(seed)):
            if kind == "load":
                policy, routing, workers = payload
                o, eng = oracle_lib.Oracle(*payload), new_engine(*payload)
            elif kind == "heartbeat" and payload is not None:
                o.update_workers(*payload)
                eng.update_workers(*payload)
            elif kind == "workers":
                workers = payload
                o.load_workers(payload)
                eng.load_workers(payload)
            elif kind == "routing":
                routing = payload
                o.load_routing(payload)
                eng.load_routing(payload)
            elif kind == "policy":
                o.load_policy(payload)
                eng.load_policy(payload, "step%d" % step)
            b = eng.batch(len(jobs))
            h = sl.SelHarness(None, routing, workers)
            n_listed += len(h.encode(jobs)["sel_ids"])
            h.close()
            for m in MODES:
                sl.assert_same(b.encode(jobs).dispatch(m).copy(), o.eval(jobs, m), "life cycle %d step %d mode %d" % (seed, step, m))
            b.free()
        eng.close()
        o.close()
    assert n_listed > 10


@pytest.mark.gpu
def test_more_listed_jobs_than_one_grid():
    """A batch of 24,000 jobs, most of them listed: route_select_kernel's grid-stride loop runs more than one sweep."""
    policy, routing, workers = wide_registry()
    table = wire.WorkerTable.from_workers(workers)
    base = wide_jobs(workers, 3000, seed=9)
    pick = np.random.default_rng(5).integers(0, len(base), 24_000)
    jobs = [base[i] for i in pick]
    n = listed(policy, routing, workers, jobs)
    assert n > GRID_JOBS and n > len(jobs) // 2, n
    o = oracle_lib.Oracle(policy, routing, table)
    eng = new_engine(policy, routing, table)
    every_path(eng, o, jobs, table.loads(), "24,000 jobs", True)
    eng.close()
    o.close()


@pytest.mark.gpu
def test_tick_graphs_follow_the_selective_list():
    """Ticks are cached CUDA graphs keyed by the routed batch's listed-job count and the table generation.  Re-encode the
    routed batch between ticks: with the same size but a different number of listed jobs, then with the same number but
    enough extra ids that the selective list outgrows its buffer (a new allocation)."""
    policy, routing, workers = pins_registry()
    table = wire.WorkerTable.from_workers(workers)
    W = len(workers)
    U = sl.UNIQUE
    n = 400
    routable = [w for w in workers if w["pool"] != "ghost"][::2]
    one = [{"topic": "job.any", "labels": {"hostname": routable[i]["labels"]["hostname"]}} for i in range(n)]
    fewer = [j if k % 2 else {"topic": "job.any", "labels": {"zone": "z1"}} for k, j in enumerate(one)]
    five = [{"topic": "job.any", "labels": {k: routable[i]["labels"][k] for k in U}} for i in range(n)]
    plain = [{"topic": "job.any", "labels": {"rack": "r%02d" % (i % 16)}} for i in range(n)]
    h = sl.SelHarness(policy, routing, workers)
    cols = [h.encode(x) for x in (one, fewer, five)]
    h.close()
    assert [len(c["sel_ids"]) for c in cols] == [n, n // 2, n]
    assert len(cols[2]["_sel_extra"]) + 2 * n > 1024 > len(cols[0]["_sel_extra"]) + 2 * n   # the second outgrows the first
    o = oracle_lib.Oracle(policy, routing, table)
    eng = new_engine(policy, routing, table)
    loads = table.loads()
    b, c = eng.batch(n), eng.batch(n)
    c.encode(plain).dispatch()
    # two ticks a round and graphs per tick phase (the tick number mod 6): rounds 0, 3 and 6 share theirs, and so do 1 and 4
    for jobs in (one, one, fewer, fewer, five, five, one):
        b.encode(jobs).dispatch()   # a tick takes a batch that is resident on the device
        b.tick(loads.ctypes.data, 0, W)
        c.tick(loads.ctypes.data, 0, W)
        b.wait()
        sl.assert_same(b.fetch().copy(), o.eval(jobs), "tick")
        eng.tick_flush()
        c.wait()
        sl.assert_same(c.fetch().copy(), o.eval(plain), "tick flush")
    eng.close()
    o.close()


@pytest.mark.gpu
def test_routing_reloads_move_pairs_across_the_line():
    """Holders are routable workers: a routing reload that adds the pool of m's five unrouted holders makes m dense (37
    holders); one that drops pool c makes n selective (20 holders).  A batch encoded before each reload is refused, and
    encoded again it matches the oracle of the new tables."""
    from cordum_b200 import engine

    policy, routing, workers = boundary_registry()
    table = wire.WorkerTable.from_workers(workers)
    jobs = boundary_jobs(workers)
    more = {"topics": {"job.any": ["a", "b", "ghost"]}, "pools": {"a": {}, "b": {}, "c": {}, "ghost": {}}}
    fewer = {"topics": {"job.any": ["a", "b"]}, "pools": {"a": {}, "b": {}}}
    eng = new_engine(policy, routing, table)
    b = eng.batch(len(jobs))
    b.encode(jobs)
    o = oracle_lib.Oracle(policy, routing, table)
    sl.assert_same(b.dispatch().copy(), o.eval(jobs), "before")
    probe = [{"topic": "job.any", "labels": {"grp": g}} for g in "mn"]
    for r, sel_m, sel_n in ((more, False, False), (fewer, True, True), (routing, True, False)):
        h = sl.SelHarness(policy, r, workers)
        assert sorted(h.encode(probe)["sel_ids"]) == [j for j, s in enumerate((sel_m, sel_n)) if s]
        h.close()
        eng.load_routing(r)
        o.load_routing(r)
        with pytest.raises(engine.CordumError) as ei:
            b.dispatch()
        assert ei.value.code == E_STALE
        sl.assert_same(b.encode(jobs).dispatch().copy(), o.eval(jobs), "after routing %s" % sorted(r["pools"]))
    eng.close()
    o.close()
    # every route path on the last tables
    o = oracle_lib.Oracle(policy, fewer, table)
    eng = new_engine(policy, fewer, table)
    every_path(eng, o, jobs, table.loads(), "pool c dropped", True)
    eng.close()
    o.close()


@pytest.mark.gpu
def test_registry_reloads_cross_1024_bits():
    from cordum_b200 import engine

    _, routing, small = threshold_registry(1024)
    _, _, large = threshold_registry(1025)
    jobs = threshold_jobs(1023)
    eng = new_engine(None, routing, small)
    o = oracle_lib.Oracle(None, routing, small)
    b = eng.batch(len(jobs))
    b.encode(jobs)
    for workers, listed_after in ((large, True), (small, False), (large, True)):
        eng.load_workers(workers)
        o.load_workers(workers)
        with pytest.raises(engine.CordumError) as ei:
            b.dispatch()
        assert ei.value.code == E_STALE
        b.encode(jobs).dispatch()
        before = eng.launch_count()
        got = b.dispatch().copy()
        assert eng.launch_count() - before == (3 if listed_after else 2)
        sl.assert_same(got, o.eval(jobs), "after loading %d workers" % len(workers))
    eng.close()
    o.close()
