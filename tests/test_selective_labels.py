"""Selective placement pairs: labels that only a few workers carry (hostname-style, `hostname=node-17342`), in a registry
whose placement labels need more than CORDUM_SEL_MIN_BITS (1,024) bits.  Such a pair gets no dense bit, bitmap row or
side-row bit per job; it gets the list of routable workers that carry it (tables.h DeviceTables.sel_*), the job records
name it by id (JobRec.sel + the batch's selective list), and route_select_kernel picks among its holders.  Reference
semantics: strategy_least_loaded.go:40-136 (route), :161-175 (matchesLabels), :241-265 (poolSatisfies).

CPU: the new tables and the host encoder's records, walked in Python the way route_select_kernel walks them, against the C++
and the Python oracle.  GPU: the kernels against the C++ oracle, both encoders, all three modes, the load paths and the
dense path forced on the same inputs.  cordum_test_set_selective moves the limits so both paths run on the same registry."""
import ctypes as C
import random

import numpy as np
import pytest

import kats
import oracle_lib
import table_walk
import test_fuzz_three_way as fuzz
from cordum_b200 import wire

FIELDS = ("decision", "sched_decision", "flags", "route_status", "reason_code", "rule_idx", "worker_slot")
JF_SELECTIVE = 0x10000
MIN_BITS, MAX_HOLDERS = 1024, 32          # tables.h CORDUM_SEL_MIN_BITS / CORDUM_SEL_MAX_HOLDERS
DENSE = (0xFFFFFFFF, MAX_HOLDERS)         # no registry has that many bits: the dense path everywhere
MODES = (wire.MODE_POLICY_AND_ROUTE, wire.MODE_POLICY_ONLY, wire.MODE_ROUTE_ONLY)


def set_selective(min_bits, max_holders):
    from cordum_b200 import _lib

    L = _lib.load()
    L.cordum_test_set_selective.argtypes = [C.c_uint32, C.c_uint32]
    L.cordum_test_set_selective.restype = None
    L.cordum_test_set_selective(min_bits, max_holders)


@pytest.fixture(autouse=True)
def default_limits():
    set_selective(MIN_BITS, MAX_HOLDERS)
    yield
    set_selective(MIN_BITS, MAX_HOLDERS)


def assert_same(got, want, what=""):
    assert len(got) == len(want)
    for f in FIELDS:
        bad = np.nonzero(got[f] != want[f])[0]
        assert len(bad) == 0, "%s field %s differs at %d jobs, first %s: got %s want %s" % (
            what, f, len(bad), bad[:8], got[f][bad[:8]], want[f][bad[:8]])


# ------------------------------------------------------------------ the Python walk of the new tables
class SelHarness(table_walk.HostHarness):
    """table_walk's host harness plus the selective tables and the batch's selective list."""

    def tables(self):
        T = super().tables()
        for name in ("sel_off", "sel_pos", "pos_sel_off", "pos_sel"):
            ptr, nbytes = C.c_void_p(), C.c_uint64()
            self._ck(self.L.cordum_test_host_table(self.h, name.encode(), C.byref(ptr), C.byref(nbytes)))
            T[name] = np.frombuffer((C.c_uint8 * nbytes.value).from_address(ptr.value), np.uint32).copy() if nbytes.value else np.zeros(0, np.uint32)
        for s in ("n_sel", "lbm_words"):
            T[s] = int(self.L.cordum_test_host_scalar(self.h, s.encode()))
        return T

    def encode(self, env):
        cols = super().encode(env)
        L = self.L
        L.cordum_test_host_sel.argtypes = [C.c_int32, C.POINTER(C.c_void_p), C.POINTER(C.c_uint64)]
        got = []
        for which in (0, 1):
            ptr, nbytes = C.c_void_p(), C.c_uint64()
            L.cordum_test_host_sel(which, C.byref(ptr), C.byref(nbytes))
            got.append(np.frombuffer((C.c_uint8 * nbytes.value).from_address(ptr.value), np.uint32).copy() if nbytes.value else np.zeros(0, np.uint32))
        cols["_sel_jobs"], cols["_sel_extra"] = got[0].reshape(-1, 2), got[1]
        cols["sel_ids"] = selective_ids(cols)
        return cols

    def evaluate(self, env, mode=wire.MODE_POLICY_AND_ROUTE):
        cols = self.encode(env)
        T = self.tables()
        return walk(T, cols, table_walk.walk(T, cols, mode))


def selective_ids(cols):
    """caller job -> its selective pair ids, from JobRec.sel and the selective list (tables.h JobRecords)."""
    job, extra = cols["_job"], cols["_sel_extra"]
    out = {}
    prev = -1
    for slot, x in cols["_sel_jobs"]:
        assert slot > prev, "the selective list is not in ascending slot order"
        prev = slot
        r = job[slot]
        assert r["flags"] & JF_SELECTIVE and r["flags"] & table_walk.JF_PLACE_UNSAT
        ids = [int(r["spare"][0]) - 1] + ([int(r["spare"][1]) - 1] if r["spare"][1] else [])
        if x:
            assert len(ids) == 2
            ids += [int(v) for v in extra[x + 1: x + 1 + extra[x]]]
        out[int(r["orig"])] = ids
    flagged = {int(o) for o, f in zip(job["orig"], job["flags"]) if f & JF_SELECTIVE}
    assert flagged == set(out), "the selective list and the JF_SELECTIVE flags disagree"
    return out


def walk(T, cols, out):
    """route_select_kernel: jobs route_kernel left at NO_WORKERS that name selective pairs."""
    key, _, _ = table_walk._worker_pools(T)
    for j, ids in cols["sel_ids"].items():
        if out[j]["route_status"] != wire.ROUTE_NO_WORKERS:
            continue
        flags, topic = int(cols["flags"][j]), int(cols["topic"][j])
        off, cnt = int(T["topic_pool_off"][topic]), int(T["topic_pool_cnt"][topic])
        pools = {int(p) for p in T["pool_list"][off:off + cnt]}
        if cols["pref_pool"][j]:
            pools = {int(cols["pref_pool"][j]) - 1}
        need_req = int(cols["req_pool"][j]) & ~T["req_blank_mask"]
        need_pl = int(cols["place"][j])

        def pool_ok(p):
            if p not in pools:
                return False
            if not flags & table_walk.JF_REQ_NONEMPTY:
                return True
            return bool(T["pool_req_nonempty"][p]) and not flags & table_walk.JF_REQ_UNKNOWN and (need_req & ~int(T["pool_req_mask"][p])) == 0

        def carries(pos):
            own = set(T["pos_sel"][T["pos_sel_off"][pos]:T["pos_sel_off"][pos + 1]].tolist())
            return (T["pos_label"][pos] & need_pl) == need_pl and set(ids) <= own

        route, slot, tie = wire.ROUTE_NO_WORKERS, -1, False
        pw = int(cols["pref_worker"][j])
        p1 = int(T["slot_pos"][pw - 1]) if pw and pw != table_walk.PREF_UNKNOWN else 0
        if p1 and pool_ok(int(T["pos_pool"][p1 - 1])) and carries(p1 - 1) and key[p1 - 1] != table_walk.KEY_NONE:
            route, slot = wire.ROUTE_OK_PREFERRED, pw - 1
        else:
            short = min(ids, key=lambda s: T["sel_off"][s + 1] - T["sel_off"][s])
            best, bcnt, total = table_walk.KEY_NONE, 0, 0
            for pos in T["sel_pos"][T["sel_off"][short]:T["sel_off"][short + 1]]:
                if pool_ok(int(T["pos_pool"][pos])) and carries(pos):
                    total += 1
                    best, bcnt = table_walk._merge(best, bcnt, key[pos], 1)
            if best != table_walk.KEY_NONE:
                route, slot, tie = wire.ROUTE_OK, int(T["rank_slot"][best & 0xFFFFFFFF]), bcnt > 1
            elif total:
                route = wire.ROUTE_POOL_OVERLOADED
        out[j]["route_status"] = route
        out[j]["worker_slot"] = slot
        out[j]["flags"] |= wire.F_TIE if tie else 0
    return out


# ------------------------------------------------------------------ registries and jobs
UNIQUE = ("hostname", "instance", "serial", "uuid", "mac")   # one value per worker each


def registry(n_workers, n_pools, seed=1, n_unique=2, n_second=None, groups=(2, 3, 7, 16, 31, 32, 33, 40)):
    """Every worker: a hostname, up to n_unique - 1 further labels of its own (the first n_second workers only, when given),
    a shared zone and rack; workers 0.. also belong to `svc` groups of the given sizes (equal loads inside a group: ties).
    A few workers sit in a pool the routing table does not know."""
    rng = random.Random(seed)
    pools = ["p%03d" % p for p in range(n_pools)]
    routing = {"topics": {"job.any": pools, "job.half": pools[: n_pools // 2], "job.one": pools[1:2]},
               "pools": {p: ({"requires": ["gpu"]} if i % 4 == 0 else {}) for i, p in enumerate(pools)}}
    svc = {}
    w = 0
    for g, size in enumerate(groups):
        for _ in range(size):
            svc[w] = "s%02d" % g
            w += 1
    workers = []
    for i in range(n_workers):
        labels = {k: "%s-%05d" % (k[:4], i) for u, k in enumerate(UNIQUE[:n_unique]) if u == 0 or n_second is None or i < n_second}
        labels["zone"], labels["rack"] = "z%d" % (i % 4), "r%02d" % (i % 16)
        if i in svc:
            labels["svc"] = svc[i]
        pool = pools[(i * 7) % n_pools] if i % 97 != 5 else "ghost"
        if i in svc:
            act, cpu = 1, 10.0
        else:
            act, cpu = rng.randrange(3), float(rng.choice([0, 10, 20, 95]))
        workers.append(kats.hb("w%05d" % i, pool, act, cpu, 0.0, 8, labels))
    return {"default_tenant": "default", "rules": [{"id": "deny-x", "decision": "deny", "match": {"topics": ["job.x"]}}]}, routing, workers


def jobs_for(workers, n_pools, n=400, seed=2, n_second=None):
    rng = random.Random(seed)
    W = len(workers)
    n_second = n_second or W
    host = lambda i: workers[i]["labels"]["hostname"]   # noqa: E731
    jobs = []
    for t in range(n):
        i = rng.randrange(W)
        lab = workers[i]["labels"]
        kind = t % 20
        topic = rng.choice(["job.any", "job.any", "job.half", "job.one"])
        j = {"topic": topic, "labels": {"hostname": host(i)}}
        if kind == 1:
            j["labels"]["zone"] = lab["zone"]                        # host + zone that match
        elif kind == 2:
            j["labels"]["zone"] = "z%d" % ((i + 1) % 4)              # ... that conflict
        elif kind == 3:
            j["labels"]["gpu"] = ""                                  # host + k: "" (nobody carries gpu)
        elif kind == 4:
            j["labels"]["rack"] = ""                                 # host + k: "" on a key everybody carries
        elif kind == 5:
            j["labels"]["instance"] = workers[rng.randrange(n_second)]["labels"]["instance"]    # two hosts, mostly
        elif kind == 6:
            j["labels"] = {"svc": "s%02d" % rng.randrange(8)}          # a shared pair: ties, the lowest rank wins
        elif kind == 7:
            j["labels"]["preferred_worker_id"] = workers[i]["worker_id"]             # preferred worker: a holder
        elif kind == 8:
            j["labels"]["preferred_worker_id"] = workers[rng.randrange(W)]["worker_id"]   # ... mostly a non-holder
        elif kind == 9:
            j["labels"]["preferred_pool"] = workers[i]["pool"] if rng.random() < 0.7 else "p%03d" % rng.randrange(n_pools)
        elif kind == 10:
            j["meta"] = {"requires": ["gpu"]}                        # behind requires
        elif kind == 11:
            j["labels"]["hostname"] = "node-unknown"                 # a pair no routable worker carries
        elif kind == 12:
            j["labels"]["other"] = "nobody"                          # selective pair + unknown pair
        elif kind == 13:
            j["labels"] = {"svc": "s%02d" % rng.randrange(8), "zone": "z%d" % rng.randrange(4), "preferred_worker_id": workers[rng.randrange(40)]["worker_id"]}
        elif kind == 14:
            j["topic"] = ""                                          # missing topic
        elif kind == 15:
            j["topic"] = "job.x"                                     # denied by policy: not routed
        elif kind == 16:
            j["labels"] = {"zone": lab["zone"]}                      # dense only
        elif kind == 17:
            j["labels"] = {}
        jobs.append(j)
    return jobs


def multi_jobs(workers, counts=(1, 2, 3, 5), n_unique=5):
    """Jobs naming 1, 2, 3 and 5 selective pairs of one worker, and the same with one pair of another worker."""
    out = []
    for c in counts:
        for i in range(0, len(workers), max(1, len(workers) // 7)):
            lab = {k: workers[i]["labels"][k] for k in UNIQUE[:c]}
            out.append({"topic": "job.any", "labels": dict(lab)})
            other = dict(lab)
            other[UNIQUE[c - 1]] = workers[(i + 1) % len(workers)]["labels"][UNIQUE[c - 1]]
            out.append({"topic": "job.any", "labels": other})
            out.append({"topic": "job.any", "labels": dict(lab, zone=workers[i]["labels"]["zone"], preferred_worker_id=workers[i]["worker_id"])})
    return out


# ------------------------------------------------------------------ CPU: tables and records
def test_holder_count_boundary_and_unknown_pools():
    """K holders: selective; K+1: dense.  Holders in a pool the routing table does not know do not count."""
    pools = ["a", "b"]
    routing = {"topics": {"job.any": pools}, "pools": {p: {} for p in pools}}
    workers = [kats.hb("u%04d" % i, pools[i % 2], 0, 0.0, 0.0, 4, {"host": "h%04d" % i}) for i in range(1100)]
    workers += [kats.hb("k%02d" % i, "a", 0, 0.0, 0.0, 4, {"grp": "k"}) for i in range(MAX_HOLDERS)]
    workers += [kats.hb("l%02d" % i, "b", 0, 0.0, 0.0, 4, {"grp": "l"}) for i in range(MAX_HOLDERS + 1)]
    # 32 routable holders plus five outside the routing table: still selective
    workers += [kats.hb("m%02d" % i, "a" if i < MAX_HOLDERS else "ghost", 0, 0.0, 0.0, 4, {"grp": "m"}) for i in range(MAX_HOLDERS + 5)]
    h = SelHarness(None, routing, workers)
    T = h.tables()
    # dense: the any bit, keys host / grp, the pair grp=l
    assert T["place_bits"] == 4 and T["n_sel"] == 1100 + 2
    lens = np.diff(T["sel_off"])
    assert sorted(lens.tolist()).count(MAX_HOLDERS) == 2 and (lens == 1).sum() == 1100
    jobs = [{"topic": "job.any", "labels": {"grp": g}} for g in "klm"] + [{"topic": "job.any", "labels": {"host": "h0007"}}]
    cols = h.encode(jobs)
    assert set(cols["sel_ids"]) == {0, 2, 3} and not cols["flags"][1] & JF_SELECTIVE
    o = oracle_lib.Oracle(None, routing, workers)
    for mode in MODES:
        assert_same(h.evaluate(jobs, mode), o.eval(jobs, mode, threads=8), "mode %d" % mode)
    o.close()
    h.close()


def dense_tables(policy, routing, workers):
    set_selective(*DENSE)
    h = SelHarness(policy, routing, workers)
    T = h.tables()
    h.close()
    set_selective(MIN_BITS, MAX_HOLDERS)
    return T


@pytest.mark.parametrize("bits", [1024, 1025])
def test_threshold_is_1024_placement_bits(bits):
    """bits = any + the host key + one pair per worker: at 1,024 the tables are the dense ones byte for byte, at 1,025 the
    host pairs are selective."""
    routing = {"topics": {"job.any": ["a", "b"]}, "pools": {"a": {}, "b": {}}}
    workers = [kats.hb("w%04d" % i, "ab"[i % 2], i % 3, 0.0, 0.0, 4, {"host": "h%04d" % i}) for i in range(bits - 2)]
    h = SelHarness(None, routing, workers)
    T, D = h.tables(), dense_tables(None, routing, workers)
    if bits == 1024:
        assert T["n_sel"] == 0 and T["place_bits"] == 1024
        for k, v in D.items():
            if isinstance(v, np.ndarray):
                assert np.array_equal(v, T[k]), k
            else:
                assert v == T[k], k
    else:
        assert T["n_sel"] == bits - 2 and T["place_bits"] == 2 and T["xw_place"] == 0 and D["xw_place"] > 0
        assert T["lbm_words"] * 500 < D["lbm_words"]   # place_bits rows per pool: 2 against 1,025
        assert np.array_equal(np.diff(T["sel_off"]), np.ones(bits - 2)) and np.array_equal(np.diff(T["pos_sel_off"]), np.ones(bits - 2))
        # pair id -> its one holder, and back
        assert np.array_equal(T["pos_sel"][T["sel_pos"]], np.arange(bits - 2))
    jobs = [{"topic": "job.any", "labels": {"host": "h%04d" % i}} for i in range(0, bits - 2, 13)]
    o = oracle_lib.Oracle(None, routing, workers)
    assert_same(h.evaluate(jobs), o.eval(jobs, threads=8))
    o.close()
    h.close()


def test_capacity_refusal_and_rollback_unchanged():
    """65,536 keys + pairs is still the limit, refused transactionally, whether or not the pairs could be selective."""
    routing = {"topics": {"job.any": ["a"]}, "pools": {"a": {}}}
    good = [kats.hb("w%04d" % i, "a", 0, 0.0, 0.0, 4, {"host": "h%04d" % i}) for i in range(1500)]
    h = SelHarness(None, routing, good)
    before = h.tables()
    assert before["n_sel"] == 1500
    big = [kats.hb("x%05d" % i, "a", 0, 0.0, 0.0, 4, {"key%05d" % i: "v"}) for i in range(33000)]
    with pytest.raises(RuntimeError, match="65536"):
        h.load_workers(big)
    after = h.tables()
    for k, v in before.items():
        assert np.array_equal(v, after[k]) if isinstance(v, np.ndarray) else v == after[k], k
    jobs = [{"topic": "job.any", "labels": {"host": "h0042"}}]
    o = oracle_lib.Oracle(None, routing, good)
    assert_same(h.evaluate(jobs), o.eval(jobs, threads=8))
    o.close()
    h.close()


def test_records_name_their_selective_pairs():
    """0/1/2/3/5 selective pairs on one job; a selective pair with an unknown pair; k: "" next to a selective pair."""
    policy, routing, workers = registry(1200, 16, n_unique=5)
    h = SelHarness(policy, routing, workers)
    T = h.tables()
    assert T["n_sel"] >= 5 * 1150 and T["place_bits"] <= 128 and T["xw_place"] == 0
    w = workers[500]["labels"]
    jobs = [{"topic": "job.any", "labels": {"zone": w["zone"]}}]
    jobs += [{"topic": "job.any", "labels": {k: w[k] for k in UNIQUE[:c]}} for c in (1, 2, 3, 5)]
    jobs += [{"topic": "job.any", "labels": {"hostname": w["hostname"], "other": "nobody"}},
             {"topic": "job.any", "labels": {"hostname": w["hostname"], "gpu": ""}}]
    cols = h.encode(jobs)
    sel = cols["sel_ids"]
    assert 0 not in sel and 5 not in sel and not cols["flags"][0] & table_walk.JF_PLACE_UNSAT
    assert cols["flags"][5] & table_walk.JF_PLACE_UNSAT and not cols["flags"][5] & JF_SELECTIVE
    assert [len(sel[j]) for j in (1, 2, 3, 4, 6)] == [1, 2, 3, 5, 1]
    pos = int(T["slot_pos"][500]) - 1
    own = set(T["pos_sel"][T["pos_sel_off"][pos]:T["pos_sel_off"][pos + 1]].tolist())
    assert set(sel[4]) == own and all(set(sel[j]) <= own for j in (1, 2, 3, 6))
    assert cols["place"][6] != 0 and cols["place"][1] == 0   # k: "" keeps its dense bit
    x = cols["_sel_jobs"][:, 1]
    assert (x != 0).sum() == 2 and cols["_sel_extra"][0] == 0   # the jobs with 3 and 5 pairs use the extra words
    jobs += multi_jobs(workers)
    o = oracle_lib.Oracle(policy, routing, workers)
    for mode in MODES:
        assert_same(h.evaluate(jobs, mode), o.eval(jobs, mode, threads=8), "mode %d" % mode)
    o.close()
    h.close()


@pytest.mark.parametrize("limits", [(MIN_BITS, MAX_HOLDERS), DENSE, (0, 3)], ids=["default", "dense", "forced"])
def test_hostname_registry_matches_the_oracle(limits):
    set_selective(*limits)
    policy, routing, workers = registry(1300, 24)
    jobs = jobs_for(workers, 24, 500) + multi_jobs(workers, (1, 2))
    h = SelHarness(policy, routing, workers)
    T = h.tables()
    assert (T["n_sel"] > 0) == (limits != DENSE)
    cols = h.encode(jobs)
    assert (len(cols["sel_ids"]) > 100) == (limits != DENSE)
    o = oracle_lib.Oracle(policy, routing, workers)
    for mode in MODES:
        want = o.eval(jobs, mode, threads=8)
        assert_same(h.evaluate(jobs, mode), want, "mode %d" % mode)
    st = want["route_status"]
    for s in (wire.ROUTE_OK, wire.ROUTE_OK_PREFERRED, wire.ROUTE_NO_WORKERS, wire.ROUTE_POOL_OVERLOADED, wire.ROUTE_NO_POOL_REQUIRES):
        assert (st == s).any(), s
    assert (want["flags"] & wire.F_TIE).any()
    o.close()
    h.close()


@pytest.mark.parametrize("seed", range(24))
def test_fuzz_three_way_with_selective_pairs(seed):
    """The three-way fuzz configurations with every pair of at most two routable holders made selective: walk == C++ oracle
    == Python oracle (oracle/py_oracle.py, through the fuzz module's py_records)."""
    set_selective(0, 2)
    policy, routing, workers, jobs = fuzz.fuzz_case(seed, 12)
    h = SelHarness(policy, routing, workers)
    got = h.evaluate(jobs, wire.MODE_POLICY_AND_ROUTE)
    o = oracle_lib.Oracle(policy, routing, workers)
    assert_same(got, o.eval(jobs, threads=8), "seed %d" % seed)
    assert fuzz.rec_tuples(got) == fuzz.py_records(policy, routing, workers, jobs)
    o.close()
    h.close()


def test_fuzz_selects_something():
    set_selective(0, 2)
    n = 0
    for seed in range(24):
        policy, routing, workers, jobs = fuzz.fuzz_case(seed, 12)
        h = SelHarness(policy, routing, workers)
        n += len(h.encode(jobs)["sel_ids"])
        h.close()
    assert n > 50


# ------------------------------------------------------------------ GPU
GPU_WORKERS, GPU_POOLS, GPU_SECOND = 60000, 256, 2000


@pytest.fixture(scope="module")
def big():
    # 60,000 hostnames and 2,000 instance ids: keys + pairs stay below the 65,536 the label dictionary holds
    policy, routing, workers = registry(GPU_WORKERS, GPU_POOLS, seed=5, n_second=GPU_SECOND)
    table = wire.WorkerTable.from_workers(workers)
    jobs = jobs_for(workers, GPU_POOLS, 2000, seed=6, n_second=GPU_SECOND) + multi_jobs(workers[:GPU_SECOND], (1, 2))
    o = oracle_lib.Oracle(policy, routing, table)
    yield policy, routing, workers, table, jobs, o
    o.close()


@pytest.fixture(scope="module")
def eng(big):
    from cordum_b200 import engine

    policy, routing, _, table, _, _ = big
    e = engine.Engine(device=0)
    e.load_policy(policy, "sel")
    e.load_routing(routing)
    e.load_workers(table)
    yield e
    e.close()


@pytest.mark.gpu
@pytest.mark.parametrize("device_encode", [False, True], ids=["host-encode", "device-encode"])
def test_hostname_registry_through_the_kernels(big, eng, device_encode):
    _, _, _, table, jobs, o = big
    h = SelHarness(*big[:2], table)
    T = h.tables()
    assert T["n_sel"] >= GPU_WORKERS + GPU_SECOND - 700 and T["place_bits"] <= 128
    assert len(h.encode(jobs)["sel_ids"]) > 1000
    h.close()
    b = eng.batch(len(jobs))
    for mode in MODES:
        before = eng.host_fallbacks()
        enc = b.encode_device(jobs) if device_encode else b.encode(jobs)
        got = enc.dispatch(mode).copy()
        assert eng.host_fallbacks() - before == (1 if device_encode else 0)
        want = o.eval(jobs, mode, threads=8)
        assert_same(got, want, "mode %d" % mode)
        if mode != wire.MODE_POLICY_ONLY:
            st = want["route_status"]
            for s in (wire.ROUTE_OK, wire.ROUTE_OK_PREFERRED, wire.ROUTE_NO_WORKERS, wire.ROUTE_POOL_OVERLOADED):
                assert (st == s).any(), s
            assert (want["flags"] & wire.F_TIE).any()
    # resident and async dispatch of the same records
    b.dispatch_resident()
    assert_same(b.fetch().copy(), o.eval(jobs, threads=8), "resident")
    b.dispatch_async()
    assert_same(b.wait().copy(), o.eval(jobs, threads=8), "async")
    b.free()


@pytest.mark.gpu
def test_device_encoder_keeps_batches_without_selective_pairs(big, eng):
    """A batch that names no selective pair stays on the device (the dense part fits the records); one that does falls back
    exactly once."""
    _, _, workers, _, _, o = big
    plain = [{"topic": "job.any", "labels": {"zone": "z%d" % (i % 4), "rack": "r%02d" % (i % 16)}} for i in range(2000)]
    # s07: 40 routable holders, a dense pair (s06 has 33 members, one of them outside the routing table: selective)
    plain += [{"topic": "job.half", "labels": {"svc": "s07"}}, {"topic": "job.any"}, {"topic": "job.any", "labels": {"gpu": ""}}]
    b = eng.batch(len(plain) + 1)
    before = eng.host_fallbacks()
    assert_same(b.encode_device(plain).dispatch().copy(), o.eval(plain), "dense only")
    assert eng.host_fallbacks() == before
    pinned = plain + [{"topic": "job.any", "labels": {"hostname": workers[77]["labels"]["hostname"]}}]
    assert_same(b.encode_device(pinned).dispatch().copy(), o.eval(pinned), "one pinned job")
    assert eng.host_fallbacks() == before + 1
    b.free()


@pytest.mark.gpu
def test_launches_heartbeats_reload_and_ticks(big, eng):
    """route_select_kernel is one more launch where a batch lists selective jobs; heartbeat deltas move the winner of a
    shared pair; a reload that moves a hostname makes encoded batches stale and then routes to the new holder; ticks."""
    policy, routing, workers, table, jobs, o = big
    W = len(workers)
    b = eng.batch(len(jobs))
    b.encode(jobs).dispatch()
    before = eng.launch_count()
    got = b.dispatch().copy()
    assert eng.launch_count() - before == 3        # policy, route, route_select
    assert_same(got, o.eval(jobs, threads=8), "baseline")
    plain = [{"topic": "job.any", "labels": {"zone": "z1"}}] * 64
    c = eng.batch(len(plain))
    c.encode(plain).dispatch()
    before = eng.launch_count()
    c.dispatch()
    assert eng.launch_count() - before == 2        # nothing listed: no route_select launch
    # heartbeats: the members of svc group s03 (7 workers, equal loads) get distinct loads, then the order flips
    grp = [i for i, w in enumerate(workers) if w["labels"].get("svc") == "s03"]
    probe = [{"topic": "job.any", "labels": {"svc": "s03"}}] * 8 + [{"topic": "job.any", "labels": {"hostname": workers[g]["labels"]["hostname"]}} for g in grp]
    p = eng.batch(len(probe))
    p.encode(probe)
    loads = table.loads()
    for flip in (False, True):
        for r, g in enumerate(grp):
            loads["active_jobs"][g] = (len(grp) - r) if flip else r
            loads["cpu_load"][g] = 0.0
        slots = np.array(grp, np.uint32)
        eng.update_workers(slots, loads[grp])
        o.update_workers(slots, loads[grp])
        got = p.dispatch().copy()
        assert_same(got, o.eval(probe), "heartbeat flip=%s" % flip)
        assert got["worker_slot"][0] == (grp[-1] if flip else grp[0])
    # ticks over the same loads
    all_slots = np.arange(W, dtype=np.uint32)
    b.dispatch()
    p.dispatch()
    b.tick(loads.ctypes.data, 0, W)
    p.tick(loads.ctypes.data, 0, W)
    o.update_workers(all_slots, loads)
    b.wait()
    assert_same(b.fetch().copy(), o.eval(jobs, threads=8), "tick")
    eng.tick_flush()
    p.wait()
    assert_same(p.fetch().copy(), o.eval(probe), "tick flush")
    # a reload that moves a hostname to another worker
    from cordum_b200 import engine

    moved = [dict(w, labels=dict(w["labels"])) for w in workers]
    a, z = grp[-1], grp[-2]                         # the two least loaded members after the flip
    moved[a]["labels"]["hostname"], moved[z]["labels"]["hostname"] = workers[z]["labels"]["hostname"], workers[a]["labels"]["hostname"]
    for w, L in zip(moved, loads):
        w["active_jobs"], w["cpu_load"] = int(L["active_jobs"]), float(L["cpu_load"])
    mt = wire.WorkerTable.from_workers(moved)
    eng.load_workers(mt)
    with pytest.raises(engine.CordumError):
        p.dispatch()                                # encoded under the previous registry
    o2 = oracle_lib.Oracle(policy, routing, mt)
    got = p.encode(probe).dispatch().copy()
    assert_same(got, o2.eval(probe), "after the reload")
    assert got["worker_slot"][8 + grp.index(a)] == z
    eng.load_workers(table)                         # the module's registry and loads again
    o.load_workers(table)
    o2.close()
    for x in (b, c, p):
        x.free()


@pytest.mark.gpu
def test_dense_path_gives_identical_records(big):
    from cordum_b200 import engine

    policy, routing, workers, table, jobs, o = big
    jobs = jobs[:1500]
    out = {}
    for name, limits in (("selective", (MIN_BITS, MAX_HOLDERS)), ("dense", DENSE)):
        set_selective(*limits)
        e = engine.Engine(device=0)
        e.load_policy(policy, name)
        e.load_routing(routing)
        e.load_workers(table)
        b = e.batch(len(jobs))
        out[name] = {m: b.encode(jobs).dispatch(m).copy() for m in MODES}
        b.free()
        e.close()
    for m in MODES:
        assert_same(out["selective"][m], out["dense"][m], "mode %d" % m)
        assert_same(out["selective"][m], o.eval(jobs, m), "oracle mode %d" % m)


@pytest.mark.gpu
@pytest.mark.slow
def test_million_jobs_against_the_hostname_registry(big, eng):
    """A batch the dense encoding refuses (7.5 KB of side row per job) completes and matches the oracle."""
    _, _, workers, _, jobs, o = big
    rng = np.random.default_rng(3)
    base = jobs_for(workers, GPU_POOLS, 4000, seed=9, n_second=GPU_SECOND)
    pick = rng.integers(0, len(base), 1_000_000)
    env = wire.EnvelopeBatch.from_jobs([base[i] for i in pick])
    b = eng.batch(env.n_jobs)
    got = b.encode(env).dispatch().copy()
    assert_same(got, o.eval(base, threads=16)[pick], "1M jobs")   # a record depends on its own job only
    b.free()
