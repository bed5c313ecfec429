"""CPU tests of the PRODUCT's host side (table compiler + encoder, cordum_b200/csrc/host.cpp):
the compiled tables + encoded columns, re-walked the way kernels.cu walks them
(tests/table_walk.py), must reproduce the oracle's decision records bit for bit.
No GPU, no compute through the C ABI's dispatch calls."""
import numpy as np
import pytest

import kats
import oracle_lib
import table_walk
from cordum_b200 import synth, wire

FIELDS = ("decision", "sched_decision", "flags", "route_status", "reason_code", "rule_idx", "worker_slot")


def assert_same(got, want, what=""):
    for f in FIELDS:
        bad = np.nonzero(got[f] != want[f])[0]
        assert len(bad) == 0, "%s field %s differs at jobs %s: got %s want %s" % (
            what, f, bad[:8], got[f][bad[:8]], want[f][bad[:8]])


@pytest.mark.parametrize("case", kats.CASES, ids=[c["name"] for c in kats.CASES])
def test_tables_reproduce_reference_kats(case):
    h = table_walk.HostHarness(case["policy"], case["routing"], case["workers"])
    o = oracle_lib.Oracle(case["policy"], case["routing"], case["workers"])
    env = wire.EnvelopeBatch.from_jobs([case["job"]])
    assert_same(h.evaluate(env, case["mode"]), o.eval(env, case["mode"]), case["name"])


@pytest.mark.parametrize("name,n,mode", [("tiny", 2000, wire.MODE_POLICY_AND_ROUTE), ("tiny", 500, wire.MODE_POLICY_ONLY),
                                         ("tiny", 500, wire.MODE_ROUTE_ONLY), ("c2", 1500, wire.MODE_POLICY_AND_ROUTE)])
def test_tables_match_oracle_on_synthetic(name, n, mode):
    cfg = synth.make_config(name, n)
    h = table_walk.HostHarness(cfg.policy, cfg.routing, cfg.workers)
    o = oracle_lib.Oracle(cfg.policy, cfg.routing, cfg.workers)
    want = o.eval(cfg.jobs, mode, threads=4)
    assert_same(h.evaluate(cfg.jobs, mode), want, name)


def test_tables_match_oracle_with_ties_and_load_updates():
    spec = synth.Spec(**{**synth.SPECS["tiny"].__dict__, "tie_fraction": 0.5, "seed": 11})
    cfg = synth.make_config(spec)
    h = table_walk.HostHarness(cfg.policy, cfg.routing, cfg.workers)
    o = oracle_lib.Oracle(cfg.policy, cfg.routing, cfg.workers)
    want = o.eval(cfg.jobs, wire.MODE_POLICY_AND_ROUTE)
    assert (want["flags"] & wire.F_TIE).astype(bool).sum() > 20
    assert_same(h.evaluate(cfg.jobs), want, "ties")
    # heartbeat deltas: new loads for a third of the workers
    rng = np.random.default_rng(1)
    slots = np.arange(0, cfg.workers.n_workers, 3, dtype=np.uint32)
    loads = np.zeros(len(slots), dtype=wire.LOAD_DTYPE)
    loads["active_jobs"] = rng.integers(0, 6, len(slots))
    loads["max_parallel_jobs"] = rng.choice([0, 4, 8], len(slots))
    loads["cpu_load"] = (rng.random(len(slots)) * 100).astype(np.float32)
    loads["gpu_utilization"] = (rng.random(len(slots)) * 100).astype(np.float32)
    h.update_workers(slots, loads)
    o.update_workers(slots, loads)
    assert_same(h.evaluate(cfg.jobs), o.eval(cfg.jobs, wire.MODE_POLICY_AND_ROUTE), "after heartbeat deltas")


def test_approved_replay_and_c5():
    c5 = kats.golden("c5_demo_guardrails.json")
    jobs, workers, kind = synth.make_c5(3000)
    h = table_walk.HostHarness(c5["policy"], c5["routing"], workers)
    o = oracle_lib.Oracle(c5["policy"], c5["routing"], workers)
    got = h.evaluate(jobs)
    assert_same(got, o.eval(jobs), "c5")
    # SURVEY §8d config 5 expectations
    assert (got["sched_decision"][kind == 0] == wire.DEC_REQUIRE_HUMAN).all()
    assert (got["decision"][kind == 1] == wire.DEC_ALLOW).all() and (got["rule_idx"][kind == 1] == -1).all()
    assert (got["decision"][kind == 2] == wire.DEC_DENY).all()
    assert (got["decision"][kind == 3] == wire.DEC_ALLOW).all() and (got["route_status"][kind == 3] == wire.ROUTE_OK).all()
    replay = jobs.with_approved(kind == 0)
    got2 = h.evaluate(replay)
    assert_same(got2, o.eval(replay), "c5 replay")
    assert (got2["route_status"][kind == 0] == wire.ROUTE_OK).all()


def test_new_topics_and_effective_configs_after_load():
    """Dictionaries grow on first sight of a topic / effective config (dynamic tables)."""
    policy = {"default_tenant": "default",
              "rules": [{"id": "r", "decision": "deny", "reason": "x", "match": {"topics": ["job.a.*"]}}]}
    routing = {"topics": {"job.b.one": ["p"]}, "pools": {"p": {}}}
    workers = [kats.hb("w", "p")]
    h = table_walk.HostHarness(policy, routing, workers)
    o = oracle_lib.Oracle(policy, routing, workers)
    jobs = [{"topic": "job.a.new1"}, {"topic": "job.b.one"}, {"topic": " job.a.padded "},
            {"topic": "job.b.one", "effective_config": b'{"safety":{"denied_topics":["job.b.*"]}}'},
            {"topic": "job.b.one", "effective_config": b'{"safety":{"allowed_topics":["job.c.*"]}}'},
            {"topic": "job.c.x", "effective_config": b'{"safety":{"allowed_topics":["job.c.*"]}}'},
            {"topic": "job.b.one", "labels": {"mcp.server": "evil"},
             "effective_config": b'{"data":{"safety":{"mcp":{"deny_servers":["EVIL"]}}}}'},
            {"topic": "job.b.one", "effective_config": b'not json'}]
    for _ in range(2):   # second pass: everything already in the dictionaries
        assert_same(h.evaluate(jobs), o.eval(jobs), "dynamic")


def test_policy_reload_changes_answers():
    routing = {"topics": {"job.x": ["p"]}, "pools": {"p": {}}}
    h = table_walk.HostHarness({"rules": [{"id": "a", "decision": "deny", "match": {"topics": ["job.x"]}}]}, routing,
                               [kats.hb("w", "p")])
    jobs = [{"topic": "job.x"}]
    assert h.evaluate(jobs)["decision"][0] == wire.DEC_DENY
    h.load_policy({"rules": [{"id": "a", "decision": "allow", "match": {"topics": ["job.x"]}}]})
    r = h.evaluate(jobs)
    assert r["decision"][0] == wire.DEC_ALLOW and r["route_status"][0] == wire.ROUTE_OK
    h.load_policy(None)   # nil policy: allow-all
    assert h.evaluate(jobs)["decision"][0] == wire.DEC_ALLOW


def test_capacity_errors_fail_closed():
    """What still has a ceiling: 16-bit dictionary ids in the job record.  (Mask widths do not: test_wide_masks.py.)"""
    rules = [{"id": "r", "decision": "deny", "match": {"capabilities": ["cap%d" % i for i in range(70000)]}}]
    h = table_walk.HostHarness({"rules": [{"id": "ok", "decision": "deny", "match": {"topics": ["job.x"]}}]})
    with pytest.raises(RuntimeError, match="65535 distinct values"):
        h.load_policy({"rules": rules})
    assert h.evaluate([{"topic": "job.x"}])["decision"][0] == wire.DEC_DENY   # the previous policy still serves


@pytest.mark.parametrize("sizes", [[0], [1], [512], [513], [1500, 3, 0, 600], [8192, 8193], [20000]])
def test_refresh_work_list(sizes):
    """Chunk table of the worker-table refresh (tables.h): every pool owns ceil(n/512) chunks (an empty pool one, empty,
    chunk); worker_merge_kernel runs all chunks of a multi-chunk pool up to 8192 workers and chunk 0 of larger pools."""
    workers, pools = [], {}
    for p, n in enumerate(sizes):
        pools["p%d" % p] = {}
        workers += [kats.hb("w-%d-%05d" % (p, i), "p%d" % p) for i in range(n)]
    routing = {"topics": {"job.x": list(pools)}, "pools": pools}
    h = table_walk.HostHarness(None, routing, workers)
    T = h.tables()
    off = T["pool_off"]
    assert [int(off[p + 1] - off[p]) for p in range(len(sizes))] == sizes
    want_chunks, want_merge, smem = [], [], 0
    for p, n in enumerate(sizes):
        m = max(1, -(-n // 512))
        g0 = len(want_chunks)
        assert int(T["pool_chunk0"][p]) == g0
        want_chunks += [p] * m
        if n > 8192:
            want_merge.append(g0)
        elif m > 1:
            want_merge += list(range(g0, g0 + m))
            smem = max(smem, n * 8)
    assert int(T["pool_chunk0"][len(sizes)]) == len(want_chunks) == int(T["n_chunks"])
    assert T["chunk_pool"][:len(want_chunks)].tolist() == want_chunks
    assert int(T["n_merge"]) == len(want_merge) and T["merge_list"][:len(want_merge)].tolist() == want_merge
    assert int(T["merge_smem"]) == smem <= 8192 * 8
    h.close()


def test_tables_match_oracle_on_config3_sample():
    """BASELINE config 3 (4,096 rules, 65,536 workers, 1M jobs): the host tables of the headline workload, walked for
    eight 100-job windows spread over the batch, against the oracle."""
    cfg = synth.make_config("c3")
    h = table_walk.HostHarness(cfg.policy, cfg.routing, cfg.workers, threads=4)
    o = oracle_lib.Oracle(cfg.policy, cfg.routing, cfg.workers)
    T = h.tables()
    assert int(T["n_rules"]) == 4096 and int(T["n_slots"]) == 65536 and int(T["n_merge"]) > 0
    rng = np.random.default_rng(5)
    seen = set()
    for s in rng.integers(0, cfg.jobs.n_jobs - 100, 8):
        env = cfg.jobs.slice(int(s), 100)
        want = o.eval(env, wire.MODE_POLICY_AND_ROUTE, threads=4)
        assert_same(h.evaluate(env), want, "c3 window at %d" % s)
        seen |= set(want["decision"].tolist())
    assert len(seen) >= 4
    h.close()
    o.close()


def test_rejected_worker_load_keeps_the_previous_registry():
    """A cordum_workers_load that fails (label dictionary over capacity, NaN load) must leave the previous registry in
    place: same tables, same encoding, same results (ADVICE round 1: a failed load used to leave n_slots / loads of the
    new registry next to slot_pos / pos_slot of the old one, and later calls indexed out of bounds)."""
    routing = {"topics": {"job.a": ["p"]}, "pools": {"p": {}}}
    good = [kats.hb("w0", "p", 1, 10.0, 0.0, 4, {"zone": "a"}), kats.hb("w1", "p", 0, 20.0, 0.0, 4, {"zone": "b"})]
    jobs = [{"topic": "job.a"}, {"topic": "job.a", "labels": {"zone": "b"}},
            {"topic": "job.a", "labels": {"preferred_worker_id": "w1"}}, {"topic": "job.a", "labels": {"preferred_worker_id": "w079"}}]
    h = table_walk.HostHarness(None, routing, good)
    o = oracle_lib.Oracle(None, routing, good)
    want = o.eval(jobs, wire.MODE_ROUTE_ONLY)
    assert_same(h.evaluate(jobs, wire.MODE_ROUTE_ONLY), want, "before")
    before = h.tables()
    too_many = [kats.hb("w%05d" % i, "p", 0, 1.0, 0.0, 0, {"host-%d" % i: "x"}) for i in range(33000)]   # 33000 keys + 33000 pairs > 65536 bits
    with pytest.raises(RuntimeError, match="placement labels"):
        h.load_workers(too_many)
    nan = [kats.hb("w0", "p", 1, float("nan"), 0.0, 4)]
    with pytest.raises(RuntimeError, match="NaN"):
        h.load_workers(nan)
    after = h.tables()
    for k in ("n_slots", "n_pos"):
        assert before[k] == after[k] == 2, k
    for k in ("slot_pos", "pos_slot", "pos_rank", "rank_slot", "pool_off", "pos_label_lo", "pos_label_hi"):
        assert np.array_equal(before[k], after[k]), k
    assert np.array_equal(before["loads"], after["loads"])
    assert_same(h.evaluate(jobs, wire.MODE_ROUTE_ONLY), want, "after the rejected loads")
    # heartbeat deltas are still bounded by the OLD registry
    with pytest.raises(RuntimeError):
        h.update_workers(np.array([2], np.uint32), np.zeros(1, wire.LOAD_DTYPE))
    h.update_workers(np.array([1], np.uint32), np.array([(3, 4, 50.0, 0.0)], wire.LOAD_DTYPE))
    o.update_workers(np.array([1], np.uint32), np.array([(3, 4, 50.0, 0.0)], wire.LOAD_DTYPE))
    assert_same(h.evaluate(jobs, wire.MODE_ROUTE_ONLY), o.eval(jobs, wire.MODE_ROUTE_ONLY), "after a delta")
    # a delta is all or nothing too: a row refused after valid rows leaves those rows unapplied (on both sides)
    loads = h.tables()["loads"].copy()
    for bad_row in ((0, 0, float("nan"), 0.0), (0, 0, 0.0, float("nan"))):
        with pytest.raises(RuntimeError, match="NaN"):
            h.update_workers(np.array([0, 1], np.uint32), np.array([(7, 8, 55.0, 0.0), bad_row], wire.LOAD_DTYPE))
        assert np.array_equal(h.tables()["loads"], loads)
    for side in (h, o):
        with pytest.raises(RuntimeError, match="out of range"):
            side.update_workers(np.array([0, 2], np.uint32), np.array([(7, 8, 55.0, 0.0), (0, 0, 0.0, 0.0)], wire.LOAD_DTYPE))
    assert np.array_equal(h.tables()["loads"], loads)
    assert_same(h.evaluate(jobs, wire.MODE_ROUTE_ONLY), o.eval(jobs, wire.MODE_ROUTE_ONLY), "after refused deltas")
    # the next accepted delta brings its own rows only
    h.update_workers(np.array([1], np.uint32), np.array([(0, 4, 5.0, 0.0)], wire.LOAD_DTYPE))
    o.update_workers(np.array([1], np.uint32), np.array([(0, 4, 5.0, 0.0)], wire.LOAD_DTYPE))
    assert tuple(h.tables()["loads"][0]) == tuple(loads[0])
    assert_same(h.evaluate(jobs, wire.MODE_ROUTE_ONLY), o.eval(jobs, wire.MODE_ROUTE_ONLY), "after an accepted delta")


SUMMARISED = ("tenant", "cap", "pack", "actor", "combo", "risk")


@pytest.mark.parametrize("case", ["fuzz-400-%d" % s for s in range(4)] + ["wide-%d" % s for s in range(4)] + ["c2", "sparse"])
def test_summaries_cover_their_rows(case, monkeypatch):
    """policy_kernel skips a word group when the AND of the job's summaries has no bit for it, so a summary that misses a
    group its row occupies drops that group's rules.  For every summarised attribute and value: summary bit g is set
    exactly when the row has a bit in words [g * sum_group, (g + 1) * sum_group) of 128 bits."""
    import test_fuzz_three_way as fuzz

    if case == "sparse":
        policy, routing, workers, _ = fuzz.sparse_summary_case()
    elif case == "c2":
        cfg = synth.make_config("c2", 10)
        policy, routing, workers = cfg.policy, cfg.routing, cfg.workers
    elif case.startswith("wide"):
        fuzz.widen(monkeypatch)
        policy, routing, workers, _ = fuzz.wide_case(int(case.split("-")[1]))
    else:
        policy, routing, workers, _ = fuzz.fuzz_case(100 + int(case.split("-")[2]), 400)
    h = table_walk.HostHarness(policy, routing, workers)
    T = h.tables()
    W, G = T["row_words"], T["sum_group"]
    n_groups = -(-(W // 4) // G)
    assert 1 <= n_groups <= 64
    for a in SUMMARISED:
        rows, sums = T["row_" + a].reshape(-1, W), T["sum_" + a]
        assert len(sums) == max(len(rows), 1), a
        for v, row in enumerate(rows):
            occupied = sum(1 << g for g in range(n_groups) if row[4 * G * g: 4 * G * (g + 1)].any())
            assert int(sums[v]) == occupied, "%s value %d: summary %x, row occupies %x" % (a, v, int(sums[v]), occupied)
    if case.startswith("wide"):
        assert T["xw_risk"] > 0 and len(T["sum_risk"]) > 65   # summaries of tags 64... (row 1 + tag)
    if case == "sparse":   # one word group per tag; four tags share a 128-bit word, so 24 distinct summaries
        risk = [int(x) for x in T["sum_risk"]]
        assert len(risk) == 97 and all(bin(x).count("1") == 1 for x in risk[1:]) and len(set(risk[1:])) == 24
    h.close()


@pytest.mark.parametrize("sum_use", [None] + [0, 1, 2, 4, 8, 16, 32, 63])
def test_sparse_summaries_match_oracle(sum_use, monkeypatch):
    """The host tables of a policy whose risk / capability / pack summaries prune word groups, walked with the summaries
    the table compiler picks and with each one forced, against the oracle."""
    import test_fuzz_three_way as fuzz

    fuzz.force_sum_use(monkeypatch, sum_use)
    policy, routing, workers, jobs = fuzz.sparse_summary_case()
    jobs = jobs[:300]
    h = table_walk.HostHarness(policy, routing, workers)
    T = h.tables()
    assert T["xw_risk"] == 1 and (sum_use is None or T["sum_use"] == sum_use)
    if sum_use is None:
        assert T["sum_use"] & table_walk.SUM_RISK   # the compiler picks the risk summaries where they pay
    o = oracle_lib.Oracle(policy, routing, workers)
    want = o.eval(jobs, wire.MODE_POLICY_AND_ROUTE)
    assert_same(h.evaluate(jobs), want, "sum_use %s" % sum_use)
    assert len(set(want["rule_idx"].tolist())) > 100
    h.close()
    o.close()


def test_rejected_routing_load_keeps_the_previous_routing():
    """A routing reload that makes more labelled workers routable than the label dictionary holds is refused whole."""
    workers = [kats.hb("a%03d" % i, "p", 0, float(i), 0.0, 0, {"zone": "z"}) for i in range(3)] + \
              [kats.hb("b%05d" % i, "q", 0, 1.0, 0.0, 0, {"host-%d" % i: "x"}) for i in range(33000)]
    r1 = {"topics": {"job.a": ["p"]}, "pools": {"p": {}}}
    r2 = {"topics": {"job.a": ["p", "q"]}, "pools": {"p": {}, "q": {}}}
    jobs = [{"topic": "job.a"}, {"topic": "job.a", "labels": {"zone": "z"}}]
    h = table_walk.HostHarness(None, r1, workers)
    o = oracle_lib.Oracle(None, r1, workers)
    want = o.eval(jobs, wire.MODE_ROUTE_ONLY)
    assert_same(h.evaluate(jobs, wire.MODE_ROUTE_ONLY), want, "before")
    with pytest.raises(RuntimeError, match="placement labels"):
        h.load_routing(r2)
    assert_same(h.evaluate(jobs, wire.MODE_ROUTE_ONLY), want, "after the rejected routing")


def test_effective_config_verdicts_survive_reloads():
    """The (effective config, topic) verdict table is kept across policy / routing reloads (ids are stable) and only
    extended: old configs on old topics, old configs on topics a reload pre-seeds, new configs after the reload."""
    p1 = {"rules": [{"id": "a", "decision": "deny", "match": {"topics": ["job.a.*"]}}]}
    p2 = {"rules": [{"id": "b", "decision": "require_approval", "reason": "r", "match": {"topics": ["job.b.*"]}}]}
    r1 = {"topics": {"job.a.one": ["p"]}, "pools": {"p": {}}}
    r2 = {"topics": {"job.a.one": ["p"], "job.b.two": ["p"], "job.c.three": ["p"]}, "pools": {"p": {}}}
    workers = [kats.hb("w", "p")]
    effs = [b'{"safety":{"denied_topics":["job.b.*"]}}', b'{"safety":{"allowed_topics":["job.a.*","job.c.*"]}}',
            b'{"data":{"safety":{"denied_topics":["job.?.one"]}}}']
    topics = ["job.a.one", "job.b.two", "job.c.three", "job.d.four"]
    jobs = [{"topic": t, "effective_config": e} for t in topics for e in effs] + [{"topic": t} for t in topics]
    h = table_walk.HostHarness(p1, r1, workers)
    o = oracle_lib.Oracle(p1, r1, workers)
    assert_same(h.evaluate(jobs[:6]), o.eval(jobs[:6]), "before")           # two topics, three configs seen
    h.load_policy(p2)
    h.load_routing(r2)                                                      # pre-seeds job.b.two (seen) and job.c.three (new)
    o2 = oracle_lib.Oracle(p2, r2, workers)
    assert_same(h.evaluate(jobs), o2.eval(jobs), "after the reloads")
    more = [{"topic": t, "effective_config": b'{"safety":{"denied_topics":["job.d.*"],"allowed_topics":["job.*"]}}'} for t in topics]
    assert_same(h.evaluate(more + jobs), o2.eval(more + jobs), "a config first seen after the reloads")
    h.load_policy(p1)
    assert_same(h.evaluate(more + jobs), oracle_lib.Oracle(p1, r2, workers).eval(more + jobs), "and back")


def test_dynamic_dictionaries_start_a_new_generation_when_full():
    """Raw topics and effective configs are dictionary-coded on first sight; the dictionaries are bounded (max_topics /
    max_effcfgs).  The reference has no such bound - it evaluates strings - so a full dictionary must not stop the
    engine: it starts a new generation (only the routing table's topics survive), and answers stay those of the oracle."""
    policy = {"rules": [{"id": "d", "decision": "deny", "match": {"topics": ["job.bad.*"]}},
                        {"id": "a", "decision": "require_approval", "reason": "r", "match": {"topics": ["job.?1.*"]}}]}
    routing = {"topics": {"job.keep.a": ["p"], "job.keep.b": ["p"]}, "pools": {"p": {}}}
    workers = [kats.hb("w", "p")]
    h = table_walk.HostHarness(policy, routing, workers, max_topics=16, max_effcfgs=6)
    o = oracle_lib.Oracle(policy, routing, workers)
    n0 = h.tables()["n_topics"]
    assert n0 == 3                                   # "", and the two routed topics
    resets = 0
    for rnd in range(12):
        jobs = [{"topic": "job.%s%d.x%d" % ("bad" if i % 3 == 0 else "t", rnd % 4, rnd * 10 + i)} for i in range(7)]
        jobs += [{"topic": "job.keep.a"}, {"topic": "job.keep.b", "effective_config": ('{"safety":{"denied_topics":["job.keep.%s"]}}' % "ab"[rnd % 2]).encode()},
                 {"topic": "job.t1.e%d" % rnd, "effective_config": ('{"safety":{"allowed_topics":["job.t%d.*"]}}' % (rnd % 5)).encode()}]
        assert_same(h.evaluate(jobs), o.eval(jobs), "round %d" % rnd)
        T = h.tables()
        assert T["n_topics"] <= 16 and T["n_effcfg"] <= 6
        assert T["dict_resets"] >= resets
        resets = T["dict_resets"]
    assert resets >= 3                               # 8 new topics per round into 13 free ids: several generations
    # one batch that needs more than a whole dictionary is refused (and only that batch)
    with pytest.raises(RuntimeError, match="more distinct topics"):
        h.evaluate([{"topic": "job.big.%d" % i} for i in range(20)])
    assert_same(h.evaluate([{"topic": "job.keep.a"}, {"topic": "job.bad.z"}]), o.eval([{"topic": "job.keep.a"}, {"topic": "job.bad.z"}]), "after the refused batch")
    with pytest.raises(RuntimeError, match="effective configs"):
        h.evaluate([{"topic": "job.keep.a", "effective_config": ('{"safety":{"denied_topics":["x%d"]}}' % i).encode()} for i in range(9)])
    o.close()


# Label pairs whose keys or values hold NUL.  Both are valid (a protobuf string, a Go map key), so "a\0b" = "c" and
# "a" = "b\0c" are different pairs; a pair key that joins key and value with a separator byte makes them one.
# (name, policy, routing, workers, jobs)
NUL_ROUTING = {"topics": {"job.x": ["p"]}, "pools": {"p": {}}}
NUL_PAIR_CASES = [
    ("job-key-holds-nul", None, NUL_ROUTING,
     [kats.hb("w0", "p", 0, 10.0, 0.0, 0, {"a": "b\0c"}), kats.hb("w1", "p", 0, 50.0, 0.0, 0, {"z": "1"})],
     [{"topic": "job.x", "labels": {"a\0b": "c"}}, {"topic": "job.x", "labels": {"a": "b\0c"}}, {"topic": "job.x", "labels": {"a": "b"}}]),
    ("job-value-holds-nul", None, NUL_ROUTING,
     [kats.hb("w0", "p", 0, 10.0, 0.0, 0, {"a\0b": "c"}), kats.hb("w1", "p", 0, 50.0, 0.0, 0, {"z": "1"})],
     [{"topic": "job.x", "labels": {"a": "b\0c"}}, {"topic": "job.x", "labels": {"a\0b": "c"}}, {"topic": "job.x", "labels": {"a\0b": ""}}]),
    ("colliding-workers", None, NUL_ROUTING,   # the less loaded worker holds the other pair of the collision
     [kats.hb("w0", "p", 0, 10.0, 0.0, 0, {"a": "b\0c"}), kats.hb("w1", "p", 0, 50.0, 0.0, 0, {"a\0b": "c"}),
      kats.hb("w2", "p", 0, 5.0, 0.0, 0, {"a\0": "\0b\0c"})],
     [{"topic": "job.x", "labels": {"a\0b": "c"}}, {"topic": "job.x", "labels": {"a": "b\0c"}}, {"topic": "job.x", "labels": {"a\0": "\0b\0c"}},
      {"topic": "job.x", "labels": {"a\0b\0": "c"}}]),
    ("rule-labels", {"default_tenant": "default", "rules": [
        {"id": "r0", "decision": "deny", "reason": "a is b-nul-c", "match": {"labels": {"a": "b\0c"}}},
        {"id": "r1", "decision": "require_approval", "reason": "a-nul-b is x", "match": {"labels": {"a\0b": "x"}}}]},
     NUL_ROUTING, [kats.hb("w0", "p")],
     [{"topic": "job.x", "labels": {"a\0b": "c"}}, {"topic": "job.x", "labels": {"a\0b": "x"}}, {"topic": "job.x", "labels": {"a": "b\0c"}},
      {"topic": "job.x", "labels": {"a": "b\0c", "a\0b": "x"}}, {"topic": "job.x", "labels": {"a": "b"}}]),
]


@pytest.mark.parametrize("name,policy,routing,workers,jobs", NUL_PAIR_CASES, ids=[c[0] for c in NUL_PAIR_CASES])
def test_label_pairs_with_nul_bytes_do_not_collide(name, policy, routing, workers, jobs):
    h = table_walk.HostHarness(policy, routing, workers)
    o = oracle_lib.Oracle(policy, routing, workers)
    for mode in (wire.MODE_POLICY_AND_ROUTE, wire.MODE_POLICY_ONLY, wire.MODE_ROUTE_ONLY):
        assert_same(h.evaluate(jobs, mode), o.eval(jobs, mode), "%s mode %d" % (name, mode))
    h.close()
    o.close()
