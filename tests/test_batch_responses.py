"""cordum_batch_responses: a dispatched batch's jobs grouped by safety response class on the device, each class's reason and
rule id rendered once.  The partition is checked against keys computed in Python from the batch's own decision records and
encoded records (each job exactly once, ascending inside a class, classes in first_job order, one key per class and
distinct keys across classes); the text against the C++ oracle's per-job response (MCP values compared case-folded: the
class quotes the canonical spelling) and, for the gateway flavour, GatewayPolicyEvaluator.  Every dispatch path, mode and
encoder, subsets and merges, fixtures that reach every reason code, one class and thousands of classes, tile and radix-pass
edges, rule indices above 4,096, reloads and new dictionary generations after the dispatch, refusals and launch counts;
and reference_api.decision_records against a per-job restatement through SafetyClient."""
import ctypes as C
import json

import numpy as np
import pytest

import kats
import oracle_lib
import test_batch_subset as tbs
from cordum_b200 import reference_api, synth, wire

pytestmark = pytest.mark.gpu

MODES = tbs.MODES
PATHS = tbs.PATHS
TILE = 2048                     # items per CTA of the response kernels (csrc/kernels.h CORDUM_SUBSET_TILE)
E_INVALID, E_STATE, E_STALE = -1, -4, -6
MCP_CODES = set(range(wire.REASON_TENANT_MCP, wire.REASON_TENANT_MCP + 8)) | set(range(wire.REASON_EFF_MCP, wire.REASON_EFF_MCP + 8))
TOPIC_CODES = {wire.REASON_EFF_DENIED_TOPIC, wire.REASON_EFF_NOT_ALLOWED_TOPIC}


@pytest.fixture(scope="module")
def eng():
    from cordum_b200 import engine

    e = engine.Engine(device=0)
    yield e
    e.close()


def refused(code, fn):
    from cordum_b200 import engine

    with pytest.raises(engine.CordumError) as ei:
        fn()
    assert ei.value.code == code
    return str(ei.value)


def launches_for(n_rules, n_topics=1, n=1):
    """8 + 3 x ceil(key bits / 8): key bits = 15 + bits(n_rules + 1 values) + max(16, bits(topic ids))."""
    if n == 0:
        return 0
    bits = 15 + int(n_rules).bit_length() + max(16, int(max(n_topics - 1, 0)).bit_length())
    return 8 + 3 * ((bits + 7) // 8)


def job_keys(b, rec):
    """The class key of every job, from its decision record and its encoded record."""
    job, _, slot = b.records()
    mine = job[slot]
    code = rec["reason_code"].astype(np.int64)
    arg = np.zeros(len(rec), np.int64)
    t = np.isin(code, list(TOPIC_CODES))
    arg[t] = mine["topic"][t]
    for base in (wire.REASON_TENANT_MCP, wire.REASON_EFF_MCP):
        m = (code >= base) & (code < base + 8)
        f = np.clip((code - base) >> 1, 0, 3)
        arg[m] = mine["mcp"][np.arange(len(rec)), f][m]
    return list(zip(rec["decision"].tolist(), rec["sched_decision"].tolist(), (rec["flags"] & wire.CLASS_FLAG_MASK).tolist(),
                    code.tolist(), rec["rule_idx"].tolist(), arg.tolist()))


def partition_checked(b, rec, resp, what):
    """The partition against the keys of the records; returns the keys per job."""
    n = len(rec)
    cls, off, jobs = resp["classes"], resp["offsets"].astype(np.int64), resp["jobs"].astype(np.int64)
    m = len(cls)
    assert len(off) == m + 1 and off[0] == 0 and off[-1] == n and len(jobs) == n, what
    assert (np.diff(off) > 0).all(), what
    assert np.array_equal(np.sort(jobs), np.arange(n)), what                       # each job exactly once
    assert np.array_equal(cls["first_job"].astype(np.int64), jobs[off[:-1]] if m else np.zeros(0, np.int64)), what
    assert (np.diff(cls["first_job"].astype(np.int64)) > 0).all(), what            # classes by first_job
    keys = job_keys(b, rec) if n else []
    seen = set()
    for c in range(m):
        members = jobs[off[c]:off[c + 1]]
        assert (np.diff(members) > 0).all(), what                                  # ascending inside a class
        k = cls[c]
        key = (int(k["decision"]), int(k["sched_decision"]), int(k["flags"]) & wire.CLASS_FLAG_MASK, int(k["reason_code"]),
               int(k["rule_idx"]), int(k["arg"]))
        assert all(keys[j] == key for j in members.tolist()), (what, c, key)
        assert key not in seen, (what, key)
        seen.add(key)
        want_flag = wire.CLASS_QUOTES_VALUE if int(k["reason_code"]) in MCP_CODES else 0
        assert int(k["flags"]) & ~wire.CLASS_FLAG_MASK == want_flag, what
    assert len(seen) == len(set(keys)), what
    return keys


def expected_text(o, env, j, flavor, mode):
    """(reason, rule_id) the front-end builds for job j, from the oracle's per-job response."""
    r = o.eval_one(env.slice(j, 1), mode, flavor)
    dec = r["decision"]
    code = int(r["reason_code"])
    reason = r["reason"] if (code != wire.REASON_NONE and dec not in ("ALLOW", "ALLOW_WITH_CONSTRAINTS")) or code == wire.REASON_APPROVAL_GRANTED else ""
    return reason, r["rule_id"] if r["has_snapshot"] else "", code


def mcp_expected(reason, k):
    """An MCP reason as a class quotes it: the value case-folded, or "" for a value no list names (dictionary id
    CORDUM_ID_OTHER = 1 keeps no spelling; the request's own needs the envelopes)."""
    if int(k["arg"]) != 1:
        return reason
    return reason[:reason.index('"')] + '""' + reason[reason.rindex('"') + 1:]


def text_checked(o, env, resp, what, flavor=wire.REASON_FLAVOR_KERNEL, per_class=3, mode=wire.MODE_POLICY_ONLY):
    """Each class's reason and rule id against the oracle for up to per_class members (first, middle, last)."""
    off, jobs = resp["offsets"], resp["jobs"]
    codes = set()
    for c, k in enumerate(resp["classes"]):
        members = jobs[off[c]:off[c + 1]]
        pick = sorted({0, len(members) // 2, len(members) - 1})[:per_class]
        for i in pick:
            reason, rule_id, code = expected_text(o, env, int(members[i]), flavor, mode)
            got = resp["reasons"][c]
            if code in MCP_CODES:
                assert oracle_lib.equal_fold(got, mcp_expected(reason, k)), (what, c, got, reason)   # the canonical value
            else:
                assert got == reason, (what, c, got, reason)
            assert resp["rule_ids"][c] == rule_id, (what, c, resp["rule_ids"][c], rule_id)
        codes.add(int(k["reason_code"]))
    return codes


def env_of(jobs):
    return jobs if isinstance(jobs, wire.EnvelopeBatch) else wire.EnvelopeBatch.from_jobs(jobs)


# ------------------------------------------------------------------ every path, mode and encoder
@pytest.mark.parametrize("encoder", ["host", "device"])
@pytest.mark.parametrize("name", ["tiny", "c2", "c5", "fuzz"])
def test_every_dispatch_path(eng, name, encoder):
    policy, routing, workers, env = tbs.config(name)
    tbs.load(eng, policy, routing, workers)
    o = oracle_lib.Oracle(policy, routing, workers)
    loads = workers.loads()
    b = eng.batch(env.n_jobs)
    b.encode_device(env.deinterned()) if encoder == "device" else b.encode(env)
    refused(E_STATE, b.responses)                            # encoded, never dispatched
    checked_text = False
    for mode in MODES:
        for path in PATHS:
            if path == "tick" and mode != wire.MODE_POLICY_AND_ROUTE:
                continue
            if path == "async":
                b.dispatch_async(mode)
                refused(E_STATE, b.responses)                # before the wait
                rec = b.wait().copy()
            else:
                rec = tbs.run(eng, b, mode, path, loads)
            before = eng.launch_count()
            resp = b.responses()
            assert eng.launch_count() - before == launches_for(eng.stats().n_rules, eng.stats().n_topics, len(rec))
            partition_checked(b, rec, resp, "%s %s mode %d %s" % (name, encoder, mode, path))
            if mode != wire.MODE_ROUTE_ONLY and not checked_text:
                text_checked(o, env, resp, "%s %s" % (name, encoder))
                checked_text = True
    b.encode(env)
    refused(E_STATE, b.responses)                            # a new encode: no responses until the next dispatch
    b.free()
    o.close()


def test_device_encode_that_falls_back_to_the_host(eng):
    cfg = synth.make_config("tiny")
    tbs.load(eng, cfg.policy, cfg.routing, cfg.workers)
    jobs = [{"topic": "job.first.seen.%d" % (i % 3)} if i % 5 == 0 else {"topic": "job.pack000.read", "labels": {"zone": "z%d" % (i % 4)}}
            for i in range(3000)]
    b = eng.batch(len(jobs))
    before = eng.host_fallbacks()
    b.encode_device(jobs)
    b.dispatch_async()
    refused(E_STATE, b.responses)
    rec = b.wait().copy()
    assert eng.host_fallbacks() == before + 1
    partition_checked(b, rec, b.responses(), "fallback")
    b.free()


# ------------------------------------------------------------------ subsets and merges
@pytest.mark.parametrize("name", ["c2", "fuzz"])
def test_subsets_and_merges(eng, name):
    policy, routing, workers, env = tbs.config(name)
    tbs.load(eng, policy, routing, workers)
    o = oracle_lib.Oracle(policy, routing, workers)
    src, sub, mrg = eng.batch(env.n_jobs), eng.batch(env.n_jobs), eng.batch(2 * env.n_jobs)
    src.encode(env).dispatch()
    pick = np.arange(0, env.n_jobs, 3)
    src.subset(sub, jobs=pick)
    refused(E_STATE, sub.responses)                          # a subset is encoded, not dispatched
    for path in PATHS:
        rec = tbs.run(eng, sub, wire.MODE_POLICY_AND_ROUTE, path, workers.loads())
        resp = sub.responses()
        partition_checked(sub, rec, resp, "%s subset %s" % (name, path))
    text_checked(o, tbs.take(env, pick), resp, name + " subset", mode=wire.MODE_POLICY_AND_ROUTE)
    src.merge(sub, mrg)
    refused(E_STATE, mrg.responses)
    rec = mrg.dispatch().copy()
    resp = mrg.responses()
    partition_checked(mrg, rec, resp, name + " merge")
    both = np.concatenate([np.arange(env.n_jobs), pick])   # the merge holds src's jobs, then the subset's
    text_checked(o, tbs.take(env, both), resp, name + " merge", mode=wire.MODE_POLICY_AND_ROUTE)
    for b in (src, sub, mrg):
        b.free()
    o.close()


# ------------------------------------------------------------------ every reason code
MCP_FIELDS = ("server", "tool", "resource", "action")
LABEL = {"server": "mcp.server", "tool": "mcp.tool", "resource": "mcp.resource", "action": "mcp.action"}


def every_code_fixture():
    """A policy, routing and jobs whose records carry every reason code, both MCP sources x 4 fields x denied / not
    allowed, effective-config topic reasons, approval granted, constraints and remediations, approval_required."""
    mcp = {}
    for f in MCP_FIELDS:
        mcp["allow_%ss" % f] = ["ok-%s" % f, "Bad-%s" % f]
        mcp["deny_%ss" % f] = ["Bad-%s" % f]
    policy = {
        "default_tenant": "default",
        "tenants": {"default": {"allow_topics": ["job.*"]}, "strict": {"allow_topics": ["job.*"], "mcp": mcp}},
        "rules": [
            {"id": "deny-x", "decision": "deny", "reason": "x is denied", "match": {"topics": ["job.x.*"]},
             "remediations": [{"id": "r1", "title": "use y", "replacement_topic": "job.y.a"}]},
            {"id": "need-human", "decision": "require_approval", "reason": "prod needs a human", "match": {"topics": ["job.prod.*"]}},
            {"id": "slow", "decision": "throttle", "reason": "slow down", "match": {"topics": ["job.slow.*"]}},
            {"id": "bounded", "decision": "allow", "match": {"topics": ["job.cap.*"]}, "constraints": {"budgets": {"max_runtime_ms": 5}}},
            {"id": "awc", "decision": "allow_with_constraints", "reason": "dropped", "match": {"topics": ["job.awc.*"]},
             "constraints": {"budgets": {"max_retries": 1}}},
            {"id": "plain", "decision": "allow", "reason": "dropped too", "match": {"topics": ["job.ok.*"]}},
        ]}
    routing = {"topics": {"job.ok.a": ["p"], "job.prod.a": ["p"]}, "pools": {"p": {}}}
    workers = [kats.hb("w1", "p"), kats.hb("w2", "p")]
    jobs = [{"topic": ""}, {"topic": "   "}, {"topic": "other.thing"}, {"topic": "job.x.a"}, {"topic": "job.prod.a"},
            {"topic": "job.slow.a"}, {"topic": "job.cap.a"}, {"topic": "job.awc.a"}, {"topic": "job.ok.a"}, {"topic": "job.none"},
            {"topic": "job.prod.a", "approved": True, "labels": {"approval_granted": "true"}}]
    for f in MCP_FIELDS:
        others = {LABEL[g]: "ok-%s" % g for g in MCP_FIELDS if g != f}
        for val in ("BAD-%s" % f, "bad-%s" % f, "nope-%s" % f, "NOPE-%s" % f):        # denied (two spellings), not allowed
            jobs.append({"topic": "job.ok.a", "tenant": "strict", "labels": dict(others, **{LABEL[f]: val})})
            deny = {"mcp": {"deny_%ss" % f: ["Bad-%s" % f], "allow_%ss" % f: ["ok-%s" % f, "Bad-%s" % f]}}
            eff = json.dumps({"safety": deny}).encode()
            jobs.append({"topic": "job.ok.a", "labels": dict(others, **{LABEL[f]: val}), "effective_config": eff})
    eff_topics = [b'{"safety":{"denied_topics":["job.ok.*"]}}', b'{"safety":{"allowed_topics":["job.zz.*"]}}']
    for i in range(6):
        jobs.append({"topic": "job.ok.%s" % "ab"[i % 2] + (" " if i % 3 == 0 else ""), "effective_config": eff_topics[i % 2]})
    # a require_approval rule overridden by an effective-config deny: approval_required on a DENY
    jobs.append({"topic": "job.prod.a", "effective_config": b'{"safety":{"denied_topics":["job.prod.*"]}}'})
    return policy, routing, workers, jobs * 3


def test_every_reason_code_and_both_flavours(eng):
    policy, routing, workers, jobs = every_code_fixture()
    tbs.load(eng, policy, routing, workers)
    o = oracle_lib.Oracle(policy, routing, workers)
    env = env_of(jobs)
    b = eng.batch(len(jobs))
    codes = set()
    for mode in (wire.MODE_POLICY_ONLY, wire.MODE_POLICY_AND_ROUTE):
        rec = b.encode(env).dispatch(mode).copy()
        for flavor in (wire.REASON_FLAVOR_KERNEL, wire.REASON_FLAVOR_GATEWAY):
            resp = b.responses(flavor)
            keys = partition_checked(b, rec, resp, "every code %d %d" % (mode, flavor))
            codes |= text_checked(o, env, resp, "every code flavor %d" % flavor, flavor, per_class=99, mode=mode)
            # the MCP classes: one per (code, value id), not per spelling: "BAD-x" and "bad-x" share the denied class,
            # "nope-x" and "NOPE-x" (named by no list) the not-allowed one
            mcp = sorted(int(k["reason_code"]) for k in resp["classes"] if int(k["reason_code"]) in MCP_CODES)
            assert mcp == sorted(MCP_CODES), mcp
        assert len(set(keys)) == len(resp["classes"])
    assert codes >= {wire.REASON_NONE, wire.REASON_RULE, wire.REASON_MISSING_TOPIC, wire.REASON_UNSUPPORTED_TOPIC,
                     wire.REASON_EFF_DENIED_TOPIC, wire.REASON_EFF_NOT_ALLOWED_TOPIC, wire.REASON_APPROVAL_GRANTED} | MCP_CODES, codes
    flags = np.bitwise_or.reduce(resp["classes"]["flags"])
    assert flags & wire.F_CONSTRAINTS and flags & wire.F_APPROVAL_REQUIRED and flags & wire.F_APPROVED_BYPASS
    b.free()
    o.close()


def test_gateway_flavour_against_the_gateway_evaluator(eng):
    policy, routing, workers, jobs = every_code_fixture()
    reqs = [dict(j, tenant=j.get("tenant", "default")) for j in jobs if not j.get("approved")]
    ev = reference_api.GatewayPolicyEvaluator(device=0)
    want = ev.evaluate_batch(policy, "", reqs)
    ev._server.engine.close()
    tbs.load(eng, policy, routing, workers)
    b = eng.batch(len(reqs))
    rec = b.encode([reference_api._envelope(r) for r in reqs]).dispatch(wire.MODE_POLICY_ONLY).copy()
    resp = b.responses(wire.REASON_FLAVOR_GATEWAY)
    partition_checked(b, rec, resp, "gateway")
    off, jb = resp["offsets"], resp["jobs"]
    for c, k in enumerate(resp["classes"]):
        for j in jb[off[c]:off[c + 1]].tolist():
            w = want[j]["reason"] if want[j]["decision"] not in ("ALLOW", "ALLOW_WITH_CONSTRAINTS") else ""
            got = resp["reasons"][c]
            assert got == w or (int(k["reason_code"]) in MCP_CODES and oracle_lib.equal_fold(got, mcp_expected(w, k))), (j, got, w)
    b.free()


# ------------------------------------------------------------------ shapes
def test_one_class(eng):
    routing = {"topics": {"job.hot": ["p"]}, "pools": {"p": {}}}
    tbs.load(eng, None, routing, [kats.hb("w%d" % i, "p") for i in range(3)])
    n = 5 * TILE + 7
    jobs = [{"topic": "job.hot"}] * n
    b = eng.batch(n)
    for mode in MODES:
        rec = b.encode(jobs).dispatch(mode).copy()
        resp = b.responses()
        partition_checked(b, rec, resp, "one class mode %d" % mode)
        assert len(resp["classes"]) == 1 and resp["reasons"] == [""] and resp["rule_ids"] == [""]
    b.free()


def test_thousands_of_classes_behind_effective_config_topics(eng):
    n = 3 * TILE + 5
    tbs.load(eng, None, {"topics": {}, "pools": {}}, [kats.hb("w", "p")])
    eff = b'{"safety":{"denied_topics":["job.*"]}}'
    order = (np.arange(n) * 4999) % n
    jobs = [{"topic": "job.t%05d" % (i % 4000), "effective_config": eff} for i in order]
    env = env_of(jobs)
    o = oracle_lib.Oracle(None, {"topics": {}, "pools": {}}, [kats.hb("w", "p")])
    b = eng.batch(n)
    rec = b.encode(env).dispatch(wire.MODE_POLICY_ONLY).copy()
    resp = b.responses()
    partition_checked(b, rec, resp, "4000 topics")
    assert len(resp["classes"]) == 4000
    text_checked(o, env, {**resp, "classes": resp["classes"][:50]}, "4000 topics", per_class=2)
    for c in range(0, 4000, 397):
        j = int(resp["classes"][c]["first_job"])
        assert resp["reasons"][c] == "topic '%s' denied by effective config" % jobs[j]["topic"]
    b.free()
    o.close()


@pytest.mark.parametrize("n", [0, 1, TILE - 1, TILE, TILE + 1, 3 * TILE + 17])
def test_tile_edges(eng, n):
    cfg = synth.make_config("c2")
    tbs.load(eng, cfg.policy, cfg.routing, cfg.workers)
    b = eng.batch(max(n, 1))
    env = cfg.jobs.slice(0, n)
    rec = b.encode(env).dispatch().copy()
    before = eng.launch_count()
    resp = b.responses()
    assert eng.launch_count() - before == launches_for(eng.stats().n_rules, eng.stats().n_topics, n)
    partition_checked(b, rec, resp, "n=%d" % n)
    if n == 0:
        assert len(resp["classes"]) == 0 and list(resp["offsets"]) == [0]
    b.free()


@pytest.mark.parametrize("n_rules", [255, 511, 512, 4500])
def test_rule_indices_and_radix_pass_edges(eng, n_rules):
    """Rule counts around a digit of the key (one more radix pass) and rule indices above 4,096."""
    rules = [{"id": "r%05d" % i, "decision": ["deny", "throttle", "require_approval", "allow"][i % 4], "reason": "rule %d" % i,
              "match": {"topics": ["job.r%05d" % i]}} for i in range(n_rules)]
    policy = {"default_tenant": "default", "rules": rules}
    tbs.load(eng, policy, {"topics": {}, "pools": {}}, [kats.hb("w", "p")])
    idx = sorted({n_rules - 1, n_rules - 2, n_rules // 2, 0, 1, 4097 % n_rules, 4099 % n_rules})
    jobs = [{"topic": "job.r%05d" % idx[i % len(idx)]} for i in range(TILE + 3)] + [{"topic": "job.none"}]
    env = env_of(jobs)
    b = eng.batch(len(jobs))
    rec = b.encode(env).dispatch(wire.MODE_POLICY_ONLY).copy()
    before = eng.launch_count()
    resp = b.responses()
    assert eng.launch_count() - before == launches_for(n_rules, eng.stats().n_topics, len(jobs))
    partition_checked(b, rec, resp, "rules %d" % n_rules)
    assert set(resp["classes"]["rule_idx"].tolist()) == set(idx) | {-1}
    for c, k in enumerate(resp["classes"]):
        r = int(k["rule_idx"])
        if r >= 0:
            assert resp["rule_ids"][c] == "r%05d" % r
            assert resp["reasons"][c] == ("" if r % 4 == 3 else "rule %d" % r)
    b.free()


@pytest.mark.slow
def test_config3_million_jobs(eng):
    cfg = synth.make_config("c3")
    tbs.load(eng, cfg.policy, cfg.routing, cfg.workers)
    o = oracle_lib.Oracle(cfg.policy, cfg.routing, cfg.workers)
    b = eng.batch(cfg.jobs.n_jobs)
    rec = b.encode(cfg.jobs).dispatch().copy()
    resp = b.responses()
    partition_checked(b, rec, resp, "config 3")
    text_checked(o, cfg.jobs, resp, "config 3", per_class=1)
    b.free()
    o.close()


# ------------------------------------------------------------------ after the dispatch
def test_reloads_and_new_dictionary_generations():
    from cordum_b200 import engine

    e = engine.Engine(device=0, max_topics=16)
    try:
        policy, routing, workers, _ = every_code_fixture()
        tbs.load(e, policy, routing, workers)
        eff = b'{"safety":{"denied_topics":["job.*"]}}'
        first = [{"topic": "job.first.%d " % (i % 6), "effective_config": eff} for i in range(300)] + \
                [{"topic": "job.x.a"}, {"topic": "job.prod.a"}]
        mcp_jobs = first + [{"topic": "job.ok.a", "tenant": "strict", "labels": {"mcp.server": "BAD-server"}}]
        b, c, d = e.batch(400), e.batch(400), e.batch(400)
        rec = b.encode(first).dispatch().copy()
        want = b.responses()
        want = {k: (v.copy() if hasattr(v, "copy") else v) for k, v in want.items()}
        d.encode(mcp_jobs).dispatch()
        d_resp = d.responses()
        assert any(int(k["reason_code"]) in MCP_CODES for k in d_resp["classes"])
        # a new dictionary generation: 12 new topics do not fit next to the first generation's
        c.encode([{"topic": "job.second.%02d" % (i % 12)} for i in range(300)]).dispatch()
        # policy, routing and workers reloads
        e.load_policy({"default_tenant": "default", "rules": [{"id": "d", "decision": "deny", "reason": "new", "match": {"topics": ["job.*"]}}]}, "r")
        e.load_routing({"topics": {"job.z": ["q"]}, "pools": {"q": {}}})
        e.load_workers([kats.hb("x%d" % i, "q") for i in range(3)])
        again = b.responses()
        partition_checked(b, rec, again, "after reloads")
        assert again["reasons"] == want["reasons"] and again["rule_ids"] == want["rule_ids"]
        assert np.array_equal(again["classes"], want["classes"]) and np.array_equal(again["jobs"], want["jobs"])
        assert "'job.first.0 ' " not in " ".join(again["reasons"]) and "topic 'job.first.0' denied by effective config" in again["reasons"]
        msg = refused(E_STALE, d.responses)                  # an MCP class: the value dictionaries were rebuilt
        assert "MCP value" in msg
        b.free()
        c.free()
        d.free()
    finally:
        e.close()


def test_buffers_survive_plan_and_topic_counts(eng):
    cfg = synth.make_config("c2")
    tbs.load(eng, cfg.policy, cfg.routing, cfg.workers)
    b = eng.batch(cfg.jobs.n_jobs)
    rec = b.encode(cfg.jobs).dispatch().copy()
    resp = b.responses()
    keep = {k: (v.copy() if hasattr(v, "copy") else list(v)) for k, v in resp.items() if k != "policy_gen"}
    offsets, jobs, _ = b.plan()
    off0, jobs0 = offsets.copy(), jobs.copy()
    b.topic_counts()
    b.plan()
    for k in ("classes", "offsets", "jobs"):
        assert np.array_equal(resp[k], keep[k]), k                   # the views after a plan and a topic-counts call
    b.responses()
    assert np.array_equal(offsets, off0) and np.array_equal(jobs, jobs0)   # the plan views after a responses call
    partition_checked(b, rec, b.responses(), "interleaved")
    b.free()


def test_refusals_and_launch_counts(eng):
    cfg = synth.make_config("tiny")
    tbs.load(eng, cfg.policy, cfg.routing, cfg.workers)
    b = eng.batch(cfg.jobs.n_jobs)
    out = wire.CordumResponses()
    L = b.L
    assert L.cordum_batch_responses(None, 0, C.byref(out)) == E_INVALID
    assert L.cordum_last_error().decode() == "null argument"
    assert L.cordum_batch_responses(b.h, 0, None) == E_INVALID
    assert L.cordum_batch_responses(b.h, 2, C.byref(out)) == E_INVALID
    assert L.cordum_last_error().decode() == "unknown reason flavor 2"
    assert L.cordum_batch_responses(b.h, 0, C.byref(out)) == E_STATE    # never encoded
    assert "no completed dispatch" in L.cordum_last_error().decode()
    b.encode(cfg.jobs)
    before = eng.launch_count()
    refused(E_STATE, b.responses)
    assert eng.launch_count() == before
    rec = b.dispatch().copy()
    for flavor in (0, 1, 0):
        before = eng.launch_count()
        partition_checked(b, rec, b.responses(flavor), "repeat")
        assert eng.launch_count() - before == launches_for(eng.stats().n_rules, eng.stats().n_topics, len(rec))
    b.free()


# ------------------------------------------------------------------ the stored records
@pytest.mark.parametrize("fixture", ["every_code", "c5"])
def test_decision_records_match_a_per_job_restatement(eng, fixture):
    if fixture == "c5":
        c5 = kats.golden("c5_demo_guardrails.json")
        policy, routing = c5["policy"], c5["routing"]
        jobs = [kats.c5_job(k, approved=(i % 7 == 0)) for i, k in enumerate(["write", "write-untagged", "dangerous", "read"] * 50)]
        workers = [kats.hb("demo-worker", "demo-guardrails", 0, maxp=8)]
    else:
        policy, routing, workers, jobs = every_code_fixture()
        jobs = [j for j in jobs if j.get("tenant") != "strict" and b"mcp" not in (j.get("effective_config") or b"")]
    tbs.load(eng, policy, routing, workers)
    server = reference_api.SafetyKernelServer(engine=eng)
    client = reference_api.SafetyClient(server)
    reqs = [{"job_id": "j%d" % i, "topic": j["topic"], "tenant_id": j.get("tenant", ""), "labels": j.get("labels") or {},
             "meta": j.get("meta"), "env": {reference_api.EFFECTIVE_CONFIG_ENV: j["effective_config"]} if j.get("effective_config") else {}}
            for i, j in enumerate(jobs)]
    per_job = client.check_batch(reqs)
    b = eng.batch(len(reqs))
    b.encode([reference_api._envelope(reference_api.policy_check_request(r)) for r in reqs]).dispatch(wire.MODE_POLICY_ONLY)
    got = reference_api.decision_records(b, eng)
    seen = 0
    for cls in got:
        for j in cls["jobs"].tolist():
            want = dict(per_job[j])
            want.pop("approval_ref")
            if want["approval_required"] and want["decision"] in ("ALLOW", "ALLOW_WITH_CONSTRAINTS"):
                want["decision"] = "REQUIRE_APPROVAL"        # engine.go:527-529
            assert cls["record"] == want, (j, cls["record"], want)
            dlq = {"DENY": "safety_denied"}.get(cls["record"]["decision"])
            assert cls["dlq_reason_code"] == dlq
            seen += 1
    assert seen == len(reqs)
    server._batch and server._batch.free()
    b.free()
