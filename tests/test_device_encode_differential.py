"""The device encoder (cordum_b200/csrc/encode.cu) against the host encoder (host.cpp Host::encode_job) and the C++ oracle,
on batches that stay on the device.

A batch the device encoder cannot finish (non-ASCII text in a field it folds, a string over 4,096 bytes, a label key plus
value over 512 bytes, an unseen topic or effective config) raises a fallback flag, and the host re-encodes the whole
batch; a wrong device record in such a batch never shows.  So every case here first checks that host_fallbacks() did not
move, then compares every JobRec / RouteRec field (but `spare`) with the host encoder's, job by job, and every decision
record field with the oracle in all three modes, from three envelope layouts (interned, deinterned, pinned).

Cases: the fuzz configurations with an ASCII-only awkward vocabulary (test_fuzz_three_way.ascii_case) and their reload /
heartbeat life cycle, repeated label keys, every length class of the folding hash in every folded dictionary, label pairs
holding NUL, batch sizes and key counts around the encoder's scan and slot shapes; and the fallback triggers themselves,
one per batch, which must raise the counter by exactly one and still give the oracle's decisions.
Run on an H100: pytest -m gpu tests/test_device_encode_differential.py."""
import os

import numpy as np
import pytest

import kats
import oracle_lib
import table_walk
import test_fuzz_three_way as fuzz
from cordum_b200 import wire
from test_device_encode import assert_records_equal
from test_host_tables import NUL_PAIR_CASES

pytestmark = pytest.mark.gpu

FIELDS = ("decision", "sched_decision", "flags", "route_status", "reason_code", "rule_idx", "worker_slot")
MODES = (wire.MODE_POLICY_AND_ROUTE, wire.MODE_POLICY_ONLY, wire.MODE_ROUTE_ONLY)
KEPT = {"batches": 0, "jobs": 0}   # device encodes this module saw complete on the device


def cores() -> int:
    try:
        return max(1, len(os.sched_getaffinity(0)))
    except AttributeError:
        return os.cpu_count() or 1


@pytest.fixture(scope="module")
def eng():
    from cordum_b200 import engine

    e = engine.Engine(device=0)
    yield e
    e.close()


def load(e, policy, routing, workers):
    e.load_policy(policy, "device-encode")
    e.load_routing(routing)
    e.load_workers(workers)


def assert_same(got, want, what):
    for f in FIELDS:
        bad = np.nonzero(got[f] != want[f])[0]
        assert len(bad) == 0, "%s: field %s differs at jobs %s: kernels %s oracle %s" % (
            what, f, bad[:8].tolist(), got[f][bad[:8]].tolist(), want[f][bad[:8]].tolist())


def check_order(job, slot, tclass, ncls, what):
    """slot_of is a permutation, orig its inverse, and the records are sorted by the encoders' key (topic id * tenant
    classes + tenant class, from the host's tables)."""
    n = len(job)
    assert np.array_equal(np.sort(slot), np.arange(n, dtype=np.uint32)), "%s: slot_of is not a permutation" % what
    assert np.array_equal(job["orig"][slot], np.arange(n, dtype=np.uint32)), "%s: slot_of / orig are not inverse" % what
    key = job["topic"].astype(np.int64) * ncls + tclass[job["tenant"].astype(np.int64)]
    bad = np.nonzero(np.diff(key) < 0)[0]
    assert len(bad) == 0, "%s: records out of key order at slots %s" % (what, bad[:8].tolist())


def check(e, config, jobs, what):
    """Host encode twice (the second sees the final dictionaries), then the device encoder from three layouts: no
    fallback, records equal to the host's, decisions equal to the oracle's in every mode."""
    policy, routing, workers = config
    env = jobs if isinstance(jobs, wire.EnvelopeBatch) else wire.EnvelopeBatch.from_jobs(jobs)
    n = env.n_jobs
    h = table_walk.HostHarness(policy, routing, workers)
    T = h.tables()
    h.close()
    o = oracle_lib.Oracle(policy, routing, workers)
    want = {m: o.eval(env, m, threads=cores()) for m in MODES}
    o.close()
    bh, bd = e.batch(n), e.batch(n)
    pinned = e.pinned_envelopes(env.deinterned())
    try:
        bh.encode(env)
        job, route, slot = bh.encode(env).records()
        host = (job[slot], route[slot])
        tclass = np.zeros(max(len(T["tenant_class"]), int(job["tenant"].max(initial=0)) + 1), np.int64)
        tclass[: len(T["tenant_class"])] = T["tenant_class"]
        for layout, name in ((env, "interned"), (env.deinterned(), "deinterned"), (pinned, "pinned")):
            for i, mode in enumerate(MODES):
                f0 = e.host_fallbacks()
                bd.encode_device(layout)
                if i == 0:
                    job, route, slot = bd.records()
                    assert e.host_fallbacks() == f0, "%s (%s): the batch fell back to the host encoder" % (what, name)
                    check_order(job, slot, tclass, T["tenant_classes"], "%s (%s)" % (what, name))
                    assert_records_equal((job[slot], route[slot]), host, "%s (%s)" % (what, name))
                got = bd.dispatch(mode).copy()
                assert e.host_fallbacks() == f0, "%s (%s): the batch fell back to the host encoder" % (what, name)
                assert_same(got, want[mode], "%s (%s, mode %d)" % (what, name, mode))
                KEPT["batches"] += 1
                KEPT["jobs"] += n
    finally:
        bh.free()
        bd.free()
        pinned.free()


# ------------------------------------------------------------------ the fuzz, ASCII only
@pytest.mark.parametrize("seed,max_rules", [(s, 12) for s in range(60)] + [(100 + s, 400) for s in range(12)])
def test_ascii_fuzz_stays_on_the_device(eng, seed, max_rules):
    policy, routing, workers, jobs = fuzz.ascii_case(seed, max_rules)
    load(eng, policy, routing, workers)
    check(eng, (policy, routing, workers), jobs, "ascii seed %d (%d rules)" % (seed, max_rules))


@pytest.mark.parametrize("seed", range(30))
def test_ascii_life_cycle_stays_on_the_device(eng, seed):
    """Every reload changes the host's dictionaries; the engine must export them again (v_dict) before the next device
    encode, or the device codes against stale ids."""
    config = None
    for step, (kind, payload, jobs) in enumerate(fuzz.ascii_life_cycle(seed)):
        if kind == "load":
            config = payload
            load(eng, *config)
        elif kind == "heartbeat" and payload is not None:
            slots, loads = payload
            eng.update_workers(slots, loads)
            w = [dict(x) for x in config[2]]
            for s, l in zip(slots.tolist(), loads):
                w[s].update(active_jobs=int(l["active_jobs"]), max_parallel_jobs=int(l["max_parallel_jobs"]),
                            cpu_load=float(l["cpu_load"]), gpu_utilization=float(l["gpu_utilization"]))
            config = (config[0], config[1], w)
        elif kind == "workers":
            eng.load_workers(payload)
            config = (config[0], config[1], payload)
        elif kind == "routing":
            eng.load_routing(payload)
            config = (config[0], payload, config[2])
        elif kind == "policy":
            eng.load_policy(payload, "device-encode")
            config = (payload, config[1], config[2])
        check(eng, config, jobs, "ascii life cycle %d after %s (step %d)" % (seed, kind, step - 1))


@pytest.mark.parametrize("seed", range(60))
def test_repeated_label_keys_stay_on_the_device(eng, seed):
    """The last of repeated keys wins for rule pairs, placement, every MCP alias, secrets_present and the routing hints."""
    policy, routing, workers, jobs = fuzz.dup_case(seed)
    load(eng, policy, routing, workers)
    check(eng, (policy, routing, workers), jobs, "repeated keys seed %d" % seed)


def test_repeated_label_keys_each_field(eng):
    """One job per special key, each key given twice or three times, the winning value last and first in turn."""
    policy = {"default_tenant": "default", "rules": [
        {"id": "lab", "decision": "deny", "reason": "l", "match": {"labels": {"env": "prod"}}},
        {"id": "srv", "decision": "require_approval", "reason": "s", "match": {"mcp": {"deny_servers": ["srv"]}}},
        {"id": "tool", "decision": "deny", "reason": "t", "match": {"mcp": {"allow_tools": ["read"]}}},
        {"id": "sec", "decision": "throttle", "reason": "x", "match": {"secrets_present": True}}],
        "tenants": {"default": {"mcp": {"deny_actions": ["write"], "deny_resources": ["db"]}}}}
    routing = {"topics": {"job.a": ["p", "q"]}, "pools": {"p": {}, "q": {}}}
    workers = [kats.hb("w0", "p", 0, 10.0, 0.0, 0, {"zone": "a"}), kats.hb("w1", "q", 0, 50.0, 0.0, 0, {"zone": "b"})]
    load(eng, policy, routing, workers)
    pairs = {"env": ("prod", "dev"), "zone": ("b", "a"), "secrets_present": ("true", "no"), "preferred_pool": ("q", "p"),
             "preferred_worker_id": ("w1", "w0")}
    pairs.update({k: ("srv", "other") for k in ("mcp.server", "mcp_server", "mcpServer")})
    pairs.update({k: ("write", "read") for k in ("mcp.tool", "mcp_tool", "mcpTool")})
    pairs.update({k: ("db", "x") for k in ("mcp.resource", "mcp_resource", "mcpResource")})
    pairs.update({k: ("WRITE", "read") for k in ("mcp.action", "mcp_action", "mcpAction")})
    jobs = []
    for k, (a, b) in pairs.items():
        for win, lose in ((a, b), (b, a)):
            jobs.append({"topic": "job.a", "labels": [(k, lose), (k, win)]})
            jobs.append({"topic": "job.a", "labels": [(k, lose), ("other", "1"), (k, ""), (k, win)]})
            jobs.append({"topic": "job.a", "labels": [(k, win)]})
    check(eng, (policy, routing, workers), jobs, "repeated special keys")


# ------------------------------------------------------------------ the folding hash, every length class
FOLD_CHARS = "aZ@[`{zA0-._q"


def fold_value(n, salt):
    """An ASCII string of n bytes, mixed case, with the bytes just outside A-Z ('@', '[', '`', '{')."""
    return "".join(FOLD_CHARS[(i * 7 + salt) % len(FOLD_CHARS)] for i in range(n))


def swap_case(s):
    return "".join(c.lower() if i % 2 else c.upper() for i, c in enumerate(s))


FOLD_LENGTHS = list(range(0, 41)) + [160, 161]
FOLD_FIELDS = ("tenant", "capability", "pack", "actor", "risk", "requires", "mcp0", "mcp1", "mcp2", "mcp3")


def fold_case():
    rules, jobs, reqs = [], [], []
    mcp_key = {"mcp0": ("servers", "mcp.server"), "mcp1": ("tools", "mcp_tool"), "mcp2": ("resources", "mcpResource"),
               "mcp3": ("actions", "mcp.action")}
    for fi, field in enumerate(FOLD_FIELDS):
        for n in FOLD_LENGTHS:
            v = fold_value(n, fi)
            m = {"tenant": {"tenants": [v]}, "capability": {"capabilities": [v]}, "pack": {"pack_ids": [v]},
                 "actor": {"actor_ids": [v]}, "risk": {"risk_tags": [v]}, "requires": {"requires": [v]}}.get(field)
            if m is None:
                m = {"mcp": {"deny_" + mcp_key[field][0]: [v]}}
            rules.append({"id": "%s-%d" % (field, n), "decision": ("deny", "require_approval", "throttle")[n % 3], "reason": field, "match": m})
            if field == "requires":
                reqs.append(v)
            # the same value in another case, a near miss ('@' <-> '`', '[' <-> '{': one bit apart, like a case fold)
            near = v.translate(str.maketrans("@[`{", "`{@["))
            for val in (swap_case(v), v.upper(), near, " \t" + swap_case(v) + "\r\n"):
                j = {"topic": "job.f", "meta": {}}
                if field == "tenant":
                    j["tenant"] = val
                elif field == "capability":
                    j["meta"]["capability"] = val
                elif field == "pack":
                    j["meta"]["pack_id"] = val
                elif field == "actor":
                    j["meta"]["actor_id"] = val
                elif field == "risk":
                    j["meta"]["risk_tags"] = [val]
                elif field == "requires":
                    j["meta"]["requires"] = [val]
                else:
                    j["labels"] = {mcp_key[field][1]: val}
                jobs.append(j)
    routing = {"topics": {"job.f": ["p"]}, "pools": {"p": {"requires": reqs[:20]}, "q": {"requires": reqs[20:]}}}
    workers = [kats.hb("w0", "p"), kats.hb("w1", "q")]
    return {"default_tenant": "default", "rules": rules}, routing, workers, jobs


def test_fold_hash_length_classes(eng):
    """Mixed-case values of every length 0-40 (the hash reads 1-3, 4-7, 8-16 and 16-byte blocks + a tail), and 160 / 161,
    in every folded dictionary: the device folds with lower8 (SWAR) and must hash to the host's canonical strings."""
    policy, routing, workers, jobs = fold_case()
    load(eng, policy, routing, workers)
    check(eng, (policy, routing, workers), jobs, "fold hash")


# ------------------------------------------------------------------ NUL inside label pairs
@pytest.mark.parametrize("name,policy,routing,workers,jobs", NUL_PAIR_CASES, ids=[c[0] for c in NUL_PAIR_CASES])
def test_label_pairs_with_nul_bytes_on_the_device(eng, name, policy, routing, workers, jobs):
    """The pair key is length-prefixed on both sides (host.hpp StrTable::pair_key, encode.cu hash_pair).  With a NUL
    separator the device's rule-label pair table (DD_LABEL_PAIR) made "a\\0b" = "c" match a rule on "a" = "b\\0c"."""
    load(eng, policy, routing, workers)
    check(eng, (policy, routing, workers), jobs * 8, name)


# ------------------------------------------------------------------ what goes back to the host, and what does not
LONG = 4096
TR_POLICY = {"default_tenant": "default", "rules": [
    {"id": "ten", "decision": "deny", "reason": "t", "match": {"tenants": ["acme", "t" * LONG]}},
    {"id": "cap", "decision": "require_approval", "reason": "c", "match": {"capabilities": ["cap.read", "c" * LONG]}},
    {"id": "risk", "decision": "throttle", "reason": "r", "match": {"risk_tags": ["write", "r" * LONG]}},
    {"id": "pack", "decision": "deny", "reason": "p", "match": {"pack_ids": ["sre", "p" * LONG]}},
    {"id": "act", "decision": "deny", "reason": "a", "match": {"actor_ids": ["alice", "a" * LONG]}},
    {"id": "lab", "decision": "deny", "reason": "l", "match": {"labels": {"env": "prød"}}},
    {"id": "mcp", "decision": "deny", "reason": "m", "match": {"mcp": {"deny_tools": ["bad", "m" * (512 - 8)]}}},
    {"id": "sec", "decision": "throttle", "reason": "s", "match": {"secrets_present": True}}]}
TR_ROUTING = {"topics": {"job.a": ["p"], "job.b": ["p", "q"], "job.ü": ["q"], "j" * LONG: ["p"], "k" * (LONG + 1): ["p"]},
              "pools": {"p": {"requires": ["git"]}, "q": {}}}
TR_WORKERS = [kats.hb("w0", "p", 0, 10.0, 0.0, 0, {"zone": "a"}), kats.hb("wö", "q", 0, 20.0, 0.0, 0, {"zöne": "ü"})]
TR_CLEAN = [{"topic": "job.a", "tenant": "acme"}, {"topic": "job.b", "meta": {"capability": "CAP.READ", "risk_tags": ["write"]}},
            {"topic": "job.a", "labels": {"zone": "a", "mcp.tool": "bad"}}, {"topic": "job.b", "meta": {"requires": ["git"]}},
            {"topic": "job.b", "labels": {"env": "prod", "preferred_pool": "q"}}]
EFF = '{"safety":{"denied_topics":["job.b"]}}'


def eff_of(n, tag=""):
    """A valid effective config of exactly n bytes (padded with spaces); `tag` makes it a different string."""
    s = '{"safety":{"denied_topics":["job.b%s"]}}' % tag
    return (s[:-1] + " " * (n - len(s)) + "}").encode()


def job_with(field, v):
    j = {"topic": "job.b", "meta": {}}
    if field == "tenant":
        j["tenant"] = v
    elif field == "meta_tenant":
        j["meta"]["tenant_id"] = v
    elif field == "capability":
        j["meta"]["capability"] = v
    elif field == "pack":
        j["meta"]["pack_id"] = v
    elif field == "actor":
        j["meta"]["actor_id"] = v
    elif field == "principal":
        j = {"topic": "job.b", "principal_id": v}
    elif field == "risk":
        j["meta"]["risk_tags"] = ["write", v]
    elif field == "requires":
        j["meta"]["requires"] = [v, "git"]
    elif field == "mcp":
        j["labels"] = {"mcp_tool": v}
    elif field == "secrets":
        j["labels"] = {"secrets_present": v}
    elif field == "topic":
        j["topic"] = v
    elif field == "effective_config":
        j["effective_config"] = v
    else:
        raise ValueError(field)
    return j


def label_of(key, n, c):
    """A job with one label `key` whose key plus value is n bytes."""
    return {"topic": "job.b", "labels": {key: c * (n - len(key))}}


# fields the device folds, and the first byte of their test values; MCP values and secrets_present are label values, so
# the 512-byte bound on a label's key plus value (the pair probe's buffer) reaches them long before kMaxStr does
STRINGS = {"tenant": "t", "meta_tenant": "t", "capability": "c", "pack": "p", "actor": "a", "principal": "a", "risk": "r",
           "requires": "g"}
LABELS = {"mcp": ("mcp_tool", "m"), "secrets": ("secrets_present", "y")}
TRIGGERS = ([("non-ascii-" + f, lambda i, f=f, c=c: job_with(f, "é" + c)) for f, c in STRINGS.items()] +
            [("non-ascii-" + f, lambda i, f=f, c=kc[1]: job_with(f, "é" + c)) for f, kc in LABELS.items()] +
            [("long-" + f, lambda i, f=f, c=c: job_with(f, c * (LONG + 1))) for f, c in STRINGS.items()] +
            [("long-topic", lambda i: job_with("topic", "k" * (LONG + 1))),
             ("long-effective-config", lambda i: job_with("effective_config", eff_of(LONG + 1)))] +
            [("label-513-" + k, lambda i, k=k: label_of(k, 513, "x")) for k in ("zone", "env", "mcp_tool", "secrets_present",
                                                                                  "preferred_pool", "preferred_worker_id")] +
            [("unseen-topic", lambda i: job_with("topic", "job.new.%d" % i)),
             ("unseen-effective-config", lambda i: job_with("effective_config", ('{"safety":{"denied_topics":["x%d"]}}' % i).encode()))])
NON_TRIGGERS = ([("exact-" + f, job_with(f, c * LONG)) for f, c in STRINGS.items()] +
                [("exact-topic", job_with("topic", "j" * LONG)), ("exact-effective-config", job_with("effective_config", eff_of(LONG)))] +
                [("label-512-" + k, label_of(k, 512, c)) for k, c in (("zone", "x"), ("env", "x"), ("mcp_tool", "M"),
                                                                        ("secrets_present", "y"), ("preferred_pool", "q"),
                                                                        ("preferred_worker_id", "w"))] +
                [("non-ascii-label", {"topic": "job.b", "labels": {"zöne": "ü", "kéy": "v"}}),
                 ("non-ascii-rule-label-value", {"topic": "job.b", "labels": {"env": "prød"}}),
                 ("non-ascii-preferred-pool", {"topic": "job.b", "labels": {"preferred_pool": "pööl"}}),
                 ("non-ascii-preferred-worker", {"topic": "job.b", "labels": {"preferred_worker_id": "wö"}}),
                 ("known-non-ascii-topic", {"topic": "job.ü"}),
                 ("known-effective-config", {"topic": "job.b", "effective_config": EFF.encode()})])


@pytest.mark.parametrize("name,make", TRIGGERS, ids=[t[0] for t in TRIGGERS])
def test_fallback_trigger_goes_to_the_host_once(eng, name, make):
    load(eng, TR_POLICY, TR_ROUTING, TR_WORKERS)
    o = oracle_lib.Oracle(TR_POLICY, TR_ROUTING, TR_WORKERS)
    clean = TR_CLEAN * 20
    b = eng.batch(len(clean) + 2)
    try:
        b.encode(clean + [job_with("topic", "j" * LONG), job_with("topic", "k" * (LONG + 1))])   # the clean vocabulary is known
        for i, mode in enumerate(MODES):
            jobs = clean[:50] + [make(i)] + clean[50:]
            f0 = eng.host_fallbacks()
            got = b.encode_device(jobs).dispatch(mode).copy()
            assert eng.host_fallbacks() == f0 + 1, "%s: expected exactly one fallback, got %d" % (name, eng.host_fallbacks() - f0)
            assert_same(got, o.eval(jobs, mode), "%s (mode %d)" % (name, mode))
            f0 = eng.host_fallbacks()
            got = b.encode_device(clean).dispatch(mode).copy()   # and the clean batch alone stays on the device
            assert eng.host_fallbacks() == f0, name
            assert_same(got, o.eval(clean, mode), "%s, clean (mode %d)" % (name, mode))
    finally:
        b.free()
        o.close()


@pytest.mark.parametrize("name,job", NON_TRIGGERS, ids=[t[0] for t in NON_TRIGGERS])
def test_non_trigger_stays_on_the_device(eng, name, job):
    load(eng, TR_POLICY, TR_ROUTING, TR_WORKERS)
    check(eng, (TR_POLICY, TR_ROUTING, TR_WORKERS), TR_CLEAN * 10 + [job] + TR_CLEAN * 3, name)


# ------------------------------------------------------------------ scan and slot shapes
N_TOPICS = 2600


def shape_config():
    """2,600 routed topics and 600 rules in one topic cluster, split by six tenants, so there are seven tenant classes and
    topics x classes (about 18,000 keys) is far above 2,048 and not a multiple of 1,024: encode_scan_kernel gives each of
    its 1,024 threads several keys."""
    rules = [{"id": "r%d" % i, "decision": ("deny", "allow", "require_approval", "throttle")[i % 4], "reason": "r",
              "match": {"topics": ["job.t.*"], "tenants": ["ten%d" % (i % 6)]}} for i in range(600)]
    policy = {"default_tenant": "default", "rules": rules}
    routing = {"topics": {"job.t.%d" % i: ["p%d" % (i % 3)] for i in range(N_TOPICS)}, "pools": {"p0": {}, "p1": {}, "p2": {}}}
    workers = [kats.hb("w%d" % i, "p%d" % (i % 3), i % 4, 10.0 * i, 0.0, 4) for i in range(12)]
    return policy, routing, workers


def shape_jobs(n, seed):
    rng = np.random.default_rng(seed)
    tids = rng.integers(0, N_TOPICS, n)
    tids[: min(n, 8)] = [N_TOPICS - 1, 0, N_TOPICS - 2, 2047, 2048, 1023, 1024, 2100][: min(n, 8)]
    tens = rng.integers(0, 8, n)
    return [{"topic": "job.t.%d" % t, "tenant": ("ten0", "TEN1", "ten2 ", "ten3", "ten4", "\tTen5", "other", "")[k]} for t, k in zip(tids, tens)]


@pytest.mark.parametrize("n", [1, 127, 128, 129, 255, 256, 257, 1023, 1024, 1025, 100_000])
def test_scan_and_slot_shapes(eng, n):
    policy, routing, workers = shape_config()
    h = table_walk.HostHarness(policy, routing, workers)
    T = h.tables()
    h.close()
    n_keys = T["n_topics"] * T["tenant_classes"]
    assert T["tenant_classes"] >= 6 and n_keys > 2048 and n_keys % 1024 != 0, (T["n_topics"], T["tenant_classes"])
    load(eng, policy, routing, workers)
    check(eng, (policy, routing, workers), shape_jobs(n, n), "%d jobs over %d keys" % (n, n_keys))


def test_every_job_on_one_key(eng):
    """Every job contends for the slot counter of one key."""
    policy, routing, workers = shape_config()
    load(eng, policy, routing, workers)
    jobs = [{"topic": "job.t.2447", "tenant": "ten1", "labels": {"i": str(i)}} for i in range(20_000)]
    check(eng, (policy, routing, workers), jobs, "one key")


def test_device_kept_the_batches(eng):
    """The cases above must really have run on the device encoder (an always-falling-back encoder passes them trivially)."""
    if KEPT["batches"] == 0:
        pytest.skip("no device-encode case ran in this session")
    print("device-encoded batches kept on the device: %d (%d jobs)" % (KEPT["batches"], KEPT["jobs"]))
