"""Adversarial randomized agreement of three independent implementations on small configurations built
from awkward strings (padding, case, glob classes / escapes / malformed patterns, empty values, duplicates,
MCP aliases, effective configs, legacy tenant rules, ties, overloaded workers):

    C++ oracle (oracle/oracle.cpp)  ==  Python oracle (oracle/py_oracle.py)  ==  the product's host tables re-walked
                                                                                 the way the kernels walk them

The reference's own tests pin none of these interactions (SURVEY.md §8c, last row); agreement of two restatements
written from the cited lines, plus the product's table compiler + encoder, is what stands in for them.  CPU only."""
import contextlib
import json
import os
import random
import sys

import numpy as np
import pytest

import kats
import oracle_lib
import table_walk
from cordum_b200 import wire

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import py_oracle  # noqa: E402

STATUS_CODE = {v: k for k, v in kats.ROUTE_NAMES.items()}
FIELDS = ("decision", "sched_decision", "flags", "route_status", "reason_code", "rule_idx", "worker_slot")

TENANTS = ["default", "t1", "T1", " t1 ", "acme", "Acme ", ""]
PACKS = ["sre", "db", "Web", "x"]
VERBS = ["collect", "delete", "a", "a.b", "*", ""]
CAPS = ["cap.read", "CAP.READ", " cap.write", "cap.write", ""]
RISKS = ["write", "Write ", "prod", "secrets", "SECRETS", "pii", ""]
REQS = ["git", "GIT", " net ", "gpu", "docker", ""]
LKEYS = ["env", "zone", "tier", "gpu"]
LVALS = ["prod", "dev", "a", "", "true"]
ACTORS = ["alice", "Alice", "svc-1", ""]
POOLS = ["p0", "p1", "p2", "gpu-pool"]
PATTERNS = ["job.*", "job.sre.*", "job.[sd]*.*", "job.[^s]*.collect", "job.db.delete", "job.?b.*", "job.\\*.x", "job.[abc",
            " job.sre.collect ", "", "*", "job.sre.c*t", "JOB.sre.*", "job.web.*", "job.*.a.b"]
MCP_VALS = ["srv", "SRV", " srv ", "other", "bad", "read", "WRITE", ""]
# non-ASCII: Unicode White_Space that TrimSpace strips (NBSP, EM SPACE, IDEOGRAPHIC SPACE, NEL, LINE SEPARATOR), characters it
# does not (ZERO WIDTH SPACE, BOM), letters that only fold outside ASCII (EqualFold is restated as ASCII-only), multi-byte
# runes under '?' and character classes of path.Match
TENANTS += ["\u00a0t1\u00a0", "\u2003acme", "t1\u3000", "\u00c9cole", "\u00e9cole", "t1\u200b", "\u0085t1\u2028"]
CAPS += ["\u00a0cap.read", "CAP.R\u00c9AD", "cap.r\u00e9ad"]
RISKS += ["\u2002write", "write\ufeff"]
REQS += ["\u00a0git", "g\u0131t"]
MCP_VALS += ["\u2003srv\u2003", "s\u0280v"]
PATTERNS += ["job.\u00e9*", "\u00a0job.sre.*\u00a0", "job.[\u00e0-\u00ff]*.*", "job.?\u00e9.*"]
PACKS += ["\u00e9t\u00e9"]
DECISIONS = ["allow", "deny", "require_approval", "throttle", "allow_with_constraints", "permit", "block", "REQUIRE-HUMAN", ""]



def _ascii_vocabulary():
    """Module globals for ascii_case: the ASCII entries of the vocabularies above plus awkward ASCII of their own - control
    bytes TrimSpace keeps (NUL, 0x1C-0x1F, DEL), \\v \\f \\r\\n padding, mixed-case values longer than 16 and than 160 bytes
    (every length class of the folding hash), and NUL inside label keys and values, where "a\\0b" = "c" and "a" = "b\\0c"
    are different pairs.  No string needs Unicode tables, so the device encoder keeps every batch (encode.cu)."""
    asc = lambda xs: [x for x in xs if x.isascii()]   # noqa: E731
    long_t, long_c = "Tenant-Of-" + "MiXeD" * 33, "Cap.Of-Mixed-Case-" + "Ab" * 80   # 175 and 178 bytes
    return dict(
        TENANTS=asc(TENANTS) + ["\vt1\f", "t1\r\n", "\x1ct1", "t1\x7f", "\x00t1", "T1\x1f", "Tenant-Mixed-Case", "tenant-mixed-case\r\n",
                                long_t, " " + long_t.lower()],
        PACKS=asc(PACKS) + ["Pack-Of-Mixed-Case", "\x1e"],
        CAPS=asc(CAPS) + ["\fcap.read\v", "cap.read\x00", "CAP.Of-Mixed-Case-Xy", "cap.of-mixed-case-xy\r\n", long_c, long_c.upper()],
        RISKS=asc(RISKS) + ["\vwrite", "WRITE\r\n", "write\x1d", "Risk-Of-Mixed-Case", "risk-of-mixed-case\f", "SeCrEtS"],
        REQS=asc(REQS) + ["\vgit\f", "Git\r\n", "git\x7f", "Requires-Mixed-Case", " requires-mixed-case"],
        LKEYS=asc(LKEYS) + ["a", "a\x00b", "Env"],
        LVALS=asc(LVALS) + ["b\x00c", "c", "\x00", "PROD", " prod"],
        ACTORS=asc(ACTORS) + ["\x1falice", "ALICE\r\n", "Actor-Of-Mixed-Case-" + "Q" * 150],
        MCP_VALS=asc(MCP_VALS) + ["\vsrv\f", "Srv\r\n", "\x1fsrv", "srv\x00", "Server-Of-Mixed-Case", "server-of-mixed-case\v"],
        PATTERNS=asc(PATTERNS) + ["\vjob.sre.*", "job.db.*\r\n", "job.\x00*"],
    )


@contextlib.contextmanager
def vocabulary(v):
    """The generators read the module's vocabulary globals: swap them for `v` inside the block."""
    me = sys.modules[__name__]
    old = {k: getattr(me, k) for k in v}
    for k, x in v.items():
        setattr(me, k, x)
    try:
        yield
    finally:
        for k, x in old.items():
            setattr(me, k, x)


def pick(rng, xs, lo=0, hi=2):
    return [rng.choice(xs) for _ in range(rng.randint(lo, hi))]


def mcp_lists(rng):
    m = {}
    for k in ("servers", "tools", "resources", "actions"):
        if rng.random() < 0.25:
            m["allow_" + k] = pick(rng, MCP_VALS, 1, 2)
        if rng.random() < 0.2:
            m["deny_" + k] = pick(rng, MCP_VALS, 1, 2)
    return m


def make_policy(rng, max_rules=12):
    if max_rules <= 12 and rng.random() < 0.15:   # legacy form: no rules, per-tenant allow / deny topic lists
        tenants = {}
        for t in rng.sample(["default", "t1", "acme"], rng.randint(1, 3)):
            tenants[t] = {"allow_topics": pick(rng, PATTERNS, 0, 2), "deny_topics": pick(rng, PATTERNS, 0, 2), "mcp": mcp_lists(rng)}
        return {"default_tenant": rng.choice(["default", " t1", ""]), "tenants": tenants}
    rules = []
    for i in range(rng.randint(max(1, max_rules // 3), max_rules)):
        m = {}
        if rng.random() < 0.5:
            m["tenants"] = pick(rng, TENANTS, 1, 2)
        if rng.random() < 0.7:
            m["topics"] = pick(rng, PATTERNS, 1, 3)
        if rng.random() < 0.3:
            m["capabilities"] = pick(rng, CAPS, 1, 2)
        if rng.random() < 0.3:
            m["risk_tags"] = pick(rng, RISKS, 1, 2)
        if rng.random() < 0.25:
            m["requires"] = pick(rng, REQS, 1, 2)
        if rng.random() < 0.2:
            m["pack_ids"] = pick(rng, PACKS, 1, 2)
        if rng.random() < 0.2:
            m["actor_ids"] = pick(rng, ACTORS, 1, 2)
        if rng.random() < 0.2:
            m["actor_types"] = pick(rng, ["human", "Service", "", "robot"], 1, 2)
        if rng.random() < 0.25:
            m["labels"] = {rng.choice(LKEYS): rng.choice(LVALS) for _ in range(rng.randint(1, 2))}
        if rng.random() < 0.15:
            m["secrets_present"] = rng.random() < 0.5
        if rng.random() < 0.2:
            m["mcp"] = mcp_lists(rng)
        r = {"id": "r%d" % i, "decision": rng.choice(DECISIONS), "reason": "because %d" % i, "match": m}
        if rng.random() < 0.2:
            r["constraints"] = {"budgets": {"max_runtime_ms": 1000 + i}}
        rules.append(r)
    pol = {"default_tenant": rng.choice(["default", "t1", ""]), "rules": rules}
    if rng.random() < 0.4:
        pol["tenants"] = {t: {"mcp": mcp_lists(rng)} for t in rng.sample(["default", "t1", "acme", "T1"], rng.randint(1, 2))}
    return pol


def make_routing(rng):
    topics = {}
    for p in PACKS + [""]:
        for v in VERBS[:4]:
            if rng.random() < 0.6:
                topics["job.%s.%s" % (p.lower(), v)] = [rng.choice(POOLS) for _ in range(rng.randint(1, 3))]
    topics[" job.sre.collect "] = ["p2"]          # the routing map is keyed by the RAW topic
    pools = {p: ({"requires": pick(rng, REQS, 0, 2)} if rng.random() < 0.5 else {}) for p in POOLS if rng.random() < 0.9}
    return {"topics": topics, "pools": pools}


def make_workers(rng):
    ws = []
    for i in range(rng.randint(0, 24)):
        labels = {k: rng.choice(LVALS) for k in rng.sample(LKEYS, rng.randint(0, 3))}
        coarse = rng.random() < 0.6   # coarse loads: ties and exact overload thresholds
        cpu = float(rng.choice([0, 25, 50, 89.5, 90, 95])) if coarse else rng.random() * 100
        gpu = float(rng.choice([0, 0, 50, 90])) if coarse else rng.random() * 100
        ws.append(kats.hb("w%02d" % rng.randint(0, 30), rng.choice(POOLS + ["orphan"]), rng.randint(0, 9), cpu, gpu,
                          rng.choice([0, 4, 10]), labels))
    return ws


def make_job(rng, workers):
    pack, verb = rng.choice(PACKS), rng.choice(VERBS)
    topic = rng.choice(["job.%s.%s" % (pack.lower(), verb), "job.%s.%s" % (pack, verb), " job.sre.collect ", "", "jobs.x", "job.", "job.sre.collect"])
    j = {"topic": topic, "tenant": rng.choice(TENANTS), "principal_id": rng.choice(ACTORS)}
    if rng.random() < 0.8:
        j["meta"] = {"tenant_id": rng.choice(TENANTS), "actor_id": rng.choice(ACTORS), "actor_type": rng.choice([0, 1, 2, 3]),
                     "capability": rng.choice(CAPS), "pack_id": rng.choice(PACKS + [""]),
                     "risk_tags": pick(rng, RISKS, 0, 3), "requires": pick(rng, REQS, 0, 2)}
    labels = {}
    for k in rng.sample(LKEYS, rng.randint(0, 3)):
        labels[k] = rng.choice(LVALS)
    if rng.random() < 0.3:
        labels[rng.choice(["mcp.server", "mcp_server", "mcpServer"])] = rng.choice(MCP_VALS)
    if rng.random() < 0.2:
        labels[rng.choice(["mcp.tool", "mcpTool"])] = rng.choice(MCP_VALS)
    if rng.random() < 0.15:
        labels[rng.choice(["mcp.action", "mcp_action"])] = rng.choice(MCP_VALS)
    if rng.random() < 0.1:
        labels["mcp.resource"] = rng.choice(MCP_VALS)
    if rng.random() < 0.2:
        labels["secrets_present"] = rng.choice(["true", "TRUE", "1", "yes", "YES", "no", " true ", ""])
    if rng.random() < 0.15:
        labels["preferred_pool"] = rng.choice(POOLS + ["nope", ""])
    if rng.random() < 0.15 and workers:
        labels["preferred_worker_id"] = rng.choice([w["worker_id"] for w in workers] + ["ghost"])
    if rng.random() < 0.3:
        labels.update({"workflow_id": "wf", "run_id": "r", "cordum.trace": "x"})
    if labels or rng.random() < 0.5:
        j["labels"] = labels
    if rng.random() < 0.2:
        eff = {}
        if rng.random() < 0.6:
            eff["denied_topics"] = pick(rng, PATTERNS, 1, 2)
        if rng.random() < 0.5:
            eff["allowed_topics"] = pick(rng, PATTERNS, 0, 2)
        if rng.random() < 0.4:
            eff["mcp"] = mcp_lists(rng)
        # ParseEffectiveSafety (effective.go:12-39): encoding/json field matching is case-insensitive, wrong types fail
        shape = rng.random()
        if shape < 0.7:
            j["effective_config"] = json.dumps({"safety": eff})
        elif shape < 0.8:
            j["effective_config"] = json.dumps({"Safety": {k.upper(): v for k, v in eff.items()}})
        elif shape < 0.9:
            j["effective_config"] = json.dumps({"safety": {"denied_topics": "job.*"}})   # not an array
        else:
            j["effective_config"] = rng.choice(["{", "null", "[]", '{"safety": null}', '{"other": 1}', '{"safety": {"denied_topics": [1]}}'])
    if rng.random() < 0.1:
        j["approved"] = True
    return j


def py_records(policy, routing, workers, jobs):
    live = list({w["worker_id"]: w for w in workers}.values())   # registry semantics: the latest heartbeat wins
    out = []
    for job in jobs:
        if isinstance(job.get("labels"), list):   # repeated keys: the map the reference decodes holds the last value
            job = dict(job, labels=dict(job["labels"]))
        r = py_oracle.process_job(policy, routing, live, job)
        rt = r["route"]
        out.append((wire.DEC_NAMES.index(r["decision"]), wire.DEC_NAMES.index(r["sched_decision"]), r["rule_idx"],
                    bool(r["approval_required"]), bool(r["has_snapshot"]), bool(r["has_constraints"]),
                    STATUS_CODE[rt["status"]] if rt else 0, bool(rt["tie"]) if rt else False))
    return out


def rec_tuples(rec):
    return [(int(r["decision"]), int(r["sched_decision"]), int(r["rule_idx"]), bool(r["flags"] & wire.F_APPROVAL_REQUIRED),
             bool(r["flags"] & wire.F_HAS_SNAPSHOT), bool(r["flags"] & wire.F_CONSTRAINTS), int(r["route_status"]),
             bool(r["flags"] & wire.F_TIE)) for r in rec]


def fuzz_case(seed, max_rules):
    """(policy, routing, workers, jobs) of one seed of the three-way fuzz."""
    rng = random.Random(7000 + seed)
    policy, routing, workers = make_policy(rng, max_rules), make_routing(rng), make_workers(rng)
    jobs = [make_job(rng, workers) for _ in range(40 if max_rules <= 12 else 120)]
    return policy, routing, workers, jobs


def widen(monkeypatch):
    """Vocabularies large enough that the risk-tag, requires-token, label-pair and placement-label dictionaries outgrow
    the mask fields of the job record (tables.h WideLayout).  The generators read these module globals."""
    me = sys.modules[__name__]
    monkeypatch.setattr(me, "RISKS", RISKS + ["tag%02d" % i for i in range(90)] + ["TAG%02d " % i for i in range(0, 90, 7)])
    monkeypatch.setattr(me, "REQS", REQS + ["req%02d" % i for i in range(100)] + [" REQ%02d" % i for i in range(0, 100, 9)])
    monkeypatch.setattr(me, "LKEYS", LKEYS + ["k%02d" % i for i in range(30)])
    monkeypatch.setattr(me, "LVALS", LVALS + ["v%d" % i for i in range(8)])


def wide_case(seed):
    """(policy, routing, workers, jobs) of one seed of the wide-universe fuzz; call widen() first."""
    me = sys.modules[__name__]
    rng = random.Random(12000 + seed)
    policy, routing, workers = make_policy(rng, 300), make_routing(rng), make_workers(rng) + make_workers(rng) + make_workers(rng)
    for r in policy.get("rules", []):   # more rules with mask predicates than the base generator makes
        if rng.random() < 0.5:
            r["match"]["risk_tags"] = pick(rng, me.RISKS, 2, 5)
        if rng.random() < 0.4:
            r["match"]["requires"] = pick(rng, me.REQS, 1, 3)
        if rng.random() < 0.4:
            r["match"]["labels"] = {rng.choice(me.LKEYS): rng.choice(me.LVALS) for _ in range(rng.randint(1, 2))}
    for p in routing["pools"].values():
        if rng.random() < 0.7:
            p["requires"] = pick(rng, me.REQS, 1, 6)
    jobs = []
    for _ in range(150):
        j = make_job(rng, workers)
        if rng.random() < 0.5:
            j.setdefault("meta", {})
            j["meta"] = dict(j["meta"] or {})
            j["meta"]["risk_tags"] = pick(rng, me.RISKS, 0, 5)
            j["meta"]["requires"] = pick(rng, me.REQS, 0, 5)
        jobs.append(j)
    return policy, routing, workers, jobs


def life_cycle(seed, steps=6):
    """The reload / heartbeat sequence of one seed.  Yields (kind, payload, jobs): first ("load", (policy, routing,
    workers), jobs), then one step at a time - ("heartbeat", (slots, loads), jobs), ("workers", workers, jobs),
    ("routing", routing, jobs) or ("policy", policy, jobs) - where `jobs` is a fresh batch to check after the step."""
    rng = random.Random(9000 + seed)
    policy, routing, workers = make_policy(rng), make_routing(rng), make_workers(rng)
    yield "load", (policy, routing, workers), [make_job(rng, workers) for _ in range(30)]
    for step in range(steps):
        kind = rng.choice(["heartbeat", "heartbeat", "workers", "routing", "policy"])
        payload = None
        if kind == "heartbeat" and workers:
            n = len(workers)
            slots = np.array(sorted(rng.sample(range(n), rng.randint(1, n))), dtype=np.uint32)
            loads = np.zeros(len(slots), dtype=wire.LOAD_DTYPE)
            loads["active_jobs"] = [rng.randint(0, 9) for _ in slots]
            loads["max_parallel_jobs"] = [rng.choice([0, 4, 10]) for _ in slots]
            loads["cpu_load"] = np.array([rng.choice([0, 50, 89.99, 90, 100 * rng.random()]) for _ in slots], dtype=np.float32)
            loads["gpu_utilization"] = np.array([rng.choice([0, 0, 90, 100 * rng.random()]) for _ in slots], dtype=np.float32)
            payload = (slots, loads)
        elif kind == "workers":
            workers = payload = make_workers(rng)
        elif kind == "routing":
            routing = payload = make_routing(rng)
        elif kind == "policy":
            policy = payload = make_policy(rng)
        yield kind, payload, [make_job(rng, workers) for _ in range(30)]


def ascii_case(seed, max_rules):
    """fuzz_case with the ASCII-only awkward vocabulary of _ascii_vocabulary."""
    with vocabulary(_ascii_vocabulary()):
        return fuzz_case(seed, max_rules)


def ascii_life_cycle(seed):
    """The steps of life_cycle(seed), drawn from the ASCII-only vocabulary."""
    with vocabulary(_ascii_vocabulary()):
        return list(life_cycle(seed))


DUP_KEYS = ["mcp.server", "mcp_server", "mcpServer", "mcp.tool", "mcp_tool", "mcpTool", "mcp.resource", "mcp_resource", "mcpResource",
            "mcp.action", "mcp_action", "mcpAction", "secrets_present", "preferred_pool", "preferred_worker_id"]


def dup_case(seed):
    """ascii_case(seed, 12) with repeated label keys spliced into most jobs: labels become a list of (key, value) pairs in
    which some keys - ordinary and rule label keys, placement keys, every MCP alias, secrets_present and the routing
    hints - occur two or three times with different values.  Only the last occurrence counts."""
    policy, routing, workers, jobs = ascii_case(seed, 12)
    voc = _ascii_vocabulary()
    rng = random.Random(21000 + seed)
    values = {"secrets_present": ["true", "TRUE", "1", "yes", "no", " true ", ""], "preferred_pool": POOLS + ["nope", ""],
              "preferred_worker_id": [w["worker_id"] for w in workers] + ["ghost", ""]}
    for j in jobs:
        if rng.random() < 0.2:
            continue
        items = list((j.get("labels") or {}).items())
        for k in rng.sample(voc["LKEYS"] + DUP_KEYS, rng.randint(1, 4)) + [k for k, _ in items if rng.random() < 0.5]:
            vals = values.get(k, voc["MCP_VALS"] if k.startswith("mcp") else voc["LVALS"])
            for _ in range(rng.randint(2, 3)):
                items.insert(rng.randint(0, len(items)), (k, rng.choice(vals)))
        j["labels"] = items
    return policy, routing, workers, jobs


def sparse_summary_case():
    """(policy, routing, workers, jobs) whose risk-tag, capability and pack rows are sparse: 96 tags (32 of them beyond the
    record's 64-bit mask), each owning one block of 32 consecutive rules, so a tag's row - and its summary - covers one
    128-bit word (shared by four tags).  A summary taken from the wrong row drops the word that holds the job's first
    match.  In the fuzz configurations most rules list no risk tag, every risk row is dense and the risk
    summaries skip nothing."""
    tags = ["tag%02d" % i for i in range(96)]
    rules = []
    for i in range(96 * 32):
        m = {"topics": ["job.r.*"], "risk_tags": [tags[i // 32]]}
        if i % 32 < 16:
            m["capabilities"] = ["cap%d" % (i % 4)]
        if i % 32 < 8:
            m["pack_ids"] = ["pack%d" % (i % 2)]
        rules.append({"id": "r%d" % i, "decision": ("deny", "require_approval", "throttle", "allow")[i % 4], "reason": "r", "match": m})
    policy = {"default_tenant": "default", "rules": rules}
    routing = {"topics": {"job.r.x": ["p"]}, "pools": {"p": {}}}
    workers = [kats.hb("w%d" % i, "p", i % 3, 10.0 * i, 0.0, 4) for i in range(8)]
    rng = random.Random(96)
    jobs = []
    for i in range(2000):
        k = rng.choice([0, 1, 1, 1, 2, 4])
        meta = {"risk_tags": rng.sample(tags, k), "capability": rng.choice(["cap0", "cap1", "cap2", "cap3", "other", ""]),
                "pack_id": rng.choice(["pack0", "pack1", ""])}
        jobs.append({"topic": "job.r.x", "meta": meta})
    return policy, routing, workers, jobs


# CORDUM_SUM_USE: which attributes' summaries policy_kernel ANDs before it visits a word group (tables.h SUM_*).  None leaves
# the choice to the table compiler; the forced values switch each summary on alone, none of them, and all of them.
SUM_USE_FORCED = [0, 1, 2, 4, 8, 16, 32, 63]


def force_sum_use(monkeypatch, sum_use):
    if sum_use is not None:
        monkeypatch.setenv("CORDUM_SUM_USE", str(sum_use))
    else:
        monkeypatch.delenv("CORDUM_SUM_USE", raising=False)


def with_sum_use(cases):
    """pytest parameters (*case, sum_use): ids name the case alone when the table compiler chooses, and add "-sum<value>"
    where CORDUM_SUM_USE is forced."""
    return [pytest.param(*c, id="-".join(str(x) for x in c[:-1]) + ("" if c[-1] is None else "-sum%d" % c[-1])) for c in cases]


@pytest.mark.parametrize("seed,max_rules,sum_use", with_sum_use([(s, 12, None) for s in range(60)] + [(100 + s, 400, None) for s in range(12)] +
                                                                [(100 + s, 400, u) for s in range(12) for u in SUM_USE_FORCED]))
def test_three_implementations_agree(seed, max_rules, sum_use, monkeypatch):
    """max_rules = 400: several 128-bit words of rule positions, so clustering by topic prefix, duplicated positions of
    multi-pattern rules, per-topic word lists and the ascending order inside a word all take part.  With sum_use forced,
    the walk skips word groups by whichever summaries the knob names (the table compiler reads it on every rebuild)."""
    force_sum_use(monkeypatch, sum_use)
    policy, routing, workers, jobs = fuzz_case(seed, max_rules)
    agree_three_ways(seed, policy, routing, workers, jobs, sum_use)


def agree_three_ways(seed, policy, routing, workers, jobs, sum_use=None):
    env = wire.EnvelopeBatch.from_jobs(jobs)
    o = oracle_lib.Oracle(policy, routing, workers)
    h = table_walk.HostHarness(policy, routing, workers)
    if sum_use is not None:
        assert h.tables()["sum_use"] == sum_use
    for mode in (wire.MODE_POLICY_AND_ROUTE, wire.MODE_POLICY_ONLY, wire.MODE_ROUTE_ONLY):
        want_m, got = o.eval(env, mode), h.evaluate(env, mode)
        for f in FIELDS:   # product host tables vs C++ oracle: every field of the record
            bad = np.nonzero(got[f] != want_m[f])[0]
            assert len(bad) == 0, "seed %d mode %d field %s job %s: tables %s oracle %s\n%s" % (
                seed, mode, f, bad[:4], got[f][bad[:4]], want_m[f][bad[:4]], json.dumps(jobs[int(bad[0])]))
    want = o.eval(env, wire.MODE_POLICY_AND_ROUTE)
    o.close()
    h.close()
    a, b = rec_tuples(want), py_records(policy, routing, workers, jobs)
    bad = [(i, x, y) for i, (x, y) in enumerate(zip(a, b)) if x != y]
    assert not bad, "seed %d C++ vs Python oracle: %s\n%s" % (seed, bad[:3], json.dumps(jobs[bad[0][0]]))


@pytest.mark.parametrize("seed,max_rules", [(s, 12) for s in range(60)] + [(100 + s, 400) for s in range(12)])
def test_three_implementations_agree_on_ascii_vocabulary(seed, max_rules):
    """The ASCII-only awkward vocabulary (_ascii_vocabulary): the inputs the device encoder keeps to itself, checked against
    both oracles here so that the GPU tests can take the host encoder as their reference."""
    agree_three_ways(seed, *ascii_case(seed, max_rules))


@pytest.mark.parametrize("seed", range(60))
def test_three_implementations_agree_on_repeated_label_keys(seed):
    """Labels with repeated keys (dup_case): the last value wins for rule label pairs, placement, every MCP alias,
    secrets_present and the routing hints."""
    policy, routing, workers, jobs = dup_case(seed)
    assert sum(len(j.get("labels") or []) > len(dict(j.get("labels") or [])) for j in jobs) >= len(jobs) // 2
    agree_three_ways(seed, policy, routing, workers, jobs)


@pytest.mark.parametrize("seed", range(30))
def test_reloads_and_heartbeats_keep_agreeing(seed):
    """The same engine-side objects across a life cycle: heartbeat deltas (loads by slot), a worker-registry reload, a
    routing reload and a policy reload, each followed by a re-evaluation of freshly encoded jobs - dictionaries are
    rebuilt, ids are reassigned and the tables must still agree with an oracle that went through the same calls."""
    check_life_cycle(seed, life_cycle(seed))


@pytest.mark.parametrize("seed", range(30))
def test_reloads_and_heartbeats_keep_agreeing_on_ascii_vocabulary(seed):
    check_life_cycle(seed, ascii_life_cycle(seed))


def check_life_cycle(seed, steps):
    o = h = None
    for step, (kind, payload, jobs) in enumerate(steps):
        if kind == "load":
            o, h = oracle_lib.Oracle(*payload), table_walk.HostHarness(*payload)
        elif kind == "heartbeat" and payload is not None:
            o.update_workers(*payload)
            h.update_workers(*payload)
        elif kind == "workers":
            o.load_workers(payload)
            h.load_workers(payload)
        elif kind == "routing":
            o.load_routing(payload)
            h.load_routing(payload)
        elif kind == "policy":
            o.load_policy(payload)
            h.load_policy(payload)
        env = wire.EnvelopeBatch.from_jobs(jobs)
        want, got = o.eval(env, wire.MODE_POLICY_AND_ROUTE), h.evaluate(env, wire.MODE_POLICY_AND_ROUTE)
        for f in FIELDS:
            bad = np.nonzero(got[f] != want[f])[0]
            assert len(bad) == 0, "seed %d after %s (step %d): field %s job %s: tables %s oracle %s\n%s" % (
                seed, kind, step - 1, f, bad[:4], got[f][bad[:4]], want[f][bad[:4]], json.dumps(jobs[int(bad[0])]))
    o.close()
    h.close()


@pytest.mark.parametrize("seed,sum_use", with_sum_use([(s, None) for s in range(16)] + [(s, u) for s in range(16) for u in SUM_USE_FORCED]))
def test_three_implementations_agree_with_wide_universes(seed, sum_use, monkeypatch):
    """The same agreement with vocabularies large enough that the risk-tag, requires-token, label-pair and placement-label
    dictionaries outgrow the mask fields of the job record (tables.h WideLayout: side rows of extra mask words), mixed
    with the awkward strings above, and across a reload back to a narrow policy.  Risk tags 64... have summaries of
    their own (row 1 + tag), which a forced SUM_RISK walks."""
    force_sum_use(monkeypatch, sum_use)
    widen(monkeypatch)
    policy, routing, workers, jobs = wide_case(seed)
    h = table_walk.HostHarness(policy, routing, workers)
    T = h.tables()
    assert T["xw_risk"] + T["xw_req"] + T["xw_lab"] + T["xw_place"] >= 2, (T["xw_risk"], T["xw_req"], T["xw_lab"], T["xw_place"])
    if sum_use is not None:
        assert T["sum_use"] == sum_use
    o = oracle_lib.Oracle(policy, routing, workers)
    env = wire.EnvelopeBatch.from_jobs(jobs)
    for mode in (wire.MODE_POLICY_AND_ROUTE, wire.MODE_POLICY_ONLY, wire.MODE_ROUTE_ONLY):
        want_m, got = o.eval(env, mode), h.evaluate(env, mode)
        for f in FIELDS:
            bad = np.nonzero(got[f] != want_m[f])[0]
            assert len(bad) == 0, "seed %d mode %d field %s job %s: tables %s oracle %s\n%s" % (
                seed, mode, f, bad[:4], got[f][bad[:4]], want_m[f][bad[:4]], json.dumps(jobs[int(bad[0])]))
    a, b = rec_tuples(o.eval(env, wire.MODE_POLICY_AND_ROUTE)), py_records(policy, routing, workers, jobs)
    bad = [(i, x, y) for i, (x, y) in enumerate(zip(a, b)) if x != y]
    assert not bad, "seed %d C++ vs Python oracle: %s\n%s" % (seed, bad[:3], json.dumps(jobs[bad[0][0]]))
    # narrow again: the side rows disappear and the same envelopes still agree
    monkeypatch.undo()
    narrow = make_policy(random.Random(seed), 12)
    h.load_policy(narrow)
    o2 = oracle_lib.Oracle(narrow, routing, workers)
    got, want = h.evaluate(env), o2.eval(env)
    for f in FIELDS:
        assert np.array_equal(got[f], want[f]), (seed, f)
    o.close(); o2.close(); h.close()
