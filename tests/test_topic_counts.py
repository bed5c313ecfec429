"""cordum_batch_topic_counts: a dispatched batch's jobs counted per TrimSpace(topic) label and plan outcome column, on the
device.  The expected table comes from the envelopes the test built (raw topic per job, trimmed by the oracle's
restatement of Go's strings.TrimSpace) and the batch's own decision records (plan outcome per job, as test_batch_plan
computes it), grouped in Python: labels, row order and every count must match, and the column sums must equal the plan's
bucket sizes.  Every dispatch path and encoder, subsets, labels that Go and Python trim differently, tile edges, one
topic and thousands of topics, reloads and new dictionary generations after the dispatch, the call order and the exact
launch count; and reference_api.topic_metrics against a per-job restatement of the engine.go increments."""
import ctypes as C

import numpy as np
import pytest

import kats
import oracle_lib
import test_batch_subset as tbs
from cordum_b200 import reference_api, synth, wire

pytestmark = pytest.mark.gpu

MODES = tbs.MODES
PATHS = tbs.PATHS
TILE = 2048            # sorted records per CTA of topic_count_kernel (csrc/kernels.h CORDUM_COUNT_TILE)
COUNT_LAUNCHES = 2     # topic_count_kernel + topic_rows_kernel
E_INVALID, E_STATE = -1, -4
NCOL = wire.COUNT_COLUMNS


@pytest.fixture(scope="module")
def eng():
    from cordum_b200 import engine

    e = engine.Engine(device=0)
    yield e
    e.close()


def raw_topics(env) -> list:
    """Each job's raw topic bytes, from the envelopes."""
    if not isinstance(env, wire.EnvelopeBatch):
        env = wire.EnvelopeBatch.from_jobs(env)
    t = env.cols["topic"][:env.n_jobs]
    arena = np.asarray(env.arena).tobytes()
    return [arena[o:o + ln] for o, ln in zip(t["off"].tolist(), t["len"].tolist())]


_TRIMMED = {}


def trimmed(raw: bytes) -> bytes:
    """Go's strings.TrimSpace (the oracle's restatement), memoised per raw topic."""
    if raw not in _TRIMMED:
        _TRIMMED[raw] = oracle_lib.trim_space(raw)
    return _TRIMMED[raw]


def columns(rec) -> np.ndarray:
    """Count column per job: the plan outcome bucket, or COUNT_ROUTED (test_batch_plan.expected's rule)."""
    k = tbs.outcome(rec)
    return np.where(k < 0, wire.COUNT_ROUTED, k)


def expected(rec, topics):
    """(labels, counts) from the raw topics and the decision records, grouped in Python."""
    labels = [trimmed(t) for t in topics]
    names = sorted(set(labels))
    row = {lab: i for i, lab in enumerate(names)}
    idx = np.fromiter((row[lab] for lab in labels), dtype=np.int64, count=len(labels))
    counts = np.bincount(idx * NCOL + columns(rec), minlength=len(names) * NCOL).reshape(len(names), NCOL)
    return names, counts.astype(np.uint32)


def counts_checked(eng, b, rec, topics, what, plan=True):
    """b.topic_counts() against the expected table, its launch count and the plan's bucket sizes; returns copies."""
    before = eng.launch_count()
    labels, counts = b.topic_counts()
    assert eng.launch_count() - before == (COUNT_LAUNCHES if len(rec) else 0), what
    want_labels, want_counts = expected(rec, topics)
    assert labels == want_labels, (what, labels[:8], want_labels[:8])
    assert counts.dtype == np.uint32 and counts.shape == (len(want_labels), NCOL), what
    assert np.array_equal(counts, want_counts), what
    assert (counts.sum(axis=1) > 0).all() and counts.sum() == len(rec), what
    if plan:
        offsets, _, ns = b.plan()
        sizes = np.diff(offsets.astype(np.int64))
        assert np.array_equal(counts[:, :wire.PLAN_OUTCOMES].sum(axis=0), sizes[ns:]), what
        assert counts[:, wire.COUNT_ROUTED].sum() == sizes[:ns].sum(), what
    return list(labels), counts.copy()


def refused(code, fn):
    from cordum_b200 import engine

    with pytest.raises(engine.CordumError) as ei:
        fn()
    assert ei.value.code == code


# ------------------------------------------------------------------ every path, mode and encoder
@pytest.mark.parametrize("encoder", ["host", "device"])
@pytest.mark.parametrize("name", ["tiny", "c2", "c5", "fuzz"])
def test_every_dispatch_path(eng, name, encoder):
    policy, routing, workers, env = tbs.config(name)
    tbs.load(eng, policy, routing, workers)
    topics = raw_topics(env)
    loads = workers.loads()
    b = eng.batch(env.n_jobs)
    b.encode_device(env.deinterned()) if encoder == "device" else b.encode(env)
    refused(E_STATE, b.topic_counts)                     # encoded, never dispatched
    cols = set()
    for mode in MODES:
        for path in PATHS:
            if path == "tick" and mode != wire.MODE_POLICY_AND_ROUTE:
                continue
            if path == "async":
                b.dispatch_async(mode)
                refused(E_STATE, b.topic_counts)         # before the wait
                rec = b.wait().copy()
            else:
                rec = tbs.run(eng, b, mode, path, loads)
            _, counts = counts_checked(eng, b, rec, topics, "%s %s mode %d %s" % (name, encoder, mode, path))
            cols |= set(np.flatnonzero(counts.sum(axis=0)).tolist())
    assert len(cols) >= 3, cols
    b.encode(env)                                        # a new encode: no counts until the next dispatch
    refused(E_STATE, b.topic_counts)
    b.free()


def test_device_encode_that_falls_back_to_the_host(eng):
    cfg = synth.make_config("tiny")
    tbs.load(eng, cfg.policy, cfg.routing, cfg.workers)
    jobs = [{"topic": "job.first.seen.%d" % (i % 3)} if i % 5 == 0 else {"topic": "job.pack000.read", "labels": {"zone": "z%d" % (i % 4)}}
            for i in range(3000)]
    b = eng.batch(len(jobs))
    before = eng.host_fallbacks()
    b.encode_device(jobs)
    b.dispatch_async()
    refused(E_STATE, b.topic_counts)
    rec = b.wait().copy()
    assert eng.host_fallbacks() == before + 1
    labels, _ = counts_checked(eng, b, rec, raw_topics(jobs), "fallback")
    assert b"job.first.seen.2" in labels
    b.free()


# ------------------------------------------------------------------ subsets
@pytest.mark.parametrize("name", ["c2", "fuzz"])
def test_subsets(eng, name):
    policy, routing, workers, env = tbs.config(name)
    tbs.load(eng, policy, routing, workers)
    topics = raw_topics(env)
    src, dst = eng.batch(env.n_jobs), eng.batch(env.n_jobs)
    rec = src.encode(env).dispatch().copy()
    labels, counts = counts_checked(eng, src, rec, topics, name + " parent")
    # the retryable jobs, dispatched again without a load change, land in the same columns
    m = src.subset(dst, outcomes=wire.SUBSET_RETRYABLE)
    assert m > 0
    refused(E_STATE, dst.topic_counts)                   # a subset is encoded, not dispatched
    for path in PATHS:
        got = tbs.run(eng, dst, wire.MODE_POLICY_AND_ROUTE, path, workers.loads())
        parent = dst.parent_index().copy()
        sub_labels, sub_counts = counts_checked(eng, dst, got, [topics[p] for p in parent], "%s retryable %s" % (name, path))
        keep = np.zeros(NCOL, bool)
        keep[[wire.PLAN_THROTTLE, wire.PLAN_NO_WORKERS, wire.PLAN_POOL_OVERLOADED]] = True
        want = np.where(keep, counts, 0)
        rows = want.sum(axis=1) > 0
        assert sub_labels == [lab for lab, r in zip(labels, rows) if r], (name, path)
        assert np.array_equal(sub_counts, want[rows]), (name, path)
    # a subset by list: every third job
    pick = np.arange(0, env.n_jobs, 3)
    src.subset(dst, jobs=pick)
    got = dst.dispatch(wire.MODE_POLICY_AND_ROUTE).copy()
    counts_checked(eng, dst, got, [topics[p] for p in pick], name + " list")
    src.free()
    dst.free()


# ------------------------------------------------------------------ labels
GO_SPACES = [" job.a", "job.a\t", " job.a ", "\u0085job.a", "\n\vjob.a\f\r", "　job.a ", "job.a"]
NOT_GO_SPACES = ["\x1cjob.a", "\x1fjob.a", "​job.a", "﻿job.a"]   # Python's str.strip trims \x1c-\x1f, Go does not
EMPTY = ["", "   ", "\t\n"]
ODD = ["job.\x00nul", "\x00", "other.topic", "job.b", "job.\xe9t\xe9"]


def test_labels_are_go_trim_space(eng):
    routing = {"topics": {"job.a": ["p"], " job.a": ["p"], "job.b": ["p"]}, "pools": {"p": {}}}
    tbs.load(eng, None, routing, [kats.hb("w1", "p"), kats.hb("w2", "p")])
    vocab = GO_SPACES + NOT_GO_SPACES + EMPTY + ODD
    jobs = [{"topic": vocab[(i * 7) % len(vocab)]} for i in range(3 * TILE + 11)]
    topics = raw_topics(jobs)
    b = eng.batch(len(jobs))
    for mode in MODES:
        rec = b.encode(jobs).dispatch(mode).copy()
        labels, counts = counts_checked(eng, b, rec, topics, "vocabulary mode %d" % mode)
        total = dict(zip(labels, counts.sum(axis=1).tolist()))
        n_of = {v: sum(1 for j in jobs if j["topic"] == v) for v in vocab}
        assert total[b"job.a"] == sum(n_of[v] for v in GO_SPACES)
        assert total[b""] == sum(n_of[v] for v in EMPTY)
        for v in NOT_GO_SPACES + ODD:
            assert total[v.encode()] == n_of[v], v
        assert labels == sorted(labels) and len(labels) == 2 + len(NOT_GO_SPACES) + len(ODD)
    b.free()


# ------------------------------------------------------------------ shapes
@pytest.mark.parametrize("n", [0, 1, TILE - 1, TILE, TILE + 1, 3 * TILE + 17])
def test_batch_sizes(eng, n):
    cfg = synth.make_config("c2")
    tbs.load(eng, cfg.policy, cfg.routing, cfg.workers)
    b = eng.batch(max(n, 1))
    env = cfg.jobs.slice(0, n)
    rec = b.encode(env).dispatch().copy()
    labels, counts = counts_checked(eng, b, rec, raw_topics(env), "n=%d" % n)
    if n == 0:
        assert labels == [] and counts.shape == (0, NCOL)
    b.free()


def test_one_topic_for_every_job(eng):
    """One label, several outcomes: " job.hot" has no pools (routing keys the raw topic) but counts under "job.hot"."""
    routing = {"topics": {"job.hot": ["p"]}, "pools": {"p": {}}}
    tbs.load(eng, None, routing, [kats.hb("w%d" % i, "p") for i in range(5)])
    n = 40 * TILE + 3
    jobs = [[{"topic": "job.hot"}, {"topic": " job.hot"}, {"topic": "job.hot", "labels": {"preferred_pool": "nope"}},
             {"topic": "job.hot", "meta": {"requires": ["tpu"]}}][i % 4] if i % 9 == 0 else {"topic": "job.hot"} for i in range(n)]
    b = eng.batch(n)
    for mode in MODES:
        rec = b.encode(jobs).dispatch(mode).copy()
        labels, counts = counts_checked(eng, b, rec, raw_topics(jobs), "one topic mode %d" % mode)
        assert labels == [b"job.hot"] and counts.sum() == n
    b.free()


def test_every_job_on_a_distinct_topic(eng):
    n = 6000
    routing = {"topics": {"job.t%05d" % i: ["p"] for i in range(0, n, 2)}, "pools": {"p": {}}}
    tbs.load(eng, None, routing, [kats.hb("w%d" % i, "p") for i in range(3)])
    order = (np.arange(n) * 4999) % n                     # first sight in a scattered order
    jobs = [{"topic": "job.t%05d" % i} for i in order]
    b = eng.batch(n)
    for mode in MODES:
        rec = b.encode(jobs).dispatch(mode).copy()
        labels, counts = counts_checked(eng, b, rec, raw_topics(jobs), "distinct topics mode %d" % mode)
        assert len(labels) == n and (counts.sum(axis=1) == 1).all()
    b.free()


@pytest.mark.slow
def test_config3_million_jobs(eng):
    cfg = synth.make_config("c3")
    tbs.load(eng, cfg.policy, cfg.routing, cfg.workers)
    b = eng.batch(cfg.jobs.n_jobs)
    rec = b.encode(cfg.jobs).dispatch().copy()
    counts_checked(eng, b, rec, raw_topics(cfg.jobs), "config 3")
    b.free()


# ------------------------------------------------------------------ life cycle
def test_labels_survive_reloads_and_new_dictionary_generations():
    from cordum_b200 import engine

    e = engine.Engine(device=0, max_topics=16)
    try:
        routing = {"topics": {"job.a": ["p"]}, "pools": {"p": {}}}
        tbs.load(e, None, routing, [kats.hb("w1", "p")])
        first = [{"topic": "job.first.%d " % (i % 6)} for i in range(500)]
        b, c = e.batch(500), e.batch(500)
        rec = b.encode(first).dispatch().copy()
        want = counts_checked(e, b, rec, raw_topics(first), "first generation")
        # a new dictionary generation: 12 new topics do not fit next to the first generation's 8; topic ids are reused
        second = [{"topic": "job.second.%02d" % (i % 12)} for i in range(500)]
        rec2 = c.encode(second).dispatch().copy()
        counts_checked(e, c, rec2, raw_topics(second), "second generation")
        d = e.batch(500)
        refused(-6, lambda: b.subset(d, outcomes=wire.SUBSET_RETRYABLE | 1 << wire.DEC_ALLOW))   # b's ids are stale now
        again = counts_checked(e, b, rec, raw_topics(first), "first generation, after the second")
        assert again[0] == want[0] and np.array_equal(again[1], want[1])
        # policy, routing and workers reloads
        e.load_policy({"default_tenant": "default", "rules": [{"id": "d", "decision": "deny", "match": {"topics": ["job.*"]}}]}, "r")
        e.load_routing({"topics": {"job.z": ["q"]}, "pools": {"q": {}}})
        e.load_workers([kats.hb("x%d" % i, "q") for i in range(3)])
        again = counts_checked(e, b, rec, raw_topics(first), "after reloads", plan=False)
        assert again[0] == want[0] and np.array_equal(again[1], want[1])
        b.free()
        c.free()
        d.free()
    finally:
        e.close()


def test_plan_and_counts_do_not_invalidate_each_other(eng):
    cfg = synth.make_config("c2")
    tbs.load(eng, cfg.policy, cfg.routing, cfg.workers)
    b = eng.batch(cfg.jobs.n_jobs)
    rec = b.encode(cfg.jobs).dispatch().copy()
    offsets, jobs, _ = b.plan()
    off0, jobs0 = offsets.copy(), jobs.copy()
    labels, counts = b.topic_counts()
    counts0 = counts.copy()
    b.plan()
    assert np.array_equal(counts, counts0)                # the counts view after a second plan
    b.topic_counts()
    assert np.array_equal(offsets, off0) and np.array_equal(jobs, jobs0)   # the plan views after a second counts call
    counts_checked(eng, b, rec, raw_topics(cfg.jobs), "interleaved")
    b.free()


def test_refusals_and_launch_counts(eng):
    cfg = synth.make_config("tiny")
    tbs.load(eng, cfg.policy, cfg.routing, cfg.workers)
    b = eng.batch(cfg.jobs.n_jobs)
    out = wire.CordumTopicCounts()
    assert b.L.cordum_batch_topic_counts(None, C.byref(out)) == E_INVALID
    assert b.L.cordum_batch_topic_counts(b.h, None) == E_INVALID
    assert b.L.cordum_batch_topic_counts(b.h, C.byref(out)) == E_STATE      # never encoded
    b.encode(cfg.jobs)
    before = eng.launch_count()
    refused(E_STATE, b.topic_counts)
    assert eng.launch_count() == before
    rec = b.dispatch().copy()
    for _ in range(3):
        counts_checked(eng, b, rec, raw_topics(cfg.jobs), "repeat", plan=False)
    b.free()


# ------------------------------------------------------------------ the four counter vectors
def per_job_metrics(rec, topics):
    """engine.go's increments, job by job: handleJobRequest (:209-218, :239) and processJob (:333, :344, :404, :435)."""
    received, denied, completed, dispatched = {}, {}, {}, {}

    def inc(d, k):
        d[k] = d.get(k, 0) + 1

    for raw, r in zip(topics, rec):
        topic = oracle_lib.trim_space(raw)
        if topic == b"":
            inc(completed, (topic, "JOB_STATUS_FAILED"))
            continue
        inc(received, topic)
        st, sched = int(r["route_status"]), int(r["sched_decision"])
        if st == wire.ROUTE_NOT_ATTEMPTED:
            if sched in (wire.DEC_DENY, wire.DEC_UNSPECIFIED):
                inc(denied, topic)
        elif st in (wire.ROUTE_OK, wire.ROUTE_OK_PREFERRED):
            inc(dispatched, topic)
        elif st not in (wire.ROUTE_NO_WORKERS, wire.ROUTE_POOL_OVERLOADED):   # not retryable: FAILED
            inc(completed, (topic, "JOB_STATUS_FAILED"))
    return {"jobs_received_total": received, "safety_denied_total": denied, "jobs_completed_total": completed,
            "jobs_dispatched_total": dispatched}


@pytest.mark.parametrize("name", ["c2", "fuzz"])
def test_topic_metrics_match_the_engine_increments(eng, name):
    policy, routing, workers, env = tbs.config(name)
    tbs.load(eng, policy, routing, workers)
    topics = raw_topics(env)
    b = eng.batch(env.n_jobs)
    b.encode(env)
    for mode in MODES:
        rec = b.dispatch(mode).copy()
        labels, counts = b.topic_counts()
        got = reference_api.topic_metrics(labels, counts)
        assert got == per_job_metrics(rec, topics), (name, mode)
        assert sum(got["jobs_received_total"].values()) + got["jobs_completed_total"].get((b"", "JOB_STATUS_FAILED"), 0) == len(rec)
    b.free()
