#!/usr/bin/env python
"""countbench.py — per-topic outcome counts (cordum_batch_topic_counts) against the two ways a bulk caller gets them
without it.

    python tools/countbench.py [--jobs 1000000] [--reps 20] [--out FILE]

Workloads, each one batch of --jobs jobs dispatched in POLICY_AND_ROUTE mode:
    c3            BASELINE config 3 (4,096 rules, 65,536 workers, Zipf topics)
    c3_one_topic  the same batch with every job's topic set to the first job's: one row, the whole batch on one topic id
Paths, run alternately --reps times after two warm-up rounds (median / min / max):
    device_ms        host clock around Batch.topic_counts() (kernels, the copy of the non-zero rows, the merge by label)
    device_event_ms  CUDA events on the batch's stream around the same call
    records_ms       cordum_batch_records (JobRec topic ids + slot_of) and cordum_batch_fetch (16 B records), a numpy bincount
                     over (topic id, column), the ids named from the envelopes and merged by TrimSpace label
    strings_ms       cordum_batch_fetch, then each job's topic string from the envelopes grouped in a dict by its
                     TrimSpace label, joined with the fetched records' columns by a bincount
All three tables must be identical.  The card's name and power limit are read in the same run.
Results: one JSON document on stdout (and --out).
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cordum_b200 import engine, synth, wire  # noqa: E402

NCOL = wire.COUNT_COLUMNS


def go_trim(raw: bytes) -> bytes:
    """Go's strings.TrimSpace, through the library's own implementation."""
    import ctypes as C

    from cordum_b200 import _lib

    off, ln = C.c_uint64(), C.c_uint64()
    _lib.load().cordum_test_trim(raw, len(raw), C.byref(off), C.byref(ln))
    return raw[off.value:off.value + ln.value]


def columns(rec):
    st = rec["route_status"].astype(np.int64)
    return np.where((st == wire.ROUTE_OK) | (st == wire.ROUTE_OK_PREFERRED), wire.COUNT_ROUTED,
                    np.where(st == wire.ROUTE_NOT_ATTEMPTED, rec["sched_decision"].astype(np.int64), 6 + st - wire.ROUTE_MISSING_TOPIC))


def topic_bytes(env, j):
    t = env.cols["topic"][j]
    return bytes(env.arena[int(t["off"]):int(t["off"]) + int(t["len"])])


def merge(names, rows):
    """Rows keyed by raw name -> (labels ascending, counts) merged by TrimSpace label."""
    acc = {}
    for name, row in zip(names, rows):
        lab = go_trim(name)
        acc[lab] = acc.get(lab, 0) + row
    labels = sorted(acc)
    return labels, np.array([acc[k] for k in labels], dtype=np.uint32).reshape(len(labels), NCOL)


def by_records(b, env):
    job, _, slot_of = b.records()
    rec = b.fetch()
    tid = job["topic"].astype(np.int64)[slot_of]
    n_ids = int(tid.max()) + 1 if len(tid) else 0
    table = np.bincount(tid * NCOL + columns(rec), minlength=n_ids * NCOL).reshape(n_ids, NCOL)
    ids = np.flatnonzero(table.sum(axis=1))
    first = np.full(n_ids, -1, np.int64)
    first[tid[::-1]] = np.arange(len(tid))[::-1]       # a job of each id, to name it from the envelopes
    return merge([topic_bytes(env, int(first[i])) for i in ids], table[ids])


def by_strings(b, env):
    rec = b.fetch()
    t = env.cols["topic"][:env.n_jobs]
    arena = env.arena.tobytes()
    label_of, row_of, idx = {}, {}, np.empty(env.n_jobs, np.int64)
    for j, (o, ln) in enumerate(zip(t["off"].tolist(), t["len"].tolist())):
        raw = arena[o:o + ln]
        lab = label_of.get(raw)
        if lab is None:
            lab = label_of[raw] = go_trim(raw)
        idx[j] = row_of.setdefault(lab, len(row_of))
    table = np.bincount(idx * NCOL + columns(rec), minlength=len(row_of) * NCOL).reshape(len(row_of), NCOL)
    return merge(list(row_of), table)


def stats(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def run(name, cfg, env, reps):
    import torch

    e = engine.Engine(device=0)
    e.load_policy(cfg.policy, name)
    e.load_routing(cfg.routing)
    e.load_workers(cfg.workers)
    b = e.batch(env.n_jobs)
    b.encode(env).dispatch(wire.MODE_POLICY_AND_ROUTE)
    before = e.launch_count()
    b.topic_counts()
    launches = e.launch_count() - before
    stream = torch.cuda.ExternalStream(b.stream)
    dev, ev, recs, strs = [], [], [], []
    same = True
    for r in range(reps + 2):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        t0 = time.perf_counter()
        labels, counts = b.topic_counts()
        t1 = time.perf_counter()
        e1.record(stream)
        e1.synchronize()
        counts = counts.copy()
        t2 = time.perf_counter()
        l2, c2 = by_records(b, env)
        t3 = time.perf_counter()
        l3, c3 = by_strings(b, env)
        t4 = time.perf_counter()
        if r >= 2:
            dev.append((t1 - t0) * 1e3)
            ev.append(e0.elapsed_time(e1))
            recs.append((t3 - t2) * 1e3)
            strs.append((t4 - t3) * 1e3)
        same = same and labels == l2 == l3 and np.array_equal(counts, c2) and np.array_equal(counts, c3)
    res = {"device_ms": stats(dev), "device_event_ms": stats(ev), "records_ms": stats(recs), "strings_ms": stats(strs),
           "rows": len(labels), "largest_row": int(counts.sum(axis=1).max()), "launches": launches, "identical": bool(same)}
    b.free()
    e.close()
    print(name, json.dumps(res), file=sys.stderr, flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    doc = {"gpu": gpu, "jobs": a.jobs, "reps": a.reps}
    cfg = synth.make_config("c3", a.jobs)
    doc["c3"] = run("c3", cfg, cfg.jobs, a.reps)
    cols = dict(cfg.jobs.cols)
    cols["topic"] = np.full_like(cols["topic"], cols["topic"][0])
    one = wire.EnvelopeBatch(cfg.jobs.n_jobs, cfg.jobs.arena, cols)
    doc["c3_one_topic"] = run("c3_one_topic", cfg, one, a.reps)
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
