#!/usr/bin/env python
"""planbench.py — the dispatch plan (cordum_batch_plan) against fetching the records and grouping them on the host.

    python tools/planbench.py [--jobs 1000000] [--reps 20] [--out FILE]

Workloads, each one dispatched batch of --jobs jobs:
    c3            BASELINE config 3 (4,096 rules, 65,536 workers), POLICY_AND_ROUTE: 65,548 buckets, three radix passes
    c3_policy     the same batch in POLICY_ONLY mode: every job in one of six outcome buckets (heavy skew)
    hostnames     the 60,000-hostname registry of tools/selbench.py (256 pools, a tenth of the jobs pinned to a host),
                  POLICY_AND_ROUTE: 60,012 buckets, two passes
Per workload, median / min / max over --reps:
    plan_ms       device time of the plan: CUDA events on the batch's stream around the call (its kernels and the D2H of the
                  offsets and job indices)
    plan_call_ms  host clock around the call (it returns once the arrays are in host memory)
    fetch_ms      host clock around cordum_batch_fetch: D2H of the 16 B records + synchronise
    group_ms      host clock of the numpy grouping of the fetched records (bucket key, stable argsort, bincount, cumsum)
and whether the plan equals the host grouping.  The card's name and power limit are read in the same run.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from cordum_b200 import engine, synth, wire  # noqa: E402


def host_grouping(rec, n_slots):
    st = rec["route_status"].astype(np.int64)
    routed = (st == wire.ROUTE_OK) | (st == wire.ROUTE_OK_PREFERRED)
    key = np.where(routed, rec["worker_slot"].astype(np.int64),
                   np.where(st == wire.ROUTE_NOT_ATTEMPTED, n_slots + rec["sched_decision"].astype(np.int64),
                            n_slots + 6 + st - wire.ROUTE_MISSING_TOPIC))
    jobs = np.argsort(key, kind="stable")
    offsets = np.zeros(n_slots + wire.PLAN_OUTCOMES + 1, np.int64)
    offsets[1:] = np.cumsum(np.bincount(key, minlength=n_slots + wire.PLAN_OUTCOMES))
    return offsets, jobs


def stats(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def measure(b, n_slots, reps):
    import torch

    stream = torch.cuda.ExternalStream(b.stream)
    plan, call, fetch, group = [], [], [], []
    same = True
    for r in range(reps + 2):   # the first two grow the scratch and warm up
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        t0 = time.perf_counter()
        offsets, jobs, ns = b.plan()
        t1 = time.perf_counter()
        e1.record(stream)
        e1.synchronize()
        t2 = time.perf_counter()
        rec = b.fetch()
        t3 = time.perf_counter()
        want_off, want_jobs = host_grouping(rec, n_slots)
        t4 = time.perf_counter()
        if r >= 2:
            plan.append(e0.elapsed_time(e1))
            call.append((t1 - t0) * 1e3)
            fetch.append((t3 - t2) * 1e3)
            group.append((t4 - t3) * 1e3)
        same = same and ns == n_slots and np.array_equal(offsets, want_off) and np.array_equal(jobs, want_jobs)
    buckets = int((np.diff(want_off) > 0).sum())
    return {"plan_ms": stats(plan), "plan_call_ms": stats(call), "fetch_ms": stats(fetch), "group_ms": stats(group),
            "n_slots": n_slots, "non_empty_buckets": buckets, "largest_bucket": int(np.diff(want_off).max()), "plan_equals_host": bool(same)}


def run(name, policy, routing, workers, env, mode, reps):
    e = engine.Engine(device=0)
    e.load_policy(policy, name)
    e.load_routing(routing)
    e.load_workers(workers)
    b = e.batch(env.n_jobs)
    b.encode(env).dispatch(mode)
    before = e.launch_count()
    b.plan()
    launches = e.launch_count() - before
    res = measure(b, workers.n_workers, reps)
    res["launches"] = launches
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
    doc["c3"] = run("c3", cfg.policy, cfg.routing, cfg.workers, cfg.jobs, wire.MODE_POLICY_AND_ROUTE, a.reps)
    doc["c3_policy"] = run("c3_policy", cfg.policy, cfg.routing, cfg.workers, cfg.jobs, wire.MODE_POLICY_ONLY, a.reps)
    del cfg
    import selbench

    policy, routing, workers = selbench.fleet(60000, 256, 1)
    table = wire.WorkerTable.from_workers(workers)
    env = wire.EnvelopeBatch.from_jobs(selbench.job_list(workers, a.jobs, 2))
    doc["hostnames"] = run("hostnames", policy, routing, table, env, wire.MODE_POLICY_AND_ROUTE, a.reps)
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
