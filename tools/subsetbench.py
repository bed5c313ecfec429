#!/usr/bin/env python
"""subsetbench.py — requeueing a dispatched batch's retryable jobs: a device subset (cordum_batch_subset) against encoding
the same jobs again.

    python tools/subsetbench.py [--jobs 1000000] [--reps 20] [--out FILE]

Workload: BASELINE config 3 at --jobs jobs.  One heartbeat (cordum_workers_update) overloads every third pool, then the
batch is dispatched (POLICY_AND_ROUTE); its THROTTLE / NO_WORKERS / POOL_OVERLOADED jobs are the retry set.  Four paths,
alternated inside every repetition, loads unchanged between them:
    subset_ms            device time of cordum_batch_subset(RETRYABLE): CUDA events on the destination's stream around the
                         call (its four kernels, the 16 B readback of the counts between them, the D2H of the parent index)
    subset_dispatch_ms   host clock: the subset + cordum_dispatch_resident of the destination, ending in its synchronise
    encode_device_ms     host clock: the selected jobs' envelopes gathered and copied into pinned staging
                         (cordum_envelopes_alloc'd once), cordum_encode_device, cordum_dispatch
    encode_host_ms       host clock: the selected jobs' envelopes gathered, cordum_encode, cordum_dispatch
    build_ms             host clock of the envelope gather + pinned copy alone (part of encode_device_ms)
Median / min / max over --reps, after two warm-up repetitions.  Every repetition checks that the parent index is the
selection and that the three dispatched paths give identical records.  The card's name and power limit are read in the
same run (nvidia-smi query, nothing is changed).  Results: one JSON document on stdout (and --out).
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

FIELDS = ("decision", "sched_decision", "flags", "route_status", "reason_code", "rule_idx", "worker_slot")


def take(env, idx):
    """The envelopes of jobs idx (ascending) as a batch of their own (CSR columns re-based, arena shared)."""
    cols = {k: env.cols[k][idx] for k in env.SCALARS + ("has_meta", "actor_type", "approved")}
    for off, vals in (("risk_off", ("risk_tags",)), ("requires_off", ("requires_",)), ("label_off", ("label_keys", "label_vals"))):
        o = env.cols[off].astype(np.int64)
        lens = o[idx + 1] - o[idx]
        new = np.zeros(len(idx) + 1, np.int64)
        np.cumsum(lens, out=new[1:])
        pick = np.repeat(o[idx] - new[:-1], lens) + np.arange(new[-1])
        cols[off] = new.astype(np.uint32)
        for v in vals:
            part = env.cols[v][pick]
            cols[v] = part if len(part) else np.zeros(1, dtype=wire.STR_DTYPE)
    return wire.EnvelopeBatch(len(idx), env.arena, cols)


def stats(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    cfg = synth.make_config("c3", a.jobs)
    e = engine.Engine(device=0)
    e.load_policy(cfg.policy, "subsetbench")
    e.load_routing(cfg.routing)
    e.load_workers(cfg.workers)
    W = cfg.workers.n_workers
    loads = cfg.workers.loads().copy()
    pools = np.array([w["pool"] for w in cfg.workers.to_workers()])
    hot = sorted(set(pools.tolist()))[::3]
    loads["cpu_load"][np.isin(pools, hot)] = 95.0
    e.update_workers(np.arange(W, dtype=np.uint32), loads)
    n = cfg.jobs.n_jobs
    src, dst, dev, host = e.batch(n), e.batch(n), e.batch(n), e.batch(n)
    rec = src.encode(cfg.jobs).dispatch().copy()
    st = rec["route_status"]
    retry = np.flatnonzero((st == wire.ROUTE_NO_WORKERS) | (st == wire.ROUTE_POOL_OVERLOADED) |
                           ((st == wire.ROUTE_NOT_ATTEMPTED) & (rec["sched_decision"] == wire.DEC_THROTTLE)))
    pinned = e.pinned_envelopes(like=take(cfg.jobs, retry))
    stream = torch.cuda.ExternalStream(dst.stream)
    t_sub, t_sub_disp, t_dev, t_host, t_build = [], [], [], [], []
    same = True
    before = e.launch_count()
    src.subset(dst, outcomes=wire.SUBSET_RETRYABLE)
    launches = e.launch_count() - before
    for r in range(a.reps + 2):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        m = src.subset(dst, outcomes=wire.SUBSET_RETRYABLE)
        e1.record(stream)
        e1.synchronize()
        ok = m == len(retry) and np.array_equal(dst.parent_index(), retry)
        t0 = time.perf_counter()
        src.subset(dst, outcomes=wire.SUBSET_RETRYABLE)
        dst.dispatch_resident()
        t1 = time.perf_counter()
        got_sub = dst.fetch().copy()
        t2 = time.perf_counter()
        pinned.fill(take(cfg.jobs, retry))
        t3 = time.perf_counter()
        dev.encode_device(pinned)
        got_dev = dev.dispatch().copy()
        t4 = time.perf_counter()
        got_host = host.encode(take(cfg.jobs, retry)).dispatch().copy()
        t5 = time.perf_counter()
        for f in FIELDS:
            ok = ok and np.array_equal(got_sub[f], got_dev[f]) and np.array_equal(got_sub[f], got_host[f]) and np.array_equal(got_sub[f], rec[f][retry])
        same = same and bool(ok)
        if r >= 2:
            t_sub.append(e0.elapsed_time(e1))
            t_sub_disp.append((t1 - t0) * 1e3)
            t_dev.append((t4 - t2) * 1e3)
            t_build.append((t3 - t2) * 1e3)
            t_host.append((t5 - t4) * 1e3)
    doc = {"gpu": gpu, "jobs": n, "reps": a.reps, "retry_jobs": int(len(retry)),
           "retry_by_status": {k: int(v) for k, v in (("THROTTLE", ((st == wire.ROUTE_NOT_ATTEMPTED) & (rec["sched_decision"] == wire.DEC_THROTTLE)).sum()),
                                                      ("NO_WORKERS", (st == wire.ROUTE_NO_WORKERS).sum()), ("POOL_OVERLOADED", (st == wire.ROUTE_POOL_OVERLOADED).sum()))},
           "subset_launches": launches, "host_fallbacks": e.host_fallbacks(),
           "subset_ms": stats(t_sub), "subset_dispatch_ms": stats(t_sub_disp), "encode_device_ms": stats(t_dev),
           "encode_host_ms": stats(t_host), "build_ms": stats(t_build), "outputs_identical": same}
    pinned.free()
    for b in (src, dst, dev, host):
        b.free()
    e.close()
    s = json.dumps(doc, indent=1)
    print(s)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(s)


if __name__ == "__main__":
    main()
