#!/usr/bin/env python
"""mergebench.py — one heartbeat epoch's retries and new arrivals as one batch: a device merge (cordum_batch_merge) of the
retry subset and the device-encoded arrivals, against dispatching the two batches back to back, and against gathering the
retry envelopes with the arrivals' and encoding them together.

    python tools/mergebench.py [--jobs 1000000] [--reps 20] [--out FILE]

Workload: BASELINE config 3 at 2 x --jobs jobs, split in two: the first --jobs are the source batch, the rest the new
arrivals.  One heartbeat (cordum_workers_update) overloads every third pool, the source is dispatched (POLICY_AND_ROUTE)
and its THROTTLE / NO_WORKERS / POOL_OVERLOADED jobs are taken as a subset (cordum_batch_subset, RETRYABLE); the
arrivals are encoded on the device once.  Four paths, alternated inside every repetition, loads unchanged between them:
    merge_ms             device time of cordum_batch_merge(retry, arrivals): CUDA events on the destination's stream
                         around the call (its three kernels)
    merge_host_ms        host clock around the same call
    merge_dispatch_ms    host clock: the merge + cordum_dispatch_resident of the destination, ending in its synchronise
    two_dispatches_ms    host clock: cordum_dispatch_resident of the retry batch, then of the arrivals
    encode_both_ms       host clock: the retry envelopes gathered and concatenated with the arrivals' into pinned staging
                         (cordum_envelopes_alloc'd once), cordum_encode_device, cordum_dispatch
Median / min / max over --reps, after two warm-up repetitions.  Every repetition checks that the three ways give identical
decision records (the merge's = the retry batch's followed by the arrivals').  merge_gbps: the bytes the merge kernels
move (merge_bytes below, from the shapes) over the median merge_ms, and its share of the H100 SXM's 3.35 TB/s.  The
card's name and power limit are read in the same run (nvidia-smi query, nothing is changed).  Results: one JSON document
on stdout (and --out).
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
from subsetbench import FIELDS, stats, take  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM5 80 GB HBM3 peak


def merge_bytes(n_a, n_b, ww=0, sel_words=0):
    """Bytes the three merge kernels read and write for sources of n_a and n_b jobs (csrc/merge.cu):
    key kernel: the first 16 B of each JobRec, a tenant-class byte, and the 4 B key written back;
    gather: each key again, one binary search over the other source's keys (counted as its 4 B leaf: the upper levels
    are shared by a warp and stay in L1 / L2), the 64 B JobRec and 32 B RouteRec read and written, 4 B of slot_of, and
    the wide rows (ww 64-bit words) read and written; the selective lists (sel_words 32-bit words together) read and
    written about twice."""
    n = n_a + n_b
    key = n * (16 + 1 + 4)
    gather = n * (4 + 4 + 2 * (64 + 32) + 4 + 2 * 8 * ww)
    return key + gather + 4 * 4 * sel_words


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    cfg = synth.make_config("c3", 2 * a.jobs)
    n = a.jobs
    src_env, new_env = take(cfg.jobs, np.arange(n)), take(cfg.jobs, np.arange(n, cfg.jobs.n_jobs))
    e = engine.Engine(device=0)
    e.load_policy(cfg.policy, "mergebench")
    e.load_routing(cfg.routing)
    e.load_workers(cfg.workers)
    W = cfg.workers.n_workers
    loads = cfg.workers.loads().copy()
    pools = np.array([w["pool"] for w in cfg.workers.to_workers()])
    hot = sorted(set(pools.tolist()))[::3]
    loads["cpu_load"][np.isin(pools, hot)] = 95.0
    e.update_workers(np.arange(W, dtype=np.uint32), loads)
    src, retry, new = e.batch(n), e.batch(n), e.batch(new_env.n_jobs)
    rec = src.encode(src_env).dispatch().copy()
    m_retry = src.subset(retry, outcomes=wire.SUBSET_RETRYABLE)
    parent = retry.parent_index().copy()
    new.encode_device(new_env.deinterned()).wait()
    if e.host_fallbacks():   # first sight of a topic: the host encoder finished it, a dispatch puts it on the device
        new.dispatch()
    m = m_retry + new_env.n_jobs
    dst, both = e.batch(m), e.batch(m)
    both_env = take(cfg.jobs, np.concatenate([parent, np.arange(n, cfg.jobs.n_jobs)]))
    pinned = e.pinned_envelopes(like=both_env)
    stream = torch.cuda.ExternalStream(dst.stream)
    before = e.launch_count()
    retry.merge(new, dst)
    launches = e.launch_count() - before
    t_dev, t_host, t_md, t_two, t_enc = [], [], [], [], []
    same = True
    for r in range(a.reps + 2):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(stream)
        t0 = time.perf_counter()
        retry.merge(new, dst)
        t1 = time.perf_counter()
        e1.record(stream)
        e1.synchronize()
        t2 = time.perf_counter()
        retry.merge(new, dst)
        dst.dispatch_resident()
        t3 = time.perf_counter()
        got_merge = dst.fetch().copy()
        t4 = time.perf_counter()
        retry.dispatch_resident()
        new.dispatch_resident()
        t5 = time.perf_counter()
        got_two = np.concatenate([retry.fetch().copy(), new.fetch().copy()])
        t6 = time.perf_counter()
        pinned.fill(take(cfg.jobs, np.concatenate([parent, np.arange(n, cfg.jobs.n_jobs)])))
        both.encode_device(pinned)
        got_enc = both.dispatch().copy()
        t7 = time.perf_counter()
        ok = len(got_merge) == m
        for f in FIELDS:
            ok = ok and np.array_equal(got_merge[f], got_two[f]) and np.array_equal(got_merge[f], got_enc[f])
        same = same and bool(ok)
        if r >= 2:
            t_dev.append(e0.elapsed_time(e1))
            t_host.append((t1 - t0) * 1e3)
            t_md.append((t3 - t2) * 1e3)
            t_two.append((t5 - t4) * 1e3)
            t_enc.append((t7 - t6) * 1e3)
    nbytes = merge_bytes(m_retry, new_env.n_jobs)
    med = statistics.median(t_dev)
    st = rec["route_status"]
    doc = {"gpu": gpu, "source_jobs": n, "new_jobs": int(new_env.n_jobs), "retry_jobs": int(m_retry), "merged_jobs": int(m),
           "retry_by_status": {k: int(v) for k, v in (("THROTTLE", ((st == wire.ROUTE_NOT_ATTEMPTED) & (rec["sched_decision"] == wire.DEC_THROTTLE)).sum()),
                                                      ("NO_WORKERS", (st == wire.ROUTE_NO_WORKERS).sum()), ("POOL_OVERLOADED", (st == wire.ROUTE_POOL_OVERLOADED).sum()))},
           "reps": a.reps, "merge_launches": launches, "host_fallbacks": e.host_fallbacks(),
           "merge_ms": stats(t_dev), "merge_host_ms": stats(t_host), "merge_dispatch_ms": stats(t_md),
           "two_dispatches_ms": stats(t_two), "encode_both_ms": stats(t_enc),
           "merge_bytes": nbytes, "merge_gbps": nbytes / (med * 1e-3) / 1e9, "merge_hbm_share": nbytes / (med * 1e-3) / HBM_BYTES_PER_S,
           "outputs_identical": same}
    pinned.free()
    for b in (src, retry, new, dst, both):
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
