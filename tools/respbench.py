#!/usr/bin/env python
"""respbench.py — batch responses (cordum_batch_responses) against the per-job host path a bulk caller has without it.

    python tools/respbench.py [--jobs 1000000] [--reps 10] [--out FILE]

Workload: BASELINE config 3 (4,096 rules, 65,536 workers, Zipf topics), one batch of --jobs jobs dispatched in
POLICY_AND_ROUTE mode.  Paths, run alternately --reps times after two warm-up rounds (median / min / max):
    device_ms        host clock around Batch.responses() (kernels, the copies of the classes and the job list, one reason
                     and one rule id rendered per class)
    device_event_ms  CUDA events on the batch's stream around the same call
    per_job_ms       cordum_batch_fetch, then cordum_reason and cordum_rule_id_at for every job (what the front-end does per
                     request), through ctypes
Both must give every job the same reason and rule id.  The card's name and power limit are read in the same run.
Results: one JSON document on stdout (and --out).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cordum_b200 import engine, synth, wire  # noqa: E402


def per_job(e, b):
    """Each job's (reason, rule id) as the front-end builds them (frontend.cpp), one library call per string."""
    L = e.L
    rec = b.fetch()
    gen = b.policy_gen()
    buf = C.create_string_buffer(4096)
    reasons, rule_ids = [], []
    dec, code, flags, rule = (rec[f].tolist() for f in ("decision", "reason_code", "flags", "rule_idx"))
    for j in range(len(rec)):
        r = ""
        if (code[j] != wire.REASON_NONE and dec[j] not in (wire.DEC_ALLOW, wire.DEC_ALLOW_WITH_CONSTRAINTS)) or code[j] == wire.REASON_APPROVAL_GRANTED:
            L.cordum_reason(e.h, b.h, j, buf, len(buf))
            r = buf.value.decode("utf-8", "replace")
        i = ""
        if flags[j] & wire.F_HAS_SNAPSHOT:
            L.cordum_rule_id_at(e.h, gen, rule[j], buf, len(buf))
            i = buf.value.decode("utf-8", "replace")
        reasons.append(r)
        rule_ids.append(i)
    return reasons, rule_ids


def expand(resp, n):
    reasons, rule_ids = [None] * n, [None] * n
    off, jobs = resp["offsets"], resp["jobs"]
    for c in range(len(resp["classes"])):
        for j in jobs[off[c]:off[c + 1]].tolist():
            reasons[j], rule_ids[j] = resp["reasons"][c], resp["rule_ids"][c]
    return reasons, rule_ids


def stats(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs)}


def main():
    import torch

    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    cfg = synth.make_config("c3", a.jobs)
    e = engine.Engine(device=0)
    e.load_policy(cfg.policy, "c3")
    e.load_routing(cfg.routing)
    e.load_workers(cfg.workers)
    b = e.batch(cfg.jobs.n_jobs)
    b.encode(cfg.jobs).dispatch(wire.MODE_POLICY_AND_ROUTE)
    before = e.launch_count()
    resp = b.responses()
    launches = e.launch_count() - before
    stream = torch.cuda.ExternalStream(b.stream)
    dev, ev, host = [], [], []
    same = True
    for r in range(a.reps + 2):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record(stream)
        t0 = time.perf_counter()
        resp = b.responses()
        t1 = time.perf_counter()
        e1.record(stream)
        e1.synchronize()
        got = expand(resp, cfg.jobs.n_jobs)
        t2 = time.perf_counter()
        want = per_job(e, b)
        t3 = time.perf_counter()
        if r >= 2:
            dev.append((t1 - t0) * 1e3)
            ev.append(e0.elapsed_time(e1))
            host.append((t3 - t2) * 1e3)
        same = same and got == want
    sizes = [int(x) for x in (resp["offsets"][1:].astype("int64") - resp["offsets"][:-1].astype("int64"))]
    doc = {"gpu": gpu, "jobs": a.jobs, "reps": a.reps, "device_ms": stats(dev), "device_event_ms": stats(ev),
           "per_job_ms": stats(host), "classes": len(resp["classes"]), "largest_class": max(sizes) if sizes else 0,
           "launches": launches, "identical": bool(same)}
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
