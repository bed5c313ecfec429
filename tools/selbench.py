#!/usr/bin/env python
"""selbench.py — selective placement pairs against the dense label encoding, on a hostname-labelled fleet.

    python tools/selbench.py [--workers 60000] [--pools 256] [--jobs 250000] [--rounds 3] [--big 1000000] [--out FILE]

Registry: --workers workers in --pools pools, each with a hostname of its own plus a shared zone (8) and rack (64).
Jobs (seeded): a tenth pinned to one hostname (half of those with the host's zone too), the rest on zone / rack labels
or none.  The same registry and jobs run through two engines, alternating, `--rounds` times:
    selective  the default limits (CORDUM_SEL_MIN_BITS / CORDUM_SEL_MAX_HOLDERS): every hostname is a selective pair
    dense      cordum_test_set_selective(2^32-1, ...): every pair keeps a dense bit, bitmap row and side-row bit
and report per engine:
    refresh_ms        one heartbeat epoch (cordum_workers_ingest of all loads, H2D + refresh kernels), host clock around
                      ingest + device synchronise, median of 20
    derived_mib       derived-table bytes per set (pos_key, ckey, skey, label bitmaps, lbest, load copy), from the table shapes
    route_ms          route_kernel + route_select_kernel of one resident dispatch (cordum_batch_kernel_times), median
    resident_rate     decisions/s of back-to-back resident dispatches (records already in HBM)
    e2e_rate          decisions/s of host encode + H2D + kernels + D2H, per step
    fallbacks         cordum_host_fallbacks added by one device encode of the batch, and of the batch without its pinned jobs
Then one --big-job batch through the selective engine alone (the dense encoding needs 7.5 KB of side row per job and
refuses it).  The card's name and power limit are read in the same run.  Results: one JSON document on stdout (and --out).
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import random
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from cordum_b200 import _lib, engine, wire  # noqa: E402

DENSE_MIN_BITS, MAX_HOLDERS, SEL_MIN_BITS = 0xFFFFFFFF, 32, 1024


def set_limits(min_bits, max_holders=MAX_HOLDERS):
    L = _lib.load()
    L.cordum_test_set_selective.argtypes = [C.c_uint32, C.c_uint32]
    L.cordum_test_set_selective.restype = None
    L.cordum_test_set_selective(min_bits, max_holders)


def fleet(n_workers, n_pools, seed):
    rng = random.Random(seed)
    pools = ["p%03d" % p for p in range(n_pools)]
    routing = {"topics": {"job.run": pools}, "pools": {p: {} for p in pools}}
    workers = [{"worker_id": "w%06d" % i, "pool": pools[i % n_pools], "active_jobs": rng.randrange(4), "max_parallel_jobs": 8,
                "cpu_load": float(rng.randrange(0, 95, 5)), "gpu_utilization": 0.0,
                "labels": {"hostname": "node-%06d" % i, "zone": "z%d" % (i % 8), "rack": "r%02d" % (i % 64)}} for i in range(n_workers)]
    policy = {"default_tenant": "default", "rules": [{"id": "deny-x", "decision": "deny", "match": {"topics": ["job.x"]}}]}
    return policy, routing, workers


def job_list(workers, n, seed, pinned=True):
    rng = random.Random(seed)
    W = len(workers)
    out = []
    for t in range(n):
        k = t % 10
        i = rng.randrange(W)
        lab = workers[i]["labels"]
        if k == 0 and pinned:
            j = {"hostname": lab["hostname"]}
            if rng.random() < 0.5:
                j["zone"] = lab["zone"]
        elif k < 5:
            j = {"zone": "z%d" % rng.randrange(8)}
        elif k < 7:
            j = {"rack": "r%02d" % rng.randrange(64)}
        else:
            j = {}
        out.append({"topic": "job.run", "labels": j})
    return out


def derived_bytes(policy, routing, table):
    """Per derived-table set, from the compiled shapes (engine.cu sync_tables)."""
    L = _lib.load()
    L.cordum_test_host_new.restype = C.c_void_p
    L.cordum_test_host_scalar.restype = C.c_uint64
    L.cordum_test_host_scalar.argtypes = [C.c_void_p, C.c_char_p]
    h = C.c_void_p(L.cordum_test_host_new(0, 0, 1))
    for fn, doc in ((L.cordum_test_host_policy, json.dumps(policy).encode()), (L.cordum_test_host_routing, json.dumps(routing).encode())):
        fn.argtypes = [C.c_void_p, C.c_char_p, C.c_uint64]
        assert fn(h, doc, len(doc)) == 0
    L.cordum_test_host_workers.argtypes = [C.c_void_p, C.c_void_p]
    assert L.cordum_test_host_workers(h, C.addressof(table.struct)) == 0
    s = {k: int(L.cordum_test_host_scalar(h, k.encode())) for k in ("n_pos", "n_pools", "n_slots", "place_bits", "lbm_words", "n_sel")}
    L.cordum_test_host_free.argtypes = [C.c_void_p]
    L.cordum_test_host_free(h)
    lbest = s["n_pools"] * s["place_bits"] * 16 if s["place_bits"] <= SEL_MIN_BITS else 0
    total = 3 * 8 * s["n_pos"] + 4 * s["lbm_words"] + lbest + 16 * s["n_slots"] + 17 * s["n_pools"]
    return total, s


def run_engine(name, min_bits, policy, routing, table, env, env_plain, steps):
    set_limits(min_bits)
    e = engine.Engine(device=0)
    e.load_policy(policy, name)
    e.load_routing(routing)
    e.load_workers(table)
    W = table.n_workers
    loads = table.loads()
    import torch

    res = {}
    b = e.batch(env.n_jobs)
    b.encode(env).dispatch()
    torch.cuda.synchronize()
    # heartbeat epochs
    t = []
    for _ in range(20):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e.ingest(loads.ctypes.data, 0, W)
        torch.cuda.synchronize()
        t.append((time.perf_counter() - t0) * 1e3)
    res["refresh_ms"] = statistics.median(t[2:])
    # route kernels of resident dispatches
    r = []
    for _ in range(steps):
        b.dispatch_resident()
        r.append(b.kernel_times()[1])
    res["route_ms"] = statistics.median(r)
    # resident rate
    for _ in range(3):
        b.dispatch_resident_async(); b.wait()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        b.dispatch_resident_async()
        b.wait()
    res["resident_rate"] = env.n_jobs * steps / (time.perf_counter() - t0)
    # end to end: host encode + H2D + kernels + D2H
    t0 = time.perf_counter()
    for _ in range(max(3, steps // 4)):
        out = b.encode(env).dispatch()
    res["e2e_rate"] = env.n_jobs * max(3, steps // 4) / (time.perf_counter() - t0)
    res["records"] = out.copy()
    # device encoder: with and without the pinned jobs
    f0 = e.host_fallbacks()
    b.encode_device(env).dispatch()
    f1 = e.host_fallbacks()
    c = e.batch(env_plain.n_jobs)
    c.encode_device(env_plain).dispatch()
    res["fallbacks"] = {"with_pinned": f1 - f0, "without": e.host_fallbacks() - f1}
    c.free()
    b.free()
    e.close()
    set_limits(SEL_MIN_BITS)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workers", type=int, default=60000)
    ap.add_argument("--pools", type=int, default=256)
    ap.add_argument("--jobs", type=int, default=250000)
    ap.add_argument("--big", type=int, default=1000000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    policy, routing, workers = fleet(a.workers, a.pools, 1)
    table = wire.WorkerTable.from_workers(workers)
    jobs = job_list(workers, a.jobs, 2)
    env = wire.EnvelopeBatch.from_jobs(jobs)
    env_plain = wire.EnvelopeBatch.from_jobs(job_list(workers, a.jobs // 4, 3, pinned=False))
    doc = {"gpu": gpu, "workers": a.workers, "pools": a.pools, "jobs": a.jobs, "pinned_jobs": sum(1 for j in jobs if "hostname" in j["labels"])}
    for name, mb in (("selective", SEL_MIN_BITS), ("dense", DENSE_MIN_BITS)):
        set_limits(mb)
        doc[name + "_derived_bytes_per_set"], doc[name + "_shape"] = derived_bytes(policy, routing, table)
    set_limits(SEL_MIN_BITS)
    runs = {"selective": [], "dense": []}
    recs = {}
    for _ in range(a.rounds):
        for name, mb in (("selective", SEL_MIN_BITS), ("dense", DENSE_MIN_BITS)):
            r = run_engine(name, mb, policy, routing, table, env, env_plain, a.steps)
            recs[name] = r.pop("records")
            runs[name].append(r)
            print(name, json.dumps(r), file=sys.stderr, flush=True)
    doc["runs"] = runs
    doc["records_identical"] = all(np.array_equal(recs["selective"][f], recs["dense"][f]) for f in recs["dense"].dtype.names)
    if a.big:
        big = wire.EnvelopeBatch.from_jobs([jobs[i % len(jobs)] for i in range(a.big)])
        e = engine.Engine(device=0)
        e.load_policy(policy, "big")
        e.load_routing(routing)
        e.load_workers(table)
        b = e.batch(big.n_jobs)
        b.encode(big).dispatch()
        t0 = time.perf_counter()
        for _ in range(3):
            b.encode(big).dispatch()
        e2e = 3 * big.n_jobs / (time.perf_counter() - t0)
        r = []
        for _ in range(a.steps):
            b.dispatch_resident()
            r.append(b.kernel_times()[1])
        doc["big"] = {"jobs": a.big, "e2e_rate": e2e, "route_ms": statistics.median(r)}
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
