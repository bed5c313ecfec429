"""Kernel launches the engine counts (cordum_launch_count) on each way worker loads reach the device, and the records each
step routes on those loads.  Every load path refreshes the derived worker tables once per heartbeat epoch; a dispatch or a
tick that finds them current launches only policy_kernel and route_kernel.  The counts are exact, so a change to the
epoch bookkeeping that drops or repeats a refresh shows up here even where the records would still agree."""
import numpy as np
import pytest

import oracle_lib
from cordum_b200 import synth

pytestmark = pytest.mark.gpu
FIELDS = ("decision", "sched_decision", "flags", "route_status", "reason_code", "rule_idx", "worker_slot")

# tiny and c2 both compile to one worker_chunk launch per refresh and no merge launch
REFRESH = 1
POLICY_AND_ROUTE = 2


@pytest.fixture(scope="module")
def eng():
    from cordum_b200 import engine

    e = engine.Engine(device=0)
    yield e
    e.close()


def assert_same(got, want, what):
    for f in FIELDS:
        assert np.array_equal(got[f], want[f]), (what, f)


@pytest.mark.parametrize("name,n", [("tiny", 2000), ("c2", None)])
def test_launch_counts_per_load_path(eng, name, n):
    cfg = synth.make_config(name, n)
    eng.load_policy(cfg.policy, "launches")
    eng.load_routing(cfg.routing)
    eng.load_workers(cfg.workers)
    o = oracle_lib.Oracle(cfg.policy, cfg.routing, cfg.workers)
    W = cfg.workers.n_workers
    half = cfg.jobs.n_jobs // 2
    jobs = [cfg.jobs.slice(0, half), cfg.jobs.slice(half, cfg.jobs.n_jobs - half)]
    a, b = (eng.batch(j.n_jobs) for j in jobs)
    a.encode(jobs[0]).dispatch()
    b.encode(jobs[1]).dispatch()                       # both resident, for the ticks
    rng = np.random.default_rng(11)
    epochs = []
    for _ in range(5):
        loads = cfg.workers.loads()
        loads["active_jobs"] = rng.integers(0, 9, W)
        loads["cpu_load"] = (rng.random(W) * 100).astype(np.float32)
        loads["gpu_utilization"] = (rng.random(W) * 100).astype(np.float32)
        epochs.append(loads)
    all_slots = np.arange(W, dtype=np.uint32)

    def delta(step):
        before = eng.launch_count()
        out = step()
        return eng.launch_count() - before, out

    def check(batch, got, loads, what):
        o.update_workers(all_slots, loads)
        assert_same(got, o.eval(jobs[batch]), what)

    # host loads: the first dispatch after cordum_workers_update refreshes from the host tables
    eng.update_workers(all_slots, epochs[0])
    d, got = delta(lambda: a.dispatch().copy())
    assert d == REFRESH + POLICY_AND_ROUTE, ("dispatch after update_workers", d)
    check(0, got, epochs[0], "update_workers")

    # cordum_workers_ingest refreshes as it is called; the dispatch after it finds the tables current
    d, _ = delta(lambda: eng.ingest(epochs[1].ctypes.data, 0, W))
    assert d == REFRESH, ("ingest", d)
    d, got = delta(lambda: a.dispatch().copy())
    assert d == POLICY_AND_ROUTE, ("dispatch after ingest", d)
    check(0, got, epochs[1], "ingest")

    # a device load table: refreshed as it is handed over
    import torch

    dev = torch.from_numpy(epochs[2].view(np.uint8).reshape(W, 16).copy()).cuda()
    torch.cuda.synchronize()

    def set_and_dispatch():
        eng.set_loads_device(dev.data_ptr(), W, torch.cuda.current_stream().cuda_stream)
        return a.dispatch().copy()

    d, got = delta(set_and_dispatch)
    assert d == REFRESH + POLICY_AND_ROUTE, ("set_loads_device + dispatch", d)
    check(0, got, epochs[2], "set_loads_device")

    # ticks: heartbeat epoch + policy of the new batch + route of the previous tick's batch
    d, _ = delta(lambda: a.tick(epochs[3].ctypes.data, 0, W))
    assert d == REFRESH + 1, ("first tick", d)
    d, _ = delta(lambda: b.tick(epochs[4].ctypes.data, 0, W))
    assert d == REFRESH + 2, ("second tick", d)
    a.wait()                                           # routed by the second tick
    check(0, a.fetch().copy(), epochs[3], "first tick")
    d, _ = delta(eng.tick_flush)
    assert d == 1, ("tick_flush", d)
    b.wait()
    check(1, b.fetch().copy(), epochs[4], "second tick")

    # a plain dispatch after ticks continues from the tables of the last tick
    d, got = delta(lambda: a.dispatch().copy())
    assert d == POLICY_AND_ROUTE, ("dispatch after ticks", d)
    check(0, got, epochs[4], "dispatch after ticks")
    a.free()
    b.free()
    o.close()
