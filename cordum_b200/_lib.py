"""ctypes binding of libcordum_b200.so (include/cordum_b200.h).

The shared library is built in-tree by `__graft_entry__.build()` (cordum_b200/csrc/Makefile).
If it is missing this module raises — there is no Python or CPU fallback for the hot path.
"""
from __future__ import annotations

import ctypes as C
import os

from . import wire

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libcordum_b200.so")

# every symbol include/cordum_b200.h declares (the CPU test-suite checks they are all exported)
API = [
    "cordum_last_error", "cordum_version", "cordum_engine_create", "cordum_engine_destroy", "cordum_policy_load",
    "cordum_policy_snapshots", "cordum_policy_snapshot", "cordum_routing_load", "cordum_workers_load", "cordum_workers_update",
    "cordum_workers_set_loads_device", "cordum_exchange_unique_id", "cordum_exchange_init", "cordum_workers_ingest",
    "cordum_tick_async", "cordum_tick_flush", "cordum_tick_stream", "cordum_peer_export", "cordum_peer_import",
    "cordum_batch_alloc", "cordum_batch_free", "cordum_encode", "cordum_encode_device", "cordum_envelopes_alloc",
    "cordum_envelopes_free", "cordum_host_fallbacks", "cordum_batch_records", "cordum_dispatch",
    "cordum_dispatch_async", "cordum_batch_wait", "cordum_dispatch_resident", "cordum_dispatch_resident_async", "cordum_batch_fetch", "cordum_batch_stream",
    "cordum_batch_size", "cordum_batch_results", "cordum_batch_timing", "cordum_batch_kernel_times", "cordum_batch_plan", "cordum_batch_topic_counts", "cordum_batch_responses", "cordum_batch_subset", "cordum_batch_parent_index", "cordum_batch_merge", "cordum_rule_id", "cordum_reason", "cordum_reason_flavor", "cordum_batch_snapshot", "cordum_batch_policy_gen", "cordum_policy_generation", "cordum_frontend_cache_stats", "cordum_rule_id_at", "cordum_rule_constraints_json_at", "cordum_rule_remediations_json_at",
    "cordum_subject", "cordum_rule_constraints_json", "cordum_rule_remediations_json", "cordum_stats",
    "cordum_launch_count", "cordum_frontend_create", "cordum_frontend_destroy", "cordum_frontend_submit", "cordum_frontend_submit_many", "cordum_frontend_stats", "cordum_frontend_loadgen",
    "cordum_test_glob", "cordum_test_trim", "cordum_test_normalize_decision",
    "cordum_test_parse_effective", "cordum_test_canon",
]

_lib = None


def load() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            "cordum_b200: %s is missing — run `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a).  There is no CPU fallback." % LIB_PATH)
    L = C.CDLL(LIB_PATH)
    vp, u32, u64, i32, i64, cp = C.c_void_p, C.c_uint32, C.c_uint64, C.c_int32, C.c_int64, C.c_char_p
    L.cordum_last_error.restype = cp
    L.cordum_version.restype = cp
    L.cordum_engine_create.argtypes = [C.POINTER(wire.CordumEngineOpts), C.POINTER(vp)]
    L.cordum_engine_destroy.argtypes = [vp]
    L.cordum_engine_destroy.restype = None
    L.cordum_policy_load.argtypes = [vp, cp, u64, cp, u64]
    L.cordum_policy_snapshots.argtypes = [vp, cp, u64, C.POINTER(u32)]
    L.cordum_policy_snapshot.argtypes = [vp, cp, u64]
    L.cordum_policy_snapshot.restype = i64
    L.cordum_routing_load.argtypes = [vp, cp, u64]
    L.cordum_workers_load.argtypes = [vp, vp]
    L.cordum_workers_update.argtypes = [vp, u32, vp, vp]
    L.cordum_workers_set_loads_device.argtypes = [vp, vp, u32, vp]
    L.cordum_exchange_unique_id.argtypes = [vp]
    L.cordum_exchange_init.argtypes = [vp, vp, i32, i32]
    L.cordum_workers_ingest.argtypes = [vp, vp, u32, u32]
    L.cordum_tick_async.argtypes = [vp, vp, u32, vp, u32, u32]
    L.cordum_tick_flush.argtypes = [vp]
    L.cordum_tick_stream.argtypes = [vp]
    L.cordum_tick_stream.restype = vp
    L.cordum_peer_export.argtypes = [vp, i32, i32, vp]
    L.cordum_peer_import.argtypes = [vp, vp]
    L.cordum_batch_alloc.argtypes = [vp, u32, C.POINTER(vp)]
    L.cordum_batch_free.argtypes = [vp]
    L.cordum_batch_free.restype = None
    L.cordum_encode.argtypes = [vp, vp, vp]
    L.cordum_encode_device.argtypes = [vp, vp, vp]
    L.cordum_envelopes_alloc.argtypes = [vp, C.POINTER(wire.CordumEnvelopeCaps), C.POINTER(vp)]
    L.cordum_envelopes_free.argtypes = [vp, vp]
    L.cordum_envelopes_free.restype = None
    L.cordum_host_fallbacks.argtypes = [vp]
    L.cordum_host_fallbacks.restype = u64
    L.cordum_batch_records.argtypes = [vp, vp, vp, vp]
    for f in ("cordum_dispatch", "cordum_dispatch_async", "cordum_dispatch_resident", "cordum_dispatch_resident_async"):
        getattr(L, f).argtypes = [vp, vp, u32]
    L.cordum_batch_wait.argtypes = [vp]
    L.cordum_batch_fetch.argtypes = [vp]
    L.cordum_batch_stream.argtypes = [vp]
    L.cordum_batch_stream.restype = vp
    L.cordum_batch_size.argtypes = [vp]
    L.cordum_batch_size.restype = u32
    L.cordum_batch_results.argtypes = [vp]
    L.cordum_batch_results.restype = vp
    L.cordum_batch_timing.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.cordum_batch_kernel_times.argtypes = [vp, C.POINTER(C.c_float), C.POINTER(C.c_float)]
    L.cordum_batch_plan.argtypes = [vp, C.POINTER(wire.CordumPlan)]
    L.cordum_batch_topic_counts.argtypes = [vp, C.POINTER(wire.CordumTopicCounts)]
    L.cordum_batch_responses.argtypes = [vp, u32, C.POINTER(wire.CordumResponses)]
    L.cordum_batch_subset.argtypes = [vp, u32, vp, u32, vp, C.POINTER(u32)]
    L.cordum_batch_parent_index.argtypes = [vp, C.POINTER(u32)]
    L.cordum_batch_parent_index.restype = vp
    L.cordum_batch_merge.argtypes = [vp, vp, vp]
    L.cordum_rule_id.argtypes = [vp, i32, cp, u64]
    L.cordum_rule_id.restype = i64
    L.cordum_rule_constraints_json.argtypes = [vp, i32, cp, u64]
    L.cordum_rule_constraints_json.restype = i64
    L.cordum_rule_remediations_json.argtypes = [vp, i32, cp, u64]
    L.cordum_rule_remediations_json.restype = i64
    L.cordum_reason.argtypes = [vp, vp, u32, cp, u64]
    L.cordum_reason.restype = i64
    L.cordum_reason_flavor.argtypes = [vp, vp, u32, u32, vp, cp, u64]
    L.cordum_reason_flavor.restype = i64
    L.cordum_batch_snapshot.argtypes = [vp, cp, u64]
    L.cordum_batch_snapshot.restype = i64
    L.cordum_batch_policy_gen.argtypes = [vp]
    L.cordum_batch_policy_gen.restype = u64
    L.cordum_policy_generation.argtypes = [vp]
    L.cordum_policy_generation.restype = u64
    L.cordum_frontend_cache_stats.argtypes = [vp, vp, vp, vp]
    for fn in (L.cordum_rule_id_at, L.cordum_rule_constraints_json_at, L.cordum_rule_remediations_json_at):
        fn.argtypes = [vp, u64, i32, cp, u64]
        fn.restype = i64
    L.cordum_subject.argtypes = [vp, vp, u32, cp, u64]
    L.cordum_subject.restype = i64
    L.cordum_stats.argtypes = [vp, C.POINTER(wire.CordumTableStats)]
    L.cordum_frontend_create.argtypes = [vp, vp, C.POINTER(vp)]
    L.cordum_frontend_destroy.argtypes = [vp]
    L.cordum_frontend_destroy.restype = None
    L.cordum_frontend_submit.argtypes = [vp, vp, vp]
    L.cordum_frontend_submit_many.argtypes = [vp, vp, u32, vp]
    L.cordum_frontend_stats.argtypes = [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    L.cordum_frontend_loadgen.argtypes = [vp, vp, u32, u32, C.c_double, vp, u64]
    L.cordum_frontend_loadgen.restype = u64
    L.cordum_launch_count.argtypes = [vp]
    L.cordum_launch_count.restype = u64
    L.cordum_test_glob.argtypes = [cp, u64, cp, u64]
    L.cordum_test_trim.argtypes = [cp, u64, C.POINTER(u64), C.POINTER(u64)]
    L.cordum_test_normalize_decision.argtypes = [cp, u64]
    L.cordum_test_canon.argtypes = [i32, cp, u64, cp, u64]
    L.cordum_test_canon.restype = i64
    L.cordum_test_parse_effective.argtypes = [cp, u64, C.POINTER(u32), C.POINTER(u32)]
    L.cordum_test_batch_side.argtypes = [vp, i32, vp, u64]
    L.cordum_test_batch_side.restype = i64
    # host-only hooks (CPU tests of the table compiler / encoder)
    L.cordum_test_last_error.restype = cp
    L.cordum_test_host_new.argtypes = [u32, u32, u32]
    L.cordum_test_host_new.restype = vp
    L.cordum_test_host_free.argtypes = [vp]
    L.cordum_test_host_free.restype = None
    L.cordum_test_host_policy.argtypes = [vp, cp, u64]
    L.cordum_test_host_routing.argtypes = [vp, cp, u64]
    L.cordum_test_host_workers.argtypes = [vp, vp]
    L.cordum_test_host_update.argtypes = [vp, u32, vp, vp]
    L.cordum_test_slab_bytes.argtypes = [u32]
    L.cordum_test_slab_bytes.restype = u64
    L.cordum_test_host_encode.argtypes = [vp, vp, vp, vp]
    L.cordum_test_host_wide_words.argtypes = [vp]
    L.cordum_test_host_wide_words.restype = u32
    L.cordum_test_host_table.argtypes = [vp, cp, C.POINTER(vp), C.POINTER(u64)]
    L.cordum_test_json_canon.argtypes = [cp, u64, cp, u64]
    L.cordum_test_json_canon.restype = i64
    L.cordum_test_host_scalar.argtypes = [vp, cp]
    L.cordum_test_host_scalar.restype = u64
    _lib = L
    return L
