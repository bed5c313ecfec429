"""CPU re-walk of the compiled tables, mirroring kernels.cu step for step.

TEST INFRASTRUCTURE.  The product evaluates jobs only on the GPU; this module lets the
CPU test-suite check the table compiler and the encoder (host C++ in
cordum_b200/csrc/host.cpp) against the oracle without a GPU: it loads the same library,
pulls the host-side tables and encoded columns out through the cordum_test_host_* hooks
and applies the kernel's algorithm (AND of pass-rows, first set bit, per-rule subset
tests, verdict tables, per-pool argmin) in plain Python/numpy.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from cordum_b200 import _lib, policy_io, wire

JF_COMBO_MASK, JF_MCP_USED, JF_HAS_LABELS, JF_APPROVED = 0x7, 0x8, 0x10, 0x20
JF_REQ_NONEMPTY, JF_REQ_UNKNOWN, JF_PLACE_UNSAT = 0x40, 0x80, 0x100
JF_TOPIC_MISSING, JF_TOPIC_UNSUPPORTED, JF_TOPIC_RAW_EMPTY = 0x200, 0x400, 0x800
PREF_UNKNOWN = 0xFFFFFFFF
KEY_NONE = (1 << 64) - 1
JOB_DTYPE = np.dtype([("topic", "<u4"), ("flags", "<u4"), ("orig", "<u4"), ("tenant", "<u2"), ("tenant_pol", "<u2"),
                      ("capability", "<u2"), ("pack", "<u2"), ("actor", "<u2"), ("effcfg", "<u2"), ("mcp", "<u2", (4,)),
                      ("risk_mask", "<u8"), ("req_mask", "<u8"), ("lab_mask", "<u8"), ("spare", "<u4", (2,))])
ROUTE_DTYPE = np.dtype([("place_lo", "<u8"), ("place_hi", "<u8"), ("req_pool", "<u8"), ("pref_pool", "<u4"), ("pref_worker", "<u4")])
assert JOB_DTYPE.itemsize == 64 and ROUTE_DTYPE.itemsize == 32
SUM_TENANT, SUM_CAP, SUM_PACK, SUM_ACTOR, SUM_COMBO, SUM_RISK = 1, 2, 4, 8, 16, 32
TABLES = {
    "row_tenant": np.uint32, "row_topic": np.uint32, "row_cap": np.uint32, "row_pack": np.uint32,
    "row_actor": np.uint32, "row_combo": np.uint32, "row_risk": np.uint32, "row_check": np.uint32,
    "row_mcp0": np.uint32, "row_mcp1": np.uint32, "row_mcp2": np.uint32, "row_mcp3": np.uint32,
    "pos2rule": np.uint32, "sum_tenant": np.uint64, "sum_topic": np.uint64, "sum_cap": np.uint64, "sum_pack": np.uint64,
    "sum_actor": np.uint64, "sum_combo": np.uint64, "sum_risk": np.uint64,
    "rule_req_need": np.uint64, "rule_lab_need": np.uint64, "rule_dec": np.uint8, "tenant_mcp": np.uint8,
    "eff_mcp": np.uint8, "eff_topic": np.uint8, "topic_pool_off": np.uint32, "topic_pool_cnt": np.uint32,
    "pool_list": np.uint32, "pool_req_mask": np.uint64, "pool_req_nonempty": np.uint8, "pool_off": np.uint32,
    "pos_pool": np.uint32, "pos_slot": np.uint32, "pos_rank": np.uint32, "slot_pos": np.uint32, "rank_slot": np.uint32,
    "pos_label_lo": np.uint64, "pos_label_hi": np.uint64, "loads": wire.LOAD_DTYPE,
    "chunk_pool": np.uint32, "pool_chunk0": np.uint32, "merge_list": np.uint32,
    "rule_need_x": np.uint64, "pool_req_x": np.uint64, "req_blank_x": np.uint64, "pos_label_x": np.uint64,
    "tenant_class": np.uint8,
}
SCALARS = ["n_rules", "n_seg", "sum_group", "sum_use", "n_chunks", "n_merge", "merge_smem", "row_words", "mcp_stride", "topic_stride", "n_effcfg", "req_blank_mask", "n_pools",
           "n_pos", "n_slots", "n_topics", "xw_risk", "xw_req", "xw_lab", "xw_place", "place_bits", "dict_resets", "tenant_classes"]


def _align16(x):
    return (x + 15) & ~15


def _orderable(score: np.float32) -> int:
    if score == 0:
        score = np.float32(0.0)
    b = int(np.float32(score).view(np.uint32))
    return (~b) & 0xFFFFFFFF if b & 0x80000000 else b | 0x80000000


class HostHarness:
    """Host (table compiler + encoder) without a GPU."""

    def __init__(self, policy=None, routing=None, workers=None, threads=2, max_topics=0, max_effcfgs=0):
        self.L = _lib.load()
        self.h = C.c_void_p(self.L.cordum_test_host_new(max_topics, max_effcfgs, threads))
        self.load_policy(policy)
        self.load_routing(routing)
        self.load_workers(workers or [])

    def close(self):
        if self.h:
            self.L.cordum_test_host_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _ck(self, rc):
        if rc:
            raise RuntimeError("host: %s" % self.L.cordum_test_last_error().decode())

    def load_policy(self, policy):
        doc = policy_io.to_json(policy)
        self._ck(self.L.cordum_test_host_policy(self.h, doc, len(doc)))

    def load_routing(self, routing):
        doc = policy_io.to_json(routing)
        self._ck(self.L.cordum_test_host_routing(self.h, doc, len(doc)))

    def load_workers(self, workers):
        wt = workers if isinstance(workers, wire.WorkerTable) else wire.WorkerTable.from_workers(workers)
        self._wt = wt
        self._ck(self.L.cordum_test_host_workers(self.h, C.addressof(wt.struct)))

    def update_workers(self, slots, loads):
        slots = np.ascontiguousarray(slots, dtype=np.uint32)
        loads = np.ascontiguousarray(loads, dtype=wire.LOAD_DTYPE)
        self._ck(self.L.cordum_test_host_update(self.h, len(slots), slots.ctypes.data, loads.ctypes.data))

    def encode(self, env) -> dict:
        """Encoded records as the batch holds them (topic-sorted), un-sorted into caller order for the walk; the
        sorted arrays are kept under "_job" / "_route" / "_slot_of" for tests of the order itself."""
        if not isinstance(env, wire.EnvelopeBatch):
            env = wire.EnvelopeBatch.from_jobs(env)
        n = env.n_jobs
        slab = np.zeros(int(self.L.cordum_test_slab_bytes(n)) + 64, dtype=np.uint8)
        base = (-slab.ctypes.data) % 16
        slab = slab[base:]
        ww = int(self.L.cordum_test_host_wide_words(self.h))
        wide = np.zeros(max(n * ww, 1), dtype=np.uint64)
        self._ck(self.L.cordum_test_host_encode(self.h, C.addressof(env.struct), slab.ctypes.data, wide.ctypes.data))
        assert int(self.L.cordum_test_host_wide_words(self.h)) == ww
        job = slab[: 64 * n].view(JOB_DTYPE).copy()
        route = slab[64 * n: 96 * n].view(ROUTE_DTYPE).copy()
        slot_of = slab[96 * n: 100 * n].view(np.uint32).copy()
        assert np.array_equal(job["orig"][slot_of], np.arange(n, dtype=np.uint32)), "slot_of / orig are not inverse"
        assert np.all(np.diff(job["topic"].astype(np.int64)) >= 0), "records are not sorted by topic id"
        # inside a topic the records are grouped by tenant class; the sort is stable, so two neighbours with the same
        # topic and the same tenant keep their batch order
        same = (np.diff(job["topic"].astype(np.int64)) == 0) & (np.diff(job["tenant"].astype(np.int64)) == 0)
        assert np.all(np.diff(job["orig"].astype(np.int64))[same] > 0), "the sort is not stable"
        j, r = job[slot_of], route[slot_of]
        cols = {k: j[k] for k in ("topic", "flags", "tenant", "tenant_pol", "capability", "pack", "actor", "effcfg",
                                  "risk_mask", "req_mask", "lab_mask")}
        for f in range(4):
            cols["mcp%d" % f] = j["mcp"][:, f]
        for k in ("place_lo", "place_hi", "req_pool", "pref_pool", "pref_worker"):
            cols[k] = r[k]
        cols["_job"], cols["_route"], cols["_slot_of"] = job, route, slot_of
        # wide masks (tables.h WideLayout): fold the extra words of each mask into one Python int per job
        xr, xq, xl, xp = (int(self.L.cordum_test_host_scalar(self.h, k)) for k in (b"xw_risk", b"xw_req", b"xw_lab", b"xw_place"))
        assert ww == xr + 2 * xq + xl + xp
        wrows = wide[: n * ww].reshape(n, ww)[slot_of] if ww else np.zeros((n, 0), np.uint64)
        cols["_wide"] = wrows

        def fold(base_cols, off, cnt):
            out = []
            for i in range(n):
                v, sh = 0, 0
                for c in base_cols:
                    v |= int(cols[c][i]) << sh
                    sh += 64
                for k in range(cnt):
                    v |= int(wrows[i, off + k]) << sh
                    sh += 64
                out.append(v)
            return out
        cols["risk_mask"] = fold(["risk_mask"], 0, xr)
        cols["req_mask"] = fold(["req_mask"], xr, xq)
        cols["lab_mask"] = fold(["lab_mask"], xr + xq, xl)
        cols["req_pool"] = fold(["req_pool"], xr + xq + xl, xq)
        cols["place"] = fold(["place_lo", "place_hi"], xr + 2 * xq + xl, xp)
        return cols

    def tables(self) -> dict:
        t = {}
        for name, dt in TABLES.items():
            ptr, nbytes = C.c_void_p(), C.c_uint64()
            self._ck(self.L.cordum_test_host_table(self.h, name.encode(), C.byref(ptr), C.byref(nbytes)))
            if nbytes.value == 0:
                t[name] = np.zeros(0, dtype=dt)
            else:
                buf = (C.c_uint8 * nbytes.value).from_address(ptr.value)
                t[name] = np.frombuffer(buf, dtype=dt).copy()
        for s in SCALARS:
            t[s] = int(self.L.cordum_test_host_scalar(self.h, s.encode()))
        # fold the wide words (tables.h WideLayout) into one Python int per rule / pool / worker
        xq, xl, xp = t["xw_req"], t["xw_lab"], t["xw_place"]

        def wide_int(arr, base, cnt):
            v = 0
            for k in range(cnt):
                v |= int(arr[base + k]) << (64 * k)
            return v
        nr = len(t["rule_req_need"])
        rx = t["rule_need_x"]
        t["rule_req_need"] = [int(t["rule_req_need"][r]) | (wide_int(rx, r * (xq + xl), xq) << 64 if (xq and (r + 1) * (xq + xl) <= len(rx)) else 0) for r in range(nr)]
        t["rule_lab_need"] = [int(t["rule_lab_need"][r]) | (wide_int(rx, r * (xq + xl) + xq, xl) << 64 if (xl and (r + 1) * (xq + xl) <= len(rx)) else 0) for r in range(nr)]
        t["pool_req_mask"] = [int(m) | (wide_int(t["pool_req_x"], p * xq, xq) << 64) for p, m in enumerate(t["pool_req_mask"])]
        t["req_blank_mask"] = int(t["req_blank_mask"]) | (wide_int(t["req_blank_x"], 0, xq) << 64)
        t["pos_label"] = [int(lo) | int(hi) << 64 | (wide_int(t["pos_label_x"], i * xp, xp) << 128)
                          for i, (lo, hi) in enumerate(zip(t["pos_label_lo"], t["pos_label_hi"]))]
        return t

    def evaluate(self, env, mode=wire.MODE_POLICY_AND_ROUTE) -> np.ndarray:
        cols = self.encode(env)      # encode first: it may register new topics / effective configs
        return walk(self.tables(), cols, mode)


def _worker_pools(T):
    """worker_pool_kernel: per-pos key, per-pool best and count at the minimum score."""
    n_pos, n_pools = T["n_pos"], T["n_pools"]
    key = [KEY_NONE] * max(n_pos, 1)
    for pos in range(n_pos):
        L = T["loads"][T["pos_slot"][pos]]
        active, maxp = np.float32(int(L["active_jobs"])), int(L["max_parallel_jobs"])
        cpu, gpu = np.float32(L["cpu_load"]), np.float32(L["gpu_utilization"])
        over = False
        if maxp > 0:
            over = np.float32(active / np.float32(maxp)) >= np.float32(0.9)
        over = over or cpu >= np.float32(90) or gpu >= np.float32(90)
        score = np.float32(np.float32(active + np.float32(cpu / np.float32(100))) + np.float32(gpu / np.float32(100)))
        key[pos] = KEY_NONE if over else (_orderable(score) << 32) | int(T["pos_rank"][pos])
    best, cnt = [KEY_NONE] * max(n_pools, 1), [0] * max(n_pools, 1)
    for p in range(n_pools):
        a, b = int(T["pool_off"][p]), int(T["pool_off"][p + 1])
        ks = key[a:b]
        if ks:
            best[p] = min(ks)
        if best[p] != KEY_NONE:
            cnt[p] = sum(1 for k in ks if k != KEY_NONE and (k >> 32) == (best[p] >> 32))
    return key, best, cnt


def _merge(key, cnt, k2, c2):
    if k2 == KEY_NONE:
        return key, cnt
    if key == KEY_NONE or (k2 >> 32) < (key >> 32):
        return k2, c2
    if (k2 >> 32) == (key >> 32):
        return min(key, k2), cnt + c2
    return key, cnt


def walk(T, cols, mode) -> np.ndarray:
    n = len(cols["flags"])
    out = np.zeros(n, dtype=wire.DECISION_DTYPE)
    out["rule_idx"] = -1
    out["worker_slot"] = -1
    W = T["row_words"]
    rows = {k: T[k].reshape(-1, W) if len(T[k]) else np.zeros((0, W), np.uint32)
            for k in ("row_tenant", "row_topic", "row_cap", "row_pack", "row_actor", "row_combo", "row_risk", "row_check",
                      "row_mcp0", "row_mcp1", "row_mcp2", "row_mcp3")}
    key, pool_best, pool_cnt = _worker_pools(T)
    stride = T["mcp_stride"]
    for j in range(n):
        flags = int(cols["flags"][j])
        topic = int(cols["topic"][j])
        mid = [int(cols["mcp%d" % f][j]) for f in range(4)]
        req_mask = int(cols["req_mask"][j])
        dec = sched = rflags = reason = route = 0
        rule, slot = -1, -1
        if mode != wire.MODE_ROUTE_ONLY:
            if mode == wire.MODE_POLICY_AND_ROUTE and flags & JF_APPROVED:
                dec = sched = wire.DEC_ALLOW
                reason, rflags = wire.REASON_APPROVAL_GRANTED, wire.F_APPROVED_BYPASS
            elif flags & JF_TOPIC_MISSING:
                dec = sched = wire.DEC_DENY
                reason = wire.REASON_MISSING_TOPIC
            elif flags & JF_TOPIC_UNSUPPORTED:
                dec = sched = wire.DEC_DENY
                reason = wire.REASON_UNSUPPORTED_TOPIC
            else:
                mcp_used, has_labels = bool(flags & JF_MCP_USED), bool(flags & JF_HAS_LABELS)
                acc = (rows["row_combo"][(flags & JF_COMBO_MASK) + ((flags >> 14) & 3) * 6] & rows["row_tenant"][cols["tenant"][j]]
                       & rows["row_topic"][topic] & rows["row_cap"][cols["capability"][j]]
                       & rows["row_pack"][cols["pack"][j]] & rows["row_actor"][cols["actor"][j]])
                risk = int(cols["risk_mask"][j])
                if risk == 0:
                    rk = rows["row_risk"][0]
                else:
                    rk = np.zeros(W, np.uint32)
                    for b in range(risk.bit_length()):
                        if risk >> b & 1:
                            rk = rk | rows["row_risk"][1 + b]
                acc = acc & rk
                if mcp_used:
                    for f in range(4):
                        acc = acc & rows["row_mcp%d" % f][mid[f]]
                chk = rows["row_check"][0]
                lab = int(cols["lab_mask"][j])
                # rule bits are permuted; the kernel ANDs the per-row summaries first and visits only the word groups
                # that survive (kernels.cu phase P): no surviving bit may lie outside them.  The first match is the
                # minimum ORIGINAL rule index over the surviving bits.
                G = int(T["sum_group"])
                use = int(T["sum_use"])
                live = int(T["sum_topic"][topic])
                if use & SUM_TENANT:
                    live &= int(T["sum_tenant"][cols["tenant"][j]])
                if use & SUM_CAP:
                    live &= int(T["sum_cap"][cols["capability"][j]])
                if use & SUM_PACK:
                    live &= int(T["sum_pack"][cols["pack"][j]])
                if use & SUM_ACTOR:
                    live &= int(T["sum_actor"][cols["actor"][j]])
                if use & SUM_COMBO:
                    live &= int(T["sum_combo"][(flags & JF_COMBO_MASK) + ((flags >> 14) & 3) * 6])
                if use & SUM_RISK:
                    rs = int(T["sum_risk"][0]) if risk == 0 else 0
                    for b in range(risk.bit_length()):
                        if risk >> b & 1:
                            rs |= int(T["sum_risk"][1 + b])
                    live &= rs
                n128 = W // 4
                listed = [w for w in range(n128) if live >> (w // G) & 1]
                outside = acc.copy()
                for wi in listed:
                    outside[4 * wi: 4 * wi + 4] = 0
                assert not outside.any(), "a surviving bit lies outside the live word groups"
                # the summaries themselves must be exact: a group is flagged iff the row has a bit there
                trow = rows["row_topic"][topic]
                for g in range((n128 + G - 1) // G):
                    assert bool(trow[4 * G * g: 4 * G * (g + 1)].any()) == bool(int(T["sum_topic"][topic]) >> g & 1)
                iw = 4
                best = 1 << 62
                for wi in listed:
                    # like the kernel: inside a word positions ascend with the rule index, so the first surviving bit
                    # that passes its subset test is the word's first match and the rest of the word is not looked at
                    word_best, prev = None, -1
                    for w in range(iw * wi, iw * wi + iw):
                        bits = int(acc[w])
                        while bits:
                            b = (bits & -bits).bit_length() - 1
                            bits &= bits - 1
                            pos = w * 32 + b
                            r = int(T["pos2rule"][pos])
                            assert r >= prev, "positions inside a word must ascend with the rule index"
                            prev = r
                            if int(chk[w]) >> b & 1:
                                need, ln = int(T["rule_req_need"][r]), int(T["rule_lab_need"][r])
                                if not ((need & ~req_mask) == 0 and (ln == 0 or (has_labels and (ln & ~lab) == 0))):
                                    continue
                            if word_best is None:
                                word_best = r
                    if word_best is not None:
                        best = min(best, word_best)
                first = best if best < (1 << 62) else -1
                rule = first
                code, hascons = wire.DEC_ALLOW, False
                if first >= 0:
                    rd = int(T["rule_dec"][first])
                    code, hascons = rd & 0x7F, bool(rd & 0x80)
                rule_approval = code == wire.DEC_REQUIRE_HUMAN
                tm = 0
                tpol = int(cols["tenant_pol"][j])
                if mcp_used and tpol:
                    base = (tpol - 1) * 4 * stride
                    for f in range(4):
                        v = int(T["tenant_mcp"][base + f * stride + mid[f]])
                        if v:
                            tm = 1 + f * 2 + (v - 1)
                            break
                    if tm:
                        code = wire.DEC_DENY
                dec = wire.DEC_ALLOW
                if code == wire.DEC_DENY:
                    dec, reason = wire.DEC_DENY, (wire.REASON_TENANT_MCP + tm - 1) if tm else wire.REASON_RULE
                elif code == wire.DEC_REQUIRE_HUMAN:
                    dec, reason = wire.DEC_REQUIRE_HUMAN, wire.REASON_RULE
                elif code == wire.DEC_THROTTLE:
                    dec, reason = wire.DEC_THROTTLE, wire.REASON_RULE
                elif code == wire.DEC_ALLOW_WITH_CONSTRAINTS or hascons:
                    dec = wire.DEC_ALLOW_WITH_CONSTRAINTS
                eff = int(cols["effcfg"][j])
                if eff:
                    tb = int(T["eff_topic"][eff * T["topic_stride"] + topic])
                    if tb & 1:
                        dec, reason = wire.DEC_DENY, wire.REASON_EFF_DENIED_TOPIC
                    if tb & 2:
                        dec, reason = wire.DEC_DENY, wire.REASON_EFF_NOT_ALLOWED_TOPIC
                    if mcp_used:
                        base = eff * 4 * stride
                        for f in range(4):
                            v = int(T["eff_mcp"][base + f * stride + mid[f]])
                            if v:
                                dec, reason = wire.DEC_DENY, wire.REASON_EFF_MCP + f * 2 + (v - 1)
                                break
                approval = rule_approval or dec == wire.DEC_REQUIRE_HUMAN
                rflags = wire.F_HAS_SNAPSHOT | (wire.F_APPROVAL_REQUIRED if approval else 0) | (wire.F_CONSTRAINTS if hascons else 0)
                sched = dec
                if approval and dec in (wire.DEC_ALLOW, wire.DEC_ALLOW_WITH_CONSTRAINTS):
                    sched = wire.DEC_REQUIRE_HUMAN
        do_route = mode == wire.MODE_ROUTE_ONLY or (mode == wire.MODE_POLICY_AND_ROUTE and sched in (wire.DEC_ALLOW, wire.DEC_ALLOW_WITH_CONSTRAINTS))
        if do_route:
            if flags & JF_TOPIC_RAW_EMPTY:
                route = wire.ROUTE_MISSING_TOPIC
            else:
                off, cnt = int(T["topic_pool_off"][topic]), int(T["topic_pool_cnt"][topic])
                pools = [int(p) for p in T["pool_list"][off:off + cnt]]
                ppool = int(cols["pref_pool"][j])
                if ppool:
                    if ppool == PREF_UNKNOWN or (ppool - 1) not in pools:
                        route = wire.ROUTE_NO_POOL_PREFERRED
                    else:
                        pools = [ppool - 1]
                if route == 0 and not pools:
                    route = wire.ROUTE_NO_POOL_TOPIC
                if route == 0:
                    req_any, req_unknown = bool(flags & JF_REQ_NONEMPTY), bool(flags & JF_REQ_UNKNOWN)
                    need_req = int(cols["req_pool"][j]) & ~T["req_blank_mask"]
                    need_pl = int(cols["place"][j])
                    unsat = bool(flags & JF_PLACE_UNSAT)
                    labelled = need_pl != 0 or unsat

                    def elig(p):
                        if not req_any:
                            return True
                        return bool(T["pool_req_nonempty"][p]) and not req_unknown and (need_req & ~int(T["pool_req_mask"][p])) == 0

                    el = [p for p in pools if elig(p)]
                    best, bcnt, total = KEY_NONE, 0, 0
                    if not labelled:
                        for p in el:
                            total += int(T["pool_off"][p + 1]) - int(T["pool_off"][p])
                            best, bcnt = _merge(best, bcnt, pool_best[p], pool_cnt[p])
                    elif not unsat:
                        for p in el:
                            for pos in range(int(T["pool_off"][p]), int(T["pool_off"][p + 1])):
                                if (T["pos_label"][pos] & need_pl) != need_pl:
                                    continue
                                total += 1
                                best, bcnt = _merge(best, bcnt, key[pos], 1)
                    if not el:
                        route = wire.ROUTE_NO_POOL_REQUIRES
                    else:
                        took = False
                        pw = int(cols["pref_worker"][j])
                        if pw and pw != PREF_UNKNOWN:
                            p1 = int(T["slot_pos"][pw - 1])
                            if p1 and int(T["pos_pool"][p1 - 1]) in el and not unsat:
                                pos = p1 - 1
                                lab_ok = (T["pos_label"][pos] & need_pl) == need_pl
                                if lab_ok and key[pos] != KEY_NONE:
                                    took, route, slot = True, wire.ROUTE_OK_PREFERRED, pw - 1
                        if not took:
                            if best != KEY_NONE:
                                route, slot = wire.ROUTE_OK, int(T["rank_slot"][best & 0xFFFFFFFF])
                                if bcnt > 1:
                                    rflags |= wire.F_TIE
                            else:
                                route = wire.ROUTE_POOL_OVERLOADED if total > 0 else wire.ROUTE_NO_WORKERS
        out[j] = (dec, sched, rflags, route, reason, (0, 0, 0), rule, slot)
    return out
