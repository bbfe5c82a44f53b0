"""Fault domains (gsim_domain_*) on the CPU: the kernels' row bodies (tests/hostemu) against the rules of
DESIGN.md §3.5 "Fault domains": the domain schedule function, the two-layer in-force rule, domain-wide
operations that equal the per-member calls over the same ids, snapshots, the read-only per-domain stats
against a numpy restatement, and validation."""
import ctypes as C
import os
import struct
import subprocess
import sys

import numpy as np
import pytest

from consul_b200 import _lib
from consul_b200.pool import (DOMAIN_MAX, FLAG_COORDINATES, FLAG_PROBE_PIGGYBACK, FLAG_PUSH_PULL, GsimError, Pool,
                              lan_config, wan_config)
from consul_b200.wan import c5_latency_matrix
import snapblob
from parity import compare_pools

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = _lib.load(os.path.join(ROOT, "tests", "hostemu", "libgsim_hostemu.so"))
ERR_INVALID, ERR_NOT_FOUND, ERR_STATE = -1, -5, -6
LAYOUT_DOM = 512
FULL = 1_000_000
PUR_FLAP, PUR_FLAP_DOMAIN = 12, 13
SCHEDULING = {"active_rows"}
LAYOUT_PIG, LAYOUT_FLAP = 128, 256
PIGK, PIG_BYTES = 4, 16 * 4 + 4 * 4 + 4 * 32 * 8  # GS_PIGK, sizeof(GsPig)


def layout(blob):
    return struct.unpack_from("<I", blob, 36)[0]


def split_dom(blob):
    """(the blob without the domain column, the schedule table and layout bit 512; the column; the table), the
    first part being what the same pool without domains writes.  Walks the blob forward from its header: the
    planes of tests/snapblob.py, the flap schedule column (bit 256) and the domain column (bit 512) before the
    pool-wide words, then the table (its length, then its words)."""
    blob = bytes(blob)
    lay = layout(blob)
    if not lay & LAYOUT_DOM:
        return blob, None, None
    cap = struct.unpack_from("<I", blob, 12)[0]
    g = snapblob.GsGlobals.from_buffer_copy(blob, snapblob._HEAD.size)
    n_sched = struct.unpack_from("<I", blob, 20)[0]
    r = snapblob.SNAP_HEADER_SIZE + snapblob.SCHED_SIZE * n_sched
    for _ in range(snapblob.MAX_RUMORS):
        nl, pl, _co = struct.unpack_from("<III", blob, r)
        r += 12 + nl + pl
    cols = snapblob.columns(lay & ~(LAYOUT_PIG | LAYOUT_FLAP | LAYOUT_DOM), g.ring_mask + 1)
    if lay & LAYOUT_PIG:  # owed answers and the piggyback words, after the push-pull columns
        at = next(x for x, c in enumerate(cols) if c[0] in ("imp_loss", "imp_recv", "pause_until", "stats"))
        cols = cols[:at] + [("pig_req", np.uint32, 2 * PIGK, True, True), ("pig", None, 1, False, False)] + cols[at:]
    at = next(x for x, c in enumerate(cols) if c[0] == "stats")
    extra = ([("imp_flap", np.uint32, 1, True, True)] if lay & LAYOUT_FLAP else []) + \
        [("imp_dom", np.uint32, 1, True, True)]
    cols = cols[:at] + extra + cols[at:]
    col, cut = None, None
    for name, dtype, nplanes, per_member, _fill in cols:
        pb = PIG_BYTES if name == "pig" else snapblob._plane_bytes(name, dtype, per_member, cap)
        for _ in range(nplanes):
            (tag,) = struct.unpack_from("<I", blob, r)
            size = 8 if tag == 1 else 4 + pb
            if name == "imp_dom":
                cut = (r, r + size)
                col = (np.full(cap, struct.unpack_from("<I", blob, r + 4)[0], np.uint32) if tag == 1 else
                       np.frombuffer(blob[r + 4:r + 4 + pb], np.uint32).copy())
            r += size
    (n_tab,) = struct.unpack_from("<I", blob, r)
    tab = np.frombuffer(blob[r + 4:r + 4 + 4 * n_tab], np.uint32).copy()
    assert r + 4 + 4 * n_tab == len(blob), "bytes left over after the domain schedule table"
    rest = blob[:cut[0]] + blob[cut[1]:r]
    return rest[:36] + struct.pack("<I", lay & ~LAYOUT_DOM) + rest[40:], col, tab


# ---- 1. the schedule function ------------------------------------------------------------------------------
def philox(seed, c0, c1, c2, c3):
    ctr, key, out = (C.c_uint32 * 4)(c0, c1, c2, c3), (C.c_uint32 * 2)(seed & 0xFFFFFFFF, seed >> 32), (C.c_uint32 * 4)()
    L.gsim_philox4x32(ctr, key, out)
    return list(out)


def domain_bad_py(seed, d, period, ppm, t):
    if period == 0 or ppm >= FULL:
        return 1
    if ppm == 0:
        return 0
    phase = philox(seed, d, 0xFFFFFFFF, PUR_FLAP_DOMAIN, 0)[1] % period
    return int(philox(seed, d, ((t + phase) // period) & 0xFFFFFFFF, PUR_FLAP_DOMAIN, 0)[0] < (ppm << 32) // FULL)


def test_domain_schedule_function_known_answers():
    for seed in (0, 0x5EED, 0xDEADBEEF12345678):
        for period in (1, 7, 4095):
            for d in (1, 129, DOMAIN_MAX):
                ticks = list(range(0, 3 * period + 2, max(1, period // 3))) + [2**32 - 1, 2**32 - period]
                for ppm in (1, 500_000, 999_999):
                    for t in ticks[::2]:
                        assert L.gsim_domain_flap_bad(seed, d, period, ppm, t) == domain_bad_py(seed, d, period, ppm, t)
                assert all(L.gsim_domain_flap_bad(seed, d, period, 0, t) == 0 for t in ticks)
                assert all(L.gsim_domain_flap_bad(seed, d, period, FULL, t) == 1 for t in ticks)
                assert L.gsim_domain_flap_bad(seed, d, 0, 0, 5) == 1          # no schedule: always in force
    for bad in ((0, 7, 10), (DOMAIN_MAX + 1, 7, 10), (1, 4096, 10), (1, 7, FULL + 1)):
        assert L.gsim_domain_flap_bad(1, bad[0], bad[1], bad[2], 5) == ERR_INVALID


def test_domain_phases_are_uniform_and_not_the_member_draw():
    seed, period = 0xD0D0, 50
    phases = np.array([philox(seed, d, 0xFFFFFFFF, PUR_FLAP_DOMAIN, 0)[1] % period for d in range(1, 5001)])
    counts = np.bincount(phases, minlength=period)
    chi2 = float(((counts - 100.0) ** 2 / 100.0).sum())
    assert chi2 < 100.0, chi2                                            # 49 degrees of freedom
    # the domain draw is its own: with the member draw's id and parameters it differs somewhere
    differs = 0
    for x in range(1, 60):
        a = [L.gsim_domain_flap_bad(seed, x, 13, 400_000, t) for t in range(0, 130, 13)]
        b = [L.gsim_flap_bad(seed, x, 13, 400_000, t) for t in range(0, 130, 13)]
        differs += a != b
    assert differs > 40


# ---- 2. equivalences -------------------------------------------------------------------------------------
def _kind(kind):
    """(config, latency matrix, impair(pool) -> ids)"""
    if kind == "lan":
        def imp(p):
            ids = list(range(0, 1500, 17))
            p.impair(ids, 300_000, 1)
            return ids
        return lan_config(L, capacity=1501, n_initial=1500, seed=0xD0A1, mailbox_depth=4), None, imp
    if kind == "one_way_no_tcp":
        def imp(p):
            a, b = list(range(3, 1200, 29)), list(range(11, 1200, 41))
            p.impair_dir(a, 0, FULL, 0, True)
            p.impair_dir(b, 600_000, 0, 0, True)
            return a + b
        return lan_config(L, capacity=1200, n_initial=1200, seed=0xD0A2, disable_tcp_pings=0), None, imp
    if kind == "wan_c5":
        def imp(p):
            p.impair_fraction(40_000, 5, 200_000, 2)
            return [i for i in range(2048) if p.impairment(i) != (0, 0)]
        return (wan_config(L, capacity=2048, n_initial=2048, seed=0xD0A3, mailbox_depth=8), c5_latency_matrix(16),
                imp)
    if kind == "push_pull":
        def imp(p):
            ids = list(range(1, 1024, 11))
            p.impair_dir(ids, 300_000, 300_000, 0, True)
            return ids
        return (lan_config(L, capacity=1024, n_initial=1024, seed=0xD0A6, flags=FLAG_PUSH_PULL,
                           push_pull_interval_ns=10**9, mailbox_depth=4), None, imp)
    if kind == "piggyback":
        def imp(p):
            ids = list(range(5, 1000, 13))
            p.impair(ids, 400_000, 1)
            return ids
        return (lan_config(L, capacity=1000, n_initial=1000, seed=0xD0A4, flags=FLAG_PROBE_PIGGYBACK,
                           mailbox_depth=4), None, imp)
    def imp(p):
        ids = list(range(2, 800, 9))
        p.impair(ids, 250_000, 2)
        return ids
    return lan_config(L, capacity=800, n_initial=800, seed=0xD0A5, flags=FLAG_COORDINATES, mailbox_depth=4), None, imp


KINDS = ["lan", "one_way_no_tcp", "wan_c5", "push_pull", "piggyback", "coordinates"]


def _pair(kind, lib):
    cfg, lat, imp = _kind(kind)
    a, b = Pool(cfg, lib), Pool(cfg, lib)
    for p in (a, b):
        if lat is not None:
            p.latency_set(lat)
    return cfg, a, b, imp


@pytest.mark.parametrize("kind", KINDS)
def test_domains_without_schedules_change_nothing(hostemu_lib, kind):
    cfg, a, b, imp = _pair(kind, hostemu_lib)
    for p in (a, b):
        imp(p)
        p.user_event(1, b"e", b"v", False)
    a.domain_set_range(0, a.stats()["n_members"], 32, 1)
    a.domain_set([1, 2, 3], 7000)
    a.domain_flap([9999], 0, 0)                                        # clearing: the table stays empty
    for k in [1, 2, 5, 13, 40, 100]:
        for p in (a, b):
            p.step(k)
        compare_pools(a, b, f"{kind} tick {a.now}")
        blob, col, tab = split_dom(a.snapshot())
        assert col is not None and int(col[40]) == 2 and int(col[2]) == 7000 and len(tab) == 0
        assert blob == b.snapshot(), f"{kind} tick {a.now}: blobs differ"


@pytest.mark.parametrize("kind", KINDS)
def test_always_bad_domains_are_the_static_impairment(hostemu_lib, kind):
    cfg, a, b, imp = _pair(kind, hostemu_lib)
    for p in (a, b):
        imp(p)
        p.user_event(1, b"e", b"v", False)
    a.domain_set_range(0, a.stats()["n_members"], 16, 3)
    doms = sorted(set(a.domains().tolist()))
    a.domain_flap(doms, 7, FULL)
    assert a.domain_flap_get(doms[0]) == (7, FULL) and a.domain_flap_get(DOMAIN_MAX) == (0, 0)
    for k in [1, 1, 2, 3, 5, 8, 13, 21, 40, 100]:
        for p in (a, b):
            p.step(k)
        compare_pools(a, b, f"{kind} tick {a.now}")
        blob, col, tab = split_dom(a.snapshot())
        assert len(tab) == doms[-1] + 1 and int(tab[doms[0]]) == 7 << 20 | FULL
        assert blob == b.snapshot(), f"{kind} tick {a.now}: blobs differ"


@pytest.mark.parametrize("kind", ["lan", "one_way_no_tcp", "wan_c5", "push_pull"])
def test_never_bad_domains_are_no_impairment(hostemu_lib, kind):
    cfg, a, b, imp = _pair(kind, hostemu_lib)
    for p in (a, b):
        p.user_event(1, b"e", b"v", False)
    imp(a)
    a.domain_set_range(0, a.stats()["n_members"], 32, 1)
    a.domain_flap(sorted(set(a.domains().tolist())), 50, 0)
    for k in [1, 2, 5, 20, 60, 150]:
        for p in (a, b):
            p.step(k)
        assert a.state_hash() == b.state_hash(), f"{kind} tick {a.now}"
        sa, sb = a.stats(), b.stats()
        for f in SCHEDULING:
            sa.pop(f), sb.pop(f)
        assert sa == sb, f"{kind} tick {a.now}"


# ---- 3. correlation: the two-layer rule ----------------------------------------------------------------
def restate(p, seed, now):
    """Per-domain stats over the pool's columns (numpy), and the per-member in-force bits."""
    n = p.stats()["n_members"]
    key, meta = p.column("key")[:n], p.column("meta")[:n]
    dom = p.domains()
    truth, rank, aw = key & 3, (key >> 2) & 3, meta & 7
    imp = np.array([any(v != 0 for v in p.impairment_dir(i)) for i in range(n)])
    paused = np.array([p.paused_until(i) != 0xFFFFFFFF for i in range(n)])
    own = np.array([L.gsim_flap_bad(seed, i, *p.impair_flap_get(i), now) for i in range(n)], bool)
    dsched = {d: p.domain_flap_get(int(d)) for d in set(dom.tolist()) if d}
    dbad = np.array([1 if d == 0 else L.gsim_domain_flap_bad(seed, int(d), *dsched[int(d)], now) for d in dom], bool)
    force = imp & own & dbad
    return dict(n=n, truth=truth, rank=rank, aw=aw, dom=dom, imp=imp, paused=paused, force=force)


def expected_stats(r, first, count):
    out = np.zeros((count, 11), np.uint64)
    for i in range(r["n"]):
        x = int(r["dom"][i]) - first
        if not 0 <= x < count or r["truth"][i] == 0:
            continue
        run = r["truth"][i] == 1
        row = out[x]
        row[0] += 1
        row[1] += run
        row[2] += r["paused"][i]
        row[3] += r["imp"][i]
        row[4] += r["force"][i]
        row[5 + int(r["rank"][i])] += 1
        if run:
            row[9] = max(row[9], r["aw"][i])
            row[10] += r["aw"][i]
    return out


def stats_rows(s):
    return np.stack([s[f].astype(np.uint64) for f in ("members", "running", "paused", "impaired", "in_force", "alive",
                                                      "suspect", "dead", "left", "awareness_max",
                                                      "awareness_sum")], axis=1)


def test_domain_bursts_hit_whole_racks_and_compose_with_member_schedules(hostemu_lib):
    seed = 0xD0C1
    cfg = lan_config(L, capacity=2048, n_initial=2048, seed=seed, disable_tcp_pings=1, mailbox_depth=4)
    p = Pool(cfg, hostemu_lib)
    p.domain_set_range(0, 2048, 32, 1)                                  # 64 racks
    racks = list(range(1, 65, 3))
    assert p.domain_impair(racks, 500_000, 500_000) == 32 * len(racks)
    p.domain_flap(racks, 10, 300_000)
    p.user_event(1, b"e", b"v", False)
    seen = set()
    for _ in range(12):
        p.step(7)
        s = p.domain_stats(1, 64)
        for d in racks:
            assert s["in_force"][d - 1] in (0, s["impaired"][d - 1]), (p.now, d)
            seen.add(int(s["in_force"][d - 1]))
        assert (stats_rows(s) == expected_stats(restate(p, seed, p.now), 1, 64)).all()
    assert seen == {0, 32}
    # member schedules as well: the AND of both layers
    p.impair_flap(list(range(0, 2048, 5)), 3, 500_000)
    for _ in range(8):
        p.step(5)
        r = restate(p, seed, p.now)
        s = p.domain_stats(1, 64)
        assert (stats_rows(s) == expected_stats(r, 1, 64)).all(), p.now
    assert p.stats()["packets_lost"] > 0


# ---- 4. domain operations equal the per-member calls -----------------------------------------------------
def _ops_pair(lib, seed):
    cfg = lan_config(L, capacity=3000, n_initial=3000, seed=seed, disable_tcp_pings=1, mailbox_depth=4)
    a, b = Pool(cfg, lib), Pool(cfg, lib)
    for p in (a, b):
        p.domain_set_range(0, 3000, 40, 1)
        p.domain_set(list(range(7, 3000, 101)), 900)
        p.user_event(1, b"e", b"v", False)
        p.step(5)
    return a, b


def _ids(p, doms):
    d = p.domains()
    return [int(i) for i in np.nonzero(np.isin(d, doms))[0]]


def test_domain_crash_is_crash_many(hostemu_lib):
    a, b = _ops_pair(hostemu_lib, 0xD0E1)
    doms = [2, 5, 900, 61]
    pz = [i for i in _ids(a, doms)][:6] + [3]
    for p in (a, b):
        assert p.pause(pz, 50) == len(pz)                              # paused members: the crash is for good
        p.step(3)
    assert a.domain_crash(doms) == len([i for i in _ids(a, doms) if i not in pz])
    b.crash_many(_ids(b, doms))
    assert a.pause_stats() == b.pause_stats() and a.pause_stats()["paused"] == 1
    for k in (1, 10, 60, 100):
        for p in (a, b):
            p.step(k)
        compare_pools(a, b, f"crash tick {a.now}")
        assert split_dom(a.snapshot())[0] == split_dom(b.snapshot())[0]
    assert a.domain_crash([3000]) == 0


def test_domain_pause_is_pause_many(hostemu_lib):
    a, b = _ops_pair(hostemu_lib, 0xD0E2)
    doms = [1, 9, 900]
    a.crash(_ids(a, doms)[4])
    b.crash(_ids(b, doms)[4])
    k = a.domain_pause(doms, 25)
    assert k == b.pause(_ids(b, doms), 25) == len(_ids(a, doms)) - 1
    for t in (1, 10, 20, 50):
        for p in (a, b):
            p.step(t)
        compare_pools(a, b, f"pause tick {a.now}")
        assert a.pause_stats() == b.pause_stats()
        assert split_dom(a.snapshot())[0] == split_dom(b.snapshot())[0]


@pytest.mark.parametrize("args", [(300_000, 300_000, 1, 0), (0, FULL, 0, 1), (600_000, 0, 2, 1)])
def test_domain_impair_is_impair_dir_many(hostemu_lib, args):
    a, b = _ops_pair(hostemu_lib, 0xD0E3)
    doms = [3, 4, 900, 70]
    send, recv, delay, no_tcp = args
    assert a.domain_impair(doms, send, recv, delay, no_tcp) == len(_ids(a, doms))
    b.impair_dir(_ids(b, doms), send, recv, delay, bool(no_tcp))
    for t in (1, 10, 60, 100):
        for p in (a, b):
            p.step(t)
        compare_pools(a, b, f"impair tick {a.now}")
        assert split_dom(a.snapshot())[0] == split_dom(b.snapshot())[0]
    # clearing again: the n_impaired bookkeeping and with it the fast-path gate follow
    a.domain_impair(doms, 0, 0, 0, 0)
    b.impair_dir(_ids(b, doms), 0, 0, 0, False)
    for p in (a, b):
        p.step(200)
    compare_pools(a, b, "cleared")
    assert split_dom(a.snapshot())[0] == split_dom(b.snapshot())[0]
    assert a.stats()["active_rows"] == b.stats()["active_rows"]


# ---- 5. snapshots -----------------------------------------------------------------------------------------
def test_snapshot_mid_flap_restores_into_a_fresh_pool(hostemu_lib):
    cfg = lan_config(L, capacity=1500, n_initial=1500, seed=0xD0F1, disable_tcp_pings=1, mailbox_depth=4)
    a = Pool(cfg, hostemu_lib)
    a.domain_set_range(0, 1500, 25, 1)
    a.domain_impair(list(range(1, 61, 4)), 500_000, 500_000, 1)
    a.domain_flap(list(range(1, 61, 2)), 37, 400_000)
    a.impair_flap(list(range(0, 1500, 11)), 5, 600_000)
    a.step(55)
    blob = a.snapshot()
    assert layout(blob) & LAYOUT_DOM
    fresh = Pool(cfg, hostemu_lib)
    fresh.restore(blob)
    assert fresh.snapshot() == blob
    assert (fresh.domains() == a.domains()).all() and fresh.domain_flap_get(59) == (37, 400_000)
    assert (stats_rows(fresh.domain_stats(1, 60)) == stats_rows(a.domain_stats(1, 60))).all()
    for _ in range(6):
        for p in (a, fresh):
            p.step(20)
        compare_pools(a, fresh, f"restored tick {a.now}")
    # a blob without domains clears the column and every domain schedule
    plain = Pool(cfg, hostemu_lib)
    fresh.restore(plain.snapshot())
    assert not fresh.domains().any() and fresh.domain_flap_get(59) == (0, 0)
    blob2, col, tab = split_dom(fresh.snapshot())
    assert not col.any() and len(tab) == 0 and fresh.state_hash() == plain.state_hash()


def test_a_pool_without_domains_writes_the_blob_it_always_did(hostemu_lib):
    cfg = lan_config(L, capacity=900, n_initial=900, seed=0xD0F2)
    a, b = Pool(cfg, hostemu_lib), Pool(cfg, hostemu_lib)
    for p in (a, b):
        p.impair(list(range(0, 900, 7)), 200_000, 0)
        p.step(30)
    assert a.domain_crash([1, 2]) == 0 and a.domain_impair([1], 5, 5) == 0 and a.domain_pause([1], 4) == 0
    assert not a.domains().any() and not a.domain_stats(1, 4)["members"].any()
    assert a.snapshot() == b.snapshot() and not layout(a.snapshot()) & LAYOUT_DOM


# ---- 6. the stats are read-only ---------------------------------------------------------------------------
def test_domain_stats_restatement_and_read_only(hostemu_lib):
    seed = 0xD0B1
    cfg = lan_config(L, capacity=3000, n_initial=2900, seed=seed, disable_tcp_pings=1, mailbox_depth=4)
    p = Pool(cfg, hostemu_lib)
    p.domain_set_range(0, 2900, 30, 5)
    p.domain_set(list(range(0, 2900, 37)), 2)
    p.domain_impair([6, 9, 2], 400_000, 400_000, 1)
    p.domain_flap([6, 2], 9, 500_000)
    p.domain_pause([11], 30)
    p.domain_crash([13, 14])
    p.user_event(1, b"e", b"v", False)
    for t in (3, 20, 40):
        p.step(t)
        h, s, blob, fs = p.state_hash(), p.stats(), p.snapshot(), p.flap_stats()
        got = p.domain_stats(1, 120)
        assert (stats_rows(got) == expected_stats(restate(p, seed, p.now), 1, 120)).all(), p.now
        assert got["members"].sum() == 2900 and got["dead"].sum() + got["suspect"].sum() > 0 or t < 40
        assert p.state_hash() == h and p.stats() == s and p.snapshot() == blob and p.flap_stats() == fs


# ---- 7. validation ---------------------------------------------------------------------------------------
def test_validation(hostemu_lib):
    p = Pool(lan_config(hostemu_lib, capacity=100, n_initial=64, seed=0xD0F3), hostemu_lib)
    invalid = (lambda: p.domain_set([1], DOMAIN_MAX + 1), lambda: p.domain_set_range(0, 10, 0, 1),
               lambda: p.domain_set_range(0, 10, 1, 0), lambda: p.domain_set_range(0, 10, 1, DOMAIN_MAX - 8),
               lambda: p.domain_flap([0], 5, 10), lambda: p.domain_flap([DOMAIN_MAX + 1], 5, 10),
               lambda: p.domain_flap([1], 4096, 10), lambda: p.domain_flap([1], 5, FULL + 1),
               lambda: p.domain_flap_get(0), lambda: p.domain_impair([0], 1, 1),
               lambda: p.domain_impair([1], FULL + 1, 0), lambda: p.domain_impair([1], 0, 0, 0, 2),
               lambda: p.domain_impair([1], 0, 0, 255), lambda: p.domain_crash([DOMAIN_MAX + 1]),
               lambda: p.domain_pause([1], 0), lambda: p.domain_pause([0], 5),
               lambda: p.domain_stats(0, 1), lambda: p.domain_stats(DOMAIN_MAX, 2))
    for fn in invalid:
        with pytest.raises(GsimError) as e:
            fn()
        assert e.value.code == ERR_INVALID
    for fn in (lambda: p.domain_set([64], 1), lambda: p.domain_set_range(60, 5, 1, 1), lambda: p.domains(60, 5)):
        with pytest.raises(GsimError) as e:
            fn()
        assert e.value.code == ERR_NOT_FOUND
    p.domain_set_range(0, 9, 1, DOMAIN_MAX - 8)                          # exactly up to the maximum
    assert int(p.domains(8, 1)[0]) == DOMAIN_MAX
    assert p.domain_stats(DOMAIN_MAX, 1)["members"][0] == 1
    p.domain_flap([DOMAIN_MAX], 4095, FULL)
    assert p.domain_flap_get(DOMAIN_MAX) == (4095, FULL)
    p.domain_flap([DOMAIN_MAX], 0, 123)
    assert p.domain_flap_get(DOMAIN_MAX) == (0, 0)


def test_sharded_pools_refuse():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29571",
           os.path.join(ROOT, "tests", "sharded_domain_worker_cpu.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "DOMAINS REFUSED" in r.stdout


# ---- 8. lockstep with the domain oracle (tests/oracle_domain/domain.patch) ------------------------------------
from test_flap_cpu import FlapLockstep  # noqa: E402
import fuzz_ops  # noqa: E402
import scenarios as sc  # noqa: E402
from oracle_domain import DomainOraclePool  # noqa: E402


class DomainLockstep(FlapLockstep):
    """A Lockstep pair whose pools also take fault-domain operations drawn for (seed, tick): assignments by list
    and by range, domain schedules, and domain-wide impairment, crashes and pauses, plus the per-domain stats.
    Both must return the same results."""

    DOMAIN = 0xD0F0

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.domain_record = {}

    def step(self, side, k):
        p = side.pool
        now, n = p.now, p.stats()["n_members"]
        rng = self._rng(self.DOMAIN, now)
        res = []
        room = max(0, self.depth - 2 - self.extra_latency)

        def doms():
            return [rng.choice([0, 1, 2, 3, 5, 8, 13, 40]) if rng.random() < 0.05 else rng.randint(1, 14)
                    for _ in range(rng.randint(1, 4))]

        def do(what, fn):
            try:
                res.append((what, fn()))
            except GsimError as e:
                res.append((what, e.code))

        if n and rng.random() < 0.6:
            x = rng.random()
            if x < 0.15:
                do("range", lambda: p.domain_set_range(0, n, rng.choice([4, 16, 50]), rng.randint(1, 3)))
            elif x < 0.3:
                do("set", lambda: p.domain_set([rng.randrange(n) for _ in range(rng.randint(1, 20))], rng.randint(0, 12)))
            elif x < 0.55:
                do("flap", lambda: p.domain_flap(doms(), rng.choice([0, 1, 3, 7, 50]),
                                                 rng.choice([0, 200_000, 600_000, FULL])))
            elif x < 0.8:
                do("impair", lambda: p.domain_impair(doms(), rng.choice([0, 300_000, FULL]),
                                                     rng.choice([0, 400_000]), rng.randint(0, min(room, 1)),
                                                     rng.choice([0, 0, 1])))
            elif x < 0.9:
                do("pause", lambda: p.domain_pause(doms(), rng.choice([0, 3, 20])))
            else:
                do("crash", lambda: p.domain_crash(doms()))
            do("stats", lambda: p.domain_stats(1, 16).tolist())
        if side.index == 0:
            self.domain_record[now] = res
        else:
            assert self.domain_record.get(now) == res, \
                f"seed {self.seed} tick {now}: {self.domain_record.get(now)} vs {res}"
        super().step(side, k)


@pytest.mark.parametrize("seed", range(6))
def test_fuzz_against_the_domain_oracle(hostemu_lib, seed):
    pair = DomainLockstep(lambda c: Pool(c, hostemu_lib), lambda c: DomainOraclePool(c), 0xD1B0 + seed, extra=True)
    assert fuzz_ops.run_sequence(pair.make, hostemu_lib, 0xD1B1000 + seed, n_ops=40) == 40


@pytest.mark.parametrize("kind", ["lan", "wan_c5"])
def test_domain_and_member_schedules_against_the_oracle(hostemu_lib, kind):
    """Racks whose loss, delay and NO_TCP flap on domain schedules, some members flapping on their own as well,
    the TCP fallback off on LAN: suspicions happen, and the kernels' row step and the oracle agree."""
    if kind == "lan":
        cfg, lat, n = lan_config(L, capacity=2049, n_initial=2048, seed=0xD1C1, disable_tcp_pings=1,
                                 mailbox_depth=4), None, 2048
    else:
        cfg, lat, n = wan_config(L, capacity=2049, n_initial=2048, seed=0xD1C2, mailbox_depth=8), c5_latency_matrix(16), 2048
    pools = [Pool(cfg, hostemu_lib), DomainOraclePool(cfg)]
    for p in pools:
        if lat is not None:
            p.latency_set(lat)
    sc.both(pools, lambda p: p.domain_set_range(0, n, 32, 1))
    sc.both(pools, lambda p: p.domain_impair(list(range(1, 65, 3)), 500_000, 400_000, 1, 1))
    sc.both(pools, lambda p: p.domain_flap(list(range(1, 65, 3)), 10, 300_000))
    sc.both(pools, lambda p: p.domain_flap(list(range(4, 65, 9)), 3, FULL))
    sc.both(pools, lambda p: p.impair_flap(list(range(0, n, 7)), 5, 500_000))
    sc.both(pools, lambda p: p.user_event(7, b"e", b"x", False))
    for _ in range(8):
        sc.step_compare(pools, 50, 25, f"{kind} domains")
        assert (stats_rows(pools[0].domain_stats(1, 64)) == stats_rows(pools[1].domain_stats(1, 64))).all()
    s = pools[0].stats()
    assert s["packets_lost"] > 0 and (kind != "lan" or s["suspects"] > 0), s
    x = sc.both(pools, lambda p: p.member_add())
    assert sc.both(pools, lambda p: p.join(x, list(range(0, n, 50)))) > 0
    sc.both(pools, lambda p: p.domain_crash([5, 6]))
    sc.both(pools, lambda p: p.domain_pause([7], 15))
    sc.step_compare(pools, 100, 20, f"{kind} after a join, a crash and a pause")


@pytest.mark.parametrize("order", ["1", "2"])
def test_row_order_does_not_matter(order):
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "from consul_b200 import _lib\n"
        "from consul_b200.pool import Pool, lan_config, FLAG_PUSH_PULL\n"
        "L = _lib.load(%r)\n"
        "p = Pool(lan_config(L, capacity=2049, n_initial=2048, seed=43, flags=FLAG_PUSH_PULL, "
        "push_pull_interval_ns=10**9, mailbox_depth=4, disable_tcp_pings=1), L)\n"
        "p.domain_set_range(0, 2048, 32, 1); p.domain_impair(list(range(1, 65, 4)), 600000, 600000, 1, 1)\n"
        "p.domain_flap(list(range(1, 65, 2)), 9, 400000); p.impair_flap(list(range(0, 2048, 11)), 4, 500000)\n"
        "x = p.member_add(); p.join(x, [1]); p.user_event(3, b'e', b'', False)\n"
        "p.step(400)\n"
        "s = p.stats(); s.pop('active_rows')\n"
        "print(p.state_hash(), sorted(s.items()), p.domain_stats(1, 64).tolist())\n"
    ) % (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "hostemu", "libgsim_hostemu.so"))
    outs = []
    for o in ("0", order):
        r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, GSIM_HOSTEMU_ORDER=o),
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        outs.append(r.stdout.strip())
    assert outs[0] == outs[1], outs


def test_snapshot_mid_flap_steps_on_like_the_oracle(hostemu_lib):
    cfg = lan_config(L, capacity=1500, n_initial=1500, seed=0xD1D1, disable_tcp_pings=1, mailbox_depth=4)
    a, ora = Pool(cfg, hostemu_lib), DomainOraclePool(cfg)
    for p in (a, ora):
        p.domain_set_range(0, 1500, 25, 1)
        p.domain_impair(list(range(1, 61, 4)), 500_000, 500_000, 1)
        p.domain_flap(list(range(1, 61, 2)), 37, 400_000)
        p.impair_flap(list(range(0, 1500, 11)), 5, 600_000)
        p.step(55)                                       # mid-epoch for most domains (period 37)
    blob = a.snapshot()
    fresh = Pool(cfg, hostemu_lib)
    fresh.restore(blob)
    for _ in range(6):
        for p in (fresh, ora):
            p.step(20)
        compare_pools(fresh, ora, f"restored vs oracle tick {fresh.now}")
    # an old blob (no domains) restored into a pool with domains clears them: it steps on like an oracle
    # without domains
    plain_cfg = lan_config(L, capacity=1500, n_initial=1500, seed=0xD1D1, disable_tcp_pings=1, mailbox_depth=4)
    old, ora2 = Pool(plain_cfg, hostemu_lib), DomainOraclePool(plain_cfg)
    for p in (old, ora2):
        p.impair(list(range(0, 1500, 13)), 400_000, 1)
        p.step(30)
    fresh.restore(old.snapshot())
    assert not fresh.domains().any() and fresh.domain_flap_get(3) == (0, 0)
    for _ in range(4):
        for p in (fresh, ora2):
            p.step(25)
        compare_pools(fresh, ora2, f"old blob vs oracle tick {fresh.now}")
