"""Intermittent impairment (gsim_impair_flap_*) on the CPU: the kernels' row bodies (tests/hostemu) against the
flap oracle (tests/oracle_flap/flap.patch), plus the rules of DESIGN.md §3.5 "Intermittent impairment": the
schedule function, a schedule that is always bad is the static impairment, one that is never bad is no
impairment, lockstep fuzz, snapshots, the read-only statistics and validation."""
import ctypes as C
import os
import random
import struct
import subprocess
import sys

import numpy as np
import pytest

import fuzz_ops
import scenarios as sc
import snapblob
from backend_fuzz import Lockstep
from consul_b200 import _lib
from consul_b200.pool import (FLAG_COORDINATES, FLAG_PROBE_PIGGYBACK, GsimError, Pool, lan_config, wan_config)
from consul_b200.wan import c5_latency_matrix
from oracle_flap import FlapOraclePool
from parity import compare_pools

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = _lib.load(os.path.join(ROOT, "tests", "hostemu", "libgsim_hostemu.so"))
ERR_INVALID, ERR_NOT_FOUND, ERR_STATE = -1, -5, -6
LAYOUT_FLAP = 256
FULL = 1_000_000
PUR_FLAP, PUR_IMPAIR = 12, 9
# counters that count scheduling work, not protocol traffic (a pool with a schedule steps every row generically)
SCHEDULING = {"active_rows"}


def layout(blob):
    return struct.unpack_from("<I", blob, 36)[0]


# the planes gsim_snapshot writes after the schedule column: stats, heard_cnt, conv_tick, crashed_alive and
# crashed_dead_tick, each stored raw behind its 4-byte tag
TAIL = (4 + 16 * 8) + 2 * (4 + 32 * 4) + 2 * (4 + 4)


def split_flap(blob):
    """(the blob without the schedule column and its layout bit, the column or None): the first part is what
    the same pool without a schedule column writes (and what tests/snapblob.py reads)"""
    blob = bytes(blob)
    lay = layout(blob)
    if not lay & LAYOUT_FLAP:
        return blob, None
    cap = struct.unpack_from("<I", blob, 12)[0]
    head, tail = blob[:-TAIL], blob[-TAIL:]
    # a column of one repeated word is stored as (tag 1, word); a schedule word is never 1 (period >= 1)
    if struct.unpack_from("<I", head, len(head) - 8)[0] == 1:
        col = np.full(cap, struct.unpack_from("<I", head, len(head) - 4)[0], np.uint32)
        head = head[:-8]
    else:
        assert struct.unpack_from("<I", head, len(head) - 4 - 4 * cap)[0] == 0
        col = np.frombuffer(head[len(head) - 4 * cap:], np.uint32).copy()
        head = head[:-(4 + 4 * cap)]
    return head[:36] + struct.pack("<I", lay & ~LAYOUT_FLAP) + head[40:] + tail, col


# ---- 1. the schedule function ------------------------------------------------------------------------------
def philox(seed, c0, c1, c2, c3):
    ctr, key, out = (C.c_uint32 * 4)(c0, c1, c2, c3), (C.c_uint32 * 2)(seed & 0xFFFFFFFF, seed >> 32), (C.c_uint32 * 4)()
    L.gsim_philox4x32(ctr, key, out)
    return list(out)


def flap_bad_py(seed, m, period, ppm, t):
    if period == 0 or ppm >= FULL:
        return 1
    if ppm == 0:
        return 0
    phase = philox(seed, m, 0xFFFFFFFF, PUR_FLAP, 0)[1] % period
    epoch = (t + phase) // period
    return int(philox(seed, m, epoch & 0xFFFFFFFF, PUR_FLAP, 0)[0] < (ppm << 32) // FULL)


def test_schedule_function_known_answers():
    rng = random.Random(0xF1A9)
    seeds = [0, 0x5EED, 0xDEADBEEF12345678]
    for seed in seeds:
        for period in (1, 7, 4095):
            for m in (0, 1, 129, 4096, 1 << 20):
                ppm = rng.choice([1, 100_000, 500_000, 999_999])
                ticks = list(range(0, 3 * period + 2, max(1, period // 5))) + [2**32 - 1, 2**32 - period]
                for t in ticks:
                    assert L.gsim_flap_bad(seed, m, period, ppm, t) == flap_bad_py(seed, m, period, ppm, t), \
                        (seed, m, period, ppm, t)
                assert all(L.gsim_flap_bad(seed, m, period, 0, t) == 0 for t in ticks)
                assert all(L.gsim_flap_bad(seed, m, period, FULL, t) == 1 for t in ticks)
    # an epoch is `period` ticks: the state changes only where (t + phase) crosses a multiple of the period
    seed, m, period = 0x5EED, 77, 7
    phase = philox(seed, m, 0xFFFFFFFF, PUR_FLAP, 0)[1] % period
    states = [L.gsim_flap_bad(seed, m, period, 500_000, t) for t in range(400)]
    assert all(states[t] == states[t - 1] for t in range(1, 400) if (t + phase) % period)
    assert 0 < sum(states) < 400
    assert L.gsim_flap_bad(seed, m, 0, 0, 5) == 1                          # no schedule: always in force
    assert L.gsim_flap_bad(seed, m, 4096, 0, 5) == ERR_INVALID
    assert L.gsim_flap_bad(seed, m, 7, FULL + 1, 5) == ERR_INVALID


# ---- 2. always bad is the static impairment ---------------------------------------------------------------
def _kind(kind):
    """(config, latency matrix, impair(pool) -> ids)"""
    if kind == "lan":
        def imp(p):
            ids = list(range(0, 1500, 17))
            p.impair(ids, 300_000, 1)
            return ids
        return lan_config(L, capacity=1501, n_initial=1500, seed=0xF1A1, mailbox_depth=4), None, imp
    if kind == "one_way_no_tcp":
        def imp(p):
            a, b = list(range(3, 1200, 29)), list(range(11, 1200, 41))
            p.impair_dir(a, 0, FULL, 0, True)
            p.impair_dir(b, 600_000, 0, 0, True)
            return a + b
        return lan_config(L, capacity=1200, n_initial=1200, seed=0xF1A2, disable_tcp_pings=0), None, imp
    if kind == "wan_c5":
        def imp(p):
            p.impair_fraction(40_000, 5, 200_000, 2)
            return [i for i in range(2048) if p.impairment(i) != (0, 0)]
        return (wan_config(L, capacity=2048, n_initial=2048, seed=0xF1A3, mailbox_depth=8), c5_latency_matrix(16),
                imp)
    if kind == "piggyback":
        def imp(p):
            ids = list(range(5, 1000, 13))
            p.impair(ids, 400_000, 1)
            return ids
        return (lan_config(L, capacity=1000, n_initial=1000, seed=0xF1A4, flags=FLAG_PROBE_PIGGYBACK,
                           mailbox_depth=4), None, imp)
    def imp(p):
        ids = list(range(2, 800, 9))
        p.impair(ids, 250_000, 2)
        return ids
    return lan_config(L, capacity=800, n_initial=800, seed=0xF1A5, flags=FLAG_COORDINATES, mailbox_depth=4), None, imp


@pytest.mark.parametrize("kind", ["lan", "one_way_no_tcp", "wan_c5", "piggyback", "coordinates"])
def test_always_bad_is_the_static_impairment(hostemu_lib, kind):
    cfg, lat, imp = _kind(kind)
    a, b = Pool(cfg, hostemu_lib), Pool(cfg, hostemu_lib)
    for p in (a, b):
        if lat is not None:
            p.latency_set(lat)
        ids = imp(p)
        p.user_event(1, b"e", b"v", False)
    a.impair_flap(ids, 7, FULL)
    assert a.impair_flap_get(ids[0]) == (7, FULL) and b.impair_flap_get(ids[0]) == (0, 0)
    for k in [1, 1, 2, 3, 5, 8, 13, 21, 40, 60, 100]:
        for p in (a, b):
            p.step(k)
        compare_pools(a, b, f"{kind} tick {a.now}")
        blob, col = split_flap(a.snapshot())
        assert col is not None and int(col[ids[0]]) == 7 << 20 | FULL
        assert blob == b.snapshot(), f"{kind} tick {a.now}: blobs differ"
    s = a.stats()
    assert s["packets_lost"] > 0 or kind == "coordinates"


# ---- 3. never bad is no impairment --------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["lan", "one_way_no_tcp", "wan_c5"])
def test_never_bad_is_no_impairment(hostemu_lib, kind):
    cfg, lat, imp = _kind(kind)
    a, b = Pool(cfg, hostemu_lib), Pool(cfg, hostemu_lib)
    for p in (a, b):
        if lat is not None:
            p.latency_set(lat)
        p.user_event(1, b"e", b"v", False)
    ids = imp(a)
    a.impair_flap(ids, 50, 0)
    for k in [1, 2, 5, 20, 60, 150]:
        for p in (a, b):
            p.step(k)
        assert a.state_hash() == b.state_hash(), f"{kind} tick {a.now}"
        sa, sb = a.stats(), b.stats()
        for f in SCHEDULING:
            sa.pop(f), sb.pop(f)
        assert sa == sb, f"{kind} tick {a.now}"
    assert a.flap_stats() == {"scheduled": len(set(ids)), "bad": 0}


# ---- 4. lockstep with the flap oracle --------------------------------------------------------------------
class FlapLockstep(Lockstep):
    """A Lockstep pair whose pools also take flap schedule operations drawn for (seed, tick): schedules set,
    changed and cleared on lists of members and on a seeded fraction.  Both must return the same results."""

    FLAP = 0xF1A9

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.flap_record = {}

    def step(self, side, k):
        p = side.pool
        now, n = p.now, p.stats()["n_members"]
        rng = self._rng(self.FLAP, now)
        res = None
        if n and rng.random() < 0.5:
            period = rng.choice([0, 1, 2, 5, 13, 50, 4095])
            ppm = rng.choice([0, 150_000, 500_000, 900_000, FULL])
            try:
                if rng.random() < 0.7:
                    ids = [rng.randrange(n) for _ in range(rng.randint(1, 30))]
                    p.impair_flap(ids, period, ppm)
                    res = ("many", period, ppm, [p.impair_flap_get(i) for i in ids[:4]])
                else:
                    res = ("fraction", p.impair_flap_fraction(rng.choice([30_000, 300_000]), rng.randrange(9),
                                                              period, ppm))
            except GsimError as e:
                res = e.code
        if side.index == 0:
            self.flap_record[now] = res
        else:
            assert self.flap_record.get(now) == res, f"seed {self.seed} tick {now}: {self.flap_record.get(now)} vs {res}"
        super().step(side, k)


@pytest.mark.parametrize("seed", range(6))
def test_fuzz_against_the_flap_oracle(hostemu_lib, seed):
    pair = FlapLockstep(lambda c: Pool(c, hostemu_lib), lambda c: FlapOraclePool(c), 0xF1B0 + seed, extra=True)
    assert fuzz_ops.run_sequence(pair.make, hostemu_lib, 0xF1B1000 + seed, n_ops=40) == 40


def test_flapping_lan_against_the_oracle(hostemu_lib):
    """Loss, delay and NO_TCP that come and go, without the TCP fallback: suspicions happen, and both agree."""
    cfg = lan_config(L, capacity=2001, n_initial=2000, seed=0xF1C1, disable_tcp_pings=1, mailbox_depth=4)
    pools = [Pool(cfg, hostemu_lib), FlapOraclePool(cfg)]
    sc.both(pools, lambda p: p.impair_dir_fraction(30_000, 1, 500_000, 500_000, 1, True))
    sc.both(pools, lambda p: p.impair_flap_fraction(30_000, 1, 10, 300_000))
    sc.both(pools, lambda p: p.impair_flap(list(range(0, 2000, 97)), 3, 500_000))
    sc.both(pools, lambda p: p.user_event(7, b"e", b"x", False))
    sc.step_compare(pools, 400, 25, "flapping LAN")
    s = pools[0].stats()
    assert s["suspects"] > 0 and s["packets_lost"] > 0, s
    x = sc.both(pools, lambda p: p.member_add())
    assert sc.both(pools, lambda p: p.join(x, list(range(0, 2000, 50)))) > 0
    sc.step_compare(pools, 100, 20, "after a join")


@pytest.mark.parametrize("order", ["1", "2"])
def test_row_order_does_not_matter(order):
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "from consul_b200 import _lib\n"
        "from consul_b200.pool import Pool, lan_config, FLAG_PUSH_PULL\n"
        "L = _lib.load(%r)\n"
        "p = Pool(lan_config(L, capacity=2049, n_initial=2048, seed=41, flags=FLAG_PUSH_PULL, "
        "push_pull_interval_ns=10**9, mailbox_depth=4, disable_tcp_pings=1), L)\n"
        "p.impair_dir_fraction(30000, 1, 600000, 600000, 1, True); p.impair_flap_fraction(30000, 1, 9, 400000)\n"
        "x = p.member_add(); p.join(x, [1]); p.user_event(3, b'e', b'', False)\n"
        "p.step(400)\n"
        "s = p.stats(); s.pop('active_rows')\n"
        "print(p.state_hash(), sorted(s.items()))\n"
    ) % (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "hostemu", "libgsim_hostemu.so"))
    outs = []
    for o in ("0", order):
        r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, GSIM_HOSTEMU_ORDER=o),
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        outs.append(r.stdout.strip())
    assert outs[0] == outs[1], outs


# ---- 5. snapshots ----------------------------------------------------------------------------------------
def test_snapshot_mid_epoch_restores_into_a_fresh_pool(hostemu_lib):
    cfg = lan_config(L, capacity=1500, n_initial=1500, seed=0xF1D1, disable_tcp_pings=1, mailbox_depth=4)
    a, ora = Pool(cfg, hostemu_lib), FlapOraclePool(cfg)
    for p in (a, ora):
        p.impair_fraction(50_000, 2, 500_000, 1)
        p.impair_flap_fraction(50_000, 2, 37, 400_000)
        p.step(55)                                      # mid-epoch for most members (period 37)
    blob = a.snapshot()
    assert layout(blob) & LAYOUT_FLAP
    fresh = Pool(cfg, hostemu_lib)
    fresh.restore(blob)
    assert fresh.flap_stats() == a.flap_stats()
    assert fresh.snapshot() == blob
    for _ in range(6):
        for p in (a, fresh, ora):
            p.step(20)
        compare_pools(a, fresh, f"restored tick {a.now}")
        compare_pools(a, ora, f"oracle tick {a.now}")
    # a blob without the column clears every schedule
    plain = Pool(cfg, hostemu_lib)
    fresh.restore(plain.snapshot())
    assert fresh.flap_stats() == {"scheduled": 0, "bad": 0}
    blob, col = split_flap(fresh.snapshot())
    assert not col.any() and fresh.state_hash() == plain.state_hash()
    snapblob.parse(blob)


def test_a_never_scheduled_pool_writes_the_blob_it_always_did(hostemu_lib):
    cfg = lan_config(L, capacity=900, n_initial=900, seed=0xF1D2)
    a, b = Pool(cfg, hostemu_lib), Pool(cfg, hostemu_lib)
    for p in (a, b):
        p.impair(list(range(0, 900, 7)), 200_000, 0)
        p.step(30)
    a.impair_flap(list(range(0, 900, 7)), 0, 0)         # clearing on a pool that never had a schedule
    assert a.flap_stats() == {"scheduled": 0, "bad": 0}
    assert a.snapshot() == b.snapshot()
    assert not layout(a.snapshot()) & LAYOUT_FLAP
    # once the column exists the blob carries it, even after every schedule is cleared
    a.impair_flap([3], 5, 100)
    a.impair_flap([3], 0, 0)
    blob, col = split_flap(a.snapshot())
    assert blob == b.snapshot() and not col.any()


# ---- 6. read-only statistics -------------------------------------------------------------------------------
def test_flap_stats_count_with_the_schedule_function(hostemu_lib):
    seed = 0xF1E1
    cfg = lan_config(L, capacity=3000, n_initial=3000, seed=seed)
    p = Pool(cfg, hostemu_lib)
    p.impair_fraction(100_000, 3, 300_000)
    k = p.impair_flap_fraction(100_000, 3, 11, 350_000)
    p.impair_flap(list(range(1, 3000, 101)), 4095, 700_000)
    sched = {i: p.impair_flap_get(i) for i in range(3000)}
    picked = [i for i, v in sched.items() if v != (0, 0)]
    assert len(picked) == len(set(picked) | set(range(1, 3000, 101))) and k > 0
    for _ in range(4):
        p.step(17)
        h, s = p.state_hash(), p.stats()
        want = [0, 0]
        for i, (per, ppm) in sched.items():
            if per:
                want[0] += 1
                want[1] += L.gsim_flap_bad(seed, i, per, ppm, p.now)
        got = p.flap_stats()
        assert [got["scheduled"], got["bad"]] == want
        assert 0 < want[1] < want[0]
        assert p.state_hash() == h and p.stats() == s and p.flap_stats() == got


def test_fraction_picks_the_members_impair_fraction_picks(hostemu_lib):
    cfg = lan_config(hostemu_lib, capacity=5000, n_initial=5000, seed=0xF1E2)
    a, b = Pool(cfg, hostemu_lib), Pool(cfg, hostemu_lib)
    ka = a.impair_fraction(50_000, 11, 1000)
    kb = b.impair_flap_fraction(50_000, 11, 20, 5000)
    assert ka == kb > 0
    assert [i for i in range(5000) if a.impairment(i) != (0, 0)] == \
        [i for i in range(5000) if b.impair_flap_get(i) != (0, 0)]
    assert b.impair_flap_fraction(50_000, 11, 0, 0) == kb          # period 0 clears them again
    assert b.flap_stats()["scheduled"] == 0


# ---- 7. validation --------------------------------------------------------------------------------------------
def test_validation(hostemu_lib):
    cfg = lan_config(hostemu_lib, capacity=100, n_initial=64, seed=0xF1F1)
    for p in (Pool(cfg, hostemu_lib), FlapOraclePool(cfg)):
        for fn in (lambda: p.impair_flap([1], 4096, 0), lambda: p.impair_flap([1], 5, FULL + 1),
                   lambda: p.impair_flap_fraction(FULL + 1, 1, 5, 0), lambda: p.impair_flap_fraction(10, 1, 4096, 0),
                   lambda: p.impair_flap_fraction(10, 1, 5, FULL + 1)):
            with pytest.raises(GsimError) as e:
                fn()
            assert e.value.code == ERR_INVALID
        for fn in (lambda: p.impair_flap([64], 5, 10), lambda: p.impair_flap_get(64)):
            with pytest.raises(GsimError) as e:
                fn()
            assert e.value.code == ERR_NOT_FOUND
        p.impair_flap([63], 4095, FULL)
        assert p.impair_flap_get(63) == (4095, FULL)
        p.impair_flap([63], 0, 123)
        assert p.impair_flap_get(63) == (0, 0)


def test_sharded_pools_refuse():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29563",
           os.path.join(ROOT, "tests", "sharded_flap_worker_cpu.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "FLAP REFUSED" in r.stdout
