"""What only the CUDA backend runs, on the H100: the tick stretch graph and its quiet probe, the window and
tick kernels' partitions of a pool over their grid, the row gather of a join, the device write batches and
the pause / resume / impair kernels.

- Schedule parity: a CUDA pool and a host-emulation pool take the same operations; after every one the
  state and every gsim_sched_counts field that counts ticks or decisions must be equal.  A stretch that
  stops late, a horizon that comes back early or quiet-probe counts that never make a pool pristine change
  no state, only the schedule, so only this sees them.
- A capped grid (GSIM_GRID_MAX) makes a pool the oracle follows column by column run what only the largest
  pools run at the full grid: several rounds of tiles per warp, uneven splits, window batches across tiles.
- Pauses and impairment fuzzed together on the device, and the primitives' edges against the oracle."""
import ctypes as C
import os
import random

import numpy as np
import pytest

import fuzz_ops
from backend_fuzz import GROWTH, SIZES, Lockstep, check_schedule, size_id
from consul_b200 import _lib
from consul_b200.pool import (FLAG_COORDINATES, FLAG_LOG_GLOBAL_EVENTS, FLAG_PUSH_PULL, Pool, lan_config,
                              wan_config)
from consul_b200.wan import c5_latency_matrix
from oracle_pause import PauseOraclePool
from parity import compare_pools

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def counted_lib():
    """the host emulation behind the counting backend: it records the last tick stretch"""
    lib = _lib.load(os.path.join(ROOT, "tests", "hostemu", "libgsim_hostemu_counted.so"))
    lib.gsim_hostemu_last_stretch.restype = None
    lib.gsim_hostemu_last_stretch.argtypes = [C.POINTER(C.c_uint32)]
    return lib


def last_stretch(lib):
    out = (C.c_uint32 * 7)()
    lib.gsim_hostemu_last_stretch(out)
    return dict(zip(("t0", "nticks", "floor", "depth", "ran", "last_active", "quiet"), list(out)))


def both(pools, fn):
    a, b = [fn(p) for p in pools]
    assert a == b, (a, b)
    return a


def events(p):
    return sorted((e.tick, e.type, e.subject, e.observer, e.ltime) for e in p.poll_events())


def same_state_and_schedule(pools, where):
    compare_pools(pools[0], pools[1], where, columns=False)
    check_schedule(pools[0], pools[1], where)


# ---- 1. schedule parity with the host emulation ----------------------------------------------------
@pytest.mark.parametrize("size", SIZES + (GROWTH,), ids=size_id)
def test_schedule_parity_fuzz(cuda_lib, hostemu_lib, size):
    n0, cap = (size, size + 24) if isinstance(size, int) else size
    seed = 0xBA0000 + n0
    pair = Lockstep(lambda c: Pool(c, cuda_lib), lambda c: Pool(c, hostemu_lib), seed, size=(n0, cap), extra=True,
                    schedule=True, grow=3 if size == GROWTH else 0)
    fuzz_ops.run_sequence(pair.make, cuda_lib, seed, n_ops=30)


@pytest.mark.parametrize("size", [None, (1025, 1049), (5000, 5024)], ids=str)
def test_schedule_parity_calm(cuda_lib, hostemu_lib, size):
    """calm pools spend most ticks in quiet windows, closed form included (the host emulation's windows cost a
    row per tick: the sizes stay small)"""
    for k in range(2):
        seed = 0xBA3000 + 17 * k + (size[0] if size else 0)
        pair = Lockstep(lambda c: Pool(c, cuda_lib), lambda c: Pool(c, hostemu_lib), seed, size=size,
                        disturb=False, schedule=True)
        fuzz_ops.run_sequence(pair.make, cuda_lib, seed, n_ops=40, calm=True)


@pytest.mark.parametrize("n", [100_000, 200_000])
def test_bench_step_schedule(cuda_lib, n):
    """bench.py's step (member_add, join, step(2048)), both parities of the joiner's slot: the stretch of the
    join cascade runs exactly up to the first quiet tick, LAST_ACTIVE + depth, as the rule says."""
    hl = counted_lib()
    cfg = dict(capacity=n + 16, n_initial=n, seed=0x5EED0001)
    pools = [Pool(lan_config(cuda_lib, **cfg), cuda_lib), Pool(lan_config(hl, **cfg), hl)]
    for p in pools:
        p.step(64)
    same_state_and_schedule(pools, "warm")
    for k in range(3):
        x = both(pools, lambda p: p.member_add())
        assert both(pools, lambda p: p.join(x, [0])) == 1
        start, c0 = pools[0].now, pools[0].sched_counts()
        for p in pools:
            p.step(2048)
        same_state_and_schedule(pools, f"bench step {k}")
        s = last_stretch(hl)
        single = pools[0].sched_counts()["tick_launches"] - c0["tick_launches"]
        assert s["t0"] == start and s["quiet"] == 1, s
        assert single == s["ran"] == s["last_active"] + s["depth"] - start, (single, s)


def test_wan_deep_ring_and_lossy_schedule(cuda_lib):
    """stretches that end by going quiet with a depth-8 ring, and by running out of ticks in a lossy pool"""
    hl = counted_lib()
    for name, fn, kw in (("wan", wan_config, dict(capacity=8194, n_initial=8192, seed=77, mailbox_depth=8)),
                         ("lossy", lan_config, dict(capacity=3002, n_initial=3000, seed=24, packet_loss_ppm=200000))):
        pools = [Pool(fn(cuda_lib, **kw), cuda_lib), Pool(fn(hl, **kw), hl)]
        if name == "wan":
            for p in pools:
                p.latency_set(c5_latency_matrix(16))
        ran_out = quiet = 0
        for k, chunk in enumerate((100, 1, 7, 333, 600, 2, 500)):
            if k == 3:
                x = both(pools, lambda p: p.member_add())
                both(pools, lambda p: p.join(x, [5]))
            if k == 5:
                both(pools, lambda p: p.user_event(9, b"e", b"p", False))
            for p in pools:
                p.step(chunk)
            same_state_and_schedule(pools, f"{name} +{chunk}")
            s = last_stretch(hl)
            quiet += s["quiet"]
            ran_out += s["ran"] == s["nticks"] and not s["quiet"]
        if name == "wan":
            assert quiet > 0 and pools[0].sched_counts()["window_ticks"] > 0
        else:
            assert ran_out > 0 and pools[0].stats()["nacks"] > 0


# ---- 2. a capped grid against the oracle -----------------------------------------------------------
def check(pools, where, sample=range(0, 1 << 30, 97)):
    compare_pools(*pools, where)
    assert pools[0].pause_stats() == pools[1].pause_stats(), where
    n = pools[0].stats()["n_members"]
    ids = [i for i in sample if i < n]
    assert [pools[0].paused_until(i) for i in ids] == [pools[1].paused_until(i) for i in ids], where


def steps(pools, chunks, where):
    for c in chunks:
        for p in pools:
            p.step(c)
        check(pools, f"{where} +{c} (tick {pools[0].now})")


def capped_workload(lib, kind):
    if kind == "lan20011":
        n = 20011
        cfg = dict(capacity=n + 8, n_initial=n, seed=0xCA9, flags=FLAG_LOG_GLOBAL_EVENTS)
        pools = [Pool(lan_config(lib, **cfg), lib), PauseOraclePool(lan_config(lib, **cfg))]
        x = both(pools, lambda p: p.member_add())
        both(pools, lambda p: p.join(x, [0]))
        check(pools, "join")
        steps(pools, (1, 3, 12, 40), "cascade")
        assert both(pools, lambda p: p.crash_fraction(20000, 5)) > 0
        steps(pools, (5, 60, 200), "crash wave")
        both(pools, lambda p: p.pause(list(range(3, n, 211)), 40))
        both(pools, lambda p: p.pause_fraction(5000, 2, 400))
        steps(pools, (20, 30, 300, 700), "pauses")
    elif kind == "wan8192":
        n = 8192
        cfg = dict(capacity=n, n_initial=n, seed=0xCA8, mailbox_depth=8, flags=FLAG_LOG_GLOBAL_EVENTS)
        pools = [Pool(wan_config(lib, **cfg), lib), PauseOraclePool(wan_config(lib, **cfg))]
        lat = c5_latency_matrix(16)
        room = 8 - 2 - (int(np.asarray(lat).max()) - 1)
        for p in pools:
            p.latency_set(lat)
        both(pools, lambda p: p.impair_fraction(20000, 3, 300000, room))
        both(pools, lambda p: p.impair(list(range(1, n, 301)), 1_000_000, 0))
        slot = both(pools, lambda p: p.user_event(0, b"e", b"x" * 16, False))
        assert slot >= 0
        steps(pools, (1, 9, 40, 150, 400, 900), "wan")
    else:
        n = 5000
        cfg = dict(capacity=n, n_initial=n, seed=0xCA7, flags=FLAG_PUSH_PULL | FLAG_COORDINATES,
                   push_pull_interval_ns=2_000_000_000, mailbox_depth=4)
        pools = [Pool(lan_config(lib, **cfg), lib), PauseOraclePool(lan_config(lib, **cfg))]
        both(pools, lambda p: p.crash_many(list(range(0, n, 53))))
        both(pools, lambda p: p.pause(list(range(7, n, 97)), 25))
        steps(pools, (1, 5, 30, 100, 300), "push-pull")
        assert pools[0].sched_counts()["window_ticks"] == 0          # only the tick kernel
    both(pools, events)
    return pools


@pytest.mark.parametrize("kind", ["lan20011", "wan8192", "push_pull"])
@pytest.mark.parametrize("cap", [1, 2, 17])
def test_capped_grid_against_the_oracle(cuda_lib, monkeypatch, cap, kind):
    monkeypatch.setenv("GSIM_GRID_MAX", str(cap))
    capped_workload(cuda_lib, kind)


@pytest.mark.parametrize("knob", ["GSIM_NO_PDL", "GSIM_WIN_CYCLIC"])
def test_capped_grid_with_knobs(cuda_lib, monkeypatch, knob):
    monkeypatch.setenv("GSIM_GRID_MAX", "2")
    monkeypatch.setenv(knob, "1")
    capped_workload(cuda_lib, "lan20011")


# ---- 3. pauses and impairment fuzzed together on the device ------------------------------------------
FUZZ_SIZES = [None, None, (129, 153), (1025, 1049), (5000, 5024), (20011, 20035), GROWTH]


@pytest.mark.parametrize("seed", range(16))
def test_fuzz_pauses_and_impairment(cuda_lib, seed):
    size = FUZZ_SIZES[seed % len(FUZZ_SIZES)]
    fseed = 0xBA4000 + seed
    pair = Lockstep(lambda c: Pool(c, cuda_lib), PauseOraclePool, fseed, size=size, extra=True,
                    grow=3 if size == GROWTH else 0)
    assert fuzz_ops.run_sequence(pair.make, cuda_lib, fseed, n_ops=30) == 30
    if size == GROWTH:
        assert pair.max_n > 1024


# ---- 4. the primitives' edges at the full grid -------------------------------------------------------
@pytest.mark.parametrize("k", [63, 64, 65, 200])
def test_join_with_many_seeds(cuda_lib, k):
    """k distinct seeds: k + 1 rows gathered in chunks of 64; 26 user events, then the joiner's alive rumor and
    join intent (28 live rumors) make the merges' writes overflow a write batch"""
    n = 5000
    cfg = lan_config(cuda_lib, capacity=n + 2, n_initial=n, seed=0x5EED + k, flags=FLAG_LOG_GLOBAL_EVENTS)
    pools = [Pool(cfg, cuda_lib), PauseOraclePool(cfg)]
    for s in range(26):
        both(pools, lambda p: p.user_event(37 * s + 1, b"ev%d" % s, b"z" * s, False))
    steps(pools, (2,), "events")
    x = both(pools, lambda p: p.member_add())
    seeds = random.Random(k).sample(range(n), k)
    seeds = seeds + seeds[:5] + [x, n + 1]
    assert both(pools, lambda p: p.join(x, seeds, False)) == k + 5
    check(pools, "join")
    y = both(pools, lambda p: p.member_add())
    assert both(pools, lambda p: p.join(y, [x] + seeds[::-1], True)) == k + 7   # x twice; n + 1 is y now
    check(pools, "second join")
    steps(pools, (1, 10, 100), "after")
    both(pools, events)


def test_long_id_lists_at_1m(cuda_lib):
    n = 1 << 20
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0x1D5, flags=FLAG_LOG_GLOBAL_EVENTS)
    pools = [Pool(cfg, cuda_lib), PauseOraclePool(cfg, threads=0)]
    rng = random.Random(3)

    def ids():
        some = rng.sample(range(n), 3500)
        return some + [rng.choice(some) for _ in range(1500)]   # 5 000 ids, duplicates included

    impaired, paused, crashed = ids(), ids(), ids()
    both(pools, lambda p: p.impair(impaired, 400000, 0))   # (a LAN ring has no room for a delay)
    assert both(pools, lambda p: p.pause(paused, 60)) == len(set(paused))
    both(pools, lambda p: p.crash_many(crashed))
    sample = sorted(set(paused))[::37] + list(range(0, n, 4099))
    check(pools, "lists", sample)
    for upto in (20, 61, 200):
        for p in pools:
            p.step(upto - p.now)
        compare_pools(*pools, f"tick {upto}", columns=upto == 200)
        assert pools[0].pause_stats() == pools[1].pause_stats()


def test_snapshot_of_an_impaired_pool(cuda_lib):
    n = 8192
    cfg = wan_config(cuda_lib, capacity=n + 4, n_initial=n, seed=0x5A1, mailbox_depth=8, flags=FLAG_LOG_GLOBAL_EVENTS)
    a = Pool(cfg, cuda_lib)
    a.latency_set(c5_latency_matrix(16))
    a.impair_fraction(30000, 4, 500000, 1)
    a.impair(list(range(5, n, 700)), 1_000_000, 0)
    a.pause(list(range(11, n, 333)), 50)
    x = a.member_add()
    a.join(x, [1, 2, 3])
    a.step(17)
    blob = a.snapshot()
    a.step(300)
    h1, s1 = a.state_hash(), a.stats()
    b = Pool(cfg, cuda_lib)                                  # a fresh pool, never impaired
    b.restore(blob)
    assert b.impairment(5) == a.impairment(5)
    b.step(300)
    s2 = b.stats()
    s1.pop("active_rows")
    s2.pop("active_rows")
    assert b.state_hash() == h1 and s2 == s1
    ora = PauseOraclePool(cfg)
    ora.latency_set(c5_latency_matrix(16))
    ora.impair_fraction(30000, 4, 500000, 1)
    ora.impair(list(range(5, n, 700)), 1_000_000, 0)
    ora.pause(list(range(11, n, 333)), 50)
    ora.member_add()
    ora.join(x, [1, 2, 3])
    ora.step(317)
    compare_pools(b, ora, "restored vs oracle")
