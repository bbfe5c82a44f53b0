"""Tick stretches (DESIGN.md §4.2): on a single-GPU pool the single ticks of a busy period run up to the
first quiet tick in one submission, and the device decides where that is: quiet at tick t when
t >= max(LAST_ACTIVE, dirty_tick + 1) + depth.  The host emulation runs GsBackend's default stretch
(one tick at a time, then the quiet probe); the counting backend counts one wait per stretch, as on CUDA,
and records the last stretch so that the rule can be checked.  Which ticks run singly and which in
windows must not show in the results: same digest, counters and columns as a pool that runs every tick
as a single launch, and as the oracle, after every operation."""
import ctypes as C
import os

from consul_b200 import _lib
from consul_b200.pool import FLAG_NO_WINDOWS, Pool, lan_config, wan_config
from oracle_binding import OraclePool
from parity import compare_pools

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MS = 1_000_000
# single ticks per bench step at 100 000 members with the host looking for quietness between chunks
# (backing off 1, 2, 4, 8 ticks), on the same pool after the same warm-up: odd steps 40, even steps 48
PARENT_SINGLE_TICKS = 48


def counted_lib():
    lib = _lib.load(os.path.join(ROOT, "tests", "hostemu", "libgsim_hostemu_counted.so"))
    lib.gsim_hostemu_waits.restype = C.c_uint64
    lib.gsim_hostemu_waits.argtypes = [C.POINTER(C.c_uint64)]
    lib.gsim_hostemu_last_stretch.restype = None
    lib.gsim_hostemu_last_stretch.argtypes = [C.POINTER(C.c_uint32)]
    return lib


def waits(lib):
    chunks = C.c_uint64()
    w = lib.gsim_hostemu_waits(C.byref(chunks))
    return w, chunks.value


def last_stretch(lib):
    out = (C.c_uint32 * 7)()
    lib.gsim_hostemu_last_stretch(out)
    return dict(zip(("t0", "nticks", "floor", "depth", "ran", "last_active", "quiet"), list(out)))


def check_rule(s):
    """A stretch stops at the first quiet tick, or runs all its ticks."""
    quiet_at = max(s["last_active"], s["floor"]) + s["depth"]
    if s["quiet"]:
        assert s["t0"] + s["ran"] == max(quiet_at, s["t0"]), s
    else:
        assert s["ran"] == s["nticks"] and s["t0"] + s["ran"] < quiet_at, s


def trio(lib, cfg_fn, **kw):
    """the pool on the counted host emulation, the same pool without windows, and the oracle"""
    return [Pool(cfg_fn(lib, **kw), lib), Pool(cfg_fn(lib, flags=FLAG_NO_WINDOWS, **kw), lib),
            OraclePool(cfg_fn(lib, **kw))]


def all3(pools, fn):
    out = [fn(p) for p in pools]
    assert out[0] == out[1] == out[2], out
    return out[0]


def step_all(pools, ticks, where, lib=None):
    for p in pools:
        p.step(ticks)
    compare_pools(pools[0], pools[2], where + " (stretches vs oracle)")
    compare_pools(pools[0], pools[1], where + " (stretches vs single ticks)")
    if lib is not None:
        check_rule(last_stretch(lib))


def test_bench_step_waits_three_times_and_runs_no_extra_single_tick():
    lib = counted_lib()
    n = 100_000
    p = Pool(lan_config(lib, capacity=n + 16, n_initial=n, seed=0x5EED0001), lib)
    p.step(64)
    for _ in range(2):  # warm-up: the step bench.py times
        x = p.member_add()
        assert p.join(x, [0]) == 1
        p.step(2048)
    for _ in range(2):  # one step of each parity
        w0, _ = waits(lib)
        x = p.member_add()
        assert p.join(x, [0]) == 1
        w1, k1 = waits(lib)
        start, c0 = p.now, p.sched_counts()
        p.step(2048)
        w2, k2 = waits(lib)
        c1 = p.sched_counts()
        assert w1 - w0 == 1                        # join: the rows it merges
        assert w2 - w1 <= 3, w2 - w1               # the stretch, the window chain, the count behind retirement
        assert k2 - k1 == 1                        # the whole cascade is one stretch
        s = last_stretch(lib)
        check_rule(s)
        assert s["t0"] == start and s["quiet"] == 1 and s["floor"] == start + 1
        single = c1["tick_launches"] - c0["tick_launches"]
        assert single == s["ran"] == s["last_active"] + s["depth"] - start
        assert single <= PARENT_SINGLE_TICKS
        assert c1["horizon_scans"] - c0["horizon_scans"] == 1
    p.close()


def test_bench_steps_same_results():
    lib = counted_lib()
    pools = trio(lib, lan_config, capacity=3003, n_initial=3000, seed=0x5EED0001)
    step_all(pools, 64, "warm", lib)
    for k in range(3):
        x = all3(pools, lambda p: p.member_add())
        assert all3(pools, lambda p: p.join(x, [0])) == 1
        step_all(pools, 2048, f"bench step {k}", lib)


def test_crash_wave():
    lib = counted_lib()
    pools = trio(lib, lan_config, capacity=4000, n_initial=4000, seed=23)
    step_all(pools, 40, "before", lib)
    assert all3(pools, lambda p: p.crash_fraction(20000, 1)) > 0
    for chunk in (7, 64, 200, 700):
        step_all(pools, chunk, f"crash wave +{chunk}", lib)
    assert pools[0].stats()["probe_failures"] > 0


def test_pool_wide_loss_runs_stretches_to_their_end():
    """With 20 % of all packets lost the pool is hardly ever quiet for long: nearly every tick runs singly,
    and the stretch that ends a step runs all its ticks."""
    lib = counted_lib()
    pools = trio(lib, lan_config, capacity=1500, n_initial=1500, seed=24, packet_loss_ppm=200000)
    for chunk in (50, 1, 333):
        step_all(pools, chunk, f"lossy +{chunk}", lib)
        s = last_stretch(lib)
        assert s["ran"] == s["nticks"] and s["t0"] + s["ran"] == pools[0].now, s
    sc = pools[0].sched_counts()
    assert sc["window_ticks"] < 40 and sc["tick_launches"] > 340, sc
    assert pools[0].stats()["nacks"] > 0


def test_wan_pool_with_a_deep_ring():
    lib = counted_lib()
    pools = trio(lib, wan_config, capacity=2002, n_initial=2000, seed=77, mailbox_depth=8)
    step_all(pools, 100, "wan steady", lib)
    assert last_stretch(lib)["depth"] == 8
    x = all3(pools, lambda p: p.member_add())
    assert all3(pools, lambda p: p.join(x, [5])) == 1
    step_all(pools, 600, "wan join", lib)
    all3(pools, lambda p: p.user_event(9, b"e", b"p", False))
    step_all(pools, 500, "wan event", lib)
    assert pools[0].sched_counts()["window_ticks"] > 0


def test_scheduled_operation_and_reaper_inside_a_step():
    """A leaving member's shutdown is scheduled for a later tick and the reaper wakes every 20 ticks: both
    split a step, so a stretch ends at them and a new one starts behind them."""
    lib = counted_lib()
    pools = trio(lib, lan_config, capacity=3000, n_initial=3000, seed=41, reap_interval_ns=2000 * MS,
                 reconnect_timeout_ns=3000 * MS, tombstone_timeout_ns=3000 * MS)
    step_all(pools, 30, "warm", lib)
    all3(pools, lambda p: p.crash_many([11, 12, 13]))
    all3(pools, lambda p: p.leave(17))
    _, k0 = waits(lib)
    step_all(pools, 900, "leave + crashes + reaps", lib)
    _, k1 = waits(lib)
    assert k1 - k0 >= 5, k1 - k0                   # stretches bounded by the schedule
    assert pools[0].stats()["probe_failures"] > 0
    step_all(pools, 300, "after", lib)


def test_host_write_just_before_a_step():
    """A host write that posts no mail (a crash) counts like mail at the tick it was made: the stretch may not
    stop before dirty_tick + 1 + depth even though LAST_ACTIVE is old."""
    lib = counted_lib()
    pools = trio(lib, lan_config, capacity=2001, n_initial=2000, seed=25)
    step_all(pools, 300, "quiet", lib)
    for k, chunk in enumerate((1, 2, 3)):  # one stretch each: none can stop before floor + depth = now + 3
        now = all3(pools, lambda p: p.now)
        all3(pools, lambda p: p.crash(100 + k))
        step_all(pools, chunk, f"crash + {chunk}", lib)
        s = last_stretch(lib)
        assert s["floor"] == now + 1 and s["t0"] == now, s
        assert s["ran"] == min(chunk, max(s["last_active"], now + 1) + s["depth"] - now), s
    all3(pools, lambda p: p.crash(200))
    step_all(pools, 50, "crash + 50", lib)
    x = all3(pools, lambda p: p.member_add())
    assert all3(pools, lambda p: p.join(x, [3])) == 1
    all3(pools, lambda p: p.user_event(4, b"deploy", b"now", False))
    step_all(pools, 400, "join + event", lib)
