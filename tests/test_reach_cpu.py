"""One-way reachability (gsim_impair_dir_*) on the CPU: the kernels' row bodies (tests/hostemu) against the
reach oracle (tests/oracle_reach/reach.patch) after every operation — digest, counters and columns — plus the
semantics of DESIGN.md §3.5 "One-way reachability": the symmetric case is gsim_impair_*, inbound-blocked,
outbound-blocked and TCP-blocked members behave as the rules say, snapshots, validation and a fuzz."""
import os
import random
import struct
import subprocess
import sys

import pytest

import fuzz_ops
import scenarios as sc
from backend_fuzz import Lockstep
from consul_b200 import _lib
from consul_b200.pool import (FLAG_NO_WINDOWS, FLAG_PUSH_PULL, IMPAIR_NO_TCP, GsimError, Pool, lan_config,
                              wan_config)
from consul_b200.wan import c5_latency_matrix
from oracle_reach import ReachOraclePool
from parity import compare_pools

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = _lib.load(os.path.join(ROOT, "tests", "hostemu", "libgsim_hostemu.so"))
ERR_INVALID, ERR_NOT_FOUND, ERR_STATE = -1, -5, -6
LAYOUT_IMPAIR, LAYOUT_REACH = 8, 64
FULL = 1_000_000


@pytest.fixture()
def make(hostemu_lib):
    return lambda cfg: [Pool(cfg, hostemu_lib), ReachOraclePool(cfg)]


def both(pools, fn):
    return sc.both(pools, fn)


def layout(blob):
    return struct.unpack_from("<I", blob, 36)[0]


def heard(p, member, slot):
    return bool(int(p.column("heard")[member]) >> slot & 1)


def inc_of(p, member):
    return int(p.column("key")[member]) >> 5


class Directional:
    """A pool whose impair / impair_fraction set a directional setting derived from their arguments (inbound
    only, outbound only, symmetric, or symmetric without TCP), so that the operation schedules of
    tests/backend_fuzz.py and tests/fuzz_ops.py exercise gsim_impair_dir_* unchanged."""

    def __init__(self, pool):
        self.pool = pool

    def __getattr__(self, name):
        return getattr(self.pool, name)

    @staticmethod
    def _dir(loss, delay):
        mode = (loss // 1000 + 7 * delay) % 4
        if mode == 0:
            return 0, loss, False
        if mode == 1:
            return loss, 0, False
        return loss, loss, mode == 3

    def impair(self, ids, loss, delay=0):
        s, r, t = self._dir(loss, delay)
        return self.pool.impair_dir(ids, s, r, delay, t)

    def impair_fraction(self, ppm, salt, loss, delay=0):
        s, r, t = self._dir(loss, delay)
        return self.pool.impair_dir_fraction(ppm, salt, s, r, delay, t)


# ---- the symmetric case is gsim_impair_* ---------------------------------------------------------------
def _setup(kind):
    if kind == "lan":
        return lan_config(L, capacity=3001, n_initial=3000, seed=0x4EAC1), None, None
    if kind == "wan_c5":
        return wan_config(L, capacity=2049, n_initial=2048, seed=0x4EAC2, mailbox_depth=8), c5_latency_matrix(16), None
    if kind == "push_pull":
        return lan_config(L, capacity=1025, n_initial=1024, seed=0x4EAC3, flags=FLAG_PUSH_PULL,
                          push_pull_interval_ns=1_000_000_000, mailbox_depth=4), None, None
    return wan_config(L, capacity=600, n_initial=600, seed=0x4EAC4, mailbox_depth=4, phase_group=1), None, "graph"


def _prepare(p, lat, extra, n):
    if lat is not None:
        p.latency_set(lat)
    if extra == "graph":
        p.graph_set(*fuzz_ops.random_graph(random.Random(9), n))


@pytest.mark.parametrize("kind", ["lan", "wan_c5", "push_pull", "graph"])
def test_symmetric_setting_is_impair(hostemu_lib, kind):
    cfg, lat, extra = _setup(kind)
    n = cfg.n_initial
    delay = 2 if lat is not None else (1 if (cfg.mailbox_depth or 2) >= 4 else 0)
    a, b = Pool(cfg, hostemu_lib), Pool(cfg, hostemu_lib)
    for p in (a, b):
        _prepare(p, lat, extra, n)
    ids = list(range(0, n, 13))
    a.impair(ids, 250000, delay)
    b.impair_dir(ids, 250000, 250000, delay)
    assert a.impair_fraction(30000, 7, 600000) == b.impair_dir_fraction(30000, 7, 600000, 600000)
    assert [a.impairment(i) for i in range(n)] == [b.impairment(i) for i in range(n)]
    assert all(b.impairment_dir(i) == (a.impairment(i)[0], a.impairment(i)[0], a.impairment(i)[1], False)
               for i in range(0, n, 7))
    for p in (a, b):
        p.user_event(1, b"e", b"v", False)
    for upto in (50, 200, 400):
        for p in (a, b):
            p.step(upto - p.now)
        compare_pools(a, b, f"{kind} tick {upto}")
    assert a.snapshot() == b.snapshot()                       # nothing directional: the blob of gsim_impair_*
    assert not layout(b.snapshot()) & LAYOUT_REACH


def test_fraction_picks_the_members_impair_fraction_picks(hostemu_lib):
    cfg = lan_config(hostemu_lib, capacity=5000, n_initial=5000, seed=0x4EAC5)
    a, b = Pool(cfg, hostemu_lib), Pool(cfg, hostemu_lib)
    ka = a.impair_fraction(50000, 11, 1000)
    kb = b.impair_dir_fraction(50000, 11, 0, FULL, 0, True)
    assert ka == kb > 0
    picked_a = [i for i in range(5000) if a.impairment(i) != (0, 0)]
    picked_b = [i for i in range(5000) if b.impairment_dir(i) != (0, 0, 0, False)]
    assert picked_a == picked_b and len(picked_a) == ka
    assert b.impairment_dir(picked_b[0]) == (0, FULL, 0, True)


# ---- behaviour on a pool with no other loss --------------------------------------------------------------
BLOCKED = [100, 400, 777]


def _lan(n, seed, **kw):
    return lan_config(L, capacity=n + 1, n_initial=n, seed=seed, **kw)


def test_inbound_blocked_with_tcp_fallback(make):
    """Inbound UDP blocked, TCP fallback on: no suspicion anywhere, and gossip never reaches the members."""
    n = 1000
    pools = make(_lan(n, 0x4EAD1))
    both(pools, lambda p: p.impair_dir(BLOCKED, 0, FULL))
    slot = both(pools, lambda p: p.user_event(5, b"deploy", b"v1", False))
    sc.step_compare(pools, 300, 50, "inbound blocked")
    for p in pools:
        s = p.stats()
        assert s["suspects"] == 0 and s["refutes"] == 0 and s["deads"] == 0, s
        assert s["packets_lost"] > 0
        assert sum(heard(p, m, slot) for m in range(n)) == n - len(BLOCKED)
        assert not any(heard(p, m, slot) for m in BLOCKED)


def test_inbound_blocked_push_pull_delivers_the_event(make):
    """... with push-pull on, the member's own push-pull (TCP) brings the event within two periods."""
    n = 1000
    pools = make(_lan(n, 0x4EAD2, flags=FLAG_PUSH_PULL, push_pull_interval_ns=1_000_000_000, mailbox_depth=4))
    # pushPullScale(1 s, 1000 members) = 6 s = 60 ticks of 100 ms
    period = 60
    both(pools, lambda p: p.impair_dir(BLOCKED, 0, FULL))
    t0 = pools[0].now
    slot = both(pools, lambda p: p.user_event(5, b"deploy", b"v1", False))
    reached = {}
    for _ in range(2 * period):
        for p in pools:
            p.step(1)
        for m in BLOCKED:
            if m not in reached and heard(pools[0], m, slot):
                reached[m] = pools[0].now - t0
        if pools[0].now % 20 == 0:
            compare_pools(*pools, f"push-pull tick {pools[0].now}")
    compare_pools(*pools, "push-pull end")
    assert sorted(reached) == BLOCKED, reached
    assert all(heard(pools[1], m, slot) for m in BLOCKED)
    assert max(reached.values()) <= 2 * period
    assert all(p.stats()["suspects"] == 0 for p in pools)


def test_inbound_blocked_without_tcp_fallback(make):
    """Without the TCP fallback the blocked members' probes all fail: their awareness saturates, they accuse
    healthy members, who refute; nobody is declared Failed."""
    n = 1000
    pools = make(_lan(n, 0x4EAD3, disable_tcp_pings=1))
    both(pools, lambda p: p.impair_dir(BLOCKED, 0, FULL))
    sc.step_compare(pools, 400, 50, "inbound blocked, no TCP fallback")
    aw_max = 8                                               # lan_config's awareness_max_multiplier
    for p in pools[:1]:
        meta = p.column("meta")
        assert all(int(meta[m]) & 7 == aw_max - 1 for m in BLOCKED)
    for p in pools:
        s = p.stats()
        assert s["suspects"] == s["refutes"] > 0 and s["deads"] == 0, s


def test_outbound_blocked_without_tcp_fallback(make):
    """Outbound UDP blocked: the member's acks never arrive, so it is suspected, and it refutes."""
    n = 1000
    pools = make(_lan(n, 0x4EAD4, disable_tcp_pings=1))
    inc0 = [inc_of(pools[0], m) for m in BLOCKED]
    both(pools, lambda p: p.impair_dir(BLOCKED, FULL, 0))
    sc.step_compare(pools, 300, 50, "outbound blocked")
    s = pools[0].stats()
    assert s["suspects"] == s["refutes"] > 0 and s["deads"] == 0, s
    assert all(inc_of(pools[0], m) > i0 for m, i0 in zip(BLOCKED, inc0))


def test_no_tcp_join_fails(make):
    n = 400
    pools = make(lan_config(L, capacity=n + 4, n_initial=n, seed=0x4EAD5))
    x = both(pools, lambda p: p.member_add())
    y = both(pools, lambda p: p.member_add())
    both(pools, lambda p: p.impair_dir([x, 7], 0, 0, 0, True))
    assert both(pools, lambda p: p.join(x, [0, 1, 2])) == 0        # the joiner has no TCP
    assert both(pools, lambda p: p.join(y, [7])) == 0              # the only seed has no TCP
    assert both(pools, lambda p: p.join(y, [7, 8, 7, 9])) == 2     # skipped like an unreachable seed
    compare_pools(*pools, "joins")
    sc.step_compare(pools, 60, 20, "after the joins")


@pytest.mark.parametrize("no_tcp", [True, False])
def test_no_tcp_member_keeps_its_event_from_push_pull(make, no_tcp):
    """An event whose origin cannot send UDP spreads only through push-pull: not at all without TCP."""
    n = 1000
    pools = make(_lan(n, 0x4EAD6, flags=FLAG_PUSH_PULL, push_pull_interval_ns=1_000_000_000, mailbox_depth=4))
    origin = 42
    both(pools, lambda p: p.impair_dir([origin], FULL, 0, 0, no_tcp))
    slot = both(pools, lambda p: p.user_event(origin, b"deploy", b"v1", False))
    sc.step_compare(pools, 180, 30, f"no_tcp={no_tcp}")
    reached = both(pools, lambda p: sum(heard(p, m, slot) for m in range(n)))
    if no_tcp:
        assert reached == 1
        assert pools[0].stats()["push_pulls"] > 0
    else:
        assert reached > 1


# ---- lockstep and scheduling ---------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
def test_lockstep_with_pauses_against_the_oracle(hostemu_lib, seed):
    pair = Lockstep(lambda c: Directional(Pool(c, hostemu_lib)), lambda c: Directional(ReachOraclePool(c)),
                    0x4EA0 + seed, extra=True)
    assert fuzz_ops.run_sequence(pair.make, hostemu_lib, 0x4EA1000 + seed, n_ops=30) == 30


def test_c5_matrix_delays_and_a_csr_graph(make):
    cfg = wan_config(L, capacity=2048, n_initial=2048, seed=0x4EAD7, mailbox_depth=8)
    pools = make(cfg)
    for p in pools:
        p.latency_set(c5_latency_matrix(16))
    both(pools, lambda p: p.impair_dir_fraction(20000, 3, 200000, 700000, 1))
    both(pools, lambda p: p.impair_dir_fraction(5000, 4, 0, 0, 0, True))
    both(pools, lambda p: p.pause(list(range(9, 2048, 97)), 40))
    slot = both(pools, lambda p: p.user_event(0, b"e", b"x" * 8, False))
    sc.step_compare(pools, 300, 30, "C5")
    assert slot >= 0
    g = make(wan_config(L, capacity=600, n_initial=600, seed=0x4EAD8, mailbox_depth=4, phase_group=1))
    for p in g:
        p.graph_set(*fuzz_ops.random_graph(random.Random(3), 600))
        p.impair_dir(list(range(0, 600, 11)), 0, FULL)
        p.impair_dir(list(range(5, 600, 23)), 400000, 0, 0, True)
    sc.step_compare(g, 300, 30, "graph")


@pytest.mark.parametrize("order", ["1", "2"])
def test_row_order_does_not_matter(order):
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "from consul_b200 import _lib\n"
        "from consul_b200.pool import Pool, lan_config, FLAG_PUSH_PULL\n"
        "L = _lib.load(%r)\n"
        "p = Pool(lan_config(L, capacity=2049, n_initial=2048, seed=37, flags=FLAG_PUSH_PULL, "
        "push_pull_interval_ns=10**9, mailbox_depth=4, disable_tcp_pings=0), L)\n"
        "p.impair_dir_fraction(30000, 1, 0, 10**6); p.impair_dir(list(range(5, 2048, 50)), 10**6, 0, 0, True)\n"
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


def test_windows_match_single_ticks_across_a_clear(hostemu_lib):
    n = 3000
    pools = [Pool(lan_config(hostemu_lib, capacity=n, n_initial=n, seed=0x4EAD9, flags=f), hostemu_lib)
             for f in (0, FLAG_NO_WINDOWS)]
    ora = ReachOraclePool(lan_config(L, capacity=n, n_initial=n, seed=0x4EAD9))
    ids = list(range(0, n, 31))
    for p in pools + [ora]:
        p.impair_dir(ids, 0, 0, 0, True)               # NO_TCP alone: the generic probe path
        p.step(200)
    compare_pools(pools[0], ora, "NO_TCP alone")
    for p in pools + [ora]:
        p.impair_dir(ids, 0, 0, 0, False)              # cleared: windows come back
        p.step(1500)
    assert pools[0].sched_counts()["window_ticks"] > 1000
    assert pools[1].sched_counts()["window_ticks"] == 0
    compare_pools(pools[0], pools[1], "windows vs single ticks")
    compare_pools(pools[0], ora, "windows vs oracle")


def test_clearing_returns_to_the_gate_off_path(hostemu_lib):
    n = 2000
    cfg = lan_config(hostemu_lib, capacity=n + 1, n_initial=n, seed=0x4EADA)
    ref, a = Pool(cfg, hostemu_lib), Pool(cfg, hostemu_lib)
    a.impair_dir([1, 2, 3], 100, 200000, 0, True)
    a.impair_dir_fraction(100000, 5, 0, 0, 0, True)
    a.step(50)
    a.impair_dir(list(range(n)), 0, 0, 0, False)
    ref.step(50)
    s0a, s0r = a.sched_counts(), ref.sched_counts()
    for p in (ref, a):
        x = p.member_add()
        p.join(x, [0])
        p.step(800)
    da = {k: a.sched_counts()[k] - s0a[k] for k in ("window_launches", "window_ticks")}
    dr = {k: ref.sched_counts()[k] - s0r[k] for k in ("window_launches", "window_ticks")}
    assert da == dr and da["window_ticks"] > 0
    assert all(a.impairment_dir(i) == (0, 0, 0, False) for i in range(0, n, 7))


# ---- snapshots -------------------------------------------------------------------------------------------
def test_snapshot_round_trip_mid_run(hostemu_lib):
    n = 2048
    cfg = wan_config(hostemu_lib, capacity=n, n_initial=n, seed=0x4EADB, mailbox_depth=8,
                     flags=FLAG_PUSH_PULL, push_pull_interval_ns=10**9)
    p = Pool(cfg, hostemu_lib)
    p.latency_set(c5_latency_matrix(16))
    p.impair_dir_fraction(30000, 3, 100000, FULL, 1, False)
    p.impair_dir(list(range(0, n, 101)), 0, 0, 0, True)
    p.user_event(2, b"e", b"", False)
    p.step(37)
    blob = p.snapshot()
    assert layout(blob) & LAYOUT_REACH and layout(blob) & LAYOUT_IMPAIR
    settings = [p.impairment_dir(i) for i in range(0, n, 3)]
    p.step(150)
    h1, s1 = p.state_hash(), p.stats()
    s1.pop("active_rows")
    q = Pool(cfg, hostemu_lib)                            # never impaired: restore brings every column
    q.restore(blob)
    assert [q.impairment_dir(i) for i in range(0, n, 3)] == settings
    q.step(150)
    s2 = q.stats()
    s2.pop("active_rows")
    assert q.state_hash() == h1 and s2 == s1


def test_a_symmetric_pool_writes_the_blob_it_always_did(hostemu_lib):
    n = 1000
    cfg = lan_config(hostemu_lib, capacity=n + 1, n_initial=n, seed=0x4EADC)
    a, b = Pool(cfg, hostemu_lib), Pool(cfg, hostemu_lib)
    a.impair([1, 5, 9], 300000, 0)
    b.impair_dir([1, 5, 9], 300000, 300000, 0, False)
    b.impair_dir([], 0, 700000)                            # nothing listed: no columns
    for p in (a, b):
        p.step(60)
    assert a.snapshot() == b.snapshot() and layout(b.snapshot()) == layout(a.snapshot())
    assert not layout(a.snapshot()) & LAYOUT_REACH


def test_restoring_a_blob_without_the_reach_columns(hostemu_lib):
    n = 1000
    cfg = lan_config(hostemu_lib, capacity=n + 1, n_initial=n, seed=0x4EADD, disable_tcp_pings=1)
    src = Pool(cfg, hostemu_lib)
    src.impair([4, 8], 500000, 0)
    src.step(20)
    plain = src.snapshot()
    assert layout(plain) & LAYOUT_IMPAIR and not layout(plain) & LAYOUT_REACH
    src.step(100)
    q = Pool(cfg, hostemu_lib)
    q.impair_dir([4, 8, 12], 0, FULL, 0, True)             # directional: its columns exist
    q.step(5)
    q.restore(plain)
    assert q.impairment_dir(4) == (500000, 500000, 0, False) and q.impairment_dir(12) == (0, 0, 0, False)
    assert q.impairment(8) == (500000, 0)
    q.step(100)
    assert q.state_hash() == src.state_hash()


# ---- validation ----------------------------------------------------------------------------------------
def test_validation(make):
    for p in make(lan_config(L, capacity=300, n_initial=300, seed=1, mailbox_depth=4)):
        for bad, code in ((lambda: p.impair_dir([1], FULL + 1, 0), ERR_INVALID),
                          (lambda: p.impair_dir([1], 0, FULL + 1), ERR_INVALID),
                          (lambda: p.impair_dir([1], 0, 0, 3), ERR_INVALID),
                          (lambda: p.impair_dir([300], 0, 10), ERR_NOT_FOUND),
                          (lambda: p.impair_dir_fraction(FULL + 1, 0, 0, 10), ERR_INVALID),
                          (lambda: p.impair_dir_fraction(1000, 0, 0, FULL + 1), ERR_INVALID),
                          (lambda: p.impairment_dir(300), ERR_NOT_FOUND)):
            with pytest.raises(GsimError) as e:
                bad()
            assert e.value.code == code
        assert p.impairment_dir(1) == (0, 0, 0, False)
        p.impair_dir([1], 1000, 2000, 2)
        p.impair_dir([2], 1000, 1000, 0, True)
        p.impair_dir([3], 1000, 1000, 0, False)
        for m in (1, 2):
            with pytest.raises(GsimError) as e:
                p.impairment(m)                               # half of a directional setting: refused
            assert e.value.code == ERR_STATE
        assert p.impairment(3) == (1000, 0)
        assert p.impairment_dir(1) == (1000, 2000, 2, False) and p.impairment_dir(2) == (1000, 1000, 0, True)


def test_unknown_flag_bits_are_refused(hostemu_lib):
    import ctypes as C
    p = Pool(lan_config(hostemu_lib, capacity=10, n_initial=10, seed=2), hostemu_lib)
    ids = (C.c_uint32 * 1)(1)
    out = C.c_uint32()
    for flags in (2, 4, 0x80, 0xFFFFFFFF, IMPAIR_NO_TCP | 2):
        assert hostemu_lib.gsim_impair_dir_many(p.h, ids, 1, 0, 0, 0, flags) == ERR_INVALID
        assert hostemu_lib.gsim_impair_dir_fraction(p.h, 1000, 0, 0, 0, 0, flags, C.byref(out)) == ERR_INVALID
    assert hostemu_lib.gsim_impair_dir_many(p.h, ids, 1, 0, 0, 0, IMPAIR_NO_TCP) == 0


# ---- fuzz ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(6))
def test_fuzz_with_directional_impairment(hostemu_lib, seed):
    pair = Lockstep(lambda c: Directional(Pool(c, hostemu_lib)), lambda c: Directional(ReachOraclePool(c)),
                    0x4EB0 + seed)
    assert fuzz_ops.run_sequence(pair.make, hostemu_lib, 0x4EB1000 + seed, n_ops=40) == 40
