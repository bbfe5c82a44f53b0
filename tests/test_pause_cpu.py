"""Paused members (gsim_pause_*) on the CPU: the kernels' row bodies (tests/hostemu) against the pause
oracle after every operation — digest, counters, columns, resume ticks and pause statistics — plus the
semantics of DESIGN.md §3.6 and every interaction with the other operations."""
import os
import random
import struct
import subprocess
import sys

import numpy as np
import pytest

import fuzz_ops
import scenarios as sc
from consul_b200 import _lib
from consul_b200.pool import (FLAG_LOG_GLOBAL_EVENTS, FLAG_NO_WINDOWS, FLAG_PUSH_PULL, NEVER,
                              PRED_CRASHED_ALL_DEAD, GsimError, Pool, lan_config, wan_config)
from consul_b200.wan import c5_latency_matrix
from oracle_pause import PauseOraclePool
from parity import active_mask, compare_pools

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
L = _lib.load(os.path.join(ROOT, "tests", "hostemu", "libgsim_hostemu.so"))
ERR_INVALID, ERR_NOT_FOUND, ERR_STATE = -1, -5, -6
TRUTH_UP, TRUTH_CRASHED = 1, 2
RANK_ALIVE, RANK_SUSPECT, RANK_DEAD = 0, 1, 2
EV_MEMBER_JOIN, EV_MEMBER_FAILED = 0, 2
LAYOUT_PAUSE = 32


@pytest.fixture()
def make(hostemu_lib):
    return lambda cfg: [Pool(cfg, hostemu_lib), PauseOraclePool(cfg)]


def both(pools, fn):
    return sc.both(pools, fn)


def check(pools, where, sample=range(0, 1 << 30, 97)):
    """Digest, counters, columns, pause statistics and sampled resume ticks are the oracle's."""
    compare_pools(*pools, where)
    assert pools[0].pause_stats() == pools[1].pause_stats(), where
    n = pools[0].stats()["n_members"]
    ids = [i for i in sample if i < n]
    assert [pools[0].paused_until(i) for i in ids] == [pools[1].paused_until(i) for i in ids], where


def step_check(pools, ticks, every, where, sample=range(0, 1 << 30, 97)):
    done = 0
    while done < ticks:
        k = min(every, ticks - done)
        for p in pools:
            p.step(k)
        done += k
        check(pools, f"{where} +{done}", sample)


def events(p):
    return sorted((e.tick, e.type, e.subject, e.observer) for e in p.poll_events())


def layout(blob):
    return struct.unpack_from("<I", blob, 36)[0]


def truth_rank(p, i):
    k = int(p.column("key")[i])
    return k & 3, (k >> 2) & 3, k >> 5


# ---- the three pause lengths of the issue's threshold question --------------------------------------
# LAN defaults at 3 000 members on 100 ms ticks: ProbeInterval 10, ProbeTimeout 5, the suspicion timeout
# 140 ticks with every confirmation and 835 without any.
@pytest.mark.parametrize("d,expect", [(3, "alive"), (50, "suspect"), (900, "dead")])
def test_pause_lengths(make, d, expect):
    n = 3000
    pools = make(lan_config(L, capacity=n + 1, n_initial=n, seed=0x9A05E, flags=FLAG_LOG_GLOBAL_EVENTS))
    victims = [7, 300, 1500, 2999]
    sc.step_compare(pools, 13, 13, "warm up")
    inc0 = [truth_rank(pools[0], v)[2] for v in victims]
    t0 = pools[0].now
    assert both(pools, lambda p: p.pause(victims, d)) == len(victims)
    sample = victims + list(range(0, n, 211))
    check(pools, "paused", sample)
    assert all(p.paused_until(v) == t0 + d for p in pools for v in victims)
    assert all(truth_rank(pools[0], v)[0] == TRUTH_CRASHED for v in victims)
    assert pools[0].stats()["n_crashed"] == len(victims)
    step_check(pools, d, max(1, d // 6), f"d={d} paused", sample)
    assert pools[0].now == t0 + d
    st = pools[0].pause_stats()
    assert st["paused"] == 0 and all(p.paused_until(v) == NEVER for p in pools for v in victims)
    assert all(truth_rank(pools[0], v)[0] == TRUTH_UP for v in victims)
    assert pools[0].stats()["n_crashed"] == 0
    ev = both(pools, events)
    s = pools[0].stats()
    if expect == "alive":
        assert st["resumed_alive"] == len(victims) and s["suspects"] == 0, (st, s)
    elif expect == "suspect":
        assert st["resumed_suspect"] > 0 and st["resumed_dead"] == 0, st
    else:
        assert st["resumed_dead"] == len(victims), st
        failed = [e for e in ev if e[1] == EV_MEMBER_FAILED]
        assert sorted(e[2] for e in failed) == victims and all(e[0] < t0 + d for e in failed)
        joins = [e for e in ev if e[1] == EV_MEMBER_JOIN]
        assert sorted(e[2] for e in joins) == victims and all(e[0] == t0 + d for e in joins), joins
    step_check(pools, 40, 5, f"d={d} resumed", sample)
    for v, i0 in zip(victims, inc0):
        truth, rank, inc = truth_rank(pools[0], v)
        assert truth == TRUTH_UP and rank == RANK_ALIVE
        assert (inc > i0) == (expect != "alive")  # a refutation bumps past the accused incarnation
    assert pools[0].stats()["refutes"] == st["resumed_suspect"] + st["resumed_dead"]


# ---- pool setups ---------------------------------------------------------------------------------
def _setup(kind):
    if kind == "lan20k":
        return lan_config(L, capacity=20001, n_initial=20000, seed=0x20C), None, None
    if kind == "wan_c5":
        return wan_config(L, capacity=2049, n_initial=2048, seed=0xC5, mailbox_depth=8, tick_ns=100_000_000), \
            c5_latency_matrix(16), None
    if kind == "push_pull":
        return lan_config(L, capacity=1025, n_initial=1024, seed=0x9911, flags=FLAG_PUSH_PULL,
                          push_pull_interval_ns=2_000_000_000, mailbox_depth=4), None, None
    if kind == "graph":
        return wan_config(L, capacity=600, n_initial=600, seed=0x6AF, mailbox_depth=4, phase_group=1), None, "graph"
    return lan_config(L, capacity=3001, n_initial=3000, seed=0x1A9), None, "impair"


@pytest.mark.parametrize("kind", ["lan20k", "wan_c5", "push_pull", "graph", "impair"])
def test_setups_match_the_oracle(make, kind):
    cfg, lat, extra = _setup(kind)
    pools = make(cfg)
    n = cfg.n_initial
    for p in pools:
        if lat is not None:
            p.latency_set(lat)
        if extra == "graph":
            p.graph_set(*fuzz_ops.random_graph(random.Random(5), n))
        if extra == "impair":
            p.impair(list(range(0, n, 17)), 300000)
    if extra != "graph":
        x = both(pools, lambda p: p.member_add())
        both(pools, lambda p: p.join(x, [0]))
    both(pools, lambda p: p.user_event(5, b"deploy", b"v1", False))
    # mixed lengths through pause_many, and a fraction (some impaired members among them)
    both(pools, lambda p: p.pause(list(range(3, n, 101)), 4))
    both(pools, lambda p: p.pause(list(range(50, n, 307)), 60))
    k = both(pools, lambda p: p.pause_fraction(10000, 3, 250))
    assert k > 0
    step_check(pools, 400, 25, kind)
    st = pools[0].pause_stats()
    assert st["paused"] == 0 and sum(st.values()) > k


def test_no_windows_matches_windows_and_a_resume_ends_a_quiet_stretch(hostemu_lib):
    """A quiet pool whose only paused members are already Dead: the resume tick lands in what would have
    been one long quiet window.  The step must stop there, refute, and match single ticks and the oracle."""
    n = 3000
    pools = []
    for flags in (FLAG_LOG_GLOBAL_EVENTS, FLAG_LOG_GLOBAL_EVENTS | FLAG_NO_WINDOWS):
        p = Pool(lan_config(hostemu_lib, capacity=n, n_initial=n, seed=0x0D1E, flags=flags), hostemu_lib)
        pools.append(p)
    ora = PauseOraclePool(lan_config(L, capacity=n, n_initial=n, seed=0x0D1E, flags=FLAG_LOG_GLOBAL_EVENTS))
    ids = [11, 222, 1333]
    for p in pools + [ora]:
        p.pause(ids, 1500)
        assert p.run_until(PRED_CRASHED_ALL_DEAD, 0, 1400, 100) != NEVER   # all Dead, long before the resume
        p.step(1200 - p.now)
    for p in pools:
        assert [truth_rank(p, i)[1] for i in ids] == [RANK_DEAD] * 3
    before = pools[0].sched_counts()
    for p in pools + [ora]:
        p.step(700)                       # one call across the resume at tick 1500
    after = pools[0].sched_counts()
    assert after["window_ticks"] - before["window_ticks"] > 500
    assert pools[1].sched_counts()["window_ticks"] == 0
    compare_pools(pools[0], pools[1], "windows vs single ticks")
    compare_pools(pools[0], ora, "windows vs oracle")
    for p in pools + [ora]:
        assert p.pause_stats() == {"paused": 0, "resumed_alive": 0, "resumed_suspect": 0, "resumed_dead": 3}
        joins = [e for e in events(p) if e[1] == EV_MEMBER_JOIN]
        assert [(e[0], e[2]) for e in joins] == [(1500, i) for i in ids]


@pytest.mark.parametrize("order", ["1", "2"])
def test_row_order_does_not_matter(order):
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "from consul_b200 import _lib\n"
        "from consul_b200.pool import Pool, wan_config\n"
        "L = _lib.load(%r)\n"
        "p = Pool(wan_config(L, capacity=2049, n_initial=2048, seed=31, mailbox_depth=8), L)\n"
        "p.pause_fraction(30000, 1, 40); p.pause(list(range(5, 2048, 50)), 300); x = p.member_add(); p.join(x, [1])\n"
        "p.step(400)\n"
        "s = p.stats(); s.pop('active_rows')\n"
        "print(p.state_hash(), sorted(s.items()), p.pause_stats())\n"
    ) % (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "hostemu", "libgsim_hostemu.so"))
    outs = []
    for o in ("0", order):
        r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, GSIM_HOSTEMU_ORDER=o),
                           capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr[-2000:]
        outs.append(r.stdout.strip())
    assert outs[0] == outs[1], outs


def test_queue_wake_invariant_across_a_pause(tmp_path):
    """tests/hostemu/pause_wake_check.cpp: the queue_wake_check build, with members paused while they have
    broadcasts queued and resumed, checked after every tick."""
    exe = str(tmp_path / "pause_wake_check")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-pthread", "-o", exe,
                    os.path.join(ROOT, "tests", "hostemu", "pause_wake_check.cpp"),
                    os.path.join(ROOT, "tests", "hostemu", "hostemu_backend.cpp")], check=True, cwd=ROOT)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr


def test_a_paused_member_keeps_its_state(make):
    n = 2000
    pools = make(lan_config(L, capacity=n + 1, n_initial=n, seed=0x57A7E))
    x = both(pools, lambda p: p.member_add())
    both(pools, lambda p: p.join(x, [0]))
    both(pools, lambda p: p.user_event(9, b"deploy", b"v1", False))
    sc.step_compare(pools, 3, 3, "spreading")
    p = pools[0]
    heard = p.column("heard")[:n + 1]
    v = [i for i in range(n) if heard[i] and i != 9][:5]
    assert len(v) == 5
    both(pools, lambda q: q.pause(v, 80))
    cols = ("heard", "queued", "tx", "ltime_member", "ltime_event", "event_min", "cursor", "pass", "meta")
    frozen = {c: p.column(c)[..., v].copy() for c in cols}
    step_check(pools, 79, 8, "paused")
    # a rumor that completes among the running members meanwhile is retired: its bit goes everywhere
    act = active_mask(p)
    assert act != 0
    for c in cols:
        now, then = p.column(c)[..., v], frozen[c]
        if c in ("heard", "queued"):
            now, then = now & act, then & act
        elif c == "tx":
            now, then = now[[r for r in range(30) if act >> r & 1]], then[[r for r in range(30) if act >> r & 1]]
        assert np.array_equal(now, then), c
    step_check(pools, 20, 1, "resumed")


# ---- interactions ----------------------------------------------------------------------------------
def test_crash_cancels_the_resume(make):
    n = 1000
    pools = make(lan_config(L, capacity=n, n_initial=n, seed=0xC4A5))
    both(pools, lambda p: p.pause([10, 20, 30], 40))
    sc.step_compare(pools, 10, 10, "paused")
    both(pools, lambda p: p.crash_many([10, 20]))
    assert all(p.paused_until(10) == NEVER and p.paused_until(30) == 40 for p in pools)
    # crash_fraction draws among running members only: paused ones are never selected
    k = both(pools, lambda p: p.crash_fraction(1_000_000, 4))
    assert k == n - 3
    step_check(pools, 50, 10, "after")
    assert pools[0].pause_stats()["paused"] == 0 and pools[0].pause_stats()["resumed_alive"] + \
        pools[0].pause_stats()["resumed_suspect"] + pools[0].pause_stats()["resumed_dead"] == 1
    assert truth_rank(pools[0], 10)[0] == TRUTH_CRASHED and truth_rank(pools[0], 30)[0] == TRUTH_UP


def test_reaped_or_pruned_paused_members_stay_gone(make):
    n = 600
    cfg = lan_config(L, capacity=n, n_initial=n, seed=0x4EA9, reconnect_timeout_ns=2 * 10**9,
                     tombstone_timeout_ns=2 * 10**9, reap_interval_ns=10**9)
    pools = make(cfg)
    both(pools, lambda p: p.pause([1, 2, 3, 4], 1500))
    assert both(pools, lambda p: p.run_until(PRED_CRASHED_ALL_DEAD, 0, 1400, 10)) != NEVER
    both(pools, lambda p: p.force_leave(0, 2, True))     # pruned
    both(pools, lambda p: p.force_leave(0, 3, False))    # listed Left
    check(pools, "forced")
    assert all(p.paused_until(2) == NEVER and p.paused_until(3) == NEVER for p in pools)
    step_check(pools, 100, 10, "reaper")                 # 1 and 4 are reaped (Dead for > 2 s)
    assert pools[0].pause_stats()["paused"] == 0
    step_check(pools, 1500 - pools[0].now + 20, 100, "past the resume")
    st = pools[0].pause_stats()
    assert st == {"paused": 0, "resumed_alive": 0, "resumed_suspect": 0, "resumed_dead": 0}, st
    assert all(truth_rank(pools[0], i)[0] != TRUTH_UP for i in (1, 2, 3, 4))


def test_operations_on_a_paused_member_fail_and_leaving_members_are_skipped(make):
    n = 500
    pools = make(lan_config(L, capacity=n + 1, n_initial=n, seed=0x0B5))
    both(pools, lambda p: p.leave(8))
    assert both(pools, lambda p: p.pause([5, 8], 30)) == 1            # LEAVING: skipped
    assert both(pools, lambda p: p.pause([5, 6], 30)) == 1            # already paused: skipped
    for p in pools:
        for op in (lambda: p.leave(5), lambda: p.join(5, [0]), lambda: p.user_event(5, b"e", b"", False),
                   lambda: p.member_update(5, 40)):
            with pytest.raises(GsimError) as e:
                op()
            assert e.value.code == ERR_STATE
    step_check(pools, 120, 15, "leave and pause")                     # 8 leaves on schedule, 5 and 6 resume


def test_impaired_and_paused(make):
    n = 2000
    pools = make(lan_config(L, capacity=n, n_initial=n, seed=0x1B9A, disable_tcp_pings=1))
    for p in pools:
        p.impair(list(range(0, n, 9)), 500000)
    both(pools, lambda p: p.pause(list(range(0, n, 27)), 70))          # every one of them impaired too
    both(pools, lambda p: p.impair(list(range(0, n, 54)), 0, 0))       # cleared while paused
    step_check(pools, 200, 20, "impaired + paused")
    assert pools[0].pause_stats()["resumed_suspect"] > 0


def test_snapshot_restore_mid_pause(hostemu_lib):
    n = 2048
    cfg = wan_config(hostemu_lib, capacity=n, n_initial=n, seed=0x5A9, mailbox_depth=8, flags=FLAG_LOG_GLOBAL_EVENTS)
    p = Pool(cfg, hostemu_lib)
    p.latency_set(c5_latency_matrix(16))
    p.pause_fraction(20000, 3, 90)
    p.pause([1, 2, 3], 30)
    p.step(11)
    blob = p.snapshot()
    assert layout(blob) & LAYOUT_PAUSE
    pu = [p.paused_until(i) for i in range(0, n, 3)]
    assert any(u != NEVER for u in pu)
    p.step(120)
    h1, s1, ps1 = p.state_hash(), p.stats(), p.pause_stats()
    s1.pop("active_rows")
    q = Pool(cfg, hostemu_lib)                             # never paused: restore brings the column
    q.restore(blob)
    assert [q.paused_until(i) for i in range(0, n, 3)] == pu
    q.step(120)
    s2 = q.stats()
    s2.pop("active_rows")
    assert q.state_hash() == h1 and s2 == s1 and q.pause_stats() == ps1
    # a blob without the pause column restores a pool nobody in it is paused
    r = Pool(cfg, hostemu_lib)
    r.latency_set(c5_latency_matrix(16))
    plain = r.snapshot()
    assert not layout(plain) & LAYOUT_PAUSE
    r.step(30)
    q.restore(plain)
    q.step(30)
    assert q.state_hash() == r.state_hash() and q.paused_until(1) == NEVER and q.pause_stats()["paused"] == 0


def test_a_never_paused_pool_is_unchanged(hostemu_lib):
    n = 1000
    cfg = lan_config(hostemu_lib, capacity=n + 1, n_initial=n, seed=77)
    ref, a = Pool(cfg, hostemu_lib), Pool(cfg, hostemu_lib)
    assert a.pause([], 10) == 0                            # nothing to pause: nothing allocated
    assert a.snapshot() == ref.snapshot() and not layout(ref.snapshot()) & LAYOUT_PAUSE
    assert a.paused_until(3) == NEVER and a.pause_stats()["paused"] == 0
    for p in (ref, a):
        x = p.member_add()
        p.join(x, [0])
        p.step(100)
    assert a.state_hash() == ref.state_hash() and a.snapshot() == ref.snapshot()


def test_validation(make):
    for p in make(lan_config(L, capacity=300, n_initial=300, seed=1)):
        for bad, code in ((lambda: p.pause([1], 0), ERR_INVALID),
                          (lambda: p.pause([300], 5), ERR_NOT_FOUND),
                          (lambda: p.pause_fraction(1_000_001, 0, 5), ERR_INVALID),
                          (lambda: p.pause_fraction(1000, 0, 0), ERR_INVALID),
                          (lambda: p.pause([1], 0xFFFFFFFF), ERR_INVALID),
                          (lambda: p.paused_until(300), ERR_NOT_FOUND)):
            with pytest.raises(GsimError) as e:
                bad()
            assert e.value.code == code
        assert p.pause_stats()["paused"] == 0 and p.paused_until(1) == NEVER


def test_sharded_pools_refuse_pausing():
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", "29561",
           os.path.join(ROOT, "tests", "sharded_pause_worker_cpu.py")]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600, cwd=ROOT)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "PAUSE REFUSED" in r.stdout


# ---- fuzz --------------------------------------------------------------------------------------------
class _Pausing:
    """One pool of a fuzz pair: before every step it applies the pause operation the shared schedule
    (seed, current tick) picks, so both pools of the pair see the same operations (a snapshot, a few ticks
    and a restore on one of them leave the schedule in step)."""

    def __init__(self, pool, seed):
        self.pool, self.seed = pool, seed

    def __getattr__(self, name):
        return getattr(self.pool, name)

    def step(self, k=1):
        now = self.pool.now
        rng = random.Random(self.seed * 7919 + now)
        n = self.pool.stats()["n_members"]
        if n and rng.random() < 0.4:
            d = rng.choice([1, 2, 4, 9, 30, 150, 700])
            if rng.random() < 0.6:
                self.pool.pause(rng.sample(range(n), min(n, rng.choice([1, 2, 5, 20]))), d)
            else:
                self.pool.pause_fraction(rng.choice([5000, 100000]), now, d)
        self.pool.step(k)


@pytest.mark.parametrize("seed", range(8))
def test_fuzz_with_pauses(hostemu_lib, seed):
    def make(cfg):
        return [_Pausing(Pool(cfg, hostemu_lib), seed), _Pausing(PauseOraclePool(cfg), seed)]

    assert fuzz_ops.run_sequence(make, hostemu_lib, 0x9A050000 + seed, n_ops=40) == 40
