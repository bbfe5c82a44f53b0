"""Degraded members (gsim_impair_*) on the CPU: the kernel's row body (tests/hostemu) against the
oracle bit for bit — columns, counters, digest, convergence ticks — plus the properties the fault
model must have and Lifeguard's effect on false suspicion."""
import os
import random
import subprocess
import sys

import numpy as np
import pytest

import fuzz_ops
import scenarios as sc
from consul_b200.pool import (FLAG_COORDINATES, FLAG_NO_WINDOWS, FLAG_PUSH_PULL, NEVER, PRED_RUMOR_CONVERGED,
                              GsimError, Pool, lan_config, wan_config)
from consul_b200.wan import c5_latency_matrix
from oracle_impair import ImpairOraclePool
from parity import compare_pools

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ERR_INVALID, ERR_NOT_FOUND = -1, -5
RANK_DEAD = 2


def slow_matrix(n_dcs, worst):
    a = np.arange(n_dcs)[:, None]
    b = np.arange(n_dcs)[None, :]
    m = 1 + (3 * a + 5 * b) % worst
    m[np.arange(n_dcs), np.arange(n_dcs)] = 1
    return m.astype(np.uint8)


@pytest.fixture()
def make(hostemu_lib):
    return lambda cfg: [Pool(cfg, hostemu_lib), ImpairOraclePool(cfg)]


def both(pools, fn):
    return sc.both(pools, fn)


def test_loss_only_parity(make, hostemu_lib):
    n = 2048
    pools = make(lan_config(hostemu_lib, capacity=n + 1, n_initial=n, seed=0x1A11))
    bad = list(range(3, n, 97))
    for p in pools:
        p.impair(bad, 300000)
    x = both(pools, lambda p: p.member_add())
    both(pools, lambda p: p.join(x, [0]))
    slot = both(pools, lambda p: p.user_event(5, b"deploy", b"v1", False))
    sc.step_compare(pools, 300, 25, "loss only")
    t = both(pools, lambda p: p.run_until(PRED_RUMOR_CONVERGED, slot, 2000, 4))
    assert t != NEVER
    compare_pools(*pools, "converged")
    s = pools[0].stats()
    assert s["packets_lost"] > 0 and s["indirect_pings"] > 0
    assert all(p.impairment(bad[0]) == (300000, 0) for p in pools)


@pytest.mark.parametrize("matrix", [None, "slow"])
def test_delay_only_parity(make, hostemu_lib, matrix):
    """WAN pool with an 8-slot mailbox ring: receive delays alone, then on top of a slow matrix."""
    n = 16 * 128
    pools = make(wan_config(hostemu_lib, capacity=n + 1, n_initial=n, seed=0xDE1A, mailbox_depth=8))
    delay = 5
    if matrix:
        for p in pools:
            p.latency_set(slow_matrix(16, 3))               # extra latency up to 2 ticks
        delay = 4
    for p in pools:
        p.impair(list(range(0, n, 37)), 0, delay)
        p.impair(list(range(11, n, 53)), 0, 2)
    slot = both(pools, lambda p: p.user_event(1, b"e", b"p", False))
    sc.step_compare(pools, 200, 20, f"delay matrix={matrix}")
    t = both(pools, lambda p: p.run_until(PRED_RUMOR_CONVERGED, slot, 2000, 4))
    assert t != NEVER
    s = pools[0].stats()
    assert s["packets_lost"] == 0 and s["indirect_pings"] > 0   # slow acks go through the indirect stage
    compare_pools(*pools, "converged")


def test_loss_and_delay_on_a_graph(make, hostemu_lib):
    n = 600
    cfg = wan_config(hostemu_lib, capacity=n, n_initial=n, seed=0x6AF, mailbox_depth=4, phase_group=1)
    pools = make(cfg)
    rp, ci = fuzz_ops.random_graph(random.Random(5), n)
    for p in pools:
        p.graph_set(rp, ci)
        p.impair(list(range(0, n, 13)), 400000, 2)
    both(pools, lambda p: p.user_event(2, b"g", b"x", False))
    sc.step_compare(pools, 250, 25, "graph")
    assert pools[0].stats()["packets_lost"] > 0


def test_coordinates_see_the_delay(make, hostemu_lib):
    n = 512
    cfg = lan_config(hostemu_lib, capacity=n, n_initial=n, seed=0xC00, flags=FLAG_COORDINATES, mailbox_depth=8,
                     phase_group=1)
    pools = make(cfg)
    for p in pools:
        p.impair(list(range(0, n, 7)), 100000, 3)
    sc.step_compare(pools, 150, 30, "coordinates")
    for m in (0, 1, 7, 300):
        assert pools[0].coordinate(m) == pools[1].coordinate(m)
    # a delayed member's coordinate moves away from the origin further than on an unimpaired pool
    q = Pool(cfg, hostemu_lib)
    q.step(150)
    assert pools[0].coordinate(0) != q.coordinate(0)


def test_push_pull_parity(make, hostemu_lib):
    n = 1024
    cfg = lan_config(hostemu_lib, capacity=n + 1, n_initial=n, seed=0x9911, flags=FLAG_PUSH_PULL,
                     push_pull_interval_ns=2_000_000_000, mailbox_depth=4)
    pools = make(cfg)
    for p in pools:
        p.impair(list(range(1, n, 41)), 500000, 1)
    x = both(pools, lambda p: p.member_add())
    both(pools, lambda p: p.join(x, [3]))
    sc.step_compare(pools, 200, 25, "push-pull")
    assert pools[0].stats()["push_pulls"] > 0


def test_set_then_cleared_mid_run(make, hostemu_lib):
    """Impair, run, clear: the pool keeps matching the oracle, and afterwards its schedule is that of an
    unimpaired pool again (long windows, closed form)."""
    n = 3000
    pools = make(lan_config(hostemu_lib, capacity=n, n_initial=n, seed=0xC1EA))
    ids = list(range(5, n, 61))
    for p in pools:
        p.impair(ids, 600000)
    sc.step_compare(pools, 400, 100, "impaired")
    impaired = pools[0].sched_counts()
    assert impaired["closed_form_launches"] == 0
    for p in pools:
        p.impair(ids, 0, 0)
        assert p.impairment(ids[0]) == (0, 0)
    sc.step_compare(pools, 2500, 500, "cleared")
    after = pools[0].sched_counts()
    assert after["closed_form_launches"] > 0 and after["closed_form_ticks"] > 1000, after


def test_snapshot_restore_of_an_impaired_pool(hostemu_lib):
    n = 2048
    cfg = wan_config(hostemu_lib, capacity=n, n_initial=n, seed=0x5A9, mailbox_depth=8)
    p = Pool(cfg, hostemu_lib)
    p.latency_set(c5_latency_matrix(16))
    p.impair_fraction(20000, 3, 250000, 2)
    slot = p.user_event(1, b"a", b"b", False)
    p.step(11)
    blob = p.snapshot()
    p.step(60)
    h1, info1, s1 = p.state_hash(), p.rumor_info(slot), p.stats()
    s1.pop("active_rows")
    q = Pool(cfg, hostemu_lib)                             # never impaired: restore brings the columns
    q.restore(blob)
    assert [q.impairment(i) for i in range(0, n, 5)] == [p.impairment(i) for i in range(0, n, 5)]
    q.step(60)
    s2 = q.stats()
    s2.pop("active_rows")
    assert q.state_hash() == h1 and q.rumor_info(slot) == info1 and s2 == s1
    # a blob without impairment restores an unimpaired pool into one that has the columns
    r = Pool(cfg, hostemu_lib)
    r.latency_set(c5_latency_matrix(16))
    plain = r.snapshot()
    r.step(30)
    q.restore(plain)
    q.step(30)
    assert q.state_hash() == r.state_hash() and q.impairment(0) == (0, 0)


@pytest.mark.parametrize("order", ["1", "2"])
def test_row_order_does_not_matter(order):
    code = (
        "import sys; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
        "from consul_b200 import _lib\n"
        "from consul_b200.pool import Pool, wan_config\n"
        "L = _lib.load(%r)\n"
        "p = Pool(wan_config(L, capacity=2049, n_initial=2048, seed=31, mailbox_depth=8), L)\n"
        "p.impair_fraction(30000, 1, 500000, 3); x = p.member_add(); p.join(x, [1]); p.step(400)\n"
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


def _script(p):
    x = p.member_add()
    p.join(x, [4])
    p.user_event(7, b"e", b"p", False)
    p.crash_many([20, 21])
    p.step(400)


def test_clearing_is_the_plain_model(hostemu_lib):
    """impair(ids, 0, 0) on a fresh pool, or impair then clear before a tick, changes nothing: same digest,
    counters and snapshot as a pool that was never impaired (a never-impaired pool allocates no columns)."""
    n = 2000
    cfg = lan_config(hostemu_lib, capacity=n + 1, n_initial=n, seed=71, packet_loss_ppm=50000)
    ref, a, b = (Pool(cfg, hostemu_lib) for _ in range(3))
    a.impair(list(range(0, n, 3)), 0, 0)
    assert a.snapshot() == ref.snapshot()
    b.impair(list(range(0, n, 3)), 700000, 0)
    b.impair(list(range(0, n, 3)), 0, 0)
    for p in (ref, a, b):
        _script(p)
    for p in (a, b):
        assert p.state_hash() == ref.state_hash() and p.stats() == ref.stats()


def test_windows_match_single_ticks_on_an_impaired_pool(hostemu_lib):
    n = 3000
    pools = []
    for flags in (0, FLAG_NO_WINDOWS):
        p = Pool(lan_config(hostemu_lib, capacity=n + 1, n_initial=n, seed=72, flags=flags), hostemu_lib)
        p.impair_fraction(10000, 9, 300000, 0)
        p.step(500)
        _script(p)
        p.step(1500)
        pools.append(p)
    compare_pools(*pools, "windows vs single ticks")
    assert pools[0].sched_counts()["window_ticks"] > 100
    assert pools[1].sched_counts()["window_ticks"] == 0


def test_a_silent_member_is_suspected_refutes_and_never_dies(make, hostemu_lib):
    n = 1024
    pools = make(lan_config(hostemu_lib, capacity=n, n_initial=n, seed=0x5111, disable_tcp_pings=1))
    victim = 300
    for p in pools:
        p.impair([victim], 1_000_000)
    for k in range(12):
        sc.step_compare(pools, 50, 50, f"silent {k}")
        for p in pools:
            key = p.column("key")
            assert ((key[victim] >> 2) & 3) != RANK_DEAD
    s = pools[0].stats()
    assert s["suspects"] > 0 and s["refutes"] > 0 and s["deads"] == 0
    assert pools[0].column("meta")[victim] & 7 > 0      # its awareness (local health) went up


def test_receive_delay_only_ever_delays(hostemu_lib):
    n = 2048
    cfg = wan_config(hostemu_lib, capacity=n, n_initial=n, seed=0xD1, mailbox_depth=8)
    ticks = []
    for delay in (0, 2, 5):
        p = Pool(cfg, hostemu_lib)
        if delay:
            p.impair(list(range(0, n, 3)), 0, delay)
        slot = p.user_event(0, b"e", b"x", False)
        ticks.append(p.run_until(PRED_RUMOR_CONVERGED, slot, 3000, 1))
    assert NEVER not in ticks and ticks[0] <= ticks[1] <= ticks[2] and ticks[0] < ticks[2], ticks


def _false_suspicions(lib, seed, aw_max):
    n = 2000
    p = Pool(lan_config(lib, capacity=n, n_initial=n, seed=seed, awareness_max_multiplier=aw_max, disable_tcp_pings=1),
             lib)
    k = p.impair_fraction(20000, seed, 600000, 0)
    p.step(1500)
    s = p.stats()
    assert s["deads"] == 0 and s["n_crashed"] == 0
    return k, s["suspects"], s["refutes"]


def test_lifeguard_reduces_false_suspicion(hostemu_lib):
    """2 000 members, 2 % of them at 60 % loss, no TCP fallback, nobody crashed: every suspicion is false.
    Lifeguard's local health (awareness_max_multiplier 8) stretches a degraded prober's probe deadline, so
    it accuses healthy members less often than with awareness off (1).  Measured over 1 500 ticks on the
    host emulation (impaired members, then suspects = refutes with 8 / with 1):
      seed 1: 37 impaired, 2388 vs 4498
      seed 2: 35 impaired, 2245 vs 4230
      seed 3: 36 impaired, 2268 vs 4347"""
    for seed in (1, 2, 3):
        k8, sus8, ref8 = _false_suspicions(hostemu_lib, seed, 8)
        k1, sus1, ref1 = _false_suspicions(hostemu_lib, seed, 1)
        assert k8 == k1 > 0
        assert sus8 < sus1, (seed, sus8, sus1)


def test_impair_fraction_parity_and_independence(make, hostemu_lib):
    n = 5000
    pools = make(lan_config(hostemu_lib, capacity=n, n_initial=n, seed=0xF4))
    k = both(pools, lambda p: p.impair_fraction(100000, 7, 123456, 0))
    assert 350 < k < 650
    got = [i for i in range(n) if pools[0].impairment(i) != (0, 0)]
    assert len(got) == k and [pools[1].impairment(i) for i in got] == [(123456, 0)] * k
    # same salt, other purpose: the crash selection is a different set of members
    crashed = both(pools, lambda p: p.crash_fraction(100000, 7))
    key = pools[0].column("key")[:n]
    down = set(np.nonzero((key & 3) == 2)[0].tolist())
    assert len(down) == crashed and len(down & set(got)) < k // 2
    # crashed members are not selected again; the count only covers UP members
    k2 = both(pools, lambda p: p.impair_fraction(1_000_000, 8, 0, 0))
    assert k2 == n - crashed
    sc.step_compare(pools, 50, 50, "after fraction")


@pytest.mark.parametrize("ppm", [0, 1, 999, 250000, 999999, 1000000])
def test_impairment_reads_back_exactly(make, hostemu_lib, ppm):
    pools = make(wan_config(hostemu_lib, capacity=300, n_initial=300, seed=1, mailbox_depth=8))
    for p in pools:
        p.impair([17], ppm, 6)
        assert p.impairment(17) == (ppm, 6)
        assert p.impairment(18) == (0, 0)


def test_validation(make, hostemu_lib):
    for p in make(lan_config(hostemu_lib, capacity=300, n_initial=300, seed=1)):   # depth 2: no delay at all
        for bad, code in ((lambda: p.impair([1], 1_000_001), ERR_INVALID),
                          (lambda: p.impair([300], 1000), ERR_NOT_FOUND),
                          (lambda: p.impair([1], 0, 1), ERR_INVALID),
                          (lambda: p.impair_fraction(1_000_001, 0, 1000), ERR_INVALID),
                          (lambda: p.impair_fraction(1000, 0, 1_000_001), ERR_INVALID),
                          (lambda: p.impairment(300), ERR_NOT_FOUND)):
            with pytest.raises(GsimError) as e:
                bad()
            assert e.value.code == code
        p.impair([1], 1_000_000, 0)
    for p in make(wan_config(hostemu_lib, capacity=300, n_initial=300, seed=1, mailbox_depth=8)):
        p.latency_set(np.full((2, 2), 4, dtype=np.uint8))   # extra 3 of the 6 the ring allows
        with pytest.raises(GsimError) as e:
            p.impair([1], 0, 4)
        assert e.value.code == ERR_INVALID
        p.impair([1], 0, 3)
        with pytest.raises(GsimError) as e:                 # the matrix must leave room for the delay present
            p.latency_set(np.full((2, 2), 5, dtype=np.uint8))
        assert e.value.code == ERR_INVALID
        p.latency_set(np.full((2, 2), 4, dtype=np.uint8))
        p.impair([1], 0, 0)
        p.latency_set(np.full((2, 2), 7, dtype=np.uint8))   # nobody delayed any more


class _Impairing:
    """One pool of a fuzz pair: before every step it applies the impairment operation the shared schedule
    (seed, current tick) picks, so both pools of the pair see the same operations (a snapshot, a few
    ticks and a restore on one of them leave the schedule in step)."""

    def __init__(self, pool, seed, depth):
        self.pool, self.seed, self.depth, self.extra = pool, seed, depth, 0

    def __getattr__(self, name):
        return getattr(self.pool, name)

    def latency_set(self, lat):
        self.pool.latency_set(lat)
        self.extra = 0 if lat is None else int(np.asarray(lat).max()) - 1

    def step(self, k=1):
        now = self.pool.now
        rng = random.Random(self.seed * 7919 + now)
        n = self.pool.stats()["n_members"]
        room = max(0, self.depth - 2 - self.extra)
        if n and rng.random() < 0.5:
            loss, delay = rng.choice([0, 0, 100000, 600000, 1_000_000]), rng.randrange(room + 1)
            if rng.random() < 0.5:
                self.pool.impair(rng.sample(range(n), min(n, rng.choice([1, 3, 20]))), loss, delay)
            else:
                self.pool.impair_fraction(rng.choice([10000, 200000]), now, loss, delay)
        self.pool.step(k)


@pytest.mark.parametrize("seed", range(8))
def test_fuzz_with_impairment(hostemu_lib, seed):
    def make(cfg):
        depth = cfg.mailbox_depth or 2
        return [_Impairing(Pool(cfg, hostemu_lib), seed, depth), _Impairing(ImpairOraclePool(cfg), seed, depth)]

    assert fuzz_ops.run_sequence(make, hostemu_lib, 0x1A9A0000 + seed, n_ops=40) == 40
