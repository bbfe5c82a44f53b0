"""Intermittent impairment (gsim_impair_flap_*) on the H100: digest and counters against the flap oracle on a
1 Mi LAN pool with flapping loss, a WAN C5 pool with flapping delay and the 4 M-member C3 crash wave with 1 %
flapping; a schedule that is always bad against the static impairment and one that is never bad against no
impairment at 1 Mi members; a device snapshot round trip; the whole state against the host emulation."""
import pytest

import fuzz_ops
import snapblob
from consul_b200.pool import (NEVER, PRED_CRASHED_ALL_DEAD, Pool, lan_config, wan_config)
from consul_b200.wan import c5_latency_matrix
from oracle_flap import FlapOraclePool
from parity import compare_pools
from test_flap_cpu import SCHEDULING, FlapLockstep, split_flap

pytestmark = pytest.mark.gpu
FULL = 1_000_000


def both(pools, fn):
    a, b = [fn(p) for p in pools]
    assert a == b, (a, b)
    return a


def run_to(pools, checkpoints, where):
    for upto in checkpoints:
        for p in pools:
            p.step(upto - p.now)
        compare_pools(*pools, f"{where} tick {upto}", columns=False)


def test_1m_lan_flapping_loss(cuda_lib):
    n = 1 << 20
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0xF1A90001, disable_tcp_pings=1)
    pools = [Pool(cfg, cuda_lib), FlapOraclePool(cfg, threads=0)]
    k = both(pools, lambda p: p.impair_fraction(10_000, 1, 500_000, 0))
    assert abs(k - n // 100) < 500
    assert both(pools, lambda p: p.impair_flap_fraction(10_000, 1, 50, 200_000)) == k
    both(pools, lambda p: p.user_event(3, b"deploy", bytes(32), False))
    run_to(pools, (10, 60, 200, 350, 500), "1M LAN flapping")
    s = pools[0].stats()
    assert s["suspects"] > 0 and s["deads"] == 0 and s["packets_lost"] > 0, s
    fs = pools[0].flap_stats()
    assert fs["scheduled"] == k and 0 < fs["bad"] < k


def test_wan_c5_flapping_delay(cuda_lib):
    n = 1 << 18
    cfg = wan_config(cuda_lib, capacity=n, n_initial=n, seed=0xF1A90002, mailbox_depth=8)
    pools = [Pool(cfg, cuda_lib), FlapOraclePool(cfg, threads=0)]
    for p in pools:
        p.latency_set(c5_latency_matrix(64))
    both(pools, lambda p: p.impair_fraction(20_000, 2, 100_000, 2))
    both(pools, lambda p: p.impair_flap_fraction(20_000, 2, 10, 400_000))
    both(pools, lambda p: p.user_event(0, b"e", b"x" * 16, False))
    run_to(pools, (20, 100, 300, 600), "WAN C5 flapping delay")


def test_c3_4m_crash_wave_with_flapping(cuda_lib):
    n = 4_000_000
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0xF1A90003)
    pools = [Pool(cfg, cuda_lib), FlapOraclePool(cfg, threads=0)]
    crashed = both(pools, lambda p: p.crash_fraction(100_000, 0))
    k = both(pools, lambda p: p.impair_fraction(10_000, 0, 300_000, 0))
    both(pools, lambda p: p.impair_flap_fraction(10_000, 0, 20, 300_000))
    assert abs(crashed - n // 10) < 5000 and abs(k - (n - crashed) // 100) < 2000
    run_to(pools, (16, 64, 200, 500, 900, 1400, 2000), "C3+flapping")
    t_dead = both(pools, lambda p: p.run_until(PRED_CRASHED_ALL_DEAD, 0, 0, 1))
    assert t_dead != NEVER
    s = pools[0].stats()
    assert s["deads"] == crashed and s["packets_lost"] > 0


def _pair(cuda_lib, seed):
    n = 1 << 20
    # a ring of 4 arrival slots, so that a receive delay of 1 fits (gsim_impair_*)
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=seed, disable_tcp_pings=1, mailbox_depth=4)
    a, b = Pool(cfg, cuda_lib), Pool(cfg, cuda_lib)
    for p in (a, b):
        p.user_event(2, b"e", b"", False)
    return a, b


def test_always_bad_is_the_static_impairment_at_1m(cuda_lib):
    a, b = _pair(cuda_lib, 0xF1A90004)
    for p in (a, b):
        p.impair_dir_fraction(10_000, 4, 400_000, 300_000, 1, True)
    a.impair_flap_fraction(10_000, 4, 13, FULL)
    for upto in (5, 40, 150, 300):
        for p in (a, b):
            p.step(upto - p.now)
        compare_pools(a, b, f"always bad tick {upto}", columns=False)
    blob, col = split_flap(a.snapshot())
    assert blob == b.snapshot() and col.any()


def test_never_bad_is_no_impairment_at_1m(cuda_lib):
    a, b = _pair(cuda_lib, 0xF1A90005)
    a.impair_dir_fraction(10_000, 5, 400_000, 300_000, 1, True)
    a.impair_flap_fraction(10_000, 5, 13, 0)
    for upto in (5, 40, 150, 300):
        for p in (a, b):
            p.step(upto - p.now)
        assert a.state_hash() == b.state_hash(), upto
        sa, sb = a.stats(), b.stats()
        for f in SCHEDULING:
            sa.pop(f), sb.pop(f)
        assert sa == sb, upto


def test_snapshot_round_trip_on_the_device(cuda_lib):
    n = 1 << 18
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0xF1A90006, disable_tcp_pings=1, mailbox_depth=4)

    def setup(p):
        p.impair_fraction(20_000, 6, 600_000, 1)
        p.impair_flap_fraction(20_000, 6, 29, 300_000)
        p.user_event(1, b"e", b"", False)

    p = Pool(cfg, cuda_lib)
    setup(p)
    p.step(43)
    blob = p.snapshot()
    p.step(200)
    h1, s1 = p.state_hash(), p.stats()
    q = Pool(cfg, cuda_lib)
    q.restore(blob)
    assert q.flap_stats()["scheduled"] > 0
    q.step(200)
    s2 = q.stats()
    for s in (s1, s2):
        s.pop("active_rows")
    assert q.state_hash() == h1 and s2 == s1
    ora = FlapOraclePool(cfg, threads=0)
    setup(ora)
    ora.step(243)
    compare_pools(q, ora, "restored vs oracle", columns=False)


@pytest.mark.parametrize("seed", range(3))
def test_whole_state_against_the_host_emulation(cuda_lib, hostemu_lib, seed):
    """Fuzzed schedules on the device and in the host emulation, the whole state compared after every
    operation (the snapshots in canonical form, tests/snapblob.py, with the schedule column compared raw)."""

    class Compared(FlapLockstep):
        def step(self, side, k):
            super().step(side, k)
            if side.index == 1:
                a, b = (s.pool for s in self.sides)
                (ba, ca), (bb, cb) = split_flap(a.snapshot()), split_flap(b.snapshot())
                snapblob.assert_same(ba, bb, f"seed {self.seed} tick {a.now}")
                assert (ca is None) == (cb is None) and (ca is None or (ca == cb).all())

        def make(self, cfg):
            self.sides = super().make(cfg)
            return self.sides

    pair = Compared(lambda c: Pool(c, cuda_lib), lambda c: Pool(c, hostemu_lib), 0xF1C0 + seed, extra=True,
                    schedule=True)
    fuzz_ops.run_sequence(pair.make, cuda_lib, 0xF1C1000 + seed, n_ops=30)
