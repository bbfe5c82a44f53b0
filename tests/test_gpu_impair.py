"""Degraded members (gsim_impair_*) on the H100 against the oracle: digest and counters at
checkpoints and the exact convergence ticks, on the generic probe path the impairment selects and
back on the fast paths once it is cleared."""
import pytest

from consul_b200.pool import NEVER, PRED_CRASHED_ALL_DEAD, PRED_RUMOR_CONVERGED, Pool, lan_config, wan_config
from consul_b200.wan import c5_latency_matrix
from oracle_impair import ImpairOraclePool
from parity import compare_pools

pytestmark = pytest.mark.gpu


def both(pools, fn):
    a, b = [fn(p) for p in pools]
    assert a == b, (a, b)
    return a


def run_to(pools, checkpoints, where):
    for upto in checkpoints:
        for p in pools:
            p.step(upto - p.now)
        compare_pools(*pools, f"{where} tick {upto}", columns=False)


def test_1m_lan_one_percent_impaired(cuda_lib):
    n = 1 << 20
    cfg = lan_config(cuda_lib, capacity=n + 1, n_initial=n, seed=0x1A9A0001)
    pools = [Pool(cfg, cuda_lib), ImpairOraclePool(cfg, threads=0)]
    k = both(pools, lambda p: p.impair_fraction(10000, 1, 300000, 0))
    assert abs(k - n // 100) < 1000
    x = both(pools, lambda p: p.member_add())
    both(pools, lambda p: p.join(x, [0]))
    slot = both(pools, lambda p: p.user_event(3, b"deploy", bytes(32), False))
    run_to(pools, (8, 40), "1M LAN")
    t = both(pools, lambda p: p.run_until(PRED_RUMOR_CONVERGED, slot, 1000, 1))
    assert t != NEVER
    run_to(pools, (t + 100, 600, 1200, 2000), "1M LAN")
    s = pools[0].stats()
    assert s["packets_lost"] > 0 and s["deads"] == 0


def test_wan_c5_matrix_with_delays(cuda_lib):
    n = 64 * 128 * 16
    cfg = wan_config(cuda_lib, capacity=n, n_initial=n, seed=0x1A9A0002, mailbox_depth=8)
    pools = [Pool(cfg, cuda_lib), ImpairOraclePool(cfg, threads=0)]
    for p in pools:
        p.latency_set(c5_latency_matrix(64))              # extra latency up to 4 ticks
    both(pools, lambda p: p.impair_fraction(20000, 2, 100000, 2))
    slot = both(pools, lambda p: p.user_event(0, b"e", b"x" * 16, False))
    t = both(pools, lambda p: p.run_until(PRED_RUMOR_CONVERGED, slot, 2000, 1))
    assert t != NEVER
    run_to(pools, (t + 50, t + 400), "WAN")


def test_cleared_mid_run_windows_come_back(cuda_lib):
    n = 1 << 20
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0x1A9A0003)
    pools = [Pool(cfg, cuda_lib), ImpairOraclePool(cfg, threads=0)]
    ids = list(range(7, n, 997))
    for p in pools:
        p.impair(ids, 500000)
    run_to(pools, (300, 800), "impaired")
    before = pools[0].sched_counts()
    assert before["closed_form_launches"] == 0
    for p in pools:
        p.impair(ids, 0, 0)
    run_to(pools, (1500, 4000), "cleared")
    after = pools[0].sched_counts()
    assert after["closed_form_ticks"] > 1000, after


def test_c3_4m_crash_wave_plus_impaired(cuda_lib):
    """BASELINE config 3's size: 4 000 000 members, ~10 % crashed and ~1 % impaired at tick 0."""
    n = 4_000_000
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0x5EED0003)
    pools = [Pool(cfg, cuda_lib), ImpairOraclePool(cfg, threads=0)]
    crashed = both(pools, lambda p: p.crash_fraction(100000, 0))
    k = both(pools, lambda p: p.impair_fraction(10000, 0, 300000, 0))
    assert abs(crashed - n // 10) < 5000 and abs(k - (n - crashed) // 100) < 2000
    run_to(pools, (16, 64, 200, 300, 500, 900, 1400, 2000), "C3+impaired")
    t_dead = both(pools, lambda p: p.run_until(PRED_CRASHED_ALL_DEAD, 0, 0, 1))
    assert t_dead != NEVER
    s = pools[0].stats()
    assert s["deads"] == crashed and s["packets_lost"] > 0
