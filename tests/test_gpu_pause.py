"""Paused members (gsim_pause_*) on the H100 against the pause oracle: digest, counters and pause
statistics at checkpoints before, at and after the resume, then until the pool is quiet again."""
import pytest

from consul_b200.pool import FLAG_LOG_GLOBAL_EVENTS, NEVER, PRED_RUMOR_CONVERGED, Pool, lan_config, wan_config
from consul_b200.wan import c5_latency_matrix
from oracle_pause import PauseOraclePool
from parity import compare_pools

pytestmark = pytest.mark.gpu


def both(pools, fn):
    a, b = [fn(p) for p in pools]
    assert a == b, (a, b)
    return a


def run_to(pools, checkpoints, where, sample=()):
    for upto in checkpoints:
        for p in pools:
            p.step(upto - p.now)
        compare_pools(*pools, f"{where} tick {upto}", columns=False)
        assert pools[0].pause_stats() == pools[1].pause_stats(), f"{where} tick {upto}"
        assert [pools[0].paused_until(i) for i in sample] == [pools[1].paused_until(i) for i in sample]


def events(p):
    return sorted((e.tick, e.type, e.subject, e.observer) for e in p.poll_events())


def test_1m_lan_one_percent_paused_for_400_ticks(cuda_lib):
    n = 1 << 20
    cfg = lan_config(cuda_lib, capacity=n + 1, n_initial=n, seed=0x9A050001, flags=FLAG_LOG_GLOBAL_EVENTS)
    pools = [Pool(cfg, cuda_lib), PauseOraclePool(cfg, threads=0)]
    k = both(pools, lambda p: p.pause_fraction(10000, 1, 400))
    assert abs(k - n // 100) < 1000
    x = both(pools, lambda p: p.member_add())
    both(pools, lambda p: p.join(x, [0]))
    slot = both(pools, lambda p: p.user_event(3, b"deploy", bytes(32), False))
    sample = list(range(0, n, 4099))
    run_to(pools, (8, 40, 200, 399, 400, 401, 420), "1M LAN paused", sample)
    st = pools[0].pause_stats()
    assert st["paused"] == 0 and st["resumed_alive"] + st["resumed_suspect"] + st["resumed_dead"] == k
    assert st["resumed_dead"] > 0        # 400 ticks is past the suspicion timeout with confirmations (241)
    run_to(pools, (800, 1500, 2500), "1M LAN resumed")
    assert both(pools, lambda p: p.run_until(PRED_RUMOR_CONVERGED, slot, 0, 1)) != NEVER
    assert both(pools, events)
    assert pools[0].stats()["n_crashed"] == 0


def test_wan_c5_mixed_pause_lengths(cuda_lib):
    n = 64 * 128 * 16
    cfg = wan_config(cuda_lib, capacity=n, n_initial=n, seed=0x9A050002, mailbox_depth=8)
    pools = [Pool(cfg, cuda_lib), PauseOraclePool(cfg, threads=0)]
    for p in pools:
        p.latency_set(c5_latency_matrix(64))
    for ids, d in ((range(5, n, 301), 3), (range(9, n, 503), 40), (range(13, n, 709), 700)):
        both(pools, lambda p: p.pause(list(ids), d))
    slot = both(pools, lambda p: p.user_event(0, b"e", b"x" * 16, False))
    run_to(pools, (3, 4, 40, 41, 300, 700, 701, 900), "WAN", list(range(0, n, 97)))
    assert both(pools, lambda p: p.run_until(PRED_RUMOR_CONVERGED, slot, 2000, 1)) != NEVER


def test_snapshot_round_trip_mid_pause(cuda_lib):
    n = 1 << 20
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0x9A050003)
    p = Pool(cfg, cuda_lib)
    p.pause_fraction(10000, 2, 300)
    p.step(100)
    blob = p.snapshot()
    p.step(400)
    h1, ps1 = p.state_hash(), p.pause_stats()
    q = Pool(cfg, cuda_lib)
    q.restore(blob)
    assert q.pause_stats()["paused"] > 0
    q.step(400)
    assert q.state_hash() == h1 and q.pause_stats() == ps1
    ora = PauseOraclePool(cfg, threads=0)
    ora.pause_fraction(10000, 2, 300)
    ora.step(500)
    assert ora.state_hash() == h1 and ora.pause_stats() == ps1


def test_c3_4m_one_percent_paused_past_the_suspicion_timeout(cuda_lib):
    """BASELINE config 3's size: 4 000 000 members, ~1 % paused for 1 700 ticks (the suspicion timeout is
    265 ticks with every confirmation and 1 585 without any)."""
    n = 4_000_000
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0x5EED0003)
    pools = [Pool(cfg, cuda_lib), PauseOraclePool(cfg, threads=0)]
    k = both(pools, lambda p: p.pause_fraction(10000, 0, 1700))
    assert abs(k - n // 100) < 2000
    run_to(pools, (64, 300, 900, 1699, 1700, 1701, 1800, 2200), "C3 paused")
    st = both(pools, lambda p: p.pause_stats())
    assert st["paused"] == 0 and st["resumed_dead"] == k, st
