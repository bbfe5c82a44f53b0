"""One-way reachability (gsim_impair_dir_*) on the H100 against the reach oracle: digest and counters at
checkpoints on inbound-blocked LAN pools and a WAN C5 pool with one-way loss and members without TCP; the
schedule against the host emulation; a snapshot round trip on the device; the selection at 16 Mi members."""
import pytest

import fuzz_ops
from backend_fuzz import Lockstep
from consul_b200.pool import FLAG_PUSH_PULL, Pool, lan_config, wan_config
from consul_b200.wan import c5_latency_matrix
from oracle_reach import ReachOraclePool
from parity import compare_pools
from test_reach_cpu import Directional

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


@pytest.mark.parametrize("tcp_fallback", [True, False])
def test_1m_lan_inbound_blocked(cuda_lib, tcp_fallback):
    n = 1 << 20
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0x4EAC0001, disable_tcp_pings=0 if tcp_fallback else 1)
    pools = [Pool(cfg, cuda_lib), ReachOraclePool(cfg, threads=0)]
    k = both(pools, lambda p: p.impair_dir_fraction(1000, 1, 0, FULL))
    assert abs(k - n // 1000) < 150
    slot = both(pools, lambda p: p.user_event(3, b"deploy", bytes(32), False))
    run_to(pools, (8, 40, 150, 300, 600), "1M LAN inbound blocked")
    s = pools[0].stats()
    assert s["deads"] == 0 and s["suspects"] == s["refutes"]
    assert (s["suspects"] == 0) == tcp_fallback, s
    heard = pools[0].column("heard")
    assert int((heard >> slot & 1).sum()) == n - k            # gossip reaches everyone but the blocked members


def test_256k_wan_c5_one_way_loss_and_no_tcp(cuda_lib):
    n = 1 << 18
    cfg = wan_config(cuda_lib, capacity=n, n_initial=n, seed=0x4EAC0002, mailbox_depth=8, flags=FLAG_PUSH_PULL,
                     push_pull_interval_ns=2_000_000_000)
    pools = [Pool(cfg, cuda_lib), ReachOraclePool(cfg, threads=0)]
    for p in pools:
        p.latency_set(c5_latency_matrix(64))
    both(pools, lambda p: p.impair_dir_fraction(20000, 2, 300000, 50000, 1))
    both(pools, lambda p: p.impair_dir_fraction(5000, 3, 0, 0, 0, True))
    slot = both(pools, lambda p: p.user_event(0, b"e", b"x" * 16, False))
    run_to(pools, (20, 100, 300, 600), "WAN C5")
    assert slot >= 0 and pools[0].stats()["push_pulls"] > 0


@pytest.mark.parametrize("seed", range(4))
def test_schedule_parity_with_the_host_emulation(cuda_lib, hostemu_lib, seed):
    pair = Lockstep(lambda c: Directional(Pool(c, cuda_lib)), lambda c: Directional(Pool(c, hostemu_lib)),
                    0x4EC0 + seed, extra=True, schedule=True)
    fuzz_ops.run_sequence(pair.make, cuda_lib, 0x4EC1000 + seed, n_ops=30)


def test_snapshot_round_trip_on_the_device(cuda_lib):
    n = 1 << 18
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0x4EAC0003, flags=FLAG_PUSH_PULL,
                     push_pull_interval_ns=2_000_000_000, mailbox_depth=4)
    p = Pool(cfg, cuda_lib)
    p.impair_dir_fraction(10000, 5, 0, FULL, 1)
    p.impair_dir_fraction(2000, 6, FULL, 0, 0, True)
    p.user_event(1, b"e", b"", False)
    p.step(33)
    blob = p.snapshot()
    p.step(200)
    h1, s1 = p.state_hash(), p.stats()
    q = Pool(cfg, cuda_lib)
    q.restore(blob)
    q.step(200)
    s2 = q.stats()
    for s in (s1, s2):
        s.pop("active_rows")
    assert q.state_hash() == h1 and s2 == s1
    ora = ReachOraclePool(cfg, threads=0)
    ora.impair_dir_fraction(10000, 5, 0, FULL, 1)
    ora.impair_dir_fraction(2000, 6, FULL, 0, 0, True)
    ora.user_event(1, b"e", b"", False)
    ora.step(233)
    compare_pools(q, ora, "restored vs oracle", columns=False)


def test_fraction_at_16m_members(cuda_lib):
    n = 1 << 24
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0x4EAC0004)
    a = Pool(cfg, cuda_lib)
    k = a.impair_dir_fraction(1000, 9, 0, FULL, 0, True)
    assert abs(k - n // 1000) < 600
    del a
    b = Pool(cfg, cuda_lib)
    assert b.impair_fraction(1000, 9, 1000) == k              # the same members: the same count
    sample = range(0, n, 4099)
    picked = [i for i in sample if b.impairment(i) != (0, 0)]
    c = Pool(cfg, cuda_lib)
    c.impair_dir_fraction(1000, 9, 0, FULL, 0, True)
    assert [i for i in sample if c.impairment_dir(i) != (0, 0, 0, False)] == picked
