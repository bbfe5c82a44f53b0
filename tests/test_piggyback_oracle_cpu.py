"""Broadcasts piggybacked on probe traffic (GSIM_FLAG_PROBE_PIGGYBACK) against independent restatements: the
kernel's row body (host emulation) against the piggyback oracle (tests/oracle_piggyback/piggyback.patch), digest,
counters and every column; and the piggyback oracle against the full-fidelity model M0 with piggyback on."""
import os
import statistics
import sys

import pytest

import piggyback_scenarios as ps
from consul_b200.pool import (FLAG_PROBE_PIGGYBACK, NEVER, PRED_RUMOR_CONVERGED, GsimError, Pool, lan_config)
from oracle_piggyback import PiggybackOraclePool
from parity import compare_pools

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle"))
import m0_memberlist as m0  # noqa: E402


@pytest.fixture()
def make(hostemu_lib):
    return lambda cfg: [Pool(cfg, hostemu_lib), PiggybackOraclePool(cfg)]


def check(pools, upto):
    compare_pools(*pools, f"tick {upto}", columns=True)
    ps.both(pools, lambda p: p.piggyback_stats())


@pytest.mark.parametrize("seed", [0x5EED0003, 7, 8])
def test_user_event(make, hostemu_lib, seed):
    pools, slot, t = ps.user_event(make, hostemu_lib, 600, check, seed=seed)
    assert pools[0].piggyback_stats()["broadcasts"] > 0


def test_user_event_with_loss(make, hostemu_lib):
    ps.user_event(make, hostemu_lib, 800, check, seed=5, packet_loss_ppm=100000)


@pytest.mark.parametrize("seed", [0x5EED0001, 3])
def test_join_cascade(make, hostemu_lib, seed):
    pools = ps.join_cascade(make, hostemu_lib, 700, check, seed=seed)
    assert pools[0].piggyback_stats()["owed_served"] > 0


@pytest.mark.parametrize("seed", [0x5EED0002, 4])
def test_crash_wave_indirect_probes_and_nacks(make, hostemu_lib, seed):
    pools = ps.crash_wave(make, hostemu_lib, 700, check, seed=seed)
    s = pools[0].stats()
    assert s["nacks"] > 0 and s["indirect_pings"] > 0


def test_wan_c5_delays_impaired_one_way_push_pull(make, hostemu_lib):
    ps.wan_impaired(make, hostemu_lib, 16 * 128, check, push_pull=True, max_ticks=200)


def test_pool_loss_and_crashes_between_ticks(make, hostemu_lib):
    """Members crash while their queues are full and probes owe them answers: the gate and the owed answers of
    members that stopped running."""
    n = 500
    pools = make(lan_config(hostemu_lib, capacity=n, n_initial=n, seed=12, flags=FLAG_PROBE_PIGGYBACK,
                            packet_loss_ppm=30000))
    ps.both(pools, lambda p: p.user_event(0, b"a", b"x" * 20, False))
    ps.run_to(pools, (3, 4), check)
    for p in pools:
        p.crash_many(list(range(10, n, 17)))
    ps.run_to(pools, (5, 6, 9, 30, 120), check)


def test_backlog_overflow(make, hostemu_lib):
    pools = make(lan_config(hostemu_lib, capacity=24, n_initial=24, seed=77, flags=FLAG_PROBE_PIGGYBACK,
                            retransmit_mult=4, indirect_checks=8))
    for p in pools:
        p.crash_many(list(range(1, 24, 3)))
    for k in range(10):
        ps.both(pools, lambda p: p.user_event(0, b"e%d" % k, b"x", False))
        ps.run_to(pools, (pools[0].now + 10,), check)
    assert pools[0].piggyback_stats()["owed_dropped"] > 0


@pytest.mark.parametrize("seed", [21, 22, 23, 24])
def test_fuzzed_operations(hostemu_lib, seed):
    """The backend fuzz's operation sequences (joins, leaves, crashes, events, injections, retirements, WAN
    matrices, loss, push-pull, coordinates, snapshots of the kernel side) with the flag, kernel body against the
    piggyback oracle after every operation."""
    import fuzz_ops

    def mk(cfg):
        cfg.flags |= FLAG_PROBE_PIGGYBACK
        return [Pool(cfg, hostemu_lib), PiggybackOraclePool(cfg)]
    fuzz_ops.run_sequence(mk, hostemu_lib, seed, n_ops=50)


def test_sharded_pools_refuse_the_flag(hostemu_lib):
    cfg = lan_config(hostemu_lib, capacity=256, n_initial=256, seed=1, flags=FLAG_PROBE_PIGGYBACK, world_size=2,
                     rank=0)
    with pytest.raises(GsimError) as e:
        Pool(cfg, hostemu_lib)
    assert e.value.code == -1  # GSIM_ERR_INVALID


# ---- M0 cross-check ---------------------------------------------------------------------------------------
# M0 and M1 draw differently, so only means over seeds can agree.  The scenario is the one of
# test_m0_crosscheck.py::test_piggyback_on_probe_traffic_shifts_dissemination_by_about_one_tick: a converged
# cluster, 7 ticks, a user event from member 3, ticks until everybody has it, then the drained queues.
SHARE_TOL = 0.03   # absolute, on the share of all transmissions that rode on probe traffic
TICKS_TOL = 1.0    # on the mean ticks to everybody
# on the shift the flag causes: a difference of two differences of 8-seed means, each with a per-seed spread of
# about a tick; measured 1.12 ticks at 200 agents (M0 0.62, oracle 1.75) and 0.38 at 400 (M0 1.38, oracle 1.00)
SHIFT_TOL = 1.25


def _m0(n, piggy):
    ticks, share = [], []
    for seed in range(1, 9):
        net = m0.Network(m0.Config(piggyback=piggy), seed=seed)
        net.converged_cluster(n)
        net.step(7)
        key = net.user_event(3, b"deploy", b"x" * 8)
        t0 = net.now
        t = net.first_tick(lambda: all(any(k == key for _, k in a.delivered) for a in net.up_agents()), 400)
        assert t is not None
        net.step(80)
        ticks.append(t - t0)
        share.append(net.stats["piggyback_msgs"] / (net.stats["msgs"] + net.stats["piggyback_msgs"]))
    return statistics.mean(ticks), statistics.mean(share)


def _m1(n, flags):
    ticks, share = [], []
    for seed in range(1, 9):
        p = PiggybackOraclePool(lan_config(capacity=n, n_initial=n, seed=seed, flags=flags))
        p.step(7)
        slot = p.user_event(3, b"deploy", b"x" * 8, False)
        t = p.run_until(PRED_RUMOR_CONVERGED, slot, 400, 1)
        assert t != NEVER
        p.step(80)
        ticks.append(t - 7)
        s = p.stats()
        pig = p.piggyback_stats()["broadcasts"] if flags else 0
        assert s["rumors_sent"] + pig == n * s["retransmit_limit"]      # budget conserved
        share.append(pig / (s["rumors_sent"] + pig))
    return statistics.mean(ticks), statistics.mean(share)


@pytest.mark.parametrize("n", [200, 400])
def test_m0_crosscheck(n):
    """The piggyback oracle against M0 with piggyback on: the share of transmissions that ride on probe traffic
    within SHARE_TOL, the mean ticks until everybody has the event within TICKS_TOL, and the flag shortens both
    models' dissemination by amounts within SHIFT_TOL of each other."""
    m0_plain, _ = _m0(n, False)
    m0_pig, m0_share = _m0(n, True)
    m1_plain, _ = _m1(n, 0)
    m1_pig, m1_share = _m1(n, FLAG_PROBE_PIGGYBACK)
    info = dict(m0=(m0_plain, m0_pig, m0_share), m1=(m1_plain, m1_pig, m1_share))
    assert abs(m1_share - m0_share) <= SHARE_TOL, info
    assert abs(m1_pig - m0_pig) <= TICKS_TOL, info
    assert m0_pig < m0_plain and m1_pig < m1_plain, info
    assert abs((m1_plain - m1_pig) - (m0_plain - m0_pig)) <= SHIFT_TOL, info
