"""Broadcasts piggybacked on probe traffic (GSIM_FLAG_PROBE_PIGGYBACK) on the H100 against the piggyback oracle
(tests/oracle_piggyback/piggyback.patch): digests and the piggyback counters at checkpoints of a user event at 1 Mi members, a join
cascade, a 4 M-member crash wave with loss and a WAN pool with delays and impaired members; and a quiet flagged
pool that still runs closed-form windows."""
import pytest

import piggyback_scenarios as ps
from consul_b200.pool import FLAG_PROBE_PIGGYBACK, Pool, lan_config
from oracle_piggyback import PiggybackOraclePool
from parity import compare_pools

pytestmark = pytest.mark.gpu


@pytest.fixture()
def make(cuda_lib):
    return lambda cfg: [Pool(cfg, cuda_lib), PiggybackOraclePool(cfg, threads=0)]


def check(pools, upto):
    compare_pools(*pools, f"tick {upto}", columns=False)
    ps.both(pools, lambda p: p.piggyback_stats())


def test_1m_lan_user_event(make, cuda_lib):
    pools, slot, t = ps.user_event(make, cuda_lib, 1 << 20, check)
    pg = pools[0].piggyback_stats()
    s = pools[0].stats()
    assert s["rumors_sent"] + pg["broadcasts"] == (1 << 20) * s["retransmit_limit"]


def test_join_cascade(make, cuda_lib):
    pools = ps.join_cascade(make, cuda_lib, 1 << 18, check)
    assert pools[0].piggyback_stats()["broadcasts"] > 0


def test_4m_crash_wave(make, cuda_lib):
    pools = ps.crash_wave(make, cuda_lib, 4_000_000, check, checkpoints=(10, 40, 120))
    assert pools[0].piggyback_stats()["owed_served"] > 0


def test_wan_c5_impaired(make, cuda_lib):
    ps.wan_impaired(make, cuda_lib, 64 * 128 * 8, check, push_pull=True)


def test_quiet_flagged_pool_runs_closed_form(cuda_lib):
    n = 1 << 20
    pools = [Pool(lan_config(cuda_lib, capacity=n, n_initial=n, seed=9, flags=f), cuda_lib)
             for f in (0, FLAG_PROBE_PIGGYBACK)]
    for p in pools:
        p.step(3000)
    assert pools[0].state_hash() == pools[1].state_hash()
    a, b = (p.sched_counts() for p in pools)
    assert b["closed_form_ticks"] > 2000 and b["closed_form_ticks"] == a["closed_form_ticks"], (a, b)
    assert pools[1].piggyback_stats()["owed_served"] == 0
