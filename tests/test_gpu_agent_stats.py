"""Per-agent serf Stats() and the health histogram on the H100 (DESIGN.md §3.8): the sm_90a kernels against
the restatement of tests/test_agent_stats_cpu.py over the device's own columns and rumor table, every field of
every agent, at pool sizes the host emulation cannot reach."""
import numpy as np
import pytest

from consul_b200.pool import NEVER, PRED_CRASHED_ALL_DEAD, Pool, lan_config
from test_agent_stats_cpu import check_agents, observables

pytestmark = pytest.mark.gpu


def test_1m_join_cascade_with_user_events(cuda_lib):
    n = 1 << 20
    p = Pool(lan_config(cuda_lib, capacity=n + 4, n_initial=n, seed=0xA6E10001), cuda_lib)
    x = p.member_add()
    assert p.join(x, [0]) == 1
    lone = p.member_add()                                      # never joins: isolated, pending
    y = p.member_add()
    assert p.join(y, [77]) == 1
    p.user_event(5, b"deploy", b"x" * 32, False)
    p.user_event(9, b"config", b"y" * 16, False)
    seen_partial = False
    for t in (0, 2, 6, 12, 24):
        p.step(t - p.now)
        before = observables(p)
        got = check_agents(p, p, f"1M cascade tick {t}", sample=(0, x, lone))
        assert observables(p) == before
        assert got["members"][lone] <= 3
        seen_partial = seen_partial or len(np.unique(got["members"][:n])) > 1
        if t == 0:
            assert got["event_queue"][5] == 1 and got["event_queue"][9] == 1 and got["intent_queue"][x] == 1
    assert seen_partial                                        # some agents listed a joiner others had not heard of


def test_4m_after_crash_wave_with_impaired(cuda_lib):
    n = 4 << 20
    p = Pool(lan_config(cuda_lib, capacity=n, n_initial=n, seed=0xA6E10002), cuda_lib)
    rng = np.random.default_rng(5)
    ids = rng.choice(n, n // 100, replace=False).astype(np.uint32)
    half = len(ids) // 2
    p.impair(ids[:half].tolist(), 300000, 0)                   # lossy both ways
    p.impair_dir(ids[half:].tolist(), 0, 1000000, 0, no_tcp=True)  # inbound blocked, no TCP fallback
    impaired = np.zeros(n, dtype=bool)
    impaired[ids] = True
    crashed = p.crash_fraction(100000, 3)
    assert crashed > 0
    t = p.run_until(PRED_CRASHED_ALL_DEAD, 0, 6000, 50)
    assert t != NEVER
    light = lambda: (p.state_hash(), p.stats(), p.sched_counts())  # (no 4M snapshot blob)
    before = light()
    got = check_agents(p, p, "4M after the crash wave", impaired=impaired, sample=(0,))
    assert light() == before
    assert (got["failed"] == crashed).all()
    h = p.health_histogram()
    assert h.sum() == n - crashed and h[1, 7] > 0
