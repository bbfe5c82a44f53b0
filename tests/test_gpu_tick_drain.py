"""The tick kernel's drain on the H100: members that need the generic row step are queued one entry each and
taken 32 at a time by whichever warp of the CTA is free, whatever tile or scanning warp they came from.
Which warp steps a member must not matter, so digests, counters and columns must equal the oracle's:

- pool sizes that are not a multiple of 32 (a tile's last group is partial) nor of the grid's split;
- capped grids (GSIM_GRID_MAX), which give each warp several rounds of tiles and so reuse the queue;
- per-member ticker phases (phase_group 1: no phase gate) and wide phase groups (phase_group 256);
- a WAN pool, whose gossip runs at every tick (GossipInterval = one tick);
- a pool with periodic push-pull, whose ticker puts members in the queue that have no mail."""
import pytest

from consul_b200.pool import FLAG_LOG_GLOBAL_EVENTS, FLAG_PUSH_PULL, Pool, lan_config, wan_config
from oracle_binding import OraclePool
from parity import compare_pools

pytestmark = pytest.mark.gpu


def both(pools, fn):
    a, b = [fn(p) for p in pools]
    assert a == b, (a, b)
    return a


def steps(pools, chunks, where):
    for c in chunks:
        for p in pools:
            p.step(c)
        compare_pools(*pools, f"{where} +{c} (tick {pools[0].now})")


def cascade(lib, make, n, extra=(), **kw):
    """a join cascade, a crash wave and its failure detection, compared with the oracle along the way; returns
    the CUDA pool's counters at the end"""
    cfg = make(lib, capacity=n + 8, n_initial=n, flags=FLAG_LOG_GLOBAL_EVENTS | kw.pop("flags", 0), **kw)
    pools = [Pool(cfg, lib), OraclePool(cfg)]
    try:
        steps(pools, (3,), "start")
        x = both(pools, lambda p: p.member_add())
        assert both(pools, lambda p: p.join(x, [0])) == 1
        steps(pools, (1, 2, 5, 9, 14, 30) + tuple(extra), "cascade")
        assert both(pools, lambda p: p.crash_fraction(20000, 7)) > 0
        steps(pools, (4, 40, 160), "crash wave")
        stats = pools[0].stats()
        assert stats["active_rows"] > 0
        return stats
    finally:
        for p in pools:
            p.close()


@pytest.mark.parametrize("n", [999, 20011])
@pytest.mark.parametrize("cap", [None, 1, 3])
def test_lan_cascade(cuda_lib, monkeypatch, n, cap):
    if cap is not None:
        monkeypatch.setenv("GSIM_GRID_MAX", str(cap))
    cascade(cuda_lib, lan_config, n, seed=0xD0A1 + n)


@pytest.mark.parametrize("phase_group", [1, 256])
@pytest.mark.parametrize("cap", [None, 2])
def test_phase_groups(cuda_lib, monkeypatch, phase_group, cap):
    if cap is not None:
        monkeypatch.setenv("GSIM_GRID_MAX", str(cap))
    cascade(cuda_lib, lan_config, 12345, seed=0xD0A2, phase_group=phase_group)


@pytest.mark.parametrize("cap", [None, 2])
def test_wan_gossip_every_tick(cuda_lib, monkeypatch, cap):
    if cap is not None:
        monkeypatch.setenv("GSIM_GRID_MAX", str(cap))
    stats = cascade(cuda_lib, wan_config, 7001, seed=0xD0A3, mailbox_depth=8)
    assert stats["gossip_interval_ticks"] == 1


@pytest.mark.parametrize("cap", [None, 3])
def test_push_pull(cuda_lib, monkeypatch, cap):
    if cap is not None:
        monkeypatch.setenv("GSIM_GRID_MAX", str(cap))
    cascade(cuda_lib, lan_config, 5003, extra=(200,), seed=0xD0A4, flags=FLAG_PUSH_PULL,
            push_pull_interval_ns=2_000_000_000)
