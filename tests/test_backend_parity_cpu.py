"""The backend parity sequences (tests/backend_fuzz.py) on the host emulation: the same operations as the
GPU file runs — pools at the CUDA partition edges, joins with many seeds, crash / pause / impair over long
id lists, rumor bursts in front of a join, pauses and impairment together — against the pause oracle with
columns after every operation.  This checks the harness and the operations' semantics before any GPU time
is spent; and the schedule (gsim_sched_counts) must not depend on the order rows are stepped in."""
import random

import pytest

import fuzz_ops
from backend_fuzz import (GROWTH, SIZES, Lockstep, size_id, tick_blocks, tick_runs, window_batch_crosses_a_tile,
                          window_blocks)
from consul_b200.pool import FLAG_LOG_GLOBAL_EVENTS, Pool, lan_config
from oracle_pause import PauseOraclePool
from parity import compare_pools

ERR_STATE = -6


@pytest.mark.parametrize("size", SIZES + (GROWTH,), ids=size_id)
def test_sizes_against_the_oracle(hostemu_lib, size):
    n0, cap = (size, size + 24) if isinstance(size, int) else size
    seed = 0xBA0000 + n0
    pair = Lockstep(lambda c: Pool(c, hostemu_lib), PauseOraclePool, seed, size=(n0, cap), extra=True,
                    grow=3 if size == GROWTH else 0)
    assert fuzz_ops.run_sequence(pair.make, hostemu_lib, seed, n_ops=30) == 30
    if size == GROWTH:
        assert pair.max_n > 1024, "the pool did not grow from one CTA to two"


@pytest.mark.parametrize("seed", range(6))
def test_small_pools_with_long_argument_lists(hostemu_lib, seed):
    pair = Lockstep(lambda c: Pool(c, hostemu_lib), PauseOraclePool, seed, extra=True)
    assert fuzz_ops.run_sequence(pair.make, hostemu_lib, 0xBA1000 + seed, n_ops=40) == 40


def test_multi_seed_join_semantics(hostemu_lib):
    """Join(x, seeds): every seed occurrence that is a running member other than x merges both ways and
    counts once (duplicates included); ids past the members, x itself and members that are not running —
    crashed, paused — are skipped, as memberlist skips an address it cannot reach."""
    n = 300
    cfg = lan_config(hostemu_lib, capacity=n + 4, n_initial=n, seed=0x5EED5, flags=FLAG_LOG_GLOBAL_EVENTS)
    pools = [Pool(cfg, hostemu_lib), PauseOraclePool(cfg)]
    for p in pools:
        for s in range(28):                                 # 28 live rumor slots for the merges to carry
            p.user_event(10 + s, b"ev%d" % s, b"z" * s, False)
        p.crash_many([20, 21])
        p.pause([30, 31], 50)
        p.step(2)
    compare_pools(*pools, "setup")
    x = 5
    seeds = [20, 7, 7, x, 30, n, n + 3, 1 << 20, 8, 21, 31, 9] + list(range(100, 170))
    want = sum(1 for s in seeds if s < n and s != x and s not in (20, 21, 30, 31))
    assert [p.join(x, seeds, False) for p in pools] == [want, want]
    compare_pools(*pools, "after the join")
    # nothing reachable: no merge, no join intent, not an error
    assert [p.join(6, [20, n + 1, 6, 30], True) for p in pools] == [0, 0]
    compare_pools(*pools, "after a join with no reachable seed")
    # a paused joiner cannot join
    for p in pools:
        with pytest.raises(Exception) as e:
            p.join(30, [1])
        assert getattr(e.value, "code", None) == ERR_STATE
    for p in pools:
        p.step(60)
    compare_pools(*pools, "after 60 ticks")


def test_schedule_does_not_depend_on_row_order(hostemu_lib, monkeypatch):
    """The host emulation steps rows in reverse order with GSIM_HOSTEMU_ORDER=1; the same sequence must give
    the same state and the same schedule after every operation."""
    rng = random.Random(7)
    for k, size in enumerate((None, (1025, 1049), GROWTH, None)):
        seed = 0xBA2000 + k

        def reversed_rows(cfg):
            monkeypatch.setenv("GSIM_HOSTEMU_ORDER", "1")
            try:
                return Pool(cfg, hostemu_lib)
            finally:
                monkeypatch.delenv("GSIM_HOSTEMU_ORDER")

        pair = Lockstep(lambda c: Pool(c, hostemu_lib), reversed_rows, seed, size=size, extra=True, schedule=True,
                        grow=3 if size == GROWTH else 0)
        fuzz_ops.run_sequence(pair.make, hostemu_lib, seed, n_ops=30, calm=rng.random() < 0.5)


def test_capped_grid_partitions():
    """What GSIM_GRID_MAX makes of a 20 011-member pool (157 tiles, 628 groups of 32)"""
    n = 20011
    for cap in (1, 2):
        runs, rounds = tick_runs(n, tick_blocks(n, cap))
        assert rounds >= 3 and len(set(runs)) == 2, (cap, rounds, set(runs))
    # windows: runs of 79 groups per warp at one CTA cross tiles; 40 at two CTAs do not
    assert window_batch_crosses_a_tile(n, window_blocks(n, 1))
    assert not window_batch_crosses_a_tile(n, window_blocks(n, 2))
    runs, rounds = tick_runs(n, tick_blocks(n, 17))
    assert len(runs) == 136 and set(runs) == {1, 2} and rounds == 1
    assert window_batch_crosses_a_tile(n, window_blocks(n, 17))
    # the full grid (132 SMs x 4 CTAs) takes one tile per warp at most, and no batch crosses a tile
    assert tick_runs(n, tick_blocks(n, 528))[1] == 1 and not window_batch_crosses_a_tile(n, window_blocks(n, 528))
