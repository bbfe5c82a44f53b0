"""Shared bodies of the backend parity tests (test_backend_parity_cpu.py on the host emulation,
test_gpu_backend_parity.py on the H100): a pair of pools that fuzz_ops.run_sequence drives in lock step,
with pauses, impairment and operations with long argument lists slipped in front of every step; the pool
sizes at the CUDA kernels' partition edges; the schedule comparison; and the arithmetic of how the tick and
window kernels split a pool over their grid."""
from __future__ import annotations

import random

import numpy as np

from consul_b200.pool import GsimError

# n_initial at the edges of a tile (128 members), of one CTA of the tick kernel (8 warps, a tile each:
# 1 024 members), and 20 011 members = 157 tiles, which a capped grid splits unevenly (GSIM_GRID_MAX)
SIZES = (127, 128, 129, 1023, 1025, 5000, 20011)
# a pool that grows from one CTA to two mid-run: new tick, stretch and window graphs
GROWTH = (1020, 1060)

# gsim_sched_counts fields that count ticks or decisions: the same operations must give the same schedule
# on every backend and in every row order.  (window_ms / tick_ms are times.)
SCHEDULE_FIELDS = ("window_launches", "window_ticks", "tick_launches", "horizon_scans", "closed_form_launches",
                   "closed_form_ticks")

TILE, WARPS, ROUND = 128, 8, 4  # gs_core.h GS_TILE; gs_cuda.cu GS_BLOCK / 32 and GS_ROUND


def size_id(size):
    """pytest id of an entry of SIZES + (GROWTH,)"""
    return str(size) if isinstance(size, int) else "x".join(map(str, size))


def schedule(pool):
    c = pool.sched_counts()
    return {k: c[k] for k in SCHEDULE_FIELDS}


def check_schedule(a, b, where=""):
    sa, sb = schedule(a), schedule(b)
    diffs = {k: (sa[k], sb[k]) for k in SCHEDULE_FIELDS if sa[k] != sb[k]}
    assert not diffs, f"schedule differs {where}: {diffs}"


# ---- the operations slipped in front of a step ------------------------------------------------------
# The pause and impairment schedules are those of the pause and impairment CPU fuzz tests.
def pause_op(do, rng: random.Random, n: int, now: int):
    if n and rng.random() < 0.4:
        d = rng.choice([1, 2, 4, 9, 30, 150, 700])
        if rng.random() < 0.6:
            ids = rng.sample(range(n), min(n, rng.choice([1, 2, 5, 20])))
            do("pause", lambda p: p.pause(ids, d))
        else:
            ppm = rng.choice([5000, 100000])
            do("pause_fraction", lambda p: p.pause_fraction(ppm, now, d))


def impair_op(do, rng: random.Random, n: int, now: int, room: int):
    """delays stay within `room` ticks"""
    if n and rng.random() < 0.5:
        loss, delay = rng.choice([0, 0, 100000, 600000, 1_000_000]), rng.randrange(room + 1)
        if rng.random() < 0.5:
            ids = rng.sample(range(n), min(n, rng.choice([1, 3, 20])))
            do("impair", lambda p: p.impair(ids, loss, delay))
        else:
            ppm = rng.choice([10000, 200000])
            do("impair_fraction", lambda p: p.impair_fraction(ppm, now, loss, delay))


def extra_op(do, rng: random.Random, n: int, room: int):
    """One of the operations with long argument lists, on a pool of n > 0 members."""
    kind = rng.random()
    if kind < 0.3:
        # Join with many seeds: 62..65 distinct rows besides the joiner straddle the 64 rows one device
        # gather takes.  Duplicates, the joiner itself and ids >= n are skipped, crashed or paused seeds too.
        x = rng.randrange(n)
        seeds = rng.sample(range(n), min(n, rng.choice([1, 3, 8, 62, 63, 64, 65, 150])))
        seeds += [rng.choice(seeds) for _ in range(rng.choice([0, 1, 5]))]
        if rng.random() < 0.5:
            seeds.append(x)
        if rng.random() < 0.5:
            seeds.append(n + rng.randrange(3))
        rng.shuffle(seeds)
        ig = rng.random() < 0.5
        do(f"join {x} <- {len(seeds)} seeds", lambda p: p.join(x, seeds, ig))
    elif kind < 0.55:
        # crash_many / pause / impair over 300..3000 ids drawn from a few members: many duplicates
        some = rng.sample(range(n), max(1, min(n, rng.choice([n // 50, n // 10, 40]))))
        ids = [rng.choice(some) for _ in range(rng.randint(300, 3000))]
        what = rng.choice(["crash", "pause", "impair"])
        if what == "crash":
            do(f"crash_many {len(ids)} ids", lambda p: p.crash_many(ids))
        elif what == "pause":
            d = rng.choice([2, 30, 300])
            do(f"pause {len(ids)} ids", lambda p: p.pause(ids, d))
        else:
            loss, delay = rng.choice([0, 200000, 1_000_000]), rng.randrange(room + 1)
            do(f"impair {len(ids)} ids", lambda p: p.impair(ids, loss, delay))
    elif kind < 0.8:
        # a burst of user events, then a join whose merges carry them all: more device writes than one
        # write batch holds, so it is flushed in the middle of the join
        for e in range(rng.randint(20, 28)):
            m = rng.randrange(n)
            do(f"burst event {m}", lambda p: p.user_event(m, b"b%d" % e, b"y" * (e % 9), False))
        x = rng.randrange(n)
        seeds = rng.sample(range(n), min(n, rng.choice([1, 3, 8])))
        do(f"join {x} <- {len(seeds)} seeds after a burst", lambda p: p.join(x, seeds, False))
    else:
        for _ in range(rng.randint(1, 8)):                 # growth (across a CTA boundary where sized so)
            do("add", lambda p: p.member_add())


class _Side:
    """One pool of a Lockstep pair, as fuzz_ops.run_sequence sees it."""

    def __init__(self, pool, pair, index):
        self.pool, self.pair, self.index = pool, pair, index

    def __getattr__(self, name):
        return getattr(self.pool, name)

    def latency_set(self, lat):
        self.pool.latency_set(lat)
        self.pair.extra_latency = 0 if lat is None else int(np.asarray(lat).max()) - 1

    def step(self, k=1):
        self.pair.step(self, k)


class Lockstep:
    """Two pools that fuzz_ops.run_sequence drives alike.  In front of every step each pool takes the
    operations drawn for (seed, current tick): a pause, an impairment (`disturb`) and one operation with a long
    argument list (`extra`), each from its own random stream so that their decisions are not correlated;
    and `grow` new members while the capacity leaves room for the fuzz's own.
    Both pools must return the same results and fail alike, and with `schedule` their step must add the same
    amounts to the schedule counters.  Keying the draws on the tick keeps the pools in step when
    run_sequence snapshots one pool, runs it a few ticks and restores it: the restore undoes those
    operations, and the counters, which are not pool state, are compared per step."""

    PAUSE, IMPAIR, EXTRA = 0, 0x1A9A, 0xE7A

    def __init__(self, make_a, make_b, seed, size=None, disturb=True, extra=False, schedule=False, grow=0):
        self.makers, self.seed, self.size = (make_a, make_b), seed, size
        self.disturb, self.extra, self.schedule, self.grow = disturb, extra, schedule, grow
        self.depth, self.capacity, self.extra_latency, self.max_n = 2, 0, 0, 0
        self.record = {}

    def make(self, cfg):
        """run_sequence's `make`: `size` = (n_initial, capacity) replaces the drawn size"""
        if self.size is not None:
            cfg.n_initial, cfg.capacity = self.size
        self.depth, self.capacity = cfg.mailbox_depth or 2, cfg.capacity
        return [_Side(m(cfg), self, i) for i, m in enumerate(self.makers)]

    def _rng(self, stream, now):
        return random.Random(((self.seed + stream) << 20) + now)

    def step(self, side, k):
        p = side.pool
        now, n = p.now, p.stats()["n_members"]
        self.max_n = max(self.max_n, n)
        results = []

        def do(what, fn):
            try:
                results.append((what, "ok", fn(p)))
            except GsimError as e:
                results.append((what, "err", e.code))

        room = max(0, self.depth - 2 - self.extra_latency)
        if n + self.grow <= self.capacity - 8:
            for _ in range(self.grow):
                do("grow", lambda q: q.member_add())
        if self.disturb:
            pause_op(do, self._rng(self.PAUSE, now), n, now)
            impair_op(do, self._rng(self.IMPAIR, now), n, now, room)
        rng = self._rng(self.EXTRA, now)
        if self.extra and n and rng.random() < 0.5:
            extra_op(do, rng, n, room)
        before = schedule(p) if self.schedule else None
        p.step(k)
        inc = {f: v - before[f] for f, v in schedule(p).items()} if self.schedule else None
        # the first pool's latest step from this tick (a snapshot's few ticks are overwritten by the real step)
        if side.index == 0:
            self.record[now] = (k, results, inc)
            return
        mine, theirs = (k, results, inc), self.record.get(now)
        where = f"seed {self.seed}: step {k} at tick {now}"
        assert theirs is not None, f"{where}: the first pool did not step from this tick"
        assert mine[1] == theirs[1], f"{where}: operations differ\n{theirs[1]}\n{mine[1]}"
        assert mine == theirs, f"{where}: schedule differs: {theirs[2]} vs {mine[2]}"


# ---- how the kernels split a single-GPU pool (gs_cuda.cu) -----------------------------------------
def tick_blocks(n: int, grid: int) -> int:
    """CudaBackend::tick_blocks: a warp per tile up to the grid"""
    return min(((n + TILE - 1) // TILE + WARPS - 1) // WARPS, grid)


def tick_runs(n: int, blocks: int):
    """gs_tick_kernel: tiles per warp (contiguous floor / ceil runs) and the rounds of up to GS_ROUND tiles the
    kernel runs for them"""
    tiles, warps = (n + TILE - 1) // TILE, blocks * WARPS
    runs = [(w + 1) * tiles // warps - w * tiles // warps for w in range(warps)]
    max_run = (tiles + warps - 1) // warps
    return runs, (max_run + ROUND - 1) // ROUND


def window_blocks(n: int, grid: int) -> int:
    """CudaBackend::run_windows: a warp per group of 32 members up to the grid"""
    return min(((n + TILE - 1) // TILE * 4 + WARPS - 1) // WARPS, grid)


def window_runs(n: int, blocks: int):
    """gs_window_kernel (contiguous mode): (first group, groups) of every warp; the warp takes its groups in
    batches of four, and a batch lies across two tiles when its first group is not a tile's first"""
    groups, warps = (n + TILE - 1) // TILE * 4, blocks * WARPS
    run = (groups + warps - 1) // warps
    out = []
    for w in range(warps):
        g0 = min(w * run, groups)
        out.append((g0, min(g0 + run, groups) - g0))
    return out


def window_batch_crosses_a_tile(n: int, blocks: int) -> bool:
    return any((g0 + b) // 4 != (min(b + 4, cnt) - 1 + g0) // 4
               for g0, cnt in window_runs(n, blocks) for b in range(0, cnt, 4))
