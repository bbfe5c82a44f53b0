"""The H100's whole pool state against the host emulation's, through snapshots.

The GPU parity tests compare pools through the state digest and the 17 readable columns.  Much device state
is in neither: the older coordinate slot, the coordinate tags and adjustment windows, the impairment,
reachability and pause columns, `reap_after`, the mailboxes the next tick does not read, and the pool-wide
counters.  A kernel that writes one of them wrongly passes those tests until the bad value reaches a digested
field.  Here a CUDA pool and a host-emulation pool (the same row bodies compiled for the CPU) take the same
operations, and their snapshots must be equal in canonical form (tests/snapblob.py) after every step:

- lockstep fuzz with directional impairment, pauses, reconnect overrides and long argument lists, at the
  partition edges and under capped grids;
- handover: a blob restored into a fresh pool of the other backend carries on in step for 2 000 ticks;
- scale: 256 Ki members with everything on, at checkpoints over 300 ticks."""
import random

import numpy as np
import pytest

import fuzz_ops
import snapblob as sb
from backend_fuzz import GROWTH, SIZES, size_id
from consul_b200.pool import FLAG_COORDINATES, FLAG_PUSH_PULL, Pool, wan_config
from consul_b200.wan import c5_latency_matrix
from fullstate_fuzz import FullStateLockstep, handover
from test_reach_cpu import Directional

pytestmark = pytest.mark.gpu


def pair(cuda_lib, hostemu_lib, seed, size=None, grow=0):
    return FullStateLockstep(lambda c: Directional(Pool(c, cuda_lib)), lambda c: Directional(Pool(c, hostemu_lib)),
                             seed, size=size, extra=True, grow=grow)


# ---- lockstep fuzz ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("grid", ["1", "17"])
@pytest.mark.parametrize("size", SIZES + (GROWTH,), ids=size_id)
def test_lockstep_full_state(cuda_lib, hostemu_lib, monkeypatch, grid, size):
    monkeypatch.setenv("GSIM_GRID_MAX", grid)
    n0, cap = (size, size + 24) if isinstance(size, int) else size
    seed = 0xF4000 + n0
    p = pair(cuda_lib, hostemu_lib, seed, size=(n0, cap), grow=3 if size == GROWTH else 0)
    assert fuzz_ops.run_sequence(p.make, cuda_lib, seed, n_ops=24) == 24
    assert p.compared > 0


# run_sequence's own configurations: coordinates, push-pull, CSR peer graphs and WAN rings of depth 8
PRESET_SEEDS = (0xF3001, 0xF3010, 0xF300B, 0xF305E, 0xF3082)


def preset_features(lib, seed):
    rng = random.Random(seed)
    cfg, lat = fuzz_ops.random_config(rng, lib)
    graph = cfg.n_initial >= 5 and rng.random() < 0.2
    return {f for f, on in (("coord", cfg.flags & FLAG_COORDINATES), ("pp", cfg.flags & FLAG_PUSH_PULL),
                            ("csr", graph), ("wan8", lat is not None and cfg.mailbox_depth == 8)) if on}


def test_presets_cover_every_feature(hostemu_lib):
    assert set().union(*(preset_features(hostemu_lib, s) for s in PRESET_SEEDS)) == {"coord", "pp", "csr", "wan8"}


@pytest.mark.parametrize("seed", PRESET_SEEDS, ids=hex)
def test_lockstep_full_state_presets(cuda_lib, hostemu_lib, seed):
    p = pair(cuda_lib, hostemu_lib, seed)
    assert fuzz_ops.run_sequence(p.make, cuda_lib, seed, n_ops=40) == 40
    assert p.compared > 0


# ---- handover between the backends ---------------------------------------------------------------------------
def everything(lib, n, seed):
    """WAN C5 at depth 8, coordinates, push-pull, directional impairment with NO_TCP, pauses, reconnect
    overrides and a crash wave (the same operations on either backend)"""
    cfg = dict(capacity=n + 8, n_initial=n, seed=seed, mailbox_depth=8, flags=FLAG_COORDINATES | FLAG_PUSH_PULL,
               push_pull_interval_ns=20 * 10**9, reap_interval_ns=10**9, reconnect_timeout_ns=30 * 10**9)
    p = Pool(wan_config(lib, **cfg), lib)
    lat = c5_latency_matrix(16)
    p.latency_set(lat)
    return p, cfg, 8 - 2 - (int(np.asarray(lat).max()) - 1)


def disturb(p, n, room, salt):
    p.impair_dir_fraction(20000, salt, 0, 1_000_000, room, False)        # inbound blocked
    p.impair_dir_fraction(20000, salt + 1, 1_000_000, 0, 0, True)        # outbound blocked, no TCP
    p.impair_dir(list(range(3 + salt, n, 97)), 200000, 50000, min(1, room), True)
    p.pause_fraction(10000, salt + 2, 60)
    for i in range(5 + salt, n, max(1, n // 3000)):
        p.member_reconnect_timeout_set(i, (i % 7 + 1) * 10**9)
    x = p.member_add()
    p.join(x, [1, 2, 3])
    p.user_event(4, b"ev%d" % salt, b"v" * 9, False)


def fresh_like(p_cfg, lib):
    p = Pool(wan_config(lib, **p_cfg), lib)
    p.latency_set(c5_latency_matrix(16))
    return p


def test_handover_both_ways(cuda_lib, hostemu_lib):
    n = 5000
    (dev, cfg, room), (host, _, _) = everything(cuda_lib, n, 0xF5), everything(hostemu_lib, n, 0xF5)
    for chunk, salt in ((30, 1), (20, 10)):
        for p in (dev, host):
            disturb(p, n, room, salt)
            p.step(chunk)
            p.crash_fraction(20000, salt)
        sb.assert_same(dev.snapshot(), host.snapshot(), f"before the handover, tick {host.now}")
    # the device's state carried on by the host emulation
    moved = handover(dev, host, fresh_like(cfg, hostemu_lib), (1, 7, 100, 400, 1500), "device -> host")
    assert host.now >= 2050
    # and the host emulation's carried on by the device, next to the same host pool
    for p in (moved, host):
        disturb(p, n, room, 20)
        p.step(3)
    handover(host, moved, fresh_like(cfg, cuda_lib), (1, 9, 300, 1700), "host -> device")


# ---- scale -----------------------------------------------------------------------------------------------
def test_everything_at_256k(cuda_lib, hostemu_lib):
    n = 256 << 10
    (dev, cfg, room), (host, _, _) = everything(cuda_lib, n, 0xF6), everything(hostemu_lib, n, 0xF6)
    pools = (dev, host)
    for p in pools:
        p.impair_dir_fraction(10000, 1, 0, 1_000_000, room, False)
        p.impair_dir_fraction(10000, 2, 1_000_000, 0, 0, True)
        p.impair_dir_fraction(5000, 3, 300000, 100000, 1, True)
        p.pause_fraction(3000, 4, 90)
        for i in range(11, n, 64):                                    # 4 096 reconnect overrides
            p.member_reconnect_timeout_set(i, (i % 5 + 1) * 10**9)
        x = p.member_add()
        p.join(x, [0, 1])
        p.user_event(7, b"scale", b"s" * 20, False)
    checkpoints = 0
    for chunk in (20, 40, 90, 150):
        for p in pools:
            p.step(chunk)
        if chunk == 40:
            for p in pools:
                assert p.crash_fraction(20000, 9) > 0                 # a crash wave
        blob = dev.snapshot()
        sb.assert_same(blob, host.snapshot(), f"256 Ki at tick {dev.now}")
        assert dev.state_hash() == host.state_hash()
        parsed = sb.parse(blob)
        assert np.array_equal(sb.newer_coordinates(parsed).view(np.uint64), dev.coordinates().view(np.uint64))
        checkpoints += 1
    assert checkpoints == 4 and dev.now == 300
