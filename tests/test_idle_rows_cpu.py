"""Rows of a join-cascade tick that have nothing to do are not stepped (host emulation of the tick kernel).

A member with a non-empty broadcast queue wakes at its next gossip tick instead of every tick, and mail
whose rumors the receiver has all heard only clears its word (gs_queue_wake_slot / gs_mail_is_stale in
consul_b200/csrc/gs_row.h; the tick kernel retires such words in its scan, the row step returns before
counting the row).  Neither changes what any row computes: every case below is compared with the oracle
tick by tick, and the cascade of bench.py's workload must end in the oracle's digest with fewer rows
stepped.
"""
import os
import subprocess

import pytest

import scenarios as sc
from consul_b200.pool import FLAG_PUSH_PULL, Pool, lan_config, wan_config
from oracle_binding import OraclePool
from parity import compare_stats

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEC = 1_000_000_000
MS = 1_000_000

# sum of active_rows over the 64 single ticks of the cascade below, before queued members woke only at
# their gossip ticks and stale mail stopped being stepped (host emulation, same workload)
ACTIVE_ROWS_BEFORE = 4_533_831


@pytest.fixture()
def make(hostemu_lib):
    return lambda cfg: [Pool(cfg, hostemu_lib), OraclePool(cfg)]


def bench_cascade(pools):
    """step(64), one bench step (member_add -> join(x, [0]) -> step(2048)), then one more member_add + join
    and 64 single ticks (tools/cascade_rows.py): active_rows of each of those ticks."""
    for p in pools:
        p.step(64)
    x = sc.both(pools, lambda p: p.member_add())
    assert sc.both(pools, lambda p: p.join(x, [0])) == 1
    for p in pools:
        p.step(2048)
    x = sc.both(pools, lambda p: p.member_add())
    assert sc.both(pools, lambda p: p.join(x, [0])) == 1
    rows = []
    for _ in range(64):
        before = pools[0].stats()["active_rows"]
        for p in pools:
            p.step(1)
        rows.append(pools[0].stats()["active_rows"] - before)
    return rows


def test_cascade_steps_fewer_rows_and_computes_the_same(make, hostemu_lib):
    n = 200_000
    pools = make(lan_config(hostemu_lib, capacity=n + 16, n_initial=n, seed=0x5EED0001))
    rows = bench_cascade(pools)
    total = sum(rows)
    print(f"\nactive rows over the cascade: {total:,} (before: {ACTIVE_ROWS_BEFORE:,}, "
          f"{total / ACTIVE_ROWS_BEFORE:.3f}); peak tick {max(rows):,}")
    assert total <= 0.8 * ACTIVE_ROWS_BEFORE
    compare_stats(*pools, "after the cascade")
    assert pools[0].state_hash() == pools[1].state_hash()


def test_queued_members_have_a_wake_by_their_next_gossip_tick(tmp_path):
    """tests/hostemu/queue_wake_check.cpp: after every tick of a cascade, on a LAN pool (GI 2, depth 2), a WAN
    pool on 100 ms ticks (GI 5, depth 8) and a pool whose GI (3) exceeds its ring depth (2)."""
    exe = str(tmp_path / "queue_wake_check")
    subprocess.run(["g++", "-O2", "-ffp-contract=off", "-std=c++17", "-pthread", "-o", exe,
                    os.path.join(ROOT, "tests", "hostemu", "queue_wake_check.cpp"),
                    os.path.join(ROOT, "tests", "hostemu", "hostemu_backend.cpp")], check=True, cwd=ROOT)
    r = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    print(r.stdout)
    assert r.returncode == 0, r.stdout + r.stderr
    assert r.stdout.count(" 0 violations") == 3


def test_user_event_dropped_by_event_min_and_buffer_window(make, hostemu_lib):
    """A dropped event is not in `heard`: its mail keeps stepping the member (and witnessing the clock)."""
    n = 64
    pools = make(lan_config(hostemu_lib, capacity=n + 4, n_initial=n, seed=31, event_buffer=4))
    sc.both(pools, lambda p: p.user_event(1, b"old", b"1", False))
    sc.step_compare(pools, 3, 1, "first event")
    x = sc.both(pools, lambda p: p.member_add(watched=True))
    sc.both(pools, lambda p: p.join(x, [2], True))              # ignore_old: eventMinTime drops "old"
    for k in range(6):
        sc.both(pools, lambda p: p.user_event(1, b"burst%d" % k, b"", False))
    sc.step_compare(pools, 50, 1, "window")
    assert pools[0].stats()["rumors_dropped"] > 0


def test_accusation_and_push_pull_riding_with_stale_bits(make, hostemu_lib):
    """Push-pull answers carry the sender's whole heard mask with GS_ACC_BIT; accusations reach crashed
    members while gossip about the same rumors is still arriving."""
    n = 400
    pools = make(lan_config(hostemu_lib, capacity=n + 2, n_initial=n, seed=0x5EED0021, flags=FLAG_PUSH_PULL,
                            push_pull_interval_ns=1 * SEC))
    sc.both(pools, lambda p: p.user_event(3, b"e", b"p", False))
    sc.step_compare(pools, 6, 1, "event spreading")
    for p in pools:
        p.crash_many([10, 11, 12, 200])
    sc.both(pools, lambda p: p.user_event(4, b"f", b"q", False))
    sc.step_compare(pools, 120, 1, "accusations and push-pulls")
    s = pools[0].stats()
    assert s["suspects"] > 0 and s["push_pulls"] > 0


def test_crashed_members_with_mail_in_flight(make, hostemu_lib):
    n = 500
    pools = make(lan_config(hostemu_lib, capacity=n + 2, n_initial=n, seed=0x5EED0031))
    x = sc.both(pools, lambda p: p.member_add())
    assert sc.both(pools, lambda p: p.join(x, [0])) == 1
    sc.step_compare(pools, 8, 1, "cascade")
    for p in pools:
        p.crash_many(list(range(0, n, 7)))                       # mid-cascade: queues and mail in flight
    sc.step_compare(pools, 80, 1, "after the crash")


def test_retired_slot_in_flight_and_reused(make, hostemu_lib):
    n = 300
    pools = make(lan_config(hostemu_lib, capacity=n + 2, n_initial=n, seed=0x5EED0041))
    slot = sc.both(pools, lambda p: p.user_event(5, b"gone", b"", False))
    sc.step_compare(pools, 5, 1, "in flight")
    for p in pools:
        p.rumor_retire(slot)                                      # retired with its packets still travelling
    sc.step_compare(pools, 2, 1, "retired")
    assert sc.both(pools, lambda p: p.user_event(9, b"reuse", b"x", False)) == slot
    sc.step_compare(pools, 40, 1, "slot reused")


def test_wan_pool_depth_eight(make, hostemu_lib):
    """WAN timing on 100 ms ticks: GossipInterval is 5 ticks, a queued member's wake lands 5 slots ahead."""
    n = 1000
    pools = make(wan_config(hostemu_lib, capacity=n + 2, n_initial=n, seed=0x5EED0051, mailbox_depth=8,
                            tick_ns=100 * MS))
    s = pools[0].stats()
    assert s["gossip_interval_ticks"] == 5
    x = sc.both(pools, lambda p: p.member_add())
    assert sc.both(pools, lambda p: p.join(x, [0])) == 1
    sc.both(pools, lambda p: p.user_event(2, b"wan", b"", False))
    sc.step_compare(pools, 60, 1, "wan cascade")


def test_gossip_interval_longer_than_the_ring(make, hostemu_lib):
    """GI = 3 ticks on a depth-2 ring: a wake three ticks ahead does not fit, so it goes to t + 1 there."""
    n = 600
    pools = make(lan_config(hostemu_lib, capacity=n + 2, n_initial=n, seed=0x5EED0061, gossip_interval_ns=300 * MS))
    assert pools[0].stats()["gossip_interval_ticks"] == 3
    x = sc.both(pools, lambda p: p.member_add())
    assert sc.both(pools, lambda p: p.join(x, [0])) == 1
    sc.step_compare(pools, 60, 1, "GI > depth")
