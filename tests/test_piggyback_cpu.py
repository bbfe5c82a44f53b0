"""Broadcasts piggybacked on probe traffic (GSIM_FLAG_PROBE_PIGGYBACK, DESIGN.md §3.7) on the host emulation of
the tick kernel's row body: budget conservation, independence from row order, snapshots with owed answers in
flight, the gate that keeps a quiet pool quiet, the owed-answer backlog, and the direction of the effect on
dissemination."""
import os
import subprocess
import sys

import pytest

import piggyback_scenarios as ps
from consul_b200.pool import (FLAG_PROBE_PIGGYBACK, NEVER, PRED_RUMOR_CONVERGED, GsimError, Pool, lan_config)

HERE = os.path.dirname(os.path.abspath(__file__))


def _digest(pools, upto):
    ps.both(pools, lambda p: (p.state_hash(), p.piggyback_stats()))


@pytest.mark.parametrize("n", [400, 2000])
def test_budget_conservation(hostemu_lib, n):
    """Lossless user event: every member transmits it exactly `limit` times, in gossip packets or on probes."""
    pools, slot, t = ps.user_event(lambda cfg: [Pool(cfg, hostemu_lib)], hostemu_lib, n, _digest)
    p = pools[0]
    p.step(200)
    s, pg = p.stats(), p.piggyback_stats()
    assert p.rumor_info(slot)["queued_count"] == 0
    assert s["rumors_sent"] + pg["broadcasts"] == n * s["retransmit_limit"]
    assert s["rumors_sent"] == s["gossip_packets"]                 # gossip packets count gossip only
    assert 0.05 < pg["broadcasts"] / (n * s["retransmit_limit"]) < 0.2, pg
    assert pg["owed_served"] > 0 and pg["packets"] == pg["broadcasts"]


def test_flag_on_a_quiet_pool_changes_nothing(hostemu_lib):
    """Nothing queued: no owed answers are posted, the digest and the launch schedule (quiet windows and their
    closed form) are the unflagged pool's."""
    n = 1000
    pools = [Pool(lan_config(hostemu_lib, capacity=n, n_initial=n, seed=9, flags=f), hostemu_lib)
             for f in (0, FLAG_PROBE_PIGGYBACK)]
    for p in pools:
        p.step(1500)
    assert pools[0].state_hash() == pools[1].state_hash()
    a, b = (p.sched_counts() for p in pools)
    keys = ("window_launches", "window_ticks", "tick_launches", "horizon_scans", "closed_form_launches",
            "closed_form_ticks")
    assert {k: a[k] for k in keys} == {k: b[k] for k in keys}
    assert b["closed_form_ticks"] > 1000
    assert pools[1].piggyback_stats() == {"packets": 0, "broadcasts": 0, "owed_served": 0, "owed_dropped": 0}
    with pytest.raises(GsimError):
        pools[0].piggyback_stats()


def test_quiet_again_after_an_event(hostemu_lib):
    """Once the event has drained the gate clears and the pool goes back to closed-form windows."""
    n = 2000
    pools, slot, t = ps.user_event(lambda cfg: [Pool(cfg, hostemu_lib)], hostemu_lib, n, _digest, seed=3)
    p = pools[0]
    before = p.sched_counts()["closed_form_ticks"]
    served = p.piggyback_stats()["owed_served"]
    p.step(1500)
    assert p.sched_counts()["closed_form_ticks"] - before > 1000
    assert p.piggyback_stats()["owed_served"] == served


def test_piggyback_shortens_dissemination(hostemu_lib):
    """Same seeds with and without the flag: the event reaches everybody sooner on average (M0 measured 0.3-2
    ticks at <= 800 agents)."""
    n = 400
    ticks = {0: [], FLAG_PROBE_PIGGYBACK: []}
    for seed in range(8):
        for f in ticks:
            p = Pool(lan_config(hostemu_lib, capacity=n, n_initial=n, seed=0x5EED0100 + seed, flags=f), hostemu_lib)
            slot = p.user_event(0, b"deploy", b"x" * 32, False)
            t = p.run_until(PRED_RUMOR_CONVERGED, slot, 600, 1)
            assert t != NEVER
            ticks[f].append(t)
    plain, pig = (sum(v) / len(v) for v in ticks.values())
    assert 0.2 <= plain - pig <= 4.0, ticks


def test_backlog_overflow_is_counted(hostemu_lib):
    """A small pool whose members all probe at the same tick, a third of them crashed and eight relays per
    indirect probe: members owe more answers in one tick than the 4 they serve; the rest are dropped and counted,
    the same in every row order (test_row_order_independence's scenarios share the counter)."""
    n = 24
    cfg = lan_config(hostemu_lib, capacity=n, n_initial=n, seed=77, flags=FLAG_PROBE_PIGGYBACK, retransmit_mult=4,
                     indirect_checks=8)
    p = Pool(cfg, hostemu_lib)
    p.crash_many(list(range(1, n, 3)))
    for k in range(10):
        p.user_event(0, b"e%d" % k, b"x", False)
        p.step(10)
    pg = p.piggyback_stats()
    assert pg["owed_dropped"] > 0 and pg["owed_served"] > 0, pg


def test_snapshot_with_owed_answers_in_flight(hostemu_lib):
    n = 2000
    cfg = lan_config(hostemu_lib, capacity=n + 1, n_initial=n, seed=21, flags=FLAG_PROBE_PIGGYBACK,
                     packet_loss_ppm=50000)
    p = Pool(cfg, hostemu_lib)
    x = p.member_add()
    p.join(x, [0])
    p.user_event(5, b"e", b"x" * 8, False)
    p.step(6)
    req = p.piggyback_stats()["owed_served"]
    p.step(1)
    assert p.piggyback_stats()["owed_served"] > req             # answers are owed across the snapshot
    blob = p.snapshot()
    q = Pool(cfg, hostemu_lib)
    q.restore(blob)
    served = p.piggyback_stats()["owed_served"]
    for x in (p, q):                                            # the blob held owed answers: served right away
        x.step(1)
        assert x.piggyback_stats()["owed_served"] > served
    for k in (1, 5, 40, 200):
        p.step(k)
        q.step(k)
        assert q.state_hash() == p.state_hash() and q.piggyback_stats() == p.piggyback_stats()
    with pytest.raises(GsimError):
        Pool(lan_config(hostemu_lib, capacity=n + 1, n_initial=n, seed=21), hostemu_lib).restore(blob)


def test_unflagged_blob_is_unchanged(hostemu_lib):
    """A pool without the flag writes the blob it wrote before: no piggyback layout bit, no extra planes."""
    n = 500
    a = Pool(lan_config(hostemu_lib, capacity=n, n_initial=n, seed=2), hostemu_lib)
    b = Pool(lan_config(hostemu_lib, capacity=n, n_initial=n, seed=2, flags=FLAG_PROBE_PIGGYBACK), hostemu_lib)
    for p in (a, b):
        p.step(20)
    ba, bb = a.snapshot(), b.snapshot()
    layout = lambda blob: int.from_bytes(blob[36:40], "little")  # SnapHeader.layout
    assert layout(ba) & 128 == 0 and layout(bb) & 128 == 128
    assert len(bb) > len(ba)


def _scenario_digests(lib):
    out = []
    rec = lambda pools, upto: out.append((upto, pools[0].state_hash(), tuple(pools[0].piggyback_stats().values())))
    mk = lambda cfg: [Pool(cfg, lib)]
    ps.user_event(mk, lib, 600, rec)
    ps.join_cascade(mk, lib, 700, rec)
    ps.crash_wave(mk, lib, 700, rec)
    ps.wan_impaired(mk, lib, 16 * 128, rec, push_pull=True, max_ticks=200)
    p = Pool(lan_config(lib, capacity=24, n_initial=24, seed=77, flags=FLAG_PROBE_PIGGYBACK, retransmit_mult=4,
                        indirect_checks=8), lib)                  # (test_backlog_overflow_is_counted's pool)
    p.crash_many(list(range(1, 24, 3)))
    for k in range(10):
        p.user_event(0, b"e%d" % k, b"x", False)
        p.step(10)
        rec([p], p.now)
    return out


def test_row_order_independence(hostemu_lib):
    """Owed answers are a commutative mailbox: reverse and odd-even row orders give the same digests and
    counters as the natural order, through a user event, a join cascade, a crash wave with loss and a WAN pool
    with delays, one-way members and push-pull."""
    ref = _scenario_digests(hostemu_lib)
    code = ("import sys; sys.path[:0]=[%r,%r]\n"
            "from consul_b200 import _lib\n"
            "import test_piggyback_cpu as t\n"
            "print(repr(t._scenario_digests(_lib.load(%r))))\n") % (
        os.path.dirname(HERE), HERE, os.path.join(HERE, "hostemu", "libgsim_hostemu.so"))
    for order in ("1", "2"):
        r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, GSIM_HOSTEMU_ORDER=order),
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stdout + r.stderr
        assert r.stdout.strip().splitlines()[-1] == repr(ref)


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_fuzz_with_the_flag(hostemu_lib, seed):
    """The fuzzed operation sequences on flagged pools: two host-emulation pools in lockstep, the first of which
    is snapshotted, stepped and restored now and then (which must be invisible), with the column invariants."""
    import fuzz_ops

    def make(cfg):
        cfg.flags |= FLAG_PROBE_PIGGYBACK
        return [Pool(cfg, hostemu_lib), Pool(cfg, hostemu_lib)]
    fuzz_ops.run_sequence(make, hostemu_lib, seed, n_ops=50)
