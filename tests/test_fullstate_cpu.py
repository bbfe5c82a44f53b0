"""The whole pool state through snapshots, on the CPU: the blob reader (tests/snapblob.py) against the blobs
libgsim writes, row-order independence of every column (not only of the digest and the readable columns),
and a handover between two host-emulation pools that backs up the canonical form's masks."""
import ctypes as C
import hashlib
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest

import fuzz_ops
import snapblob as sb
from consul_b200.pool import FLAG_COORDINATES, FLAG_PUSH_PULL, Pool, lan_config, wan_config
from consul_b200.wan import c5_latency_matrix
from fullstate_fuzz import FullStateLockstep, handover
from test_reach_cpu import Directional

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def busy_pool(lib, coord=False, pp=False, impair=False, reach=False, pause=False, n=300, seed=0xF5):
    """a pool with some of everything its layout carries, 40 ticks into a run"""
    flags = (FLAG_COORDINATES if coord else 0) | (FLAG_PUSH_PULL if pp else 0)
    p = Pool(lan_config(lib, capacity=n + 20, n_initial=n, seed=seed, flags=flags, mailbox_depth=4,
                        push_pull_interval_ns=10**9), lib)
    if impair:
        p.impair(list(range(0, n, 9)), 200000, 1)
    if reach:
        p.impair_dir(list(range(4, n, 11)), 0, 300000, 0, True)
    if pause:
        p.pause(list(range(2, n, 17)), 25)
        p.pause([5], 400)                                # still paused at the snapshot: a Sched entry
    p.member_reconnect_timeout_set(7, 3 * 10**9)
    x = p.member_add()
    p.join(x, [1, 2])
    p.user_event(3, b"ev", b"payload", False)
    p.crash(11)
    p.step(40)
    return p


LAYOUTS = [c for c in itertools.product((False, True), repeat=5) if not (c[3] and not c[2])]  # reach needs impair


def layout_id(c):
    return "-".join(n for n, on in zip(("coord", "pp", "impair", "reach", "pause"), c) if on) or "plain"


@pytest.mark.parametrize("combo", LAYOUTS, ids=layout_id)
def test_parse_and_reserialise_every_layout(hostemu_lib, combo):
    p = busy_pool(hostemu_lib, *combo)
    blob = p.snapshot()
    s = sb.parse(blob)
    want = (sb.LAYOUT_KST | (sb.LAYOUT_COORD if combo[0] else 0) | (sb.LAYOUT_PP if combo[1] else 0) |
            (sb.LAYOUT_IMPAIR if combo[2] else 0) | (sb.LAYOUT_REACH if combo[3] else 0) |
            (sb.LAYOUT_PAUSE if combo[4] else 0))
    assert s["header"]["layout"] == want
    assert sb.serialise(s) == blob
    # the columns gsim_column_read exposes, and the bulk coordinates, are the parsed planes
    n, cap = s["globals"].n, p.capacity
    assert np.array_equal(p.column("key"), s["cols"]["key"][p.now & 1][:cap])
    assert np.array_equal(p.column("sus_from"), s["cols"]["sus_from"][:, :cap])
    assert np.array_equal(p.column("tx"), s["cols"]["tx"][:, :cap])
    assert np.array_equal(p.column("ltime_event"), s["cols"]["ltime_event"][0][:cap])
    assert s["cols"]["reap_after"][0][7] != 0 and not s["cols"]["reap_after"][0][8:].any()
    if combo[0]:
        assert np.array_equal(sb.newer_coordinates(s).view(np.uint64), p.coordinates().view(np.uint64))
    if combo[2]:
        assert s["cols"]["imp_loss"][0][9] != 0 and s["cols"]["imp_delay"][0][9] == 1
    if combo[3]:
        assert s["cols"]["imp_flags"][0][4] == 1 and s["cols"]["imp_recv"][0][4] != 0 and s["cols"]["imp_loss"][0][4] == 0
    if combo[4]:
        assert s["cols"]["pause_until"][0][5] == 400 and list(s["cols"]["pause_cnt"][0][:1]) == [p.pause_stats()["paused"]]
        assert [tuple(e) for e in s["sched"]] == [(400, 0, 2)]
    assert (b"ev", b"payload", 0) in s["rumors"]
    # restore accepts the re-serialised blob, and the pool then writes it again
    q = Pool(lan_config(hostemu_lib, capacity=n + 19, n_initial=300, seed=0xF5,
                        flags=(FLAG_COORDINATES if combo[0] else 0) | (FLAG_PUSH_PULL if combo[1] else 0),
                        mailbox_depth=4, push_pull_interval_ns=10**9), hostemu_lib)
    q.restore(sb.serialise(s))
    assert q.snapshot() == blob
    for r in (p, q):
        r.step(60)
    sb.assert_same(p.snapshot(), q.snapshot(), "60 ticks after the restore")


def test_pinned_sizes(hostemu_lib):
    """gsim_snapshot_size = header + Sched entries + rumor headers + every plane stored raw"""
    for combo in ((False,) * 5, (True,) * 5):
        p = busy_pool(hostemu_lib, *combo)
        blob = p.snapshot()
        s = sb.parse(blob)
        raw = sum(v.nbytes for v in s["cols"].values())
        rum = sum(12 + len(a) + len(b) for a, b, _ in s["rumors"])
        # every SnapCol is one plane per entry of columns(), tx counted as its 15 two-byte planes
        n_planes = sum(e[2] for e in sb.columns(s["header"]["layout"], s["globals"].ring_mask + 1))
        want = sb.SNAP_HEADER_SIZE + sb.SCHED_SIZE * len(s["sched"]) + rum + raw + 4 * n_planes
        size = C.c_size_t()
        assert hostemu_lib.gsim_snapshot_size(p.h, C.byref(size)) == 0
        assert size.value == want, (size.value, want)
        assert len(blob) <= want


def test_fill_planes(hostemu_lib):
    """a plane of one repeated word is stored as tag 1 and read back as the full plane; one word off and it is raw"""
    p = Pool(lan_config(hostemu_lib, capacity=256, n_initial=256, seed=3), hostemu_lib)
    blob = p.snapshot()
    s = sb.parse(blob)
    tags = dict()
    for name, tag in s["tags"]:
        tags.setdefault(name, set()).add(tag)
    assert tags["sus_from"] == {1} and tags["acc"] == {1} and tags["key"] == {0} and tags["stats"] == {0}
    assert (s["cols"]["sus_from"] == 0xFFFFFFFF).all() and (s["cols"]["acc"] == 2**64 - 1).all()
    assert (s["cols"]["ltime_member"] == 1).all()
    assert len(blob) < sb.SNAP_HEADER_SIZE + 256 * 4 * 30      # most planes are fills
    s["cols"]["sus_start"][0][200] = 5                         # one word off: stored raw
    out = sb.serialise(s)
    assert len(out) == len(blob) + 256 * 4 - 4
    assert sb.parse(out)["cols"]["sus_start"][0][200] == 5
    q = Pool(lan_config(hostemu_lib, capacity=256, n_initial=256, seed=3), hostemu_lib)
    q.restore(out)
    assert q.column("sus_start")[200] == 5 and q.snapshot() == out


def test_blob_without_impairment_into_an_impaired_pool(hostemu_lib):
    src = busy_pool(hostemu_lib, coord=True, pause=True)
    plain = src.snapshot()
    assert not sb.parse(plain)["header"]["layout"] & (sb.LAYOUT_IMPAIR | sb.LAYOUT_REACH)
    q = busy_pool(hostemu_lib, coord=True, impair=True, reach=True, pause=True, seed=0xF6)
    q.restore(plain)
    mine = sb.parse(q.snapshot())
    assert mine["header"]["layout"] & sb.LAYOUT_REACH
    for c in ("imp_loss", "imp_delay", "imp_recv", "imp_flags"):
        assert not mine["cols"][c].any(), c                    # nobody impaired
    for r in (src, q):
        r.step(150)
    a, b = sb.canonical(src.snapshot()), sb.canonical(q.snapshot())
    for c in ("imp_loss", "imp_delay", "imp_recv", "imp_flags"):
        del b["cols"][c]
    b["header"] = dict(b["header"], layout=a["header"]["layout"])
    assert sb.first_difference(a, b) is None
    assert src.state_hash() == q.state_hash()


def test_canonical_masks_follow_the_digest(hostemu_lib):
    """A field the digest folds changes the canonical state; a masked field, only where the digest ignores it"""
    p = busy_pool(hostemu_lib, coord=True, pp=True, impair=True, reach=True, pause=True)
    s = sb.parse(p.snapshot())
    base = sb.canonical(s)
    key = s["cols"]["key"][p.now & 1]
    up = np.nonzero((key & 3) == 1)[0]
    idle = [i for i in up if ((s["cols"]["meta"][0][i] >> 3) & 3) == 0 and i < s["globals"].n]
    for name, plane, i, live in (("probe_tgt", 0, idle[0], False), ("due", 0, up[0], True),
                                 ("adj", 3, up[0], True), ("coord", 11 + 2, up[1], True),
                                 ("reap_after", 0, up[2], True), ("imp_flags", 0, 1000 % s["header"]["cap"], True),
                                 ("meta", 0, up[0], True)):
        t = {k: (v.copy() if k == "cols" else v) for k, v in s.items()}
        t["cols"] = {k: v.copy() for k, v in s["cols"].items()}
        v = t["cols"][name]
        v[plane, i] = v[plane, i] + (1 if v.dtype != np.float64 else 0.5)
        d = sb.first_difference(base, sb.canonical(t))
        assert (d is not None) == live, (name, d)
    t = dict(s, cols={k: v.copy() for k, v in s["cols"].items()})
    t["cols"]["meta"][0][up[0]] ^= sb.META_DIRTY              # stripped like gsim_column_read does
    assert sb.first_difference(base, sb.canonical(t)) is None


# ---- row order -----------------------------------------------------------------------------------------
def state_digest(blob) -> str:
    c = sb.canonical(blob)
    h = hashlib.sha256(repr(sorted(c["header"].items())).encode() + c["globals"] + c["sched"].tobytes())
    for name, payload, co in c["rumors"]:
        h.update(name + payload + bytes([co]))
    for k in sorted(c["cols"]):
        h.update(k.encode() + np.ascontiguousarray(c["cols"][k]).tobytes())
    return h.hexdigest()


class Recording(Directional):
    """records the canonical state after every step"""

    def __init__(self, pool, log):
        super().__init__(pool)
        self.log = log

    def step(self, k=1):
        self.pool.step(k)
        self.log.append(state_digest(self.pool.snapshot()))


def recorded_fuzz(lib, seed, n_ops=30):
    """one host-emulation pool through a fuzzed sequence (the second pool of the pair is its twin): the
    canonical state after every step"""
    log = []
    pair = FullStateLockstep(lambda c: Recording(Pool(c, lib), log), lambda c: Directional(Pool(c, lib)), seed,
                             extra=True)
    fuzz_ops.run_sequence(pair.make, lib, seed, n_ops=n_ops)
    return log


ORDER_SEEDS = (0xF0001, 0xF0002, 0xF0007)


@pytest.mark.parametrize("order", ["1", "2"])
def test_full_state_does_not_depend_on_row_order(order):
    code = ("import sys, json; sys.path.insert(0, %r); sys.path.insert(0, %r)\n"
            "from consul_b200 import _lib\n"
            "import test_fullstate_cpu as t\n"
            "L = _lib.load(%r)\n"
            "print(json.dumps([t.recorded_fuzz(L, s) for s in t.ORDER_SEEDS]))\n"
            ) % (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tests", "hostemu", "libgsim_hostemu.so"))
    outs = []
    for o in ("0", order):
        r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, GSIM_HOSTEMU_ORDER=o),
                           capture_output=True, text=True, timeout=900)
        assert r.returncode == 0, r.stderr[-3000:]
        outs.append(r.stdout.strip().splitlines()[-1])
    assert outs[0] == outs[1]
    assert len(outs[0]) > 1000                                 # states were recorded


# ---- lockstep and handover between two host-emulation pools ------------------------------------------------
@pytest.mark.parametrize("seed", range(4))
def test_lockstep_full_state(hostemu_lib, seed):
    pair = FullStateLockstep(lambda c: Directional(Pool(c, hostemu_lib)), lambda c: Directional(Pool(c, hostemu_lib)),
                             0xF1000 + seed, extra=True)
    assert fuzz_ops.run_sequence(pair.make, hostemu_lib, 0xF1000 + seed, n_ops=30) == 30
    assert pair.compared > 0


def everything_pool(lib, n, seed=0xF2):
    """WAN C5 at depth 8, coordinates, push-pull, directional impairment with NO_TCP, pauses, reconnect
    overrides and a crash wave"""
    p = Pool(wan_config(lib, capacity=n + 8, n_initial=n, seed=seed, mailbox_depth=8,
                        flags=FLAG_COORDINATES | FLAG_PUSH_PULL, push_pull_interval_ns=20 * 10**9,
                        reap_interval_ns=10**9, reconnect_timeout_ns=30 * 10**9), lib)
    p.latency_set(c5_latency_matrix(16))
    room = 8 - 2 - (int(np.asarray(c5_latency_matrix(16)).max()) - 1)
    p.impair_dir_fraction(20000, 1, 0, 1_000_000, room, False)       # inbound blocked
    p.impair_dir_fraction(20000, 2, 1_000_000, 0, 0, True)           # outbound blocked, no TCP
    p.impair_dir(list(range(3, n, 97)), 200000, 50000, 1, True)
    p.pause_fraction(10000, 3, 60)
    for i in range(5, n, max(1, n // 300)):
        p.member_reconnect_timeout_set(i, (i % 7 + 1) * 10**9)
    x = p.member_add()
    p.join(x, [1, 2, 3])
    p.user_event(4, b"ev", b"v" * 9, False)
    p.step(30)
    p.crash_fraction(30000, 4)
    p.step(20)
    return p


def test_handover_between_host_pools(hostemu_lib):
    n = 3000
    a, stay = everything_pool(hostemu_lib, n), everything_pool(hostemu_lib, n)
    sb.assert_same(a.snapshot(), stay.snapshot(), "twins")
    fresh = Pool(wan_config(hostemu_lib, capacity=n + 8, n_initial=n, seed=0xF2, mailbox_depth=8,
                            flags=FLAG_COORDINATES | FLAG_PUSH_PULL, push_pull_interval_ns=20 * 10**9,
                            reap_interval_ns=10**9, reconnect_timeout_ns=30 * 10**9), hostemu_lib)
    fresh.latency_set(c5_latency_matrix(16))
    handover(a, stay, fresh, (1, 7, 100, 400, 1500), "host -> host")
    assert stay.now >= 2050
