"""Per-agent serf Stats() and Lifeguard health scores (gsim_agent_stats_read, gsim_health_histogram; DESIGN.md
§3.8) on the host emulation, run in lockstep with the oracle.  Every field of every agent is compared with an
independent restatement over the ORACLE's columns and rumor table, sampled agents also with gsim_members /
gsim_num_nodes, and both calls are checked to be read-only.  The restatement is shared with
tests/test_gpu_agent_stats.py."""
import ctypes as C

import numpy as np
import pytest

import scenarios as sc
from consul_b200.pool import (AGENT_STATS_DTYPE, NEVER, PRED_ALL_RUMORS_CONVERGED, PRED_CRASHED_ALL_DEAD, GsimError,
                              Pool, consul_test_config, lan_config, wan_config)
from consul_b200.wan import c5_latency_matrix
from oracle_binding import OraclePool
from oracle_pause import PauseOraclePool
from oracle_reach import ReachOraclePool

ERR_INVALID, ERR_NOT_FOUND = -1, -5
RUMOR_ALIVE = 1
QCLASS = {1: 0, 2: 1, 3: 1, 4: 2, 5: 0}  # rumor kind -> queue: memberlist, serf intents, serf events
STATUS_LEFT, STATUS_FAILED = 3, 4
ISOLATED = 1 << 11


# ---- restatement ----------------------------------------------------------------------------------------
def rumor_table(pool):
    """[(slot, kind, subject)] of the tracked broadcasts."""
    out = []
    for slot in range(30):
        try:
            info = pool.rumor_info(slot)
        except GsimError:
            continue
        out.append((slot, info["kind"], info["subject"]))
    return out


def popcount(x):
    return np.bitwise_count(x.astype(np.uint32)).astype(np.int64)


def restate(cols, rumors, n, graph=None, impaired=None):
    """(stats, histogram) as serf and memberlist define them, from the columns and the rumor table.

    cols: {key, meta, heard, queued, ltime_member, ltime_event} (the current key buffer), rumors: rumor_table,
    graph: (row_ptr, col_idx) of a CSR pool, impaired: bool per member (None: nobody)."""
    key, meta, heard, queued = (cols[c][:n].astype(np.int64) for c in ("key", "meta", "heard", "queued"))
    truth, rank, pending = key & 3, (key >> 2) & 3, (key >> 4) & 1
    isolated = (meta & ISOLATED) != 0
    listed = truth != 0
    first_slot = {}                           # Members() looks a pending member up by its first alive rumor
    for slot, kind, subj in sorted(rumors):
        if kind == RUMOR_ALIVE and subj not in first_slot:
            first_slot[subj] = slot
    cnt = np.zeros((n, 4), dtype=np.int64)
    ids = np.arange(n)
    cnt[ids[listed], rank[listed]] += 1       # the agent itself
    if graph is None:
        est = listed & (pending == 0)
        total = np.bincount(rank[est], minlength=4)
        others = total[None, :] - (est[:, None] & (rank[:, None] == np.arange(4)[None, :]))
        cnt += np.where(isolated[:, None], 0, others)
        for subj, slot in first_slot.items():
            if subj >= n or not listed[subj] or not pending[subj]:
                continue
            sees = ((heard >> slot) & 1) != 0
            sees[subj] = False
            cnt[sees, rank[subj]] += 1
    else:
        rp, col = graph
        for i in range(n):
            for m in set(int(c) for c in col[rp[i]:rp[i + 1]]) - {i}:
                if not listed[m]:
                    continue
                if pending[m]:
                    ok = m in first_slot and (heard[i] >> first_slot[m]) & 1
                else:
                    ok = not isolated[i]
                if ok:
                    cnt[i, rank[m]] += 1
    mask = [0, 0, 0]
    for slot, kind, _ in rumors:
        mask[QCLASS[kind]] |= 1 << slot
    s = np.zeros(n, dtype=AGENT_STATS_DTYPE)
    s["members"] = cnt.sum(1)
    s["failed"] = cnt[:, 2]
    s["left"] = cnt[:, 3]
    s["health_score"] = meta & 7
    s["member_time"] = cols["ltime_member"][:n]
    s["event_time"] = cols["ltime_event"][:n]
    s["query_time"] = 1
    s["intent_queue"] = popcount(queued & mask[1])
    s["event_queue"] = popcount(queued & mask[2])
    s["query_queue"] = 0
    s["memberlist_queue"] = popcount(queued & mask[0])
    s["running"] = truth == 1
    imp = np.zeros(n, dtype=bool) if impaired is None else np.asarray(impaired[:n], dtype=bool)
    hist = np.zeros((2, 8), dtype=np.uint64)
    run = truth == 1
    np.add.at(hist, (imp[run].astype(np.int64), (meta[run] & 7)), 1)
    return s, hist


STAT_COLUMNS = ("key", "meta", "heard", "queued", "ltime_member", "ltime_event")


def check_agents(p, o, where, graph=None, impaired=None, sample=(0, 1)):
    """Every field of every agent and the histogram against the restatement over the oracle's state."""
    n = p.stats()["n_members"]
    cols = {c: o.column(c) for c in STAT_COLUMNS}
    want, want_hist = restate(cols, rumor_table(o), n, graph, impaired)
    got = p.agent_stats()
    assert got.dtype == AGENT_STATS_DTYPE and len(got) == n
    for f in AGENT_STATS_DTYPE.names:
        bad = np.nonzero(got[f] != want[f])[0]
        assert len(bad) == 0, (where, f, bad[:8], got[f][bad[:8]], want[f][bad[:8]])
    assert (p.health_histogram() == want_hist).all(), (where, p.health_histogram(), want_hist)
    for i in set(sample) | {n - 1}:
        ms = p.members(i)
        assert (got["members"][i], got["failed"][i], got["left"][i]) == (
            len(ms), sum(m[1] == STATUS_FAILED for m in ms), sum(m[1] == STATUS_LEFT for m in ms)), (where, i)
        assert p.num_nodes(i) == got["members"][i]
        assert p.agent_stats(i, 1)[0] == got[i]
    return got


def observables(p):
    return p.state_hash(), p.stats(), p.sched_counts(), p.snapshot()


# ---- scenarios ------------------------------------------------------------------------------------------
def test_join_cascade_pending_isolated_and_merged(hostemu_lib):
    n = 300
    cfg = lan_config(hostemu_lib, capacity=n + 4, n_initial=n, seed=0xA6E1)
    pools = [Pool(cfg, hostemu_lib), OraclePool(cfg)]
    x = sc.both(pools, lambda p: p.member_add())
    assert sc.both(pools, lambda p: p.join(x, [0])) == 1
    lone = sc.both(pools, lambda p: p.member_add())           # created, never joined: isolated, pending
    y = sc.both(pools, lambda p: p.member_add())
    assert sc.both(pools, lambda p: p.join(y, [5])) == 1
    sc.both(pools, lambda p: p.user_event(7, b"deploy", b"x" * 20, False))
    sc.both(pools, lambda p: p.user_event(7, b"again", b"y" * 10, False))
    for k in range(12):
        got = check_agents(*pools, f"cascade tick {k}", sample=(0, 5, 7, x, lone, y))
        assert got["members"][lone] <= 3                      # itself and the joiners it has heard of
        if k == 0:
            assert got["members"][0] == n + 1 and got["members"][5] == n + 1 and got["members"][1] == n
            assert got["event_queue"][7] == 2 and got["intent_queue"][x] == 1 and got["memberlist_queue"][lone] == 1
        sc.step_compare(pools, 1, 1, f"cascade {k}")
    sc.step_compare(pools, 100, 50, "cascade settled")
    got = check_agents(*pools, "settled", sample=(0, x, lone, y))
    assert got["members"][0] >= n + 2 and got["event_queue"].sum() == 0
    assert got["member_time"][:n].min() >= 2 and got["event_time"][:n].min() >= 3


def test_leave_crash_wave_and_dead(hostemu_lib):
    n = 400
    cfg = lan_config(hostemu_lib, capacity=n, n_initial=n, seed=0xA6E2, flags=1)
    pools = [Pool(cfg, hostemu_lib), OraclePool(cfg)]
    for p in pools:
        p.leave(3)
    sc.step_compare(pools, 5, 5, "leaving")
    check_agents(*pools, "leaving", sample=(0, 3))
    sc.step_compare(pools, 60, 20, "left")
    got = check_agents(*pools, "left", sample=(0, 3))
    assert (got["left"] == 1).all() and got["running"][3] == 0
    crashed = sc.both(pools, lambda p: p.crash_fraction(100000, 3))
    sc.step_compare(pools, 30, 30, "crash wave")
    check_agents(*pools, "crash wave", sample=(0, 5))
    t = sc.both(pools, lambda p: p.run_until(PRED_CRASHED_ALL_DEAD, 0, 4000, 25))
    assert t != NEVER
    got = check_agents(*pools, "all dead", sample=(0, 5))
    assert (got["failed"] == crashed).all() and got["running"].sum() == n - 1 - crashed


def test_reap_and_force_leave_prune(hostemu_lib):
    MS = 1_000_000
    cfg = consul_test_config(hostemu_lib, capacity=8, n_initial=0, seed=3, flags=1, phase_group=1,
                             reconnect_timeout_ns=250 * MS, tombstone_timeout_ns=250 * MS, reap_interval_ns=300 * MS)
    pools = [Pool(cfg, hostemu_lib), OraclePool(cfg)]
    for _ in range(5):
        sc.both(pools, lambda p: p.member_add())
    for j in range(1, 5):
        sc.both(pools, lambda p: p.join(j, [0]))
    check_agents(*pools, "joined", sample=range(5))
    assert sc.both(pools, lambda p: p.run_until(PRED_ALL_RUMORS_CONVERGED, 0, 400, 1)) != NEVER
    check_agents(*pools, "converged", sample=range(5))
    for p in pools:
        p.crash_many([1, 2])
    assert sc.both(pools, lambda p: p.run_until(PRED_CRASHED_ALL_DEAD, 0, 2000, 1)) != NEVER
    got = check_agents(*pools, "dead", sample=range(5))
    assert got["failed"][0] == 2
    for k in range(20):                                        # the reaper erases both
        sc.step_compare(pools, 1, 1, f"reap {k}")
        got = check_agents(*pools, f"reap {k}", sample=(0, 1, 3))
        if got["members"][0] == 3:
            break
    assert got["members"][0] == 3 and got["failed"][0] == 0
    for p in pools:
        p.crash(4)
    assert sc.both(pools, lambda p: p.run_until(PRED_CRASHED_ALL_DEAD, 0, 2000, 1)) != NEVER
    for p in pools:
        p.force_leave(0, 4)
    got = check_agents(*pools, "force-leave", sample=(0, 3, 4))
    assert got["left"][0] == 1
    for p in pools:
        p.force_leave(0, 4, prune=True)
    got = check_agents(*pools, "prune", sample=(0, 3, 4))
    assert got["members"][0] == 2 and got["left"][0] == 0


def test_csr_pool(hostemu_lib):
    n = 260
    cfg = lan_config(hostemu_lib, capacity=n + 1, n_initial=n, seed=0xA6E4)
    pools = [Pool(cfg, hostemu_lib), OraclePool(cfg)]
    x = sc.both(pools, lambda p: p.member_add())
    assert sc.both(pools, lambda p: p.join(x, [0])) == 1
    rng = np.random.default_rng(4)
    deg = rng.integers(0, 24, n + 1)
    deg[10], deg[20] = 5, 6
    rp = np.concatenate([[0], np.cumsum(deg)]).astype(np.uint32)
    col = rng.integers(0, n + 1, int(rp[-1])).astype(np.uint32)
    col[rp[10]:rp[10] + 3] = 10                                # itself, and duplicates
    col[rp[20]:rp[20] + 4] = [x, x, 3, 3]                      # the pending joiner twice
    for p in pools:
        p.graph_set(rp, col)
    graph = (rp, col)
    check_agents(*pools, "csr pending", graph=graph, sample=(0, 10, 20, x))
    for p in pools:
        p.crash_many([3, 50, 51])
    for k in range(4):
        sc.step_compare(pools, 60, 60, f"csr {k}")
        check_agents(*pools, f"csr {k}", graph=graph, sample=(0, 10, 20, x))


def test_impaired_and_one_way_members(hostemu_lib):
    n = 600
    cfg = lan_config(hostemu_lib, capacity=n, n_initial=n, seed=0xA6E5)
    pools = [Pool(cfg, hostemu_lib), ReachOraclePool(cfg)]
    k1 = sc.both(pools, lambda p: p.impair_fraction(30000, 1, 600000, 0))
    k2 = sc.both(pools, lambda p: p.impair_dir_fraction(30000, 2, 0, 1000000, 0, no_tcp=True))
    assert k1 > 0 and k2 > 0
    sc.both(pools, lambda p: p.impair_dir([9], 0, 0, 0, no_tcp=True))
    sc.both(pools, lambda p: p.impair([11], 0, 0))             # set back to nothing: unimpaired
    sc.step_compare(pools, 150, 50, "impaired")
    impaired = np.array([any(pools[1].impairment_dir(i)) for i in range(n)])
    assert impaired[9] and not impaired[11]
    got = check_agents(*pools, "impaired", impaired=impaired, sample=(0, 9, 11))
    h = pools[0].health_histogram()
    assert h[1].sum() == impaired.sum() and h.sum() == n
    assert h[1, 7] >= k2 // 2 and got["health_score"][impaired].mean() > got["health_score"][~impaired].mean()


def test_paused_members(hostemu_lib):
    n = 400
    cfg = lan_config(hostemu_lib, capacity=n, n_initial=n, seed=0xA6E6)
    pools = [Pool(cfg, hostemu_lib), PauseOraclePool(cfg)]
    k = sc.both(pools, lambda p: p.pause_fraction(50000, 1, 40))
    k += sc.both(pools, lambda p: p.pause([2], 40))
    assert k > 1
    sc.step_compare(pools, 20, 10, "paused")
    got = check_agents(*pools, "paused", sample=(0, 2))
    assert got["running"].sum() == n - k and got["running"][2] == 0
    assert pools[0].health_histogram().sum() == n - k
    sc.step_compare(pools, 40, 20, "resumed")
    got = check_agents(*pools, "resumed", sample=(0, 2))
    assert got["running"].sum() == n and pools[0].health_histogram().sum() == n


def test_wan_pool_c5_matrix(hostemu_lib):
    n_dcs = 8
    n = n_dcs * 128 + 40
    cfg = wan_config(hostemu_lib, capacity=n + 2, n_initial=n, seed=0xA6E7, mailbox_depth=8)
    pools = [Pool(cfg, hostemu_lib), OraclePool(cfg)]
    for p in pools:
        p.latency_set(c5_latency_matrix(n_dcs))
    x = sc.both(pools, lambda p: p.member_add())
    assert sc.both(pools, lambda p: p.join(x, [130])) == 1
    sc.both(pools, lambda p: p.user_event(300, b"wan", b"z" * 16, False))
    for p in pools:
        p.crash_many([5, 700])
    for k in range(5):
        sc.step_compare(pools, 7, 7, f"wan {k}")
        check_agents(*pools, f"wan {k}", sample=(0, x, 300))


# ---- read-only and validation ---------------------------------------------------------------------------
def test_calls_are_read_only(hostemu_lib):
    n = 300
    cfg = lan_config(hostemu_lib, capacity=n + 2, n_initial=n, seed=0xA6E8)
    p = Pool(cfg, hostemu_lib)
    p.impair_fraction(50000, 1, 500000, 0)
    p.pause([4], 30)
    x = p.member_add()
    p.join(x, [0])
    p.user_event(1, b"e", b"p", False)
    p.step(3)
    before = observables(p)
    p.agent_stats()
    p.agent_stats(7, 3)
    p.health_histogram()
    assert observables(p) == before
    p.step(50)                                                 # and the pool carries on as it would have


def test_errors(hostemu_lib):
    cfg = lan_config(hostemu_lib, capacity=40, n_initial=32, seed=1)
    p = Pool(cfg, hostemu_lib)
    lib = hostemu_lib
    buf = np.zeros(64, dtype=AGENT_STATS_DTYPE)
    ptr = buf.ctypes.data_as(C.c_void_p)
    assert lib.gsim_agent_stats_read(p.h, 0, 32, ptr) == 0
    assert lib.gsim_agent_stats_read(p.h, 31, 1, ptr) == 0
    assert lib.gsim_agent_stats_read(p.h, 0, 33, ptr) == ERR_NOT_FOUND
    assert lib.gsim_agent_stats_read(p.h, 32, 1, ptr) == ERR_NOT_FOUND
    assert lib.gsim_agent_stats_read(p.h, 0xFFFFFFFF, 2, ptr) == ERR_NOT_FOUND
    assert lib.gsim_agent_stats_read(p.h, 0, 0, ptr) == ERR_INVALID
    assert lib.gsim_agent_stats_read(p.h, 0, 4, None) == ERR_INVALID
    assert lib.gsim_agent_stats_read(None, 0, 4, ptr) == ERR_INVALID
    assert lib.gsim_health_histogram(p.h, None) == ERR_INVALID
    assert lib.gsim_health_histogram(None, None) == ERR_INVALID
    with pytest.raises(GsimError):
        p.agent_stats(30, 5)
    assert (p.health_histogram() == np.array([[32] + [0] * 7, [0] * 8])).all()
