"""Fault domains (gsim_domain_*) on the H100: a 1 Mi LAN pool in racks of 32 with a flapping rack schedule and a
256 Ki WAN C5 pool with flapping rack delay against the domain oracle, the 4 M-member C3 crash wave with 1 % of
racks crashed by gsim_domain_crash against the oracle and gsim_crash_many over the same ids, a domain schedule that is
always bad against the static impairment and one that is never bad against no impairment at 1 Mi members,
gsim_domain_stats_read against a numpy restatement at 16 Mi members, and a device snapshot round trip."""
import numpy as np
import pytest

from consul_b200.pool import (NEVER, PRED_CRASHED_ALL_DEAD, Pool, lan_config, wan_config)
from consul_b200.wan import c5_latency_matrix
from oracle_domain import DomainOraclePool
from parity import compare_pools
from test_domain_cpu import SCHEDULING, split_dom, stats_rows

pytestmark = pytest.mark.gpu
FULL = 1_000_000


def _racks(p, n, per, share_ppm, salt):
    """Racks of `per` members; the racks whose index draws below share_ppm (a fixed numpy stream)."""
    p.domain_set_range(0, n, per, 1)
    n_racks = (n + per - 1) // per
    rng = np.random.default_rng(salt)
    return sorted(int(d) + 1 for d in np.nonzero(rng.random(n_racks) < share_ppm / FULL)[0])


def both(pools, fn):
    a, b = [fn(p) for p in pools]
    assert a == b, (a, b)
    return a


def test_1m_lan_racks_flapping_against_the_oracle(cuda_lib):
    """1 Mi members in racks of 32, 1 % of racks at 50 % loss under a rack schedule (period 50, 10 % bad), and
    a user event: digest and counters against the domain oracle; a rack's members are in force together."""
    n = 1 << 20
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0xD0A90002, disable_tcp_pings=1)
    pools = [Pool(cfg, cuda_lib), DomainOraclePool(cfg, threads=0)]
    racks = [_racks(p, n, 32, 10_000, 2) for p in pools][0]
    assert both(pools, lambda p: p.domain_impair(racks, 500_000, 500_000)) == 32 * len(racks)
    both(pools, lambda p: p.domain_flap(racks, 50, 100_000))
    both(pools, lambda p: p.user_event(3, b"deploy", bytes(32), False))
    seen = set()
    for upto in (10, 60, 200, 350, 500):
        for p in pools:
            p.step(upto - p.now)
        compare_pools(*pools, f"1M LAN racks tick {upto}", columns=False)
        s = pools[0].domain_stats(1, n // 32)
        assert (stats_rows(s) == stats_rows(pools[1].domain_stats(1, n // 32))).all(), upto
        for d in racks:
            assert s["in_force"][d - 1] in (0, 32)
            seen.add(int(s["in_force"][d - 1]))
    assert seen == {0, 32}
    st = pools[0].stats()
    assert st["packets_lost"] > 0 and st["suspects"] > 0 and st["deads"] == 0, st


def test_wan_c5_flapping_domain_delay_against_the_oracle(cuda_lib):
    n = 1 << 18
    cfg = wan_config(cuda_lib, capacity=n, n_initial=n, seed=0xD0A90003, mailbox_depth=8)
    pools = [Pool(cfg, cuda_lib), DomainOraclePool(cfg, threads=0)]
    for p in pools:
        p.latency_set(c5_latency_matrix(64))
    racks = [_racks(p, n, 64, 20_000, 3) for p in pools][0]
    both(pools, lambda p: p.domain_impair(racks, 100_000, 100_000, 2))
    both(pools, lambda p: p.domain_flap(racks, 10, 400_000))
    both(pools, lambda p: p.impair_flap(list(range(0, n, 97)), 7, 500_000))
    both(pools, lambda p: p.user_event(0, b"e", b"x" * 16, False))
    for upto in (20, 100, 300, 600):
        for p in pools:
            p.step(upto - p.now)
        compare_pools(*pools, f"WAN C5 tick {upto}", columns=False)


def test_c3_4m_racks_crashed_by_domain(cuda_lib):
    """4 M members, 1 % of racks of 32 crashed by gsim_domain_crash: the all-dead tick, digest and counters equal
    the domain oracle's, and the device pool equals one crashed by gsim_crash_many over the same ids."""
    n = 4_000_000
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0xD0A90004)
    a, b, ora = Pool(cfg, cuda_lib), Pool(cfg, cuda_lib), DomainOraclePool(cfg, threads=0)
    racks = _racks(a, n, 32, 10_000, 4)
    _racks(ora, n, 32, 10_000, 4)
    b.domain_set_range(0, n, 32, 1)
    ids = np.nonzero(np.isin(b.domains(), racks))[0].tolist()
    assert a.domain_crash(racks) == ora.domain_crash(racks) == len(ids)
    b.crash_many(ids)
    ta = a.run_until(PRED_CRASHED_ALL_DEAD, 0, 2000, 16)
    to = ora.run_until(PRED_CRASHED_ALL_DEAD, 0, 2000, 16)
    tb = b.run_until(PRED_CRASHED_ALL_DEAD, 0, 2000, 16)
    assert ta == to == tb != NEVER
    compare_pools(a, ora, "all dead vs oracle", columns=False)
    compare_pools(a, b, "all dead vs crash_many", columns=False)


def _pair_1m(cuda_lib, seed):
    n = 1 << 20
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=seed, disable_tcp_pings=1, mailbox_depth=4)
    a, b = Pool(cfg, cuda_lib), Pool(cfg, cuda_lib)
    for p in (a, b):
        p.impair_dir_fraction(10_000, 4, 400_000, 300_000, 1, True)
        p.user_event(1, b"e", b"", False)
    a.domain_set_range(0, n, 32, 1)
    return a, b, list(range(1, n // 32 + 1))


def test_always_bad_domains_are_the_static_impairment_at_1m(cuda_lib):
    a, b, doms = _pair_1m(cuda_lib, 0xD0A90005)
    a.domain_flap(doms, 13, FULL)
    for upto in (5, 40, 150, 300):
        for p in (a, b):
            p.step(upto - p.now)
        compare_pools(a, b, f"always bad tick {upto}", columns=False)
    assert split_dom(a.snapshot())[0] == b.snapshot()


def test_never_bad_domains_are_no_impairment_at_1m(cuda_lib):
    a, b, doms = _pair_1m(cuda_lib, 0xD0A90006)
    b.impair_dir_fraction(10_000, 4, 0, 0, 0, False)
    a.domain_flap(doms, 13, 0)
    for upto in (5, 40, 150, 300):
        for p in (a, b):
            p.step(upto - p.now)
        assert a.state_hash() == b.state_hash(), upto
        sa, sb = a.stats(), b.stats()
        for f in SCHEDULING:
            sa.pop(f), sb.pop(f)
        assert sa == sb, upto


def test_domain_stats_at_16m(cuda_lib, hostemu_lib):
    n = 16 << 20
    seed = 0xD0A90007
    p = Pool(lan_config(cuda_lib, capacity=n, n_initial=n, seed=seed, mailbox_depth=4), cuda_lib)
    racks = _racks(p, n, 40, 10_000, 7)
    crashed = racks[::3]
    p.domain_impair(racks, 300_000, 300_000, 1)
    p.domain_flap(racks[::2], 20, 500_000)
    p.domain_crash(crashed)
    p.step(30)
    n_dom = (n + 39) // 40
    h, s = p.state_hash(), p.stats()
    got = p.domain_stats(1, n_dom)
    assert p.state_hash() == h and p.stats() == s
    key, meta, dom = p.column("key")[:n], p.column("meta")[:n], p.domains()
    truth, rank, aw = key & 3, (key >> 2) & 3, (meta & 7).astype(np.uint64)
    run = truth == 1
    x = dom.astype(np.int64) - 1
    want = {"members": np.bincount(x, minlength=n_dom), "running": np.bincount(x, run, n_dom),
            "paused": np.zeros(n_dom)}
    imp_dom = np.zeros(n_dom + 1, bool)
    imp_dom[racks] = True
    bad = np.ones(n_dom + 1, bool)
    for d in racks[::2]:
        bad[d] = hostemu_lib.gsim_domain_flap_bad(seed, d, 20, 500_000, p.now) == 1
    want["impaired"] = np.bincount(x, imp_dom[dom], n_dom)
    want["in_force"] = np.bincount(x, imp_dom[dom] & bad[dom], n_dom)
    for r, f in enumerate(("alive", "suspect", "dead", "left")):
        want[f] = np.bincount(x, rank == r, n_dom)
    want["awareness_sum"] = np.bincount(x, np.where(run, aw, 0), n_dom)
    mx = np.zeros(n_dom, np.uint64)
    np.maximum.at(mx, x, np.where(run, aw, 0))
    want["awareness_max"] = mx
    for f, v in want.items():
        assert (got[f].astype(np.int64) == np.asarray(v).astype(np.int64)).all(), f
    assert got["running"][np.array(crashed) - 1].sum() == 0


def test_snapshot_round_trip_on_the_device(cuda_lib):
    n = 1 << 18
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0xD0A90008, disable_tcp_pings=1, mailbox_depth=4)
    p = Pool(cfg, cuda_lib)
    racks = _racks(p, n, 32, 20_000, 8)
    p.domain_impair(racks, 600_000, 600_000, 1)
    p.domain_flap(racks, 29, 300_000)
    p.user_event(1, b"e", b"", False)
    p.step(43)
    blob = p.snapshot()
    p.step(200)
    h1, s1 = p.state_hash(), p.stats()
    q = Pool(cfg, cuda_lib)
    q.restore(blob)
    assert (q.domains() == p.domains()).all() and q.domain_flap_get(racks[0]) == (29, 300_000)
    q.step(200)
    s2 = q.stats()
    for s in (s1, s2):
        s.pop("active_rows")
    assert q.state_hash() == h1 and s2 == s1
