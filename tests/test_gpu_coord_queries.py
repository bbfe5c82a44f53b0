"""Network-coordinate queries on the H100 (DESIGN.md §3.4 "Queries"): the sm_90a gather, pair, sort, median and
sampling kernels against the oracle's coordinates and the restatements of tests/test_coord_queries_cpu.py, at
pool scale; the pool's digest still equals the oracle's after the queries."""
import time

import numpy as np
import pytest
from scipy.stats import spearmanr

import test_coord_queries_cpu as tq
from consul_b200.pool import FLAG_COORDINATES, Pool, lan_config, wan_config
from consul_b200.wan import c5_latency_matrix
from oracle_binding import OraclePool
from oracle_impair import ImpairOraclePool

pytestmark = pytest.mark.gpu
MI = 1 << 20


def lockstep(pools, ticks):
    for p in pools:
        p.step(ticks)
    assert pools[0].state_hash() == pools[1].state_hash()


def check_all(p, o, lat, delay, frm, n_dcs=0, draws=MI):
    n = p.stats()["n_members"]
    tick_s = tq.tick_seconds(p)
    coords = p.coordinates()
    ref = tq.oracle_coords(o, n)
    assert coords.tobytes() == ref.tobytes()
    keys = tq.view_keys(p)
    # the full ?near= order of every member
    ids, dist = p.sort_by_distance(frm)
    e_ids, e_dist = tq.stable_order(np.arange(n), tq.distance(ref[frm], ref))
    assert (ids == e_ids).all() and dist.tobytes() == e_dist.tobytes()
    # pair estimates and true round trips
    rng = np.random.default_rng(5)
    a, b = rng.integers(0, n, 100000), rng.integers(0, n, 100000)
    est, tru = p.rtt(a, b, true_rtt=True)
    assert est.tobytes() == tq.distance(ref[a], ref[b]).tobytes()
    assert tru.tobytes() == tq.model_rtt(lat, delay, tick_s, a, b).tobytes()
    if n_dcs:
        order, rtt = p.dcs_by_distance(frm)
        e_order, e_rtt = tq.router_dcs(ref, keys, frm, n_dcs)
        assert (order == e_order).all() and rtt.tobytes() == e_rtt.tobytes()
    got = p.coordinate_error(min(draws, p.capacity), 1)
    exp = tq.error_stats(ref, keys, lat, delay, tick_s, p.cfg.seed, n, min(draws, p.capacity), 1)
    assert np.array([got[k] for k in ("pairs", "mean", "p50", "p90", "p99", "max")]).tobytes() == np.array(exp).tobytes()
    return got


def test_lan_1mi(cuda_lib):
    n = MI
    cfg = lan_config(cuda_lib, capacity=n, n_initial=n, seed=0xC0, flags=FLAG_COORDINATES)
    pools = [Pool(cfg, cuda_lib), OraclePool(cfg, threads=0)]
    pools[0].crash_many([9, 70000])
    pools[1].crash_many([9, 70000])
    lockstep(pools, 120)
    before = tq.observables(pools[0])
    check_all(*pools, None, None, 4242)
    assert tq.observables(pools[0]) == before
    lockstep(pools, 10)


def test_wan_c5_2mi(cuda_lib):
    n = 2 * MI
    cfg = wan_config(cuda_lib, capacity=n, n_initial=n, seed=0xC5, flags=FLAG_COORDINATES, mailbox_depth=8)
    pools = [Pool(cfg, cuda_lib), OraclePool(cfg, threads=0)]
    lat = c5_latency_matrix(64)
    for p in pools:
        p.latency_set(lat)
        p.leave(300)
    lockstep(pools, 60)
    check_all(*pools, lat, None, 77, n_dcs=64)
    lockstep(pools, 5)


def test_impaired_delays(cuda_lib):
    n = 256 * 1024
    cfg = wan_config(cuda_lib, capacity=n, n_initial=n, seed=0x1D, flags=FLAG_COORDINATES, mailbox_depth=8)
    pools = [Pool(cfg, cuda_lib), ImpairOraclePool(cfg, threads=0)]
    lat = c5_latency_matrix(16)
    for p in pools:
        p.latency_set(lat)
        p.impair_fraction(50000, 3, 0, 1)
    delay = np.array([pools[0].impairment(i)[1] for i in range(n)], dtype=np.int64)
    assert delay.sum() > 0
    lockstep(pools, 100)
    check_all(*pools, lat, delay, 1000, n_dcs=16)
    lockstep(pools, 5)


def test_c5_8mi_sort_and_ranking(cuda_lib):
    """8 Mi members on the C5 matrix, the embedding run long enough to settle: the full sort and the DC
    ranking against restatements over the pool's own coordinates (bulk-read, equal to the per-member getter),
    and the ranking property of the matrix seen from DC0.  No oracle runs beside it: 2000 ticks of 8 Mi
    members with coordinates are over a hundred times the oracle work of the 2 Mi case (60 ticks of 2 Mi); the bulk read and the query kernels are checked against
    the oracle at 1 Mi, 2 Mi and on the unaligned pool below, and this pool's digest stays unchanged by the
    queries (checked against its own digest before them)."""
    n = 8 * MI
    cfg = wan_config(cuda_lib, capacity=n, n_initial=n, seed=0x8C5, flags=FLAG_COORDINATES, mailbox_depth=8)
    p = Pool(cfg, cuda_lib)
    lat = c5_latency_matrix(64)
    p.latency_set(lat)
    p.step(2000)
    digest = p.state_hash()
    coords = p.coordinates()
    for i in (0, 12345, n - 1):
        vec, err, adj, h = p.coordinate(i)
        assert coords[i].tobytes() == np.array(vec + [err, adj, h]).tobytes()
    keys = tq.view_keys(p)
    frm = 5
    t0 = time.perf_counter()
    ids, dist = p.sort_by_distance(frm)
    t_sort = time.perf_counter() - t0
    e_ids, e_dist = tq.stable_order(np.arange(n), tq.distance(coords[frm], coords))
    assert (ids == e_ids).all() and dist.tobytes() == e_dist.tobytes()
    order, rtt = p.dcs_by_distance(frm)
    e_order, e_rtt = tq.router_dcs(coords, keys, frm, 64)
    assert (order == e_order).all() and rtt.tobytes() == e_rtt.tobytes()
    # seen from DC0, the DCs b = 0 (mod 5) are 5 ticks nearer than every other one, there and back
    near = [b for b in range(64) if b % 5 == 0]
    assert set(order[: len(near)]) == set(near), (list(order), list(rtt))
    true_rtt = [0.0005 + (int(lat[0][b]) - 1 + int(lat[b][0]) - 1) * tq.tick_seconds(p) for b in order]
    rho = spearmanr(rtt, true_rtt).correlation
    err = p.coordinate_error(MI, 0)
    assert p.state_hash() == digest
    print(f"8Mi C5 after 2000 ticks: full sort {t_sort * 1e3:.1f} ms wall, DC rank correlation {rho:.3f}, "
          f"error {err}")


def test_unaligned_shapes_against_the_oracle(cuda_lib):
    """The radix sort's and the gather's edges on the device: a pool whose size is a multiple of neither the
    sort's 4096-pair tile nor the 256-thread CTA (partial last tile, partial last round with idle lanes, fewer
    tiles than digits in the scan), explicit id lists of every awkward length with duplicates and k < n,
    a servers subset for the DC ranking, a partial row block and a partial last chunk of error draws."""
    n = 300007
    cfg = wan_config(cuda_lib, capacity=n, n_initial=n, seed=0x0DD, flags=FLAG_COORDINATES, mailbox_depth=8)
    pools = [Pool(cfg, cuda_lib), OraclePool(cfg, threads=0)]
    lat = c5_latency_matrix(64)
    for q in pools:
        q.latency_set(lat)
        q.leave(4099)
    lockstep(pools, 60)
    p, o = pools
    check_all(p, o, lat, None, 4097, n_dcs=64)             # full sort, DC ranking, n_draws = n (n % 256 != 0)
    ref = tq.oracle_coords(o, n)
    keys = tq.view_keys(p)
    tick_s = tq.tick_seconds(p)
    for first, count in ((0, 1), (1000, 12345), (n - 300, 300), (n - 1, 1), (255, 257)):
        assert p.coordinates(first, count).tobytes() == ref[first:first + count].tobytes()
    rng = np.random.default_rng(11)
    for m in (1, 2, 255, 256, 257, 4095, 4096, 4097, 65537):
        sel = rng.integers(0, n, m).astype(np.uint32)
        sel[m // 2:] = sel[: m - m // 2]                       # duplicates: the second half repeats the first
        e_ids, e_dist = tq.stable_order(sel, tq.distance(ref[77], ref[sel]))
        for k in sorted({1, m // 2, m} - {0}):
            ids, dist = p.sort_by_distance(77, sel, k)
            assert (ids == e_ids[:k]).all() and dist.tobytes() == e_dist[:k].tobytes(), (m, k)
    servers = np.sort(rng.choice(n, 5000, replace=False)).astype(np.uint32)
    servers[:3] = [4099, 4098, 9]                             # one Left, in arbitrary order
    order, rtt = p.dcs_by_distance(4097, servers)
    e_order, e_rtt = tq.router_dcs(ref, keys, 4097, 64, servers)
    assert (order == e_order).all() and rtt.tobytes() == e_rtt.tobytes()
    for n_draws, salt in ((1, 0), (255, 1), (257, 2), (100003, 3)):
        got = p.coordinate_error(n_draws, salt)
        exp = tq.error_stats(ref, keys, lat, None, tick_s, cfg.seed, n, n_draws, salt)
        vals = [got[x] for x in ("pairs", "mean", "p50", "p90", "p99", "max")]
        assert np.array(vals).tobytes() == np.array(exp).tobytes(), (n_draws, vals, exp)
    lockstep(pools, 5)                                         # the queries changed nothing


def test_fresh_pool_every_key_ties(cuda_lib):
    """A pool that has not run: every member sits at the origin, every distance is the same, so every digit
    pass of the sort is skipped and the result is the input order; the DC ranking breaks its ties by index."""
    n = 70001
    cfg = wan_config(cuda_lib, capacity=n, n_initial=n, seed=3, flags=FLAG_COORDINATES, mailbox_depth=8)
    p = Pool(cfg, cuda_lib)
    p.latency_set(c5_latency_matrix(8))
    ids, dist = p.sort_by_distance(5)
    assert (ids == np.arange(n)).all() and (dist == 2.0e-5).all()
    rng = np.random.default_rng(4)
    for m in (1, 257, 4097, 65537):
        sel = rng.integers(0, n, m).astype(np.uint32)
        ids, dist = p.sort_by_distance(5, sel, m)
        assert (ids == sel).all() and (dist == 2.0e-5).all()
    order, rtt = p.dcs_by_distance(3 * 128)
    assert list(order) == [3, 0, 1, 2, 4, 5, 6, 7] and rtt[0] == 0.0 and (rtt[1:] == 2.0e-5).all()
    coords = p.coordinates()
    assert (coords == coords[0]).all()
    for n_draws in (n, 4097):                                  # errors tie within each pair class as well
        r = p.coordinate_error(n_draws, 0)
        exp = tq.error_stats(coords, tq.view_keys(p), c5_latency_matrix(8), None, tq.tick_seconds(p), cfg.seed, n,
                             n_draws, 0)
        got = [r[x] for x in ("pairs", "mean", "p50", "p90", "p99", "max")]
        assert np.array(got).tobytes() == np.array(exp).tobytes(), (got, exp)
