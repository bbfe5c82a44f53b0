"""Network-coordinate queries (DESIGN.md §3.4 "Queries") on the host emulation: bulk coordinates, RTT
estimates, the ?near= order, the datacenter ranking of the router and the accuracy of the embedding, each
against an independent restatement over the ORACLE's coordinates (oracle pool run in lockstep), and each
read-only.  The restatements are shared with tests/test_gpu_coord_queries.py."""
import ctypes as C

import numpy as np
import pytest

import scenarios as sc
from consul_b200.pool import FLAG_COORDINATES, GsimError, Pool, lan_config, wan_config
from consul_b200.wan import c5_latency_matrix
from oracle_binding import OraclePool, oracle_lib
from oracle_impair import ImpairOraclePool

ERR_INVALID, ERR_NOT_FOUND, ERR_STATE = -1, -5, -6
TILE = 128


# ---- restatements ---------------------------------------------------------------------------------
def oracle_coords(o, n):
    """(n, 11) array of the oracle's coordinates (oracle_coordinate_get, one member at a time)."""
    out = np.zeros((n, 11))
    buf = (C.c_double * 11)()
    for i in range(n):
        assert o.lib.oracle_coordinate_get(o.h, i, buf) == 0
        out[i] = buf[:]
    return out


def distance(ca, cb):
    """Coordinate.DistanceTo(other).Seconds() for rows of 11 doubles, in upstream's textual operation order
    (elementwise IEEE doubles: numpy never fuses a multiply and an add), through time.Duration."""
    ca, cb = np.atleast_2d(ca), np.atleast_2d(cb)
    s = np.zeros(max(len(ca), len(cb)))
    for x in range(8):
        d = ca[:, x] - cb[:, x]
        s = s + d * d
    raw = np.sqrt(s) + ca[:, 10] + cb[:, 10]
    adj = raw + ca[:, 9] + cb[:, 9]
    dist = np.where(adj > 0.0, adj, raw)
    ns = (dist * 1.0e9).astype(np.int64)                     # int64(float) truncates, as Go's conversion
    return (ns // 1000000000).astype(np.float64) + (ns % 1000000000).astype(np.float64) / 1.0e9


def extra(lat, delay, src, dst):
    """Extra one-way ticks from src to dst: the matrix entry - 1 between their datacenters, plus dst's delay."""
    e = np.zeros(len(src), dtype=np.int64)
    if lat is not None:
        nd = lat.shape[0]
        e += lat[(src // TILE) % nd, (dst // TILE) % nd].astype(np.int64) - 1
    if delay is not None:
        e += delay[dst]
    return e


def model_rtt(lat, delay, tick_s, a, b):
    return 0.0005 + (extra(lat, delay, a, b) + extra(lat, delay, b, a)).astype(np.float64) * tick_s


def stable_order(ids, dist):
    idx = np.argsort(dist, kind="stable")
    return np.asarray(ids)[idx], dist[idx]


def router_dcs(coords, keys, frm, n_dcs, servers=None):
    """GetDatacentersByDistance for one area: (dc order, median RTTs) of the datacenters with a counted server."""
    servers = np.arange(len(keys)) if servers is None else np.asarray(servers)
    truth, rank = keys[servers] & 3, (keys[servers] >> 2) & 3
    keep = servers[(truth != 0) & (rank != 3)]
    dc = (keep // TILE) % n_dcs
    mine = (frm // TILE) % n_dcs
    rtt = distance(coords[frm][None, :].repeat(len(keep), 0), coords[keep]) if len(keep) else np.zeros(0)
    rtt = np.where(dc == mine, 0.0, rtt)
    med = {}
    for c in range(n_dcs):
        r = np.sort(rtt[dc == c])
        if len(r):
            med[c] = r[len(r) // 2]
    names = sorted(med)                                        # synthetic names ordered by index
    names = sorted(names, key=lambda c: med[c])                # then the stable sort by median RTT
    return np.array(names, dtype=np.uint32), np.array([med[c] for c in names])


def philox(seed, c0, c1, c2, c3):
    """Philox4x32-10 over arrays of counters (Salmon et al. 2011)."""
    M0, M1, W0, W1 = np.uint64(0xD2511F53), np.uint64(0xCD9E8D57), 0x9E3779B9, 0xBB67AE85
    k0, k1 = seed & 0xFFFFFFFF, seed >> 32
    c = [np.asarray(v, dtype=np.uint64) & np.uint64(0xFFFFFFFF) for v in np.broadcast_arrays(c0, c1, c2, c3)]
    mask = np.uint64(0xFFFFFFFF)
    for _ in range(10):
        p0, p1 = M0 * c[0], M1 * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ np.uint64(k0), p1 & mask, (p0 >> np.uint64(32)) ^ c[3] ^ np.uint64(k1),
             p0 & mask]
        k0, k1 = (k0 + W0) & 0xFFFFFFFF, (k1 + W1) & 0xFFFFFFFF
    return c


def error_stats(coords, keys, lat, delay, tick_s, seed, n, n_draws, salt):
    """gsim_coordinate_error restated: draws, kept pairs, relative errors, chunked mean, order statistics."""
    k = np.arange(n_draws, dtype=np.uint64)
    r = philox(seed, k, salt, 11, 0)
    i, j = (r[0] % np.uint64(n)).astype(np.int64), (r[1] % np.uint64(n)).astype(np.int64)
    up = (keys & 3) == 1
    kept = (i != j) & up[i] & up[j]
    i, j = i[kept], j[kept]
    est = distance(coords[i], coords[j])
    tru = model_rtt(lat, delay, tick_s, i, j)
    err = np.abs(est - tru) / tru
    m = len(err)
    if m == 0:
        return [0.0] + [float("nan")] * 5
    chunk = np.arange(n_draws)[kept] // 256
    total = 0.0
    for c in np.unique(chunk):
        part = np.cumsum(err[chunk == c])[-1]                  # cumsum adds strictly in order
        total = total + float(part)
    s = np.sort(err)
    q = lambda f: s[int(f * (m - 1))]
    return [float(m), total / m, q(0.5), q(0.9), q(0.99), s[-1]]


def tick_seconds(pool):
    """The pool's tick in seconds, as libgsim derives it (whole nanoseconds / 1e9)."""
    return (pool.cfg.probe_interval_ns // pool.stats()["probe_interval_ticks"]) / 1.0e9


def view_keys(pool, now=None):
    """The key column the queries read at `now` (key buffer now & 1)."""
    return pool.column("key").astype(np.int64)


def observables(p):
    cols = {c: p.column(c).tobytes() for c in ("key", "meta", "due", "cursor", "heard", "queued", "inbox")}
    return p.state_hash(), p.stats(), p.sched_counts(), cols


# ---- pools ----------------------------------------------------------------------------------------------
def lan_pool(lib, n=3 * TILE + 40, seed=3):
    cfg = lan_config(lib, capacity=n + 4, n_initial=n, seed=seed, flags=FLAG_COORDINATES)
    return cfg, None, None


def wan_slow_pool(lib, n=6 * TILE + 17, seed=7):
    # one-way latencies up to 4 ticks: some round trips exceed WAN's ProbeTimeout and take the slow path
    cfg = wan_config(lib, capacity=n + 4, n_initial=n, seed=seed, flags=FLAG_COORDINATES, mailbox_depth=8,
                     packet_loss_ppm=50000)
    a, b = np.arange(4)[:, None], np.arange(4)[None, :]
    m = (1 + (3 * a + 5 * b) % 4).astype(np.uint8)
    m[np.arange(4), np.arange(4)] = 1
    return cfg, m, None


def run_pools(lib, kind, ticks=300):
    cfg, lat, _ = {"lan": lan_pool, "wan": wan_slow_pool, "impaired": lambda l: wan_slow_pool(l, seed=9)}[kind](lib)
    pools = [Pool(cfg, lib), (ImpairOraclePool if kind == "impaired" else OraclePool)(cfg)]
    delay = None
    for p in pools:
        if lat is not None:
            p.latency_set(lat)
    if kind == "impaired":
        ids = list(range(3, cfg.n_initial, 11))
        for p in pools:
            p.impair(ids, 0, 1)
        delay = np.zeros(cfg.capacity, dtype=np.int64)
        delay[ids] = 1
    sc.step_compare(pools, ticks, 100, kind)
    tick_s = tick_seconds(pools[0])
    return pools, cfg, lat, delay, tick_s


@pytest.fixture(scope="module", params=["lan", "wan", "impaired"])
def world(request, hostemu_lib):
    return run_pools(hostemu_lib, request.param)


def test_coordinates_bulk_equals_getter_and_oracle(world):
    (p, o), cfg, *_ = world
    n = cfg.n_initial
    got = p.coordinates()
    assert got.shape == (n, 11)
    ref = oracle_coords(o, n)
    assert got.tobytes() == ref.tobytes()
    for i in (0, 1, n // 2, n - 1):
        vec, err, adj, h = p.coordinate(i)
        assert got[i].tobytes() == np.array(vec + [err, adj, h]).tobytes()
    assert p.coordinates(5, 7).tobytes() == got[5:12].tobytes()
    assert p.coordinates(n, 0).shape == (0, 11)


def test_rtt_equals_restated_distance_and_model(world):
    (p, o), cfg, lat, delay, tick_s = world
    n = cfg.n_initial
    coords = oracle_coords(o, n)
    rng = np.random.default_rng(1)
    a, b = rng.integers(0, n, 3000), rng.integers(0, n, 3000)
    a[:5] = b[:5]                                              # a member to itself
    est, tru = p.rtt(a, b, true_rtt=True)
    assert est.tobytes() == distance(coords[a], coords[b]).tobytes()
    assert tru.tobytes() == model_rtt(lat, delay, tick_s, a, b).tobytes()
    assert p.rtt(a, b).tobytes() == est.tobytes()


def test_sort_by_distance_is_a_stable_sort(world):
    (p, o), cfg, *_ = world
    n = cfg.n_initial
    coords = oracle_coords(o, n)
    rng = np.random.default_rng(2)
    for frm in (0, 200, n - 1):
        ids, dist = p.sort_by_distance(frm)
        e_ids, e_dist = stable_order(np.arange(n), distance(coords[frm], coords))
        assert (ids == e_ids).all() and dist.tobytes() == e_dist.tobytes()
        assert (np.diff(dist) >= 0).all()
        # duplicates and an arbitrary input order; every k
        sel = rng.integers(0, n, 300)
        sel[:40] = sel[40:80]
        e_ids, e_dist = stable_order(sel, distance(coords[frm], coords[sel]))
        for k in (1, 2, 17, 299, 300):
            ids, dist = p.sort_by_distance(frm, sel, k)
            assert (ids == e_ids[:k]).all() and dist.tobytes() == e_dist[:k].tobytes()
    assert p.sort_by_distance(0, [], 0)[0].shape == (0,)


def test_sort_ties_keep_input_order(hostemu_lib):
    """Members of one datacenter that were never probed share the origin: every distance ties."""
    cfg = lan_config(hostemu_lib, capacity=70000, n_initial=65537, seed=1, flags=FLAG_COORDINATES)
    p = Pool(cfg, hostemu_lib)
    rng = np.random.default_rng(3)
    for n in (0, 1, 255, 256, 257, 4096, 4097, 65537):
        sel = rng.integers(0, 65537, n).astype(np.uint32)
        ids, dist = p.sort_by_distance(7, sel, n)
        assert (ids == sel).all() and (dist == 2.0e-5).all()
    ids, _ = p.sort_by_distance(7)
    assert (ids == np.arange(65537)).all()
    p.step(30)                                                 # some members have moved, most still tie
    coords = p.coordinates()
    for n in (255, 256, 257, 65537):
        sel = rng.integers(0, 65537, n).astype(np.uint32)
        e_ids, e_dist = stable_order(sel, distance(coords[9], coords[sel]))
        ids, dist = p.sort_by_distance(9, sel, n)
        assert (ids == e_ids).all() and dist.tobytes() == e_dist.tobytes()


def test_dcs_by_distance_restates_the_router(hostemu_lib):
    n = 8 * TILE * 3
    cfg = wan_config(hostemu_lib, capacity=n + 4, n_initial=n, seed=13, flags=FLAG_COORDINATES, mailbox_depth=8)
    pools = [Pool(cfg, hostemu_lib), OraclePool(cfg)]
    lat = c5_latency_matrix(8)
    for q in pools:
        q.latency_set(lat)
    sc.step_compare(pools, 200, 100, "dcs")
    for q in pools:
        q.leave(130)
        q.crash_many([131, 300])
    sc.step_compare(pools, 200, 100, "dcs after leave")
    p, o = pools
    keys = view_keys(p)
    assert (keys[130] >> 2) & 3 == 3 and keys[300] & 3 == 2   # listed Left; crashed and still counted
    coords = oracle_coords(o, n)
    for frm in (0, 129, 1000):
        order, rtt = p.dcs_by_distance(frm)
        e_order, e_rtt = router_dcs(coords, keys, frm, 8)
        assert (order == e_order).all() and rtt.tobytes() == e_rtt.tobytes()
        assert order[0] == (frm // TILE) % 8 and rtt[0] == 0.0
    sel = [1, 2, 130, 131, 300, 700, 701, 702, 1020]
    order, rtt = p.dcs_by_distance(5, sel)
    e_order, e_rtt = router_dcs(coords, keys, 5, 8, sel)
    assert (order == e_order).all() and rtt.tobytes() == e_rtt.tobytes()
    # ties between datacenters break by index: every member at the origin
    q = Pool(cfg, hostemu_lib)
    q.latency_set(lat)
    order, rtt = q.dcs_by_distance(3 * TILE)
    assert list(order) == [3, 0, 1, 2, 4, 5, 6, 7] and rtt[0] == 0.0 and (rtt[1:] == 2.0e-5).all()


def test_dcs_by_distance_skips_reaped_members(hostemu_lib):
    n = 4 * TILE
    cfg = wan_config(hostemu_lib, capacity=n + 4, n_initial=n, seed=21, flags=FLAG_COORDINATES, mailbox_depth=8,
                     reconnect_timeout_ns=30 * 10**9, reap_interval_ns=5 * 10**9, tombstone_timeout_ns=30 * 10**9)
    p = Pool(cfg, hostemu_lib)
    p.latency_set(c5_latency_matrix(4))
    gone = list(range(TILE, 2 * TILE))                         # all of datacenter 1
    p.crash_many(gone)
    p.step(600)
    keys = view_keys(p)
    assert (keys[gone] & 3 == 0).all()                         # reaped: no such member any more
    order, rtt = p.dcs_by_distance(0)
    assert 1 not in order and len(order) == 3
    e_order, e_rtt = router_dcs(p.coordinates(), keys, 0, 4)
    assert (order == e_order).all() and rtt.tobytes() == e_rtt.tobytes()


def test_coordinate_error_restated(world):
    (p, o), cfg, lat, delay, tick_s = world
    n = cfg.n_initial
    coords = oracle_coords(o, n)
    keys = view_keys(p)
    for n_draws, salt in ((1, 0), (255, 3), (256, 3), (257, 3), (n, 9)):
        got = p.coordinate_error(n_draws, salt)
        exp = error_stats(coords, keys, lat, delay, tick_s, cfg.seed, n, n_draws, salt)
        vals = [got[k] for k in ("pairs", "mean", "p50", "p90", "p99", "max")]
        assert np.array(vals, dtype=np.float64).tobytes() == np.array(exp).tobytes(), (n_draws, vals, exp)


def test_philox_restatement_matches_the_oracle():
    lib = oracle_lib()
    out = (C.c_uint32 * 4)()
    for ctr, seed in (([5, 7, 11, 0], 3), ([0xFFFFFFFF, 1, 11, 0], 0x123456789ABCDEF)):
        lib.oracle_philox4x32((C.c_uint32 * 4)(*ctr), (C.c_uint32 * 2)(seed & 0xFFFFFFFF, seed >> 32), out)
        assert [int(v) for v in philox(seed, *ctr)] == list(out)


def test_queries_are_read_only(world):
    (p, o), cfg, lat, *_ = world
    before = observables(p)
    p.coordinates()
    p.rtt([0, 1], [2, 3], true_rtt=True)
    p.sort_by_distance(1)
    p.sort_by_distance(1, [4, 4, 2], 2)
    p.coordinate_error(500, 1)
    if lat is not None:
        p.dcs_by_distance(2)
    assert observables(p) == before
    p.step(50)
    o.step(50)
    assert p.state_hash() == o.state_hash()


def test_validation(hostemu_lib):
    p = Pool(lan_config(hostemu_lib, capacity=300, n_initial=300, seed=1), hostemu_lib)
    for call in (lambda: p.coordinates(), lambda: p.rtt([0], [1]), lambda: p.sort_by_distance(0),
                 lambda: p.dcs_by_distance(0), lambda: p.coordinate_error(10)):
        with pytest.raises(GsimError) as e:
            call()
        assert e.value.code == ERR_STATE                       # created without GSIM_FLAG_COORDINATES
    q = Pool(lan_config(hostemu_lib, capacity=300, n_initial=300, seed=1, flags=FLAG_COORDINATES), hostemu_lib)
    for call, code in ((lambda: q.coordinates(299, 2), ERR_NOT_FOUND), (lambda: q.rtt([0, 300], [1, 2]), ERR_NOT_FOUND),
                       (lambda: q.rtt([0], [300]), ERR_NOT_FOUND), (lambda: q.sort_by_distance(300), ERR_NOT_FOUND),
                       (lambda: q.sort_by_distance(0, [1, 300]), ERR_NOT_FOUND),
                       (lambda: q.sort_by_distance(0, [1, 2], 3), ERR_INVALID),
                       (lambda: q.sort_by_distance(0, [1] * 100000), ERR_INVALID),
                       (lambda: q.dcs_by_distance(0), ERR_STATE),  # no latency matrix
                       (lambda: q.coordinate_error(0), ERR_INVALID), (lambda: q.coordinate_error(100000), ERR_INVALID)):
        with pytest.raises(GsimError) as e:
            call()
        assert e.value.code == code
    q.latency_set(np.ones((2, 2), dtype=np.uint8))
    with pytest.raises(GsimError) as e:
        q.dcs_by_distance(300)
    assert e.value.code == ERR_NOT_FOUND
    with pytest.raises(GsimError) as e:
        q.dcs_by_distance(0, [0, 400])
    assert e.value.code == ERR_NOT_FOUND
    assert q.rtt([], []).shape == (0,)
    r = q.coordinate_error(300, 0)                             # every member at the origin: 2e-5 s vs 0.5 ms
    assert r["pairs"] > 250 and r["max"] == r["p50"] == abs(2.0e-5 - 0.0005) / 0.0005
