"""Pool — one simulated gossip pool (LAN or WAN) of virtual members on one H100.

Thin object wrapper over the C ABI; all simulation state lives in HBM behind libgsim.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import _lib
from ._lib import (AGENT_STATS_FIELDS, COLUMNS, GSIM_MAX_RUMORS, GSIM_MAX_SUSPICION_SLOTS, STAT_NAMES,
                   GsimConfig, GsimEvent, GsimMember, GsimMemberDesc, GsimRumorInfo, GsimStats)

# gsim_agent_stats, one uint32 per field
AGENT_STATS_DTYPE = np.dtype([(n, np.uint32) for n in AGENT_STATS_FIELDS])

IMPAIR_NO_TCP = 1  # GSIM_IMPAIR_NO_TCP

# gsim_domain_stats (fault domains, DESIGN.md §3.5)
DOMAIN_MAX = (1 << 22) - 1  # GSIM_DOMAIN_MAX
DOMAIN_STATS_DTYPE = np.dtype([(n, np.uint32) for n in ("members", "running", "paused", "impaired", "in_force",
                                                        "alive", "suspect", "dead", "left", "awareness_max")]
                              + [("awareness_sum", np.uint64)])

PRED_RUMOR_CONVERGED = 1
PRED_ALL_RUMORS_CONVERGED = 2
PRED_CRASHED_ALL_DEAD = 3
NEVER = 0xFFFFFFFF

FLAG_LOG_GLOBAL_EVENTS = 1
FLAG_NO_GRAPH = 2
FLAG_NO_WINDOWS = 16
FLAG_PUSH_PULL = 32
FLAG_COORDINATES = 64
FLAG_PROBE_PIGGYBACK = 256  # broadcasts ride on pings, acks, indirect pings and nacks (DESIGN.md 3.7)
MEMBER_WATCHED = 1
MAX_DCS = 64  # datacenters of a latency matrix


def _uptr(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_uint32))


def _dptr(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(C.c_double))


class GsimError(RuntimeError):
    def __init__(self, code: int, msg: str):
        super().__init__(f"gsim error {code}: {msg}")
        self.code = code


def lan_config(lib=None, **kw) -> GsimConfig:
    lib = lib or _lib.lib()
    c = GsimConfig()
    lib.gsim_config_default_lan(C.byref(c))
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def wan_config(lib=None, **kw) -> GsimConfig:
    lib = lib or _lib.lib()
    c = GsimConfig()
    lib.gsim_config_default_wan(C.byref(c))
    for k, v in kw.items():
        setattr(c, k, v)
    return c


def consul_test_config(lib=None, **kw) -> GsimConfig:
    lib = lib or _lib.lib()
    c = GsimConfig()
    lib.gsim_config_consul_test(C.byref(c))
    for k, v in kw.items():
        setattr(c, k, v)
    return c


@dataclass
class Event:
    tick: int
    type: int
    subject: int
    observer: int
    ltime: int


class Pool:
    def __init__(self, cfg: GsimConfig, lib=None):
        self.lib = lib or _lib.lib()
        self.cfg = cfg
        h = C.c_void_p()
        rc = self.lib.gsim_pool_create(C.byref(cfg), C.byref(h))
        if rc != 0:
            raise GsimError(rc, self.lib.gsim_strerror(rc).decode())
        self.h = h
        self.capacity = cfg.capacity

    # -- lifecycle -----------------------------------------------------------
    def close(self):
        if getattr(self, "h", None):
            self.lib.gsim_pool_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _ck(self, rc: int):
        if rc != 0:
            msg = self.lib.gsim_last_error(self.h).decode() or self.lib.gsim_strerror(rc).decode()
            raise GsimError(rc, msg)

    # -- membership operations --------------------------------------------------
    def member_add(self, alive_msg_size: int = 0, watched: bool = False, name_len: int = 0, meta_len: int = 0) -> int:
        d = GsimMemberDesc(alive_msg_size, MEMBER_WATCHED if watched else 0, name_len, meta_len)
        out = C.c_uint32()
        self._ck(self.lib.gsim_member_add(self.h, C.byref(d), C.byref(out)))
        return out.value

    def join(self, member: int, seeds, ignore_old: bool = True) -> int:
        arr = (C.c_uint32 * len(seeds))(*seeds)
        n_ok = C.c_int()
        self._ck(self.lib.gsim_join(self.h, member, arr, len(seeds), int(ignore_old), C.byref(n_ok)))
        return n_ok.value

    def leave(self, member: int):
        self._ck(self.lib.gsim_leave(self.h, member))

    def crash(self, member: int):
        self._ck(self.lib.gsim_crash(self.h, member))

    def crash_many(self, ids):
        arr = (C.c_uint32 * len(ids))(*ids)
        self._ck(self.lib.gsim_crash_many(self.h, arr, len(ids)))

    def crash_fraction(self, ppm: int, salt: int = 0) -> int:
        out = C.c_uint32()
        self._ck(self.lib.gsim_crash_fraction(self.h, ppm, salt, C.byref(out)))
        return out.value

    def force_leave(self, via: int, target: int, prune: bool = False):
        self._ck(self.lib.gsim_force_leave(self.h, via, target, int(prune)))

    def user_event(self, member: int, name: bytes, payload: bytes, coalesce: bool = False) -> int:
        out = C.c_uint32()
        self._ck(self.lib.gsim_user_event(self.h, member, name, len(name), payload, len(payload),
                                          int(coalesce), C.byref(out)))
        return out.value

    def rumor_inject(self, slot: int, member: int) -> bool:
        """Out-of-band delivery of tracked broadcast `slot` to `member` (WAN bridges)."""
        out = C.c_int()
        self._ck(self.lib.gsim_rumor_inject(self.h, slot, member, C.byref(out)))
        return bool(out.value)

    def member_watch(self, member: int, on: bool = True):
        self._ck(self.lib.gsim_member_watch(self.h, member, int(on)))

    def member_update(self, member: int, alive_msg_size: int = 0) -> int:
        """(*Serf).SetTags: re-announce under the next incarnation; returns the rumor slot."""
        out = C.c_uint32()
        self._ck(self.lib.gsim_member_update(self.h, member, alive_msg_size, C.byref(out)))
        return out.value

    def graph_set(self, row_ptr, col_idx):
        """CSR peer graph: member i's memberlist = col_idx[row_ptr[i]:row_ptr[i+1]]; None removes it."""
        if row_ptr is None:
            self._ck(self.lib.gsim_graph_set(self.h, 0, None, None))
            return
        rp = np.ascontiguousarray(row_ptr, dtype=np.uint32)
        ci = np.ascontiguousarray(col_idx, dtype=np.uint32)
        self._ck(self.lib.gsim_graph_set(self.h, len(rp) - 1, rp.ctypes.data_as(C.POINTER(C.c_uint32)),
                                         ci.ctypes.data_as(C.POINTER(C.c_uint32))))

    def member_reconnect_timeout_set(self, member: int, timeout_ns: int):
        """serf.Config.ReconnectTimeoutOverride result for one member (0 = the pool's value)."""
        self._ck(self.lib.gsim_member_reconnect_timeout_set(self.h, member, timeout_ns))

    def coordinate(self, member: int):
        """(*Serf).GetCoordinate: (vec[8], error, adjustment, height) in seconds."""
        out = (C.c_double * 11)()
        self._ck(self.lib.gsim_coordinate_get(self.h, member, out))
        v = [float(x) for x in out]
        return v[:8], v[8], v[9], v[10]

    # -- network-coordinate queries (read-only; DESIGN.md §3.4 "Queries") ---------------------------
    def coordinates(self, first: int = 0, count: int | None = None) -> np.ndarray:
        """Coordinates of members [first, first + count) as rows of (vec[8], error, adjustment, height)."""
        if count is None:
            count = self.stats()["n_members"] - first
        out = np.zeros((max(count, 0), 11), dtype=np.float64)
        self._ck(self.lib.gsim_coordinates_read(self.h, first, count, _dptr(out)))
        return out

    def rtt(self, a, b, true_rtt: bool = False):
        """ComputeDistance between a[k] and b[k] in seconds (`consul rtt`); with true_rtt also the round trip
        a direct probe samples in the model: (est, true)."""
        a = np.ascontiguousarray(a, dtype=np.uint32).ravel()
        b = np.ascontiguousarray(b, dtype=np.uint32).ravel()
        if a.shape != b.shape:
            raise ValueError("a and b must have the same length")
        est = np.zeros(len(a), dtype=np.float64)
        tru = np.zeros(len(a), dtype=np.float64) if true_rtt else None
        self._ck(self.lib.gsim_rtt_many(self.h, _uptr(a), _uptr(b), len(a), _dptr(est),
                                        _dptr(tru) if true_rtt else None))
        return (est, tru) if true_rtt else est

    def sort_by_distance(self, frm: int, ids=None, k: int | None = None):
        """sortNodesByDistanceFrom: (ids, distances) of the k nearest of `ids` (None: every member), stable."""
        if ids is None:
            n = self.stats()["n_members"]
            arr = None
        else:
            arr = np.ascontiguousarray(ids, dtype=np.uint32).ravel()
            n = len(arr)
        k = n if k is None else k
        out = np.zeros(k, dtype=np.uint32)
        dist = np.zeros(k, dtype=np.float64)
        self._ck(self.lib.gsim_sort_by_distance(self.h, frm, _uptr(arr) if arr is not None else None,
                                                n if arr is not None else 0, k, _uptr(out), _dptr(dist)))
        return out, dist

    def dcs_by_distance(self, frm: int, servers=None):
        """Router.GetDatacentersByDistance seen from `frm`: (datacenter indices, median RTTs), nearest first;
        datacenters without a counted server are left out, as upstream."""
        order = np.zeros(MAX_DCS, dtype=np.uint32)
        rtt = np.full(MAX_DCS, np.nan)                 # entries past n_dcs stay NaN
        arr = None if servers is None else np.ascontiguousarray(servers, dtype=np.uint32).ravel()
        self._ck(self.lib.gsim_dcs_by_distance(self.h, frm, _uptr(arr) if arr is not None else None,
                                               0 if arr is None else len(arr), _uptr(order), _dptr(rtt)))
        keep = np.isfinite(rtt)
        return order[keep], rtt[keep]

    def coordinate_error(self, n_draws: int, salt: int = 0) -> dict:
        """Relative error of the embedding against the model's round trips over seeded member pairs."""
        out = (C.c_double * 6)()
        self._ck(self.lib.gsim_coordinate_error(self.h, n_draws, salt, out))
        return dict(zip(("pairs", "mean", "p50", "p90", "p99", "max"), [int(out[0])] + [float(x) for x in out[1:]]))

    def latency_set(self, lat):
        """lat: square matrix (n_dcs x n_dcs) of one-way latencies in ticks (>= 1), or None."""
        if lat is None:
            self._ck(self.lib.gsim_latency_set(self.h, 0, None))
            return
        m = np.ascontiguousarray(lat, dtype=np.uint8)
        assert m.ndim == 2 and m.shape[0] == m.shape[1]
        self._ck(self.lib.gsim_latency_set(self.h, m.shape[0], m.ctypes.data_as(C.POINTER(C.c_uint8))))

    def impair(self, ids, loss_ppm: int, delay_ticks: int = 0):
        """Degrade the listed members: UDP loss to and from each (ppm) and a receive delay (ticks);
        (0, 0) clears it."""
        arr = (C.c_uint32 * max(1, len(ids)))(*ids)
        self._ck(self.lib.gsim_impair_many(self.h, arr, len(ids), loss_ppm, delay_ticks))

    def impair_fraction(self, member_ppm: int, salt: int, loss_ppm: int, delay_ticks: int = 0) -> int:
        """Degrade a seeded fraction (ppm) of the running members; returns how many were selected."""
        out = C.c_uint32()
        self._ck(self.lib.gsim_impair_fraction(self.h, member_ppm, salt, loss_ppm, delay_ticks, C.byref(out)))
        return out.value

    def impairment(self, member: int):
        """(loss_ppm, delay_ticks) of one member, as set."""
        loss, delay = C.c_uint32(), C.c_uint32()
        self._ck(self.lib.gsim_impair_get(self.h, member, C.byref(loss), C.byref(delay)))
        return loss.value, delay.value

    def impair_dir(self, ids, send_loss_ppm: int, recv_loss_ppm: int, delay_ticks: int = 0, no_tcp: bool = False):
        """One-way reachability for the listed members: UDP loss of what each sends and of what it
        receives (ppm), a receive delay (ticks) and, with no_tcp, no TCP to or from it (no fallback
        ping, no push-pull, no join through it).  (0, 0, 0, False) clears it."""
        arr = (C.c_uint32 * max(1, len(ids)))(*ids)
        self._ck(self.lib.gsim_impair_dir_many(self.h, arr, len(ids), send_loss_ppm, recv_loss_ppm, delay_ticks,
                                               IMPAIR_NO_TCP if no_tcp else 0))

    def impair_dir_fraction(self, member_ppm: int, salt: int, send_loss_ppm: int, recv_loss_ppm: int,
                            delay_ticks: int = 0, no_tcp: bool = False) -> int:
        """impair_dir on the members impair_fraction selects for the same salt; returns how many."""
        out = C.c_uint32()
        self._ck(self.lib.gsim_impair_dir_fraction(self.h, member_ppm, salt, send_loss_ppm, recv_loss_ppm,
                                                   delay_ticks, IMPAIR_NO_TCP if no_tcp else 0, C.byref(out)))
        return out.value

    def impairment_dir(self, member: int):
        """(send_loss_ppm, recv_loss_ppm, delay_ticks, no_tcp) of one member, as set."""
        send, recv, delay, flags = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_uint32()
        self._ck(self.lib.gsim_impair_dir_get(self.h, member, C.byref(send), C.byref(recv), C.byref(delay),
                                              C.byref(flags)))
        return send.value, recv.value, delay.value, bool(flags.value & IMPAIR_NO_TCP)

    def impair_flap(self, ids, period_ticks: int, bad_ppm: int):
        """Make the impairment of the listed members intermittent: in force only during bad epochs of
        `period_ticks` ticks, each bad with probability bad_ppm / 1e6.  period_ticks 0 clears the schedule
        (impairment always in force)."""
        arr = (C.c_uint32 * max(1, len(ids)))(*ids)
        self._ck(self.lib.gsim_impair_flap_many(self.h, arr, len(ids), period_ticks, bad_ppm))

    def impair_flap_fraction(self, member_ppm: int, salt: int, period_ticks: int, bad_ppm: int) -> int:
        """impair_flap on the members impair_fraction selects for the same salt; returns how many."""
        out = C.c_uint32()
        self._ck(self.lib.gsim_impair_flap_fraction(self.h, member_ppm, salt, period_ticks, bad_ppm, C.byref(out)))
        return out.value

    def impair_flap_get(self, member: int):
        """(period_ticks, bad_ppm) of one member's schedule, (0, 0) without one."""
        period, ppm = C.c_uint32(), C.c_uint32()
        self._ck(self.lib.gsim_impair_flap_get(self.h, member, C.byref(period), C.byref(ppm)))
        return period.value, ppm.value

    def flap_stats(self):
        """{'scheduled', 'bad'}: members with a schedule, and those of them in a bad epoch now."""
        out = (C.c_uint64 * 2)()
        self._ck(self.lib.gsim_impair_flap_stats(self.h, out))
        return {"scheduled": out[0], "bad": out[1]}

    def pause(self, ids, ticks: int) -> int:
        """Stop the listed members (running, not leaving) for `ticks` ticks; returns how many were paused."""
        arr = (C.c_uint32 * max(1, len(ids)))(*ids)
        out = C.c_uint32()
        self._ck(self.lib.gsim_pause_many(self.h, arr, len(ids), ticks, C.byref(out)))
        return out.value

    def pause_fraction(self, member_ppm: int, salt: int, ticks: int) -> int:
        """Stop a seeded fraction (ppm) of the running members for `ticks` ticks; returns how many."""
        out = C.c_uint32()
        self._ck(self.lib.gsim_pause_fraction(self.h, member_ppm, salt, ticks, C.byref(out)))
        return out.value

    def paused_until(self, member: int) -> int:
        """The tick the member resumes at, NEVER when it is not paused."""
        out = C.c_uint32()
        self._ck(self.lib.gsim_pause_get(self.h, member, C.byref(out)))
        return out.value

    def pause_stats(self):
        """{'paused', 'resumed_alive', 'resumed_suspect', 'resumed_dead'}"""
        out = (C.c_uint64 * 4)()
        self._ck(self.lib.gsim_pause_stats(self.h, out))
        return dict(zip(("paused", "resumed_alive", "resumed_suspect", "resumed_dead"), out))

    # -- fault domains (DESIGN.md §3.5 "Fault domains") -------------------------------
    def domain_set(self, ids, domain: int):
        """Put the listed members in fault domain `domain` (1 .. DOMAIN_MAX); 0 takes them out of any."""
        arr = (C.c_uint32 * max(1, len(ids)))(*ids)
        self._ck(self.lib.gsim_domain_set_many(self.h, arr, len(ids), domain))

    def domain_set_range(self, first: int, count: int, per_domain: int, first_domain: int = 1):
        """Member first + x goes to domain first_domain + x // per_domain: racks of per_domain members."""
        self._ck(self.lib.gsim_domain_set_range(self.h, first, count, per_domain, first_domain))

    def domains(self, first: int = 0, count: int | None = None) -> np.ndarray:
        """The domain of members [first, first + count) as a uint32 array (0 = none)."""
        if count is None:
            count = self.stats()["n_members"] - first
        out = np.zeros(max(count, 0), dtype=np.uint32)
        self._ck(self.lib.gsim_domain_get(self.h, first, count, out.ctypes.data_as(C.c_void_p)))
        return out

    def domain_flap(self, domains, period_ticks: int, bad_ppm: int):
        """Give the listed domains a flap schedule: their members' impairments are in force only during the
        domain's bad epochs (and their own, if they have one).  period_ticks 0 clears it."""
        arr = (C.c_uint32 * max(1, len(domains)))(*domains)
        self._ck(self.lib.gsim_domain_flap_set(self.h, arr, len(domains), period_ticks, bad_ppm))

    def domain_flap_get(self, domain: int):
        """(period_ticks, bad_ppm) of one domain's schedule, (0, 0) without one."""
        period, ppm = C.c_uint32(), C.c_uint32()
        self._ck(self.lib.gsim_domain_flap_get(self.h, domain, C.byref(period), C.byref(ppm)))
        return period.value, ppm.value

    def domain_impair(self, domains, send_loss_ppm: int, recv_loss_ppm: int, delay_ticks: int = 0,
                      flags: int = 0) -> int:
        """impair_dir_many over every member of the listed domains; returns how many members."""
        arr = (C.c_uint32 * max(1, len(domains)))(*domains)
        out = C.c_uint32()
        self._ck(self.lib.gsim_domain_impair(self.h, arr, len(domains), send_loss_ppm, recv_loss_ppm, delay_ticks,
                                             flags, C.byref(out)))
        return out.value

    def domain_crash(self, domains) -> int:
        """crash_many over every member of the listed domains; returns how many running members crashed."""
        arr = (C.c_uint32 * max(1, len(domains)))(*domains)
        out = C.c_uint32()
        self._ck(self.lib.gsim_domain_crash(self.h, arr, len(domains), C.byref(out)))
        return out.value

    def domain_pause(self, domains, ticks: int) -> int:
        """pause_many over every member of the listed domains; returns how many were paused."""
        arr = (C.c_uint32 * max(1, len(domains)))(*domains)
        out = C.c_uint32()
        self._ck(self.lib.gsim_domain_pause(self.h, arr, len(domains), ticks, C.byref(out)))
        return out.value

    def domain_stats(self, first: int, count: int) -> np.ndarray:
        """Per-domain counts of domains [first, first + count), read on the device, as a structured array with
        the fields of DOMAIN_STATS_DTYPE."""
        out = np.zeros(max(count, 0), dtype=DOMAIN_STATS_DTYPE)
        self._ck(self.lib.gsim_domain_stats_read(self.h, first, count, out.ctypes.data_as(C.c_void_p)))
        return out

    # -- time ---------------------------------------------------------------------
    def step(self, ticks: int = 1):
        self._ck(self.lib.gsim_step(self.h, ticks))

    def run_until(self, predicate: int, arg: int = 0, max_ticks: int = 10000,
                  check_every: int = 16) -> int:
        out = C.c_uint32()
        self._ck(self.lib.gsim_run_until(self.h, predicate, arg, max_ticks, check_every,
                                         C.byref(out)))
        return out.value

    @property
    def now(self) -> int:
        return self.lib.gsim_now(self.h)

    # -- observation ------------------------------------------------------------------
    def members(self, observer: int):
        n = C.c_size_t()
        self._ck(self.lib.gsim_members(self.h, observer, None, 0, C.byref(n)))
        buf = (GsimMember * max(1, n.value))()
        self._ck(self.lib.gsim_members(self.h, observer, buf, n.value, C.byref(n)))
        return [(m.id, m.status, m.incarnation, m.rank) for m in buf[: n.value]]

    def num_nodes(self, observer: int) -> int:
        out = C.c_uint32()
        self._ck(self.lib.gsim_num_nodes(self.h, observer, C.byref(out)))
        return out.value

    def agent_stats(self, first: int = 0, count: int | None = None) -> np.ndarray:
        """(*Serf).Stats() of members [first, first + count), computed on the device, as a structured array
        with the fields of AGENT_STATS_DTYPE (DESIGN.md §3.8)."""
        if count is None:
            count = self.stats()["n_members"] - first
        out = np.zeros(max(count, 0), dtype=AGENT_STATS_DTYPE)
        self._ck(self.lib.gsim_agent_stats_read(self.h, first, count, out.ctypes.data_as(C.c_void_p)))
        return out

    def health_histogram(self) -> np.ndarray:
        """Running members by health score (awareness): row 0 without an impairment, row 1 with one."""
        out = np.zeros((2, 8), dtype=np.uint64)
        self._ck(self.lib.gsim_health_histogram(self.h, out.ctypes.data_as(C.POINTER(C.c_uint64))))
        return out

    def poll_events(self, cap: int = 65536):
        buf = (GsimEvent * cap)()
        n = C.c_size_t()
        self._ck(self.lib.gsim_poll_events(self.h, buf, cap, C.byref(n)))
        return [Event(e.tick, e.type, e.subject, e.observer, e.ltime) for e in buf[: n.value]]

    def rumor_info(self, slot: int) -> dict:
        out = GsimRumorInfo()
        self._ck(self.lib.gsim_rumor_info_get(self.h, slot, C.byref(out)))
        return {n: getattr(out, n) for n, _ in GsimRumorInfo._fields_}

    def rumor_retire(self, slot: int):
        self._ck(self.lib.gsim_rumor_retire(self.h, slot))

    def user_event_get(self, slot: int):
        nl, pl = C.c_size_t(), C.c_size_t()
        nb, pb = C.create_string_buffer(1024), C.create_string_buffer(1024)
        self._ck(self.lib.gsim_user_event_get(self.h, slot, nb, 1024, C.byref(nl), pb, 1024,
                                              C.byref(pl)))
        return nb.raw[: nl.value], pb.raw[: pl.value]

    def stats(self) -> dict:
        s = GsimStats()
        self._ck(self.lib.gsim_stats_get(self.h, C.byref(s)))
        out = {n: int(s.counters[i]) for i, n in enumerate(STAT_NAMES)}
        for n, _ in GsimStats._fields_:
            if n == "counters":
                continue
            v = getattr(s, n)
            out[n] = list(v) if n == "suspicion_ticks" else int(v)
        return out

    def state_hash(self):
        out = (C.c_uint64 * 4)()
        self._ck(self.lib.gsim_state_hash(self.h, out))
        return tuple(int(x) for x in out)

    def column(self, name: str) -> np.ndarray:
        cap = self.capacity
        if name == "tx":
            arr = np.zeros((GSIM_MAX_RUMORS, cap), dtype=np.uint8)
        elif name == "sus_from":
            arr = np.zeros((GSIM_MAX_SUSPICION_SLOTS, cap), dtype=np.uint32)
        else:
            arr = np.zeros(cap, dtype=np.uint32)
        n = C.c_size_t()
        self._ck(self.lib.gsim_column_read(self.h, COLUMNS[name], arr.ctypes.data_as(C.c_void_p),
                                           arr.nbytes, C.byref(n)))
        return arr

    # -- checkpoint -----------------------------------------------------------------------
    def snapshot(self) -> bytes:
        n = C.c_size_t()
        self._ck(self.lib.gsim_snapshot_size(self.h, C.byref(n)))
        buf = C.create_string_buffer(n.value)
        self._ck(self.lib.gsim_snapshot(self.h, buf, n.value, C.byref(n)))
        return buf.raw[: n.value]

    def restore(self, blob: bytes):
        self._ck(self.lib.gsim_restore(self.h, blob, len(blob)))

    # -- measurement ----------------------------------------------------------------------
    def last_step_timing(self):
        ms = C.c_double()
        n = C.c_uint64()
        self._ck(self.lib.gsim_last_step_timing(self.h, C.byref(ms), C.byref(n)))
        return ms.value, n.value

    def sched_counts(self) -> dict:
        out = (C.c_uint64 * 8)()
        self._ck(self.lib.gsim_sched_counts(self.h, out))
        return {"window_launches": int(out[0]), "window_ticks": int(out[1]), "tick_launches": int(out[2]),
                "horizon_scans": int(out[3]), "window_ms": out[4] / 1e6, "tick_ms": out[5] / 1e6,
                "closed_form_launches": int(out[6]), "closed_form_ticks": int(out[7])}

    def piggyback_stats(self) -> dict:
        """Probe traffic that carried broadcasts (pools created with FLAG_PROBE_PIGGYBACK)."""
        out = (C.c_uint64 * 4)()
        self._ck(self.lib.gsim_piggyback_stats(self.h, out))
        return {"packets": int(out[0]), "broadcasts": int(out[1]), "owed_served": int(out[2]),
                "owed_dropped": int(out[3])}

    def launch_count(self) -> int:
        return int(self.lib.gsim_launch_count(self.h))
