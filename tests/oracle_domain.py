"""ctypes binding of tests/oracle_domain/liboracle_domain.so — TEST INFRASTRUCTURE.

That library is the oracle with degraded, paused, one-way and flapping members (impair.patch, pause.patch,
reach.patch, flap.patch) and fault domains (tests/oracle_domain/domain.patch) restated on top, applied by
`__graft_entry__.build()`; `DomainOraclePool` drives it with the methods of `FlapOraclePool` plus those of
`consul_b200.pool.Pool` for fault domains.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from consul_b200.pool import DOMAIN_STATS_DTYPE, GsimError
from oracle_binding import _SIGS
from oracle_flap import _FLAP_SIGS, FlapOraclePool
from oracle_impair import _IMPAIR_SIGS
from oracle_pause import _PAUSE_SIGS
from oracle_reach import _REACH_SIGS

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBORACLE_DOMAIN = os.path.join(ROOT, "tests", "oracle_domain", "liboracle_domain.so")

_u32, _sz, _P = C.c_uint32, C.c_size_t, C.c_void_p
_DOMAIN_SIGS = [
    ("oracle_domain_set_many", C.c_int, [_P, C.POINTER(_u32), _sz, _u32]),
    ("oracle_domain_set_range", C.c_int, [_P, _u32, _u32, _u32, _u32]),
    ("oracle_domain_get", C.c_int, [_P, _u32, _u32, _P]),
    ("oracle_domain_flap_set", C.c_int, [_P, C.POINTER(_u32), _sz, _u32, _u32]),
    ("oracle_domain_flap_get", C.c_int, [_P, _u32, C.POINTER(_u32), C.POINTER(_u32)]),
    ("oracle_domain_impair", C.c_int, [_P, C.POINTER(_u32), _sz, _u32, _u32, _u32, _u32, C.POINTER(_u32)]),
    ("oracle_domain_crash", C.c_int, [_P, C.POINTER(_u32), _sz, C.POINTER(_u32)]),
    ("oracle_domain_pause", C.c_int, [_P, C.POINTER(_u32), _sz, _u32, C.POINTER(_u32)]),
    ("oracle_domain_stats", C.c_int, [_P, _u32, _u32, _P]),
]
_LIB = None


def domain_oracle_lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIBORACLE_DOMAIN):
            raise OSError(f"{LIBORACLE_DOMAIN} missing: run `python __graft_entry__.py`")
        lib = C.CDLL(LIBORACLE_DOMAIN)
        for name, res, args in _SIGS + _IMPAIR_SIGS + _PAUSE_SIGS + _REACH_SIGS + _FLAP_SIGS + _DOMAIN_SIGS:
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _LIB = lib
    return _LIB


def _arr(xs):
    return (_u32 * max(1, len(xs)))(*xs)


class DomainOraclePool(FlapOraclePool):
    def __init__(self, cfg, threads: int = 1):
        self.lib = domain_oracle_lib()
        self.cfg = cfg
        self.capacity = cfg.capacity
        self.h = self.lib.oracle_create(C.byref(cfg), threads)
        if not self.h:
            raise GsimError(-1, "oracle_create failed")

    def domain_set(self, ids, domain):
        self._ck(self.lib.oracle_domain_set_many(self.h, _arr(ids), len(ids), domain))

    def domain_set_range(self, first, count, per_domain, first_domain=1):
        self._ck(self.lib.oracle_domain_set_range(self.h, first, count, per_domain, first_domain))

    def domains(self, first=0, count=None):
        if count is None:
            count = self.stats()["n_members"] - first
        out = np.zeros(max(count, 0), dtype=np.uint32)
        self._ck(self.lib.oracle_domain_get(self.h, first, count, out.ctypes.data_as(C.c_void_p)))
        return out

    def domain_flap(self, domains, period_ticks, bad_ppm):
        self._ck(self.lib.oracle_domain_flap_set(self.h, _arr(domains), len(domains), period_ticks, bad_ppm))

    def domain_flap_get(self, domain):
        period, ppm = _u32(), _u32()
        self._ck(self.lib.oracle_domain_flap_get(self.h, domain, C.byref(period), C.byref(ppm)))
        return period.value, ppm.value

    def domain_impair(self, domains, send_loss_ppm, recv_loss_ppm, delay_ticks=0, flags=0):
        out = _u32()
        self._ck(self.lib.oracle_domain_impair(self.h, _arr(domains), len(domains), send_loss_ppm, recv_loss_ppm,
                                               delay_ticks, flags, C.byref(out)))
        return out.value

    def domain_crash(self, domains):
        out = _u32()
        self._ck(self.lib.oracle_domain_crash(self.h, _arr(domains), len(domains), C.byref(out)))
        return out.value

    def domain_pause(self, domains, ticks):
        out = _u32()
        self._ck(self.lib.oracle_domain_pause(self.h, _arr(domains), len(domains), ticks, C.byref(out)))
        return out.value

    def domain_stats(self, first, count):
        out = np.zeros(max(count, 0), dtype=DOMAIN_STATS_DTYPE)
        self._ck(self.lib.oracle_domain_stats(self.h, first, count, out.ctypes.data_as(C.c_void_p)))
        return out
