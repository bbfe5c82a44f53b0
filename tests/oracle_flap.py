"""ctypes binding of tests/oracle_flap/liboracle_flap.so — TEST INFRASTRUCTURE.

That library is the oracle with degraded members (impair.patch), paused members (pause.patch), one-way
reachability (reach.patch) and intermittent impairment (tests/oracle_flap/flap.patch) restated on top, applied
by `__graft_entry__.build()`; `FlapOraclePool` drives it with the methods of `ReachOraclePool` plus those of
`consul_b200.pool.Pool` for flap schedules.
"""
from __future__ import annotations

import ctypes as C
import os

from consul_b200.pool import GsimError
from oracle_binding import _SIGS
from oracle_impair import _IMPAIR_SIGS
from oracle_pause import _PAUSE_SIGS
from oracle_reach import _REACH_SIGS, ReachOraclePool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBORACLE_FLAP = os.path.join(ROOT, "tests", "oracle_flap", "liboracle_flap.so")

_u32, _sz = C.c_uint32, C.c_size_t
_FLAP_SIGS = [
    ("oracle_impair_flap_many", C.c_int, [C.c_void_p, C.POINTER(_u32), _sz, _u32, _u32]),
    ("oracle_impair_flap_fraction", C.c_int, [C.c_void_p, _u32, _u32, _u32, _u32, C.POINTER(_u32)]),
    ("oracle_impair_flap_get", C.c_int, [C.c_void_p, _u32, C.POINTER(_u32), C.POINTER(_u32)]),
]
_LIB = None


def flap_oracle_lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIBORACLE_FLAP):
            raise OSError(f"{LIBORACLE_FLAP} missing: run `python __graft_entry__.py`")
        lib = C.CDLL(LIBORACLE_FLAP)
        for name, res, args in _SIGS + _IMPAIR_SIGS + _PAUSE_SIGS + _REACH_SIGS + _FLAP_SIGS:
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _LIB = lib
    return _LIB


class FlapOraclePool(ReachOraclePool):
    def __init__(self, cfg, threads: int = 1):
        self.lib = flap_oracle_lib()
        self.cfg = cfg
        self.capacity = cfg.capacity
        self.h = self.lib.oracle_create(C.byref(cfg), threads)
        if not self.h:
            raise GsimError(-1, "oracle_create failed")

    def impair_flap(self, ids, period_ticks, bad_ppm):
        arr = (_u32 * max(1, len(ids)))(*ids)
        self._ck(self.lib.oracle_impair_flap_many(self.h, arr, len(ids), period_ticks, bad_ppm))

    def impair_flap_fraction(self, member_ppm, salt, period_ticks, bad_ppm):
        out = _u32()
        self._ck(self.lib.oracle_impair_flap_fraction(self.h, member_ppm, salt, period_ticks, bad_ppm, C.byref(out)))
        return out.value

    def impair_flap_get(self, member):
        period, ppm = _u32(), _u32()
        self._ck(self.lib.oracle_impair_flap_get(self.h, member, C.byref(period), C.byref(ppm)))
        return period.value, ppm.value
