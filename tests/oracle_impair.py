"""ctypes binding of tests/oracle_impair/liboracle_impair.so — TEST INFRASTRUCTURE.

That library is the oracle (oracle/oracle.cpp) with degraded members restated on top
(tests/oracle_impair/impair.patch, applied by `__graft_entry__.build()`); `ImpairOraclePool` drives it
with the methods of `OraclePool` plus those of `consul_b200.pool.Pool` for impairment.
"""
from __future__ import annotations

import ctypes as C
import os

from consul_b200.pool import GsimError
from oracle_binding import _SIGS, OraclePool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBORACLE_IMPAIR = os.path.join(ROOT, "tests", "oracle_impair", "liboracle_impair.so")

_u32, _sz = C.c_uint32, C.c_size_t
_IMPAIR_SIGS = [
    ("oracle_impair_many", C.c_int, [C.c_void_p, C.POINTER(_u32), _sz, _u32, _u32]),
    ("oracle_impair_fraction", C.c_int, [C.c_void_p, _u32, _u32, _u32, _u32, C.POINTER(_u32)]),
    ("oracle_impair_get", C.c_int, [C.c_void_p, _u32, C.POINTER(_u32), C.POINTER(_u32)]),
]
_LIB = None


def impair_oracle_lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIBORACLE_IMPAIR):
            raise OSError(f"{LIBORACLE_IMPAIR} missing: run `python __graft_entry__.py`")
        lib = C.CDLL(LIBORACLE_IMPAIR)
        for name, res, args in _SIGS + _IMPAIR_SIGS:
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _LIB = lib
    return _LIB


class ImpairOraclePool(OraclePool):
    def __init__(self, cfg, threads: int = 1):
        self.lib = impair_oracle_lib()
        self.cfg = cfg
        self.capacity = cfg.capacity
        self.h = self.lib.oracle_create(C.byref(cfg), threads)
        if not self.h:
            raise GsimError(-1, "oracle_create failed")

    def impair(self, ids, loss_ppm, delay_ticks=0):
        arr = (_u32 * max(1, len(ids)))(*ids)
        self._ck(self.lib.oracle_impair_many(self.h, arr, len(ids), loss_ppm, delay_ticks))

    def impair_fraction(self, member_ppm, salt, loss_ppm, delay_ticks=0):
        out = _u32()
        self._ck(self.lib.oracle_impair_fraction(self.h, member_ppm, salt, loss_ppm, delay_ticks, C.byref(out)))
        return out.value

    def impairment(self, member):
        loss, delay = _u32(), _u32()
        self._ck(self.lib.oracle_impair_get(self.h, member, C.byref(loss), C.byref(delay)))
        return loss.value, delay.value
