"""ctypes binding of tests/oracle_pause/liboracle_pause.so — TEST INFRASTRUCTURE.

That library is the oracle with degraded members (impair.patch) and paused members
(tests/oracle_pause/pause.patch) restated on top, applied by `__graft_entry__.build()`;
`PauseOraclePool` drives it with the methods of `ImpairOraclePool` plus those of
`consul_b200.pool.Pool` for pausing.
"""
from __future__ import annotations

import ctypes as C
import os

from consul_b200.pool import GsimError
from oracle_binding import _SIGS
from oracle_impair import _IMPAIR_SIGS, ImpairOraclePool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBORACLE_PAUSE = os.path.join(ROOT, "tests", "oracle_pause", "liboracle_pause.so")

_u32, _sz = C.c_uint32, C.c_size_t
_PAUSE_SIGS = [
    ("oracle_pause_many", C.c_int, [C.c_void_p, C.POINTER(_u32), _sz, _u32, C.POINTER(_u32)]),
    ("oracle_pause_fraction", C.c_int, [C.c_void_p, _u32, _u32, _u32, C.POINTER(_u32)]),
    ("oracle_pause_get", C.c_int, [C.c_void_p, _u32, C.POINTER(_u32)]),
    ("oracle_pause_stats", C.c_int, [C.c_void_p, C.POINTER(C.c_uint64)]),
]
_LIB = None


def pause_oracle_lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIBORACLE_PAUSE):
            raise OSError(f"{LIBORACLE_PAUSE} missing: run `python __graft_entry__.py`")
        lib = C.CDLL(LIBORACLE_PAUSE)
        for name, res, args in _SIGS + _IMPAIR_SIGS + _PAUSE_SIGS:
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _LIB = lib
    return _LIB


class PauseOraclePool(ImpairOraclePool):
    def __init__(self, cfg, threads: int = 1):
        self.lib = pause_oracle_lib()
        self.cfg = cfg
        self.capacity = cfg.capacity
        self.h = self.lib.oracle_create(C.byref(cfg), threads)
        if not self.h:
            raise GsimError(-1, "oracle_create failed")

    def pause(self, ids, ticks):
        arr = (_u32 * max(1, len(ids)))(*ids)
        out = _u32()
        self._ck(self.lib.oracle_pause_many(self.h, arr, len(ids), ticks, C.byref(out)))
        return out.value

    def pause_fraction(self, member_ppm, salt, ticks):
        out = _u32()
        self._ck(self.lib.oracle_pause_fraction(self.h, member_ppm, salt, ticks, C.byref(out)))
        return out.value

    def paused_until(self, member):
        out = _u32()
        self._ck(self.lib.oracle_pause_get(self.h, member, C.byref(out)))
        return out.value

    def pause_stats(self):
        out = (C.c_uint64 * 4)()
        self._ck(self.lib.oracle_pause_stats(self.h, out))
        return dict(zip(("paused", "resumed_alive", "resumed_suspect", "resumed_dead"), out))
