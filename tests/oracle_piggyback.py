"""ctypes binding of tests/oracle_piggyback/liboracle_piggyback.so — TEST INFRASTRUCTURE.

That library is the oracle with degraded, paused and one-way members (impair.patch, pause.patch, reach.patch) and
broadcasts piggybacked on probe traffic (tests/oracle_piggyback/piggyback.patch) restated on top, applied by
`__graft_entry__.build()`; `PiggybackOraclePool` drives it with the methods of `ReachOraclePool` plus
`piggyback_stats`.
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
LIBORACLE_PIGGYBACK = os.path.join(ROOT, "tests", "oracle_piggyback", "liboracle_piggyback.so")

_PIG_SIGS = [("oracle_piggyback_stats", C.c_int, [C.c_void_p, C.POINTER(C.c_uint64)])]
_LIB = None


def piggyback_oracle_lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIBORACLE_PIGGYBACK):
            raise OSError(f"{LIBORACLE_PIGGYBACK} missing: run `python __graft_entry__.py`")
        lib = C.CDLL(LIBORACLE_PIGGYBACK)
        for name, res, args in _SIGS + _IMPAIR_SIGS + _PAUSE_SIGS + _REACH_SIGS + _PIG_SIGS:
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _LIB = lib
    return _LIB


class PiggybackOraclePool(ReachOraclePool):
    def __init__(self, cfg, threads: int = 1):
        self.lib = piggyback_oracle_lib()
        self.cfg = cfg
        self.capacity = cfg.capacity
        self.h = self.lib.oracle_create(C.byref(cfg), threads)
        if not self.h:
            raise GsimError(-1, "oracle_create failed")

    def piggyback_stats(self) -> dict:
        out = (C.c_uint64 * 4)()
        self._ck(self.lib.oracle_piggyback_stats(self.h, out))
        return {"packets": int(out[0]), "broadcasts": int(out[1]), "owed_served": int(out[2]),
                "owed_dropped": int(out[3])}
