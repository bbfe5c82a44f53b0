"""ctypes binding of tests/oracle_reach/liboracle_reach.so — TEST INFRASTRUCTURE.

That library is the oracle with degraded members (impair.patch), paused members (pause.patch) and
one-way reachability (tests/oracle_reach/reach.patch) restated on top, applied by
`__graft_entry__.build()`; `ReachOraclePool` drives it with the methods of `PauseOraclePool` plus those
of `consul_b200.pool.Pool` for directional impairment.
"""
from __future__ import annotations

import ctypes as C
import os

from consul_b200.pool import IMPAIR_NO_TCP, GsimError
from oracle_binding import _SIGS
from oracle_impair import _IMPAIR_SIGS
from oracle_pause import _PAUSE_SIGS, PauseOraclePool

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIBORACLE_REACH = os.path.join(ROOT, "tests", "oracle_reach", "liboracle_reach.so")

_u32, _sz = C.c_uint32, C.c_size_t
_REACH_SIGS = [
    ("oracle_impair_dir_many", C.c_int, [C.c_void_p, C.POINTER(_u32), _sz, _u32, _u32, _u32, _u32]),
    ("oracle_impair_dir_fraction", C.c_int, [C.c_void_p, _u32, _u32, _u32, _u32, _u32, _u32, C.POINTER(_u32)]),
    ("oracle_impair_dir_get", C.c_int, [C.c_void_p, _u32, C.POINTER(_u32), C.POINTER(_u32), C.POINTER(_u32),
                                        C.POINTER(_u32)]),
]
_LIB = None


def reach_oracle_lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(LIBORACLE_REACH):
            raise OSError(f"{LIBORACLE_REACH} missing: run `python __graft_entry__.py`")
        lib = C.CDLL(LIBORACLE_REACH)
        for name, res, args in _SIGS + _IMPAIR_SIGS + _PAUSE_SIGS + _REACH_SIGS:
            fn = getattr(lib, name)
            fn.restype = res
            fn.argtypes = args
        _LIB = lib
    return _LIB


class ReachOraclePool(PauseOraclePool):
    def __init__(self, cfg, threads: int = 1):
        self.lib = reach_oracle_lib()
        self.cfg = cfg
        self.capacity = cfg.capacity
        self.h = self.lib.oracle_create(C.byref(cfg), threads)
        if not self.h:
            raise GsimError(-1, "oracle_create failed")

    def impair_dir(self, ids, send_loss_ppm, recv_loss_ppm, delay_ticks=0, no_tcp=False):
        arr = (_u32 * max(1, len(ids)))(*ids)
        self._ck(self.lib.oracle_impair_dir_many(self.h, arr, len(ids), send_loss_ppm, recv_loss_ppm, delay_ticks,
                                                 IMPAIR_NO_TCP if no_tcp else 0))

    def impair_dir_fraction(self, member_ppm, salt, send_loss_ppm, recv_loss_ppm, delay_ticks=0, no_tcp=False):
        out = _u32()
        self._ck(self.lib.oracle_impair_dir_fraction(self.h, member_ppm, salt, send_loss_ppm, recv_loss_ppm,
                                                     delay_ticks, IMPAIR_NO_TCP if no_tcp else 0, C.byref(out)))
        return out.value

    def impairment_dir(self, member):
        s, r, d, f = _u32(), _u32(), _u32(), _u32()
        self._ck(self.lib.oracle_impair_dir_get(self.h, member, C.byref(s), C.byref(r), C.byref(d), C.byref(f)))
        return s.value, r.value, d.value, bool(f.value & IMPAIR_NO_TCP)
