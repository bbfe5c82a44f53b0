"""Host round trips of the benchmark's step: member_add + join(x, [0]) + step(2048).

tests/hostemu/libgsim_hostemu_counted.so is the host emulation behind a backend that counts every call
which would wait for the device on the CUDA backend (a synchronous copy, a readback, a stream
synchronisation).  Each one leaves the GPU idle while the host waits, so the host side of an
operation may wait only where it needs a value to decide what to do next: the rows a join merges, the end of each chunk of single ticks, one look for quietness, the
window chain and the count behind rumor retirement.  Writes to device state are queued and applied
on the device in order (GsWriteBatch) without a wait.
"""
import ctypes as C
import os

from consul_b200 import _lib
from consul_b200.pool import Pool, lan_config

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

N = 100_000
# the same calls before device write batches (host emulation, this pool, after the same warm-up)
BEFORE = {"member_add + join": 22, "step(2048)": 25}


def test_bench_step_waits_for_the_device_only_where_it_needs_a_value():
    lib = _lib.load(os.path.join(ROOT, "tests", "hostemu", "libgsim_hostemu_counted.so"))
    waits = lib.gsim_hostemu_waits
    waits.restype = C.c_uint64
    waits.argtypes = [C.POINTER(C.c_uint64)]
    chunks = C.c_uint64()

    def count():
        w = waits(C.byref(chunks))
        return w, chunks.value

    p = Pool(lan_config(lib, capacity=N + 16, n_initial=N, seed=0x5EED0001), lib)
    p.step(64)
    for _ in range(2):  # warm-up: the step bench.py times
        x = p.member_add()
        assert p.join(x, [0]) == 1
        p.step(2048)
    w0, _ = count()
    x = p.member_add()
    assert p.join(x, [0]) == 1
    w1, k1 = count()
    p.step(2048)
    w2, k2 = count()
    join_waits, step_waits, tick_chunks = w1 - w0, w2 - w1, k2 - k1
    print(f"\nwaits for the device, {N:,} members: member_add + join {join_waits} (before: "
          f"{BEFORE['member_add + join']}), step(2048) {step_waits} with {tick_chunks} single-tick chunks "
          f"(before: {BEFORE['step(2048)']})")
    assert join_waits <= 1
    assert step_waits <= tick_chunks + 3
    p.close()
