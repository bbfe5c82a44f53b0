"""Where the end-to-end step of bench.py goes on one GPU: wall time of each C-ABI call (dev tool).
restore (snapshot blob in pinned host memory) -> member_add -> join -> step(2048) -> Members() -> stats.
An optional argument names the libgsim build to time (default: the package's)."""
import ctypes as C
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from consul_b200 import _lib  # noqa: E402
from consul_b200._lib import GsimMember  # noqa: E402
from consul_b200.pool import Pool, lan_config  # noqa: E402

lib = _lib.load(sys.argv[1]) if len(sys.argv) > 1 else _lib.lib()
n = 1_000_000
p = Pool(lan_config(lib, capacity=n + 4096, n_initial=n, seed=0x5EED0001), lib)
p.step(64)
blob = p.snapshot()
pinned = torch.empty(len(blob), dtype=torch.uint8, pin_memory=True)
pinned.numpy()[:] = memoryview(blob)
ptr = C.c_void_p(pinned.data_ptr())
buf = (GsimMember * (n + 4096))()
k = C.c_size_t()
names = ["restore", "member_add", "join", "step", "members", "stats"]
acc = dict.fromkeys(names, 0.0)
REP = 8
for it in range(REP + 2):
    ts = [time.perf_counter()]
    assert p.lib.gsim_restore(p.h, ptr, len(blob)) == 0; ts.append(time.perf_counter())
    x = p.member_add(); ts.append(time.perf_counter())
    p.join(x, [0]); ts.append(time.perf_counter())
    p.step(2048); ts.append(time.perf_counter())
    assert p.lib.gsim_members(p.h, 0, buf, n + 4096, C.byref(k)) == 0; ts.append(time.perf_counter())
    p.stats(); ts.append(time.perf_counter())
    if it >= 2:
        for i, nm in enumerate(names):
            acc[nm] += (ts[i + 1] - ts[i]) * 1e3 / REP
print(json.dumps({"lib": lib._name, "blob_bytes": len(blob), "members": k.value, "threads": os.environ.get("GSIM_MEMBERS_THREADS"),
                  "wall_ms": {a: round(b, 3) for a, b in acc.items()}, "sum_ms": round(sum(acc.values()), 3)}))
