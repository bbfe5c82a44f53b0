"""Wall time of bench.py's resident step for two or more libgsim builds, alternating (dev tool).

One pool per build (1 M converged members, BASELINE config 2, seed 0x5EED0001), all resident at once;
rounds of STEPS steps (member_add -> join(x, [0]) -> step(2048)) run build after build, so drift of the
machine lands on every build alike.  A step's wall time minus its kernel time is what the host adds.
Every pool runs the same steps, so the state digests at the end must be equal.

    python tools/step_compare.py OLD/libgsim.so consul_b200/libgsim.so [--rounds 4] [--steps 20]
"""
import argparse
import json
import os
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from consul_b200 import _lib  # noqa: E402
from consul_b200.pool import Pool, lan_config  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("libs", nargs="+")
ap.add_argument("--members", type=int, default=1_000_000)
ap.add_argument("--ticks", type=int, default=2048)
ap.add_argument("--rounds", type=int, default=4)
ap.add_argument("--steps", type=int, default=20)
ap.add_argument("--warmup", type=int, default=3)
args = ap.parse_args()
n = args.members
pools = []
for path in args.libs:
    lib = _lib.load(path)
    pools.append(Pool(lan_config(lib, capacity=n + 4096, n_initial=n, seed=0x5EED0001), lib))


def step(p):
    x = p.member_add()
    assert p.join(x, [0]) == 1
    p.step(args.ticks)


for p in pools:
    for _ in range(args.warmup):
        step(p)
res = [{"lib": path, "ms_per_step": [], "kernel_ms_per_step": [], "value": []} for path in args.libs]
for _ in range(args.rounds):
    for p, r in zip(pools, res):
        members = p.stats()["n_members"]
        kms = 0.0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            step(p)
            kms += p.last_step_timing()[0]
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        r["ms_per_step"].append(round(dt * 1e3 / args.steps, 4))
        r["kernel_ms_per_step"].append(round(kms / args.steps, 4))
        # node-ticks per second, as bench.py's `value` (members grow by one per step)
        r["value"].append(round((members + (args.steps + 1) / 2) * args.ticks * args.steps / dt / 1e6, 1))
for p, r in zip(pools, res):
    r["digest"] = "%016x" % p.state_hash()[0]
    r["host_ms_per_step"] = [round(a - b, 4) for a, b in zip(r["ms_per_step"], r["kernel_ms_per_step"])]
    print(json.dumps(r), flush=True)
    p.close()
