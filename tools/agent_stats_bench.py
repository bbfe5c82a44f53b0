"""Time the per-agent observation calls (DESIGN.md §3.8) against the member count they replace.

  python tools/agent_stats_bench.py [--sizes 1,64] [--reps 5]

For each pool size (Mi members, LAN, one joiner pending and one user event queued) it prints one JSON line with
the wall time (host clock around the call, which ends in its one device wait) of:
  - gsim_agent_stats_read over every member, and for one member (one agent's Stats()),
  - gsim_health_histogram,
  - one gsim_num_nodes call (the key column copied to the host and counted there),
each the median of --reps calls after one warm-up call, plus the device time of the kernels and copies of one
call of each (torch.profiler's CUDA activity).  The GPU's name, power limit and SM clocks are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from consul_b200.pool import Pool, lan_config  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from coord_query_bench import device_ms, gpu_info  # noqa: E402

MI = 1 << 20


def wall_ms(fn, reps):
    fn()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        times.append((time.perf_counter() - t0) * 1e3)
    return round(statistics.median(times), 3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,64")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    print(json.dumps({"gpu": gpu_info()}), flush=True)
    for mi in (int(s) for s in args.sizes.split(",")):
        n = mi * MI
        p = Pool(lan_config(capacity=n + 1, n_initial=n, seed=0xA6E1B000 + mi))
        x = p.member_add()
        p.join(x, [0])
        p.user_event(1, b"bench", b"x" * 32, False)
        p.step(4)
        calls = {
            "agent_stats_all": lambda: p.agent_stats(0, n + 1),
            "agent_stats_one": lambda: p.agent_stats(12345, 1),
            "health_histogram": p.health_histogram,
            "num_nodes": lambda: p.num_nodes(12345),
        }
        row = {"members": n + 1}
        for name, fn in calls.items():
            row[name + "_ms"] = wall_ms(fn, args.reps)
            kern, copy, top = device_ms(fn)
            row[name + "_device"] = {"kernel_ms": round(kern, 4), "copy_ms": round(copy, 4),
                                     "kernels": {k: round(v, 4) for k, v in top.items()}}
        print(json.dumps(row), flush=True)
        p.close()
    print(json.dumps({"gpu": gpu_info()}), flush=True)


if __name__ == "__main__":
    main()
