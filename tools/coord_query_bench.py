"""Time the network-coordinate queries (DESIGN.md §3.4 "Queries") and follow the embedding's accuracy.

  python tools/coord_query_bench.py [--sizes 1,8,64] [--error-ticks 0,100,500,1000,2000]

For each pool size (Mi members, C5 latency matrix, coordinates on, a few ticks run) it prints, for every
query call, the device time of its kernels (CUDA kernel activity recorded by torch.profiler, copies excluded)
and of its three costliest kernels, the device time of its copies, and its wall time including the readback;
then the bulk read against the per-member getter at the first size (the getter timed
on a sample of 20 000 members and extrapolated), and the error statistics of gsim_coordinate_error over
probe time on the C5 matrix at 1 Mi members.  The GPU's power limit and SM clock are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from consul_b200.pool import FLAG_COORDINATES, Pool, wan_config  # noqa: E402
from consul_b200.wan import c5_latency_matrix  # noqa: E402

MI = 1 << 20


def gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"unavailable ({e})"


def device_ms(fn):
    """(kernel ms, copy ms) of one call: the CUDA activity torch.profiler records in this process, which
    includes libgsim's kernels on its own stream."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
    kern = copy = 0.0
    by_kernel = {}
    for e in prof.events():
        if e.device_type != torch.autograd.DeviceType.CUDA:
            continue
        us = e.time_range.elapsed_us()
        if e.name.startswith(("Memcpy", "Memset")):
            copy += us
        else:
            kern += us
            by_kernel[e.name] = by_kernel.get(e.name, 0.0) + us / 1e3
    top = dict(sorted(by_kernel.items(), key=lambda kv: -kv[1])[:3])
    return kern / 1e3, copy / 1e3, top


def timed(fn, reps=3):
    fn()                                                      # first call allocates the query buffers
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        best = min(best, time.perf_counter() - t0)
    try:
        kern, copy, top = device_ms(fn)
    except Exception as e:  # noqa: BLE001
        kern = copy = top = f"unavailable ({e})"
    return {"kernels_ms": kern, "copies_ms": copy, "wall_ms": best * 1e3, "top_kernels_ms": top}


def c5_pool(n, seed=0xC5):
    p = Pool(wan_config(capacity=n, n_initial=n, seed=seed, flags=FLAG_COORDINATES, mailbox_depth=8))
    p.latency_set(c5_latency_matrix(64))
    return p


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1,8,64")
    ap.add_argument("--error-ticks", default="0,100,500,1000,2000")
    a = ap.parse_args()
    out = {"gpu": gpu_info(), "calls_ms": {}}
    sizes = [int(s) for s in a.sizes.split(",")]
    for mi in sizes:
        n = mi * MI
        p = c5_pool(n)
        p.step(20)
        rng = np.random.default_rng(1)
        pa, pb = rng.integers(0, n, MI), rng.integers(0, n, MI)
        r = {
            "coordinates(all)": timed(lambda: p.coordinates()),
            "rtt(1Mi pairs, true)": timed(lambda: p.rtt(pa, pb, true_rtt=True)),
            "sort_by_distance(all)": timed(lambda: p.sort_by_distance(7)),
            "sort_by_distance(all, k=10)": timed(lambda: p.sort_by_distance(7, k=10)),
            "dcs_by_distance(all)": timed(lambda: p.dcs_by_distance(7)),
            "coordinate_error(1Mi draws)": timed(lambda: p.coordinate_error(MI, 1)),
        }
        if mi == sizes[0]:
            sample = 20000
            t0 = time.perf_counter()
            for i in range(sample):
                p.coordinate(i)
            per = (time.perf_counter() - t0) / sample
            r["coordinate(i) x n, extrapolated wall_ms"] = per * n * 1e3
            r["bulk speed-up (wall)"] = r["coordinate(i) x n, extrapolated wall_ms"] / r["coordinates(all)"]["wall_ms"]
        out["calls_ms"][f"{mi}Mi"] = r
        print(json.dumps({f"{mi}Mi": r}), flush=True)
        p.close()
    p = c5_pool(MI, seed=0xE5)
    done, series = 0, []
    for t in [int(x) for x in a.error_ticks.split(",")]:
        p.step(t - done)
        done = t
        e = p.coordinate_error(MI, 0)
        series.append({"tick": t, **e})
        print(json.dumps(series[-1]), flush=True)
    out["error_over_time_1Mi_c5"] = series
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
