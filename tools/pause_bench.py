"""Paused members on one H100: how long may a member stall before the cluster declares it Failed, and what
pausing costs.

(a) Threshold curve: a 1 Mi-member LAN pool, 1 % of its members paused for d ticks (100 ms each), d in
    {3, 10, 30, 100, 200, 300, 500, 1500}: how many came back Alive (the pause went unnoticed), Suspect
    (a false suspicion, refuted) and Dead (declared Failed).  With awareness_max_multiplier 8 and 1.
(b) Kernel time per tick while 1 % of 1 Mi members are paused, next to the same pool with nobody paused.
(c) Device time of the resume kernel (and of the pause kernel) at 1 Mi and 64 Mi members, from
    torch.profiler's CUDA activity records.

Prints the card's name and power limit (read in the same run) and one JSON line per row.

  python tools/pause_bench.py [--out DIR] [--skip-64m]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def threshold_row(n, d, aw_max):
    from consul_b200.pool import Pool, lan_config
    p = Pool(lan_config(capacity=n, n_initial=n, seed=0x9A05B001, awareness_max_multiplier=aw_max))
    p.step(16)
    k = p.pause_fraction(10000, 1, d)
    p.step(d)
    st = p.pause_stats()
    assert st["paused"] == 0
    return {"row": "threshold", "members": n, "awareness_max_multiplier": aw_max, "pause_ticks": d, "paused": k,
            "alive": st["resumed_alive"], "suspect": st["resumed_suspect"], "dead": st["resumed_dead"]}


def cost_row(n, ppm, ticks):
    from consul_b200.pool import Pool, lan_config
    p = Pool(lan_config(capacity=n, n_initial=n, seed=0x9A05B002))
    p.step(64)
    k = p.pause_fraction(ppm, 2, ticks + 64) if ppm else 0
    p.step(64)                                        # the cascade of probes of the paused members starts
    before = p.sched_counts()
    p.step(ticks)
    ms, launches = p.last_step_timing()
    after = p.sched_counts()
    sched = {key: after[key] - before[key] for key in ("window_launches", "window_ticks", "tick_launches")}
    return {"row": "cost", "members": n, "paused": k, "ticks": ticks, "kernel_ms_per_tick": ms / ticks,
            "launches": launches, "sched": sched}


def resume_row(n, reps=5):
    """Device time of gs_pause_kernel (gsim_pause_fraction, 1 % of the members) and of gs_resume_kernel (one
    resume tick), from torch.profiler's CUDA activity records: median of `reps` rounds."""
    from torch.profiler import ProfilerActivity, profile
    from consul_b200.pool import Pool, lan_config
    p = Pool(lan_config(capacity=n, n_initial=n, seed=0x9A05B003))
    p.step(16)
    t_pause, t_resume = [], []
    for r in range(reps + 1):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            p.pause_fraction(10000, r, 4)
            p.step(5)                                 # the resume runs before the 4th tick of this step
        us = {e.key: e.device_time_total / max(1, e.count) for e in prof.key_averages()}
        if r:                                         # (round 0 warms up the profiler)
            t_pause.append(next(v for k, v in us.items() if "gs_pause_kernel" in k))
            t_resume.append(next(v for k, v in us.items() if "gs_resume_kernel" in k))
    return {"row": "kernels", "members": n, "pause_kernel_us": sorted(t_pause)[reps // 2],
            "resume_kernel_us": sorted(t_resume)[reps // 2], "rounds": reps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--members", type=int, default=1 << 20)
    ap.add_argument("--out", default=None, help="also write the rows to DIR/pause_bench.jsonl")
    ap.add_argument("--skip-64m", action="store_true")
    a = ap.parse_args()
    c = card()
    print("card:", c, flush=True)
    rows = []

    def emit(r):
        rows.append(r)
        print(json.dumps(r), flush=True)

    for aw in (8, 1):
        for d in (3, 10, 30, 100, 200, 300, 500, 1500):
            emit(threshold_row(a.members, d, aw))
    for ppm in (0, 10000):
        emit(cost_row(a.members, ppm, 400))
    emit(resume_row(a.members))
    if not a.skip_64m:
        emit(resume_row(64 << 20))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "pause_bench.jsonl"), "w") as f:
            f.write("card: %s\n" % c)
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
