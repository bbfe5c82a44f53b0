"""Degraded members on one H100: what the generic probe path costs, and what Lifeguard buys.

1. Cost: a 1 Mi-member LAN pool with 0 %, 0.1 % and 1 % of its members impaired (30 % loss, no delay),
   2 048 ticks each: kernel ms per tick (gsim_last_step_timing), launches by kind (gsim_sched_counts)
   and node-ticks per second of kernel time.  Any impaired member turns the probe fast paths and the
   long / closed-form quiet windows off for the whole pool, so the 0 % row is the baseline.
2. Lifeguard: 1 % impaired at 50 % loss, no TCP fallback, 3 000 ticks, with awareness_max_multiplier 8
   and 1 (local health off).  Nobody crashes, so every suspicion is false.

Prints the card's name and power limit (read in the same run) and one JSON line per row.

  python tools/impair_bench.py [--members N] [--out DIR]
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


def cost_row(n, frac_ppm, ticks):
    from consul_b200.pool import Pool, lan_config
    p = Pool(lan_config(capacity=n, n_initial=n, seed=0x1A9B0001))
    k = p.impair_fraction(frac_ppm, 1, 300000, 0) if frac_ppm else 0
    p.step(64)                                        # warm-up: modules loaded, graphs captured
    before = p.sched_counts()
    p.step(ticks)
    ms, launches = p.last_step_timing()
    after = p.sched_counts()
    sched = {key: after[key] - before[key] for key in ("window_launches", "window_ticks", "tick_launches",
                                                       "closed_form_launches", "closed_form_ticks")}
    return {"row": "cost", "members": n, "impaired": k, "ticks": ticks, "kernel_ms_per_tick": ms / ticks,
            "launches": launches, "sched": sched, "node_ticks_per_s": n * ticks / (ms / 1e3)}


def lifeguard_row(n, aw_max, ticks):
    from consul_b200.pool import Pool, lan_config
    p = Pool(lan_config(capacity=n, n_initial=n, seed=0x1A9B0002, awareness_max_multiplier=aw_max, disable_tcp_pings=1))
    k = p.impair_fraction(10000, 2, 500000, 0)
    p.step(ticks)
    s = p.stats()
    return {"row": "lifeguard", "members": n, "impaired": k, "ticks": ticks, "awareness_max_multiplier": aw_max,
            "refutes": s["refutes"], "suspects": s["suspects"], "probe_failures": s["probe_failures"],
            "nacks": s["nacks"], "deads": s["deads"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--members", type=int, default=1 << 20)
    ap.add_argument("--out", default=None, help="also write the rows to DIR/impair_bench.jsonl")
    a = ap.parse_args()
    print("card:", card(), flush=True)
    rows = [cost_row(a.members, ppm, 2048) for ppm in (0, 1000, 10000)]
    rows += [lifeguard_row(a.members, aw, 3000) for aw in (8, 1)]
    for r in rows:
        print(json.dumps(r), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "impair_bench.jsonl"), "w") as f:
            f.write("card: %s\n" % card())
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
