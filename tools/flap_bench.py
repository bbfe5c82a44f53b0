"""Intermittent impairment on one H100: steady loss against flapping loss of the same mean, at 1 Mi LAN members.

1 % of the members are impaired, the TCP fallback ping is off (with it on, loss alone suspects nobody,
DESIGN.md §3.5).  The steady row gives them loss L all the time; each flapping row gives them loss L / f in bad
epochs that occur with probability f, for epoch periods of 10, 50 and 200 ticks of 100 ms: the same mean loss.
Per row, over the run: false suspicions (GSIM_STAT_SUSPECTS; nobody crashes), refutes, the final health
histogram (gsim_health_histogram, impaired members) and kernel ms per tick (gsim_last_step_timing).

One more line compares the kernel time of the steady row with the same pool whose impaired members all carry a
schedule with bad_ppm = 1e6, which behaves identically: the difference is the cost of the schedule lookups.

Prints the card's name, power limit and max SM clock (read in the same run) and one JSON line per row.

  python tools/flap_bench.py [--members N] [--ticks T] [--loss PPM] [--bad PPM] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FULL = 1_000_000


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def row(n, ticks, loss_ppm, period, bad_ppm, chunk=50):
    """period 0: the steady impairment; else loss_ppm in force only in bad epochs"""
    from consul_b200.pool import Pool, lan_config
    cfg = lan_config(capacity=n, n_initial=n, seed=0xF1AB0001, disable_tcp_pings=1)
    p = Pool(cfg)
    k = p.impair_fraction(10_000, 1, loss_ppm, 0)
    if period:
        p.impair_flap_fraction(10_000, 1, period, bad_ppm)
    kernel_ms = 0.0
    while p.now < ticks:
        p.step(min(chunk, ticks - p.now))
        kernel_ms += p.last_step_timing()[0]
    s = p.stats()
    hist = p.health_histogram()
    out = {"members": n, "impaired": k, "ticks": ticks, "loss_ppm": loss_ppm, "period": period,
           "bad_ppm": bad_ppm if period else None, "mean_loss_ppm": loss_ppm * (bad_ppm if period else FULL) // FULL,
           "suspects": s["suspects"], "refutes": s["refutes"], "deads": s["deads"],
           "packets_lost": s["packets_lost"], "health_hist_impaired": [int(x) for x in hist[1]],
           "kernel_ms_per_tick": kernel_ms / ticks}
    if period:
        out["flap_stats_end"] = p.flap_stats()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--members", type=int, default=1 << 20)
    ap.add_argument("--ticks", type=int, default=1000)
    ap.add_argument("--loss", type=int, default=50_000, help="steady loss L (ppm)")
    ap.add_argument("--bad", type=int, default=100_000, help="bad-epoch fraction f (ppm); flapping loss is L / f")
    ap.add_argument("--out", default=None, help="also write the rows to DIR/flap_bench.jsonl")
    a = ap.parse_args()
    c = card()
    print("card:", c, flush=True)
    flap_loss = min(FULL, a.loss * FULL // a.bad)
    rows = [row(a.members, a.ticks, a.loss, 0, 0)]
    print(json.dumps(rows[-1]), flush=True)
    for period in (10, 50, 200):
        rows.append(row(a.members, a.ticks, flap_loss, period, a.bad))
        print(json.dumps(rows[-1]), flush=True)
    # the schedule lookups: the steady row again, with every impaired member's schedule always bad
    always = row(a.members, a.ticks, a.loss, 7, FULL)
    assert always["suspects"] == rows[0]["suspects"] and always["packets_lost"] == rows[0]["packets_lost"]
    rows.append({"lookup_cost": True, "static_kernel_ms_per_tick": rows[0]["kernel_ms_per_tick"],
                 "always_bad_kernel_ms_per_tick": always["kernel_ms_per_tick"]})
    print(json.dumps(rows[-1]), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "flap_bench.jsonl"), "w") as f:
            f.write("card: %s\n" % c)
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
