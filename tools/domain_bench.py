"""Fault domains on one H100: correlated bursts against independent ones of the same mean loss, at 1 Mi LAN members.

The members are in racks of 32 (gsim_domain_set_range); 1 % of the racks are impaired, the same members in
every row, and the TCP fallback ping is off (with it on, loss alone suspects nobody, DESIGN.md §3.5).
  steady       loss L all the time
  independent  loss L / f in bad epochs of each member's own schedule (period P, bad with probability f)
  racks        loss L / f in bad epochs of the rack's schedule (period P, f): a rack's members burst together
Per row, over the run: false suspicions (GSIM_STAT_SUSPECTS; nobody crashes), refutes, members with a health
score above 0 at the end (gsim_health_histogram), the peak fraction of one impaired rack that is Suspect at once
(gsim_domain_stats_read every --every ticks) and kernel ms per tick (gsim_last_step_timing).

Two more lines: the kernel time of the steady row with every impaired member on an always-bad member schedule
against the same with an always-bad rack schedule (identical results; the difference is what the domain lookup
adds to the member one), and at --big members the time of one gsim_domain_stats_read over every rack and of one
gsim_domain_crash of 1 % of the racks (host clock around the call, which ends in a readback).

Prints the card's name, power limit and max SM clock (read in the same run) and one JSON line per row.

  python tools/domain_bench.py [--members N] [--ticks T] [--loss PPM] [--bad PPM] [--period P] [--big N] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

FULL = 1_000_000
RACK = 32


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def racks_of(n, share_ppm=10_000, salt=0xD0B):
    n_racks = (n + RACK - 1) // RACK
    return [int(d) + 1 for d in np.nonzero(np.random.default_rng(salt).random(n_racks) < share_ppm / FULL)[0]]


def row(n, ticks, mode, loss_ppm, period, bad_ppm, every):
    """mode: 'steady', 'independent' (member schedules) or 'racks' (domain schedules)"""
    from consul_b200.pool import Pool, lan_config
    p = Pool(lan_config(capacity=n, n_initial=n, seed=0xD0AB0001, disable_tcp_pings=1))
    p.domain_set_range(0, n, RACK, 1)
    racks = racks_of(n)
    k = p.domain_impair(racks, loss_ppm, loss_ppm)
    if mode == "independent":
        ids = np.nonzero(np.isin(p.domains(), racks))[0].tolist()
        p.impair_flap(ids, period, bad_ppm)
    elif mode == "racks":
        p.domain_flap(racks, period, bad_ppm)
    idx = np.array(racks) - 1
    kernel_ms, peak = 0.0, 0.0
    while p.now < ticks:
        p.step(min(every, ticks - p.now))
        kernel_ms += p.last_step_timing()[0]
        s = p.domain_stats(1, (n + RACK - 1) // RACK)
        peak = max(peak, float((s["suspect"][idx] / np.maximum(s["members"][idx], 1)).max()))
    st = p.stats()
    hist = p.health_histogram()
    return {"mode": mode, "members": n, "impaired": k, "racks": len(racks), "ticks": ticks, "loss_ppm": loss_ppm,
            "period": period if mode != "steady" else None, "bad_ppm": bad_ppm if mode != "steady" else None,
            "suspects": st["suspects"], "refutes": st["refutes"], "deads": st["deads"],
            "packets_lost": st["packets_lost"], "health_above_0": int(hist[:, 1:].sum()),
            "peak_rack_suspect_fraction": peak, "kernel_ms_per_tick": kernel_ms / ticks}


def lookup_cost(n, ticks, loss_ppm, every):
    """kernel ms per tick of the steady row on always-bad member schedules and on always-bad rack schedules"""
    from consul_b200.pool import Pool, lan_config
    out = {}
    for mode in ("member", "racks"):
        p = Pool(lan_config(capacity=n, n_initial=n, seed=0xD0AB0001, disable_tcp_pings=1))
        p.domain_set_range(0, n, RACK, 1)
        racks = racks_of(n)
        p.domain_impair(racks, loss_ppm, loss_ppm)
        if mode == "member":
            p.impair_flap(np.nonzero(np.isin(p.domains(), racks))[0].tolist(), 7, FULL)
        else:
            p.domain_flap(racks, 7, FULL)
        ms = 0.0
        while p.now < ticks:
            p.step(min(every, ticks - p.now))
            ms += p.last_step_timing()[0]
        out[mode] = (ms / ticks, p.state_hash())
    assert out["member"][1] == out["racks"][1], "always-bad member and rack schedules must behave alike"
    return {"lookup_cost": True, "member_schedule_kernel_ms_per_tick": out["member"][0],
            "rack_schedule_kernel_ms_per_tick": out["racks"][0]}


def big_calls(n, reps=5):
    """host ms of one gsim_domain_stats_read over every rack and of one gsim_domain_crash of 1 % of the racks"""
    from consul_b200.pool import Pool, lan_config
    p = Pool(lan_config(capacity=n, n_initial=n, seed=0xD0AB0002))
    p.domain_set_range(0, n, RACK, 1)
    n_racks = (n + RACK - 1) // RACK
    p.domain_stats(1, n_racks)                                  # warm up
    t = []
    for _ in range(reps):
        t0 = time.perf_counter()
        p.domain_stats(1, n_racks)
        t.append((time.perf_counter() - t0) * 1e3)
    racks = racks_of(n)
    t0 = time.perf_counter()
    crashed = p.domain_crash(racks)
    crash_ms = (time.perf_counter() - t0) * 1e3
    return {"big": True, "members": n, "racks": n_racks, "domain_stats_ms": min(t), "domain_stats_ms_all": t,
            "domain_crash_ms": crash_ms, "crashed": crashed}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--members", type=int, default=1 << 20)
    ap.add_argument("--ticks", type=int, default=500)
    ap.add_argument("--loss", type=int, default=50_000, help="steady loss L (ppm)")
    ap.add_argument("--bad", type=int, default=100_000, help="bad-epoch fraction f (ppm); bursty loss is L / f")
    ap.add_argument("--period", type=int, default=50)
    ap.add_argument("--every", type=int, default=10, help="ticks between domain_stats samples")
    ap.add_argument("--big", type=int, default=64 << 20, help="members for the domain_stats / domain_crash timing")
    ap.add_argument("--out", default=None, help="also write the rows to DIR/domain_bench.jsonl")
    a = ap.parse_args()
    c = card()
    print("card:", c, flush=True)
    burst = min(FULL, a.loss * FULL // a.bad)
    rows = [row(a.members, a.ticks, "steady", a.loss, 0, 0, a.every)]
    print(json.dumps(rows[-1]), flush=True)
    for mode in ("independent", "racks"):
        rows.append(row(a.members, a.ticks, mode, burst, a.period, a.bad, a.every))
        print(json.dumps(rows[-1]), flush=True)
    rows.append(lookup_cost(a.members, a.ticks, a.loss, a.every))
    print(json.dumps(rows[-1]), flush=True)
    if a.big:
        rows.append(big_calls(a.big))
        print(json.dumps(rows[-1]), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "domain_bench.jsonl"), "w") as f:
            f.write("card: %s\n" % c)
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
