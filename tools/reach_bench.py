"""One-way reachability on one H100: what half-broken members do to a 1 Mi-member LAN pool.

For 0.1 % and 1 % of the members with inbound UDP blocked (receive loss 100 %) or outbound UDP blocked (send
loss 100 %), with the TCP fallback ping on and off and periodic push-pull on and off, over 3 000 ticks of
100 ms: suspicions and refutes (nobody crashes, so every suspicion is false), the awareness (local health)
histogram of the blocked members at the end, when a user event fired at tick 10 by an unblocked member has
reached every blocked member (or the fraction it reached), and kernel ms per tick (gsim_last_step_timing).

Prints the card's name, power limit and max SM clock (read in the same run) and one JSON line per row.

  python tools/reach_bench.py [--members N] [--ticks T] [--out DIR]
"""
import argparse
import json
import os
import random
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


def card():
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def row(n, frac_ppm, direction, tcp_fallback, push_pull, ticks, chunk=50):
    from consul_b200.pool import FLAG_PUSH_PULL, Pool, lan_config
    cfg = lan_config(capacity=n, n_initial=n, seed=0x4EAB0001, disable_tcp_pings=0 if tcp_fallback else 1,
                     flags=FLAG_PUSH_PULL if push_pull else 0, mailbox_depth=4 if push_pull else 0)
    p = Pool(cfg)
    rng = random.Random(frac_ppm * 7 + (direction == "in"))
    blocked = sorted(rng.sample(range(8, n), n * frac_ppm // 1_000_000))
    send, recv = (0, 1_000_000) if direction == "in" else (1_000_000, 0)
    p.impair_dir(blocked, send, recv)
    ids = np.asarray(blocked, dtype=np.int64)
    p.step(10)
    slot = p.user_event(3, b"deploy", bytes(32), False)
    kernel_ms, reached_at, frac = 0.0, None, 0.0
    while p.now < ticks:
        p.step(min(chunk, ticks - p.now))
        kernel_ms += p.last_step_timing()[0]
        if reached_at is None:
            got = (p.column("heard")[ids] >> slot) & 1
            frac = float(got.mean())
            if got.all():
                reached_at = p.now - 10       # ticks after the event, to the chunk
    s = p.stats()
    aw = np.bincount(p.column("meta")[ids] & 7, minlength=8).tolist()
    return {"members": n, "blocked": len(blocked), "direction": direction, "tcp_fallback": tcp_fallback,
            "push_pull": push_pull, "ticks": ticks, "suspects": s["suspects"], "refutes": s["refutes"],
            "deads": s["deads"], "probe_failures": s["probe_failures"], "push_pulls": s["push_pulls"],
            "awareness_hist": aw, "event_reached_all_after_ticks": reached_at, "event_fraction_reached": frac,
            "kernel_ms_per_tick": kernel_ms / (ticks - 10)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--members", type=int, default=1 << 20)
    ap.add_argument("--ticks", type=int, default=3000)
    ap.add_argument("--out", default=None, help="also write the rows to DIR/reach_bench.jsonl")
    a = ap.parse_args()
    c = card()
    print("card:", c, flush=True)
    rows = []
    for frac in (1000, 10000):
        for direction in ("in", "out"):
            for tcp in (True, False):
                for pp in (False, True):
                    rows.append(row(a.members, frac, direction, tcp, pp, a.ticks))
                    print(json.dumps(rows[-1]), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "reach_bench.jsonl"), "w") as f:
            f.write("card: %s\n" % c)
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
