"""Rows per tick of one join cascade: where the tick kernel's generic row steps go (dev tool).

Runs on the host emulation (or any libgsim build): a LAN pool, step(64), WARMUP bench steps
(member_add -> join(x, [0]) -> step(2048)), then one more member_add + join followed by TICKS single
ticks, reading the counters after each.  `active_rows` counts the members that left the 4-byte mailbox
scan (staged probes included); probes, gossip packets and accepted rumors say what they did.  With the
CUDA build (--lib consul_b200/libgsim.so, on an H100) `kernel_us` is each tick's kernel time.

    python tools/cascade_rows.py [--lib tests/hostemu/libgsim_hostemu.so] [--members 200000] [--ticks 64]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from consul_b200 import _lib  # noqa: E402
from consul_b200.pool import Pool, lan_config  # noqa: E402

KEYS = ("active_rows", "probes", "gossip_packets", "rumors_accepted")


def cascade_rows(lib, members=200_000, ticks=64, warmup=1, seed=0x5EED0001):
    """Per-tick counter deltas of one bench-step cascade, and the pool's digest at the end."""
    p = Pool(lan_config(lib, capacity=members + 16, n_initial=members, seed=seed), lib)
    try:
        p.step(64)
        for _ in range(warmup):
            x = p.member_add()
            assert p.join(x, [0]) == 1
            p.step(2048)
        x = p.member_add()
        assert p.join(x, [0]) == 1
        rows = []
        prev = p.stats()
        for _ in range(ticks):
            p.step(1)
            s = p.stats()
            rows.append({k: s[k] - prev[k] for k in KEYS})
            rows[-1]["kernel_us"] = round(p.last_step_timing()[0] * 1e3, 2)
            prev = s
        return rows, prev, p.state_hash()
    finally:
        p.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "tests", "hostemu", "libgsim_hostemu.so"))
    ap.add_argument("--members", type=int, default=200_000)
    ap.add_argument("--ticks", type=int, default=64)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--json", action="store_true", help="one JSON line instead of the table")
    args = ap.parse_args()
    rows, stats, digest = cascade_rows(_lib.load(args.lib), args.members, args.ticks, args.warmup)
    total = {k: sum(r[k] for r in rows) for k in KEYS + ("kernel_us",)}
    if args.json:
        print(json.dumps({"lib": args.lib, "members": args.members, "per_tick": rows, "total": total,
                          "digest": "%016x" % digest[0]}))
        return
    print("tick " + " ".join("%15s" % k for k in KEYS) + "       kernel_us")
    for t, r in enumerate(rows):
        print("%4d " % t + " ".join("%15d" % r[k] for k in KEYS) + "%16.2f" % r["kernel_us"])
    print("sum  " + " ".join("%15d" % total[k] for k in KEYS) + "%16.2f" % total["kernel_us"])
    print("digest %016x" % digest[0])


if __name__ == "__main__":
    main()
