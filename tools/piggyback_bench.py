"""Broadcasts piggybacked on probe traffic (GSIM_FLAG_PROBE_PIGGYBACK) on one H100: what the flag does to
dissemination and what it costs.

Rows, each with and without the flag on the same seed:
  * C4 user event (BASELINE config 4's shape) at 1 Mi and 16 Mi LAN members: ticks until every member has it,
    and the share of its transmissions that rode on probe traffic;
  * C2 joiner (config 2's shape) at 1 Mi members: ticks until its alive rumor and join intent reached everybody,
    and the tick kernels' CUDA-event time over the cascade's first 64 ticks (gsim_last_step_timing).

Prints the card's name, power limit and max SM clock (read in the same run) and one JSON line per row.

  python tools/piggyback_bench.py [--sizes 1048576,16777216] [--seeds 2] [--out DIR]
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


def share(p, flag):
    if not flag:
        return 0.0
    s, pg = p.stats(), p.piggyback_stats()
    return pg["broadcasts"] / max(1, pg["broadcasts"] + s["rumors_sent"])


def c4_row(n, seed, flag):
    from consul_b200.pool import NEVER, PRED_RUMOR_CONVERGED, Pool, lan_config
    p = Pool(lan_config(capacity=n, n_initial=n, seed=seed, flags=flag))
    slot = p.user_event(0, b"deploy", b"x" * 32, False)
    t = p.run_until(PRED_RUMOR_CONVERGED, slot, 1000, 1)
    p.step(120)                                               # the retransmission tail
    return {"row": "c4_user_event", "members": n, "seed": hex(seed), "flag": bool(flag),
            "ticks_to_all": None if t == NEVER else t, "probe_share": round(share(p, flag), 4),
            "digest": "%016x" % p.state_hash()[0]}


def c2_row(n, seed, flag, timed=64):
    from consul_b200.pool import NEVER, PRED_ALL_RUMORS_CONVERGED, Pool, lan_config
    cfg = lan_config(capacity=n + 1, n_initial=n, seed=seed, flags=flag)
    q = Pool(cfg)                                             # ticks until the joiner's rumors reached everybody
    q.step(2)
    q.join(q.member_add(), [0])
    t = q.run_until(PRED_ALL_RUMORS_CONVERGED, 0, 1000, 1)
    t = None if t == NEVER else t - 2
    del q
    p = Pool(cfg)                                             # the same cascade, one timed tick at a time
    p.step(2)
    x = p.member_add()
    p.join(x, [0])
    ms = 0.0
    for _ in range(timed):
        p.step(1)
        k, _n = p.last_step_timing()
        ms += k
    p.run_until(PRED_ALL_RUMORS_CONVERGED, 0, 1000, 1)
    return {"row": "c2_joiner", "members": n + 1, "seed": hex(seed), "flag": bool(flag),
            "ticks_to_all": t, "kernel_ms_first_%d_ticks" % timed: round(ms, 3),
            "probe_share": round(share(p, flag), 4), "digest": "%016x" % p.state_hash()[0]}


def main():
    from consul_b200.pool import FLAG_PROBE_PIGGYBACK
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1048576,16777216")
    ap.add_argument("--seeds", type=int, default=2)
    ap.add_argument("--c2-rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    rows = [{"card": card()}]
    print(json.dumps(rows[0]), flush=True)
    for n in [int(x) for x in a.sizes.split(",")]:
        for s in range(a.seeds):
            for flag in (0, FLAG_PROBE_PIGGYBACK):
                rows.append(c4_row(n, 0x5EED0003 + s, flag))
                print(json.dumps(rows[-1]), flush=True)
    for r in range(a.c2_rounds):                              # alternating, same process: the spread is visible
        for flag in (0, FLAG_PROBE_PIGGYBACK):
            rows.append(c2_row(1 << 20, 0x5EED0001, flag))
            print(json.dumps(rows[-1]), flush=True)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "piggyback_bench.jsonl"), "w") as f:
            for r in rows:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
