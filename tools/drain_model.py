"""Model of the tick kernel's drain over one bench-step join cascade (dev tool, host emulation).

A LAN pool, step(64), WARMUP bench steps (member_add -> join(x, [0]) -> step(2048)), one more member_add +
join, then single ticks until the cascade is over.  Before each tick the columns say which members need the
generic row step (mail, a gossip turn at this tick, a suspect or dead view; probes mostly go through the
staged fast path in the scan and are left out); the model
splits the scan positions over CTAS x 8 warps as gs_tick_kernel does (contiguous, floor or ceil of
tiles / warps each) and counts, per tick, the warp-steps of the busiest CTA's warps:

  groups   one warp-step per 32-member group with an active member, tiles in order (the drain before
           members were queued one by one)
  rows     active members packed 32 per warp-step, tiles in order (gs_tick_kernel's drain)
  dealt    packed, and the scan positions dealt to tiles so that runs of tiles of different gossip phase
           alternate (deal_tiles below): every CTA gets an even share of the gossiping tiles

It assumes that a warp-step costs the same whether its lanes are a sparse group or 32 packed members, and
that a tick waits for its busiest CTA; the kernel time per tick on an H100 is what tools/cascade_rows.py
measures.  The second assumption does not hold in the plateau of the cascade (DESIGN.md §6): a tick kernel
with the dealing took as long there as without it, so the kernel does not deal.

    python tools/drain_model.py [--members 1000000] [--ctas 528] [--per-tick]
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from consul_b200 import _lib  # noqa: E402
from consul_b200.pool import Pool, lan_config  # noqa: E402

TILE, WARPS_PER_CTA = 128, 8


def deal_alternate(j, L, R):
    """tile j of a stretch of L tiles that starts a run of R and alternates between its runs: q = L // R whole
    runs and one of rem = L % R tiles; the first rem * (q + 1) positions alternate over all q + 1 runs, the rest
    over the q whole ones"""
    q, rem = L // R, L % R
    first = j < rem * (q + 1)
    j2 = j - rem * (q + 1)
    return np.where(first, (j % (q + 1)) * R + j // (q + 1),
                    (j2 % max(q, 1)) * R + rem + j2 // max(q, 1))


def deal_tiles(lo, hi, P, shift, GI):
    """The tile scanned at every position of [lo, hi) when positions are dealt: gossip phases come in runs of
    R = P << phase_shift tiles; the positions alternate between the runs of every whole block of GI * R tiles
    (run k entered 2k phase groups in, so neighbours do not share their probe phase either), and the E tiles
    outside whole blocks take E positions spread evenly over the range.  A bijection of [lo, hi)."""
    s = np.arange(lo, hi, dtype=np.int64)
    if P == 0 or GI <= 1:
        return s
    R = P << shift
    B = GI * R
    a0 = min(-(-lo // B) * B, hi)
    a1 = max(hi // B * B, a0)
    n, head = hi - lo, a0 - lo
    E = head + (hi - a1)
    r = s - lo
    out = np.empty_like(s)
    before = np.zeros_like(s)
    extra = np.zeros(len(s), dtype=bool)
    if E:
        k = (r * E) // n
        pk = ((2 * k + 1) * n) // (2 * E)
        extra = pk == r
        before = k + (pk < r)
        kh = k[extra]
        out[extra] = np.where(kh < head, lo + deal_alternate(kh, head, R),
                              a1 + deal_alternate(kh - head, hi - a1, R))
    b = (r - before)[~extra]
    j = b % B
    kk = j % GI
    out[~extra] = a0 + (b - j) + kk * R + (j // GI + ((2 * kk) << shift)) % R
    return out


def ceil_div(a, b):
    return -(-a // b)


def busiest(per_pos, bounds):
    """the most any CTA has of per_pos summed over its positions"""
    return int(np.add.reduceat(per_pos, bounds[:-1]).max()) if per_pos.any() else 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=os.path.join(ROOT, "tests", "hostemu", "libgsim_hostemu.so"))
    ap.add_argument("--members", type=int, default=1_000_000)
    ap.add_argument("--ctas", type=int, default=132 * 4, help="CTAs of the tick grid (SMs x resident CTAs)")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--per-tick", action="store_true")
    args = ap.parse_args()
    n = args.members
    lib = _lib.load(args.lib)
    p = Pool(lan_config(lib, capacity=n + 16, n_initial=n, seed=0x5EED0001), lib)
    try:
        p.step(64)
        for _ in range(args.warmup):
            x = p.member_add()
            assert p.join(x, [0]) == 1
            p.step(2048)
        x = p.member_add()
        assert p.join(x, [0]) == 1
        s = p.stats()
        P, GI = s["probe_interval_ticks"], s["gossip_interval_ticks"]
        members = s["n_members"]
        n_tiles = (members + TILE - 1) // TILE
        warps = args.ctas * WARPS_PER_CTA
        bounds = ((np.arange(warps + 1, dtype=np.int64) * n_tiles) // warps)[::WARPS_PER_CTA]
        dealt = deal_tiles(0, n_tiles, P, 0, GI)  # lan_config: one tile per phase group
        m = n_tiles * TILE
        rows = []
        for k in range(400):
            t = p.now
            col = {}
            for name in ("inbox", "heard", "queued", "meta", "key"):
                a = p.column(name)
                b = np.zeros(m, dtype=np.uint64)
                b[:min(m, len(a))] = a[:m]
                col[name] = b
            mail = ((col["inbox"] & 0x3FFFFFFF & ~col["heard"]) != 0) | ((col["inbox"] & 0x80000000) != 0)
            gossip = (col["queued"] != 0) & (((col["meta"] >> 16) & 0xFF) == t % GI)
            other = ((col["key"] >> 2) & 3) != 0
            act = mail | gossip | other
            act[members:] = False
            per_tile = act.reshape(n_tiles, TILE).sum(axis=1)
            groups = act.reshape(n_tiles * 4, 32).any(axis=1).reshape(n_tiles, 4).sum(axis=1)
            row = (k, int(act.sum()), int(groups.sum()),
                   ceil_div(busiest(groups, bounds), WARPS_PER_CTA),
                   ceil_div(ceil_div(busiest(per_tile, bounds), 32), WARPS_PER_CTA),
                   ceil_div(ceil_div(busiest(per_tile[dealt], bounds), 32), WARPS_PER_CTA))
            rows.append(row)
            p.step(1)
            if k > 8 and not act.any():
                break
    finally:
        p.close()
    if args.per_tick:
        print("tick     rows  groups | busiest-CTA warp-steps: groups  rows  dealt")
        for r in rows:
            print("%4d %8d %7d | %30d %5d %6d" % r)
    tot = [sum(r[i] for r in rows) for i in (3, 4, 5)]
    print("%d members, %d CTAs x %d warps, %d ticks: busiest-warp steps per cascade: groups %d, rows %d, "
          "rows dealt %d" % ((members, args.ctas, WARPS_PER_CTA, len(rows)) + tuple(tot)))


if __name__ == "__main__":
    main()
