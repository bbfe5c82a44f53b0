"""A test-side reader of gsim_snapshot blobs (version 3, single-GPU layouts), and their canonical form.

`parse(blob)` reads a blob in the order gs_api.cpp gsim_snapshot writes it: the SnapHeader (with GsGlobals),
the Sched entries, the 30 rumor headers, then every column plane in snap_cols order.  Columns come back as
named numpy arrays shaped [planes][cap] (tx: [rumor][cap], two rumors per 16-bit element as in gs_core.h
GS_TX); the pool-wide words (stats, heard_cnt, ...) as [1][count].  `serialise(state)` writes the same bytes
back, so a parse that drifted from the writer's layout cannot go unnoticed.

`canonical(blob)` is the parsed state with the fields zeroed that no later tick or host call can read, so that
two pools which took the same operations on different backends give equal canonical states:

- the fields gs_aux.h gs_hash_row folds are masked exactly as it masks them (`due` while up, the probe while
  probing, the suspicion record while Suspect, `change_tick` from Dead, `tx` of heard rumors, `heard`,
  `queued` and the mailboxes under the active rumor mask and the ACC bit), with GS_META_DIRTY and
  GS_WAKE_BIT stripped as gsim_column_read strips them;
- every other column, the counters, the Sched entries, the rumor headers and GsGlobals are compared raw.  The
  few masks beyond the digest's rules are listed in EXTRA_MASKS, each with the code that shows the field is
  written before it is read."""
from __future__ import annotations

import ctypes as C
import struct

import numpy as np

MAGIC = 0x4753494D534E4150           # "GSIMSNAP"
VERSION = 3
SNAP_HEADER_SIZE = 5312              # sizeof(SnapHeader), gs_api.cpp
SCHED_SIZE = 12                      # sizeof(Sched): tick, id, action
GLOBALS_SIZE = 5264                  # sizeof(GsGlobals), gs_core.h
MAX_RUMORS, K1, PPK, COORD_WORDS, ADJ_WINDOW, STAT_COUNT = 30, 5, 4, 11, 20, 16
STAT_ACTIVE_ROWS = 14                # GSIM_STAT_ACTIVE_ROWS

LAYOUT_COORD, LAYOUT_PP, LAYOUT_KST, LAYOUT_IMPAIR, LAYOUT_SHARDED, LAYOUT_PAUSE, LAYOUT_REACH = 1, 2, 4, 8, 16, 32, 64

# key word / meta word / inbox bits (gs_core.h)
META_DIRTY, ACC_BIT, WAKE_BIT = 1 << 8, 0x80000000, 0x40000000
TRUTH_NONE, TRUTH_UP = 0, 1
RANK_SUSPECT, RANK_DEAD = 1, 2


class GsRumor(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("kind", "subject", "inc", "ltime", "origin", "size", "qclass", "start_tick")]


class GsGlobals(C.Structure):
    """gs_core.h GsGlobals, field for field"""
    _fields_ = ([(n, C.c_uint32) for n in ("n", "cap", "up_count", "P", "T", "GI", "gossip_nodes", "indirect_checks",
                                           "awareness_max", "retransmit_limit", "sus_k")]
                + [("sus_ticks", C.c_uint32 * K1)]
                + [(n, C.c_uint32) for n in ("gtd_ticks", "udp_avail", "disable_tcp", "loss_thr", "event_buffer",
                                             "seed_lo", "seed_hi", "active_mask")]
                + [("class_mask", C.c_uint32 * 3)]
                + [(n, C.c_uint32) for n in ("perm_bits", "flags", "evlog_cap", "world", "rank", "phase_group",
                                             "phase_gate", "phase_shift", "rot_p", "rot_g", "rows_per_rank",
                                             "key_stride", "ring_mask", "n_dcs")]
                + [("lat", C.c_uint8 * (64 * 64))]
                + [(n, C.c_uint32) for n in ("pp_interval", "rot_pp", "graph_n", "reap_min_override", "active_bytes")]
                + [("coord_base_rtt_s", C.c_double), ("tick_seconds", C.c_double), ("n_magic", C.c_uint64),
                   ("rumors", GsRumor * MAX_RUMORS)])


assert C.sizeof(GsGlobals) == GLOBALS_SIZE
_HEAD = struct.Struct("<QIIIIQIIQ")  # magic, version, cap, now, n_sched, node_ticks, n_established, layout, graph_hash
assert _HEAD.size + GLOBALS_SIZE == SNAP_HEADER_SIZE


def columns(layout: int, depth: int):
    """snap_cols for a blob of this layout and mailbox ring depth: (name, dtype, planes, per_member, may_fill)
    entries in blob order; name repeats for columns stored as several SnapCols (the two key buffers, the ring)"""
    u32, u64, u8, f64 = np.uint32, np.uint64, np.uint8, np.float64
    v = [("key", u32, 1, True, False), ("key", u32, 1, True, False)]
    v += [("inbox", u32, 1, True, True)] * depth
    v += [(n, u32, 1, True, True) for n in ("due", "meta", "cursor", "pass", "probe_tgt", "probe_inc", "sus_start")]
    v += [("sus_from", u32, K1, True, True), ("acc", u64, 2 * K1, True, True), ("change_tick", u32, 1, True, True),
          ("reap_after", u32, 1, True, True)]
    v += [(n, u32, 1, True, True) for n in ("ltime_member", "ltime_event", "event_min", "heard", "queued")]
    v += [("tx", u8, MAX_RUMORS // 2, True, True)]                      # planes of 2 bytes per member
    if layout & LAYOUT_KST:
        v += [("kst", u8, 1, True, True)]
    if layout & LAYOUT_COORD:
        v += [("coord", f64, 2 * COORD_WORDS, True, True), ("ctag", u32, 2, True, True),
              ("adj", f64, ADJ_WINDOW, True, True), ("adj_idx", u32, 1, True, True)]
    if layout & LAYOUT_PP:
        v += [("ppreq", u32, 2 * PPK, True, True), ("pp_clk", u32, 4, True, True)]
    if layout & LAYOUT_IMPAIR:
        v += [("imp_loss", u32, 1, True, True), ("imp_delay", u8, 1, True, True)]
    if layout & LAYOUT_REACH:
        v += [("imp_recv", u32, 1, True, True), ("imp_flags", u8, 1, True, True)]
    if layout & LAYOUT_PAUSE:
        v += [("pause_until", u32, 1, True, True), ("pause_cnt", u64, 1, False, False)]
    v += [("stats", u64, 1, False, False), ("heard_cnt", u32, 1, False, False), ("conv_tick", u32, 1, False, False),
          ("crashed_alive", u32, 1, False, False), ("crashed_dead_tick", u32, 1, False, False)]
    return v


WORDS = {"pause_cnt": 4, "stats": STAT_COUNT, "heard_cnt": 32, "conv_tick": 32, "crashed_alive": 1,
         "crashed_dead_tick": 1}


def _plane_bytes(name, dtype, per_member, cap):
    if name == "tx":
        return 2 * cap
    return (cap if per_member else WORDS[name]) * np.dtype(dtype).itemsize


def parse(blob: bytes) -> dict:
    """The blob's state: {'header': {...}, 'globals': GsGlobals, 'sched': [n][3] u32, 'rumors': [(name, payload,
    coalesce)], 'cols': {name: [planes][cap] array}, 'tags': [(name, tag)] per plane in blob order}"""
    blob = bytes(blob)
    if len(blob) < SNAP_HEADER_SIZE:
        raise ValueError("shorter than a snapshot header")
    magic, version, cap, now, n_sched, node_ticks, n_est, layout, graph_hash = _HEAD.unpack_from(blob, 0)
    if magic != MAGIC or version != VERSION:
        raise ValueError(f"not a version {VERSION} gsim snapshot")
    if layout & LAYOUT_SHARDED:
        raise ValueError("sharded blobs are not read here")
    g = GsGlobals.from_buffer_copy(blob, _HEAD.size)
    header = dict(cap=cap, now=now, n_sched=n_sched, node_ticks=node_ticks, n_established=n_est, layout=layout,
                  graph_hash=graph_hash)
    r = SNAP_HEADER_SIZE
    sched = np.frombuffer(blob, np.uint32, 3 * n_sched, r).reshape(n_sched, 3).copy()
    r += SCHED_SIZE * n_sched
    rumors = []
    for _ in range(MAX_RUMORS):
        nl, pl, co = struct.unpack_from("<III", blob, r)
        r += 12
        rumors.append((blob[r:r + nl], blob[r + nl:r + nl + pl], co))
        r += nl + pl
    planes, tags = {}, []
    for name, dtype, nplanes, per_member, may_fill in columns(layout, g.ring_mask + 1):
        pb = _plane_bytes(name, dtype, per_member, cap)
        for _ in range(nplanes):
            (tag,) = struct.unpack_from("<I", blob, r)
            if tag == 1:
                assert may_fill and pb >= 8, f"{name}: a fill where the writer never stores one"
                raw = blob[r + 4:r + 8] * (pb // 4)
                r += 8
            else:
                assert tag == 0, f"{name}: corrupt plane tag {tag}"
                raw = blob[r + 4:r + 4 + pb]
                assert len(raw) == pb, f"{name}: truncated"
                r += 4 + pb
            tags.append((name, tag))
            planes.setdefault(name, []).append(np.frombuffer(raw, dtype).copy())
    assert r == len(blob), f"{len(blob) - r} bytes left over after the last plane"
    cols = {name: np.stack(p) for name, p in planes.items()}
    # two rumors per 16-bit element: plane q holds (rumor 2q, rumor 2q + 1) of member i at bytes 2i, 2i + 1
    cols["tx"] = cols["tx"].reshape(MAX_RUMORS // 2, cap, 2).transpose(0, 2, 1).reshape(MAX_RUMORS, cap)
    return dict(header=header, globals=g, sched=sched, rumors=rumors, cols=cols, tags=tags)


def serialise(state: dict) -> bytes:
    """The blob gsim_snapshot writes for this state (planes of one repeated word stored as a fill)"""
    h, g = state["header"], state["globals"]
    out = [_HEAD.pack(MAGIC, VERSION, h["cap"], h["now"], len(state["sched"]), h["node_ticks"], h["n_established"],
                      h["layout"], h["graph_hash"]), bytes(g), np.ascontiguousarray(state["sched"], np.uint32).tobytes()]
    for name, payload, co in state["rumors"]:
        out += [struct.pack("<III", len(name), len(payload), co), bytes(name), bytes(payload)]
    cols = dict(state["cols"])
    cap = h["cap"]
    cols["tx"] = np.ascontiguousarray(cols["tx"]).reshape(MAX_RUMORS // 2, 2, cap).transpose(0, 2, 1).reshape(
        MAX_RUMORS // 2, 2 * cap)
    seen = {}
    for name, dtype, nplanes, per_member, may_fill in columns(h["layout"], g.ring_mask + 1):
        for _ in range(nplanes):
            q = seen.get(name, 0)
            seen[name] = q + 1
            raw = np.ascontiguousarray(cols[name][q], dtype).tobytes()
            if may_fill and len(raw) >= 8 and raw[:-4] == raw[4:]:
                out += [struct.pack("<I", 1), raw[:4]]
            else:
                out += [struct.pack("<I", 0), raw]
    return b"".join(out)


# ---- canonical form ---------------------------------------------------------------------------------
# Masks beyond gs_hash_row's rules, each with the code that writes the field before anything reads it:
EXTRA_MASKS = {
    # gs_row.h gs_row_step_body counts GS_ST_ACTIVE_ROWS for rows that leave the tick kernel's scan, and the
    # CUDA kernels count whole probing tiles there (gs_cuda.cu): a scheduling diagnostic that no tick reads
    # and gsim_stats_get only reports (tests/parity.py compare_stats skips it too).
    "stats[ACTIVE_ROWS]": "scheduling diagnostic",
    # Rows of ids >= n have not been created.  gs_aux.h gs_init_row writes every per-member column of the core
    # set, the coordinates and the push-pull mailboxes when member_add creates the row, and
    # gs_api.cpp init_device_state leaves the coordinate columns of those rows unset (uninitialised device
    # memory on CUDA, zeros in the host emulation).  The impairment, reachability and pause columns, which
    # gs_init_row does not write, stay compared on every row.
    "rows >= n": "written by gs_init_row before any read",
}
_NOT_INIT = ("imp_loss", "imp_delay", "imp_recv", "imp_flags", "pause_until")


def canonical(blob) -> dict:
    """parse(blob) with the dead fields zeroed (see the module docstring and EXTRA_MASKS)"""
    s = parse(blob) if isinstance(blob, (bytes, bytearray)) else blob
    g, now = s["globals"], s["header"]["now"]
    cols = {k: v.copy() for k, v in s["cols"].items()}
    cap, n = s["header"]["cap"], g.n
    act, depth = g.active_mask, g.ring_mask + 1
    cur = now & 1
    key = cols["key"][cur]
    truth, rank = key & 3, (key >> 2) & 3
    exists = truth != TRUTH_NONE
    up = truth == TRUTH_UP
    meta = cols["meta"][0] & ~np.uint32(META_DIRTY)
    probing = up & (((meta >> 3) & 3) != 0)

    def keep(name, mask):
        cols[name] = np.where(mask, cols[name], 0).astype(cols[name].dtype)

    # gs_hash_row's rules.  A row whose key (in the buffer the next tick reads) has truth NONE folds nothing
    # of these fields; for one that exists, they are folded under these masks.
    cols["meta"][0] = meta
    for name in ("meta", "cursor", "pass", "ltime_member", "ltime_event", "event_min"):
        keep(name, exists)
    keep("due", up)
    keep("probe_tgt", probing)
    keep("probe_inc", probing)
    keep("sus_start", exists & (rank == RANK_SUSPECT))
    keep("sus_from", (exists & (rank == RANK_SUSPECT))[None, :])
    keep("change_tick", exists & (rank >= RANK_DEAD))
    for name in ("heard", "queued"):
        keep(name, exists)
        cols[name] &= np.uint32(act)
    heard_bits = ((cols["heard"][0][None, :] >> np.arange(MAX_RUMORS, dtype=np.uint32)[:, None]) & 1).astype(bool)
    keep("tx", heard_bits)
    inbox = cols["inbox"]
    live = np.zeros_like(inbox)
    slot = now & g.ring_mask
    live[slot] = inbox[slot] & np.uint32(act | ACC_BIT)                # stripped of GS_WAKE_BIT
    for d in range(1, g.ring_mask):                                    # packets in flight
        live[(now + d) & g.ring_mask] = inbox[(now + d) & g.ring_mask] & np.uint32(act)
    cols["inbox"] = np.where(exists[None, :], live, 0).astype(np.uint32)
    # the mailboxes of the buffer the next tick reads, while the ACC bit says there is mail in them (the other
    # buffer, emptied entry by entry by the tick that read it, is compared raw)
    accbit = exists & ((inbox[slot] & np.uint32(ACC_BIT)) != 0)
    acc = cols["acc"].reshape(2, K1, cap)
    acc[cur] = np.where(accbit[None, :], acc[cur], 0)
    if "ppreq" in cols and g.pp_interval != 0:
        req = cols["ppreq"].reshape(2, PPK, cap)
        req[cur] = np.where(accbit[None, :], req[cur], 0)
        clk = cols["pp_clk"].reshape(2, 2, cap)
        clk[cur] = np.where(accbit[None, :], clk[cur], 0)
    # EXTRA_MASKS
    cols["stats"][0][STAT_ACTIVE_ROWS] = 0
    for name, v in cols.items():
        if v.shape[-1] == cap and name not in _NOT_INIT:
            v[..., n:] = 0
    if "coord" in cols:
        cols["coord"] = cols["coord"].view(np.uint64)                  # bit for bit
        cols["adj"] = cols["adj"].view(np.uint64)
    return dict(header=s["header"], globals=bytes(s["globals"]), sched=s["sched"], rumors=s["rumors"], cols=cols,
                n=n)


def newer_coordinates(state: dict) -> np.ndarray:
    """[n][11] float64 of a parsed state: each member's newer coordinate slot (gs_hash_row's choice:
    ctag[1] > ctag[0])"""
    cols, n, cap = state["cols"], state["globals"].n, state["header"]["cap"]
    c = cols["coord"].reshape(2, COORD_WORDS, cap)
    slot = (cols["ctag"][1] > cols["ctag"][0]).astype(np.intp)
    return np.where(slot[None, :] == 1, c[1], c[0])[:, :n].T.copy()


def first_difference(a: dict, b: dict):
    """None if two canonical states are equal, else a one-line description of the first difference: the
    column, plane and member with both values"""
    for part in ("header", "globals"):
        if a[part] != b[part]:
            if part == "header":
                diff = {k: (a[part][k], b[part][k]) for k in a[part] if a[part][k] != b[part][k]}
                return f"header differs: {diff}"
            x, y = np.frombuffer(a[part], np.uint8), np.frombuffer(b[part], np.uint8)
            off = int(np.nonzero(x != y)[0][0])
            return f"GsGlobals differs at byte {off}"
    if not np.array_equal(a["sched"], b["sched"]):
        return f"Sched differs: {a['sched'].tolist()} vs {b['sched'].tolist()}"
    for r, (x, y) in enumerate(zip(a["rumors"], b["rumors"])):
        if x != y:
            return f"rumor header {r} differs: {x} vs {y}"
    if a["cols"].keys() != b["cols"].keys():
        return f"column sets differ: {sorted(a['cols'])} vs {sorted(b['cols'])}"
    for name, x in a["cols"].items():
        y = b["cols"][name]
        if not np.array_equal(x, y):
            plane, member = (int(v) for v in np.argwhere(x != y)[0])
            count = int(np.count_nonzero(x != y))
            return (f"column {name} plane {plane} member {member}: {x[plane, member]:#x} vs {y[plane, member]:#x}"
                    f" ({count} elements differ)")
    return None


def assert_same(blob_a, blob_b, where=""):
    d = first_difference(canonical(blob_a), canonical(blob_b))
    assert d is None, f"full state differs {where}: {d}"
