"""ctypes binding of the libgsim C ABI (include/gsim.h).

The product library is ``consul_b200/libgsim.so`` (CUDA, sm_90a).  It is loaded lazily and
there is no fallback: if the shared object is missing or no H100-class device is usable the
calls raise.  ``load(path)`` exists so the test-suite can bind the same signatures to the
host-emulation build under ``tests/hostemu`` (test infrastructure, never used by the package).
"""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
DEFAULT_LIB = os.path.join(HERE, "libgsim.so")

GSIM_MAX_RUMORS = 30
GSIM_MAX_SUSPICION_SLOTS = 5
GSIM_STAT_COUNT = 16

STAT_NAMES = [
    "probes", "acks", "indirect_pings", "nacks", "probe_failures", "suspects", "confirmations",
    "deads", "refutes", "gossip_packets", "rumors_sent", "rumors_accepted", "rumors_dropped",
    "packets_lost", "active_rows", "push_pulls",
]

COLUMNS = {
    "key": 0, "meta": 1, "due": 2, "cursor": 3, "pass": 4, "probe_tgt": 5, "probe_inc": 6,
    "sus_start": 7, "sus_from": 8, "change_tick": 9, "ltime_member": 10, "ltime_event": 11,
    "event_min": 12, "heard": 13, "queued": 14, "tx": 15, "inbox": 16,
}


class GsimConfig(C.Structure):
    _fields_ = [
        ("struct_size", C.c_uint32), ("flags", C.c_uint32), ("seed", C.c_uint64),
        ("capacity", C.c_uint32), ("n_initial", C.c_uint32), ("tick_ns", C.c_uint64),
        ("probe_interval_ns", C.c_uint64), ("probe_timeout_ns", C.c_uint64),
        ("gossip_interval_ns", C.c_uint64), ("gossip_to_the_dead_ns", C.c_uint64),
        ("push_pull_interval_ns", C.c_uint64),
        ("gossip_nodes", C.c_uint32), ("indirect_checks", C.c_uint32),
        ("retransmit_mult", C.c_uint32), ("suspicion_mult", C.c_uint32),
        ("suspicion_max_timeout_mult", C.c_uint32), ("awareness_max_multiplier", C.c_uint32),
        ("udp_buffer_size", C.c_uint32), ("disable_tcp_pings", C.c_uint32),
        ("packet_loss_ppm", C.c_uint32),
        ("event_buffer", C.c_uint32), ("user_event_size_limit", C.c_uint32),
        ("leave_propagate_delay_ns", C.c_uint64), ("broadcast_timeout_ns", C.c_uint64),
        ("reap_interval_ns", C.c_uint64), ("reconnect_timeout_ns", C.c_uint64),
        ("tombstone_timeout_ns", C.c_uint64),
        ("world_size", C.c_uint32), ("rank", C.c_uint32), ("device", C.c_int32),
        ("event_log_capacity", C.c_uint32), ("phase_group", C.c_uint32), ("mailbox_depth", C.c_uint32),
    ]


class GsimMemberDesc(C.Structure):
    _fields_ = [("alive_msg_size", C.c_uint32), ("flags", C.c_uint32), ("name_len", C.c_uint32),
                ("meta_len", C.c_uint32)]


class GsimMember(C.Structure):
    _fields_ = [("id", C.c_uint32), ("status", C.c_int32), ("incarnation", C.c_uint32),
                ("rank", C.c_uint32)]


class GsimEvent(C.Structure):
    _fields_ = [("tick", C.c_uint32), ("type", C.c_uint32), ("subject", C.c_uint32),
                ("observer", C.c_uint32), ("ltime", C.c_uint32), ("reserved", C.c_uint32)]


class GsimRumorInfo(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in (
        "kind", "subject", "incarnation", "ltime", "origin", "size_bytes", "start_tick",
        "heard_count", "converged_tick", "queued_count")]


# gsim_agent_stats, in order (every field a uint32_t)
AGENT_STATS_FIELDS = ("members", "failed", "left", "health_score", "member_time", "event_time", "query_time",
                      "intent_queue", "event_queue", "query_queue", "memberlist_queue", "running")


class GsimStats(C.Structure):
    _fields_ = [
        ("counters", C.c_uint64 * GSIM_STAT_COUNT), ("node_ticks", C.c_uint64),
        ("tick", C.c_uint32), ("n_members", C.c_uint32),
        ("n_up", C.c_uint32), ("n_crashed", C.c_uint32), ("n_gone", C.c_uint32),
        ("n_view_alive", C.c_uint32), ("n_view_suspect", C.c_uint32),
        ("n_view_dead", C.c_uint32), ("n_view_left", C.c_uint32),
        ("retransmit_limit", C.c_uint32), ("suspicion_k", C.c_uint32),
        ("suspicion_ticks", C.c_uint32 * GSIM_MAX_SUSPICION_SLOTS),
        ("probe_interval_ticks", C.c_uint32), ("probe_timeout_ticks", C.c_uint32),
        ("gossip_interval_ticks", C.c_uint32), ("events_dropped", C.c_uint32),
    ]


# every symbol include/gsim.h declares: (name, restype, argtypes)
_P = C.c_void_p
_u32, _u64, _i32, _sz = C.c_uint32, C.c_uint64, C.c_int, C.c_size_t
SIGNATURES = [
    ("gsim_config_default_lan", None, [C.POINTER(GsimConfig)]),
    ("gsim_config_default_wan", None, [C.POINTER(GsimConfig)]),
    ("gsim_config_consul_test", None, [C.POINTER(GsimConfig)]),
    ("gsim_retransmit_limit", _u32, [_u32, _u32]),
    ("gsim_suspicion_timeout_ns", _u64, [_u32, _u32, _u64]),
    ("gsim_remaining_suspicion_ns", C.c_int64, [_u32, _u32, _u64, _u64, _u64]),
    ("gsim_push_pull_scale_ns", _u64, [_u64, _u32]),
    ("gsim_lamport_witness", _u32, [_u32, _u32]),
    ("gsim_refute_incarnation", _u32, [_u32, _u32]),
    ("gsim_philox4x32", None, [C.POINTER(_u32), C.POINTER(_u32), C.POINTER(_u32)]),
    ("gsim_pool_create", _i32, [C.POINTER(GsimConfig), C.POINTER(_P)]),
    ("gsim_pool_destroy", None, [_P]),
    ("gsim_strerror", C.c_char_p, [_i32]),
    ("gsim_last_error", C.c_char_p, [_P]),
    ("gsim_abi_version", _i32, []),
    ("gsim_member_add", _i32, [_P, C.POINTER(GsimMemberDesc), C.POINTER(_u32)]),
    ("gsim_join", _i32, [_P, _u32, C.POINTER(_u32), _sz, _i32, C.POINTER(_i32)]),
    ("gsim_leave", _i32, [_P, _u32]),
    ("gsim_crash", _i32, [_P, _u32]),
    ("gsim_crash_many", _i32, [_P, C.POINTER(_u32), _sz]),
    ("gsim_crash_fraction", _i32, [_P, _u32, _u32, C.POINTER(_u32)]),
    ("gsim_force_leave", _i32, [_P, _u32, _u32, _i32]),
    ("gsim_user_event", _i32, [_P, _u32, C.c_char_p, _sz, C.c_char_p, _sz, _i32, C.POINTER(_u32)]),
    ("gsim_rumor_inject", _i32, [_P, _u32, _u32, C.POINTER(_i32)]),
    ("gsim_latency_set", _i32, [_P, _u32, C.POINTER(C.c_uint8)]),
    ("gsim_impair_many", _i32, [_P, C.POINTER(_u32), _sz, _u32, _u32]),
    ("gsim_impair_fraction", _i32, [_P, _u32, _u32, _u32, _u32, C.POINTER(_u32)]),
    ("gsim_impair_get", _i32, [_P, _u32, C.POINTER(_u32), C.POINTER(_u32)]),
    ("gsim_impair_dir_many", _i32, [_P, C.POINTER(_u32), _sz, _u32, _u32, _u32, _u32]),
    ("gsim_impair_dir_fraction", _i32, [_P, _u32, _u32, _u32, _u32, _u32, _u32, C.POINTER(_u32)]),
    ("gsim_impair_dir_get", _i32, [_P, _u32, C.POINTER(_u32), C.POINTER(_u32), C.POINTER(_u32), C.POINTER(_u32)]),
    ("gsim_impair_flap_many", _i32, [_P, C.POINTER(_u32), _sz, _u32, _u32]),
    ("gsim_impair_flap_fraction", _i32, [_P, _u32, _u32, _u32, _u32, C.POINTER(_u32)]),
    ("gsim_impair_flap_get", _i32, [_P, _u32, C.POINTER(_u32), C.POINTER(_u32)]),
    ("gsim_impair_flap_stats", _i32, [_P, C.POINTER(_u64)]),
    ("gsim_flap_bad", _i32, [_u64, _u32, _u32, _u32, _u32]),
    ("gsim_domain_set_many", _i32, [_P, C.POINTER(_u32), _sz, _u32]),
    ("gsim_domain_set_range", _i32, [_P, _u32, _u32, _u32, _u32]),
    ("gsim_domain_get", _i32, [_P, _u32, _u32, _P]),
    ("gsim_domain_flap_set", _i32, [_P, C.POINTER(_u32), _sz, _u32, _u32]),
    ("gsim_domain_flap_get", _i32, [_P, _u32, C.POINTER(_u32), C.POINTER(_u32)]),
    ("gsim_domain_flap_bad", _i32, [_u64, _u32, _u32, _u32, _u32]),
    ("gsim_domain_impair", _i32, [_P, C.POINTER(_u32), _sz, _u32, _u32, _u32, _u32, C.POINTER(_u32)]),
    ("gsim_domain_crash", _i32, [_P, C.POINTER(_u32), _sz, C.POINTER(_u32)]),
    ("gsim_domain_pause", _i32, [_P, C.POINTER(_u32), _sz, _u32, C.POINTER(_u32)]),
    ("gsim_domain_stats_read", _i32, [_P, _u32, _u32, _P]),
    ("gsim_pause_many", _i32, [_P, C.POINTER(_u32), _sz, _u32, C.POINTER(_u32)]),
    ("gsim_pause_fraction", _i32, [_P, _u32, _u32, _u32, C.POINTER(_u32)]),
    ("gsim_pause_get", _i32, [_P, _u32, C.POINTER(_u32)]),
    ("gsim_pause_stats", _i32, [_P, C.POINTER(_u64)]),
    ("gsim_graph_set", _i32, [_P, _u32, C.POINTER(_u32), C.POINTER(_u32)]),
    ("gsim_member_reconnect_timeout_set", _i32, [_P, _u32, _u64]),
    ("gsim_coordinate_get", _i32, [_P, _u32, C.POINTER(C.c_double)]),
    ("gsim_coordinates_read", _i32, [_P, _u32, _u32, C.POINTER(C.c_double)]),
    ("gsim_rtt_many", _i32, [_P, C.POINTER(_u32), C.POINTER(_u32), _sz, C.POINTER(C.c_double),
                             C.POINTER(C.c_double)]),
    ("gsim_sort_by_distance", _i32, [_P, _u32, C.POINTER(_u32), _sz, _sz, C.POINTER(_u32),
                                     C.POINTER(C.c_double)]),
    ("gsim_dcs_by_distance", _i32, [_P, _u32, C.POINTER(_u32), _sz, C.POINTER(_u32), C.POINTER(C.c_double)]),
    ("gsim_coordinate_error", _i32, [_P, _u32, _u32, C.POINTER(C.c_double)]),
    ("gsim_member_watch", _i32, [_P, _u32, _i32]),
    ("gsim_member_update", _i32, [_P, _u32, _u32, C.POINTER(_u32)]),
    ("gsim_step", _i32, [_P, _u32]),
    ("gsim_run_until", _i32, [_P, _i32, _u32, _u32, _u32, C.POINTER(_u32)]),
    ("gsim_now", _u32, [_P]),
    ("gsim_members", _i32, [_P, _u32, C.POINTER(GsimMember), _sz, C.POINTER(_sz)]),
    ("gsim_num_nodes", _i32, [_P, _u32, C.POINTER(_u32)]),
    ("gsim_agent_stats_read", _i32, [_P, _u32, _u32, _P]),
    ("gsim_health_histogram", _i32, [_P, C.POINTER(_u64)]),
    ("gsim_poll_events", _i32, [_P, C.POINTER(GsimEvent), _sz, C.POINTER(_sz)]),
    ("gsim_rumor_info_get", _i32, [_P, _u32, C.POINTER(GsimRumorInfo)]),
    ("gsim_rumor_retire", _i32, [_P, _u32]),
    ("gsim_user_event_get", _i32, [_P, _u32, _P, _sz, C.POINTER(_sz), _P, _sz, C.POINTER(_sz)]),
    ("gsim_stats_get", _i32, [_P, C.POINTER(GsimStats)]),
    ("gsim_state_hash", _i32, [_P, C.POINTER(_u64)]),
    ("gsim_column_read", _i32, [_P, _i32, _P, _sz, C.POINTER(_sz)]),
    ("gsim_snapshot_size", _i32, [_P, C.POINTER(_sz)]),
    ("gsim_snapshot", _i32, [_P, _P, _sz, C.POINTER(_sz)]),
    ("gsim_restore", _i32, [_P, _P, _sz]),
    ("gsim_shard_export_fds", _i32, [_P, C.POINTER(_i32), _sz, C.POINTER(_sz)]),
    ("gsim_shard_attach", _i32, [_P, _u32, C.POINTER(_i32), _sz]),
    ("gsim_shard_ready", _i32, [_P]),
    ("gsim_last_step_timing", _i32, [_P, C.POINTER(C.c_double), C.POINTER(_u64)]),
    ("gsim_launch_count", _u64, [_P]),
    ("gsim_sched_counts", _i32, [_P, C.POINTER(_u64)]),
    ("gsim_piggyback_stats", _i32, [_P, C.POINTER(_u64)]),
    ("gsim_ring_entry", _u32, [_u64, _u32, _u32, _u32, _u32]),
    ("gsim_ring_position", _u32, [_u64, _u32, _u32, _u32, _u32]),
    ("gsim_wire_alive", _sz, [_P, _sz, _u32, C.c_char_p, _P, _sz, C.c_uint16, _P, _sz, C.POINTER(C.c_uint8)]),
    ("gsim_wire_suspect", _sz, [_P, _sz, _u32, C.c_char_p, C.c_char_p]),
    ("gsim_wire_dead", _sz, [_P, _sz, _u32, C.c_char_p, C.c_char_p]),
    ("gsim_wire_join_intent", _sz, [_P, _sz, _u64, C.c_char_p]),
    ("gsim_wire_leave_intent", _sz, [_P, _sz, _u64, C.c_char_p, _i32]),
    ("gsim_wire_user_event", _sz, [_P, _sz, _u64, _P, _sz, _P, _sz, _i32]),
    ("gsim_wire_compound", _sz, [_P, _sz, C.POINTER(_P), C.POINTER(_sz), _sz]),
    ("gsim_wire_wanfed_frame", _sz, [_P, _sz, _P, _sz]),
    ("gsim_wire_ping", _sz, [_P, _sz, _u32, C.c_char_p, _P, _sz, C.c_uint16, C.c_char_p]),
    ("gsim_wire_indirect_ping", _sz, [_P, _sz, _u32, _P, _sz, C.c_uint16, C.c_char_p, _i32, _P, _sz, C.c_uint16,
                                      C.c_char_p]),
    ("gsim_wire_ack", _sz, [_P, _sz, _u32, _P, _sz]),
    ("gsim_wire_nack", _sz, [_P, _sz, _u32]),
    ("gsim_wire_consul_user_event", _sz, [_P, _sz, C.c_char_p, C.c_char_p, _P, _sz, C.c_char_p, C.c_char_p,
                                          C.c_char_p, _i32]),
]


def load(path: str = DEFAULT_LIB) -> C.CDLL:
    """dlopen a libgsim build and attach the header's signatures.  Raises if missing."""
    if not os.path.exists(path):
        raise OSError(
            f"{path} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(libgsim has no CPU fallback)")
    lib = C.CDLL(path)
    for name, res, args in SIGNATURES:
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    return lib


_LIB = None


def lib() -> C.CDLL:
    global _LIB
    if _LIB is None:
        _LIB = load(DEFAULT_LIB)
    return _LIB
