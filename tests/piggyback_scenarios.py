"""Scenarios for broadcasts piggybacked on probe traffic (GSIM_FLAG_PROBE_PIGGYBACK, DESIGN.md §3.7), shared by
the host-emulation tests and the H100 tests.  Each takes a list of pools built from one config and drives them
through the same operations; `check` compares them wherever it is called."""
from consul_b200.pool import FLAG_PROBE_PIGGYBACK, NEVER, PRED_RUMOR_CONVERGED, lan_config, wan_config
from consul_b200.wan import c5_latency_matrix

SEC = 1_000_000_000


def both(pools, fn):
    out = [fn(p) for p in pools]
    assert all(o == out[0] for o in out), out
    return out[0]


def run_to(pools, checkpoints, check):
    for upto in checkpoints:
        for p in pools:
            p.step(upto - p.now)
        check(pools, upto)


def user_event(make, lib, n, check, seed=0x5EED0003, flags=0, **kw):
    """BASELINE config 4's shape: one user event from member 0; runs until everybody has it, then drains."""
    pools = make(lan_config(lib, capacity=n, n_initial=n, seed=seed, flags=FLAG_PROBE_PIGGYBACK | flags, **kw))
    slot = both(pools, lambda p: p.user_event(0, b"deploy", b"x" * 32, False))
    run_to(pools, (1, 2, 5), check)
    t = both(pools, lambda p: p.run_until(PRED_RUMOR_CONVERGED, slot, 600, 1))
    assert t != NEVER
    run_to(pools, (t + 1, t + 60), check)
    return pools, slot, t


def join_cascade(make, lib, n, check, seed=0x5EED0001, **kw):
    """BASELINE config 2's shape: one joiner through seed 0, its alive rumor and join intent spread."""
    pools = make(lan_config(lib, capacity=n + 1, n_initial=n, seed=seed, flags=FLAG_PROBE_PIGGYBACK, **kw))
    x = both(pools, lambda p: p.member_add())
    both(pools, lambda p: p.join(x, [0]))
    run_to(pools, (3, 10, 20, 40, 80), check)
    return pools


def crash_wave(make, lib, n, check, seed=0x5EED0002, ppm=100000, loss_ppm=20000, checkpoints=(10, 40, 120, 300), **kw):
    """BASELINE config 3's shape: ~10 % crash at tick 0 (indirect probes, nacks, suspicion and dead rumors),
    with pool-wide packet loss."""
    pools = make(lan_config(lib, capacity=n, n_initial=n, seed=seed, flags=FLAG_PROBE_PIGGYBACK,
                            packet_loss_ppm=loss_ppm, **kw))
    both(pools, lambda p: p.crash_fraction(ppm, 7))
    both(pools, lambda p: p.user_event(0, b"during", b"x" * 16, False))   # queues while the indirect stage runs
    run_to(pools, checkpoints[:2], check)
    both(pools, lambda p: p.user_event(3, b"later", b"y" * 16, False))
    run_to(pools, checkpoints[2:], check)
    return pools


def wan_impaired(make, lib, n, check, seed=0x5EED0005, push_pull=False, max_ticks=1500):
    """BASELINE config 5's latency matrix, members with loss and receive delays, one-way members, a user event."""
    from consul_b200.pool import FLAG_PUSH_PULL
    flags = FLAG_PROBE_PIGGYBACK | (FLAG_PUSH_PULL if push_pull else 0)
    pools = make(wan_config(lib, capacity=n, n_initial=n, seed=seed, mailbox_depth=8, flags=flags,
                            push_pull_interval_ns=2 * SEC))
    for p in pools:
        p.latency_set(c5_latency_matrix(64))
    both(pools, lambda p: p.impair_fraction(20000, 2, 100000, 2))
    ids = list(range(5, n, 211))
    for p in pools:
        p.impair_dir(ids[0::2], 1000000, 0)        # outbound UDP lost
        p.impair_dir(ids[1::2], 0, 1000000)        # inbound UDP lost
    slot = both(pools, lambda p: p.user_event(1, b"e", b"x" * 16, False))
    run_to(pools, (2, 7, 30), check)
    t = both(pools, lambda p: p.run_until(PRED_RUMOR_CONVERGED, slot, max_ticks, 1))
    end = pools[0].now
    run_to(pools, (end + 50, end + 300), check)
    return pools
