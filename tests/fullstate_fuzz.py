"""Whole-state lockstep fuzz and backend handover, shared by tests/test_fullstate_cpu.py (two host-emulation
pools) and tests/test_gpu_fullstate.py (the H100 against the host emulation): two pools compared through
their snapshots in canonical form (tests/snapblob.py), not only through the digest and the readable columns."""
from __future__ import annotations

import snapblob
from backend_fuzz import Lockstep
from consul_b200.pool import GsimError


class FullStateLockstep(Lockstep):
    """A Lockstep pair whose pools are also compared through their snapshots after every step: the canonical
    state (snapblob.canonical) and the events logged since the last step.  In front of every step both pools
    also take the same ReconnectTimeout override (`member_reconnect_timeout_set`, the device write of
    `reap_after`), from a random stream of its own."""

    RECONNECT = 0x4EC0

    def __init__(self, *a, **kw):
        super().__init__(*a, **kw)
        self.sides, self.compared, self.overrides = None, 0, {}

    def make(self, cfg):
        self.sides = super().make(cfg)
        return self.sides

    def step(self, side, k):
        p = side.pool
        n, now = p.stats()["n_members"], p.now
        rng = self._rng(self.RECONNECT, now)
        rc = None
        if n and rng.random() < 0.3:
            m, t = rng.randrange(n + 2), rng.choice([0, 1, 150, 900, 40_000]) * 1_000_000
            try:
                p.member_reconnect_timeout_set(m, t)
                rc = (m, t, "ok")
            except GsimError as e:
                rc = (m, t, e.code)
        super().step(side, k)
        if side.index == 0:
            self.overrides[now] = rc
            return
        assert self.overrides[now] == rc, f"seed {self.seed} tick {now}: reconnect override {self.overrides[now]} vs {rc}"
        self.compare(f"seed {self.seed}: step {k} from tick {now}")

    def compare(self, where):
        a, b = (s.pool for s in self.sides)
        snapblob.assert_same(a.snapshot(), b.snapshot(), where)
        ea, eb = (sorted((e.tick, e.type, e.subject, e.observer, e.ltime) for e in q.poll_events()) for q in (a, b))
        assert ea == eb, f"{where}: events differ"
        self.compared += 1


def handover(src, stay, fresh, chunks, where=""):
    """Restore src's snapshot into `fresh` (a new pool of the same configuration, possibly on another backend)
    and step it next to `stay`, a pool that took the same operations as src and never switched: their digests
    and canonical states must stay equal after every chunk of ticks."""
    fresh.restore(src.snapshot())
    snapblob.assert_same(fresh.snapshot(), stay.snapshot(), f"{where} right after the restore")
    for c in chunks:
        fresh.step(c)
        stay.step(c)
        assert fresh.state_hash() == stay.state_hash(), f"{where}: digests differ at tick {stay.now}"
        snapblob.assert_same(fresh.snapshot(), stay.snapshot(), f"{where} at tick {stay.now}")
    return fresh
