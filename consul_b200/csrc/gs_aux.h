// gs_aux.h — per-row bodies of the auxiliary kernels (row init, crash injection,
// recount, state digest).  Same sharing arrangement as gs_row.h.
#pragma once
#include "gs_backend.h"
#include "gs_row.h"

// A converged member as serf.Create + a finished join leaves it ([U] memberlist.setAlive:
// incarnation 1; [U] serf.Create: the three Lamport clocks incremented once).
// Probe/gossip ticker phases mirror triggerFunc's random stagger ([U] state.go).
GS_DEV void gs_init_row(const GsDev& d, const GsGlobals& g, uint32_t i, uint32_t now) {
  const size_t cap = g.cap;
  // one stagger draw per phase group (default: per tile of 128 members, so that the
  // failure-detector path is uniform per CTA); phase_group == 1 draws it per member
  const uint32_t group = i / g.phase_group;
  const uint32_t pp = gs_probe_phase(g.rot_p, group, g.P), gp = gs_gossip_phase(g.rot_g, group, g.P, g.GI);
  const uint32_t k = gs_key_make(1u, 0u, GS_RANK_ALIVE, GS_TRUTH_UP);
  gs_key_store(d, g, 0u, i, k);
  gs_key_store(d, g, 1u, i, k);
  for (uint32_t s = 0; s <= g.ring_mask; ++s) d.inbox[s][i] = 0u;
  d.meta[i] = gp << GS_META_GPHASE_SHIFT;
  d.due[i] = now + (pp + g.P - now % g.P) % g.P;  // first tick >= now congruent to the phase
  d.cursor[i] = 0u;
  d.pass[i] = 0u;
  d.probe_tgt[i] = 0u;
  d.probe_inc[i] = 0u;
  d.sus_start[i] = 0u;
  for (uint32_t q = 0; q < GS_K1MAX; ++q) {
    d.sus_from[(size_t)q * cap + i] = GS_EMPTY32;
    d.acc[(size_t)q * cap + i] = GS_EMPTY64;
    d.acc[((size_t)GS_K1MAX + q) * cap + i] = GS_EMPTY64;
  }
  d.change_tick[i] = 0u;
  d.reap_after[i] = 0u;
  d.ltime_member[i] = 1u;
  d.ltime_event[i] = 1u;
  d.event_min[i] = 0u;
  d.heard[i] = 0u;
  d.queued[i] = 0u;
  if (d.coord != nullptr) {  // [U] coordinate.NewCoordinate: the origin, maximal error, minimal height
    GsCoord o;
    gs_coord_origin(o);
    for (uint32_t slot = 0; slot < 2u; ++slot) {
      double* out = d.coord + ((size_t)slot * GS_COORD_WORDS) * cap + i;
      for (uint32_t x = 0; x < GS_COORD_DIM; ++x) out[(size_t)x * cap] = o.vec[x];
      out[(size_t)8 * cap] = o.error;
      out[(size_t)9 * cap] = o.adjustment;
      out[(size_t)10 * cap] = o.height;
      d.ctag[(size_t)slot * cap + i] = 0u;
    }
    for (uint32_t s = 0; s < GS_ADJ_WINDOW; ++s) d.adj[(size_t)s * cap + i] = 0.0;
    d.adj_idx[i] = 0u;
  }
  if (d.ppreq != nullptr) {
    for (uint32_t q = 0; q < 2u * GS_PPK; ++q) d.ppreq[(size_t)q * cap + i] = GS_EMPTY32;
    for (uint32_t q = 0; q < 4u; ++q) d.pp_clk[(size_t)q * cap + i] = 0u;
  }
}

// Member i (key word k0 in buffer 0) crashes: truth CRASHED in both key buffers.
GS_DEV void gs_crash_keys(const GsDev& d, const GsGlobals& g, uint32_t i, uint32_t k0) {
  gs_key_store(d, g, 0u, i, (k0 & ~3u) | GS_TRUTH_CRASHED);
  gs_key_store(d, g, 1u, i, (d.key[1][i] & ~3u) | GS_TRUTH_CRASHED);
}

// BASELINE config 3: crash every UP member whose Philox draw is below the threshold.
GS_DEV bool gs_crash_row(const GsDev& d, const GsGlobals& g, uint32_t i, uint32_t thr,
                         uint32_t salt) {
  uint32_t k = d.key[0][i];
  if (gs_key_truth(k) != GS_TRUTH_UP) return false;
  GsU4 r = gs_philox(g.seed_lo, g.seed_hi, i, salt, GS_PUR_CRASH, 0u);
  if (r.x >= thr) return false;
  gs_crash_keys(d, g, i, k);
  return true;
}

// ---- paused members (gsim_pause_*, DESIGN.md §3.6) ---------------------------------------------
// pause_until[i] = the tick member i resumes at, 0 = not paused.  While paused its truth is CRASHED: every
// kernel treats it as it treats a crashed process.

// gsim_pause_fraction's draw for member i: its own purpose word, so the selection is independent of the
// crash and impairment selections for the same salt.
GS_DEV bool gs_pause_pick(const GsGlobals& g, uint32_t i, uint32_t thr, uint32_t salt) {
  return gs_philox(g.seed_lo, g.seed_hi, i, salt, GS_PUR_PAUSE, 0u).x < thr;
}

// Pause member i until tick `until` if it runs and is not leaving (a leaving member's scheduled shutdown
// only fires for a running process).  A paused member is not running, so it is never paused twice.
GS_DEV bool gs_pause_row(const GsDev& d, const GsGlobals& g, uint32_t* pause_until, uint32_t i, uint32_t until) {
  const uint32_t k0 = d.key[0][i];
  if (gs_key_truth(k0) != GS_TRUTH_UP || (d.meta[i] & GS_META_LEAVING)) return false;
  gs_key_store(d, g, 0u, i, (k0 & ~3u) | GS_TRUTH_CRASHED);
  gs_key_store(d, g, 1u, i, (d.key[1][i] & ~3u) | GS_TRUTH_CRASHED);
  pause_until[i] = until;
  return true;
}

// Resume codes of gs_resume_row (0 = nothing to do).
enum { GS_RESUMED_ALIVE = 1, GS_RESUMED_SUSPECT = 2, GS_RESUMED_DEAD = 3, GS_PAUSE_FORGOTTEN = 4 };

// Tick t, before it runs (resume = true): member i resumes if its pause ends now.  The process carries on
// with the state it had: truth goes back to UP in both key buffers and nothing else of the member's state
// changes, except that a probe in flight is abandoned (stage IDLE, no missed nacks) and its ticker fires next
// at the first tick >= t on its phase (a `due` off the phase would never fire, gs_tile_probe_gate).  A wake
// in the slot tick t reads steps the row at once: section B refutes a Suspect or Dead record, and a member
// with broadcasts queued has its wake again (the GS_WAKE_BIT invariant).  Returns the rank it comes back to.
// A paused member that is gone (reaped, pruned, or listed Left by force_leave) never resumes: its pause is
// forgotten (GS_PAUSE_FORGOTTEN), at its resume tick or by a sweep with resume = false.
GS_DEV uint32_t gs_resume_row(const GsDev& d, const GsGlobals& g, uint32_t* pause_until, uint32_t i, uint32_t t,
                              bool resume) {
  const uint32_t until = pause_until[i];
  if (until == 0u) return 0u;
  const uint32_t k = d.key[t & 1u][i];
  if (gs_key_truth(k) == GS_TRUTH_CRASHED && gs_key_rank(k) != GS_RANK_LEFT) {
    if (!resume || until != t) return 0u;
    gs_key_store(d, g, 0u, i, (d.key[0][i] & ~3u) | GS_TRUTH_UP);
    gs_key_store(d, g, 1u, i, (d.key[1][i] & ~3u) | GS_TRUTH_UP);
    d.meta[i] = gs_meta_set_nmiss(gs_meta_set_stage(d.meta[i], GS_STAGE_IDLE), 0u);
    const uint32_t pp = gs_probe_phase(g.rot_p, i / g.phase_group, g.P);
    d.due[i] = t + (pp + g.P - t % g.P) % g.P;
    d.inbox[t & g.ring_mask][i] |= GS_WAKE_BIT;
    pause_until[i] = 0u;
    return GS_RESUMED_ALIVE + gs_key_rank(k);
  }
  pause_until[i] = 0u;
  return GS_PAUSE_FORGOTTEN;
}

// ---- fault domains (gsim_domain_*, DESIGN.md §3.5 "Fault domains") -----------------------------------
// dom = the domain column; bits = a bitmap of the listed domains (domain x is bit x & 31 of word x >> 5,
// n_words words).  The one selection rule of gsim_domain_impair, _crash and _pause: member i's domain is listed.
GS_HD bool gs_domain_listed(const uint32_t* dom, const uint32_t* bits, uint32_t n_words, uint32_t i) {
  const uint32_t x = dom[i];
  return x != 0u && (x >> 5) < n_words && ((bits[x >> 5] >> (x & 31u)) & 1u) != 0u;
}

// One listed member of a domain operation, as the per-member call would treat it.  Returns bit 0 = counted in
// counts[0] (IMPAIR: written; CRASH: crashed; PAUSE: paused), bit 1 = counted in counts[1] (IMPAIR: it was
// impaired before; CRASH: a paused member whose resume was cancelled).  COUNT writes nothing and counts it.
GS_DEV uint32_t gs_domain_op_row(const GsDev& d, const GsGlobals& g, const GsDomainOp& a, uint32_t i) {
  if (a.op == GS_DOMAIN_OP_COUNT) return 1u;
  if (a.op == GS_DOMAIN_OP_IMPAIR) return gs_impair_write(a.imp, i, a.v) ? 3u : 1u;  // gsim_impair_dir_many
  if (a.op == GS_DOMAIN_OP_PAUSE) return gs_pause_row(d, g, a.pause_until, i, a.until) ? 1u : 0u;
  const uint32_t k = d.key[0][i];  // gsim_crash_many: a running member crashes, a paused one crashes for good
  if (gs_key_truth(k) == GS_TRUTH_UP) {
    gs_crash_keys(d, g, i, k);
    return 1u;
  }
  if (gs_key_truth(k) == GS_TRUTH_CRASHED && a.pause_until != nullptr && a.pause_until[i] != 0u) {
    a.pause_until[i] = 0u;
    return 2u;
  }
  return 0u;
}

// Member i's contribution to its domain's stats at tick now, packed as the stats kernel sums them: c[0] =
// members | running << 6 | paused << 12 | impaired << 18 | in_force << 24, c[1] = alive | suspect << 6 | dead
// << 12 | left << 18, c[2] = its awareness when it runs (else 0).  Returns false when it is not counted (truth
// NONE).
GS_HD bool gs_domain_stats_row(const GsDev& d, uint32_t seed_lo, uint32_t seed_hi, const GsDomainCols& c, uint32_t i,
                               uint32_t now, uint32_t out[3]) {
  const uint32_t k = c.key[i];
  if (gs_key_truth(k) == GS_TRUTH_NONE) return false;
  const bool run = gs_key_truth(k) == GS_TRUTH_UP;
  const bool paused = c.pause_until != nullptr && c.pause_until[i] != 0u;
  const GsImpairCols& m = c.imp;
  const bool impaired = (m.loss != nullptr && m.loss[i] != 0u) || (m.recv != nullptr && m.recv[i] != 0u) ||
                        (m.delay != nullptr && m.delay[i] != 0u) || (m.flags != nullptr && m.flags[i] != 0u);
  const bool in_force = impaired && gs_imp_in_force(d, seed_lo, seed_hi, i, now);
  out[0] = 1u | (run ? 1u << 6 : 0u) | (paused ? 1u << 12 : 0u) | (impaired ? 1u << 18 : 0u) |
           (in_force ? 1u << 24 : 0u);
  out[1] = 1u << (6u * gs_key_rank(k));
  out[2] = run ? gs_meta_aw(c.meta[i]) : 0u;
  return true;
}
GS_HD void gs_domain_stats_add(GsDomainStats& s, const uint32_t c[3], uint32_t aw_max) {
  s.members += c[0] & 63u;
  s.running += (c[0] >> 6) & 63u;
  s.paused += (c[0] >> 12) & 63u;
  s.impaired += (c[0] >> 18) & 63u;
  s.in_force += (c[0] >> 24) & 63u;
  s.alive += c[1] & 63u;
  s.suspect += (c[1] >> 6) & 63u;
  s.dead += (c[1] >> 12) & 63u;
  s.left += (c[1] >> 18) & 63u;
  s.awareness_sum += c[2];
  if (aw_max > s.awareness_max) s.awareness_max = aw_max;
}

// [U] serf.handleReap -> reap(failedMembers, ReconnectTimeout) / reap(leftMembers, TombstoneTimeout):
// a member that has been Failed (Left) for longer than the timeout is erased from the member
// list (EventMemberReap).  Row a17 of SURVEY 8a; Consul shortens the timeouts in
// agent/consul/server_test.go:675-677.  Returns bit 0 = reaped, bit 1 = it was an established
// (non-pending) member; the caller logs the event.
GS_DEV uint32_t gs_reap_row(const GsDev& d, const GsGlobals& g, uint32_t i, uint32_t now,
                            uint32_t reconnect_ticks, uint32_t tombstone_ticks) {
  const uint32_t k = d.key[now & 1u][i];
  const uint32_t truth = gs_key_truth(k), rank = gs_key_rank(k);
  if (truth == GS_TRUTH_NONE || truth == GS_TRUTH_UP) return 0u;
  uint32_t limit;
  if (rank == GS_RANK_DEAD) limit = d.reap_after[i] != 0u ? d.reap_after[i] : reconnect_ticks;  // ReconnectTimeoutOverride
  else if (rank == GS_RANK_LEFT) limit = tombstone_ticks;
  else return 0u;
  if (now - d.change_tick[i] <= limit) return 0u;
  gs_key_store(d, g, 0u, i, d.key[0][i] & ~3u);
  gs_key_store(d, g, 1u, i, d.key[1][i] & ~3u);
  return 1u | (gs_key_pending(k) ? 0u : 2u);
}

// Canonical digest of one row: only fields that are semantically live are folded, so
// that stale scratch in cold columns never matters (the oracle folds the same fields).
GS_DEV uint64_t gs_hash_row(const GsDev& d, const GsGlobals& g, uint32_t i, uint32_t now) {
  const uint32_t cur = now & 1u;  // buffer the next tick will read
  const size_t cap = g.cap;
  const uint32_t k = d.key[cur][i];
  const uint32_t truth = gs_key_truth(k);
  if (truth == GS_TRUTH_NONE) return 0ull;
  const uint32_t m = d.meta[i] & ~GS_META_DIRTY;
  const uint32_t rank = gs_key_rank(k);
  const bool up = truth == GS_TRUTH_UP;
  const bool probing = up && gs_meta_stage(m) != GS_STAGE_IDLE;
  uint64_t h = 0x9E3779B97F4A7C15ull;
  h = gs_mix64(h, i);
  h = gs_mix64(h, k);
  h = gs_mix64(h, m);
  h = gs_mix64(h, up ? d.due[i] : 0u);
  h = gs_mix64(h, d.cursor[i]);
  h = gs_mix64(h, d.pass[i]);
  h = gs_mix64(h, probing ? d.probe_tgt[i] : 0u);
  h = gs_mix64(h, probing ? d.probe_inc[i] : 0u);
  h = gs_mix64(h, rank == GS_RANK_SUSPECT ? d.sus_start[i] : 0u);
  for (uint32_t q = 0; q < GS_K1MAX; ++q)
    h = gs_mix64(h, rank == GS_RANK_SUSPECT ? d.sus_from[(size_t)q * cap + i] : 0u);
  h = gs_mix64(h, rank >= GS_RANK_DEAD ? d.change_tick[i] : 0u);
  h = gs_mix64(h, d.ltime_member[i]);
  h = gs_mix64(h, d.ltime_event[i]);
  h = gs_mix64(h, d.event_min[i]);
  const uint32_t heard = d.heard[i] & g.active_mask;
  h = gs_mix64(h, heard);
  h = gs_mix64(h, d.queued[i] & g.active_mask);
  const uint32_t inb = d.inbox[now & g.ring_mask][i];
  h = gs_mix64(h, inb & (g.active_mask | GS_ACC_BIT));
  // latency pools: packets still in flight, by ticks until arrival (slot now-1 was just consumed)
  for (uint32_t s = 1; s < g.ring_mask; ++s)
    h = gs_mix64(h, d.inbox[(now + s) & g.ring_mask][i] & g.active_mask);
  uint32_t hm = heard;
  while (hm) {
#if defined(__CUDA_ARCH__)
    uint32_t r = __ffs(hm) - 1;
#else
    uint32_t r = (uint32_t)__builtin_ctz(hm);
#endif
    hm &= hm - 1;
    h = gs_mix64(h, (r << 8) | d.tx[GS_TX(r, cap, i)]);
  }
  if (d.coord != nullptr) {  // the member's current coordinate, bit for bit, and its adjustment window
    const uint32_t slot = d.ctag[cap + i] > d.ctag[i] ? 1u : 0u;
    const double* c = d.coord + ((size_t)slot * GS_COORD_WORDS) * cap + i;
    for (uint32_t x = 0; x < GS_COORD_WORDS; ++x) {
      uint64_t bits;
      memcpy(&bits, &c[(size_t)x * cap], 8);
      h = gs_mix64(h, bits);
    }
    h = gs_mix64(h, d.adj_idx[i]);
  }
  if (inb & GS_ACC_BIT) {
    const uint64_t* acc = d.acc + (size_t)cur * GS_K1MAX * cap;
    for (uint32_t s = 0; s < GS_K1MAX; ++s) h = gs_mix64(h, acc[(size_t)s * cap + i]);
    if (g.pp_interval != 0u) {  // push-pull requests and partner clocks waiting in the mailbox
      const uint32_t* req = d.ppreq + (size_t)cur * GS_PPK * cap;
      for (uint32_t s = 0; s < GS_PPK; ++s) h = gs_mix64(h, req[(size_t)s * cap + i]);
      const uint32_t* clk = d.pp_clk + (size_t)cur * 2u * cap;
      h = gs_mix64(h, clk[i]);
      h = gs_mix64(h, clk[cap + i]);
    }
    if (d.pig_req != nullptr) {  // probe-path answers this member owes (GSIM_FLAG_PROBE_PIGGYBACK)
      const uint32_t* req = d.pig_req + (size_t)cur * GS_PIGK * cap;
      for (uint32_t s = 0; s < GS_PIGK; ++s) h = gs_mix64(h, req[(size_t)s * cap + i]);
    }
  }
  return h;
}

