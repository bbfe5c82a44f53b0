// gs_agent.h — read-only per-agent observation (DESIGN.md §3.8): the bodies of gsim_agent_stats_read and
// gsim_health_histogram, shared by the host defaults of GsBackend (gs_api.cpp) and the sm_90a kernels
// (gs_cuda.cu).  Nothing here writes pool state.
//
// [U] serf/serf.go Stats, memberlist/memberlist.go GetHealthScore, memberlist/queue.go NumQueued.
#pragma once
#include "gs_core.h"

GS_HD uint32_t gs_popc(uint32_t x) {
#if defined(__CUDA_ARCH__)
  return (uint32_t)__popc(x);
#else
  return (uint32_t)__builtin_popcount(x);
#endif
}

// One agent's serf Stats(), field for field gsim_agent_stats.
struct GsAgentStats {
  uint32_t members, failed, left;
  uint32_t health_score;
  uint32_t member_time, event_time, query_time;
  uint32_t intent_queue, event_queue, query_queue;
  uint32_t memberlist_queue;
  uint32_t running;
};

// The subjects of the tracked alive rumors, each with the first such slot (the one gsim_members looks
// up): a pending member c is in observer i's list iff bit slot[x] of heard[i] is set.
struct GsPendingAlive {
  uint32_t n;
  uint32_t slot[GS_MAX_RUMORS];
  uint32_t subject[GS_MAX_RUMORS];
};

GS_HD void gs_pending_alive(const GsGlobals& g, GsPendingAlive& pa) {
  pa.n = 0;
  for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r) {
    if (!((g.active_mask >> r) & 1u) || g.rumors[r].kind != GS_RUMOR_ALIVE) continue;
    bool seen = false;
    for (uint32_t x = 0; x < pa.n; ++x) seen = seen || pa.subject[x] == g.rumors[r].subject;
    if (seen) continue;
    pa.slot[pa.n] = r;
    pa.subject[pa.n] = g.rumors[r].subject;
    pa.n++;
  }
}

// The columns the stats read (device pointers in the kernels, host copies in the default), all indexed by
// member id.  key = the key buffer of the current tick; row_ptr / col_idx null on complete-graph pools.
struct GsAgentCols {
  const uint32_t* key;
  const uint32_t* meta;
  const uint32_t* heard;
  const uint32_t* queued;
  const uint32_t* ltime_member;
  const uint32_t* ltime_event;
  const uint32_t* row_ptr;
  const uint32_t* col_idx;
};

// Member c as everybody outside the pending rule sees it: listed (truth not NONE) and established.
// Returns its rank + 1, 0 when it is not such a member.
GS_HD uint32_t gs_established_rank1(uint32_t kc) {
  return gs_key_truth(kc) != GS_TRUTH_NONE && !gs_key_pending(kc) ? gs_key_rank(kc) + 1u : 0u;
}

// Member c != i as observer i lists it in Members() (gs_api.cpp members_locked): rank + 1, or 0 when hidden.
GS_HD uint32_t gs_agent_sees(const GsAgentCols& c, const GsPendingAlive& pa, uint32_t i, uint32_t heard_i,
                             uint32_t meta_i, uint32_t m) {
  const uint32_t km = c.key[m];
  if (gs_key_truth(km) == GS_TRUTH_NONE) return 0u;
  if (!gs_key_pending(km)) return (meta_i & GS_META_ISOLATED) ? 0u : gs_key_rank(km) + 1u;
  for (uint32_t x = 0; x < pa.n; ++x)
    if (pa.subject[x] == m) return ((heard_i >> pa.slot[x]) & 1u) ? gs_key_rank(km) + 1u : 0u;
  return 0u;
}

// Stats of agent i.  est[r] = established members of rank r over the whole pool (gs_established_rank1),
// unused on a CSR pool, where the list is the agent plus its row (each member once).
GS_HD GsAgentStats gs_agent_stats_row(const GsAgentCols& c, const uint32_t class_mask[3], const uint32_t est[4],
                                      const GsPendingAlive& pa, uint32_t i) {
  const uint32_t ki = c.key[i], meta = c.meta[i], heard = c.heard[i], queued = c.queued[i];
  uint32_t cnt[4] = {0u, 0u, 0u, 0u};
  if (gs_key_truth(ki) != GS_TRUTH_NONE) cnt[gs_key_rank(ki)]++;
  if (c.row_ptr != nullptr) {
    const uint32_t e0 = c.row_ptr[i], e1 = c.row_ptr[i + 1];
    for (uint32_t e = e0; e < e1; ++e) {
      const uint32_t m = c.col_idx[e];
      if (m == i) continue;
      bool dup = false;
      for (uint32_t f = e0; f < e && !dup; ++f) dup = c.col_idx[f] == m;
      if (dup) continue;
      const uint32_t r1 = gs_agent_sees(c, pa, i, heard, meta, m);
      if (r1) cnt[r1 - 1u]++;
    }
  } else {
    if (!(meta & GS_META_ISOLATED)) {
      const uint32_t self = gs_established_rank1(ki);
      for (uint32_t r = 0; r < 4u; ++r) cnt[r] += est[r] - (self == r + 1u ? 1u : 0u);
    }
    for (uint32_t x = 0; x < pa.n; ++x) {
      const uint32_t m = pa.subject[x];
      if (m == i || !gs_key_pending(c.key[m])) continue;  // established: counted in est
      const uint32_t r1 = gs_agent_sees(c, pa, i, heard, meta, m);
      if (r1) cnt[r1 - 1u]++;
    }
  }
  GsAgentStats s;
  s.members = cnt[0] + cnt[1] + cnt[2] + cnt[3];
  s.failed = cnt[GS_RANK_DEAD];
  s.left = cnt[GS_RANK_LEFT];
  s.health_score = gs_meta_aw(meta);
  s.member_time = c.ltime_member[i];
  s.event_time = c.ltime_event[i];
  s.query_time = 1u;  // queries are not simulated: the clock member_add started stays at 1
  s.intent_queue = gs_popc(queued & class_mask[1]);
  s.event_queue = gs_popc(queued & class_mask[2]);
  s.query_queue = 0u;
  s.memberlist_queue = gs_popc(queued & class_mask[0]);
  s.running = gs_key_truth(ki) == GS_TRUTH_UP ? 1u : 0u;
  return s;
}

// Histogram bin of member i: impaired * 8 + awareness for a running member, GS_HIST_NONE otherwise.
// imp = the impairment columns of the pool (any of them may be null: not allocated, zero for everybody).
#define GS_HIST_BINS 16u
#define GS_HIST_NONE GS_HIST_BINS
GS_HD uint32_t gs_health_bin(uint32_t key, uint32_t meta, const GsImpairCols& imp, uint32_t i) {
  if (gs_key_truth(key) != GS_TRUTH_UP) return GS_HIST_NONE;
  const bool impaired = (imp.loss != nullptr && imp.loss[i] != 0u) || (imp.recv != nullptr && imp.recv[i] != 0u) ||
                        (imp.delay != nullptr && imp.delay[i] != 0u) || (imp.flags != nullptr && imp.flags[i] != 0u);
  return (impaired ? 8u : 0u) + gs_meta_aw(meta);
}
