// gs_backend.h — the narrow device interface the host side of libgsim drives.
// libgsim.so links exactly one implementation: the CUDA backend (gs_cuda.cu).  A second
// implementation exists only under tests/hostemu/ (the same row function compiled by g++
// and looped sequentially) so kernel logic can be debugged in a GPU-less container; it is
// test infrastructure and is never linked into or loaded by the product library.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <stdlib.h>

#include <vector>

#include "gs_agent.h"
#include "gs_core.h"

struct GsRecount {
  uint32_t heard_cnt[GS_MAX_RUMORS];
  uint32_t queued_cnt[GS_MAX_RUMORS];
  uint32_t truth_cnt[4];
  uint32_t rank_cnt[4];
  uint32_t crashed_alive;
  uint32_t isolated_up;  // running members that have not joined the established set
  uint32_t pending;           // members not yet folded into the established set (known through their alive rumor only)
  uint32_t unreachable_live;  // members whose process is gone (crashed / shut down) but whom the cluster
                              // still lists as alive or suspect: the targets an unanswered probe can hit
};

// What GsBackend::run_tick_stretch did: read back in one piece.
struct GsStretch {
  uint32_t ran;          // ticks run
  uint32_t launches;     // tick launches, including those that found the stretch over and ran nothing
  uint32_t last_active;  // GS_Q_LAST_ACTIVE at the end
  uint32_t quiet;        // 1: stopped at a quiet tick, and the two fields below are set
  uint32_t horizon;      // quiet_probe's horizon at t0 + ran
  GsRecount counts;      // ... and its counts (when asked for)
};

// ---- device write batches -------------------------------------------------------------------
// The host side of an operation (a new member, a join, a retired rumor) is a few dozen small writes,
// several of them read-modify-writes of a word the host does not keep.  They are queued as an ordered
// list and applied on the device in that order by one thread, after everything the pool enqueued
// before and before everything it enqueues after: no host round trip per word.
enum : uint32_t {
  GS_WR_STORE32 = 0,  // *a = v
  GS_WR_STORE8 = 1,   // byte *a = v
  GS_WR_OR32 = 2,     // *a |= v
  GS_WR_AND32 = 3,    // *a &= v
  GS_WR_KST = 4,      // status byte a (gs_kst_code): nibble v (0 = low, key[0]; 1 = high, key[1]) := code of key word b
  GS_WR_HEARD = 5,    // heard_cnt[r] at a += v; if that makes it w (up_count) and conv_tick[r] at b is empty, it := x (now)
};
struct GsWriteOp {
  uint64_t a, b;  // device addresses
  uint32_t op, v, w, x;
};
#define GS_WB_MAX 120u  // ops per launch: the batch travels as one kernel parameter (< 4 KB)
struct GsWriteBatch {
  uint32_t n, pad;
  GsWriteOp op[GS_WB_MAX];
};

GS_HD void gs_apply_write(const GsWriteOp& o) {
  uint32_t* a = reinterpret_cast<uint32_t*>(o.a);
  switch (o.op) {
    case GS_WR_STORE32: *a = o.v; break;
    case GS_WR_STORE8: *reinterpret_cast<uint8_t*>(o.a) = (uint8_t)o.v; break;
    case GS_WR_OR32: *a |= o.v; break;
    case GS_WR_AND32: *a &= o.v; break;
    case GS_WR_KST: {
      uint8_t* s = reinterpret_cast<uint8_t*>(o.a);
      const uint32_t code = gs_kst_code(*reinterpret_cast<const uint32_t*>(o.b));
      *s = (uint8_t)(o.v ? ((*s & 0x0Fu) | (code << 4)) : ((*s & 0xF0u) | code));
      break;
    }
    case GS_WR_HEARD: {
      const uint32_t c = *a + o.v;
      *a = c;
      uint32_t* conv = reinterpret_cast<uint32_t*>(o.b);
      if (c == o.w && *conv == GS_EMPTY32) *conv = o.x;
      break;
    }
  }
}

class GsBackend {
 public:
  virtual ~GsBackend() {}
  virtual const char* name() const = 0;
  virtual void* alloc(size_t bytes) = 0;  // returns nullptr on failure
  virtual void release(void* p) = 0;
  virtual bool h2d(void* dst, const void* src, size_t bytes) = 0;
  virtual bool d2h(void* dst, const void* src, size_t bytes) = 0;
  // A few KB at most host -> device, ordered on the pool's stream but NOT waited for: the source may be
  // reused as soon as the call returns (the driver stages small pageable copies before returning),
  // everything the pool launches or reads later comes after it.  Used for the globals upload.
  virtual bool h2d_word(void* dst, const void* src, size_t bytes) { return h2d(dst, src, bytes); }
  // The ops of `b` in order, on the pool's stream (see GsWriteBatch).  The CUDA backend applies them in
  // one launch that is not waited for and ends in a system-scope fence, so peers of a sharded pool see
  // every op once a barrier that comes after it on this stream has let them go on.  Defined here
  // through the copy primitives every backend has, which is what the host emulation runs.
  virtual bool write_batch(const GsWriteBatch& b) {
    for (uint32_t k = 0; k < b.n; ++k) {
      const GsWriteOp& o = b.op[k];
      const size_t na = (o.op == GS_WR_STORE8 || o.op == GS_WR_KST) ? 1u : 4u;
      const bool use_b = o.op == GS_WR_KST || o.op == GS_WR_HEARD;
      uint32_t a = 0u, bw = 0u;  // host copies of the words the op touches
      if (!d2h(&a, reinterpret_cast<const void*>(o.a), na)) return false;
      if (use_b && !d2h(&bw, reinterpret_cast<const void*>(o.b), 4)) return false;
      const uint32_t b0 = bw;
      GsWriteOp h = o;
      h.a = (uint64_t)(uintptr_t)&a;
      h.b = (uint64_t)(uintptr_t)&bw;
      gs_apply_write(h);
      if (!h2d(reinterpret_cast<void*>(o.a), &a, na)) return false;
      if (bw != b0 && !h2d(reinterpret_cast<void*>(o.b), &bw, 4)) return false;
    }
    return true;
  }
  // Bulk host -> device, enqueued only: the caller keeps `src` alive and calls sync() before it returns
  // (gsim_restore streams its planes back to back and waits once).
  // host staging memory for bulk copies (page-locked where that makes the copy a plain DMA)
  virtual void* host_alloc(size_t bytes) { return malloc(bytes); }
  virtual void host_free(void* q) { free(q); }
  virtual bool h2d_async(void* dst, const void* src, size_t bytes) { return h2d(dst, src, bytes); }
  // The per-member words the host side of a state exchange needs, in one round trip:
  // out = {key[0], key[1], meta, heard, queued, ltime_member, ltime_event, event_min}
  virtual bool row_read(const GsDev& d, uint32_t i, uint32_t out[8]) = 0;
  // ... for `n` members, out[8 * x ..] = the words of ids[x] (the CUDA backend: one round trip per 64 rows)
  virtual bool rows_read(const GsDev& d, const uint32_t* ids, uint32_t n, uint32_t* out) {
    for (uint32_t x = 0; x < n; ++x)
      if (!row_read(d, ids[x], out + 8 * (size_t)x)) return false;
    return true;
  }
  virtual bool fill32(uint32_t* dst, uint32_t value, size_t count) = 0;
  virtual bool fill8(uint8_t* dst, uint8_t value, size_t count) = 0;
  // rows [first, first+count): converged members, inc=1, clocks=1, phases from Philox (not waited for)
  virtual bool init_rows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t first,
                         uint32_t count, uint32_t now) = 0;
  // advance `nticks` ticks starting at tick t0 (tick_base on the device == t0 on entry and
  // t0+nticks on exit).  kernel_ms accumulates CUDA-event time of the tick launches.
  virtual bool run_ticks(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t t0,
                         uint32_t nticks, bool use_graph, double* kernel_ms, uint64_t* launches,
                         const GsXbar* xbar = nullptr) = 0;
  // run_ticks, then *last_active = this rank's GS_Q_LAST_ACTIVE.  The CUDA backend reads it back with
  // the launches' own synchronisation; by default it is a readback of its own.
  virtual bool run_ticks_read(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t t0, uint32_t nticks,
                              bool use_graph, double* kernel_ms, uint64_t* launches, const GsXbar* xbar,
                              uint32_t* last_active) {
    return run_ticks(d, g_dev, g, t0, nticks, use_graph, kernel_ms, launches, xbar) &&
           d2h(last_active, d.qstate[g.rank] + GS_Q_LAST_ACTIVE, 4);
  }
  // Single ticks until the pool is quiet (DESIGN.md §4.2), single-GPU pools: tick t0 + k runs unless
  // t0 + k >= t0 + nticks or t0 + k >= max(GS_Q_LAST_ACTIVE, floor) + depth (depth = g.ring_mask + 1: every
  // arrival slot has been scanned empty once since the last mail).  When it stopped at such a quiet tick,
  // out->horizon and (counts) out->counts are quiet_probe's at that tick.  The CUDA backend decides on the
  // device and waits once; by default it is run_ticks_read one tick at a time, then quiet_probe.
  virtual bool run_tick_stretch(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t t0,
                                uint32_t nticks, uint32_t floor, bool counts, double* kernel_ms, GsStretch* out) {
    const uint32_t depth = g.ring_mask + 1u;
    *out = GsStretch();
    if (!d2h(&out->last_active, d.qstate[0] + GS_Q_LAST_ACTIVE, 4)) return false;
    for (;;) {
      const uint32_t la = out->last_active > floor ? out->last_active : floor;
      if (t0 + out->ran >= la + depth) {
        out->quiet = 1u;
        break;
      }
      if (out->ran == nticks) break;
      uint64_t nl = 0;
      if (!run_ticks_read(d, g_dev, g, t0 + out->ran, 1u, true, kernel_ms, &nl, nullptr, &out->last_active))
        return false;
      out->ran++;
      out->launches++;
    }
    return !out->quiet || quiet_probe(d, g_dev, g, t0 + out->ran, &out->horizon, counts ? &out->counts : nullptr);
  }
  // Quiet windows (DESIGN.md §4.2): advance up to `nticks` ticks starting at t0 as a chain of launches
  // of <= ProbeInterval ticks each, on a pool whose mailboxes are known to be empty.  The chain stops at
  // the horizon (GS_Q_HORIZON); *ticks_done = how far it got (tick_base == t0 + *ticks_done on exit).
  // `per_launch` = ticks one launch may cover: ProbeInterval in general; more when the caller knows that
  // no probe can go unanswered (every listed member runs, no loss, no slow link), so the horizon cannot move.
  virtual bool run_windows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t t0, uint32_t nticks,
                           uint32_t per_launch, bool use_graph, double* kernel_ms, uint64_t* launches,
                           uint32_t* ticks_done, const GsXbar* xbar, bool pristine) = 0;
  // lowers GS_Q_HORIZON (every rank's copy) to the earliest accusation the probes in flight of rows
  // [first, first+count) can produce
  virtual bool quiet_scan(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now, uint32_t first,
                          uint32_t count) = 0;
  // Single-GPU pools: GS_Q_HORIZON := GS_NEVER, quiet_scan over every member, *horizon = the result, and
  // (counts != nullptr) recount over every member into *counts.  The CUDA backend makes it one submission
  // with one readback; by default it is the primitives one after the other.
  virtual bool quiet_probe(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now,
                           uint32_t* horizon, GsRecount* counts) {
    const uint32_t never = GS_NEVER;
    return h2d(d.qstate[0] + GS_Q_HORIZON, &never, 4) && quiet_scan(d, g_dev, g, now, 0u, g.n) &&
           d2h(horizon, d.qstate[0] + GS_Q_HORIZON, 4) && (!counts || recount(d, g_dev, g, now, 0u, g.n, counts));
  }
  // ---- sharded (multi-GPU) pools, see gs_vmm.h; unsupported by default ------------------------
  virtual bool shard_begin(uint32_t, uint32_t) { return false; }
  virtual size_t shard_granularity() { return 0; }
  virtual void* shard_alloc(size_t /*slice_bytes*/, size_t /*planes*/) { return nullptr; }
  virtual bool shard_commit(const int** /*fds*/, size_t* /*n*/) { return false; }
  virtual bool shard_attach(uint32_t /*peer*/, const int* /*fds*/, size_t /*n*/) { return false; }
  virtual bool xbar_host(const GsXbar&) { return false; }  // arrive, wait for every rank, sync
  virtual bool crash_fraction(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g,
                              uint32_t thr, uint32_t salt, uint32_t now, uint32_t* n_crashed) = 0;
  // gs_impair_row over every member, writing setting v into the impairment columns c (allocated by the
  // caller, who may not have published them in `d` yet; c.recv and c.flags may be null); counts[0] =
  // members selected, counts[1] = how many of them were impaired before.  Defined here through the copy
  // primitives every backend has, which is what the host emulation runs; the CUDA backend replaces it with
  // gs_impair_kernel.
  virtual bool impair_dir_fraction(const GsDev& d, const GsGlobals* /*g_dev*/, const GsGlobals& g,
                                   const GsImpairCols& c, uint32_t thr, uint32_t salt, const GsImpairVal& v,
                                   uint32_t counts[2]) {
    counts[0] = counts[1] = 0u;
    if (!g.n) return true;
    std::vector<uint32_t> key(g.n), lc(g.n), rc(c.recv ? g.n : 0u);
    std::vector<uint8_t> dc(g.n), fc(c.flags ? g.n : 0u);
    if (!d2h(key.data(), d.key[0], (size_t)g.n * 4) || !d2h(lc.data(), c.loss, (size_t)g.n * 4) ||
        !d2h(dc.data(), c.delay, g.n) || (c.recv && !d2h(rc.data(), c.recv, (size_t)g.n * 4)) ||
        (c.flags && !d2h(fc.data(), c.flags, g.n)))
      return false;
    const GsImpairCols hc = {lc.data(), c.recv ? rc.data() : nullptr, dc.data(), c.flags ? fc.data() : nullptr};
    for (uint32_t i = 0; i < g.n; ++i) {
      const uint32_t r = gs_impair_row(key[i], hc, g.seed_lo, g.seed_hi, i, thr, salt, v);
      counts[0] += r & 1u;
      counts[1] += (r >> 1) & 1u;
    }
    return h2d(c.loss, lc.data(), (size_t)g.n * 4) && h2d(c.delay, dc.data(), g.n) &&
           (!c.recv || h2d(c.recv, rc.data(), (size_t)g.n * 4)) && (!c.flags || h2d(c.flags, fc.data(), g.n));
  }
  // The symmetric case (loss, loss, delay, no flags) on the two columns every impaired pool has.
  virtual bool impair_fraction(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t* loss_col,
                               uint8_t* delay_col, uint32_t thr, uint32_t salt, uint32_t loss, uint32_t delay,
                               uint32_t counts[2]) {
    const GsImpairCols c = {loss_col, nullptr, delay_col, nullptr};
    const GsImpairVal v = {loss, loss, delay, 0u};
    return impair_dir_fraction(d, g_dev, g, c, thr, salt, v, counts);
  }
  // Intermittent impairment (gs_core.h; col is the caller's schedule column).  flap_fraction: gs_flap_row(w)
  // over every member, counts as for impair_dir_fraction; flap_stats: out[0] = members with a schedule, out[1]
  // = those of them in a bad epoch at tick now.  Defined here through the copy primitives every backend has,
  // which is what the host emulation runs; the CUDA backend replaces them with gs_flap_kernel and
  // gs_flap_stats_kernel.
  virtual bool flap_fraction(const GsDev& d, const GsGlobals* /*g_dev*/, const GsGlobals& g, uint32_t* col,
                             uint32_t thr, uint32_t salt, uint32_t w, uint32_t counts[2]) {
    counts[0] = counts[1] = 0u;
    if (!g.n) return true;
    std::vector<uint32_t> key(g.n), fc(g.n);
    if (!d2h(key.data(), d.key[0], (size_t)g.n * 4) || !d2h(fc.data(), col, (size_t)g.n * 4)) return false;
    for (uint32_t i = 0; i < g.n; ++i) {
      const uint32_t r = gs_flap_row(key[i], fc.data(), g.seed_lo, g.seed_hi, i, thr, salt, w);
      counts[0] += r & 1u;
      counts[1] += (r >> 1) & 1u;
    }
    return h2d(col, fc.data(), (size_t)g.n * 4);
  }
  virtual bool flap_stats(const GsGlobals& g, const uint32_t* col, uint32_t now, uint64_t out[2]) {
    out[0] = out[1] = 0u;
    if (!g.n) return true;
    std::vector<uint32_t> fc(g.n);
    if (!d2h(fc.data(), col, (size_t)g.n * 4)) return false;
    for (uint32_t i = 0; i < g.n; ++i) {
      if (fc[i] == 0u) continue;
      out[0]++;
      out[1] += gs_flap_bad(g.seed_lo, g.seed_hi, i, fc[i], now) ? 1u : 0u;
    }
    return true;
  }
  // Paused members (gs_aux.h; pause_until is the caller's column).  pause_rows: gs_pause_row(until) over the
  // `n` distinct members ids[] when ids != nullptr, otherwise over every member whose gs_pause_pick(thr, salt)
  // draw selects it; *n_paused = members paused.  resume_rows: gs_resume_row(t, resume) over every member,
  // logging a pool-wide EventMemberJoin at t for each member that comes back from Dead when `log_events`;
  // counts[0..2] = resumed Alive / Suspect / Dead, counts[3] = pauses forgotten.  Both are defined in
  // gs_api.cpp through the copy primitives every backend has, which is what the host emulation runs; the CUDA
  // backend replaces them with one kernel each.
  virtual bool pause_rows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t* pause_until,
                          const uint32_t* ids, uint32_t n, uint32_t thr, uint32_t salt, uint32_t until,
                          uint32_t* n_paused);
  virtual bool resume_rows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t* pause_until,
                           uint32_t t, bool resume, bool log_events, uint32_t counts[4]);
  // Fault domains (gs_aux.h; dom is the caller's domain column).  domain_range: dom[first + x] = first_domain +
  // x / per_domain for x < count.  domain_rows: gs_domain_op_row(a) over every member gs_domain_listed selects,
  // `bits` a host bitmap of n_words words; counts[0] and counts[1] sum its two result bits.  domain_stats: out[x]
  // (host memory) = the stats of domain first_domain + x at tick now, gs_domain_stats_row summed over its
  // members.  Defined in gs_api.cpp through the copy primitives every backend has, which is what the host
  // emulation runs; the CUDA backend replaces each with one sm_90a kernel.
  virtual bool domain_range(uint32_t* dom, uint32_t first, uint32_t count, uint32_t per_domain, uint32_t first_domain);
  virtual bool domain_rows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, const uint32_t* dom,
                           const uint32_t* bits, uint32_t n_words, const GsDomainOp& a, uint32_t counts[2]);
  virtual bool domain_stats(const GsDev& d, const GsGlobals& g, const GsDomainCols& c, uint32_t now,
                            uint32_t first_domain, uint32_t count, GsDomainStats* out);
  // ---- network-coordinate queries (gs_query.h, DESIGN.md §3.4 "Queries"; single-GPU pools) ----------
  // Read-only.  Every pointer is device memory and nothing is waited for: the caller reads the result
  // back once.  Defined in gs_api.cpp through the copy primitives every backend has, which is what the
  // host emulation runs; the CUDA backend replaces each with sm_90a kernels.
  // rows[11 x ..] = the published coordinate (gs_coord_pick) of member first + x
  virtual bool coord_rows(const GsDev& d, const GsGlobals& g, uint32_t first, uint32_t count, double* rows);
  // est[k] = the distance between a[k] and b[k]; tru[k] (tru may be null) = gs_model_rtt(a[k], b[k]) at tick now
  virtual bool coord_pairs(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now, const uint32_t* a,
                           const uint32_t* b, uint32_t n, double* est, double* tru);
  // key[x] = gs_dist_key of the distance from `from` to ids[x] (ids null: to member x), val[x] = that id; or
  // (router) gs_router_entry at tick now.  ids may be val.
  virtual bool coord_dist_from(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now, uint32_t from,
                               const uint32_t* ids, uint32_t n, bool router, uint64_t* key, uint32_t* val);
  // stable sort of the n pairs (key[x], val[x]) by key, or (n_dcs != 0) by (gs_dc_digit(val), key)
  virtual bool sort_pairs(const GsGlobals& g, uint64_t* key, uint32_t* val, uint32_t n, uint32_t n_dcs);
  // over pairs sorted by (datacenter, key): cnt[c] = entries of datacenter c < n_dcs, med[c] = the distance of
  // its entry cnt[c] / 2 (+inf when it has none)
  virtual bool dc_medians(const GsGlobals& g, const uint64_t* key, const uint32_t* val, uint32_t n, uint32_t n_dcs,
                          double* med, uint32_t* cnt);
  // gsim_coordinate_error: draws [0, n_draws) at tick now into key (gs_dist_key of the relative error, all ones
  // when skipped) and val (the draw), sorted by sort_pairs; then out = {kept, mean, p50, p90, p99, max}, the
  // mean = (sum over chunks of GS_ERR_CHUNK draws, in chunk order, of the chunk's errors summed in draw order) /
  // kept.  `part` has room for 2 ceil(n_draws / GS_ERR_CHUNK) doubles.
  virtual bool coord_error(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now, uint32_t n_draws,
                           uint32_t salt, uint64_t* key, uint32_t* val, double* part, double* out);
  // ---- per-agent observation (gs_agent.h, DESIGN.md §3.8) ------------------------------------------
  // Read-only; `key` is the key buffer of the current tick and `out` host memory.  Defined in gs_api.cpp
  // through the copy primitives every backend has, which is what the host emulation runs; the CUDA backend
  // replaces each with sm_90a kernels in one submission and one wait.
  // out[x] = gs_agent_stats_row of member first + x (est[] counted over every member first)
  virtual bool agent_stats(const GsDev& d, const GsGlobals& g, const uint32_t* key, const GsPendingAlive& pa,
                           uint32_t first, uint32_t count, GsAgentStats* out);
  // out[b] = members in bin b of gs_health_bin, over every member
  virtual bool health_histogram(const GsDev& d, const GsGlobals& g, const uint32_t* key, const GsImpairCols& imp,
                                uint64_t out[GS_HIST_BINS]);
  // counts over members [first, first + count) (a rank of a sharded pool counts its own rows)
  virtual bool recount(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now, uint32_t first,
                       uint32_t count, GsRecount* out) = 0;
  virtual bool state_hash(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now,
                          uint64_t out[4]) = 0;
  // serf's reaper (gs_aux.h gs_reap_row) over every row; counts[0] = members erased, counts[1] =
  // how many of them were established; logs EventMemberReap when `log_events`
  virtual bool reap_rows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now,
                         uint32_t reconnect_ticks, uint32_t tombstone_ticks, bool log_events,
                         uint32_t counts[2]) = 0;
  // clear rumor bits outside `keep` in the heard / queued / mailbox columns (slot retirement; not waited for)
  virtual bool and_columns(const GsDev& d, const GsGlobals& g, uint32_t keep, uint32_t first, uint32_t count) = 0;
  virtual bool sync() = 0;
  virtual const char* last_error() const = 0;
  virtual uint64_t total_launches() const = 0;
};

// Implemented by gs_cuda.cu (product) — returns nullptr and fills err when no usable
// sm_90 device exists.  There is deliberately no CPU implementation in libgsim.
GsBackend* gs_make_cuda_backend(int device, char* err, size_t err_cap);

// ---- state digest shared by every implementation of state_hash -----------------
GS_HD uint64_t gs_mix64(uint64_t h, uint64_t w) {
  h = (h ^ w) * 0xff51afd7ed558ccdull;
  h ^= h >> 32;
  return h;
}
GS_HD void gs_hash_lanes(uint64_t h, uint64_t lanes[4]) {
  lanes[0] = h;
  lanes[1] = gs_mix64(h, 1);
  lanes[2] = gs_mix64(h, 2);
  lanes[3] = gs_mix64(h, 3);
}
