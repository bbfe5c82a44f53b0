// gs_api.cpp — host side of libgsim: the C ABI declared in include/gsim.h.
//
// Everything here is control plane: configuration, the N-dependent scalar tables
// (SURVEY §8a row a11, evaluated in double exactly like [U] memberlist/util.go and
// suspicion.go and then quantised to ticks so no floating point runs on the GPU), the
// serf-level operations that happen between ticks (Create/Join/Leave/UserEvent), and the
// rumor-slot bookkeeping.  The data plane is gs_cuda.cu.
#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <mutex>
#include <string>
#include <type_traits>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <thread>
#include <vector>

#include "../../include/gsim.h"
#include "gs_aux.h"
#include "gs_backend.h"
#include "gs_wire.h"
#include "gs_coord.h"
#include "gs_query.h"

#ifndef GS_MAKE_BACKEND
#define GS_MAKE_BACKEND gs_make_cuda_backend
#endif
GsBackend* GS_MAKE_BACKEND(int device, char* err, size_t err_cap);

// ---------------------------------------------------------------------------
// pure formulas
// ---------------------------------------------------------------------------
extern "C" uint32_t gsim_retransmit_limit(uint32_t retransmit_mult, uint32_t n) {
  // [U] memberlist/util.go retransmitLimit: mult * ceil(log10(n+1));
  // doc form pinned by /root/reference/agent/config/runtime.go:1328-1330
  double node_scale = ceil(log10((double)n + 1.0));
  return retransmit_mult * (uint32_t)(int64_t)node_scale;
}

extern "C" uint64_t gsim_suspicion_timeout_ns(uint32_t suspicion_mult, uint32_t n,
                                              uint64_t interval_ns) {
  // [U] memberlist/util.go suspicionTimeout: mult * max(1, log10(max(1,n))) * interval,
  // computed as mult * Duration(nodeScale*1000) * interval / 1000 in int64;
  // doc form pinned by agent/config/runtime.go:1310-1312
  double node_scale = fmax(1.0, log10(fmax(1.0, (double)n)));
  int64_t scaled = (int64_t)(node_scale * 1000.0);
  return (uint64_t)((int64_t)suspicion_mult * scaled * (int64_t)interval_ns / 1000);
}

static uint64_t suspicion_total_ns(uint32_t n_confirm, uint32_t k, uint64_t min_ns,
                                   uint64_t max_ns) {
  // [U] memberlist/suspicion.go remainingSuspicionTime without the elapsed term
  if (k < 1) return min_ns;
  double frac = log((double)n_confirm + 1.0) / log((double)k + 1.0);
  double max_s = (double)max_ns / 1e9, min_s = (double)min_ns / 1e9;
  double raw = max_s - frac * (max_s - min_s);
  int64_t timeout = (int64_t)floor(1000.0 * raw) * 1000000ll;
  if (timeout < (int64_t)min_ns) timeout = (int64_t)min_ns;
  return (uint64_t)timeout;
}

extern "C" int64_t gsim_remaining_suspicion_ns(uint32_t n_confirm, uint32_t k, uint64_t elapsed_ns,
                                               uint64_t min_ns, uint64_t max_ns) {
  return (int64_t)suspicion_total_ns(n_confirm, k, min_ns, max_ns) - (int64_t)elapsed_ns;
}

extern "C" uint64_t gsim_push_pull_scale_ns(uint64_t interval_ns, uint32_t n) {
  // [U] memberlist/util.go pushPullScale, threshold 32
  if (n <= 32) return interval_ns;
  double mult = ceil(log2((double)n) - log2(32.0)) + 1.0;
  return (uint64_t)((int64_t)mult * (int64_t)interval_ns);
}

extern "C" uint32_t gsim_lamport_witness(uint32_t clock, uint32_t v) {
  // [U] serf/lamport.go Witness: if v >= cur, cur = v + 1
  return v < clock ? clock : v + 1u;
}

extern "C" uint32_t gsim_refute_incarnation(uint32_t cur, uint32_t accused) {
  // [U] memberlist/state.go refute: inc = nextIncarnation(); if accused >= inc,
  // inc = skipIncarnation(accused - inc + 1)
  uint32_t inc = cur + 1u;
  if (accused >= inc) inc += accused - inc + 1u;
  return inc;
}

extern "C" uint32_t gsim_ring_entry(uint64_t seed, uint32_t n, uint32_t member, uint32_t pass, uint32_t position) {
  if (n == 0 || position >= n) return GS_EMPTY32;
  const GsU4 rk = gs_perm_keys((uint32_t)seed, (uint32_t)(seed >> 32), member, pass);
  return gs_perm(position, n, gs_perm_bits_of(n), rk);
}

extern "C" uint32_t gsim_ring_position(uint64_t seed, uint32_t n, uint32_t member, uint32_t pass, uint32_t entry) {
  if (n == 0 || entry >= n) return GS_EMPTY32;
  const GsU4 rk = gs_perm_keys((uint32_t)seed, (uint32_t)(seed >> 32), member, pass);
  return gs_perm_inv(entry, n, gs_perm_bits_of(n), rk);
}

extern "C" void gsim_philox4x32(const uint32_t ctr[4], const uint32_t key[2], uint32_t out[4]) {
  GsU4 r = gs_philox(key[0], key[1], ctr[0], ctr[1], ctr[2], ctr[3]);
  out[0] = r.x;
  out[1] = r.y;
  out[2] = r.z;
  out[3] = r.w;
}

// ---------------------------------------------------------------------------
// config presets
// ---------------------------------------------------------------------------
static const uint64_t MS = 1000000ull, SEC = 1000000000ull;

extern "C" void gsim_config_default_lan(gsim_config* c) {
  memset(c, 0, sizeof(*c));
  c->struct_size = sizeof(*c);
  c->seed = 0x5EED0001ull;
  c->capacity = 1024;
  // [U] memberlist DefaultLANConfig, pinned by agent/config/runtime.go:1271-1336
  c->probe_interval_ns = 1 * SEC;
  c->probe_timeout_ns = 500 * MS;
  c->gossip_interval_ns = 200 * MS;
  c->gossip_to_the_dead_ns = 30 * SEC;
  c->push_pull_interval_ns = 30 * SEC;
  c->gossip_nodes = 3;
  c->indirect_checks = 3;
  c->retransmit_mult = 4;
  c->suspicion_mult = 4;
  c->suspicion_max_timeout_mult = 6;
  c->awareness_max_multiplier = 8;
  c->udp_buffer_size = 1400;
  // [U] serf DefaultConfig with Consul's overrides: libserf/serf.go:19-36,
  // agent/consul/config.go:622-623 (ReconnectTimeout 72h)
  c->event_buffer = 512;
  c->user_event_size_limit = 512;
  c->leave_propagate_delay_ns = 3 * SEC;
  c->broadcast_timeout_ns = 5 * SEC;
  c->reap_interval_ns = 15 * SEC;
  c->reconnect_timeout_ns = 72ull * 3600 * SEC;
  c->tombstone_timeout_ns = 24ull * 3600 * SEC;
  c->world_size = 1;
  c->rank = 0;
  c->device = -1;
}

extern "C" void gsim_config_default_wan(gsim_config* c) {
  gsim_config_default_lan(c);
  // [U] memberlist DefaultWANConfig, pinned by agent/config/runtime.go:1348-1413;
  // gossip_nodes stays 3: agent/config/default.go:88-89 seeds gossip_wan from the LAN struct
  c->probe_interval_ns = 5 * SEC;
  c->probe_timeout_ns = 3 * SEC;
  c->gossip_interval_ns = 500 * MS;
  c->gossip_to_the_dead_ns = 60 * SEC;
  c->push_pull_interval_ns = 60 * SEC;
  c->suspicion_mult = 6;
}

extern "C" void gsim_config_consul_test(gsim_config* c) {
  gsim_config_default_lan(c);
  // agent/consul/server_test.go:221-237
  c->probe_interval_ns = 100 * MS;
  c->probe_timeout_ns = 50 * MS;
  c->gossip_interval_ns = 100 * MS;
  c->suspicion_mult = 2;
}

// ---------------------------------------------------------------------------
// pool
// ---------------------------------------------------------------------------
struct RumorHost {
  std::string name, payload;
  int coalesce = 0;
};
struct Sched {
  uint32_t tick, id, action;  // action 1 = shut down member `id` after Leave(); 2 = resume the members paused until `tick`
};

// A few host threads that stay around between calls (Members() of a large pool splits the id range over
// them): creating threads per call costs more than the work in a process that has a GPU context mapped.
class HostWorkers {
 public:
  explicit HostWorkers(unsigned n) : n_(n) {
    for (unsigned w = 1; w < n_; ++w) th_.emplace_back([this, w] { loop(w); });
  }
  ~HostWorkers() {
    {
      std::lock_guard<std::mutex> lk(m_);
      stop_ = true;
    }
    start_.notify_all();
    for (auto& t : th_) t.join();
  }
  unsigned size() const { return n_; }
  // job(w) on every worker w in [0, n); the caller is worker 0; returns when all are done
  void run(const std::function<void(unsigned)>& job) {
    {
      std::lock_guard<std::mutex> lk(m_);
      job_ = &job;
      pending_ = n_ - 1;
      ++gen_;
    }
    start_.notify_all();
    job(0);
    std::unique_lock<std::mutex> lk(m_);
    done_.wait(lk, [this] { return pending_ == 0; });
    job_ = nullptr;
  }

 private:
  void loop(unsigned w) {
    uint64_t seen = 0;
    for (;;) {
      const std::function<void(unsigned)>* job;
      {
        std::unique_lock<std::mutex> lk(m_);
        start_.wait(lk, [&] { return stop_ || gen_ != seen; });
        if (stop_) return;
        seen = gen_;
        job = job_;
      }
      (*job)(w);
      {
        std::lock_guard<std::mutex> lk(m_);
        if (--pending_ == 0) done_.notify_one();
      }
    }
  }
  unsigned n_;
  std::vector<std::thread> th_;
  std::mutex m_;
  std::condition_variable start_, done_;
  const std::function<void(unsigned)>* job_ = nullptr;
  uint64_t gen_ = 0;
  unsigned pending_ = 0;
  bool stop_ = false;
};

struct gsim_pool {
  gsim_config cfg;
  GsBackend* be = nullptr;
  GsDev d;
  GsGlobals g;
  GsGlobals* g_dev = nullptr;
  bool g_dirty = true;
  bool counts_stale = true;
  uint32_t now = 0;
  uint64_t node_ticks = 0;
  std::mutex mu;
  RumorHost rh[GS_MAX_RUMORS];
  std::vector<Sched> sched;
  std::vector<void*> allocs;
  GsRecount rc;
  double last_ms = 0;
  uint64_t last_launches = 0;
  uint32_t events_dropped = 0;
  std::string err;
  uint64_t tick_ns = 0;
  uint32_t n_established = 0;  // members folded into the base set (not pending)
  // sharded (multi-GPU) pools: DESIGN.md §7
  bool sharded = false;
  uint32_t world = 1, rank = 0;
  size_t rows_per_rank = 0;
  uint8_t* pages = nullptr;  // page column: rank r's pool-wide words at pages + r*GS_PAGE_BYTES
  const int* shard_fds = nullptr;  // one exported descriptor per column slice
  size_t n_shard_fds = 0;
  uint32_t attached = 1;     // ranks whose memory is mapped here (including this one)
  bool ready = true;         // false between gsim_pool_create and gsim_shard_ready
  uint32_t call_seq = 0;     // controller calls so far (selects the blob slot)
  // rank-local counting: every rank counts its own rows, rank 0 sums (collective_recount)
  HostWorkers* workers = nullptr;  // created by the first bulk read that wants them
  uint32_t* stage = nullptr;  // pinned host staging for bulk reads (host_stage)
  size_t stage_words = 0;
  uint32_t quiet_fails = 0;  // consecutive looks at a pool that was still busy (try_quiet backs off)
  bool partials_fresh = false;  // (rank 0) the partial counts in its page describe (partials_seq, partials_now)
  uint32_t partials_seq = 0, partials_now = 0;
  // retirement at a step boundary clears the freed slots' bits rank by rank: the controller only collects
  // the mask (defer_and), every rank applies it to its own rows after the call (pending_keep)
  bool defer_and = false;
  uint32_t pending_keep = 0xFFFFFFFFu;
  std::vector<uint32_t> graph_rp, graph_col;  // host copy of the CSR peer graph (gsim_graph_set)
  GsXbar xb;
  std::vector<std::pair<uint32_t, uint32_t>> name_lens;  // (member, bytes of its node name) where not canonical
  // quiet-window scheduling (DESIGN.md §4.2)
  bool quiet = false;        // the pool is known to be quiet at p->now: windows may run
  bool healthy = false;      // ... and no probe can go unanswered: a launch may cover many ProbeIntervals
  bool pristine = false;     // ... and every member is up, listed alive and established: probes have a closed form
  uint32_t dirty_seq = 0;    // bumped by every host-side write to device state (quiet no longer known)
  uint32_t dirty_tick = 0;   // p->now at that write
  uint32_t retry_at = 0;     // do not look for quietness again before this tick
  // window launches, ticks run in windows, single-tick launches, horizon scans, ns of window kernels, ns of tick kernels
  uint64_t sched_counts[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  // degraded members (gsim_impair_*): the columns, allocated on first use, and how many members have a
  // non-zero impairment.  d.imp_loss / d.imp_delay point at the columns only while that count is > 0.
  uint32_t* imp_loss = nullptr;
  uint8_t* imp_delay = nullptr;
  uint32_t n_impaired = 0;
  // ... and the two columns of one-way reachability (gsim_impair_dir_*), allocated by the first setting
  // whose receive threshold differs from its send threshold or that has a flag: imp_loss is then the send
  // threshold, imp_recv the receive threshold.  Until then the receive threshold is imp_loss itself.
  uint32_t* imp_recv = nullptr;
  uint8_t* imp_flags = nullptr;
  // ... and intermittent impairment (gsim_impair_flap_*): the schedule column (gs_flap_word per member, 0 =
  // none), allocated by the first schedule call, and how many members have a schedule.  d.imp_flap points at
  // the column only while that count and n_impaired are > 0 (a schedule gates an impairment).
  uint32_t* imp_flap = nullptr;
  uint32_t n_flap = 0;
  // ... and fault domains (gsim_domain_*): the domain column (0 = none), allocated by the first domain call;
  // the domain schedule table, dom_tab[x] = gs_flap_word of domain x (0 = none), as long as the highest id
  // ever given a schedule, with its device copy (dom_tab_cap entries) and how many entries are non-zero.
  // d.imp_dom / d.dom_flap point at them only while that count and n_impaired are > 0.
  uint32_t* imp_dom = nullptr;
  std::vector<uint32_t> dom_tab;
  uint32_t* dom_tab_dev = nullptr;
  size_t dom_tab_cap = 0;
  uint32_t n_dom_sched = 0;
  // paused members (gsim_pause_*): the resume-tick column (0 = not paused) and {paused now, resumed Alive,
  // Suspect, Dead}; the first pause allocates the column and pause_cnt_dev, a device copy of the counts that
  // exists only so that snapshots carry them
  uint32_t* pause_until = nullptr;
  uint64_t* pause_cnt_dev = nullptr;
  uint64_t pause_cnt[4] = {0, 0, 0, 0};
  // network-coordinate queries (gsim_coordinates_read ...): (key, value) pairs for `capacity` entries and
  // room for partial sums and small results, allocated by the first query that needs them
  uint64_t* q_key = nullptr;
  uint32_t* q_val = nullptr;
  double* q_aux = nullptr;
  // host writes to device state not yet handed to the backend (see dev()), and whether handing an
  // earlier batch over failed (reported by the API call it belonged to)
  GsWriteBatch wb = {};
  bool wb_failed = false;
  uint32_t last_active = 0;  // GS_Q_LAST_ACTIVE as the last run_ticks left it (single-GPU pools)
};

static void counts_invalidate(gsim_pool* p) {
  p->counts_stale = true;
  p->partials_fresh = false;
}

static void mark_dirty(gsim_pool* p) {
  p->quiet = false;
  p->healthy = false;
  p->pristine = false;
  p->retry_at = 0;  // (the clock may have gone back: restore)
  p->quiet_fails = 0;
  p->dirty_seq++;
  p->dirty_tick = p->now;
}

static uint64_t gcd64(uint64_t a, uint64_t b) {
  while (b) {
    uint64_t t = a % b;
    a = b;
    b = t;
  }
  return a;
}
static uint32_t ceil_ticks(uint64_t ns, uint64_t tick) { return (uint32_t)((ns + tick - 1) / tick); }
static uint32_t clamp_ticks(uint64_t ns, uint64_t tick);

static int fail(gsim_pool* p, int code, const char* msg) {
  p->err = msg ? msg : "";
  if (code == GSIM_ERR_CUDA && p->be) p->err += std::string(": ") + p->be->last_error();
  return code;
}

// ---- host writes to device state ------------------------------------------------------------
// Queued as ops of one GsWriteBatch and handed to the backend, in order, right before the next thing
// the host asks of the device (dev()) or at the end of the API call: a write costs no round trip, and
// the read-modify-writes happen on the device, so the host never reads a word only to change it.
static bool flush_writes(gsim_pool* p) {
  if (!p->wb.n) return true;
  const bool okk = p->be->write_batch(p->wb);
  p->wb.n = 0;
  if (!okk) p->wb_failed = true;
  return okk;
}

// The backend, for anything that launches, copies or reads: every queued write comes before it.
static GsBackend* dev(gsim_pool* p) {
  flush_writes(p);
  return p->be;
}

// End of an API call: its writes are on the stream, or the call fails.
static int finish_writes(gsim_pool* p, int rc) {
  const bool okk = flush_writes(p) && !p->wb_failed;
  p->wb_failed = false;
  if (!okk && rc == GSIM_OK) rc = fail(p, GSIM_ERR_CUDA, "device write batch");
  return rc;
}

static bool put_op(gsim_pool* p, uint32_t op, const void* a, uint32_t v, const void* b = nullptr, uint32_t w = 0u,
                   uint32_t x = 0u) {
  mark_dirty(p);  // a host write to device state: whatever was known about quietness is void
  if (p->wb.n == GS_WB_MAX && !flush_writes(p)) return false;
  GsWriteOp& o = p->wb.op[p->wb.n++];
  o.a = (uint64_t)(uintptr_t)a;
  o.b = (uint64_t)(uintptr_t)b;
  o.op = op;
  o.v = v;
  o.w = w;
  o.x = x;
  return true;
}

template <class T>
static bool peek(gsim_pool* p, const T* col, size_t i, T* out) {
  return dev(p)->d2h(out, col + i, sizeof(T));
}
template <class T>
static bool poke(gsim_pool* p, T* col, size_t i, T v) {
  static_assert(sizeof(T) == 4 || sizeof(T) == 1, "device writes are words or bytes");
  return put_op(p, sizeof(T) == 4 ? GS_WR_STORE32 : GS_WR_STORE8, col + i, (uint32_t)v);
}
static bool poke_or(gsim_pool* p, uint32_t* col, size_t i, uint32_t bits) { return put_op(p, GS_WR_OR32, col + i, bits); }

// Host-side write of a member's key word (k, or the word AND k when and_mask): every replica on a
// sharded pool, and the member's status byte in step (see gs_kst_code), derived on the device.
static bool write_key(gsim_pool* p, uint32_t buf, uint32_t i, uint32_t k, bool and_mask) {
  const uint32_t op = and_mask ? GS_WR_AND32 : GS_WR_STORE32;
  for (uint32_t r = 0; r < (p->sharded ? p->world : 1u); ++r)
    if (!put_op(p, op, p->d.key_rep[buf] + (size_t)r * p->g.key_stride + i, k)) return false;
  return !p->d.kst || put_op(p, GS_WR_KST, p->d.kst + i, buf, p->d.key[buf] + i);
}
static bool poke_key(gsim_pool* p, uint32_t buf, uint32_t i, uint32_t k) { return write_key(p, buf, i, k, false); }

// One more member has heard rumor r (`add` of them): heard_cnt[r] += add, and the rumor's convergence
// tick is now if that makes every running member
static bool heard_add(gsim_pool* p, uint32_t r, uint32_t add) {
  return put_op(p, GS_WR_HEARD, p->d.heard_cnt + r, add, p->d.conv_tick + r, p->g.up_count, p->now);
}

// N-dependent scalars, recomputed whenever the member count changes (a11).
static void recompute_tables(gsim_pool* p) {
  GsGlobals& g = p->g;
  const gsim_config& c = p->cfg;
  const uint32_t n = g.n;
  g.retransmit_limit = gsim_retransmit_limit(c.retransmit_mult, n);
  if (g.retransmit_limit > 255u) g.retransmit_limit = 255u;
  // [U] memberlist/state.go suspectNode: k = SuspicionMult - 2, 0 if n-2 < k
  int k = (int)c.suspicion_mult - 2;
  if ((int)n - 2 < k) k = 0;
  if (k < 0) k = 0;
  if (k > GS_K1MAX - 1) k = GS_K1MAX - 1;
  g.sus_k = (uint32_t)k;
  uint64_t min_ns = gsim_suspicion_timeout_ns(c.suspicion_mult, n, c.probe_interval_ns);
  uint64_t max_ns = (uint64_t)c.suspicion_max_timeout_mult * min_ns;
  for (uint32_t q = 0; q < GS_K1MAX; ++q) {
    uint32_t cc = q > g.sus_k ? g.sus_k : q;
    g.sus_ticks[q] = ceil_ticks(suspicion_total_ns(cc, g.sus_k, min_ns, max_ns), p->tick_ns);
  }
  g.perm_bits = gs_perm_bits_of(n);
  g.n_magic = n ? 0xFFFFFFFFFFFFFFFFull / n + 1ull : 0ull;
  // [U] memberlist/state.go schedule: the push-pull ticker runs every pushPullScale(PushPullInterval, n)
  g.pp_interval = 0;
  g.rot_pp = 0;
  if ((c.flags & GSIM_FLAG_PUSH_PULL) && c.push_pull_interval_ns) {
    g.pp_interval = ceil_ticks(gsim_push_pull_scale_ns(c.push_pull_interval_ns, n), p->tick_ns);
    if (g.pp_interval < 2u) g.pp_interval = 2u;  // the exchange itself takes two ticks
    g.rot_pp = (gs_phase_rot(g.seed_lo, g.seed_hi) >> 8) % g.pp_interval;
  }
  p->g_dirty = true;
}

// Ordered before every later launch on the pool's stream, not waited for (the copy is staged).
static bool upload_globals(gsim_pool* p) {
  if (!p->g_dirty) return true;
  GsBackend* be = dev(p);
  if (p->sharded) {
    // the controller (rank 0) writes every rank's device copy; only `rank` differs
    for (uint32_t r = 0; r < p->world; ++r) {
      GsGlobals tmp = p->g;
      tmp.rank = r;
      if (!be->h2d_word(p->pages + (size_t)r * GS_PAGE_BYTES + GS_PG_GLOBALS, &tmp, sizeof(GsGlobals))) return false;
    }
  } else if (!be->h2d_word(p->g_dev, &p->g, sizeof(GsGlobals))) {
    return false;
  }
  p->g_dirty = false;
  return true;
}

// ---- sharded pools: the controller protocol ---------------------------------------------------
// Every rank calls every API function in the same order.  Rank 0 (the controller) executes the
// host-side operation — all device pokes go through the unified address space, to whichever GPU
// owns the row — then publishes the resulting host state (GsGlobals incl. the rumor table, clock,
// schedule, return code, small out-parameters) in a blob in its page and enters the device
// barrier; the other ranks enter the barrier, read the blob and adopt the state.
struct BlobHdr {
  int32_t rc;
  uint32_t now, n_established, n_sched, out_bytes, dirty_seq;
  uint64_t node_ticks;
  uint32_t call_seq, want_bytes;  // which call this blob answers: a rank out of step must fail, not adopt
  uint32_t pending_keep;          // bit columns every rank still has to AND on its own rows (~0 = nothing)
};

template <class F>
static int controller_call(gsim_pool* p, void* out, size_t out_bytes, F f) {
  if (!p->sharded) return finish_writes(p, f());
  const uint32_t seq = p->call_seq++;
  const uint32_t slot = seq & 1u;
  uint8_t* blob_dev = p->pages + GS_PG_BLOB + (size_t)slot * GS_BLOB_BYTES;  // in rank 0's page
  std::vector<uint8_t> blob(GS_BLOB_BYTES, 0);
  BlobHdr h;
  memset(&h, 0, sizeof(h));
  if (p->rank == 0) {
    h.rc = finish_writes(p, f());  // (the blob copy below waits for them: done before any rank goes on)
    if (p->g_dirty && !upload_globals(p)) h.rc = h.rc ? h.rc : GSIM_ERR_CUDA;
    h.now = p->now;
    h.n_established = p->n_established;
    h.n_sched = (uint32_t)p->sched.size();
    h.out_bytes = (uint32_t)(out ? out_bytes : 0);
    h.node_ticks = p->node_ticks;
    h.dirty_seq = p->dirty_seq;
    h.call_seq = seq;
    h.want_bytes = (uint32_t)out_bytes;
    h.pending_keep = p->pending_keep;
    uint8_t* w = blob.data();
    if (sizeof(h) + sizeof(GsGlobals) + (size_t)h.n_sched * sizeof(Sched) + h.out_bytes > GS_BLOB_BYTES) {
      // every rank must still leave the barrier: publish the error instead of the state
      fail(p, GSIM_ERR_INVALID, "state blob overflow (too many scheduled shutdowns for a sharded pool)");
      h.rc = GSIM_ERR_INVALID;
      h.n_sched = 0;
      h.out_bytes = 0;
    }
    memcpy(w, &h, sizeof(h)); w += sizeof(h);
    memcpy(w, &p->g, sizeof(GsGlobals)); w += sizeof(GsGlobals);
    if (h.n_sched) memcpy(w, p->sched.data(), h.n_sched * sizeof(Sched));
    w += h.n_sched * sizeof(Sched);
    if (out && h.out_bytes) memcpy(w, out, h.out_bytes);
    w += h.out_bytes;
    if (!dev(p)->h2d(blob_dev, blob.data(), (size_t)(w - blob.data()))) return fail(p, GSIM_ERR_CUDA, "blob h2d");
    if (!dev(p)->xbar_host(p->xb)) return fail(p, GSIM_ERR_CUDA, "barrier");
    return h.rc;
  }
  if (!dev(p)->xbar_host(p->xb)) return fail(p, GSIM_ERR_CUDA, "barrier");
  if (!dev(p)->d2h(blob.data(), blob_dev, GS_BLOB_BYTES)) return fail(p, GSIM_ERR_CUDA, "blob d2h");
  const uint8_t* r = blob.data();
  memcpy(&h, r, sizeof(h)); r += sizeof(h);
  if (h.call_seq != seq || h.want_bytes != (uint32_t)out_bytes) {
    char msg[160];
    snprintf(msg, sizeof(msg), "controller protocol out of step: call %u (%zu bytes out) met the blob of call %u (%u bytes out)",
             seq, out_bytes, h.call_seq, h.want_bytes);
    if (getenv("GSIM_DEBUG_PROTOCOL")) fprintf(stderr, "libgsim rank %u: %s\n", p->rank, msg);
    return fail(p, GSIM_ERR_STATE, msg);
  }
  memcpy(&p->g, r, sizeof(GsGlobals)); r += sizeof(GsGlobals);
  p->g.rank = p->rank;
  p->sched.resize(h.n_sched);
  if (h.n_sched) memcpy(p->sched.data(), r, h.n_sched * sizeof(Sched));
  r += h.n_sched * sizeof(Sched);
  if (out && h.out_bytes == out_bytes && out_bytes) memcpy(out, r, out_bytes);
  p->now = h.now;
  p->n_established = h.n_established;
  p->node_ticks = h.node_ticks;
  p->pending_keep = h.pending_keep;
  if (h.dirty_seq != p->dirty_seq) {  // the controller wrote device state: same consequence on every rank
    p->dirty_seq = h.dirty_seq;
    p->dirty_tick = p->now;
    p->quiet = false;
    p->healthy = false;
    p->pristine = false;
    p->retry_at = 0;
    p->quiet_fails = 0;
  }
  p->g_dirty = false;
  counts_invalidate(p);
  if (h.rc) p->err = "controller reported an error";
  return h.rc;
}

#define GS_CONTROLLER_ONLY(p)                                                                        \
  if ((p)->sharded && (p)->rank != 0)                                                                \
    return fail((p), GSIM_ERR_STATE, "bulk observation of a sharded pool is served by rank 0 only")

static void rebuild_class_masks(gsim_pool* p) {
  GsGlobals& g = p->g;
  g.class_mask[0] = g.class_mask[1] = g.class_mask[2] = 0;
  g.active_bytes = 0;
  for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r)
    if ((g.active_mask >> r) & 1u) {
      g.class_mask[g.rumors[r].qclass] |= 1u << r;
      g.active_bytes += g.rumors[r].size + (g.rumors[r].qclass ? 3u : 2u);
    }
  p->g_dirty = true;
}

template <class T>
static bool alloc_col(gsim_pool* p, T** out, size_t count) {
  void* q = dev(p)->alloc(count * sizeof(T));
  if (!q) return false;
  p->allocs.push_back(q);
  *out = reinterpret_cast<T*>(q);
  return true;
}

// Sharded pools: every rank's progress words say "all ticks < now are done" (controller only).
static bool reset_tick_flags(gsim_pool* p) {
  if (!p->sharded) return true;
  uint32_t words[GS_MAX_WORLD];
  for (uint32_t r = 0; r < GS_MAX_WORLD; ++r) words[r] = p->now;
  const uint32_t zero = 0;
  for (uint32_t r = 0; r < p->world; ++r) {
    uint8_t* page = p->pages + (size_t)r * GS_PAGE_BYTES;
    if (!dev(p)->h2d(page + GS_PG_TICK_FLAGS, words, sizeof(words))) return false;
    if (!dev(p)->h2d(page + GS_PG_DONE_CTR, &zero, 4)) return false;
    if (!dev(p)->h2d(page + GS_PG_TICK_BASE, &p->now, 4)) return false;
  }
  return true;
}

// Quiet-window words of every rank: nothing known (controller only).
static bool reset_qstate(gsim_pool* p) {
  const uint32_t words[GS_Q_WORDS] = {p->now, GS_NEVER, p->now, 0u};  // last-active+1 = now: tick now-1 counts as active
  for (uint32_t r = 0; r < (p->sharded ? p->world : 1u); ++r)
    if (!dev(p)->h2d(p->d.qstate[r], words, sizeof(words))) return false;
  mark_dirty(p);
  return true;
}

// Bytes a probe message leaves to piggybacked broadcasts ([U] memberlist/net.go sendMsg: UDPBufferSize -
// len(msg) - compoundHeaderOverhead), by GS_PIG_*.  The messages as memberlist's probeNode / handleIndirectPing
// send them: IPv4 address, port 8301, the name of the pool's last member id, "node-<capacity - 1>", on both ends,
// a sequence number past 2^16 (5 bytes, a member that has probed for a day), acks without a ping-delegate payload.
static void pig_budgets(const gsim_pool* p, uint32_t out[4]) {
  char name[32];
  const int len = snprintf(name, sizeof(name), "node-%u", p->cfg.capacity ? p->cfg.capacity - 1u : 0u);
  const uint8_t addr[4] = {10, 0, 0, 1};
  const uint32_t seq = 0x10000u;
  size_t msg[4];
  msg[GS_PIG_PING] = gsw::ping(nullptr, 0, seq, name, (size_t)len, addr, 4, 8301, name, (size_t)len);
  msg[GS_PIG_ACK] = gsw::ack(nullptr, 0, seq, nullptr, 0);
  msg[GS_PIG_NACK] = gsw::nack(nullptr, 0, seq);
  msg[GS_PIG_INDREQ] = gsw::indirect_ping(nullptr, 0, seq, addr, 4, 8301, name, (size_t)len, true, addr, 4, 8301, name,
                                          (size_t)len);
  for (int k = 0; k < 4; ++k) out[k] = p->g.udp_avail > msg[k] ? p->g.udp_avail - (uint32_t)msg[k] : 0u;
}

// Device-side initial state: empty columns, zeroed counters, the converged initial members.
// On a sharded pool this runs on rank 0 only and reaches every GPU through the unified columns.
static int init_device_state(gsim_pool* p) {
  GsBackend* be = dev(p);
  GsDev& d = p->d;
  GsGlobals& g = p->g;
  const size_t cap = g.cap;
  bool okk = true;
  // key = 0 means truth NONE for rows that were never created
  const size_t key_words = p->sharded ? (size_t)g.key_stride * p->world : cap;
  okk = okk && be->fill32(d.key_rep[0], 0, key_words) && be->fill32(d.key_rep[1], 0, key_words);
  for (uint32_t s = 0; s <= g.ring_mask; ++s) okk = okk && be->fill32(d.inbox[s], 0, cap);
  if (d.kst) okk = okk && be->fill8(d.kst, 0, cap);
  okk = okk && be->fill32(d.due, GS_NEVER, cap);  // rows that do not exist are never due
  okk = okk && be->fill32(d.reap_after, 0, cap);
  // rows that were never created hold the same defaults gs_init_row writes, so that a column
  // nobody has touched is one repeated word (gsim_snapshot stores such planes as a fill)
  okk = okk && be->fill32(d.cursor, 0, cap) && be->fill32(d.pass, 0, cap) && be->fill32(d.probe_tgt, 0, cap) &&
        be->fill32(d.probe_inc, 0, cap) && be->fill32(d.sus_start, 0, cap) && be->fill32(d.change_tick, 0, cap) &&
        be->fill32(d.event_min, 0, cap) && be->fill32(d.heard, 0, cap) && be->fill32(d.queued, 0, cap) &&
        be->fill32(d.ltime_member, 1, cap) && be->fill32(d.ltime_event, 1, cap) && be->fill32(d.meta, 0, cap) &&
        be->fill32(d.sus_from, GS_EMPTY32, cap * GS_K1MAX) &&
        be->fill32(reinterpret_cast<uint32_t*>(d.acc), GS_EMPTY32, cap * GS_K1MAX * 2 * 2);
  okk = okk && be->fill8(d.tx, 0, cap * GS_MAX_RUMORS);
  if (d.ppreq) okk = okk && be->fill32(d.ppreq, GS_EMPTY32, cap * 2 * GS_PPK) && be->fill32(d.pp_clk, 0, cap * 4);
  if (d.pig) {
    GsPig pig;
    memset(&pig, 0, sizeof(pig));
    pig_budgets(p, pig.budget);
    okk = okk && be->fill32(d.pig_req, GS_EMPTY32, cap * 2 * GS_PIGK) && be->h2d(d.pig, &pig, sizeof(pig));
  }
  okk = okk && be->fill32(reinterpret_cast<uint32_t*>(d.stats), 0, GSIM_STAT_COUNT * 2);
  okk = okk && be->fill32(d.heard_cnt, 0, 32) && be->fill32(d.conv_tick, GS_EMPTY32, 32);
  okk = okk && be->fill32(d.view_cnt, 0, 4) && be->fill32(d.crashed_alive, 0, 1);
  okk = okk && be->fill32(d.crashed_dead_tick, GS_EMPTY32, 1);
  okk = okk && be->fill32(d.evlog_cursor, 0, 2) && be->fill32(d.tick_base, 0, 1);
  if (!p->sharded) okk = okk && be->fill32(d.done_ctr, 0, 1);
  okk = okk && reset_qstate(p);

  p->g_dirty = true;
  okk = okk && upload_globals(p);
  okk = okk && reset_tick_flags(p);
  okk = okk && be->init_rows(d, p->g_dev, g, 0, p->cfg.n_initial, 0);
  return okk ? GSIM_OK : GSIM_ERR_CUDA;
}

extern "C" int gsim_abi_version(void) { return GSIM_ABI_VERSION; }

extern "C" const char* gsim_strerror(int code) {
  switch (code) {
    case GSIM_OK: return "ok";
    case GSIM_ERR_INVALID: return "invalid argument";
    case GSIM_ERR_NO_DEVICE: return "no usable sm_90 CUDA device (libgsim has no CPU fallback)";
    case GSIM_ERR_CUDA: return "CUDA error";
    case GSIM_ERR_CAPACITY: return "capacity exhausted";
    case GSIM_ERR_NOT_FOUND: return "not found";
    case GSIM_ERR_STATE: return "illegal state";
    case GSIM_ERR_TOO_LARGE: return "user event too large";
    case GSIM_ERR_NOMEM: return "out of memory";
  }
  return "unknown error";
}

extern "C" const char* gsim_last_error(gsim_pool* p) { return p ? p->err.c_str() : ""; }

static_assert(GS_PG_GLOBALS + sizeof(GsGlobals) <= GS_PG_SCRATCH, "GsGlobals outgrew its page slot");
static_assert(sizeof(BlobHdr) + sizeof(GsGlobals) + 4096 <= GS_BLOB_BYTES, "state blob too small");
static thread_local std::string g_create_err;

extern "C" int gsim_pool_create(const gsim_config* cfg, gsim_pool** out) {
  if (!cfg || !out || cfg->struct_size != sizeof(gsim_config)) return GSIM_ERR_INVALID;
  if (cfg->capacity == 0 || cfg->n_initial > cfg->capacity) return GSIM_ERR_INVALID;
  if (!cfg->probe_interval_ns || !cfg->probe_timeout_ns || !cfg->gossip_interval_ns)
    return GSIM_ERR_INVALID;
  if (cfg->probe_timeout_ns >= cfg->probe_interval_ns) return GSIM_ERR_INVALID;
  if (cfg->world_size < 1 || cfg->world_size > GS_MAX_WORLD || cfg->rank >= cfg->world_size) return GSIM_ERR_INVALID;
  const bool sharded = cfg->world_size > 1;
  uint64_t tick = cfg->tick_ns;
  if (!tick) tick = gcd64(gcd64(cfg->probe_interval_ns, cfg->probe_timeout_ns), cfg->gossip_interval_ns);
  if (cfg->probe_interval_ns % tick || cfg->probe_timeout_ns % tick || cfg->gossip_interval_ns % tick)
    return GSIM_ERR_INVALID;
  if (cfg->gossip_interval_ns / tick > 255 || cfg->awareness_max_multiplier < 1 ||
      cfg->awareness_max_multiplier > 8 || cfg->gossip_nodes > 8 || cfg->indirect_checks > 8)
    return GSIM_ERR_INVALID;
  const uint32_t phase_group = cfg->phase_group ? cfg->phase_group : GS_TILE;
  // 1 (per member) or 128 * 2^k (whole tiles)
  if (phase_group != 1 && (phase_group % GS_TILE != 0 || ((phase_group / GS_TILE) & (phase_group / GS_TILE - 1)) != 0))
    return GSIM_ERR_INVALID;
  // mailbox ring: 2 arrival slots unless the pool is going to carry a latency matrix
  const uint32_t ring_depth = cfg->mailbox_depth ? cfg->mailbox_depth : 2u;
  if (ring_depth < 2 || ring_depth > GS_RING_MAX || (ring_depth & (ring_depth - 1u)) != 0) return GSIM_ERR_INVALID;

  if (sharded && (cfg->flags & GSIM_FLAG_PROBE_PIGGYBACK)) {
    g_create_err = "GSIM_FLAG_PROBE_PIGGYBACK is not supported on sharded pools";
    fprintf(stderr, "libgsim: %s\n", g_create_err.c_str());
    return GSIM_ERR_INVALID;
  }

  char errbuf[256] = {0};
  GsBackend* be = GS_MAKE_BACKEND(cfg->device, errbuf, sizeof(errbuf));
  if (!be) {
    g_create_err = errbuf;
    fprintf(stderr, "libgsim: %s\n", errbuf);
    return GSIM_ERR_NO_DEVICE;
  }
  gsim_pool* p = new gsim_pool();
  p->cfg = *cfg;
  p->be = be;
  p->tick_ns = tick;
  memset(&p->d, 0, sizeof(p->d));
  memset(&p->g, 0, sizeof(p->g));
  memset(&p->rc, 0, sizeof(p->rc));
  // column stride: padded to whole tiles so the tick kernel never needs a bounds check
  size_t cap = ((size_t)cfg->capacity + GS_TILE - 1) / GS_TILE * GS_TILE;
  GsDev& d = p->d;
  GsGlobals& g = p->g;
  if (sharded) {
    // one virtual address range per column, physically sharded over the GPUs (gs_vmm.h);
    // rows per rank is a multiple of the 2 MB mapping granularity so byte columns align too
    if (!be->shard_begin(cfg->world_size, cfg->rank)) {
      g_create_err = be->last_error();
      fprintf(stderr, "libgsim: sharded pools unavailable: %s\n", be->last_error());
      gsim_pool_destroy(p);
      return GSIM_ERR_CUDA;
    }
    const size_t gran = be->shard_granularity();
    size_t per = ((size_t)cfg->capacity + cfg->world_size - 1) / cfg->world_size;
    const size_t gran_rows = gran / 2;  // the narrowest column has 2-byte elements (GS_TX)
    per = (per + gran_rows - 1) / gran_rows * gran_rows;
    p->sharded = true;
    p->world = cfg->world_size;
    p->rank = cfg->rank;
    p->rows_per_rank = per;
    p->ready = false;
    cap = per * cfg->world_size;
  }
  const size_t per_rank = p->rows_per_rank;
  auto acol = [&](auto** out, size_t planes) -> bool {
    typedef typename std::remove_pointer<typename std::remove_pointer<decltype(out)>::type>::type T;
    if (!sharded) return alloc_col(p, out, cap * planes);
    void* q = be->shard_alloc(per_rank * sizeof(T), planes);
    *out = reinterpret_cast<T*>(q);
    return q != nullptr;
  };
  bool okk = true;
  if (!sharded) {
    okk = okk && alloc_col(p, &d.key[0], cap) && alloc_col(p, &d.key[1], cap);
    d.key_rep[0] = d.key[0];
    d.key_rep[1] = d.key[1];
  } else {
    // one full replica of the key column per rank (gathers stay local; writers update all)
    const size_t gran = be->shard_granularity();
    const size_t rep_bytes = (cap * 4 + gran - 1) / gran * gran;
    g.key_stride = (uint32_t)(rep_bytes / 4);
    for (int b = 0; b < 2 && okk; ++b) {
      d.key_rep[b] = reinterpret_cast<uint32_t*>(be->shard_alloc(rep_bytes, 1));
      okk = d.key_rep[b] != nullptr;
      d.key[b] = okk ? d.key_rep[b] + (size_t)cfg->rank * g.key_stride : nullptr;
    }
  }
  if (!sharded) okk = okk && alloc_col(p, &d.kst, cap);  // performance variant: status replica
  g.ring_mask = ring_depth - 1u;
  for (uint32_t s = 0; s < ring_depth; ++s) okk = okk && acol(&d.inbox[s], 1);
  okk = okk && acol(&d.due, 1) && acol(&d.meta, 1);
  okk = okk && acol(&d.cursor, 1) && acol(&d.pass, 1);
  okk = okk && acol(&d.probe_tgt, 1) && acol(&d.probe_inc, 1);
  okk = okk && acol(&d.sus_start, 1) && acol(&d.sus_from, GS_K1MAX);
  okk = okk && acol(&d.acc, GS_K1MAX * 2);
  okk = okk && acol(&d.change_tick, 1) && acol(&d.reap_after, 1);
  okk = okk && acol(&d.ltime_member, 1) && acol(&d.ltime_event, 1);
  okk = okk && acol(&d.event_min, 1);
  okk = okk && acol(&d.heard, 1) && acol(&d.queued, 1);
  {  // two rumors per 16-bit element (GS_TX): the narrowest sharded slice is 2 bytes per member
    uint16_t* tx16 = nullptr;
    okk = okk && acol(&tx16, GS_MAX_RUMORS / 2);
    d.tx = reinterpret_cast<uint8_t*>(tx16);
  }
  if (cfg->flags & GSIM_FLAG_COORDINATES) {  // Vivaldi state: 348 B per member, only when asked for
    if (sharded) {
      g_create_err = "network coordinates are not supported on sharded pools yet";
      fprintf(stderr, "libgsim: %s\n", g_create_err.c_str());
      gsim_pool_destroy(p);
      return GSIM_ERR_INVALID;
    }
    okk = okk && alloc_col(p, &d.coord, cap * 2 * GS_COORD_WORDS) && alloc_col(p, &d.ctag, cap * 2) &&
          alloc_col(p, &d.adj, cap * GS_ADJ_WINDOW) && alloc_col(p, &d.adj_idx, cap);
  }
  if (cfg->flags & GSIM_FLAG_PUSH_PULL)  // push-pull mailboxes: 48 B per member, only when asked for
    okk = okk && acol(&d.ppreq, 2 * GS_PPK) && acol(&d.pp_clk, 4);
  if (cfg->flags & GSIM_FLAG_PROBE_PIGGYBACK)  // owed answers: 32 B per member, only when asked for
    okk = okk && alloc_col(p, &d.pig_req, cap * 2 * GS_PIGK) && alloc_col(p, &d.pig, (size_t)1);
  uint32_t evcap = cfg->event_log_capacity ? cfg->event_log_capacity : 65536u;
  if (!sharded) {
    okk = okk && alloc_col(p, &d.stats, (size_t)GSIM_STAT_COUNT);
    okk = okk && alloc_col(p, &d.heard_cnt, (size_t)32) && alloc_col(p, &d.conv_tick, (size_t)32);
    okk = okk && alloc_col(p, &d.view_cnt, (size_t)4);
    okk = okk && alloc_col(p, &d.crashed_alive, (size_t)1) && alloc_col(p, &d.crashed_dead_tick, (size_t)1);
    okk = okk && alloc_col(p, &d.evlog, (size_t)evcap) && alloc_col(p, &d.evlog_cursor, (size_t)2);
    okk = okk && alloc_col(p, &d.tick_base, (size_t)1);
    okk = okk && alloc_col(p, &d.done_ctr, (size_t)1);  // grid barrier of multi-tick launches
    okk = okk && alloc_col(p, &d.qstate[0], (size_t)GS_Q_WORDS);
    okk = okk && alloc_col(p, &p->g_dev, (size_t)1);
  } else if (okk) {
    // pool-wide words: one 2 MB page per rank; counters and the event log live in rank 0's
    p->pages = reinterpret_cast<uint8_t*>(be->shard_alloc(GS_PAGE_BYTES, 1));
    okk = p->pages != nullptr && be->shard_commit(&p->shard_fds, &p->n_shard_fds);
    if (okk) {
      uint8_t* page0 = p->pages;
      uint8_t* mine = p->pages + (size_t)p->rank * GS_PAGE_BYTES;
      d.stats = reinterpret_cast<unsigned long long*>(mine + GS_PG_STATS);  // per rank, summed on read
      d.heard_cnt = reinterpret_cast<uint32_t*>(page0 + GS_PG_HEARD_CNT);
      d.conv_tick = reinterpret_cast<uint32_t*>(page0 + GS_PG_CONV_TICK);
      d.view_cnt = reinterpret_cast<uint32_t*>(page0 + GS_PG_VIEW_CNT);
      d.crashed_alive = reinterpret_cast<uint32_t*>(page0 + GS_PG_CRASHED_ALIVE);
      d.crashed_dead_tick = reinterpret_cast<uint32_t*>(page0 + GS_PG_CRASHED_DEAD_TICK);
      d.evlog_cursor = reinterpret_cast<uint32_t*>(page0 + GS_PG_EVLOG_CURSOR);
      d.evlog = reinterpret_cast<GsEventRec*>(page0 + GS_PG_EVLOG);
      const uint32_t room = (GS_PAGE_BYTES - GS_PG_EVLOG) / (uint32_t)sizeof(GsEventRec);
      if (evcap > room) evcap = room;
      d.tick_base = reinterpret_cast<uint32_t*>(mine + GS_PG_TICK_BASE);
      p->g_dev = reinterpret_cast<GsGlobals*>(mine + GS_PG_GLOBALS);
      for (uint32_t r = 0; r < GS_MAX_WORLD; ++r)
        p->xb.flags[r] = reinterpret_cast<uint32_t*>(p->pages + (size_t)(r < p->world ? r : 0) * GS_PAGE_BYTES + GS_PG_XBAR_FLAGS);
      for (uint32_t r = 0; r < GS_MAX_WORLD; ++r)
        d.tick_flags[r] = reinterpret_cast<uint32_t*>(p->pages + (size_t)(r < p->world ? r : 0) * GS_PAGE_BYTES + GS_PG_TICK_FLAGS);
      d.done_ctr = reinterpret_cast<uint32_t*>(mine + GS_PG_DONE_CTR);
      for (uint32_t r = 0; r < p->world; ++r)
        d.qstate[r] = reinterpret_cast<uint32_t*>(p->pages + (size_t)r * GS_PAGE_BYTES + GS_PG_QSTATE);
      p->xb.epoch = reinterpret_cast<uint32_t*>(mine + GS_PG_XBAR_EPOCH);
      p->xb.rank = p->rank;
      p->xb.world = p->world;
      // peers write barrier flags into this page as soon as they have mapped it: zero it now
      okk = be->fill8(mine, 0, GS_PAGE_BYTES) && be->sync();
    }
  }
  if (!okk) {
    g_create_err = be->last_error();
    fprintf(stderr, "libgsim: allocation failed: %s\n", be->last_error());
    gsim_pool_destroy(p);
    return GSIM_ERR_NOMEM;
  }

  g.n = cfg->n_initial;
  p->n_established = cfg->n_initial;
  g.cap = (uint32_t)cap;
  g.up_count = cfg->n_initial;
  g.P = (uint32_t)(cfg->probe_interval_ns / tick);
  g.T = (uint32_t)(cfg->probe_timeout_ns / tick);
  g.GI = (uint32_t)(cfg->gossip_interval_ns / tick);
  g.gossip_nodes = cfg->gossip_nodes;
  g.indirect_checks = cfg->indirect_checks;
  g.awareness_max = cfg->awareness_max_multiplier;
  g.gtd_ticks = ceil_ticks(cfg->gossip_to_the_dead_ns, tick);
  // [U] memberlist/state.go gossip(): bytesAvail = UDPBufferSize - compoundHeaderOverhead(2)
  g.udp_avail = cfg->udp_buffer_size > 2 ? cfg->udp_buffer_size - 2 : 0;
  g.disable_tcp = cfg->disable_tcp_pings;
  g.loss_thr = (uint32_t)(((uint64_t)cfg->packet_loss_ppm << 32) / 1000000ull);
  if (cfg->packet_loss_ppm >= 1000000u) g.loss_thr = 0xFFFFFFFFu;
  g.event_buffer = cfg->event_buffer;
  g.seed_lo = (uint32_t)cfg->seed;
  g.seed_hi = (uint32_t)(cfg->seed >> 32);
  g.flags = cfg->flags;
  g.evlog_cap = evcap;
  g.world = cfg->world_size;
  g.rank = cfg->rank;
  g.phase_group = phase_group;
  g.phase_gate = (phase_group % GS_TILE == 0) ? 1u : 0u;
  g.phase_shift = 0;
  while (g.phase_gate && (GS_TILE << g.phase_shift) < phase_group) g.phase_shift++;
  {
    const uint32_t rot = gs_phase_rot(g.seed_lo, g.seed_hi);
    g.rot_p = rot % g.P;
    g.rot_g = (rot >> 16) % g.GI;
  }
  g.rows_per_rank = (uint32_t)p->rows_per_rank;
  g.tick_seconds = (double)tick / 1.0e9;
  g.coord_base_rtt_s = 0.0005;  // a direct ack inside one tick: half a millisecond on top of the matrix
  recompute_tables(p);
  if (!sharded && init_device_state(p) != GSIM_OK) {  // sharded pools: gsim_shard_ready
    g_create_err = be->last_error();
    fprintf(stderr, "libgsim: pool init failed: %s\n", be->last_error());
    gsim_pool_destroy(p);
    return GSIM_ERR_CUDA;
  }
  *out = p;
  return GSIM_OK;
}

// ---- sharded pools: wiring the ranks together ------------------------------------------------------
extern "C" int gsim_shard_export_fds(gsim_pool* p, int* fds, size_t cap, size_t* n) {
  if (!p || !n || !p->sharded) return GSIM_ERR_INVALID;
  *n = p->n_shard_fds;
  if (fds) {
    if (cap < p->n_shard_fds) return GSIM_ERR_INVALID;
    memcpy(fds, p->shard_fds, p->n_shard_fds * sizeof(int));
  }
  return GSIM_OK;
}

extern "C" int gsim_shard_attach(gsim_pool* p, uint32_t peer_rank, const int* fds, size_t n) {
  if (!p || !p->sharded || p->ready || !fds) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (!dev(p)->shard_attach(peer_rank, fds, n)) return fail(p, GSIM_ERR_CUDA, "shard_attach");
  p->attached += 1;
  return GSIM_OK;
}

extern "C" int gsim_shard_ready(gsim_pool* p) {
  if (!p) return GSIM_ERR_INVALID;
  if (!p->sharded) return GSIM_OK;
  std::lock_guard<std::mutex> lk(p->mu);
  if (p->ready) return GSIM_OK;
  if (p->attached != p->world) return fail(p, GSIM_ERR_STATE, "not every peer rank has been attached");
  if (!dev(p)->xbar_host(p->xb)) return fail(p, GSIM_ERR_CUDA, "barrier");  // every page is mapped and zeroed
  int rc = controller_call(p, nullptr, 0, [&]() -> int { return init_device_state(p); });
  if (rc) return fail(p, rc, "init");
  p->ready = true;
  return GSIM_OK;
}

extern "C" void gsim_pool_destroy(gsim_pool* p) {
  if (!p) return;
  if (p->be) {
    dev(p)->sync();
    if (p->stage) dev(p)->host_free(p->stage);
    delete p->workers;
    p->workers = nullptr;
    for (void* q : p->allocs) dev(p)->release(q);
    delete p->be;
  }
  delete p;
}

// ---- rumor slots --------------------------------------------------------------
static void shard_rows(const gsim_pool* p, uint32_t* first, uint32_t* count) {
  const uint32_t n = p->g.n;
  *first = 0;
  *count = n;
  if (p->sharded) {
    const uint64_t f = (uint64_t)p->rank * p->rows_per_rank;
    *first = f < n ? (uint32_t)f : n;
    *count = *first + p->rows_per_rank < n ? (uint32_t)p->rows_per_rank : n - *first;
  }
}

// Sharded pools count rank by rank: every rank runs the count over ITS rows (local HBM instead of a
// walk of the whole pool over NVLink from GPU 0) and leaves the partial in rank 0's page; the
// controller sums them in do_recount as long as nothing was written since.  Called by every rank,
// outside controller_call, right before a call whose controller side wants counts.
static int collective_recount(gsim_pool* p) {
  if (!p->sharded || !p->ready) return GSIM_OK;
  static_assert(sizeof(GsRecount) <= 512 && GS_PG_SCRATCH + 512u * GS_MAX_WORLD_ <= GS_PG_BLOB, "partial counts");
  GsRecount part;
  uint32_t first, count;
  shard_rows(p, &first, &count);
  // (the device copy of the globals is current: every controller call ends with the upload)
  const bool usable = !(p->rank == 0 && p->g_dirty);
  if (!dev(p)->recount(p->d, p->g_dev, p->g, p->now, first, count, &part)) return GSIM_ERR_CUDA;
  if (!dev(p)->h2d(p->pages + GS_PG_SCRATCH + 512u * p->rank, &part, sizeof(part))) return GSIM_ERR_CUDA;
  if (!dev(p)->xbar_host(p->xb)) return GSIM_ERR_CUDA;
  if (p->rank == 0) {
    p->partials_fresh = usable;
    p->partials_seq = p->dirty_seq;
    p->partials_now = p->now;
  }
  return GSIM_OK;
}

static bool do_recount(gsim_pool* p) {
  if (!p->counts_stale) return true;
  if (!upload_globals(p)) return false;
  if (p->sharded && p->partials_fresh && p->partials_seq == p->dirty_seq && p->partials_now == p->now) {
    std::vector<uint8_t> raw(512u * p->world);
    if (!dev(p)->d2h(raw.data(), p->pages + GS_PG_SCRATCH, raw.size())) return false;
    memset(&p->rc, 0, sizeof(p->rc));
    uint32_t* sum = reinterpret_cast<uint32_t*>(&p->rc);
    for (uint32_t r = 0; r < p->world; ++r) {
      GsRecount part;
      memcpy(&part, raw.data() + 512u * r, sizeof(part));
      const uint32_t* w = reinterpret_cast<const uint32_t*>(&part);
      for (size_t x = 0; x < sizeof(GsRecount) / 4; ++x) sum[x] += w[x];
    }
  } else if (!dev(p)->recount(p->d, p->g_dev, p->g, p->now, 0u, p->g.n, &p->rc)) {
    return false;
  }
  p->counts_stale = false;
  return true;
}

static bool and_bit_columns(gsim_pool* p, uint32_t keep);

// Free a rumor slot, all but clearing its bits from the heard / queued / mailbox columns (the caller
// does that, for every slot it frees at once: and_bit_columns).
static int release_slot(gsim_pool* p, uint32_t slot) {
  GsGlobals& g = p->g;
  GsRumor& ru = g.rumors[slot];
  if (ru.kind == GSIM_RUMOR_ALIVE) {
    // fold into the base state: the subject becomes known to every non-isolated member.  The subject
    // of a tracked alive rumor is pending in both key buffers: gsim_member_add sets the bit, nothing
    // but this clears it, and reaping or pruning a member keeps it.
    p->n_established += 1;
    if (!write_key(p, 0, ru.subject, ~(1u << 4), true) || !write_key(p, 1, ru.subject, ~(1u << 4), true))
      return GSIM_ERR_CUDA;
  }
  g.active_mask &= ~(1u << slot);
  memset(&ru, 0, sizeof(ru));
  p->rh[slot] = RumorHost();
  rebuild_class_masks(p);
  if (!poke(p, p->d.heard_cnt, slot, 0u) || !poke(p, p->d.conv_tick, slot, GS_EMPTY32))
    return GSIM_ERR_CUDA;
  counts_invalidate(p);
  return GSIM_OK;
}

static int retire_slot(gsim_pool* p, uint32_t slot) {
  const int rc = release_slot(p, slot);
  if (rc) return rc;
  return and_bit_columns(p, ~(1u << slot)) ? GSIM_OK : GSIM_ERR_CUDA;
}

// heard/queued/inbox bits of a freed slot must be zero before the slot is reused.
static bool and_bit_columns(gsim_pool* p, uint32_t keep) {
  mark_dirty(p);
  if (p->sharded && p->defer_and) {  // step boundary: every rank clears its own rows after the call
    p->pending_keep &= keep;
    return true;
  }
  return dev(p)->and_columns(p->d, p->g, keep, 0u, p->g.n);
}

// ... which is this, on every rank, right after the controller call that collected the mask.
static int apply_pending_and(gsim_pool* p) {
  if (!p->sharded || p->pending_keep == 0xFFFFFFFFu) return GSIM_OK;
  uint32_t first, count;
  shard_rows(p, &first, &count);
  const bool ok = dev(p)->and_columns(p->d, p->g, p->pending_keep, first, count) && dev(p)->sync();
  p->pending_keep = 0xFFFFFFFFu;
  // nobody goes on (to reuse a freed slot, to tick) before every rank's rows are clean
  if (!ok || !dev(p)->xbar_host(p->xb)) return GSIM_ERR_CUDA;
  return GSIM_OK;
}

// Retire finished membership rumors (alive / intents): every UP member has heard them and
// nobody is retransmitting any more.  Runs at step boundaries only.
static int auto_retire(gsim_pool* p) {
  GsGlobals& g = p->g;
  uint32_t cand = 0;
  for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r)
    if (((g.active_mask >> r) & 1u) && g.rumors[r].kind != GSIM_RUMOR_USER_EVENT) cand |= 1u << r;
  if (!cand) return GSIM_OK;
  if (!do_recount(p)) return GSIM_ERR_CUDA;
  uint32_t keep = 0xFFFFFFFFu;
  for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r) {
    if (!((cand >> r) & 1u)) continue;
    // an alive rumor folds into the base set only when nobody still depends on having
    // heard it individually (members that have not joined the base set yet)
    if (g.rumors[r].kind == GSIM_RUMOR_ALIVE && p->rc.isolated_up != 0) continue;
    if (p->rc.heard_cnt[r] == g.up_count && p->rc.queued_cnt[r] == 0) {
      int rcode = release_slot(p, r);
      if (rcode) return rcode;
      keep &= ~(1u << r);
    }
  }
  // one pass over the bit columns for every slot freed
  if (keep != 0xFFFFFFFFu && !and_bit_columns(p, keep)) return GSIM_ERR_CUDA;
  return GSIM_OK;
}

static int alloc_slot(gsim_pool* p, uint32_t* slot_out) {
  GsGlobals& g = p->g;
  for (int attempt = 0; attempt < 2; ++attempt) {
    for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r)
      if (!((g.active_mask >> r) & 1u)) {
        *slot_out = r;
        return GSIM_OK;
      }
    if (attempt == 0) {
      int rc = auto_retire(p);
      if (rc) return rc;
    }
  }
  return GSIM_ERR_CAPACITY;
}

// A member whose broadcast queue became non-empty between ticks must be looked at by the
// next tick: set the wake bit in the mailbox that tick will read.
// A piggybacking pool also stamps its gate for that tick (GsPig::gate).
static bool post_wake(gsim_pool* p, uint32_t row) {
  if (p->d.pig && !poke(p, reinterpret_cast<uint32_t*>(p->d.pig), p->now % GS_PIG_GATES, p->now + 1u)) return false;
  return poke_or(p, p->d.inbox[p->now & p->g.ring_mask], row, GS_WAKE_BIT);
}

// ---- message sizes: what the encoder (gs_wire.h) produces for this member ------------------------
// A virtual member is called "node-<id>" unless gsim_member_desc.name_len said otherwise.
static uint32_t member_name_len(const gsim_pool* p, uint32_t id) {
  for (const auto& kv : p->name_lens)
    if (kv.first == id) return kv.second;
  uint32_t digits = 1;
  for (uint32_t v = id; v >= 10u; v /= 10u) ++digits;
  return 5u + digits;
}
static uint32_t alive_size(const gsim_pool* p, uint32_t id, uint32_t inc, uint32_t meta_len) {
  static const uint8_t vsn[6] = {1, 5, 2, 2, 5, 4}, addr[4] = {10, 0, 0, 1};
  static const char none = 0;
  return (uint32_t)gsw::alive(nullptr, 0, inc, nullptr, member_name_len(p, id), addr, 4, 8301, &none, meta_len, vsn);
}
static uint32_t intent_size(const gsim_pool* p, uint32_t id, bool leave, uint32_t ltime) {
  return (uint32_t)gsw::serf_intent(nullptr, 0, leave, ltime, nullptr, member_name_len(p, id), false, false);
}

static int start_rumor(gsim_pool* p, uint32_t slot, uint32_t kind, uint32_t subject, uint32_t inc,
                       uint32_t ltime, uint32_t origin, uint32_t size, uint32_t qclass) {
  GsGlobals& g = p->g;
  GsRumor& ru = g.rumors[slot];
  ru.kind = kind;
  ru.subject = subject;
  ru.inc = inc;
  ru.ltime = ltime;
  ru.origin = origin;
  ru.size = size;
  ru.qclass = qclass;
  ru.start_tick = p->now;
  g.active_mask |= 1u << slot;
  rebuild_class_masks(p);
  // the origin holds it with transmits = 0
  if (!poke_or(p, p->d.heard, origin, 1u << slot) || !poke_or(p, p->d.queued, origin, 1u << slot)) return GSIM_ERR_CUDA;
  if (!poke(p, p->d.tx, GS_TX(slot, g.cap, origin), (uint8_t)0)) return GSIM_ERR_CUDA;
  if (!post_wake(p, origin)) return GSIM_ERR_CUDA;
  if (!poke(p, p->d.heard_cnt, slot, 1u)) return GSIM_ERR_CUDA;
  if (!poke(p, p->d.conv_tick, slot, g.up_count == 1u ? p->now : GS_EMPTY32)) return GSIM_ERR_CUDA;
  counts_invalidate(p);
  return GSIM_OK;
}

static void log_host_event(gsim_pool* p, uint32_t type, uint32_t subject, uint32_t observer,
                           uint32_t ltime) {
  uint32_t cur[2];
  if (!dev(p)->d2h(cur, p->d.evlog_cursor, 8)) return;
  if (cur[0] < p->g.evlog_cap) {
    GsEventRec e = {p->now, type, subject, observer, ltime, 0u};
    dev(p)->h2d(p->d.evlog + cur[0], &e, sizeof(e));
    cur[0]++;
  } else {
    cur[1]++;
  }
  dev(p)->h2d(p->d.evlog_cursor, cur, 8);
}

// ---- membership operations -------------------------------------------------------
extern "C" int gsim_member_add(gsim_pool* p, const gsim_member_desc* desc, uint32_t* id_out) {
  if (!p || !id_out) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  return controller_call(p, id_out, sizeof(uint32_t), [&]() -> int {
  GsGlobals& g = p->g;
  if (g.graph_n) return fail(p, GSIM_ERR_STATE, "the peer graph of this pool is static (gsim_graph_set)");
  if (g.n >= p->cfg.capacity) return fail(p, GSIM_ERR_CAPACITY, "member capacity exhausted");
  uint32_t slot;
  int rc = alloc_slot(p, &slot);
  if (rc) return fail(p, rc, "no free rumor slot for the member's alive broadcast");
  const uint32_t id = g.n;
  if (!upload_globals(p)) return fail(p, GSIM_ERR_CUDA, "upload");
  if (!dev(p)->init_rows(p->d, p->g_dev, g, id, 1, p->now)) return fail(p, GSIM_ERR_CUDA, "init_rows");
  // [U] memberlist.Create -> setAlive: incarnation 1, alive{} queued on the new member;
  // pending: other members learn of it only through that rumor (aliveNode).
  const uint32_t k = gs_key_make(1u, 1u, GS_RANK_ALIVE, GS_TRUTH_UP);
  uint32_t flags = 0;
  // it knows nobody yet; with an empty base set there is nothing it could be missing
  if (p->n_established > 0) flags |= GS_META_ISOLATED;
  if (desc && (desc->flags & GSIM_MEMBER_WATCHED)) flags |= GS_META_WATCHED;
  if (!poke_key(p, 0, id, k) || !poke_key(p, 1, id, k) || (flags && !poke_or(p, p->d.meta, id, flags)))
    return fail(p, GSIM_ERR_CUDA, "poke");
  g.n += 1;
  g.up_count += 1;
  recompute_tables(p);
  if (desc && desc->name_len) p->name_lens.push_back(std::make_pair(id, desc->name_len));
  uint32_t size = desc && desc->alive_msg_size ? desc->alive_msg_size : alive_size(p, id, 1u, desc ? desc->meta_len : 0u);
  rc = start_rumor(p, slot, GSIM_RUMOR_ALIVE, id, 1u, 0u, id, size, 0u);
  if (rc) return fail(p, rc, "start_rumor");
  *id_out = id;
  return GSIM_OK;
  });
}

// One direction of a join push-pull: `dst` merges what `src` knows
// ([U] memberlist.mergeState -> aliveNode; [U] serf/delegate.go MergeRemoteState).
// rs / rd: the rows of both ends as rows_read gave them, brought up to date with every write of the
// join so far; rd gets this merge's writes.
static int merge_remote(gsim_pool* p, uint32_t dst, const uint32_t* rs, uint32_t* rd, bool ignore_old_events) {
  GsGlobals& g = p->g;
  uint32_t hs = rs[3], hd = rd[3], qd = rd[4], lm_s = rs[5], le_s = rs[6], lm_d = rd[5], le_d = rd[6], emin = rd[7], md = rd[2];
  // clocks: Witness(remote - 1)  ==  max(local, remote)
  if (lm_s > lm_d) lm_d = lm_s;
  if (le_s > le_d) le_d = le_s;
  if (ignore_old_events && le_s > emin) emin = le_s;  // eventMinTime = pp.EventLTime
  uint32_t fresh = hs & ~hd & g.active_mask;
  uint32_t accepted = 0;
  for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r) {
    if (!((fresh >> r) & 1u)) continue;
    const GsRumor& ru = g.rumors[r];
    bool accept = true;
    if (ru.kind == GSIM_RUMOR_USER_EVENT) {
      if (ru.ltime >= le_d) le_d = ru.ltime + 1u;
      if (ru.ltime < emin) accept = false;
      else if (le_d > g.event_buffer && ru.ltime < le_d - g.event_buffer) accept = false;
      if (accept && (md & GS_META_WATCHED)) log_host_event(p, GSIM_EVENT_USER, r, dst, ru.ltime);
    } else if (ru.kind == GSIM_RUMOR_JOIN_INTENT || ru.kind == GSIM_RUMOR_LEAVE_INTENT) {
      if (ru.ltime >= lm_d) lm_d = ru.ltime + 1u;
    } else if (ru.kind == GSIM_RUMOR_ALIVE) {
      if (md & GS_META_WATCHED) log_host_event(p, GSIM_EVENT_MEMBER_JOIN, ru.subject, dst, 0u);
    } else if (ru.kind == GSIM_RUMOR_UPDATE) {
      if (md & GS_META_WATCHED) log_host_event(p, GSIM_EVENT_MEMBER_UPDATE, ru.subject, dst, 0u);
    }
    if (accept) {
      accepted |= 1u << r;
      if (!poke(p, p->d.tx, GS_TX(r, g.cap, dst), (uint8_t)0) || !heard_add(p, r, 1u)) return GSIM_ERR_CUDA;
    }
  }
  hd |= accepted;
  qd |= accepted;
  if (accepted && !post_wake(p, dst)) return GSIM_ERR_CUDA;
  if (!poke(p, p->d.heard, dst, hd) || !poke(p, p->d.queued, dst, qd) ||
      !poke(p, p->d.ltime_member, dst, lm_d) || !poke(p, p->d.ltime_event, dst, le_d) ||
      !poke(p, p->d.event_min, dst, emin))
    return GSIM_ERR_CUDA;
  rd[3] = hd;
  rd[4] = qd;
  rd[5] = lm_d;
  rd[6] = le_d;
  rd[7] = emin;
  counts_invalidate(p);
  return GSIM_OK;
}

extern "C" int gsim_join(gsim_pool* p, uint32_t id, const uint32_t* seeds, size_t n_seeds,
                         int ignore_old, int* n_ok) {
  if (!p || (!seeds && n_seeds)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  int n_ok_local = 0;
  if (!n_ok) n_ok = &n_ok_local;
  return controller_call(p, n_ok, sizeof(int), [&]() -> int {
  GsGlobals& g = p->g;
  if (id >= g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  // the joiner's and every seed's row in one round trip; the join works on this copy from here on,
  // writing to it what it writes to the device
  std::vector<uint32_t> ids(1, id);
  for (size_t s = 0; s < n_seeds; ++s)
    if (seeds[s] < g.n && std::find(ids.begin(), ids.end(), seeds[s]) == ids.end()) ids.push_back(seeds[s]);
  std::vector<uint32_t> rows(ids.size() * 8);
  if (!dev(p)->rows_read(p->d, ids.data(), (uint32_t)ids.size(), rows.data())) return fail(p, GSIM_ERR_CUDA, "rows_read");
  auto row = [&](uint32_t m) { return rows.data() + 8 * (std::find(ids.begin(), ids.end(), m) - ids.begin()); };
  const uint32_t cur = p->now & 1u;  // (rows hold key[0] and key[1])
  uint32_t* ri = row(id);
  if (gs_key_truth(ri[cur]) != GS_TRUTH_UP) return fail(p, GSIM_ERR_STATE, "member is not running");
  // GSIM_IMPAIR_NO_TCP at the joiner or at a seed: the push-pull to that seed cannot connect (only pools
  // that have the flag column read it; a member with a flap schedule of its own or of its domain only while
  // its impairment is in force now, gs_in_force)
  std::vector<uint8_t> no_tcp(ids.size(), 0u);
  for (size_t x = 0; p->imp_flags && x < ids.size(); ++x) {
    if (!peek(p, p->imp_flags, ids[x], &no_tcp[x])) return fail(p, GSIM_ERR_CUDA, "peek");
    no_tcp[x] &= GSIM_IMPAIR_NO_TCP;
    uint32_t w = 0u, dom = 0u, wd = 0u;
    if (no_tcp[x] && p->d.imp_flap && !peek(p, p->imp_flap, ids[x], &w)) return fail(p, GSIM_ERR_CUDA, "peek");
    if (no_tcp[x] && p->d.dom_flap && !peek(p, p->imp_dom, ids[x], &dom)) return fail(p, GSIM_ERR_CUDA, "peek");
    if (p->d.dom_flap && dom < p->dom_tab.size()) wd = p->dom_tab[dom];
    if (!gs_in_force(g.seed_lo, g.seed_hi, ids[x], w, dom, wd, p->now)) no_tcp[x] = 0u;
  }
  auto tcp_blocked = [&](uint32_t m) { return no_tcp[std::find(ids.begin(), ids.end(), m) - ids.begin()] != 0u; };
  int okc = 0;
  for (size_t s = 0; s < n_seeds; ++s) {
    uint32_t sd = seeds[s];
    if (sd >= g.n || sd == id) continue;
    uint32_t* rsd = row(sd);
    if (gs_key_truth(rsd[cur]) != GS_TRUTH_UP) continue;  // unreachable seed: Join skips it
    if (tcp_blocked(id) || tcp_blocked(sd)) continue;     // ... and so does a seed it cannot connect to
    // push-pull in both directions; eventJoinIgnore applies to the joiner only
    int rc = merge_remote(p, id, rsd, ri, ignore_old != 0);
    if (!rc) rc = merge_remote(p, sd, ri, rsd, false);
    if (rc) return fail(p, rc, "merge");
    uint32_t mi = ri[2], ms = rsd[2];
    uint32_t iso = mi & ms & GS_META_ISOLATED;
    mi = (mi & ~GS_META_ISOLATED) | iso;
    ms = (ms & ~GS_META_ISOLATED) | iso;
    if (!poke(p, p->d.meta, id, mi) || !poke(p, p->d.meta, sd, ms)) return fail(p, GSIM_ERR_CUDA, "poke");
    ri[2] = mi;
    rsd[2] = ms;
    ++okc;
  }
  if (okc > 0) {
    // [U] serf.Join -> broadcastJoin(clock.Time()): Witness(ltime), join intent queued
    const uint32_t lm = ri[5];
    uint32_t slot;
    int rc = alloc_slot(p, &slot);
    if (rc == GSIM_OK) {
      rc = start_rumor(p, slot, GSIM_RUMOR_JOIN_INTENT, id, 0u, lm, id, intent_size(p, id, false, lm), 1u);
      if (rc) return fail(p, rc, "start_rumor");
    } else if (rc != GSIM_ERR_CAPACITY) {
      return fail(p, rc, "alloc_slot");
    }
    if (!poke(p, p->d.ltime_member, id, lm + 1u)) return fail(p, GSIM_ERR_CUDA, "poke");
  }
  if (n_ok) *n_ok = okc;
  return GSIM_OK;
  });
}

static int set_truth(gsim_pool* p, uint32_t id, uint32_t truth) {
  for (int b = 0; b < 2; ++b) {
    uint32_t k;
    if (!peek(p, p->d.key[b], id, &k)) return GSIM_ERR_CUDA;
    k = (k & ~3u) | truth;
    if (!poke_key(p, b, id, k)) return GSIM_ERR_CUDA;
  }
  return GSIM_OK;
}

// Member id is not paused any more (crashed for good, or gone): clear its resume tick.
static bool pause_forget(gsim_pool* p, uint32_t id) {
  if (!p->pause_cnt[0]) return true;
  uint32_t until = 0;
  if (!peek(p, p->pause_until, id, &until)) return false;
  if (!until) return true;
  p->pause_cnt[0]--;
  return poke(p, p->pause_until, id, 0u);
}

static int refresh_after_truth_change(gsim_pool* p) {
  counts_invalidate(p);
  if (!do_recount(p)) return GSIM_ERR_CUDA;
  GsGlobals& g = p->g;
  g.up_count = p->rc.truth_cnt[GS_TRUTH_UP];
  p->g_dirty = true;
  if (!poke(p, p->d.crashed_alive, 0, p->rc.crashed_alive)) return GSIM_ERR_CUDA;
  uint32_t cdt = GS_EMPTY32;
  if (p->rc.crashed_alive == 0 && p->rc.truth_cnt[GS_TRUTH_CRASHED] > 0) cdt = p->now;
  if (!poke(p, p->d.crashed_dead_tick, 0, cdt)) return GSIM_ERR_CUDA;
  // heard counters are over UP members only
  for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r) {
    if (!((g.active_mask >> r) & 1u)) continue;
    if (!poke(p, p->d.heard_cnt, r, p->rc.heard_cnt[r])) return GSIM_ERR_CUDA;
    if (p->rc.heard_cnt[r] == g.up_count && !heard_add(p, r, 0u)) return GSIM_ERR_CUDA;  // (converged now?)
  }
  return GSIM_OK;
}

extern "C" int gsim_crash_many(gsim_pool* p, const uint32_t* ids, size_t n) {
  if (!p || (!ids && n)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  return controller_call(p, nullptr, 0, [&]() -> int {
  for (size_t x = 0; x < n; ++x) {
    if (ids[x] >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
    uint32_t k;
    if (!peek(p, p->d.key[p->now & 1u], ids[x], &k)) return fail(p, GSIM_ERR_CUDA, "peek");
    if (gs_key_truth(k) != GS_TRUTH_UP) {
      // a paused member crashes for good: its resume is cancelled
      if (gs_key_truth(k) == GS_TRUTH_CRASHED && !pause_forget(p, ids[x])) return fail(p, GSIM_ERR_CUDA, "peek");
      continue;
    }
    int rc = set_truth(p, ids[x], GS_TRUTH_CRASHED);
    if (rc) return fail(p, rc, "set_truth");
  }
  int rc = refresh_after_truth_change(p);
  return rc ? fail(p, rc, "recount") : GSIM_OK;
  });
}

extern "C" int gsim_crash(gsim_pool* p, uint32_t id) { return gsim_crash_many(p, &id, 1); }

extern "C" int gsim_crash_fraction(gsim_pool* p, uint32_t ppm, uint32_t salt, uint32_t* n_crashed) {
  if (!p || ppm > 1000000u) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  uint32_t n_crashed_local = 0;
  if (!n_crashed) n_crashed = &n_crashed_local;
  return controller_call(p, n_crashed, sizeof(uint32_t), [&]() -> int {
  uint32_t thr = ppm >= 1000000u ? 0xFFFFFFFFu : (uint32_t)(((uint64_t)ppm << 32) / 1000000ull);
  uint32_t cnt = 0;
  if (!upload_globals(p)) return fail(p, GSIM_ERR_CUDA, "upload");
  mark_dirty(p);
  if (!dev(p)->crash_fraction(p->d, p->g_dev, p->g, thr, salt, p->now, &cnt))
    return fail(p, GSIM_ERR_CUDA, "crash_fraction");
  if (n_crashed) *n_crashed = cnt;
  int rc = refresh_after_truth_change(p);
  return rc ? fail(p, rc, "recount") : GSIM_OK;
  });
}

// (*Serf).SetTags -> [U] memberlist.UpdateNode: the member re-announces itself with new meta under
// the next incarnation; every receiver's aliveNode takes the higher incarnation and raises
// NotifyUpdate -> serf EventMemberUpdate.  The tags themselves stay on the host (SURVEY 8b).
extern "C" int gsim_member_update(gsim_pool* p, uint32_t id, uint32_t alive_msg_size, uint32_t* slot_out) {
  if (!p) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  uint32_t slot_local = 0;
  if (!slot_out) slot_out = &slot_local;
  return controller_call(p, slot_out, sizeof(uint32_t), [&]() -> int {
  GsGlobals& g = p->g;
  if (id >= g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  uint32_t k, m;
  if (!peek(p, p->d.key[p->now & 1u], id, &k) || !peek(p, p->d.meta, id, &m))
    return fail(p, GSIM_ERR_CUDA, "peek");
  if (gs_key_truth(k) != GS_TRUTH_UP || (m & GS_META_LEAVING))
    return fail(p, GSIM_ERR_STATE, "member is not running");
  uint32_t slot;
  int rc = alloc_slot(p, &slot);
  if (rc) return fail(p, rc, "no free rumor slot");
  const uint32_t inc = gs_key_inc(k) + 1u;  // nextIncarnation
  for (int b = 0; b < 2; ++b) {
    uint32_t kk;
    if (!peek(p, p->d.key[b], id, &kk)) return fail(p, GSIM_ERR_CUDA, "peek");
    if (!poke_key(p, b, id, gs_key_with_inc(kk, inc))) return fail(p, GSIM_ERR_CUDA, "poke");
  }
  rc = start_rumor(p, slot, GSIM_RUMOR_UPDATE, id, inc, 0u, id, alive_msg_size ? alive_msg_size : alive_size(p, id, inc, 0u), 0u);
  if (rc) return fail(p, rc, "start_rumor");
  *slot_out = slot;
  return GSIM_OK;
  });
}

extern "C" int gsim_leave(gsim_pool* p, uint32_t id) {
  if (!p) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  return controller_call(p, nullptr, 0, [&]() -> int {
  GsGlobals& g = p->g;
  if (id >= g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  uint32_t k, m;
  if (!peek(p, p->d.key[p->now & 1u], id, &k) || !peek(p, p->d.meta, id, &m))
    return fail(p, GSIM_ERR_CUDA, "peek");
  if (gs_key_truth(k) != GS_TRUTH_UP || (m & GS_META_LEAVING))
    return fail(p, GSIM_ERR_STATE, "member is not running or already leaving");
  // [U] serf.Leave: leave intent with the member clock, then memberlist.Leave broadcasts
  // dead{Node == From} which every receiver records as StateLeft.
  uint32_t lm;
  if (!peek(p, p->d.ltime_member, id, &lm)) return fail(p, GSIM_ERR_CUDA, "peek");
  uint32_t slot;
  int rc = alloc_slot(p, &slot);
  if (rc == GSIM_OK) {
    rc = start_rumor(p, slot, GSIM_RUMOR_LEAVE_INTENT, id, 0u, lm, id, intent_size(p, id, true, lm), 1u);
    if (rc) return fail(p, rc, "start_rumor");
  } else if (rc != GSIM_ERR_CAPACITY) {
    return fail(p, rc, "alloc_slot");
  }
  if (!poke(p, p->d.ltime_member, id, lm + 1u)) return fail(p, GSIM_ERR_CUDA, "poke");
  for (int b = 0; b < 2; ++b) {
    uint32_t kk;
    if (!peek(p, p->d.key[b], id, &kk)) return fail(p, GSIM_ERR_CUDA, "peek");
    kk = gs_key_with_rank(kk, GS_RANK_LEFT);
    if (!poke_key(p, b, id, kk)) return fail(p, GSIM_ERR_CUDA, "poke");
  }
  m |= GS_META_LEAVING;
  if (!poke(p, p->d.meta, id, m) || !poke(p, p->d.change_tick, id, p->now))
    return fail(p, GSIM_ERR_CUDA, "poke");
  if (g.flags & GSIM_FLAG_LOG_GLOBAL_EVENTS) log_host_event(p, GSIM_EVENT_MEMBER_LEAVE, id, GS_EMPTY32, 0);
  // the process lingers while its two broadcasts drain, then LeavePropagateDelay
  uint32_t rounds = g.gossip_nodes ? (g.retransmit_limit + g.gossip_nodes - 1) / g.gossip_nodes : 0;
  uint32_t drain = rounds * g.GI;
  uint32_t bt = ceil_ticks(p->cfg.broadcast_timeout_ns, p->tick_ns);
  if (drain > bt) drain = bt;
  uint32_t linger = 2 * drain + ceil_ticks(p->cfg.leave_propagate_delay_ns, p->tick_ns);
  Sched s = {p->now + linger, id, 1u};
  p->sched.push_back(s);
  counts_invalidate(p);
  return GSIM_OK;
  });
}

extern "C" int gsim_force_leave(gsim_pool* p, uint32_t via, uint32_t target, int prune) {
  if (!p) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  return controller_call(p, nullptr, 0, [&]() -> int {
  if (via >= p->g.n || target >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  // [U] serf.RemoveFailedNode: a forged leave intent turns Failed into Left.  The decision is
  // taken on the member's CURRENT record (the buffer the next tick reads); the other buffer may
  // still hold the previous state (DIRTY), so the result is written to both and DIRTY is dropped.
  uint32_t k, m;
  if (!peek(p, p->d.key[p->now & 1u], target, &k) || !peek(p, p->d.meta, target, &m))
    return fail(p, GSIM_ERR_CUDA, "peek");
  const uint32_t k_before = k;
  if (gs_key_rank(k) == GS_RANK_DEAD) k = gs_key_with_rank(k, GS_RANK_LEFT);
  if (prune && gs_key_rank(k) == GS_RANK_LEFT && gs_key_truth(k) != GS_TRUTH_UP && gs_key_truth(k) != GS_TRUTH_NONE) {
    if (!gs_key_pending(k)) p->n_established -= 1;
    k &= ~3u;
  }
  if (k != k_before) {
    if (!poke_key(p, 0, target, k) || !poke_key(p, 1, target, k)) return fail(p, GSIM_ERR_CUDA, "poke");
    if ((m & GS_META_DIRTY) && !poke(p, p->d.meta, target, m & ~GS_META_DIRTY)) return fail(p, GSIM_ERR_CUDA, "poke");
    // a paused member that is pruned or listed Left stays gone: it will not resume
    if (gs_key_truth(k_before) == GS_TRUTH_CRASHED && !pause_forget(p, target)) return fail(p, GSIM_ERR_CUDA, "peek");
  }
  int rc = refresh_after_truth_change(p);
  return rc ? fail(p, rc, "recount") : GSIM_OK;
  });
}

extern "C" int gsim_user_event(gsim_pool* p, uint32_t id, const void* name, size_t name_len,
                               const void* payload, size_t payload_len, int coalesce,
                               uint32_t* slot_out) {
  if (!p || (!name && name_len) || (!payload && payload_len)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  uint32_t slot_local = 0;
  if (!slot_out) slot_out = &slot_local;
  return controller_call(p, slot_out, sizeof(uint32_t), [&]() -> int {
  GsGlobals& g = p->g;
  if (id >= g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  // [U] serf.UserEvent: size limit on name+payload (agent side: user_event.go:82-113)
  if (name_len + payload_len > p->cfg.user_event_size_limit)
    return fail(p, GSIM_ERR_TOO_LARGE, "user event exceeds UserEventSizeLimit");
  uint32_t k, m;
  if (!peek(p, p->d.key[p->now & 1u], id, &k) || !peek(p, p->d.meta, id, &m))
    return fail(p, GSIM_ERR_CUDA, "peek");
  if (gs_key_truth(k) != GS_TRUTH_UP) return fail(p, GSIM_ERR_STATE, "member is not running");
  uint32_t le;
  if (!peek(p, p->d.ltime_event, id, &le)) return fail(p, GSIM_ERR_CUDA, "peek");
  std::string nm((const char*)name, name_len), pl((const char*)payload, payload_len);
  // identical (LTime, Name, Payload) is the same event for serf's de-dup ring
  for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r) {
    if (!((g.active_mask >> r) & 1u) || g.rumors[r].kind != GSIM_RUMOR_USER_EVENT) continue;
    if (g.rumors[r].ltime == le && p->rh[r].name == nm && p->rh[r].payload == pl) {
      // [U] serf.UserEvent -> handleUserEvent on the caller's own buffer, then QueueBroadcast: a
      // member that had not seen this (LTime, Name, Payload) delivers it now; either way its copy
      // is (re)queued with transmits = 0.
      uint32_t h, q;
      if (!peek(p, p->d.heard, id, &h) || !peek(p, p->d.queued, id, &q)) return fail(p, GSIM_ERR_CUDA, "peek");
      if (!((h >> r) & 1u)) {
        if (!poke(p, p->d.heard, id, h | (1u << r)) || !heard_add(p, r, 1u)) return fail(p, GSIM_ERR_CUDA, "poke");
        if (m & GS_META_WATCHED) log_host_event(p, GSIM_EVENT_USER, r, id, le);
      }
      if (!poke(p, p->d.queued, id, q | (1u << r)) || !poke(p, p->d.tx, GS_TX(r, g.cap, id), (uint8_t)0) ||
          !post_wake(p, id) || !poke(p, p->d.ltime_event, id, le + 1u))
        return fail(p, GSIM_ERR_CUDA, "poke");
      counts_invalidate(p);
      if (slot_out) *slot_out = r;
      return GSIM_OK;
    }
  }
  // the encoded messageUserEvent{LTime,Name,Payload,CC} behind its serf type byte
  static const char some = 0;  // (a non-nil payload slice; sizing reads no bytes)
  uint32_t size = (uint32_t)gsw::serf_user_event(nullptr, 0, le, nullptr, name_len, &some, payload_len, coalesce != 0, false);
  // [U] serf.UserEvent checks the limit a second time on the ENCODED message
  if (size > p->cfg.user_event_size_limit)
    return fail(p, GSIM_ERR_TOO_LARGE, "encoded user event exceeds UserEventSizeLimit");
  uint32_t slot;
  int rc = alloc_slot(p, &slot);
  if (rc) return fail(p, rc, "no free rumor slot");
  rc = start_rumor(p, slot, GSIM_RUMOR_USER_EVENT, id, 0u, le, id, size, 2u);
  if (rc) return fail(p, rc, "start_rumor");
  p->rh[slot].name = nm;
  p->rh[slot].payload = pl;
  p->rh[slot].coalesce = coalesce;
  if (!poke(p, p->d.ltime_event, id, le + 1u)) return fail(p, GSIM_ERR_CUDA, "poke");
  if (m & GS_META_WATCHED) log_host_event(p, GSIM_EVENT_USER, slot, id, le);
  if (slot_out) *slot_out = slot;
  return GSIM_OK;
  });
}

// Out-of-band delivery of a tracked broadcast to one member: what arrival by gossip would do, but
// now and by name.  BASELINE config 5's bridge members use it to re-fire an event they delivered
// in one WAN pool into the other (models ForwardRPC, agent/consul/internal_endpoint.go:839).
extern "C" int gsim_rumor_inject(gsim_pool* p, uint32_t slot, uint32_t id, int* accepted_out) {
  if (!p || slot >= GS_MAX_RUMORS) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  int acc_local = 0;
  if (!accepted_out) accepted_out = &acc_local;
  return controller_call(p, accepted_out, sizeof(int), [&]() -> int {
  GsGlobals& g = p->g;
  *accepted_out = 0;
  if (!((g.active_mask >> slot) & 1u)) return fail(p, GSIM_ERR_NOT_FOUND, "slot is free");
  if (id >= g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  uint32_t k, m, h, q, le, lm, emin;
  if (!peek(p, p->d.key[p->now & 1u], id, &k) || !peek(p, p->d.meta, id, &m) ||
      !peek(p, p->d.heard, id, &h) || !peek(p, p->d.queued, id, &q) ||
      !peek(p, p->d.ltime_event, id, &le) || !peek(p, p->d.ltime_member, id, &lm) ||
      !peek(p, p->d.event_min, id, &emin))
    return fail(p, GSIM_ERR_CUDA, "peek");
  if (gs_key_truth(k) != GS_TRUTH_UP) return fail(p, GSIM_ERR_STATE, "member is not running");
  if ((h >> slot) & 1u) return GSIM_OK;  // already delivered: serf's de-dup ring drops it
  const GsRumor& ru = g.rumors[slot];
  bool accept = true;
  if (ru.kind == GSIM_RUMOR_USER_EVENT) {
    if (ru.ltime >= le) le = ru.ltime + 1u;
    if (ru.ltime < emin) accept = false;
    else if (le > g.event_buffer && ru.ltime < le - g.event_buffer) accept = false;
    if (accept && (m & GS_META_WATCHED)) log_host_event(p, GSIM_EVENT_USER, slot, id, ru.ltime);
    if (!poke(p, p->d.ltime_event, id, le)) return fail(p, GSIM_ERR_CUDA, "poke");
  } else if (ru.kind == GSIM_RUMOR_JOIN_INTENT || ru.kind == GSIM_RUMOR_LEAVE_INTENT) {
    if (ru.ltime >= lm) lm = ru.ltime + 1u;
    if (!poke(p, p->d.ltime_member, id, lm)) return fail(p, GSIM_ERR_CUDA, "poke");
  } else if (ru.kind == GSIM_RUMOR_ALIVE) {
    if (m & GS_META_WATCHED) log_host_event(p, GSIM_EVENT_MEMBER_JOIN, ru.subject, id, 0u);
  } else if (ru.kind == GSIM_RUMOR_UPDATE) {
    if (m & GS_META_WATCHED) log_host_event(p, GSIM_EVENT_MEMBER_UPDATE, ru.subject, id, 0u);
  }
  if (!accept) return GSIM_OK;
  if (!poke(p, p->d.heard, id, h | (1u << slot)) || !poke(p, p->d.queued, id, q | (1u << slot)) ||
      !poke(p, p->d.tx, GS_TX(slot, g.cap, id), (uint8_t)0) || !post_wake(p, id) || !heard_add(p, slot, 1u))
    return fail(p, GSIM_ERR_CUDA, "poke");
  counts_invalidate(p);
  *accepted_out = 1;
  return GSIM_OK;
  });
}

// Peer graph in CSR form (north_star: "message-passing kernel over a CSR peer graph"; SURVEY 7):
// member i's memberlist becomes col_idx[row_ptr[i] .. row_ptr[i+1]) — peer selection for gossip,
// indirect-probe relays, push-pull and the probe ring all draw from that row instead of [0, n).
// A graph whose every row is [0, n) reproduces the complete-graph results bit for bit.  Static
// topology: rows for exactly the current members; gsim_member_add is refused while a graph is set.
extern "C" int gsim_graph_set(gsim_pool* p, uint32_t n_rows, const uint32_t* row_ptr, const uint32_t* col_idx) {
  if (!p || (n_rows && (!row_ptr || !col_idx))) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (p->sharded) return fail(p, GSIM_ERR_STATE, "peer graphs are not supported on sharded pools");
  GsGlobals& g = p->g;
  if (n_rows == 0) {
    g.graph_n = 0;
    p->d.row_ptr = p->d.col_idx = nullptr;
    p->graph_rp.clear();
    p->graph_col.clear();
    p->g_dirty = true;
    return GSIM_OK;
  }
  if (n_rows != g.n) return fail(p, GSIM_ERR_INVALID, "the graph must have one row per member");
  if (row_ptr[0] != 0) return fail(p, GSIM_ERR_INVALID, "row_ptr[0] must be 0");
  for (uint32_t i = 0; i < n_rows; ++i)
    if (row_ptr[i + 1] < row_ptr[i]) return fail(p, GSIM_ERR_INVALID, "row_ptr must be non-decreasing");
  const uint32_t nnz = row_ptr[n_rows];
  for (uint32_t e = 0; e < nnz; ++e)
    if (col_idx[e] >= g.n) return fail(p, GSIM_ERR_INVALID, "col_idx out of range");
  uint32_t *rp_dev = nullptr, *col_dev = nullptr;
  if (!alloc_col(p, &rp_dev, (size_t)n_rows + 1) || !alloc_col(p, &col_dev, (size_t)(nnz ? nnz : 1)))
    return fail(p, GSIM_ERR_NOMEM, "graph allocation");
  if (!dev(p)->h2d(rp_dev, row_ptr, ((size_t)n_rows + 1) * 4) || (nnz && !dev(p)->h2d(col_dev, col_idx, (size_t)nnz * 4)))
    return fail(p, GSIM_ERR_CUDA, "h2d");
  p->graph_rp.assign(row_ptr, row_ptr + n_rows + 1);
  p->graph_col.assign(col_idx, col_idx + nnz);
  p->d.row_ptr = rp_dev;
  p->d.col_idx = col_dev;
  g.graph_n = n_rows;
  p->g_dirty = true;
  return GSIM_OK;
}

// serf.Config.ReconnectTimeoutOverride (internal/gossip/libserf/serf.go:68-85: a member may
// advertise its own reconnect timeout in a tag; agent/consul/client_test.go:862-894).  The callback
// is host code; its result for one member is stored here and used by the reaper instead of the
// pool's ReconnectTimeout.  0 restores the default.
extern "C" int gsim_member_reconnect_timeout_set(gsim_pool* p, uint32_t id, uint64_t timeout_ns) {
  if (!p) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  return controller_call(p, nullptr, 0, [&]() -> int {
  if (id >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  uint32_t ticks = timeout_ns ? clamp_ticks(timeout_ns, p->tick_ns) : 0u;
  if (timeout_ns && ticks == 0u) ticks = 1u;
  if (!poke(p, p->d.reap_after, id, ticks)) return fail(p, GSIM_ERR_CUDA, "poke");
  if (ticks && (p->g.reap_min_override == 0u || ticks < p->g.reap_min_override)) {
    p->g.reap_min_override = ticks;
    p->g_dirty = true;
  }
  return GSIM_OK;
  });
}

// (*Serf).GetCoordinate / GetCachedCoordinate(name) — agent/router/router.go:62-67: the member's
// current network coordinate (vec[8], error, adjustment, height; seconds).
extern "C" int gsim_coordinate_get(gsim_pool* p, uint32_t id, double out[11]) {
  if (!p || !out) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GS_CONTROLLER_ONLY(p);
  if (!p->d.coord) return fail(p, GSIM_ERR_STATE, "the pool was created without GSIM_FLAG_COORDINATES");
  if (id >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  const size_t cap = p->g.cap;
  uint32_t ta, tb;
  if (!peek(p, p->d.ctag, id, &ta) || !peek(p, p->d.ctag, cap + id, &tb)) return fail(p, GSIM_ERR_CUDA, "peek");
  const size_t slot = tb > ta ? 1 : 0;
  for (size_t x = 0; x < GS_COORD_WORDS; ++x)
    if (!peek(p, p->d.coord, (slot * GS_COORD_WORDS + x) * cap + id, &out[x])) return fail(p, GSIM_ERR_CUDA, "peek");
  return GSIM_OK;
}

// ---- network-coordinate queries (DESIGN.md §3.4 "Queries", gs_query.h) -----------------------------
// The backend defaults (gs_backend.h): the coordinate columns copied to the host behind a GsDev of host
// pointers, the query bodies of gs_query.h run there, the results copied back.
namespace {
struct HostCoords {
  std::vector<double> coord;
  std::vector<uint32_t> ctag, key;
  std::vector<uint8_t> delay;
  std::vector<uint32_t> flap, dom, dom_flap;
  GsDev d;
  bool load(GsBackend* be, const GsDev& dd, const GsGlobals& g, uint32_t now, bool keys) {
    const size_t cap = g.cap;
    d = dd;
    coord.resize(cap * 2 * GS_COORD_WORDS);
    ctag.resize(cap * 2);
    if (!be->d2h(coord.data(), dd.coord, coord.size() * 8) || !be->d2h(ctag.data(), dd.ctag, ctag.size() * 4))
      return false;
    d.coord = coord.data();
    d.ctag = ctag.data();
    if (dd.imp_delay) {
      delay.resize(cap);
      if (!be->d2h(delay.data(), dd.imp_delay, cap)) return false;
      d.imp_delay = delay.data();
    }
    if (dd.imp_flap) {
      flap.resize(cap);
      if (!be->d2h(flap.data(), dd.imp_flap, cap * 4)) return false;
      d.imp_flap = flap.data();
    }
    if (dd.dom_flap) {
      dom.resize(cap);
      dom_flap.resize(dd.dom_flap_n);
      if (!be->d2h(dom.data(), dd.imp_dom, cap * 4) || !be->d2h(dom_flap.data(), dd.dom_flap, (size_t)dd.dom_flap_n * 4))
        return false;
      d.imp_dom = dom.data();
      d.dom_flap = dom_flap.data();
    }
    if (keys) {
      key.resize(g.n);
      if (g.n && !be->d2h(key.data(), dd.key[now & 1u], (size_t)g.n * 4)) return false;
      d.key[now & 1u] = key.data();
    }
    return true;
  }
};
}  // namespace

static_assert(sizeof(GsCoord) == GS_COORD_WORDS * sizeof(double), "a coordinate row is its 11 doubles");

bool GsBackend::coord_rows(const GsDev& d, const GsGlobals& g, uint32_t first, uint32_t count, double* rows) {
  if (!count) return true;
  HostCoords h;
  if (!h.load(this, d, g, 0u, false)) return false;
  std::vector<GsCoord> out(count);
  for (uint32_t x = 0; x < count; ++x) gs_coord_pick(h.d.coord, h.d.ctag, g.cap, first + x, out[x]);
  return h2d(rows, out.data(), out.size() * sizeof(GsCoord));
}

bool GsBackend::coord_pairs(const GsDev& d, const GsGlobals*, const GsGlobals& g, uint32_t now, const uint32_t* a, const uint32_t* b,
                            uint32_t n, double* est, double* tru) {
  if (!n) return true;
  HostCoords h;
  std::vector<uint32_t> ha(n), hb(n);
  std::vector<double> he(n), ht(n);
  if (!h.load(this, d, g, 0u, false) || !d2h(ha.data(), a, (size_t)n * 4) || !d2h(hb.data(), b, (size_t)n * 4))
    return false;
  for (uint32_t k = 0; k < n; ++k) {
    GsCoord ca, cb;
    gs_coord_pick(h.d.coord, h.d.ctag, g.cap, ha[k], ca);
    gs_coord_pick(h.d.coord, h.d.ctag, g.cap, hb[k], cb);
    he[k] = gs_coord_distance_seconds(ca, cb);
    ht[k] = gs_model_rtt(g, h.d, ha[k], hb[k], now);
  }
  return h2d(est, he.data(), (size_t)n * 8) && (!tru || h2d(tru, ht.data(), (size_t)n * 8));
}

bool GsBackend::coord_dist_from(const GsDev& d, const GsGlobals*, const GsGlobals& g, uint32_t now, uint32_t from,
                                const uint32_t* ids, uint32_t n, bool router, uint64_t* key, uint32_t* val) {
  if (!n) return true;
  HostCoords h;
  std::vector<uint32_t> hi(n);
  std::vector<uint64_t> hk(n);
  if (!h.load(this, d, g, now, router) || (ids && !d2h(hi.data(), ids, (size_t)n * 4))) return false;
  GsCoord cf;
  gs_coord_pick(h.d.coord, h.d.ctag, g.cap, from, cf);
  for (uint32_t x = 0; x < n; ++x) {
    const uint32_t s = ids ? hi[x] : x;
    if (router) {
      gs_router_entry(h.d, g, now, from, cf, s, &hk[x], &hi[x]);
    } else {
      GsCoord c;
      gs_coord_pick(h.d.coord, h.d.ctag, g.cap, s, c);
      hk[x] = gs_dist_key(gs_coord_distance_seconds(cf, c));
      hi[x] = s;
    }
  }
  return h2d(key, hk.data(), (size_t)n * 8) && h2d(val, hi.data(), (size_t)n * 4);
}

bool GsBackend::sort_pairs(const GsGlobals&, uint64_t* key, uint32_t* val, uint32_t n, uint32_t n_dcs) {
  if (n < 2u) return true;
  std::vector<uint64_t> hk(n), sk(n);
  std::vector<uint32_t> hv(n), sv(n), ord(n);
  if (!d2h(hk.data(), key, (size_t)n * 8) || !d2h(hv.data(), val, (size_t)n * 4)) return false;
  for (uint32_t x = 0; x < n; ++x) ord[x] = x;
  std::stable_sort(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) {
    if (n_dcs) {
      const uint32_t da = gs_dc_digit(hv[a], n_dcs), db = gs_dc_digit(hv[b], n_dcs);
      if (da != db) return da < db;
    }
    return hk[a] < hk[b];
  });
  for (uint32_t x = 0; x < n; ++x) {
    sk[x] = hk[ord[x]];
    sv[x] = hv[ord[x]];
  }
  return h2d(key, sk.data(), (size_t)n * 8) && h2d(val, sv.data(), (size_t)n * 4);
}

bool GsBackend::dc_medians(const GsGlobals&, const uint64_t* key, const uint32_t* val, uint32_t n, uint32_t n_dcs,
                           double* med, uint32_t* cnt) {
  std::vector<uint64_t> hk(n);
  std::vector<uint32_t> hv(n), hc(n_dcs, 0u), first(n_dcs, 0u);
  std::vector<double> hm(n_dcs);
  if (n && (!d2h(hk.data(), key, (size_t)n * 8) || !d2h(hv.data(), val, (size_t)n * 4))) return false;
  for (uint32_t x = 0; x < n; ++x) {
    const uint32_t c = gs_dc_digit(hv[x], n_dcs);
    if (c >= n_dcs) continue;
    if (!hc[c]) first[c] = x;
    hc[c]++;
  }
  for (uint32_t c = 0; c < n_dcs; ++c) hm[c] = hc[c] ? gs_key_dist(hk[first[c] + hc[c] / 2u]) : gs_key_dist(0x7FF0000000000000ull);
  return h2d(med, hm.data(), (size_t)n_dcs * 8) && h2d(cnt, hc.data(), (size_t)n_dcs * 4);
}

bool GsBackend::coord_error(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now, uint32_t n_draws,
                            uint32_t salt, uint64_t* key, uint32_t* val, double* part, double* out) {
  const uint32_t nch = (n_draws + GS_ERR_CHUNK - 1u) / GS_ERR_CHUNK;
  HostCoords h;
  if (!h.load(this, d, g, now, true)) return false;
  std::vector<uint64_t> hk(n_draws);
  std::vector<uint32_t> hv(n_draws);
  std::vector<double> hp(2 * (size_t)nch, 0.0);
  for (uint32_t k = 0; k < n_draws; ++k) {
    const double e = gs_error_draw(h.d, g, now, k, salt);
    hv[k] = k;
    hk[k] = ~0ull;
    if (e < 0.0) continue;
    hk[k] = gs_dist_key(e);
    hp[k / GS_ERR_CHUNK] = hp[k / GS_ERR_CHUNK] + e;
    hp[nch + k / GS_ERR_CHUNK] += 1.0;
  }
  if (!h2d(key, hk.data(), (size_t)n_draws * 8) || !h2d(val, hv.data(), (size_t)n_draws * 4) ||
      !sort_pairs(g, key, val, n_draws, 0u) || !d2h(hk.data(), key, (size_t)n_draws * 8))
    return false;
  double ho[6];
  gs_error_finish(hk.data(), n_draws, hp.data(), ho);
  (void)g_dev;
  return h2d(part, hp.data(), hp.size() * 8) && h2d(out, ho, sizeof(ho));
}

static int coord_query_check(gsim_pool* p) {
  if (!p->d.coord) return fail(p, GSIM_ERR_STATE, "the pool was created without GSIM_FLAG_COORDINATES");
  return GSIM_OK;
}

// q_aux: chunk sums and counts of gsim_coordinate_error (2 per GS_ERR_CHUNK draws of `capacity`), then
// room for the small results (its 6 statistics; the per-datacenter medians and counts)
static size_t query_aux_small(const gsim_pool* p) { return 2 * ((size_t)p->g.cap / GS_ERR_CHUNK + 1); }

static bool query_alloc(gsim_pool* p) {
  if (p->q_key) return true;
  const size_t cap = p->g.cap;
  uint64_t* k = nullptr;
  uint32_t* v = nullptr;
  double* a = nullptr;
  if (!alloc_col(p, &k, cap) || !alloc_col(p, &v, cap) || !alloc_col(p, &a, query_aux_small(p) + 2 * GS_MAX_DCS))
    return false;
  p->q_key = k;
  p->q_val = v;
  p->q_aux = a;
  return true;
}

static int check_ids(gsim_pool* p, const uint32_t* ids, size_t n) {
  for (size_t x = 0; x < n; ++x)
    if (ids[x] >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  return GSIM_OK;
}

// (*Serf).GetCoordinate for members [first, first + count) — what `consul rtt` and the catalog's
// Coordinate.ListNodes read (agent/consul/coordinate_endpoint.go): out[11 x ..] is exactly what
// gsim_coordinate_get returns for member first + x.
extern "C" int gsim_coordinates_read(gsim_pool* p, uint32_t first, uint32_t count, double* out) {
  if (!p || (!out && count)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GS_CONTROLLER_ONLY(p);
  int rc = coord_query_check(p);
  if (rc) return rc;
  if (first > p->g.n || count > p->g.n - first) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  if (!count) return GSIM_OK;
  const size_t bytes = (size_t)count * sizeof(GsCoord);
  double* rows = reinterpret_cast<double*>(dev(p)->alloc(bytes));
  if (!rows) return fail(p, GSIM_ERR_NOMEM, "coordinate rows");
  const bool okk = dev(p)->coord_rows(p->d, p->g, first, count, rows) && dev(p)->d2h(out, rows, bytes);
  dev(p)->release(rows);
  return okk ? GSIM_OK : fail(p, GSIM_ERR_CUDA, "coord_rows");
}

// librtt.ComputeDistance (internal/gossip/librtt/rtt.go:16-22), what `consul rtt` prints, for n pairs; and the
// round trip a direct probe between them samples in the model (§3.5), to measure the embedding against.
extern "C" int gsim_rtt_many(gsim_pool* p, const uint32_t* a, const uint32_t* b, size_t n, double* est_s,
                             double* true_s) {
  if (!p || (n && (!a || !b || !est_s)) || n > 0x7FFFFFFFu) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GS_CONTROLLER_ONLY(p);
  int rc = coord_query_check(p);
  if (!rc) rc = check_ids(p, a, n);
  if (!rc) rc = check_ids(p, b, n);
  if (rc || !n) return rc;
  if (!upload_globals(p)) return fail(p, GSIM_ERR_CUDA, "upload");
  // one buffer: a, b, then the estimates and the true round trips next to each other (one readback)
  uint8_t* buf = reinterpret_cast<uint8_t*>(dev(p)->alloc(n * 24));
  if (!buf) return fail(p, GSIM_ERR_NOMEM, "pair buffers");
  uint32_t* da = reinterpret_cast<uint32_t*>(buf);
  uint32_t* db = da + n;
  double* de = reinterpret_cast<double*>(buf + n * 8);
  double* dt = true_s ? de + n : nullptr;
  std::vector<double> back(true_s ? 2 * n : 0);
  bool okk = dev(p)->h2d_async(da, a, n * 4) && dev(p)->h2d_async(db, b, n * 4) &&
             dev(p)->coord_pairs(p->d, p->g_dev, p->g, p->now, da, db, (uint32_t)n, de, dt);
  if (okk && true_s) {
    okk = dev(p)->d2h(back.data(), de, n * 16);
    if (okk) {
      memcpy(est_s, back.data(), n * 8);
      memcpy(true_s, back.data() + n, n * 8);
    }
  } else if (okk) {
    okk = dev(p)->d2h(est_s, de, n * 8);
  }
  dev(p)->release(buf);
  return okk ? GSIM_OK : fail(p, GSIM_ERR_CUDA, "coord_pairs");
}

// sortNodesByDistanceFrom (agent/consul/rtt.go:14-52, 190-220): the ?near= order of catalog and health results,
// a sort.Stable of `ids` (NULL: every created member, in id order) by ComputeDistance from `from`.  The first k
// results are written (k = n for the whole order, small k for NearestN); ties keep input order.
extern "C" int gsim_sort_by_distance(gsim_pool* p, uint32_t from, const uint32_t* ids, size_t n, size_t k,
                                     uint32_t* out_ids, double* out_dist) {
  if (!p) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GS_CONTROLLER_ONLY(p);
  int rc = coord_query_check(p);
  if (rc) return rc;
  const size_t count = ids ? n : p->g.n;
  if (from >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  if (ids && (rc = check_ids(p, ids, n))) return rc;
  if (count > p->g.cap) return fail(p, GSIM_ERR_INVALID, "more ids than the pool's capacity");
  if (k > count || (k && !out_ids)) return fail(p, GSIM_ERR_INVALID, "k must be <= the number of ids");
  if (!count) return GSIM_OK;
  if (!query_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "query buffers");
  if (!upload_globals(p)) return fail(p, GSIM_ERR_CUDA, "upload");
  GsBackend* be = dev(p);
  bool okk = (!ids || be->h2d_async(p->q_val, ids, count * 4)) &&
             be->coord_dist_from(p->d, p->g_dev, p->g, p->now, from, ids ? p->q_val : nullptr, (uint32_t)count, false,
                                 p->q_key, p->q_val) &&
             be->sort_pairs(p->g, p->q_key, p->q_val, (uint32_t)count, 0u);
  if (okk && k) okk = be->d2h(out_ids, p->q_val, k * 4) && (!out_dist || be->d2h(out_dist, p->q_key, k * 8));
  if (okk && !k) okk = be->sync();
  return okk ? GSIM_OK : fail(p, GSIM_ERR_CUDA, "sort_by_distance");
}

// Router.GetDatacentersByDistance (agent/router/router.go:537-615) for one area, seen from `from`: every server
// (servers == NULL: every member, as in a WAN pool) that the view does not list Left and that still exists
// counts, in datacenter (i / 128) % n_dcs; one in from's own datacenter at 0.0, every other at ComputeDistance.
// A datacenter's RTT is rtts[len / 2] of its sorted RTTs; datacenters are stable-sorted by it, ties in index
// order (where upstream's sort.Strings pass over DC names stands).  dc_order / dc_rtt hold n_dcs entries; a
// datacenter without a counted server (upstream: absent) comes last with dc_rtt = +inf.
extern "C" int gsim_dcs_by_distance(gsim_pool* p, uint32_t from, const uint32_t* servers, size_t n_servers,
                                    uint32_t* dc_order, double* dc_rtt) {
  if (!p || !dc_order || !dc_rtt || (!servers && n_servers)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GS_CONTROLLER_ONLY(p);
  int rc = coord_query_check(p);
  if (rc) return rc;
  const uint32_t n_dcs = p->g.n_dcs;
  if (!n_dcs) return fail(p, GSIM_ERR_STATE, "the pool has no latency matrix (no datacenters)");
  if (from >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  if (servers && (rc = check_ids(p, servers, n_servers))) return rc;
  const size_t count = servers ? n_servers : p->g.n;
  if (count > p->g.cap) return fail(p, GSIM_ERR_INVALID, "more servers than the pool's capacity");
  if (!query_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "query buffers");
  if (!upload_globals(p)) return fail(p, GSIM_ERR_CUDA, "upload");
  GsBackend* be = dev(p);
  double* med = p->q_aux;
  uint32_t* cnt = reinterpret_cast<uint32_t*>(p->q_aux + GS_MAX_DCS);
  double m[GS_MAX_DCS];
  const bool okk = (!servers || be->h2d_async(p->q_val, servers, count * 4)) &&
                   be->coord_dist_from(p->d, p->g_dev, p->g, p->now, from, servers ? p->q_val : nullptr, (uint32_t)count,
                                       true, p->q_key, p->q_val) &&
                   be->sort_pairs(p->g, p->q_key, p->q_val, (uint32_t)count, n_dcs) &&
                   be->dc_medians(p->g, p->q_key, p->q_val, (uint32_t)count, n_dcs, med, cnt) &&
                   be->d2h(m, med, (size_t)n_dcs * 8);
  if (!okk) return fail(p, GSIM_ERR_CUDA, "dcs_by_distance");
  uint32_t ord[GS_MAX_DCS];
  for (uint32_t c = 0; c < n_dcs; ++c) ord[c] = c;
  std::stable_sort(ord, ord + n_dcs, [&](uint32_t a, uint32_t b) { return m[a] < m[b]; });
  for (uint32_t c = 0; c < n_dcs; ++c) {
    dc_order[c] = ord[c];
    dc_rtt[c] = m[ord[c]];
  }
  return GSIM_OK;
}

// How well the embedding predicts the model's round trips (SURVEY §8f N3): over the draws k < n_draws of
// philox(seed; k, salt, GS_PUR_COORD_SAMPLE) = (x, y, ..), the pairs (x mod n, y mod n) of two different running
// members; out = {pairs kept, mean, p50, p90, p99, max} of |ComputeDistance - true| / true (gs_query.h).
extern "C" int gsim_coordinate_error(gsim_pool* p, uint32_t n_draws, uint32_t salt, double out[6]) {
  if (!p || !out) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GS_CONTROLLER_ONLY(p);
  int rc = coord_query_check(p);
  if (rc) return rc;
  if (n_draws == 0u || n_draws > p->g.cap) return fail(p, GSIM_ERR_INVALID, "n_draws must be in [1, capacity]");
  if (!p->g.n) return fail(p, GSIM_ERR_STATE, "the pool has no members");
  if (!query_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "query buffers");
  if (!upload_globals(p)) return fail(p, GSIM_ERR_CUDA, "upload");
  double* dout = p->q_aux + query_aux_small(p);
  if (!dev(p)->coord_error(p->d, p->g_dev, p->g, p->now, n_draws, salt, p->q_key, p->q_val, p->q_aux, dout) ||
      !dev(p)->d2h(out, dout, 6 * sizeof(double)))
    return fail(p, GSIM_ERR_CUDA, "coordinate_error");
  return GSIM_OK;
}

// Turn event logging for one member on or off after creation (gsim_member_desc.flags does it at
// creation): the EventCh of that agent, polled through gsim_poll_events.
extern "C" int gsim_member_watch(gsim_pool* p, uint32_t id, int on) {
  if (!p) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  return controller_call(p, nullptr, 0, [&]() -> int {
  if (id >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  uint32_t m;
  if (!peek(p, p->d.meta, id, &m)) return fail(p, GSIM_ERR_CUDA, "peek");
  m = on ? (m | GS_META_WATCHED) : (m & ~GS_META_WATCHED);
  if (!poke(p, p->d.meta, id, m)) return fail(p, GSIM_ERR_CUDA, "poke");
  return GSIM_OK;
  });
}

// ---- degraded members (DESIGN.md §3) -------------------------------------------------------
// Loss in ppm -> the Philox threshold (the rule of packet_loss_ppm), and back: thr = floor(ppm 2^32 / 1e6)
// is one-to-one because 2^32 / 1e6 > 1, so ppm = ceil(thr 1e6 / 2^32).
static uint32_t ppm_to_thr(uint32_t ppm) {
  return ppm >= 1000000u ? 0xFFFFFFFFu : (uint32_t)(((uint64_t)ppm << 32) / 1000000ull);
}
static uint32_t thr_to_ppm(uint32_t thr) { return (uint32_t)(((uint64_t)thr * 1000000ull + 0xFFFFFFFFull) >> 32); }

// largest extra one-way latency of the datacenter matrix (0 without one)
static uint32_t max_dc_extra(const GsGlobals& g) {
  uint32_t m = 0;
  for (uint32_t a = 0; a < g.n_dcs; ++a)
    for (uint32_t b = 0; b < g.n_dcs; ++b) m = g.lat[a * GS_MAX_DCS + b] > m ? g.lat[a * GS_MAX_DCS + b] : m;
  return m;
}

static bool impair_max_delay(gsim_pool* p, uint32_t* out) {
  *out = 0;
  if (!p->imp_delay || !p->g.n) return true;
  std::vector<uint8_t> v(p->g.n);
  if (!dev(p)->d2h(v.data(), p->imp_delay, v.size())) return false;
  for (uint8_t x : v) *out = x > *out ? x : *out;
  return true;
}

static bool impair_alloc(gsim_pool* p) {
  if (p->imp_loss) return true;
  const size_t cap = p->g.cap;
  uint32_t* loss = nullptr;
  uint8_t* delay = nullptr;
  if (!alloc_col(p, &loss, cap) || !alloc_col(p, &delay, cap)) return false;
  if (!dev(p)->fill32(loss, 0, cap) || !dev(p)->fill8(delay, 0, cap)) return false;
  p->imp_loss = loss;
  p->imp_delay = delay;
  return true;
}

// The receive-threshold and flag columns, the receive thresholds a copy of the send thresholds (the
// impairment columns exist already).
static bool reach_alloc(gsim_pool* p) {
  if (p->imp_recv) return true;
  const size_t cap = p->g.cap;
  uint32_t* recv = nullptr;
  uint8_t* flags = nullptr;
  if (!alloc_col(p, &recv, cap) || !alloc_col(p, &flags, cap)) return false;
  std::vector<uint32_t> loss(cap);
  if (!dev(p)->d2h(loss.data(), p->imp_loss, cap * 4) || !dev(p)->h2d(recv, loss.data(), cap * 4) ||
      !dev(p)->fill8(flags, 0, cap))
    return false;
  p->imp_recv = recv;
  p->imp_flags = flags;
  return true;
}

// The kernels see the columns only while somebody is impaired: with none, every path (fast paths, long
// windows, closed form) is exactly the one of a pool that never was.
static void impair_publish(gsim_pool* p) {
  p->d.imp_loss = p->n_impaired ? p->imp_loss : nullptr;
  p->d.imp_delay = p->n_impaired ? p->imp_delay : nullptr;
  p->d.imp_recv = p->n_impaired ? (p->imp_recv ? p->imp_recv : p->imp_loss) : nullptr;
  p->d.imp_flags = p->n_impaired ? p->imp_flags : nullptr;
  p->d.imp_flap = p->n_impaired && p->n_flap ? p->imp_flap : nullptr;
  const bool dom_on = p->n_impaired && p->n_dom_sched;
  p->d.imp_dom = dom_on ? p->imp_dom : nullptr;
  p->d.dom_flap = dom_on ? p->dom_tab_dev : nullptr;
  p->d.dom_flap_n = dom_on ? (uint32_t)p->dom_tab.size() : 0u;
  mark_dirty(p);
}

// a member is impaired when any of its four values is non-zero
static bool impair_recount(gsim_pool* p) {
  p->n_impaired = 0;
  if (p->imp_loss && p->g.n) {
    std::vector<uint32_t> loss(p->g.n), recv(p->imp_recv ? p->g.n : 0u);
    std::vector<uint8_t> delay(p->g.n), flags(p->imp_recv ? p->g.n : 0u);
    if (!dev(p)->d2h(loss.data(), p->imp_loss, loss.size() * 4) || !dev(p)->d2h(delay.data(), p->imp_delay, delay.size()))
      return false;
    if (p->imp_recv && (!dev(p)->d2h(recv.data(), p->imp_recv, recv.size() * 4) ||
                        !dev(p)->d2h(flags.data(), p->imp_flags, flags.size())))
      return false;
    for (uint32_t i = 0; i < p->g.n; ++i)
      p->n_impaired += (loss[i] | delay[i] | (p->imp_recv ? recv[i] | flags[i] : 0u)) != 0u ? 1u : 0u;
  }
  impair_publish(p);
  return true;
}

static int impair_check(gsim_pool* p, uint32_t loss_ppm, uint32_t delay_ticks, uint32_t recv_ppm = 0u,
                        uint32_t flags = 0u) {
  if (p->sharded) return fail(p, GSIM_ERR_STATE, "member impairment is not supported on sharded pools");
  if (loss_ppm > 1000000u || recv_ppm > 1000000u) return fail(p, GSIM_ERR_INVALID, "loss_ppm must be <= 1000000");
  if (flags & ~(uint32_t)GSIM_IMPAIR_NO_TCP) return fail(p, GSIM_ERR_INVALID, "unknown impairment flag");
  // a packet to the member arrives 1 + extra + delay ticks after it was sent: that slot must not wrap the ring
  if ((uint64_t)max_dc_extra(p->g) + delay_ticks + 2u > (uint64_t)p->g.ring_mask + 1u)
    return fail(p, GSIM_ERR_INVALID, "latency plus receive delay must stay below mailbox_depth - 1 extra ticks");
  return GSIM_OK;
}

// gsim_impair_many and gsim_impair_dir_many: setting v (thresholds) for the listed members.  A symmetric
// setting on a pool without the reachability columns touches the two columns it always had.
static int impair_set_many(gsim_pool* p, const uint32_t* ids, size_t n, const GsImpairVal& v) {
  for (size_t x = 0; x < n; ++x)
    if (ids[x] >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  const bool now_impaired = (v.send | v.recv | v.delay | v.flags) != 0u;
  if (!p->imp_loss && !now_impaired) return GSIM_OK;  // clearing on a pool that never was impaired
  if (!impair_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "impairment columns");
  if (n && (v.recv != v.send || v.flags != 0u) && !reach_alloc(p))
    return fail(p, GSIM_ERR_NOMEM, "reachability columns");
  for (size_t x = 0; x < n; ++x) {
    uint32_t old_loss, old_recv = 0u;
    uint8_t old_delay, old_flags = 0u;
    if (!peek(p, p->imp_loss, ids[x], &old_loss) || !peek(p, p->imp_delay, ids[x], &old_delay))
      return fail(p, GSIM_ERR_CUDA, "peek");
    if (p->imp_recv && (!peek(p, p->imp_recv, ids[x], &old_recv) || !peek(p, p->imp_flags, ids[x], &old_flags)))
      return fail(p, GSIM_ERR_CUDA, "peek");
    const bool was = (old_loss | old_delay | old_recv | old_flags) != 0u;
    if (!poke(p, p->imp_loss, ids[x], v.send) || !poke(p, p->imp_delay, ids[x], (uint8_t)v.delay))
      return fail(p, GSIM_ERR_CUDA, "poke");
    if (p->imp_recv && (!poke(p, p->imp_recv, ids[x], v.recv) || !poke(p, p->imp_flags, ids[x], (uint8_t)v.flags)))
      return fail(p, GSIM_ERR_CUDA, "poke");
    p->n_impaired = p->n_impaired - (was ? 1u : 0u) + (now_impaired ? 1u : 0u);
  }
  impair_publish(p);
  return GSIM_OK;
}

// gsim_impair_fraction and gsim_impair_dir_fraction: the selection of gs_impair_row, one backend call.
static int impair_set_fraction(gsim_pool* p, uint32_t member_ppm, uint32_t salt, const GsImpairVal& v,
                               uint32_t* n_impaired) {
  if (!impair_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "impairment columns");
  if ((v.recv != v.send || v.flags != 0u) && !reach_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "reachability columns");
  if (!upload_globals(p)) return fail(p, GSIM_ERR_CUDA, "upload");
  uint32_t counts[2] = {0, 0};
  const GsImpairCols c = {p->imp_loss, p->imp_recv, p->imp_delay, p->imp_flags};
  if (!dev(p)->impair_dir_fraction(p->d, p->g_dev, p->g, c, ppm_to_thr(member_ppm), salt, v, counts))
    return fail(p, GSIM_ERR_CUDA, "impair_fraction");
  p->n_impaired = p->n_impaired - counts[1] + ((v.send | v.recv | v.delay | v.flags) != 0u ? counts[0] : 0u);
  if (n_impaired) *n_impaired = counts[0];
  impair_publish(p);
  return GSIM_OK;
}

extern "C" int gsim_impair_many(gsim_pool* p, const uint32_t* ids, size_t n, uint32_t loss_ppm, uint32_t delay_ticks) {
  if (!p || (!ids && n)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  int rc = impair_check(p, loss_ppm, delay_ticks);
  if (rc) return rc;
  const uint32_t thr = ppm_to_thr(loss_ppm);
  return impair_set_many(p, ids, n, GsImpairVal{thr, thr, delay_ticks, 0u});
}

extern "C" int gsim_impair_dir_many(gsim_pool* p, const uint32_t* ids, size_t n, uint32_t send_loss_ppm,
                                    uint32_t recv_loss_ppm, uint32_t delay_ticks, uint32_t flags) {
  if (!p || (!ids && n)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  int rc = impair_check(p, send_loss_ppm, delay_ticks, recv_loss_ppm, flags);
  if (rc) return rc;
  return impair_set_many(p, ids, n, GsImpairVal{ppm_to_thr(send_loss_ppm), ppm_to_thr(recv_loss_ppm), delay_ticks, flags});
}

extern "C" int gsim_impair_fraction(gsim_pool* p, uint32_t member_ppm, uint32_t salt, uint32_t loss_ppm,
                                    uint32_t delay_ticks, uint32_t* n_impaired) {
  if (!p || member_ppm > 1000000u) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  int rc = impair_check(p, loss_ppm, delay_ticks);
  if (rc) return rc;
  const uint32_t thr = ppm_to_thr(loss_ppm);
  return impair_set_fraction(p, member_ppm, salt, GsImpairVal{thr, thr, delay_ticks, 0u}, n_impaired);
}

extern "C" int gsim_impair_dir_fraction(gsim_pool* p, uint32_t member_ppm, uint32_t salt, uint32_t send_loss_ppm,
                                        uint32_t recv_loss_ppm, uint32_t delay_ticks, uint32_t flags,
                                        uint32_t* n_impaired) {
  if (!p || member_ppm > 1000000u) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  int rc = impair_check(p, send_loss_ppm, delay_ticks, recv_loss_ppm, flags);
  if (rc) return rc;
  return impair_set_fraction(p, member_ppm, salt,
                             GsImpairVal{ppm_to_thr(send_loss_ppm), ppm_to_thr(recv_loss_ppm), delay_ticks, flags},
                             n_impaired);
}

// the four values of member `id` (thresholds), all zero on a pool that never was impaired
static int impair_read(gsim_pool* p, uint32_t id, GsImpairVal* v) {
  if (id >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  uint8_t delay = 0, flags = 0;
  *v = GsImpairVal{0u, 0u, 0u, 0u};
  if (p->imp_loss && (!peek(p, p->imp_loss, id, &v->send) || !peek(p, p->imp_delay, id, &delay)))
    return fail(p, GSIM_ERR_CUDA, "peek");
  v->recv = v->send;
  if (p->imp_recv && (!peek(p, p->imp_recv, id, &v->recv) || !peek(p, p->imp_flags, id, &flags)))
    return fail(p, GSIM_ERR_CUDA, "peek");
  v->delay = delay;
  v->flags = flags;
  return GSIM_OK;
}

extern "C" int gsim_impair_get(gsim_pool* p, uint32_t id, uint32_t* loss_ppm, uint32_t* delay_ticks) {
  if (!p) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GsImpairVal v;
  if (int rc = impair_read(p, id, &v)) return rc;
  if (v.recv != v.send || v.flags != 0u)
    return fail(p, GSIM_ERR_STATE, "the member's impairment is directional: use gsim_impair_dir_get");
  if (loss_ppm) *loss_ppm = thr_to_ppm(v.send);
  if (delay_ticks) *delay_ticks = v.delay;
  return GSIM_OK;
}

extern "C" int gsim_impair_dir_get(gsim_pool* p, uint32_t id, uint32_t* send_loss_ppm, uint32_t* recv_loss_ppm,
                                   uint32_t* delay_ticks, uint32_t* flags) {
  if (!p) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GsImpairVal v;
  if (int rc = impair_read(p, id, &v)) return rc;
  if (send_loss_ppm) *send_loss_ppm = thr_to_ppm(v.send);
  if (recv_loss_ppm) *recv_loss_ppm = thr_to_ppm(v.recv);
  if (delay_ticks) *delay_ticks = v.delay;
  if (flags) *flags = v.flags;
  return GSIM_OK;
}

// ---- intermittent impairment (DESIGN.md §3.5 "Intermittent impairment") ----------------------------
extern "C" int gsim_flap_bad(uint64_t seed, uint32_t member, uint32_t period_ticks, uint32_t bad_ppm, uint32_t tick) {
  if (period_ticks == 0u) return 1;  // no schedule: the impairment is always in force
  if (period_ticks > GS_FLAP_MAX_PERIOD || bad_ppm > 1000000u) return GSIM_ERR_INVALID;
  return gs_flap_bad((uint32_t)seed, (uint32_t)(seed >> 32), member, gs_flap_word(period_ticks, bad_ppm), tick) ? 1 : 0;
}

static int flap_check(gsim_pool* p, uint32_t period_ticks, uint32_t bad_ppm) {
  if (p->sharded) return fail(p, GSIM_ERR_STATE, "intermittent impairment is not supported on sharded pools");
  if (period_ticks > GS_FLAP_MAX_PERIOD) return fail(p, GSIM_ERR_INVALID, "period_ticks must be <= 4095");
  if (bad_ppm > 1000000u) return fail(p, GSIM_ERR_INVALID, "bad_ppm must be <= 1000000");
  return GSIM_OK;
}

static bool flap_alloc(gsim_pool* p) {
  if (p->imp_flap) return true;
  uint32_t* col = nullptr;
  if (!alloc_col(p, &col, p->g.cap) || !dev(p)->fill32(col, 0u, p->g.cap)) return false;
  p->imp_flap = col;
  return true;
}

// members with a schedule, counted from the column (after a restore)
static bool flap_recount(gsim_pool* p) {
  p->n_flap = 0;
  if (p->imp_flap && p->g.n) {
    std::vector<uint32_t> col(p->g.n);
    if (!dev(p)->d2h(col.data(), p->imp_flap, col.size() * 4)) return false;
    for (uint32_t w : col) p->n_flap += w != 0u ? 1u : 0u;
  }
  impair_publish(p);
  return true;
}

static uint32_t flap_word_of(uint32_t period_ticks, uint32_t bad_ppm) {
  return period_ticks ? gs_flap_word(period_ticks, bad_ppm) : 0u;
}

extern "C" int gsim_impair_flap_many(gsim_pool* p, const uint32_t* ids, size_t n, uint32_t period_ticks,
                                     uint32_t bad_ppm) {
  if (!p || (!ids && n)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (int rc = flap_check(p, period_ticks, bad_ppm)) return rc;
  for (size_t x = 0; x < n; ++x)
    if (ids[x] >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  const uint32_t w = flap_word_of(period_ticks, bad_ppm);
  if (!p->imp_flap && w == 0u) return GSIM_OK;  // clearing on a pool that never had a schedule
  if (!flap_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "schedule column");
  for (size_t x = 0; x < n; ++x) {
    uint32_t old;
    if (!peek(p, p->imp_flap, ids[x], &old)) return fail(p, GSIM_ERR_CUDA, "peek");
    if (!poke(p, p->imp_flap, ids[x], w)) return fail(p, GSIM_ERR_CUDA, "poke");
    p->n_flap = p->n_flap - (old != 0u ? 1u : 0u) + (w != 0u ? 1u : 0u);
  }
  impair_publish(p);
  return GSIM_OK;
}

extern "C" int gsim_impair_flap_fraction(gsim_pool* p, uint32_t member_ppm, uint32_t salt, uint32_t period_ticks,
                                         uint32_t bad_ppm, uint32_t* n_selected) {
  if (!p || member_ppm > 1000000u) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (int rc = flap_check(p, period_ticks, bad_ppm)) return rc;
  const uint32_t w = flap_word_of(period_ticks, bad_ppm);
  if (!flap_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "schedule column");
  if (!upload_globals(p)) return fail(p, GSIM_ERR_CUDA, "upload");
  uint32_t counts[2] = {0, 0};
  if (!dev(p)->flap_fraction(p->d, p->g_dev, p->g, p->imp_flap, ppm_to_thr(member_ppm), salt, w, counts))
    return fail(p, GSIM_ERR_CUDA, "flap_fraction");
  p->n_flap = p->n_flap - counts[1] + (w != 0u ? counts[0] : 0u);
  if (n_selected) *n_selected = counts[0];
  impair_publish(p);
  return GSIM_OK;
}

extern "C" int gsim_impair_flap_get(gsim_pool* p, uint32_t id, uint32_t* period_ticks, uint32_t* bad_ppm) {
  if (!p) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (p->sharded) return fail(p, GSIM_ERR_STATE, "intermittent impairment is not supported on sharded pools");
  if (id >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  uint32_t w = 0u;
  if (p->imp_flap && !peek(p, p->imp_flap, id, &w)) return fail(p, GSIM_ERR_CUDA, "peek");
  if (period_ticks) *period_ticks = w >> GS_FLAP_PPM_BITS;
  if (bad_ppm) *bad_ppm = w & ((1u << GS_FLAP_PPM_BITS) - 1u);
  return GSIM_OK;
}

extern "C" int gsim_impair_flap_stats(gsim_pool* p, uint64_t out[2]) {
  if (!p || !out) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (p->sharded) return fail(p, GSIM_ERR_STATE, "intermittent impairment is not supported on sharded pools");
  out[0] = out[1] = 0u;
  if (!p->imp_flap) return GSIM_OK;
  if (!dev(p)->flap_stats(p->g, p->imp_flap, p->now, out)) return fail(p, GSIM_ERR_CUDA, "flap_stats");
  return GSIM_OK;
}

// ---- paused members (DESIGN.md §3.6) ---------------------------------------------------------
// The backend defaults (gs_backend.h): the columns gs_pause_row and gs_resume_row touch, copied to the host
// behind a GsDev of host pointers, stepped there and copied back.
namespace {
struct HostRows {
  std::vector<uint32_t> key0, key1, meta, due, inbox, pause;
  std::vector<uint8_t> kst;
  GsDev d;
  uint32_t slot = 0;
  bool load(GsBackend* be, const GsDev& dd, const GsGlobals& g, const uint32_t* pause_until, uint32_t t) {
    const size_t n = g.n;
    d = dd;
    slot = t & g.ring_mask;
    key0.resize(n), key1.resize(n), meta.resize(n), due.resize(n), inbox.resize(n), pause.resize(n);
    if (!be->d2h(key0.data(), dd.key[0], n * 4) || !be->d2h(key1.data(), dd.key[1], n * 4) ||
        !be->d2h(meta.data(), dd.meta, n * 4) || !be->d2h(due.data(), dd.due, n * 4) ||
        !be->d2h(inbox.data(), dd.inbox[slot], n * 4) || (pause_until && !be->d2h(pause.data(), pause_until, n * 4)))
      return false;
    if (dd.kst) {
      kst.resize(n);
      if (!be->d2h(kst.data(), dd.kst, n)) return false;
      d.kst = kst.data();
    }
    d.key[0] = d.key_rep[0] = key0.data();
    d.key[1] = d.key_rep[1] = key1.data();
    d.meta = meta.data();
    d.due = due.data();
    d.inbox[slot] = inbox.data();
    return true;
  }
  bool store(GsBackend* be, const GsDev& dd, const GsGlobals& g, uint32_t* pause_until) {
    const size_t n = g.n;
    return be->h2d(dd.key[0], key0.data(), n * 4) && be->h2d(dd.key[1], key1.data(), n * 4) &&
           be->h2d(dd.meta, meta.data(), n * 4) && be->h2d(dd.due, due.data(), n * 4) &&
           be->h2d(dd.inbox[slot], inbox.data(), n * 4) && (!pause_until || be->h2d(pause_until, pause.data(), n * 4)) &&
           (!dd.kst || be->h2d(dd.kst, kst.data(), n));
  }
};
}  // namespace

bool GsBackend::pause_rows(const GsDev& d, const GsGlobals*, const GsGlobals& g, uint32_t* pause_until,
                           const uint32_t* ids, uint32_t n, uint32_t thr, uint32_t salt, uint32_t until,
                           uint32_t* n_paused) {
  *n_paused = 0;
  if (!g.n) return true;
  HostRows h;
  if (!h.load(this, d, g, pause_until, 0u)) return false;
  if (ids) {
    for (uint32_t x = 0; x < n; ++x) *n_paused += gs_pause_row(h.d, g, h.pause.data(), ids[x], until) ? 1u : 0u;
  } else {
    for (uint32_t i = 0; i < g.n; ++i)
      if (gs_pause_pick(g, i, thr, salt)) *n_paused += gs_pause_row(h.d, g, h.pause.data(), i, until) ? 1u : 0u;
  }
  return h.store(this, d, g, pause_until);
}

bool GsBackend::resume_rows(const GsDev& d, const GsGlobals*, const GsGlobals& g, uint32_t* pause_until, uint32_t t,
                            bool resume, bool log_events, uint32_t counts[4]) {
  counts[0] = counts[1] = counts[2] = counts[3] = 0u;
  if (!g.n) return true;
  HostRows h;
  if (!h.load(this, d, g, pause_until, t)) return false;
  std::vector<uint32_t> back_from_dead;
  for (uint32_t i = 0; i < g.n; ++i) {
    const uint32_t r = gs_resume_row(h.d, g, h.pause.data(), i, t, resume);
    if (r) counts[r - 1u]++;
    if (r == GS_RESUMED_DEAD && log_events) back_from_dead.push_back(i);
  }
  if (!h.store(this, d, g, pause_until)) return false;
  if (back_from_dead.empty()) return true;
  uint32_t cur[2];
  if (!d2h(cur, d.evlog_cursor, 8)) return false;
  for (uint32_t i : back_from_dead) {
    if (cur[0] < g.evlog_cap) {
      const GsEventRec e = {t, GS_EV_MEMBER_JOIN, i, GS_EMPTY32, 0u, 0u};
      if (!h2d(d.evlog + cur[0], &e, sizeof(e))) return false;
      cur[0]++;
    } else {
      cur[1]++;
    }
  }
  return h2d(d.evlog_cursor, cur, 8);
}

static bool pause_alloc(gsim_pool* p) {
  if (p->pause_until) return true;
  uint32_t* col = nullptr;
  uint64_t* cnt = nullptr;
  if (!alloc_col(p, &col, p->g.cap) || !alloc_col(p, &cnt, 4)) return false;
  if (!dev(p)->fill32(col, 0u, p->g.cap) || !dev(p)->fill32(reinterpret_cast<uint32_t*>(cnt), 0u, 8)) return false;
  p->pause_until = col;
  p->pause_cnt_dev = cnt;
  return true;
}

static int pause_check(gsim_pool* p, uint32_t ticks) {
  if (p->sharded) return fail(p, GSIM_ERR_STATE, "pausing members is not supported on sharded pools");
  if (ticks == 0u) return fail(p, GSIM_ERR_INVALID, "ticks must be >= 1");
  if (ticks >= GS_NEVER - p->now) return fail(p, GSIM_ERR_INVALID, "the resume tick must fit in 32 bits");
  return GSIM_OK;
}

static int pause_done(gsim_pool* p, uint32_t until, uint32_t k, uint32_t* n_paused);

// The selected members (ids[0..n), or the draw below thr) stop now and resume at now + ticks: one resume
// entry in the schedule per distinct tick, which also makes gsim_step end its chunks (windows, tick
// stretches) there.
static int pause_run(gsim_pool* p, const uint32_t* ids, uint32_t n, uint32_t thr, uint32_t salt, uint32_t ticks,
                     uint32_t* n_paused) {
  if (!pause_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "pause column");
  if (!upload_globals(p)) return fail(p, GSIM_ERR_CUDA, "upload");
  mark_dirty(p);
  const uint32_t until = p->now + ticks;
  uint32_t k = 0;
  if (!dev(p)->pause_rows(p->d, p->g_dev, p->g, p->pause_until, ids, n, thr, salt, until, &k))
    return fail(p, GSIM_ERR_CUDA, "pause_rows");
  return pause_done(p, until, k, n_paused);
}

// After k members were paused until tick `until`: the counts, the resume entry and the recount.
static int pause_done(gsim_pool* p, uint32_t until, uint32_t k, uint32_t* n_paused) {
  *n_paused = k;
  if (!k) return GSIM_OK;
  p->pause_cnt[0] += k;
  bool have = false;
  for (const Sched& s : p->sched) have = have || (s.action == 2u && s.tick == until);
  if (!have) p->sched.push_back(Sched{until, 0u, 2u});
  int rc = refresh_after_truth_change(p);
  return rc ? fail(p, rc, "recount") : GSIM_OK;
}

// Tick p->now, before it runs: the members whose pause ends now resume (resume = true), and the pauses of
// members that are gone meanwhile are forgotten.  Returns whether anybody's truth changed.
static int pause_resume(gsim_pool* p, bool resume, bool* any) {
  uint32_t c[4];
  if (!upload_globals(p)) return GSIM_ERR_CUDA;
  mark_dirty(p);
  if (!dev(p)->resume_rows(p->d, p->g_dev, p->g, p->pause_until, p->now, resume,
                           (p->cfg.flags & GSIM_FLAG_LOG_GLOBAL_EVENTS) != 0, c))
    return GSIM_ERR_CUDA;
  p->pause_cnt[0] -= (uint64_t)c[0] + c[1] + c[2] + c[3];
  for (int x = 0; x < 3; ++x) p->pause_cnt[1 + x] += c[x];
  *any = *any || c[0] + c[1] + c[2] != 0u;
  return GSIM_OK;
}

extern "C" int gsim_pause_many(gsim_pool* p, const uint32_t* ids, size_t n, uint32_t ticks, uint32_t* n_paused) {
  if (!p || (!ids && n)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  uint32_t local = 0;
  if (!n_paused) n_paused = &local;
  *n_paused = 0;
  return controller_call(p, n_paused, sizeof(uint32_t), [&]() -> int {
    int rc = pause_check(p, ticks);
    if (rc) return rc;
    std::vector<uint32_t> v(ids, ids + n);
    for (uint32_t id : v)
      if (id >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
    std::sort(v.begin(), v.end());  // (the CUDA kernel takes one row per thread: no id twice)
    v.erase(std::unique(v.begin(), v.end()), v.end());
    if (v.empty()) return GSIM_OK;
    return pause_run(p, v.data(), (uint32_t)v.size(), 0u, 0u, ticks, n_paused);
  });
}

extern "C" int gsim_pause_fraction(gsim_pool* p, uint32_t member_ppm, uint32_t salt, uint32_t ticks,
                                   uint32_t* n_paused) {
  if (!p || member_ppm > 1000000u) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  uint32_t local = 0;
  if (!n_paused) n_paused = &local;
  *n_paused = 0;
  return controller_call(p, n_paused, sizeof(uint32_t), [&]() -> int {
    int rc = pause_check(p, ticks);
    if (rc) return rc;
    return pause_run(p, nullptr, 0u, ppm_to_thr(member_ppm), salt, ticks, n_paused);
  });
}

extern "C" int gsim_pause_get(gsim_pool* p, uint32_t id, uint32_t* resume_tick) {
  if (!p) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (id >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  uint32_t until = 0;
  if (p->pause_until && !peek(p, p->pause_until, id, &until)) return fail(p, GSIM_ERR_CUDA, "peek");
  if (resume_tick) *resume_tick = until ? until : 0xFFFFFFFFu;
  return GSIM_OK;
}

extern "C" int gsim_pause_stats(gsim_pool* p, uint64_t out[4]) {
  if (!p || !out) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  memcpy(out, p->pause_cnt, sizeof(p->pause_cnt));
  return GSIM_OK;
}

// ---- fault domains (DESIGN.md §3.5 "Fault domains") -------------------------------------------------
// The backend defaults (gs_backend.h): the columns the rows read and write, copied to the host, stepped there
// and copied back.
bool GsBackend::domain_range(uint32_t* dom, uint32_t first, uint32_t count, uint32_t per_domain, uint32_t first_domain) {
  if (!count) return true;
  std::vector<uint32_t> v(count);
  for (uint32_t x = 0; x < count; ++x) v[x] = first_domain + x / per_domain;
  return h2d(dom + first, v.data(), (size_t)count * 4);
}

bool GsBackend::domain_rows(const GsDev& d, const GsGlobals*, const GsGlobals& g, const uint32_t* dom,
                            const uint32_t* bits, uint32_t n_words, const GsDomainOp& a, uint32_t counts[2]) {
  counts[0] = counts[1] = 0u;
  if (!g.n) return true;
  std::vector<uint32_t> dc(g.n);
  if (!d2h(dc.data(), dom, (size_t)g.n * 4)) return false;
  GsDomainOp ha = a;
  HostRows h;
  std::vector<uint32_t> lc, rc;
  std::vector<uint8_t> delay, fc;
  if (a.op == GS_DOMAIN_OP_IMPAIR) {
    lc.resize(g.n), delay.resize(g.n), rc.resize(a.imp.recv ? g.n : 0u), fc.resize(a.imp.flags ? g.n : 0u);
    if (!d2h(lc.data(), a.imp.loss, (size_t)g.n * 4) || !d2h(delay.data(), a.imp.delay, g.n) ||
        (a.imp.recv && !d2h(rc.data(), a.imp.recv, (size_t)g.n * 4)) || (a.imp.flags && !d2h(fc.data(), a.imp.flags, g.n)))
      return false;
    ha.imp = {lc.data(), a.imp.recv ? rc.data() : nullptr, delay.data(), a.imp.flags ? fc.data() : nullptr};
  } else if (a.op != GS_DOMAIN_OP_COUNT) {
    if (!h.load(this, d, g, a.pause_until, 0u)) return false;
    ha.pause_until = a.pause_until ? h.pause.data() : nullptr;
  }
  for (uint32_t i = 0; i < g.n; ++i) {
    if (!gs_domain_listed(dc.data(), bits, n_words, i)) continue;
    const uint32_t r = gs_domain_op_row(h.d, g, ha, i);
    counts[0] += r & 1u;
    counts[1] += (r >> 1) & 1u;
  }
  if (a.op == GS_DOMAIN_OP_IMPAIR)
    return h2d(a.imp.loss, lc.data(), (size_t)g.n * 4) && h2d(a.imp.delay, delay.data(), g.n) &&
           (!a.imp.recv || h2d(a.imp.recv, rc.data(), (size_t)g.n * 4)) && (!a.imp.flags || h2d(a.imp.flags, fc.data(), g.n));
  return a.op == GS_DOMAIN_OP_COUNT || h.store(this, d, g, a.pause_until);
}

bool GsBackend::domain_stats(const GsDev& d, const GsGlobals& g, const GsDomainCols& c, uint32_t now,
                             uint32_t first_domain, uint32_t count, GsDomainStats* out) {
  memset(out, 0, (size_t)count * sizeof(GsDomainStats));
  if (!g.n || !count) return true;
  const size_t n = g.n;
  std::vector<uint32_t> key(n), meta(n), dom(n), pause(c.pause_until ? n : 0u), loss(c.imp.loss ? n : 0u),
      recv(c.imp.recv ? n : 0u);
  std::vector<uint8_t> delay(c.imp.delay ? n : 0u), flags(c.imp.flags ? n : 0u);
  if (!d2h(key.data(), c.key, n * 4) || !d2h(meta.data(), c.meta, n * 4) || !d2h(dom.data(), c.dom, n * 4) ||
      (c.pause_until && !d2h(pause.data(), c.pause_until, n * 4)) || (c.imp.loss && !d2h(loss.data(), c.imp.loss, n * 4)) ||
      (c.imp.recv && !d2h(recv.data(), c.imp.recv, n * 4)) || (c.imp.delay && !d2h(delay.data(), c.imp.delay, n)) ||
      (c.imp.flags && !d2h(flags.data(), c.imp.flags, n)))
    return false;
  HostCoords hc;  // the published schedule columns gs_imp_in_force reads
  hc.d = d;
  if (d.imp_flap) {
    hc.flap.resize(g.cap);
    if (!d2h(hc.flap.data(), d.imp_flap, (size_t)g.cap * 4)) return false;
    hc.d.imp_flap = hc.flap.data();
  }
  if (d.dom_flap) {
    hc.dom_flap.resize(d.dom_flap_n);
    if (!d2h(hc.dom_flap.data(), d.dom_flap, (size_t)d.dom_flap_n * 4)) return false;
    hc.d.imp_dom = dom.data();
    hc.d.dom_flap = hc.dom_flap.data();
  }
  const GsDomainCols h = {key.data(), meta.data(), dom.data(), c.pause_until ? pause.data() : nullptr,
                          {c.imp.loss ? loss.data() : nullptr, c.imp.recv ? recv.data() : nullptr,
                           c.imp.delay ? delay.data() : nullptr, c.imp.flags ? flags.data() : nullptr}};
  for (uint32_t i = 0; i < g.n; ++i) {
    const uint32_t x = dom[i] - first_domain;
    uint32_t v[3];
    if (x >= count || !gs_domain_stats_row(hc.d, g.seed_lo, g.seed_hi, h, i, now, v)) continue;
    gs_domain_stats_add(out[x], v, v[2]);
  }
  return true;
}

static_assert(sizeof(GsDomainStats) == sizeof(gsim_domain_stats), "GsDomainStats is gsim_domain_stats field for field");

static int domain_sharded(gsim_pool* p) {
  return fail(p, GSIM_ERR_STATE, "fault domains are not supported on sharded pools");
}

static bool domain_alloc(gsim_pool* p) {
  if (p->imp_dom) return true;
  uint32_t* col = nullptr;
  if (!alloc_col(p, &col, p->g.cap) || !dev(p)->fill32(col, 0u, p->g.cap)) return false;
  p->imp_dom = col;
  return true;
}

// The device copy of the schedule table, reallocated when the table outgrows it.
static bool domain_tab_upload(gsim_pool* p) {
  if (p->dom_tab.size() > p->dom_tab_cap) {
    size_t cap = p->dom_tab_cap ? p->dom_tab_cap : 1024u;
    while (cap < p->dom_tab.size()) cap *= 2u;
    uint32_t* t = nullptr;
    if (!alloc_col(p, &t, cap)) return false;
    if (p->dom_tab_dev) {
      if (!dev(p)->sync()) return false;  // no launch still reads the old copy
      p->allocs.erase(std::find(p->allocs.begin(), p->allocs.end(), (void*)p->dom_tab_dev));
      dev(p)->release(p->dom_tab_dev);
    }
    p->dom_tab_dev = t;
    p->dom_tab_cap = cap;
  }
  p->n_dom_sched = 0;
  for (uint32_t w : p->dom_tab) p->n_dom_sched += w != 0u ? 1u : 0u;
  if (!p->dom_tab.empty() && !dev(p)->h2d(p->dom_tab_dev, p->dom_tab.data(), p->dom_tab.size() * 4)) return false;
  impair_publish(p);
  return true;
}

// A domain list: every id in 1 .. GS_DOMAIN_MAX, as a bitmap (bit x & 31 of word x >> 5).
static int domain_bits(gsim_pool* p, const uint32_t* domains, size_t n, std::vector<uint32_t>* bits) {
  uint32_t hi = 0;
  for (size_t x = 0; x < n; ++x) {
    if (domains[x] == 0u || domains[x] > GS_DOMAIN_MAX) return fail(p, GSIM_ERR_INVALID, "domain ids are 1 .. GSIM_DOMAIN_MAX");
    hi = std::max(hi, domains[x]);
  }
  bits->assign(n ? hi / 32u + 1u : 0u, 0u);
  for (size_t x = 0; x < n; ++x) (*bits)[domains[x] >> 5] |= 1u << (domains[x] & 31u);
  return GSIM_OK;
}

// One domain operation over the members of the listed domains (none on a pool without a domain column).
static int domain_run(gsim_pool* p, const std::vector<uint32_t>& bits, const GsDomainOp& a, uint32_t counts[2]) {
  counts[0] = counts[1] = 0u;
  if (!p->imp_dom || bits.empty()) return GSIM_OK;
  if (!upload_globals(p)) return fail(p, GSIM_ERR_CUDA, "upload");
  if (a.op != GS_DOMAIN_OP_COUNT) mark_dirty(p);
  if (!dev(p)->domain_rows(p->d, p->g_dev, p->g, p->imp_dom, bits.data(), (uint32_t)bits.size(), a, counts))
    return fail(p, GSIM_ERR_CUDA, "domain_rows");
  return GSIM_OK;
}

extern "C" int gsim_domain_set_many(gsim_pool* p, const uint32_t* ids, size_t n, uint32_t domain) {
  if (!p || (!ids && n)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (p->sharded) return domain_sharded(p);
  if (domain > GS_DOMAIN_MAX) return fail(p, GSIM_ERR_INVALID, "domain must be <= GSIM_DOMAIN_MAX");
  for (size_t x = 0; x < n; ++x)
    if (ids[x] >= p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  if (!domain_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "domain column");
  for (size_t x = 0; x < n; ++x)
    if (!poke(p, p->imp_dom, ids[x], domain)) return fail(p, GSIM_ERR_CUDA, "poke");
  mark_dirty(p);
  return GSIM_OK;
}

extern "C" int gsim_domain_set_range(gsim_pool* p, uint32_t first, uint32_t count, uint32_t per_domain,
                                     uint32_t first_domain) {
  if (!p) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (p->sharded) return domain_sharded(p);
  if (per_domain == 0u) return fail(p, GSIM_ERR_INVALID, "per_domain must be >= 1");
  if (first_domain == 0u || (count && (uint64_t)first_domain + (count - 1u) / per_domain > GS_DOMAIN_MAX))
    return fail(p, GSIM_ERR_INVALID, "the domains must lie in 1 .. GSIM_DOMAIN_MAX");
  if ((uint64_t)first + count > p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  if (!domain_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "domain column");
  if (!dev(p)->domain_range(p->imp_dom, first, count, per_domain, first_domain)) return fail(p, GSIM_ERR_CUDA, "domain_range");
  mark_dirty(p);
  return GSIM_OK;
}

extern "C" int gsim_domain_get(gsim_pool* p, uint32_t first, uint32_t count, uint32_t* out) {
  if (!p || (!out && count)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (p->sharded) return domain_sharded(p);
  if ((uint64_t)first + count > p->g.n) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  if (!p->imp_dom) {
    memset(out, 0, (size_t)count * 4);
    return GSIM_OK;
  }
  if (count && !dev(p)->d2h(out, p->imp_dom + first, (size_t)count * 4)) return fail(p, GSIM_ERR_CUDA, "d2h");
  return GSIM_OK;
}

extern "C" int gsim_domain_flap_set(gsim_pool* p, const uint32_t* domains, size_t n, uint32_t period_ticks,
                                    uint32_t bad_ppm) {
  if (!p || (!domains && n)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (p->sharded) return domain_sharded(p);
  if (int rc = flap_check(p, period_ticks, bad_ppm)) return rc;
  std::vector<uint32_t> bits;
  if (int rc = domain_bits(p, domains, n, &bits)) return rc;
  if (!domain_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "domain column");
  const uint32_t w = flap_word_of(period_ticks, bad_ppm);
  for (size_t x = 0; x < n; ++x) {
    if (domains[x] >= p->dom_tab.size()) {
      if (w == 0u) continue;
      p->dom_tab.resize((size_t)domains[x] + 1u, 0u);
    }
    p->dom_tab[domains[x]] = w;
  }
  if (!domain_tab_upload(p)) return fail(p, GSIM_ERR_NOMEM, "domain schedule table");
  return GSIM_OK;
}

extern "C" int gsim_domain_flap_get(gsim_pool* p, uint32_t domain, uint32_t* period_ticks, uint32_t* bad_ppm) {
  if (!p) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (p->sharded) return domain_sharded(p);
  if (domain == 0u || domain > GS_DOMAIN_MAX) return fail(p, GSIM_ERR_INVALID, "domain ids are 1 .. GSIM_DOMAIN_MAX");
  const uint32_t w = domain < p->dom_tab.size() ? p->dom_tab[domain] : 0u;
  if (period_ticks) *period_ticks = w >> GS_FLAP_PPM_BITS;
  if (bad_ppm) *bad_ppm = w & ((1u << GS_FLAP_PPM_BITS) - 1u);
  return GSIM_OK;
}

extern "C" int gsim_domain_flap_bad(uint64_t seed, uint32_t domain, uint32_t period_ticks, uint32_t bad_ppm,
                                    uint32_t tick) {
  if (domain == 0u || domain > GS_DOMAIN_MAX) return GSIM_ERR_INVALID;
  if (period_ticks == 0u) return 1;  // no schedule: the impairment is always in force
  if (period_ticks > GS_FLAP_MAX_PERIOD || bad_ppm > 1000000u) return GSIM_ERR_INVALID;
  return gs_domain_flap_bad((uint32_t)seed, (uint32_t)(seed >> 32), domain, gs_flap_word(period_ticks, bad_ppm), tick)
             ? 1 : 0;
}

extern "C" int gsim_domain_impair(gsim_pool* p, const uint32_t* domains, size_t n, uint32_t send_loss_ppm,
                                  uint32_t recv_loss_ppm, uint32_t delay_ticks, uint32_t flags, uint32_t* n_members) {
  if (!p || (!domains && n)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (p->sharded) return domain_sharded(p);
  if (int rc = impair_check(p, send_loss_ppm, delay_ticks, recv_loss_ppm, flags)) return rc;
  std::vector<uint32_t> bits;
  if (int rc = domain_bits(p, domains, n, &bits)) return rc;
  const GsImpairVal v = {ppm_to_thr(send_loss_ppm), ppm_to_thr(recv_loss_ppm), delay_ticks, flags};
  const bool now_impaired = (v.send | v.recv | v.delay | v.flags) != 0u;
  uint32_t counts[2] = {0, 0};
  GsDomainOp a = {};
  a.op = GS_DOMAIN_OP_COUNT;
  // gsim_impair_dir_many allocates columns only for a non-empty id list: count the members first where that
  // decides it (clearing on a pool that never was impaired, or a first directional setting)
  if (!p->imp_loss || ((v.recv != v.send || v.flags != 0u) && !p->imp_recv)) {
    if (int rc = domain_run(p, bits, a, counts)) return rc;
    if (n_members) *n_members = counts[0];
    if (!p->imp_loss && !now_impaired) return GSIM_OK;
    if (!impair_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "impairment columns");
    if (counts[0] && (v.recv != v.send || v.flags != 0u) && !reach_alloc(p))
      return fail(p, GSIM_ERR_NOMEM, "reachability columns");
  }
  a.op = GS_DOMAIN_OP_IMPAIR;
  a.imp = {p->imp_loss, p->imp_recv, p->imp_delay, p->imp_flags};
  a.v = v;
  if (int rc = domain_run(p, bits, a, counts)) return rc;
  p->n_impaired = p->n_impaired - counts[1] + (now_impaired ? counts[0] : 0u);
  if (n_members) *n_members = counts[0];
  impair_publish(p);
  return GSIM_OK;
}

extern "C" int gsim_domain_crash(gsim_pool* p, const uint32_t* domains, size_t n, uint32_t* n_crashed) {
  if (!p || (!domains && n)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (p->sharded) return domain_sharded(p);
  std::vector<uint32_t> bits;
  if (int rc = domain_bits(p, domains, n, &bits)) return rc;
  GsDomainOp a = {};
  a.op = GS_DOMAIN_OP_CRASH;
  a.pause_until = p->pause_cnt[0] ? p->pause_until : nullptr;  // (a resume to cancel only while somebody is paused)
  uint32_t counts[2] = {0, 0};
  if (int rc = domain_run(p, bits, a, counts)) return rc;
  p->pause_cnt[0] -= counts[1];
  if (n_crashed) *n_crashed = counts[0];
  int rc = refresh_after_truth_change(p);
  return rc ? fail(p, rc, "recount") : GSIM_OK;
}

extern "C" int gsim_domain_pause(gsim_pool* p, const uint32_t* domains, size_t n, uint32_t ticks, uint32_t* n_paused) {
  if (!p || (!domains && n)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  uint32_t local = 0;
  if (!n_paused) n_paused = &local;
  *n_paused = 0;
  if (p->sharded) return domain_sharded(p);
  if (int rc = pause_check(p, ticks)) return rc;
  std::vector<uint32_t> bits;
  if (int rc = domain_bits(p, domains, n, &bits)) return rc;
  if (!p->imp_dom || bits.empty()) return GSIM_OK;
  if (!pause_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "pause column");
  GsDomainOp a = {};
  a.op = GS_DOMAIN_OP_PAUSE;
  a.pause_until = p->pause_until;
  a.until = p->now + ticks;
  uint32_t counts[2] = {0, 0};
  if (int rc = domain_run(p, bits, a, counts)) return rc;
  return pause_done(p, a.until, counts[0], n_paused);
}

extern "C" int gsim_domain_stats_read(gsim_pool* p, uint32_t first_domain, uint32_t count, gsim_domain_stats* out) {
  if (!p || (!out && count)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (p->sharded) return domain_sharded(p);
  if (first_domain == 0u || (uint64_t)first_domain + count > (uint64_t)GS_DOMAIN_MAX + 1u)
    return fail(p, GSIM_ERR_INVALID, "the domains must lie in 1 .. GSIM_DOMAIN_MAX");
  if (!p->imp_dom) {
    memset(out, 0, (size_t)count * sizeof(gsim_domain_stats));
    return GSIM_OK;
  }
  const GsDomainCols c = {p->d.key[p->now & 1u], p->d.meta, p->imp_dom, p->pause_until,
                          {p->imp_loss, p->imp_recv, p->imp_delay, p->imp_flags}};
  if (!dev(p)->domain_stats(p->d, p->g, c, p->now, first_domain, count, reinterpret_cast<GsDomainStats*>(out)))
    return fail(p, GSIM_ERR_CUDA, "domain_stats");
  return GSIM_OK;
}

// WAN latency pools (BASELINE config 5, SURVEY 8d C5): n_dcs synthetic datacenters, member i
// lives in datacenter (i / 128) % n_dcs; a packet from datacenter a to b takes lat[a*n_dcs+b]
// ticks (>= 1; 1 is the latency every packet has on a pool without a matrix).
extern "C" int gsim_latency_set(gsim_pool* p, uint32_t n_dcs, const uint8_t* lat_ticks) {
  if (!p || n_dcs > GS_MAX_DCS || (n_dcs && !lat_ticks)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  return controller_call(p, nullptr, 0, [&]() -> int {
  GsGlobals& g = p->g;
  uint32_t max_delay = 0;
  if (p->n_impaired && !impair_max_delay(p, &max_delay)) return fail(p, GSIM_ERR_CUDA, "d2h");
  for (uint32_t x = 0; x < n_dcs * n_dcs; ++x)
    if (lat_ticks[x] < 1u || lat_ticks[x] > g.ring_mask)
      return fail(p, GSIM_ERR_INVALID, "latency must be in [1, mailbox_depth - 1] ticks");
    else if (lat_ticks[x] + max_delay > g.ring_mask)
      return fail(p, GSIM_ERR_INVALID, "latency plus the largest receive delay must stay below mailbox_depth");
  memset(g.lat, 0, sizeof(g.lat));
  for (uint32_t a = 0; a < n_dcs; ++a)
    for (uint32_t b = 0; b < n_dcs; ++b) g.lat[a * GS_MAX_DCS + b] = (uint8_t)(lat_ticks[a * n_dcs + b] - 1u);
  g.n_dcs = n_dcs;
  p->g_dirty = true;
  mark_dirty(p);  // what a probe round trip costs has changed
  return GSIM_OK;
  });
}

// ---- time -----------------------------------------------------------------------
static int apply_sched(gsim_pool* p) {
  bool any = false, resume = false;
  for (size_t x = 0; x < p->sched.size();) {
    if (p->sched[x].tick <= p->now) {
      resume = resume || p->sched[x].action == 2u;
      if (p->sched[x].action == 1u) {
        uint32_t k;
        if (!peek(p, p->d.key[p->now & 1u], p->sched[x].id, &k)) return GSIM_ERR_CUDA;
        if (gs_key_truth(k) == GS_TRUTH_UP) {
          int rc = set_truth(p, p->sched[x].id, GS_TRUTH_GONE);
          if (rc) return rc;
          any = true;
        }
      }
      p->sched.erase(p->sched.begin() + x);
    } else {
      ++x;
    }
  }
  if (resume && p->pause_until) {
    int rc = pause_resume(p, true, &any);
    if (rc) return rc;
  }
  if (any) return refresh_after_truth_change(p);
  return GSIM_OK;
}

// Advance `ticks` ticks.  On a sharded pool every rank runs this together: the host-side parts
// (scheduled shutdowns, globals upload, rumor retirement) are controller calls, the tick kernels
// run on every rank with a device barrier after each tick.
// [U] serf.handleReap: every ReapInterval, erase members that have been Failed for longer than
// ReconnectTimeout or Left for longer than TombstoneTimeout (SURVEY 8a row a17).  The reaper's
// ticker fires at ticks that are multiples of ReapInterval; with Consul's production values
// (72 h / 24 h, agent/consul/config.go:622-623) nothing can be old enough within any simulated
// horizon and no pass is ever scheduled — only test timings (server_test.go:675-677) reach it.
struct ReapPlan {
  uint32_t every, reconnect, tombstone;
};
static uint32_t clamp_ticks(uint64_t ns, uint64_t tick) {
  const uint64_t t = (ns + tick - 1) / tick;
  return t > 0xFFFFFFF0ull ? 0xFFFFFFF0u : (uint32_t)t;
}
static ReapPlan reap_plan(const gsim_pool* p) {
  ReapPlan r;
  r.every = p->cfg.reap_interval_ns ? clamp_ticks(p->cfg.reap_interval_ns, p->tick_ns) : 0u;
  r.reconnect = clamp_ticks(p->cfg.reconnect_timeout_ns, p->tick_ns);
  r.tombstone = clamp_ticks(p->cfg.tombstone_timeout_ns, p->tick_ns);
  return r;
}
// first tick > now at which a reap pass can possibly find something, or GS_NEVER
static uint32_t next_reap_tick(const gsim_pool* p, uint32_t now) {
  const ReapPlan r = reap_plan(p);
  if (!r.every) return GS_NEVER;
  uint32_t youngest = r.reconnect < r.tombstone ? r.reconnect : r.tombstone;
  if (p->g.reap_min_override && p->g.reap_min_override < youngest) youngest = p->g.reap_min_override;
  uint64_t t = (uint64_t)(now / r.every + 1u) * r.every;
  if (t <= youngest) t = ((uint64_t)youngest / r.every + 1u) * r.every;  // nobody is that old before
  return t >= GS_NEVER ? GS_NEVER : (uint32_t)t;
}
static int reap_pass(gsim_pool* p) {
  const ReapPlan r = reap_plan(p);
  if (!r.every || p->now == 0 || p->now % r.every != 0) return GSIM_OK;
  uint32_t youngest = r.reconnect < r.tombstone ? r.reconnect : r.tombstone;
  if (p->g.reap_min_override && p->g.reap_min_override < youngest) youngest = p->g.reap_min_override;
  if (p->now <= youngest) return GSIM_OK;
  uint32_t counts[2] = {0, 0};
  if (!upload_globals(p)) return GSIM_ERR_CUDA;
  mark_dirty(p);
  if (!dev(p)->reap_rows(p->d, p->g_dev, p->g, p->now, r.reconnect, r.tombstone,
                        (p->cfg.flags & GSIM_FLAG_LOG_GLOBAL_EVENTS) != 0, counts))
    return GSIM_ERR_CUDA;
  if (!counts[0]) return GSIM_OK;
  p->n_established -= counts[1];
  if (p->pause_cnt[0]) {  // a reaped member that was paused stays gone
    bool any = false;
    int rc = pause_resume(p, false, &any);
    if (rc) return rc;
  }
  return refresh_after_truth_change(p);
}

// ---- quiet-window scheduling (DESIGN.md §4.2) --------------------------------------------------
static bool windows_possible(const gsim_pool* p) {
  static const bool env_off = getenv("GSIM_NO_WINDOWS") != nullptr;
  const GsGlobals& g = p->g;
  // per-tile ticker phases (the window kernel derives a tile's due ticks from its phase), no
  // per-member periodic tickers besides the probe (push-pull), no coordinate exchange on acks
  return !env_off && !(p->cfg.flags & GSIM_FLAG_NO_WINDOWS) && g.phase_gate != 0u && g.pp_interval == 0u &&
         p->d.coord == nullptr && g.P >= 2u && g.T < g.P && g.n != 0u;
}

#define GS_LONG_WINDOW 32u  // ProbeIntervals one launch covers on a healthy quiet pool
#define GS_PRISTINE_WINDOW 256u  // ... and on a pristine one (every probe a prompt ack: gs_pristine_probes)
static bool pristine_windows_on() {
  static const bool off = getenv("GSIM_NO_PRISTINE_WINDOWS") != nullptr;
  return !off;
}
static bool long_windows_on() {
  static const bool off = getenv("GSIM_NO_LONG_WINDOWS") != nullptr;
  return !off;
}

// No probe in flight, and can one fail at all?  Not if every member the cluster lists as alive or
// suspect is actually running, no packet is lost and no link is slower than ProbeTimeout: then the
// horizon cannot move and one launch may run many ProbeIntervals (the controller counts, every
// rank adopts the answer).
static bool probes_always_answered(const gsim_pool* p) {
  const GsGlobals& g = p->g;
  bool links_ok = true;  // every round trip of the latency matrix fits ProbeTimeout
  for (uint32_t a = 0; a < g.n_dcs && links_ok; ++a)
    for (uint32_t b = 0; b < g.n_dcs; ++b)
      if ((uint32_t)g.lat[a * GS_MAX_DCS + b] + g.lat[b * GS_MAX_DCS + a] > g.T) links_ok = false;
  return g.loss_thr == 0u && p->n_impaired == 0u && links_ok;
}
static int quiet_decision(gsim_pool* p, uint32_t hz, bool can_long);

// After single ticks (sharded pools, and pools without CUDA graphs): has the pool been quiet long
// enough, and how far is the horizon?
static int try_quiet(gsim_pool* p) {
  GsBackend* be = dev(p);
  const GsGlobals& g = p->g;
  const uint32_t depth = g.ring_mask + 1u;
  uint32_t* qs = p->d.qstate[p->sharded ? p->rank : 0u];
  uint32_t la = p->last_active;  // single GPU: the word run_ticks read back with its own synchronisation
  if (p->sharded) {
    if (!be->xbar_host(p->xb)) return GSIM_ERR_CUDA;  // every rank's last tick has published
    if (!be->d2h(&la, qs + GS_Q_LAST_ACTIVE, 4)) return GSIM_ERR_CUDA;
    // ... and nobody runs on (and writes this rank's copy from its next tick) before everybody has read
    if (!be->xbar_host(p->xb)) return GSIM_ERR_CUDA;
  }
  if (p->dirty_tick + 1u > la) la = p->dirty_tick + 1u;  // a host write at tick T counts like mail at T
  // every arrival slot has been scanned empty once and nobody posted meanwhile: `depth` quiet ticks
  if (p->now < la + depth) {
    // Still busy.  Looking again after every tick would put a host round trip (on a sharded pool: two
    // barriers) behind each tick of a cascade: back off 1, 2, 4, 8 ticks.  Finding the quiet a few ticks
    // late only means those ticks ran as single launches.
    const uint32_t wait = 1u << (p->quiet_fails < 3u ? p->quiet_fails : 3u);
    if (p->quiet_fails < 3u) p->quiet_fails++;
    p->retry_at = la + depth > p->now + wait ? la + depth : p->now + wait;
    return GSIM_OK;
  }
  p->quiet_fails = 0;
  const bool can_long = probes_always_answered(p);
  uint32_t hz = 0;
  if (!p->sharded) {
    // horizon reset, scan and readback in one round trip, with the counts a long window needs
    counts_invalidate(p);  // (ticks have run since the last count)
    if (!upload_globals(p)) return GSIM_ERR_CUDA;
    if (!be->quiet_probe(p->d, p->g_dev, g, p->now, &hz, can_long ? &p->rc : nullptr)) return GSIM_ERR_CUDA;
    p->counts_stale = !can_long;
  } else {
    const uint32_t never = GS_NEVER;
    if (!be->h2d(qs + GS_Q_HORIZON, &never, 4)) return GSIM_ERR_CUDA;
    if (!be->xbar_host(p->xb)) return GSIM_ERR_CUDA;
    uint32_t first, count;
    shard_rows(p, &first, &count);
    if (!be->quiet_scan(p->d, p->g_dev, g, p->now, first, count)) return GSIM_ERR_CUDA;
    if (!be->xbar_host(p->xb)) return GSIM_ERR_CUDA;
    if (!be->d2h(&hz, qs + GS_Q_HORIZON, 4)) return GSIM_ERR_CUDA;
    if (!be->xbar_host(p->xb)) return GSIM_ERR_CUDA;  // (same: read before anybody moves on)
  }
  return quiet_decision(p, hz, can_long);
}

// The pool is quiet at p->now and the horizon is `hz`: windows from here, or single ticks up to a near
// probe deadline.  On a single-GPU pool p->rc holds the counts when `can_long`.
static int quiet_decision(gsim_pool* p, uint32_t hz, bool can_long) {
  const GsGlobals& g = p->g;
  const uint32_t depth = g.ring_mask + 1u;
  p->sched_counts[3]++;
  if (hz >= p->now + g.P / 2u + 1u) {
    p->quiet = true;
    uint32_t ok_long = 0;
    if (hz == GS_NEVER && can_long) {
      int rc = GSIM_OK;
      if (p->sharded) {
        counts_invalidate(p);  // (ticks have run since the last count)
        rc = collective_recount(p);
        if (rc) return rc;
      }
      rc = controller_call(p, &ok_long, sizeof(ok_long), [&]() -> int {
        if (!do_recount(p)) return GSIM_ERR_CUDA;
        ok_long = p->rc.unreachable_live == 0u ? 1u : 0u;
        // everybody running, listed alive by everybody, folded into the established set
        // (members still pending are the subjects of tracked alive rumors: the closed form stops in front
        // of their ring entries as it does in front of a member's own)
        uint32_t spec[GS_MAX_SPECIAL];
        const uint32_t n_spec = gs_special_members(g, spec);
        if (ok_long && p->rc.truth_cnt[GS_TRUTH_UP] == g.n && p->rc.rank_cnt[GS_RANK_ALIVE] == g.n &&
            n_spec <= GS_MAX_SPECIAL && p->rc.pending <= n_spec && p->rc.isolated_up == 0u && pristine_windows_on())
          ok_long |= 2u;
        return GSIM_OK;
      });
      if (rc) return rc;
    }
    p->healthy = (ok_long & 1u) != 0u;
    p->pristine = (ok_long & 2u) != 0u;
  } else {  // a probe deadline is upon us: single ticks until it has passed, then look again
    p->retry_at = (hz > p->now ? hz : p->now) + depth + 1u;
  }
  return GSIM_OK;
}

// `chunk` ticks, as quiet windows where the pool allows it and as single ticks where it does not.
static int advance_ticks(gsim_pool* p, uint32_t chunk, bool use_graph) {
  GsBackend* be = dev(p);
  const GsXbar* xb = p->sharded ? &p->xb : nullptr;
  uint32_t left = chunk;
  const bool can_window = windows_possible(p);
  // sharded pools and pools without graphs look for quietness from the host, between chunks (try_quiet)
  const bool stretch = can_window && !p->sharded && use_graph;
  while (left) {
    if (can_window && p->quiet) {
      uint32_t done = 0;
      uint64_t nl = 0;
      double wms = 0;
      // ticks per launch: one ProbeInterval; up to GS_LONG_WINDOW of them on a healthy pool
      const bool lng = p->healthy && long_windows_on();
      const bool prist = lng && p->pristine;  // (the closed form costs the same for any number of probes)
      const uint32_t per_launch = prist ? p->g.P * GS_PRISTINE_WINDOW : lng ? p->g.P * GS_LONG_WINDOW : p->g.P;
      if (!be->run_windows(p->d, p->g_dev, p->g, p->now, left, per_launch, use_graph, &wms, &nl, &done, xb, prist))
        return GSIM_ERR_CUDA;
      p->last_ms += wms;
      p->sched_counts[4] += (uint64_t)(wms * 1e6);
      p->last_launches += nl;
      p->sched_counts[0] += nl;
      p->sched_counts[1] += done;
      if (prist) {
        p->sched_counts[6] += nl;
        p->sched_counts[7] += done;
      }
      p->now += done;
      p->node_ticks += (uint64_t)done * p->g.n;
      left -= done;
      if (left) {  // the chain stopped at the horizon: single ticks from here
        p->quiet = false;
        p->healthy = false;
        p->pristine = false;
        p->retry_at = p->now + 1u;
      }
      continue;
    }
    if (stretch) {
      // Single ticks up to the first quiet tick, found by the device (run_tick_stretch): one submission and
      // one readback for the whole busy stretch, with the quiet probe behind it when it stopped quiet.
      // A host write at tick T counts like mail at T; after a near probe deadline nobody looks before retry_at.
      const uint32_t depth = p->g.ring_mask + 1u;
      uint32_t floor = p->dirty_tick + 1u;
      if (p->retry_at > floor + depth) floor = p->retry_at - depth;
      const bool can_long = probes_always_answered(p);
      counts_invalidate(p);
      if (!upload_globals(p)) return GSIM_ERR_CUDA;
      GsStretch s;
      double tms = 0;
      if (!be->run_tick_stretch(p->d, p->g_dev, p->g, p->now, left, floor, can_long, &tms, &s)) return GSIM_ERR_CUDA;
      p->last_active = s.last_active;
      p->last_ms += tms;
      p->last_launches += s.launches;
      p->sched_counts[5] += (uint64_t)(tms * 1e6);
      p->sched_counts[2] += s.ran;
      p->now += s.ran;
      p->node_ticks += (uint64_t)s.ran * p->g.n;
      left -= s.ran;
      if (s.quiet) {
        if (can_long) p->rc = s.counts;
        p->counts_stale = !can_long;
        int rc = quiet_decision(p, s.horizon, can_long);
        if (rc) return rc;
      }
      continue;
    }
    uint32_t c = left;
    if (can_window && c > 16u) c = 16u;  // look for quietness every few ticks
    if (can_window && p->retry_at > p->now && p->retry_at - p->now < c) c = p->retry_at - p->now;
    double tms = 0;
    if (!be->run_ticks_read(p->d, p->g_dev, p->g, p->now, c, use_graph, &tms, &p->last_launches, xb, &p->last_active))
      return GSIM_ERR_CUDA;
    p->last_ms += tms;
    p->sched_counts[5] += (uint64_t)(tms * 1e6);
    p->sched_counts[2] += c;
    p->now += c;
    p->node_ticks += (uint64_t)c * p->g.n;
    left -= c;
    if (can_window && left && p->now >= p->retry_at) {
      int rc = try_quiet(p);
      if (rc) return rc;
    }
  }
  return GSIM_OK;
}

extern "C" int gsim_piggyback_stats(gsim_pool* p, uint64_t out[4]) {
  if (!p || !out) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (!p->d.pig) return fail(p, GSIM_ERR_STATE, "the pool was created without GSIM_FLAG_PROBE_PIGGYBACK");
  GsPig pig;
  if (!flush_writes(p) || !dev(p)->d2h(&pig, p->d.pig, sizeof(pig))) return fail(p, GSIM_ERR_CUDA, "d2h");
  for (int k = 0; k < 4; ++k) {
    out[k] = 0;
    for (int l = 0; l < 32; ++l) out[k] += pig.stats[k][l];
  }
  return GSIM_OK;
}

extern "C" int gsim_sched_counts(gsim_pool* p, uint64_t out[8]) {
  if (!p || !out) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  memcpy(out, p->sched_counts, sizeof(p->sched_counts));
  return GSIM_OK;
}

static int step_locked(gsim_pool* p, uint32_t ticks) {
  if (!p->ready) return GSIM_ERR_STATE;
  p->last_ms = 0;
  p->last_launches = 0;
  uint32_t left = ticks;
  const bool use_graph = !(p->cfg.flags & GSIM_FLAG_NO_GRAPH);
  while (left) {
    int rc = controller_call(p, nullptr, 0, [&]() -> int {
      int r = apply_sched(p);
      if (r) return r;
      r = reap_pass(p);
      if (r) return r;
      return upload_globals(p) ? GSIM_OK : GSIM_ERR_CUDA;
    });
    if (rc) return rc;
    uint32_t chunk = left;
    for (const Sched& s : p->sched)
      if (s.tick > p->now && s.tick - p->now < chunk) chunk = s.tick - p->now;
    const uint32_t reap_at = next_reap_tick(p, p->now);
    if (reap_at != GS_NEVER && reap_at - p->now < chunk) chunk = reap_at - p->now;
    rc = advance_ticks(p, chunk, use_graph);
    if (rc) return rc;
    left -= chunk;
    counts_invalidate(p);
  }
  // (the mask is the same on every rank: the loop's last controller call published it)
  bool cand = false;
  for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r)
    if (((p->g.active_mask >> r) & 1u) && p->g.rumors[r].kind != GSIM_RUMOR_USER_EVENT) cand = true;
  if (cand) {
    int rc = collective_recount(p);
    if (rc) return rc;
  }
  int rc = controller_call(p, nullptr, 0, [&]() -> int {
    int r = apply_sched(p);
    if (r) return r;
    p->defer_and = true;
    r = auto_retire(p);
    p->defer_and = false;
    return r;
  });
  if (rc) return rc;
  return apply_pending_and(p);
}

extern "C" int gsim_step(gsim_pool* p, uint32_t ticks) {
  if (!p) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  int rc = step_locked(p, ticks);
  return rc ? fail(p, rc, "step") : GSIM_OK;
}

extern "C" uint32_t gsim_now(gsim_pool* p) { return p ? p->now : 0; }

extern "C" int gsim_run_until(gsim_pool* p, int predicate, uint32_t arg, uint32_t max_ticks,
                              uint32_t check_every, uint32_t* tick_out) {
  if (!p || !check_every) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (tick_out) *tick_out = GS_EMPTY32;
  uint32_t done = 0;
  double ms = 0;
  uint64_t launches = 0;
  for (;;) {
    uint32_t result = GS_EMPTY32;
    if (predicate == GSIM_PRED_RUMOR_CONVERGED) {
      if (arg >= GS_MAX_RUMORS) return fail(p, GSIM_ERR_INVALID, "bad slot");
      if (!peek(p, p->d.conv_tick, arg, &result)) return fail(p, GSIM_ERR_CUDA, "peek");
    } else if (predicate == GSIM_PRED_ALL_RUMORS_CONVERGED) {
      uint32_t ct[32];
      if (!dev(p)->d2h(ct, p->d.conv_tick, sizeof(ct))) return fail(p, GSIM_ERR_CUDA, "d2h");
      uint32_t mx = 0;
      bool all = true;
      for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r)
        if ((p->g.active_mask >> r) & 1u) {
          if (ct[r] == GS_EMPTY32) all = false;
          else if (ct[r] > mx) mx = ct[r];
        }
      if (all) result = mx;
    } else if (predicate == GSIM_PRED_CRASHED_ALL_DEAD) {
      if (!peek(p, p->d.crashed_dead_tick, 0, &result)) return fail(p, GSIM_ERR_CUDA, "peek");
    } else {
      return fail(p, GSIM_ERR_INVALID, "unknown predicate");
    }
    if (result != GS_EMPTY32) {
      if (tick_out) *tick_out = result;
      break;
    }
    if (done >= max_ticks) break;
    uint32_t chunk = max_ticks - done < check_every ? max_ticks - done : check_every;
    int rc = step_locked(p, chunk);
    if (rc) return fail(p, rc, "step");
    ms += p->last_ms;
    launches += p->last_launches;
    done += chunk;
  }
  p->last_ms = ms;
  p->last_launches = launches;
  return GSIM_OK;
}

// ---- observation ------------------------------------------------------------------
static bool host_knows(const GsGlobals& g, uint32_t i, uint32_t c, uint32_t kc, uint32_t heard_i,
                       uint32_t meta_i) {
  if (c == i) return true;
  if (!gs_key_pending(kc)) return !(meta_i & GS_META_ISOLATED);
  for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r)
    if (((g.active_mask >> r) & 1u) && g.rumors[r].kind == GSIM_RUMOR_ALIVE && g.rumors[r].subject == c)
      return (heard_i >> r) & 1u;
  return false;
}

// Pinned staging for bulk reads (Members() pulls one key per member): grown on demand, freed with the pool.
static uint32_t* host_stage(gsim_pool* p, size_t words) {
  if (words > p->stage_words) {
    if (p->stage) dev(p)->host_free(p->stage);
    p->stage_words = 0;
    p->stage = static_cast<uint32_t*>(dev(p)->host_alloc(words * 4u));
    if (p->stage) p->stage_words = words;
  }
  return p->stage;
}

static int members_locked(gsim_pool* p, uint32_t observer, gsim_member* out, size_t cap, size_t* n) {
  const GsGlobals& g = p->g;
  if (observer >= g.n) return GSIM_ERR_NOT_FOUND;
  uint32_t* keys = host_stage(p, g.n);
  uint32_t heard, meta;
  if (!keys || !dev(p)->d2h(keys, p->d.key[p->now & 1u], (size_t)g.n * 4) ||
      !peek(p, p->d.heard, observer, &heard) || !peek(p, p->d.meta, observer, &meta))
    return GSIM_ERR_CUDA;
  // on a CSR peer graph a member's list is itself plus its row
  std::vector<uint8_t> in_row;
  if (g.graph_n) {
    in_row.assign(g.n, 0);
    in_row[observer] = 1;
    for (uint32_t e = p->graph_rp[observer]; e < p->graph_rp[observer + 1]; ++e) in_row[p->graph_col[e]] = 1;
  }
  auto visible = [&](uint32_t c) -> bool {
    const uint32_t kc = keys[c];
    if (gs_key_truth(kc) == GS_TRUTH_NONE) return false;
    if (g.graph_n && !in_row[c]) return false;
    return host_knows(g, observer, c, kc, heard, meta);
  };
  auto emit = [&](uint32_t c, gsim_member& mm) {
    const uint32_t kc = keys[c];
    mm.id = c;
    mm.incarnation = gs_key_inc(kc);
    mm.rank = gs_key_rank(kc);
    // memberlist suspect is still serf alive; dead -> failed; left -> left
    mm.status = mm.rank == GS_RANK_DEAD   ? GSIM_STATUS_FAILED
                : mm.rank == GS_RANK_LEFT ? GSIM_STATUS_LEFT
                                          : GSIM_STATUS_ALIVE;
  };
  // The list is 16 B per member: at a million members the host loop, not the 4 MB copy, is the cost of
  // the call.  Large pools split the id range over a few threads (count, exclusive scan, fill).
  unsigned nt = 1;
  if (g.n >= (1u << 17)) {
    nt = std::thread::hardware_concurrency();
    nt = nt > 8u ? 8u : nt < 1u ? 1u : nt;
    if (const char* e = getenv("GSIM_MEMBERS_THREADS")) nt = (unsigned)atoi(e) ? (unsigned)atoi(e) : 1u;
  }
  if (!out) cap = 0;
  if (nt <= 1) {
    size_t cnt = 0;
    for (uint32_t c = 0; c < g.n; ++c) {
      if (!visible(c)) continue;
      if (cnt < cap) emit(c, out[cnt]);
      ++cnt;
    }
    if (n) *n = cnt;
    return GSIM_OK;
  }
  if (p->workers && p->workers->size() != nt) {
    delete p->workers;
    p->workers = nullptr;
  }
  if (!p->workers) p->workers = new HostWorkers(nt);
  std::vector<size_t> part(nt, 0);
  std::atomic<unsigned> counted{0};
  const uint32_t chunk = (g.n + nt - 1) / nt;
  const std::function<void(unsigned)> work = [&](unsigned w) {
    const uint32_t lo = w * chunk < g.n ? w * chunk : g.n, hi = lo + chunk < g.n ? lo + chunk : g.n;
    size_t mine = 0;
    for (uint32_t c = lo; c < hi; ++c) mine += visible(c) ? 1u : 0u;
    part[w] = mine;
    counted.fetch_add(1, std::memory_order_release);
    while (counted.load(std::memory_order_acquire) < nt) std::this_thread::yield();
    size_t at = 0;
    for (unsigned q = 0; q < w; ++q) at += part[q];
    if (at >= cap) return;
    for (uint32_t c = lo; c < hi && at < cap; ++c)
      if (visible(c)) emit(c, out[at++]);
  };
  p->workers->run(work);
  size_t cnt = 0;
  for (unsigned w = 0; w < nt; ++w) cnt += part[w];
  if (n) *n = cnt;
  return GSIM_OK;
}

extern "C" int gsim_members(gsim_pool* p, uint32_t observer, gsim_member* out, size_t cap, size_t* n) {
  if (!p) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GS_CONTROLLER_ONLY(p);
  int rc = members_locked(p, observer, out, cap, n);
  return rc ? fail(p, rc, "members") : GSIM_OK;
}

extern "C" int gsim_num_nodes(gsim_pool* p, uint32_t observer, uint32_t* n) {
  if (!p || !n) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  return controller_call(p, n, sizeof(uint32_t), [&]() -> int {
  size_t cnt = 0;
  int rc = members_locked(p, observer, nullptr, 0, &cnt);
  *n = (uint32_t)cnt;
  return rc ? fail(p, rc, "num_nodes") : GSIM_OK;
  });
}

// ---- per-agent observation (DESIGN.md §3.8, gs_agent.h) ---------------------------------------------
static_assert(sizeof(GsAgentStats) == sizeof(gsim_agent_stats), "GsAgentStats is gsim_agent_stats field for field");

bool GsBackend::agent_stats(const GsDev& d, const GsGlobals& g, const uint32_t* key, const GsPendingAlive& pa,
                            uint32_t first, uint32_t count, GsAgentStats* out) {
  const size_t n = g.n;
  std::vector<uint32_t> k(n), meta(n), heard(n), queued(n), lm(n), le(n), rp, col;
  if (!d2h(k.data(), key, n * 4) || !d2h(meta.data(), d.meta, n * 4) || !d2h(heard.data(), d.heard, n * 4) ||
      !d2h(queued.data(), d.queued, n * 4) || !d2h(lm.data(), d.ltime_member, n * 4) ||
      !d2h(le.data(), d.ltime_event, n * 4))
    return false;
  uint32_t est[4] = {0u, 0u, 0u, 0u};
  if (g.graph_n) {
    rp.resize(n + 1);
    if (!d2h(rp.data(), d.row_ptr, (n + 1) * 4)) return false;
    col.resize(rp[n]);
    if (rp[n] && !d2h(col.data(), d.col_idx, (size_t)rp[n] * 4)) return false;
  } else {
    for (size_t i = 0; i < n; ++i)
      if (const uint32_t r1 = gs_established_rank1(k[i])) est[r1 - 1u]++;
  }
  const GsAgentCols c = {k.data(), meta.data(), heard.data(), queued.data(), lm.data(), le.data(),
                         g.graph_n ? rp.data() : nullptr, g.graph_n ? col.data() : nullptr};
  for (uint32_t x = 0; x < count; ++x) out[x] = gs_agent_stats_row(c, g.class_mask, est, pa, first + x);
  return true;
}

bool GsBackend::health_histogram(const GsDev& d, const GsGlobals& g, const uint32_t* key, const GsImpairCols& imp,
                                 uint64_t out[GS_HIST_BINS]) {
  const size_t n = g.n;
  for (uint32_t b = 0; b < GS_HIST_BINS; ++b) out[b] = 0u;
  std::vector<uint32_t> k(n), meta(n), loss(imp.loss ? n : 0u), recv(imp.recv ? n : 0u);
  std::vector<uint8_t> delay(imp.delay ? n : 0u), flags(imp.flags ? n : 0u);
  if (!d2h(k.data(), key, n * 4) || !d2h(meta.data(), d.meta, n * 4) || (imp.loss && !d2h(loss.data(), imp.loss, n * 4)) ||
      (imp.recv && !d2h(recv.data(), imp.recv, n * 4)) || (imp.delay && !d2h(delay.data(), imp.delay, n)) ||
      (imp.flags && !d2h(flags.data(), imp.flags, n)))
    return false;
  const GsImpairCols h = {imp.loss ? loss.data() : nullptr, imp.recv ? recv.data() : nullptr,
                          imp.delay ? delay.data() : nullptr, imp.flags ? flags.data() : nullptr};
  for (uint32_t i = 0; i < n; ++i) {
    const uint32_t b = gs_health_bin(k[i], meta[i], h, i);
    if (b < GS_HIST_BINS) out[b]++;
  }
  return true;
}

// (*Serf).Stats() of members [first, first + count) — what `consul info` prints as serf_lan / serf_wan
// (agent/consul/client.go:417, server.go:1733,1744).  Read-only.
extern "C" int gsim_agent_stats_read(gsim_pool* p, uint32_t first, uint32_t count, gsim_agent_stats* out) {
  if (!p || !out || count == 0u) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GS_CONTROLLER_ONLY(p);
  if (first >= p->g.n || count > p->g.n - first) return fail(p, GSIM_ERR_NOT_FOUND, "unknown member");
  GsPendingAlive pa;
  gs_pending_alive(p->g, pa);
  if (!dev(p)->agent_stats(p->d, p->g, p->d.key[p->now & 1u], pa, first, count, reinterpret_cast<GsAgentStats*>(out)))
    return fail(p, GSIM_ERR_CUDA, "agent_stats");
  return GSIM_OK;
}

// memberlist GetHealthScore() of every running member, counted by score: out[0] unimpaired, out[1] impaired.
extern "C" int gsim_health_histogram(gsim_pool* p, uint64_t out[2][8]) {
  if (!p || !out) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GS_CONTROLLER_ONLY(p);
  const GsImpairCols imp = {p->imp_loss, p->imp_recv, p->imp_delay, p->imp_flags};
  uint64_t h[GS_HIST_BINS];
  if (!dev(p)->health_histogram(p->d, p->g, p->d.key[p->now & 1u], imp, h))
    return fail(p, GSIM_ERR_CUDA, "health_histogram");
  memcpy(out, h, sizeof(h));
  return GSIM_OK;
}

extern "C" int gsim_poll_events(gsim_pool* p, gsim_event* out, size_t cap, size_t* n) {
  if (!p || !n || (!out && cap)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GS_CONTROLLER_ONLY(p);
  uint32_t cur[2];
  if (!dev(p)->d2h(cur, p->d.evlog_cursor, 8)) return fail(p, GSIM_ERR_CUDA, "d2h");
  uint32_t have = cur[0] < p->g.evlog_cap ? cur[0] : p->g.evlog_cap;
  std::vector<GsEventRec> ev(have);
  if (have && !dev(p)->d2h(ev.data(), p->d.evlog, (size_t)have * sizeof(GsEventRec)))
    return fail(p, GSIM_ERR_CUDA, "d2h");
  // the device appends in scheduling order; canonical order is (tick, type, subject, observer)
  std::sort(ev.begin(), ev.end(), [](const GsEventRec& a, const GsEventRec& b) {
    if (a.tick != b.tick) return a.tick < b.tick;
    if (a.type != b.type) return a.type < b.type;
    if (a.subject != b.subject) return a.subject < b.subject;
    return a.observer < b.observer;
  });
  size_t take = have < cap ? have : cap;
  for (size_t x = 0; x < take; ++x) {
    out[x].tick = ev[x].tick;
    out[x].type = ev[x].type;
    out[x].subject = ev[x].subject;
    out[x].observer = ev[x].observer;
    out[x].ltime = ev[x].ltime;
    out[x].reserved = 0;
  }
  *n = take;
  // keep what did not fit
  uint32_t rest = have - (uint32_t)take;
  if (rest && !dev(p)->h2d(p->d.evlog, ev.data() + take, (size_t)rest * sizeof(GsEventRec)))
    return fail(p, GSIM_ERR_CUDA, "h2d");
  p->events_dropped += cur[1];
  uint32_t reset[2] = {rest, 0};
  if (!dev(p)->h2d(p->d.evlog_cursor, reset, 8)) return fail(p, GSIM_ERR_CUDA, "h2d");
  return GSIM_OK;
}

extern "C" int gsim_rumor_info_get(gsim_pool* p, uint32_t slot, gsim_rumor_info* out) {
  if (!p || !out || slot >= GS_MAX_RUMORS) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (int rcc = collective_recount(p)) return fail(p, rcc, "recount");
  return controller_call(p, out, sizeof(gsim_rumor_info), [&]() -> int {
  const GsGlobals& g = p->g;
  if (!((g.active_mask >> slot) & 1u)) return fail(p, GSIM_ERR_NOT_FOUND, "slot is free");
  if (!do_recount(p)) return fail(p, GSIM_ERR_CUDA, "recount");
  const GsRumor& ru = g.rumors[slot];
  out->kind = ru.kind;
  out->subject = ru.subject;
  out->incarnation = ru.inc;
  out->ltime = ru.ltime;
  out->origin = ru.origin;
  out->size_bytes = ru.size;
  out->start_tick = ru.start_tick;
  out->heard_count = p->rc.heard_cnt[slot];
  out->queued_count = p->rc.queued_cnt[slot];
  if (!peek(p, p->d.conv_tick, slot, &out->converged_tick)) return fail(p, GSIM_ERR_CUDA, "peek");
  return GSIM_OK;
  });
}

extern "C" int gsim_rumor_retire(gsim_pool* p, uint32_t slot) {
  if (!p || slot >= GS_MAX_RUMORS) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  return controller_call(p, nullptr, 0, [&]() -> int {
  if (!((p->g.active_mask >> slot) & 1u)) return fail(p, GSIM_ERR_NOT_FOUND, "slot is free");
  if (p->g.rumors[slot].kind == GSIM_RUMOR_ALIVE) {
    if (!do_recount(p)) return fail(p, GSIM_ERR_CUDA, "recount");
    if (p->rc.heard_cnt[slot] != p->g.up_count || p->rc.isolated_up != 0)
      return fail(p, GSIM_ERR_STATE, "alive rumor has not reached every running member");
  }
  int rc = retire_slot(p, slot);
  return rc ? fail(p, rc, "retire") : GSIM_OK;
  });
}

extern "C" int gsim_user_event_get(gsim_pool* p, uint32_t slot, void* name, size_t name_cap,
                                   size_t* name_len, void* payload, size_t payload_cap,
                                   size_t* payload_len) {
  if (!p || slot >= GS_MAX_RUMORS) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GS_CONTROLLER_ONLY(p);
  if (!((p->g.active_mask >> slot) & 1u) || p->g.rumors[slot].kind != GSIM_RUMOR_USER_EVENT)
    return fail(p, GSIM_ERR_NOT_FOUND, "not a user event slot");
  const RumorHost& rh = p->rh[slot];
  if (name_len) *name_len = rh.name.size();
  if (payload_len) *payload_len = rh.payload.size();
  if (name && name_cap) memcpy(name, rh.name.data(), std::min(name_cap, rh.name.size()));
  if (payload && payload_cap) memcpy(payload, rh.payload.data(), std::min(payload_cap, rh.payload.size()));
  return GSIM_OK;
}

extern "C" int gsim_stats_get(gsim_pool* p, gsim_stats* out) {
  if (!p || !out) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  if (int rcc = collective_recount(p)) return fail(p, rcc, "recount");
  return controller_call(p, out, sizeof(gsim_stats), [&]() -> int {
  memset(out, 0, sizeof(*out));
  if (!do_recount(p)) return fail(p, GSIM_ERR_CUDA, "recount");
  if (!p->sharded) {
    if (!dev(p)->d2h(out->counters, p->d.stats, sizeof(out->counters))) return fail(p, GSIM_ERR_CUDA, "d2h");
  } else {
    // message counters are accumulated per rank (no cross-GPU atomics in the tick): sum the pages
    for (uint32_t r = 0; r < p->world; ++r) {
      uint64_t part[GSIM_STAT_COUNT];
      if (!dev(p)->d2h(part, p->pages + (size_t)r * GS_PAGE_BYTES + GS_PG_STATS, sizeof(part)))
        return fail(p, GSIM_ERR_CUDA, "d2h");
      for (int q = 0; q < GSIM_STAT_COUNT; ++q) out->counters[q] += part[q];
    }
  }
  const GsGlobals& g = p->g;
  out->node_ticks = p->node_ticks;
  out->tick = p->now;
  out->n_members = g.n;
  out->n_up = p->rc.truth_cnt[GS_TRUTH_UP];
  out->n_crashed = p->rc.truth_cnt[GS_TRUTH_CRASHED];
  out->n_gone = p->rc.truth_cnt[GS_TRUTH_GONE];
  out->n_view_alive = p->rc.rank_cnt[GS_RANK_ALIVE];
  out->n_view_suspect = p->rc.rank_cnt[GS_RANK_SUSPECT];
  out->n_view_dead = p->rc.rank_cnt[GS_RANK_DEAD];
  out->n_view_left = p->rc.rank_cnt[GS_RANK_LEFT];
  out->retransmit_limit = g.retransmit_limit;
  out->suspicion_k = g.sus_k;
  for (int q = 0; q < GS_K1MAX; ++q) out->suspicion_ticks[q] = g.sus_ticks[q];
  out->probe_interval_ticks = g.P;
  out->probe_timeout_ticks = g.T;
  out->gossip_interval_ticks = g.GI;
  uint32_t cur[2] = {0, 0};
  dev(p)->d2h(cur, p->d.evlog_cursor, 8);
  out->events_dropped = p->events_dropped + cur[1];
  return GSIM_OK;
  });
}

extern "C" int gsim_state_hash(gsim_pool* p, uint64_t out[4]) {
  if (!p || !out) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  return controller_call(p, out, 4 * sizeof(uint64_t), [&]() -> int {
  if (!upload_globals(p)) return fail(p, GSIM_ERR_CUDA, "upload");
  if (!dev(p)->state_hash(p->d, p->g_dev, p->g, p->now, out)) return fail(p, GSIM_ERR_CUDA, "hash");
  // pool-wide scalars
  uint64_t h = gs_mix64(0x243F6A8885A308D3ull, p->now);
  h = gs_mix64(h, p->g.n);
  h = gs_mix64(h, p->g.up_count);
  h = gs_mix64(h, p->g.active_mask);
  for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r)
    if ((p->g.active_mask >> r) & 1u) {
      const GsRumor& ru = p->g.rumors[r];
      h = gs_mix64(h, ((uint64_t)r << 32) | ru.kind);
      h = gs_mix64(h, ((uint64_t)ru.subject << 32) | ru.ltime);
    }
  uint64_t lanes[4];
  gs_hash_lanes(h, lanes);
  for (int q = 0; q < 4; ++q) out[q] += lanes[q];
  return GSIM_OK;
  });
}

extern "C" int gsim_column_read(gsim_pool* p, int column, void* out, size_t cap_bytes, size_t* n_bytes) {
  if (!p || !out) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GS_CONTROLLER_ONLY(p);
  const GsDev& d = p->d;
  const size_t cap = p->g.cap;
  const void* src = nullptr;
  size_t bytes = cap * 4;
  switch (column) {
    case GSIM_COL_KEY: src = d.key[p->now & 1u]; break;
    case GSIM_COL_META: src = d.meta; break;
    case GSIM_COL_DUE: src = d.due; break;
    case GSIM_COL_CURSOR: src = d.cursor; break;
    case GSIM_COL_PASS: src = d.pass; break;
    case GSIM_COL_PROBE_TGT: src = d.probe_tgt; break;
    case GSIM_COL_PROBE_INC: src = d.probe_inc; break;
    case GSIM_COL_SUS_START: src = d.sus_start; break;
    case GSIM_COL_SUS_FROM: src = d.sus_from; bytes = cap * 4 * GS_K1MAX; break;
    case GSIM_COL_CHANGE_TICK: src = d.change_tick; break;
    case GSIM_COL_LTIME_MEMBER: src = d.ltime_member; break;
    case GSIM_COL_LTIME_EVENT: src = d.ltime_event; break;
    case GSIM_COL_EVENT_MIN: src = d.event_min; break;
    case GSIM_COL_HEARD: src = d.heard; break;
    case GSIM_COL_QUEUED: src = d.queued; break;
    case GSIM_COL_TX: src = d.tx; bytes = cap * GS_MAX_RUMORS; break;
    case GSIM_COL_INBOX: src = d.inbox[p->now & p->g.ring_mask]; break;
    default: return fail(p, GSIM_ERR_INVALID, "unknown column");
  }
  // the caller sees rows of `capacity` elements; the device stride is padded to whole tiles
  const size_t ucap = p->cfg.capacity;
  const size_t planes = column == GSIM_COL_SUS_FROM ? GS_K1MAX : column == GSIM_COL_TX ? GS_MAX_RUMORS : 1;
  const size_t elem = column == GSIM_COL_TX ? 1 : 4;
  const size_t out_bytes = planes * ucap * elem;
  (void)bytes;
  if (n_bytes) *n_bytes = out_bytes;
  if (cap_bytes < out_bytes) return fail(p, GSIM_ERR_INVALID, "buffer too small");
  if (column == GSIM_COL_TX) {
    // device layout: two rumors per 16-bit element (GS_TX); the caller sees [rumor][capacity] bytes
    std::vector<uint8_t> pair(ucap * 2);
    uint8_t* o = reinterpret_cast<uint8_t*>(out);
    for (size_t q = 0; q < GS_MAX_RUMORS / 2; ++q) {
      if (!dev(p)->d2h(pair.data(), reinterpret_cast<const uint8_t*>(src) + q * cap * 2, ucap * 2))
        return fail(p, GSIM_ERR_CUDA, "d2h");
      for (size_t i = 0; i < ucap; ++i) {
        o[(2 * q) * ucap + i] = pair[2 * i];
        o[(2 * q + 1) * ucap + i] = pair[2 * i + 1];
      }
    }
    return GSIM_OK;
  }
  for (size_t q = 0; q < planes; ++q)
    if (!dev(p)->d2h(reinterpret_cast<uint8_t*>(out) + q * ucap * elem,
                    reinterpret_cast<const uint8_t*>(src) + q * cap * elem, ucap * elem))
      return fail(p, GSIM_ERR_CUDA, "d2h");
  if (column == GSIM_COL_META) {
    uint32_t* mm = reinterpret_cast<uint32_t*>(out);
    for (size_t i = 0; i < ucap; ++i) mm[i] &= ~GS_META_DIRTY;  // implementation detail
  }
  if (column == GSIM_COL_INBOX) {
    uint32_t* mm = reinterpret_cast<uint32_t*>(out);
    for (size_t i = 0; i < ucap; ++i) mm[i] &= ~GS_WAKE_BIT;  // implementation detail
  }
  return GSIM_OK;
}

// ---- checkpoint / resume ------------------------------------------------------------
// A snapshot is a header followed by the columns, plane by plane.  Most planes of the cold columns
// hold one repeated 32-bit word (empty accusation slots, untouched retransmit counters, zero
// change ticks ...): such a plane is stored as (tag 1, word) and restored with a device fill
// instead of a host->device copy; everything else is (tag 0, raw bytes).
struct SnapCol {
  void* ptr;
  size_t bytes;      // all planes together
  uint32_t planes;   // equally sized, each a multiple of 4 bytes
  bool may_fill;     // planes may be stored as a repeated word
};
static std::vector<SnapCol> snap_cols(gsim_pool* p, bool with_impairment, bool with_pause, bool with_reach,
                                      bool with_flap, bool with_dom) {
  const GsDev& d = p->d;
  const size_t cap = p->g.cap;
  std::vector<SnapCol> v;
  auto add = [&](void* q, size_t b, uint32_t planes = 1, bool may_fill = true) { v.push_back(SnapCol{q, b, planes, may_fill}); };
  add(d.key[0], cap * 4, 1, false); add(d.key[1], cap * 4, 1, false);  // (replicated per rank when sharded)
  for (uint32_t s = 0; s <= p->g.ring_mask; ++s) add(d.inbox[s], cap * 4);
  add(d.due, cap * 4); add(d.meta, cap * 4); add(d.cursor, cap * 4); add(d.pass, cap * 4);
  add(d.probe_tgt, cap * 4); add(d.probe_inc, cap * 4); add(d.sus_start, cap * 4);
  add(d.sus_from, cap * 4 * GS_K1MAX, GS_K1MAX); add(d.acc, cap * 8 * GS_K1MAX * 2, GS_K1MAX * 2); add(d.change_tick, cap * 4);
  add(d.reap_after, cap * 4);
  add(d.ltime_member, cap * 4); add(d.ltime_event, cap * 4); add(d.event_min, cap * 4);
  add(d.heard, cap * 4); add(d.queued, cap * 4); add(d.tx, cap * GS_MAX_RUMORS, GS_MAX_RUMORS / 2);
  if (d.kst) add(d.kst, cap);
  if (d.coord) {
    add(d.coord, cap * 8 * 2 * GS_COORD_WORDS, 2 * GS_COORD_WORDS);
    add(d.ctag, cap * 4 * 2, 2);
    add(d.adj, cap * 8 * GS_ADJ_WINDOW, GS_ADJ_WINDOW);
    add(d.adj_idx, cap * 4);
  }
  if (d.ppreq) {
    add(d.ppreq, cap * 4 * 2 * GS_PPK, 2 * GS_PPK);
    add(d.pp_clk, cap * 4 * 4, 4);
  }
  if (d.pig) {
    add(d.pig_req, cap * 4 * 2 * GS_PIGK, 2 * GS_PIGK);
    add(d.pig, sizeof(GsPig), 1, false);
  }
  if (with_impairment) {
    add(p->imp_loss, cap * 4);
    add(p->imp_delay, cap);
  }
  if (with_reach) {
    add(p->imp_recv, cap * 4);
    add(p->imp_flags, cap);
  }
  if (with_pause) {
    add(p->pause_until, cap * 4);
    add(p->pause_cnt_dev, 4 * 8, 1, false);
  }
  if (with_flap) add(p->imp_flap, cap * 4);
  if (with_dom) add(p->imp_dom, cap * 4);  // (the schedule table follows the columns: its length, then its words)
  add(d.stats, GSIM_STAT_COUNT * 8, 1, false); add(d.heard_cnt, 32 * 4, 1, false); add(d.conv_tick, 32 * 4, 1, false);
  add(d.crashed_alive, 4, 1, false); add(d.crashed_dead_tick, 4, 1, false);
  return v;
}
struct SnapHeader {
  uint64_t magic;
  uint32_t version, cap;
  uint32_t now, n_sched;
  uint64_t node_ticks;
  uint32_t n_established;
  uint32_t layout;       // which optional column sets the blob carries (snap_layout)
  uint64_t graph_hash;   // FNV-1a of the CSR peer graph the state was produced on (0: complete graph)
  GsGlobals g;
};
static const uint64_t SNAP_MAGIC = 0x4753494D534E4150ull;  // "GSIMSNAP"
static const uint32_t SNAP_VERSION = 3;

// The optional column sets of a pool, as a bit mask: a blob is only ever parsed by a pool with the
// same set (the planes follow each other without per-plane names).
static uint32_t snap_layout(const gsim_pool* p) {
  uint32_t m = 0;
  if (p->d.coord) m |= 1u;
  if (p->d.ppreq) m |= 2u;
  if (p->d.kst) m |= 4u;
  if (p->imp_loss) m |= 8u;  // impairment columns (restore allocates them when the pool has none)
  if (p->sharded) m |= 16u;
  if (p->pause_until) m |= 32u;  // the pause column and statistics (restore allocates them when the pool has none)
  if (p->imp_recv) m |= 64u;     // the reachability columns (with bit 8; restore allocates them when the pool has none)
  if (p->d.pig) m |= 128u;       // owed answers and the piggyback words (GSIM_FLAG_PROBE_PIGGYBACK)
  if (p->imp_flap) m |= 256u;    // the flap schedule column (restore allocates it when the pool has none)
  if (p->imp_dom) m |= 512u;     // the domain column and schedule table (restore allocates the column)
  return m;
}
static uint64_t snap_graph_hash(const gsim_pool* p) {
  if (p->g.graph_n == 0u) return 0ull;
  uint64_t h = 0xCBF29CE484222325ull;
  auto mix = [&](const std::vector<uint32_t>& v) {
    for (uint32_t x : v) {
      h ^= x;
      h *= 0x100000001B3ull;
    }
  };
  mix(p->graph_rp);
  mix(p->graph_col);
  return h ? h : 1ull;
}

static size_t snap_size(gsim_pool* p) {
  size_t s = sizeof(SnapHeader) + p->sched.size() * sizeof(Sched);
  for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r) s += 12 + p->rh[r].name.size() + p->rh[r].payload.size();
  for (const SnapCol& c : snap_cols(p, p->imp_loss != nullptr, p->pause_until != nullptr, p->imp_recv != nullptr,
                                    p->imp_flap != nullptr, p->imp_dom != nullptr))
    s += c.bytes + 4u * c.planes;  // upper bound: every plane raw
  if (p->imp_dom) s += 4u + p->dom_tab.size() * 4u;
  return s;
}

extern "C" int gsim_snapshot_size(gsim_pool* p, size_t* n_bytes) {
  if (!p || !n_bytes) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GS_CONTROLLER_ONLY(p);
  *n_bytes = snap_size(p);
  return GSIM_OK;
}

extern "C" int gsim_snapshot(gsim_pool* p, void* out, size_t cap_bytes, size_t* n_bytes) {
  if (!p || !out) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  GS_CONTROLLER_ONLY(p);
  size_t need = snap_size(p);
  if (n_bytes) *n_bytes = need;
  if (cap_bytes < need) return fail(p, GSIM_ERR_INVALID, "buffer too small");
  uint8_t* w = reinterpret_cast<uint8_t*>(out);
  uint8_t* const w0 = w;
  SnapHeader h;
  memset(&h, 0, sizeof(h));
  h.magic = SNAP_MAGIC;
  h.version = SNAP_VERSION;
  h.layout = snap_layout(p);
  h.graph_hash = snap_graph_hash(p);
  h.cap = p->g.cap;
  h.now = p->now;
  h.n_sched = (uint32_t)p->sched.size();
  h.node_ticks = p->node_ticks;
  h.n_established = p->n_established;
  h.g = p->g;
  memcpy(w, &h, sizeof(h));
  w += sizeof(h);
  if (!p->sched.empty()) memcpy(w, p->sched.data(), p->sched.size() * sizeof(Sched));
  w += p->sched.size() * sizeof(Sched);
  for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r) {
    uint32_t hdr[3] = {(uint32_t)p->rh[r].name.size(), (uint32_t)p->rh[r].payload.size(),
                       (uint32_t)p->rh[r].coalesce};
    memcpy(w, hdr, 12);
    w += 12;
    memcpy(w, p->rh[r].name.data(), hdr[0]);
    w += hdr[0];
    memcpy(w, p->rh[r].payload.data(), hdr[1]);
    w += hdr[1];
  }
  if (p->pause_cnt_dev && !dev(p)->h2d(p->pause_cnt_dev, p->pause_cnt, sizeof(p->pause_cnt)))
    return fail(p, GSIM_ERR_CUDA, "h2d");
  for (const SnapCol& c : snap_cols(p, p->imp_loss != nullptr, p->pause_until != nullptr, p->imp_recv != nullptr,
                                    p->imp_flap != nullptr, p->imp_dom != nullptr)) {
    const size_t pb = c.bytes / c.planes;
    for (uint32_t q = 0; q < c.planes; ++q) {
      uint8_t* raw = w + 4;
      if (!dev(p)->d2h(raw, reinterpret_cast<uint8_t*>(c.ptr) + (size_t)q * pb, pb)) return fail(p, GSIM_ERR_CUDA, "d2h");
      // one repeated word?  (buf[0..n-4) == buf[4..n) iff all 32-bit words are equal)
      const bool uniform = c.may_fill && pb >= 8 && memcmp(raw, raw + 4, pb - 4) == 0;
      const uint32_t tag = uniform ? 1u : 0u;
      memcpy(w, &tag, 4);
      w += 4 + (uniform ? 4 : pb);
    }
  }
  if (p->imp_dom) {
    const uint32_t len = (uint32_t)p->dom_tab.size();
    memcpy(w, &len, 4);
    if (len) memcpy(w + 4, p->dom_tab.data(), (size_t)len * 4);
    w += 4 + (size_t)len * 4;
  }
  if (n_bytes) *n_bytes = (size_t)(w - w0);  // what was actually written (<= gsim_snapshot_size)
  return GSIM_OK;
}

extern "C" int gsim_restore(gsim_pool* p, const void* blob, size_t n_bytes) {
  if (!p || !blob || n_bytes < sizeof(SnapHeader)) return GSIM_ERR_INVALID;
  std::lock_guard<std::mutex> lk(p->mu);
  const int rc_all = controller_call(p, nullptr, 0, [&]() -> int {
  const uint8_t* r = reinterpret_cast<const uint8_t*>(blob);
  const uint8_t* end = r + n_bytes;
  SnapHeader h;
  memcpy(&h, r, sizeof(h));
  r += sizeof(h);
  if (h.magic != SNAP_MAGIC || h.version != SNAP_VERSION) return fail(p, GSIM_ERR_INVALID, "not a gsim snapshot of this version");
  // The blob is trusted for nothing that selects memory: stride, member count, column set, sharding
  // geometry and peer graph must be this pool's before a single plane is copied.
  if (h.cap != p->g.cap || h.g.cap != p->g.cap || h.g.n > p->cfg.capacity || h.g.n > p->g.cap ||
      h.g.ring_mask != p->g.ring_mask || (h.g.pp_interval != 0u) != (p->g.pp_interval != 0u) ||
      (h.layout & ~872u) != (snap_layout(p) & ~872u) || (h.layout & 72u) == 64u || h.g.world != p->g.world || h.g.key_stride != p->g.key_stride ||
      h.g.rows_per_rank != p->g.rows_per_rank || h.g.phase_group != p->g.phase_group ||
      h.g.graph_n != p->g.graph_n || h.graph_hash != snap_graph_hash(p) || h.n_established > h.g.n)
    return fail(p, GSIM_ERR_INVALID, "snapshot does not match this pool (capacity, column set, sharding or peer graph)");
  if ((size_t)(end - r) < (size_t)h.n_sched * sizeof(Sched)) return fail(p, GSIM_ERR_INVALID, "truncated");
  p->sched.resize(h.n_sched);
  if (h.n_sched) memcpy(p->sched.data(), r, (size_t)h.n_sched * sizeof(Sched));
  r += (size_t)h.n_sched * sizeof(Sched);
  for (uint32_t x = 0; x < GS_MAX_RUMORS; ++x) {
    if (end - r < 12) return fail(p, GSIM_ERR_INVALID, "truncated");
    uint32_t hdr[3];
    memcpy(hdr, r, 12);
    r += 12;
    if ((size_t)(end - r) < (size_t)hdr[0] + hdr[1]) return fail(p, GSIM_ERR_INVALID, "truncated");
    p->rh[x].name.assign((const char*)r, hdr[0]);
    r += hdr[0];
    p->rh[x].payload.assign((const char*)r, hdr[1]);
    r += hdr[1];
    p->rh[x].coalesce = (int)hdr[2];
  }
  const bool blob_impaired = (h.layout & 8u) != 0u;
  if (blob_impaired && !impair_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "impairment columns");
  const bool blob_reach = (h.layout & 64u) != 0u;
  if (blob_reach && !reach_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "reachability columns");
  const bool blob_paused = (h.layout & 32u) != 0u;
  if (blob_paused && !pause_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "pause column");
  const bool blob_flap = (h.layout & 256u) != 0u;
  if (blob_flap && !flap_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "schedule column");
  const bool blob_dom = (h.layout & 512u) != 0u;
  if (blob_dom && !domain_alloc(p)) return fail(p, GSIM_ERR_NOMEM, "domain column");
  for (const SnapCol& c : snap_cols(p, blob_impaired, blob_paused, blob_reach, blob_flap, blob_dom)) {
    if (c.may_fill) {  // plane by plane: a device fill or a copy
      const size_t pb = c.bytes / c.planes;
      for (uint32_t q = 0; q < c.planes; ++q) {
        if (end - r < 8) return fail(p, GSIM_ERR_INVALID, "truncated");
        uint32_t tag, word;
        memcpy(&tag, r, 4);
        memcpy(&word, r + 4, 4);
        uint8_t* dst = reinterpret_cast<uint8_t*>(c.ptr) + (size_t)q * pb;
        if (tag == 1u) {
          if (!dev(p)->fill32(reinterpret_cast<uint32_t*>(dst), word, pb / 4)) return fail(p, GSIM_ERR_CUDA, "fill");
          r += 8;
        } else if (tag == 0u) {
          if ((size_t)(end - r) < 4 + pb) return fail(p, GSIM_ERR_INVALID, "truncated");
          if (!dev(p)->h2d_async(dst, r + 4, pb)) return fail(p, GSIM_ERR_CUDA, "h2d");
          r += 4 + pb;
        } else {
          return fail(p, GSIM_ERR_INVALID, "corrupt snapshot");
        }
      }
      continue;
    }
    if ((size_t)(end - r) < 4 + c.bytes) return fail(p, GSIM_ERR_INVALID, "truncated");
    r += 4;  // tag 0 (these columns are always stored raw)
    if (!dev(p)->h2d_async(c.ptr, r, c.bytes)) return fail(p, GSIM_ERR_CUDA, "h2d");
    if (p->sharded && (c.ptr == p->d.key[0] || c.ptr == p->d.key[1])) {
      // the key column is replicated per rank: restore every replica
      uint32_t* rep0 = c.ptr == p->d.key[0] ? p->d.key_rep[0] : p->d.key_rep[1];
      for (uint32_t q = 0; q < p->world; ++q)
        if (!dev(p)->h2d_async(rep0 + (size_t)q * p->g.key_stride, r, c.bytes)) return fail(p, GSIM_ERR_CUDA, "h2d");
    }
    if (p->sharded && c.ptr == (void*)p->d.stats) {
      // counters restore into rank 0's page; the other ranks' partial sums restart at zero
      std::vector<uint8_t> zeros(c.bytes, 0);
      for (uint32_t q = 1; q < p->world; ++q)
        if (!dev(p)->h2d(p->pages + (size_t)q * GS_PAGE_BYTES + GS_PG_STATS, zeros.data(), c.bytes)) return fail(p, GSIM_ERR_CUDA, "h2d");
    }
    r += c.bytes;
  }
  // a blob without impairment columns restores a pool nobody in it is impaired
  if (!blob_impaired && p->imp_loss &&
      (!dev(p)->fill32(p->imp_loss, 0, p->g.cap) || !dev(p)->fill8(p->imp_delay, 0, p->g.cap)))
    return fail(p, GSIM_ERR_CUDA, "fill");
  // ... and one without the pause column a pool nobody in it is paused
  if (!blob_paused && p->pause_until && !dev(p)->fill32(p->pause_until, 0u, p->g.cap)) return fail(p, GSIM_ERR_CUDA, "fill");
  // ... and one without the schedule column a pool in which nobody has a schedule
  if (!blob_flap && p->imp_flap && !dev(p)->fill32(p->imp_flap, 0u, p->g.cap)) return fail(p, GSIM_ERR_CUDA, "fill");
  // ... and one without domains a pool in which nobody has a domain and no domain a schedule
  p->dom_tab.clear();
  if (blob_dom) {
    uint32_t len = 0;
    if (end - r < 4) return fail(p, GSIM_ERR_INVALID, "truncated");
    memcpy(&len, r, 4);
    if (len > GS_DOMAIN_MAX + 1u || (size_t)(end - r - 4) < (size_t)len * 4) return fail(p, GSIM_ERR_INVALID, "truncated");
    p->dom_tab.assign(len, 0u);
    if (len) memcpy(p->dom_tab.data(), r + 4, (size_t)len * 4);
    r += 4 + (size_t)len * 4;
  } else if (p->imp_dom && !dev(p)->fill32(p->imp_dom, 0u, p->g.cap)) {
    return fail(p, GSIM_ERR_CUDA, "fill");
  }
  if (!dev(p)->sync()) return fail(p, GSIM_ERR_CUDA, "sync");  // every plane has left the caller's blob
  // ... and one without the reachability columns a pool whose settings are all symmetric
  if (!blob_reach && p->imp_recv) {
    std::vector<uint32_t> loss(p->g.cap);
    if (!dev(p)->d2h(loss.data(), p->imp_loss, loss.size() * 4) || !dev(p)->h2d(p->imp_recv, loss.data(), loss.size() * 4) ||
        !dev(p)->fill8(p->imp_flags, 0, p->g.cap))
      return fail(p, GSIM_ERR_CUDA, "copy");
  }
  memset(p->pause_cnt, 0, sizeof(p->pause_cnt));
  if (blob_paused && !dev(p)->d2h(p->pause_cnt, p->pause_cnt_dev, sizeof(p->pause_cnt))) return fail(p, GSIM_ERR_CUDA, "d2h");
  {
    // topology fields stay the live pool's (they were checked equal above, except the rank, which is
    // this process's own on a sharded pool)
    const uint32_t world = p->g.world, rank = p->g.rank, stride = p->g.key_stride, rpr = p->g.rows_per_rank;
    p->g = h.g;
    p->g.world = world;
    p->g.rank = rank;
    p->g.key_stride = stride;
    p->g.rows_per_rank = rpr;
  }
  p->now = h.now;
  p->node_ticks = h.node_ticks;
  p->n_established = h.n_established;
  p->g_dirty = true;
  counts_invalidate(p);
  if (!impair_recount(p) || !flap_recount(p) || !domain_tab_upload(p)) return fail(p, GSIM_ERR_CUDA, "d2h");
  if (!poke(p, p->d.tick_base, 0, p->now) || !reset_tick_flags(p) || !reset_qstate(p)) return fail(p, GSIM_ERR_CUDA, "poke");
  uint32_t zero2[2] = {0, 0};
  if (!dev(p)->h2d(p->d.evlog_cursor, zero2, 8)) return fail(p, GSIM_ERR_CUDA, "h2d");
  return GSIM_OK;
  });
  dev(p)->sync();  // whatever happened, no copy out of the caller's blob is still in flight
  return rc_all;
}

// ---- measurement hooks ------------------------------------------------------------
extern "C" int gsim_last_step_timing(gsim_pool* p, double* kernel_ms, uint64_t* launches) {
  if (!p) return GSIM_ERR_INVALID;
  if (kernel_ms) *kernel_ms = p->last_ms;
  if (launches) *launches = p->last_launches;
  return GSIM_OK;
}

extern "C" uint64_t gsim_launch_count(gsim_pool* p) { return p && p->be ? dev(p)->total_launches() : 0; }

// ---- wire formats (include/gsim.h; encoders in gs_wire.h) ---------------------------------------
static size_t zlen(const char* s) { return s ? strlen(s) : 0; }
extern "C" size_t gsim_wire_alive(void* out, size_t cap, uint32_t incarnation, const char* node, const void* addr,
                                  size_t addr_len, uint16_t port, const void* meta, size_t meta_len, const uint8_t vsn[6]) {
  static const uint8_t vsn0[6] = {0, 0, 0, 0, 0, 0};
  return gsw::alive(out, cap, incarnation, node, zlen(node), addr, addr_len, port, meta, meta_len, vsn ? vsn : vsn0);
}
extern "C" size_t gsim_wire_suspect(void* out, size_t cap, uint32_t incarnation, const char* node, const char* from) {
  return gsw::suspect_or_dead(out, cap, false, incarnation, node, zlen(node), from, zlen(from));
}
extern "C" size_t gsim_wire_dead(void* out, size_t cap, uint32_t incarnation, const char* node, const char* from) {
  return gsw::suspect_or_dead(out, cap, true, incarnation, node, zlen(node), from, zlen(from));
}
extern "C" size_t gsim_wire_join_intent(void* out, size_t cap, uint64_t ltime, const char* node) {
  return gsw::serf_intent(out, cap, false, ltime, node, zlen(node), false, false);
}
extern "C" size_t gsim_wire_leave_intent(void* out, size_t cap, uint64_t ltime, const char* node, int prune) {
  return gsw::serf_intent(out, cap, true, ltime, node, zlen(node), prune != 0, false);
}
extern "C" size_t gsim_wire_user_event(void* out, size_t cap, uint64_t ltime, const void* name, size_t name_len,
                                       const void* payload, size_t payload_len, int coalesce) {
  return gsw::serf_user_event(out, cap, ltime, name, name_len, payload, payload_len, coalesce != 0, false);
}
extern "C" size_t gsim_wire_compound(void* out, size_t cap, const void* const* msgs, const size_t* lens, size_t count) {
  if (count > 255 || (count && (!msgs || !lens))) return 0;
  return gsw::compound(out, cap, msgs, lens, count);
}
extern "C" size_t gsim_wire_wanfed_frame(void* out, size_t cap, const void* packet, size_t len) {
  return gsw::wanfed_frame(out, cap, packet, len);
}
extern "C" size_t gsim_wire_ping(void* out, size_t cap, uint32_t seq_no, const char* node, const void* source_addr,
                                 size_t source_addr_len, uint16_t source_port, const char* source_node) {
  return gsw::ping(out, cap, seq_no, node, zlen(node), source_addr, source_addr_len, source_port, source_node,
                   zlen(source_node));
}
extern "C" size_t gsim_wire_indirect_ping(void* out, size_t cap, uint32_t seq_no, const void* target, size_t target_len,
                                          uint16_t port, const char* node, int nack, const void* source_addr,
                                          size_t source_addr_len, uint16_t source_port, const char* source_node) {
  return gsw::indirect_ping(out, cap, seq_no, target, target_len, port, node, zlen(node), nack != 0, source_addr,
                            source_addr_len, source_port, source_node, zlen(source_node));
}
extern "C" size_t gsim_wire_ack(void* out, size_t cap, uint32_t seq_no, const void* payload, size_t payload_len) {
  return gsw::ack(out, cap, seq_no, payload, payload_len);
}
extern "C" size_t gsim_wire_nack(void* out, size_t cap, uint32_t seq_no) { return gsw::nack(out, cap, seq_no); }
extern "C" size_t gsim_wire_consul_user_event(void* out, size_t cap, const char* id, const char* name,
                                              const void* payload, size_t payload_len, const char* node_filter,
                                              const char* service_filter, const char* tag_filter, int version) {
  return gsw::consul_user_event(out, cap, id ? id : "", name ? name : "", payload, payload_len, node_filter,
                                service_filter, tag_filter, version);
}
