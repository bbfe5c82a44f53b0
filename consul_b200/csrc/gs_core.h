// gs_core.h — state layout, packing helpers and counter-based RNG shared by the CUDA
// kernels (gs_kernels.cu) and the host side of libgsim (gs_api.cpp).
//
// Data layout in HBM (SoA, one element per virtual member, index = member id):
//   HOT, read by every row every tick (16 B / node-tick):
//     key[2][N]   u32  double-buffered cluster view of the member as SUBJECT:
//                      inc<<5 | pending<<4 | rank<<2 | truth     (a1, a6-a9 in SURVEY 8a)
//     inbox[2][N] u32  per-arrival-tick mailbox: bit r = rumor r delivered, bit 31 =
//                      accusation(s) pending in acc[][][]         (transport, §5)
//     due[N]      u32  tick of the member's next probe action      (a2, a3)
//     meta[N]     u32  awareness | probe stage | nack misses | dirty | flags | gossip phase
//   COLD, touched only by rows that act in this tick:
//     cursor/pass/probe_tgt/probe_inc   probe ring position and the in-flight probe
//     sus_start, sus_from[K1][N]        Lifeguard suspicion record of the subject (a7)
//     acc[2][K1][N] u64                 accusation mailbox, (~inc<<32 | from), kept as the
//                                       K1 smallest by an atomicMin chain (commutative)
//     change_tick                       tick the subject became Dead/Left
//     ltime_member, ltime_event, event_min   serf Lamport clocks (a13)
//     heard, queued (u32 masks), tx[R][N] u8 TransmitLimitedQueue per tracked rumor (a5)
#pragma once
#include <stdint.h>

#if defined(__CUDACC__)
#define GS_HD __host__ __device__ __forceinline__
#else
#define GS_HD inline
#endif

#define GS_MAX_RUMORS 30
#define GS_MAX_WORLD_ 8
#define GS_K1MAX 5
#define GS_RING_MAX 8            // deepest mailbox ring (WAN latency pools): latency <= GS_RING_MAX - 1
#define GS_MAX_DCS 64u           // synthetic datacenters of a latency pool (BASELINE config 5)
#define GS_ACC_BIT 0x80000000u   // inbox: auxiliary mail — accusation(s) pending in acc[][][] and/or
                                 // push-pull requests / clocks in ppreq[][][] / pp_clk[][][]
#define GS_PPK 4                 // push-pull requests one member serves per tick (smallest ids win)
#define GS_WAKE_BIT 0x40000000u  // inbox: "process this row" (self-posted or by the host)
// Invariant: a member with queued != 0 has a wake pending at or before its next gossip tick (the row
// step posts it for that tick, gs_queue_wake_slot; the host posts it for `now` whenever it queues).
// A running suspicion timer or a stale key buffer (GS_META_DIRTY) has a wake pending for the next tick.
#define GS_TILE 128u             // rows per CTA; ticker phases are uniform per tile
#define GS_NEVER 0xFFFFFFFFu
#define GS_EMPTY32 0xFFFFFFFFu
#define GS_EMPTY64 0xFFFFFFFFFFFFFFFFull
#define GS_KR_MAX_TRIES 32u  // kRandomNodes tries = min(3n, 32); upstream: 3n
#define GS_PROBE_SKIP_CAP 1024u

// truth / rank values are the public GSIM_TRUTH_* / GSIM_RANK_* constants.
enum { GS_TRUTH_NONE = 0, GS_TRUTH_UP = 1, GS_TRUTH_CRASHED = 2, GS_TRUTH_GONE = 3 };
enum { GS_RANK_ALIVE = 0, GS_RANK_SUSPECT = 1, GS_RANK_DEAD = 2, GS_RANK_LEFT = 3 };
enum { GS_STAGE_IDLE = 0, GS_STAGE_WAIT_T = 1, GS_STAGE_WAIT_P = 2 };
// tracked-broadcast kinds and event types: the public GSIM_RUMOR_* / GSIM_EVENT_* values
enum { GS_RUMOR_ALIVE = 1, GS_RUMOR_JOIN_INTENT = 2, GS_RUMOR_LEAVE_INTENT = 3, GS_RUMOR_USER_EVENT = 4, GS_RUMOR_UPDATE = 5 };
enum { GS_EV_MEMBER_JOIN = 0, GS_EV_MEMBER_FAILED = 2, GS_EV_MEMBER_UPDATE = 3, GS_EV_MEMBER_REAP = 4, GS_EV_USER = 5 };

// Philox counter "purpose" words.
enum {
  GS_PUR_PHASE = 1,
  GS_PUR_PERM = 2,
  GS_PUR_GOSSIP = 3,
  GS_PUR_RELAY = 4,
  GS_PUR_LOSS = 5,
  GS_PUR_CRASH = 6,
  GS_PUR_PUSHPULL = 7,
  // 8 = GS_PUR_COORD (gs_coord.h)
  GS_PUR_IMPAIR = 9,
  GS_PUR_PAUSE = 10,
  // 11 = gsim_coordinate_error's sample draws (GS_PUR_COORD_SAMPLE)
  GS_PUR_FLAP = 12,
  GS_PUR_FLAP_DOMAIN = 13
};
// Loss "kind" (folded into the counter) — one draw per simulated UDP packet.
enum {
  GS_LK_PING = 0,
  GS_LK_ACK = 1,
  GS_LK_INDREQ = 2,
  GS_LK_INDPING = 3,
  GS_LK_INDACK = 4,
  GS_LK_INDFWD = 5,
  GS_LK_NACK = 6,
  GS_LK_GOSSIP = 7
};

// ---- key word -------------------------------------------------------------
GS_HD uint32_t gs_key_make(uint32_t inc, uint32_t pending, uint32_t rank, uint32_t truth) {
  return (inc << 5) | (pending << 4) | (rank << 2) | truth;
}
GS_HD uint32_t gs_key_truth(uint32_t k) { return k & 3u; }
GS_HD uint32_t gs_key_rank(uint32_t k) { return (k >> 2) & 3u; }
GS_HD uint32_t gs_key_pending(uint32_t k) { return (k >> 4) & 1u; }
GS_HD uint32_t gs_key_inc(uint32_t k) { return k >> 5; }
GS_HD uint32_t gs_key_with_rank(uint32_t k, uint32_t rank) { return (k & ~(3u << 2)) | (rank << 2); }
GS_HD uint32_t gs_key_with_inc(uint32_t k, uint32_t inc) { return (k & 31u) | (inc << 5); }
// Status replica: what a prober or gossiper needs to know about a peer is its
// truth and rank — 4 bits — not its 27-bit incarnation.  At 64 Mi members the key column is 256 MB
// per buffer and every random 4-byte gather costs a DRAM sector; one status byte per member holds
// both buffers' views in 64 MB, a quarter of the key column (the 50 MB L2 of an H100 holds most of
// it, and the backend pins what fits with a persisting access-policy window).  Code = rank<<2 | truth,
// 0 = no such member, GS_KST_PENDING (rank 1, truth 0: otherwise meaningless) = "pending joiner,
// read the full key".
#define GS_KST_PENDING 4u
GS_HD uint32_t gs_kst_code(uint32_t k) {
  if ((k & 3u) == 0u) return 0u;
  if ((k >> 4) & 1u) return GS_KST_PENDING;
  return k & 15u;
}

// ---- meta word ------------------------------------------------------------
#define GS_META_AW_MASK 0x7u
#define GS_META_STAGE_SHIFT 3
#define GS_META_NMISS_SHIFT 5
#define GS_META_DIRTY (1u << 8)
#define GS_META_LEAVING (1u << 9)
#define GS_META_WATCHED (1u << 10)
#define GS_META_ISOLATED (1u << 11)  // created but has not completed a Join yet
#define GS_META_GPHASE_SHIFT 16
GS_HD uint32_t gs_meta_aw(uint32_t m) { return m & GS_META_AW_MASK; }
GS_HD uint32_t gs_meta_stage(uint32_t m) { return (m >> GS_META_STAGE_SHIFT) & 3u; }
GS_HD uint32_t gs_meta_nmiss(uint32_t m) { return (m >> GS_META_NMISS_SHIFT) & 7u; }
GS_HD uint32_t gs_meta_gphase(uint32_t m) { return (m >> GS_META_GPHASE_SHIFT) & 0xFFu; }
GS_HD uint32_t gs_meta_set_aw(uint32_t m, uint32_t aw) { return (m & ~GS_META_AW_MASK) | aw; }
GS_HD uint32_t gs_meta_set_stage(uint32_t m, uint32_t s) {
  return (m & ~(3u << GS_META_STAGE_SHIFT)) | (s << GS_META_STAGE_SHIFT);
}
GS_HD uint32_t gs_meta_set_nmiss(uint32_t m, uint32_t n) {
  return (m & ~(7u << GS_META_NMISS_SHIFT)) | ((n & 7u) << GS_META_NMISS_SHIFT);
}

// ---- Philox4x32-10 (Salmon et al., SC'11), counter based: no RNG state in HBM ----
GS_HD uint32_t gs_mulhi(uint32_t a, uint32_t b) {
#if defined(__CUDA_ARCH__)
  return __umulhi(a, b);
#else
  return (uint32_t)(((uint64_t)a * (uint64_t)b) >> 32);
#endif
}
struct GsU4 {
  uint32_t x, y, z, w;
};
GS_HD GsU4 gs_philox(uint32_t k0, uint32_t k1, uint32_t c0, uint32_t c1, uint32_t c2,
                     uint32_t c3) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t hi0 = gs_mulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    uint32_t hi1 = gs_mulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0;
    c1 = n1;
    c2 = n2;
    c3 = n3;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  GsU4 o;
  o.x = c0;
  o.y = c1;
  o.z = c2;
  o.w = c3;
  return o;
}
// ---- ticker stagger ([U] memberlist/state.go triggerFunc: rand % interval per agent) ----
// The stagger only has to spread the tickers evenly over their interval, so phases are
// dealt round-robin over consecutive phase groups, rotated by a seed-derived offset:
//   probe phase  = (group + rot_p) mod P,   gossip phase = (group / P + rot_g) mod GI.
// Any run of consecutive tiles then holds every phase equally often, which is what lets the
// tick kernel give each warp a contiguous chunk of tiles with a perfectly balanced number of
// probing tiles — no work stealing, no atomics.
GS_HD uint32_t gs_fmix32(uint32_t x) {  // murmur3 finaliser
  x ^= x >> 16;
  x *= 0x85EBCA6Bu;
  x ^= x >> 13;
  x *= 0xC2B2AE35u;
  x ^= x >> 16;
  return x;
}
GS_HD uint32_t gs_phase_rot(uint32_t seed_lo, uint32_t seed_hi) {
  return gs_fmix32(seed_lo * 0x9E3779B1u + seed_hi);
}
GS_HD uint32_t gs_probe_phase(uint32_t rot_p, uint32_t group, uint32_t P) {
  return (group % P + rot_p) % P;
}
GS_HD uint32_t gs_gossip_phase(uint32_t rot_g, uint32_t group, uint32_t P, uint32_t GI) {
  return ((group / P) % GI + rot_g) % GI;
}

// Push-pull ticker of a phase group ([U] memberlist/state.go schedule: pushPullTrigger with a random
// stagger): groups are dealt round-robin over the interval like the probe phases.
GS_HD bool gs_pp_due(uint32_t pp_interval, uint32_t rot_pp, uint32_t group, uint32_t t) {
  return pp_interval != 0u && (t + rot_pp) % pp_interval == group % pp_interval;
}

// x mod n with the precomputed magic = ceil(2^64 / n)
GS_HD uint32_t gs_fastmod(uint32_t x, uint32_t n, uint64_t magic) {
  const uint64_t low = magic * (uint64_t)x;
#if defined(__CUDA_ARCH__)
  return (uint32_t)__umul64hi(low, (uint64_t)n);
#else
  return (uint32_t)(((unsigned __int128)low * n) >> 64);
#endif
}

GS_HD uint32_t gs_u4_get(const GsU4& v, uint32_t idx) {
  return idx == 0 ? v.x : idx == 1 ? v.y : idx == 2 ? v.z : v.w;
}

// ---- probe ring: keyed Feistel permutation of [0, n) with cycle walking ------
// Replaces the O(N)-per-member shuffled `nodes` slice ([U] memberlist/state.go
// resetNodes/shuffleNodes): every member visits every peer exactly once per pass,
// in a per-(member, pass) pseudo-random order, with O(1) state (cursor, pass).
GS_HD uint32_t gs_feistel_round(uint32_t r, uint32_t k) {
  uint32_t x = (r + k) * 0x9E3779B1u;
  x ^= x >> 15;
  x *= 0x85EBCA77u;
  x ^= x >> 13;
  return x;
}
// Round keys of one (member, pass) ring: two murmur finalisers, two cheap combinations.
GS_HD GsU4 gs_perm_keys(uint32_t seed_lo, uint32_t seed_hi, uint32_t member, uint32_t pass) {
  GsU4 k;
  k.x = gs_fmix32(member * 0x9E3779B1u + pass * 0x85EBCA77u + seed_lo);
  k.y = gs_fmix32(k.x ^ seed_hi ^ 0xC2B2AE3Du);
  k.z = k.x * 0x9E3779B1u + k.y;
  k.w = (k.y * 0x85EBCA77u) ^ k.x;
  return k;
}
// bit width of the smallest power of two >= n (>= 4): the Feistel domain.  The two halves may differ by
// one bit (an "unbalanced" Feistel network: each round XORs one half with a keyed function of the other,
// halves alternating — a bijection for any pair of widths), so the domain is never more than twice n and
// cycle walking takes < 2 rounds on average for every n, not only for those just below an even power of
// two.  With equal halves this is exactly the classic swap-and-XOR network.
GS_HD uint32_t gs_perm_bits_of(uint32_t n) {
  uint32_t bits = 2u;
  while (bits < 32u && (1ull << bits) < (unsigned long long)n) ++bits;
  return bits;
}
GS_HD uint32_t gs_perm(uint32_t x, uint32_t n, uint32_t bits, const GsU4& rk) {
  const uint32_t lo_bits = bits >> 1, hi_bits = bits - lo_bits;
  const uint32_t lo_mask = (1u << lo_bits) - 1u, hi_mask = (1u << hi_bits) - 1u;
  do {
    uint32_t hi = x >> lo_bits, lo = x & lo_mask;
    hi ^= gs_feistel_round(lo, rk.x) & hi_mask;
    lo ^= gs_feistel_round(hi, rk.y) & lo_mask;
    hi ^= gs_feistel_round(lo, rk.z) & hi_mask;
    lo ^= gs_feistel_round(hi, rk.w) & lo_mask;
    x = (hi << lo_bits) | lo;
  } while (x >= n);
  return x;
}

// The position of ring entry y: the inverse network, walked the same way (F^-1 until it lands inside [0, n)).
GS_HD uint32_t gs_perm_inv(uint32_t y, uint32_t n, uint32_t bits, const GsU4& rk) {
  const uint32_t lo_bits = bits >> 1, hi_bits = bits - lo_bits;
  const uint32_t lo_mask = (1u << lo_bits) - 1u, hi_mask = (1u << hi_bits) - 1u;
  do {
    uint32_t hi = y >> lo_bits, lo = y & lo_mask;
    lo ^= gs_feistel_round(hi, rk.w) & lo_mask;
    hi ^= gs_feistel_round(lo, rk.z) & hi_mask;
    lo ^= gs_feistel_round(hi, rk.y) & lo_mask;
    hi ^= gs_feistel_round(lo, rk.x) & hi_mask;
    y = (hi << lo_bits) | lo;
  } while (y >= n);
  return y;
}

// Quiet windows of a PRISTINE pool (every member running, listed alive by everybody, established, every
// link within ProbeTimeout, no loss): whoever a probe hits, it is acknowledged at once, so the outcome of
// a member's next k probes does not depend on the k ring entries — cursor + k, due + k ProbeIntervals,
// awareness - k (floored at 0) — and k is bounded by the launch, by the end of the ring pass, and by the
// member's own entry in its ring (which the generic step skips): one inverse permutation instead of k
// forward ones and k status gathers.  Returns k for a member whose ticker fires at `due` < w1.
// (`k` on entry = ticker firings inside the launch, ceil((w1 - due) / P))
GS_HD uint32_t gs_pristine_probes_k(uint32_t n, uint32_t bits, const GsU4& rk, uint32_t self, uint32_t cursor, uint32_t k,
                                    const uint32_t* special, uint32_t n_special) {
  if (cursor >= n) return 0u;  // ring wrap: re-keyed by the generic step
  if (n - cursor < k) k = n - cursor;
  uint32_t pos = gs_perm_inv(self, n, bits, rk);
  if (pos >= cursor && pos - cursor < k) k = pos - cursor;
  // members that are not established yet (subjects of alive rumors still tracked): whether a prober
  // knows them is in its heard mask — the generic step's business, like the prober's own entry
  for (uint32_t x = 0; x < n_special; ++x) {
    if (special[x] >= n || special[x] == self) continue;
    pos = gs_perm_inv(special[x], n, bits, rk);
    if (pos >= cursor && pos - cursor < k) k = pos - cursor;
  }
  return k;
}
GS_HD uint32_t gs_pristine_probes(uint32_t n, uint32_t bits, const GsU4& rk, uint32_t self, uint32_t cursor,
                                  uint32_t due, uint32_t w1, uint32_t P, const uint32_t* special, uint32_t n_special) {
  return gs_pristine_probes_k(n, bits, rk, self, cursor, (w1 - due + P - 1u) / P, special, n_special);
}

#define GS_IMPAIR_NO_TCP 1u  // GSIM_IMPAIR_NO_TCP: every TCP exchange to or from the member fails

// The impairment columns of a pool (gsim_impair_*, gsim_impair_dir_*): loss = the send threshold, recv and
// flags null until the first directional setting allocates them (then recv = loss is the symmetric case).
struct GsImpairCols {
  uint32_t* loss;
  uint32_t* recv;
  uint8_t* delay;
  uint8_t* flags;
};
// The setting written into them: send / receive thresholds, receive delay, GSIM_IMPAIR_* flags.
struct GsImpairVal {
  uint32_t send, recv, delay, flags;
};

// gsim_impair_fraction / gsim_impair_dir_fraction for member i whose key word (either buffer: truth is in
// both) is key: a member that runs and whose Philox draw (its own purpose word, so the selection is
// independent of gs_crash_row's for the same salt) is below thr gets the impairment v (recv and flags only
// where those columns exist, gs_impair_write: returns whether member i was impaired before).  Returns bit 0 =
// selected, bit 1 = it was impaired before.
GS_HD bool gs_impair_write(const GsImpairCols& c, uint32_t i, const GsImpairVal& v) {
  const bool was = c.loss[i] != 0u || c.delay[i] != 0u || (c.recv != nullptr && c.recv[i] != 0u) ||
                   (c.flags != nullptr && c.flags[i] != 0u);
  c.loss[i] = v.send;
  c.delay[i] = (uint8_t)v.delay;
  if (c.recv != nullptr) c.recv[i] = v.recv;
  if (c.flags != nullptr) c.flags[i] = (uint8_t)v.flags;
  return was;
}
GS_HD uint32_t gs_impair_row(uint32_t key, const GsImpairCols& c, uint32_t seed_lo, uint32_t seed_hi, uint32_t i,
                             uint32_t thr, uint32_t salt, const GsImpairVal& v) {
  if ((key & 3u) != GS_TRUTH_UP) return 0u;
  if (gs_philox(seed_lo, seed_hi, i, salt, GS_PUR_IMPAIR, 0u).x >= thr) return 0u;
  return gs_impair_write(c, i, v) ? 3u : 1u;
}

// Intermittent impairment (gsim_impair_flap_*): a member's schedule word is period << 20 | bad_ppm, 0 for
// none.  Time is cut into epochs of `period` ticks, shifted per member by a phase drawn once; each epoch is
// bad with probability bad_ppm / 1e6, and the member's impairment is in force only during bad epochs.
#define GS_FLAP_PPM_BITS 20u
#define GS_FLAP_MAX_PERIOD 4095u
GS_HD uint32_t gs_flap_word(uint32_t period, uint32_t bad_ppm) { return period << GS_FLAP_PPM_BITS | bad_ppm; }

// Is the epoch of tick t bad under schedule word w (w != 0) for key k drawn under purpose word pur?  phase =
// philox(k, ~0, pur).y mod period; epoch = (t + phase) / period in 64 bits; bad iff philox(k, epoch, pur).x <
// thr(bad_ppm), the ppm threshold floor(ppm 2^32 / 1e6), except that 1e6 is bad in every epoch.  Members
// (gs_flap_bad) and fault domains (gs_domain_flap_bad) draw their epochs here, each under its own purpose word.
GS_HD bool gs_epoch_bad(uint32_t seed_lo, uint32_t seed_hi, uint32_t k, uint32_t pur, uint32_t w, uint32_t t) {
  const uint32_t period = w >> GS_FLAP_PPM_BITS, ppm = w & ((1u << GS_FLAP_PPM_BITS) - 1u);
  if (ppm >= 1000000u) return true;
  if (ppm == 0u) return false;
  const uint32_t phase = gs_philox(seed_lo, seed_hi, k, 0xFFFFFFFFu, pur, 0u).y % period;
  // (t + phase) / period without a 64-bit division: t = q period + r, and r + phase < 2 period
  const uint32_t q = t / period, r = t - q * period;
  const uint32_t epoch = q + (r + phase >= period ? 1u : 0u);
  const uint32_t thr = (uint32_t)(((uint64_t)ppm << 32) / 1000000u);
  return gs_philox(seed_lo, seed_hi, k, epoch, pur, 0u).x < thr;
}

// Is member m in a bad epoch of its own schedule w at tick t?
GS_HD bool gs_flap_bad(uint32_t seed_lo, uint32_t seed_hi, uint32_t m, uint32_t w, uint32_t t) {
  return gs_epoch_bad(seed_lo, seed_hi, m, GS_PUR_FLAP, w, t);
}

// Fault domains (gsim_domain_*): each member has a domain id (0 = none, 1 .. GS_DOMAIN_MAX), and a domain may
// have a schedule word of the same format as a member's.  Is domain dom in a bad epoch of w at tick t?
#define GS_DOMAIN_MAX ((1u << 22) - 1u)
GS_HD bool gs_domain_flap_bad(uint32_t seed_lo, uint32_t seed_hi, uint32_t dom, uint32_t w, uint32_t t) {
  return gs_epoch_bad(seed_lo, seed_hi, dom, GS_PUR_FLAP_DOMAIN, w, t);
}

// The two layers of intermittent impairment: member m's impairment is in force at t iff its own schedule wm
// is absent (0) or bad at t, and its domain's schedule wd is absent (0: no domain, or a domain without one)
// or bad at t.
GS_HD bool gs_in_force(uint32_t seed_lo, uint32_t seed_hi, uint32_t m, uint32_t wm, uint32_t dom, uint32_t wd,
                       uint32_t t) {
  return (wm == 0u || gs_flap_bad(seed_lo, seed_hi, m, wm, t)) &&
         (wd == 0u || gs_domain_flap_bad(seed_lo, seed_hi, dom, wd, t));
}

// gsim_impair_flap_fraction for member i: the selection of gs_impair_row (same draw, so a salt picks the
// same members), writing schedule word w.  Returns bit 0 = selected, bit 1 = it had a schedule before.
GS_HD uint32_t gs_flap_row(uint32_t key, uint32_t* col, uint32_t seed_lo, uint32_t seed_hi, uint32_t i, uint32_t thr,
                           uint32_t salt, uint32_t w) {
  if ((key & 3u) != GS_TRUTH_UP) return 0u;
  if (gs_philox(seed_lo, seed_hi, i, salt, GS_PUR_IMPAIR, 0u).x >= thr) return 0u;
  const bool was = col[i] != 0u;
  col[i] = w;
  return was ? 3u : 1u;
}

// Retransmit counter of rumor r at member i.  Two rumors share one 16-bit element so that the
// narrowest column has 2-byte elements: a sharded pool maps every (column, rank) slice with the
// 2 MB granularity of the virtual-memory API, which then allows 1 Mi members per GPU (1-byte
// planes would need 2 Mi).
#define GS_TX(r, cap, i) ((((size_t)((r) >> 1) * (size_t)(cap) + (size_t)(i)) << 1) + ((r) & 1u))

// ---- tracked rumor table ------------------------------------------------------
struct GsRumor {
  uint32_t kind;     // GSIM_RUMOR_*
  uint32_t subject;  // member id (ALIVE / intents) or origin (user event)
  uint32_t inc;      // incarnation carried by an alive rumor
  uint32_t ltime;    // Lamport time carried by serf messages
  uint32_t origin;
  uint32_t size;     // encoded message bytes (for the UDP budget)
  uint32_t qclass;   // 0 memberlist queue, 1 serf intent queue, 2 serf event queue
  uint32_t start_tick;
};

// Device-resident pool constants; rewritten by the host between steps only.
struct GsGlobals {
  uint32_t n;         // created member ids [0, n)
  uint32_t cap;       // column stride
  uint32_t up_count;  // members with truth == UP
  uint32_t P, T, GI;  // probe interval, probe timeout, gossip interval (ticks)
  uint32_t gossip_nodes, indirect_checks, awareness_max;
  uint32_t retransmit_limit;
  uint32_t sus_k;                // confirmations that shorten the timer
  uint32_t sus_ticks[GS_K1MAX];  // timeout in ticks after c confirmations
  uint32_t gtd_ticks;            // GossipToTheDeadTime
  uint32_t udp_avail;            // UDPBufferSize - compoundHeaderOverhead
  uint32_t disable_tcp;
  uint32_t loss_thr;  // packet lost iff philox < loss_thr (0 = lossless fast path)
  uint32_t event_buffer;
  uint32_t seed_lo, seed_hi;
  uint32_t active_mask;    // non-free rumor slots
  uint32_t class_mask[3];  // rumor slots by queue class
  uint32_t perm_bits;    // gs_perm_bits_of(n)
  uint32_t flags;
  uint32_t evlog_cap;
  uint32_t world, rank;
  uint32_t phase_group;  // members per ticker-phase group (1 or a multiple of GS_TILE)
  uint32_t phase_gate;   // 1: phases are uniform per tile, whole tiles can skip the `due` column
  uint32_t phase_shift;  // phase_group == GS_TILE << phase_shift when phase_gate
  uint32_t rot_p, rot_g; // seed-derived rotation of the probe / gossip phases
  uint32_t rows_per_rank; // sharded pools: rank r owns members [r*rows_per_rank, (r+1)*rows_per_rank)
  uint32_t key_stride;    // sharded pools: elements between the per-rank replicas of the key column
  // WAN latency pools (BASELINE config 5, SURVEY 8d C5).  A packet sent at tick t from a member
  // of datacenter a to one of datacenter b arrives at tick t + 1 + lat[a][b]; mailboxes are a
  // ring of ring_mask + 1 arrival slots.  n_dcs == 0: every packet arrives at t + 1.
  uint32_t ring_mask;     // mailbox ring depth - 1 (depth is a power of two, 2 by default)
  uint32_t n_dcs;         // datacenter of member i = (i / GS_TILE) % n_dcs
  uint8_t lat[GS_MAX_DCS * GS_MAX_DCS];  // EXTRA one-way latency in ticks (matrix entry - 1)
  // Periodic push-pull anti-entropy (SURVEY 8f N1; [U] memberlist/state.go pushPull): the members
  // of phase group q run theirs at ticks t with (t + rot_pp) % pp_interval == q % pp_interval.
  uint32_t pp_interval;   // pushPullScale(PushPullInterval, n) in ticks; 0 = disabled
  uint32_t rot_pp;
  // Peer graph (north_star "CSR peer graph", SURVEY 7): 0 = the complete graph, every member may
  // pick any other; otherwise member i's memberlist is col_idx[row_ptr[i] .. row_ptr[i+1]) and
  // graph_n == n rows are described (static topology: restricted segments, partial views).
  uint32_t graph_n;
  uint32_t reap_min_override;  // smallest per-member ReconnectTimeout override so far (ticks), 0 = none
  uint32_t active_bytes;       // every tracked broadcast with its per-message overhead: <= udp_avail means the
                               // byte budget of a packet can never bind (the common case), whatever is queued
  // network coordinates (gs_coord.h, GSIM_FLAG_COORDINATES): round trip fed to Vivaldi on a direct
  // ack = coord_base_rtt_s + (extra latency there and back) * tick_seconds
  double coord_base_rtt_s, tick_seconds;
  // ceil(2^64 / n): `x % n` for the complete graph's peer draws as two multiplications (Lemire, Kaser &
  // Kurz 2019, exact for every 32-bit x and n) instead of an emulated 32-bit division per draw
  uint64_t n_magic;
  GsRumor rumors[GS_MAX_RUMORS];
};

// Members that may still be "pending" (known only through their alive rumor): the subjects of the
// tracked alive rumors.  Fills out[0 .. GS_MAX_SPECIAL) and returns how many there are in all
// (more than GS_MAX_SPECIAL: the closed form of a pristine window is not used, see gs_api.cpp).
#define GS_MAX_SPECIAL 8u
GS_HD uint32_t gs_special_members(const GsGlobals& g, uint32_t* out) {
  uint32_t cnt = 0;
  for (uint32_t r = 0; r < GS_MAX_RUMORS; ++r)
    if (((g.active_mask >> r) & 1u) && g.rumors[r].kind == GS_RUMOR_ALIVE) {
      if (cnt < GS_MAX_SPECIAL) out[cnt] = g.rumors[r].subject;
      ++cnt;
    }
  return cnt;
}

struct GsEventRec {
  uint32_t tick, type, subject, observer, ltime, reserved;
};

struct GsPig;

// Device column pointers.
struct GsDev {
  uint32_t* key[2];      // the key column this rank READS (its own replica when sharded)
  uint32_t* key_rep[2];  // replica 0; replica r at + r*key_stride.  Writers update every replica.
  uint32_t* inbox[GS_RING_MAX];  // arrival-tick ring; slots >= ring depth are null
  uint32_t* due;
  uint32_t* meta;
  uint32_t* cursor;
  uint32_t* pass;
  uint32_t* probe_tgt;
  uint32_t* probe_inc;
  uint32_t* sus_start;
  uint32_t* sus_from;  // [GS_K1MAX][cap]
  uint64_t* acc;       // [2][GS_K1MAX][cap]
  uint32_t* change_tick;
  uint32_t* reap_after;  // per-member ReconnectTimeout override in ticks, 0 = the pool's (cold: reaper only)
  uint32_t* ltime_member;
  uint32_t* ltime_event;
  uint32_t* event_min;
  uint32_t* heard;
  uint32_t* queued;
  uint8_t* tx;  // retransmit counters, [GS_MAX_RUMORS / 2][cap][2]: see GS_TX
  // network coordinates (gs_coord.h; null unless GSIM_FLAG_COORDINATES)
  double* coord;        // [2 slots][GS_COORD_WORDS][cap]
  uint32_t* ctag;       // [2 slots][cap]  tick the slot was written + 1 (0 = initial origin)
  double* adj;          // [GS_ADJ_WINDOW][cap] adjustment samples
  uint32_t* adj_idx;    // [cap]
  // push-pull mailboxes (null unless the pool runs periodic push-pull), by arrival-tick parity
  // status replica (see gs_kst_code): one byte per member with the 4-bit view of key[0] (low nibble)
  // and key[1] (high nibble) that peer selection needs; null on sharded pools (they gather from their
  // own full key replica)
  uint8_t* kst;
  const uint32_t* row_ptr;  // [graph_n + 1] CSR peer graph, null on complete-graph pools
  const uint32_t* col_idx;  // [row_ptr[graph_n]]
  uint32_t* ppreq;   // [2][GS_PPK][cap] requester ids, kept as the GS_PPK smallest (atomicMin chain)
  uint32_t* pp_clk;  // [2][2][cap] max of the senders' {member, event} Lamport clocks (atomicMax)
  // degraded members (gsim_impair_*): per-member UDP loss threshold and receive delay in ticks.  Both
  // null unless at least one member is impaired right now, which is also what turns the probe fast
  // paths off (the host keeps the columns and the count; a pool that was never impaired has neither).
  const uint32_t* imp_loss;  // [cap] packet from the member lost iff Philox word y < imp_loss (send threshold)
  const uint8_t* imp_delay;  // [cap] extra ticks before the member handles what it receives
  // pool-wide device words
  unsigned long long* stats;  // [GSIM_STAT_COUNT]
  uint32_t* heard_cnt;        // [GS_MAX_RUMORS]
  uint32_t* conv_tick;        // [GS_MAX_RUMORS]
  uint32_t* view_cnt;         // [4] alive/suspect/dead/left transitions bookkeeping
  uint32_t* crashed_alive;    // CRASHED members not yet Dead in the view
  uint32_t* crashed_dead_tick;
  GsEventRec* evlog;
  uint32_t* evlog_cursor;  // [0]=written, [1]=dropped
  uint32_t* tick_base;
  // sharded pools: inter-tick barrier state (gs_tick_kernel); null on single-GPU pools
  uint32_t* tick_flags[GS_MAX_WORLD_];  // tick_flags[r] = rank r's array of per-rank progress words
  uint32_t* done_ctr;
  // quiet-window scheduling (DESIGN.md §4.2): qstate[r] = rank r's copy of the GS_Q_* words; this
  // rank reads qstate[rank], writers update every rank's copy (like key_rep)
  uint32_t* qstate[GS_MAX_WORLD_];
  // one-way reachability (gsim_impair_dir_*), set exactly when imp_loss is: packet to the member lost iff
  // Philox word z < imp_recv (imp_recv == imp_loss until some member's receive threshold differs from its
  // send threshold or has a flag), and GSIM_IMPAIR_* flags per member (null until the first directional
  // setting).  Last in the struct, so every other field keeps its offset.
  const uint32_t* imp_recv;
  const uint8_t* imp_flags;
  // broadcasts piggybacked on probe traffic (GSIM_FLAG_PROBE_PIGGYBACK), both null without the flag:
  // owed answers by arrival-tick parity, [2][GS_PIGK][cap] entries receiver << 3 | kind << 1 | lost, kept as
  // the GS_PIGK smallest by an atomicMin chain; and the pool-wide words
  uint32_t* pig_req;
  GsPig* pig;
  // intermittent impairment (gsim_impair_flap_*): schedule words (gs_flap_bad), null while no member has a
  // schedule or nobody is impaired.  Only the impaired row step reads it; last in the struct, so every other
  // field keeps its offset.
  const uint32_t* imp_flap;
  // fault domains (gsim_domain_*): the domain column and the domain schedule table (dom_flap[x] = schedule
  // word of domain x, dom_flap_n entries), both null while no domain has a schedule or nobody is impaired
  const uint32_t* imp_dom;
  const uint32_t* dom_flap;
  uint32_t dom_flap_n;
};

// Fault-domain operations and observation (bodies in gs_aux.h).
enum { GS_DOMAIN_OP_IMPAIR = 0, GS_DOMAIN_OP_CRASH = 1, GS_DOMAIN_OP_PAUSE = 2, GS_DOMAIN_OP_COUNT = 3 };
// What a domain operation writes: the impairment columns and setting (IMPAIR), the pause column (CRASH: null
// while nobody was ever paused; PAUSE) and the resume tick (PAUSE).
struct GsDomainOp {
  uint32_t op;
  GsImpairCols imp;
  GsImpairVal v;
  uint32_t* pause_until;
  uint32_t until;
};

// Per-domain observation (gsim_domain_stats_read), field for field gsim_domain_stats.
struct GsDomainStats {
  uint32_t members, running, paused, impaired, in_force;
  uint32_t alive, suspect, dead, left;
  uint32_t awareness_max;
  uint64_t awareness_sum;
};
// The columns it reads: key = the key buffer of the current tick; imp = the impairment columns (any may be
// null); pause_until may be null; d = the published columns gs_imp_in_force reads.
struct GsDomainCols {
  const uint32_t* key;
  const uint32_t* meta;
  const uint32_t* dom;
  const uint32_t* pause_until;
  GsImpairCols imp;
};
// Member m's domain schedule word under the published columns of d (0 without one).
GS_HD uint32_t gs_dom_word(const GsDev& d, uint32_t m, uint32_t* dom) {
  if (d.dom_flap == nullptr) return 0u;
  *dom = d.imp_dom[m];
  return *dom < d.dom_flap_n ? d.dom_flap[*dom] : 0u;
}

// Is member m's impairment in force at tick t under the published columns of d (gs_in_force)?
GS_HD bool gs_imp_in_force(const GsDev& d, uint32_t seed_lo, uint32_t seed_hi, uint32_t m, uint32_t t) {
  uint32_t dom = 0u;
  const uint32_t wm = d.imp_flap != nullptr ? d.imp_flap[m] : 0u, wd = gs_dom_word(d, m, &dom);
  return gs_in_force(seed_lo, seed_hi, m, wm, dom, wd, t);
}

// Broadcasts piggybacked on probe traffic (GSIM_FLAG_PROBE_PIGGYBACK, DESIGN.md §3.7).
#define GS_PIGK 4u       // owed answers one member serves per tick (smallest entries win), like GS_PPK
#define GS_PIG_GATES 16u // gate words: tick s is gated iff gate[s % 16] == s + 1
// The probe messages whose remaining UDP room carries broadcasts, and what an owed answer entry names.
enum { GS_PIG_PING = 0, GS_PIG_ACK = 1, GS_PIG_NACK = 2, GS_PIG_INDREQ = 3 };
// gsim_piggyback_stats counters
enum { GS_PIG_ST_PACKETS = 0, GS_PIG_ST_BCASTS = 1, GS_PIG_ST_SERVED = 2, GS_PIG_ST_DROPPED = 3 };
// Pool-wide words of a piggybacking pool (one device allocation, carried whole by snapshots).
struct GsPig {
  // "some member's broadcast queue was non-empty when tick s began" <=> gate[s % 16] == s + 1.  A row that
  // ends tick t with a non-empty queue stamps every tick up to the one it is stepped at again (at most the
  // mailbox ring depth, <= 8, ahead), the host stamps `now` when it queues something: the word a tick
  // reads is never one that tick writes, and nobody has to clear a word.
  uint32_t gate[GS_PIG_GATES];
  uint32_t budget[4];                  // bytes left for broadcasts in a ping / ack / nack / indirect-ping request
  unsigned long long stats[4][32];     // GS_PIG_ST_* per member id % 32 (summed on read)
};

// Pool-wide scheduling words (one copy per rank).  A pool is QUIET when every mailbox slot is empty
// and nothing time-driven is pending except probe tickers: then a tick changes nothing but the rows
// whose ticker fires, those rows write only themselves, and the first tick at which any member can
// touch another one again is known in advance (the deadline of an unanswered probe, >= ProbeInterval
// after it started).  Up to that HORIZON the ticks of a tile are independent of every other tile, so
// one launch may run a whole window of them without looking at a single mailbox word.
enum {
  GS_Q_LAST_ACTIVE = 0,  // last tick at which a mailbox word was non-zero or a member posted one (+1; 0 = never)
  GS_Q_HORIZON = 1,      // lower bound of the next tick at which a member may post (deadline of a failed probe)
  GS_Q_WIN_END = 2,      // tick the chain of window launches has reached (windows stop at the horizon)
  GS_Q_VIOLATION = 3,    // set if a window launch ever met mail or posted: internal error, checked by the host
  GS_Q_WORDS = 4
};

// Per-row outputs that the launch wrapper reduces (warp/block aggregated atomics).
#define GS_NSTAT 16
struct GsRowOut {
  uint32_t st[GS_NSTAT];
  uint32_t new_heard;     // rumor bits accepted by this row in this tick
  int32_t crashed_alive;  // delta of the "crashed but not yet dead" count
};

// ---- multi-GPU (sharded) pools: DESIGN.md §7, gs_vmm.h ---------------------------------------
// Every rank has one 2 MB "page" of pool-wide words in its own HBM, mapped by all ranks.
// Counters and the event log live in rank 0's page (the other ranks update them with
// remote atomics over NVLink); tick_base, the device copy of GsGlobals and the barrier flags
// are per rank.
#define GS_PAGE_BYTES (2u << 20)
#define GS_PG_STATS 0u
#define GS_PG_HEARD_CNT 256u
#define GS_PG_CONV_TICK 512u
#define GS_PG_VIEW_CNT 768u
#define GS_PG_CRASHED_ALIVE 800u
#define GS_PG_CRASHED_DEAD_TICK 804u
#define GS_PG_EVLOG_CURSOR 808u
#define GS_PG_TICK_BASE 816u
#define GS_PG_XBAR_EPOCH 820u
#define GS_PG_XBAR_FLAGS 832u
#define GS_PG_TICK_FLAGS 896u   // [GS_MAX_WORLD] "rank r has completed every tick < value"
#define GS_PG_DONE_CTR 960u     // CTAs of this rank that have finished the current tick
#define GS_PG_QSTATE 976u       // [GS_Q_WORDS] quiet-window scheduling words of this rank
#define GS_PG_GLOBALS 1024u
#define GS_PG_SCRATCH 8192u
#define GS_PG_BLOB 16384u      // 2 slots of GS_BLOB_BYTES
#define GS_BLOB_BYTES 32768u
#define GS_PG_EVLOG 131072u
#define GS_MAX_WORLD 8

// Cross-GPU barrier between ticks: rank r stores its epoch into slot r of every rank's flag
// array (st.release.sys over NVLink) and spins on its own array until all slots caught up.
struct GsXbar {
  uint32_t* flags[GS_MAX_WORLD];  // flags[r] = rank r's array of GS_MAX_WORLD words
  uint32_t* epoch;                // this rank's last completed epoch
  uint32_t rank, world;
};
