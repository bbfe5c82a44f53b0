// gs_cuda.cu — sm_90a kernels and the CUDA backend of libgsim.
//
// Kernels (all HBM/L2-bound integer work; no tensor cores by design — there is no dense
// contraction anywhere on this path):
//   gs_tick_kernel      one launch = one lock-step tick of every virtual member
//                       (SURVEY §7 K1+K2 fused: emit and apply are separated by the
//                       double-buffered mailbox instead of a grid barrier)
//   gs_advance_kernel   bumps the device tick counter at the end of a CUDA-graph chunk
//   gs_stretch_*        drive a tick stretch: single ticks until the pool is quiet, decided on the device
//   gs_init_kernel, gs_crash_kernel, gs_recount_kernel, gs_hash_kernel   control plane
//   gs_pause_kernel, gs_resume_kernel   paused members (gsim_pause_*, DESIGN.md §3.6)
//   gs_coord_*_kernel, gs_rs_*_kernel   network-coordinate queries and their stable LSD radix sort
//                                       (DESIGN.md §3.4 "Queries")
//
// Launch shape of the tick: a persistent grid (SMs x resident CTAs) of 256-thread CTAs; every warp
// owns a contiguous chunk of 128-member tiles, scans their 4-byte mailbox words through a
// shared-memory ring and works only on tiles with mail or a due probe ticker (DESIGN.md §4).
// Ticks are chained inside a CUDA graph of GS_GRAPH_TICKS launches with programmatic dependent
// launch, so the per-launch host cost is off the critical path.
#include <cuda_runtime.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <map>

#include "gs_aux.h"
#include "gs_backend.h"
#include "gs_query.h"
#include "gs_vmm.h"

#define GS_BLOCK 256
#define GS_GRAPH_TICKS 64
#define GS_WIN_GRAPH 8   // quiet windows per CUDA graph
#ifndef GS_STRETCH_TICKS
#define GS_STRETCH_TICKS 16  // tick launches per pass of a tick stretch's loop (at most this many - 1 run nothing)
#endif

namespace {

// COORDS selects the tick-kernel instantiation that carries the network-coordinate update
// (gs_coord.h, ~150 double-precision operations per direct ack) and the row step of pools with flap
// schedules (gsim_impair_flap_*: Philox draws at the register limit).  The default instantiation
// contains none of that code, so pools with neither pay nothing for it; a pool with schedules runs the
// COORDS instantiation whether or not it has coordinates (the update is skipped without them).
template <bool COORDS>
struct DevSinkT {
  static constexpr bool kCoords = COORDS;
  uint32_t* s_stat;
  uint32_t* s_heard;
  uint32_t* s_q;  // [0] this CTA saw mail or posted some, [1] min horizon raised by its members
  __device__ __forceinline__ void activity() { s_q[0] = 1u; }
  __device__ __forceinline__ void horizon(uint32_t h) { atomicMin(&s_q[1], h); }
  // Counters are kept per lane (one shared-memory bank each): the 32 members of a group bump the same
  // counter at the same instruction, and 32 atomics on ONE shared word replay 32 times.
  __device__ __forceinline__ void stat(int idx, uint32_t v) { atomicAdd(&s_stat[idx * 32 + (threadIdx.x & 31u)], v); }
  __device__ __forceinline__ void heard(uint32_t r) { atomicAdd(&s_heard[r * 32u + (threadIdx.x & 31u)], 1u); }
  // Pool-wide words (crashed_alive, the event-log cursor, heard_cnt) live in rank 0's page on a
  // sharded pool and are updated by every GPU: system-scope atomics (device scope is not atomic
  // across GPUs).  They are rare — one per event, not per member — so single-GPU pools pay nothing
  // measurable for the wider scope.
  __device__ __forceinline__ void crashed_dead(const GsDev& d, uint32_t t) {
    uint32_t old = atomicSub_system(d.crashed_alive, 1u);
    if (old == 1u) *d.crashed_dead_tick = t;
  }
  __device__ __forceinline__ void log_event(const GsDev& d, const GsGlobals& g, uint32_t t,
                                            uint32_t type, uint32_t subject, uint32_t observer,
                                            uint32_t ltime) {
    uint32_t pos = atomicAdd_system(&d.evlog_cursor[0], 1u);
    if (pos < g.evlog_cap) {
      GsEventRec e;
      e.tick = t;
      e.type = type;
      e.subject = subject;
      e.observer = observer;
      e.ltime = ltime;
      e.reserved = 0u;
      d.evlog[pos] = e;
    } else {
      atomicAdd_system(&d.evlog_cursor[1], 1u);
    }
  }
};
typedef DevSinkT<false> DevSink;

#ifndef GS_MIN_BLOCKS
#define GS_MIN_BLOCKS 4
#endif
#define GS_WARPS (GS_BLOCK / 32)
#define GS_ROUND 4                   // tiles a warp brings in with one bulk copy and scans between two drains of the CTA's queue

// Bulk asynchronous copies (TMA, 1-D): ONE lane moves a whole run of tiles global -> shared with a single
// instruction (cp.async.bulk: SASS UBLKCP) and the data's arrival is counted in bytes on an mbarrier in
// shared memory (expect_tx / complete_tx: SASS SYNCS), which the warp then waits on.  The round-1 scan
// issued a 16-byte cp.async per lane and tile (LDGSTS.128): ~40 warp instructions per idle tile, most of
// them address arithmetic and commit/wait bookkeeping.
__device__ __forceinline__ uint32_t gs_smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void gs_mbar_init(uint64_t* bar, uint32_t arrivals) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(gs_smem_addr(bar)), "r"(arrivals) : "memory");
}
__device__ __forceinline__ void gs_mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(gs_smem_addr(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void gs_bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   gs_smem_addr(smem_dst)),
               "l"(gsrc), "r"(bytes), "r"(gs_smem_addr(bar))
               : "memory");
}
// true once the phase with this parity has completed; bounded (a byte-count bug must not hang the device:
// the caller raises the pool's VIOLATION word instead)
__device__ __forceinline__ bool gs_mbar_wait(uint64_t* bar, uint32_t parity) {
  for (uint32_t spin = 0; spin < (1u << 24); ++spin) {
    uint32_t done;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(gs_smem_addr(bar)), "r"(parity)
        : "memory");
    if (done) return true;
  }
  return false;
}

// ---- sharded pools: the inter-tick barrier lives inside the kernels ---------------------------
// Acquire side: tick t may start once every rank has published "all ticks < t done" in this rank's
// progress array (written by the peers over NVLink with st.release.sys at the end of their
// previous launch).
__device__ __forceinline__ void gs_ranks_wait(const GsDev& d, const GsGlobals& g, uint32_t t) {
  if (threadIdx.x < g.world) {
    uint32_t v;
    do {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(d.tick_flags[g.rank] + threadIdx.x) : "memory");
    } while ((int32_t)(v - t) < 0);
  }
  __syncthreads();
}
// Release side.  Every thread that delivered something fenced at system scope, so its mailbox
// clears, key updates and remote deliveries are performed; CTAs count in with a device-scope atomic
// and the last one publishes `t_done` to every rank.  The chain (write -> fence.sys -> bar -> atomic
// ... atomic -> fence.sys -> st.release.sys) does not rely on kernel boundaries, which is what
// makes it safe inside a CUDA graph.
__device__ __forceinline__ void gs_ranks_release(const GsDev& d, const GsGlobals& g, uint32_t t_done) {
  __syncthreads();
  if (threadIdx.x == 0u) {
    __threadfence_system();
    const uint32_t arrived = atomicAdd(d.done_ctr, 1u);
    if (arrived == gridDim.x - 1u) {
      __threadfence_system();
      *d.done_ctr = 0u;
      __threadfence_system();
      for (uint32_t r = 0; r < g.world; ++r)
        asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(d.tick_flags[r] + g.rank), "r"(t_done) : "memory");
    }
  }
}

// Quiet-window scheduling words (GS_Q_*): every rank keeps a copy, writers update all of them.
__device__ __forceinline__ void gs_q_publish(const GsDev& d, const GsGlobals& g, const uint32_t* s_q, uint32_t t) {
  if (s_q[0] != 0u) {
    if (g.world <= 1u) atomicMax(d.qstate[0] + GS_Q_LAST_ACTIVE, t + 1u);
    else for (uint32_t r = 0; r < g.world; ++r) atomicMax_system(d.qstate[r] + GS_Q_LAST_ACTIVE, t + 1u);
  }
  if (s_q[1] != GS_NEVER) {
    if (g.world <= 1u) atomicMin(d.qstate[0] + GS_Q_HORIZON, s_q[1]);
    else for (uint32_t r = 0; r < g.world; ++r) atomicMin_system(d.qstate[r] + GS_Q_HORIZON, s_q[1]);
  }
}

// The generic row step, out of line.  Inlined into the persistent loops it costs every launch its
// registers (80 -> 3 resident CTAs per SM); as a call it costs the members that take it ~30
// instructions on top of several hundred, and the loops around it fit 64 registers (4 CTAs per SM:
// a quarter more warps to hide the L2 round trips, and at 1 M members two tiles per warp, not three).
// Pools with degraded members step through an instantiation of their own, so the one every other pool runs
// carries none of the impairment terms.
template <bool COORDS>
__device__ __noinline__ void gs_row_step_impaired_call(const GsDev* dp, const GsGlobals* gp, uint32_t i, uint32_t t,
                                                       uint32_t inb, uint32_t* s_stat, uint32_t* s_heard, uint32_t* s_q) {
  DevSinkT<COORDS> sink{s_stat, s_heard, s_q};
  gs_row_step_body<true>(*dp, *gp, i, t, t % gp->GI, inb, sink);
}
// Pools that piggyback broadcasts on probe traffic (GSIM_FLAG_PROBE_PIGGYBACK) likewise.
template <bool COORDS, bool IMPAIRED>
__device__ __noinline__ void gs_row_step_pig_call(const GsDev* dp, const GsGlobals* gp, uint32_t i, uint32_t t,
                                                  uint32_t inb, uint32_t* s_stat, uint32_t* s_heard, uint32_t* s_q) {
  DevSinkT<COORDS> sink{s_stat, s_heard, s_q};
  gs_row_step_body<IMPAIRED, true>(*dp, *gp, i, t, t % gp->GI, inb, sink);
}
template <bool COORDS>
__device__ __noinline__ void gs_row_step_call(const GsDev* dp, const GsGlobals* gp, uint32_t i, uint32_t t,
                                              uint32_t inb, uint32_t* s_stat, uint32_t* s_heard, uint32_t* s_q) {
  if (dp->imp_loss != nullptr) {
    gs_row_step_impaired_call<COORDS>(dp, gp, i, t, inb, s_stat, s_heard, s_q);
    return;
  }
  DevSinkT<COORDS> sink{s_stat, s_heard, s_q};
  gs_row_step_body<false>(*dp, *gp, i, t, t % gp->GI, inb, sink);
}

// Pools whose impaired members have flap schedules (GsDev::imp_flap or dom_flap set, only with imp_loss) likewise; only
// the COORDS kernels call it (gs_kernel_extras).
template <bool COORDS, bool PIG>
__device__ __noinline__ void gs_row_step_flap_call(const GsDev* dp, const GsGlobals* gp, uint32_t i, uint32_t t,
                                                   uint32_t inb, uint32_t* s_stat, uint32_t* s_heard, uint32_t* s_q) {
  DevSinkT<COORDS> sink{s_stat, s_heard, s_q};
  gs_row_step_body<true, PIG, true>(*dp, *gp, i, t, t % gp->GI, inb, sink);
}

// Every generic row step of the tick and window kernels: piggybacking and flapping pools call their own step from
// here, not from inside gs_row_step_call, so that its frame does not stack on top of the default step's.
template <bool COORDS>
__device__ __forceinline__ void gs_row_step_any(const GsDev* dp, const GsGlobals* gp, uint32_t i, uint32_t t,
                                                uint32_t inb, uint32_t* s_stat, uint32_t* s_heard, uint32_t* s_q) {
  if constexpr (COORDS) {
    if (dp->imp_flap != nullptr || dp->dom_flap != nullptr) {
      if (dp->pig == nullptr) gs_row_step_flap_call<COORDS, false>(dp, gp, i, t, inb, s_stat, s_heard, s_q);
      else gs_row_step_flap_call<COORDS, true>(dp, gp, i, t, inb, s_stat, s_heard, s_q);
      return;
    }
  }
  if (dp->pig == nullptr) gs_row_step_call<COORDS>(dp, gp, i, t, inb, s_stat, s_heard, s_q);
  else if (dp->imp_loss != nullptr) gs_row_step_pig_call<COORDS, true>(dp, gp, i, t, inb, s_stat, s_heard, s_q);
  else gs_row_step_pig_call<COORDS, false>(dp, gp, i, t, inb, s_stat, s_heard, s_q);
}

// Tick stretches (run_tick_stretch): the control block on the device, in the backend's scratch.
struct GsStretchCtl {
  GsStretch out;               // read back at the end
  uint32_t violation;          // GS_Q_VIOLATION at the end (read back with `out`)
  uint32_t end, floor, depth;  // ticks before `end` run until the first tick >= max(LAST_ACTIVE, floor) + depth
};
// the tick at which the stretch stops, given GS_Q_LAST_ACTIVE
__device__ __forceinline__ uint32_t gs_stretch_stop(const GsStretchCtl& c, uint32_t last_active) {
  const uint32_t quiet_at = (last_active > c.floor ? last_active : c.floor) + c.depth;
  return quiet_at < c.end ? quiet_at : c.end;
}

// Persistent, warp-centric tick.  Every warp owns a CONTIGUOUS chunk of tiles (128 members
// each); because ticker phases are dealt round-robin over tiles, every chunk holds the same
// number of probing tiles (+-1) at every tick, so the static split is balanced.
//   Scan: each lane moves the mailbox words of 4 members (16 B; a tile is one 512-byte
// request) into a per-warp shared-memory ring with cp.async, GS_STAGES-1 tiles ahead; tiles
// whose ticker phase can be due at this tick also bring their `due` words.  An idle tile
// costs ~40 warp instructions and 4 bytes per member.
//   Work: a tile with activity is re-read from shared memory one member per lane (coalesced
// column accesses).  The four 32-member groups of a probing tile go through the staged fast
// path together — own columns, target gathers and commits are each issued for all four
// before the first is consumed — so the tile pays two dependent memory latencies, not eight.
// Whatever the fast path declines goes to the generic gs_row_step.
template <bool COORDS>
__global__ void __launch_bounds__(GS_BLOCK, GS_MIN_BLOCKS)
    gs_tick_kernel(const __grid_constant__ GsDev d, const GsGlobals* __restrict__ gp, uint32_t k_off,
                   const GsStretchCtl* __restrict__ stretch) {
  __shared__ uint32_t s_stat[GS_NSTAT * 32];  // [counter][lane]
  __shared__ uint32_t s_heard[32 * 32];       // [broadcast slot][lane]
  __shared__ __align__(128) uint32_t s_inb[GS_WARPS][GS_ROUND][GS_TILE];  // a warp's round of mailbox words ...
  __shared__ __align__(128) uint32_t s_due[GS_WARPS][GS_ROUND][GS_TILE];  // ... and `due` words (gated tiles only)
  __shared__ __align__(8) uint64_t s_bar[GS_WARPS];                       // one transaction barrier per warp
  __shared__ uint32_t s_q[2];
  // members that need the generic step, queued one entry each by the scanning warps and taken 32 at a time
  // by whichever warp of the CTA is free (two counters each: rounds alternate, see below).  An entry is
  // (scanning warp << 9) | (tile in its round << 7) | member in tile; s_rtile[w] is warp w's first tile
  // of the round.
  __shared__ uint16_t s_work[GS_WARPS * GS_ROUND * GS_TILE];
  __shared__ uint32_t s_rtile[GS_WARPS];
  __shared__ uint32_t s_wn[2], s_wtake[2];
  static_assert(GS_WARPS <= 8 && GS_ROUND <= 4 && GS_TILE == 128, "s_work entries are 3 + 2 + 7 bits");
  const uint32_t tid = threadIdx.x;
  for (uint32_t x = tid; x < GS_NSTAT * 32u; x += GS_BLOCK) s_stat[x] = 0u;
  for (uint32_t x = tid; x < 32u * 32u; x += GS_BLOCK) s_heard[x] = 0u;
  if (tid == 64u) s_q[0] = 0u;
  if (tid == 65u) s_q[1] = GS_NEVER;
  if (tid >= 66u && tid < 68u) s_wn[tid - 66u] = 0u;
  if (tid >= 68u && tid < 70u) s_wtake[tid - 68u] = 0u;
  if (tid >= 96u && tid < 96u + GS_WARPS) gs_mbar_init(&s_bar[tid - 96u], 1u);  // one arrival per phase: the issuing lane
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  // Programmatic dependent launch: let the next tick's grid start launching now; it blocks in
  // its own griddepcontrol.wait until this grid has completed and flushed.  Everything above
  // this line touches no global memory.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  // Inside a tick stretch (single-GPU pools) a launch whose tick is past the stretch's end or at its first
  // quiet tick runs nothing: it neither scans nor publishes.  Every thread of every CTA decides the same
  // without a barrier, although CTAs of this tick may raise GS_Q_LAST_ACTIVE while others still read it:
  // the word only grows, and a tick that stops publishes nothing, so the only raised value a thread can
  // read comes from a CTA of this tick that runs, and a higher LAST_ACTIVE only makes "run" more certain.
  if (stretch != nullptr && *d.tick_base + k_off >= gs_stretch_stop(*stretch, __ldcg(d.qstate[0] + GS_Q_LAST_ACTIVE)))
    return;
  __syncthreads();
  const GsGlobals& g = *gp;
  const uint32_t t = *d.tick_base + k_off;
  if (g.world > 1u) gs_ranks_wait(d, g, t);
  const uint32_t cur = t & 1u, P = g.P, pslot = t % P, gslot = t % g.GI;
  const uint32_t pslot_t = (t + P - g.T % P) % P;
  const uint32_t lane = tid & 31u, wib = tid >> 5;
  // this rank's tiles: everything on one GPU, a contiguous range of members when sharded
  uint32_t tile_lo = 0, tile_hi = (g.n + GS_TILE - 1u) / GS_TILE;
  if (g.world > 1u) {
    const uint32_t per = g.rows_per_rank / GS_TILE;
    tile_lo = g.rank * per < tile_hi ? g.rank * per : tile_hi;
    tile_hi = tile_lo + per < tile_hi ? tile_lo + per : tile_hi;
  }
  // contiguous runs of tiles, floor or ceil of tiles / warps each: every warp (and so every SM) gets
  // its share — with ceil-sized chunks the last quarter of the grid had nothing to do at 1 M members
  const uint32_t n_warps = gridDim.x * GS_WARPS, n_tiles = tile_hi - tile_lo;
  const uint32_t wid = blockIdx.x * GS_WARPS + wib;
  const uint32_t t_begin = tile_lo + (uint32_t)(((uint64_t)wid * n_tiles) / n_warps);
  const uint32_t t_end = tile_lo + (uint32_t)(((uint64_t)(wid + 1u) * n_tiles) / n_warps);
  const uint32_t* __restrict__ inbox_cur = d.inbox[t & g.ring_mask];  // this tick's arrival slot
  const bool gated = g.phase_gate != 0u;
  const uint32_t shift = g.phase_shift;
  DevSinkT<COORDS> sink{s_stat, s_heard, s_q};

  // Rounds.  A warp scans up to GS_ROUND of its tiles and runs the staged probe fast path inline;
  // every member that needs the generic step goes into the CTA's queue instead.  Then the whole CTA
  // drains the queue, 32 members per warp at a time: a warp whose tiles were idle helps the warp whose
  // tiles all gossip (gossip phases come in runs of ProbeInterval tiles, so consecutive tiles are
  // busy together and a static split leaves half the warps waiting at the closing barrier), and in the
  // rise and the tail of a join cascade, when a few active members are spread over every 32-member
  // group, a warp-step still steps 32 of them.  Results do not depend on who steps a member:
  // everything a member sends is a commutative atomic and counters are summed per lane.
  const uint32_t max_run = (n_tiles + n_warps - 1u) / n_warps, n_rounds = (max_run + GS_ROUND - 1u) / GS_ROUND;
  bool did_work = false;  // this thread touched global state (needs the closing fence when sharded)
  const bool sys_scan = g.world > 1u && (g.flags & 4u);  // GSIM_FLAG_SHARD_SYNC_SCAN (debug): system-scope loads, no bulk copy
  // Bring round r of this warp's tiles into its shared-memory buffers: ONE bulk copy for the mailbox words of
  // the whole round, one per tile that can have a probe action due at this tick (2 of every P phases) for its
  // `due` words; the other tiles' `due` reads as "never".  Issued for round r + 1 as soon as the warp has
  // scanned round r, so the copy flies while the CTA drains its queue.
  auto bring = [&](uint32_t r) {
    const uint32_t b0 = t_begin + r * GS_ROUND < t_end ? t_begin + r * GS_ROUND : t_end;
    const uint32_t b1 = b0 + GS_ROUND < t_end ? b0 + GS_ROUND : t_end;
    const uint32_t tiles = b1 - b0;
    if (!tiles) return;
    uint32_t gate_mask = 0;
    for (uint32_t x = 0; x < tiles; ++x) {
      bool gate = true;
      if (gated) {
        const uint32_t pp = gs_probe_phase(g.rot_p, (b0 + x) >> shift, P);
        gate = pp == pslot || pp == pslot_t;
      }
      gate_mask |= gate ? 1u << x : 0u;
    }
    const size_t off0 = (size_t)b0 * GS_TILE;  // columns are padded to whole tiles
    if (sys_scan) {
      for (uint32_t x = 0; x < tiles; ++x) {
        uint4 v;
        asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                     : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(inbox_cur + off0 + x * GS_TILE + lane * 4u) : "memory");
        *reinterpret_cast<uint4*>(&s_inb[wib][x][lane * 4u]) = v;
        const uint4 dv = (gate_mask >> x) & 1u ? *reinterpret_cast<const uint4*>(d.due + off0 + x * GS_TILE + lane * 4u)
                                               : make_uint4(GS_NEVER, GS_NEVER, GS_NEVER, GS_NEVER);
        *reinterpret_cast<uint4*>(&s_due[wib][x][lane * 4u]) = dv;
      }
      __syncwarp();
      return;
    }
    for (uint32_t x = 0; x < tiles; ++x)
      if (!((gate_mask >> x) & 1u))
        *reinterpret_cast<uint4*>(&s_due[wib][x][lane * 4u]) = make_uint4(GS_NEVER, GS_NEVER, GS_NEVER, GS_NEVER);
    __syncwarp();
    if (lane == 0u) {
      // the buffers were last touched through the generic proxy: order that before the bulk writes
      asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
      gs_mbar_expect_tx(&s_bar[wib], (tiles + __popc(gate_mask)) * GS_TILE * 4u);
      gs_bulk_g2s(&s_inb[wib][0][0], inbox_cur + off0, tiles * GS_TILE * 4u, &s_bar[wib]);
      for (uint32_t x = 0; x < tiles; ++x)
        if ((gate_mask >> x) & 1u) gs_bulk_g2s(&s_due[wib][x][0], d.due + off0 + x * GS_TILE, GS_TILE * 4u, &s_bar[wib]);
    }
  };
  bring(0u);
  for (uint32_t round = 0; round < n_rounds; ++round) {
  const uint32_t par = round & 1u;
  const uint32_t r_begin = t_begin + round * GS_ROUND < t_end ? t_begin + round * GS_ROUND : t_end;
  const uint32_t r_end = r_begin + GS_ROUND < t_end ? r_begin + GS_ROUND : t_end;
  if (r_end > r_begin && !sys_scan && !gs_mbar_wait(&s_bar[wib], round & 1u)) {  // (every lane waits: the data is then visible to it)
    if (lane == 0u) atomicExch(d.qstate[g.rank] + GS_Q_VIOLATION, t + 1u);
  }
  for (uint32_t tile = r_begin; tile < r_end; ++tile) {
    const uint32_t st = tile - r_begin;
    uint4 i4 = *reinterpret_cast<const uint4*>(&s_inb[wib][st][lane * 4u]);
    const uint4 d4 = *reinterpret_cast<const uint4*>(&s_due[wib][st][lane * 4u]);
    if (__any_sync(0xFFFFFFFFu, (i4.x | i4.y | i4.z | i4.w) != 0u)) {
      // Stale mail (gs_mail_is_stale): retired here without a row step — the word is cleared (in global
      // memory before the __syncthreads that closes the round, so the drain below reads it as empty, and
      // in the round buffer, so the member stays out of act[] and the fast-path candidates) and counted
      // as activity.  Not an ACTIVE_ROWS row: it never leaves the scan.
      const uint32_t m0 = tile * GS_TILE + lane * 4u;
      const uint4 h4 = __ldcg(reinterpret_cast<const uint4*>(d.heard + m0));
      uint32_t* const w_cur = d.inbox[t & g.ring_mask] + m0;
      uint32_t* const w4 = &i4.x;
      const uint32_t* const h = &h4.x;
      const uint32_t* const du = &d4.x;
      bool stale_any = false;
#pragma unroll
      for (uint32_t u = 0; u < 4u; ++u) {
        const bool pp = g.pp_interval != 0u && gs_pp_due(g.pp_interval, g.rot_pp, (m0 + u) / g.phase_group, t);
        if (w4[u] != 0u && gs_mail_is_stale(g, w4[u], h[u], du[u] == t, pp)) {
          w_cur[u] = 0u;
          s_inb[wib][st][lane * 4u + u] = 0u;
          w4[u] = 0u;
          stale_any = true;
        }
      }
      if (stale_any) sink.activity();
    }
    bool mine = (i4.x | i4.y | i4.z | i4.w) != 0u || d4.x == t || d4.y == t || d4.z == t || d4.w == t;
    // periodic push-pull (opt-in): the ticker of this tile's phase group (or, with per-member
    // phases, of one of its members) fires at this tick
    bool pp_tile = false;
    if (g.pp_interval != 0u) {
      if (gated) {
        pp_tile = gs_pp_due(g.pp_interval, g.rot_pp, tile >> shift, t);
      } else {
#pragma unroll
        for (uint32_t u = 0; u < 4u; ++u)
          pp_tile |= gs_pp_due(g.pp_interval, g.rot_pp, (tile * GS_TILE + lane * 4u + u) / g.phase_group, t);
      }
      mine |= pp_tile;
    }
    if (__any_sync(0xFFFFFFFFu, mine)) {
      did_work = true;
      __syncwarp();  // other lanes' copies are now visible: re-read one member per lane
      const uint32_t base = tile * GS_TILE + lane;
      bool act[4], cand[4];
      bool any_cand = false;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const uint32_t w = s_inb[wib][st][u * 32 + lane];
        const bool due_now = s_due[wib][st][u * 32 + lane] == t;
        act[u] = w != 0u || due_now ||
                 (g.pp_interval != 0u && gs_pp_due(g.pp_interval, g.rot_pp, (base + 32u * u) / g.phase_group, t));
        cand[u] = w == 0u && due_now;  // empty mailbox + ticker fired
        any_cand |= cand[u];
      }
      if (__any_sync(0xFFFFFFFFu, any_cand)) {
        GsFastProbe f[4];
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (cand[u]) gs_fast_load(d, cur, base + 32u * u, f[u]);               // A: own columns
#pragma unroll
        for (int u = 0; u < 4; ++u)
          if (cand[u]) cand[u] = gs_fast_target(d, g, cur, base + 32u * u, f[u]);  // B: gathers
        uint32_t n_probe = 0, n_ack = 0;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          bool acked = false;
          const bool done = cand[u] && gs_fast_finish(d, g, sink, base + 32u * u, t, f[u], &acked);  // C
          if (done) act[u] = false;
          n_probe += __popc(__ballot_sync(0xFFFFFFFFu, done));
          n_ack += __popc(__ballot_sync(0xFFFFFFFFu, done && acked));
        }
        if (lane == 0u && n_probe) {
          atomicAdd(&s_stat[GS_ST_PROBES * 32], n_probe);
          atomicAdd(&s_stat[GS_ST_ACTIVE_ROWS * 32], n_probe);
          if (n_ack) atomicAdd(&s_stat[GS_ST_ACKS * 32], n_ack);
        }
      }
      // queue the members left (mail, a probe action the fast path declined, the push-pull ticker): one
      // shared atomic reserves the tile's entries, each active lane writes its own at its prefix position
      uint32_t bal[4], n_act = 0;
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        bal[u] = __ballot_sync(0xFFFFFFFFu, act[u]);
        n_act += __popc(bal[u]);
      }
      if (n_act) {
        uint32_t pos = 0;
        if (lane == 0u) pos = atomicAdd(&s_wn[par], n_act);
        pos = __shfl_sync(0xFFFFFFFFu, pos, 0);
        const uint32_t below = (1u << lane) - 1u, key = (wib << 9) | (st << 7) | lane;
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (act[u]) s_work[pos + __popc(bal[u] & below)] = (uint16_t)(key | ((uint32_t)u << 5));
          pos += __popc(bal[u]);
        }
      }
    }
  }
  if (lane == 0u) s_rtile[wib] = r_begin;
  __syncwarp();                              // this warp is done with its round buffers:
  if (round + 1u < n_rounds) bring(round + 1u);  // the next round's copy flies while the CTA drains its queue
  __syncthreads();  // the queue of this round is complete
  if (tid == 0u) s_wn[par ^ 1u] = s_wtake[par ^ 1u] = 0u;  // the next round's counters (nobody uses them now)
  const uint32_t n_work = s_wn[par];
  // Drain: 32 queued members per warp-step, whichever tiles and scanning warps they came from.  Every lane
  // with an entry steps its member.  The mailbox word is re-read: the round buffer may already hold the next
  // round's copy, and stale mail was cleared in global memory before the barrier above.
  for (;;) {
    uint32_t idx = 0;
    if (lane == 0u) idx = atomicAdd(&s_wtake[par], 32u);
    idx = __shfl_sync(0xFFFFFFFFu, idx, 0);
    if (idx >= n_work) break;
    did_work = true;
    if (idx + lane < n_work) {
      const uint32_t e = s_work[idx + lane];
      const uint32_t i = (s_rtile[e >> 9] + ((e >> 7) & 3u)) * GS_TILE + (e & 127u);
      gs_row_step_any<COORDS>(&d, gp, i, t, __ldcg(inbox_cur + i), s_stat, s_heard, s_q);
    }
  }
  __syncthreads();  // the queue is drained (and its counters may be reused two rounds from now)
  }  // rounds
  // Sharded pools: mailbox deliveries to other GPUs are fire-and-forget reductions over NVLink;
  // a system-scope fence by the issuing thread is what guarantees they have been performed at
  // the owner before this rank can signal the inter-tick barrier.
  if (g.world > 1u && did_work && !(g.flags & 8u)) __threadfence_system();  // 8: GSIM_FLAG_SHARD_LEAN_FENCE
  __syncthreads();
  // one global atomic per counter per CTA, and only for CTAs that saw activity
  if (tid < GS_NSTAT) {
    uint32_t v = 0;
    for (uint32_t x = 0; x < 32u; ++x) v += s_stat[tid * 32u + ((x + tid) & 31u)];
    if (v) atomicAdd(&d.stats[tid], (unsigned long long)v);
  } else if (tid >= 32u && tid < 32u + GS_MAX_RUMORS) {
    uint32_t r = tid - 32u, c = 0;
    for (uint32_t x = 0; x < 32u; ++x) c += s_heard[r * 32u + ((x + r) & 31u)];
    if (c) {
      uint32_t old = atomicAdd_system(&d.heard_cnt[r], c);  // rank 0's page on a sharded pool
      if (old + c == g.up_count) d.conv_tick[r] = t;  // every UP member has heard rumor r
    }
  }
  if (tid == 0u) gs_q_publish(d, g, s_q, t);  // (after the CTA barrier above: every warp's flags are in)
  if (g.world > 1u) gs_ranks_release(d, g, t + 1u);
}

// ---------------------------------------------------------------------------------------------
// Quiet window: up to ProbeInterval ticks in ONE launch (DESIGN.md §4.2).
//
// On a quiet pool (every mailbox slot empty, nothing time-driven pending but probe tickers) a tick
// changes only the members whose ticker fires, and those write only their own row: the probe is
// pull-evaluated from the target's published key, which nobody changes.  The first tick at which a
// member can touch another one again is the deadline of an unanswered probe, at least
// ProbeInterval after it started; the minimum over all members is the HORIZON word.  Up to the
// horizon the ticks of a tile are independent of every other tile, so a warp runs all the ticks of
// the window for its tiles back to back: no mailbox scan (the words are known to be zero), no
// grid-wide synchronisation, and on a sharded pool one inter-rank barrier per window instead of one
// per tick.  Results are bit-identical to running the ticks one by one — the per-row code is the
// same gs_fast_* / gs_row_step — which tests/test_windows_cpu.py and the GPU parity tests check.
//
// A tile's members are due only at ticks congruent to its ticker phase (probe start, probe
// deadline) or to phase + ProbeTimeout (indirect stage): at most two ticks of a window.
// The generic path of a window for one batch of four groups: one ProbeInterval after the other (rows are
// independent inside a quiet window, so a warp finishes all the ticks of its groups before it looks at
// the next ones), staged probe fast path first, then the generic row step for whatever it declines.
template <bool COORDS>
__device__ __noinline__ void gs_window_generic(const GsDev* dp, const GsGlobals* gp, uint32_t gb, uint32_t g_end,
                                               uint32_t tf00, uint32_t tf01, uint32_t tf02, uint32_t tf03,
                                               uint32_t tx00, uint32_t tx01, uint32_t tx02, uint32_t tx03,
                                               uint32_t t0, uint32_t w1, uint32_t* s_stat, uint32_t* s_heard,
                                               uint32_t* s_q, uint32_t* counts) {
  const GsDev& d = *dp;
  const GsGlobals& g = *gp;
  const GsHot h = gs_hot(g);
  const uint32_t P = h.P, T = h.T, lane = threadIdx.x & 31u;
  const uint32_t tf0[4] = {tf00, tf01, tf02, tf03}, tx0[4] = {tx00, tx01, tx02, tx03};
  const bool fast_ok =
      h.loss_thr == 0u && h.graph_n == 0u && d.coord == nullptr && d.imp_loss == nullptr && h.pp_interval == 0u;
  DevSinkT<COORDS> sink{s_stat, s_heard, s_q};
  uint32_t n_probe = 0, n_ack = 0;
  bool did_work = false;
  (void)did_work;
#pragma unroll 1
    for (uint32_t s0 = t0; s0 < w1; s0 += P) {
    const uint32_t off = s0 - t0;
    uint32_t tf[4], tx[4], due[4];
    bool cand[4], slow[4];
    bool any_slow = false;
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      if (gb + u < g_end) {
        tf[u] = tf0[u] + off;
        tx[u] = tx0[u] + off;
        due[u] = __ldcg(d.due + (gb + u) * 32u + lane);
      } else {
        tf[u] = tx[u] = GS_NEVER;
        due[u] = GS_NEVER - 1u;
      }
      cand[u] = fast_ok && due[u] == tf[u] && tf[u] < w1;
      // anything else that is due inside the window takes the generic step below
      slow[u] = (due[u] == tf[u] && tf[u] < w1 && !fast_ok) || (due[u] == tx[u] && tx[u] < w1);
    }
    // ---- A. own columns of every candidate (independent loads, issued together) ----
    GsFastProbe f[4];
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (cand[u]) gs_fast_load(d, tf[u] & 1u, (gb + u) * 32u + lane, f[u]);
    // ---- B. ring entry -> target, status gathers ----
#pragma unroll
    for (int u = 0; u < 4; ++u)
      if (cand[u]) {
        const bool okk = gs_fast_target(d, h, tf[u] & 1u, (gb + u) * 32u + lane, f[u]);
        if (!okk) { cand[u] = false; slow[u] = true; }
      }
    // ---- C. commit ----
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      bool acked = false, done = false;
      if (cand[u]) {
        done = gs_fast_finish(d, h, sink, (gb + u) * 32u + lane, tf[u], f[u], &acked);
        if (!done) slow[u] = true;
        // an unanswered probe reaches its indirect stage at tf + T: inside this window it is stepped below
        else if (!acked && tf[u] + T < w1) slow[u] = true;
      }
      n_probe += done ? 1u : 0u;  // (per lane; summed over the warp at the end)
      n_ack += done && acked ? 1u : 0u;
      any_slow |= slow[u];
    }
    // ---- D. whatever is left: the generic step, tick by tick in ascending order ----
    if (__any_sync(0xFFFFFFFFu, any_slow)) {
      did_work = true;
#pragma unroll 1
      for (int u = 0; u < 4; ++u) {
        const bool sl = u == 0 ? slow[0] : u == 1 ? slow[1] : u == 2 ? slow[2] : slow[3];
        if (!__any_sync(0xFFFFFFFFu, sl)) continue;
        const uint32_t a = u == 0 ? tf[0] : u == 1 ? tf[1] : u == 2 ? tf[2] : tf[3];
        const uint32_t b = u == 0 ? tx[0] : u == 1 ? tx[1] : u == 2 ? tx[2] : tx[3];
        const uint32_t i = (gb + u) * 32u + lane;
#pragma unroll 1
        for (int which = 0; which < 2; ++which) {
          const uint32_t t = which == 0 ? (a < b ? a : b) : (a < b ? b : a);
          if (t >= w1) break;
          // (a member the fast path finished at `a` has moved its `due` on: it is not stepped twice)
          if (sl && __ldcg(d.due + i) == t) gs_row_step_any<COORDS>(&d, gp, i, t, 0u, s_stat, s_heard, s_q);
        }
      }
    }
    }  // ProbeIntervals of this launch
  counts[0] = n_probe;
  counts[1] = n_ack;
}

#ifndef GS_WIN_BLOCKS
#define GS_WIN_BLOCKS 4
#endif
// (resident CTAs per SM the window kernel is compiled for: 4 = 64 registers per thread)
#ifndef GS_WIN_BLOCKS_CLOSED
#define GS_WIN_BLOCKS_CLOSED 4
#endif

// PRISTINE = the instantiation for pools whose probes have a closed form (its own register allocation: it
// contains neither the per-probe loop nor that loop's arrays).
template <bool COORDS, bool PRISTINE>
__global__ void __launch_bounds__(GS_BLOCK, PRISTINE ? GS_WIN_BLOCKS_CLOSED : GS_WIN_BLOCKS)
    gs_window_kernel(const __grid_constant__ GsDev d, const GsGlobals* __restrict__ gp, uint32_t k_off, uint32_t n_ticks,
                     uint32_t mode) {
  __shared__ uint32_t s_stat[GS_NSTAT * 32];  // [counter][lane]
  __shared__ uint32_t s_heard[32 * 32];       // [broadcast slot][lane]
  __shared__ uint32_t s_q[2];
  __shared__ uint32_t s_spec[GS_MAX_SPECIAL + 1];  // [GS_MAX_SPECIAL] = how many
  const uint32_t tid = threadIdx.x;
  for (uint32_t x = tid; x < GS_NSTAT * 32u; x += GS_BLOCK) s_stat[x] = 0u;
  for (uint32_t x = tid; x < 32u * 32u; x += GS_BLOCK) s_heard[x] = 0u;
  if (tid == 64u) s_q[0] = 0u;
  if (tid == 65u) s_q[1] = GS_NEVER;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (tid == 66u) s_spec[GS_MAX_SPECIAL] = gs_special_members(*gp, s_spec);
  __syncthreads();
  const GsGlobals& g = *gp;
  const GsHot h = gs_hot(g);
  // mode bit 1: batches of four groups are dealt to the warps round-robin (neighbouring warps stream
  // neighbouring lines) instead of one contiguous run per warp
  const bool cyclic = (mode & 2u) != 0u;
  const uint32_t world = g.world, rank = g.rank, n_spec = s_spec[GS_MAX_SPECIAL];
  uint32_t* const qs = d.qstate[rank];
  const uint32_t t0 = *d.tick_base + k_off;
  // Where the chain of windows stands and how far it may go.  Both words are stable for the whole
  // launch: siblings only raise WIN_END to this window's own end, and lower HORIZON to ticks
  // >= t0 + ProbeInterval >= t0 + n_ticks.
  const uint32_t reached = __ldcg(qs + GS_Q_WIN_END), horizon = __ldcg(qs + GS_Q_HORIZON);
  if (reached < t0) return;  // an earlier window of this chain stopped at the horizon
  uint32_t w1 = t0 + n_ticks;
  if (horizon < w1) w1 = horizon;  // (GS_NEVER = no probe in flight anywhere)
  if (w1 <= t0) return;            // the horizon is here: the host goes back to single ticks
  if (world > 1u) gs_ranks_wait(d, g, t0);
  const uint32_t P = h.P, T = h.T, lane = tid & 31u, wib = tid >> 5;
  // this rank's groups of 32 members (4 per tile), dealt to the warps in contiguous runs: inside a
  // window rows are independent, so the unit of work need not be the 128-member phase tile
  uint32_t tile_lo = 0, tile_hi = (h.n + GS_TILE - 1u) / GS_TILE;
  if (world > 1u) {
    const uint32_t per = g.rows_per_rank / GS_TILE;
    tile_lo = rank * per < tile_hi ? rank * per : tile_hi;
    tile_hi = tile_lo + per < tile_hi ? tile_lo + per : tile_hi;
  }
  const uint32_t n_warps = gridDim.x * GS_WARPS, grp_lo = tile_lo * 4u, grp_hi = tile_hi * 4u;
  const uint32_t run = (grp_hi - grp_lo + n_warps - 1u) / n_warps;
  const uint32_t wid = blockIdx.x * GS_WARPS + wib;
  const uint32_t g_begin = grp_lo + wid * run < grp_hi ? grp_lo + wid * run : grp_hi;
  const uint32_t g_end = g_begin + run < grp_hi ? g_begin + run : grp_hi;
  const uint32_t shift = g.phase_shift + 2u, t0_mod = t0 % P, rot_p = g.rot_p;
  const uint32_t win_q = (w1 - t0) / P, win_r = (w1 - t0) - win_q * P;
  // the batch is taken through the probe fast path together if the pool allows the fast path at all
  const bool fast_ok =
      h.loss_thr == 0u && h.graph_n == 0u && d.coord == nullptr && d.imp_loss == nullptr && h.pp_interval == 0u;
  DevSinkT<COORDS> sink{s_stat, s_heard, s_q};
  bool did_work = false;
  uint32_t n_probe = 0, n_ack = 0;
  // phase of the first group, then incrementally (one division per warp, not per tile)
  uint32_t pg = g_begin >> shift;              // phase group of the current group
  uint32_t pp = (pg % P + rot_p) % P;          // its probe phase
  const uint32_t g_first = cyclic ? (grp_lo + wid * 4u < grp_hi ? grp_lo + wid * 4u : grp_hi) : g_begin;
  const uint32_t g_step = cyclic ? n_warps * 4u : 4u, g_lim = cyclic ? grp_hi : g_end;
  for (uint32_t gb = g_first; gb < g_lim; gb += g_step) {
    if (cyclic) {  // (a division per batch instead of one per warp)
      pg = gb >> shift;
      pp = (pg % P + rot_p) % P;
    }
    uint32_t tf0[4], tx0[4];
    // ---- 0. the first ticks >= t0 at which each group of the batch can be due ----
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const uint32_t grp = gb + u;
      if (grp < g_lim) {
        const uint32_t q = grp >> shift;
        if (q != pg) {                                   // groups are consecutive: the next phase group, phase + 1 (mod P)
          pp = pp + 1u == P ? 0u : pp + 1u;
          pg = q;
        }
        uint32_t a = pp + P - t0_mod;                    // first tick >= t0 congruent to the phase ...
        a = a >= P ? a - P : a;
        uint32_t b = a + T;                              // ... and to phase + ProbeTimeout
        b = b >= P ? b - P : b;
        tf0[u] = t0 + a;
        tx0[u] = t0 + b;
      } else {
        tf0[u] = tx0[u] = GS_NEVER;
      }
    }
    // ---- 1. fast-forward.  A member that is up, listed alive, idle and due at its ticker phase keeps its
    // probe state in registers and runs ALL its probes of the launch in a row: ring entry -> target ->
    // the target's status byte -> ack -> awareness - 1, due + ProbeInterval, cursor + 1.  A launch covers
    // one ProbeInterval in general and many when the host knows that no probe can go unanswered; either
    // way the loop stops at the first thing that is not this common case (ring wrap, a target that is
    // not up-alive-established, a slow link), writes the member's state back as it stood BEFORE that
    // probe, and the generic code below carries on from there.  Four groups in lock step: four
    // independent permutations and four gathers in flight per lane.
    // After an obstacle the generic path (2.) takes the ONE ProbeInterval that contains it and the
    // fast-forward resumes behind it: `lo` = the tick up to which this batch has been through 2.
    uint32_t lo = t0;
#pragma unroll 1
    for (;;) {
      uint32_t stuck = GS_NEVER;  // earliest ticker firing still inside the launch after the fast-forward
      if constexpr (PRISTINE) {
        // Closed form (gs_pristine_probes_k): every own column of the batch in ONE round of loads, then per
        // member one inverse ring permutation, no ring entries, no gathers; written back at once.
        uint32_t cnt = 0;
        uint32_t du[4], kk[4], mm[4], cu[4], pa[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          const uint32_t i = (gb + u) * 32u + lane;
          du[u] = GS_NEVER;
          kk[u] = mm[u] = cu[u] = pa[u] = 0u;
          if (gb + u < g_lim) {
            du[u] = __ldcg(d.due + i);
            if (fast_ok) {
              kk[u] = d.key[tf0[u] & 1u][i];  // (parity of the group's first firing; the rare other case reloads)
              mm[u] = d.meta[i];
              cu[u] = d.cursor[i];
              pa[u] = d.pass[i];
            }
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (gb + u >= g_lim) continue;
          const uint32_t i = (gb + u) * 32u + lane;
          uint32_t due = du[u];
          if (fast_ok && due >= lo && due < w1) {
            // on the ticker schedule of its group: the first firing of the launch, or (after an obstacle) a later one
            uint32_t later = 0u;
            bool on_phase = due == tf0[u];
            if (!on_phase && due > tf0[u]) {
              later = (due - tf0[u]) / P;
              on_phase = later * P == due - tf0[u];
            }
            if (on_phase) {
              const uint32_t k0 = ((due ^ tf0[u]) & 1u) ? d.key[due & 1u][i] : kk[u];
              const uint32_t m = mm[u];
              if (gs_key_truth(k0) == GS_TRUTH_UP && gs_key_rank(k0) == GS_RANK_ALIVE && gs_meta_stage(m) == GS_STAGE_IDLE &&
                  !(m & (GS_META_DIRTY | GS_META_ISOLATED))) {
                const GsU4 rk = gs_perm_keys(h.seed_lo, h.seed_hi, i, pa[u]);
                // firings inside the launch: ceil((w1 - tf0) / P) without a division (w1 - t0 = win_q P + win_r)
                const uint32_t kt = win_q + (win_r > tf0[u] - t0 ? 1u : 0u) - later;
                const uint32_t k = gs_pristine_probes_k(h.n, h.perm_bits, rk, i, cu[u], kt, s_spec, n_spec);
                if (k) {
                  const uint32_t aw = gs_meta_aw(m);
                  if (aw) d.meta[i] = gs_meta_set_aw(m, aw > k ? aw - k : 0u);
                  d.cursor[i] = cu[u] + k;
                  due += k * P;
                  d.due[i] = due;
                  cnt += k;
                }
              }
            }
          }
          if (due >= lo && due < w1 && due < stuck) stuck = due;  // still something due inside the launch
        }
        n_probe += cnt;  // per lane; summed over the warp once, at the end
        n_ack += cnt;
      } else
      {
        uint32_t mm[4], cu[4], du[4], m_in[4], cu_in[4], du_in[4], kt[4];
        GsU4 rk[4];
        bool live[4], in_rng[4];
        uint32_t cnt = 0;
        {
          // every own column of the batch in ONE round of loads (a member that turns out not to be due costs
          // 16 bytes it did not need; waiting for `due` first would cost every member a second round trip).
          // The key is read at the parity of the group's first firing and again in the rare other case.
          uint32_t kk[4], pa[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const uint32_t i = (gb + u) * 32u + lane;
            in_rng[u] = gb + u < g_lim;
            du[u] = GS_NEVER;
            kk[u] = mm[u] = cu[u] = pa[u] = 0u;
            if (in_rng[u]) {
              du[u] = __ldcg(d.due + i);
              if (fast_ok) {
                kk[u] = d.key[tf0[u] & 1u][i];
                mm[u] = d.meta[i];
                cu[u] = d.cursor[i];
                pa[u] = d.pass[i];
              }
            }
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            const uint32_t i = (gb + u) * 32u + lane;
            live[u] = false;
            kt[u] = 0u;
            m_in[u] = mm[u];
            cu_in[u] = cu[u];
            du_in[u] = du[u];
            if (!in_rng[u] || !fast_ok || du[u] < lo || du[u] >= w1) continue;
            // on the ticker schedule of its group: the first firing of the launch, or (after an obstacle) a later one
            uint32_t later = 0u;
            if (du[u] != tf0[u]) {
              if (du[u] < tf0[u]) continue;
              later = (du[u] - tf0[u]) / P;
              if (later * P != du[u] - tf0[u]) continue;
            }
            const uint32_t k = ((du[u] ^ tf0[u]) & 1u) ? d.key[du[u] & 1u][i] : kk[u];
            live[u] = gs_key_truth(k) == GS_TRUTH_UP && gs_key_rank(k) == GS_RANK_ALIVE &&
                      gs_meta_stage(mm[u]) == GS_STAGE_IDLE && !(mm[u] & (GS_META_DIRTY | GS_META_ISOLATED));
            rk[u] = gs_perm_keys(h.seed_lo, h.seed_hi, i, pa[u]);
            // firings inside the launch: ceil((w1 - tf0) / P) without a division (w1 - t0 = win_q P + win_r)
            kt[u] = win_q + (win_r > tf0[u] - t0 ? 1u : 0u) - later;
          }
        }
        for (;;) {
          bool go[4];
          bool any = false;
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            go[u] = live[u] && du[u] < w1;
            any |= go[u];
          }
          if (!__any_sync(0xFFFFFFFFu, any)) break;
          uint32_t c[4], kc[4];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            c[u] = 0u;
            if (go[u]) {
              if (cu[u] >= h.n) {  // ring wrap: re-keyed by the generic step
                live[u] = go[u] = false;
              } else {
                c[u] = gs_perm(cu[u], h.n, h.perm_bits, rk[u]);
                if (c[u] == (gb + u) * 32u + lane) live[u] = go[u] = false;  // own entry: skipped by the generic step
              }
            }
          }
#pragma unroll
          for (int u = 0; u < 4; ++u) kc[u] = go[u] ? gs_peer_key(d, du[u] & 1u, c[u], false) : 0u;
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            if (!go[u]) continue;
            const uint32_t i = (gb + u) * 32u + lane;
            if (gs_key_truth(kc[u]) != GS_TRUTH_UP || gs_key_rank(kc[u]) != GS_RANK_ALIVE || gs_key_pending(kc[u]) ||
                gs_extra(h, nullptr, i, c[u]) + gs_extra(h, nullptr, c[u], i) > T) {
              live[u] = false;  // anything but a prompt ack: the generic step decides
              continue;
            }
            const uint32_t aw = gs_meta_aw(mm[u]);
            mm[u] = gs_meta_set_aw(mm[u], aw ? aw - 1u : 0u);
            du[u] += P;
            cu[u] += 1u;
            ++cnt;
          }
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
          if (!in_rng[u]) continue;
          const uint32_t i = (gb + u) * 32u + lane;
          if (cu[u] != cu_in[u]) d.cursor[i] = cu[u];
          if (du[u] != du_in[u]) d.due[i] = du[u];
          if (mm[u] != m_in[u]) d.meta[i] = mm[u];
          if (du[u] >= lo && du[u] < w1 && du[u] < stuck) stuck = du[u];  // still something due inside the launch
        }
        n_probe += cnt;  // per lane; summed over the warp once, at the end
        n_ack += cnt;
      }
      stuck = __reduce_min_sync(0xFFFFFFFFu, stuck);
      if (stuck == GS_NEVER) break;
      // ---- 2. the ProbeInterval of the earliest obstacle takes the generic path (out of line: it is rare,
      // and its staging arrays would cost the loop above its registers)
      {
        const uint32_t off = (stuck - t0) / P * P, s_lo = t0 + off, s_hi = s_lo + P < w1 ? s_lo + P : w1;
        uint32_t add[2] = {0u, 0u};
        gs_window_generic<COORDS>(&d, gp, gb, g_lim, tf0[0] + off, tf0[1] + off, tf0[2] + off, tf0[3] + off, tx0[0] + off,
                                  tx0[1] + off, tx0[2] + off, tx0[3] + off, s_lo, s_hi, s_stat, s_heard, s_q, add);
        n_probe += add[0];
        n_ack += add[1];
        did_work = true;
        lo = s_lo + P;
        if (lo >= w1) break;
      }
    }
  }
  did_work |= n_probe != 0u;
  if (n_probe) {  // one shared-memory counter per lane (DevSinkT::stat)
    atomicAdd(&s_stat[GS_ST_PROBES * 32 + lane], n_probe);
    atomicAdd(&s_stat[GS_ST_ACTIVE_ROWS * 32 + lane], n_probe);
    if (n_ack) atomicAdd(&s_stat[GS_ST_ACKS * 32 + lane], n_ack);
  }
  if (world > 1u && did_work) __threadfence_system();  // horizon words on the peers, before the release
  __syncthreads();
  if (tid < GS_NSTAT) {
    uint32_t v = 0;
    for (uint32_t x = 0; x < 32u; ++x) v += s_stat[tid * 32u + ((x + tid) & 31u)];
    if (v) atomicAdd(&d.stats[tid], (unsigned long long)v);
  }
  if (tid == 0u) {
    // a quiet window never meets mail and never posts: if it did, the scheduling invariant is broken
    // ... and a launch that covers several ProbeIntervals was promised that no probe goes unanswered
    if (s_q[0] != 0u || (n_ticks > P && s_q[1] != GS_NEVER)) atomicExch(qs + GS_Q_VIOLATION, t0 + 1u);
    s_q[0] = 0u;
    gs_q_publish(d, g, s_q, t0);
    atomicMax(qs + GS_Q_WIN_END, w1);
  }
  if (world > 1u) gs_ranks_release(d, g, w1);
}

// Horizon of the pool as it stands (run before the first window after single ticks): the minimum,
// over running members with a probe in flight, of the tick at which it can end in an accusation.
__global__ void __launch_bounds__(GS_BLOCK)
    gs_quiet_scan_kernel(GsDev d, const GsGlobals* __restrict__ gp, uint32_t now, const uint32_t* now_at, uint32_t first,
                         uint32_t count) {
  __shared__ uint32_t s_min;
  if (threadIdx.x == 0u) s_min = GS_NEVER;
  __syncthreads();
  const GsGlobals& g = *gp;
  if (now_at != nullptr) now = *now_at;  // (inside a graph: the device clock)
  uint32_t h = GS_NEVER;
  for (uint32_t x = blockIdx.x * GS_BLOCK + threadIdx.x; x < count; x += gridDim.x * GS_BLOCK) {
    const uint32_t i = first + x;
    if (i >= g.n) break;
    if (gs_key_truth(d.key[now & 1u][i]) != GS_TRUTH_UP) continue;
    const uint32_t stage = gs_meta_stage(d.meta[i]);
    if (stage == GS_STAGE_IDLE) continue;
    const uint32_t due = d.due[i];
    const uint32_t e = stage == GS_STAGE_WAIT_T ? due - g.T + g.P : due;  // probe start + P, or the deadline itself
    if (e < h) h = e;
  }
  h = __reduce_min_sync(0xFFFFFFFFu, h);
  if ((threadIdx.x & 31u) == 0u && h != GS_NEVER) atomicMin(&s_min, h);
  __syncthreads();
  if (threadIdx.x == 0u && s_min != GS_NEVER) {
    if (g.world <= 1u) atomicMin(d.qstate[0] + GS_Q_HORIZON, s_min);
    else for (uint32_t r = 0; r < g.world; ++r) atomicMin_system(d.qstate[r] + GS_Q_HORIZON, s_min);
  }
}

// End of a chain of windows: the device clock moves to wherever the chain got.
__global__ void gs_window_advance_kernel(uint32_t* tick_base, const uint32_t* qs) { *tick_base = qs[GS_Q_WIN_END]; }

__global__ void gs_advance_kernel(uint32_t* tick_base, uint32_t k, uint32_t* done_ctr) {
  *tick_base += k;
  if (done_ctr) *done_ctr = 0u;
}

// A tick stretch (CudaBackend::run_tick_stretch): begin, the end of each pass of its loop, and its end.
__global__ void gs_stretch_begin_kernel(GsStretchCtl* c, uint32_t end, uint32_t floor, uint32_t depth) {
  c->out = GsStretch();
  c->violation = 0u;
  c->end = end;
  c->floor = floor;
  c->depth = depth;
}
// After a pass of `k` tick launches: the device clock moves on by the ticks that ran (the launches of the
// pass apply the same rule: every tick before the stop ran, none after it), and the loop ends at the stop.
__global__ void gs_stretch_pass_kernel(uint32_t* tick_base, const uint32_t* qs, GsStretchCtl* c, uint32_t k,
                                       cudaGraphConditionalHandle loop) {
  const uint32_t t = *tick_base, la = qs[GS_Q_LAST_ACTIVE];
  const uint32_t stop = gs_stretch_stop(*c, la);
  const uint32_t ran = stop <= t ? 0u : stop - t < k ? stop - t : k;
  *tick_base = t + ran;
  c->out.ran += ran;
  c->out.launches += k;
  if (t + ran >= stop || qs[GS_Q_VIOLATION] != 0u) {
    c->out.last_active = la;
    c->out.quiet = t + ran >= (la > c->floor ? la : c->floor) + c->depth ? 1u : 0u;
    c->violation = qs[GS_Q_VIOLATION];
    cudaGraphSetConditional(loop, 0u);
  }
}
// Stopped at a quiet tick: the quiet probe runs (horizon reset here, then scan and counts).
__global__ void gs_stretch_end_kernel(const GsStretchCtl* c, uint32_t* qs, cudaGraphConditionalHandle probe) {
  if (c->out.quiet && !c->violation) {
    qs[GS_Q_HORIZON] = GS_NEVER;
    cudaGraphSetConditional(probe, 1u);
  }
}

// Cross-GPU barrier (sharded pools).  One warp: lane r publishes this rank's new epoch into
// slot `rank` of rank r's flag array (release, system scope, over NVLink) and then spins on
// slot r of its own array until rank r has published the same epoch.  Everything the preceding
// tick kernel wrote — including remote atomics into peers' mailboxes — happens-before the
// release, so a rank that leaves the barrier sees every delivery addressed to it.
__global__ void gs_xbar_kernel(GsXbar xb) {
  const uint32_t lane = threadIdx.x;
  const uint32_t e = *xb.epoch + 1u;
  __threadfence_system();
  if (lane < xb.world) {
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(xb.flags[lane] + xb.rank), "r"(e) : "memory");
    uint32_t v;
    do {
      asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(xb.flags[xb.rank] + lane) : "memory");
    } while ((int32_t)(v - e) < 0);
  }
  __syncwarp();
  __threadfence_system();
  if (lane == 0) *xb.epoch = e;
}

__global__ void __launch_bounds__(GS_BLOCK)
    gs_init_kernel(GsDev d, const GsGlobals* __restrict__ gp, uint32_t first, uint32_t count,
                   uint32_t now) {
  uint32_t x = blockIdx.x * GS_BLOCK + threadIdx.x;
  if (x < count) gs_init_row(d, *gp, first + x, now);
}

__global__ void __launch_bounds__(GS_BLOCK)
    gs_crash_kernel(GsDev d, const GsGlobals* __restrict__ gp, uint32_t thr, uint32_t salt,
                    uint32_t* n_crashed) {
  uint32_t i = blockIdx.x * GS_BLOCK + threadIdx.x;
  bool c = false;
  if (i < gp->n) c = gs_crash_row(d, *gp, i, thr, salt);
  unsigned b = __ballot_sync(0xFFFFFFFFu, c);
  if ((threadIdx.x & 31u) == 0u && b) atomicAdd(n_crashed, (uint32_t)__popc(b));
}

// gsim_impair_fraction / gsim_impair_dir_fraction: gs_impair_row for member i, counts[0] += selected,
// counts[1] += selected members that were impaired before.
__global__ void __launch_bounds__(GS_BLOCK)
    gs_impair_kernel(GsDev d, const GsGlobals* __restrict__ gp, GsImpairCols c, uint32_t thr, uint32_t salt,
                     GsImpairVal v, uint32_t* counts) {
  const uint32_t i = blockIdx.x * GS_BLOCK + threadIdx.x;
  uint32_t r = 0u;
  if (i < gp->n) r = gs_impair_row(d.key[0][i], c, gp->seed_lo, gp->seed_hi, i, thr, salt, v);
  const unsigned sel = __ballot_sync(0xFFFFFFFFu, r & 1u), was = __ballot_sync(0xFFFFFFFFu, r & 2u);
  if ((threadIdx.x & 31u) == 0u && sel) {
    atomicAdd(&counts[0], (uint32_t)__popc(sel));
    if (was) atomicAdd(&counts[1], (uint32_t)__popc(was));
  }
}

// gsim_impair_flap_fraction: gs_flap_row for member i, counts[0] += selected, counts[1] += selected members
// that had a schedule before.
__global__ void __launch_bounds__(GS_BLOCK)
    gs_flap_kernel(GsDev d, const GsGlobals* __restrict__ gp, uint32_t* col, uint32_t thr, uint32_t salt, uint32_t w,
                   uint32_t* counts) {
  const uint32_t i = blockIdx.x * GS_BLOCK + threadIdx.x;
  uint32_t r = 0u;
  if (i < gp->n) r = gs_flap_row(d.key[0][i], col, gp->seed_lo, gp->seed_hi, i, thr, salt, w);
  const unsigned sel = __ballot_sync(0xFFFFFFFFu, r & 1u), was = __ballot_sync(0xFFFFFFFFu, r & 2u);
  if ((threadIdx.x & 31u) == 0u && sel) {
    atomicAdd(&counts[0], (uint32_t)__popc(sel));
    if (was) atomicAdd(&counts[1], (uint32_t)__popc(was));
  }
}

// gsim_impair_flap_stats: out[0] += members with a schedule, out[1] += those in a bad epoch at tick now,
// aggregated per warp (a ballot) and per CTA (one global atomic per count).
__global__ void __launch_bounds__(GS_BLOCK)
    gs_flap_stats_kernel(const uint32_t* __restrict__ col, uint32_t n, uint32_t seed_lo, uint32_t seed_hi, uint32_t now,
                         unsigned long long* out) {
  __shared__ uint32_t s[2];
  if (threadIdx.x < 2u) s[threadIdx.x] = 0u;
  __syncthreads();
  for (size_t i0 = (size_t)blockIdx.x * GS_BLOCK; i0 < n; i0 += (size_t)gridDim.x * GS_BLOCK) {
    const size_t i = i0 + threadIdx.x;
    const uint32_t w = i < n ? col[i] : 0u;
    const bool bad = w != 0u && gs_flap_bad(seed_lo, seed_hi, (uint32_t)i, w, now);
    const unsigned has = __ballot_sync(0xFFFFFFFFu, w != 0u), b = __ballot_sync(0xFFFFFFFFu, bad);
    if ((threadIdx.x & 31u) == 0u && has) {
      atomicAdd(&s[0], (uint32_t)__popc(has));
      if (b) atomicAdd(&s[1], (uint32_t)__popc(b));
    }
  }
  __syncthreads();
  if (threadIdx.x < 2u && s[threadIdx.x]) atomicAdd(&out[threadIdx.x], (unsigned long long)s[threadIdx.x]);
}

// gsim_domain_set_range: dom[first + x] = first_domain + x / per_domain.
__global__ void __launch_bounds__(GS_BLOCK)
    gs_domain_range_kernel(uint32_t* dom, uint32_t first, uint32_t count, uint32_t per_domain, uint32_t first_domain) {
  const uint32_t x = blockIdx.x * GS_BLOCK + threadIdx.x;
  if (x < count) dom[first + x] = first_domain + x / per_domain;
}

// gsim_domain_impair / _crash / _pause: gs_domain_op_row for member i when its domain is listed; counts[0] and
// counts[1] += the two result bits, aggregated per warp.
__global__ void __launch_bounds__(GS_BLOCK)
    gs_domain_op_kernel(GsDev d, const GsGlobals* __restrict__ gp, const uint32_t* __restrict__ dom,
                        const uint32_t* __restrict__ bits, uint32_t n_words, GsDomainOp a, uint32_t* counts) {
  const uint32_t i = blockIdx.x * GS_BLOCK + threadIdx.x;
  uint32_t r = 0u;
  if (i < gp->n && gs_domain_listed(dom, bits, n_words, i)) r = gs_domain_op_row(d, *gp, a, i);
  const unsigned c0 = __ballot_sync(0xFFFFFFFFu, r & 1u), c1 = __ballot_sync(0xFFFFFFFFu, r & 2u);
  if ((threadIdx.x & 31u) == 0u) {
    if (c0) atomicAdd(&counts[0], (uint32_t)__popc(c0));
    if (c1) atomicAdd(&counts[1], (uint32_t)__popc(c1));
  }
}

// gsim_domain_stats_read: out[dom[i] - first_domain] += gs_domain_stats_row of member i, grid-stride.  Lanes
// whose members share a domain (the usual case: gsim_domain_set_range gives neighbours one domain) are summed
// in the warp first (__match_any_sync, then one reduction per packed word), so each domain a warp touches
// takes one set of atomics.
__global__ void __launch_bounds__(GS_BLOCK)
    gs_domain_stats_kernel(GsDev d, GsDomainCols c, uint32_t n, uint32_t seed_lo, uint32_t seed_hi, uint32_t now,
                           uint32_t first_domain, uint32_t count, GsDomainStats* out) {
  const uint32_t lane = threadIdx.x & 31u;
  for (size_t i0 = (size_t)blockIdx.x * GS_BLOCK; i0 < n; i0 += (size_t)gridDim.x * GS_BLOCK) {
    const uint32_t i = (uint32_t)(i0 + threadIdx.x);
    uint32_t v[3] = {0u, 0u, 0u}, x = 0xFFFFFFFFu;
    bool on = false;
    if (i < n) {
      x = c.dom[i] - first_domain;
      on = x < count && gs_domain_stats_row(d, seed_lo, seed_hi, c, i, now, v);
    }
    const unsigned act = __ballot_sync(0xFFFFFFFFu, on);
    if (!on) continue;
    const unsigned peers = __match_any_sync(act, x);
    const uint32_t s0 = __reduce_add_sync(peers, v[0]), s1 = __reduce_add_sync(peers, v[1]);
    const uint32_t s2 = __reduce_add_sync(peers, v[2]), mx = __reduce_max_sync(peers, v[2]);
    if (lane != (uint32_t)__ffs(peers) - 1u) continue;
    GsDomainStats& o = out[x];
    atomicAdd(&o.members, s0 & 63u);
    if ((s0 >> 6) & 63u) atomicAdd(&o.running, (s0 >> 6) & 63u);
    if ((s0 >> 12) & 63u) atomicAdd(&o.paused, (s0 >> 12) & 63u);
    if ((s0 >> 18) & 63u) atomicAdd(&o.impaired, (s0 >> 18) & 63u);
    if ((s0 >> 24) & 63u) atomicAdd(&o.in_force, (s0 >> 24) & 63u);
    if (s1 & 63u) atomicAdd(&o.alive, s1 & 63u);
    if ((s1 >> 6) & 63u) atomicAdd(&o.suspect, (s1 >> 6) & 63u);
    if ((s1 >> 12) & 63u) atomicAdd(&o.dead, (s1 >> 12) & 63u);
    if ((s1 >> 18) & 63u) atomicAdd(&o.left, (s1 >> 18) & 63u);
    if (mx) atomicMax(&o.awareness_max, mx);
    if (s2) atomicAdd(reinterpret_cast<unsigned long long*>(&o.awareness_sum), (unsigned long long)s2);
  }
}

// gsim_pause_many (ids != nullptr: thread x takes member ids[x], no id twice) and gsim_pause_fraction (thread i
// takes member i): gs_pause_row, *n_paused += members paused.
__global__ void __launch_bounds__(GS_BLOCK)
    gs_pause_kernel(GsDev d, const GsGlobals* __restrict__ gp, uint32_t* pause_until, const uint32_t* __restrict__ ids,
                    uint32_t n, uint32_t thr, uint32_t salt, uint32_t until, uint32_t* n_paused) {
  const uint32_t x = blockIdx.x * GS_BLOCK + threadIdx.x;
  const GsGlobals& g = *gp;
  bool c = false;
  if (ids != nullptr) {
    if (x < n) c = gs_pause_row(d, g, pause_until, ids[x], until);
  } else if (x < g.n && gs_pause_pick(g, x, thr, salt)) {
    c = gs_pause_row(d, g, pause_until, x, until);
  }
  const unsigned b = __ballot_sync(0xFFFFFFFFu, c);
  if ((threadIdx.x & 31u) == 0u && b) atomicAdd(n_paused, (uint32_t)__popc(b));
}

// gs_resume_row over every member at tick t; counts[c - 1] += members with resume code c.
__global__ void __launch_bounds__(GS_BLOCK)
    gs_resume_kernel(GsDev d, const GsGlobals* __restrict__ gp, uint32_t* pause_until, uint32_t t, uint32_t resume,
                     uint32_t log_events, uint32_t* counts) {
  const uint32_t i = blockIdx.x * GS_BLOCK + threadIdx.x;
  uint32_t r = 0u;
  if (i < gp->n) r = gs_resume_row(d, *gp, pause_until, i, t, resume != 0u);
  if (r == GS_RESUMED_DEAD && log_events) {  // serf's handleNodeJoin of a Failed member
    DevSink sink{nullptr, nullptr, nullptr};
    sink.log_event(d, *gp, t, GS_EV_MEMBER_JOIN, i, GS_EMPTY32, 0u);
  }
  if (__ballot_sync(0xFFFFFFFFu, r != 0u) == 0u) return;
  for (uint32_t c = 0; c < 4u; ++c) {
    const unsigned b = __ballot_sync(0xFFFFFFFFu, r == c + 1u);
    if ((threadIdx.x & 31u) == 0u && b) atomicAdd(&counts[c], (uint32_t)__popc(b));
  }
}

__global__ void __launch_bounds__(GS_BLOCK)
    gs_reap_kernel(GsDev d, const GsGlobals* __restrict__ gp, uint32_t now, uint32_t reconnect_ticks,
                   uint32_t tombstone_ticks, uint32_t log_events, uint32_t* counts) {
  const uint32_t i = blockIdx.x * GS_BLOCK + threadIdx.x;
  uint32_t r = 0;
  if (i < gp->n) r = gs_reap_row(d, *gp, i, now, reconnect_ticks, tombstone_ticks);
  if (r && log_events) {
    DevSink sink{nullptr, nullptr, nullptr};
    sink.log_event(d, *gp, now, GS_EV_MEMBER_REAP, i, GS_EMPTY32, 0u);
  }
  const unsigned b0 = __ballot_sync(0xFFFFFFFFu, (r & 1u) != 0u), b1 = __ballot_sync(0xFFFFFFFFu, (r & 2u) != 0u);
  if ((threadIdx.x & 31u) == 0u) {
    if (b0) atomicAdd(&counts[0], (uint32_t)__popc(b0));
    if (b1) atomicAdd(&counts[1], (uint32_t)__popc(b1));
  }
}

__global__ void __launch_bounds__(GS_BLOCK)
    gs_recount_kernel(GsDev d, const GsGlobals* __restrict__ gp, uint32_t now, const uint32_t* now_at, uint32_t first,
                      uint32_t count, GsRecount* out) {
  __shared__ GsRecount s;
  uint32_t* sw = reinterpret_cast<uint32_t*>(&s);
  for (uint32_t x = threadIdx.x; x < sizeof(GsRecount) / 4; x += GS_BLOCK) sw[x] = 0u;
  __syncthreads();
  const GsGlobals& g = *gp;
  if (now_at != nullptr) now = *now_at;  // (inside a graph: the device clock)
  const uint32_t x = blockIdx.x * GS_BLOCK + threadIdx.x, i = first + x;
  if (x < count && i < g.n) {
    uint32_t k = d.key[now & 1u][i];
    uint32_t truth = gs_key_truth(k), rank = gs_key_rank(k);
    atomicAdd(&s.truth_cnt[truth], 1u);
    if (truth != GS_TRUTH_NONE) atomicAdd(&s.rank_cnt[rank], 1u);
    if (truth == GS_TRUTH_CRASHED && rank < GS_RANK_DEAD) atomicAdd(&s.crashed_alive, 1u);
    if ((truth == GS_TRUTH_CRASHED || truth == GS_TRUTH_GONE) && rank < GS_RANK_DEAD) atomicAdd(&s.unreachable_live, 1u);
    if (truth == GS_TRUTH_UP && (d.meta[i] & GS_META_ISOLATED)) atomicAdd(&s.isolated_up, 1u);
    if (truth != GS_TRUTH_NONE && gs_key_pending(k)) atomicAdd(&s.pending, 1u);
    if (truth == GS_TRUTH_UP && g.active_mask) {
      uint32_t h = d.heard[i] & g.active_mask, q = d.queued[i] & g.active_mask;
      while (h) {
        uint32_t r = __ffs(h) - 1;
        h &= h - 1;
        atomicAdd(&s.heard_cnt[r], 1u);
      }
      while (q) {
        uint32_t r = __ffs(q) - 1;
        q &= q - 1;
        atomicAdd(&s.queued_cnt[r], 1u);
      }
    }
  }
  __syncthreads();
  uint32_t* ow = reinterpret_cast<uint32_t*>(out);
  for (uint32_t x = threadIdx.x; x < sizeof(GsRecount) / 4; x += GS_BLOCK)
    if (sw[x]) atomicAdd(&ow[x], sw[x]);
}

__global__ void __launch_bounds__(GS_BLOCK)
    gs_hash_kernel(GsDev d, const GsGlobals* __restrict__ gp, uint32_t now,
                   unsigned long long* out) {
  __shared__ unsigned long long s[4];
  if (threadIdx.x < 4) s[threadIdx.x] = 0ull;
  __syncthreads();
  uint32_t i = blockIdx.x * GS_BLOCK + threadIdx.x;
  if (i < gp->n) {
    uint64_t h = gs_hash_row(d, *gp, i, now);
    if (h) {
      uint64_t lanes[4];
      gs_hash_lanes(h, lanes);
      for (int q = 0; q < 4; ++q) atomicAdd(&s[q], (unsigned long long)lanes[q]);
    }
  }
  __syncthreads();
  if (threadIdx.x < 4 && s[threadIdx.x]) atomicAdd(&out[threadIdx.x], s[threadIdx.x]);
}

// ---- per-agent observation (gs_agent.h): read-only ----------------------------------------------------
// gsim_agent_stats_read, first pass over the key column: est[r] += established members of rank r.
__global__ void __launch_bounds__(GS_BLOCK)
    gs_agent_est_kernel(const uint32_t* __restrict__ key, uint32_t n, uint32_t* est) {
  uint32_t c[4] = {0u, 0u, 0u, 0u};
  for (size_t i = (size_t)blockIdx.x * GS_BLOCK + threadIdx.x; i < n; i += (size_t)gridDim.x * GS_BLOCK) {
    const uint32_t r1 = gs_established_rank1(key[i]);
#pragma unroll
    for (uint32_t r = 0; r < 4u; ++r) c[r] += r1 == r + 1u ? 1u : 0u;
  }
#pragma unroll
  for (uint32_t r = 0; r < 4u; ++r) {
    const uint32_t s = __reduce_add_sync(0xFFFFFFFFu, c[r]);
    if ((threadIdx.x & 31u) == 0u && s) atomicAdd(&est[r], s);
  }
}

struct GsClassMasks {
  uint32_t m[3];
};

// ... second pass: thread x computes the stats of member first + x.
__global__ void __launch_bounds__(GS_BLOCK)
    gs_agent_stats_kernel(GsAgentCols c, GsClassMasks cm, const uint32_t* __restrict__ est,
                          const __grid_constant__ GsPendingAlive pa, uint32_t first, uint32_t count, GsAgentStats* out) {
  const uint32_t x = blockIdx.x * GS_BLOCK + threadIdx.x;
  if (x >= count) return;
  const uint32_t e[4] = {est[0], est[1], est[2], est[3]};
  out[x] = gs_agent_stats_row(c, cm.m, e, pa, first + x);
}

// gsim_health_histogram: out[b] += members in bin b, aggregated per warp (one shared atomic per distinct bin
// of 32 members) and per CTA (one global atomic per bin).
__global__ void __launch_bounds__(GS_BLOCK)
    gs_health_hist_kernel(const uint32_t* __restrict__ key, const uint32_t* __restrict__ meta, GsImpairCols imp,
                          uint32_t n, unsigned long long* out) {
  __shared__ uint32_t s[GS_HIST_BINS];
  if (threadIdx.x < GS_HIST_BINS) s[threadIdx.x] = 0u;
  __syncthreads();
  const uint32_t lane = threadIdx.x & 31u;
  for (size_t i0 = (size_t)blockIdx.x * GS_BLOCK; i0 < n; i0 += (size_t)gridDim.x * GS_BLOCK) {
    const size_t i = i0 + threadIdx.x;
    const uint32_t b = i < n ? gs_health_bin(key[i], meta[i], imp, (uint32_t)i) : GS_HIST_NONE;
    const unsigned peers = __match_any_sync(0xFFFFFFFFu, b);
    if (b != GS_HIST_NONE && lane == (uint32_t)__ffs(peers) - 1u) atomicAdd(&s[b], (uint32_t)__popc(peers));
  }
  __syncthreads();
  if (threadIdx.x < GS_HIST_BINS && s[threadIdx.x]) atomicAdd(&out[threadIdx.x], (unsigned long long)s[threadIdx.x]);
}

// The tick and window kernels with COORDS = true: pools with network coordinates or flap schedules (member or domain).
static bool gs_kernel_extras(const GsDev& d) {
  return d.coord != nullptr || d.imp_flap != nullptr || d.dom_flap != nullptr;
}

// Tick launches use programmatic stream serialization (PDL) so consecutive ticks overlap
// launch latency and prologue with the previous tick's tail.
static cudaError_t gs_launch_tick(uint32_t blocks, cudaStream_t stream, const GsDev& d,
                                  const GsGlobals* g_dev, uint32_t k, bool pdl,
                                  const GsStretchCtl* stretch = nullptr) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(blocks);
  cfg.blockDim = dim3(GS_BLOCK);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  return gs_kernel_extras(d) ? cudaLaunchKernelEx(&cfg, gs_tick_kernel<true>, d, g_dev, k, stretch)
                 : cudaLaunchKernelEx(&cfg, gs_tick_kernel<false>, d, g_dev, k, stretch);
}

static cudaError_t gs_launch_window(uint32_t blocks, cudaStream_t stream, const GsDev& d, const GsGlobals* g_dev,
                                    uint32_t k_off, uint32_t n_ticks, bool pdl, uint32_t mode) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(blocks);
  cfg.blockDim = dim3(GS_BLOCK);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl ? 1 : 0;
  if (mode & 1u)  // pristine pool: the closed-form instantiation
    return gs_kernel_extras(d) ? cudaLaunchKernelEx(&cfg, gs_window_kernel<true, true>, d, g_dev, k_off, n_ticks, mode)
                   : cudaLaunchKernelEx(&cfg, gs_window_kernel<false, true>, d, g_dev, k_off, n_ticks, mode);
  return gs_kernel_extras(d) ? cudaLaunchKernelEx(&cfg, gs_window_kernel<true, false>, d, g_dev, k_off, n_ticks, mode)
                 : cudaLaunchKernelEx(&cfg, gs_window_kernel<false, false>, d, g_dev, k_off, n_ticks, mode);
}

#define GS_ROWS_MAX 64u  // rows one gs_rows_read_kernel launch gathers (8 words each: 2 KB of scratch)
struct GsRowIds {
  uint32_t n;
  uint32_t id[GS_ROWS_MAX];
};
__global__ void gs_rows_read_kernel(GsDev d, GsRowIds r, uint32_t* out) {
  const uint32_t* col[8] = {d.key[0], d.key[1], d.meta, d.heard, d.queued, d.ltime_member, d.ltime_event, d.event_min};
  const uint32_t t = threadIdx.x;
  if (t < r.n * 8u) out[t] = col[t & 7u][r.id[t >> 3]];
}

// A host operation's small writes (GsWriteBatch), in order; the fence makes them visible to the other
// GPUs of a sharded pool before anything this stream runs later (their barrier) can let those go on.
__global__ void gs_write_batch_kernel(const __grid_constant__ GsWriteBatch b) {
  for (uint32_t k = 0; k < b.n; ++k) gs_apply_write(b.op[k]);
  __threadfence_system();
}

// The quiet probe's horizon, next to its counts in scratch: one readback for both
__global__ void gs_copy_word_kernel(uint32_t* dst, const uint32_t* src) { *dst = *src; }

__global__ void __launch_bounds__(GS_BLOCK) gs_fill32_kernel(uint32_t* dst, uint32_t value, size_t count) {
  for (size_t x = (size_t)blockIdx.x * GS_BLOCK + threadIdx.x; x < count; x += (size_t)gridDim.x * GS_BLOCK)
    dst[x] = value;
}

__global__ void __launch_bounds__(GS_BLOCK) gs_and_kernel(GsDev d, uint32_t first, uint32_t count, uint32_t keep) {
  const uint32_t x = blockIdx.x * GS_BLOCK + threadIdx.x, i = first + x;
  if (x >= count) return;
  uint32_t v;
  v = d.heard[i];
  if (v & ~keep) d.heard[i] = v & keep;
  v = d.queued[i];
  if (v & ~keep) d.queued[i] = v & keep;
  for (uint32_t s = 0; s < GS_RING_MAX && d.inbox[s] != nullptr; ++s) {
    v = d.inbox[s][i];
    if (v & ~keep) d.inbox[s][i] = v & keep;
  }
}

// ---- network-coordinate queries (gs_query.h, DESIGN.md §3.4 "Queries") ------------------------------
// Rows of 11 doubles for GS_BLOCK members per CTA: each member's published slot is read coalesced over the
// SoA planes into shared memory, then the CTA writes its rows out contiguously.
__global__ void __launch_bounds__(GS_BLOCK)
    gs_coord_rows_kernel(GsDev d, uint32_t cap, uint32_t first, uint32_t count, double* rows) {
  __shared__ GsCoord s[GS_BLOCK];
  const uint32_t x0 = blockIdx.x * GS_BLOCK;
  const uint32_t m = count - x0 < GS_BLOCK ? count - x0 : GS_BLOCK;
  if (threadIdx.x < m) gs_coord_pick(d.coord, d.ctag, cap, first + x0 + threadIdx.x, s[threadIdx.x]);
  __syncthreads();
  const double* sw = reinterpret_cast<const double*>(s);
  double* out = rows + (size_t)x0 * GS_COORD_WORDS;
  for (uint32_t t = threadIdx.x; t < m * GS_COORD_WORDS; t += GS_BLOCK) out[t] = sw[t];
}

__global__ void __launch_bounds__(GS_BLOCK)
    gs_coord_pairs_kernel(GsDev d, const GsGlobals* __restrict__ gp, uint32_t now, const uint32_t* a, const uint32_t* b,
                          uint32_t n, double* est, double* tru) {
  const uint32_t k = blockIdx.x * GS_BLOCK + threadIdx.x;
  if (k >= n) return;
  const GsGlobals& g = *gp;
  const uint32_t i = a[k], j = b[k];
  GsCoord ci, cj;
  gs_coord_pick(d.coord, d.ctag, g.cap, i, ci);
  gs_coord_pick(d.coord, d.ctag, g.cap, j, cj);
  est[k] = gs_coord_distance_seconds(ci, cj);
  if (tru != nullptr) tru[k] = gs_model_rtt(g, d, i, j, now);
}

__global__ void __launch_bounds__(GS_BLOCK)
    gs_coord_dist_kernel(GsDev d, const GsGlobals* __restrict__ gp, uint32_t now, uint32_t from, const uint32_t* ids,
                         uint32_t n, uint32_t router, uint64_t* key, uint32_t* val) {
  const uint32_t x = blockIdx.x * GS_BLOCK + threadIdx.x;
  if (x >= n) return;
  const GsGlobals& g = *gp;
  GsCoord cf;
  gs_coord_pick(d.coord, d.ctag, g.cap, from, cf);  // (the same 11 words for every thread: L1 broadcasts)
  const uint32_t s = ids != nullptr ? ids[x] : x;
  uint64_t k;
  uint32_t v = s;
  if (router) {
    gs_router_entry(d, g, now, from, cf, s, &k, &v);
  } else {
    GsCoord c;
    gs_coord_pick(d.coord, d.ctag, g.cap, s, c);
    k = gs_dist_key(gs_coord_distance_seconds(cf, c));
  }
  // device assertion: the radix sort orders these bits as unsigned integers, which is the order of the
  // distances only for finite values with the sign clear (__trap, not assert: no host-call machinery)
  if (v != GS_EMPTY32 && !gs_dist_key_ok(k)) __trap();
  key[x] = k;
  val[x] = v;
}

// Chunk c of gsim_coordinate_error's draws is CTA c: every thread takes one draw, thread 0 adds the kept
// errors in draw order.
__global__ void __launch_bounds__(GS_BLOCK)
    gs_coord_error_kernel(GsDev d, const GsGlobals* __restrict__ gp, uint32_t now, uint32_t n_draws, uint32_t salt,
                          uint64_t* key, uint32_t* val, double* part) {
  static_assert(GS_ERR_CHUNK == GS_BLOCK, "one CTA per chunk of draws");
  __shared__ double s[GS_BLOCK];
  const uint32_t k = blockIdx.x * GS_BLOCK + threadIdx.x;
  double e = -1.0;
  if (k < n_draws) {
    e = gs_error_draw(d, *gp, now, k, salt);
    const uint64_t bits = e < 0.0 ? ~0ull : gs_dist_key(e);
    if (e >= 0.0 && !gs_dist_key_ok(bits)) __trap();  // device assertion, as in gs_coord_dist_kernel
    key[k] = bits;
    val[k] = k;
  }
  s[threadIdx.x] = e;
  __syncthreads();
  if (threadIdx.x == 0) {
    double sum = 0.0, kept = 0.0;
    for (uint32_t x = 0; x < GS_BLOCK; ++x)
      if (s[x] >= 0.0) {
        sum = sum + s[x];
        kept += 1.0;
      }
    part[blockIdx.x] = sum;
    part[gridDim.x + blockIdx.x] = kept;
  }
}

__global__ void gs_coord_error_finish_kernel(const uint64_t* sorted, uint32_t n_draws, const double* part, double* out) {
  gs_error_finish(sorted, n_draws, part, out);
}

// Per-datacenter medians over pairs sorted by (gs_dc_digit, key): thread c finds datacenter c's run by binary
// search.
__global__ void gs_dc_medians_kernel(const uint64_t* key, const uint32_t* val, uint32_t n, uint32_t n_dcs, double* med,
                                     uint32_t* cnt) {
  const uint32_t c = threadIdx.x;
  if (c >= n_dcs) return;
  uint32_t lo = 0, hi = n;  // first entry with digit >= c
  while (lo < hi) {
    const uint32_t mid = lo + (hi - lo) / 2u;
    if (gs_dc_digit(val[mid], n_dcs) < c) lo = mid + 1u; else hi = mid;
  }
  uint32_t end = lo, top = n;  // first entry with digit > c
  while (end < top) {
    const uint32_t mid = end + (top - end) / 2u;
    if (gs_dc_digit(val[mid], n_dcs) <= c) end = mid + 1u; else top = mid;
  }
  cnt[c] = end - lo;
  med[c] = end > lo ? gs_key_dist(key[lo + (end - lo) / 2u]) : gs_key_dist(0x7FF0000000000000ull);
}

// ---- stable LSD radix sort of (u64 key, u32 value) pairs ---------------------------------------------
// 8-bit digits: passes 0..7 over the key from the least significant byte, then (by datacenter) pass 8 over
// gs_dc_digit(value).  Per pass: an upsweep histogram per tile of GS_RS_TILE pairs, an exclusive scan of every
// digit's counts over the tiles, and a scatter that ranks each tile's pairs stably (warp match + per-warp
// digit counts, rounds of GS_BLOCK pairs in input order).  One histogram of every pass up front lets the
// device skip a pass whose digit is the same for every pair; which buffer each pass reads is decided there too.
#define GS_RS_TILE 4096u
#define GS_RS_PASSES 9u
struct GsRsCtl {
  uint32_t skip[GS_RS_PASSES];
  uint32_t src[GS_RS_PASSES];  // buffer (0 = the caller's, 1 = the backend's) pass p reads
  uint32_t fin;                // buffer holding the result
};
struct GsRsBufs {
  uint64_t* key[2];
  uint32_t* val[2];
};

__device__ __forceinline__ uint32_t gs_rs_digit(uint64_t k, uint32_t v, uint32_t p, uint32_t n_dcs) {
  return p < 8u ? (uint32_t)(k >> (8u * p)) & 255u : gs_dc_digit(v, n_dcs);
}

__global__ void __launch_bounds__(GS_BLOCK)
    gs_rs_hist_kernel(const uint64_t* key, const uint32_t* val, uint32_t n, uint32_t n_dcs, uint32_t np, uint32_t* ghist) {
  __shared__ uint32_t s[GS_RS_PASSES * 256];
  for (uint32_t x = threadIdx.x; x < np * 256u; x += GS_BLOCK) s[x] = 0u;
  __syncthreads();
  for (size_t x = (size_t)blockIdx.x * GS_BLOCK + threadIdx.x; x < n; x += (size_t)gridDim.x * GS_BLOCK) {
    const uint64_t k = key[x];
    const uint32_t v = np > 8u ? val[x] : 0u;
    for (uint32_t p = 0; p < np; ++p) atomicAdd(&s[p * 256u + gs_rs_digit(k, v, p, n_dcs)], 1u);
  }
  __syncthreads();
  for (uint32_t x = threadIdx.x; x < np * 256u; x += GS_BLOCK)
    if (s[x]) atomicAdd(&ghist[x], s[x]);
}

__global__ void gs_rs_plan_kernel(const uint32_t* ghist, uint32_t n, uint32_t np, GsRsCtl* c) {
  uint32_t src = 0u;
  for (uint32_t p = 0; p < np; ++p) {
    uint32_t top = 0u;
    for (uint32_t dg = 0; dg < 256u; ++dg) top = ghist[p * 256u + dg] > top ? ghist[p * 256u + dg] : top;
    c->skip[p] = top == n ? 1u : 0u;
    c->src[p] = src;
    if (top != n) src ^= 1u;
  }
  c->fin = src;
}

__global__ void __launch_bounds__(GS_BLOCK)
    gs_rs_upsweep_kernel(GsRsBufs b, const GsRsCtl* c, uint32_t p, uint32_t n, uint32_t n_dcs, uint32_t* hist) {
  if (c->skip[p]) return;
  __shared__ uint32_t s[256];
  s[threadIdx.x] = 0u;
  __syncthreads();
  const uint64_t* key = b.key[c->src[p]];
  const uint32_t* val = b.val[c->src[p]];
  const size_t t0 = (size_t)blockIdx.x * GS_RS_TILE, t1 = t0 + GS_RS_TILE < n ? t0 + GS_RS_TILE : n;
  for (size_t x = t0 + threadIdx.x; x < t1; x += GS_BLOCK)
    atomicAdd(&s[gs_rs_digit(key[x], p == 8u ? val[x] : 0u, p, n_dcs)], 1u);
  __syncthreads();
  hist[(size_t)threadIdx.x * gridDim.x + blockIdx.x] = s[threadIdx.x];
}

// Exclusive scan of GS_BLOCK values across the CTA; *total = their sum.
__device__ __forceinline__ uint32_t gs_block_scan(uint32_t v, uint32_t* sw, uint32_t* total) {
  const uint32_t lane = threadIdx.x & 31u, w = threadIdx.x >> 5;
  uint32_t incl = v;
  for (uint32_t o = 1; o < 32u; o <<= 1) {
    const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, incl, o);
    if (lane >= o) incl += y;
  }
  if (lane == 31u) sw[w] = incl;
  __syncthreads();
  if (w == 0) {
    uint32_t t = lane < GS_WARPS ? sw[lane] : 0u, ti = t;
    for (uint32_t o = 1; o < 32u; o <<= 1) {
      const uint32_t y = __shfl_up_sync(0xFFFFFFFFu, ti, o);
      if (lane >= o) ti += y;
    }
    if (lane < GS_WARPS) sw[lane] = ti - t;
    if (lane == GS_WARPS - 1u) sw[GS_WARPS] = ti;
  }
  __syncthreads();
  const uint32_t r = sw[w] + incl - v;
  *total = sw[GS_WARPS];
  __syncthreads();
  return r;
}

// CTA dg scans digit dg's counts over the nb tiles in place.
__global__ void __launch_bounds__(GS_BLOCK) gs_rs_scan_kernel(const GsRsCtl* c, uint32_t p, uint32_t nb, uint32_t* hist) {
  if (c->skip[p]) return;
  __shared__ uint32_t sw[GS_WARPS + 1];
  uint32_t* row = hist + (size_t)blockIdx.x * nb;
  uint32_t carry = 0u;
  for (uint32_t x0 = 0; x0 < nb; x0 += GS_BLOCK) {
    const uint32_t x = x0 + threadIdx.x;
    const uint32_t v = x < nb ? row[x] : 0u;
    uint32_t total;
    const uint32_t e = gs_block_scan(v, sw, &total);
    if (x < nb) row[x] = carry + e;
    carry += total;
  }
}

__global__ void __launch_bounds__(GS_BLOCK)
    gs_rs_scatter_kernel(GsRsBufs b, const GsRsCtl* c, uint32_t p, uint32_t n, uint32_t n_dcs, const uint32_t* hist,
                         const uint32_t* ghist) {
  if (c->skip[p]) return;
  __shared__ uint32_t base[256];
  __shared__ uint32_t wcnt[GS_WARPS][256];
  __shared__ uint32_t woff[GS_WARPS][256];
  __shared__ uint32_t sw[GS_WARPS + 1];
  const uint32_t tid = threadIdx.x, lane = tid & 31u, w = tid >> 5;
  // where this tile's pairs of digit tid start: pairs of smaller digits, then earlier tiles' of this digit
  uint32_t total;
  const uint32_t before = gs_block_scan(ghist[p * 256u + tid], sw, &total);
  base[tid] = before + hist[(size_t)tid * gridDim.x + blockIdx.x];
  for (uint32_t q = 0; q < GS_WARPS; ++q) wcnt[q][tid] = 0u;
  __syncthreads();
  const uint32_t s = c->src[p];
  const uint64_t* ks = b.key[s];
  const uint32_t* vs = b.val[s];
  uint64_t* kd = b.key[s ^ 1u];
  uint32_t* vd = b.val[s ^ 1u];
  const size_t t0 = (size_t)blockIdx.x * GS_RS_TILE, t1 = t0 + GS_RS_TILE < n ? t0 + GS_RS_TILE : n;
  const uint32_t lt = (1u << lane) - 1u;
  for (size_t r0 = t0; r0 < t1; r0 += GS_BLOCK) {
    const size_t x = r0 + tid;
    const bool valid = x < t1;
    uint64_t k = 0;
    uint32_t v = 0, dg = 256u;  // (an out-of-range pair matches only its own kind)
    if (valid) {
      k = ks[x];
      v = vs[x];
      dg = gs_rs_digit(k, v, p, n_dcs);
    }
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, dg);
    const uint32_t rank = __popc(peers & lt);
    if (valid && rank == 0u) wcnt[w][dg] = __popc(peers);
    __syncthreads();
    {  // thread tid: digit tid's offsets per warp, in warp order
      uint32_t acc = base[tid];
      for (uint32_t q = 0; q < GS_WARPS; ++q) {
        const uint32_t cq = wcnt[q][tid];
        woff[q][tid] = acc;
        acc += cq;
        wcnt[q][tid] = 0u;
      }
      base[tid] = acc;
    }
    __syncthreads();
    if (valid) {
      const uint32_t pos = woff[w][dg] + rank;
      kd[pos] = k;
      vd[pos] = v;
    }
  }
}

// The result back into the caller's buffers when the last pass wrote the backend's.
__global__ void __launch_bounds__(GS_BLOCK) gs_rs_copyback_kernel(GsRsBufs b, const GsRsCtl* c, uint32_t n) {
  if (c->fin == 0u) return;
  for (size_t x = (size_t)blockIdx.x * GS_BLOCK + threadIdx.x; x < n; x += (size_t)gridDim.x * GS_BLOCK) {
    b.key[0][x] = b.key[1][x];
    b.val[0][x] = b.val[1][x];
  }
}

class CudaBackend : public GsBackend {
 public:
  explicit CudaBackend(int dev) : dev_(dev) {
    err_[0] = 0;
    cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking);
    cudaEventCreate(&ev0_);
    cudaEventCreate(&ev1_);
    int sms = 132, occ = 4;
    cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    sms_ = (uint32_t)sms;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gs_tick_kernel<false>, GS_BLOCK, 0) != cudaSuccess || occ < 1)
      occ = 4;
    full_grid_ = (uint32_t)(sms * occ);
    int wocc = GS_WIN_BLOCKS;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&wocc, gs_window_kernel<false, false>, GS_BLOCK, 0) != cudaSuccess || wocc < 1)
      wocc = GS_WIN_BLOCKS;
    win_grid_ = (uint32_t)(sms * wocc);
    // GSIM_GRID_MAX=<CTAs>: fewer CTAs for the tick and window kernels (their partitions depend on gridDim
    // only), so that a pool small enough for the oracle to follow runs several rounds and batches per warp
    if (const char* e = getenv("GSIM_GRID_MAX")) {
      const long cap = atol(e);
      if (cap > 0 && (unsigned long)cap < full_grid_) full_grid_ = (uint32_t)cap;
      if (cap > 0 && (unsigned long)cap < win_grid_) win_grid_ = (uint32_t)cap;
    }
    scratch_ = nullptr;
    cudaMalloc(&scratch_, 4096);
  }
  ~CudaBackend() override {
    cudaSetDevice(dev_);
    for (auto& kv : graphs_) cudaGraphExecDestroy(kv.second);
    for (auto& kv : wgraphs_) cudaGraphExecDestroy(kv.second);
    for (auto& kv : sgraphs_) cudaGraphExecDestroy(kv.second);
    if (sharded_) vmm_.destroy();
    if (scratch_) cudaFree(scratch_);
    if (rs_mem_) cudaFree(rs_mem_);
    cudaEventDestroy(ev0_);
    cudaEventDestroy(ev1_);
    cudaStreamDestroy(stream_);
  }
  const char* name() const override { return "cuda-sm_90a"; }
  void* alloc(size_t bytes) override {
    cudaSetDevice(dev_);
    void* p = nullptr;
    if (!ok(cudaMalloc(&p, bytes ? bytes : 4), "cudaMalloc")) return nullptr;
    return p;
  }
  void release(void* p) override {
    cudaSetDevice(dev_);
    if (p && !sharded_) cudaFree(p);
  }
  bool h2d(void* dst, const void* src, size_t bytes) override {
    cudaSetDevice(dev_);
    return ok(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream_), "h2d") &&
           ok(cudaStreamSynchronize(stream_), "h2d sync");
  }
  bool d2h(void* dst, const void* src, size_t bytes) override {
    cudaSetDevice(dev_);
    return ok(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, stream_), "d2h") &&
           ok(cudaStreamSynchronize(stream_), "d2h sync");
  }
  void* host_alloc(size_t bytes) override {
    void* q = nullptr;
    cudaSetDevice(dev_);
    return cudaHostAlloc(&q, bytes, cudaHostAllocDefault) == cudaSuccess ? q : nullptr;
  }
  void host_free(void* q) override { cudaFreeHost(q); }
  bool h2d_word(void* dst, const void* src, size_t bytes) override {
    if (bytes > 16384) return h2d(dst, src, bytes);
    cudaSetDevice(dev_);
    return ok(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream_), "h2d");
  }
  bool write_batch(const GsWriteBatch& b) override {
    if (!b.n) return true;
    cudaSetDevice(dev_);
    gs_write_batch_kernel<<<1, 1, 0, stream_>>>(b);
    ++launches_;
    return ok(cudaGetLastError(), "write batch launch");
  }
  bool h2d_async(void* dst, const void* src, size_t bytes) override {
    cudaSetDevice(dev_);
    return ok(cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, stream_), "h2d");
  }
  bool row_read(const GsDev& d, uint32_t i, uint32_t out[8]) override { return rows_read(d, &i, 1u, out); }
  bool rows_read(const GsDev& d, const uint32_t* ids, uint32_t n, uint32_t* out) override {
    cudaSetDevice(dev_);
    uint32_t* w = reinterpret_cast<uint32_t*>(scratch_) + 256;  // (the first KB of scratch belongs to the counters)
    for (uint32_t x0 = 0; x0 < n; x0 += GS_ROWS_MAX) {
      GsRowIds r;
      r.n = n - x0 < GS_ROWS_MAX ? n - x0 : GS_ROWS_MAX;
      memcpy(r.id, ids + x0, r.n * 4);
      gs_rows_read_kernel<<<1, GS_ROWS_MAX * 8, 0, stream_>>>(d, r, w);
      ++launches_;
      if (!ok(cudaGetLastError(), "rows read launch") || !d2h(out + (size_t)x0 * 8, w, (size_t)r.n * 32)) return false;
    }
    return true;
  }
  bool fill32(uint32_t* dst, uint32_t value, size_t count) override {
    cudaSetDevice(dev_);
    if ((value & 0xFFu) == ((value >> 8) & 0xFFu) && (value & 0xFFFFu) == (value >> 16))
      return ok(cudaMemsetAsync(dst, (int)(value & 0xFFu), count * 4, stream_), "memset");
    return ok(cudaMemsetD32Async_(dst, value, count), "memset32");
  }
  bool fill8(uint8_t* dst, uint8_t value, size_t count) override {
    cudaSetDevice(dev_);
    return ok(cudaMemsetAsync(dst, value, count, stream_), "memset8");
  }
  bool init_rows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals&, uint32_t first,
                 uint32_t count, uint32_t now) override {
    if (!count) return true;
    cudaSetDevice(dev_);
    gs_init_kernel<<<(count + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(d, g_dev, first,
                                                                                count, now);
    ++launches_;
    return ok(cudaGetLastError(), "init launch");
  }
  bool run_ticks(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t t0,
                 uint32_t nticks, bool use_graph, double* kernel_ms, uint64_t* launches,
                 const GsXbar* xbar) override {
    uint32_t last_active = 0;
    return run_ticks_read(d, g_dev, g, t0, nticks, use_graph, kernel_ms, launches, xbar, &last_active);
  }
  bool run_ticks_read(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t t0, uint32_t nticks,
                      bool use_graph, double* kernel_ms, uint64_t* launches, const GsXbar* xbar,
                      uint32_t* last_active) override {
    (void)t0;
    if (!nticks || !g.n) {
      if (nticks) {  // no members: just advance time
        gs_advance_kernel<<<1, 1, 0, stream_>>>(d.tick_base, nticks, nullptr);
        ++launches_;
        return ok(cudaGetLastError(), "advance") && d2h(last_active, d.qstate[g.rank] + GS_Q_LAST_ACTIVE, 4);
      }
      return d2h(last_active, d.qstate[g.rank] + GS_Q_LAST_ACTIVE, 4);
    }
    cudaSetDevice(dev_);
    l2_window(d, g);
    const uint32_t blocks = tick_blocks(g);
    if (!ok(cudaEventRecord(ev0_, stream_), "event")) return false;
    uint32_t left = nticks;
    if (use_graph && (!xbar || !no_shard_graph_) && left >= GS_GRAPH_TICKS) {
      cudaGraphExec_t ge = graph_for(d, g_dev, blocks, xbar);
      if (!ge) return false;
      while (left >= GS_GRAPH_TICKS) {
        if (!ok(cudaGraphLaunch(ge, stream_), "graph launch")) return false;
        left -= GS_GRAPH_TICKS;
        launches_ += GS_GRAPH_TICKS + 1;
      }
    }
    if (left) {
      for (uint32_t k = 0; k < left; ++k) {
        if (!ok(gs_launch_tick(blocks, stream_, d, g_dev, k, pdl_ && !xbar), "tick launch")) return false;
      }
      gs_advance_kernel<<<1, 1, 0, stream_>>>(d.tick_base, left, nullptr);
      launches_ += left + 1;
      if (!ok(cudaGetLastError(), "tick launch")) return false;
    }
    if (!ok(cudaEventRecord(ev1_, stream_), "event")) return false;
    // the word a kernel raises when one of its internal invariants breaks (a bulk copy that never
    // completed): read back with the synchronisation that happens anyway, so that it fails loudly;
    // the same 16 bytes carry the last active tick the host's quiet detection needs
    uint32_t qs[GS_Q_WORDS] = {0, 0, 0, 0};
    if (!ok(cudaMemcpyAsync(qs, d.qstate[g.rank], sizeof(qs), cudaMemcpyDeviceToHost, stream_), "tick d2h"))
      return false;
    if (!ok(cudaStreamSynchronize(stream_), "tick sync")) return false;
    const uint32_t violation = qs[GS_Q_VIOLATION];
    *last_active = qs[GS_Q_LAST_ACTIVE];
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev0_, ev1_);
    if (kernel_ms) *kernel_ms += ms;
    if (launches) *launches += nticks;
    if (violation != 0u) {
      snprintf(err_, sizeof(err_), "tick %u: a bulk copy of the mailbox scan did not complete (kernel invariant broken)", violation - 1u);
      return false;
    }
    return true;
  }
  // A tick stretch is one CUDA graph: a WHILE loop whose body is GS_STRETCH_TICKS tick launches chained with
  // PDL plus gs_stretch_pass_kernel, which moves the clock by the ticks that ran and ends the loop at the
  // stop; then, when the stretch stopped quiet, the quiet probe (an IF node).  The control block is set by
  // one launch in front of the graph and read back in one copy behind it.
  bool run_tick_stretch(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t t0, uint32_t nticks,
                        uint32_t floor, bool counts, double* kernel_ms, GsStretch* out) override {
    if (!g.n) return GsBackend::run_tick_stretch(d, g_dev, g, t0, nticks, floor, counts, kernel_ms, out);
    cudaSetDevice(dev_);
    l2_window(d, g);
    cudaGraphExec_t ge = stretch_graph_for(d, g_dev, g, tick_blocks(g), counts);
    if (!ge) return false;
    GsStretchCtl* c = stretch_ctl();
    if (!ok(cudaEventRecord(ev0_, stream_), "event")) return false;
    gs_stretch_begin_kernel<<<1, 1, 0, stream_>>>(c, t0 + nticks, floor, g.ring_mask + 1u);
    if (!ok(cudaGetLastError(), "stretch begin") || !ok(cudaGraphLaunch(ge, stream_), "stretch graph launch")) return false;
    // (the graph records ev1_ when its loop is done: the quiet probe is not tick time)
    uint8_t back[sizeof(GsStretch) + 4];
    if (!ok(cudaMemcpyAsync(back, c, sizeof(back), cudaMemcpyDeviceToHost, stream_), "stretch d2h") ||
        !ok(cudaStreamSynchronize(stream_), "stretch sync"))
      return false;
    memcpy(out, back, sizeof(GsStretch));
    uint32_t violation;
    memcpy(&violation, back + sizeof(GsStretch), 4);
    const uint32_t passes = out->launches / GS_STRETCH_TICKS;
    launches_ += 1u + out->launches + passes + 1u + (out->quiet ? (counts ? 3u : 2u) : 0u);
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev0_, ev1_);
    if (kernel_ms) *kernel_ms += ms;
    if (violation != 0u) {
      snprintf(err_, sizeof(err_), "tick %u: a bulk copy of the mailbox scan did not complete (kernel invariant broken)", violation - 1u);
      return false;
    }
    return true;
  }
  // Quiet windows (gs_window_kernel): `nticks` ticks as a chain of launches of up to ProbeInterval
  // ticks each.  The chain stops by itself at the horizon; *ticks_done says how far it got.
  bool run_windows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t t0, uint32_t nticks,
                   uint32_t per_launch, bool use_graph, double* kernel_ms, uint64_t* launches, uint32_t* ticks_done,
                   const GsXbar* xbar, bool pristine) override {
    cudaSetDevice(dev_);
    *ticks_done = 0;
    if (!nticks || !g.n) return true;
    uint32_t* qs = d.qstate[g.rank];
    uint32_t init[2] = {t0, 0u};  // WIN_END = t0, VIOLATION = 0
    if (!ok(cudaMemcpyAsync(qs + GS_Q_WIN_END, init, 8, cudaMemcpyHostToDevice, stream_), "window init")) return false;
    uint32_t tiles = (g.n + GS_TILE - 1) / GS_TILE;
    if (g.world > 1 && tiles > g.rows_per_rank / GS_TILE) tiles = g.rows_per_rank / GS_TILE;
    uint32_t blocks = (tiles * 4u + GS_WARPS - 1) / GS_WARPS;  // a warp per group of 32 members, up to a full machine
    if (blocks > win_grid_) blocks = win_grid_;
    const uint32_t K = per_launch < g.P ? g.P : per_launch;
    const bool sharded = xbar != nullptr;
    const bool pdl = pdl_ && !sharded;
    if (!ok(cudaEventRecord(ev0_, stream_), "event")) return false;
    uint32_t left = nticks, n_launch = 0;
    if (use_graph && K == g.P && (!sharded || !no_shard_graph_)) {
      while (left >= GS_WIN_GRAPH * K) {
        cudaGraphExec_t ge = window_graph_for(d, g_dev, blocks, K, pdl, g.rank);
        if (!ge) return false;
        if (!ok(cudaGraphLaunch(ge, stream_), "window graph launch")) return false;
        left -= GS_WIN_GRAPH * K;
        n_launch += GS_WIN_GRAPH;
        launches_ += GS_WIN_GRAPH + 1;
      }
    }
    if (left) {
      uint32_t k = 0;
      while (left) {
        const uint32_t c = left < K ? left : K;
        if (!ok(gs_launch_window(blocks, stream_, d, g_dev, k, c, pdl, (pristine ? 1u : 0u) | win_mode_), "window launch"))
          return false;
        k += c;
        left -= c;
        ++n_launch;
        ++launches_;
      }
      gs_window_advance_kernel<<<1, 1, 0, stream_>>>(d.tick_base, qs);
      ++launches_;
      if (!ok(cudaGetLastError(), "window launch")) return false;
    }
    if (!ok(cudaEventRecord(ev1_, stream_), "event")) return false;
    uint32_t back[2] = {0, 0};
    if (!ok(cudaMemcpyAsync(back, qs + GS_Q_WIN_END, 8, cudaMemcpyDeviceToHost, stream_), "window d2h")) return false;
    if (!ok(cudaStreamSynchronize(stream_), "window sync")) return false;
    float ms = 0.f;
    cudaEventElapsedTime(&ms, ev0_, ev1_);
    if (kernel_ms) *kernel_ms += ms;
    if (launches) *launches += n_launch;
    if (back[1] != 0u) {
      snprintf(err_, sizeof(err_), "quiet window starting at tick %u met mail or posted some (scheduling invariant broken)", back[1] - 1u);
      return false;
    }
    if (back[0] < t0 || back[0] > t0 + nticks) {
      snprintf(err_, sizeof(err_), "window chain ended at tick %u outside [%u, %u]", back[0], t0, t0 + nticks);
      return false;
    }
    *ticks_done = back[0] - t0;
    return true;
  }
  bool quiet_scan(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now, uint32_t first,
                  uint32_t count) override {
    cudaSetDevice(dev_);
    if (!count) return true;
    uint32_t blocks = (count + GS_BLOCK - 1) / GS_BLOCK;
    if (blocks > sms_ * 8u) blocks = sms_ * 8u;
    gs_quiet_scan_kernel<<<blocks, GS_BLOCK, 0, stream_>>>(d, g_dev, now, nullptr, first, count);
    ++launches_;
    (void)g;
    return ok(cudaGetLastError(), "quiet scan launch") && ok(cudaStreamSynchronize(stream_), "quiet scan");
  }
  bool quiet_probe(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now, uint32_t* horizon,
                   GsRecount* counts) override {
    cudaSetDevice(dev_);
    // scratch: [0, sizeof(GsRecount)) the counts, then the horizon word
    GsRecount* dr = reinterpret_cast<GsRecount*>(scratch_);
    uint32_t* dh = reinterpret_cast<uint32_t*>(dr + 1);
    uint32_t* qh = d.qstate[0] + GS_Q_HORIZON;
    if (!ok(cudaMemsetAsync(qh, 0xFF, 4, stream_), "memset")) return false;  // GS_NEVER
    if (g.n) {
      uint32_t blocks = (g.n + GS_BLOCK - 1) / GS_BLOCK;
      if (blocks > sms_ * 8u) blocks = sms_ * 8u;
      gs_quiet_scan_kernel<<<blocks, GS_BLOCK, 0, stream_>>>(d, g_dev, now, nullptr, 0u, g.n);
      ++launches_;
    }
    gs_copy_word_kernel<<<1, 1, 0, stream_>>>(dh, qh);
    ++launches_;
    if (counts) {
      if (!ok(cudaMemsetAsync(dr, 0, sizeof(GsRecount), stream_), "memset")) return false;
      if (g.n) {
        gs_recount_kernel<<<(g.n + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(d, g_dev, now, nullptr, 0u, g.n, dr);
        ++launches_;
      }
    }
    if (!ok(cudaGetLastError(), "quiet probe launch")) return false;
    uint8_t back[sizeof(GsRecount) + 4];
    const size_t off = counts ? 0 : sizeof(GsRecount);
    if (!d2h(back + off, reinterpret_cast<uint8_t*>(scratch_) + off, sizeof(back) - off)) return false;
    if (counts) memcpy(counts, back, sizeof(GsRecount));
    memcpy(horizon, back + sizeof(GsRecount), 4);
    return true;
  }
  bool crash_fraction(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t thr,
                      uint32_t salt, uint32_t, uint32_t* n_crashed) override {
    cudaSetDevice(dev_);
    uint32_t* cnt = reinterpret_cast<uint32_t*>(scratch_);
    if (!ok(cudaMemsetAsync(cnt, 0, 4, stream_), "memset")) return false;
    if (g.n) {
      gs_crash_kernel<<<(g.n + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(d, g_dev, thr,
                                                                                 salt, cnt);
      ++launches_;
    }
    return ok(cudaGetLastError(), "crash launch") && d2h(n_crashed, cnt, 4);
  }
  bool impair_dir_fraction(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, const GsImpairCols& c,
                           uint32_t thr, uint32_t salt, const GsImpairVal& v, uint32_t counts[2]) override {
    cudaSetDevice(dev_);
    uint32_t* cnt = reinterpret_cast<uint32_t*>(scratch_);
    if (!ok(cudaMemsetAsync(cnt, 0, 8, stream_), "memset")) return false;
    if (g.n) {
      gs_impair_kernel<<<(g.n + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(d, g_dev, c, thr, salt, v, cnt);
      ++launches_;
    }
    return ok(cudaGetLastError(), "impair launch") && d2h(counts, cnt, 8);
  }
  bool flap_fraction(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t* col, uint32_t thr,
                     uint32_t salt, uint32_t w, uint32_t counts[2]) override {
    cudaSetDevice(dev_);
    uint32_t* cnt = reinterpret_cast<uint32_t*>(scratch_);
    if (!ok(cudaMemsetAsync(cnt, 0, 8, stream_), "memset")) return false;
    if (g.n) {
      gs_flap_kernel<<<(g.n + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(d, g_dev, col, thr, salt, w, cnt);
      ++launches_;
    }
    return ok(cudaGetLastError(), "flap launch") && d2h(counts, cnt, 8);
  }
  bool flap_stats(const GsGlobals& g, const uint32_t* col, uint32_t now, uint64_t out[2]) override {
    cudaSetDevice(dev_);
    unsigned long long* h = reinterpret_cast<unsigned long long*>(scratch_);
    if (!ok(cudaMemsetAsync(h, 0, 16, stream_), "memset")) return false;
    if (g.n) {
      const uint32_t blocks = (g.n + GS_BLOCK - 1) / GS_BLOCK < sms_ * 8u ? (g.n + GS_BLOCK - 1) / GS_BLOCK : sms_ * 8u;
      gs_flap_stats_kernel<<<blocks, GS_BLOCK, 0, stream_>>>(col, g.n, g.seed_lo, g.seed_hi, now, h);
      ++launches_;
    }
    return ok(cudaGetLastError(), "flap stats launch") && d2h(out, h, 16);
  }
  bool pause_rows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t* pause_until,
                  const uint32_t* ids, uint32_t n, uint32_t thr, uint32_t salt, uint32_t until,
                  uint32_t* n_paused) override {
    cudaSetDevice(dev_);
    uint32_t* cnt = reinterpret_cast<uint32_t*>(scratch_);
    if (!ok(cudaMemsetAsync(cnt, 0, 4, stream_), "memset")) return false;
    const uint32_t rows = ids ? n : g.n;
    uint32_t* dids = nullptr;
    if (ids && n) {  // the id list travels with the launch (pageable source: copied before the call returns)
      if (!ok(cudaMallocAsync(reinterpret_cast<void**>(&dids), (size_t)n * 4, stream_), "malloc")) return false;
      if (!ok(cudaMemcpyAsync(dids, ids, (size_t)n * 4, cudaMemcpyHostToDevice, stream_), "h2d")) {
        cudaFreeAsync(dids, stream_);
        return false;
      }
    }
    if (rows) {
      gs_pause_kernel<<<(rows + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(d, g_dev, pause_until, dids, n, thr,
                                                                                 salt, until, cnt);
      ++launches_;
    }
    const bool launched = ok(cudaGetLastError(), "pause launch");
    if (dids) cudaFreeAsync(dids, stream_);
    return launched && d2h(n_paused, cnt, 4);
  }
  bool domain_range(uint32_t* dom, uint32_t first, uint32_t count, uint32_t per_domain, uint32_t first_domain) override {
    cudaSetDevice(dev_);
    if (!count) return true;
    gs_domain_range_kernel<<<(count + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(dom, first, count, per_domain,
                                                                                       first_domain);
    ++launches_;
    return ok(cudaGetLastError(), "domain range launch");
  }
  bool domain_rows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, const uint32_t* dom, const uint32_t* bits,
                   uint32_t n_words, const GsDomainOp& a, uint32_t counts[2]) override {
    cudaSetDevice(dev_);
    uint32_t* cnt = reinterpret_cast<uint32_t*>(scratch_);
    if (!ok(cudaMemsetAsync(cnt, 0, 8, stream_), "memset")) return false;
    uint32_t* dbits = nullptr;
    if (g.n && n_words) {  // the bitmap travels with the launch (pageable source: copied before the call returns)
      if (!ok(cudaMallocAsync(reinterpret_cast<void**>(&dbits), (size_t)n_words * 4, stream_), "malloc")) return false;
      if (!ok(cudaMemcpyAsync(dbits, bits, (size_t)n_words * 4, cudaMemcpyHostToDevice, stream_), "h2d")) {
        cudaFreeAsync(dbits, stream_);
        return false;
      }
      gs_domain_op_kernel<<<(g.n + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(d, g_dev, dom, dbits, n_words, a,
                                                                                     cnt);
      ++launches_;
    }
    const bool launched = ok(cudaGetLastError(), "domain launch");
    if (dbits) cudaFreeAsync(dbits, stream_);
    return launched && d2h(counts, cnt, 8);
  }
  bool domain_stats(const GsDev& d, const GsGlobals& g, const GsDomainCols& c, uint32_t now, uint32_t first_domain,
                    uint32_t count, GsDomainStats* out) override {
    cudaSetDevice(dev_);
    if (!count) return true;
    const size_t bytes = (size_t)count * sizeof(GsDomainStats);
    GsDomainStats* dout = nullptr;
    if (!ok(cudaMallocAsync(reinterpret_cast<void**>(&dout), bytes, stream_), "malloc")) return false;
    bool okk = ok(cudaMemsetAsync(dout, 0, bytes, stream_), "memset");
    if (okk && g.n) {
      const uint32_t blocks = (g.n + GS_BLOCK - 1) / GS_BLOCK < sms_ * 8u ? (g.n + GS_BLOCK - 1) / GS_BLOCK : sms_ * 8u;
      gs_domain_stats_kernel<<<blocks, GS_BLOCK, 0, stream_>>>(d, c, g.n, g.seed_lo, g.seed_hi, now, first_domain, count,
                                                               dout);
      ++launches_;
      okk = ok(cudaGetLastError(), "domain stats launch");
    }
    okk = okk && d2h(out, dout, bytes);
    cudaFreeAsync(dout, stream_);
    return okk;
  }
  bool resume_rows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t* pause_until, uint32_t t,
                   bool resume, bool log_events, uint32_t counts[4]) override {
    cudaSetDevice(dev_);
    uint32_t* cnt = reinterpret_cast<uint32_t*>(scratch_);
    if (!ok(cudaMemsetAsync(cnt, 0, 16, stream_), "memset")) return false;
    if (g.n) {
      gs_resume_kernel<<<(g.n + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(
          d, g_dev, pause_until, t, resume ? 1u : 0u, log_events ? 1u : 0u, cnt);
      ++launches_;
    }
    return ok(cudaGetLastError(), "resume launch") && d2h(counts, cnt, 16);
  }
  // ---- network-coordinate queries: enqueued only, the caller reads back -----------------------------
  bool coord_rows(const GsDev& d, const GsGlobals& g, uint32_t first, uint32_t count, double* rows) override {
    cudaSetDevice(dev_);
    if (!count) return true;
    gs_coord_rows_kernel<<<(count + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(d, g.cap, first, count, rows);
    ++launches_;
    return ok(cudaGetLastError(), "coordinate rows launch");
  }
  bool coord_pairs(const GsDev& d, const GsGlobals* g_dev, const GsGlobals&, uint32_t now, const uint32_t* a,
                   const uint32_t* b, uint32_t n, double* est, double* tru) override {
    cudaSetDevice(dev_);
    if (!n) return true;
    gs_coord_pairs_kernel<<<(n + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(d, g_dev, now, a, b, n, est, tru);
    ++launches_;
    return ok(cudaGetLastError(), "coordinate pairs launch");
  }
  bool coord_dist_from(const GsDev& d, const GsGlobals* g_dev, const GsGlobals&, uint32_t now, uint32_t from,
                       const uint32_t* ids, uint32_t n, bool router, uint64_t* key, uint32_t* val) override {
    cudaSetDevice(dev_);
    if (!n) return true;
    gs_coord_dist_kernel<<<(n + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(d, g_dev, now, from, ids, n,
                                                                                 router ? 1u : 0u, key, val);
    ++launches_;
    return ok(cudaGetLastError(), "coordinate distance launch");
  }
  bool sort_pairs(const GsGlobals& g, uint64_t* key, uint32_t* val, uint32_t n, uint32_t n_dcs) override {
    cudaSetDevice(dev_);
    if (n < 2u) return true;
    if (!rs_reserve(g.cap > n ? g.cap : n)) return false;
    const uint32_t np = n_dcs ? GS_RS_PASSES : 8u, nb = (n + GS_RS_TILE - 1u) / GS_RS_TILE;
    uint32_t hb = nb < sms_ * 4u ? nb : sms_ * 4u;
    if (!ok(cudaMemsetAsync(rs_ghist_, 0, GS_RS_PASSES * 256 * 4, stream_), "memset")) return false;
    gs_rs_hist_kernel<<<hb, GS_BLOCK, 0, stream_>>>(key, val, n, n_dcs, np, rs_ghist_);
    gs_rs_plan_kernel<<<1, 1, 0, stream_>>>(rs_ghist_, n, np, rs_ctl_);
    GsRsBufs b;
    b.key[0] = key;
    b.key[1] = rs_key_;
    b.val[0] = val;
    b.val[1] = rs_val_;
    for (uint32_t p = 0; p < np; ++p) {
      gs_rs_upsweep_kernel<<<nb, GS_BLOCK, 0, stream_>>>(b, rs_ctl_, p, n, n_dcs, rs_hist_);
      gs_rs_scan_kernel<<<256, GS_BLOCK, 0, stream_>>>(rs_ctl_, p, nb, rs_hist_);
      gs_rs_scatter_kernel<<<nb, GS_BLOCK, 0, stream_>>>(b, rs_ctl_, p, n, n_dcs, rs_hist_, rs_ghist_);
    }
    hb = (n + GS_BLOCK - 1) / GS_BLOCK < sms_ * 8u ? (n + GS_BLOCK - 1) / GS_BLOCK : sms_ * 8u;
    gs_rs_copyback_kernel<<<hb, GS_BLOCK, 0, stream_>>>(b, rs_ctl_, n);
    launches_ += 3u + 3u * np;
    return ok(cudaGetLastError(), "radix sort launch");
  }
  bool dc_medians(const GsGlobals&, const uint64_t* key, const uint32_t* val, uint32_t n, uint32_t n_dcs, double* med,
                  uint32_t* cnt) override {
    cudaSetDevice(dev_);
    gs_dc_medians_kernel<<<1, GS_MAX_DCS, 0, stream_>>>(key, val, n, n_dcs, med, cnt);
    ++launches_;
    return ok(cudaGetLastError(), "medians launch");
  }
  bool coord_error(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now, uint32_t n_draws,
                   uint32_t salt, uint64_t* key, uint32_t* val, double* part, double* out) override {
    cudaSetDevice(dev_);
    const uint32_t nch = (n_draws + GS_ERR_CHUNK - 1u) / GS_ERR_CHUNK;
    gs_coord_error_kernel<<<nch, GS_BLOCK, 0, stream_>>>(d, g_dev, now, n_draws, salt, key, val, part);
    ++launches_;
    if (!ok(cudaGetLastError(), "error sample launch") || !sort_pairs(g, key, val, n_draws, 0u)) return false;
    gs_coord_error_finish_kernel<<<1, 1, 0, stream_>>>(key, n_draws, part, out);
    ++launches_;
    return ok(cudaGetLastError(), "error finish launch");
  }
  bool reap_rows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now,
                 uint32_t reconnect_ticks, uint32_t tombstone_ticks, bool log_events,
                 uint32_t counts[2]) override {
    cudaSetDevice(dev_);
    uint32_t* cnt = reinterpret_cast<uint32_t*>(scratch_);
    if (!ok(cudaMemsetAsync(cnt, 0, 8, stream_), "memset")) return false;
    if (g.n) {
      gs_reap_kernel<<<(g.n + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(
          d, g_dev, now, reconnect_ticks, tombstone_ticks, log_events ? 1u : 0u, cnt);
      ++launches_;
    }
    return ok(cudaGetLastError(), "reap launch") && d2h(counts, cnt, 8);
  }
  bool recount(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now, uint32_t first, uint32_t count,
               GsRecount* out) override {
    cudaSetDevice(dev_);
    GsRecount* dr = reinterpret_cast<GsRecount*>(scratch_);
    if (!ok(cudaMemsetAsync(dr, 0, sizeof(GsRecount), stream_), "memset")) return false;
    if (first < g.n && count) {
      if (count > g.n - first) count = g.n - first;
      gs_recount_kernel<<<(count + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(d, g_dev, now, nullptr, first, count, dr);
      ++launches_;
    }
    return ok(cudaGetLastError(), "recount launch") && d2h(out, dr, sizeof(GsRecount));
  }
  // ---- per-agent observation: one submission, one wait -------------------------------------------------
  bool agent_stats(const GsDev& d, const GsGlobals& g, const uint32_t* key, const GsPendingAlive& pa, uint32_t first,
                   uint32_t count, GsAgentStats* out) override {
    cudaSetDevice(dev_);
    uint32_t* est = reinterpret_cast<uint32_t*>(scratch_);
    if (!ok(cudaMemsetAsync(est, 0, 16, stream_), "memset")) return false;
    if (!g.graph_n && g.n) {  // a CSR pool's list is the agent's row: no pool-wide counts
      const uint32_t blocks = (g.n + GS_BLOCK - 1) / GS_BLOCK < sms_ * 8u ? (g.n + GS_BLOCK - 1) / GS_BLOCK : sms_ * 8u;
      gs_agent_est_kernel<<<blocks, GS_BLOCK, 0, stream_>>>(key, g.n, est);
      ++launches_;
    }
    const size_t bytes = (size_t)count * sizeof(GsAgentStats);
    GsAgentStats* dout = nullptr;
    if (!ok(cudaGetLastError(), "agent counts launch") ||
        !ok(cudaMallocAsync(reinterpret_cast<void**>(&dout), bytes, stream_), "malloc"))
      return false;
    const GsAgentCols c = {key, d.meta, d.heard, d.queued, d.ltime_member, d.ltime_event,
                           g.graph_n ? d.row_ptr : nullptr, g.graph_n ? d.col_idx : nullptr};
    GsClassMasks cm;
    memcpy(cm.m, g.class_mask, sizeof(cm.m));
    gs_agent_stats_kernel<<<(count + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(c, cm, est, pa, first, count, dout);
    ++launches_;
    const bool okk = ok(cudaGetLastError(), "agent stats launch") &&
                     ok(cudaMemcpyAsync(out, dout, bytes, cudaMemcpyDeviceToHost, stream_), "d2h");
    cudaFreeAsync(dout, stream_);
    return ok(cudaStreamSynchronize(stream_), "agent stats sync") && okk;
  }
  bool health_histogram(const GsDev& d, const GsGlobals& g, const uint32_t* key, const GsImpairCols& imp,
                        uint64_t out[GS_HIST_BINS]) override {
    cudaSetDevice(dev_);
    unsigned long long* h = reinterpret_cast<unsigned long long*>(scratch_);
    if (!ok(cudaMemsetAsync(h, 0, GS_HIST_BINS * 8, stream_), "memset")) return false;
    if (g.n) {
      const uint32_t blocks = (g.n + GS_BLOCK - 1) / GS_BLOCK < sms_ * 8u ? (g.n + GS_BLOCK - 1) / GS_BLOCK : sms_ * 8u;
      gs_health_hist_kernel<<<blocks, GS_BLOCK, 0, stream_>>>(key, d.meta, imp, g.n, h);
      ++launches_;
    }
    return ok(cudaGetLastError(), "health histogram launch") && d2h(out, h, GS_HIST_BINS * 8);
  }
  bool state_hash(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now,
                  uint64_t out[4]) override {
    cudaSetDevice(dev_);
    unsigned long long* dh = reinterpret_cast<unsigned long long*>(scratch_);
    if (!ok(cudaMemsetAsync(dh, 0, 32, stream_), "memset")) return false;
    if (g.n) {
      gs_hash_kernel<<<(g.n + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(d, g_dev, now, dh);
      ++launches_;
    }
    return ok(cudaGetLastError(), "hash launch") && d2h(out, dh, 32);
  }
  // ---- sharded pools -----------------------------------------------------------------------
  bool shard_begin(uint32_t world, uint32_t rank) override {
    cudaSetDevice(dev_);
    cudaFree(0);  // make sure the primary context exists before driver-API calls
    sharded_ = vmm_.init(dev_, world, rank, err_, sizeof(err_));
    return sharded_;
  }
  size_t shard_granularity() override { return vmm_.granularity(); }
  void* shard_alloc(size_t slice_bytes, size_t planes) override {
    void* q = vmm_.reserve(slice_bytes, planes);
    if (!q) snprintf(err_, sizeof(err_), "%s", vmm_.last_error());
    return q;
  }
  bool shard_commit(const int** fds, size_t* n) override {
    if (!vmm_.commit()) {
      snprintf(err_, sizeof(err_), "%s", vmm_.last_error());
      return false;
    }
    *fds = vmm_.export_fds().data();
    *n = vmm_.export_fds().size();
    return true;
  }
  bool shard_attach(uint32_t peer, const int* fds, size_t n) override {
    cudaSetDevice(dev_);
    if (!vmm_.attach(peer, fds, n)) {
      snprintf(err_, sizeof(err_), "%s", vmm_.last_error());
      return false;
    }
    return true;
  }
  bool xbar_host(const GsXbar& xb) override {
    cudaSetDevice(dev_);
    gs_xbar_kernel<<<1, 32, 0, stream_>>>(xb);
    ++launches_;
    return ok(cudaGetLastError(), "xbar launch") && ok(cudaStreamSynchronize(stream_), "xbar");
  }
  bool and_columns(const GsDev& d, const GsGlobals& g, uint32_t keep, uint32_t first, uint32_t count) override {
    cudaSetDevice(dev_);
    if (first >= g.n || !count) return true;
    if (count > g.n - first) count = g.n - first;
    gs_and_kernel<<<(count + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(d, first, count, keep);
    ++launches_;
    return ok(cudaGetLastError(), "and launch");
  }
  bool sync() override {
    cudaSetDevice(dev_);
    return ok(cudaStreamSynchronize(stream_), "sync");
  }
  const char* last_error() const override { return err_; }
  uint64_t total_launches() const override { return launches_; }

 private:
  // performance variant: keep the status replica (1 byte per member, gathered at random by every
  // prober) resident in L2 — persisting hits for the window, streaming for everything else.
  // Set on the stream before any capture, so graph kernel nodes inherit it.
  void l2_window(const GsDev& d, const GsGlobals& g) {
    if (d.kst != nullptr && !l2_window_set_ && getenv("GSIM_NO_L2_WINDOW") == nullptr) {
      l2_window_set_ = true;
      cudaDeviceProp prop;
      if (cudaGetDeviceProperties(&prop, dev_) == cudaSuccess && prop.persistingL2CacheMaxSize > 0) {
        size_t bytes = g.cap;
        if (bytes > (size_t)prop.accessPolicyMaxWindowSize) bytes = (size_t)prop.accessPolicyMaxWindowSize;
        size_t carve = bytes < (size_t)prop.persistingL2CacheMaxSize ? bytes : (size_t)prop.persistingL2CacheMaxSize;
        cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, carve);
        cudaStreamAttrValue v;
        memset(&v, 0, sizeof(v));
        v.accessPolicyWindow.base_ptr = d.kst;
        v.accessPolicyWindow.num_bytes = bytes;
        v.accessPolicyWindow.hitRatio = bytes <= carve ? 1.0f : (float)carve / (float)bytes;
        v.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
        v.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
        cudaStreamSetAttribute(stream_, cudaStreamAttributeAccessPolicyWindow, &v);
        cudaGetLastError();  // best effort: an unsupported attribute must not fail the step
      }
    }
  }
  // persistent launch of the tick: one warp per 128-member tile up to a full machine (SMs x resident CTAs)
  uint32_t tick_blocks(const GsGlobals& g) const {
    uint32_t tiles = (g.n + GS_TILE - 1) / GS_TILE;
    if (g.world > 1 && tiles > g.rows_per_rank / GS_TILE) tiles = g.rows_per_rank / GS_TILE;
    uint32_t blocks = (tiles + GS_WARPS - 1) / GS_WARPS;
    return blocks < full_grid_ ? blocks : full_grid_;
  }
  cudaError_t cudaMemsetD32Async_(uint32_t* dst, uint32_t value, size_t count) {
    // the runtime API has no 32-bit memset: a grid-stride fill kernel on the pool's stream
    if (!count) return cudaSuccess;
    size_t blocks = (count + GS_BLOCK - 1) / GS_BLOCK;
    if (blocks > sms_ * 16u) blocks = sms_ * 16u;
    gs_fill32_kernel<<<(unsigned)blocks, GS_BLOCK, 0, stream_>>>(dst, value, count);
    ++launches_;
    return cudaGetLastError();
  }
  // the column pointers are baked into the captured launches: if they changed (a peer graph was
  // attached or removed), every cached graph is stale
  void drop_stale_graphs(const GsDev& d) {
    if (have_graph_dev_ && memcmp(&graph_dev_, &d, sizeof(GsDev)) != 0) {
      for (auto& kv : graphs_) cudaGraphExecDestroy(kv.second);
      graphs_.clear();
      for (auto& kv : wgraphs_) cudaGraphExecDestroy(kv.second);
      wgraphs_.clear();
      for (auto& kv : sgraphs_) cudaGraphExecDestroy(kv.second);
      sgraphs_.clear();
    }
    graph_dev_ = d;
    have_graph_dev_ = true;
  }
  cudaGraphExec_t graph_for(const GsDev& d, const GsGlobals* g_dev, uint32_t blocks, const GsXbar* xbar) {
    drop_stale_graphs(d);
    auto it = graphs_.find(blocks);
    if (it != graphs_.end()) return it->second;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t ge = nullptr;
    if (!ok(cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal), "capture"))
      return nullptr;
    for (uint32_t k = 0; k < GS_GRAPH_TICKS; ++k)
      if (!ok(gs_launch_tick(blocks, stream_, d, g_dev, k, pdl_ && !xbar), "tick capture")) {
        cudaGraph_t dead = nullptr;
        cudaStreamEndCapture(stream_, &dead);
        if (dead) cudaGraphDestroy(dead);
        return nullptr;
      }

    gs_advance_kernel<<<1, 1, 0, stream_>>>(d.tick_base, GS_GRAPH_TICKS, nullptr);
    if (!ok(cudaStreamEndCapture(stream_, &graph), "end capture")) return nullptr;
    if (!ok(cudaGraphInstantiate(&ge, graph, 0), "instantiate")) {
      cudaGraphDestroy(graph);
      return nullptr;
    }
    cudaGraphDestroy(graph);
    graphs_[blocks] = ge;
    return ge;
  }
  GsStretchCtl* stretch_ctl() { return reinterpret_cast<GsStretchCtl*>(reinterpret_cast<uint8_t*>(scratch_) + 3072); }
  // The graph of run_tick_stretch for this grid, with or without the counts in its quiet probe.
  cudaGraphExec_t stretch_graph_for(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t blocks, bool counts) {
    drop_stale_graphs(d);
    const uint64_t key = ((uint64_t)blocks << 1) | (counts ? 1u : 0u);
    auto it = sgraphs_.find(key);
    if (it != sgraphs_.end()) return it->second;
    GsStretchCtl* c = stretch_ctl();
    uint32_t* qs = d.qstate[0];
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t ge = nullptr;
    if (!ok(cudaGraphCreate(&graph, 0), "stretch graph")) return nullptr;
    cudaGraphConditionalHandle loop = 0, probe = 0;
    cudaGraphNode_t wn = nullptr, rn = nullptr, en = nullptr, pn = nullptr;
    cudaGraphNodeParams wp = {};
    wp.type = cudaGraphNodeTypeConditional;
    cudaGraphNodeParams pp = wp;
    bool good = ok(cudaGraphConditionalHandleCreate(&loop, graph, 1u, cudaGraphCondAssignDefault), "loop handle") &&
                ok(cudaGraphConditionalHandleCreate(&probe, graph, 0u, cudaGraphCondAssignDefault), "probe handle");
    if (good) {
      wp.conditional.handle = loop;
      wp.conditional.type = cudaGraphCondTypeWhile;
      wp.conditional.size = 1;
      good = ok(cudaGraphAddNode(&wn, graph, nullptr, 0, &wp), "while node");
    }
    // the loop's body: the tick launches of one pass, then the pass kernel
    if (good && ok(cudaStreamBeginCaptureToGraph(stream_, wp.conditional.phGraph_out[0], nullptr, nullptr, 0,
                                                 cudaStreamCaptureModeThreadLocal), "capture")) {
      for (uint32_t k = 0; k < GS_STRETCH_TICKS && good; ++k)
        good = ok(gs_launch_tick(blocks, stream_, d, g_dev, k, pdl_, c), "tick capture");
      if (good) {
        gs_stretch_pass_kernel<<<1, 1, 0, stream_>>>(d.tick_base, qs, c, GS_STRETCH_TICKS, loop);
        good = ok(cudaGetLastError(), "pass capture");
      }
      cudaGraph_t body = nullptr;
      good = ok(cudaStreamEndCapture(stream_, &body), "end capture") && good;
    } else {
      good = false;
    }
    if (good) good = ok(cudaGraphAddEventRecordNode(&rn, graph, &wn, 1, ev1_), "event node");
    if (good) {
      void* args[] = {&c, &qs, &probe};
      cudaKernelNodeParams kp = {};
      kp.func = reinterpret_cast<void*>(gs_stretch_end_kernel);
      kp.gridDim = dim3(1);
      kp.blockDim = dim3(1);
      kp.kernelParams = args;
      good = ok(cudaGraphAddKernelNode(&en, graph, &rn, 1, &kp), "end node");
    }
    if (good) {
      pp.conditional.handle = probe;
      pp.conditional.type = cudaGraphCondTypeIf;
      pp.conditional.size = 1;
      good = ok(cudaGraphAddNode(&pn, graph, &en, 1, &pp), "if node");
    }
    // the quiet probe at the tick the stretch stopped at (the device clock): scan, horizon, counts
    if (good && ok(cudaStreamBeginCaptureToGraph(stream_, pp.conditional.phGraph_out[0], nullptr, nullptr, 0,
                                                 cudaStreamCaptureModeThreadLocal), "capture")) {
      uint32_t sblocks = (g.cap + GS_BLOCK - 1) / GS_BLOCK;
      if (sblocks > sms_ * 8u) sblocks = sms_ * 8u;
      gs_quiet_scan_kernel<<<sblocks, GS_BLOCK, 0, stream_>>>(d, g_dev, 0u, d.tick_base, 0u, g.cap);
      gs_copy_word_kernel<<<1, 1, 0, stream_>>>(&c->out.horizon, qs + GS_Q_HORIZON);
      if (counts)
        gs_recount_kernel<<<(g.cap + GS_BLOCK - 1) / GS_BLOCK, GS_BLOCK, 0, stream_>>>(d, g_dev, 0u, d.tick_base, 0u, g.cap,
                                                                                      &c->out.counts);
      good = ok(cudaGetLastError(), "probe capture");
      cudaGraph_t body = nullptr;
      good = ok(cudaStreamEndCapture(stream_, &body), "end capture") && good;
    } else {
      good = false;
    }
    if (good) good = ok(cudaGraphInstantiate(&ge, graph, 0), "instantiate");
    cudaGraphDestroy(graph);
    if (!good) return nullptr;
    sgraphs_[key] = ge;
    return ge;
  }
  cudaGraphExec_t window_graph_for(const GsDev& d, const GsGlobals* g_dev, uint32_t blocks, uint32_t K, bool pdl, uint32_t rank) {
    drop_stale_graphs(d);
    const uint64_t key = ((uint64_t)blocks << 32) | K;
    auto it = wgraphs_.find(key);
    if (it != wgraphs_.end()) return it->second;
    cudaGraph_t graph = nullptr;
    cudaGraphExec_t ge = nullptr;
    if (!ok(cudaStreamBeginCapture(stream_, cudaStreamCaptureModeThreadLocal), "capture")) return nullptr;
    bool good = true;
    for (uint32_t j = 0; j < GS_WIN_GRAPH && good; ++j)
      good = ok(gs_launch_window(blocks, stream_, d, g_dev, j * K, K, pdl, win_mode_), "window capture");
    if (good) gs_window_advance_kernel<<<1, 1, 0, stream_>>>(d.tick_base, d.qstate[rank]);
    if (!ok(cudaStreamEndCapture(stream_, &graph), "end capture") || !good) {
      if (graph) cudaGraphDestroy(graph);
      return nullptr;
    }
    if (!ok(cudaGraphInstantiate(&ge, graph, 0), "instantiate")) {
      cudaGraphDestroy(graph);
      return nullptr;
    }
    cudaGraphDestroy(graph);
    wgraphs_[key] = ge;
    return ge;
  }
  // The radix sort's scratch, for up to `n` pairs (the pool's capacity): the second key and value buffers,
  // the per-tile digit counts, every pass's histogram and the plan.  Allocated by the first sort, kept until
  // the pool is destroyed.
  bool rs_reserve(size_t n) {
    if (n <= rs_n_) return true;
    if (rs_mem_) cudaFree(rs_mem_);
    rs_mem_ = nullptr;
    rs_n_ = 0;
    const size_t nb = (n + GS_RS_TILE - 1) / GS_RS_TILE;
    const size_t kb = n * 8, vb = (n * 4 + 255) / 256 * 256, hb = (256 * nb * 4 + 255) / 256 * 256;
    const size_t gb = GS_RS_PASSES * 256 * 4;
    if (!ok(cudaMalloc(&rs_mem_, kb + vb + hb + gb + sizeof(GsRsCtl)), "radix sort scratch")) {
      rs_mem_ = nullptr;
      return false;
    }
    uint8_t* q = reinterpret_cast<uint8_t*>(rs_mem_);
    rs_key_ = reinterpret_cast<uint64_t*>(q);
    rs_val_ = reinterpret_cast<uint32_t*>(q + kb);
    rs_hist_ = reinterpret_cast<uint32_t*>(q + kb + vb);
    rs_ghist_ = reinterpret_cast<uint32_t*>(q + kb + vb + hb);
    rs_ctl_ = reinterpret_cast<GsRsCtl*>(q + kb + vb + hb + gb);
    rs_n_ = n;
    return true;
  }
  bool ok(cudaError_t e, const char* what) {
    if (e == cudaSuccess) return true;
    snprintf(err_, sizeof(err_), "%s: %s", what, cudaGetErrorString(e));
    return false;
  }
  int dev_;
  cudaStream_t stream_;
  cudaEvent_t ev0_, ev1_;
  void* scratch_;
  void* rs_mem_ = nullptr;  // radix sort scratch (rs_reserve)
  size_t rs_n_ = 0;
  uint64_t* rs_key_ = nullptr;
  uint32_t* rs_val_ = nullptr;
  uint32_t* rs_hist_ = nullptr;
  uint32_t* rs_ghist_ = nullptr;
  GsRsCtl* rs_ctl_ = nullptr;
  uint32_t sms_ = 132;
  uint32_t full_grid_ = 528;
  uint32_t win_grid_ = 528;
  GsVmm vmm_;
  bool sharded_ = false;
  bool pdl_ = getenv("GSIM_NO_PDL") == nullptr;
  // sharded pools: stream launches by default (all ranks' graph launches drift and the barrier at the head
  // of every node serialises on the slowest rank); GSIM_SHARD_GRAPH=1 turns the graph path on
  bool no_shard_graph_ = getenv("GSIM_SHARD_GRAPH") == nullptr;
  // window kernel: how groups are dealt to the warps (bit 1 of the kernel's mode word); GSIM_WIN_CYCLIC=0/1
  uint32_t win_mode_ = getenv("GSIM_WIN_CYCLIC") && atoi(getenv("GSIM_WIN_CYCLIC")) ? 2u : 0u;
  std::map<uint32_t, cudaGraphExec_t> graphs_;
  std::map<uint64_t, cudaGraphExec_t> wgraphs_;
  std::map<uint64_t, cudaGraphExec_t> sgraphs_;  // tick stretches, by grid and whether the probe counts
  GsDev graph_dev_;
  bool have_graph_dev_ = false;
  bool l2_window_set_ = false;
  uint64_t launches_ = 0;
  char err_[256];
};

}  // namespace

GsBackend* gs_make_cuda_backend(int device, char* err, size_t err_cap) {
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    snprintf(err, err_cap, "no CUDA device: %s (libgsim has no CPU fallback)",
             e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    return nullptr;
  }
  if (device < 0) {
    if (cudaGetDevice(&device) != cudaSuccess) device = 0;
  }
  if (device >= count) {
    snprintf(err, err_cap, "CUDA device %d out of range (%d devices)", device, count);
    return nullptr;
  }
  cudaDeviceProp prop;
  if (cudaGetDeviceProperties(&prop, device) != cudaSuccess || prop.major != 9 || prop.minor != 0) {
    snprintf(err, err_cap, "device %d is not sm_90 (libgsim ships sm_90a SASS only)", device);
    return nullptr;
  }
  if (cudaSetDevice(device) != cudaSuccess) {
    snprintf(err, err_cap, "cudaSetDevice(%d) failed", device);
    return nullptr;
  }
  return new CudaBackend(device);
}
