// gs_query.h — read-only network-coordinate queries (DESIGN.md §3.4 "Queries"): the per-element bodies
// shared by the host defaults of GsBackend (gs_api.cpp) and the sm_90a query kernels (gs_cuda.cu).
//
// [U] internal/gossip/librtt/rtt.go ComputeDistance, agent/consul/rtt.go sortNodesByDistanceFrom,
// agent/router/router.go GetDatacentersByDistance.  Nothing here writes pool state.
#pragma once
#include "gs_row.h"

#define GS_PUR_COORD_SAMPLE 11  // Philox purpose word of gsim_coordinate_error's pair draws
#define GS_ERR_CHUNK 256u       // draws per partial sum of gsim_coordinate_error's mean
#define GS_DC_SKIPPED 255u      // datacenter digit of an entry the router skips (sorts after every datacenter)

// The coordinate member j publishes: its newer slot, the rule gsim_coordinate_get reads it by.  (Between
// steps every tag is <= now, so the newer slot is also the one gs_coord_slot_for_reader picks at now.)
GS_DEV void gs_coord_pick(const double* coord, const uint32_t* ctag, size_t cap, uint32_t j, GsCoord& c) {
  const size_t slot = ctag[cap + j] > ctag[j] ? 1u : 0u;
  const double* base = coord + slot * GS_COORD_WORDS * cap + j;
  for (int x = 0; x < GS_COORD_DIM; ++x) c.vec[x] = base[(size_t)x * cap];
  c.error = base[(size_t)8 * cap];
  c.adjustment = base[(size_t)9 * cap];
  c.height = base[(size_t)10 * cap];
}

// Is member m's impairment in force at tick `now` (gs_imp_in_force), for pools with member or domain
// schedules only: out of line, so that the query kernels of pools without schedules do not carry the
// schedule lookups (column pointers by value: taking the address of the kernel's GsDev parameter would copy
// it to the stack).
#if defined(__CUDA_ARCH__)
__device__ __noinline__
#else
inline
#endif
uint32_t gs_rtt_on(uint32_t seed_lo, uint32_t seed_hi, const uint32_t* flap, const uint32_t* dom,
                   const uint32_t* dom_flap, uint32_t dom_flap_n, uint32_t m, uint32_t now) {
  const uint32_t wm = flap != nullptr ? flap[m] : 0u;
  const uint32_t x = dom_flap != nullptr ? dom[m] : 0u, wd = x != 0u && x < dom_flap_n ? dom_flap[x] : 0u;
  return gs_in_force(seed_lo, seed_hi, m, wm, x, wd, now) ? 1u : 0u;
}

// The round trip a direct probe between a and b would sample at tick `now` (gs_coord_on_ack): the latency matrix and
// the receivers' delays there and back, each while that receiver's impairment is in force (d.imp_delay is null
// while nobody is impaired; without member or domain schedules every impairment is in force).
GS_DEV double gs_model_rtt(const GsGlobals& g, const GsDev& d, uint32_t a, uint32_t b, uint32_t now) {
  uint32_t on_a = 1u, on_b = 1u;
  if (d.imp_flap != nullptr || d.dom_flap != nullptr) {
    on_a = gs_rtt_on(g.seed_lo, g.seed_hi, d.imp_flap, d.imp_dom, d.dom_flap, d.dom_flap_n, a, now);
    on_b = gs_rtt_on(g.seed_lo, g.seed_hi, d.imp_flap, d.imp_dom, d.dom_flap, d.dom_flap_n, b, now);
  }
  return g.coord_base_rtt_s + (double)(gs_extra(g, d.imp_delay, a, b, on_b) + gs_extra(g, d.imp_delay, b, a, on_a)) *
                                  g.tick_seconds;
}

// Sort key of a distance: its IEEE bits.  gs_coord_distance_seconds never returns a negative value, -0 or
// NaN, so these bits order like the distances.
GS_HD uint64_t gs_dist_key(double s) {
  uint64_t k;
  memcpy(&k, &s, 8);
  return k;
}
GS_HD double gs_key_dist(uint64_t k) {
  double s;
  memcpy(&s, &k, 8);
  return s;
}
GS_HD bool gs_dist_key_ok(uint64_t k) { return k < 0x7FF0000000000000ull; }  // finite, sign clear

// Datacenter of a router entry (§3.1: member i is in (i / 128) % n_dcs), GS_DC_SKIPPED for a skipped one.
GS_HD uint32_t gs_dc_digit(uint32_t val, uint32_t n_dcs) {
  return val == GS_EMPTY32 ? GS_DC_SKIPPED : (val / GS_TILE) % n_dcs;
}

// GetDatacentersByDistance's entry for server `s` seen from `from` at tick `now`: skipped (val = GS_EMPTY32)
// when the view lists it Left or it no longer exists; 0.0 in from's own datacenter; else ComputeDistance.
GS_DEV void gs_router_entry(const GsDev& d, const GsGlobals& g, uint32_t now, uint32_t from, const GsCoord& cf,
                            uint32_t s, uint64_t* key, uint32_t* val) {
  const uint32_t k = d.key[now & 1u][s];
  if (gs_key_truth(k) == GS_TRUTH_NONE || gs_key_rank(k) == GS_RANK_LEFT) {
    *key = ~0ull;
    *val = GS_EMPTY32;
    return;
  }
  *val = s;
  if ((s / GS_TILE) % g.n_dcs == (from / GS_TILE) % g.n_dcs) {
    *key = 0ull;
    return;
  }
  GsCoord c;
  gs_coord_pick(d.coord, d.ctag, g.cap, s, c);
  *key = gs_dist_key(gs_coord_distance_seconds(cf, c));
}

// Draw k of gsim_coordinate_error: the pair (x mod n, y mod n) of philox(seed; k, salt, 11); kept iff the two
// differ and both run at tick now.  Returns the relative error |est - true| / true, or -1.0 for a skipped draw.
GS_DEV double gs_error_draw(const GsDev& d, const GsGlobals& g, uint32_t now, uint32_t k, uint32_t salt) {
  const GsU4 r = gs_philox(g.seed_lo, g.seed_hi, k, salt, GS_PUR_COORD_SAMPLE, 0u);
  const uint32_t i = r.x % g.n, j = r.y % g.n;
  if (i == j || gs_key_truth(d.key[now & 1u][i]) != GS_TRUTH_UP || gs_key_truth(d.key[now & 1u][j]) != GS_TRUTH_UP)
    return -1.0;
  GsCoord a, b;
  gs_coord_pick(d.coord, d.ctag, g.cap, i, a);
  gs_coord_pick(d.coord, d.ctag, g.cap, j, b);
  const double est = gs_coord_distance_seconds(a, b), tru = gs_model_rtt(g, d, i, j, now);
  return fabs(est - tru) / tru;
}

// The order statistic of `m` ascending values at quantile q: the element at floor(q (m - 1)).
GS_HD size_t gs_quantile_index(double q, size_t m) { return (size_t)(q * (double)(m - 1u)); }

// gsim_coordinate_error's result from the sorted keys (kept draws first, ascending) and the chunk sums:
// part[c] = sum of chunk c's kept errors in draw order, part[nch + c] = how many it kept.  The mean adds the
// chunk sums in chunk order.  With nothing kept, every statistic is NaN.
GS_HD void gs_error_finish(const uint64_t* sorted, uint32_t n_draws, const double* part, double out[6]) {
  const uint32_t nch = (n_draws + GS_ERR_CHUNK - 1u) / GS_ERR_CHUNK;
  double sum = 0.0, kept = 0.0;
  for (uint32_t c = 0; c < nch; ++c) {
    sum = sum + part[c];
    kept = kept + part[nch + c];
  }
  const size_t m = (size_t)kept;
  out[0] = kept;
  if (m == 0u) {
    for (int x = 1; x < 6; ++x) out[x] = gs_key_dist(0x7FF8000000000000ull);
    return;
  }
  out[1] = sum / kept;
  out[2] = gs_key_dist(sorted[gs_quantile_index(0.5, m)]);
  out[3] = gs_key_dist(sorted[gs_quantile_index(0.9, m)]);
  out[4] = gs_key_dist(sorted[gs_quantile_index(0.99, m)]);
  out[5] = gs_key_dist(sorted[m - 1u]);
}
