// queue_wake_check.cpp — TEST INFRASTRUCTURE ONLY (tests/test_idle_rows_cpu.py compiles it with the host
// emulation backend into a temporary directory and runs it).
//
// Checks the invariant next to GS_WAKE_BIT in consul_b200/csrc/gs_core.h after every single tick of a
// join cascade with a user event on top: every running member with a non-empty broadcast queue has
// GS_WAKE_BIT in the mailbox slot of its next gossip tick or an earlier one.  The pool's columns are read
// directly (the host emulation keeps them in host memory); the wake bit is an implementation detail that
// the C ABI masks out of every column it returns.
//
//   queue_wake_check            prints one line per case and exits non-zero on any violation
#define GS_MAKE_BACKEND gs_make_hostemu_backend
#include "../../consul_b200/csrc/gs_api.cpp"

#include <stdio.h>

namespace {

uint64_t violations(const gsim_pool* p) {
  const GsDev& d = p->d;
  const GsGlobals& g = p->g;
  const uint32_t now = p->now, depth = g.ring_mask + 1u;
  uint64_t bad = 0;
  for (uint32_t i = 0; i < g.n; ++i) {
    if (gs_key_truth(d.key[now & 1u][i]) != GS_TRUTH_UP || (d.queued[i] & g.active_mask) == 0u) continue;
    const uint32_t gphase = gs_meta_gphase(d.meta[i]);
    uint32_t tg = now;
    while (tg % g.GI != gphase) ++tg;  // the member's next gossip tick
    bool ok = false;
    for (uint32_t s = now; s <= tg && s < now + depth; ++s) ok = ok || (d.inbox[s & g.ring_mask][i] & GS_WAKE_BIT);
    if (!ok) ++bad;
  }
  return bad;
}

// One case: n members, a joiner, a user event, `ticks` single ticks; returns the violations seen.
int run_case(const char* name, gsim_config cfg, uint32_t n, uint32_t ticks) {
  cfg.capacity = n + 4;
  cfg.n_initial = n;
  gsim_pool* p = nullptr;
  if (gsim_pool_create(&cfg, &p) != GSIM_OK) {
    printf("%s: pool_create failed\n", name);
    return -1;
  }
  uint32_t x = 0, slot = 0;
  const uint32_t seed = 0;
  int n_ok = 0;
  if (gsim_member_add(p, nullptr, &x) != GSIM_OK || gsim_join(p, x, &seed, 1, 1, &n_ok) != GSIM_OK ||
      gsim_user_event(p, 7, "deploy", 6, "v2", 2, 0, &slot) != GSIM_OK) {
    printf("%s: setup failed: %s\n", name, gsim_last_error(p));
    gsim_pool_destroy(p);
    return -1;
  }
  uint64_t bad = 0, queued_rows = 0;
  for (uint32_t k = 0; k < ticks; ++k) {
    if (gsim_step(p, 1) != GSIM_OK) {
      printf("%s: step failed: %s\n", name, gsim_last_error(p));
      gsim_pool_destroy(p);
      return -1;
    }
    bad += violations(p);
    for (uint32_t i = 0; i < p->g.n; ++i) queued_rows += (p->d.queued[i] & p->g.active_mask) != 0u;
  }
  printf("%s: GI %u, ring depth %u, %u ticks, %llu queued member-ticks, %llu violations\n", name, p->g.GI,
         p->g.ring_mask + 1u, ticks, (unsigned long long)queued_rows, (unsigned long long)bad);
  gsim_pool_destroy(p);
  return queued_rows > 0 && bad == 0 ? 0 : 1;
}

}  // namespace

int main() {
  gsim_config lan, wan, slow;
  gsim_config_default_lan(&lan);
  lan.seed = 0x5EED0011;
  gsim_config_default_wan(&wan);  // WAN timing on 100 ms ticks: GossipInterval = 5 ticks, depth-8 ring
  wan.seed = 0x5EED0051;
  wan.tick_ns = 100 * MS;
  wan.mailbox_depth = 8;
  gsim_config_default_lan(&slow);  // GossipInterval 3 ticks on a depth-2 ring: the wake goes to t + 1
  slow.seed = 0x5EED0061;
  slow.gossip_interval_ns = 300 * MS;
  int rc = 0;
  rc |= run_case("lan", lan, 3000, 40);
  rc |= run_case("wan", wan, 1000, 60);
  rc |= run_case("gi>depth", slow, 600, 60);
  return rc ? 1 : 0;
}
