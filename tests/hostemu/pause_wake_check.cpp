// pause_wake_check.cpp — TEST INFRASTRUCTURE ONLY (tests/test_pause_cpu.py compiles it with the host
// emulation backend into a temporary directory and runs it).
//
// The queue_wake_check build (its violations() check of the invariant next to GS_WAKE_BIT) across paused
// members: members that have broadcasts queued are paused for several lengths (shorter than ProbeTimeout,
// past ProbeInterval, past the suspicion timeout), and the invariant is checked after every single tick,
// through every resume.
//
//   pause_wake_check            prints one line per case and exits non-zero on any violation
#define main queue_wake_check_main
#include "queue_wake_check.cpp"
#undef main

namespace {

int run_pause_case(const char* name, gsim_config cfg, uint32_t n, uint32_t ticks) {
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
  uint64_t bad = 0, queued_paused = 0, resumed = 0;
  for (uint32_t k = 0; k < ticks; ++k) {
    if (k % 7 == 2) {  // pause some members that have broadcasts queued right now
      std::vector<uint32_t> ids;
      for (uint32_t i = k; i < p->g.n && ids.size() < 16; i += 37)
        if ((p->d.queued[i] & p->g.active_mask) != 0u) ids.push_back(i);
      static const uint32_t lengths[4] = {2, 13, 60, 400};
      uint32_t paused = 0;
      if (!ids.empty() && gsim_pause_many(p, ids.data(), ids.size(), lengths[(k / 7) % 4], &paused) != GSIM_OK) {
        printf("%s: pause failed: %s\n", name, gsim_last_error(p));
        gsim_pool_destroy(p);
        return -1;
      }
      queued_paused += paused;
    }
    if (gsim_step(p, 1) != GSIM_OK) {
      printf("%s: step failed: %s\n", name, gsim_last_error(p));
      gsim_pool_destroy(p);
      return -1;
    }
    bad += violations(p);
  }
  uint64_t st[4];
  gsim_pause_stats(p, st);
  resumed = st[1] + st[2] + st[3];
  printf("%s: %u ticks, %llu members paused with broadcasts queued, %llu resumed, %llu violations\n", name, ticks,
         (unsigned long long)queued_paused, (unsigned long long)resumed, (unsigned long long)bad);
  gsim_pool_destroy(p);
  return queued_paused > 0 && resumed > 0 && bad == 0 ? 0 : 1;
}

}  // namespace

int main() {
  gsim_config lan, wan;
  gsim_config_default_lan(&lan);
  lan.seed = 0x5EED0111;
  gsim_config_default_wan(&wan);  // WAN timing on 100 ms ticks: GossipInterval = 5 ticks, depth-8 ring
  wan.seed = 0x5EED0151;
  wan.tick_ns = 100 * MS;
  wan.mailbox_depth = 8;
  int rc = 0;
  rc |= run_pause_case("lan", lan, 3000, 120);
  rc |= run_pause_case("wan", wan, 1000, 160);
  return rc ? 1 : 0;
}
