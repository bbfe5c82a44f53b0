// Serf::Stats() through the C++ serf facade (include/gsim_serf.hpp): serf's key set for one agent
// (agent/consul/server.go:1733), read on the device with gsim_agent_stats_read.  On a two-agent pool the Lamport
// member clock rises when the other agent's join intent arrives, an intent and a user event sit in their queues
// until they have been retransmitted, and an agent whose probes go unanswered (its only peer crashed: nobody to
// relay a probe, so no nack either) loses health (memberlist GetHealthScore).
#include <cstdio>
#include <cstdlib>
#include <string>

#include "gsim_serf.hpp"

using namespace serf;

#define CHECK(c)                                                      \
  do {                                                                \
    if (!(c)) {                                                       \
      std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c);        \
      std::exit(1);                                                   \
    }                                                                 \
  } while (0)

// retry.Run in simulated time, as tests/facade/facade_check.cpp does
template <class F>
static bool eventually(Pool& p, uint32_t max_ticks, F f) {
  for (uint32_t t = 0; t < max_ticks; ++t) {
    if (f()) return true;
    p.Step(1);
  }
  return f();
}

static unsigned long stat(Serf& s, const char* key) { return std::stoul(s.Stats().at(key)); }

int main() {
  gsim_config c = Pool::TestConfig();
  c.capacity = 16;
  c.n_initial = 0;
  c.seed = 42;
  c.flags = GSIM_FLAG_LOG_GLOBAL_EVENTS;
  try {
    Pool pool(c);
    Config c1, c2;
    c1.NodeName = "s1";
    c2.NodeName = "s2";
    auto s1 = Serf::Create(pool, c1), s2 = Serf::Create(pool, c2);
    auto st = s1->Stats();
    for (const char* k : {"members", "failed", "left", "health_score", "member_time", "event_time", "query_time",
                          "intent_queue", "event_queue", "query_queue", "encrypted", "coordinate_resets", "tick"})
      CHECK(st.count(k) == 1);
    CHECK(st.at("members") == "1" && st.at("member_time") == "1" && st.at("query_time") == "1");
    CHECK(st.at("health_score") == "0" && st.at("event_queue") == "0" && st.at("encrypted") == "false");
    CHECK(s2->Join({"s1/x"}, true) == 1);
    CHECK(s2->Stats().at("intent_queue") == "1");
    CHECK(eventually(pool, 140, [&] { return s1->NumNodes() == 2 && s2->NumNodes() == 2; }));
    CHECK(eventually(pool, 140, [&] { return stat(*s1, "member_time") > 1; }));
    CHECK(s1->Stats().at("members") == "2" && s2->Stats().at("members") == "2");
    s1->UserEvent("deploy", "v2", false);
    CHECK(s1->Stats().at("event_queue") == "1" && s2->Stats().at("event_queue") == "0");
    CHECK(eventually(pool, 140, [&] { return stat(*s2, "event_time") > 1; }));
    s2->Shutdown();
    CHECK(eventually(pool, 400, [&] { return stat(*s1, "health_score") > 0; }));
    CHECK(eventually(pool, 400, [&] { return s1->Stats().at("failed") == "1"; }));
    CHECK(s1->Stats().at("members") == "2" && s1->Stats().at("left") == "0");
    std::puts("PASS Serf.Stats per agent");
  } catch (const Error& e) {
    std::printf("gsim error %d: %s\n", e.code, e.what());
    return 2;
  }
  std::puts("ALL PASS");
  return 0;
}
