// The coordinate queries through the C++ serf facade (include/gsim_serf.hpp): Serf::DistanceTo(name), the
// librtt.ComputeDistance of `consul rtt`, and Serf::DatacentersByDistance(), Router.GetDatacentersByDistance.
// A WAN pool of four datacenters (128 members each, §3.1) whose one-way latency grows with the distance
// between datacenter indices; two named agents live in the last datacenter.
#include <cstdio>
#include <cstdlib>

#include "gsim_serf.hpp"

using namespace serf;

#define CHECK(c)                                                      \
  do {                                                                \
    if (!(c)) {                                                       \
      std::printf("FAIL %s:%d: %s\n", __FILE__, __LINE__, #c);        \
      std::exit(1);                                                   \
    }                                                                 \
  } while (0)

int main() {
  gsim_config c = Pool::DefaultWANConfig();
  c.capacity = 512;
  c.n_initial = 510;  // datacenters 0..3; ids 510, 511 (the named agents) are in datacenter 3
  c.seed = 17;
  c.flags = GSIM_FLAG_COORDINATES;
  c.mailbox_depth = 8;
  Pool pool(c);
  uint8_t lat[16];
  for (int a = 0; a < 4; ++a)
    for (int b = 0; b < 4; ++b) lat[a * 4 + b] = (uint8_t)(1 + (a > b ? a - b : b - a));
  CHECK(gsim_latency_set(pool.handle(), 4, lat) == 0);
  Config ca, cb;
  ca.NodeName = "a.dc3";
  cb.NodeName = "b.dc3";
  auto a = Serf::Create(pool, ca), b = Serf::Create(pool, cb);
  uint32_t seed = 0;
  int n_ok = 0;
  CHECK(gsim_join(pool.handle(), a->id(), &seed, 1, 1, &n_ok) == 0 && n_ok == 1);
  CHECK(gsim_join(pool.handle(), b->id(), &seed, 1, 1, &n_ok) == 0 && n_ok == 1);
  pool.Step(3000);

  // DistanceTo(name): the coordinates' DistanceTo through time.Duration (whole nanoseconds, truncated)
  const double d = a->DistanceTo("b.dc3");
  Coordinate here = a->GetCoordinate(), there;
  CHECK(a->GetCachedCoordinate("b.dc3", &there));
  const double raw = here.DistanceTo(there);
  CHECK(d <= raw && raw - d < 1.0e-9);
  CHECK(d < 0.2);  // same datacenter: well under one WAN tick
  CHECK(std::isinf(a->DistanceTo("nosuch")));
  std::puts("PASS Serf.DistanceTo");

  // DatacentersByDistance(): the agent's own datacenter first, then by latency: dc2, dc1, dc0
  const std::vector<std::string> dcs = a->DatacentersByDistance();
  CHECK(dcs.size() == 4);
  CHECK(dcs[0] == "dc3" && dcs[1] == "dc2" && dcs[2] == "dc1" && dcs[3] == "dc0");
  std::puts("PASS Serf.DatacentersByDistance");
  std::puts("ALL PASS");
  return 0;
}
