// gsim_serf.hpp — header-only C++ host side above the C ABI, mirroring the serf surface Consul
// calls (SURVEY.md §1/§8b).  The reference is Go; no Go toolchain exists in this image, so the
// host side is C++ with the reference's names, argument meaning and error behaviour:
//
//   serf::Create(conf)                      agent/consul/server_serf.go:63, client_serf.go:76
//   Serf::Join(existing, ignoreOld) -> n    server_ce.go:44, client.go:222, serf_flooder.go:72
//   Serf::Leave(), Shutdown()               server.go:1360,1367,1261; client.go:205,188
//   Serf::UserEvent(name, payload, coalesce) server_ce.go:125
//   Serf::Members(), LocalMember(), NumNodes()  server.go:1485-1500, router.go:62-67
//   Serf::RemoveFailedNode[Prune](node)     server.go:1510-1534
//   Serf::Stats()                           server.go:1733
//   conf.EventCh                            server_serf.go:270-297 (here: Pool::PumpEvents)
//
// One serf::Pool = one gossip pool (LAN or WAN) = one gsim_pool on the device; every
// serf::Create on it adds a virtual agent.  Time is explicit: Pool::Step(ticks).
#pragma once
#include <cmath>
#include <cstdint>
#include <cstring>
#include <deque>
#include <functional>
#include <limits>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "gsim.h"

namespace serf {

enum MemberStatus { StatusNone = 0, StatusAlive = 1, StatusLeaving = 2, StatusLeft = 3, StatusFailed = 4 };
enum EventType { EventMemberJoin = 0, EventMemberLeave, EventMemberFailed, EventMemberUpdate, EventMemberReap, EventUser, EventQuery };

inline const char* StatusString(int s) {  // serf.MemberStatus.String(), command/members/members.go:112
  switch (s) {
    case StatusNone: return "none";
    case StatusAlive: return "alive";
    case StatusLeaving: return "leaving";
    case StatusLeft: return "left";
    case StatusFailed: return "failed";
  }
  return "unknown";
}

struct Member {
  std::string Name;
  std::map<std::string, std::string> Tags;
  int Status = StatusNone;
  uint32_t Incarnation = 0;
};

struct Event {
  EventType Type;
  std::vector<Member> Members;  // member events
  uint32_t LTime = 0;           // user events
  std::string Name, Payload;
  uint32_t Tick = 0;
};

// coordinate.Coordinate ([U] serf/coordinate/coordinate.go), seconds
struct Coordinate {
  double Vec[8];
  double Error, Adjustment, Height;
  // Coordinate.DistanceTo(other) in seconds
  double DistanceTo(const Coordinate& o) const {
    double sum = 0.0;
    for (int k = 0; k < 8; ++k) sum += (Vec[k] - o.Vec[k]) * (Vec[k] - o.Vec[k]);
    const double raw = std::sqrt(sum) + Height + o.Height, adjusted = raw + Adjustment + o.Adjustment;
    return adjusted > 0.0 ? adjusted : raw;
  }
};

struct Config {
  std::string NodeName;
  std::map<std::string, std::string> Tags;
  std::deque<Event>* EventCh = nullptr;  // serf.Config.EventCh (server.go:504-505)
  // serf.Config.Merge (agent/consul/server_serf.go:234-239 installs lanMergeDelegate /
  // wanMergeDelegate, agent/consul/merge.go:34,111): called on BOTH sides of a join's push-pull
  // with the other side's member list; a non-empty return value is the error that cancels the
  // merge with that peer.  The delegate itself is Consul code and stays on the host.
  std::function<std::string(const std::vector<Member>&)> Merge;
  // serf.Config.ReconnectTimeoutOverride (libserf/serf.go:68-85 reads the member's "rc_tm" tag):
  // given a member and the pool's ReconnectTimeout in ns, returns the timeout to use for it.
  // Evaluated for this agent's own member record at Create and after SetTags.
  std::function<uint64_t(const Member&, uint64_t)> ReconnectTimeoutOverride;
};

class Error : public std::runtime_error {
 public:
  Error(int code, const std::string& msg) : std::runtime_error(msg), code(code) {}
  int code;
};

class Serf;

class Pool {
 public:
  explicit Pool(const gsim_config& cfg) : default_reconnect_ns_(cfg.reconnect_timeout_ns) {
    int rc = gsim_pool_create(&cfg, &h_);
    if (rc != 0) throw Error(rc, gsim_strerror(rc));
  }
  ~Pool() { gsim_pool_destroy(h_); }
  Pool(const Pool&) = delete;
  Pool& operator=(const Pool&) = delete;

  static gsim_config DefaultLANConfig() {  // [U] memberlist.DefaultLANConfig + libserf.DefaultConfig
    gsim_config c;
    gsim_config_default_lan(&c);
    return c;
  }
  static gsim_config DefaultWANConfig() {
    gsim_config c;
    gsim_config_default_wan(&c);
    return c;
  }
  static gsim_config TestConfig() {  // agent/consul/server_test.go:221-237
    gsim_config c;
    gsim_config_consul_test(&c);
    c.phase_group = 1;
    return c;
  }
  // memberlist piggybacks queued broadcasts on pings, acks, indirect pings and nacks ([U] net.go sendMsg); the
  // simulation does so for pools created from a config passed through here (GSIM_FLAG_PROBE_PIGGYBACK, off by default).
  static gsim_config WithProbePiggyback(gsim_config c, bool on = true) {
    c.flags = on ? (c.flags | GSIM_FLAG_PROBE_PIGGYBACK) : (c.flags & ~GSIM_FLAG_PROBE_PIGGYBACK);
    return c;
  }

  void Step(uint32_t ticks) { check(gsim_step(h_, ticks)); }
  uint32_t Now() const { return gsim_now(h_); }
  // Deliver pending serf events to the EventCh of every agent created on this pool.
  void PumpEvents();
  Member describe(uint32_t id, int status, uint32_t inc);
  Coordinate coordinate_of(uint32_t id) {
    double w[11];
    check(gsim_coordinate_get(h_, id, w));
    Coordinate c;
    for (int k = 0; k < 8; ++k) c.Vec[k] = w[k];
    c.Error = w[8];
    c.Adjustment = w[9];
    c.Height = w[10];
    return c;
  }
  gsim_pool* handle() { return h_; }
  void check(int rc) {
    if (rc != 0) throw Error(rc, std::string(gsim_last_error(h_)).empty() ? gsim_strerror(rc) : gsim_last_error(h_));
  }

 private:
  friend class Serf;
  gsim_pool* h_ = nullptr;
  uint64_t default_reconnect_ns_ = 0;
  std::map<std::string, uint32_t> by_name_;
  std::vector<Serf*> by_id_;
};

class Serf {
 public:
  // serf.Create(conf): one more virtual agent on `pool`.
  static std::unique_ptr<Serf> Create(Pool& pool, const Config& conf) {
    if (pool.by_name_.count(conf.NodeName)) throw Error(GSIM_ERR_STATE, "node name conflict: " + conf.NodeName);
    // The alive{} broadcast is sized by libgsim's encoder (gsim_wire_alive) from the real name and the
    // real Meta: [U] serf.encodeTags = the magic byte 255 + msgpack(map[string]string) of the tags.
    auto raw = [](size_t n) { return (uint32_t)(n < 32 ? 1 + n : n < 65536 ? 3 + n : 5 + n); };
    gsim_member_desc d;
    d.alive_msg_size = 0;
    d.name_len = (uint32_t)conf.NodeName.size();
    d.meta_len = 1u + (conf.Tags.size() < 16 ? 1u : 3u);
    for (auto& kv : conf.Tags) d.meta_len += raw(kv.first.size()) + raw(kv.second.size());
    d.flags = GSIM_MEMBER_WATCHED;
    uint32_t id = 0;
    pool.check(gsim_member_add(pool.h_, &d, &id));
    std::unique_ptr<Serf> s(new Serf(pool, id, conf));
    pool.by_name_[conf.NodeName] = id;
    if (pool.by_id_.size() <= id) pool.by_id_.resize(id + 1, nullptr);
    pool.by_id_[id] = s.get();
    s->apply_reconnect_override();
    return s;
  }

  // Join(existing, ignoreOld) -> number of nodes contacted; throws if none could be.
  int Join(const std::vector<std::string>& existing, bool ignoreOld) {
    std::vector<uint32_t> seeds;
    std::string merge_err;
    for (const std::string& a : existing) {
      std::string node = a.substr(0, a.find('/'));  // "node/ip:port", "node.dc/ip:port"
      auto it = p_.by_name_.find(node);
      if (it == p_.by_name_.end()) continue;
      // [U] memberlist pushPullNode -> MergeDelegate.NotifyMerge on both ends before any state is merged
      Serf* peer = it->second < p_.by_id_.size() ? p_.by_id_[it->second] : nullptr;
      if (peer && peer != this) {
        std::string err;
        if (conf_.Merge) err = conf_.Merge(peer->Members());
        if (err.empty() && peer->conf_.Merge) err = peer->conf_.Merge(Members());
        if (!err.empty()) {  // this peer refused (or was refused): not contacted
          merge_err = err;
          continue;
        }
      }
      seeds.push_back(it->second);
    }
    if (seeds.empty() && !merge_err.empty()) throw Error(GSIM_ERR_STATE, "Failed to join: " + merge_err);
    int n_ok = 0;
    p_.check(gsim_join(p_.h_, id_, seeds.data(), seeds.size(), ignoreOld ? 1 : 0, &n_ok));
    if (n_ok == 0 && !existing.empty()) throw Error(GSIM_ERR_NOT_FOUND, "Failed to join: no seeds could be contacted");
    return n_ok;
  }
  // SetTags(tags) — internal/gossip/libserf/serf.go:51: the tags live here on the host; the
  // re-announcement under the next incarnation (and every other member's EventMemberUpdate) is
  // simulated.  Encoded size of the alive message grows with the tags (UDP budget).
  void SetTags(const std::map<std::string, std::string>& tags) {
    conf_.Tags = tags;
    uint32_t bytes = 64;
    for (auto& kv : tags) bytes += (uint32_t)(kv.first.size() + kv.second.size() + 2);
    if (bytes > 512) bytes = 512;  // memberlist.MetaMaxSize
    p_.check(gsim_member_update(p_.h_, id_, bytes, nullptr));
    apply_reconnect_override();
  }
  // GetCoordinate() / GetCachedCoordinate(name) — agent/router/router.go:62-67: Vivaldi network
  // coordinates (pools created with GSIM_FLAG_COORDINATES).
  Coordinate GetCoordinate() { return p_.coordinate_of(id_); }
  bool GetCachedCoordinate(const std::string& name, Coordinate* out) {
    auto it = p_.by_name_.find(name);
    if (it == p_.by_name_.end()) return false;
    *out = p_.coordinate_of(it->second);
    return true;
  }
  // librtt.ComputeDistance(GetCoordinate(), GetCachedCoordinate(name)) — internal/gossip/librtt/rtt.go:16-22,
  // what `consul rtt` prints: seconds through time.Duration; +inf for a name without a coordinate.
  double DistanceTo(const std::string& name) {
    auto it = p_.by_name_.find(name);
    if (it == p_.by_name_.end()) return std::numeric_limits<double>::infinity();
    double s = 0.0;
    p_.check(gsim_rtt_many(p_.h_, &id_, &it->second, 1, &s, nullptr));
    return s;
  }
  // Router.GetDatacentersByDistance() — agent/router/router.go:537-615, for the area of this agent's pool:
  // datacenter names nearest first by median server RTT (synthetic names "dc<index>", ordered by index on
  // ties).  Datacenters without a server that counts are left out, as upstream.
  std::vector<std::string> DatacentersByDistance() {
    uint32_t order[64];
    double rtt[64];
    for (double& r : rtt) r = std::numeric_limits<double>::quiet_NaN();  // entries past n_dcs stay NaN
    p_.check(gsim_dcs_by_distance(p_.h_, id_, nullptr, 0, order, rtt));
    std::vector<std::string> out;
    for (int c = 0; c < 64; ++c)
      if (std::isfinite(rtt[c])) out.push_back("dc" + std::to_string(order[c]));
    return out;
  }
  void Leave() { p_.check(gsim_leave(p_.h_, id_)); }
  void Shutdown() { p_.check(gsim_crash(p_.h_, id_)); }  // without Leave(): a crash (server_test.go:725)
  void UserEvent(const std::string& name, const std::string& payload, bool coalesce) {
    uint32_t slot = 0;
    p_.check(gsim_user_event(p_.h_, id_, name.data(), name.size(), payload.data(), payload.size(), coalesce ? 1 : 0, &slot));
  }
  std::vector<Member> Members() {
    size_t n = 0;
    p_.check(gsim_members(p_.h_, id_, nullptr, 0, &n));
    std::vector<gsim_member> raw(n ? n : 1);
    p_.check(gsim_members(p_.h_, id_, raw.data(), raw.size(), &n));
    std::vector<Member> out;
    for (size_t x = 0; x < n; ++x) out.push_back(p_.describe(raw[x].id, raw[x].status, raw[x].incarnation));
    return out;
  }
  Member LocalMember() {
    for (Member& m : Members())
      if (m.Name == conf_.NodeName) return m;
    return Member();
  }
  int NumNodes() {
    uint32_t n = 0;
    p_.check(gsim_num_nodes(p_.h_, id_, &n));
    return (int)n;
  }
  void RemoveFailedNode(const std::string& node) { force_leave(node, 0); }
  void RemoveFailedNodePrune(const std::string& node) { force_leave(node, 1); }
  // serf's key set for this agent ([U] serf.Stats), computed on the device, plus the pool's tick.  Nothing is
  // encrypted inside the simulator and the model never resets a coordinate.
  std::map<std::string, std::string> Stats() {
    gsim_agent_stats a;
    p_.check(gsim_agent_stats_read(p_.h_, id_, 1, &a));
    auto u = [](uint32_t v) { return std::to_string(v); };
    return {{"members", u(a.members)},           {"failed", u(a.failed)},
            {"left", u(a.left)},                 {"health_score", u(a.health_score)},
            {"member_time", u(a.member_time)},   {"event_time", u(a.event_time)},
            {"query_time", u(a.query_time)},     {"intent_queue", u(a.intent_queue)},
            {"event_queue", u(a.event_queue)},   {"query_queue", u(a.query_queue)},
            {"encrypted", "false"},              {"coordinate_resets", "0"},
            {"tick", u(gsim_now(p_.h_))}};
  }
  const Config& config() const { return conf_; }
  uint32_t id() const { return id_; }

 private:
  friend class Pool;
  Serf(Pool& p, uint32_t id, const Config& c) : p_(p), id_(id), conf_(c) {}
  void apply_reconnect_override() {
    if (!conf_.ReconnectTimeoutOverride) return;
    const uint64_t dflt = p_.default_reconnect_ns_;
    const uint64_t t = conf_.ReconnectTimeoutOverride(p_.describe(id_, StatusAlive, 0), dflt);
    p_.check(gsim_member_reconnect_timeout_set(p_.h_, id_, t == dflt ? 0 : t));
  }
  void force_leave(const std::string& node, int prune) {
    auto it = p_.by_name_.find(node);
    if (it == p_.by_name_.end()) return;
    p_.check(gsim_force_leave(p_.h_, id_, it->second, prune));
  }
  Pool& p_;
  uint32_t id_;
  Config conf_;
};

inline Member Pool_describe(const std::vector<Serf*>& by_id, uint32_t id, int status, uint32_t inc) {
  Member m;
  m.Status = status;
  m.Incarnation = inc;
  if (id < by_id.size() && by_id[id]) {
    m.Name = by_id[id]->config().NodeName;
    m.Tags = by_id[id]->config().Tags;
  } else {
    m.Name = "member-" + std::to_string(id);
  }
  return m;
}

}  // namespace serf

// --- out-of-class definitions that need the complete Serf type --------------------------------
namespace serf {
inline Member Pool::describe(uint32_t id, int status, uint32_t inc) { return Pool_describe(by_id_, id, status, inc); }

inline void Pool::PumpEvents() {
  std::vector<gsim_event> buf(4096);
  size_t n = 0;
  check(gsim_poll_events(h_, buf.data(), buf.size(), &n));
  for (size_t x = 0; x < n; ++x) {
    const gsim_event& e = buf[x];
    Event ev;
    ev.Type = (EventType)e.type;
    ev.Tick = e.tick;
    if (e.type == GSIM_EVENT_USER) {
      char name[1024], payload[1024];
      size_t nl = 0, pl = 0;
      if (gsim_user_event_get(h_, e.subject, name, sizeof(name), &nl, payload, sizeof(payload), &pl) == 0) {
        ev.Name.assign(name, nl);
        ev.Payload.assign(payload, pl);
      }
      ev.LTime = e.ltime;
    } else {
      int st = e.type == GSIM_EVENT_MEMBER_FAILED ? StatusFailed : e.type == GSIM_EVENT_MEMBER_LEAVE ? StatusLeft : StatusAlive;
      ev.Members.push_back(describe(e.subject, st, 0));
    }
    for (Serf* s : by_id_) {
      if (!s || !s->config().EventCh) continue;
      if (e.observer == 0xFFFFFFFFu || e.observer == s->id()) s->config().EventCh->push_back(ev);
    }
  }
}
}  // namespace serf
