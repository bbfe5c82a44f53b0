// gs_wire.h — wire formats of the gossip path (SURVEY §8f N4), host side only.
//
// What memberlist and serf put on the wire decides how many broadcasts fit into one UDP packet
// ([U] memberlist/queue.go GetBroadcasts against UDPBufferSize), i.e. the byte budget that
// gs_select_packet enforces.  This file is the encoder those sizes come from:
//   * msgpack as hashicorp/go-msgpack v2 writes it ([U] codec/msgpack.go; pinned go.mod:213):
//     structs are maps keyed by the Go field name (or the `codec` tag), unsigned integers take the
//     shortest of fixint/uint8/16/32/64, and — for memberlist and serf, whose handle is the zero
//     codec.MsgpackHandle{} (WriteExt false) — strings AND byte slices are "raw": fixraw up to 31
//     bytes, then raw16/raw32, no str8 and no bin.  Consul's own user-event payload uses
//     MsgpackHandle{RawToString: true, WriteExt: true} (agent/user_event.go:291-296): str8 and bin.
//   * memberlist messages alive / suspect / dead behind a 1-byte message type, the compound packet
//     ([U] memberlist/util.go makeCompoundMessage: type, count, count big-endian u16 lengths, bodies);
//   * serf's join / leave intents and user events behind a 1-byte serf type, framed by memberlist's
//     userMsg byte when they travel as gossip ([U] memberlist/net.go, serf/messages.go);
//   * the WAN federation frame (agent/consul/wanfed/wanfed.go:112-121: big-endian u32 length, then
//     the packet) and Consul's UserEvent payload (agent/user_event.go:27-52).
// None of the bytes ever enter device memory: the device carries sizes (GsRumor::size).
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string.h>

namespace gsw {

// [U] memberlist/net.go messageType, [U] serf/messages.go messageType
enum { ML_PING = 0, ML_INDIRECT_PING = 1, ML_ACK = 2, ML_SUSPECT = 3, ML_ALIVE = 4, ML_DEAD = 5, ML_PUSH_PULL = 6,
       ML_COMPOUND = 7, ML_USER = 8, ML_COMPRESS = 9, ML_ENCRYPT = 10, ML_NACK = 11 };
enum { SERF_LEAVE = 0, SERF_JOIN = 1, SERF_PUSH_PULL = 2, SERF_USER_EVENT = 3, SERF_QUERY = 4 };

struct Buf {
  uint8_t* p;
  size_t cap, n;
  Buf(void* out, size_t c) : p(static_cast<uint8_t*>(out)), cap(out ? c : 0), n(0) {}
  void put(uint8_t b) {  // counts past the end: n is always the size needed
    if (n < cap) p[n] = b;
    ++n;
  }
  void put(const void* s, size_t len) {  // (sizing calls pass no buffer and possibly no source)
    if (s != nullptr && len && n + len <= cap) memcpy(p + n, s, len);
    n += len;
  }
  void be16(uint32_t v) { put((uint8_t)(v >> 8)); put((uint8_t)v); }
  void be32(uint32_t v) { be16(v >> 16); be16(v & 0xFFFFu); }
  void be64(uint64_t v) { be32((uint32_t)(v >> 32)); be32((uint32_t)v); }
};

// ---- msgpack primitives -------------------------------------------------------------------
inline void mp_uint(Buf& b, uint64_t v) {
  if (v <= 0x7Fu) b.put((uint8_t)v);
  else if (v <= 0xFFu) { b.put(0xCC); b.put((uint8_t)v); }
  else if (v <= 0xFFFFu) { b.put(0xCD); b.be16((uint32_t)v); }
  else if (v <= 0xFFFFFFFFull) { b.put(0xCE); b.be32((uint32_t)v); }
  else { b.put(0xCF); b.be64(v); }
}
inline void mp_bool(Buf& b, bool v) { b.put(v ? 0xC3 : 0xC2); }
inline void mp_nil(Buf& b) { b.put(0xC0); }
inline void mp_map(Buf& b, uint32_t n) {
  if (n < 16) b.put((uint8_t)(0x80u | n));
  else { b.put(0xDE); b.be16(n); }
}
// a string; `ext` = the handle has WriteExt (str8 exists)
inline void mp_str(Buf& b, const void* s, size_t len, bool ext) {
  if (len < 32) b.put((uint8_t)(0xA0u | len));
  else if (ext && len < 256) { b.put(0xD9); b.put((uint8_t)len); }
  else if (len < 65536) { b.put(0xDA); b.be16((uint32_t)len); }
  else { b.put(0xDB); b.be32((uint32_t)len); }
  b.put(s, len);
}
// a []byte: raw (= string form) without WriteExt, bin8/16/32 with it; a nil slice is nil
inline void mp_bytes(Buf& b, const void* s, size_t len, bool ext) {
  if (s == nullptr) return mp_nil(b);
  if (!ext) return mp_str(b, s, len, false);
  if (len < 256) { b.put(0xC4); b.put((uint8_t)len); }
  else if (len < 65536) { b.put(0xC5); b.be16((uint32_t)len); }
  else { b.put(0xC6); b.be32((uint32_t)len); }
  b.put(s, len);
}
inline void mp_key(Buf& b, const char* k) { mp_str(b, k, strlen(k), false); }  // field names are short

// ---- memberlist ---------------------------------------------------------------------------
// alive{Incarnation uint32; Node string; Addr []byte; Port uint16; Meta []byte; Vsn []uint8}
inline size_t alive(void* out, size_t cap, uint32_t inc, const char* node, size_t node_len, const void* addr,
                    size_t addr_len, uint16_t port, const void* meta, size_t meta_len, const uint8_t vsn[6]) {
  Buf b(out, cap);
  b.put(ML_ALIVE);
  mp_map(b, 6);
  mp_key(b, "Incarnation"); mp_uint(b, inc);
  mp_key(b, "Node"); mp_str(b, node, node_len, false);
  mp_key(b, "Addr"); mp_bytes(b, addr, addr_len, false);
  mp_key(b, "Port"); mp_uint(b, port);
  mp_key(b, "Meta"); mp_bytes(b, meta, meta_len, false);
  mp_key(b, "Vsn"); mp_bytes(b, vsn, 6, false);
  return b.n;
}
// suspect{Incarnation; Node; From} and dead{Incarnation; Node; From} differ in the type byte only
inline size_t suspect_or_dead(void* out, size_t cap, bool dead, uint32_t inc, const char* node, size_t node_len,
                              const char* from, size_t from_len) {
  Buf b(out, cap);
  b.put(dead ? ML_DEAD : ML_SUSPECT);
  mp_map(b, 3);
  mp_key(b, "Incarnation"); mp_uint(b, inc);
  mp_key(b, "Node"); mp_str(b, node, node_len, false);
  mp_key(b, "From"); mp_str(b, from, from_len, false);
  return b.n;
}
// Probe messages ([U] memberlist/net.go).  ping{SeqNo uint32; Node string; SourceAddr []byte; SourcePort
// uint16; SourceNode string}, the three source fields `codec:",omitempty"`.
inline void probe_source(Buf& b, const void* addr, size_t addr_len, uint16_t port, const char* src, size_t src_len) {
  if (addr != nullptr && addr_len) { mp_key(b, "SourceAddr"); mp_bytes(b, addr, addr_len, false); }
  if (port) { mp_key(b, "SourcePort"); mp_uint(b, port); }
  if (src_len) { mp_key(b, "SourceNode"); mp_str(b, src, src_len, false); }
}
inline uint32_t probe_source_fields(const void* addr, size_t addr_len, uint16_t port, size_t src_len) {
  return (addr != nullptr && addr_len ? 1u : 0u) + (port ? 1u : 0u) + (src_len ? 1u : 0u);
}
inline size_t ping(void* out, size_t cap, uint32_t seq, const char* node, size_t node_len, const void* addr,
                   size_t addr_len, uint16_t port, const char* src, size_t src_len) {
  Buf b(out, cap);
  b.put(ML_PING);
  mp_map(b, 2 + probe_source_fields(addr, addr_len, port, src_len));
  mp_key(b, "SeqNo"); mp_uint(b, seq);
  mp_key(b, "Node"); mp_str(b, node, node_len, false);
  probe_source(b, addr, addr_len, port, src, src_len);
  return b.n;
}
// indirectPingReq{SeqNo uint32; Target []byte; Port uint16; Node string; Nack bool; SourceAddr; SourcePort;
// SourceNode}, the source fields omitempty
inline size_t indirect_ping(void* out, size_t cap, uint32_t seq, const void* target, size_t target_len, uint16_t port,
                            const char* node, size_t node_len, bool nack, const void* addr, size_t addr_len,
                            uint16_t src_port, const char* src, size_t src_len) {
  Buf b(out, cap);
  b.put(ML_INDIRECT_PING);
  mp_map(b, 5 + probe_source_fields(addr, addr_len, src_port, src_len));
  mp_key(b, "SeqNo"); mp_uint(b, seq);
  mp_key(b, "Target"); mp_bytes(b, target, target_len, false);
  mp_key(b, "Port"); mp_uint(b, port);
  mp_key(b, "Node"); mp_str(b, node, node_len, false);
  mp_key(b, "Nack"); mp_bool(b, nack);
  probe_source(b, addr, addr_len, src_port, src, src_len);
  return b.n;
}
// ackResp{SeqNo uint32; Payload []byte} and nackResp{SeqNo uint32}
inline size_t ack(void* out, size_t cap, uint32_t seq, const void* payload, size_t payload_len) {
  Buf b(out, cap);
  b.put(ML_ACK);
  mp_map(b, 2);
  mp_key(b, "SeqNo"); mp_uint(b, seq);
  mp_key(b, "Payload"); mp_bytes(b, payload, payload_len, false);
  return b.n;
}
inline size_t nack(void* out, size_t cap, uint32_t seq) {
  Buf b(out, cap);
  b.put(ML_NACK);
  mp_map(b, 1);
  mp_key(b, "SeqNo"); mp_uint(b, seq);
  return b.n;
}

// [U] memberlist/util.go makeCompoundMessage
inline size_t compound(void* out, size_t cap, const void* const* msgs, const size_t* lens, size_t count) {
  Buf b(out, cap);
  b.put(ML_COMPOUND);
  b.put((uint8_t)count);
  for (size_t i = 0; i < count; ++i) b.be16((uint32_t)lens[i]);
  for (size_t i = 0; i < count; ++i) b.put(msgs[i], lens[i]);
  return b.n;
}

// ---- serf (as gossip payload: `framed` adds memberlist's userMsg byte) ------------------------
// messageJoin{LTime LamportTime; Node string} / messageLeave{LTime; Node; Prune bool}
inline size_t serf_intent(void* out, size_t cap, bool leave, uint64_t ltime, const char* node, size_t node_len,
                          bool prune, bool framed) {
  Buf b(out, cap);
  if (framed) b.put(ML_USER);
  b.put(leave ? SERF_LEAVE : SERF_JOIN);
  mp_map(b, leave ? 3 : 2);
  mp_key(b, "LTime"); mp_uint(b, ltime);
  mp_key(b, "Node"); mp_str(b, node, node_len, false);
  if (leave) { mp_key(b, "Prune"); mp_bool(b, prune); }
  return b.n;
}
// messageUserEvent{LTime; Name string; Payload []byte; CC bool}
inline size_t serf_user_event(void* out, size_t cap, uint64_t ltime, const void* name, size_t name_len,
                              const void* payload, size_t payload_len, bool cc, bool framed) {
  Buf b(out, cap);
  if (framed) b.put(ML_USER);
  b.put(SERF_USER_EVENT);
  mp_map(b, 4);
  mp_key(b, "LTime"); mp_uint(b, ltime);
  mp_key(b, "Name"); mp_str(b, name, name_len, false);
  mp_key(b, "Payload"); mp_bytes(b, payload ? payload : "", payload_len, false);
  mp_key(b, "CC"); mp_bool(b, cc);
  return b.n;
}

// ---- Consul ---------------------------------------------------------------------------------
// agent/user_event.go:27-52 UserEvent through msgpackHandleUserEvent (WriteExt): the payload of the
// serf user event "consul:event:<name>".  omitempty drops empty p / nf / sf / tf.
inline size_t consul_user_event(void* out, size_t cap, const char* id, const char* name, const void* payload,
                                size_t payload_len, const char* node_filter, const char* service_filter,
                                const char* tag_filter, int version) {
  Buf b(out, cap);
  uint32_t fields = 3;  // ID, n, v
  if (payload_len) ++fields;
  if (node_filter && *node_filter) ++fields;
  if (service_filter && *service_filter) ++fields;
  if (tag_filter && *tag_filter) ++fields;
  mp_map(b, fields);
  mp_key(b, "ID"); mp_str(b, id, strlen(id), true);
  mp_key(b, "n"); mp_str(b, name, strlen(name), true);
  if (payload_len) { mp_key(b, "p"); mp_bytes(b, payload, payload_len, true); }
  if (node_filter && *node_filter) { mp_key(b, "nf"); mp_str(b, node_filter, strlen(node_filter), true); }
  if (service_filter && *service_filter) { mp_key(b, "sf"); mp_str(b, service_filter, strlen(service_filter), true); }
  if (tag_filter && *tag_filter) { mp_key(b, "tf"); mp_str(b, tag_filter, strlen(tag_filter), true); }
  mp_key(b, "v"); mp_uint(b, (uint64_t)version);
  return b.n;
}
// agent/consul/wanfed/wanfed.go:112-121: a gossip packet relayed through a mesh gateway
inline size_t wanfed_frame(void* out, size_t cap, const void* packet, size_t len) {
  Buf b(out, cap);
  b.be32((uint32_t)len);
  b.put(packet, len);
  return b.n;
}

}  // namespace gsw
