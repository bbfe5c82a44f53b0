// counting_backend.cpp — TEST INFRASTRUCTURE ONLY.  Never linked into libgsim.so.
//
// The host emulation (hostemu_backend.cpp) behind a pass-through backend that counts the calls which
// wait for the device on the CUDA backend: a synchronous copy, a readback, a stream synchronisation.
// Each such call leaves the GPU idle while the host waits.  Built with gs_api.cpp and the host
// emulation into tests/hostemu/libgsim_hostemu_counted.so by `__graft_entry__.build()`;
// tests/test_host_round_trips.py holds the host side of the C ABI to its budget of round trips with it.
#include <atomic>

#include "../../consul_b200/csrc/gs_backend.h"

GsBackend* gs_make_hostemu_backend(int device, char* err, size_t err_cap);

// over every pool of the process: waits, and how many of them ended a chunk of single ticks
static std::atomic<uint64_t> g_waits{0}, g_tick_chunks{0};
extern "C" uint64_t gsim_hostemu_waits(uint64_t* tick_chunks) {
  if (tick_chunks) *tick_chunks = g_tick_chunks.load();
  return g_waits.load();
}

namespace {

// What waits on the CUDA backend (gs_cuda.cu) is counted once per call; the calls it only enqueues
// (small staged copies, fills, init, write batches, the bit-column pass) are not.
class CountingBackend : public GsBackend {
 public:
  explicit CountingBackend(GsBackend* in) : in_(in) {}
  ~CountingBackend() override { delete in_; }
  const char* name() const override { return in_->name(); }
  void* alloc(size_t bytes) override { return in_->alloc(bytes); }
  void release(void* p) override { in_->release(p); }
  bool h2d(void* dst, const void* src, size_t bytes) override { return wait(), in_->h2d(dst, src, bytes); }
  bool d2h(void* dst, const void* src, size_t bytes) override { return wait(), in_->d2h(dst, src, bytes); }
  bool h2d_word(void* dst, const void* src, size_t bytes) override {
    if (bytes > 16384) wait();  // (the CUDA backend waits for larger copies)
    return in_->h2d_word(dst, src, bytes);
  }
  bool write_batch(const GsWriteBatch& b) override { return in_->write_batch(b); }
  void* host_alloc(size_t bytes) override { return in_->host_alloc(bytes); }
  void host_free(void* q) override { in_->host_free(q); }
  bool h2d_async(void* dst, const void* src, size_t bytes) override { return in_->h2d_async(dst, src, bytes); }
  bool row_read(const GsDev& d, uint32_t i, uint32_t out[8]) override { return wait(), in_->row_read(d, i, out); }
  bool rows_read(const GsDev& d, const uint32_t* ids, uint32_t n, uint32_t* out) override {
    for (uint32_t x = 0; x < n; x += 64u) wait();  // one readback per 64 rows
    return in_->rows_read(d, ids, n, out);
  }
  bool fill32(uint32_t* dst, uint32_t value, size_t count) override { return in_->fill32(dst, value, count); }
  bool fill8(uint8_t* dst, uint8_t value, size_t count) override { return in_->fill8(dst, value, count); }
  bool init_rows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t first, uint32_t count,
                 uint32_t now) override {
    return in_->init_rows(d, g_dev, g, first, count, now);
  }
  bool run_ticks(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t t0, uint32_t nticks,
                 bool use_graph, double* kernel_ms, uint64_t* launches, const GsXbar* xbar) override {
    wait();
    ++g_tick_chunks;
    return in_->run_ticks(d, g_dev, g, t0, nticks, use_graph, kernel_ms, launches, xbar);
  }
  bool run_ticks_read(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t t0, uint32_t nticks,
                      bool use_graph, double* kernel_ms, uint64_t* launches, const GsXbar* xbar,
                      uint32_t* last_active) override {
    wait();  // the launches' readback carries the word
    ++g_tick_chunks;
    return in_->run_ticks_read(d, g_dev, g, t0, nticks, use_graph, kernel_ms, launches, xbar, last_active);
  }
  bool run_windows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t t0, uint32_t nticks,
                   uint32_t per_launch, bool use_graph, double* kernel_ms, uint64_t* launches, uint32_t* ticks_done,
                   const GsXbar* xbar, bool pristine) override {
    wait();
    return in_->run_windows(d, g_dev, g, t0, nticks, per_launch, use_graph, kernel_ms, launches, ticks_done, xbar,
                            pristine);
  }
  bool quiet_scan(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now, uint32_t first,
                  uint32_t count) override {
    wait();
    return in_->quiet_scan(d, g_dev, g, now, first, count);
  }
  bool quiet_probe(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now, uint32_t* horizon,
                   GsRecount* counts) override {
    wait();  // one submission, one readback
    return in_->quiet_probe(d, g_dev, g, now, horizon, counts);
  }
  bool shard_begin(uint32_t world, uint32_t rank) override { return in_->shard_begin(world, rank); }
  size_t shard_granularity() override { return in_->shard_granularity(); }
  void* shard_alloc(size_t slice_bytes, size_t planes) override { return in_->shard_alloc(slice_bytes, planes); }
  bool shard_commit(const int** fds, size_t* n) override { return in_->shard_commit(fds, n); }
  bool shard_attach(uint32_t peer, const int* fds, size_t n) override { return in_->shard_attach(peer, fds, n); }
  bool xbar_host(const GsXbar& xb) override { return wait(), in_->xbar_host(xb); }
  bool crash_fraction(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t thr, uint32_t salt,
                      uint32_t now, uint32_t* n_crashed) override {
    wait();
    return in_->crash_fraction(d, g_dev, g, thr, salt, now, n_crashed);
  }
  bool impair_fraction(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t* loss_col,
                       uint8_t* delay_col, uint32_t thr, uint32_t salt, uint32_t loss, uint32_t delay,
                       uint32_t counts[2]) override {
    wait();
    return in_->impair_fraction(d, g_dev, g, loss_col, delay_col, thr, salt, loss, delay, counts);
  }
  bool recount(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now, uint32_t first,
               uint32_t count, GsRecount* out) override {
    wait();
    return in_->recount(d, g_dev, g, now, first, count, out);
  }
  bool state_hash(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now,
                  uint64_t out[4]) override {
    wait();
    return in_->state_hash(d, g_dev, g, now, out);
  }
  bool reap_rows(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t now, uint32_t reconnect_ticks,
                 uint32_t tombstone_ticks, bool log_events, uint32_t counts[2]) override {
    wait();
    return in_->reap_rows(d, g_dev, g, now, reconnect_ticks, tombstone_ticks, log_events, counts);
  }
  bool and_columns(const GsDev& d, const GsGlobals& g, uint32_t keep, uint32_t first, uint32_t count) override {
    return in_->and_columns(d, g, keep, first, count);
  }
  bool sync() override { return wait(), in_->sync(); }
  const char* last_error() const override { return in_->last_error(); }
  uint64_t total_launches() const override { return in_->total_launches(); }

 private:
  static void wait() { ++g_waits; }
  GsBackend* in_;
};

}  // namespace

GsBackend* gs_make_counting_backend(int device, char* err, size_t err_cap) {
  GsBackend* in = gs_make_hostemu_backend(device, err, err_cap);
  return in ? new CountingBackend(in) : nullptr;
}
