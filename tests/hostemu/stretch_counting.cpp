// stretch_counting.cpp — TEST INFRASTRUCTURE ONLY.  Never linked into libgsim.so.
//
// The counting backend (counting_backend.cpp, compiled into this translation unit) with one more call that
// waits for the device on CUDA: a tick stretch (GsBackend::run_tick_stretch).  On CUDA it is one submission
// and one readback, so it counts one wait and one chunk of single ticks, whatever it runs.  The host emulation
// underneath runs GsBackend's default (one tick at a time, then the quiet probe) without being counted again.
// Built with gs_api.cpp and the host emulation into tests/hostemu/libgsim_hostemu_counted.so by
// `__graft_entry__.build()`; the last stretch is recorded so that tests/test_tick_stretch_cpu.py can check
// where it stopped.
#include "counting_backend.cpp"

// the last run_tick_stretch of the process: {t0, nticks, floor, depth, ticks run, GS_Q_LAST_ACTIVE, quiet}
static uint32_t g_stretch[7];
extern "C" void gsim_hostemu_last_stretch(uint32_t out[7]) {
  for (int k = 0; k < 7; ++k) out[k] = g_stretch[k];
}

namespace {

class StretchCountingBackend : public CountingBackend {
 public:
  explicit StretchCountingBackend(GsBackend* emu) : CountingBackend(emu), emu_(emu) {}
  bool run_tick_stretch(const GsDev& d, const GsGlobals* g_dev, const GsGlobals& g, uint32_t t0, uint32_t nticks,
                        uint32_t floor, bool counts, double* kernel_ms, GsStretch* out) override {
    ++g_waits;  // the ticks, the quiet probe and their readback are one submission
    ++g_tick_chunks;
    if (!emu_->run_tick_stretch(d, g_dev, g, t0, nticks, floor, counts, kernel_ms, out)) return false;
    const uint32_t rec[7] = {t0, nticks, floor, g.ring_mask + 1u, out->ran, out->last_active, out->quiet};
    for (int k = 0; k < 7; ++k) g_stretch[k] = rec[k];
    return true;
  }

 private:
  GsBackend* emu_;  // the host emulation (owned by CountingBackend)
};

}  // namespace

GsBackend* gs_make_stretch_counting_backend(int device, char* err, size_t err_cap) {
  GsBackend* emu = gs_make_hostemu_backend(device, err, err_cap);
  return emu ? new StretchCountingBackend(emu) : nullptr;
}
