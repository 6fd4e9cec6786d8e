// TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT.
//
// Host emulation of the Modular stream kernel (kernels/modular_lanes.cuh). The oracle backend is reused for
// everything else; decode_modular() builds its launch with the CUDA backend's own code (launch_tables.cc:
// build_modular_launch: compacted, renumbered and shared channel subtrees, or the whole-tree plans past the node limit)
// over host memory and runs decode_stream_channels() -- the code of the kernel's warp -- with one lane that does every
// column of the weighted predictor's row prologues; like the device, it enables the fast loop only in a launch that
// stages every table. tests/test_emu_modular.py compares samples, end positions and pixels with the oracle.
#include <atomic>
#include <cstring>
#include <vector>

#include "cuda_shim.h"

#include <cstdlib>
#include <type_traits>
// device-side names the per-stream code uses beyond cuda_shim.h
static inline int64_t min(int64_t a, int64_t b) { return a < b ? a : b; }
static inline int64_t max(int64_t a, int64_t b) { return a > b ? a : b; }
#define __noinline__

namespace {
// [0] streams decoded, [1] channels that ran the weighted-predictor fast loop, [2] of those, channels decoded again
// after a range trip, [3] single-leaf channels, [4] jobs built with compacted channel subtrees, [5] jobs built with the
// whole-tree plans, [6] channels that share an earlier channel's subtree copy, [7] jobs of launches without the fast loop
std::atomic<uint64_t> g_stats[8];
// > 0: the fast loop reports a range trip on the row where a channel reaches this many samples (tests the fallback,
// which real LF data never takes)
std::atomic<uint64_t> g_force_trip{0};
}  // namespace
#define JXLB_MODULAR_EVENT(k) (++g_stats[k])
#define JXLB_WP_FAST_FORCE_TRIP(samples) \
  ((g_force_trip.load() && (samples) >= g_force_trip.load()) ? 1u : 0u)
#include "../../jxl_oxide_b200/csrc/kernels/modular_lanes.cuh"
#include "../../oracle/oracle_backend.h"
#include "host_sink.h"

namespace {
std::atomic<uint64_t> g_max_channel_tree_nodes{jxlb::kMaxChannelTreeNodes};

struct HostWarp {
  static constexpr uint32_t kLanes = 1;
  uint32_t lane = 0;
  void sync() const {}
  template <typename T>
  T bcast(T v) const {
    return v;
  }
  bool all(bool p) const { return p; }
};
}  // namespace

extern "C" void jxlme_stats(uint64_t out[8], int reset) {
  for (int i = 0; i < 8; ++i) out[i] = reset ? g_stats[i].exchange(0) : g_stats[i].load();
}
extern "C" void jxlme_force_trip(uint64_t samples) { g_force_trip = samples; }
// Sets the node limit of a compacted channel subtree and returns the previous one. 0: every job with a channel subtree of
// more than one node is built with the whole-tree plans.
extern "C" uint64_t jxlme_max_channel_tree_nodes(uint64_t n) { return g_max_channel_tree_nodes.exchange(n); }

namespace jxlo {

class ModularEmuBackend : public OracleBackend {
 public:
  explicit ModularEmuBackend(int threads) : OracleBackend(threads) {}
  void set_codestream(const uint8_t* data, size_t size) override {
    OracleBackend::set_codestream(data, size);
    storage_.assign((size + 64 + 7) / 8 + 1, 0);  // zero padded like the device copy
    std::memcpy(storage_.data(), data, size);
  }
  void decode_modular(std::vector<ModularStreamJob>& jobs) override;

 private:
  size_t decode_one(const ModularLaunch& L, size_t i);  // job i of the launch; returns its end position
  std::vector<uint64_t> storage_;
};

void ModularEmuBackend::decode_modular(std::vector<ModularStreamJob>& jobs) {
  HostTableSink sink;
  const ModularLaunch L = build_modular_launch(
      jobs,
      [this](const View& v) {
        DevView d{nullptr, 0, v.w, v.h};
        if (v.w && v.h) {
          Plane& p = plane(v.plane);
          d.ptr = p.i32() + size_t(v.y0) * p.w + v.x0;
          d.stride = p.w;
        }
        return d;
      },
      sink, g_max_channel_tree_nodes.load());
  for (size_t i = 0; i < jobs.size(); ++i) {
    ++g_stats[L.needs[i].whole_tree ? 5 : 4];
    if (!L.all_staged) ++g_stats[7];
    const DevModularJob& d = L.jobs[i];
    const DevChannelPlan* plans = L.plans.data() + d.first_channel;
    for (uint32_t ci = 1; ci < d.num_channels && !L.needs[i].whole_tree; ++ci)
      for (uint32_t pj = 0; pj < ci; ++pj)
        if (plans[pj].root == plans[ci].root) {
          ++g_stats[6];
          break;
        }
    jobs[i].end_bit = decode_one(L, i);
  }
}

size_t ModularEmuBackend::decode_one(const ModularLaunch& L, size_t i) {
  DevModularJob d = L.jobs[i];
  std::vector<uint32_t> window(L.needs[i].lz_window_bytes / 4 + 1);
  d.lz_window = window.data();
  uint32_t div[65];
  for (uint32_t k = 0; k < 65; ++k) div[k] = k ? (1u << 24) / k : 0;
  // 16-byte aligned like the shared-memory arrays (accessed as uint4 / int4)
  std::vector<int4> wp_rows(L.needs[i].wp_scratch_bytes / 16 + 1), rows_b(L.needs[i].wp_scratch_bytes / 16 + 1);
  std::vector<int4> pro(kFastChunk * 4);
  std::vector<uint4> leaves(kFastMaxLeaves);
  CodeView cv;
  cv.configs = d.code.configs;
  cv.ans = d.code.ans;
  cv.prefix = d.code.prefix;
  cv.prefix_meta = d.code.prefix_meta;
  cv.log_alphabet_size = d.code.log_alphabet_size;
  cv.use_prefix = d.code.use_prefix;
  StreamState s;
  s.br.init(reinterpret_cast<const uint8_t*>(storage_.data()), d.bit_pos, d.bit_limit);
  s.ans_state = d.code.use_prefix ? 0x130000u : s.br.read(32);
  s.window = d.lz_window;
  s.lz_to_copy = s.lz_copy_pos = s.lz_decoded = 0;
  s.err = kDevOk;
  // the device enables the fast loop only in a launch that stages every table
  WpFastScratch fs = {nullptr, nullptr, nullptr};
  if (L.all_staged) fs = {pro.data(), leaves.data(), reinterpret_cast<int32_t*>(rows_b.data())};
  decode_stream_channels(HostWarp{}, d, cv, d.tree, d.luts, L.channels.data() + d.first_channel, L.plans.data() + d.first_channel,
                         reinterpret_cast<int32_t*>(wp_rows.data()), div, fs, s);
  ++g_stats[0];
  if (s.err == kDevOverrun) jxlb::fail(jxlb::kErrBitstream, "modular stream reads past the end of its section");
  if (s.err != kDevOk) jxlb::fail(jxlb::kErrBitstream, "invalid modular stream");
  return size_t(s.br.pos());
}

OracleBackend* make_modular_emu_backend(int threads) { return new ModularEmuBackend(threads); }

}  // namespace jxlo
