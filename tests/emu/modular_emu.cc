// TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT.
//
// Host emulation of the Modular stream kernel (kernels/modular_lanes.cuh). The oracle backend is reused for
// everything else; decode_modular() builds the job, channel and plan tables the CUDA backend uploads
// (cuda_backend.cu: decode_modular, with the whole-tree plans of kernels/modular_plan.cuh) over host memory and runs
// decode_stream_channels() -- the code of the kernel's warp -- with one lane that does every column of the weighted
// predictor's row prologues. tests/test_emu_modular.py compares samples, end positions and pixels with the oracle.
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
// after a range trip, [3] single-leaf channels
std::atomic<uint64_t> g_stats[4];
// > 0: the fast loop reports a range trip on the row where a channel reaches this many samples (tests the fallback,
// which real LF data never takes)
std::atomic<uint64_t> g_force_trip{0};
}  // namespace
#define JXLB_MODULAR_EVENT(k) (++g_stats[k])
#define JXLB_WP_FAST_FORCE_TRIP(samples) \
  ((g_force_trip.load() && (samples) >= g_force_trip.load()) ? 1u : 0u)
#include "../../jxl_oxide_b200/csrc/kernels/modular_lanes.cuh"
#include "../../jxl_oxide_b200/csrc/kernels/modular_plan.cuh"
#include "../../oracle/oracle_backend.h"

namespace {
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

extern "C" void jxlme_stats(uint64_t out[4], int reset) {
  for (int i = 0; i < 4; ++i) out[i] = reset ? g_stats[i].exchange(0) : g_stats[i].load();
}
extern "C" void jxlme_force_trip(uint64_t samples) { g_force_trip = samples; }

namespace jxlo {

class ModularEmuBackend : public OracleBackend {
 public:
  explicit ModularEmuBackend(int threads) : OracleBackend(threads) {}
  void set_codestream(const uint8_t* data, size_t size) override {
    OracleBackend::set_codestream(data, size);
    storage_.assign((size + 64 + 7) / 8 + 1, 0);  // zero padded like the device copy
    std::memcpy(storage_.data(), data, size);
  }
  void decode_modular(std::vector<ModularStreamJob>& jobs) override {
    for (ModularStreamJob& j : jobs) decode_one(j);
  }

 private:
  void decode_one(ModularStreamJob& j);
  std::vector<uint64_t> storage_;
};

void ModularEmuBackend::decode_one(ModularStreamJob& j) {
  const EntropyCode& c = j.tree->code;
  DevModularJob d;
  std::memset(&d, 0, sizeof(d));
  std::vector<uint32_t> cfg;
  for (const HybridUintConfig& h : c.configs) cfg.push_back(h.packed());
  std::vector<uint32_t> meta;
  for (const PrefixMeta& m : c.prefix_meta) {
    meta.push_back(m.table_offset);
    meta.push_back(m.root_bits);
  }
  d.code.cluster_map = c.cluster_map.data();
  d.code.configs = cfg.data();
  d.code.log_alphabet_size = c.log_alphabet_size;
  d.code.use_prefix = c.use_prefix ? 1 : 0;
  d.code.num_clusters = c.num_clusters;
  d.code.cluster_map_size = uint32_t(c.cluster_map.size());
  d.code.prefix_table_size = uint32_t(c.prefix_table.size());
  d.code.prefix = c.prefix_table.data();
  d.code.prefix_meta = meta.data();
  d.code.ans = c.ans_table.data();
  d.code.lz77_enabled = c.lz77_enabled ? 1 : 0;
  d.code.lz77_min_symbol = c.lz77_min_symbol;
  d.code.lz77_min_length = c.lz77_min_length;
  d.code.lz_len_conf = c.lz_len_conf.packed();
  d.code.lz_dist_cluster = c.cluster_map.empty() ? 0 : c.cluster_map.back();
  d.bit_pos = j.bit_pos;
  d.bit_limit = j.bit_limit;
  const WpHeader& w = j.wp;
  const uint32_t wpv[11] = {w.p1, w.p2, w.p3a, w.p3b, w.p3c, w.p3d, w.p3e, w.w[0], w.w[1], w.w[2], w.w[3]};
  std::memcpy(d.wp, wpv, sizeof(wpv));
  d.stream_index = j.stream_index;
  d.num_channels = uint32_t(j.channels.size());
  std::vector<DevChannel> chans;
  std::vector<DevChannelPlan> plans;
  std::vector<uint16_t> luts;
  uint32_t max_w = 0;
  uint64_t samples = 0;
  for (size_t ci = 0; ci < j.channels.size(); ++ci) {
    const ModularChannelTarget& t = j.channels[ci];
    int32_t* ptr = nullptr;
    uint32_t stride = 0;
    if (t.view.w && t.view.h) {
      Plane& p = plane(t.view.plane);
      ptr = p.i32() + size_t(t.view.y0) * p.w + t.view.x0;
      stride = p.w;
    }
    chans.push_back({ptr, stride, t.view.w, t.view.h, t.hshift, t.vshift});
    max_w = std::max(max_w, t.view.w);
    samples += uint64_t(t.view.w) * t.view.h;
    int nprev = 0;
    for (size_t pj = 0; pj < ci; ++pj) {
      const ModularChannelTarget& q = j.channels[pj];
      if (q.view.w && q.view.h && q.view.w == t.view.w && q.view.h == t.view.h && q.hshift == t.hshift && q.vshift == t.vshift) ++nprev;
    }
    plans.push_back(jxlb::build_channel_plan(*j.tree, uint32_t(ci), j.stream_index, std::min(nprev, 16), &luts));
  }
  luts.push_back(0);
  luts.push_back(0);
  d.dist_multiplier = max_w;
  d.use_wp = jxlb::tree_uses_wp(*j.tree) ? 1 : 0;
  d.tree = j.tree->nodes.data();
  d.num_tree_nodes = uint32_t(j.tree->nodes.size());
  d.luts = luts.data();
  d.lut_total = uint32_t(luts.size() - 2);
  std::vector<uint32_t> window(d.code.lz77_enabled ? size_t(std::min<uint64_t>(1u << 20, std::max<uint64_t>(samples, 1))) : 1);
  d.lz_window = window.data();
  uint32_t div[65];
  for (uint32_t i = 0; i < 65; ++i) div[i] = i ? (1u << 24) / i : 0;
  // 16-byte aligned like the shared-memory arrays (accessed as uint4 / int4)
  std::vector<int4> wp_rows(std::max<uint32_t>(max_w, 1) * 5 / 4 + 1), rows_b(std::max<uint32_t>(max_w, 1) * 5 / 4 + 1);
  std::vector<int4> pro(kFastChunk * 4);
  std::vector<uint4> leaves(kFastMaxLeaves);
  CodeView cv;
  cv.configs = cfg.data();
  cv.ans = d.code.ans;
  cv.prefix = d.code.prefix;
  cv.prefix_meta = meta.data();
  cv.log_alphabet_size = d.code.log_alphabet_size;
  cv.use_prefix = d.code.use_prefix;
  StreamState s;
  s.br.init(reinterpret_cast<const uint8_t*>(storage_.data()), d.bit_pos, d.bit_limit);
  s.ans_state = d.code.use_prefix ? 0x130000u : s.br.read(32);
  s.window = d.lz_window;
  s.lz_to_copy = s.lz_copy_pos = s.lz_decoded = 0;
  s.err = kDevOk;
  const WpFastScratch fs = {pro.data(), leaves.data(), reinterpret_cast<int32_t*>(rows_b.data())};
  decode_stream_channels(HostWarp{}, d, cv, d.tree, d.luts, chans.data(), plans.data(), reinterpret_cast<int32_t*>(wp_rows.data()),
                         div, fs, s);
  ++g_stats[0];
  if (s.err == kDevOverrun) jxlb::fail(jxlb::kErrBitstream, "modular stream reads past the end of its section");
  if (s.err != kDevOk) jxlb::fail(jxlb::kErrBitstream, "invalid modular stream");
  j.end_bit = size_t(s.br.pos());
}

OracleBackend* make_modular_emu_backend(int threads) { return new ModularEmuBackend(threads); }

}  // namespace jxlo
