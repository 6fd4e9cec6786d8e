// TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT.
//
// The host emulation of the thread-per-stream HF coefficient kernel (emu_backend.cc) with a SIMT model for every number
// of streams per warp the device launch can use (K = 4, 8, 16, 32; launch_decode_hf_lanes): make -f lanes_k.mk.
// Every loop trip of a stream is recorded (which kind of symbol it decodes), and after each decode_hf() the trips of K
// consecutive streams of the launch order are lined up the way a warp of the device runs them. tools/lanes_model.py and
// tests/test_hf_packing.py read the result through jxle_lane_k_stats().
#include <algorithm>
#include <cstdint>
#include <mutex>
#include <vector>

#include "cuda_shim.h"

namespace {
void lanes_k_trip(bool is_coefficient);
}  // namespace
// hf_lanes.cuh's loop trips report here; the hook is undefined again for emu_backend.cc to define its own (its include of
// hf_lanes.cuh is then a no-op), and lanes_k_trip() passes every trip on to it
#define JXLB_LANE_TRIP(c) lanes_k_trip(c)
#include "../../jxl_oxide_b200/csrc/kernels/hf_lanes.cuh"
#undef JXLB_LANE_TRIP
#include "emu_backend.cc"

namespace {
constexpr int kKs[4] = {4, 8, 16, 32};
// per K, accumulated over all decode_hf() calls since the last reset: [0] streams, [1] symbols (= lane trips), [2] warp
// trips (sum over warps of the longest lane), [3] warp trips with at least one lane on a non-zero count, [4] warp trips
// with at least one lane on a coefficient, [5] warps
uint64_t g_k_stats[4][6];
std::mutex g_k_mutex;

// the streams of the decode_hf() call running on this thread, in launch order
struct StreamTrips {
  const std::vector<unsigned char>* first = nullptr;  // emu_backend.cc's trip log of launch-order stream 0
  std::vector<std::vector<unsigned char>> trips;
};
thread_local StreamTrips* g_streams = nullptr;

void lanes_k_trip(bool is_coefficient) {
  emu_trip(is_coefficient);  // emu_backend.cc's own 32-stream model
  if (!g_streams || !g_trip_log) return;
  // emu_backend.cc logs launch-order stream i into the i-th element of one vector: the distance from stream 0's log
  // is the stream's index (stream 0 always decodes at least one symbol: every group holds a varblock)
  if (!g_streams->first) g_streams->first = g_trip_log;
  const size_t i = size_t(g_trip_log - g_streams->first);
  if (g_streams->trips.size() <= i) g_streams->trips.resize(i + 1);
  g_streams->trips[i].push_back(is_coefficient ? 1 : 0);
}
}  // namespace

extern "C" void jxle_lane_k_stats(int k, uint64_t out[6], int reset) {
  std::lock_guard<std::mutex> lock(g_k_mutex);
  for (int j = 0; j < 4; ++j)
    if (kKs[j] == k)
      for (int i = 0; i < 6; ++i) {
        out[i] = g_k_stats[j][i];
        if (reset) g_k_stats[j][i] = 0;
      }
}

namespace jxlo {

class LanesKBackend : public EmuBackend {
 public:
  using EmuBackend::EmuBackend;
  void decode_hf(VarDctState& st, std::vector<HfGroupJob>& jobs) override {
    StreamTrips rec;
    g_streams = &rec;
    try {
      EmuBackend::decode_hf(st, jobs);
    } catch (...) {
      g_streams = nullptr;
      throw;
    }
    g_streams = nullptr;
    rec.trips.resize(std::max(rec.trips.size(), jobs.size()));
    std::lock_guard<std::mutex> lock(g_k_mutex);
    for (int j = 0; j < 4; ++j) {
      const size_t k = size_t(kKs[j]);
      uint64_t* s = g_k_stats[j];
      for (size_t w0 = 0; w0 < rec.trips.size(); w0 += k) {
        const size_t w1 = std::min(rec.trips.size(), w0 + k);
        size_t longest = 0;
        for (size_t i = w0; i < w1; ++i) longest = std::max(longest, rec.trips[i].size()), s[1] += rec.trips[i].size();
        for (size_t t = 0; t < longest; ++t) {
          bool any_header = false, any_coeff = false;
          for (size_t i = w0; i < w1; ++i)
            if (t < rec.trips[i].size()) (rec.trips[i][t] ? any_coeff : any_header) = true;
          s[3] += any_header, s[4] += any_coeff;
        }
        s[2] += longest, ++s[5];
      }
      s[0] += rec.trips.size();
    }
  }
};

OracleBackend* make_lanes_k_backend(int threads) { return new LanesKBackend(threads); }

}  // namespace jxlo
