// TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT.
//
// Host emulation of the thread-per-stream HF coefficient kernel (kernels/hf_lanes.cuh). The oracle backend
// is reused for everything else; decode_hf() builds its DevFrame, DevHfParams and launch order with the CUDA
// backend's own code (launch_tables.cc), over host memory and the same natural-order table, and then runs
// hf_lane_decode() -- the very function every device thread runs -- once per stream, with the interleaved
// non-zero-row layout of a 32-thread CTA. tests/test_emu_lanes.py compares the resulting coefficient planes,
// end positions and final pixels with the plain oracle.
#include <algorithm>
#include <cstring>

#include "cuda_shim.h"

#include <vector>
// SIMT model: every loop trip of hf_lane_decode() reports whether it decodes a coefficient (1) or a block's non-zero
// count (0); decode_hf() below lines the trips of 32 consecutive streams up the way a warp would execute them.
namespace {
thread_local std::vector<unsigned char>* g_trip_log = nullptr;
inline void emu_trip(bool is_coefficient) {
  if (g_trip_log) g_trip_log->push_back(is_coefficient ? 1 : 0);
}
}  // namespace
#define JXLB_LANE_TRIP(c) emu_trip(c)
#include "../../jxl_oxide_b200/csrc/kernels/hf_lanes.cuh"
#include "../../jxl_oxide_b200/csrc/kernels/filter_strip.cuh"
#include "../../oracle/oracle_backend.h"
#include "../../jxl_oxide_b200/csrc/host/planner.h"
#include "host_sink.h"

namespace {
// strip filter emulation: [0] frames that took the path, [1] pixels compared, [2] pixels that differ from the oracle's stages
std::atomic<uint64_t> g_strip_stats[3];
std::atomic<uint64_t> g_hf_streams{0};
// accumulated over all decode_hf() calls since the last reset:
//   [0] streams, [1] symbols (= lane trips), [2] warp trips (sum over warps of the longest lane), [3] warp trips with
//   at least one lane on a non-zero count (the divergent block walk runs), [4] warp trips with at least one lane on a
//   coefficient, [5] warps
uint64_t g_lane_stats[6] = {0, 0, 0, 0, 0, 0};
}
extern "C" void jxle_lane_stats(uint64_t out[6], int reset) {
  for (int i = 0; i < 6; ++i) out[i] = g_lane_stats[i];
  if (reset)
    for (int i = 0; i < 6; ++i) g_lane_stats[i] = 0;
}

// how many HF streams went through hf_lane_decode() so far (the test checks that the emulated path really ran)
extern "C" uint64_t jxle_hf_streams() { return g_hf_streams.load(); }

// Known-answer check of the device bit reader (common.cuh: word-ahead, 64-bit buffer) against the host reader
// (host/bitreader.h) that the planner and the oracle use: random start offsets, random read widths 0..32, peeks,
// and pos() after every step. Returns 0 when every step agreed, otherwise 1 + the index of the first mismatch.
extern "C" uint64_t jxle_bitreader_selftest(uint64_t seed, uint32_t steps) {
  std::vector<uint64_t> store(4096 + 8, 0);
  uint64_t x = seed * 0x9e3779b97f4a7c15ull + 1;
  auto rnd = [&]() {
    x ^= x << 13, x ^= x >> 7, x ^= x << 17;
    return x;
  };
  for (size_t i = 0; i < 4096; ++i) store[i] = rnd();
  const uint8_t* bytes = reinterpret_cast<const uint8_t*>(store.data());
  const uint64_t start = rnd() % 4096;
  jxlb::BitReader host(bytes, 4096 * 8, start);
  jxlb::DevBitReader dev;
  dev.init(bytes, start);
  for (uint32_t i = 0; i < steps; ++i) {
    if (host.pos() + 64 > 4096ull * 8 * 8) break;
    if (dev.pos() != host.pos()) return 1 + i;
    const uint32_t n = uint32_t(rnd() % 33);
    if (rnd() & 1) {
      if (dev.peek(n) != host.peek(n)) return 1 + i;
    }
    if (dev.read(n) != host.read(n)) return 1 + i;
  }
  return 0;
}

// cv_read_uint (stream_common.cuh) against the closed form of the hybrid integer coding (jxl-coding/src/lib.rs:572-605):
// token < split -> token; otherwise n extra bits follow, value = (((1 << msb | mid) << n | extra) << lsb) | low.
extern "C" uint64_t jxle_hybrid_uint_selftest(uint64_t seed, uint32_t steps) {
  std::vector<uint64_t> store(1024 + 8, 0);
  uint64_t x = seed * 0x9e3779b97f4a7c15ull + 7;
  auto rnd = [&]() {
    x ^= x << 13, x ^= x >> 7, x ^= x << 17;
    return x;
  };
  for (size_t i = 0; i < 1024; ++i) store[i] = rnd();
  const uint8_t* bytes = reinterpret_cast<const uint8_t*>(store.data());
  for (uint32_t i = 0; i < steps; ++i) {
    const uint32_t split_exponent = uint32_t(rnd() % 9);           // log_alphabet_size <= 8
    const uint32_t msb = split_exponent ? uint32_t(rnd() % (split_exponent + 1)) : 0;
    const uint32_t lsb = uint32_t(rnd() % (split_exponent - msb + 1));
    const uint32_t cfg = split_exponent | msb << 8 | lsb << 16;
    const uint32_t token = uint32_t(rnd() % 256);
    const uint64_t pos = rnd() % (1024 * 64 - 128);
    jxlb::BitReader host(bytes, 1024 * 8, pos);
    jxlb::DevBitReader dev;
    dev.init(bytes, pos);
    const uint32_t got = jxlb::cv_read_uint(dev, cfg, token);
    uint32_t want;
    const uint32_t split = 1u << split_exponent;
    if (token < split) {
      want = token;
    } else {
      const uint32_t in_token = msb + lsb;
      const uint32_t n = (split_exponent - in_token + ((token - split) >> in_token)) & 31;
      const uint32_t low = token & ((1u << lsb) - 1);
      const uint32_t mid = (token >> lsb) & ((1u << msb) - 1);
      const uint64_t extra = host.read(n);
      want = uint32_t(((((uint64_t(1) << msb | mid) << n) | extra) << lsb) | low);
    }
    if (got != want || dev.pos() != host.pos()) return 1 + i;
  }
  return 0;
}

// The packed records of the thread-per-stream HF decoder read back to what they were packed from: the transform-type
// record of every type against kTransformInfo, and the varblock record at the largest values its fields can take
// (type 26; context offset hf_idx * lf_idx_mul + lf_idx with 15 quant-field and 3 x 15 LF thresholds; x, y inside a
// 1024-sample group). Returns 0 when all agree, otherwise 1 + the type that differs, or 100 + which record check failed.
extern "C" int jxle_hf_record_check() {
  using namespace jxlb;
  for (uint32_t t = 0; t < kNumTransformTypes; ++t) {
    const HfTinfo ti = hf_unpack_tinfo(hf_pack_tinfo(t));
    const TransformTypeInfo& want = kTransformInfo[t];
    if (ti.w8 != want.w8 || (1u << ti.num_blocks_log) != uint32_t(want.w8) * want.h8 || ti.order_id != want.order_id ||
        ti.transpose != want.transpose)
      return int(1 + t);
  }
  const uint32_t max_offset = 15u * (16u * 16u * 16u) + (16u * 16u * 16u - 1u);
  const uint32_t max_type = kNumTransformTypes - 1, max_xy = 1024 / 8 - 1;
  const uint2 rec = hf_block_rec(max_type | max_offset << 8, max_xy, max_xy);
  if (rec.x == kHfNoBlock) return 100;
  if ((rec.x & 0xff) != max_type || (rec.x >> 8) != max_offset) return 101;
  if ((rec.y & 0xffff) != max_xy || (rec.y >> 16) != max_xy) return 102;
  return 0;
}

namespace jxlo {

class EmuBackend : public OracleBackend {
 public:
  explicit EmuBackend(int threads) : OracleBackend(threads), natural_orders_(natural_order_table(natural_offset_)) {}
  void set_codestream(const uint8_t* data, size_t size) override {
    OracleBackend::set_codestream(data, size);
    // the device copy is zero padded (the word-ahead bit reader touches up to 3 words past the last bit)
    storage_.assign((size + 64 + 7) / 8 + 1, 0);
    std::memcpy(storage_.data(), data, size);
  }
  void decode_hf(VarDctState& st, std::vector<HfGroupJob>& jobs) override;
  bool filters_colour_fused(const View v[3], const RestorationFilter& rf, const View& sigma, bool sigma_is_constant,
                            const ColorParams* colour) override;

 private:
  std::vector<uint64_t> storage_;  // 8-byte aligned
  uint32_t natural_offset_[13];
  std::vector<uint32_t> natural_orders_;  // the device-resident natural-order table
};

void EmuBackend::decode_hf(VarDctState& st, std::vector<HfGroupJob>& jobs) {
  if (jobs.empty()) return;
  const uint8_t* cs = reinterpret_cast<const uint8_t*>(storage_.data());
  const DevFrame f = make_dev_frame(st, [this](int id) -> void* { return id < 0 ? nullptr : plane(id).data.data(); });
  const uint32_t pass = jobs[0].pass_idx;
  HostTableSink sink;
  const DevHfParams p = build_hf_params(st, pass, sink, natural_orders_.data(), natural_offset_);
  if (std::getenv("JXLE_TRACE")) std::fprintf(stderr, "[emu] decode_hf pass %u: %zu streams, %s, %u clusters, %u presets, subsampled %d\n", pass, jobs.size(), p.code.use_prefix ? "prefix" : "ANS", p.code.num_clusters, st.hfg->num_hf_presets, int(st.subsampled));

  // "shared memory" tables of one CTA
  uint8_t ctx[128] = {0};
  for (int i = 0; i < 63; ++i) {
    ctx[i] = hftab::kCoeffFreqContext[i];
    ctx[64 + i] = hftab::kCoeffNumNonzeroContext[i];
  }
  uint32_t tinfo[27];
  for (uint32_t t = 0; t < 27; ++t) tinfo[t] = hf_pack_tinfo(t);
  HfLaneTables T;
  T.tinfo = tinfo;
  T.order_offset = p.order_offset;
  T.ctx = ctx;
  T.cfg = p.code.configs;
  T.bctx = p.block_ctx_map;
  T.cmap = p.code.cluster_map;
  T.cmap_stride = 495 * p.num_block_clusters;
  T.cv.configs = p.code.configs;
  T.cv.ans = p.code.ans;
  T.cv.prefix = p.code.prefix;
  T.cv.prefix_meta = p.code.prefix_meta;
  T.cv.log_alphabet_size = p.code.log_alphabet_size;
  T.cv.use_prefix = p.code.use_prefix;

  const std::vector<uint32_t> perm = hf_launch_order(jobs, true);
  // the pre-pass kernel: one "thread" per 8x8 cell
  std::vector<uint32_t> blk_ctx(size_t(f.bw) * f.bh);
  for (uint32_t by = 0; by < f.bh; ++by)
    for (uint32_t bx = 0; bx < f.bw; ++bx)
      blk_ctx[size_t(by) * f.bw + bx] = f.subsampled ? hf_block_ctx_cell<true>(f, p, bx, by) : hf_block_ctx_cell<false>(f, p, bx, by);
  constexpr uint32_t kThreads = 32;
  std::vector<uint8_t> nz(96 * kThreads, 0xee);
  std::vector<std::vector<unsigned char>> trips(perm.size());
  for (size_t i = 0; i < perm.size(); ++i) {
    g_trip_log = &trips[i];
    HfGroupJob& job = jobs[perm[i]];
    DevHfJob dj{job.bit_pos, job.bit_limit, job.group_idx};
    uint64_t end = 0;
    int status = 0;
    const uint32_t tid = uint32_t(i % kThreads);
    if (f.subsampled) hf_lane_decode<true>(cs, f, p, T, blk_ctx.data(), dj, nz.data() + tid, kThreads, pass == 0 ? 1 : 0, &end, &status);
    else hf_lane_decode<false>(cs, f, p, T, blk_ctx.data(), dj, nz.data() + tid, kThreads, pass == 0 ? 1 : 0, &end, &status);
    if (status != kDevOk)
      throw Error(status == kDevOverrun ? kErrEof : (status == kDevUnsupported ? kErrUnsupported : kErrDeviceDecode),
                  "emulated HF lane: status " + std::to_string(status) + " in group " + std::to_string(job.group_idx));
    job.end_bit = size_t(end);
    ++g_hf_streams;
  }
  g_trip_log = nullptr;
  for (size_t w0 = 0; w0 < trips.size(); w0 += 32) {  // one warp = 32 consecutive streams of the launch order
    const size_t w1 = std::min(trips.size(), w0 + 32);
    size_t longest = 0;
    for (size_t i = w0; i < w1; ++i) longest = std::max(longest, trips[i].size()), g_lane_stats[1] += trips[i].size();
    for (size_t t = 0; t < longest; ++t) {
      bool any_header = false, any_coeff = false;
      for (size_t i = w0; i < w1; ++i)
        if (t < trips[i].size()) (trips[i][t] ? any_coeff : any_header) = true;
      g_lane_stats[3] += any_header, g_lane_stats[4] += any_coeff;
    }
    g_lane_stats[2] += longest, ++g_lane_stats[5];
  }
  g_lane_stats[0] += trips.size();
}

OracleBackend* make_emu_backend(int threads) { return new EmuBackend(threads); }

}  // namespace jxlo

// ---- the column-strip filter kernel (kernels/filter_strip.cuh) on the host ------------------------------------------
// Every CTA of the launch is run thread by thread, phase by phase (the phases are separated by __syncthreads() on the
// device, so running all threads of a phase before the next one is an admissible schedule); the window is filled the way
// the TMA copy fills it. The oracle's own stages then process the planes in place, the interior rectangle is compared
// pixel for pixel (bit patterns) and replaced by the emulated kernel's output.
extern "C" void jxle_strip_stats(uint64_t out[3], int reset) {
  for (int i = 0; i < 3; ++i) {
    out[i] = g_strip_stats[i].load();
    if (reset) g_strip_stats[i].store(0);
  }
}

// Host-side check of the filter launch geometry (launch_filters_fused): the strip kernel's rectangle is the union of the general
// kernel's interior tiles, and the 1-D border grid enumerates every other tile exactly once. Returns 0 when the frame size
// checks out, otherwise a code that says what is wrong.
extern "C" int jxle_filter_geometry_check(int width, int height) {
  using namespace jxlb::fstrip;
  const StripRect r = strip_rect(width, height);
  const int nbx = (width + 31) / 32, nby = (height + 31) / 32;
  if (r.x1 <= r.x0 || r.y1 <= r.y0) return 0;  // no strip launch: the general kernel takes the whole frame
  if (r.x0 != 32 || r.y0 != 32 || r.x1 % 32 || r.y1 % 32) return 1;
  if (r.x1 + kM > width || r.y1 + kM > height) return 2;  // every pixel of the rectangle is a margin away from the border
  const int bx_last = r.x1 / 32 - 1, by_last = r.y1 / 32 - 1;
  // interior tiles are exactly those whose 40 x 40 window lies inside the image
  for (int ty = 0; ty < nby; ++ty)
    for (int tx = 0; tx < nbx; ++tx) {
      const bool inside = tx * 32 - 4 >= 0 && ty * 32 - 4 >= 0 && tx * 32 + 36 <= width && ty * 32 + 36 <= height;
      const bool in_rect = tx >= 1 && tx <= bx_last && ty >= 1 && ty <= by_last;
      if (inside != in_rect) return 3;
    }
  std::vector<int> seen(size_t(nbx) * nby, 0);
  const int n_border = nbx * nby - bx_last * by_last;
  for (int i = 0; i < n_border; ++i) {
    int tx = -1, ty = -1;
    border_tile_index(nbx, nby, bx_last, by_last, i, tx, ty);
    if (tx < 0 || tx >= nbx || ty < 0 || ty >= nby) return 4;
    if (tx >= 1 && tx <= bx_last && ty >= 1 && ty <= by_last) return 5;  // an interior tile in the border grid
    if (seen[size_t(ty) * nbx + tx]++) return 6;                            // twice
  }
  for (int ty = 0; ty < nby; ++ty)
    for (int tx = 0; tx < nbx; ++tx) {
      const bool in_rect = tx >= 1 && tx <= bx_last && ty >= 1 && ty <= by_last;
      if (!in_rect && !seen[size_t(ty) * nbx + tx]) return 7;  // a border tile nobody takes
    }
  // strip tiles: origins inside the image, 16-byte aligned when the width is a multiple of four, outputs cover the rectangle
  const int ntx = (r.x1 - r.x0 + kTX - 1) / kTX, nty = (r.y1 - r.y0 + kTY - 1) / kTY;
  std::vector<int> cover(size_t(r.x1 - r.x0) * (r.y1 - r.y0), 0);
  for (int ty = 0; ty < nty; ++ty)
    for (int tx = 0; tx < ntx; ++tx) {
      const StripGeom g = strip_geom(width, height, r.x0, r.y0, r.x1, r.y1, tx, ty);
      if (g.gx0 < 0 || g.gy0 < 0 || g.gx0 + kWX > width || g.gy0 + kWY > height) return 8;
      if ((width & 3) == 0 && (g.gx0 & 3)) return 9;
      for (int y = g.gy0 + kM; y < g.gy0 + kWY - kM; ++y)
        for (int x = g.gx0 + kM; x < g.gx0 + kWX - kM; ++x)
          if (x >= r.x0 && x < r.x1 && y >= r.y0 && y < r.y1) cover[size_t(y - r.y0) * (r.x1 - r.x0) + (x - r.x0)] = 1;
    }
  for (int c : cover)
    if (!c) return 10;
  return 0;
}

// The kernels' sRGB transfer function (pixel_math.cuh) on n samples, so that a test can bound its distance from the exact curve
extern "C" void jxle_linear_to_srgb(const float* in, float* out, size_t n) {
  for (size_t i = 0; i < n; ++i) out[i] = jxlb::linear_to_srgb(in[i], jxlb::kSrgbPow);
}

namespace jxlo {

bool EmuBackend::filters_colour_fused(const View v[3], const RestorationFilter& rf, const View& sigma, bool sigma_is_constant,
                                      const ColorParams* colour) {
  using namespace jxlb::fstrip;
  const int width = int(v[0].w), height = int(v[0].h);
  const StripRect r = strip_rect(width, height);
  const bool colour_ok = !colour || (!colour->second_stage && colour->gamma == 0.0f);
  if (std::getenv("JXLE_TRACE"))
    std::fprintf(stderr, "[emu] filters: %d x %d, gab %d, epf iters %u, colour %d\n", width, height, int(rf.gab_enabled), rf.epf.iters, int(colour != nullptr));
  if (!rf.gab_enabled || (rf.epf.iters != 1 && rf.epf.iters != 2) || r.x1 <= r.x0 || r.y1 <= r.y0 || !colour_ok) return false;
  for (int c = 0; c < 3; ++c)
    if (v[c].x0 != 0 || v[c].y0 != 0 || int(v[c].w) != width || int(v[c].h) != height) return false;

  const DevFusedFilterParams p = fused_filter_params(rf, sigma_is_constant ? nullptr : plane(sigma.plane).f32(),
                                                     sigma_is_constant ? 0 : plane(sigma.plane).w, colour);
  float gw[3];
  strip_gab_norm(p, gw);

  const float* in[3];
  uint32_t in_stride[3], out_stride[3];
  std::vector<std::vector<float>> out_store(3);
  float* out[3];
  for (int c = 0; c < 3; ++c) {
    Plane& pl_c = plane(v[c].plane);
    in[c] = pl_c.f32();
    in_stride[c] = pl_c.w;
    out_store[c].assign(size_t(width) * height, 0.0f);
    out[c] = out_store[c].data();
    out_stride[c] = uint32_t(width);
  }
  const int ntx = (r.x1 - r.x0 + kTX - 1) / kTX, nty = (r.y1 - r.y0 + kTY - 1) / kTY;
  parallel_for(size_t(ntx) * nty, [&](size_t t) {
    const int tx = int(t % ntx), ty = int(t / ntx);
    const StripGeom g = strip_geom(width, height, r.x0, r.y0, r.x1, r.y1, tx, ty);
    std::vector<float> s(kSmemFloats, std::nanf(""));
    for (int c = 0; c < 3; ++c)  // the TMA box: kWX x kWY cells at (gx0, gy0)
      for (int y = 0; y < kWY; ++y)
        for (int x = 0; x < kWX; ++x) s[c * kPlane + y * kWX + x] = in[c][size_t(g.gy0 + y) * in_stride[c] + g.gx0 + x];
    for (int tid = 0; tid < kThreads; ++tid) phase_sigma(tid, s.data(), g, p);
    for (int tid = 0; tid < kThreads; ++tid) phase_gab(tid, s.data(), p, gw);
    for (int tid = 0; tid < kThreads; ++tid) phase_dist1(tid, s.data(), p);
    const int tf = strip_tf_of(p);
    for (int tid = 0; tid < kThreads; ++tid) {
      if (p.epf_iters == 1) {
        if (tf == 1) phase_apply1<true, 1>(tid, s.data(), g, p, out, out_stride);
        else if (tf == 2) phase_apply1<true, 2>(tid, s.data(), g, p, out, out_stride);
        else phase_apply1<true, 0>(tid, s.data(), g, p, out, out_stride);
      } else {
        phase_apply1<false, 0>(tid, s.data(), g, p, out, out_stride);
      }
    }
    if (p.epf_iters == 2)
      for (int tid = 0; tid < kThreads; ++tid) {
        if (tf == 1) phase_apply2<1>(tid, s.data(), g, p, out, out_stride);
        else if (tf == 2) phase_apply2<2>(tid, s.data(), g, p, out, out_stride);
        else phase_apply2<0>(tid, s.data(), g, p, out, out_stride);
      }
  });

  OracleBackend::gaborish(v, rf.gab_weights);
  OracleBackend::epf(v, sigma, rf.epf, sigma_is_constant);
  if (colour) OracleBackend::xyb_to_rgb(v, *colour);
  uint64_t compared = 0, differ = 0;
  for (int c = 0; c < 3; ++c) {
    Plane& pl_c = plane(v[c].plane);
    for (int y = r.y0; y < r.y1; ++y)
      for (int x = r.x0; x < r.x1; ++x) {
        uint32_t& want = pl_c.data[size_t(y) * pl_c.w + x];
        uint32_t got;
        std::memcpy(&got, &out[c][size_t(y) * width + x], 4);
        ++compared;
        if (got != want) {
          if (!differ && std::getenv("JXLE_TRACE")) std::fprintf(stderr, "[emu] strip filter: first difference at c=%d x=%d y=%d: %08x vs %08x\n", c, x, y, got, want);
          ++differ;
        }
        want = got;
      }
  }
  g_strip_stats[0] += 1, g_strip_stats[1] += compared, g_strip_stats[2] += differ;
  return true;
}

}  // namespace jxlo
