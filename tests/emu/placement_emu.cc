// TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT.
//
// Host emulation of the varblock placement (kernels/placement.cuh): the warp's steps run lane by lane for 32 lanes, and
// the result is compared with the oracle's serial scan (OracleBackend::build_block_info).
//   * As a backend (JXLO_BACKEND_FACTORY=make_placement_emu_backend): every LF group the planner hands to the oracle's
//     placement is first placed by the emulation on copies of the grids; status and grids are compared and counted.
//     jxlpe_stop_after_placement(1) ends a decode right after its first placement (an 8K frame's LF stage is all the
//     test needs).
//   * As functions on one LF group (jxlpe_place): synthetic tilings and their corruptions.
// tests/test_emu_placement.py drives both.
#include <atomic>
#include <cstring>
#include <vector>

#include "cuda_shim.h"

#include "../../jxl_oxide_b200/csrc/kernels/placement.cuh"
#include "../../oracle/oracle_backend.h"

namespace {

struct HostPlaceWarp {
  template <class F>
  void each(F f) const {
    for (uint32_t lane = 0; lane < 32; ++lane) f(lane);
  }
  void or_shared(uint32_t* p, uint32_t v) const { *p |= v; }
};

// [0] LF groups compared, [1] of those with an invalid layout, [2] groups whose status or grids differ
std::atomic<uint64_t> g_stats[3];
std::atomic<int> g_stop{0};

// The emulated placement of `job` into the given (bw x bh, stride bw) grids.
int emu_place(jxlo::OracleBackend& be, const jxlb::VarDctState& st, const jxlb::BlockInfoJob& job, int32_t* type,
              int32_t* mul, float* sigma, uint32_t stride) {
  jxlb::VarblockPlacement vp = jxlb::varblock_placement(st, job);
  jxlo::Plane& raw = be.plane(job.raw_plane);
  jxlo::Plane& sharp = be.plane(st.sharpness);
  const size_t off = size_t(job.rect.by0) * stride + job.rect.bx0;
  jxlb::DevPlacement p;
  std::memset(&p, 0, sizeof(p));
  p.raw = raw.i32();
  p.raw_stride = raw.w;
  p.nb_blocks = job.nb_blocks;
  p.bw = job.rect.bw;
  p.bh = job.rect.bh;
  p.grid_stride = stride;
  p.blk_type = type + off;
  p.blk_mul = mul + off;
  p.epf_sigma = sigma + off;
  p.sharpness = sharp.i32() + size_t(job.rect.by0) * sharp.w + job.rect.bx0;
  p.quant_mul_base = vp.quant_mul_base;
  for (int i = 0; i < 8; ++i) p.sharp_lut[i] = vp.sharp_lut[i];
  p.has_epf = vp.has_epf;
  std::vector<jxlb::PlaceShared> s(1);
  return jxlb::place_varblocks(HostPlaceWarp{}, s[0], p);
}

// Emulation and oracle on one LF group; returns the oracle's outcome (true: valid layout).
bool compare_group(jxlo::OracleBackend& be, jxlb::VarDctState& st, const jxlb::BlockInfoJob& job) {
  jxlo::Plane& type = be.plane(st.blk_type);
  std::vector<uint32_t> t(type.data), m(be.plane(st.blk_mul).data), g(be.plane(st.epf_sigma).data);
  const int emu = emu_place(be, st, job, reinterpret_cast<int32_t*>(t.data()), reinterpret_cast<int32_t*>(m.data()),
                            reinterpret_cast<float*>(g.data()), type.w);
  bool ok = true;
  try {
    be.OracleBackend::build_block_info(st, {job});
  } catch (const jxlb::Error&) {
    ok = false;
  }
  bool same = ok == (emu == jxlb::kDevOk);
  if (same && ok) {
    const bool epf = st.fh->restoration_filter.epf.iters > 0;
    const jxlo::Plane& mp = be.plane(st.blk_mul);
    const jxlo::Plane& sp = be.plane(st.epf_sigma);
    for (uint32_t y = job.rect.by0; y < job.rect.by0 + job.rect.bh; ++y)
      for (uint32_t x = job.rect.bx0; x < job.rect.bx0 + job.rect.bw; ++x) {
        const size_t i = size_t(y) * type.w + x;
        same = same && t[i] == type.data[i] && m[i] == mp.data[i] && (!epf || g[i] == sp.data[i]);
      }
  }
  ++g_stats[0];
  if (!ok) ++g_stats[1];
  if (!same) ++g_stats[2];
  return ok;
}

}  // namespace

extern "C" void jxlpe_stats(uint64_t out[3], int reset) {
  for (int i = 0; i < 3; ++i) out[i] = reset ? g_stats[i].exchange(0) : g_stats[i].load();
}
extern "C" void jxlpe_stop_after_placement(int on) { g_stop = on; }

// One LF group of bw x bh cells at the origin: raw = nb x 2 (dct_select, hf_mul - 1), sharpness = bw x bh. Places it with
// the emulation (emu != 0) or the oracle into type / mul / sigma (bw x bh; cells no varblock reached keep their input
// value in the emulation, INT32_MIN in the oracle's type grid). Returns 0 for a valid layout, 1 for an invalid one.
extern "C" int jxlpe_place(int emu, uint32_t bw, uint32_t bh, uint32_t nb, const int32_t* raw, const int32_t* sharpness,
                           int has_epf, int32_t* type, int32_t* mul, float* sigma) {
  jxlo::OracleBackend be(1);
  jxlb::FrameHeader fh;
  fh.restoration_filter.epf.iters = has_epf ? 1 : 0;
  jxlb::LfGlobalSyntax lfg;
  lfg.global_scale = 2048;
  jxlb::VarDctState st;
  st.fh = &fh;
  st.lfg = &lfg;
  st.bw = bw;
  st.bh = bh;
  st.blk_type = be.alloc_plane(bw, bh, true);
  st.blk_mul = be.alloc_plane(bw, bh, true);
  st.epf_sigma = be.alloc_plane(bw, bh, true);
  st.sharpness = be.alloc_plane(bw, bh, true);
  const int raw_plane = be.alloc_plane(nb, 2, true);
  std::memcpy(be.plane(raw_plane).data.data(), raw, size_t(nb) * 2 * 4);
  std::memcpy(be.plane(st.sharpness).data.data(), sharpness, size_t(bw) * bh * 4);
  const jxlb::BlockInfoJob job{jxlb::LfGroupRect{0, 0, bw, bh}, raw_plane, nb};
  int status;
  if (emu) {
    status = emu_place(be, st, job, type, mul, sigma, bw) == jxlb::kDevOk ? 0 : 1;
  } else {
    status = 0;
    try {
      be.build_block_info(st, {job});
    } catch (const jxlb::Error&) {
      status = 1;
    }
    std::memcpy(type, be.plane(st.blk_type).data.data(), size_t(bw) * bh * 4);
    std::memcpy(mul, be.plane(st.blk_mul).data.data(), size_t(bw) * bh * 4);
    std::memcpy(sigma, be.plane(st.epf_sigma).data.data(), size_t(bw) * bh * 4);
  }
  return status;
}

namespace jxlo {

class PlacementEmuBackend : public OracleBackend {
 public:
  explicit PlacementEmuBackend(int threads) : OracleBackend(threads) {}
  void build_block_info(VarDctState& st, const std::vector<BlockInfoJob>& jobs) override {
    bool all_ok = true;
    for (const BlockInfoJob& job : jobs) all_ok = compare_group(*this, st, job) && all_ok;
    if (g_stop) fail(kErrUnsupported, "stopped after the varblock placement");
    JXLB_CHECK(all_ok, kErrBitstream, "invalid HfMetadata block layout");
  }
};

OracleBackend* make_placement_emu_backend(int threads) { return new PlacementEmuBackend(threads); }

}  // namespace jxlo
