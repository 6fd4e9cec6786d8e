// See planner.h.
#include "planner.h"

#include "icc.h"

#include <algorithm>
#include <array>
#include <cmath>
#include <cstring>
#include <deque>
#include <map>
#include <memory>

namespace jxlb {

std::vector<uint8_t> extract_codestream(const uint8_t* data, size_t size) {
  static const uint8_t kSig[12] = {0, 0, 0, 0x0c, 'J', 'X', 'L', ' ', 0x0d, 0x0a, 0x87, 0x0a};
  if (size < 12 || std::memcmp(data, kSig, 12) != 0) return std::vector<uint8_t>(data, data + size);
  std::vector<uint8_t> out;
  size_t pos = 0;
  while (pos + 8 <= size) {
    uint64_t box_size = (uint64_t(data[pos]) << 24) | (uint64_t(data[pos + 1]) << 16) | (uint64_t(data[pos + 2]) << 8) | data[pos + 3];
    const uint8_t* ty = data + pos + 4;
    size_t header = 8;
    if (box_size == 1) {
      JXLB_CHECK(pos + 16 <= size, kErrEof, "truncated container box");
      box_size = 0;
      for (int i = 0; i < 8; ++i) box_size = (box_size << 8) | data[pos + 8 + i];
      header = 16;
    }
    size_t end = box_size == 0 ? size : pos + size_t(box_size);
    JXLB_CHECK(end <= size && end >= pos + header, kErrEof, "truncated container box");
    if (std::memcmp(ty, "jxlc", 4) == 0) {
      out.insert(out.end(), data + pos + header, data + end);
    } else if (std::memcmp(ty, "jxlp", 4) == 0) {
      JXLB_CHECK(end >= pos + header + 4, kErrBitstream, "invalid jxlp box");
      out.insert(out.end(), data + pos + header + 4, data + end);
    }
    pos = end;
  }
  JXLB_CHECK(!out.empty(), kErrBitstream, "container without codestream");
  return out;
}

namespace {

struct ChanBuf {
  View view;
  bool owned = false;
};

struct GroupChannel {
  View view;
  int32_t hshift, vshift;
};

// Rendered LF frames by level (RenderContext::lf_frame, jxl-render/src/lib.rs:46, 294-318): slot k holds
// the frame whose lf_level is k + 1; a frame with use_lf_frame reads slot `lf_level`.
struct LfFrameStore {
  bool valid = false;
  View planes[3];  // X, Y, B (f32)
};

// Splines: dequantisation, centripetal Catmull-Rom upsampling, unit arc-length resampling and the per-arc colour /
// thickness (jxl-render/src/features/spline.rs:41-178 and the head of render_spline :180-218). Scalar host work - a
// few thousand samples per frame - whose output is the arc list both backends splat.
namespace {
struct Pt {
  float x, y;
};
inline Pt operator+(Pt a, Pt b) { return {a.x + b.x, a.y + b.y}; }
inline Pt operator-(Pt a, Pt b) { return {a.x - b.x, a.y - b.y}; }
inline Pt operator*(Pt a, float k) { return {a.x * k, a.y * k}; }
inline float norm2(Pt a) { return a.x * a.x + a.y * a.y; }
inline float norm(Pt a) { return std::sqrt(norm2(a)); }
inline Pt mirror(Pt p, Pt centre) { return {centre.x + centre.x - p.x, centre.y + centre.y - p.y}; }

// value of a 32-point DCT-II series at the fractional position t (spline.rs:303-310)
float continuous_idct(const float dct[32], float t) {
  float res = dct[0];
  for (int i = 1; i < 32; ++i) {
    const float theta = float(i) * (3.14159265358979323846f / 32.0f) * (t + 0.5f);
    res += 1.41421356237309504880f * dct[i] * std::cos(theta);
  }
  return res;
}

// Rust's saturating `as i32` (NaN -> 0)
int32_t to_i32_sat(float v) {
  if (v != v) return 0;
  if (v >= 2147483648.0f) return INT32_MAX;
  if (v <= -2147483648.0f) return INT32_MIN;
  return int32_t(v);
}

std::vector<Pt> catmull_rom_points(const std::vector<Pt>& s) {
  if (s.size() == 1) return {s[0]};
  std::vector<Pt> ext;
  ext.reserve(s.size() + 2);
  ext.push_back(mirror(s[1], s[0]));
  ext.insert(ext.end(), s.begin(), s.end());
  ext.push_back(mirror(s[s.size() - 2], s[s.size() - 1]));
  std::vector<Pt> up;
  up.reserve(16 * (ext.size() - 3) + 1);
  for (size_t i = 0; i + 3 < ext.size(); ++i) {
    const Pt* p = &ext[i];
    up.push_back(p[1]);
    float t[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    for (int k = 1; k < 4; ++k) t[k] = t[k - 1] + std::pow(norm2(p[k] - p[k - 1]), 0.25f);  // knots, alpha = 1/4
    for (int step = 1; step < 16; ++step) {
      const float knot = t[1] + (float(step) / 16.0f) * (t[2] - t[1]);
      Pt a[3], b[2];
      for (int k = 0; k < 3; ++k) a[k] = p[k] + (p[k + 1] - p[k]) * ((knot - t[k]) / (t[k + 1] - t[k]));
      for (int k = 0; k < 2; ++k) b[k] = a[k] + (a[k + 1] - a[k]) * ((knot - t[k]) / (t[k + 2] - t[k]));
      up.push_back(b[0] + (b[1] - b[0]) * ((knot - t[1]) / (t[2] - t[1])));
    }
  }
  up.push_back(s.back());
  return up;
}

struct ArcSample {
  Pt point;
  float length;
};

// walk the polyline in unit steps; the last sample carries the remaining length
std::vector<ArcSample> unit_arc_samples(const std::vector<Pt>& up) {
  Pt current = up[0];
  size_t next = 0;
  std::vector<ArcSample> out{{current, 1.0f}};
  while (next < up.size()) {
    Pt prev = current;
    float arclength = 0.0f;
    for (;;) {
      if (next >= up.size()) {
        out.push_back({prev, arclength});
        break;
      }
      const Pt nx = up[next];
      const float to_next = norm(nx - prev);
      if (arclength + to_next >= 1.0f) {
        current = prev + (nx - prev) * ((1.0f - arclength) / to_next);
        out.push_back({current, 1.0f});
        break;
      }
      arclength += to_next;
      prev = nx;
      ++next;
    }
  }
  return out;
}
}  // namespace

std::vector<Backend::SplineArc> build_spline_arcs(const LfGlobalSyntax& g, bool /*vardct*/, float corr_x, float corr_b, uint32_t width,
                                                  uint32_t height) {
  std::vector<Backend::SplineArc> arcs;
  const float qa = float(g.spline_quant_adjust);
  const float inverted_qa = qa >= 0.0f ? 1.0f / (1.0f + qa / 8.0f) : 1.0f - qa / 8.0f;
  static const float kChannelWeights[4] = {0.0042f, 0.075f, 0.07f, 0.3333f};
  for (const QuantSpline& q : g.splines) {
    std::vector<Pt> pts;
    for (const auto& xy : q.points) pts.push_back({float(xy.first), float(xy.second)});
    float xyb[3][32], sigma_dct[32];
    for (int c = 0; c < 3; ++c)
      for (int i = 0; i < 32; ++i) xyb[c][i] = float(q.xyb_dct[c][i]) * kChannelWeights[c] * inverted_qa;
    for (int i = 0; i < 32; ++i) {
      xyb[0][i] += corr_x * xyb[1][i];
      xyb[2][i] += corr_b * xyb[1][i];
    }
    for (int i = 0; i < 32; ++i) sigma_dct[i] = float(q.sigma_dct[i]) * kChannelWeights[3] * inverted_qa;

    // the area limit does not bound the polygon's length when all colour coefficients are zero; the walk below is
    // linear in that length, so refuse absurd ones (the reference would allocate a sample per unit of length)
    JXLB_CHECK(q.manhattan_distance < (uint64_t(1) << 24), kErrUnsupported, "spline control polygon longer than 2^24 samples");
    const std::vector<ArcSample> samples = unit_arc_samples(catmull_rom_points(pts));
    const float arclength = float(samples.size()) - 2.0f + samples.back().length;
    for (size_t i = 0; i < samples.size(); ++i) {
      const float from_start = std::fmin(1.0f, float(i) / arclength);
      const float t = 31.0f * from_start;
      Backend::SplineArc a;
      a.x = samples[i].point.x;
      a.y = samples[i].point.y;
      a.sigma = continuous_idct(sigma_dct, t);
      a.inv_sigma = 1.0f / a.sigma;
      for (int c = 0; c < 3; ++c) a.value[c] = continuous_idct(xyb[c], t) * samples[i].length;
      // f32::max semantics: a NaN operand is ignored
      const float max_colour = std::fmax(0.01f, std::fmax(std::fmax(a.value[0], a.value[1]), a.value[2]));
      const float max_distance = std::sqrt(2.0f * (std::log(10.0f) * 3.0f + max_colour)) * std::fabs(a.sigma);
      a.xbegin = std::max<int32_t>(0, to_i32_sat(std::floor(a.x - max_distance + 0.5f)));
      a.xend = std::min<int32_t>(int32_t(width), to_i32_sat(std::floor(a.x + max_distance + 1.5f)));
      a.ybegin = std::max<int32_t>(0, to_i32_sat(std::floor(a.y - max_distance + 0.5f)));
      a.yend = std::min<int32_t>(int32_t(height), to_i32_sat(std::floor(a.y + max_distance + 1.5f)));
      if (a.xbegin < a.xend && a.ybegin < a.yend) arcs.push_back(a);
    }
  }
  return arcs;
}

// Reference slots (jxl-render/src/state.rs, lib.rs:296-330): a frame saved for later frames' patches. Only
// reference-only frames saved before the colour transform are kept (what libjxl's patch detector emits).
struct RefFrameStore {
  bool valid = false;
  bool ct_done = false;  // saved after the colour transform (regular frames) or before it (reference-only)
  uint32_t width = 0, height = 0;
  std::vector<View> channels;  // colour (XYB / as coded, f32) then extra channels (f32)
};

// A parsed Modular stream whose channel data is about to be (or has been) decoded.
struct PendingStream {
  std::unique_ptr<ModularStreamSyntax> syntax;
  std::vector<ChanBuf> coded;    // buffers of the coded channels
  std::vector<View> targets;     // where image channels must end up (empty view = stay in `coded`)
  bool direct = true;            // coded channels alias the targets (no local transforms)
  size_t job_index = 0;
};

class FramePlanner {
 public:
  FramePlanner(Backend& be, const uint8_t* cs, size_t size, const ImageHeader& ih, const DecodeOptions& opt,
               LfFrameStore (*lf_store)[4], RefFrameStore (*ref_store)[4], uint64_t visible_before,
               uint64_t invisible_before)
      : be_(be), cs_(cs), size_(size), ih_(ih), opt_(opt), lf_store_(lf_store), ref_store_(ref_store),
        visible_before_(visible_before), invisible_before_(invisible_before) {}

  DecodedFrame decode_frame(size_t frame_begin_byte, size_t* frame_end_byte);
  // A frame that fails half way (malformed or unsupported stream) must not keep its planes: they are
  // cleared from the list once exported or freed at the end of decode_frame().
  ~FramePlanner() {
    for (int id : frame_planes_) {
      try {
        be_.free_plane(id);
      } catch (...) {  // already unwinding: nothing more to do for this plane
      }
    }
  }

 private:
  BitReader reader_at(size_t bit_pos, size_t limit_byte) const { return BitReader(cs_, limit_byte, bit_pos); }
  void section(size_t logical_idx, size_t* bit_begin, size_t* byte_limit) const {
    const TocEntry& e = toc_.entries[logical_idx];
    JXLB_CHECK(e.offset + e.size <= size_, kErrEof, "frame section beyond end of codestream");
    *bit_begin = e.offset * 8;
    *byte_limit = e.offset + e.size;
  }
  const MaTree* tree_for(const ModularStreamSyntax& s) const {
    return s.has_local_tree ? &s.local_tree : &lfg_.global_tree;
  }

  // Prepares a stream: parses its header at `br`, allocates coded buffers, appends a job.
  PendingStream prepare_stream(BitReader& br, size_t limit_byte, const std::vector<GroupChannel>& image_channels,
                               uint32_t stream_index, std::vector<ModularStreamJob>* jobs);
  void finish_stream(PendingStream& ps);
  void run_inverse_transforms(const ModularStreamSyntax& s, std::vector<ChanBuf>& bufs);
  void setup_gmodular();
  std::vector<LfGroupRect> lf_rect_;
  void render_vardct(DecodedFrame* out);
  bool colour_params(bool is_xyb, size_t num_colour, ColorParams* p);
  void finish_colour(std::vector<View>& colour, bool is_xyb, bool already_converted, DecodedFrame* out);

  Backend& be_;
  const uint8_t* cs_;
  size_t size_;
  const ImageHeader& ih_;
  DecodeOptions opt_;
  LfFrameStore (*lf_store_)[4];
  RefFrameStore (*ref_store_)[4];
  // frames shown before this one / hidden frames since the last shown one: the noise generator's seed
  // (jxl-render/src/lib.rs:563-585, features/noise.rs:180-185)
  uint64_t visible_before_, invisible_before_;
  FrameHeader fh_;
  Toc toc_;
  LfGlobalSyntax lfg_;
  HfGlobalSyntax hfg_;
  VarDctState st_;
  std::vector<int> frame_planes_;  // freed at the end of the frame unless exported
  // global modular
  std::vector<ChanBuf> gm_coded_;
  size_t gm_global_count_ = 0;
  std::vector<std::vector<GroupChannel>> gm_lf_groups_;               // [lf_group]
  std::vector<std::vector<std::vector<GroupChannel>>> gm_pass_groups_;  // [pass][group]
  std::vector<uint32_t> extra_precision_;

  int new_plane(uint32_t w, uint32_t h, bool zero = false) {
    int id = be_.alloc_plane(std::max(w, 1u), std::max(h, 1u), zero);
    frame_planes_.push_back(id);
    return id;
  }
  void drop_plane(int id) {
    auto it = std::find(frame_planes_.begin(), frame_planes_.end(), id);
    if (it != frame_planes_.end()) frame_planes_.erase(it);
    be_.free_plane(id);
  }
};

PendingStream FramePlanner::prepare_stream(BitReader& br, size_t limit_byte,
                                           const std::vector<GroupChannel>& image_channels, uint32_t stream_index,
                                           std::vector<ModularStreamJob>* jobs) {
  PendingStream ps;
  std::vector<ChannelInfo> infos;
  for (const GroupChannel& g : image_channels) infos.push_back({g.view.w, g.view.h, g.hshift, g.vshift});
  ps.syntax.reset(new ModularStreamSyntax(parse_modular_stream_header(br, infos, lfg_.has_global_tree)));
  const ModularStreamSyntax& s = *ps.syntax;
  ps.direct = s.header.transforms.empty();
  for (const GroupChannel& g : image_channels) ps.targets.push_back(g.view);
  ModularStreamJob job;
  job.bit_pos = br.pos();
  job.bit_limit = limit_byte * 8;
  job.tree = tree_for(s);
  job.wp = s.header.wp;
  job.stream_index = stream_index;
  if (ps.direct) {
    for (const GroupChannel& g : image_channels) {
      ps.coded.push_back({g.view, false});
      job.channels.push_back({g.view, g.hshift, g.vshift});
    }
  } else {
    for (const ChannelInfo& c : s.channels) {
      View v;
      v.w = c.width;
      v.h = c.height;
      v.plane = (c.width && c.height) ? new_plane(c.width, c.height) : -1;
      ps.coded.push_back({v, true});
      job.channels.push_back({v, c.hshift, c.vshift});
    }
  }
  ps.job_index = jobs->size();
  jobs->push_back(std::move(job));
  return ps;
}

void FramePlanner::run_inverse_transforms(const ModularStreamSyntax& s, std::vector<ChanBuf>& bufs) {
  // TransformedModularSubimage::finish (image.rs:447-452): transforms are undone last to first.
  for (size_t ti = s.header.transforms.size(); ti-- > 0;) {
    const Transform& t = s.header.transforms[ti];
    if (t.kind == Transform::kSqueeze) {  // transform.rs:439-455
      for (size_t si = t.squeeze.size(); si-- > 0;) {
        const SqueezeStep& sp = t.squeeze[si];
        size_t begin = sp.begin_c, n = sp.num_c, end = begin + n;
        size_t res0 = sp.in_place ? end : bufs.size() - n;
        std::vector<std::pair<View, View>> pairs;
        for (size_t c = 0; c < n; ++c) pairs.push_back({bufs[begin + c].view, bufs[res0 + c].view});
        const std::vector<int> merged_ids = be_.squeeze_inverse_many(pairs, sp.horizontal);
        for (size_t c = 0; c < n; ++c) {
          ChanBuf& avg = bufs[begin + c];
          ChanBuf& res = bufs[res0 + c];
          int merged = merged_ids[c];
          frame_planes_.push_back(merged);
          View mv;
          mv.plane = merged;
          mv.w = sp.horizontal ? avg.view.w + res.view.w : avg.view.w;
          mv.h = sp.horizontal ? avg.view.h : avg.view.h + res.view.h;
          if (avg.owned && avg.view.plane >= 0) drop_plane(avg.view.plane);
          if (res.owned && res.view.plane >= 0) drop_plane(res.view.plane);
          avg.view = mv;
          avg.owned = true;
        }
        bufs.erase(bufs.begin() + res0, bufs.begin() + res0 + n);
      }
    } else if (t.kind == Transform::kRct) {
      View v[3] = {bufs[t.begin_c].view, bufs[t.begin_c + 1].view, bufs[t.begin_c + 2].view};
      if (v[0].w && v[0].h) be_.rct_inverse(v, t.rct_type);
    } else {  // palette, transform.rs:265-283
      ChanBuf pal = bufs[0];
      bufs.erase(bufs.begin());
      std::vector<View> targets;
      targets.push_back(bufs[t.begin_c].view);
      std::vector<ChanBuf> added;
      for (uint32_t c = 1; c < t.num_c; ++c) {
        View v = bufs[t.begin_c].view;
        v.plane = new_plane(v.w, v.h);
        v.x0 = v.y0 = 0;
        targets.push_back(v);
        added.push_back({v, true});
      }
      // an empty index channel has nothing to look up (palette.rs: the loops run zero times)
      if (targets[0].w && targets[0].h && targets[0].plane >= 0) {
        // a palette without explicit colours (nb_colours == 0) has no plane: only implicit and delta entries
        be_.palette_inverse(pal.view, targets, t, s.header.wp, fh_.bit_depth.bits_per_sample);
      }
      bufs.insert(bufs.begin() + t.begin_c + 1, added.begin(), added.end());
      if (pal.owned && pal.view.plane >= 0) drop_plane(pal.view.plane);
    }
  }
}

void FramePlanner::finish_stream(PendingStream& ps) {
  if (ps.direct) return;
  run_inverse_transforms(*ps.syntax, ps.coded);
  JXLB_CHECK(ps.coded.size() == ps.targets.size(), kErrBitstream, "modular transform channel mismatch");
  for (size_t i = 0; i < ps.coded.size(); ++i) {
    const View& src = ps.coded[i].view;
    const View& dst = ps.targets[i];
    JXLB_CHECK(src.w == dst.w && src.h == dst.h, kErrBitstream, "modular transform size mismatch");
    if (src.w && src.h) be_.copy_rect(src, dst);
    if (ps.coded[i].owned && src.plane >= 0) drop_plane(src.plane);
  }
}

void FramePlanner::setup_gmodular() {
  // ModularImageDestination::{prepare_gmodular,prepare_groups} (image.rs:187-345)
  const ModularStreamSyntax& s = lfg_.gmodular;
  const uint32_t gd = fh_.group_dim();
  const uint32_t gshift = ceil_log2_nonzero(gd);
  for (const ChannelInfo& c : s.channels) {
    View v;
    v.w = c.width;
    v.h = c.height;
    v.plane = (c.width && c.height) ? new_plane(c.width, c.height) : -1;
    gm_coded_.push_back({v, true});
  }
  size_t i = 0;
  for (; i < s.channels.size(); ++i) {
    const ChannelInfo& c = s.channels[i];
    if (!(i < s.nb_meta_channels || (c.width <= gd && c.height <= gd))) break;
  }
  gm_global_count_ = i;
  // pass shifts (jxl-frame/src/lib.rs:218-226)
  std::map<uint32_t, std::pair<int32_t, int32_t>> pass_shifts;
  int32_t maxshift = 3;
  for (size_t k = 0; k < fh_.passes.downsample.size() && k < fh_.passes.last_pass.size(); ++k) {
    int32_t minshift = int32_t(ceil_log2_nonzero(fh_.passes.downsample[k]));
    pass_shifts[fh_.passes.last_pass[k]] = {minshift, maxshift};
    maxshift = minshift;
  }
  pass_shifts[fh_.passes.num_passes - 1] = {0, maxshift};
  const uint32_t num_passes = fh_.passes.num_passes;
  const uint32_t cw = fh_.color_sample_width(), chh = fh_.color_sample_height();
  gm_lf_groups_.assign(fh_.num_lf_groups(), {});
  gm_pass_groups_.assign(num_passes, std::vector<std::vector<GroupChannel>>(fh_.num_groups()));
  for (; i < s.channels.size(); ++i) {
    const ChannelInfo& c = s.channels[i];
    JXLB_CHECK(c.hshift >= 0 && c.vshift >= 0, kErrBitstream, "unshiftable channel outside the global stream");
    // original size of the image channel this coded channel derives from: every non-meta channel
    // of a frame-level Modular image spans the colour sample grid (possibly dim-shifted extra
    // channels, whose original size is still the colour size; lf_global.rs:270-290).
    uint32_t ow = cw, oh = chh;
    if (c.hshift < 3 || c.vshift < 3) {
      int32_t shift = std::min(c.hshift, c.vshift);
      int pass = -1;
      for (auto& kv : pass_shifts)
        if (shift >= kv.second.first && shift < kv.second.second) {
          pass = int(kv.first);
          break;
        }
      JXLB_CHECK(pass >= 0 && uint32_t(pass) < num_passes, kErrBitstream, "no pass for modular channel shift");
      uint32_t gw = gd >> c.hshift, gh = gd >> c.vshift;
      JXLB_CHECK(gw && gh, kErrBitstream, "channel shift too large after transform");
      uint32_t nx = (ow + gd - 1) >> gshift, ny = (oh + gd - 1) >> gshift;
      JXLB_CHECK(nx * ny == fh_.num_groups(), kErrBitstream, "modular group count mismatch");
      for (uint32_t gy = 0; gy < ny; ++gy)
        for (uint32_t gx = 0; gx < nx; ++gx) {
          uint32_t x0 = gx * gw, y0 = gy * gh;
          if (x0 >= c.width || y0 >= c.height) continue;
          View v{gm_coded_[i].view.plane, x0, y0, std::min(gw, c.width - x0), std::min(gh, c.height - y0)};
          gm_pass_groups_[pass][gy * nx + gx].push_back({v, c.hshift, c.vshift});
        }
    } else {
      uint32_t gw = gd >> (c.hshift - 3), gh = gd >> (c.vshift - 3);
      JXLB_CHECK(gw && gh, kErrBitstream, "channel shift too large after transform");
      uint32_t nx = (ow + (gd << 3) - 1) >> (gshift + 3), ny = (oh + (gd << 3) - 1) >> (gshift + 3);
      JXLB_CHECK(nx * ny == fh_.num_lf_groups(), kErrBitstream, "modular LF group count mismatch");
      for (uint32_t gy = 0; gy < ny; ++gy)
        for (uint32_t gx = 0; gx < nx; ++gx) {
          uint32_t x0 = gx * gw, y0 = gy * gh;
          if (x0 >= c.width || y0 >= c.height) continue;
          View v{gm_coded_[i].view.plane, x0, y0, std::min(gw, c.width - x0), std::min(gh, c.height - y0)};
          gm_lf_groups_[gy * nx + gx].push_back({v, c.hshift, c.vshift});
        }
    }
  }
}

DecodedFrame FramePlanner::decode_frame(size_t frame_begin_byte, size_t* frame_end_byte) {
  BitReader br(cs_, size_, frame_begin_byte * 8);
  be_.phase_mark(nullptr);
  be_.new_frame();
  fh_ = parse_frame_header(br, ih_);
  toc_ = parse_toc(br, fh_);
  *frame_end_byte = toc_.data_begin + toc_.total_size;
  JXLB_CHECK(*frame_end_byte <= size_, kErrEof, "frame data beyond end of codestream");

  const bool vardct = fh_.encoding == Encoding::kVarDct;
  const bool is_lf_frame = fh_.frame_type == FrameType::kLfFrame;
  const bool is_ref_frame = fh_.frame_type == FrameType::kReferenceOnly;
  if (is_ref_frame) {
    JXLB_CHECK(fh_.save_before_ct, kErrUnsupported, "reference frames saved after the colour transform are not supported");
    JXLB_CHECK(fh_.upsampling == 1, kErrUnsupported, "upsampled reference frames are not supported");
  } else if (!is_lf_frame) {
    // regular frames are composed onto the canvas after the colour transform (jxl-render/src/blend.rs:178-415)
    JXLB_CHECK(!fh_.save_before_ct || fh_.is_last, kErrUnsupported, "regular frames saved before the colour transform are not supported");
  } else {
    JXLB_CHECK(fh_.lf_level >= 1 && fh_.lf_level <= 4 && fh_.upsampling == 1, kErrBitstream, "invalid LF frame header");
  }
  if (fh_.use_lf_frame()) {
    JXLB_CHECK(vardct, kErrBitstream, "use_lf_frame on a Modular frame");
    JXLB_CHECK(fh_.lf_level < 4 && (*lf_store_)[fh_.lf_level].valid, kErrBitstream, "frame refers to an LF frame that was not decoded");
  }
  // JPEG chroma subsampling: per-channel shifts (ChannelShift::from_jpeg_upsampling, jxl-modular/src/param.rs:105-122)
  bool h_subsampling = false, v_subsampling = false;
  uint32_t chan_hshift[3] = {0, 0, 0}, chan_vshift[3] = {0, 0, 0};
  for (uint32_t j : fh_.jpeg_upsampling) {
    h_subsampling |= j == 1 || j == 2;
    v_subsampling |= j == 1 || j == 3;
  }
  for (int c = 0; c < 3; ++c) {
    const uint32_t j = fh_.jpeg_upsampling[c];
    chan_hshift[c] = (j == 0 || j == 3) && h_subsampling;
    chan_vshift[c] = (j == 0 || j == 2) && v_subsampling;
  }
  const bool chroma_subsampled = h_subsampling || v_subsampling;
  JXLB_CHECK(!chroma_subsampled || vardct, kErrUnsupported, "chroma-subsampled Modular frames are not implemented");
  JXLB_CHECK(!chroma_subsampled || fh_.skip_adaptive_lf_smoothing(), kErrUnsupported, "adaptive LF smoothing of a chroma-subsampled frame");
  // block counts are rounded up to even in a subsampled direction (hf_metadata.rs:70-80, vardct/mod.rs:83-95)
  auto blocks_w = [&](uint32_t px) { return h_subsampling ? ((px + 7) / 8 + 1) / 2 * 2 : (px + 7) / 8; };
  auto blocks_h = [&](uint32_t px) { return v_subsampling ? ((px + 7) / 8 + 1) / 2 * 2 : (px + 7) / 8; };
  for (uint32_t u : fh_.ec_upsampling) JXLB_CHECK(u == fh_.upsampling, kErrUnsupported, "extra-channel upsampling differs from colour");
  for (const auto& ec : ih_.ec_info) JXLB_CHECK(ec.dim_shift == 0, kErrUnsupported, "dim_shift extra channels not supported");

  const uint32_t num_lf_groups = fh_.num_lf_groups(), num_groups = fh_.num_groups();
  const uint32_t num_passes = fh_.passes.num_passes;
  const bool single = toc_.single_entry();
  const uint32_t cw = fh_.color_sample_width(), chh = fh_.color_sample_height();

  // ---- LfGlobal ----
  size_t pos, limit;
  section(0, &pos, &limit);
  {
    BitReader r = reader_at(pos, limit);
    lfg_ = parse_lf_global(r, ih_, fh_);
    pos = r.pos();
  }
  if (lfg_.has_gmodular) {
    // a Modular image allocates its full-size channels up front (coded channels, then one plane per inverse transform)
    if (!vardct) be_.begin_heavy_stage(size_t(cw) * chh * 4 * 2 * (lfg_.gmodular.channels.size() + 2) + (size_t(64) << 20));
    setup_gmodular();
    std::vector<ModularStreamJob> jobs(1);
    ModularStreamJob& job = jobs[0];
    job.bit_pos = pos;
    job.bit_limit = limit * 8;
    job.tree = tree_for(lfg_.gmodular);
    job.wp = lfg_.gmodular.header.wp;
    job.stream_index = 0;
    for (size_t i = 0; i < gm_global_count_; ++i) {
      const ChannelInfo& c = lfg_.gmodular.channels[i];
      job.channels.push_back({gm_coded_[i].view, c.hshift, c.vshift});
    }
    be_.decode_modular(jobs);
    pos = jobs[0].end_bit;
  } else {
    gm_lf_groups_.assign(num_lf_groups, {});
    gm_pass_groups_.assign(num_passes, std::vector<std::vector<GroupChannel>>(num_groups));
  }

  be_.phase_mark("lf_global");
  // ---- VarDCT frame state ----
  if (vardct) {
    st_ = VarDctState();
    st_.width = cw;
    st_.height = chh;
    st_.bw = blocks_w(cw);
    st_.bh = blocks_h(chh);
    st_.subsampled = chroma_subsampled;
    for (int c = 0; c < 3; ++c) st_.hshift[c] = chan_hshift[c], st_.vshift[c] = chan_vshift[c];
    st_.group_dim = fh_.group_dim();
    st_.groups_per_row = fh_.groups_per_row();
    st_.num_groups = num_groups;
    st_.lfg = &lfg_;
    st_.hfg = &hfg_;
    st_.fh = &fh_;
    st_.ih = &ih_;
    st_.use_lf_frame = fh_.use_lf_frame();
    if (st_.use_lf_frame) {
      const LfFrameStore& lf = (*lf_store_)[fh_.lf_level];
      JXLB_CHECK(lf.planes[0].w == st_.bw && lf.planes[0].h == st_.bh, kErrBitstream, "LF frame size does not match the frame");
    }
    for (int c = 0; c < 3; ++c) {
      st_.lf_quant[c] = new_plane(st_.bw, st_.bh);
      st_.lf[c] = new_plane(st_.bw, st_.bh);
    }  // the coefficient planes are allocated when the pass groups are reached (begin_heavy_stage)
    st_.x_from_y = new_plane((cw + 63) / 64, (chh + 63) / 64);
    st_.b_from_y = new_plane((cw + 63) / 64, (chh + 63) / 64);
    st_.sharpness = new_plane(st_.bw, st_.bh);
    st_.blk_type = new_plane(st_.bw, st_.bh);
    st_.blk_mul = new_plane(st_.bw, st_.bh);
    st_.epf_sigma = new_plane(st_.bw, st_.bh);
  }

  be_.phase_mark("alloc");
  // ---- LfGroups: three entropy-coded streams each, at data-dependent bit offsets ----
  std::vector<size_t> lf_pos(num_lf_groups), lf_limit(num_lf_groups);
  std::vector<LfGroupRect> lf_rect(num_lf_groups);
  for (uint32_t g = 0; g < num_lf_groups; ++g) {
    if (single) {
      lf_pos[g] = pos;
      lf_limit[g] = limit;
    } else {
      section(1 + g, &lf_pos[g], &lf_limit[g]);
    }
    uint32_t gx = g % fh_.lf_groups_per_row(), gy = g / fh_.lf_groups_per_row();
    uint32_t lfd = fh_.lf_group_dim();
    uint32_t lw = std::min(lfd, cw - gx * lfd), lh = std::min(lfd, chh - gy * lfd);
    lf_rect[g] = {gx * (lfd / 8), gy * (lfd / 8), blocks_w(lw), blocks_h(lh)};
  }
  lf_rect_ = lf_rect;
  extra_precision_.assign(num_lf_groups, 0);
  if (vardct && !fh_.use_lf_frame()) {  // LfCoeff (jxl-vardct/src/lf.rs:138-181; absent with an LF frame)
    std::vector<ModularStreamJob> jobs;
    std::vector<PendingStream> pend;
    for (uint32_t g = 0; g < num_lf_groups; ++g) {
      BitReader r = reader_at(lf_pos[g], lf_limit[g]);
      extra_precision_[g] = r.read(2);
      const LfGroupRect& rc = lf_rect[g];
      std::vector<GroupChannel> chans;
      for (int mc : {1, 0, 2}) {  // modular channel order is Y, X, B
        const LfGroupRect sr = shifted_rect(rc, st_.hshift[mc], st_.vshift[mc]);
        chans.push_back({View{st_.lf_quant[mc], sr.bx0, sr.by0, sr.bw, sr.bh}, int32_t(st_.hshift[mc]), int32_t(st_.vshift[mc])});
      }
      pend.push_back(prepare_stream(r, lf_limit[g], chans, 1 + g, &jobs));
    }
    be_.decode_modular(jobs);
    for (uint32_t g = 0; g < num_lf_groups; ++g) {
      finish_stream(pend[g]);
      lf_pos[g] = jobs[pend[g].job_index].end_bit;
    }
  }
  be_.phase_mark("lf_coeff");
  {  // Modular LF-group channels (jxl-frame/src/data/lf_group.rs:76-91)
    std::vector<ModularStreamJob> jobs;
    std::vector<PendingStream> pend;
    std::vector<uint32_t> owner;
    for (uint32_t g = 0; g < num_lf_groups; ++g) {
      if (gm_lf_groups_[g].empty()) continue;
      BitReader r = reader_at(lf_pos[g], lf_limit[g]);
      pend.push_back(prepare_stream(r, lf_limit[g], gm_lf_groups_[g], 1 + num_lf_groups + g, &jobs));
      owner.push_back(g);
    }
    if (!jobs.empty()) be_.decode_modular(jobs);
    for (size_t k = 0; k < pend.size(); ++k) {
      finish_stream(pend[k]);
      lf_pos[owner[k]] = jobs[pend[k].job_index].end_bit;
    }
  }
  be_.phase_mark("mlf");
  if (vardct) {  // HfMetadata (jxl-vardct/src/hf_metadata.rs:52-230)
    std::vector<ModularStreamJob> jobs;
    std::vector<PendingStream> pend;
    std::vector<BlockInfoJob> bjobs;
    for (uint32_t g = 0; g < num_lf_groups; ++g) {
      BitReader r = reader_at(lf_pos[g], lf_limit[g]);
      const LfGroupRect& rc = lf_rect[g];
      uint32_t nb_blocks = 1 + r.read(ceil_log2_nonzero(rc.bw * rc.bh));
      uint32_t w64 = (rc.bw + 7) / 8, h64 = (rc.bh + 7) / 8;
      int raw = new_plane(nb_blocks, 2);
      std::vector<GroupChannel> chans;
      chans.push_back({View{st_.x_from_y, rc.bx0 / 8, rc.by0 / 8, w64, h64}, 0, 0});
      chans.push_back({View{st_.b_from_y, rc.bx0 / 8, rc.by0 / 8, w64, h64}, 0, 0});
      chans.push_back({View{raw, 0, 0, nb_blocks, 2}, 0, 0});
      chans.push_back({View{st_.sharpness, rc.bx0, rc.by0, rc.bw, rc.bh}, 0, 0});
      pend.push_back(prepare_stream(r, lf_limit[g], chans, 1 + 2 * num_lf_groups + g, &jobs));
      bjobs.push_back({rc, raw, nb_blocks});
      // without Modular transforms the stream's own output is final: the backend may place right after the stream
      if (pend.back().direct) jobs[pend.back().job_index].placement = varblock_placement(st_, bjobs.back());
    }
    be_.decode_modular(jobs);
    for (uint32_t g = 0; g < num_lf_groups; ++g) {
      finish_stream(pend[g]);
      lf_pos[g] = jobs[pend[g].job_index].end_bit;
    }
    std::vector<BlockInfoJob> rest;  // LF groups the backend did not place with their stream
    for (uint32_t g = 0; g < num_lf_groups; ++g) {
      const ModularStreamJob& j = jobs[pend[g].job_index];
      if (j.placed) JXLB_CHECK(j.layout_ok, kErrBitstream, "invalid HfMetadata block layout");
      else rest.push_back(bjobs[g]);
    }
    if (!rest.empty()) be_.build_block_info(st_, rest);
    for (auto& b : bjobs) drop_plane(b.raw_plane);
  }
  be_.phase_mark("hf_metadata");
  if (single) pos = lf_pos[0];

  // ---- HfGlobal ----
  if (vardct) {
    size_t hpos = pos, hlimit = limit;
    if (!single) section(1 + num_lf_groups, &hpos, &hlimit);
    BitReader r = reader_at(hpos, hlimit);
    // raw dequant tables (JPEG transcodes): an inline Modular image per table, decoded by the backend like any other
    // stream and read back - the matrices are built on the host
    RawTableDecoder raw_decoder = [&](BitReader& br, uint32_t w, uint32_t h, uint32_t stream_index, std::vector<int32_t> out[3]) {
      std::vector<GroupChannel> chans;
      std::vector<int> planes;
      for (int c = 0; c < 3; ++c) {
        planes.push_back(new_plane(w, h));
        chans.push_back({View{planes[c], 0, 0, w, h}, 0, 0});
      }
      std::vector<ModularStreamJob> jobs;
      PendingStream ps = prepare_stream(br, hlimit, chans, stream_index, &jobs);
      be_.decode_modular(jobs);
      finish_stream(ps);
      for (int c = 0; c < 3; ++c) {
        out[c].resize(size_t(w) * h);
        be_.download_rect(chans[c].view, out[c].data());
        drop_plane(planes[c]);
      }
      br = BitReader(cs_, hlimit, jobs[ps.job_index].end_bit);
    };
    hfg_ = parse_hf_global(r, ih_, fh_, lfg_, raw_decoder);
    if (single) pos = r.pos();
  }

  be_.phase_mark("hf_global");
  if (vardct) {
    // Everything so far worked on 1/64 of the samples; from here on the frame needs its full-resolution planes
    // (3 coefficient planes that become the pixels in place + 3 planes of filter output).
    be_.begin_heavy_stage(size_t(st_.bw) * st_.bh * 64 * 4 * 6 + (size_t(64) << 20));
    be_.phase_mark("heavy_wait");
    for (int c = 0; c < 3; ++c) st_.coeff[c] = new_plane(st_.bw * 8, st_.bh * 8, /*zero=*/true);
  }
  // ---- PassGroups ----
  for (uint32_t p = 0; p < num_passes; ++p) {
    std::vector<size_t> gpos(num_groups), glimit(num_groups);
    for (uint32_t g = 0; g < num_groups; ++g) {
      if (single) {
        gpos[g] = pos;
        glimit[g] = limit;
      } else {
        section(2 + num_lf_groups + p * num_groups + g, &gpos[g], &glimit[g]);
      }
    }
    if (vardct) {
      std::vector<HfGroupJob> jobs(num_groups);
      for (uint32_t g = 0; g < num_groups; ++g) jobs[g] = {gpos[g], glimit[g] * 8, g, p, 0};
      be_.decode_hf(st_, jobs);
      for (uint32_t g = 0; g < num_groups; ++g) gpos[g] = jobs[g].end_bit;
    }
    std::vector<ModularStreamJob> jobs;
    std::vector<PendingStream> pend;
    for (uint32_t g = 0; g < num_groups; ++g) {
      if (gm_pass_groups_[p][g].empty()) continue;
      BitReader r = reader_at(gpos[g], glimit[g]);
      pend.push_back(prepare_stream(r, glimit[g], gm_pass_groups_[p][g],
                                    1 + 3 * num_lf_groups + 17 + p * num_groups + g, &jobs));
    }
    if (!jobs.empty()) be_.decode_modular(jobs);
    for (auto& ps : pend) finish_stream(ps);
  }

  be_.phase_mark("pass_groups");
  {  // the decoded (still transformed) channels of the frame's Modular image, coding order; none when it has no such image
    std::vector<View> coded;
    if (lfg_.has_gmodular)
      for (const ChanBuf& c : gm_coded_) coded.push_back(c.view);
    be_.stage_marker("modular_coded", coded.data(), int(coded.size()));
  }
  // ---- global inverse transforms ----
  std::vector<ChanBuf> gm_image = gm_coded_;
  if (lfg_.has_gmodular) run_inverse_transforms(lfg_.gmodular, gm_image);

  be_.phase_mark("inverse_transforms");
  // ---- render ----
  DecodedFrame out;
  out.header = fh_;
  out.width = cw;
  out.height = chh;
  std::vector<View> colour;
  size_t ec_from = 0;
  if (vardct) {
    render_vardct(&out);
    for (int c = 0; c < 3; ++c) {
      if (st_.hshift[c] || st_.vshift[c]) {  // upsample_jpeg (jxl-render/src/image.rs:448-486, filter/ycbcr.rs)
        const View sub{st_.coeff[c], 0, 0, (cw + st_.hshift[c]) >> st_.hshift[c], (chh + st_.vshift[c]) >> st_.vshift[c]};
        const int id = be_.upsample_jpeg(sub, st_.hshift[c] != 0, st_.vshift[c] != 0, cw, chh);
        frame_planes_.push_back(id);
        colour.push_back(View{id, 0, 0, cw, chh});
      } else {
        colour.push_back(View{st_.coeff[c], 0, 0, cw, chh});
      }
    }
    if (st_.subsampled) be_.stage_marker("jpeg_upsampled", colour.data(), 3);
  } else {
    ec_from = fh_.encoded_color_channels;
    JXLB_CHECK(gm_image.size() >= ec_from, kErrBitstream, "missing modular colour channels");
    for (size_t c = 0; c < ec_from; ++c) colour.push_back(gm_image[c].view);
    if (ih_.xyb_encoded) {
      JXLB_CHECK(colour.size() == 3, kErrBitstream, "XYB modular frame needs three channels");
      View yxb[3] = {colour[0], colour[1], colour[2]};
      const float m[3] = {lfg_.m_x_lf / 128.0f, lfg_.m_y_lf / 128.0f, lfg_.m_b_lf / 128.0f};
      be_.modular_xyb_to_float(yxb, m);
    } else {
      for (View& v : colour) be_.int_to_float(v, ih_.bit_depth);
    }
  }
  be_.phase_mark("render_vardct");
  be_.stage_marker("pre_filter", colour.data(), int(colour.size()));

  // restoration filters (render.rs:76-131)
  const RestorationFilter& rf = fh_.restoration_filter;
  const bool upsampled = fh_.upsampling > 1;
  // an LF frame stays in XYB (it is the next frame's LF image), so does a reference frame saved before the
  // colour transform
  bool colour_done = is_lf_frame || is_ref_frame;
  if (rf.gab_enabled || rf.epf.iters > 0) {
    // a grayscale frame is filtered as three identical channels and truncated again (render.rs:74-134)
    JXLB_CHECK(colour.size() == 3 || colour.size() == 1, kErrUnsupported, "restoration filters need one or three colour channels");
    View v[3];
    for (int c = 0; c < 3; ++c) {
      if (size_t(c) < colour.size()) {
        v[c] = colour[c];
      } else {
        int id = new_plane(colour[0].w, colour[0].h);
        v[c] = View{id, 0, 0, colour[0].w, colour[0].h};
        be_.copy_rect(colour[0], v[c]);
      }
    }
    View sigma_view;
    if (vardct) sigma_view = View{st_.epf_sigma, 0, 0, st_.bw, st_.bh};
    if (vardct && rf.epf.iters > 0) be_.stage_marker("epf_sigma", &sigma_view, 1);
    ColorParams cp;
    // colour conversion follows upsampling (render.rs:136-149), so it is fused only without it
    const bool want_colour = !upsampled && !colour_done && !lfg_.has_noise && !lfg_.has_patches && !lfg_.has_splines &&
                             colour_params(ih_.xyb_encoded, colour.size(), &cp) && !cp.second_stage && cp.gamma == 0.0f &&
                             cp.pq_intensity_target == 0.0f;
    if (be_.filters_colour_fused(v, rf, sigma_view, !vardct, want_colour ? &cp : nullptr)) {
      colour_done = want_colour;
      if (want_colour) be_.stage_marker("rgb", v, 3);
    } else {
      if (rf.gab_enabled) {
        be_.gaborish(v, rf.gab_weights);
        be_.stage_marker("gaborish", v, 3);
      }
      if (rf.epf.iters > 0) {
        be_.epf(v, sigma_view, rf.epf, !vardct);
        be_.stage_marker("epf", v, 3);
      }
    }
  }

  be_.phase_mark("filters");
  // non-separable upsampling of every channel (render.rs:136-183), cropped to the frame size
  auto upsample_view = [&](View& v) {
    const uint32_t factor_log2 = ceil_log2_nonzero(fh_.upsampling);
    int id = be_.upsample(v, factor_log2, ih_);
    frame_planes_.push_back(id);
    v = View{id, 0, 0, std::min(v.w << factor_log2, fh_.width), std::min(v.h << factor_log2, fh_.height)};
  };
  if (upsampled) {
    for (View& v : colour) upsample_view(v);
    out.width = fh_.width;
    out.height = fh_.height;
    be_.stage_marker("upsampled", colour.data(), int(colour.size()));
  }
  // extra channels as floats (they take part in patch blending), upsampled like the colour channels
  std::vector<View> extra;
  for (size_t c = ec_from; c < gm_image.size() && (c - ec_from) < ih_.ec_info.size(); ++c) {
    View v = gm_image[c].view;
    be_.int_to_float(v, ih_.ec_info[c - ec_from].bit_depth);
    if (upsampled) upsample_view(v);
    extra.push_back(v);
  }
  // render_features (jxl-render/src/render.rs:159-225): patches, (splines,) noise - after upsampling, before colour
  if (lfg_.has_patches) {
    std::vector<View> all = colour;
    all.insert(all.end(), extra.begin(), extra.end());
    std::vector<Backend::PatchJob> jobs;
    for (const PatchRef& pr : lfg_.patches) {
      const RefFrameStore& ref = (*ref_store_)[pr.ref_idx];
      JXLB_CHECK(ref.valid, kErrBitstream, "patch refers to a reference frame that was not decoded");
      JXLB_CHECK(ref.channels.size() == all.size(), kErrBitstream, "patch reference has a different channel count");
      for (const PatchTarget& t : pr.targets)
        for (size_t idx = 0; idx < all.size(); ++idx) {  // blend.rs:418-545
          const PatchBlending& b = idx < colour.size() ? t.blending[0] : t.blending[1 + idx - colour.size()];
          if (b.mode == 0) continue;
          // BlendParams::from_patch_blending_info (blend.rs:104-163)
          uint32_t job_mode = b.mode;
          bool with_alpha = false, swapped = false;
          const size_t alpha_view = colour.size() + b.alpha_channel;
          if (b.mode >= 4) {
            JXLB_CHECK(alpha_view < all.size(), kErrBitstream, "patch blending refers to a missing alpha channel");
            swapped = b.mode == 5 || b.mode == 7;
            const bool is_alpha = idx == alpha_view;
            if (b.mode <= 5) {  // BlendAbove / BlendBelow
              job_mode = is_alpha ? 6 : 4;
            } else {  // MulAddAbove / MulAddBelow: the alpha channel itself is replaced (below) or kept (above)
              if (is_alpha && !swapped) continue;
              job_mode = is_alpha ? 1 : 5;
            }
            with_alpha = !is_alpha;
          }
          // target rectangle clipped to the frame, then the matching reference rectangle clipped to the reference
          const int64_t fw = all[idx].w, fhh = all[idx].h;
          const int64_t tl = std::max<int64_t>(t.x, 0), tt = std::max<int64_t>(t.y, 0);
          const int64_t tr = std::min<int64_t>(int64_t(t.x) + pr.width, fw), tb = std::min<int64_t>(int64_t(t.y) + pr.height, fhh);
          if (tr <= tl || tb <= tt) continue;
          const int64_t left = tl - t.x, top = tt - t.y;
          const int64_t rl = int64_t(pr.x0) + left, rt = int64_t(pr.y0) + top;
          const int64_t rr = std::min<int64_t>(rl + (tr - tl), ref.width), rb = std::min<int64_t>(rt + (tb - tt), ref.height);
          if (rr <= rl || rb <= rt) continue;
          const View& rv = ref.channels[idx];
          const View& dv = all[idx];
          Backend::PatchJob j;
          j.src = View{rv.plane, rv.x0 + uint32_t(rl), rv.y0 + uint32_t(rt), uint32_t(rr - rl), uint32_t(rb - rt)};
          j.dst = View{dv.plane, dv.x0 + uint32_t(tl), dv.y0 + uint32_t(tt), uint32_t(rr - rl), uint32_t(rb - rt)};
          j.mode = job_mode;
          j.clamp = b.clamp;
          j.swapped = swapped && job_mode != 1;
          if (with_alpha) {  // the frame's and the reference's alpha over the same rectangles (blend.rs:470-505)
            const View& fa = all[alpha_view];
            const View& ra = ref.channels[alpha_view];
            j.base_alpha = View{fa.plane, fa.x0 + uint32_t(tl), fa.y0 + uint32_t(tt), j.dst.w, j.dst.h};
            j.new_alpha = View{ra.plane, ra.x0 + uint32_t(rl), ra.y0 + uint32_t(rt), j.dst.w, j.dst.h};
            j.premultiplied = ih_.ec_info[b.alpha_channel].alpha_associated;
          }
          jobs.push_back(j);
        }
    }
    be_.blend_patches(jobs);
    be_.stage_marker("patches", colour.data(), int(colour.size()));
  }
  if (lfg_.has_splines) {
    JXLB_CHECK(colour.size() == 3, kErrUnsupported, "splines need three colour channels");
    // the reference draws splines on the grid as it stands after patches (render.rs:182-205); with upsampling and no
    // patches that is the pre-upsampling grid - not restated here
    JXLB_CHECK(!upsampled, kErrUnsupported, "splines together with upsampling are not implemented");
    const std::vector<Backend::SplineArc> arcs =
        build_spline_arcs(lfg_, vardct, vardct ? lfg_.base_correlation_x : 0.0f, vardct ? lfg_.base_correlation_b : 1.0f, fh_.width, fh_.height);
    View v[3] = {colour[0], colour[1], colour[2]};
    be_.splat_splines(v, arcs);
    be_.stage_marker("splines", v, 3);
  }
  if (lfg_.has_noise) {
    JXLB_CHECK(colour.size() == 3 && ih_.xyb_encoded, kErrUnsupported, "noise synthesis is implemented for XYB colour frames");
    JXLB_CHECK(!upsampled, kErrUnsupported, "noise synthesis together with upsampling is not implemented");
    View v[3] = {colour[0], colour[1], colour[2]};
    const float corr_x = vardct ? lfg_.base_correlation_x : 0.0f, corr_b = vardct ? lfg_.base_correlation_b : 1.0f;
    // a shown frame counts itself among the visible ones; a hidden one among the invisible ones
    const bool shown = !is_lf_frame && !is_ref_frame;
    const uint64_t seed0 = shown ? ((visible_before_ + 1) << 32) : (visible_before_ << 32) + invisible_before_ + 1;
    be_.add_noise(v, lfg_.noise_lut, fh_.group_dim(), seed0, corr_x, corr_b);
    be_.stage_marker("noise", v, 3);
  }
  if (fh_.do_ycbcr && !colour_done) {  // jxl-render/src/lib.rs:950-954, util.rs:320-329
    JXLB_CHECK(colour.size() == 3, kErrBitstream, "YCbCr needs three channels");
    View v[3] = {colour[0], colour[1], colour[2]};
    be_.ycbcr_to_rgb(v, Backend::YcbcrParams());
    be_.stage_marker("rgb", v, 3);
    if (ih_.colour_encoding.colour_space == ColourSpace::kGrey) colour.resize(1);
  }
  finish_colour(colour, ih_.xyb_encoded, colour_done, &out);
  out.channels.insert(out.channels.end(), extra.begin(), extra.end());
  if (is_lf_frame) {
    JXLB_CHECK(colour.size() == 3, kErrUnsupported, "grayscale LF frames are not supported");
    LfFrameStore& slot = (*lf_store_)[fh_.lf_level - 1];
    if (slot.valid)
      for (const View& v : slot.planes) be_.free_plane(v.plane);
    for (int c = 0; c < 3; ++c) slot.planes[c] = colour[c];
    slot.valid = true;
    out.internal = true;
  }
  const bool normal_frame = !is_lf_frame && !is_ref_frame;
  const bool can_reference = !fh_.is_last && (fh_.duration == 0 || fh_.save_as_reference != 0) && !is_lf_frame;  // header.rs:221-225
  if (normal_frame && !(fh_.resets_canvas && out.width == ih_.width && out.height == ih_.height)) {
    // ---- composition onto the image canvas (blend.rs:178-415 as a full-canvas model): every channel starts from
    // its source slot's canvas (transparent black when the slot is empty) and the frame's rectangle is blended in
    const size_t ncol = colour.size();
    const bool has_extra = !fh_.ec_blending_info.empty();
    std::vector<View> frame_ch = out.channels;
    std::vector<View> canvas(frame_ch.size());
    std::vector<Backend::PatchJob> colour_jobs, extra_jobs;
    // the frame's rectangle clipped to the canvas
    const int64_t fx0 = std::max<int64_t>(fh_.x0, 0), fy0 = std::max<int64_t>(fh_.y0, 0);
    const int64_t fx1 = std::min<int64_t>(int64_t(fh_.x0) + out.width, ih_.width), fy1 = std::min<int64_t>(int64_t(fh_.y0) + out.height, ih_.height);
    for (size_t idx = 0; idx < frame_ch.size(); ++idx) {
      const BlendingInfo& bi = idx < ncol ? fh_.blending_info : fh_.ec_blending_info[idx - ncol];
      const RefFrameStore& base = (*ref_store_)[bi.source];
      int id = new_plane(ih_.width, ih_.height, /*zero=*/true);
      canvas[idx] = View{id, 0, 0, ih_.width, ih_.height};
      const bool have_base = base.valid && idx < base.channels.size();
      if (have_base) {
        JXLB_CHECK(base.ct_done || !ih_.xyb_encoded, kErrUnsupported, "blending onto a frame saved before the colour transform");
        const View& bv = base.channels[idx];
        const uint32_t cw = std::min(bv.w, ih_.width), chh = std::min(bv.h, ih_.height);
        be_.copy_rect(View{bv.plane, bv.x0, bv.y0, cw, chh}, View{id, 0, 0, cw, chh});
      }
      if (fx1 <= fx0 || fy1 <= fy0) continue;
      Backend::PatchJob j;
      const uint32_t rw = uint32_t(fx1 - fx0), rh = uint32_t(fy1 - fy0);
      const uint32_t sx = uint32_t(fx0 - fh_.x0), sy = uint32_t(fy0 - fh_.y0);
      j.src = View{frame_ch[idx].plane, frame_ch[idx].x0 + sx, frame_ch[idx].y0 + sy, rw, rh};
      j.dst = View{id, uint32_t(fx0), uint32_t(fy0), rw, rh};
      j.clamp = bi.clamp;
      const bool uses_alpha = (bi.mode == BlendMode::kBlend || bi.mode == BlendMode::kMulAdd) && has_extra;
      const size_t alpha_ch = ncol + bi.alpha_channel;
      if (uses_alpha) {
        JXLB_CHECK(alpha_ch < frame_ch.size(), kErrBitstream, "blend alpha channel out of range");
        j.new_alpha = View{frame_ch[alpha_ch].plane, frame_ch[alpha_ch].x0 + sx, frame_ch[alpha_ch].y0 + sy, rw, rh};
        if (base.valid && alpha_ch < base.channels.size()) {
          const View& av = base.channels[alpha_ch];
          if (uint32_t(fx1) <= av.w && uint32_t(fy1) <= av.h) j.base_alpha = View{av.plane, av.x0 + uint32_t(fx0), av.y0 + uint32_t(fy0), rw, rh};
          else JXLB_CHECK(false, kErrUnsupported, "blend base smaller than the frame rectangle");
        }
        j.premultiplied = ih_.ec_info[bi.alpha_channel].alpha_associated;
      }
      switch (bi.mode) {  // BlendParams::from_blending_info (blend.rs:55-103)
        case BlendMode::kReplace: j.mode = 1; break;
        case BlendMode::kAdd: j.mode = 2; break;
        case BlendMode::kMul: j.mode = 3; break;
        case BlendMode::kBlend: j.mode = !uses_alpha ? 1 : (idx == alpha_ch ? 6 : 4); break;
        default: j.mode = !uses_alpha ? 2 : (idx == alpha_ch ? 0 : 5); break;  // MulAdd; Skip on its alpha channel
      }
      if (j.mode == 6) j.new_alpha = j.base_alpha = View();
      if (j.mode == 0) continue;
      (idx < ncol ? colour_jobs : extra_jobs).push_back(j);
    }
    be_.blend_patches(colour_jobs);
    be_.blend_patches(extra_jobs);
    out.channels = canvas;
    out.width = ih_.width;
    out.height = ih_.height;
  }
  if (is_ref_frame || (normal_frame && can_reference)) {
    RefFrameStore& slot = (*ref_store_)[fh_.save_as_reference];
    if (slot.valid)
      for (const View& v : slot.channels) be_.free_plane(v.plane);
    slot.channels.clear();
    if (is_ref_frame) {
      slot.channels = out.channels;  // never shown: the slot takes the planes over
    } else {
      for (const View& v : out.channels) {  // the frame may also be shown: the slot keeps a copy
        int id = be_.alloc_plane(std::max(v.w, 1u), std::max(v.h, 1u), false);
        if (v.w && v.h) be_.copy_rect(v, View{id, 0, 0, v.w, v.h});
        slot.channels.push_back(View{id, 0, 0, v.w, v.h});
      }
    }
    slot.width = out.width;
    slot.height = out.height;
    slot.ct_done = !is_ref_frame;
    slot.valid = true;
  }
  if (is_ref_frame || (normal_frame && !fh_.is_keyframe())) out.internal = true;
  // release everything not exported
  for (int id : frame_planes_) {
    bool exported = false;
    for (const View& v : out.channels) exported |= (v.plane == id);
    if (!exported) be_.free_plane(id);
  }
  frame_planes_.clear();
  gm_coded_.clear();
  be_.phase_mark("filters_colour");
  return out;
}

void FramePlanner::render_vardct(DecodedFrame*) {
  be_.vardct_coefficients(st_);
  // LF: dequant, chroma-from-luma, adaptive smoothing (vardct/mod.rs:163-201, util.rs:254-290)
  std::vector<LfDequantJob> jobs;
  const uint32_t lfd = fh_.lf_group_dim();
  for (uint32_t g = 0; g < fh_.num_lf_groups(); ++g) {
    LfDequantJob j;
    j.rect = lf_rect_[g];
    const float m[3] = {lfg_.m_x_lf, lfg_.m_y_lf, lfg_.m_b_lf};
    int32_t precision_scale = 1 << (9 - extra_precision_[g]);
    uint64_t scale_inv = uint64_t(lfg_.global_scale) * lfg_.quant_lf;
    for (int c = 0; c < 3; ++c) j.scale[c] = float(double(m[c]) * double(precision_scale) / double(scale_inv));
    jobs.push_back(j);
  }
  if (st_.use_lf_frame) {
    // the LF image is the rendered LF frame, used as is (jxl-render/src/vardct/mod.rs:175-180)
    const LfFrameStore& lf = (*lf_store_)[fh_.lf_level];
    for (int c = 0; c < 3; ++c) be_.copy_rect(lf.planes[c], View{st_.lf[c], 0, 0, st_.bw, st_.bh});
  } else {
    be_.lf_dequant(st_, jobs);
    if (!st_.subsampled) be_.lf_chroma_from_luma(st_);  // vardct/mod.rs:184-191
    if (!fh_.skip_adaptive_lf_smoothing()) be_.lf_adaptive_smoothing(st_);
  }
  {
    View v[3], cf[3];
    for (int c = 0; c < 3; ++c) {
      v[c] = View{st_.lf[c], 0, 0, st_.bw >> st_.hshift[c], st_.bh >> st_.vshift[c]};
      cf[c] = View{st_.coeff[c], 0, 0, (st_.bw >> st_.hshift[c]) * 8, (st_.bh >> st_.vshift[c]) * 8};
    }
    be_.stage_marker("lf", v, 3);
    be_.stage_marker("hf_coeff", cf, 3);
    be_.hf_dequant_cfl(st_);
    be_.stage_marker("hf_dequant", cf, 3);
    be_.hf_transform(st_);
    be_.stage_marker("idct", cf, 3);
  }
}

// postprocess_keyframe (jxl-render/src/lib.rs:925-998) for the supported colour set: fills the
// XYB -> (linear) sRGB parameters; false when the planes are left as they are.
namespace {
// jxl-color/src/ciexyz.rs:76-179 and consts.rs: every expression evaluated in f32, left to right
typedef std::array<float, 9> Mat3;
Mat3 matmul3(const Mat3& a, const Mat3& b) {
  Mat3 r;
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) r[i * 3 + j] = a[i * 3] * b[j] + a[i * 3 + 1] * b[3 + j] + a[i * 3 + 2] * b[6 + j];
  return r;
}
std::array<float, 3> matmul3vec(const Mat3& a, const std::array<float, 3>& b) {
  return {a[0] * b[0] + a[1] * b[1] + a[2] * b[2], a[3] * b[0] + a[4] * b[1] + a[5] * b[2], a[6] * b[0] + a[7] * b[1] + a[8] * b[2]};
}
Mat3 matinv(const Mat3& m) {
  const float det = m[0] * (m[4] * m[8] - m[5] * m[7]) + m[1] * (m[5] * m[6] - m[3] * m[8]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
  return {(m[4] * m[8] - m[5] * m[7]) / det, (m[7] * m[2] - m[8] * m[1]) / det, (m[1] * m[5] - m[2] * m[4]) / det,
          (m[5] * m[6] - m[3] * m[8]) / det, (m[8] * m[0] - m[6] * m[2]) / det, (m[2] * m[3] - m[0] * m[5]) / det,
          (m[3] * m[7] - m[4] * m[6]) / det, (m[6] * m[1] - m[7] * m[0]) / det, (m[0] * m[4] - m[1] * m[3]) / det};
}
std::array<float, 3> illuminant_to_xyz(const float xy[2]) { return {xy[0] / xy[1], 1.0f, (1.0f - xy[0]) / xy[1] - 1.0f}; }
Mat3 primaries_grid(const float p[3][2]) {
  return {p[0][0], p[1][0], p[2][0], p[0][1], p[1][1], p[2][1], (1.0f - p[0][0] - p[0][1]), (1.0f - p[1][0] - p[1][1]),
          (1.0f - p[2][0] - p[2][1])};
}
Mat3 primaries_to_xyz_mat(const float p[3][2], const float wp[2]) {
  Mat3 m = primaries_grid(p);
  const std::array<float, 3> mul = matmul3vec(matinv(m), illuminant_to_xyz(wp));
  for (int i = 0; i < 9; ++i) m[i] *= mul[i % 3];
  return m;
}
Mat3 xyz_to_primaries_mat(const float p[3][2], const float wp[2]) {
  Mat3 inv = matinv(primaries_grid(p));
  const std::array<float, 3> mul = matmul3vec(inv, illuminant_to_xyz(wp));
  for (int i = 0; i < 9; ++i) inv[i] /= mul[i / 3];
  return inv;
}
Mat3 adapt_mat(const float from[2], const float to[2]) {  // Bradford
  static const Mat3 kBradford = {0.8951f, 0.2664f, -0.1614f, -0.7502f, 1.7135f, 0.0367f, 0.0389f, -0.0685f, 1.0296f};
  static const Mat3 kBradfordInv = {0.9869929f, -0.1470543f, 0.1599627f, 0.4323053f, 0.5183603f,
                                    0.0492912f, -0.0085287f, 0.0400428f, 0.9684867f};
  const std::array<float, 3> from_w = illuminant_to_xyz(from), to_w = illuminant_to_xyz(to);
  if (from_w == to_w) return {1, 0, 0, 0, 1, 0, 0, 0, 1};
  const std::array<float, 3> from_lms = matmul3vec(kBradford, from_w), to_lms = matmul3vec(kBradford, to_w);
  const float mul[3] = {to_lms[0] / from_lms[0], to_lms[1] / from_lms[1], to_lms[2] / from_lms[2]};
  Mat3 multiplied;
  for (int i = 0; i < 9; ++i) multiplied[i] = kBradford[i] * mul[i / 3];
  return matmul3(kBradfordInv, multiplied);
}

const float kIlluminantD65[2] = {0.3127f, 0.329f};
const float kPrimariesSrgb[3][2] = {{0.639998686f, 0.330010138f}, {0.300003784f, 0.600003357f}, {0.150002046f, 0.059997204f}};

// The tail of ColorTransform::new for a linear-sRGB source (convert.rs:397-466) with its Matrix ops merged as
// optimize() does (convert.rs:662-690): M = xyz_to_target * (adapt * srgb_to_xyz), or adapt * srgb_to_xyz for Grey.
void target_matrix(const ColourEncoding& ce, bool grey, ColorParams* p) {
  float wp[2] = {kIlluminantD65[0], kIlluminantD65[1]};
  switch (ce.white_point) {
    case WhitePointKind::kD65: break;
    case WhitePointKind::kCustom: wp[0] = float(ce.white_xy[0]) / 1e6f, wp[1] = float(ce.white_xy[1]) / 1e6f; break;
    case WhitePointKind::kE: wp[0] = 1.0f / 3.0f, wp[1] = 1.0f / 3.0f; break;
    case WhitePointKind::kDci: wp[0] = 0.314f, wp[1] = 0.351f; break;
  }
  float prim[3][2];
  const float (*src)[2] = kPrimariesSrgb;
  static const float kBt2100[3][2] = {{0.708f, 0.292f}, {0.170f, 0.797f}, {0.131f, 0.046f}};
  static const float kP3[3][2] = {{0.680f, 0.320f}, {0.265f, 0.690f}, {0.150f, 0.060f}};
  if (ce.primaries == PrimariesKind::kBt2100) src = kBt2100;
  if (ce.primaries == PrimariesKind::kP3) src = kP3;
  for (int i = 0; i < 3; ++i)
    for (int k = 0; k < 2; ++k)
      prim[i][k] = ce.primaries == PrimariesKind::kCustom ? float(ce.primaries_xy[i][k]) / 1e6f : src[i][k];
  const Mat3 to_xyz = primaries_to_xyz_mat(kPrimariesSrgb, kIlluminantD65);
  p->second_stage = true;
  for (int i = 0; i < 3; ++i) p->luminances[i] = to_xyz[3 + i];
  Mat3 m = matmul3(adapt_mat(kIlluminantD65, wp), to_xyz);
  if (!grey) m = matmul3(xyz_to_primaries_mat(prim, wp), m);
  for (int i = 0; i < 9; ++i) p->matrix2[i] = m[i];
  p->to_luma = grey;
}
}  // namespace

bool FramePlanner::colour_params(bool is_xyb, size_t num_colour, ColorParams* p) {
  if (!is_xyb || opt_.output_colour == 2) return false;
  JXLB_CHECK(num_colour == 3, kErrBitstream, "XYB needs three channels");
  // with an embedded ICC profile the target is the equivalent enum encoding, or sRGB (jxl-render/src/lib.rs:104-150)
  const ColourEncoding& ce = ih_.colour_encoding.want_icc ? ih_.icc_encoding : ih_.colour_encoding;
  const bool linear_srgb_out = opt_.output_colour == 1;
  if (!linear_srgb_out) {
    JXLB_CHECK(ce.colour_space == ColourSpace::kRgb || ce.colour_space == ColourSpace::kGrey, kErrUnsupported,
               "unsupported output colour space");
    // HLG needs libm's powf / ln on the device; its results would not be reproducible bit for bit
    JXLB_CHECK(ce.tf != TransferFunctionKind::kHlg, kErrUnsupported, "the HLG output transfer function is not implemented");
  }
  // an HDR target keeps the image's range (convert.rs:478-499: tone mapping only towards non-HDR targets)
  const bool hdr_target = !linear_srgb_out && ce.tf == TransferFunctionKind::kPq;
  JXLB_CHECK(ih_.tone_mapping.intensity_target <= 255.0f || opt_.output_colour == 1 || hdr_target, kErrUnsupported,
             "HDR tone mapping is outside the implemented hot path");
  const OpsinInverseMatrix& oim = ih_.opsin_inverse_matrix;
  for (int i = 0; i < 3; ++i) {
    p->opsin_bias[i] = oim.opsin_bias[i];
    p->cbrt_opsin_bias[i] = cbrtf(oim.opsin_bias[i]);
    for (int j = 0; j < 3; ++j) p->matrix[i * 3 + j] = oim.inv_mat[i][j];
  }
  p->itscale = 255.0f / ih_.tone_mapping.intensity_target;
  p->apply_srgb_tf = (opt_.output_colour == 0) && ce.tf == TransferFunctionKind::kSrgb;
  p->apply_bt709_tf = (opt_.output_colour == 0) && ce.tf == TransferFunctionKind::kBt709;
  if (!linear_srgb_out) {
    if (ce.tf == TransferFunctionKind::kGamma)  // convert.rs:972-989
      p->gamma = ce.gamma_inverted ? float(ce.gamma) / 1e7f : 1e7f / float(ce.gamma);
    if (ce.tf == TransferFunctionKind::kDci) p->gamma = 1.0f / 2.6f;
    if (ce.tf == TransferFunctionKind::kPq) p->pq_intensity_target = ih_.tone_mapping.intensity_target;
    const bool grey = ce.colour_space == ColourSpace::kGrey;
    if (grey || ce.white_point != WhitePointKind::kD65 || ce.primaries != PrimariesKind::kSrgb) target_matrix(ce, grey, p);
  }
  return true;
}

void FramePlanner::finish_colour(std::vector<View>& colour, bool is_xyb, bool already_converted, DecodedFrame* out) {
  ColorParams p;
  if (!already_converted && colour_params(is_xyb, colour.size(), &p)) {
    View v[3] = {colour[0], colour[1], colour[2]};
    be_.xyb_to_rgb(v, p);
    if (p.to_luma) colour.resize(1);  // XyzToLuma leaves Y in the first channel (convert.rs:866-872)
    be_.stage_marker("rgb", colour.data(), int(colour.size()));
  }
  out->num_color = uint32_t(colour.size());
  out->channels = colour;
}

}  // namespace

StreamLayout stream_layout(const ImageHeader& ih, const DecodedFrame& f) {
  StreamLayout l;
  for (size_t c = 0; c < f.num_color && c < f.channels.size(); ++c) l.channels.push_back(c);
  if (ih.icc_is_cmyk)  // fb.rs:211-226
    for (size_t e = 0; e < ih.ec_info.size() && f.num_color + e < f.channels.size(); ++e)
      if (ih.ec_info[e].type == ExtraChannelType::kBlack) {
        l.channels.push_back(f.num_color + e);
        break;
      }
  for (size_t e = 0; e < ih.ec_info.size() && f.num_color + e < f.channels.size(); ++e)
    if (ih.ec_info[e].type == ExtraChannelType::kAlpha) {
      l.channels.push_back(f.num_color + e);
      break;
    }
  if (f.num_color == 3 && !ih.grayscale())
    for (size_t e = 0; e < ih.ec_info.size() && f.num_color + e < f.channels.size(); ++e)
      if (ih.ec_info[e].type == ExtraChannelType::kSpotColour) {
        const float* s = ih.ec_info[e].spot;
        l.spots.push_back(StreamSpot{f.num_color + e, {s[0], s[1], s[2]}, s[3]});
      }
  return l;
}

DecodeResult decode_codestream(Backend& be, const uint8_t* cs, size_t size, const DecodeOptions& opt) {
  DecodeResult res;
  be.set_codestream(cs, size);
  BitReader br(cs, size);
  res.image_header = parse_image_header(br);
  const ImageHeader& ih = res.image_header;
  if (ih.colour_encoding.want_icc) {  // jxl-oxide/src/lib.rs:365-372, jxl-render/src/lib.rs:100-150
    ImageHeader& mih = res.image_header;
    mih.icc_profile = decode_icc_stream(read_icc_stream(br));
    IccInfo info;
    const IccStatus st = icc_to_enum(mih.icc_profile, &info);
    const bool header_gray = mih.colour_encoding.colour_space == ColourSpace::kGrey;
    if (st != IccStatus::kMalformed)
      JXLB_CHECK(header_gray == info.is_gray, kErrBitstream, "colour channel mismatch between header and ICC profile");
    mih.icc_is_enum = st == IccStatus::kEnum;
    mih.icc_is_cmyk = st != IccStatus::kMalformed && info.is_cmyk;
    if (mih.icc_is_enum) {
      mih.icc_encoding = info.encoding;
    } else {  // EnumColourEncoding::{gray_srgb, srgb}
      mih.icc_encoding = ColourEncoding();
      if (header_gray) mih.icc_encoding.colour_space = ColourSpace::kGrey;
    }
  }
  br.zero_pad_to_byte();
  size_t pos = br.pos() / 8;
  if (ih.have_preview) {  // skipped, like jxl-oxide/src/lib.rs:384-411
    BitReader pr(cs, size, pos * 8);
    FrameHeader pfh = parse_frame_header(pr, ih);
    (void)pfh;
    fail(kErrUnsupported, "preview frames are not supported");
  }
  LfFrameStore lf_store[4];
  RefFrameStore ref_store[4];
  uint64_t visible_frames = 0, invisible_frames = 0;
  auto drop_lf_frames = [&] {
    for (LfFrameStore& s : lf_store)
      if (s.valid)
        for (const View& v : s.planes) be.free_plane(v.plane);
    for (RefFrameStore& s : ref_store)
      if (s.valid)
        for (const View& v : s.channels) be.free_plane(v.plane);
  };
  try {
    while (pos < size && res.frames.size() < opt.max_frames) {
      FramePlanner planner(be, cs, size, ih, opt, &lf_store, &ref_store, visible_frames, invisible_frames);
      size_t end = 0;
      DecodedFrame f = planner.decode_frame(pos, &end);
      bool last = f.header.is_last;
      if (f.internal) {  // an LF / reference / hidden frame: what later frames need lives in the stores
        if (f.header.frame_type == FrameType::kLfFrame)
          for (size_t c = 3; c < f.channels.size(); ++c) be.free_plane(f.channels[c].plane);
        else if (f.header.frame_type != FrameType::kReferenceOnly)
          for (const View& v : f.channels) be.free_plane(v.plane);
        ++invisible_frames;
      } else {
        res.frames.push_back(std::move(f));
        ++visible_frames;
        invisible_frames = 0;
      }
      pos = end;
      if (last) break;
    }
  } catch (...) {
    drop_lf_frames();
    for (DecodedFrame& f : res.frames)  // frames finished before the failing one
      for (const View& v : f.channels) be.free_plane(v.plane);
    throw;
  }
  drop_lf_frames();
  return res;
}

}  // namespace jxlb
