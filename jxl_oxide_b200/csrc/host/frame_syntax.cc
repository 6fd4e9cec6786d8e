// See frame_syntax.h.
#include "frame_syntax.h"

#include <algorithm>
#include <climits>
#include <cstdlib>
#include <cmath>

namespace jxlb {

const TransformTypeInfo kTransformInfo[kNumTransformTypes] = {
    // w8 h8 param order transpose
    {1, 1, 0, 0, 1},     // Dct8
    {1, 1, 1, 1, 0},     // Hornuss
    {1, 1, 2, 1, 0},     // Dct2
    {1, 1, 3, 1, 0},     // Dct4
    {2, 2, 4, 2, 1},     // Dct16
    {4, 4, 5, 3, 1},     // Dct32
    {1, 2, 6, 4, 1},     // Dct16x8
    {2, 1, 6, 4, 0},     // Dct8x16
    {1, 4, 7, 5, 1},     // Dct32x8
    {4, 1, 7, 5, 0},     // Dct8x32
    {2, 4, 8, 6, 1},     // Dct32x16
    {4, 2, 8, 6, 0},     // Dct16x32
    {1, 1, 9, 1, 0},     // Dct4x8
    {1, 1, 9, 1, 0},     // Dct8x4
    {1, 1, 10, 1, 0},    // Afv0
    {1, 1, 10, 1, 0},    // Afv1
    {1, 1, 10, 1, 0},    // Afv2
    {1, 1, 10, 1, 0},    // Afv3
    {8, 8, 11, 7, 1},    // Dct64
    {4, 8, 12, 8, 1},    // Dct64x32
    {8, 4, 12, 8, 0},    // Dct32x64
    {16, 16, 13, 9, 1},  // Dct128
    {8, 16, 14, 10, 1},  // Dct128x64
    {16, 8, 14, 10, 0},  // Dct64x128
    {32, 32, 15, 11, 1}, // Dct256
    {16, 32, 16, 12, 1}, // Dct256x128
    {32, 16, 16, 12, 0}, // Dct128x256
};

const uint16_t kOrderBlockSize[13][2] = {{8, 8},   {8, 8},   {16, 16},   {32, 32},  {16, 8},
                                         {32, 8},  {32, 16}, {64, 64},   {64, 32},  {128, 128},
                                         {128, 64}, {256, 256}, {256, 128}};

float powi_f32(float a, int32_t b) {  // compiler-rt __powisf2
  const bool recip = b < 0;
  float r = 1.0f;
  while (true) {
    if (b & 1) r *= a;
    b /= 2;
    if (b == 0) break;
    a *= a;
  }
  return recip ? 1.0f / r : r;
}

namespace {

HfBlockContext parse_hf_block_context(BitReader& br) {  // lf.rs:61-121
  HfBlockContext c;
  if (br.read_bool()) {
    c.num_block_clusters = 15;
    c.block_ctx_map = {0, 1, 2, 2, 3, 3, 4, 5, 6, 6, 6, 6, 6, 7, 8, 9, 9, 10, 11, 12,
                       13, 14, 14, 14, 14, 14, 7, 8, 9, 9, 10, 11, 12, 13, 14, 14, 14, 14, 14};
    return c;
  }
  uint32_t bsize = 1;
  for (auto& thr : c.lf_thresholds) {
    uint32_t n = br.read(4);
    bsize *= n + 1;
    for (uint32_t i = 0; i < n; ++i)
      thr.push_back(unpack_signed(br.read_u32({0, 4}, {16, 8}, {272, 16}, {65808, 32})));
  }
  uint32_t nq = br.read(4);
  bsize *= nq + 1;
  for (uint32_t i = 0; i < nq; ++i) c.qf_thresholds.push_back(1 + br.read_u32({0, 2}, {4, 3}, {12, 5}, {44, 8}));
  br.check();
  read_clusters(br, bsize * 39, &c.block_ctx_map, &c.num_block_clusters);
  return c;
}

}  // namespace

LfGlobalSyntax parse_lf_global(BitReader& br, const ImageHeader& ih, const FrameHeader& fh) {
  LfGlobalSyntax g;
  if (fh.patches()) {  // Patches::parse (jxl-frame/src/data/patch.rs:83-205)
    g.has_patches = true;
    std::vector<uint32_t> alpha_idx;
    for (size_t i = 0; i < ih.ec_info.size(); ++i)
      if (ih.ec_info[i].type == ExtraChannelType::kAlpha) alpha_idx.push_back(uint32_t(i));
    EntropyCode code = parse_entropy_code(br, 10);
    EntropyReader dec(&code);
    dec.begin(br);
    const uint32_t max_refs = uint32_t(std::min<uint64_t>(1u << 24, uint64_t(fh.width) * fh.height / 16));
    const uint64_t max_patches = uint64_t(max_refs) * 4;
    const uint32_t num_refs = dec.read_varint(br, 0);
    JXLB_CHECK(num_refs <= max_refs, kErrBitstream, "too many patches");
    uint64_t total = 0;
    for (uint32_t r = 0; r < num_refs; ++r) {
      PatchRef pr;
      pr.ref_idx = dec.read_varint(br, 1);
      JXLB_CHECK(pr.ref_idx < 4, kErrBitstream, "PatchRef index out of bounds");
      pr.x0 = dec.read_varint(br, 3);
      pr.y0 = dec.read_varint(br, 3);
      pr.width = dec.read_varint(br, 2) + 1;
      pr.height = dec.read_varint(br, 2) + 1;
      const uint32_t count = dec.read_varint(br, 7) + 1;
      total += count;
      JXLB_CHECK(total <= max_patches, kErrBitstream, "too many patches");
      int32_t px = 0, py = 0;
      for (uint32_t k = 0; k < count; ++k) {
        PatchTarget t;
        if (k) {
          const int64_t x = int64_t(unpack_signed(dec.read_varint(br, 6))) + px;
          const int64_t y = int64_t(unpack_signed(dec.read_varint(br, 6))) + py;
          JXLB_CHECK(x >= INT32_MIN && x <= INT32_MAX && y >= INT32_MIN && y <= INT32_MAX, kErrBitstream, "patch coord overflow");
          t.x = int32_t(x), t.y = int32_t(y);
        } else {
          t.x = int32_t(dec.read_varint(br, 4));
          t.y = int32_t(dec.read_varint(br, 4));
        }
        px = t.x, py = t.y;
        for (size_t c = 0; c < ih.ec_info.size() + 1; ++c) {
          PatchBlending b;
          b.mode = dec.read_varint(br, 5);
          JXLB_CHECK(b.mode <= 7, kErrBitstream, "invalid patch blend mode");
          if (b.mode >= 4 && alpha_idx.size() >= 2) b.alpha_channel = dec.read_varint(br, 8);
          else b.alpha_channel = alpha_idx.empty() ? 0 : alpha_idx[0];
          if (b.mode >= 3) b.clamp = dec.read_varint(br, 9) != 0;
          t.blending.push_back(b);
        }
        pr.targets.push_back(std::move(t));
      }
      g.patches.push_back(std::move(pr));
    }
    JXLB_CHECK(dec.finalize_ok(), kErrBitstream, "invalid ANS stream (patches)");
  }
  if (fh.splines()) {  // Splines::parse + QuantSpline::parse (jxl-frame/src/data/spline.rs:18-66, 155-224)
    g.has_splines = true;
    EntropyCode code = parse_entropy_code(br, 6);
    EntropyReader dec(&code);
    dec.begin(br);
    const uint64_t num_pixels = uint64_t(fh.width) * fh.height;
    size_t num_splines = dec.read_varint(br, 2);
    JXLB_CHECK(num_splines < std::min<uint64_t>(1u << 24, num_pixels / 4), kErrBitstream, "too many splines");
    ++num_splines;
    std::vector<std::pair<int64_t, int64_t>> start(num_splines);
    std::pair<int64_t, int64_t> prev;
    prev.first = dec.read_varint(br, 1);
    prev.second = dec.read_varint(br, 1);
    start[0] = prev;
    for (size_t i = 1; i < num_splines; ++i) {
      const uint32_t x = dec.read_varint(br, 1), y = dec.read_varint(br, 1);
      prev.first += unpack_signed(x);
      prev.second += unpack_signed(y);
      start[i] = prev;
    }
    g.spline_quant_adjust = unpack_signed(dec.read_varint(br, 0));
    size_t acc_points = 0;
    const size_t max_points = size_t(std::min<uint64_t>(1u << 20, num_pixels / 2));
    for (size_t i = 0; i < num_splines; ++i) {
      QuantSpline q;
      const size_t num_points = dec.read_varint(br, 3);
      acc_points += num_points;
      JXLB_CHECK(acc_points <= max_points, kErrBitstream, "too many spline points");
      std::pair<int64_t, int64_t> cur = start[i], delta{0, 0};
      q.points.push_back(cur);
      for (size_t k = 0; k < num_points; ++k) {
        const std::pair<int64_t, int64_t> before = cur;
        delta.first += unpack_signed(dec.read_varint(br, 4));
        delta.second += unpack_signed(dec.read_varint(br, 4));
        q.manhattan_distance += uint64_t(std::llabs(delta.first)) + uint64_t(std::llabs(delta.second));
        cur.first += delta.first;
        cur.second += delta.second;
        JXLB_CHECK(std::llabs(cur.first) < (int64_t(1) << 40) && std::llabs(cur.second) < (int64_t(1) << 40), kErrBitstream, "control point overflowed");
        JXLB_CHECK(cur != before, kErrBitstream, "two consecutive control points have the same value");
        q.points.push_back(cur);
      }
      for (auto& ch : q.xyb_dct)
        for (int32_t& v : ch) v = unpack_signed(dec.read_varint(br, 5));
      for (int32_t& v : q.sigma_dct) v = unpack_signed(dec.read_varint(br, 5));
      g.splines.push_back(std::move(q));
    }
    JXLB_CHECK(dec.finalize_ok(), kErrBitstream, "invalid ANS stream (splines)");
  }
  if (fh.noise()) {  // lf_global.rs:96-105
    g.has_noise = true;
    for (float& v : g.noise_lut) v = float(br.read(10)) / float(1 << 10);
  }
  if (!br.read_bool()) {
    g.m_x_lf = br.read_f16();
    g.m_y_lf = br.read_f16();
    g.m_b_lf = br.read_f16();
  }
  JXLB_CHECK(g.m_x_lf / 128.0f >= 1e-8f && g.m_y_lf / 128.0f >= 1e-8f && g.m_b_lf / 128.0f >= 1e-8f,
             kErrBitstream, "modular dequant weight too small");
  if (fh.encoding == Encoding::kVarDct) {
    g.global_scale = br.read_u32({1, 11}, {2049, 11}, {4097, 12}, {8193, 16});
    g.quant_lf = br.read_u32({16, 0}, {1, 5}, {1, 8}, {1, 16});
    g.hf_block_ctx = parse_hf_block_context(br);
    if (!br.read_bool()) {
      g.colour_factor = br.read_u32({84, 0}, {256, 0}, {2, 8}, {258, 16});
      g.base_correlation_x = br.read_f16();
      g.base_correlation_b = br.read_f16();
      g.x_factor_lf = br.read(8);
      g.b_factor_lf = br.read(8);
    }
  }
  if (g.has_splines) {  // Splines::estimate_area and the Level 10 limit (spline.rs:70-118, lf_global.rs:124-147)
    const bool vardct = fh.encoding == Encoding::kVarDct;
    const uint64_t corr_x = vardct ? uint64_t(std::ceil(std::fabs(g.base_correlation_x))) : 0;
    const uint64_t corr_b = vardct ? uint64_t(std::ceil(std::fabs(g.base_correlation_b))) : 1;
    const int32_t qa = g.spline_quant_adjust;
    auto div_ceil_qa = [qa](uint32_t v) -> uint64_t {
      const uint64_t d = v;
      if (qa >= 0) return (8 * d + 7 + uint64_t(qa)) / (8 + uint64_t(qa));
      const uint64_t a = uint64_t(-int64_t(qa));
      return d + (d * a + 7) / 8;
    };
    uint64_t total_area = 0;
    for (const QuantSpline& q : g.splines) {
      uint64_t colour[3] = {0, 0, 0};
      for (int c = 0; c < 3; ++c)
        for (int32_t v : q.xyb_dct[c]) colour[c] += div_ceil_qa(uint32_t(std::llabs(int64_t(v))));
      colour[0] += corr_x * colour[1];
      colour[2] += corr_b * colour[1];
      const uint64_t m = 1 + std::max(colour[0], std::max(colour[1], colour[2]));
      uint64_t log_colour = 0;
      while ((uint64_t(1) << log_colour) < m) ++log_colour;
      uint64_t width_estimate = 0;
      for (int32_t v : q.sigma_dct) {
        const uint64_t weight = 1 + div_ceil_qa(uint32_t(std::llabs(int64_t(v))));
        width_estimate += weight * weight * log_colour;
      }
      total_area += width_estimate * q.manhattan_distance;
    }
    const uint64_t image_size = uint64_t(fh.width) * fh.height;
    JXLB_CHECK(total_area <= std::min<uint64_t>(uint64_t(1) << 42, 1024 * image_size + (uint64_t(1) << 32)), kErrBitstream,
               "too large estimated area for splines");
  }
  br.check();
  // GlobalModular (lf_global.rs:204-313)
  uint64_t num_channels = fh.encoded_color_channels + ih.ec_info.size();
  uint64_t max_nodes = std::min<uint64_t>(1u << 22, 1024 + uint64_t(fh.width) * fh.height * num_channels / 16);
  g.has_global_tree = br.read_bool();
  if (g.has_global_tree) g.global_tree = parse_ma_tree(br, size_t(max_nodes));
  uint32_t cw = fh.color_sample_width(), ch = fh.color_sample_height();
  if (fh.encoding == Encoding::kModular && fh.do_ycbcr) {
    // Cb, Y, Cr with ChannelShift::from_jpeg_upsampling and shift_size (jxl-modular/src/param.rs:105-165): in a
    // direction where any channel is subsampled, a subsampled channel is ceil(n / 2) long and the others are rounded
    // up to twice that
    bool h_any = false, v_any = false;
    for (uint32_t j : fh.jpeg_upsampling) {
      h_any |= j == 1 || j == 2;
      v_any |= j == 1 || j == 3;
    }
    for (int i = 0; i < 3; ++i) {
      const uint32_t j = fh.jpeg_upsampling[i];
      const bool hs = h_any && (j == 0 || j == 3), vs = v_any && (j == 0 || j == 2);
      const uint32_t w = h_any ? (hs ? (cw + 1) / 2 : (cw + 1) / 2 * 2) : cw;
      const uint32_t h = v_any ? (vs ? (ch + 1) / 2 : (ch + 1) / 2 * 2) : ch;
      g.gmodular_image_channels.push_back({w, h, int32_t(hs), int32_t(vs)});
    }
  } else if (fh.encoding == Encoding::kModular) {
    for (uint32_t i = 0; i < fh.encoded_color_channels; ++i) g.gmodular_image_channels.push_back({cw, ch, 0, 0});
  }
  uint32_t color_shift = ceil_log2_nonzero(fh.upsampling);
  for (size_t i = 0; i < ih.ec_info.size(); ++i) {
    uint32_t s = ceil_log2_nonzero(fh.ec_upsampling[i]) + ih.ec_info[i].dim_shift - color_shift;
    uint32_t add = (1u << s) - 1;
    g.gmodular_image_channels.push_back({(cw + add) >> s, (ch + add) >> s, int32_t(s), int32_t(s)});
  }
  if (!g.gmodular_image_channels.empty()) {
    g.has_gmodular = true;
    g.gmodular = parse_modular_stream_header(br, g.gmodular_image_channels, g.has_global_tree);
  }
  br.check();
  return g;
}

void DequantMatrices::matrix_size(uint32_t set, uint32_t* w, uint32_t* h) {  // dct_select.rs:103-122
  static const uint16_t sizes[17][2] = {{8, 8},   {8, 8},    {8, 8},     {8, 8},     {16, 16},  {32, 32},
                                        {16, 8},  {32, 8},   {32, 16},   {8, 8},     {8, 8},    {64, 64},
                                        {64, 32}, {128, 128}, {128, 64}, {256, 256}, {256, 128}};
  *w = sizes[set][0];
  *h = sizes[set][1];
}

namespace {

// DequantMatrixParamsEncoding (dequant.rs:17-37)
struct MatrixParams {
  enum Mode { kHornuss, kDct2, kDct4, kDct4x8, kAfv, kDct, kRaw } mode = kDct;
  float raw_denominator = 0.0f;        // Raw: weight = sample * denominator, no reciprocal (dequant.rs:367-381)
  std::vector<int32_t> raw[3];
  float fixed[3][9] = {};              // Hornuss[3], Dct2[6], Dct4[2], Dct4x8[1], Afv[9]
  std::vector<float> dct_params[3];
  std::vector<float> dct4x4_params[3];
};

const float kSeqA[7] = {-1.025f, -0.78f, -0.65012f, -0.19041574f, -0.20819396f, -0.421064f, -0.32733846f};
const float kSeqB[7] = {-0.30419582f, -0.36330363f, -0.3566038f, -0.34430745f, -0.33699593f, -0.30180866f, -0.27321684f};
const float kSeqC[7] = {-1.2f, -1.2f, -0.8f, -0.7f, -0.7f, -0.4f, -0.5f};
const float kDct4x8Params[3][4] = {{2198.0505f, -0.96269625f, -0.7619425f, -0.65511405f},
                                   {764.36554f, -0.926302f, -0.967523f, -0.2784529f},
                                   {527.10754f, -1.4594386f, -1.4500821f, -1.5843723f}};
const float kDct4Params[3][4] = {{2200.0f, 0.0f, 0.0f, 0.0f}, {392.0f, 0.0f, 0.0f, 0.0f}, {112.0f, -0.25f, -0.25f, -0.5f}};

MatrixParams common_seq(float a, float b, float c) {  // dequant.rs:57-75
  MatrixParams p;
  p.mode = MatrixParams::kDct;
  p.dct_params[0] = {a};
  p.dct_params[0].insert(p.dct_params[0].end(), kSeqA, kSeqA + 7);
  p.dct_params[1] = {b};
  p.dct_params[1].insert(p.dct_params[1].end(), kSeqB, kSeqB + 7);
  p.dct_params[2] = {c};
  p.dct_params[2].insert(p.dct_params[2].end(), kSeqC, kSeqC + 7);
  return p;
}

MatrixParams dct_params3(std::vector<float> a, std::vector<float> b, std::vector<float> c) {
  MatrixParams p;
  p.mode = MatrixParams::kDct;
  p.dct_params[0] = std::move(a);
  p.dct_params[1] = std::move(b);
  p.dct_params[2] = std::move(c);
  return p;
}

MatrixParams default_params(uint32_t set) {  // dequant.rs:77-148, indexed by parameter set
  MatrixParams p;
  switch (set) {
    case 0:
      return dct_params3({3150.0f, 0.0f, -0.4f, -0.4f, -0.4f, -2.0f}, {560.0f, 0.0f, -0.3f, -0.3f, -0.3f, -0.3f},
                         {512.0f, -2.0f, -1.0f, 0.0f, -1.0f, -2.0f});
    case 1: {
      p.mode = MatrixParams::kHornuss;
      const float v[3][3] = {{280.0f, 3160.0f, 3160.0f}, {60.0f, 864.0f, 864.0f}, {18.0f, 200.0f, 200.0f}};
      for (int c = 0; c < 3; ++c)
        for (int i = 0; i < 3; ++i) p.fixed[c][i] = v[c][i];
      return p;
    }
    case 2: {
      p.mode = MatrixParams::kDct2;
      const float v[3][6] = {{3840.0f, 2560.0f, 1280.0f, 640.0f, 480.0f, 300.0f},
                             {960.0f, 640.0f, 320.0f, 180.0f, 140.0f, 120.0f},
                             {640.0f, 320.0f, 128.0f, 64.0f, 32.0f, 16.0f}};
      for (int c = 0; c < 3; ++c)
        for (int i = 0; i < 6; ++i) p.fixed[c][i] = v[c][i];
      return p;
    }
    case 3:
      p.mode = MatrixParams::kDct4;
      for (int c = 0; c < 3; ++c) {
        p.fixed[c][0] = p.fixed[c][1] = 1.0f;
        p.dct_params[c].assign(kDct4Params[c], kDct4Params[c] + 4);
      }
      return p;
    case 4:
      return dct_params3({8996.873f, -1.3000778f, -0.4942453f, -0.43909377f, -0.6350102f, -0.9017726f, -1.6162099f},
                         {3191.4836f, -0.67424583f, -0.80745816f, -0.4492584f, -0.3586544f, -0.3132239f, -0.37615025f},
                         {1157.504f, -2.0531423f, -1.4f, -0.5068713f, -0.4270873f, -1.4856834f, -4.920914f});
    case 5:
      return dct_params3({15718.408f, -1.025f, -0.98f, -0.9012f, -0.4f, -0.48819396f, -0.421064f, -0.27f},
                         {7305.7637f, -0.8041958f, -0.76330364f, -0.5566038f, -0.49785304f, -0.43699592f, -0.40180868f, -0.27321684f},
                         {3803.5317f, -3.0607336f, -2.041327f, -2.023565f, -0.54953897f, -0.4f, -0.4f, -0.3f});
    case 6:
      return dct_params3({7240.7734f, -0.7f, -0.7f, -0.2f, -0.2f, -0.2f, -0.5f}, {1448.1547f, -0.5f, -0.5f, -0.5f, -0.2f, -0.2f, -0.2f},
                         {506.85413f, -1.4f, -0.2f, -0.5f, -0.5f, -1.5f, -3.6f});
    case 7:
      return dct_params3({16283.249f, -1.7812846f, -1.6309059f, -1.0382179f, -0.85f, -0.7f, -0.9f, -1.2360638f},
                         {5089.1577f, -0.3200494f, -0.3536285f, -0.3034f, -0.61f, -0.5f, -0.5f, -0.6f},
                         {3397.7761f, -0.32132736f, -0.3450762f, -0.7034f, -0.9f, -1.0f, -1.0f, -1.1754606f});
    case 8:
      return dct_params3({13844.971f, -0.971138f, -0.658f, -0.42026f, -0.22712f, -0.2206f, -0.226f, -0.6f},
                         {4798.964f, -0.6112531f, -0.8377079f, -0.7901486f, -0.26927274f, -0.38272768f, -0.22924222f, -0.20719099f},
                         {1807.2369f, -1.2f, -1.2f, -0.7f, -0.7f, -0.7f, -0.4f, -0.5f});
    case 9:
      p.mode = MatrixParams::kDct4x8;
      for (int c = 0; c < 3; ++c) {
        p.fixed[c][0] = 1.0f;
        p.dct_params[c].assign(kDct4x8Params[c], kDct4x8Params[c] + 4);
      }
      return p;
    case 10: {
      p.mode = MatrixParams::kAfv;
      const float v[3][9] = {{3072.0f, 3072.0f, 256.0f, 256.0f, 256.0f, 414.0f, 0.0f, 0.0f, 0.0f},
                             {1024.0f, 1024.0f, 50.0f, 50.0f, 50.0f, 58.0f, 0.0f, 0.0f, 0.0f},
                             {384.0f, 384.0f, 12.0f, 12.0f, 12.0f, 22.0f, -0.25f, -0.25f, -0.25f}};
      for (int c = 0; c < 3; ++c) {
        for (int i = 0; i < 9; ++i) p.fixed[c][i] = v[c][i];
        p.dct_params[c].assign(kDct4x8Params[c], kDct4x8Params[c] + 4);
        p.dct4x4_params[c].assign(kDct4Params[c], kDct4Params[c] + 4);
      }
      return p;
    }
    case 11: return common_seq(23966.166f, 8380.191f, 4493.024f);
    case 12: return common_seq(15358.898f, 5597.3604f, 2919.9617f);
    case 13: return common_seq(47932.332f, 16760.383f, 8986.048f);
    case 14: return common_seq(30717.797f, 11194.721f, 5839.9233f);
    case 15: return common_seq(95864.664f, 33520.766f, 17972.096f);
    default: return common_seq(61435.594f, 24209.441f, 12979.847f);
  }
}

float interpolate(float pos, float max, const float* bands, size_t len) {  // dequant.rs:162-179
  if (len == 1) return bands[0];
  float scaled_pos = pos * float(len - 1) / max;
  size_t idx = size_t(scaled_pos);
  float frac = scaled_pos - float(idx);
  float a = bands[idx], b = bands[idx + 1];
  return a * powf(b / a, frac);
}

float mult(float x) { return x > 0.0f ? 1.0f + x : 1.0f / (1.0f - x); }

std::vector<float> dct_quant_weights(const std::vector<float>& params, uint32_t width, uint32_t height) {  // dequant.rs:185-215
  JXLB_CHECK(!params.empty(), kErrBitstream, "empty DCT dequant params");
  std::vector<float> bands;
  float last = params[0];
  bands.push_back(last);
  for (size_t i = 1; i < params.size(); ++i) {
    float band = last * mult(params[i]);
    JXLB_CHECK(band > 0.0f, kErrBitstream, "DCT dequant matrix: band <= 0");
    bands.push_back(band);
    last = band;
  }
  std::vector<float> ret;
  ret.reserve(size_t(width) * height);
  const float maxd = 1.41421356237309504880f + 1e-6f;
  for (uint32_t y = 0; y < height; ++y)
    for (uint32_t x = 0; x < width; ++x) {
      float dx = float(x) / float(width - 1);
      float dy = float(y) / float(height - 1);
      float distance = sqrtf(dx * dx + dy * dy);
      ret.push_back(interpolate(distance, maxd, bands.data(), bands.size()));
    }
  return ret;
}

void build_matrix(const MatrixParams& p, uint32_t set, std::vector<float> out[3]) {  // dequant.rs:156-402
  uint32_t width, height;
  DequantMatrices::matrix_size(set, &width, &height);
  for (int c = 0; c < 3; ++c) {
    std::vector<float>& ret = out[c];
    const float* params = p.fixed[c];
    switch (p.mode) {
      case MatrixParams::kDct: ret = dct_quant_weights(p.dct_params[c], width, height); break;
      case MatrixParams::kRaw:
        ret.assign(size_t(width) * height, 0.0f);
        for (size_t i = 0; i < ret.size() && i < p.raw[c].size(); ++i) ret[i] = float(p.raw[c][i]) * p.raw_denominator;
        break;
      case MatrixParams::kHornuss:
        ret.assign(64, params[0]);
        ret[0] = 1.0f;
        ret[1] = params[1];
        ret[8] = params[1];
        ret[9] = params[2];
        break;
      case MatrixParams::kDct2:
        ret.assign(64, 0.0f);
        ret[0] = 1.0f;
        for (size_t idx = 0; idx < 6; ++idx) {
          float val = params[idx];
          size_t dim = size_t(1) << (idx / 2);
          if (idx % 2 == 0) {
            for (size_t y = 0; y < dim; ++y)
              for (size_t x = dim; x < dim * 2; ++x) {
                ret[y * 8 + x] = val;
                ret[x * 8 + y] = val;
              }
          } else {
            for (size_t y = dim; y < dim * 2; ++y)
              for (size_t x = dim; x < dim * 2; ++x) ret[y * 8 + x] = val;
          }
        }
        break;
      case MatrixParams::kDct4: {
        std::vector<float> mat = dct_quant_weights(p.dct_params[c], 4, 4);
        ret.assign(64, 0.0f);
        for (size_t y = 0; y < 4; ++y)
          for (size_t x = 0; x < 4; ++x) {
            ret[y * 16 + x * 2] = mat[y * 4 + x];
            ret[y * 16 + x * 2 + 1] = mat[y * 4 + x];
            ret[(y * 2 + 1) * 8 + x * 2] = mat[y * 4 + x];
            ret[(y * 2 + 1) * 8 + x * 2 + 1] = mat[y * 4 + x];
          }
        ret[1] /= params[0];
        ret[8] /= params[0];
        ret[9] /= params[1];
        break;
      }
      case MatrixParams::kDct4x8: {
        std::vector<float> mat = dct_quant_weights(p.dct_params[c], 8, 4);
        ret.clear();
        for (size_t r = 0; r < 4; ++r)
          for (int rep = 0; rep < 2; ++rep) ret.insert(ret.end(), mat.begin() + r * 8, mat.begin() + r * 8 + 8);
        ret[8] /= params[0];
        break;
      }
      case MatrixParams::kAfv: {
        static const float kFreqs[16] = {0.0f,      0.0f, 0.8517779f, 5.3777843f, 0.0f,       0.0f,       4.734748f, 5.4492455f,
                                         1.659827f, 4.0f, 7.275749f,  10.423227f, 2.6629324f, 7.6306577f, 8.962389f, 12.971662f};
        const float lo = kFreqs[2], hi = kFreqs[15];
        std::vector<float> w4x8 = dct_quant_weights(p.dct_params[c], 8, 4);
        std::vector<float> w4x4 = dct_quant_weights(p.dct4x4_params[c], 4, 4);
        float bands[4] = {params[5], 0.0f, 0.0f, 0.0f};
        float prev = bands[0];
        for (int i = 1; i < 4; ++i) {
          bands[i] = prev * mult(params[5 + i]);
          prev = bands[i];
        }
        ret.assign(64, 0.0f);
        for (size_t y = 0; y < 4; ++y)
          for (size_t x = 0; x < 4; ++x) {
            float v;
            if (x == 0 && y == 0) v = 1.0f;
            else if (x == 0 && y == 1) v = params[2];
            else if (x == 1 && y == 0) v = params[3];
            else if (x == 1 && y == 1) v = params[4];
            else v = interpolate(kFreqs[y * 4 + x] - lo, hi - lo + 1e-6f, bands, 4);
            ret[16 * y + 2 * x] = v;
          }
        for (size_t y = 0; y < 4; ++y) {
          float* row0 = &ret[16 * y];
          float* row1 = row0 + 8;
          for (size_t x = 0; x < 8; ++x) row1[x] = (y == 0 && x == 0) ? params[0] : w4x8[y * 8 + x];
          for (size_t x = 0; x < 4; ++x) row0[2 * x + 1] = (y == 0 && x == 0) ? params[1] : w4x4[y * 4 + x];
        }
        break;
      }
    }
    if (p.mode != MatrixParams::kRaw)
      for (float& w : ret) w = 1.0f / w;
    for (float w : ret)
      JXLB_CHECK(!(w >= 1e8f || w <= 0.0f), kErrBitstream, "dequant matrix element out of range");
  }
}

void read_fixed(BitReader& br, int n, float out[3][9], int scale_first_n = 0) {
  for (int c = 0; c < 3; ++c)
    for (int i = 0; i < n; ++i) out[c][i] = br.read_f16();
  for (int c = 0; c < 3; ++c)
    for (int i = 0; i < scale_first_n; ++i) out[c][i] *= 64.0f;
}

void read_dct_params(BitReader& br, std::vector<float> out[3]) {  // dequant.rs:469-483
  uint32_t n = br.read(4) + 1;
  for (int c = 0; c < 3; ++c) {
    out[c].resize(n);
    for (float& v : out[c]) v = br.read_f16();
  }
  for (int c = 0; c < 3; ++c) out[c][0] *= 64.0f;
}

MatrixParams parse_matrix_params(BitReader& br, uint32_t set, uint32_t stream_index, const RawTableDecoder& raw_decoder) {  // dequant.rs:450-577
  uint32_t mode = br.read(3);
  bool small = set == 0 || set == 1 || set == 2 || set == 3 || set == 9 || set == 10;
  JXLB_CHECK(!(mode >= 1 && mode <= 5 && !small), kErrBitstream, "invalid dequant encoding mode for DctSelect");
  MatrixParams p;
  switch (mode) {
    case 0: return default_params(set);
    case 1:
      p.mode = MatrixParams::kHornuss;
      read_fixed(br, 3, p.fixed);
      break;
    case 2:
      p.mode = MatrixParams::kDct2;
      read_fixed(br, 6, p.fixed);
      break;
    case 3:
      p.mode = MatrixParams::kDct4;
      read_fixed(br, 2, p.fixed);
      read_dct_params(br, p.dct_params);
      break;
    case 4:
      p.mode = MatrixParams::kDct4x8;
      read_fixed(br, 1, p.fixed);
      read_dct_params(br, p.dct_params);
      break;
    case 5:
      p.mode = MatrixParams::kAfv;
      read_fixed(br, 9, p.fixed, 6);
      read_dct_params(br, p.dct_params);
      read_dct_params(br, p.dct4x4_params);
      break;
    case 6:
      p.mode = MatrixParams::kDct;
      read_dct_params(br, p.dct_params);
      break;
    default: {  // 7: Raw
      p.mode = MatrixParams::kRaw;
      p.raw_denominator = br.read_f16();
      uint32_t w, h;
      DequantMatrices::matrix_size(set, &w, &h);
      JXLB_CHECK(bool(raw_decoder), kErrUnsupported, "raw dequant tables need a Modular decoder");
      raw_decoder(br, w, h, stream_index, p.raw);
      break;
    }
  }
  br.check();
  return p;
}

}  // namespace

std::vector<uint32_t> natural_order(uint32_t order_id) {  // hf_pass.rs:156-231
  uint32_t bw = kOrderBlockSize[order_id][0], bh = kOrderBlockSize[order_id][1];
  uint32_t y_scale = bw / bh, lbw = bw / 8, lbh = bh / 8;
  std::vector<uint32_t> ret;
  ret.reserve(size_t(bw) * bh);
  for (uint32_t idx = 0; idx < lbw * lbh; ++idx) ret.push_back((idx % lbw) | ((idx / lbw) << 16));
  for (uint32_t dist = 1; dist < 2 * bw; ++dist) {
    uint32_t margin = dist > bw ? dist - bw : 0;
    for (uint32_t order = margin; order < dist - margin; ++order) {
      uint32_t x, y;
      if (dist % 2 == 1) {
        x = order;
        y = dist - 1 - order;
      } else {
        x = dist - 1 - order;
        y = order;
      }
      if (x < lbw && y < lbw) continue;
      if (y % y_scale != 0) continue;
      ret.push_back(x | ((y / y_scale) << 16));
    }
  }
  return ret;
}

HfGlobalSyntax parse_hf_global(BitReader& br, const ImageHeader& ih, const FrameHeader& fh, const LfGlobalSyntax& lfg,
                               const RawTableDecoder& raw_decoder) {
  (void)ih;
  HfGlobalSyntax g;
  // DequantMatrixSet (dequant.rs:586-658)
  const bool all_default = br.read_bool();
  auto build_all = [&](bool defaults) {
    auto dq = std::make_shared<DequantMatrices>();
    for (uint32_t set = 0; set < 17; ++set) {
      MatrixParams p = defaults ? default_params(set) : parse_matrix_params(br, set, 1 + 3 * fh.num_lf_groups() + set, raw_decoder);
      build_matrix(p, set, dq->matrices[set]);
      if (set == 0 && p.mode == MatrixParams::kRaw && std::round(1.0f / p.raw_denominator) == 2040.0f)
        for (int c = 0; c < 3; ++c) dq->jpeg[c] = p.raw[c];
      uint32_t w, h;
      DequantMatrices::matrix_size(set, &w, &h);
      for (int c = 0; c < 3; ++c) {
        const std::vector<float>& m = dq->matrices[set][c];
        std::vector<float>& t = dq->matrices_tr[set][c];
        t.resize(m.size());
        for (size_t idx = 0; idx < m.size(); ++idx) {
          size_t mx = idx % h, my = idx / h;
          t[idx] = m[mx * w + my];
        }
      }
    }
    return std::shared_ptr<const DequantMatrices>(std::move(dq));
  };
  if (all_default) {
    static const std::shared_ptr<const DequantMatrices> kDefault = build_all(true);  // thread-safe one-time init
    g.dequant = kDefault;
  } else {
    g.dequant = build_all(false);
  }
  g.dequant_all_default = all_default;
  uint32_t num_groups = fh.num_groups();
  g.num_hf_presets = br.read(ceil_log2_nonzero(num_groups)) + 1;
  for (uint32_t pass = 0; pass < fh.passes.num_passes; ++pass) {  // hf_pass.rs:34-76
    HfPassSyntax hp;
    uint32_t used_orders = br.read_u32({0x5F, 0}, {0x13, 0}, {0x00, 0}, {0, 13});
    if (used_orders != 0) {
      EntropyCode code = parse_entropy_code(br, 8);
      EntropyReader dec(&code);
      for (uint32_t id = 0; id < 13; ++id) {
        if (used_orders & 1) {
          uint32_t size = uint32_t(kOrderBlockSize[id][0]) * kOrderBlockSize[id][1];
          uint32_t skip = size / 64;
          std::vector<uint32_t> nat = natural_order(id);
          for (int c = 0; c < 3; ++c) {
            std::vector<uint32_t> perm = read_permutation(br, dec, size, skip);
            hp.order[id][c].reserve(size);
            for (uint32_t i : perm) hp.order[id][c].push_back(nat[i]);
          }
        }
        used_orders >>= 1;
      }
      JXLB_CHECK(dec.finalize_ok(), kErrBitstream, "invalid ANS stream (coefficient orders)");
    }
    const size_t code_begin = br.pos();
    hp.code = parse_entropy_code(br, 495 * g.num_hf_presets * lfg.hf_block_ctx.num_block_clusters);
#ifdef JXLB_ENTROPY_TRACE
    entropy_trace_hf_code(pass, code_begin, br.pos(), hp.code);
#endif
    (void)code_begin;
    g.passes.push_back(std::move(hp));
  }
  br.check();
  return g;
}

}  // namespace jxlb
