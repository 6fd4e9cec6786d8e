// Image header, frame header and TOC parsing. See headers.h for the reference citations.
#include "headers.h"

#include <algorithm>
#include <cmath>

#include "entropy.h"

namespace jxlb {

namespace {

// Default upsampling weights are fixed tables in the spec (jxl-image/src/lib.rs:493-594);
// they live in upsampling_weights.inc to keep this file readable.
#include "upsampling_weights.inc"

using D = BitReader::U32Dist;

void parse_size(BitReader& br, uint32_t* width, uint32_t* height) {  // jxl-image/src/lib.rs:98-128
  bool div8 = br.read_bool();
  uint32_t h_div8 = div8 ? 1 + br.read(5) : 0;
  uint32_t h = div8 ? 8 * h_div8 : br.read_u32({1, 9}, {1, 13}, {1, 18}, {1, 30});
  uint32_t ratio = br.read(3);
  uint32_t w_div8 = (div8 && ratio == 0) ? 1 + br.read(5) : 0;
  uint32_t w;
  if (!div8 && ratio == 0) {
    w = br.read_u32({1, 9}, {1, 13}, {1, 18}, {1, 30});
  } else {
    uint64_t hh = h;
    uint64_t res;
    switch (ratio) {
      case 0: res = 8ull * w_div8; break;
      case 1: res = hh; break;
      case 2: res = hh * 12 / 10; break;
      case 3: res = hh * 4 / 3; break;
      case 4: res = hh * 3 / 2; break;
      case 5: res = hh * 16 / 9; break;
      case 6: res = hh * 5 / 4; break;
      default: res = hh * 2; break;
    }
    w = uint32_t(res);
  }
  *width = w;
  *height = h;
}

void parse_preview_size(BitReader& br, uint32_t* width, uint32_t* height) {  // lib.rs:172-187
  bool div8 = br.read_bool();
  uint32_t h_div8 = div8 ? br.read_u32({16, 0}, {32, 0}, {1, 5}, {33, 9}) : 1;
  uint32_t h = div8 ? 8 * h_div8 : br.read_u32({1, 6}, {65, 8}, {321, 10}, {1345, 12});
  uint32_t ratio = br.read(3);
  uint32_t w_div8 = div8 ? br.read_u32({16, 0}, {32, 0}, {1, 5}, {33, 9}) : 1;
  uint32_t w;
  if (!div8) {
    w = br.read_u32({1, 6}, {65, 8}, {321, 10}, {1345, 12});
  } else {
    uint64_t hh = h, res;
    switch (ratio) {
      case 0: res = 8ull * w_div8; break;
      case 1: res = hh; break;
      case 2: res = hh * 12 / 10; break;
      case 3: res = hh * 4 / 3; break;
      case 4: res = hh * 3 / 2; break;
      case 5: res = hh * 16 / 9; break;
      case 6: res = hh * 5 / 4; break;
      default: res = hh * 2; break;
    }
    w = uint32_t(res);
  }
  *width = w;
  *height = h;
}

BitDepth parse_bit_depth(BitReader& br) {  // lib.rs:437-474
  BitDepth d;
  if (br.read_bool()) {
    d.float_sample = true;
    d.bits_per_sample = br.read_u32({32, 0}, {16, 0}, {24, 0}, {1, 6});
    d.exp_bits = br.read(4) + 1;
    JXLB_CHECK(d.exp_bits >= 2 && d.exp_bits <= 8, kErrBitstream, "invalid exp_bits");
    uint32_t mant = d.bits_per_sample - (d.exp_bits + 1);
    JXLB_CHECK(mant >= 2 && mant <= 23, kErrBitstream, "invalid mantissa bits");
  } else {
    d.bits_per_sample = br.read_u32({8, 0}, {10, 0}, {12, 0}, {1, 6});
    JXLB_CHECK(d.bits_per_sample <= 31, kErrBitstream, "invalid bits_per_sample");
  }
  return d;
}

std::string parse_name(BitReader& br) {  // jxl-oxide-common/src/lib.rs:296-309
  uint32_t len = br.read_u32({0, 0}, {0, 4}, {16, 5}, {48, 10});
  std::string s;
  for (uint32_t i = 0; i < len; ++i) s.push_back(char(br.read(8)));
  return s;
}

void parse_extensions(BitReader& br) {  // jxl-image/src/lib.rs:216-240
  uint64_t bits = br.read_u64();
  std::vector<uint64_t> lens;
  for (int i = 0; i < 64; ++i) {
    if (bits & 1) lens.push_back(br.read_u64());
    bits >>= 1;
  }
  for (uint64_t l : lens) br.skip(size_t(l));
  br.check();
}

ExtraChannelInfo parse_ec_info(BitReader& br) {  // lib.rs:303-345
  ExtraChannelInfo e;
  if (br.read_bool()) return e;  // default alpha channel
  uint32_t ty = br.read_enum();
  JXLB_CHECK(ty <= 6 || ty == 15 || ty == 16, kErrBitstream, "invalid extra channel type");
  e.type = ExtraChannelType(ty);
  e.bit_depth = parse_bit_depth(br);
  e.dim_shift = br.read_u32({0, 0}, {3, 0}, {4, 0}, {1, 3});
  e.name = parse_name(br);
  switch (e.type) {
    case ExtraChannelType::kAlpha: e.alpha_associated = br.read_bool(); break;
    case ExtraChannelType::kSpotColour:
      for (float& f : e.spot) f = br.read_f16();
      break;
    case ExtraChannelType::kCfa: e.cfa_channel = br.read_u32({1, 0}, {0, 2}, {3, 4}, {19, 8}); break;
    default: break;
  }
  return e;
}

int32_t parse_customxy_coord(BitReader& br) {
  return unpack_signed(br.read_u32({0, 19}, {524288, 19}, {1048576, 20}, {2097152, 21}));
}

ColourEncoding parse_colour_encoding(BitReader& br) {  // color.rs:21-58
  ColourEncoding c;
  if (br.read_bool()) return c;  // all_default
  c.want_icc = br.read_bool();
  uint32_t cs = br.read_enum();
  JXLB_CHECK(cs <= 3, kErrBitstream, "invalid colour space");
  c.colour_space = ColourSpace(cs);
  if (c.want_icc) return c;
  if (c.colour_space != ColourSpace::kXyb) {
    uint32_t wp = br.read_enum();
    JXLB_CHECK(wp == 1 || wp == 2 || wp == 10 || wp == 11, kErrBitstream, "invalid white point");
    c.white_point = WhitePointKind(wp);
    if (c.white_point == WhitePointKind::kCustom) {
      c.white_xy[0] = parse_customxy_coord(br);
      c.white_xy[1] = parse_customxy_coord(br);
    }
  }
  if (c.colour_space != ColourSpace::kXyb && c.colour_space != ColourSpace::kGrey) {
    uint32_t p = br.read_enum();
    JXLB_CHECK(p == 1 || p == 2 || p == 9 || p == 11, kErrBitstream, "invalid primaries");
    c.primaries = PrimariesKind(p);
    if (c.primaries == PrimariesKind::kCustom)
      for (auto& xy : c.primaries_xy) {
        xy[0] = parse_customxy_coord(br);
        xy[1] = parse_customxy_coord(br);
      }
  }
  if (br.read_bool()) {  // has_gamma
    c.tf = TransferFunctionKind::kGamma;
    c.gamma = br.read(24);
  } else {
    uint32_t tf = br.read_enum();
    JXLB_CHECK(tf == 1 || tf == 2 || tf == 8 || tf == 13 || tf == 16 || tf == 17 || tf == 18,
               kErrBitstream, "invalid transfer function");
    c.tf = TransferFunctionKind(tf);
  }
  c.rendering_intent = br.read_enum();
  JXLB_CHECK(c.rendering_intent <= 3, kErrBitstream, "invalid rendering intent");
  return c;
}

}  // namespace

OpsinInverseMatrix::OpsinInverseMatrix() {  // color.rs:610-628 (f32 literal arithmetic)
  const float m[3][3] = {{11.031566901960783f, -9.866943921568629f, -0.16462299647058826f},
                         {-3.254147380392157f, 4.418770392156863f, -0.16462299647058826f},
                         {-3.6588512862745097f, 2.7129230470588235f, 1.9459282392156863f}};
  for (int i = 0; i < 3; ++i)
    for (int j = 0; j < 3; ++j) inv_mat[i][j] = m[i][j];
  for (float& b : opsin_bias) b = -0.0037930732552754493f;
  quant_bias[0] = 1.0f - 0.05465007330715401f;
  quant_bias[1] = 1.0f - 0.07005449891748593f;
  quant_bias[2] = 1.0f - 0.049935103337343655f;
  quant_bias_numerator = 0.145f;
}

EpfParams::EpfParams() {  // filter.rs:79-103, 184-193
  const float lut[8] = {0.0f, 1.0f / 7.0f, 2.0f / 7.0f, 3.0f / 7.0f, 4.0f / 7.0f, 5.0f / 7.0f, 6.0f / 7.0f, 1.0f};
  for (int i = 0; i < 8; ++i) sharp_lut[i] = lut[i];
  channel_scale[0] = 40.0f, channel_scale[1] = 5.0f, channel_scale[2] = 3.5f;
  quant_mul = 0.46f, pass0_sigma_scale = 0.9f, pass2_sigma_scale = 6.5f, border_sad_mul = 2.0f / 3.0f;
  sigma_for_modular = 1.0f;
}

RestorationFilter::RestorationFilter() {
  for (auto& w : gab_weights) w[0] = 0.115169525f, w[1] = 0.061248592f;
}

ImageHeader default_image_header() {  // all-default metadata with the default upsampling weight tables
  ImageHeader h;
  h.up2_weight.assign(kDefaultUp2, kDefaultUp2 + 15);
  h.up4_weight.assign(kDefaultUp4, kDefaultUp4 + 55);
  h.up8_weight.assign(kDefaultUp8, kDefaultUp8 + 210);
  return h;
}

ImageHeader parse_image_header(BitReader& br) {
  ImageHeader h;
  JXLB_CHECK(br.read(16) == 0x0aff, kErrBitstream, "JPEG XL signature mismatch");
  parse_size(br, &h.width, &h.height);
  h.up2_weight.assign(kDefaultUp2, kDefaultUp2 + 15);
  h.up4_weight.assign(kDefaultUp4, kDefaultUp4 + 55);
  h.up8_weight.assign(kDefaultUp8, kDefaultUp8 + 210);
  bool all_default = br.read_bool();
  bool extra_fields = !all_default && br.read_bool();
  if (extra_fields) {
    h.orientation = 1 + br.read(3);
    h.have_intrinsic_size = br.read_bool();
    if (h.have_intrinsic_size) {
      uint32_t w, hh;
      parse_size(br, &w, &hh);
    }
    h.have_preview = br.read_bool();
    if (h.have_preview) parse_preview_size(br, &h.preview_width, &h.preview_height);
    h.have_animation = br.read_bool();
    if (h.have_animation) {
      h.tps_numerator = br.read_u32({100, 0}, {1000, 0}, {1, 10}, {1, 30});
      h.tps_denominator = br.read_u32({1, 0}, {1001, 0}, {1, 8}, {1, 10});
      h.num_loops = br.read_u32({0, 0}, {0, 3}, {0, 16}, {0, 32});
      h.have_timecodes = br.read_bool();
    }
  }
  if (!all_default) {
    h.bit_depth = parse_bit_depth(br);
    h.modular_16bit_buffers = br.read_bool();
    uint32_t num_extra = br.read_u32({0, 0}, {1, 0}, {2, 4}, {1, 12});
    for (uint32_t i = 0; i < num_extra; ++i) h.ec_info.push_back(parse_ec_info(br));
    h.xyb_encoded = br.read_bool();
    h.colour_encoding = parse_colour_encoding(br);
  }
  if (extra_fields) {  // ToneMapping (color.rs:312-319)
    if (!br.read_bool()) {
      h.tone_mapping.intensity_target = br.read_f16();
      h.tone_mapping.min_nits = br.read_f16();
      h.tone_mapping.relative_to_max_display = br.read_bool();
      h.tone_mapping.linear_below = br.read_f16();
    }
  }
  if (!all_default) parse_extensions(br);
  bool default_m = br.read_bool();
  if (!default_m && h.xyb_encoded) {
    if (!br.read_bool()) {  // OpsinInverseMatrix !all_default
      for (auto& row : h.opsin_inverse_matrix.inv_mat)
        for (float& v : row) v = br.read_f16();
      for (float& v : h.opsin_inverse_matrix.opsin_bias) v = br.read_f16();
      for (float& v : h.opsin_inverse_matrix.quant_bias) v = br.read_f16();
      h.opsin_inverse_matrix.quant_bias_numerator = br.read_f16();
    }
  }
  uint32_t cw_mask = default_m ? 0 : br.read(3);
  if (cw_mask & 1)
    for (float& v : h.up2_weight) v = br.read_f16();
  if (cw_mask & 2)
    for (float& v : h.up4_weight) v = br.read_f16();
  if (cw_mask & 4)
    for (float& v : h.up8_weight) v = br.read_f16();
  br.check();
  JXLB_CHECK(h.ec_info.size() <= 256, kErrBitstream, "num_extra too large");
  const ToneMapping& tm = h.tone_mapping;
  JXLB_CHECK(tm.intensity_target > 0.0f, kErrBitstream, "invalid intensity target");
  JXLB_CHECK(tm.min_nits >= 0.0f && tm.min_nits <= tm.intensity_target, kErrBitstream, "invalid min_nits");
  JXLB_CHECK(tm.linear_below >= 0.0f && !(tm.relative_to_max_display && tm.linear_below > 1.0f),
             kErrBitstream, "invalid linear_below");
  return h;
}

// jxl-color/src/icc/decode.rs:9-105 — the encoded ICC stream is entropy-decoded only to find
// where it ends; ICC colour management is outside the hot path (SURVEY §2.1 row 7).
void skip_icc_profile(BitReader& br) { read_icc_stream(br); }

std::vector<uint8_t> read_icc_stream(BitReader& br) {
  uint64_t enc_size = br.read_u64();
  JXLB_CHECK(enc_size <= (1u << 28), kErrBitstream, "encoded ICC profile too large");
  JXLB_CHECK(enc_size <= br.size_bits(), kErrEof, "encoded ICC profile larger than the codestream");
  std::vector<uint8_t> encoded;
  encoded.reserve(size_t(enc_size));
  EntropyCode code = parse_entropy_code(br, 41);
  EntropyReader dec(&code);
  dec.begin(br);
  uint8_t b1 = 0, b2 = 0;
  auto ctx = [](size_t idx, uint8_t b1, uint8_t b2) -> uint32_t {
    if (idx <= 128) return 0;
    auto is_alpha = [](uint8_t b) { return (b >= 'a' && b <= 'z') || (b >= 'A' && b <= 'Z'); };
    auto is_num = [](uint8_t b) { return (b >= '0' && b <= '9') || b == '.' || b == ','; };
    uint32_t p1, p2;
    if (is_alpha(b1)) p1 = 0;
    else if (is_num(b1)) p1 = 1;
    else if (b1 <= 1) p1 = 2 + b1;
    else if (b1 <= 15) p1 = 4;
    else if (b1 >= 241 && b1 <= 254) p1 = 5;
    else if (b1 == 255) p1 = 6;
    else p1 = 7;
    if (is_alpha(b2)) p2 = 0;
    else if (is_num(b2)) p2 = 1;
    else if (b2 <= 15) p2 = 2;
    else if (b2 >= 241) p2 = 3;
    else p2 = 4;
    return 1 + p1 + 8 * p2;
  };
  for (uint64_t idx = 0; idx < enc_size; ++idx) {
    uint32_t sym = dec.read_varint(br, ctx(size_t(idx), b1, b2));
    JXLB_CHECK(sym < 256, kErrBitstream, "invalid ICC stream");
    b2 = b1;
    b1 = uint8_t(sym);
    encoded.push_back(b1);
    br.check();
  }
  JXLB_CHECK(dec.finalize_ok(), kErrBitstream, "invalid ANS stream (ICC)");
  return encoded;
}

uint32_t FrameHeader::sample_width(uint32_t ups) const {  // header.rs:227-245
  uint32_t w = width;
  if (ups > 1) w = (w + ups - 1) / ups;
  if (lf_level > 0) {
    uint32_t div = 1u << (3 * lf_level);
    w = (w + div - 1) >> (3 * lf_level);
  }
  return w;
}
uint32_t FrameHeader::sample_height(uint32_t ups) const {
  uint32_t h = height;
  if (ups > 1) h = (h + ups - 1) / ups;
  if (lf_level > 0) {
    uint32_t div = 1u << (3 * lf_level);
    h = (h + div - 1) >> (3 * lf_level);
  }
  return h;
}

namespace {

bool test_full_image(int32_t x0, int32_t y0, uint32_t w, uint32_t h, const ImageHeader& ih) {  // header.rs:179-196
  if (x0 > 0 || y0 > 0) return false;
  int64_t right = int64_t(x0) + w, bottom = int64_t(y0) + h;
  return right >= int64_t(ih.width) && bottom >= int64_t(ih.height);
}
bool resets_canvas(BlendMode mode, bool have_crop, int32_t x0, int32_t y0, uint32_t w, uint32_t h,
                   const ImageHeader& ih) {  // header.rs:198-201
  return mode == BlendMode::kReplace && (!have_crop || test_full_image(x0, y0, w, h, ih));
}

BlendingInfo parse_blending_info(BitReader& br, bool has_extra, bool have_base, BlendMode base_mode,
                                 const FrameHeader& fh, const ImageHeader& ih) {  // header.rs:144-160
  BlendingInfo b;
  uint32_t m = br.read_u32({0, 0}, {1, 0}, {2, 0}, {3, 2});
  JXLB_CHECK(m <= 4, kErrBitstream, "invalid blend mode");
  b.mode = BlendMode(m);
  bool uses_alpha = has_extra && (b.mode == BlendMode::kBlend || b.mode == BlendMode::kMulAdd);
  if (uses_alpha) b.alpha_channel = br.read_u32({0, 0}, {1, 0}, {2, 0}, {3, 3});
  if (uses_alpha || b.mode == BlendMode::kMul) b.clamp = br.read_bool();
  BlendMode rm = have_base ? base_mode : b.mode;
  if (!resets_canvas(rm, fh.have_crop, fh.x0, fh.y0, fh.width, fh.height, ih)) b.source = br.read(2);
  return b;
}

}  // namespace

FrameHeader parse_frame_header(BitReader& br, const ImageHeader& ih) {
  FrameHeader f;
  const size_t num_ec = ih.ec_info.size();
  bool all_default = br.read_bool();
  if (!all_default) {
    f.frame_type = FrameType(br.read(2));
    f.encoding = Encoding(br.read(1));
    f.flags = br.read_u64();
    if (!ih.xyb_encoded) f.do_ycbcr = br.read_bool();
  }
  {
    bool actually_gray = f.encoding == Encoding::kModular && !f.do_ycbcr && !ih.xyb_encoded && ih.grayscale();
    f.encoded_color_channels = actually_gray ? 1 : 3;
  }
  if (f.do_ycbcr && !f.use_lf_frame())
    for (uint32_t& j : f.jpeg_upsampling) j = br.read(2);
  f.ec_upsampling.assign(num_ec, 1);
  if (!all_default && !f.use_lf_frame()) {
    f.upsampling = br.read_u32({1, 0}, {2, 0}, {4, 0}, {8, 0});
    for (size_t i = 0; i < num_ec; ++i) f.ec_upsampling[i] = br.read_u32({1, 0}, {2, 0}, {4, 0}, {8, 0});
  }
  f.group_size_shift = (f.encoding == Encoding::kModular) ? br.read(2) : 1;
  bool xyb_vardct = ih.xyb_encoded && f.encoding == Encoding::kVarDct;
  f.x_qm_scale = xyb_vardct ? 3 : 2;
  f.b_qm_scale = 2;
  if (!all_default && xyb_vardct) {
    f.x_qm_scale = br.read(3);
    f.b_qm_scale = br.read(3);
  }
  if (!all_default && f.frame_type != FrameType::kReferenceOnly) {  // Passes (header.rs:135-142)
    Passes& p = f.passes;
    p.num_passes = br.read_u32({1, 0}, {2, 0}, {3, 0}, {4, 3});
    if (p.num_passes != 1) {
      p.num_ds = br.read_u32({0, 0}, {1, 0}, {2, 0}, {3, 1});
      for (uint32_t i = 0; i + 1 < p.num_passes; ++i) p.shift.push_back(br.read(2));
      for (uint32_t i = 0; i < p.num_ds; ++i) p.downsample.push_back(br.read_u32({1, 0}, {2, 0}, {4, 0}, {8, 0}));
      for (uint32_t i = 0; i < p.num_ds; ++i) p.last_pass.push_back(br.read_u32({0, 0}, {1, 0}, {2, 0}, {0, 3}));
    }
  }
  if (f.frame_type == FrameType::kLfFrame) f.lf_level = 1 + br.read(2);
  if (!all_default && f.frame_type != FrameType::kLfFrame) f.have_crop = br.read_bool();
  const D cropd[4] = {{0, 8}, {256, 11}, {2304, 14}, {18688, 30}};
  if (f.have_crop && f.frame_type != FrameType::kReferenceOnly) {
    f.x0 = unpack_signed(br.read_u32(cropd[0], cropd[1], cropd[2], cropd[3]));
    f.y0 = unpack_signed(br.read_u32(cropd[0], cropd[1], cropd[2], cropd[3]));
  }
  f.width = ih.width;
  f.height = ih.height;
  if (f.have_crop) {
    f.width = br.read_u32(cropd[0], cropd[1], cropd[2], cropd[3]);
    f.height = br.read_u32(cropd[0], cropd[1], cropd[2], cropd[3]);
  }
  bool normal = f.frame_type == FrameType::kRegular || f.frame_type == FrameType::kSkipProgressive;
  f.ec_blending_info.assign(num_ec, BlendingInfo());
  if (!all_default && normal) {
    f.blending_info = parse_blending_info(br, num_ec != 0, false, BlendMode::kReplace, f, ih);
    for (size_t i = 0; i < num_ec; ++i)
      f.ec_blending_info[i] = parse_blending_info(br, num_ec != 0, true, f.blending_info.mode, f, ih);
    if (ih.have_animation) {
      f.duration = br.read_u32({0, 0}, {1, 0}, {0, 8}, {0, 32});
      if (ih.have_timecodes) f.timecode = br.read(32);
    }
    f.is_last = br.read_bool();
  } else {
    f.is_last = f.frame_type == FrameType::kRegular;
  }
  if (!all_default && f.frame_type != FrameType::kLfFrame && !f.is_last) f.save_as_reference = br.read(2);
  f.resets_canvas = resets_canvas(f.blending_info.mode, f.have_crop, f.x0, f.y0, f.width, f.height, ih);
  f.save_before_ct = !normal;
  if (!all_default &&
      (f.frame_type == FrameType::kReferenceOnly ||
       (f.resets_canvas && (!f.is_last && (f.duration == 0 || f.save_as_reference != 0) &&
                            f.frame_type != FrameType::kLfFrame)))) {
    f.save_before_ct = br.read_bool();
  }
  if (!all_default) {
    f.name = parse_name(br);
    // RestorationFilter (header.rs:162-167, filter.rs)
    RestorationFilter& rf = f.restoration_filter;
    if (!br.read_bool()) {
      rf.gab_enabled = br.read_bool();
      if (rf.gab_enabled && br.read_bool()) {  // custom
        for (auto& w : rf.gab_weights) {
          w[0] = br.read_f16();
          w[1] = br.read_f16();
          float s = 1.0f + (w[0] + w[1]) * 4.0f;
          JXLB_CHECK(!(std::abs(s) < 1.1920929e-7f), kErrBitstream, "gaborish weights sum to ~0");
        }
      }
      EpfParams& e = rf.epf;
      e.iters = br.read(2);
      if (e.iters != 0) {
        bool sharp_custom = (f.encoding == Encoding::kVarDct) ? br.read_bool() : false;
        if (sharp_custom)
          for (float& v : e.sharp_lut) v = br.read_f16();
        if (br.read_bool()) {  // weight_custom
          for (float& v : e.channel_scale) v = br.read_f16();
          br.read(32);
        }
        if (br.read_bool()) {  // sigma_custom
          if (f.encoding == Encoding::kVarDct) e.quant_mul = br.read_f16();
          e.pass0_sigma_scale = br.read_f16();
          e.pass2_sigma_scale = br.read_f16();
          e.border_sad_mul = br.read_f16();
        }
        if (f.encoding == Encoding::kModular) e.sigma_for_modular = br.read_f16();
      }
      parse_extensions(br);
    }
    parse_extensions(br);
  }
  f.bit_depth = ih.bit_depth;
  br.check();

  // Validation (jxl-frame/src/lib.rs:120-207)
  JXLB_CHECK(uint64_t(f.width) <= (1u << 30) && uint64_t(f.height) <= (1u << 30), kErrBitstream, "frame too large");
  JXLB_CHECK(uint64_t(f.width) * f.height <= (1ull << 40), kErrBitstream, "frame area too large");
  JXLB_CHECK(f.width != 0 && f.height != 0, kErrBitstream, "zero-sized frame");
  JXLB_CHECK(!(f.use_lf_frame() && f.lf_level >= 4), kErrBitstream, "lf_level out of range");
  uint32_t color_shift = ceil_log2_nonzero(f.upsampling);
  for (size_t i = 0; i < num_ec; ++i) {
    uint32_t es = ceil_log2_nonzero(f.ec_upsampling[i]), ds = ih.ec_info[i].dim_shift;
    JXLB_CHECK(es + ds >= color_shift, kErrBitstream, "EC upsampling < colour upsampling");
    JXLB_CHECK(es + ds <= 6, kErrBitstream, "cumulative EC upsampling too large");
    JXLB_CHECK(es + ds - color_shift <= 7 + f.group_size_shift, kErrBitstream, "dim_shift too large");
  }
  return f;
}

Toc parse_toc(BitReader& br, const FrameHeader& fh) {  // data/toc.rs:177-271
  Toc toc;
  uint32_t num_groups = fh.num_groups(), num_passes = fh.passes.num_passes;
  uint64_t entry_count = (num_groups == 1 && num_passes == 1)
                             ? 1
                             : 1ull + fh.num_lf_groups() + 1 + uint64_t(num_groups) * num_passes;
  JXLB_CHECK(entry_count <= 65536, kErrBitstream, "too many TOC entries");
  std::vector<uint32_t> perm;
  if (br.read_bool()) {
    EntropyCode code = parse_entropy_code(br, 8);
    EntropyReader dec(&code);
    dec.begin(br);
    perm = read_permutation(br, dec, uint32_t(entry_count), 0);
    JXLB_CHECK(dec.finalize_ok(), kErrBitstream, "invalid ANS stream (TOC permutation)");
  }
  br.zero_pad_to_byte();
  std::vector<uint32_t> sizes(entry_count);
  for (auto& s : sizes) s = br.read_u32({0, 10}, {1024, 14}, {17408, 22}, {4211712, 30});
  br.zero_pad_to_byte();
  br.check();
  std::vector<size_t> offsets(entry_count);
  size_t acc = br.pos() / 8;
  toc.data_begin = acc;
  for (size_t i = 0; i < entry_count; ++i) {
    offsets[i] = acc;
    acc += sizes[i];
    toc.total_size += sizes[i];
  }
  toc.entries.resize(entry_count);
  if (!perm.empty()) {
    // toc.rs:232-243: logical entry `idx` lives at bitstream position perm[idx]
    for (size_t idx = 0; idx < entry_count; ++idx) toc.entries[idx] = {offsets[perm[idx]], sizes[perm[idx]]};
  } else {
    for (size_t idx = 0; idx < entry_count; ++idx) toc.entries[idx] = {offsets[idx], sizes[idx]};
  }
  return toc;
}

size_t skip_preview_frame(const uint8_t* cs, size_t size, const ImageHeader& ih, size_t pos) {
  if (!ih.have_preview) return pos;
  BitReader br(cs, size, pos * 8);
  const FrameHeader fh = parse_frame_header(br, ih);
  const Toc toc = parse_toc(br, fh);
  const size_t end = toc.data_begin + toc.total_size;
  JXLB_CHECK(end <= size, kErrEof, "preview frame beyond end of codestream");
  return end;
}

}  // namespace jxlb
