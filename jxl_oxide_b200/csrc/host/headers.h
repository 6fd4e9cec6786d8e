// Codestream syntax structures produced by the host-side parser: image header, frame header,
// TOC. Field names follow the reference bundles so that a reader can line them up:
//   crates/jxl-image/src/{lib.rs,color.rs}, crates/jxl-frame/src/{header.rs,filter.rs,data/toc.rs}
#pragma once
#include <array>
#include <cstdint>
#include <string>
#include <vector>

#include "bitreader.h"

namespace jxlb {

struct BitDepth {  // jxl-image/src/lib.rs:430-436
  bool float_sample = false;
  uint32_t bits_per_sample = 8;
  uint32_t exp_bits = 0;
};

enum class ExtraChannelType : uint32_t {
  kAlpha = 0, kDepth, kSpotColour, kSelectionMask, kBlack, kCfa, kThermal, kNonOptional = 15, kOptional = 16
};

struct ExtraChannelInfo {  // jxl-image/src/lib.rs:289-345
  ExtraChannelType type = ExtraChannelType::kAlpha;
  BitDepth bit_depth;
  uint32_t dim_shift = 0;
  std::string name;
  bool alpha_associated = false;
  float spot[4] = {0, 0, 0, 0};
  uint32_t cfa_channel = 0;
};

enum class ColourSpace : uint32_t { kRgb = 0, kGrey = 1, kXyb = 2, kUnknown = 3 };
enum class WhitePointKind : uint32_t { kD65 = 1, kCustom = 2, kE = 10, kDci = 11 };
enum class PrimariesKind : uint32_t { kSrgb = 1, kCustom = 2, kBt2100 = 9, kP3 = 11 };
enum class TransferFunctionKind : uint32_t {
  kGamma = 0, kBt709 = 1, kUnknown = 2, kLinear = 8, kSrgb = 13, kPq = 16, kDci = 17, kHlg = 18
};

struct ColourEncoding {  // jxl-image/src/color.rs:9-58
  bool want_icc = false;
  ColourSpace colour_space = ColourSpace::kRgb;
  WhitePointKind white_point = WhitePointKind::kD65;
  int32_t white_xy[2] = {0, 0};
  PrimariesKind primaries = PrimariesKind::kSrgb;
  int32_t primaries_xy[3][2] = {};
  TransferFunctionKind tf = TransferFunctionKind::kSrgb;
  uint32_t gamma = 0;
  bool gamma_inverted = true;  // Gamma { g, inverted }: the bitstream codes 1/gamma (color.rs:582-587), an ICC 'para' curve gamma
  uint32_t rendering_intent = 1;
};

struct OpsinInverseMatrix {  // jxl-image/src/color.rs:606-628
  float inv_mat[3][3];
  float opsin_bias[3];
  float quant_bias[3];
  float quant_bias_numerator;
  OpsinInverseMatrix();
};

struct ToneMapping {
  float intensity_target = 255.0f, min_nits = 0.0f, linear_below = 0.0f;
  bool relative_to_max_display = false;
};

struct ImageHeader {  // jxl-image/src/lib.rs:17-60, 130-170
  uint32_t width = 0, height = 0;
  uint32_t orientation = 1;
  bool have_intrinsic_size = false, have_preview = false, have_animation = false;
  uint32_t preview_width = 0, preview_height = 0;
  uint32_t tps_numerator = 0, tps_denominator = 0, num_loops = 0;
  bool have_timecodes = false;
  BitDepth bit_depth;
  bool modular_16bit_buffers = true;
  std::vector<ExtraChannelInfo> ec_info;
  bool xyb_encoded = true;
  ColourEncoding colour_encoding;
  ToneMapping tone_mapping;
  OpsinInverseMatrix opsin_inverse_matrix;
  std::vector<float> up2_weight, up4_weight, up8_weight;  // 15 / 55 / 210
  bool grayscale() const { return colour_encoding.colour_space == ColourSpace::kGrey; }
  // Embedded ICC profile (want_icc): the decoded bytes, and the encoding an XYB image is rendered into - the enum
  // encoding equivalent to the profile when there is one, else sRGB / gray sRGB (jxl-render/src/lib.rs:104-150).
  std::vector<uint8_t> icc_profile;
  bool icc_is_enum = false;
  bool icc_is_cmyk = false;  // the profile's data colour space is CMYK: the black channel joins the image stream
  ColourEncoding icc_encoding;
};

enum class FrameType : uint32_t { kRegular = 0, kLfFrame = 1, kReferenceOnly = 2, kSkipProgressive = 3 };
enum class Encoding : uint32_t { kVarDct = 0, kModular = 1 };
enum class BlendMode : uint32_t { kReplace = 0, kAdd, kBlend, kMulAdd, kMul };

struct BlendingInfo {
  BlendMode mode = BlendMode::kReplace;
  uint32_t alpha_channel = 0;
  bool clamp = false;
  uint32_t source = 0;
};

struct Passes {
  uint32_t num_passes = 1, num_ds = 0;
  std::vector<uint32_t> shift, downsample, last_pass;
};

struct EpfParams {  // jxl-frame/src/filter.rs:60-103, 162-177
  uint32_t iters = 2;  // 0 = disabled
  float sharp_lut[8];
  float channel_scale[3];
  float quant_mul, pass0_sigma_scale, pass2_sigma_scale, border_sad_mul;
  float sigma_for_modular;
  EpfParams();
};

struct RestorationFilter {
  bool gab_enabled = true;
  float gab_weights[3][2];
  EpfParams epf;
  RestorationFilter();
};

struct FrameHeader {  // jxl-frame/src/header.rs:9-134
  FrameType frame_type = FrameType::kRegular;
  Encoding encoding = Encoding::kVarDct;
  uint64_t flags = 0;
  bool do_ycbcr = false;
  uint32_t encoded_color_channels = 3;
  uint32_t jpeg_upsampling[3] = {0, 0, 0};
  uint32_t upsampling = 1;
  std::vector<uint32_t> ec_upsampling;
  uint32_t group_size_shift = 1;
  uint32_t x_qm_scale = 3, b_qm_scale = 2;
  Passes passes;
  uint32_t lf_level = 0;
  bool have_crop = false;
  int32_t x0 = 0, y0 = 0;
  uint32_t width = 0, height = 0;
  BlendingInfo blending_info;
  std::vector<BlendingInfo> ec_blending_info;
  uint32_t duration = 0, timecode = 0;
  bool is_last = true;
  uint32_t save_as_reference = 0;
  bool resets_canvas = true;
  bool save_before_ct = false;
  std::string name;
  RestorationFilter restoration_filter;
  BitDepth bit_depth;

  // flags (header.rs:402-434)
  bool noise() const { return flags & 0x1; }
  bool patches() const { return flags & 0x2; }
  bool splines() const { return flags & 0x10; }
  bool use_lf_frame() const { return flags & 0x20; }
  bool skip_adaptive_lf_smoothing() const { return flags & 0x80; }

  // geometry helpers (header.rs:227-355)
  uint32_t sample_width(uint32_t ups) const;
  uint32_t sample_height(uint32_t ups) const;
  uint32_t color_sample_width() const { return sample_width(upsampling); }
  uint32_t color_sample_height() const { return sample_height(upsampling); }
  uint32_t group_dim() const { return 128u << group_size_shift; }
  uint32_t lf_group_dim() const { return group_dim() * 8; }
  uint32_t groups_per_row() const { return (color_sample_width() + group_dim() - 1) / group_dim(); }
  uint32_t group_rows() const { return (color_sample_height() + group_dim() - 1) / group_dim(); }
  uint32_t lf_groups_per_row() const { return (color_sample_width() + lf_group_dim() - 1) / lf_group_dim(); }
  uint32_t lf_group_rows() const { return (color_sample_height() + lf_group_dim() - 1) / lf_group_dim(); }
  uint32_t num_groups() const { return groups_per_row() * group_rows(); }
  uint32_t num_lf_groups() const { return lf_groups_per_row() * lf_group_rows(); }
  bool is_keyframe() const {
    return (frame_type == FrameType::kRegular || frame_type == FrameType::kSkipProgressive) &&
           (is_last || duration != 0);
  }
};

struct TocEntry {
  size_t offset = 0;  // byte offset from the start of the codestream
  uint32_t size = 0;
};

// TOC in *logical* order: [LfGlobal, LfGroup*, HfGlobal, GroupPass*] or a single entry (toc.rs).
struct Toc {
  std::vector<TocEntry> entries;
  size_t data_begin = 0, total_size = 0;
  bool single_entry() const { return entries.size() <= 1; }
};

ImageHeader parse_image_header(BitReader& br);
ImageHeader default_image_header();
// Parses an ICC profile's *presence* only: the encoded ICC stream is skipped (not decoded).
void skip_icc_profile(BitReader& br);
// The entropy-decoded (still command-coded) ICC stream (jxl-color/src/icc/decode.rs:9-81)
std::vector<uint8_t> read_icc_stream(BitReader& br);
FrameHeader parse_frame_header(BitReader& br, const ImageHeader& ih);
Toc parse_toc(BitReader& br, const FrameHeader& fh);
// The byte after the preview frame that starts at byte `pos` (the first byte after the image header), or `pos` when the
// image has no preview. Only its frame header and TOC are read, as jxl-oxide/src/lib.rs:384-411 does; the header's
// size fields default to the image's size, not the preview's.
size_t skip_preview_frame(const uint8_t* cs, size_t size, const ImageHeader& ih, size_t pos);

}  // namespace jxlb
