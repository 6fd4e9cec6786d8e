// Frame-section syntax: LfGlobal, HfGlobal (dequantisation matrices, coefficient orders, HF
// entropy codes). Everything here is table construction; no sample/coefficient is decoded.
//
// Reference: crates/jxl-frame/src/data/{lf_global.rs,hf_global.rs},
//            crates/jxl-vardct/src/{lf.rs,dequant.rs,hf_pass.rs,dct_select.rs}.
#pragma once
#include <array>
#include <cstdint>
#include <functional>
#include <memory>
#include <vector>

#include "bitreader.h"
#include "entropy.h"
#include "headers.h"
#include "modular_syntax.h"

namespace jxlb {

// TransformType (dct_select.rs:1-33). Values are the bitstream's dct_select codes.
enum TransformType : uint8_t {
  kDct8 = 0, kHornuss, kDct2, kDct4, kDct16, kDct32, kDct16x8, kDct8x16, kDct32x8, kDct8x32,
  kDct32x16, kDct16x32, kDct4x8, kDct8x4, kAfv0, kAfv1, kAfv2, kAfv3, kDct64, kDct64x32, kDct32x64,
  kDct128, kDct128x64, kDct64x128, kDct256, kDct256x128, kDct128x256, kNumTransformTypes
};

struct TransformTypeInfo {
  uint8_t w8, h8;        // size in 8x8 blocks (dct_select_size, dct_select.rs:53-77)
  uint8_t param_index;   // dequant matrix set index (dct_select.rs:79-101)
  uint8_t order_id;      // coefficient order id (dct_select.rs:124-142)
  uint8_t transpose;     // need_transpose (dct_select.rs:144-154)
};
extern const TransformTypeInfo kTransformInfo[kNumTransformTypes];

struct HfBlockContext {  // lf.rs:52-121
  std::vector<uint32_t> qf_thresholds;
  std::vector<int32_t> lf_thresholds[3];
  std::vector<uint8_t> block_ctx_map;
  uint32_t num_block_clusters = 0;
};

// Patches (jxl-frame/src/data/patch.rs): rectangles of a reference frame blended onto this frame.
struct PatchBlending {
  uint32_t mode = 0;  // 0 None, 1 Replace, 2 Add, 3 Mul, 4 BlendAbove, 5 BlendBelow, 6 MulAddAbove, 7 MulAddBelow
  uint32_t alpha_channel = 0;
  bool clamp = false;
};
struct PatchTarget {
  int32_t x = 0, y = 0;
  std::vector<PatchBlending> blending;  // [0]: colour channels, [1 + i]: extra channel i
};
struct PatchRef {
  uint32_t ref_idx = 0, x0 = 0, y0 = 0, width = 0, height = 0;
  std::vector<PatchTarget> targets;
};

// Splines (jxl-frame/src/data/spline.rs): quantised control points + DCT32 of colour and thickness.
struct QuantSpline {
  std::vector<std::pair<int64_t, int64_t>> points;  // absolute control points
  int32_t xyb_dct[3][32];
  int32_t sigma_dct[32];
  uint64_t manhattan_distance = 0;  // of the control polygon; feeds the area limit
};

struct LfGlobalSyntax {
  bool has_splines = false;
  int32_t spline_quant_adjust = 0;
  std::vector<QuantSpline> splines;
  bool has_patches = false;
  std::vector<PatchRef> patches;
  // NoiseParameters (jxl-frame/src/data/noise.rs:2-17): strength LUT over intensity
  bool has_noise = false;
  float noise_lut[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  // LfChannelDequantization (lf.rs:8-16)
  float m_x_lf = 1.0f / 32.0f, m_y_lf = 1.0f / 4.0f, m_b_lf = 1.0f / 2.0f;
  // Quantizer (lf.rs:18-23)
  uint32_t global_scale = 0, quant_lf = 0;
  HfBlockContext hf_block_ctx;
  // LfChannelCorrelation (lf.rs:25-34)
  uint32_t colour_factor = 84;
  float base_correlation_x = 0.0f, base_correlation_b = 1.0f;
  uint32_t x_factor_lf = 128, b_factor_lf = 128;
  // GlobalModular (lf_global.rs:204-313)
  bool has_global_tree = false;
  MaTree global_tree;
  std::vector<ChannelInfo> gmodular_image_channels;  // before transforms
  bool has_gmodular = false;
  ModularStreamSyntax gmodular;  // header; channel data follows at the reader position
};
// Parses LfGlobal up to (not including) the GlobalModular channel data.
LfGlobalSyntax parse_lf_global(BitReader& br, const ImageHeader& ih, const FrameHeader& fh);

// 17 dequant matrix parameter sets -> raster weight matrices (dequant.rs:159-402, 586-658).
struct DequantMatrices {
  // matrices[set][channel] : width*height floats (row-major, `width` = dequant_matrix_size().0)
  std::vector<float> matrices[17][3];
  std::vector<float> matrices_tr[17][3];
  // JPEG transcodes: the raw DCT8 table's integer values per channel when its denominator is 1/2040, else empty
  // (jpeg_quant_values, dequant.rs:616-629, 718-720)
  std::vector<int32_t> jpeg[3];
  static void matrix_size(uint32_t set, uint32_t* w, uint32_t* h);
};

struct HfPassSyntax {  // hf_pass.rs:26-76
  // order[order_id][channel]: (x, y) pairs in the wide orientation; packed x | y << 16
  std::vector<uint32_t> order[13][3];
  EntropyCode code;
};

struct HfGlobalSyntax {
  // Shared, immutable: the all-default set (the usual case) is built once per process.
  std::shared_ptr<const DequantMatrices> dequant;
  bool dequant_all_default = false;
  uint32_t num_hf_presets = 0;
  std::vector<HfPassSyntax> passes;
};
// Decodes the inline three-channel Modular image of a raw dequant table (dequant.rs:537-559): `br` stands at the
// Modular header on entry and behind the channel data on return.
using RawTableDecoder = std::function<void(BitReader& br, uint32_t width, uint32_t height, uint32_t stream_index, std::vector<int32_t> out[3])>;
HfGlobalSyntax parse_hf_global(BitReader& br, const ImageHeader& ih, const FrameHeader& fh, const LfGlobalSyntax& lfg,
                               const RawTableDecoder& raw_decoder);

// Natural coefficient order for an order id (hf_pass.rs:156-231).
std::vector<uint32_t> natural_order(uint32_t order_id);
extern const uint16_t kOrderBlockSize[13][2];  // (bw, bh) in the wide orientation, hf_pass.rs:95-109

// x.powi(n) as computed by Rust on this target (compiler-rt __powisf2).
float powi_f32(float a, int32_t b);

}  // namespace jxlb
