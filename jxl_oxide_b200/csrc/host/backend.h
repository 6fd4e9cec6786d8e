// The seam between the host-side frame planner (syntax parsing + orchestration, this directory)
// and whatever executes the sample-level work. The product implements it with sm_90a CUDA
// kernels (csrc/cuda_backend.cu); the test oracle implements it with a scalar CPU restatement
// of the reference (oracle/). It plays the role of the reference's arch-dispatched `impls::`
// modules (crates/jxl-render/src/vardct/mod.rs:25-46, filter/impls.rs:3-25) plus the entropy
// seam `decode_pass_group` (crates/jxl-frame/src/data/pass_group.rs:31).
//
// All sample storage lives behind the backend as 32-bit "planes" (row-major, stride == width),
// the device mirror of jxl-grid's AlignedGrid (crates/jxl-grid/src/lib.rs:43-103).
#pragma once
#include <cstddef>
#include <cstdint>
#include <utility>
#include <vector>

#include "frame_syntax.h"
#include "headers.h"
#include "modular_syntax.h"

namespace jxlb {

struct View {  // rectangular window into a plane (MutableSubgrid, mutable_subgrid.rs:7-14)
  int plane = -1;
  uint32_t x0 = 0, y0 = 0, w = 0, h = 0;
};

struct ModularChannelTarget {
  View view;
  int32_t hshift = 0, vshift = 0;
};

struct LfGroupRect {  // geometry of one LF group in 8x8-block units
  uint32_t bx0 = 0, by0 = 0, bw = 0, bh = 0;
};

struct BlockInfoJob {  // HfMetadata post-processing (jxl-vardct/src/hf_metadata.rs:99-230)
  LfGroupRect rect;
  int raw_plane = -1;  // nb_blocks x 2
  uint32_t nb_blocks = 0;
};

// The varblock placement of one LF group with everything it writes: the group's rectangle of the frame's blk_type /
// blk_mul / epf_sigma planes (epf_sigma = quant_mul_base / hf_mul * sharp_lut[sharpness] when has_epf).
struct VarblockPlacement {
  BlockInfoJob group;  // nb_blocks == 0: no placement
  int blk_type = -1, blk_mul = -1, epf_sigma = -1, sharpness = -1;
  float quant_mul_base = 0.0f;
  float sharp_lut[8] = {};
  bool has_epf = false;
};

// One entropy-coded Modular channel-data stream (jxl-modular/src/image.rs:456-593).
struct ModularStreamJob {
  size_t bit_pos = 0;        // absolute bit offset into the codestream where channel data begins
  size_t bit_limit = 0;      // absolute end (bits) of the enclosing TOC section
  const MaTree* tree = nullptr;
  WpHeader wp;
  uint32_t stream_index = 0;  // MA property 1
  std::vector<ModularChannelTarget> channels;
  size_t end_bit = 0;         // out: absolute bit offset after the stream
  // HfMetadata stream without Modular transforms: its LF group's varblock placement, which a backend may run right
  // after the stream (the list and the sharpness rectangle are final then). It reports that in `placed`, and the
  // outcome in `layout_ok`; the planner runs the placements no backend ran through build_block_info().
  VarblockPlacement placement;
  bool placed = false;     // out
  bool layout_ok = true;   // out
};

// One HF coefficient stream (one pass of one 256x256 group), jxl-vardct/src/hf_coeff.rs:21-252.
struct HfGroupJob {
  size_t bit_pos = 0, bit_limit = 0;
  uint32_t group_idx = 0, pass_idx = 0;
  size_t end_bit = 0;  // out
};

// Frame-level state of a VarDCT frame. Planes are allocated by the planner.
struct VarDctState {
  uint32_t width = 0, height = 0;      // colour sample size
  uint32_t bw = 0, bh = 0;             // size in 8x8 blocks (ceil)
  uint32_t group_dim = 256, groups_per_row = 0, num_groups = 0;
  // LfGlobal / headers
  const LfGlobalSyntax* lfg = nullptr;
  const HfGlobalSyntax* hfg = nullptr;
  const FrameHeader* fh = nullptr;
  const ImageHeader* ih = nullptr;
  // planes
  // The frame takes its LF image from an earlier LF frame (FrameHeader flag use_lf_frame): there is no
  // quantised LF, hence no LF-threshold contexts (hf_coeff.rs:110-127) and no LF dequant / CfL / smoothing
  // (jxl-render/src/vardct/mod.rs:175-201).
  bool use_lf_frame = false;
  // JPEG chroma subsampling (ChannelShift::from_jpeg_upsampling, jxl-modular/src/param.rs:105-140): channel c (Cb, Y,
  // Cr) keeps one sample per (1 << hshift[c]) x (1 << vshift[c]) luma samples. Every VarDCT plane keeps its full
  // bw x bh allocation; a subsampled channel lives in the top-left part, block (bx, by) at (bx >> hshift, by >> vshift).
  // bw / bh are rounded up to even in a subsampled direction (hf_metadata.rs:70-80, vardct/mod.rs:83-95).
  uint32_t hshift[3] = {0, 0, 0}, vshift[3] = {0, 0, 0};
  bool subsampled = false;
  int lf_quant[3] = {-1, -1, -1};  // i32, X/Y/B, bw x bh
  int x_from_y = -1, b_from_y = -1;  // i32, ceil(w/64) x ceil(h/64)
  int sharpness = -1;                // i32, bw x bh
  int blk_type = -1;   // i32, bw x bh: dct_select at a varblock's top-left cell, else -(1 + dx + 32*dy)
  int blk_mul = -1;    // i32, bw x bh: hf_mul at the top-left cell
  int epf_sigma = -1;  // f32, bw x bh
  int lf[3] = {-1, -1, -1};     // f32 dequantised LF, bw x bh
  int coeff[3] = {-1, -1, -1};  // i32 coefficients -> f32 samples in place, (bw*8) x (bh*8)
};

inline VarblockPlacement varblock_placement(const VarDctState& st, const BlockInfoJob& group) {
  const EpfParams& epf = st.fh->restoration_filter.epf;
  VarblockPlacement p;
  p.group = group;
  p.blk_type = st.blk_type;
  p.blk_mul = st.blk_mul;
  p.epf_sigma = st.epf_sigma;
  p.sharpness = st.sharpness;
  p.quant_mul_base = epf.quant_mul * 65536.0f / float(st.lfg->global_scale);
  for (int i = 0; i < 8; ++i) p.sharp_lut[i] = epf.sharp_lut[i];
  p.has_epf = epf.iters > 0;
  return p;
}

// The part of an LF-group rectangle channel c covers (shift_size of an even-sized rectangle).
inline LfGroupRect shifted_rect(const LfGroupRect& r, uint32_t hshift, uint32_t vshift) {
  return LfGroupRect{r.bx0 >> hshift, r.by0 >> vshift, (r.bw + (1u << hshift) - 1) >> hshift, (r.bh + (1u << vshift) - 1) >> vshift};
}

struct LfDequantJob {  // copy_lf_dequant (jxl-render/src/vardct/mod.rs:387-412)
  LfGroupRect rect;
  float scale[3];  // X, Y, B
};

struct ColorParams {  // XYB -> (linear) sRGB, jxl-color/src/{xyb.rs,ciexyz.rs:81,tf/srgb.rs}
  float opsin_bias[3], cbrt_opsin_bias[3];
  float itscale;        // 255 / intensity_target
  float matrix[9];      // opsin inverse
  bool apply_srgb_tf;
  bool apply_bt709_tf = false;  // BT.709 OETF (jxl-color/src/tf/bt709.rs, generic fast_powf)
  // Output encodings other than D65 / sRGB primaries (jxl-color/src/convert.rs:397-466): gamut mapping of the linear
  // sRGB triple (gamut.rs:4-46; the XYB source is tagged Perceptual), then one matrix (linear sRGB -> XYZ -> adapted
  // white point -> target primaries, pre-multiplied like ColorTransform::optimize) and, for a Grey target, Y alone.
  bool second_stage = false;
  float luminances[3] = {0, 0, 0};  // of the sRGB primaries: the gamut mapper's luma weights
  float matrix2[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1};
  bool to_luma = false;             // XyzToLuma: channel 0 := Y, one output channel
  float gamma = 0.0f;               // > 0: v <= 1e-7 ? 0 : fast_powf(v, gamma) (tf.rs:11-70; Gamma and DCI)
  // PQ inverse EOTF (tf/pq.rs:126-142): linear 1.0 = `pq_intensity_target` nits; 0 = off
  float pq_intensity_target = 0.0f;
};

class Backend {
 public:
  virtual ~Backend() {}
  virtual void set_codestream(const uint8_t* data, size_t size) = 0;
  // Called at the start of every frame: table pointers handed over earlier may be stale now.
  virtual void new_frame() {}
  // Called once per frame right before the planner allocates the frame's full-resolution planes (coefficients,
  // Modular image channels), with an estimate of the bytes the rest of the frame needs. Everything before it (headers,
  // LF groups: 1/64 of the samples) is cheap in memory but long in latency; a backend may hold a frame here until a
  // heavy-stage slot is free.
  virtual void begin_heavy_stage(size_t /*bytes_hint*/) {}
  // planes
  virtual int alloc_plane(uint32_t w, uint32_t h, bool zero) = 0;
  virtual void free_plane(int id) = 0;
  virtual void download_rect(const View& v, void* dst) = 0;  // tightly packed w*h 32-bit words
  virtual void copy_rect(const View& src, const View& dst) = 0;
  // Modular (bit-exact integer path)
  virtual void decode_modular(std::vector<ModularStreamJob>& jobs) = 0;
  // returns a new plane holding the merged channel (jxl-modular/src/transform/squeeze.rs)
  virtual int squeeze_inverse(const View& avg, const View& residual, bool horizontal) = 0;
  // All channels of one Squeeze step (they are independent): a backend may run them as one launch.
  virtual std::vector<int> squeeze_inverse_many(const std::vector<std::pair<View, View>>& avg_res, bool horizontal) {
    std::vector<int> ids;
    for (const auto& p : avg_res) ids.push_back(squeeze_inverse(p.first, p.second, horizontal));
    return ids;
  }
  virtual void rct_inverse(const View v[3], uint32_t rct_type) = 0;  // transform/rct.rs
  // palette (transform/palette.rs): `targets[0]` holds indices on entry
  virtual void palette_inverse(const View& palette, const std::vector<View>& targets, const Transform& t,
                               const WpHeader& wp, uint32_t bit_depth) = 0;
  // int -> float sample conversion (jxl-render/src/image.rs:93-120, convert_modular_xyb)
  virtual void int_to_float(const View& v, const BitDepth& depth) = 0;
  virtual void modular_xyb_to_float(const View yxb[3], const float m_lf_unscaled[3]) = 0;
  // VarDCT
  // Varblock placement as a pass of its own, for the LF groups whose HfMetadata stream did not place them (see
  // ModularStreamJob::placement).
  virtual void build_block_info(VarDctState& st, const std::vector<BlockInfoJob>& jobs) = 0;
  virtual void decode_hf(VarDctState& st, std::vector<HfGroupJob>& jobs) = 0;
  virtual void lf_dequant(VarDctState& st, const std::vector<LfDequantJob>& jobs) = 0;
  virtual void lf_chroma_from_luma(VarDctState& st) = 0;   // vardct/mod.rs:544-568
  virtual void lf_adaptive_smoothing(VarDctState& st) = 0; // vardct/generic/mod.rs:11-103
  virtual void hf_dequant_cfl(VarDctState& st) = 0;        // vardct/mod.rs:442-542, 570-603
  virtual void hf_transform(VarDctState& st) = 0;          // vardct/transform_common.rs:11-75
  // restoration filters and colour, on the (width x height) window of three planes
  virtual void gaborish(const View v[3], const float weights[3][2]) = 0;
  virtual void epf(const View v[3], const View& sigma, const EpfParams& p, bool sigma_is_constant) = 0;
  // features/upsampling.rs: returns a new plane of (v.w << factor_log2) x (v.h << factor_log2) f32 samples
  virtual int upsample(const View& v, uint32_t factor_log2, const ImageHeader& ih) = 0;
  // Chroma upsampling of JPEG-transcoded frames (jxl-render/src/filter/ycbcr.rs:6-78): a 2x triangle filter
  // (0.75 / 0.25, edges replicated) horizontally and/or vertically; returns a new out_w x out_h f32 plane.
  virtual int upsample_jpeg(const View& v, bool horizontal, bool vertical, uint32_t out_w, uint32_t out_h) = 0;
  // Blending of equally sized f32 rectangles, in place on `dst` (jxl-render/src/blend.rs:550-727):
  //   op 1 Replace, 2 Add, 3 Mul (`clamp`: src clamped to [0, 1] first),
  //   op 4 Blend (alpha over), 5 MulAdd (dst + alpha * src), 6 MixAlpha (dst + src * (1 - dst)).
  // `base_alpha` / `new_alpha` (plane < 0 = absent -> 0.0) are read, never written, by a job.
  struct PatchJob {
    View src, dst;
    uint32_t mode;
    bool clamp;
    bool premultiplied = false;
    bool swapped = false;  // patch modes BlendBelow / MulAddBelow: the patch goes under the frame (blend.rs:119-152)
    View base_alpha, new_alpha;
  };
  virtual void blend_patches(const std::vector<PatchJob>& jobs) = 0;
  // Spline rendering (jxl-render/src/features/spline.rs:180-254): every arc sample adds a Gaussian-like blob
  // 0.25 * value[c] * sigma * factor^2 to the pixels of its bounding box, arcs in list order.
  struct SplineArc {
    float x, y, sigma, inv_sigma, value[3];
    int32_t xbegin, xend, ybegin, yend;
  };
  virtual void splat_splines(const View v[3], const std::vector<SplineArc>& arcs) = 0;
  // Noise synthesis (jxl-render/src/features/noise.rs:12-86): pseudo-random field per group_dim x group_dim
  // group (XorShift128+ seeded by `seed0` and the group origin), 5x5 high-pass, intensity-dependent strength
  // from `lut`, added to the XYB planes `v` (frame_w x frame_h).
  virtual void add_noise(const View v[3], const float lut[8], uint32_t group_dim, uint64_t seed0, float corr_x,
                         float corr_b) = 0;
  // The same with the field (its groups, seeds and mirroring) generated over field_w x field_h, of which the
  // top-left v[0].w x v[0].h part is added to `v`: an upsampled frame takes its noise at the coded resolution from the
  // field of the upsampled size (noise.rs:21-33, 94-100). The default runs add_noise() over field-sized copies of `v`.
  virtual void add_noise_in_frame(const View v[3], uint32_t field_w, uint32_t field_h, const float lut[8], uint32_t group_dim,
                                  uint64_t seed0, float corr_x, float corr_b);
  virtual void xyb_to_rgb(const View v[3], const ColorParams& p) = 0;
  // YCbCr -> RGB of JPEG-transcoded frames, planes in Cb, Y, Cr order (jxl-color/src/ycbcr.rs:40-56)
  struct YcbcrParams {
    float y_offset, cr_to_r, cb_to_g, cr_to_g, cb_to_b;
    YcbcrParams() {
      y_offset = 128.0f / 255.0f;
      cr_to_r = 1.402f;
      cb_to_g = -0.114f * 1.772f / 0.587f;
      cr_to_g = -0.299f * 1.402f / 0.587f;
      cb_to_b = 1.772f;
    }
  };
  virtual void ycbcr_to_rgb(const View v[3], const YcbcrParams& p) = 0;
  // Optional single-pass form of gaborish() + epf() + xyb_to_rgb() (`colour` may be null). Returns
  // false when the backend wants the stages issued one by one.
  virtual bool filters_colour_fused(const View /*v*/[3], const RestorationFilter& /*rf*/, const View& /*sigma*/,
                                    bool /*sigma_is_constant*/, const ColorParams* /*colour*/) {
    return false;
  }
  // Called once the quantised LF and HF coefficients of a VarDCT frame are complete, before anything dequantises them:
  // where JPEG reconstruction (host/jbrd.h) takes the frame.
  virtual void vardct_coefficients(const VarDctState& /*st*/) {}
  // Called by the planner at stage boundaries; a backend may snapshot planes for tests.
  virtual void stage_marker(const char* /*name*/, const View* /*views*/, int /*n*/) {}
  // Profiling hook: the planner finished the named host phase (wall clock since the previous mark).
  virtual void phase_mark(const char* /*name*/) {}
};

}  // namespace jxlb
