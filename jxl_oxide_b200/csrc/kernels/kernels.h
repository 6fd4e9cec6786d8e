// Launch wrappers for the sm_90a kernels. Plain C++ signatures over raw device pointers so that
// both the CUDA backend (cuda_backend.cu) and the stage-level C ABI (capi.cu) can call them.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

#include "../host/frame_syntax.h"
#include "../host/headers.h"
#include "../host/modular_syntax.h"
#include "common.cuh"
#include "jpeg_blocks.cuh"

namespace jxlb {

struct DevChannel {
  int32_t* ptr;  // top-left of the view
  uint32_t stride, w, h;
  int32_t hshift, vshift;
};

// Host-built per-channel decision plan: MA-tree nodes on the static properties (channel index,
// stream index, unavailable previous channels) are resolved ahead of time; when the remaining
// subtree tests a single property it is flattened to a lookup table (the reference does the same
// in FlatMaTree, crates/jxl-modular/src/ma.rs:241-330, 424-470).
struct DevChannelPlan {
  uint32_t root;                 // first node that needs a sample-dependent property
  int32_t lut_prop;              // -1: walk the tree from `root`; else property index of the LUT
  int32_t lut_base;
  uint32_t lut_len, lut_offset;  // u16 leaf-node indices at job.luts[lut_offset ...]
};

// Varblock placement of one LF group (HfMetadata post-processing, jxl-vardct/src/hf_metadata.rs:99-230; see
// placement.cuh): the (dct_select, hf_mul - 1) list in, the group's rectangle of the frame's block grids out.
struct DevPlacement {
  const int32_t* raw;  // nb_blocks x 2 (stride raw_stride); null: no placement
  uint32_t raw_stride, nb_blocks;
  uint32_t bw, bh;     // the LF group in 8x8 blocks
  uint32_t grid_stride;  // of the four grids below, which point at the group's top-left cell
  int32_t* blk_type;
  int32_t* blk_mul;
  float* epf_sigma;
  const int32_t* sharpness;
  float quant_mul_base;
  float sharp_lut[8];
  uint32_t has_epf;
};
// Shared memory one placement warp needs (placement.cuh: PlaceShared); a Modular launch with HfMetadata jobs reserves at
// least this much per CTA.
constexpr size_t kPlaceSharedBytes = 2112;

struct DevModularJob {
  uint64_t bit_pos, bit_limit;
  const MaNode* tree;
  uint32_t num_tree_nodes;
  const uint16_t* luts;
  uint32_t lut_total;
  DevEntropyCode code;
  uint32_t wp[11];  // p1 p2 p3a p3b p3c p3d p3e w0..w3
  uint32_t stream_index;
  uint32_t first_channel, num_channels;
  uint32_t dist_multiplier;
  uint32_t use_wp;
  int32_t* wp_scratch;   // 5 * max_width ints when use_wp
  uint32_t* lz_window;   // when code.lz77_enabled
  DevPlacement place;    // HfMetadata streams: the LF group's varblock placement, run by the stream's warp after the decode
};

struct DevView {
  void* ptr;  // top-left element
  uint32_t stride, w, h;
};

struct DevChannel;
struct DevChannelPlan;
// One CTA of a batched Modular launch: job `job` of the frame these tables belong to.
struct DevModularBatchRef {
  const uint8_t* cs;
  const DevModularJob* jobs;
  const DevChannel* channels;
  const DevChannelPlan* plans;
  uint64_t* end_bits;   // may be mapped host memory: each stream writes its two result words once, at its end
  int* status;
  uint32_t job;
  // Per-frame completion inside a shared launch: the stream that finishes last (device counter, zero on entry) writes
  // `done_seq` to the mapped host word `done_flag`. NULL counter: the launch's end is the only signal.
  uint32_t num_jobs;
  uint32_t* counter;
  uint32_t* done_flag;
  uint32_t done_seq, pad;
};

// Modular ------------------------------------------------------------------------------------
void launch_modular_decode(const uint8_t* codestream, const DevModularJob* jobs, const DevChannel* channels,
                           const DevChannelPlan* plans, uint64_t* end_bits, int* status, int num_jobs,
                           size_t smem_bytes, bool all_tables_staged, cudaStream_t stream,
                           unsigned long long* trace = nullptr);
void launch_signal_word(uint32_t* host_mapped_word, uint32_t value, cudaStream_t stream);
void launch_modular_decode_batch(const DevModularBatchRef* refs, int total, size_t smem_bytes, bool all_tables_staged,
                                 cudaStream_t stream);
// tracing aid: writes the device's %globaltimer (ns)
void launch_read_globaltimer(unsigned long long* out, cudaStream_t stream);
void launch_squeeze_inverse(DevView avg, DevView res, DevView out, bool horizontal, cudaStream_t stream);
// The channels of one Squeeze step in one launch (channels may differ in size; zero-sized outputs are skipped).
void launch_squeeze_inverse_batch(const DevView* avg, const DevView* res, const DevView* out, int n, bool horizontal,
                                  cudaStream_t stream);
void launch_rct_inverse(DevView a, DevView b, DevView c, uint32_t rct_type, cudaStream_t stream);
// Second pass of a delta palette (palette.rs:120-152): every channel is scanned in raster order and the samples marked
// in `mask` get `d_pred`'s prediction (from already final neighbours) added - a serial recurrence per channel.
constexpr int kMaxPaletteChannels = 16;  // colour + extra channels one palette transform may cover on the device
struct DevPaletteDeltaParams {
  DevView target[kMaxPaletteChannels];
  const uint8_t* mask;  // width x height, 1 = add the prediction
  uint32_t d_pred;
  uint32_t wp[11];      // WpHeader p1, p2, p3a..p3e, w0..w3 (d_pred == 6)
  int32_t* wp_rows;     // num_c * 5 * width ints of scratch (d_pred == 6)
};
void launch_palette_delta(DevPaletteDeltaParams p, int num_c, cudaStream_t stream);
void launch_palette_inverse(DevView palette, const DevView* targets, int num_c, int nb_colours, int bit_depth, int nb_deltas,
                            uint8_t* mask, int* status, cudaStream_t stream);
void launch_int_to_float(DevView v, uint32_t bits_per_sample, uint32_t exp_bits, bool float_sample, cudaStream_t stream);
void launch_modular_xyb(DevView y, DevView x, DevView b, float mx, float my, float mb, cudaStream_t stream);
void launch_fill_u32(uint32_t* p, size_t n, uint32_t value, cudaStream_t stream);

// VarDCT -------------------------------------------------------------------------------------
struct DevLfGroupRect {
  uint32_t bx0, by0, bw, bh;
};
struct DevFrame {  // frame-global grids (device pointers), all with stride == their width
  uint32_t width, height, bw, bh;      // pixels / 8x8 blocks
  uint32_t cw, ch;                     // coefficient plane size (bw*8, bh*8)
  uint32_t w64;                        // x_from_y / b_from_y stride
  int32_t* lf_quant[3];
  int32_t* x_from_y;
  int32_t* b_from_y;
  int32_t* sharpness;
  int32_t* blk_type;
  int32_t* blk_mul;
  float* epf_sigma;
  float* lf[3];
  uint32_t* coeff[3];
  // JPEG chroma subsampling (VarDctState::hshift / vshift): channel c keeps block (bx, by) at (bx >> hshift[c],
  // by >> vshift[c]) of its (full-size) planes
  uint32_t group_blocks;  // group_dim / 8
  uint8_t hshift[3], vshift[3], subsampled;
};
// The placement of HfMetadata streams with Modular transforms, whose lists are only final after the inverse transforms
// (the other HfMetadata streams place their varblocks in the stream kernel): one warp per job; status kDevBadLayout or
// kDevOk per job.
void launch_place_varblocks(const DevPlacement* jobs, int num_jobs, int* status, cudaStream_t stream);

struct DevHfParams {
  DevEntropyCode code;
  const uint32_t* orders;         // concatenated order tables (x | y << 16)
  uint32_t order_offset[13 * 3];  // [order_id * 3 + channel] into `orders`
  const uint8_t* block_ctx_map;
  uint32_t block_ctx_map_size;
  const int32_t* lf_thresholds;   // concatenated X, Y, B
  uint32_t num_lf_thr[3];
  uint32_t has_lf_quant;  // 0: the frame uses an LF frame, the LF part of every block context is 0
  const uint32_t* qf_thresholds;
  uint32_t num_qf_thr;
  uint32_t num_block_clusters, num_hf_presets, coeff_shift;
  uint32_t group_dim_blocks, groups_per_row;
};
struct DevHfJob {
  uint64_t bit_pos, bit_limit;
  uint32_t group_idx;
};
// Shared memory of the HF coefficient kernels: the ANS alias tables are staged when they take at most kHfAnsSmemBytes,
// the cluster maps of all HF presets together when they take at most kLaneCmapSmemBytes. The one-warp-per-stream kernel
// always stages the cluster maps, so larger ones run one thread per stream (hf_schedule in launch_tables.h).
constexpr uint32_t kHfAnsSmemBytes = 128 * 1024;
constexpr uint32_t kLaneCmapSmemBytes = 32 * 1024;
// One warp per stream, `warps_per_cta` (8, 16 or 32) streams per CTA sharing the staged tables.
void launch_decode_hf(const uint8_t* codestream, DevFrame f, DevHfParams p, const DevHfJob* jobs, uint64_t* end_bits,
                      int* status, int num_jobs, int first_pass, int warps_per_cta, cudaStream_t stream);
// Same contract, one thread per stream (kernels/hf_lanes.cuh); `streams_per_cta` in {64, 128}, `streams_per_warp` in
// {4, 8, 16, 32}: a CTA runs streams_per_cta * 32 / streams_per_warp threads, and the lanes past the first
// streams_per_warp of each warp only help stage the tables.
// `list` / `counts` come from launch_hf_block_list: per group (hf_block_list_count of them), its varblock origins in
// raster order with their transform type and context offset, group_dim_blocks^2 records apart, and their number.
// A code with LZ77 needs `lz_windows`: num_jobs windows of `lz_window_len` entries
// (hf_lz77_window_entries in launch_tables.h), stream i's at lz_windows + i * lz_window_len.
size_t hf_block_list_count(DevFrame f, DevHfParams p);
void launch_hf_block_list(DevFrame f, DevHfParams p, uint2* list, uint32_t* counts, cudaStream_t stream);
void launch_decode_hf_lanes(const uint8_t* codestream, DevFrame f, DevHfParams p, const uint2* list, const uint32_t* counts,
                            const DevHfJob* jobs, uint64_t* end_bits, int* status, int num_jobs, int first_pass,
                            int streams_per_cta, int streams_per_warp, cudaStream_t stream, uint32_t* lz_windows = nullptr,
                            uint32_t lz_window_len = 0);

struct DevLfDequantJob {
  DevLfGroupRect rect;
  float scale[3];
};
void launch_lf_dequant(DevFrame f, const DevLfDequantJob* jobs, int num_jobs, cudaStream_t stream);
void launch_lf_cfl(DevFrame f, float kx, float kb, cudaStream_t stream);
void launch_lf_smooth(DevFrame f, float* tmp[3], float lf_x, float lf_y, float lf_b, cudaStream_t stream);

struct DevDequantParams {
  const float* matrices;          // all 17 sets x 3 channels x {normal, transposed}
  uint32_t matrix_offset[17 * 3 * 2];  // [(set * 3 + c) * 2 + transposed]
  float quant_bias[3], quant_bias_numerator;
  float qm_scale[3];
  float global_scale;             // as f32
  float base_correlation_x, base_correlation_b, colour_factor;
};
void launch_hf_dequant_cfl(DevFrame f, DevDequantParams p, cudaStream_t stream);
// chroma upsampling of JPEG-transcoded frames (jxl-render/src/filter/ycbcr.rs:6-78); `in` is the subsampled part
void launch_upsample_jpeg(DevView in, DevView out, int horizontal, int vertical, cudaStream_t stream);
// `scratch`: hf_transform_scratch_bytes() of device memory for the per-size-class work lists
void launch_hf_transform(DevFrame f, void* scratch, const DevDequantParams* fused_dequant, cudaStream_t stream);
size_t hf_transform_scratch_bytes(uint32_t bw, uint32_t bh);

// Filters / colour ----------------------------------------------------------------------------
void launch_gaborish(DevView in, DevView out, float w0, float w1, cudaStream_t stream);
struct DevEpfParams {
  float channel_scale[3];
  float pass0_sigma_scale, pass2_sigma_scale, border_sad_mul, sigma_for_modular;
};
void launch_epf_step(const DevView in[3], const DevView out[3], const float* sigma, uint32_t sigma_stride,
                     DevEpfParams p, int step, cudaStream_t stream);
struct DevColorParams {
  float opsin_bias[3], cbrt_opsin_bias[3], itscale, matrix[9];
  int apply_srgb_tf;
  int apply_bt709_tf;
  // non-sRGB targets (ColorParams::second_stage): gamut map, second matrix, optional XyzToLuma, gamma TF
  int second_stage, to_luma;
  float luminances[3], matrix2[9], gamma;
  float pq_intensity_target;  // > 0: PQ inverse EOTF (tf/pq.rs:126-142)
};
void launch_xyb_to_rgb(DevView x, DevView y, DevView b, DevColorParams p, cudaStream_t stream);
// YCbCr -> RGB in place, planes Cb, Y, Cr (jxl-color/src/ycbcr.rs:40-56)
struct DevYcbcrParams {
  float y_offset, cr_to_r, cb_to_g, cr_to_g, cb_to_b;
};
void launch_ycbcr_to_rgb(DevView cb, DevView y, DevView cr, DevYcbcrParams p, cudaStream_t stream);
void launch_copy_rect(DevView src, DevView dst, cudaStream_t stream);
// One k-times upsampling pass (k = 2, 4, 8); `quarter`: (k/2)^2 kernels of 25 weights (device).
void launch_upsample(DevView in, DevView out, int k, const float* quarter, cudaStream_t stream);
// Every output layout of a frame (pack.cu, per-sample rules in pack.cuh): any number of f32 planes, read through channel
// and spot tables, to u8 / u16 / f32 samples interleaved (channel fastest) or planar (channel-major), with the orientation
// applied.
struct DevPackChannel {
  const float* plane;
  uint32_t stride;
};
struct DevPackSpot {
  const float* plane;
  uint32_t stride;
  float rgb[3];
  float solidity;
};
struct DevPackSpec {
  uint32_t num_channels, num_spots;
  uint32_t width, height;  // of the stored (un-oriented) planes
  uint32_t orientation;    // 1..8
  uint32_t sample_type;    // 0: u8, 1: u16, 2: f32
  uint32_t planar;         // 0: interleaved, 1: one plane per channel
};
// `channels` and `spots` are host tables of p.num_channels and p.num_spots entries. Up to kPackParamEntries of each go to
// the kernel by value; when either table is longer, the kernel reads `d_channels` and `d_spots`, their copies in device
// memory, instead (null otherwise).
constexpr uint32_t kPackParamEntries = 8;
void launch_pack(const DevPackSpec& p, const DevPackChannel* channels, const DevPackSpot* spots, const DevPackChannel* d_channels,
                 const DevPackSpot* d_spots, void* out, cudaStream_t stream);
// Rectangle blending (jxl-render/src/blend.rs:550-727), one CTA per job; modes 1 Replace, 2 Add, 3 Mul,
// 4 Blend, 5 MulAdd, 6 MixAlpha.
struct DevPatchJob {
  const float* src;
  float* dst;
  const float* base_alpha;  // nullptr: 0.0
  const float* new_alpha;   // nullptr: 0.0
  uint32_t src_stride, dst_stride, base_alpha_stride, new_alpha_stride, w, h, mode, clamp, premultiplied;
  uint32_t swapped;  // the patch sample takes the base role (BlendBelow / MulAddBelow, blend.rs:119-152)
};
void launch_blend_patches(const DevPatchJob* jobs, int num_jobs, cudaStream_t stream);
// Spline splatting (jxl-render/src/features/spline.rs:218-252): one thread per pixel walks the arc list in order.
struct DevSplineArc {
  float x, y, sigma, inv_sigma, value[3];
  int32_t xbegin, xend, ybegin, yend;
};
void launch_splat_splines(const DevView v[3], const DevSplineArc* arcs, int num_arcs, cudaStream_t stream);
// Noise synthesis (crates/jxl-render/src/features/noise.rs). `field`: three frame-sized scratch planes.
struct DevNoiseParams {
  float lut[9];
  float corr_x, corr_b;
  uint32_t group_dim;
  unsigned long long seed0;
};
// `field` holds three field_w x field_h planes (the frame size); noise is added over the views, which lie in the field's
// top-left corner.
void launch_add_noise(const DevView v[3], float* const field[3], uint32_t field_w, uint32_t field_h, DevNoiseParams p,
                      cudaStream_t stream);
// Gaborish -> EPF -> colour in one kernel (kernels/filters_fused.cu); `in` and `out` must not alias.
struct DevFusedFilterParams {
  int gab_enabled;
  float gab_w[3][2];
  int epf_iters;  // 0..3
  DevEpfParams epf;
  const float* sigma;  // per-8x8-block sigma grid, or nullptr for the constant sigma_for_modular
  uint32_t sigma_stride;
  int colour;  // apply XYB -> RGB to the final pixels
  DevColorParams col;
};
void launch_filters_fused(const DevView in[3], const DevView out[3], DevFusedFilterParams p, cudaStream_t stream);
bool fused_filters_supported(uint32_t width, uint32_t height);

// JPEG reconstruction: scan encoding of one scan (kernels/jpeg.cu, per-block code in jpeg_blocks.cuh). Bit offsets and
// byte counts are 64-bit exclusive sums over n + 1 entries (the last one is the total).
size_t jpeg_scan_temp_bytes(uint32_t max_items);
void launch_jpeg_lengths(const DevJpegScan& p, const uint32_t* huff, const uint32_t* ezr_block, const uint32_t* ezr_count,
                         uint64_t* lens, uint32_t* err, cudaStream_t s);
void launch_jpeg_scan_u64(const uint64_t* in, uint64_t* out, uint32_t n, void* temp, size_t temp_bytes, cudaStream_t s);
void launch_jpeg_scan_u32(const uint32_t* in, uint32_t* out, uint32_t n, void* temp, size_t temp_bytes, cudaStream_t s);
void launch_jpeg_intervals(const DevJpegScan& p, const uint64_t* boff, uint64_t* ibytes, uint64_t* ipad, cudaStream_t s);
void launch_jpeg_emit(const DevJpegScan& p, const uint32_t* huff, const uint32_t* ezr_block, const uint32_t* ezr_count,
                      const uint64_t* boff, const uint64_t* ibx, const uint64_t* ipx, const uint8_t* pad, uint32_t* words,
                      uint32_t* err, cudaStream_t s);
void launch_jpeg_ff_count(const uint32_t* words, uint64_t total_bytes, uint32_t nw, uint32_t* cnt, cudaStream_t s);
void launch_jpeg_stuff(const uint32_t* words, uint64_t total_bytes, uint32_t nw, const uint32_t* ffoff, const uint64_t* ibx,
                       uint32_t nint, uint8_t* out, cudaStream_t s);

}  // namespace jxlb
