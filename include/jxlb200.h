/* jxlb200 — C ABI of the H100-native JPEG XL decode hot path (libjxlb200.so).
 *
 * This is the boundary a jxl-oxide maintainer binds from Rust (`extern "C"`, see INTEGRATION.md).
 * No C++/torch types cross it: plain pointers, sizes and int status codes. All entry points are
 * re-entrant per decoder object; one decoder owns one CUDA stream and its HBM planes
 * (the reference renders frames concurrently behind `&self`, crates/jxl-render/src/state.rs:72-228).
 *
 * Error convention (reference: Result<T, jxl_render::Error>, crates/jxl-render/src/error.rs):
 *   0 = ok, JXLB_ERR_* otherwise; jxlb_last_error() returns the message. JXLB_ERR_UNSUPPORTED
 *   marks valid streams outside the implemented hot path — the Rust shim would route those to
 *   its own CPU renderer; this library itself has NO CPU fallback.
 */
#ifndef JXLB200_H_
#define JXLB200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

enum {
  JXLB_OK = 0,
  JXLB_ERR_BITSTREAM = 1,
  JXLB_ERR_UNSUPPORTED = 2,
  JXLB_ERR_EOF = 3,
  JXLB_ERR_CUDA = 4,
  JXLB_ERR_INVALID_ARG = 5,
  JXLB_ERR_DEVICE_DECODE = 6,
  JXLB_ERR_OUT_OF_MEMORY = 7 /* the allocation budget given to jxlb_decoder_create_ex would be exceeded */
};

typedef struct jxlb_decoder jxlb_decoder;

typedef struct {
  /* 0: the image's signalled colour encoding (sRGB transfer), 1: linear sRGB, 2: leave XYB.
   * Mirrors JxlImage::request_color_encoding (crates/jxl-oxide/src/lib.rs). */
  int32_t output_colour;
  uint32_t max_frames; /* 0 = all keyframes */
} jxlb_options;

typedef struct {
  uint32_t width, height;
  uint32_t num_channels; /* colour + extra */
  uint32_t num_color;
  uint32_t is_vardct;
  uint32_t duration;
} jxlb_frame_info;

typedef struct {
  uint32_t width, height, bits_per_sample, num_extra_channels, xyb_encoded, grayscale, orientation;
} jxlb_image_info;

/* Context lifetime. Replaces JxlImageBuilder/RenderContext construction
 * (crates/jxl-oxide/src/lib.rs:205-279, crates/jxl-render/src/lib.rs:35-130). */
int32_t jxlb_decoder_create(int32_t cuda_device, jxlb_decoder** out);
/* Same with an allocation budget in bytes of HBM for planes and temporaries (0 = unlimited): the counterpart of
 * AllocTracker::with_limit (crates/jxl-grid/src/alloc_tracker.rs:8-74, JxlImageBuilder::alloc_tracker). A decode that
 * would exceed it fails with JXLB_ERR_OUT_OF_MEMORY (the reference's Error::OutOfMemory) and frees what it had. */
int32_t jxlb_decoder_create_ex(int32_t cuda_device, uint64_t mem_limit_bytes, jxlb_decoder** out);
void jxlb_decoder_destroy(jxlb_decoder* dec);
const char* jxlb_last_error(const jxlb_decoder* dec);

/* Decode every keyframe of a codestream/container held in HOST memory. Replaces
 * JxlImage::render_frame -> jxl_render::render::render_frame
 * (crates/jxl-oxide/src/lib.rs:710-740, crates/jxl-render/src/render.rs:14-156) plus
 * RenderContext::postprocess_keyframe (crates/jxl-render/src/lib.rs:925-998).
 * Decoded planes (f32, planar, row-major) stay resident in HBM until jxlb_release_frames(). */
int32_t jxlb_decode(jxlb_decoder* dec, const uint8_t* data, size_t size, const jxlb_options* opt);
/* Keep an encoded image resident in HBM (slot id chosen by the caller) and decode from it: the
 * timed region of a device-resident benchmark then contains no host->device copy of the input. */
int32_t jxlb_preload(jxlb_decoder* dec, int32_t slot, const uint8_t* data, size_t size);
int32_t jxlb_decode_slot(jxlb_decoder* dec, int32_t slot, const jxlb_options* opt);
int32_t jxlb_image_get_info(const jxlb_decoder* dec, jxlb_image_info* info);
/* JxlImage::original_icc (crates/jxl-oxide/src/lib.rs:536-540): the embedded ICC profile, reconstructed from the
 * codestream (crates/jxl-color/src/icc/decode.rs). Returns its size in bytes (0 = none, -1 = bad argument) and copies
 * it when `dst` holds at least that many bytes. */
int64_t jxlb_image_original_icc(const jxlb_decoder* dec, uint8_t* dst, size_t dst_bytes);
int32_t jxlb_num_frames(const jxlb_decoder* dec);
int32_t jxlb_frame_get_info(const jxlb_decoder* dec, int32_t frame, jxlb_frame_info* info);
/* Render::image_planar equivalent (crates/jxl-oxide/src/lib.rs:1178-1203): copy one channel to
 * host memory, `dst_stride` in floats (>= width). */
int32_t jxlb_frame_channel_to_host(jxlb_decoder* dec, int32_t frame, int32_t channel, float* dst, size_t dst_stride);
/* Number of interleaved channels ImageStream::from_render selects (crates/jxl-oxide/src/fb.rs:184-283): the colour
 * channels plus the first alpha channel; -1 on a bad argument. */
int32_t jxlb_frame_stream_channels(const jxlb_decoder* dec, int32_t frame);
/* ImageStream::write_to_buffer::<u8 | u16 | f32> (crates/jxl-oxide/src/fb.rs:309-410): the stream's channels
 * interleaved (channel fastest) with the image orientation applied and spot-colour channels mixed into RGB
 * (fb.rs:335-362). sample_type 0 = u8, 1 = u16, 2 = f32; orientation 1..8 or 0 for the image header's. The
 * conversion runs on the device and `dst` (host) receives width*height*jxlb_frame_stream_channels() samples. */
int32_t jxlb_frame_write_to_buffer(jxlb_decoder* dec, int32_t frame, int32_t sample_type, int32_t orientation, void* dst,
                                   size_t dst_bytes);
/* Same conversion with a DEVICE destination (memory of this decoder's GPU, e.g. a torch tensor): the packed frame
 * never touches the host, which is how BASELINE config #5 hands decoded frames to an NCCL gather over NVLink. The call
 * returns after the packing kernel has finished, so the buffer may be used on any stream. */
int32_t jxlb_frame_write_to_device(jxlb_decoder* dec, int32_t frame, int32_t sample_type, int32_t orientation,
                                   void* device_dst, size_t dst_bytes);
/* Device-resident access: pointer to the channel's top-left sample and its row stride (floats). */
int32_t jxlb_frame_channel_device(jxlb_decoder* dec, int32_t frame, int32_t channel, float** dptr, uint32_t* stride);
int32_t jxlb_release_frames(jxlb_decoder* dec);
/* Blocks until all work queued on the decoder's stream has finished. */
int32_t jxlb_sync(jxlb_decoder* dec);
/* Number of kernels this decoder has launched so far. */
uint64_t jxlb_launch_count(const jxlb_decoder* dec);

/* Per-kernel device timing: when on, every launch is bracketed by CUDA events on the decoder's
 * stream; jxlb_profile_get returns launches and accumulated milliseconds for a kernel family
 * ("modular_decode", "decode_hf", "hf_transform", "epf_step", ...). Used by bench.py's roofline.
 * on == 2 selects a lighter trace instead: no events, the Modular stream kernels stamp the device
 * clock and the host logs launch / return times (see jxlb_timeline_get). on == 3: only the host wall clock per
 * planner phase ("host:lf_coeff", "host:pass_groups", ...; device waits included), no events at all. */
int32_t jxlb_set_profile(jxlb_decoder* dec, int32_t on);
int32_t jxlb_profile_get(jxlb_decoder* dec, const char* name, uint64_t* launches, double* total_ms);
int32_t jxlb_profile_reset(jxlb_decoder* dec);
/* Timeline of the profiled launches / host phases since the last reset: returns the number of
 * entries; when `index` is valid also its name and [t0, t1] in ms since a process-wide origin that
 * is common to all decoders (tracing aid, mirrors the reference's `tracing` spans). */
int32_t jxlb_timeline_get(jxlb_decoder* dec, int32_t index, char* name, size_t name_cap, double* t0_ms, double* t1_ms);

/* Test / debugging hook: snapshot intermediate stages ("lf", "hf_coeff", "hf_dequant", "idct",
 * "pre_filter", "gaborish", "epf", "rgb") of the LAST decoded frame to host memory. */
int32_t jxlb_set_capture(jxlb_decoder* dec, int32_t on);
/* Restoration filters + colour as one fused kernel (default, on) or stage by stage (off): the
 * stage-by-stage form also emits the "gaborish" / "epf" snapshots for stage-level parity tests. */
int32_t jxlb_set_fuse_filters(jxlb_decoder* dec, int32_t on);
/* Scheduling of the HF coefficient streams (one per 256x256 group and pass, jxl-frame/src/data/pass_group.rs:31): how
 * many streams share one CTA and its staged tables. 0 (default, = 16), 4 (= 8), 8, 16, 32: one warp per stream, all
 * presets' tables staged once per CTA - the shortest time for ONE frame; 64 / 128: one thread per stream (32 streams
 * per warp): slower for a frame alone, but 16 warps instead of 510, which is what a GPU full of frames wants
 * (jxlb_pipeline_create's default). Frames whose HF presets' cluster maps together exceed 32 KB always run one thread per
 * stream, 128 per CTA. Results are identical; the process-wide default comes from the environment variable JXLB_HF_LANES. */
int32_t jxlb_set_hf_streams_per_cta(jxlb_decoder* dec, int32_t streams);
int32_t jxlb_stage_count(const jxlb_decoder* dec, const char* name);
int32_t jxlb_stage_get(const jxlb_decoder* dec, const char* name, int32_t idx, uint32_t* width, uint32_t* height,
                       uint32_t* out /* may be NULL */);

/* ---- Stage-level entry points on DEVICE memory (planar f32 / i32, row-major, stride in elements).
 * They replace the reference's arch-dispatched `impls::` functions one-to-one. ---- */

/* filter::impls::apply_gabor_like (crates/jxl-render/src/filter/impls/generic.rs:39).
 * In-place on three planes; weights[c][0..1]. */
int32_t jxlb_gaborish(jxlb_decoder* dec, float* const planes[3], uint32_t width, uint32_t height, uint32_t stride,
                      const float weights[6]);
/* filter::impls::epf::<STEP> chain as driven by apply_epf (crates/jxl-render/src/filter/epf.rs:10-104).
 * sigma: one f32 per 8x8 block (stride sigma_stride) or NULL to use sigma_for_modular. */
typedef struct {
  uint32_t iters;
  float channel_scale[3];
  float pass0_sigma_scale, pass2_sigma_scale, border_sad_mul, sigma_for_modular;
} jxlb_epf_params;
int32_t jxlb_epf(jxlb_decoder* dec, float* const planes[3], uint32_t width, uint32_t height, uint32_t stride,
                 const float* sigma, uint32_t sigma_stride, const jxlb_epf_params* params);
/* ColorTransform XybToMixedLms + Matrix (+ sRGB OETF) (crates/jxl-color/src/convert.rs:287-308). */
int32_t jxlb_xyb_to_rgb(jxlb_decoder* dec, float* const planes[3], uint32_t width, uint32_t height, uint32_t stride,
                        const float opsin_bias[3], const float inv_matrix[9], float intensity_target, int32_t srgb_tf);
/* squeeze::inverse_h / inverse_v (crates/jxl-modular/src/transform/squeeze.rs:11, 755). `out` is a
 * separate (avg_w + res_w) x h (horizontal) or w x (avg_h + res_h) plane. */
int32_t jxlb_squeeze_inverse(jxlb_decoder* dec, const int32_t* avg, uint32_t avg_w, uint32_t avg_h, uint32_t avg_stride,
                             const int32_t* res, uint32_t res_w, uint32_t res_h, uint32_t res_stride, int32_t* out,
                             uint32_t out_stride, int32_t horizontal);
/* blend_single (crates/jxl-render/src/blend.rs:550-727) on one rectangle, in place on `base`: mode 1 Replace, 2 Add,
 * 3 Mul, 4 Blend, 5 MulAdd, 6 MixAlpha; `swapped` gives the patch the base role (the *Below patch modes). The alpha
 * planes (device pointers, same stride) may be null (read as 0). */
int32_t jxlb_blend(jxlb_decoder* dec, float* base, const float* patch, const float* base_alpha, const float* new_alpha,
                   uint32_t width, uint32_t height, uint32_t stride, int32_t mode, int32_t clamp, int32_t premultiplied,
                   int32_t swapped);
/* ---- Stage entry points of the decode seams (SURVEY 8b). Each decodes the first frame of `data` up to and including
 * one stage, copies that stage's planes into caller-owned DEVICE buffers (row pitch `stride` 32-bit words, NULL entries
 * skipped) and stops there: what a Rust-side test of the corresponding reference function compares against.
 * JXLB_ERR_UNSUPPORTED when the frame has no such stage (e.g. a Modular frame has no HF groups). ---- */
/* decode_pass_group -> write_hf_coeff for every group and pass (crates/jxl-frame/src/data/pass_group.rs:11-46,
 * crates/jxl-vardct/src/hf_coeff.rs:21-252): the accumulated quantised coefficients, i32, X / Y / B planes of
 * (8 * ceil(w / 8)) x (8 * ceil(h / 8)) samples (`width`, `height` out; call with coeff = NULL to size the buffers). */
int32_t jxlb_decode_hf_groups(jxlb_decoder* dec, const uint8_t* data, size_t size, int32_t* const coeff[3], uint32_t stride,
                              uint32_t* width, uint32_t* height);
/* dequant_hf_varblock_grouped + chroma_from_luma_hf_grouped + transform_varblocks
 * (crates/jxl-render/src/vardct/mod.rs:442-603, 681): the XYB samples before the restoration filters, f32. */
int32_t jxlb_dequant_idct(jxlb_decoder* dec, const uint8_t* data, size_t size, float* const planes[3], uint32_t stride,
                          uint32_t* width, uint32_t* height);
/* Modular channel decode of a frame's Modular image (global, LF-group and pass-group streams,
 * crates/jxl-modular/src/image.rs:456-593) BEFORE the inverse transforms: the coded channels in coding order, i32.
 * `dims` receives width, height per coded channel (up to dims_cap / 2), `num_coded` their number; call with
 * channels = NULL first to size the buffers. */
int32_t jxlb_modular_decode_groups(jxlb_decoder* dec, const uint8_t* data, size_t size, int32_t* const* channels,
                                   uint32_t num_channels, uint32_t stride, uint32_t* num_coded, uint32_t* dims, uint32_t dims_cap);
/* features::upsample (crates/jxl-render/src/features/upsampling.rs:45-132) with the default weight tables
 * (crates/jxl-image/src/lib.rs upsampling weights): `in` (w x h, stride in floats) -> `out` ((w * factor) x (h * factor)),
 * factor 2, 4 or 8; both DEVICE pointers. */
int32_t jxlb_upsample(jxlb_decoder* dec, const float* in, uint32_t width, uint32_t height, uint32_t stride, uint32_t factor,
                      float* out, uint32_t out_stride);
/* Decode a frame whose pieces come from separate buffers (what jxl-frame hands out: Frame::data(TocGroupKind) slices,
 * crates/jxl-frame/src/lib.rs:264-275, possibly straight from `jxlp` boxes): `header` holds the codestream from its
 * signature up to and including the frame's TOC, `sections[i]` the TOC entries in bitstream order. The library joins
 * them (one copy into the pinned staging buffer it uploads from anyway) and decodes as jxlb_decode does; it still parses
 * the headers and entropy-code tables itself, because the device tables are built from them. */
typedef struct {
  const uint8_t* data;
  size_t size;
} jxlb_section;
int32_t jxlb_decode_frame_sections(jxlb_decoder* dec, const uint8_t* header, size_t header_size, const jxlb_section* sections,
                                   size_t num_sections, const jxlb_options* opt);
/* rct::inverse_rct (crates/jxl-modular/src/transform/rct.rs:15). In place on three planes. */
int32_t jxlb_rct_inverse(jxlb_decoder* dec, int32_t* const planes[3], uint32_t width, uint32_t height, uint32_t stride,
                         uint32_t rct_type);

/* ---- Frame pipeline: many independent frames through one GPU ----
 * Replaces the reference's frame-level concurrency: jxl-oxide-cli renders keyframes through rayon's par_iter
 * (crates/jxl-oxide-cli/src/decode.rs:285-320), jxl-render spawns reference / LF frames eagerly
 * (crates/jxl-render/src/lib.rs:496-509). `workers` frames are in flight (one host thread each, pinned to the CPUs
 * local to the GPU). A frame's LF stage - two long, narrow entropy kernels - holds no CUDA stream: it rides in the
 * kernels of a batch service that merges the LF streams of all frames that are ready. Past the LF stage a frame holds
 * one of `heavy_frames` slots (a pre-allocated slab of HBM for its full-resolution planes + a CUDA stream). HBM use
 * grows with both counts: heavy_frames slabs of ~25 B/px, and per worker an LF arena and a memory pool. Frames are reported in completion order. */
typedef struct jxlb_pipeline jxlb_pipeline;
typedef struct {
  int32_t workers;            /* frames in flight (host threads); 0 = default (64) */
  int32_t heavy_frames;       /* heavy slots = slabs = CUDA streams for everything but the LF stage; 0 = default (16) */
  int32_t hf_streams_per_cta; /* 0 = 128 (one thread per HF stream), see jxlb_set_hf_streams_per_cta */
  int32_t no_affinity;        /* 1 = leave the worker threads' CPU affinity alone */
  int32_t batch_streams;      /* CUDA streams of the LF batch service; 0 = default (6). heavy_frames + batch_streams
                                 should stay below 32, the number of hardware queues a process can use concurrently */
} jxlb_pipeline_config;
int32_t jxlb_pipeline_create(int32_t cuda_device, const jxlb_pipeline_config* cfg, jxlb_pipeline** out);
void jxlb_pipeline_destroy(jxlb_pipeline* p);
const char* jxlb_pipeline_last_error(const jxlb_pipeline* p);
/* Encoded image kept resident in HBM for jxlb_pipeline_submit(data = NULL, slot). */
int32_t jxlb_pipeline_preload(jxlb_pipeline* p, int32_t slot, const uint8_t* data, size_t size);
/* Queue one frame: `data`/`size` host bytes (kept alive by the caller until the frame is reported) or data = NULL
 * and a preloaded `slot`. out_mode 0: decode only (planes are produced in HBM and released), 1: all channels as
 * planar f32 (channel-major, Render::image_planar), 2 / 3: ImageStream::write_to_buffer::<u8 / u16> (interleaved, image
 * orientation, packed on the device). The pixels go to host `dst` or, with dst = NULL, into a pinned buffer of the
 * pipeline's own ring (allocated NUMA-local to the GPU by the worker threads) that jxlb_pipeline_wait hands out and
 * jxlb_pipeline_release_output takes back. out_mode 4 / 5: the same u8 / u16 packing into DEVICE memory `dst` (of the
 * pipeline's GPU) - how BASELINE config #5 feeds an NCCL gather without touching the host. `tag` comes back from
 * jxlb_pipeline_wait. Never blocks. */
int32_t jxlb_pipeline_submit(jxlb_pipeline* p, const uint8_t* data, size_t size, int32_t slot, int32_t out_mode, void* dst,
                             size_t dst_bytes, uint64_t tag);
/* Blocks until a submitted frame has finished (its output, if any, is complete in `dst`); returns its tag and decode
 * status (+ message), and where its pixels are (`out`, `out_bytes`; may be NULL pointers when not wanted).
 * JXLB_ERR_INVALID_ARG when nothing is in flight. */
int32_t jxlb_pipeline_wait(jxlb_pipeline* p, uint64_t* tag, int32_t* status, void** out, size_t* out_bytes, char* err,
                           size_t err_cap);
/* Returns a pipeline-owned output buffer (from jxlb_pipeline_wait) to the ring. */
int32_t jxlb_pipeline_release_output(jxlb_pipeline* p, void* out);
uint64_t jxlb_pipeline_launch_count(const jxlb_pipeline* p);
int32_t jxlb_pipeline_workers(const jxlb_pipeline* p);
/* The i-th worker's decoder context (profiling knobs: jxlb_set_profile / jxlb_profile_get); NULL when out of range.
 * Must not be used to decode while frames are in flight. */
jxlb_decoder* jxlb_pipeline_decoder(jxlb_pipeline* p, int32_t index);

#ifdef __cplusplus
}
#endif
#endif /* JXLB200_H_ */
