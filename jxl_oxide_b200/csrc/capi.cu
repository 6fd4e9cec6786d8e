// extern "C" boundary of libjxlb200.so — see include/jxlb200.h for the contract.
#include <cmath>
#include <cstdio>
#include <cstring>

#include "capi_internal.h"

using namespace jxlb;

namespace {

template <typename F>
int32_t guarded(jxlb_decoder* dec, F f) {
  try {
    f();
    return JXLB_OK;
  } catch (const Error& e) {
    if (dec) dec->error = e.what();
    return e.code;
  } catch (const std::exception& e) {
    if (dec) dec->error = e.what();
    return JXLB_ERR_INVALID_ARG;
  }
}

void release(jxlb_decoder* dec) {
  dec->jpeg.clear();
  dec->jpeg.shrink_to_fit();
  if (!dec->have_result) return;
  for (DecodedFrame& f : dec->res.frames)
    for (View& v : f.channels) dec->be->free_plane(v.plane);
  dec->res = DecodeResult();
  dec->have_result = false;
}

DevView raw_view(void* p, uint32_t w, uint32_t h, uint32_t stride) {
  DevView v;
  v.ptr = p;
  v.w = w;
  v.h = h;
  v.stride = stride;
  return v;
}

// Queues the copy of plane `v` to host `dst`, whose rows are `dst_stride` floats apart: one linear copy when both sides
// are contiguous, else a 2-D copy.
void plane_to_host(jxlb_decoder* dec, const View& v, float* dst, size_t dst_stride) {
  const DevView d = dec->be->dev_view(v);
  const cudaError_t e =
      d.stride == v.w && dst_stride == v.w
          ? cudaMemcpyAsync(dst, d.ptr, size_t(v.w) * v.h * 4, cudaMemcpyDeviceToHost, dec->be->stream())
          : cudaMemcpy2DAsync(dst, dst_stride * 4, d.ptr, size_t(d.stride) * 4, size_t(v.w) * 4, v.h, cudaMemcpyDeviceToHost,
                              dec->be->stream());
  JXLB_CHECK(e == cudaSuccess, kErrCuda, cudaGetErrorString(e));
}

}  // namespace

namespace jxlb {
jxlb_decoder* create_decoder_internal(int32_t device, uint64_t mem_limit, bool own_stream, int32_t* code) {
  auto dec = std::make_unique<jxlb_decoder>();
  try {
    dec->be.reset(new CudaBackend(device, own_stream));
    dec->be->set_mem_limit(mem_limit);
  } catch (const Error& e) {
    if (code) *code = e.code;
    return nullptr;
  }
  if (code) *code = JXLB_OK;
  return dec.release();
}

int32_t decode_resident(jxlb_decoder* dec, const uint8_t* cs, size_t size, const uint8_t* dptr, const jxlb_options* opt) {
  if (!dec || !cs || !dptr) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    release(dec);
    DecodeOptions o;
    if (opt) {
      o.output_colour = opt->output_colour;
      if (opt->max_frames) o.max_frames = opt->max_frames;
    }
    dec->be->use_resident_once(dptr);
    dec->res = decode_codestream(*dec->be, cs, size, o);
    dec->have_result = true;
  });
}

namespace {
struct KeyframeStop {  // thrown through decode_segment when the caller's keyframe callback fails
  int32_t code;
};
}  // namespace

int32_t decode_segment_keyframes(jxlb_decoder* dec, const uint8_t* cs, size_t size, const uint8_t* dptr, const FrameIndex& index,
                                 size_t seg, uint32_t last_keyframe, const jxlb_options* opt, bool keep_last,
                                 const std::function<int32_t(uint32_t)>& on_keyframe) {
  if (!dec || !cs) return JXLB_ERR_INVALID_ARG;
  int32_t stop = JXLB_OK;
  const int32_t rc = guarded(dec, [&] {
    release(dec);
    DecodeOptions o;
    if (opt) o.output_colour = opt->output_colour;
    if (dptr) dec->be->use_resident_once(dptr);
    try {
      decode_segment(*dec->be, cs, size, o, index, seg, last_keyframe, [&](uint32_t k, const ImageHeader& ih, DecodedFrame&& f) {
        dec->res.image_header = ih;
        dec->res.frames.push_back(std::move(f));
        dec->have_result = true;
        const int32_t r = on_keyframe(k);
        if (r != JXLB_OK) throw KeyframeStop{r};
        if (!(keep_last && k == last_keyframe)) release(dec);
      });
    } catch (const KeyframeStop& s) {
      stop = s.code;
    }
  });
  if (rc != JXLB_OK || stop != JXLB_OK) release(dec);
  return stop != JXLB_OK ? stop : rc;
}

int32_t frame_planar_to_host(jxlb_decoder* dec, int32_t frame, float* dst, size_t dst_bytes) {
  if (!dec || !dst || !dec->have_result || frame < 0 || size_t(frame) >= dec->res.frames.size()) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    const DecodedFrame& f = dec->res.frames[frame];
    size_t off = 0;  // in floats
    for (const View& v : f.channels) {
      const size_t n = size_t(v.w) * v.h;
      JXLB_CHECK((off + n) * 4 <= dst_bytes, kErrInvalidArg, "destination buffer too small");
      plane_to_host(dec, v, dst + off, v.w);
      off += n;
    }
    dec->be->sync();
  });
}
}  // namespace jxlb

extern "C" {

int32_t jxlb_decoder_create_ex(int32_t device, uint64_t mem_limit_bytes, jxlb_decoder** out) {
  if (!out) return JXLB_ERR_INVALID_ARG;
  int32_t code = JXLB_OK;
  *out = create_decoder_internal(device, mem_limit_bytes, true, &code);
  return code;
}

int32_t jxlb_decoder_create(int32_t device, jxlb_decoder** out) { return jxlb_decoder_create_ex(device, 0, out); }

int32_t jxlb_decode_frame_sections(jxlb_decoder* dec, const uint8_t* header, size_t header_size, const jxlb_section* sections,
                                   size_t num_sections, const jxlb_options* opt) {
  if (!dec || !header || (!sections && num_sections)) return JXLB_ERR_INVALID_ARG;
  size_t total = header_size;
  for (size_t i = 0; i < num_sections; ++i) {
    if (!sections[i].data && sections[i].size) return JXLB_ERR_INVALID_ARG;
    total += sections[i].size;
  }
  std::vector<uint8_t> joined;
  joined.reserve(total);
  joined.insert(joined.end(), header, header + header_size);
  for (size_t i = 0; i < num_sections; ++i) joined.insert(joined.end(), sections[i].data, sections[i].data + sections[i].size);
  return jxlb_decode(dec, joined.data(), joined.size(), opt);
}

namespace {
// Decodes `data` up to the named stage and copies that stage's planes into the caller's device buffers.
int32_t decode_until(jxlb_decoder* dec, const uint8_t* data, size_t size, const char* stage, void* const* dst, uint32_t num_dst,
                     uint32_t dst_stride, uint32_t* num_planes, uint32_t* dims, uint32_t dims_cap) {
  if (!dec || !data) return JXLB_ERR_INVALID_ARG;
  CudaBackend& be = *dec->be;
  be.stop_stage = stage;
  be.stop_dst.assign(dst ? dst : nullptr, dst ? dst + num_dst : nullptr);
  be.stop_stride = dst_stride;
  be.stop_dims.clear();
  bool reached = false;
  int32_t rc = guarded(dec, [&] {
    release(dec);
    dec->codestream = extract_codestream(data, size);
    DecodeOptions o;
    o.max_frames = 1;
    try {
      DecodeResult res = decode_codestream(be, dec->codestream.data(), dec->codestream.size(), o);
      for (DecodedFrame& f : res.frames)  // the stage does not exist in this frame: nothing to hand out
        for (View& v : f.channels) be.free_plane(v.plane);
    } catch (const StopDecode&) {
      reached = true;
    }
  });
  be.stop_stage.clear();
  be.stop_dst.clear();
  if (rc != JXLB_OK) return rc;
  if (!reached) {
    dec->error = std::string("the frame has no stage '") + stage + "'";
    return JXLB_ERR_UNSUPPORTED;
  }
  if (num_planes) *num_planes = uint32_t(be.stop_dims.size());
  for (size_t i = 0; dims && i < be.stop_dims.size() && 2 * i + 1 < dims_cap; ++i) {
    dims[2 * i] = be.stop_dims[i].first;
    dims[2 * i + 1] = be.stop_dims[i].second;
  }
  return JXLB_OK;
}
}  // namespace

int32_t jxlb_decode_hf_groups(jxlb_decoder* dec, const uint8_t* data, size_t size, int32_t* const coeff[3], uint32_t stride,
                              uint32_t* width, uint32_t* height) {
  uint32_t dims[6] = {0, 0, 0, 0, 0, 0}, n = 0;
  const int32_t rc = decode_until(dec, data, size, "hf_coeff", reinterpret_cast<void* const*>(coeff), coeff ? 3 : 0, stride, &n, dims, 6);
  if (rc == JXLB_OK && width) *width = dims[0];
  if (rc == JXLB_OK && height) *height = dims[1];
  return rc;
}

int32_t jxlb_jpeg_reconstruction_status(const uint8_t* data, size_t size) {
  if (!data) return JXLB_ERR_INVALID_ARG;
  try {
    return jpeg_reconstruction_status(data, size);
  } catch (const Error&) {  // a malformed container
    return 2;
  }
}

int32_t jxlb_reconstruct_jpeg(jxlb_decoder* dec, const uint8_t* data, size_t size, size_t* jpeg_size) {
  if (!dec || !data) return JXLB_ERR_INVALID_ARG;
  if (jpeg_size) *jpeg_size = 0;
  CudaBackend& be = *dec->be;
  const int32_t rc = guarded(dec, [&] {
    release(dec);
    JpegJob job = prepare_jpeg_job(data, size);
    dec->codestream = extract_codestream(data, size);
    DecodeOptions o;
    o.max_frames = 1;
    be.jpeg_job = &job;
    bool done = false;
    try {
      DecodeResult res = decode_codestream(be, dec->codestream.data(), dec->codestream.size(), o);
      for (DecodedFrame& f : res.frames)
        for (View& v : f.channels) be.free_plane(v.plane);
    } catch (const JpegDone&) {
      done = true;
    }
    be.jpeg_job = nullptr;
    JXLB_CHECK(done, kErrBitstream, "the first frame is not a VarDCT frame: its JPEG reconstruction data is invalid");
    dec->jpeg = std::move(job.out);
  });
  be.jpeg_job = nullptr;
  if (rc == JXLB_OK && jpeg_size) *jpeg_size = dec->jpeg.size();
  return rc;
}

int32_t jxlb_jpeg_copy(const jxlb_decoder* dec, uint8_t* dst, size_t dst_bytes) {
  if (!dec || !dst || dec->jpeg.empty() || dst_bytes < dec->jpeg.size()) return JXLB_ERR_INVALID_ARG;
  std::memcpy(dst, dec->jpeg.data(), dec->jpeg.size());
  return JXLB_OK;
}

int32_t jxlb_dequant_idct(jxlb_decoder* dec, const uint8_t* data, size_t size, float* const planes[3], uint32_t stride,
                          uint32_t* width, uint32_t* height) {
  uint32_t dims[6] = {0, 0, 0, 0, 0, 0}, n = 0;
  const int32_t rc = decode_until(dec, data, size, "idct", reinterpret_cast<void* const*>(planes), planes ? 3 : 0, stride, &n, dims, 6);
  if (rc == JXLB_OK && width) *width = dims[0];
  if (rc == JXLB_OK && height) *height = dims[1];
  return rc;
}

int32_t jxlb_modular_decode_groups(jxlb_decoder* dec, const uint8_t* data, size_t size, int32_t* const* channels,
                                   uint32_t num_channels, uint32_t stride, uint32_t* num_coded, uint32_t* dims, uint32_t dims_cap) {
  return decode_until(dec, data, size, "modular_coded", reinterpret_cast<void* const*>(channels), channels ? num_channels : 0, stride,
                      num_coded, dims, dims_cap);
}

int32_t jxlb_upsample(jxlb_decoder* dec, const float* in, uint32_t width, uint32_t height, uint32_t stride, uint32_t factor,
                      float* out, uint32_t out_stride) {
  if (!dec || !in || !out || (factor != 2 && factor != 4 && factor != 8) || !width || !height) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    ImageHeader ih = default_image_header();
    const std::vector<float>& weights = factor == 2 ? ih.up2_weight : (factor == 4 ? ih.up4_weight : ih.up8_weight);
    // per-phase 5x5 kernels from the symmetric weight list (upsampling.rs:66-92)
    const uint32_t k = factor, mat_n = k / 2;
    std::vector<float> quarter(size_t(k) * k / 4 * 25, 0.0f);
    size_t weight_idx = 0;
    for (uint32_t y = 0; y < 5 * mat_n; ++y) {
      const uint32_t mat_y = y / 5, ky = y % 5;
      for (uint32_t x = y; x < 5 * mat_n; ++x) {
        const uint32_t mat_x = x / 5, kx = x % 5;
        const float wv = weights[weight_idx++];
        quarter[size_t(mat_y * mat_n + mat_x) * 25 + ky * 5 + kx] = wv;
        quarter[size_t(mat_x * mat_n + mat_y) * 25 + kx * 5 + ky] = wv;
      }
    }
    cudaStream_t s = dec->be->stream();
    float* d_quarter = nullptr;
    JXLB_CHECK(cudaMallocAsync(&d_quarter, quarter.size() * 4, s) == cudaSuccess, kErrCuda, "cudaMallocAsync failed");
    JXLB_CHECK(cudaMemcpyAsync(d_quarter, quarter.data(), quarter.size() * 4, cudaMemcpyHostToDevice, s) == cudaSuccess, kErrCuda, "upload failed");
    launch_upsample(raw_view(const_cast<float*>(in), width, height, stride), raw_view(out, width * k, height * k, out_stride), int(k), d_quarter, s);
    cudaFreeAsync(d_quarter, s);
    dec->be->launches++;
    dec->be->sync();
  });
}

void jxlb_decoder_destroy(jxlb_decoder* dec) { delete dec; }

const char* jxlb_last_error(const jxlb_decoder* dec) { return dec ? dec->error.c_str() : "null decoder"; }

int32_t jxlb_decode(jxlb_decoder* dec, const uint8_t* data, size_t size, const jxlb_options* opt) {
  if (!dec || !data) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    release(dec);
    dec->codestream = extract_codestream(data, size);
    DecodeOptions o;
    if (opt) {
      o.output_colour = opt->output_colour;
      if (opt->max_frames) o.max_frames = opt->max_frames;
    }
    dec->res = decode_codestream(*dec->be, dec->codestream.data(), dec->codestream.size(), o);
    dec->have_result = true;
  });
}

int32_t jxlb_image_keyframes(const uint8_t* data, size_t size, int32_t* num_keyframes, int32_t* num_segments) {
  if (num_keyframes) *num_keyframes = 0;
  if (num_segments) *num_segments = 0;
  if (!data) return JXLB_ERR_INVALID_ARG;
  try {
    const std::vector<uint8_t> cs = extract_codestream(data, size);
    const FrameIndex index = index_frames(cs.data(), cs.size());
    if (num_keyframes) *num_keyframes = int32_t(index.num_keyframes);
    if (num_segments) *num_segments = int32_t(index.segments.size());
    return index.error;
  } catch (const Error& e) {
    return e.code;
  } catch (const std::exception&) {
    return JXLB_ERR_INVALID_ARG;
  }
}

int32_t jxlb_decode_keyframe(jxlb_decoder* dec, const uint8_t* data, size_t size, const jxlb_options* opt, int32_t keyframe) {
  if (!dec || !data || keyframe < 0) return JXLB_ERR_INVALID_ARG;
  FrameIndex index;
  const int32_t rc = guarded(dec, [&] {
    release(dec);
    dec->codestream = extract_codestream(data, size);
    index = index_frames(dec->codestream.data(), dec->codestream.size());
    JXLB_CHECK(uint32_t(keyframe) < index.num_keyframes, kErrInvalidArg, "keyframe index out of range");
  });
  if (rc != JXLB_OK) return rc;
  return decode_segment_keyframes(dec, dec->codestream.data(), dec->codestream.size(), nullptr, index,
                                  index.segment_of(uint32_t(keyframe)), uint32_t(keyframe), opt, true,
                                  [](uint32_t) { return JXLB_OK; });
}

int32_t jxlb_preload(jxlb_decoder* dec, int32_t slot, const uint8_t* data, size_t size) {
  if (!dec || !data) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    // build the new copy first: a failure (malformed container, out of memory) leaves the slot as it was
    std::vector<uint8_t> cs = extract_codestream(data, size);
    uint8_t* dptr = dec->be->upload_resident(cs.data(), cs.size());
    jxlb_decoder::Slot& s = dec->slots[slot];
    if (s.dptr) cudaFree(s.dptr);
    s.codestream = std::move(cs);
    s.dptr = dptr;
  });
}

int32_t jxlb_decode_slot(jxlb_decoder* dec, int32_t slot, const jxlb_options* opt) {
  if (!dec) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    auto it = dec->slots.find(slot);
    JXLB_CHECK(it != dec->slots.end(), kErrInvalidArg, "unknown preload slot");
    release(dec);
    DecodeOptions o;
    if (opt) {
      o.output_colour = opt->output_colour;
      if (opt->max_frames) o.max_frames = opt->max_frames;
    }
    dec->be->use_resident_once(it->second.dptr);
    dec->res = decode_codestream(*dec->be, it->second.codestream.data(), it->second.codestream.size(), o);
    dec->have_result = true;
  });
}

int32_t jxlb_image_get_info(const jxlb_decoder* dec, jxlb_image_info* info) {
  if (!dec || !info || !dec->have_result) return JXLB_ERR_INVALID_ARG;
  const ImageHeader& ih = dec->res.image_header;
  info->width = ih.width;
  info->height = ih.height;
  info->bits_per_sample = ih.bit_depth.bits_per_sample;
  info->num_extra_channels = uint32_t(ih.ec_info.size());
  info->xyb_encoded = ih.xyb_encoded;
  info->grayscale = ih.grayscale();
  info->orientation = ih.orientation;
  return JXLB_OK;
}

int64_t jxlb_image_original_icc(const jxlb_decoder* dec, uint8_t* dst, size_t dst_bytes) {
  if (!dec || !dec->have_result) return -1;
  const std::vector<uint8_t>& icc = dec->res.image_header.icc_profile;
  if (dst && dst_bytes >= icc.size() && !icc.empty()) std::memcpy(dst, icc.data(), icc.size());
  return int64_t(icc.size());
}

int32_t jxlb_num_frames(const jxlb_decoder* dec) { return (dec && dec->have_result) ? int32_t(dec->res.frames.size()) : 0; }

int32_t jxlb_frame_get_info(const jxlb_decoder* dec, int32_t frame, jxlb_frame_info* info) {
  if (!dec || !info || !dec->have_result || frame < 0 || size_t(frame) >= dec->res.frames.size()) return JXLB_ERR_INVALID_ARG;
  const DecodedFrame& f = dec->res.frames[frame];
  info->width = f.width;
  info->height = f.height;
  info->num_channels = uint32_t(f.channels.size());
  info->num_color = f.num_color;
  info->is_vardct = f.header.encoding == Encoding::kVarDct;
  info->duration = f.header.duration;
  return JXLB_OK;
}

int32_t jxlb_frame_channel_to_host(jxlb_decoder* dec, int32_t frame, int32_t channel, float* dst, size_t dst_stride) {
  if (!dec || !dst || !dec->have_result || frame < 0 || size_t(frame) >= dec->res.frames.size()) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    const DecodedFrame& f = dec->res.frames[frame];
    JXLB_CHECK(channel >= 0 && size_t(channel) < f.channels.size(), kErrInvalidArg, "channel out of range");
    const View& v = f.channels[channel];
    JXLB_CHECK(dst_stride >= v.w, kErrInvalidArg, "dst_stride too small");
    plane_to_host(dec, v, dst, dst_stride);
    dec->be->sync();
  });
}

static_assert(int(JXLB_LAYOUT_STREAM) == kWriteStream && int(JXLB_LAYOUT_STREAM_NO_ALPHA) == kWriteStreamNoAlpha &&
                  int(JXLB_LAYOUT_ALL_INTERLEAVED) == kWriteAllInterleaved && int(JXLB_LAYOUT_ALL_PLANAR) == kWriteAllPlanar,
              "the ABI's layout numbers are the planner's");

namespace {
WritePlan frame_write_plan(const jxlb_decoder* dec, int32_t frame, const jxlb_write_spec& spec) {
  JXLB_CHECK(dec->have_result && frame >= 0 && size_t(frame) < dec->res.frames.size(), kErrInvalidArg, "no such frame");
  return plan_write(dec->res.image_header, dec->res.frames[size_t(frame)], spec.layout, spec.sample_type, spec.orientation,
                    spec.render_spot_colour != 0);
}
}  // namespace

int32_t jxlb_frame_write_size(jxlb_decoder* dec, int32_t frame, const jxlb_write_spec* spec, uint32_t* num_channels,
                              uint64_t* bytes) {
  if (!dec || !spec) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    const WritePlan w = frame_write_plan(dec, frame, *spec);
    if (num_channels) *num_channels = uint32_t(w.layout.channels.size());
    if (bytes) *bytes = w.bytes;
  });
}

int32_t jxlb_frame_write_ex(jxlb_decoder* dec, int32_t frame, const jxlb_write_spec* spec, void* dst, size_t dst_bytes,
                            int32_t dst_on_device) {
  if (!dec || !spec || !dst) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    const WritePlan w = frame_write_plan(dec, frame, *spec);
    JXLB_CHECK(dst_bytes >= w.bytes, kErrInvalidArg, "destination buffer too small");
    const DecodedFrame& f = dec->res.frames[size_t(frame)];
    DevPackSpec p;
    p.num_channels = uint32_t(w.layout.channels.size());
    p.num_spots = uint32_t(w.layout.spots.size());
    p.width = w.width;
    p.height = w.height;
    p.orientation = w.orientation;
    p.sample_type = w.sample_type;
    p.planar = w.planar ? 1 : 0;
    std::vector<DevPackChannel> channels;
    for (size_t c : w.layout.channels) {
      const DevView d = dec->be->dev_view(f.channels[c]);
      channels.push_back(DevPackChannel{static_cast<const float*>(d.ptr), d.stride});
    }
    std::vector<DevPackSpot> spots;
    for (const StreamSpot& s : w.layout.spots) {
      const DevView d = dec->be->dev_view(f.channels[s.channel]);
      spots.push_back(DevPackSpot{static_cast<const float*>(d.ptr), d.stride, {s.rgb[0], s.rgb[1], s.rgb[2]}, s.solidity});
    }
    dec->be->pack(p, channels, spots, dst, w.bytes, dst_on_device != 0);
  });
}

// ImageStream::write_to_buffer is the stream layout with spot colours mixed.
int32_t jxlb_frame_write_to_buffer(jxlb_decoder* dec, int32_t frame, int32_t sample_type, int32_t orientation, void* dst,
                                   size_t dst_bytes) {
  const jxlb_write_spec spec{JXLB_LAYOUT_STREAM, sample_type, orientation, 1};
  return jxlb_frame_write_ex(dec, frame, &spec, dst, dst_bytes, 0);
}

int32_t jxlb_frame_write_to_device(jxlb_decoder* dec, int32_t frame, int32_t sample_type, int32_t orientation, void* device_dst,
                                   size_t dst_bytes) {
  const jxlb_write_spec spec{JXLB_LAYOUT_STREAM, sample_type, orientation, 1};
  return jxlb_frame_write_ex(dec, frame, &spec, device_dst, dst_bytes, 1);
}

int32_t jxlb_frame_stream_channels(const jxlb_decoder* dec, int32_t frame) {
  if (!dec || !dec->have_result || frame < 0 || size_t(frame) >= dec->res.frames.size()) return -1;
  return int32_t(stream_layout(dec->res.image_header, dec->res.frames[frame]).channels.size());
}

int32_t jxlb_frame_channel_device(jxlb_decoder* dec, int32_t frame, int32_t channel, float** dptr, uint32_t* stride) {
  if (!dec || !dptr || !stride || !dec->have_result || frame < 0 || size_t(frame) >= dec->res.frames.size()) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    const DecodedFrame& f = dec->res.frames[frame];
    JXLB_CHECK(channel >= 0 && size_t(channel) < f.channels.size(), kErrInvalidArg, "channel out of range");
    DevView d = dec->be->dev_view(f.channels[channel]);
    *dptr = static_cast<float*>(d.ptr);
    *stride = d.stride;
  });
}

int32_t jxlb_release_frames(jxlb_decoder* dec) {
  if (!dec) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] { release(dec); });
}

int32_t jxlb_sync(jxlb_decoder* dec) {
  if (!dec) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] { dec->be->sync(); });
}

uint64_t jxlb_launch_count(const jxlb_decoder* dec) { return dec ? dec->be->launches : 0; }

int32_t jxlb_set_profile(jxlb_decoder* dec, int32_t on) {
  if (!dec) return JXLB_ERR_INVALID_ARG;
  dec->be->host_phases = on == 3;   // host wall clock per planner phase only
  dec->be->profile = on == 1;       // CUDA events around every launch + host phase clock
  dec->be->trace_device = on == 2;  // no events: device-clock stamps in the stream kernels + host launch/return times
  return JXLB_OK;
}

int32_t jxlb_profile_get(jxlb_decoder* dec, const char* name, uint64_t* launches, double* total_ms) {
  if (!dec || !name || !launches || !total_ms) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    dec->be->sync();
    auto it = dec->be->profile_acc.find(name);
    *launches = it == dec->be->profile_acc.end() ? 0 : it->second.first;
    *total_ms = it == dec->be->profile_acc.end() ? 0.0 : it->second.second;
  });
}

int32_t jxlb_timeline_get(jxlb_decoder* dec, int32_t index, char* name, size_t name_cap, double* t0_ms, double* t1_ms) {
  if (!dec) return -1;
  int32_t n = -1;
  guarded(dec, [&] {
    dec->be->sync();
    n = int32_t(dec->be->timeline.size());
    if (index >= 0 && index < n && name && name_cap && t0_ms && t1_ms) {
      const auto& e = dec->be->timeline[size_t(index)];
      std::snprintf(name, name_cap, "%s", e.name.c_str());
      *t0_ms = e.t0_ms;
      *t1_ms = e.t1_ms;
    }
  });
  return n;
}

int32_t jxlb_profile_reset(jxlb_decoder* dec) {
  if (!dec) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    dec->be->sync();
    dec->be->profile_acc.clear();
    dec->be->timeline.clear();
  });
}

int32_t jxlb_set_capture(jxlb_decoder* dec, int32_t on) {
  if (!dec) return JXLB_ERR_INVALID_ARG;
  dec->be->capture = on != 0;
  return JXLB_OK;
}

int32_t jxlb_set_fuse_filters(jxlb_decoder* dec, int32_t on) {
  if (!dec) return JXLB_ERR_INVALID_ARG;
  dec->be->fuse_filters = on != 0;
  return JXLB_OK;
}

int32_t jxlb_set_hf_streams_per_cta(jxlb_decoder* dec, int32_t streams) {
  if (!dec || (streams != 0 && streams != 4 && streams != 8 && streams != 16 && streams != 32 && streams != 64 && streams != 128))
    return JXLB_ERR_INVALID_ARG;
  dec->be->hf_streams_per_cta = streams;
  return JXLB_OK;
}

int32_t jxlb_set_hf_streams_per_warp(jxlb_decoder* dec, int32_t streams) {
  if (!dec || (streams != 0 && streams != 4 && streams != 8 && streams != 16 && streams != 32)) return JXLB_ERR_INVALID_ARG;
  dec->be->hf_streams_per_warp = streams;
  return JXLB_OK;
}

int32_t jxlb_stage_count(const jxlb_decoder* dec, const char* name) {
  if (!dec || !name) return 0;
  auto it = dec->be->stages.find(name);
  return it == dec->be->stages.end() ? 0 : int32_t(it->second.size());
}

int32_t jxlb_stage_get(const jxlb_decoder* dec, const char* name, int32_t idx, uint32_t* width, uint32_t* height, uint32_t* out) {
  if (!dec || !name || !width || !height) return JXLB_ERR_INVALID_ARG;
  auto it = dec->be->stages.find(name);
  if (it == dec->be->stages.end() || idx < 0 || size_t(idx) >= it->second.size()) return JXLB_ERR_INVALID_ARG;
  const auto& dims = dec->be->stage_dims.at(name)[idx];
  *width = dims.first;
  *height = dims.second;
  if (out) std::memcpy(out, it->second[idx].data(), it->second[idx].size() * 4);
  return JXLB_OK;
}

int32_t jxlb_gaborish(jxlb_decoder* dec, float* const planes[3], uint32_t width, uint32_t height, uint32_t stride,
                      const float weights[6]) {
  if (!dec || !planes || !weights) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    cudaStream_t s = dec->be->stream();
    for (int c = 0; c < 3; ++c) {
      float* tmp = nullptr;
      JXLB_CHECK(cudaMallocAsync(&tmp, size_t(stride) * height * 4, s) == cudaSuccess, kErrCuda, "cudaMallocAsync failed");
      launch_gaborish(raw_view(planes[c], width, height, stride), raw_view(tmp, width, height, stride), weights[c * 2],
                      weights[c * 2 + 1], s);
      launch_copy_rect(raw_view(tmp, width, height, stride), raw_view(planes[c], width, height, stride), s);
      cudaFreeAsync(tmp, s);
      dec->be->launches += 2;
    }
  });
}

int32_t jxlb_epf(jxlb_decoder* dec, float* const planes[3], uint32_t width, uint32_t height, uint32_t stride,
                 const float* sigma, uint32_t sigma_stride, const jxlb_epf_params* params) {
  if (!dec || !planes || !params) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    cudaStream_t s = dec->be->stream();
    DevView cur[3], alt[3];
    float* tmp[3];
    for (int c = 0; c < 3; ++c) {
      JXLB_CHECK(cudaMallocAsync(&tmp[c], size_t(stride) * height * 4, s) == cudaSuccess, kErrCuda, "cudaMallocAsync failed");
      cur[c] = raw_view(planes[c], width, height, stride);
      alt[c] = raw_view(tmp[c], width, height, stride);
    }
    DevEpfParams dp;
    for (int c = 0; c < 3; ++c) dp.channel_scale[c] = params->channel_scale[c];
    dp.pass0_sigma_scale = params->pass0_sigma_scale;
    dp.pass2_sigma_scale = params->pass2_sigma_scale;
    dp.border_sad_mul = params->border_sad_mul;
    dp.sigma_for_modular = params->sigma_for_modular;
    bool in_alt = false;
    auto run = [&](int step) {
      launch_epf_step(in_alt ? alt : cur, in_alt ? cur : alt, sigma, sigma_stride, dp, step, s);
      dec->be->launches++;
      in_alt = !in_alt;
    };
    if (params->iters == 3) run(0);
    if (params->iters >= 1) run(1);
    if (params->iters >= 2) run(2);
    for (int c = 0; c < 3; ++c) {
      if (in_alt) launch_copy_rect(alt[c], cur[c], s);
      cudaFreeAsync(tmp[c], s);
    }
  });
}

int32_t jxlb_xyb_to_rgb(jxlb_decoder* dec, float* const planes[3], uint32_t width, uint32_t height, uint32_t stride,
                        const float opsin_bias[3], const float inv_matrix[9], float intensity_target, int32_t srgb_tf) {
  if (!dec || !planes || !opsin_bias || !inv_matrix) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    DevColorParams p{};  // sRGB-gamut target: no second stage, no gamma / PQ curve
    for (int i = 0; i < 3; ++i) {
      p.opsin_bias[i] = opsin_bias[i];
      p.cbrt_opsin_bias[i] = cbrtf(opsin_bias[i]);
    }
    for (int i = 0; i < 9; ++i) p.matrix[i] = inv_matrix[i];
    p.itscale = 255.0f / intensity_target;
    p.apply_srgb_tf = srgb_tf;
    p.apply_bt709_tf = 0;
    launch_xyb_to_rgb(raw_view(planes[0], width, height, stride), raw_view(planes[1], width, height, stride),
                      raw_view(planes[2], width, height, stride), p, dec->be->stream());
    dec->be->launches++;
  });
}

int32_t jxlb_squeeze_inverse(jxlb_decoder* dec, const int32_t* avg, uint32_t avg_w, uint32_t avg_h, uint32_t avg_stride,
                             const int32_t* res, uint32_t res_w, uint32_t res_h, uint32_t res_stride, int32_t* out,
                             uint32_t out_stride, int32_t horizontal) {
  if (!dec || !avg || !out) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    uint32_t ow = horizontal ? avg_w + res_w : avg_w, oh = horizontal ? avg_h : avg_h + res_h;
    launch_squeeze_inverse(raw_view(const_cast<int32_t*>(avg), avg_w, avg_h, avg_stride),
                           raw_view(const_cast<int32_t*>(res), res_w, res_h, res_stride), raw_view(out, ow, oh, out_stride),
                           horizontal != 0, dec->be->stream());
    dec->be->launches++;
  });
}

int32_t jxlb_rct_inverse(jxlb_decoder* dec, int32_t* const planes[3], uint32_t width, uint32_t height, uint32_t stride,
                         uint32_t rct_type) {
  if (!dec || !planes) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    launch_rct_inverse(raw_view(planes[0], width, height, stride), raw_view(planes[1], width, height, stride),
                       raw_view(planes[2], width, height, stride), rct_type, dec->be->stream());
    dec->be->launches++;
  });
}

int32_t jxlb_blend(jxlb_decoder* dec, float* base, const float* patch, const float* base_alpha, const float* new_alpha,
                   uint32_t width, uint32_t height, uint32_t stride, int32_t mode, int32_t clamp, int32_t premultiplied,
                   int32_t swapped) {
  if (!dec || !base || !patch || mode < 1 || mode > 6) return JXLB_ERR_INVALID_ARG;
  return guarded(dec, [&] {
    const DevPatchJob j{patch, base, base_alpha, new_alpha, stride, stride, stride, stride, width, height, uint32_t(mode),
                        clamp ? 1u : 0u, premultiplied ? 1u : 0u, swapped ? 1u : 0u};
    dec->be->blend_raw(j);
  });
}

}  // extern "C"
