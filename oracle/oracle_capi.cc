// TEST INFRASTRUCTURE — see oracle_backend.h. C entry points for ctypes (tests/, bench.py).
#include <cstring>
#include <memory>
#include <string>

#include "../jxl_oxide_b200/csrc/host/planner.h"
#include "oracle_backend.h"
#include "../jxl_oxide_b200/csrc/host/icc.h"

// tests/emu/ builds this file a second time with a backend whose entropy stages run the host-compiled device code
#ifdef JXLO_BACKEND_FACTORY
namespace jxlo {
OracleBackend* JXLO_BACKEND_FACTORY(int threads);
}
#define JXLO_NEW_BACKEND(threads) jxlo::JXLO_BACKEND_FACTORY(threads)
#else
#define JXLO_NEW_BACKEND(threads) new jxlo::OracleBackend(threads)
#endif

namespace {
struct Handle {
  std::unique_ptr<jxlo::OracleBackend> be;
  jxlb::DecodeResult res;
  std::vector<uint8_t> codestream;
};
void set_err(char* err, size_t n, const std::string& s) {
  if (err && n) {
    std::strncpy(err, s.c_str(), n - 1);
    err[n - 1] = 0;
  }
}
}  // namespace

extern "C" {

void* jxlo_decode(const uint8_t* data, size_t size, int output_colour, int threads, int capture, int* status,
                  char* err, size_t errlen) {
  auto h = std::make_unique<Handle>();
  try {
    h->codestream = jxlb::extract_codestream(data, size);
    h->be.reset(JXLO_NEW_BACKEND(threads));
    h->be->capture = capture != 0;
    jxlb::DecodeOptions opt;
    opt.output_colour = output_colour;
    h->res = jxlb::decode_codestream(*h->be, h->codestream.data(), h->codestream.size(), opt);
    if (status) *status = 0;
    return h.release();
  } catch (const jxlb::Error& e) {
    if (status) *status = e.code;
    set_err(err, errlen, e.what());
  } catch (const std::exception& e) {
    if (status) *status = -1;
    set_err(err, errlen, e.what());
  }
  return nullptr;
}

int jxlo_num_frames(void* hp) { return int(static_cast<Handle*>(hp)->res.frames.size()); }

void jxlo_image_info(void* hp, uint32_t* width, uint32_t* height, uint32_t* bits, uint32_t* num_extra,
                     uint32_t* xyb, uint32_t* gray) {
  const jxlb::ImageHeader& ih = static_cast<Handle*>(hp)->res.image_header;
  *width = ih.width, *height = ih.height, *bits = ih.bit_depth.bits_per_sample;
  *num_extra = uint32_t(ih.ec_info.size()), *xyb = ih.xyb_encoded, *gray = ih.grayscale();
}

// Known-answer hook for the ICC recognition rules (host/icc.cc, shared with the product): status 0 enum / 1
// unsupported / 2 malformed; out = colour space, white point, primaries, transfer function, gamma, gamma_inverted,
// rendering intent.
int jxlo_icc_to_enum(const uint8_t* icc, size_t size, uint32_t out[7]) {
  jxlb::IccInfo info;
  const jxlb::IccStatus st = jxlb::icc_to_enum(std::vector<uint8_t>(icc, icc + size), &info);
  const jxlb::ColourEncoding& e = info.encoding;
  out[0] = uint32_t(e.colour_space), out[1] = uint32_t(e.white_point), out[2] = uint32_t(e.primaries), out[3] = uint32_t(e.tf);
  out[4] = e.gamma, out[5] = e.gamma_inverted ? 1 : 0, out[6] = e.rendering_intent;
  return int(st);
}

// Known-answer hook: the PQ inverse EOTF as the colour stage applies it (replays tf/pq.rs:460-478)
void jxlo_linear_to_pq(float* samples, size_t n, float intensity_target) {
  for (size_t i = 0; i < n; ++i) samples[i] = jxlo::linear_to_pq(samples[i], intensity_target);
}

// Known-answer hooks: the restoration filters on three caller planes of width x height f32 samples (tightly packed),
// filtered in place, default parameters. jxlo_epf takes the per-8x8-block sigma grid ((w + 7) / 8 x (h + 7) / 8), or
// NULL for the constant sigma of a Modular frame.
void jxlo_gaborish(float* p0, float* p1, float* p2, uint32_t w, uint32_t h, const float weights[6]) {
  jxlo::OracleBackend be(1);
  float* p[3] = {p0, p1, p2};
  jxlb::View v[3];
  float wt[3][2];
  for (int c = 0; c < 3; ++c) {
    v[c] = jxlb::View{be.alloc_plane(w, h, false), 0, 0, w, h};
    std::memcpy(be.plane(v[c].plane).f32(), p[c], size_t(w) * h * 4);
    wt[c][0] = weights[2 * c], wt[c][1] = weights[2 * c + 1];
  }
  be.gaborish(v, wt);
  for (int c = 0; c < 3; ++c) std::memcpy(p[c], be.plane(v[c].plane).f32(), size_t(w) * h * 4);
}

void jxlo_epf(float* p0, float* p1, float* p2, uint32_t w, uint32_t h, const float* sigma, float sigma_const, uint32_t iters) {
  jxlo::OracleBackend be(1);
  float* p[3] = {p0, p1, p2};
  jxlb::View v[3], sv;
  for (int c = 0; c < 3; ++c) {
    v[c] = jxlb::View{be.alloc_plane(w, h, false), 0, 0, w, h};
    std::memcpy(be.plane(v[c].plane).f32(), p[c], size_t(w) * h * 4);
  }
  const uint32_t bw = (w + 7) / 8, bh = (h + 7) / 8;
  if (sigma) {
    sv = jxlb::View{be.alloc_plane(bw, bh, false), 0, 0, bw, bh};
    std::memcpy(be.plane(sv.plane).f32(), sigma, size_t(bw) * bh * 4);
  }
  jxlb::EpfParams prm;
  prm.iters = iters;
  prm.sigma_for_modular = sigma_const;
  be.epf(v, sv, prm, sigma == nullptr);
  for (int c = 0; c < 3; ++c) std::memcpy(p[c], be.plane(v[c].plane).f32(), size_t(w) * h * 4);
}

// features::upsample with the default weights: `in` (width x height, tightly packed) -> `out` (width * factor x
// height * factor), factor 2, 4 or 8.
void jxlo_upsample(const float* in, uint32_t w, uint32_t h, uint32_t factor, float* out) {
  jxlo::OracleBackend be(1);
  const jxlb::View v{be.alloc_plane(w, h, false), 0, 0, w, h};
  std::memcpy(be.plane(v.plane).f32(), in, size_t(w) * h * 4);
  const int id = be.upsample(v, factor == 2 ? 1 : (factor == 4 ? 2 : 3), jxlb::default_image_header());
  std::memcpy(out, be.plane(id).f32(), size_t(w) * h * factor * factor * 4);
}

// The restoration filters a decoded frame's header asks for: Gaborish on / off and the EPF iteration count.
void jxlo_frame_filters(void* hp, int frame, uint32_t* gab_enabled, uint32_t* epf_iters) {
  const jxlb::RestorationFilter& rf = static_cast<Handle*>(hp)->res.frames.at(frame).header.restoration_filter;
  *gab_enabled = rf.gab_enabled ? 1 : 0;
  *epf_iters = rf.epf.iters;
}

size_t jxlo_image_original_icc(void* hp, uint8_t* dst, size_t cap) {
  const std::vector<uint8_t>& icc = static_cast<Handle*>(hp)->res.image_header.icc_profile;
  if (dst && cap >= icc.size() && !icc.empty()) std::memcpy(dst, icc.data(), icc.size());
  return icc.size();
}

uint32_t jxlo_image_orientation(void* hp) { return static_cast<Handle*>(hp)->res.image_header.orientation; }

void jxlo_frame_info(void* hp, int frame, uint32_t* width, uint32_t* height, uint32_t* num_channels,
                     uint32_t* num_color, uint32_t* is_vardct) {
  const jxlb::DecodedFrame& f = static_cast<Handle*>(hp)->res.frames.at(frame);
  *width = f.width, *height = f.height, *num_channels = uint32_t(f.channels.size()), *num_color = f.num_color;
  *is_vardct = f.header.encoding == jxlb::Encoding::kVarDct;
}

void jxlo_frame_channel(void* hp, int frame, int channel, float* out) {
  Handle* h = static_cast<Handle*>(hp);
  const jxlb::DecodedFrame& f = h->res.frames.at(frame);
  h->be->download_rect(f.channels.at(channel), out);
}

// Returns the number of planes captured for `name` (0 if absent). With out != NULL copies plane idx.
int jxlo_stage(void* hp, const char* name, int idx, uint32_t* w, uint32_t* hgt, uint32_t* out) {
  Handle* h = static_cast<Handle*>(hp);
  auto it = h->be->stages.find(name);
  if (it == h->be->stages.end()) return 0;
  if (idx >= 0 && idx < int(it->second.size())) {
    *w = h->be->stage_dims[name][idx].first;
    *hgt = h->be->stage_dims[name][idx].second;
    if (out) std::memcpy(out, it->second[idx].data(), it->second[idx].size() * 4);
  }
  return int(it->second.size());
}

// ImageStream::write_to_buffer::<u8 | u16 | f32> (crates/jxl-oxide/src/fb.rs:309-410, 387-401, 436-520):
// channel-interleaved samples with the orientation applied. sample_type 0 = u8, 1 = u16, 2 = f32;
// orientation 0 = the image header's. Returns the number of samples written.
uint32_t jxlo_frame_stream_channels(void* hp, int frame) {
  Handle* h = static_cast<Handle*>(hp);
  return uint32_t(jxlb::stream_layout(h->res.image_header, h->res.frames.at(frame)).channels.size());
}

size_t jxlo_frame_write_to_buffer(void* hp, int frame, int sample_type, int orientation, void* dst) {
  Handle* h = static_cast<Handle*>(hp);
  const jxlb::DecodedFrame& f = h->res.frames.at(frame);
  const uint32_t orient = orientation ? uint32_t(orientation) : h->res.image_header.orientation;
  const uint32_t width = f.channels.at(0).w, height = f.channels.at(0).h;
  const uint32_t ow = orient >= 5 ? height : width, oh = orient >= 5 ? width : height;
  const jxlb::StreamLayout layout = jxlb::stream_layout(h->res.image_header, f);
  const size_t nc = layout.channels.size();
  std::vector<std::vector<float>> planes(nc), spots(layout.spots.size());
  for (size_t c = 0; c < nc; ++c) {
    planes[c].resize(size_t(width) * height);
    h->be->download_rect(f.channels[layout.channels[c]], planes[c].data());
  }
  for (size_t s = 0; s < spots.size(); ++s) {
    spots[s].resize(size_t(width) * height);
    h->be->download_rect(f.channels[layout.spots[s].channel], spots[s].data());
  }
  size_t count = 0;
  for (uint32_t y = 0; y < oh; ++y)
    for (uint32_t x = 0; x < ow; ++x) {
      uint32_t sx, sy;
      switch (orient) {
        case 1: sx = x, sy = y; break;
        case 2: sx = ow - x - 1, sy = y; break;
        case 3: sx = ow - x - 1, sy = oh - y - 1; break;
        case 4: sx = x, sy = oh - y - 1; break;
        case 5: sx = y, sy = x; break;
        case 6: sx = y, sy = ow - x - 1; break;
        case 7: sx = oh - y - 1, sy = ow - x - 1; break;
        default: sx = oh - y - 1, sy = x; break;
      }
      for (size_t c = 0; c < nc; ++c, ++count) {
        float v = planes[c][size_t(sy) * width + sx];
        if (c < 3)  // spot colours (fb.rs:335-362)
          for (size_t s = 0; s < spots.size(); ++s) {
            const float mix = spots[s][size_t(sy) * width + sx] * layout.spots[s].solidity;
            v = layout.spots[s].rgb[c] * mix + v * (1.0f - mix);
          }
        if (sample_type == 2) {
          static_cast<float*>(dst)[count] = v;
        } else {
          const float hi = sample_type == 0 ? 255.0f : 65535.0f;
          float t = v * hi + 0.5f;
          t = t < 0.0f ? 0.0f : (t > hi ? hi : t);  // f32::clamp keeps NaN, `as uN` then yields 0
          const uint32_t q = (t == t) ? uint32_t(t) : 0u;
          if (sample_type == 0) static_cast<uint8_t*>(dst)[count] = uint8_t(q);
          else static_cast<uint16_t*>(dst)[count] = uint16_t(q);
        }
      }
    }
  return count;
}

void jxlo_free(void* hp) { delete static_cast<Handle*>(hp); }

}  // extern "C"
