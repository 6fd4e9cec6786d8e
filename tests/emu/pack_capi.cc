// TEST INFRASTRUCTURE. C entry points (pack.mk) for tests/test_write_layouts.py: a frame decoded by the oracle, the
// planner's write plan for it (host/planner.cc plan_write, the same code jxlb_frame_write_ex runs) and the frame packed
// on the host by the per-sample functions of the device packer (kernels/pack.cuh), thread by thread in a plain loop.
#include <cstring>
#include <memory>
#include <string>

#include "cuda_shim.h"

#include "../../jxl_oxide_b200/csrc/kernels/pack.cuh"
#include "../../jxl_oxide_b200/csrc/host/planner.h"
#include "../../oracle/oracle_backend.h"

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

void* jxlw_decode(const uint8_t* data, size_t size, int threads, int* status, char* err, size_t errlen) {
  auto h = std::make_unique<Handle>();
  try {
    h->codestream = jxlb::extract_codestream(data, size);
    h->be.reset(new jxlo::OracleBackend(threads));
    h->res = jxlb::decode_codestream(*h->be, h->codestream.data(), h->codestream.size(), jxlb::DecodeOptions());
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

// The image header alone (no frame is decoded): enough for the channel selection of a frame decoded elsewhere.
void* jxlw_read_header(const uint8_t* data, size_t size) {
  auto h = std::make_unique<Handle>();
  try {
    h->codestream = jxlb::extract_codestream(data, size);
    jxlb::parse_codestream_header(h->codestream.data(), h->codestream.size(), &h->res.image_header);
    return h.release();
  } catch (const std::exception&) {
    return nullptr;
  }
}

// What the channel selection reads from the image header.
void jxlw_header(void* hp, uint32_t* icc_is_cmyk, uint32_t* grayscale, uint32_t* orientation, uint32_t* num_extra) {
  const jxlb::ImageHeader& ih = static_cast<Handle*>(hp)->res.image_header;
  *icc_is_cmyk = ih.icc_is_cmyk, *grayscale = ih.grayscale(), *orientation = ih.orientation;
  *num_extra = uint32_t(ih.ec_info.size());
}

void jxlw_extra_channel(void* hp, int e, uint32_t* type, float spot[4]) {
  const jxlb::ExtraChannelInfo& ec = static_cast<Handle*>(hp)->res.image_header.ec_info.at(size_t(e));
  *type = uint32_t(ec.type);
  for (int k = 0; k < 4; ++k) spot[k] = ec.spot[k];
}

int jxlw_num_frames(void* hp) { return int(static_cast<Handle*>(hp)->res.frames.size()); }

void jxlw_frame_info(void* hp, int frame, uint32_t* width, uint32_t* height, uint32_t* num_channels, uint32_t* num_color) {
  const jxlb::DecodedFrame& f = static_cast<Handle*>(hp)->res.frames.at(size_t(frame));
  *width = f.channels.at(0).w, *height = f.channels.at(0).h, *num_channels = uint32_t(f.channels.size()), *num_color = f.num_color;
}

void jxlw_frame_channel(void* hp, int frame, int channel, float* out) {
  Handle* h = static_cast<Handle*>(hp);
  h->be->download_rect(h->res.frames.at(size_t(frame)).channels.at(size_t(channel)), out);
}

// plan_write: status 0 or the error code (message in err); the selected channels (up to cap), the spot channels (up to
// cap), their count and the output's byte count.
int jxlw_plan(void* hp, int frame, int layout, int sample_type, int orientation, int spot_colours, uint32_t* channels,
              uint32_t* num_channels, uint32_t* spots, uint32_t* num_spots, uint32_t cap, uint64_t* bytes, char* err, size_t errlen) {
  Handle* h = static_cast<Handle*>(hp);
  try {
    const jxlb::WritePlan w =
        jxlb::plan_write(h->res.image_header, h->res.frames.at(size_t(frame)), layout, sample_type, orientation, spot_colours != 0);
    *num_channels = uint32_t(w.layout.channels.size());
    *num_spots = uint32_t(w.layout.spots.size());
    for (size_t i = 0; i < w.layout.channels.size() && i < cap; ++i) channels[i] = uint32_t(w.layout.channels[i]);
    for (size_t i = 0; i < w.layout.spots.size() && i < cap; ++i) spots[i] = uint32_t(w.layout.spots[i].channel);
    *bytes = w.bytes;
    return 0;
  } catch (const jxlb::Error& e) {
    set_err(err, errlen, e.what());
    return e.code;
  }
}

// The frame written as jxlb_frame_write_ex would, by pack.cuh on the host; `out` holds the plan's byte count.
int jxlw_pack(void* hp, int frame, int layout, int sample_type, int orientation, int spot_colours, void* out) {
  Handle* h = static_cast<Handle*>(hp);
  const jxlb::DecodedFrame& f = h->res.frames.at(size_t(frame));
  try {
    const jxlb::WritePlan w = jxlb::plan_write(h->res.image_header, f, layout, sample_type, orientation, spot_colours != 0);
    const size_t n = size_t(w.width) * w.height;
    std::vector<std::vector<float>> planes(w.layout.channels.size()), spot_planes(w.layout.spots.size());
    std::vector<jxlb::DevPackChannel> channels;
    std::vector<jxlb::DevPackSpot> spots;
    for (size_t c = 0; c < planes.size(); ++c) {
      planes[c].resize(n);
      h->be->download_rect(f.channels[w.layout.channels[c]], planes[c].data());
      channels.push_back(jxlb::DevPackChannel{planes[c].data(), w.width});
    }
    for (size_t s = 0; s < spot_planes.size(); ++s) {
      const jxlb::StreamSpot& sp = w.layout.spots[s];
      spot_planes[s].resize(n);
      h->be->download_rect(f.channels[sp.channel], spot_planes[s].data());
      spots.push_back(jxlb::DevPackSpot{spot_planes[s].data(), w.width, {sp.rgb[0], sp.rgb[1], sp.rgb[2]}, sp.solidity});
    }
    jxlb::DevPackSpec p;
    p.num_channels = uint32_t(channels.size());
    p.num_spots = uint32_t(spots.size());
    p.width = w.width;
    p.height = w.height;
    p.orientation = w.orientation;
    p.sample_type = w.sample_type;
    p.planar = w.planar ? 1 : 0;
    const uint32_t ow = p.orientation >= 5 ? p.height : p.width, oh = p.orientation >= 5 ? p.width : p.height;
    for (uint32_t c = 0; c < p.num_channels; ++c)
      for (uint32_t y = 0; y < oh; ++y)
        for (uint32_t x = 0; x < ow; ++x) {
          uint32_t sx, sy;
          jxlb::pack_source_xy(p.orientation, ow, oh, x, y, &sx, &sy);
          jxlb::pack_store(out, jxlb::pack_index(p, ow, oh, c, x, y), p.sample_type,
                           jxlb::pack_sample(p, channels.data(), spots.data(), c, sx, sy));
        }
    return 0;
  } catch (const jxlb::Error& e) {
    return e.code;
  }
}

void jxlw_free(void* hp) { delete static_cast<Handle*>(hp); }

}  // extern "C"
