// TEST INFRASTRUCTURE. C entry points of the oracle's keyframe decode (keyframes.mk), for tests/keyframe_lib.py.
#include <cstring>
#include <memory>
#include <string>

#include "../../jxl_oxide_b200/csrc/host/frame_index.h"
#include "../../oracle/oracle_backend.h"

namespace {
struct Handle {
  std::unique_ptr<jxlo::OracleBackend> be;
  jxlb::DecodedFrame frame;
};
void set_err(char* err, size_t n, const std::string& s) {
  if (err && n) {
    std::strncpy(err, s.c_str(), n - 1);
    err[n - 1] = 0;
  }
}
}  // namespace

extern "C" {

// The index: returns the number of segments (-1 when the image header cannot be read) and fills, up to `cap` of
// each, the first keyframe and the keyframe count of every segment; *error receives the index's error code.
int jxlk_segments(const uint8_t* data, size_t size, uint32_t* first_keyframe, uint32_t* num_keyframes, int cap, int* error) {
  try {
    const std::vector<uint8_t> cs = jxlb::extract_codestream(data, size);
    const jxlb::FrameIndex idx = jxlb::index_frames(cs.data(), cs.size());
    for (size_t s = 0; s < idx.segments.size() && int(s) < cap; ++s) {
      first_keyframe[s] = idx.segments[s].keyframes.empty() ? 0 : idx.segments[s].keyframes.front();
      num_keyframes[s] = uint32_t(idx.segments[s].keyframes.size());
    }
    if (error) *error = idx.error;
    return int(idx.segments.size());
  } catch (const jxlb::Error& e) {
    if (error) *error = e.code;
    return -1;
  }
}

// Keyframe `keyframe` decoded from its own segment on the oracle; NULL and *status on failure.
void* jxlk_decode_keyframe(const uint8_t* data, size_t size, int keyframe, int threads, int* status, char* err, size_t errlen) {
  auto h = std::make_unique<Handle>();
  try {
    const std::vector<uint8_t> cs = jxlb::extract_codestream(data, size);
    const jxlb::FrameIndex idx = jxlb::index_frames(cs.data(), cs.size());
    JXLB_CHECK(keyframe >= 0 && uint32_t(keyframe) < idx.num_keyframes, jxlb::kErrInvalidArg, "keyframe index out of range");
    h->be.reset(new jxlo::OracleBackend(threads));
    bool got = false;
    jxlb::decode_segment(*h->be, cs.data(), cs.size(), jxlb::DecodeOptions(), idx, idx.segment_of(uint32_t(keyframe)), uint32_t(keyframe),
                         [&](uint32_t k, const jxlb::ImageHeader&, jxlb::DecodedFrame&& f) {
                           if (k == uint32_t(keyframe)) {
                             h->frame = std::move(f);
                             got = true;
                           } else {
                             for (const jxlb::View& v : f.channels) h->be->free_plane(v.plane);
                           }
                         });
    JXLB_CHECK(got, jxlb::kErrBitstream, "keyframe not decoded");
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

void jxlk_frame_info(void* hp, uint32_t* width, uint32_t* height, uint32_t* num_channels) {
  const jxlb::DecodedFrame& f = static_cast<Handle*>(hp)->frame;
  *width = f.width, *height = f.height, *num_channels = uint32_t(f.channels.size());
}

void jxlk_frame_channel(void* hp, int channel, float* out) {
  Handle* h = static_cast<Handle*>(hp);
  h->be->download_rect(h->frame.channels.at(channel), out);
}

void jxlk_free(void* hp) { delete static_cast<Handle*>(hp); }

}  // extern "C"
