// Internals shared by the C-ABI translation units (capi.cu, pipeline.cu). Not part of the public boundary.
#pragma once
#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/jxlb200.h"
#include "cuda_backend.h"
#include "host/frame_index.h"
#include "host/planner.h"

struct jxlb_decoder {
  std::unique_ptr<jxlb::CudaBackend> be;
  jxlb::DecodeResult res;
  bool have_result = false;
  std::string error;
  std::vector<uint8_t> codestream;
  std::vector<uint8_t> jpeg;  // the last jxlb_reconstruct_jpeg result
  struct Slot {
    std::vector<uint8_t> codestream;
    uint8_t* dptr = nullptr;
  };
  std::map<int32_t, Slot> slots;
  ~jxlb_decoder() {
    for (auto& kv : slots) cudaFree(kv.second.dptr);
  }
};

namespace jxlb {
// A decoder without a CUDA stream of its own (pipeline workers: CudaBackend(own_stream = false)); nullptr + code on failure.
jxlb_decoder* create_decoder_internal(int32_t device, uint64_t mem_limit, bool own_stream, int32_t* code);
// Decodes a codestream whose bytes already live in HBM at `dptr` (zero-padded like upload_resident() does) and on the
// host at `cs` (the planner parses headers, TOC and entropy-code tables from the host copy).
int32_t decode_resident(jxlb_decoder* dec, const uint8_t* cs, size_t size, const uint8_t* dptr, const jxlb_options* opt);
// Decodes segment `seg` of `index` (codestream `cs`; `dptr` its HBM copy from upload_resident() or NULL) up to keyframe
// `last_keyframe`. Each keyframe becomes frame 0 of the decoder while `on_keyframe(k)` runs, so the frame accessors and
// packers work on it; it is released afterwards, except the last one when `keep_last` is set. A nonzero return of
// `on_keyframe` stops the segment with that status (dec->error holds its message).
int32_t decode_segment_keyframes(jxlb_decoder* dec, const uint8_t* cs, size_t size, const uint8_t* dptr, const FrameIndex& index,
                                 size_t seg, uint32_t last_keyframe, const jxlb_options* opt, bool keep_last,
                                 const std::function<int32_t(uint32_t)>& on_keyframe);
// All channels of a frame to host memory, channel-major (c, h, w) f32, one synchronisation at the end.
int32_t frame_planar_to_host(jxlb_decoder* dec, int32_t frame, float* dst, size_t dst_bytes);
}  // namespace jxlb
