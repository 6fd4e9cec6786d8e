// Keyframe index of a codestream: one header-only pass (image header, ICC stream skipped, every frame header and TOC;
// no section is decoded) that records what each frame reads from and writes to the state frames share - the four
// reference slots and the four LF stores - and cuts the frame list into segments that decode independently. It is
// how keyframes are rendered concurrently (jxl-oxide-cli's par_iter over render_frame(k), decode.rs:285-320) without
// decoding a keyframe's predecessors more than once: a segment needs nothing from the frames before it.
#pragma once
#include <cstdint>
#include <functional>
#include <string>
#include <vector>

#include "planner.h"

namespace jxlb {

struct IndexedFrame {
  size_t begin = 0, end = 0;  // byte range in the codestream
  FrameType type = FrameType::kRegular;
  bool shown = false;  // a keyframe: what decode_codestream puts into DecodeResult::frames
  // shown / hidden frames before this one, counted as decode_codestream counts them (the noise seed)
  uint64_t visible_before = 0, invisible_before = 0;
  // bit i < 4: reference slot i, bit 4 + i: LF store i (the frame whose lf_level is i + 1)
  uint32_t reads = 0, writes = 0;
  // the header, the TOC or the frame's data is malformed or cut off: decoding stops with an error at this frame,
  // which is counted as a keyframe so that the error has a keyframe to be reported on
  bool broken = false;
};

struct FrameSegment {
  size_t first_frame = 0, num_frames = 0;  // into FrameIndex::frames
  size_t begin = 0;                        // byte offset of the first frame
  uint64_t visible_before = 0, invisible_before = 0;
  std::vector<uint32_t> keyframes;  // keyframe indices, ascending
};

struct FrameIndex {
  ImageHeader image_header;  // ICC profile not decoded
  std::vector<IndexedFrame> frames;
  std::vector<FrameSegment> segments;
  uint32_t num_keyframes = 0;
  int error = 0;  // != 0 when the last frame is broken: its error code and message
  std::string message;

  size_t segment_of(uint32_t keyframe) const;
};

// Indexes `cs` (a bare codestream). Throws when the image header itself cannot be read; a frame that cannot be
// read or is cut off ends the index as a broken frame (FrameIndex::error) instead, so the frames before it keep
// their segments.
FrameIndex index_frames(const uint8_t* cs, size_t size);

// Decodes segment `seg` of `index` from `cs` through `be`, starting from empty reference slots and LF stores and the
// segment's frame counts, and hands each keyframe to `sink` (keyframe index, image header with its ICC profile decoded,
// frame) as soon as it is finished; the sink owns the frame's planes. Stops after keyframe `last_keyframe` or at the
// segment's end. Keyframe k decoded this way equals keyframe k of decode_codestream bit for bit. Calls
// be.set_codestream() itself.
using KeyframeSink = std::function<void(uint32_t keyframe, const ImageHeader& ih, DecodedFrame&& frame)>;
void decode_segment(Backend& be, const uint8_t* cs, size_t size, const DecodeOptions& opt, const FrameIndex& index,
                    size_t seg, uint32_t last_keyframe, const KeyframeSink& sink);

}  // namespace jxlb
