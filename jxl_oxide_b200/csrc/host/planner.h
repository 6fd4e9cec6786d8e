// Host-side frame planner: walks the codestream syntax (image header, frame header, TOC,
// LfGlobal, LfGroups, HfGlobal, PassGroups), builds the tables the sample-level stages need and
// drives a `Backend` through the stages in the order of the reference's render_frame
// (crates/jxl-render/src/render.rs:14-156, vardct/mod.rs:48-385, modular.rs:6-147,
// lib.rs:925-998). It never touches a sample itself.
#pragma once
#include <cstdint>
#include <functional>
#include <string>
#include <vector>

#include "backend.h"

namespace jxlb {

struct DecodeOptions {
  // Output colour: 0 = image's signalled encoding (sRGB transfer for the supported set),
  // 1 = linear sRGB, 2 = leave XYB.
  int output_colour = 0;
  uint32_t max_frames = 0xffffffffu;
};

// What a frame is to the frames around it (jxl-render/src/lib.rs:294-330, jxl-frame/src/header.rs:221-225): the
// decoder and the keyframe index (frame_index.h) both take it from here.
struct FrameRole {
  FrameType kind = FrameType::kRegular;
  // blended onto the canvas: a regular frame that does not replace the whole canvas
  bool composes = false;
  int saved_to = -1;   // the reference slot the frame is saved to, -1 when it is not saved
  bool shown = false;  // a keyframe: one of the frames of the decoded image
  int lf_read = -1;    // the LF store the frame takes its LF image from (use_lf_frame), or -1
  int lf_write = -1;   // the LF store an LF frame is kept in (lf_level - 1), or -1
  bool regular() const { return kind != FrameType::kLfFrame && kind != FrameType::kReferenceOnly; }
};

inline FrameRole frame_role(const FrameHeader& fh, const ImageHeader& ih) {
  FrameRole r;
  r.kind = fh.frame_type;
  r.composes = r.regular() && !(fh.resets_canvas && fh.width == ih.width && fh.height == ih.height);
  const bool can_reference = !fh.is_last && (fh.duration == 0 || fh.save_as_reference != 0);
  if (r.kind == FrameType::kReferenceOnly || (r.regular() && can_reference)) r.saved_to = int(fh.save_as_reference);
  r.shown = fh.is_keyframe();
  if (fh.use_lf_frame()) r.lf_read = int(fh.lf_level);
  if (r.kind == FrameType::kLfFrame) r.lf_write = int(fh.lf_level) - 1;
  return r;
}

struct DecodedFrame {
  bool internal = false;  // an LF frame: consumed by later frames, never shown (jxl-render/src/lib.rs:294-318)
  uint32_t width = 0, height = 0;
  uint32_t num_color = 0;
  std::vector<View> channels;  // f32 planes: colour channels then extra channels
  FrameHeader header;
};

// What ImageStream::from_render puts into an interleaved buffer (jxl-oxide/src/fb.rs:184-283): the colour channels,
// then the first alpha channel; spot-colour channels are mixed into a three-channel colour image while it is written
// (fb.rs:335-362) unless the image is grayscale (lib.rs:416). The black channel of a CMYK image (recognised by its
// ICC profile's data colour space) follows the colour channels; the samples stay CMYK - no CMS here.
struct StreamSpot {
  size_t channel;  // index into DecodedFrame::channels
  float rgb[3];
  float solidity;
};
struct StreamLayout {
  std::vector<size_t> channels;  // indices into DecodedFrame::channels, in output order
  std::vector<StreamSpot> spots;
};
// `skip_alpha` leaves the alpha channel out (Render::stream_no_alpha); `render_spot_colour` off leaves the spot colours
// unmixed (JxlImage::set_render_spot_color(false), fb.rs:247).
StreamLayout stream_layout(const ImageHeader& ih, const DecodedFrame& f, bool skip_alpha = false, bool render_spot_colour = true);
// Render::image_all_channels / image_planar (lib.rs:1150-1198): the colour channels, then every extra channel in header
// order; nothing is mixed.
StreamLayout all_channels_layout(const DecodedFrame& f);

// One write of a frame's samples (jxlb_write_spec, include/jxlb200.h): which planes go where, and the output's size.
enum WriteLayout : int32_t { kWriteStream = 0, kWriteStreamNoAlpha = 1, kWriteAllInterleaved = 2, kWriteAllPlanar = 3 };
struct WritePlan {
  StreamLayout layout;
  uint32_t orientation = 1;  // 1..8
  uint32_t sample_type = 0;  // 0: u8, 1: u16, 2: f32
  bool planar = false;
  uint32_t width = 0, height = 0;  // of the stored planes; the output is height x width for orientations 5..8
  size_t bytes = 0;
};
// Throws kErrInvalidArg for a layout, sample type or orientation (0 = the image's, else 1..8) out of range, and
// kErrUnsupported when the selected planes differ in size. `render_spot_colour` matters to the stream layouts only.
WritePlan plan_write(const ImageHeader& ih, const DecodedFrame& f, int32_t layout, int32_t sample_type, int32_t orientation,
                     bool render_spot_colour);

struct DecodeResult {
  ImageHeader image_header;
  std::vector<DecodedFrame> frames;
};

// Strips an ISOBMFF container if present (crates/jxl-bitstream/src/container*). Returns the bare
// codestream (a copy when boxes had to be concatenated).
std::vector<uint8_t> extract_codestream(const uint8_t* data, size_t size);

// Decodes every keyframe of `codestream` (bare) through `be`. Planes referenced by the result
// stay alive in the backend until the caller frees them.
DecodeResult decode_codestream(Backend& be, const uint8_t* codestream, size_t size, const DecodeOptions& opt);

// The two halves of decode_codestream. parse_codestream_header reads the image header and ICC profile, skips the
// preview frame if there is one, and returns the byte offset of the first frame. decode_frames decodes the frames from byte `begin` on, as if `visible_before` shown
// and `invisible_before` hidden frames had come before and left every reference slot and LF store empty; each shown
// frame goes to `sink` as soon as it is finished (the sink owns its planes), up to `max_shown` of them. The stores are
// freed when it returns or throws. The caller has called be.set_codestream().
size_t parse_codestream_header(const uint8_t* codestream, size_t size, ImageHeader* ih);
void decode_frames(Backend& be, const uint8_t* codestream, size_t size, const ImageHeader& ih, const DecodeOptions& opt,
                   size_t begin, uint64_t visible_before, uint64_t invisible_before, uint32_t max_shown,
                   const std::function<void(DecodedFrame&&)>& sink);

}  // namespace jxlb
