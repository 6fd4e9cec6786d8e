// See frame_index.h.
#include "frame_index.h"

#include <algorithm>

namespace jxlb {

namespace {

// The state a frame reads and writes (frame_role, planner.h).
void frame_state(const FrameHeader& fh, const ImageHeader& ih, IndexedFrame* f) {
  const FrameRole role = frame_role(fh, ih);
  if (role.lf_read >= 0) f->reads |= 1u << (4 + role.lf_read);
  if (fh.patches()) f->reads |= 0xfu;  // the patch list (in LfGlobal) may name any slot
  if (role.composes) {  // composition onto the canvas reads the blending sources
    f->reads |= 1u << fh.blending_info.source;
    for (const BlendingInfo& b : fh.ec_blending_info) f->reads |= 1u << b.source;
  }
  if (role.lf_write >= 0) f->writes |= 1u << (4 + role.lf_write);
  if (role.saved_to >= 0) f->writes |= 1u << role.saved_to;
  f->shown = role.shown;
}

}  // namespace

size_t FrameIndex::segment_of(uint32_t keyframe) const {
  for (size_t s = 0; s < segments.size(); ++s)
    if (!segments[s].keyframes.empty() && keyframe <= segments[s].keyframes.back()) return s;
  fail(kErrInvalidArg, "keyframe index out of range");
}

FrameIndex index_frames(const uint8_t* cs, size_t size) {
  FrameIndex idx;
  BitReader br(cs, size);
  idx.image_header = parse_image_header(br);
  const ImageHeader& ih = idx.image_header;
  if (ih.colour_encoding.want_icc) skip_icc_profile(br);
  br.check();
  br.zero_pad_to_byte();
  // the preview is neither a visible nor an invisible frame: it takes no part in the noise seeds
  size_t pos = skip_preview_frame(cs, size, ih, br.pos() / 8);

  uint64_t visible = 0, invisible = 0;
  while (pos < size) {
    IndexedFrame f;
    f.begin = pos;
    f.visible_before = visible;
    f.invisible_before = invisible;
    bool last = false;
    try {
      BitReader fr(cs, size, pos * 8);
      const FrameHeader fh = parse_frame_header(fr, ih);
      f.type = fh.frame_type;
      frame_state(fh, ih, &f);
      last = fh.is_last;
      const Toc toc = parse_toc(fr, fh);
      f.end = toc.data_begin + toc.total_size;
      JXLB_CHECK(f.end <= size, kErrEof, "frame data beyond end of codestream");
    } catch (const Error& e) {
      f.broken = true;
      f.shown = true;
      f.reads = f.writes = 0;
      f.end = size;
      idx.error = e.code;
      idx.message = e.what();
    }
    idx.frames.push_back(f);
    if (f.broken || last) break;
    if (f.shown) {
      ++visible;
      invisible = 0;
    } else {
      ++invisible;
    }
    pos = f.end;
  }

  // A segment may start at frame i when the frame before it is shown and no frame from i on reads a slot or store
  // whose last writer lies before i: for every such read (writer w, reader j), no cut falls in (w, j].
  const size_t n = idx.frames.size();
  std::vector<int> covered(n + 1, 0);
  int last_writer[8];
  std::fill(last_writer, last_writer + 8, -1);
  for (size_t j = 0; j < n; ++j) {
    const IndexedFrame& f = idx.frames[j];
    for (int b = 0; b < 8; ++b)
      if ((f.reads >> b & 1) && last_writer[b] >= 0) {
        ++covered[size_t(last_writer[b]) + 1];
        --covered[j + 1];
      }
    for (int b = 0; b < 8; ++b)
      if (f.writes >> b & 1) last_writer[b] = int(j);
  }
  int open = 0;
  uint32_t keyframe = 0;
  for (size_t i = 0; i < n; ++i) {
    open += covered[i];
    const IndexedFrame& f = idx.frames[i];
    if (i == 0 || (idx.frames[i - 1].shown && open == 0)) {
      FrameSegment s;
      s.first_frame = i;
      s.begin = f.begin;
      s.visible_before = f.visible_before;
      s.invisible_before = f.invisible_before;
      idx.segments.push_back(s);
    }
    FrameSegment& s = idx.segments.back();
    ++s.num_frames;
    if (f.shown) s.keyframes.push_back(keyframe++);
  }
  // trailing frames that show nothing (a stream that ends in hidden frames) need no decoding
  if (!idx.segments.empty() && idx.segments.back().keyframes.empty()) idx.segments.pop_back();
  idx.num_keyframes = keyframe;
  return idx;
}

void decode_segment(Backend& be, const uint8_t* cs, size_t size, const DecodeOptions& opt, const FrameIndex& index,
                    size_t seg, uint32_t last_keyframe, const KeyframeSink& sink) {
  JXLB_CHECK(seg < index.segments.size(), kErrInvalidArg, "segment index out of range");
  const FrameSegment& s = index.segments[seg];
  // nothing after the segment's last frame is read: a backend that uploads the codestream uploads only up to there
  size = std::min(size, index.frames[s.first_frame + s.num_frames - 1].end);
  be.set_codestream(cs, size);
  ImageHeader ih;
  parse_codestream_header(cs, size, &ih);
  uint32_t count = 0;
  for (uint32_t k : s.keyframes) count += k <= last_keyframe;
  if (count == 0) return;
  uint32_t next = s.keyframes.front();
  decode_frames(be, cs, size, ih, opt, s.begin, s.visible_before, s.invisible_before, count,
                [&](DecodedFrame&& f) { sink(next++, ih, std::move(f)); });
  if (next < s.keyframes.front() + count) {  // the frames ran out before the keyframe: report it as the index did
    const IndexedFrame& last = index.frames[s.first_frame + s.num_frames - 1];
    fail(last.broken ? index.error : kErrBitstream, last.broken ? index.message : "keyframe not found in its segment");
  }
}

}  // namespace jxlb
