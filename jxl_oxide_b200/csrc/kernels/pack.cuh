// Per-sample rules of the frame packer (pack.cu): where an output sample comes from, how spot colours are mixed into it and
// how it is stored. Parity with the reference's ImageStream / FrameBuffer is bit equality, so these are the float
// operations of crates/jxl-oxide/src/fb.rs in its order. tests/emu compiles this header for the host
// (tests/test_write_layouts.py), where the operators of pixel_math.cuh are plain C++ under -ffp-contract=off.
#pragma once
#include "pixel_math.cuh"

namespace jxlb {

// Output sample (x, y) of an image shown with `orientation` (1..8) reads stored sample (sx, sy); ow x oh are the output
// dimensions, swapped against the stored ones for orientations 5..8 (to_original_coord, fb.rs:383-397).
JXLB_PX void pack_source_xy(uint32_t orientation, uint32_t ow, uint32_t oh, uint32_t x, uint32_t y, uint32_t* sx, uint32_t* sy) {
  switch (orientation) {
    case 2: *sx = ow - x - 1, *sy = y; break;
    case 3: *sx = ow - x - 1, *sy = oh - y - 1; break;
    case 4: *sx = x, *sy = oh - y - 1; break;
    case 5: *sx = y, *sy = x; break;
    case 6: *sx = y, *sy = ow - x - 1; break;
    case 7: *sx = oh - y - 1, *sy = ow - x - 1; break;
    case 8: *sx = oh - y - 1, *sy = x; break;
    default: *sx = x, *sy = y; break;
  }
}

// Colour channel c (< 3) of stored sample (sx, sy) with every spot colour of the table mixed in, in table order
// (fb.rs:335-362): v = rgb[c] * mix + v * (1 - mix), mix = spot sample * solidity.
JXLB_PX float pack_sample(const DevPackSpec& p, const DevPackChannel* channels, const DevPackSpot* spots, uint32_t c, uint32_t sx,
                          uint32_t sy) {
  float v = channels[c].plane[size_t(sy) * channels[c].stride + sx];
  if (c < 3)
    for (uint32_t s = 0; s < p.num_spots; ++s) {
      const float mix = fmul(spots[s].plane[size_t(sy) * spots[s].stride + sx], spots[s].solidity);
      v = fadd(fmul(spots[s].rgb[c], mix), fmul(v, fsub(1.0f, mix)));
    }
  return v;
}

// Stores `v` as element i of `out`: f32 as is, u8 / u16 as round(v * max) clamped to [0, max], NaN -> 0 (fb.rs:436-520).
JXLB_PX void pack_store(void* out, size_t i, uint32_t sample_type, float v) {
  if (sample_type == 2) {
    static_cast<float*>(out)[i] = v;
    return;
  }
  const float hi = sample_type == 0 ? 255.0f : 65535.0f;
  float t = fadd(fmul(v, hi), 0.5f);
  t = t < 0.0f ? 0.0f : (t > hi ? hi : t);  // f32::clamp; NaN falls through and casts to 0
  const uint32_t q = (t == t) ? uint32_t(t) : 0u;
  if (sample_type == 0) static_cast<uint8_t*>(out)[i] = uint8_t(q);
  else static_cast<uint16_t*>(out)[i] = uint16_t(q);
}

// Element index of channel c of output sample (x, y): interleaved (channel fastest) or planar (one oriented plane per
// channel, channel-major).
JXLB_PX size_t pack_index(const DevPackSpec& p, uint32_t ow, uint32_t oh, uint32_t c, uint32_t x, uint32_t y) {
  return p.planar ? (size_t(c) * oh + y) * ow + x : (size_t(y) * ow + x) * p.num_channels + c;
}

}  // namespace jxlb
