// Column-strip form of the fused restoration filters for windows that lie wholly inside the image:
// Gaborish -> EPF step 1 -> EPF step 2 -> XYB->RGB (the libjxl default at d <= ~1.5). The per-pixel formulas are those of
// every other filter kernel (pixel_math.cuh, the reference's generic path).
//
// What differs is who computes what. A CTA of 256 threads owns a 64 x 32 window (56 x 24 output pixels, margin 4 =
// Gaborish 1 + step 1's 2 + step 2's 1) in shared memory. A thread owns ONE COLUMN of the window and a run of 6-8
// rows of it and walks down that run:
//   * the 3 x 3 / plus-shaped neighbourhoods slide through registers: one shared-memory row (3-4 loads per channel)
//     per output instead of 9-15, no per-pixel index arithmetic (row offsets are immediates after unrolling), the
//     8x8-block border flags of the column are per-thread constants;
//   * step 1's patch distances are plus-sums of per-pixel absolute differences V_d(r) = |a[r+d] - a[r]|:
//     dist_d(q) = sum_c scale_c * sum_o V_d,c(q+o), summed in the reference's order of o. Each V is formed once per
//     column triple instead of five times (exact: the same subtraction, the same additions in the same order);
//   * step 2's distances are single differences of the values the weighted sum loads anyway, so step 2 has no distance
//     pass at all: the vertical one rolls down the column, the horizontal pair comes from the left / centre / right samples.
//
// The phase functions are plain functions of (thread id, window) so that tests/emu can run them on the host, thread by
// thread and phase by phase, and compare with the oracle without a GPU (tests/test_emu_filters.py).
#pragma once
#include "pixel_math.cuh"

namespace jxlb {
namespace fstrip {

// The Gaborish and distance phases walk the three channels with the same code (a loop, not three unrolled copies): the
// kernel is straight-line code that every warp executes once, so its size is instruction-fetch traffic (the fully unrolled
// body stalls on instruction fetch).
constexpr int kChanUnroll = 1;

constexpr int kWX = 64, kWY = 32;        // window (shared-memory plane) size
constexpr int kM = 4;                    // margin
constexpr int kTX = kWX - 2 * kM;        // 56 output columns
constexpr int kTY = kWY - 2 * kM;        // 24 output rows
constexpr int kThreads = 256, kSegs = kThreads / kWX;  // 4 row runs per column
constexpr int kPlane = kWX * kWY;
constexpr int kSigX = 9, kSigY = 5;      // 8x8 blocks an unaligned 64 x 32 window can touch
// shared-memory floats: in/B [3], A [3], D [2] planes, then sigma, 6.6 (1/sqrt2 - 1) / sigma, sRGB exponent table
constexpr int kOffA = 3 * kPlane, kOffD = 6 * kPlane, kOffSigma = 8 * kPlane, kOffInv = kOffSigma + kSigX * kSigY,
              kOffPow = kOffInv + kSigX * kSigY, kSmemFloats = kOffPow + 16;

struct StripGeom {
  int width, height;      // image
  int x0, y0, x1, y1;     // output rectangle of this launch (every pixel of it is >= kM away from the image border)
  int gx0, gy0;           // image pixel of window cell (0, 0) for this CTA
  int bx_first, by_first; // first 8x8 block under the window
};

// Window origin of tile (tx, ty): tiles are anchored at (x0, y0); the last ones are pulled back inside the image (their
// outputs then overlap the previous tile's: same values written twice).
JXLB_PX StripGeom strip_geom(int width, int height, int x0, int y0, int x1, int y1, int tx, int ty) {
  StripGeom g;
  g.width = width, g.height = height, g.x0 = x0, g.y0 = y0, g.x1 = x1, g.y1 = y1;
  int gx = x0 + tx * kTX - kM, gy = y0 + ty * kTY - kM;
  if (gx + kWX > width) gx = width - kWX;
  if (gy + kWY > height) gy = height - kWY;
  g.gx0 = gx, g.gy0 = gy;
  g.bx_first = gx >> 3, g.by_first = gy >> 3;
  return g;
}

// ---- phase 0: per-block sigma and the division it feeds (one per 8x8 block instead of one per pixel and step) ----------
JXLB_PX void phase_sigma(int tid, float* s, const StripGeom& g, const DevFusedFilterParams& p) {
  if (tid < kSigX * kSigY) {
    const int bx = g.bx_first + tid % kSigX, by = g.by_first + tid / kSigX;
    float sg = p.epf.sigma_for_modular;
    if (p.sigma) sg = (bx < ((g.width + 7) >> 3) && by < ((g.height + 7) >> 3)) ? p.sigma[size_t(by) * p.sigma_stride + bx] : 1.0f;
    s[kOffSigma + tid] = sg;
    s[kOffInv + tid] = epf_inv_sigma(sg);
  } else if (tid >= 64 && tid < 80) {
    s[kOffPow + tid - 64] = kSrgbPow[tid - 64];
  }
}

// ---- phase 1: Gaborish, in -> A on [1, 63) x [1, 31) ------------------------------------------------------------------
JXLB_PX void phase_gab(int tid, float* s, const DevFusedFilterParams& p, const float gw[3]) {
  const int col = tid & (kWX - 1), seg = tid / kWX;
  if (col < 1 || col >= kWX - 1) return;
  constexpr int L = 8;
  const int y0 = 1 + seg * L;
  const int n = (kWY - 1 - y0) < L ? (kWY - 1 - y0) : L;
#pragma unroll kChanUnroll
  for (int c = 0; c < 3; ++c) {
    const float* a = s + c * kPlane + y0 * kWX + col;
    float* o = s + kOffA + c * kPlane + y0 * kWX + col;
    const float w0 = p.gab_w[c][0], w1 = p.gab_w[c][1], g = gw[c];
    float tl = a[-kWX - 1], tc = a[-kWX], tr = a[-kWX + 1];
    float ml = a[-1], mc = a[0], mr = a[1];
#pragma unroll
    for (int i = 0; i < L; ++i) {
      if (i < n) {
        const float bl = a[(i + 1) * kWX - 1], bc = a[(i + 1) * kWX], br = a[(i + 1) * kWX + 1];
        o[i * kWX] = gaborish_3x3(tl, tc, tr, ml, mc, mr, bl, bc, br, w0, w1, g);
        tl = ml, tc = mc, tr = mr;
        ml = bl, mc = bc, mr = br;
      }
    }
  }
}

// ---- phase 2: step-1 distance maps D[0] = dist_(0,1), D[1] = dist_(1,0) on [2, 61) x [2, 29) ---------------------------
JXLB_PX void phase_dist1(int tid, float* s, const DevFusedFilterParams& p) {
  const int col = tid & (kWX - 1), seg = tid / kWX;
  if (col < 2 || col >= kWX - 3) return;
  constexpr int L = 7;
  constexpr int yend = kWY - 3;  // 29
  const int y0 = 2 + seg * L;
  const int n = (yend - y0) < L ? (yend - y0) : L;
  // epf.rs starts every distance at 0.0 and adds the channels' terms: the same here (0.0 + t is t for the non-negative t)
  float d01[L], d10[L];
#pragma unroll
  for (int i = 0; i < L; ++i) d01[i] = d10[i] = 0.0f;
#pragma unroll kChanUnroll
  for (int c = 0; c < 3; ++c) {
    const float* a = s + kOffA + c * kPlane + y0 * kWX + col;  // (col, y0)
    const float sc = p.epf.channel_scale[c];
    // rows y0 - 1, y0, y0 + 1; columns col - 1 .. col + 2
    float r0[4], r1[4], vc[3], hc[3];
    {
      const float pm1 = a[-kWX], pp1 = a[-kWX + 1];
#pragma unroll
      for (int j = 0; j < 4; ++j) r0[j] = a[j - 1], r1[j] = a[kWX + j - 1];
      vc[0] = absdiff(r0[1], pm1);      // V01(col, y0 - 1)
      vc[1] = absdiff(r1[1], r0[1]);    // V01(col, y0)
      hc[0] = absdiff(pp1, pm1);        // V10(col, y0 - 1)
      hc[1] = absdiff(r0[2], r0[1]);    // V10(col, y0)
    }
#pragma unroll
    for (int i = 0; i < L; ++i) {
      if (i < n) {
        float r2[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) r2[j] = a[(i + 2) * kWX + j - 1];
        vc[2] = absdiff(r2[1], r1[1]);  // V01(col, y + 1)
        hc[2] = absdiff(r1[2], r1[1]);  // V10(col, y + 1)
        const float vl = absdiff(r1[0], r0[0]), vr = absdiff(r1[2], r0[2]);  // V01(col -+ 1, y)
        const float hl = absdiff(r0[1], r0[0]), hr = absdiff(r0[3], r0[2]);  // V10(col -+ 1, y)
        // plus order of step 1: (0,-1) (0,0) (0,1) (-1,0) (1,0)
        const float p01 = fadd(fadd(fadd(fadd(vc[0], vc[1]), vc[2]), vl), vr);
        const float p10 = fadd(fadd(fadd(fadd(hc[0], hc[1]), hc[2]), hl), hr);
        const float t01 = fmul(sc, p01), t10 = fmul(sc, p10);
        d01[i] = fadd(d01[i], t01);
        d10[i] = fadd(d10[i], t10);
        vc[0] = vc[1], vc[1] = vc[2];
        hc[0] = hc[1], hc[1] = hc[2];
#pragma unroll
        for (int j = 0; j < 4; ++j) r0[j] = r1[j], r1[j] = r2[j];
      }
    }
  }
  float* d = s + kOffD + y0 * kWX + col;
#pragma unroll
  for (int i = 0; i < L; ++i)
    if (i < n) d[i * kWX] = d01[i], d[kPlane + i * kWX] = d10[i];
}

// weights and weighted sums of one pixel from its four distances (neighbour order (0,-1) (0,1) (-1,0) (1,0))
JXLB_PX void epf_combine(const float du, const float dd, const float dl, const float dr, float nis, const float ce[3],
                         const float up[3], const float dn[3], const float le[3], const float ri[3], float o[3]) {
  const float wu = epf_weight(du, nis), wd = epf_weight(dd, nis), wl = epf_weight(dl, nis), wr = epf_weight(dr, nis);
  const float sw = fadd(fadd(fadd(fadd(1.0f, wu), wd), wl), wr);
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float sum = fadd(ce[c], fmul(wu, up[c]));
    sum = fadd(sum, fmul(wd, dn[c]));
    sum = fadd(sum, fmul(wl, le[c]));
    sum = fadd(sum, fmul(wr, ri[c]));
    o[c] = fdiv(sum, sw);
  }
}

// phase_dist1 and epf_combine spell step 1's plus and neighbour orders out in registers; these tie them to pixel_math.cuh's
static_assert(epf_plus_x(1, 0) == 0 && epf_plus_y(1, 0) == -1 && epf_plus_x(1, 1) == 0 && epf_plus_y(1, 1) == 0 &&
                  epf_plus_x(1, 2) == 0 && epf_plus_y(1, 2) == 1 && epf_plus_x(1, 3) == -1 && epf_plus_y(1, 3) == 0 &&
                  epf_plus_x(1, 4) == 1 && epf_plus_y(1, 4) == 0,
              "phase_dist1 sums the plus in epf_plus order");
static_assert(epf_nb_x(1, 0) == 0 && epf_nb_y(1, 0) == -1 && epf_nb_x(1, 1) == 0 && epf_nb_y(1, 1) == 1 && epf_nb_x(1, 2) == -1 &&
                  epf_nb_y(1, 2) == 0 && epf_nb_x(1, 3) == 1 && epf_nb_y(1, 3) == 0,
              "epf_combine takes the neighbours in epf_nb order");

// TF: the colour stage's transfer function (colour_tf), a template parameter so that a kernel carries the code of its own
// curve only (the row loops are unrolled: every pixel row holds a copy of the colour stage).
static inline int strip_tf_of(const DevFusedFilterParams& p) {  // host side: which instantiation a frame needs
  return p.colour ? colour_tf(p.col) : 0;
}
static inline void strip_gab_norm(const DevFusedFilterParams& p, float gw[3]) {  // host side: phase_gab's `gw` argument
  for (int c = 0; c < 3; ++c) gw[c] = 1.0f / ((1.0f + p.gab_w[c][0] * 4.0f) + p.gab_w[c][1] * 4.0f);
}

// ---- phase 3: step-1 weighted sums, A + D -> B (the dead `in` planes) on [3, 61) x [3, 29); when step 1 is the frame's last
// EPF step (LAST: epf_iters == 1) the output tile [4, 60) x [4, 28) goes through the colour stage to the output planes ----
template <bool LAST, int TF>
JXLB_PX void phase_apply1(int tid, float* s, const StripGeom& g, const DevFusedFilterParams& p, float* const out[3],
                          const uint32_t out_stride[3]) {
  const int col = tid & (kWX - 1), seg = tid / kWX;
  constexpr int lo = LAST ? kM : 3;
  if (col < lo || col >= kWX - lo) return;
  constexpr int L = LAST ? 6 : 7;
  constexpr int yend = kWY - lo;  // 29 / 28
  const int y0 = lo + seg * L;
  const int n = (yend - y0) < L ? (yend - y0) : L;
  const int gx = g.gx0 + col;
  const bool x_in = gx >= g.x0 && gx < g.x1;
  const bool x_border = epf_col_border(gx);
  const float sm_plain = epf_step_mul(p.epf, 1, false), sm_border = epf_step_mul(p.epf, 1, true);
  const int bxi = (gx >> 3) - g.bx_first;
  const float* a = s + kOffA + y0 * kWX + col;
  const float* d = s + kOffD + y0 * kWX + col;
  float* o = s + y0 * kWX + col;
  float up[3], ce[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) up[c] = a[c * kPlane - kWX], ce[c] = a[c * kPlane];
  float du = d[-kWX];  // dist_(0,1)(col, y - 1) = distance to the neighbour (0, -1)
#pragma unroll
  for (int i = 0; i < L; ++i) {
    if (i < n) {
      const int gy = g.gy0 + y0 + i;
      const int bi = ((gy >> 3) - g.by_first) * kSigX + bxi;
      const float sigma = s[kOffSigma + bi];
      float dn[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) dn[c] = a[c * kPlane + (i + 1) * kWX];
      const float dd = d[i * kWX];
      float res[3];
      if (sigma < 0.3f) {
#pragma unroll
        for (int c = 0; c < 3; ++c) res[c] = ce[c];
      } else {
        const bool border = x_border || epf_row_border(gy);
        const float nis = fmul(s[kOffInv + bi], border ? sm_border : sm_plain);
        float le[3], ri[3];
#pragma unroll
        for (int c = 0; c < 3; ++c) le[c] = a[c * kPlane + i * kWX - 1], ri[c] = a[c * kPlane + i * kWX + 1];
        const float dl = d[kPlane + i * kWX - 1], dr = d[kPlane + i * kWX];
        epf_combine(du, dd, dl, dr, nis, ce, up, dn, le, ri, res);
      }
      if (LAST) {
        if (p.colour) xyb_to_rgb_px(res, p.col, TF, s + kOffPow);
        if (x_in && gy >= g.y0 && gy < g.y1) {
#pragma unroll
          for (int c = 0; c < 3; ++c) out[c][size_t(gy) * out_stride[c] + gx] = res[c];
        }
      } else {
#pragma unroll
        for (int c = 0; c < 3; ++c) o[c * kPlane + i * kWX] = res[c];
      }
      du = dd;
#pragma unroll
      for (int c = 0; c < 3; ++c) up[c] = ce[c], ce[c] = dn[c];
    }
  }
}

// ---- phase 4: step 2 (distances on the fly) + colour, B -> the output planes on [4, 60) x [4, 28) ---------------------
// out[c] points at image pixel (0, 0) of the output plane c, stride in floats.
template <int TF>
JXLB_PX void phase_apply2(int tid, float* s, const StripGeom& g, const DevFusedFilterParams& p, float* const out[3],
                          const uint32_t out_stride[3]) {
  const int col = tid & (kWX - 1), seg = tid / kWX;
  if (col < kM || col >= kWX - kM) return;
  constexpr int L = kTY / kSegs;  // 6
  const int y0 = kM + seg * L;
  const int gx = g.gx0 + col;
  const bool x_in = gx >= g.x0 && gx < g.x1;
  const bool x_border = epf_col_border(gx);
  const float sm_plain = epf_step_mul(p.epf, 2, false), sm_border = epf_step_mul(p.epf, 2, true);
  const int bxi = (gx >> 3) - g.bx_first;
  const float s0 = p.epf.channel_scale[0], s1 = p.epf.channel_scale[1], s2 = p.epf.channel_scale[2];
  const float* b = s + y0 * kWX + col;
  float up[3], ce[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) up[c] = b[c * kPlane - kWX], ce[c] = b[c * kPlane];
  // dist_(0,1)(col, y - 1): |B(y) - B(y - 1)| per channel, scaled and added in channel order
  float du = fadd(fadd(fmul(s0, absdiff(ce[0], up[0])), fmul(s1, absdiff(ce[1], up[1]))), fmul(s2, absdiff(ce[2], up[2])));
#pragma unroll
  for (int i = 0; i < L; ++i) {
    const int gy = g.gy0 + y0 + i;
    const int bi = ((gy >> 3) - g.by_first) * kSigX + bxi;
    const float sigma = s[kOffSigma + bi];
    float dn[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) dn[c] = b[c * kPlane + (i + 1) * kWX];
    const float dd = fadd(fadd(fmul(s0, absdiff(dn[0], ce[0])), fmul(s1, absdiff(dn[1], ce[1]))), fmul(s2, absdiff(dn[2], ce[2])));
    float res[3];
    if (sigma < 0.3f) {
#pragma unroll
      for (int c = 0; c < 3; ++c) res[c] = ce[c];
    } else {
      const bool border = x_border || epf_row_border(gy);
      const float nis = fmul(s[kOffInv + bi], border ? sm_border : sm_plain);
      float le[3], ri[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) le[c] = b[c * kPlane + i * kWX - 1], ri[c] = b[c * kPlane + i * kWX + 1];
      const float dl = fadd(fadd(fmul(s0, absdiff(ce[0], le[0])), fmul(s1, absdiff(ce[1], le[1]))), fmul(s2, absdiff(ce[2], le[2])));
      const float dr = fadd(fadd(fmul(s0, absdiff(ri[0], ce[0])), fmul(s1, absdiff(ri[1], ce[1]))), fmul(s2, absdiff(ri[2], ce[2])));
      epf_combine(du, dd, dl, dr, nis, ce, up, dn, le, ri, res);
    }
    if (p.colour) xyb_to_rgb_px(res, p.col, TF, s + kOffPow);
    if (x_in && gy >= g.y0 && gy < g.y1) {
#pragma unroll
      for (int c = 0; c < 3; ++c) out[c][size_t(gy) * out_stride[c] + gx] = res[c];
    }
    du = dd;
#pragma unroll
    for (int c = 0; c < 3; ++c) up[c] = ce[c], ce[c] = dn[c];
  }
}

// The rectangle the strip kernel covers: the union of fused_filter_kernel's 32 x 32 tiles whose 40 x 40 window lies inside
// the image (tiles bx in [1, bx_last], by in [1, by_last]). Empty (x1 <= x0) when the image is too small.
struct StripRect {
  int x0, y0, x1, y1;
};
static inline StripRect strip_rect(int width, int height) {
  StripRect r{32, 32, 0, 0};
  if (width < kWX + 2 * 32 || height < kWY + 2 * 32) return r;
  const int bx_last = (width - 36) / 32, by_last = (height - 36) / 32;
  r.x1 = 32 * (bx_last + 1), r.y1 = 32 * (by_last + 1);
  return r;
}

// The general kernel's launch over the tiles the strip kernel does not cover (a 1-D grid): tile `i` of nbx x nby tiles minus
// the interior [1, bx_last] x [1, by_last] - row 0, then the rows below by_last, then the left column and the columns right of
// bx_last of the rows in between. Count: nbx * nby - bx_last * by_last.
JXLB_PX void border_tile_index(int nbx, int nby, int bx_last, int by_last, int i, int& tx, int& ty) {
  if (i < nbx) {
    tx = i, ty = 0;
    return;
  }
  i -= nbx;
  const int n_bottom = nbx * (nby - 1 - by_last);
  if (i < n_bottom) {
    ty = by_last + 1 + i / nbx, tx = i % nbx;
    return;
  }
  i -= n_bottom;
  const int per_row = 1 + (nbx - 1 - bx_last);
  ty = 1 + i / per_row;
  const int j = i % per_row;
  tx = j == 0 ? 0 : bx_last + j;
}

}  // namespace fstrip
}  // namespace jxlb
