// Per-pixel formulas of the restoration filters and the colour stage, each defined once for every kernel that evaluates it:
// the stage kernels (filters.cu), fused_filter_kernel (filters_fused.cu) and the column-strip kernel (filter_strip.cuh).
// Parity with the oracle is bit equality, so the float operations and their order are those of the reference's generic path
// (crates/jxl-render/src/filter/impls/generic/{gabor,epf}.rs, crates/jxl-color/src/{xyb.rs, tf/*.rs, gamut.rs, convert.rs}).
//
// Device code rounds every operation explicitly (the kernels are compiled with -fmad=false); ffma stands exactly where the
// reference calls mul_add. tests/emu compiles the same functions for the host, where the operators are plain C++ under
// -ffp-contract=off and std::fmaf is the same correctly rounded operation as the device's FFMA. A formula that reads a table
// takes it as an argument: the strip kernel reads its copy from shared memory, the other kernels read kSrgbPow.
#pragma once
#include "kernels.h"

#include <cmath>
#include <cstdint>
#include <cstring>

namespace jxlb {
// Their own namespace, imported into jxlb at the end. (nvcc places a nested namespace's __constant__ tables ahead of the
// including file's: kSrgbPow at offset 0 of its bank lets the strip kernel index it without adding a base.)
namespace px {

#if defined(__CUDACC__)
#define JXLB_PX __device__ __forceinline__
JXLB_PX float fadd(float a, float b) { return __fadd_rn(a, b); }
JXLB_PX float fsub(float a, float b) { return __fsub_rn(a, b); }
JXLB_PX float fmul(float a, float b) { return __fmul_rn(a, b); }
JXLB_PX float fdiv(float a, float b) { return __fdiv_rn(a, b); }
JXLB_PX float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }
JXLB_PX float fsqrt(float a) { return __fsqrt_rn(a); }
JXLB_PX uint32_t float_bits(float a) { return __float_as_uint(a); }
JXLB_PX float bits_float(uint32_t a) { return __uint_as_float(a); }
JXLB_PX int32_t float_to_int_rz(float a) { return __float2int_rz(a); }  // saturating, NaN -> 0
#else
#define JXLB_PX static inline
JXLB_PX float fadd(float a, float b) { return a + b; }
JXLB_PX float fsub(float a, float b) { return a - b; }
JXLB_PX float fmul(float a, float b) { return a * b; }
JXLB_PX float fdiv(float a, float b) { return a / b; }
JXLB_PX float ffma(float a, float b, float c) { return std::fmaf(a, b, c); }
JXLB_PX float fsqrt(float a) { return std::sqrt(a); }
JXLB_PX uint32_t float_bits(float a) {
  uint32_t u;
  std::memcpy(&u, &a, 4);
  return u;
}
JXLB_PX float bits_float(uint32_t a) {
  float f;
  std::memcpy(&f, &a, 4);
  return f;
}
JXLB_PX int32_t float_to_int_rz(float a) {  // the device conversion: saturating, NaN -> 0
  return a != a ? 0 : (a >= 2147483648.0f ? INT32_MAX : (a < -2147483648.0f ? INT32_MIN : int32_t(a)));
}
#endif
JXLB_PX float absdiff(float a, float b) { return fabsf(fsub(a, b)); }

// ---- colour ------------------------------------------------------------------------------------------------------------

// linear_to_srgb's per-exponent factor: tf/srgb.rs:31-44 assembles it from an upper and a lower byte table as
// 0x40000000 | upper << 18 | lower << 10; the 16 results are listed here.
#if defined(__CUDACC__)
__device__ __constant__ const float kSrgbPow[16] = {
#else
static const float kSrgbPow[16] = {
#endif
    0x1p+1f,       0x1.55b8p+1f, 0x1.c82p+1f, 0x1.3068p+2f, 0x1.9658p+2f, 0x1.0f38p+3f, 0x1.6a08p+3f, 0x1.e34p+3f,
    0x1.4288p+4f, 0x1.ae88p+4f, 0x1.1f58p+5f, 0x1.7f9p+5f, 0x1p+6f,       0x1.55b8p+6f, 0x1.c82p+6f, 0x1.3068p+7f};

// sRGB OETF (tf/srgb.rs:28-47, scalar path); `pow_tab` holds the values of kSrgbPow
JXLB_PX float linear_to_srgb(float v, const float* pow_tab) {
  const uint32_t bits = float_bits(v);
  const uint32_t vb = bits & 0x7fffffffu;
  const float v_adj = bits_float((vb | 0x3e800000u) & 0x3effffffu);
  float pw = 0.059914046f;
  pw = fsub(fmul(pw, v_adj), 0.10889456f);
  pw = fadd(fmul(pw, v_adj), 0.107963754f);
  pw = fadd(fmul(pw, v_adj), 0.018092343f);
  const uint32_t idx = ((vb >> 23) - 118) & 0xf;
  const float mul = pow_tab[idx];
  const float av = bits_float(vb);
  const float small = fmul(av, 12.92f);
  const float acc = fsub(fmul(pw, mul), 0.055f);
  const float res = av <= 0.0031308f ? small : acc;
  return bits_float((float_bits(res) & 0x7fffffffu) | (bits & 0x80000000u));  // copysignf(res, v)
}

// fast_powf_generic (fastmath/powf.rs:7-22, 147-156 with rational_poly.rs:2-6): rational-polynomial log2 and pow2, un-fused
JXLB_PX float fast_powf(float a, float power) {
  const int32_t x_bits = int32_t(float_bits(a));
  const int32_t exp_shifted = (x_bits - 0x3f2aaaab) >> 23;
  const float mantissa = bits_float(uint32_t(x_bits - (exp_shifted << 23)));
  const float exp_val = float(exp_shifted);
  const float x = fsub(mantissa, 1.0f);
  const float yp = fadd(fmul(fadd(fmul(7.4245873327820566e-1f, x), 1.4287160470083755f), x), -1.8503833400518310e-6f);
  const float yq = fadd(fmul(fadd(fmul(1.7409343003366853e-1f, x), 1.0096718572241148f), x), 9.9032814277590719e-1f);
  const float e = fmul(fadd(fdiv(yp, yq), exp_val), power);
  const float x_floor = floorf(e);
  const float ex = bits_float((uint32_t(float_to_int_rz(x_floor)) + 127u) << 23);
  const float frac = fsub(e, x_floor);
  float num = fadd(frac, 1.01749063e1f);
  num = fadd(fmul(num, frac), 4.88687798e1f);
  num = fadd(fmul(num, frac), 9.85506591e1f);
  num = fmul(num, ex);
  float den = fadd(fmul(2.10242958e-1f, frac), -2.22328856e-2f);
  den = fadd(fmul(den, frac), -1.94414990e1f);
  den = fadd(fmul(den, frac), 9.85506633e1f);
  return fdiv(num, den);
}

// BT.709 OETF (tf/bt709.rs:61-68)
JXLB_PX float linear_to_bt709(float a) {
  if (a <= 0.018f) return fmul(4.5f, a);
  return ffma(fast_powf(a, 0.45f), 1.099f, -0.099f);
}

// apply_gamma's scalar tail (tf.rs:62-69)
JXLB_PX float gamma_tf(float a, float gamma) { return a <= 1e-7f ? 0.0f : fast_powf(a, gamma); }

// linear_to_pq_generic (tf/pq.rs:126-142): fourth root, then a 4/4 rational polynomial (Horner, un-fused)
JXLB_PX float pq_tf(float s, float y_mult) {
  const float a = fabsf(s);
  const float a_1_4 = fsqrt(fsqrt(fmul(a, y_mult)));
  float yp, yq;
  if (a < 1e-4f) {
    yp = fadd(fmul(fadd(fmul(fadd(fmul(fadd(fmul(-2.864824e5f, a_1_4), 6.889862e4f), a_1_4), 1.352821e2f), a_1_4), 3.881234e-1f), a_1_4), 9.863406e-6f);
    yq = fadd(fmul(fadd(fmul(fadd(fmul(fadd(fmul(-2.072546e5f, a_1_4), -4.389884e4f), a_1_4), 1.608477e4f), a_1_4), 1.477719e3f), a_1_4), 3.371868e1f);
  } else {
    yp = fadd(fmul(fadd(fmul(fadd(fmul(fadd(fmul(4.838434e1f, a_1_4), 1.492516e2f), a_1_4), 5.522776e1f), a_1_4), -1.095778f), a_1_4), 1.351392e-2f);
    yq = fadd(fmul(fadd(fmul(fadd(fmul(fadd(fmul(2.590418e1f, a_1_4), 1.120607e2f), a_1_4), 9.26371e1f), a_1_4), 2.016708e1f), a_1_4), 1.012416f);
  }
  return copysignf(fdiv(yp, yq), s);
}

// XYB -> linear RGB: opsin inverse and matrix (xyb.rs:35-60, ciexyz.rs:81-87)
JXLB_PX void xyb_to_linear(float o[3], const DevColorParams& p) {
  const float xx = o[0], yy = o[1], bb = o[2];
  const float g_l = fsub(fadd(yy, xx), p.cbrt_opsin_bias[0]);
  const float g_m = fsub(fsub(yy, xx), p.cbrt_opsin_bias[1]);
  const float g_s = fsub(bb, p.cbrt_opsin_bias[2]);
  const float a = fmul(ffma(fmul(g_l, g_l), g_l, p.opsin_bias[0]), p.itscale);
  const float b = fmul(ffma(fmul(g_m, g_m), g_m, p.opsin_bias[1]), p.itscale);
  const float c = fmul(ffma(fmul(g_s, g_s), g_s, p.opsin_bias[2]), p.itscale);
  const float* m = p.matrix;
  o[0] = fadd(fadd(fmul(m[0], a), fmul(m[1], b)), fmul(m[2], c));
  o[1] = fadd(fadd(fmul(m[3], a), fmul(m[4], b)), fmul(m[5], c));
  o[2] = fadd(fadd(fmul(m[6], a), fmul(m[7], b)), fmul(m[8], c));
}

// The transfer function of an sRGB or BT.709 target: 0 none (linear), 1 sRGB, 2 BT.709
__host__ __device__ inline int colour_tf(const DevColorParams& p) { return p.apply_srgb_tf ? 1 : (p.apply_bt709_tf ? 2 : 0); }

JXLB_PX void encode_tf(float o[3], int tf, const float* srgb_pow) {
  if (tf == 1) {
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = linear_to_srgb(o[c], srgb_pow);
  } else if (tf == 2) {
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = linear_to_bt709(o[c]);
  }
}

// The filter kernels' colour stage: XYB -> linear RGB -> transfer function `tf`
JXLB_PX void xyb_to_rgb_px(float o[3], const DevColorParams& p, int tf, const float* srgb_pow) {
  xyb_to_linear(o, p);
  encode_tf(o, tf, srgb_pow);
}

// map_gamut_generic (gamut.rs:4-46) followed by the merged target matrix (convert.rs:397-466)
JXLB_PX void second_colour_stage(float o[3], const DevColorParams& p) {
  const float yl = fadd(fadd(fmul(o[0], p.luminances[0]), fmul(o[1], p.luminances[1])), fmul(o[2], p.luminances[2]));
  float gray_saturation = 0.0f, gray_luminance = 0.0f;
#pragma unroll
  for (int i = 0; i < 3; ++i) {
    const float v_sub_y = fsub(o[i], yl);
    const float inv = fdiv(1.0f, v_sub_y == 0.0f ? 1.0f : v_sub_y);
    const float v_over = fmul(o[i], inv);
    if (!(v_sub_y >= 0.0f)) gray_saturation = fmaxf(gray_saturation, v_over);
    gray_luminance = fmaxf(v_sub_y <= 0.0f ? gray_saturation : fsub(v_over, inv), gray_luminance);
  }
  float gray_mix = fadd(fmul(0.3f, fsub(gray_saturation, gray_luminance)), gray_luminance);
  gray_mix = gray_mix < 0.0f ? 0.0f : (gray_mix > 1.0f ? 1.0f : gray_mix);
  const float max_colour = fmaxf(o[2], fmaxf(o[1], fmaxf(o[0], 1.0f)));
#pragma unroll
  for (int i = 0; i < 3; ++i) o[i] = fdiv(fadd(fmul(gray_mix, fsub(yl, o[i])), o[i]), max_colour);
  const float* m = p.matrix2;
  const float t0 = fadd(fadd(fmul(m[0], o[0]), fmul(m[1], o[1])), fmul(m[2], o[2]));
  const float t1 = fadd(fadd(fmul(m[3], o[0]), fmul(m[4], o[1])), fmul(m[5], o[2]));
  const float t2 = fadd(fadd(fmul(m[6], o[0]), fmul(m[7], o[1])), fmul(m[8], o[2]));
  o[0] = p.to_luma ? t1 : t0;
  o[1] = t1;
  o[2] = t2;
}

// ---- Gaborish (gabor.rs:3-167) -----------------------------------------------------------------------------------------

// 1 / (1 + 4 w0 + 4 w1): the normalisation every output of a channel is multiplied by
JXLB_PX float gaborish_norm(float w0, float w1) { return fdiv(1.0f, fadd(fadd(1.0f, fmul(w0, 4.0f)), fmul(w1, 4.0f))); }

// A pixel none of whose eight neighbours lies outside the image, from its 3 x 3 neighbourhood (top, middle, bottom row)
JXLB_PX float gaborish_3x3(float tl, float tc, float tr, float ml, float mc, float mr, float bl, float bc, float br, float w0,
                           float w1, float gw) {
  const float sum_side = fadd(fadd(fadd(tc, ml), mr), bc);
  const float sum_diag = fadd(fadd(fadd(tl, tr), bl), br);
  return fmul(fadd(fadd(mc, fmul(sum_side, w0)), fmul(sum_diag, w1)), gw);
}

// Any pixel (x, y) of a width x height image: the formulas differ between interior pixels, the first / last row and column
// and the degenerate 1-row / 1-column images; each is the reference's. at(dx, dy) returns the sample at (x + dx, y + dy).
template <typename At>
JXLB_PX float gaborish_px(const At& at, int x, int y, int width, int height, float w0, float w1, float gw) {
  if (height == 1) {
    if (width == 1) return at(0, 0);
    const float merged_w0 = fadd(fadd(1.0f, 2.0f), w0);
    const float merged_w1 = fadd(w0, fmul(2.0f, w1));
    if (x == 0) return fmul(fadd(fmul(at(0, 0), fadd(merged_w0, merged_w1)), fmul(at(1, 0), merged_w1)), gw);
    if (x == width - 1) return fmul(fadd(fmul(at(0, 0), fadd(merged_w0, merged_w1)), fmul(at(-1, 0), merged_w1)), gw);
    return fmul(fadd(fmul(at(0, 0), merged_w0), fmul(fadd(at(-1, 0), at(1, 0)), merged_w1)), gw);
  }
  if (y == 0 || y == height - 1) {
    const int ya = (y == 0) ? 1 : -1;  // the one adjacent row
    if (width == 1) {
      const float u = at(0, ya), c = at(0, 0);
      return fmul(fadd(fmul(c, fadd(fadd(1.0f, fmul(3.0f, w0)), fmul(2.0f, w1))), fmul(u, fadd(w0, fmul(2.0f, w1)))), gw);
    }
    if (x == 0 || x == width - 1) {
      const int xo = (x == 0) ? 1 : -1;
      const float a1 = at(0, ya), a0 = at(xo, ya), c1 = at(0, 0), c0 = at(xo, 0);
      return fmul(fadd(fadd(fmul(c1, fadd(fadd(1.0f, fmul(2.0f, w0)), w1)), fmul(fadd(a1, c0), fadd(w0, w1))), fmul(a0, w1)), gw);
    }
    const float a0 = at(-1, ya), a1 = at(0, ya), a2 = at(1, ya);
    const float c0 = at(-1, 0), c1 = at(0, 0), c2 = at(1, 0);
    return fmul(fadd(fadd(c1, fmul(fadd(fadd(fadd(a1, c0), c1), c2), w0)), fmul(fadd(fadd(fadd(a0, a2), c0), c2), w1)), gw);
  }
  if (width == 1) {
    const float t = at(0, -1), c = at(0, 0), b = at(0, 1);
    const float sum_side = fadd(fadd(t, fmul(2.0f, c)), b);
    const float sum_diag = fmul(2.0f, fadd(t, b));
    return fmul(fadd(fadd(c, fmul(sum_side, w0)), fmul(sum_diag, w1)), gw);
  }
  if (x == 0 || x == width - 1) {
    const int xo = (x == 0) ? 1 : -1;
    const float t1 = at(0, -1), c1 = at(0, 0), b1 = at(0, 1);
    const float t0 = at(xo, -1), c0 = at(xo, 0), b0 = at(xo, 1);
    const float sum_side = fadd(fadd(fadd(t1, c0), c1), b1);
    const float sum_diag = fadd(fadd(fadd(t0, t1), b0), b1);
    return fmul(fadd(fadd(c1, fmul(sum_side, w0)), fmul(sum_diag, w1)), gw);
  }
  return gaborish_3x3(at(-1, -1), at(0, -1), at(1, -1), at(-1, 0), at(0, 0), at(1, 0), at(-1, 1), at(0, 1), at(1, 1), w0, w1, gw);
}

// ---- edge-preserving filter (epf.rs) -----------------------------------------------------------------------------------

// 6.6 * (1/sqrt(2) - 1) / sigma: the reference computes it for every pixel, the kernels once per 8x8 block (same operands)
JXLB_PX float epf_inv_sigma(float sigma) { return fdiv(fmul(6.6f, fsub(0.70710678118654752440f, 1.0f)), sigma); }

// Pixels in the first or last column or row of their 8x8 block take the border multiplier
JXLB_PX bool epf_col_border(int x) { return (x & 7) == 0 || (x & 7) == 7; }
JXLB_PX bool epf_row_border(int y) { return ((y + 1) & 6) == 0; }

// The factor of step `step` (0, 1, 2) that multiplies epf_inv_sigma, with the border multiplier on 8x8-block borders
JXLB_PX float epf_step_mul(const DevEpfParams& p, int step, bool border) {
  const float sm = step == 0 ? p.pass0_sigma_scale : (step == 2 ? p.pass2_sigma_scale : 1.0f);
  return border ? fmul(sm, p.border_sad_mul) : sm;
}

// Weight of a neighbour at patch distance `dist`; nis = epf_inv_sigma * epf_step_mul
JXLB_PX float epf_weight(float dist, float nis) { return fmaxf(fadd(1.0f, fmul(dist, nis)), 0.0f); }

// Neighbour offsets in the reference's order: 12 for step 0, 4 for steps 1 and 2. Offsets of the plus whose absolute
// differences make a patch distance, in the reference's summation order: 5 for steps 0 and 1 (the orders differ), the centre
// only for step 2. constexpr, so that in an unrolled loop every offset folds into an immediate address.
__host__ __device__ constexpr int epf_neighbours(int step) { return step == 0 ? 12 : 4; }
__host__ __device__ constexpr int epf_nb_x(int step, int k) {
  constexpr int k0[12] = {0, -1, 0, 1, -2, -1, 1, 2, -1, 0, 1, 0}, k1[4] = {0, 0, -1, 1};
  return step == 0 ? k0[k] : k1[k];
}
__host__ __device__ constexpr int epf_nb_y(int step, int k) {
  constexpr int k0[12] = {-2, -1, -1, -1, 0, 0, 0, 0, 1, 1, 1, 2}, k1[4] = {-1, 1, 0, 0};
  return step == 0 ? k0[k] : k1[k];
}
__host__ __device__ constexpr int epf_plus_size(int step) { return step == 2 ? 1 : 5; }
__host__ __device__ constexpr int epf_plus_x(int step, int i) {
  constexpr int p0[5] = {0, 1, 0, -1, 0}, p1[5] = {0, 0, 0, -1, 1};
  return step == 2 ? 0 : (step == 0 ? p0[i] : p1[i]);
}
__host__ __device__ constexpr int epf_plus_y(int step, int i) {
  constexpr int p0[5] = {-1, 0, 0, 0, 1}, p1[5] = {-1, 0, 1, 0, 0};
  return step == 2 ? 0 : (step == 0 ? p0[i] : p1[i]);
}

}  // namespace px
using namespace px;
}  // namespace jxlb
