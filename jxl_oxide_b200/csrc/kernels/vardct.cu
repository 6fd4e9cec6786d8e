// VarDCT stages on the device: LF dequant / chroma-from-luma / adaptive smoothing, HF dequant + chroma-from-luma, LLF insertion
// and the 27 inverse transforms. Float op order follows the reference's generic code path
// (crates/jxl-render/src/vardct/{mod.rs,transform_common.rs,generic/*.rs}); this file is
// compiled with -fmad=false and fuses only where the reference calls mul_add.
#include "kernels.h"

#include <algorithm>
#include <cstring>

namespace jxlb {

#define JXLB_TABLE_QUAL __device__ __constant__ const
#include "../host/jxl_tables.inc"
#undef JXLB_TABLE_QUAL

// TransformTypeInfo (host/frame_syntax.cc kTransformInfo): w8, h8, param, order, transpose
__device__ __constant__ const uint8_t kDevTransformInfo[27][5] = {
    {1, 1, 0, 0, 1},  {1, 1, 1, 1, 0},  {1, 1, 2, 1, 0},   {1, 1, 3, 1, 0},    {2, 2, 4, 2, 1},   {4, 4, 5, 3, 1},
    {1, 2, 6, 4, 1},  {2, 1, 6, 4, 0},  {1, 4, 7, 5, 1},   {4, 1, 7, 5, 0},    {2, 4, 8, 6, 1},   {4, 2, 8, 6, 0},
    {1, 1, 9, 1, 0},  {1, 1, 9, 1, 0},  {1, 1, 10, 1, 0},  {1, 1, 10, 1, 0},   {1, 1, 10, 1, 0},  {1, 1, 10, 1, 0},
    {8, 8, 11, 7, 1}, {4, 8, 12, 8, 1}, {8, 4, 12, 8, 0},  {16, 16, 13, 9, 1}, {8, 16, 14, 10, 1}, {16, 8, 14, 10, 0},
    {32, 32, 15, 11, 1}, {16, 32, 16, 12, 1}, {32, 16, 16, 12, 0},
};

// sec_half tables for n = 64, 128, 256 (computed on the host with cosf, dct_common.rs:57-67)
__device__ __constant__ float kSecLarge[32 + 64 + 128];
void upload_sec_large(const float* host224) { cudaMemcpyToSymbol(kSecLarge, host224, sizeof(float) * 224); }

namespace {

__device__ __forceinline__ const float* sec_half(int n) {
  switch (n) {
    case 4: return kSecHalf4;
    case 8: return kSecHalf8;
    case 16: return kSecHalf16;
    case 32: return kSecHalf32;
    case 64: return kSecLarge;
    case 128: return kSecLarge + 32;
    default: return kSecLarge + 96;
  }
}

// ---------------------------------------------------------------------------------------------
// LF (vardct/mod.rs:387-412, 544-568; generic/mod.rs:11-103)
__global__ void lf_dequant_kernel(DevFrame f, const DevLfDequantJob* jobs) {
  const DevLfDequantJob j = jobs[blockIdx.z];
  uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= j.rect.bw || y >= j.rect.bh) return;
#pragma unroll
  for (int c = 0; c < 3; ++c) {  // a subsampled channel covers the shifted part of the rectangle
    const uint32_t hs = f.hshift[c], vs = f.vshift[c];
    if (x >= ((j.rect.bw + hs) >> hs) || y >= ((j.rect.bh + vs) >> vs)) continue;
    const size_t i = size_t((j.rect.by0 >> vs) + y) * f.bw + (j.rect.bx0 >> hs) + x;
    f.lf[c][i] = __fmul_rn(float(f.lf_quant[c][i]), j.scale[c]);
  }
}

// for_each_varblocks (vardct/mod.rs:693-730): where channel c keeps the varblock starting at (bx, by); false when a
// subsampled channel skips it. The second look-up is group-local, like the reference's.
__device__ __forceinline__ bool channel_block(const DevFrame& f, uint32_t c, uint32_t bx, uint32_t by, uint32_t& dbx, uint32_t& dby) {
  dbx = bx;
  dby = by;
  if (!f.subsampled) return true;
  const uint32_t hs = f.hshift[c], vs = f.vshift[c];
  if (!(hs | vs)) return true;
  const uint32_t gx0 = bx / f.group_blocks * f.group_blocks, gy0 = by / f.group_blocks * f.group_blocks;
  const uint32_t lx = bx - gx0, ly = by - gy0;
  if (((lx >> hs) << hs) != lx || ((ly >> vs) << vs) != ly) return false;
  if (f.blk_type[size_t(gy0 + (ly >> vs)) * f.bw + gx0 + (lx >> hs)] < 0) return false;
  dbx = (gx0 >> hs) + (lx >> hs);
  dby = (gy0 >> vs) + (ly >> vs);
  return true;
}

// dequant_hf_varblock_grouped for one channel of a chroma-subsampled frame (no chroma from luma, vardct/mod.rs:353):
// one thread per coefficient of the channel's own (shifted) grid. Subsampled channels hold 8x8 varblocks only.
__global__ void hf_dequant_channel_kernel(DevFrame f, DevDequantParams p, int c) {
  const uint32_t hs = f.hshift[c], vs = f.vshift[c];
  const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= (f.cw >> hs) || y >= (f.ch >> vs)) return;
  const uint32_t sbx = x >> 3, sby = y >> 3;
  uint32_t bx = sbx, by = sby, ix, iy;
  int32_t t;
  if (hs | vs) {
    const uint32_t gbx = f.group_blocks >> hs, gby = f.group_blocks >> vs;
    bx = sbx / gbx * f.group_blocks + ((sbx % gbx) << hs);
    by = sby / gby * f.group_blocks + ((sby % gby) << vs);
    if (bx >= f.bw || by >= f.bh) return;
    t = f.blk_type[size_t(by) * f.bw + bx];
    uint32_t dbx, dby;
    if (t < 0 || !channel_block(f, c, bx, by, dbx, dby)) return;
    if (kDevTransformInfo[t][0] * kDevTransformInfo[t][1] != 1) return;
    ix = x & 7, iy = y & 7;
  } else {
    t = f.blk_type[size_t(by) * f.bw + bx];
    if (t < 0) {
      const uint32_t code = uint32_t(-t - 1);
      bx -= code & 31;
      by -= code >> 5;
      t = f.blk_type[size_t(by) * f.bw + bx];
    }
    ix = x - bx * 8, iy = y - by * 8;
  }
  const uint32_t w = uint32_t(kDevTransformInfo[t][0]) * 8;
  const uint32_t set = kDevTransformInfo[t][2], tr = kDevTransformInfo[t][4];
  const float hf_mul = float(f.blk_mul[size_t(by) * f.bw + bx]);
  const size_t i = size_t(y) * f.cw + x;
  const float mul = __fmul_rn(__fdiv_rn(65536.0f, __fmul_rn(p.global_scale, hf_mul)), p.qm_scale[c]);
  const float m = __ldg(p.matrices + p.matrix_offset[(set * 3 + c) * 2 + tr] + iy * w + ix);
  float q = float(int32_t(f.coeff[c][i]));
  if (fabsf(q) <= 1.0f) q = __fmul_rn(q, p.quant_bias[c]);
  else q = __fsub_rn(q, __fdiv_rn(p.quant_bias_numerator, q));
  q = __fmul_rn(q, m);
  q = __fmul_rn(q, mul);
  f.coeff[c][i] = __float_as_uint(q);
}

__global__ void lf_cfl_kernel(DevFrame f, float kx, float kb) {
  size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= size_t(f.bw) * f.bh) return;
  float y = f.lf[1][i];
  f.lf[0][i] = __fadd_rn(f.lf[0][i], __fmul_rn(kx, y));
  f.lf[2][i] = __fadd_rn(f.lf[2][i], __fmul_rn(kb, y));
}

// Reads the original planes `f.lf`, writes `out` (the reference updates in place but only ever
// reads original values: left neighbour is saved, up/down sums are precomputed).
__global__ void lf_smooth_kernel(DevFrame f, float* out0, float* out1, float* out2, float lf_x, float lf_y, float lf_b) {
  uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= f.bw) return;
  const size_t w = f.bw;
  const size_t i = size_t(y) * w + x;
  float* out[3] = {out0, out1, out2};
  const float lfs[3] = {lf_x, lf_y, lf_b};
  if (f.bw <= 2 || f.bh <= 2 || x == 0 || y == 0 || x + 1 >= f.bw || y + 1 >= f.bh) {
#pragma unroll
    for (int c = 0; c < 3; ++c) out[c][i] = f.lf[c][i];
    return;
  }
  const float kSelf = 0.052262735f, kSide = 0.2034514f, kDiag = 0.03348292f;
  float self[3], wa[3], gap = 0.5f;
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* p = f.lf[c];
    self[c] = p[i];
    float ud_c = __fadd_rn(p[i - w], p[i + w]);
    float ud_l = __fadd_rn(p[i - w - 1], p[i + w - 1]);
    float ud_r = __fadd_rn(p[i - w + 1], p[i + w + 1]);
    float side = __fadd_rn(__fadd_rn(p[i - 1], p[i + 1]), ud_c);
    float diag = __fadd_rn(ud_l, ud_r);
    wa[c] = __fadd_rn(__fadd_rn(__fmul_rn(self[c], kSelf), __fmul_rn(side, kSide)), __fmul_rn(diag, kDiag));
    float gap_t = __fdiv_rn(fabsf(__fsub_rn(wa[c], self[c])), lfs[c]);
    gap = fmaxf(gap, gap_t);
  }
  float gap_scale = fmaxf(__fsub_rn(3.0f, __fmul_rn(4.0f, gap)), 0.0f);
#pragma unroll
  for (int c = 0; c < 3; ++c) out[c][i] = __fadd_rn(__fmul_rn(__fsub_rn(wa[c], self[c]), gap_scale), self[c]);
}

// ---------------------------------------------------------------------------------------------
// dequant_hf_varblock_grouped + chroma_from_luma_hf_grouped (vardct/mod.rs:442-542, 570-603),
// one thread per coefficient position, all three channels.
__global__ void hf_dequant_cfl_kernel(DevFrame f, DevDequantParams p) {
  uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= f.cw || y >= f.ch) return;
  uint32_t bx = x >> 3, by = y >> 3;
  int32_t t = f.blk_type[size_t(by) * f.bw + bx];
  uint32_t ox = bx, oy = by;
  if (t < 0) {
    uint32_t code = uint32_t(-t - 1);
    ox = bx - (code & 31);
    oy = by - (code >> 5);
    t = f.blk_type[size_t(oy) * f.bw + ox];
  }
  const uint32_t w = uint32_t(kDevTransformInfo[t][0]) * 8;
  const uint32_t set = kDevTransformInfo[t][2], tr = kDevTransformInfo[t][4];
  const uint32_t ix = x - ox * 8, iy = y - oy * 8;
  const float hf_mul = float(f.blk_mul[size_t(oy) * f.bw + ox]);
  const size_t i = size_t(y) * f.cw + x;
  float v[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    float mul = __fmul_rn(__fdiv_rn(65536.0f, __fmul_rn(p.global_scale, hf_mul)), p.qm_scale[c]);
    float m = __ldg(p.matrices + p.matrix_offset[(set * 3 + c) * 2 + tr] + iy * w + ix);
    float q = float(int32_t(f.coeff[c][i]));
    if (fabsf(q) <= 1.0f) q = __fmul_rn(q, p.quant_bias[c]);
    else q = __fsub_rn(q, __fdiv_rn(p.quant_bias_numerator, q));
    q = __fmul_rn(q, m);
    q = __fmul_rn(q, mul);
    v[c] = q;
  }
  size_t ti = size_t(y >> 6) * f.w64 + (x >> 6);
  float kx = __fadd_rn(p.base_correlation_x, __fdiv_rn(float(f.x_from_y[ti]), p.colour_factor));
  float kb = __fadd_rn(p.base_correlation_b, __fdiv_rn(float(f.b_from_y[ti]), p.colour_factor));
  v[0] = __fadd_rn(v[0], __fmul_rn(kx, v[1]));
  v[2] = __fadd_rn(v[2], __fmul_rn(kb, v[1]));
#pragma unroll
  for (int c = 0; c < 3; ++c) f.coeff[c][i] = __float_as_uint(v[c]);
}

// ---------------------------------------------------------------------------------------------
// 1-D DCT (generic/dct.rs:143-293). `io` and `scratch` hold N floats each.
#define SQRT2F 1.41421356237309504880f

__device__ __forceinline__ void dct4(float* io, bool forward) {
  const float sec0 = 0.5411961f, sec1 = 1.306563f;
  float i0 = io[0], i1 = io[1], i2 = io[2], i3 = io[3];
  if (forward) {
    float sum03 = __fadd_rn(i0, i3), sum12 = __fadd_rn(i1, i2);
    float tmp0 = __fmul_rn(__fsub_rn(i0, i3), sec0), tmp1 = __fmul_rn(__fsub_rn(i1, i2), sec1);
    float out0 = __fdiv_rn(__fadd_rn(tmp0, tmp1), 4.0f), out1 = __fdiv_rn(__fsub_rn(tmp0, tmp1), 4.0f);
    io[0] = __fdiv_rn(__fadd_rn(sum03, sum12), 4.0f);
    io[1] = __fadd_rn(__fmul_rn(out0, SQRT2F), out1);
    io[2] = __fdiv_rn(__fsub_rn(sum03, sum12), 4.0f);
    io[3] = out1;
  } else {
    float tmp0 = __fmul_rn(i1, SQRT2F), tmp1 = __fadd_rn(i1, i3);
    float out0 = __fmul_rn(__fadd_rn(tmp0, tmp1), sec0), out1 = __fmul_rn(__fsub_rn(tmp0, tmp1), sec1);
    float sum02 = __fadd_rn(i0, i2), sub02 = __fsub_rn(i0, i2);
    io[0] = __fadd_rn(sum02, out0);
    io[1] = __fadd_rn(sub02, out1);
    io[2] = __fsub_rn(sub02, out1);
    io[3] = __fsub_rn(sum02, out0);
  }
}

template <int N>
struct Dct1D {
  static __device__ __noinline__ void run(float* io, float* scratch, bool forward) {
    constexpr int h = N / 2;
    float* in0 = scratch;
    float* in1 = scratch + h;
    const float* sec = sec_half(N);
    if (forward) {
      for (int i = 0; i < h; ++i) {
        in0[i] = __fdiv_rn(__fadd_rn(io[i], io[N - i - 1]), 2.0f);
        in1[i] = __fdiv_rn(__fsub_rn(io[i], io[N - i - 1]), 2.0f);
      }
      for (int i = 0; i < h; ++i) in1[i] = __fmul_rn(in1[i], sec[i]);
      Dct1D<h>::run(in0, io, true);
      Dct1D<h>::run(in1, io + h, true);
      in1[0] = __fmul_rn(in1[0], SQRT2F);
      for (int i = 0; i + 1 < h; ++i) in1[i] = __fadd_rn(in1[i], in1[i + 1]);
      for (int i = 0; i < h; ++i) io[i * 2] = in0[i];
      for (int i = 0; i < h; ++i) io[i * 2 + 1] = in1[i];
    } else {
      for (int i = 0; i < h; ++i) {
        in0[i] = io[i * 2];
        in1[i] = io[i * 2 + 1];
      }
      for (int i = 1; i < h; ++i) in1[h - i] = __fadd_rn(in1[h - i], in1[h - i - 1]);
      in1[0] = __fmul_rn(in1[0], SQRT2F);
      Dct1D<h>::run(in0, io, false);
      Dct1D<h>::run(in1, io + h, false);
      for (int i = 0; i < h; ++i) in1[i] = __fmul_rn(in1[i], sec[i]);
      for (int i = 0; i < h; ++i) {
        float a = scratch[i], b = scratch[i + h];
        io[i] = __fadd_rn(a, b);
        io[N - i - 1] = __fsub_rn(a, b);
      }
    }
  }
};

template <>
struct Dct1D<8> {
  static __device__ __forceinline__ void run(float* io, float*, bool forward) {
    const float* sec = kSecHalf8;
    if (forward) {
      float in0[4], in1[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        in0[i] = __fdiv_rn(__fadd_rn(io[i], io[7 - i]), 2.0f);
        in1[i] = __fdiv_rn(__fmul_rn(__fsub_rn(io[i], io[7 - i]), sec[i]), 2.0f);
      }
      dct4(in0, true);
#pragma unroll
      for (int i = 0; i < 4; ++i) io[i * 2] = in0[i];
      dct4(in1, true);
      in1[0] = __fmul_rn(in1[0], SQRT2F);
#pragma unroll
      for (int i = 0; i < 3; ++i) io[i * 2 + 1] = __fadd_rn(in1[i], in1[i + 1]);
      io[7] = in1[3];
    } else {
      float in0[4] = {io[0], io[2], io[4], io[6]};
      float in1[4] = {__fmul_rn(io[1], SQRT2F), __fadd_rn(io[3], io[1]), __fadd_rn(io[5], io[3]), __fadd_rn(io[7], io[5])};
      dct4(in0, false);
      dct4(in1, false);
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        float r = __fmul_rn(in1[i], sec[i]);
        io[i] = __fadd_rn(in0[i], r);
        io[7 - i] = __fsub_rn(in0[i], r);
      }
    }
  }
};

__device__ void dct1d(float* io, float* scratch, int n, bool forward) {
  switch (n) {
    case 1: return;
    case 2: {
      float t0 = __fadd_rn(io[0], io[1]), t1 = __fsub_rn(io[0], io[1]);
      if (forward) {
        io[0] = __fdiv_rn(t0, 2.0f);
        io[1] = __fdiv_rn(t1, 2.0f);
      } else {
        io[0] = t0;
        io[1] = t1;
      }
      return;
    }
    case 4: dct4(io, forward); return;
    case 8: Dct1D<8>::run(io, scratch, forward); return;
    case 16: Dct1D<16>::run(io, scratch, forward); return;
    case 32: Dct1D<32>::run(io, scratch, forward); return;
    case 64: Dct1D<64>::run(io, scratch, forward); return;
    case 128: Dct1D<128>::run(io, scratch, forward); return;
    default: Dct1D<256>::run(io, scratch, forward); return;
  }
}

struct Grid {
  float* p;
  int stride, w, h;
  __device__ __forceinline__ float& at(int x, int y) { return p[y * stride + x]; }
};

// dct_2d (generic/dct.rs:5-141), executed by a single thread on a small grid. `tmp` must hold
// 3 * max(w, h) floats.
__device__ void dct_2d_serial(Grid io, bool forward, float* tmp) {
  const int width = io.w, height = io.h;
  if (width * height <= 1) return;
  const float mul = forward ? 0.5f : 1.0f;
  if (width == 2 && height == 1) {
    float v0 = io.at(0, 0), v1 = io.at(1, 0);
    io.at(0, 0) = __fmul_rn(__fadd_rn(v0, v1), mul);
    io.at(1, 0) = __fmul_rn(__fsub_rn(v0, v1), mul);
    return;
  }
  if (width == 1 && height == 2) {
    float v0 = io.at(0, 0), v1 = io.at(0, 1);
    io.at(0, 0) = __fmul_rn(__fadd_rn(v0, v1), mul);
    io.at(0, 1) = __fmul_rn(__fsub_rn(v0, v1), mul);
    return;
  }
  if (width == 2 && height == 2) {
    float v00 = io.at(0, 0), v01 = io.at(1, 0), v10 = io.at(0, 1), v11 = io.at(1, 1);
    io.at(0, 0) = __fmul_rn(__fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(v00, v01), v10), v11), mul), mul);
    io.at(1, 0) = __fmul_rn(__fmul_rn(__fsub_rn(__fadd_rn(__fsub_rn(v00, v01), v10), v11), mul), mul);
    io.at(0, 1) = __fmul_rn(__fmul_rn(__fsub_rn(__fsub_rn(__fadd_rn(v00, v01), v10), v11), mul), mul);
    io.at(1, 1) = __fmul_rn(__fmul_rn(__fadd_rn(__fsub_rn(__fsub_rn(v00, v01), v10), v11), mul), mul);
    return;
  }
  float* line = tmp;
  float* scratch = tmp + (width > height ? width : height);
  if (height == 1) {
    for (int x = 0; x < width; ++x) line[x] = io.at(x, 0);
    dct1d(line, scratch, width, forward);
    for (int x = 0; x < width; ++x) io.at(x, 0) = line[x];
    return;
  }
  if (width == 1) {
    for (int y = 0; y < height; ++y) line[y] = io.at(0, y);
    dct1d(line, scratch, height, forward);
    for (int y = 0; y < height; ++y) io.at(0, y) = line[y];
    return;
  }
  if (height == 2) {
    for (int x = 0; x < width; ++x) {
      float t0 = io.at(x, 0), t1 = io.at(x, 1);
      io.at(x, 0) = __fmul_rn(__fadd_rn(t0, t1), mul);
      io.at(x, 1) = __fmul_rn(__fsub_rn(t0, t1), mul);
    }
    for (int r = 0; r < 2; ++r) {
      for (int x = 0; x < width; ++x) line[x] = io.at(x, r);
      dct1d(line, scratch, width, forward);
      for (int x = 0; x < width; ++x) io.at(x, r) = line[x];
    }
    return;
  }
  if (width == 2) {
    for (int y = 0; y < height; ++y) {
      float v0 = io.at(0, y), v1 = io.at(1, y);
      io.at(0, y) = __fmul_rn(__fadd_rn(v0, v1), mul);
      io.at(1, y) = __fmul_rn(__fsub_rn(v0, v1), mul);
    }
    for (int c = 0; c < 2; ++c) {
      for (int y = 0; y < height; ++y) line[y] = io.at(c, y);
      dct1d(line, scratch, height, forward);
      for (int y = 0; y < height; ++y) io.at(c, y) = line[y];
    }
    return;
  }
  for (int y = 0; y < height; ++y) {
    for (int x = 0; x < width; ++x) line[x] = io.at(x, y);
    dct1d(line, scratch, width, forward);
    for (int x = 0; x < width; ++x) io.at(x, y) = line[x];
  }
  for (int x = 0; x < width; ++x) {
    for (int y = 0; y < height; ++y) line[y] = io.at(x, y);
    dct1d(line, scratch, height, forward);
    for (int y = 0; y < height; ++y) io.at(x, y) = line[y];
  }
}

// generic/transform.rs -------------------------------------------------------------------------
__device__ void aux_idct2(Grid b, int size, float* s /* size*size */) {
  const int n = size / 2;
  for (int y = 0; y < n; ++y)
    for (int x = 0; x < n; ++x) {
      float c00 = b.at(x, y), c01 = b.at(x + n, y), c10 = b.at(x, y + n), c11 = b.at(x + n, y + n);
      s[(2 * y) * size + 2 * x] = __fadd_rn(__fadd_rn(__fadd_rn(c00, c01), c10), c11);
      s[(2 * y) * size + 2 * x + 1] = __fsub_rn(__fsub_rn(__fadd_rn(c00, c01), c10), c11);
      s[(2 * y + 1) * size + 2 * x] = __fsub_rn(__fadd_rn(__fsub_rn(c00, c01), c10), c11);
      s[(2 * y + 1) * size + 2 * x + 1] = __fadd_rn(__fsub_rn(__fsub_rn(c00, c01), c10), c11);
    }
  for (int y = 0; y < size; ++y)
    for (int x = 0; x < size; ++x) b.at(x, y) = s[y * size + x];
}

// All 8x8 "special" transforms, executed by one thread on an 8x8 grid in shared memory.
__device__ void transform_special(Grid c, int type, float* scratch /* 64 + 48 floats */) {
  float* tmp = scratch + 64;
  if (type == 2) {  // Dct2
    aux_idct2(c, 2, scratch);
    aux_idct2(c, 4, scratch);
    aux_idct2(c, 8, scratch);
  } else if (type == 3) {  // Dct4
    aux_idct2(c, 2, scratch);
    for (int y = 0; y < 2; ++y)
      for (int x = 0; x < 2; ++x) {
        Grid s{scratch + (y * 2 + x) * 16, 4, 4, 4};
        for (int iy = 0; iy < 4; ++iy)
          for (int ix = 0; ix < 4; ++ix) s.at(iy, ix) = c.at(x + ix * 2, y + iy * 2);
      }
    for (int k = 0; k < 4; ++k) dct_2d_serial(Grid{scratch + k * 16, 4, 4, 4}, false, tmp);
    for (int y = 0; y < 2; ++y)
      for (int x = 0; x < 2; ++x)
        for (int iy = 0; iy < 4; ++iy)
          for (int ix = 0; ix < 4; ++ix) c.at(x * 4 + ix, y * 4 + iy) = scratch[(y * 2 + x) * 16 + iy * 4 + ix];
  } else if (type == 1) {  // Hornuss
    aux_idct2(c, 2, scratch);
    for (int y = 0; y < 2; ++y)
      for (int x = 0; x < 2; ++x) {
        float* s = scratch + (y * 2 + x) * 16;
        for (int iy = 0; iy < 4; ++iy)
          for (int ix = 0; ix < 4; ++ix) s[iy * 4 + ix] = c.at(x + ix * 2, y + iy * 2);
        float residual_sum = 0.0f;
        for (int i = 1; i < 16; ++i) residual_sum = __fadd_rn(residual_sum, s[i]);
        float avg = __fsub_rn(s[0], __fdiv_rn(residual_sum, 16.0f));
        s[0] = s[5];
        s[5] = 0.0f;
        for (int i = 0; i < 16; ++i) s[i] = __fadd_rn(s[i], avg);
      }
    for (int y = 0; y < 2; ++y)
      for (int x = 0; x < 2; ++x)
        for (int iy = 0; iy < 4; ++iy)
          for (int ix = 0; ix < 4; ++ix) c.at(x * 4 + ix, y * 4 + iy) = scratch[(y * 2 + x) * 16 + iy * 4 + ix];
  } else if (type == 12 || type == 13) {  // Dct4x8 / Dct8x4
    float coeff0 = c.at(0, 0), coeff1 = c.at(0, 1);
    c.at(0, 0) = __fadd_rn(coeff0, coeff1);
    c.at(0, 1) = __fsub_rn(coeff0, coeff1);
    for (int idx = 0; idx < 2; ++idx) {
      Grid s{scratch + idx * 32, 8, 8, 4};
      for (int iy = 0; iy < 4; ++iy)
        for (int ix = 0; ix < 8; ++ix) s.at(ix, iy) = c.at(ix, iy * 2 + idx);
      dct_2d_serial(s, false, tmp);
    }
    if (type == 13) {
      for (int y = 0; y < 8; ++y)
        for (int x = 0; x < 8; ++x) c.at(y, x) = scratch[y * 8 + x];
    } else {
      for (int y = 0; y < 8; ++y)
        for (int x = 0; x < 8; ++x) c.at(x, y) = scratch[y * 8 + x];
    }
  } else {  // Afv0..3
    const int n = type - 14;
    const int flip_x = n % 2, flip_y = n / 2;
    float* coeff_afv = scratch;        // 16
    float* samples_afv = scratch + 16; // 16
    float* s4x4 = scratch + 32;        // 16
    float* s4x8 = scratch + 48;        // 32
    float* tmp2 = scratch + 80;        // 24 (3 * 8)
    coeff_afv[0] = __fmul_rn(__fadd_rn(__fadd_rn(c.at(0, 0), c.at(1, 0)), c.at(0, 1)), 4.0f);
    for (int idx = 1; idx < 16; ++idx) coeff_afv[idx] = c.at(2 * (idx % 4), 2 * (idx / 4));
    for (int j = 0; j < 16; ++j) samples_afv[j] = 0.0f;
    for (int i = 0; i < 16; ++i)
      for (int j = 0; j < 16; ++j) samples_afv[j] = __fmaf_rn(coeff_afv[i], kAfvBasis[i][j], samples_afv[j]);
    for (int i = 0; i < 16; ++i) s4x4[i] = 0.0f;
    for (int i = 0; i < 32; ++i) s4x8[i] = 0.0f;
    s4x4[0] = __fadd_rn(__fsub_rn(c.at(0, 0), c.at(1, 0)), c.at(0, 1));
    for (int iy = 0; iy < 4; ++iy)
      for (int ix = 0; ix < 4; ++ix) {
        if ((ix | iy) == 0) continue;
        s4x4[ix * 4 + iy] = c.at(2 * ix + 1, 2 * iy);
      }
    dct_2d_serial(Grid{s4x4, 4, 4, 4}, false, tmp2);
    s4x8[0] = __fsub_rn(c.at(0, 0), c.at(0, 1));
    for (int iy = 0; iy < 4; ++iy)
      for (int ix = 0; ix < 8; ++ix) {
        if ((ix | iy) == 0) continue;
        s4x8[iy * 8 + ix] = c.at(ix, 2 * iy + 1);
      }
    dct_2d_serial(Grid{s4x8, 8, 8, 4}, false, tmp2);
    for (int iy = 0; iy < 4; ++iy) {
      int afv_y = flip_y == 0 ? iy : 3 - iy;
      for (int ix = 0; ix < 4; ++ix) {
        int afv_x = flip_x == 0 ? ix : 3 - ix;
        c.at(flip_x * 4 + ix, flip_y * 4 + iy) = samples_afv[afv_y * 4 + afv_x];
      }
    }
    for (int iy = 0; iy < 4; ++iy)
      for (int ix = 0; ix < 4; ++ix) c.at((1 - flip_x) * 4 + ix, flip_y * 4 + iy) = s4x4[iy * 4 + ix];
    for (int iy = 0; iy < 4; ++iy)
      for (int ix = 0; ix < 8; ++ix) c.at(ix, (1 - flip_y) * 4 + iy) = s4x8[iy * 8 + ix];
  }
}

// transform_varblocks_inner (transform_common.rs:11-75): one CTA per (8x8 cell, channel); cells
// that are not a varblock origin exit immediately. First, correctness-oriented version: rows then
// columns straight on the coefficient plane (L1/L2 resident), one thread per line.
//
// Varblocks are independent, so the frame is first sorted into three work lists by size class and
// each class gets a persistent (grid-stride) kernel shaped for it:
//   small  (8x8 cells: DCT8 and the nine "special" 8x8 transforms): 8 threads per block, one row /
//          column per thread in registers, 32 blocks per CTA;
//   medium (16x8 ... 32x32): one warp per block, tile staged in shared memory (stride 33), one
//          row / column per lane in registers;
//   large  (64x64 ... 256x256): one 64-thread CTA per block, line buffers in shared memory.
// Every variant performs exactly the reference's operations per line (rows first, then columns,
// generic/dct.rs:93-140), so results are bit-identical to the single-threaded formulation.

// Medium class, by shape (width x height in 8x8 cells): 2x1 1x2 2x2 4x1 1x4 4x2 2x4 4x4. The medium kernel walks the shapes
// one after the other so that the warps of an SM execute the same transform sizes at the same time (its unrolled
// 8 / 16 / 32-point transforms do not fit the instruction cache together: instruction fetch was the top stall).
constexpr int kMediumShapes = 8;
__host__ __device__ inline int medium_shape(int w8, int h8) {
  return w8 == 2 ? (h8 == 1 ? 0 : (h8 == 2 ? 2 : 6)) : (w8 == 1 ? (h8 == 2 ? 1 : 4) : (h8 == 1 ? 3 : (h8 == 2 ? 5 : 7)));
}
// The ten transform types of one 8x8 cell (DCT8, Hornuss, DCT2, DCT4, DCT4x8, DCT8x4, AFV0-3) each get their own list:
// the 8-thread groups of a warp then work on the same type and take the same branch of the transform.
constexpr int kSmallTypes = 10;
__host__ __device__ inline int small_type_index(int t) { return t < 4 ? t : t - 8; }  // types 0-3 and 12-17
struct TransformLists {
  uint32_t* counts;  // [0]: unused, [2], [3]: large64, large256; [4..11]: medium shapes; [12..21]: small types
  uint32_t* items[4];
  uint32_t* shape_items[kMediumShapes];
  uint32_t* small_items[kSmallTypes];
};

// One list slot per varblock. The lanes of a warp that append to the same list reserve their slots with ONE atomic
// (match_any): a frame has half a million cells and a dozen counters, and one atomic per cell serialises on them.
__global__ void classify_varblocks_kernel(DevFrame f, TransformLists L) {
  const uint32_t bx = blockIdx.x * blockDim.x + threadIdx.x, by = blockIdx.y * blockDim.y + threadIdx.y;
  int key = -1;  // counter index: 2 / 3 large, 4 + shape medium, 12 + type small
  if (bx < f.bw && by < f.bh) {
    const int32_t t = f.blk_type[size_t(by) * f.bw + bx];
    if (t >= 0) {
      const int m = max(int(kDevTransformInfo[t][0]), int(kDevTransformInfo[t][1]));
      const int cls = m == 1 ? 0 : (m <= 4 ? 1 : (m == 8 ? 2 : 3));
      key = cls == 1 ? 4 + medium_shape(kDevTransformInfo[t][0], kDevTransformInfo[t][1]) : (cls == 0 ? 12 + small_type_index(t) : cls);
    }
  }
  const uint32_t peers = __match_any_sync(0xffffffffu, key);
  if (key < 0) return;
  const uint32_t lane = (threadIdx.y * blockDim.x + threadIdx.x) & 31;
  const int leader = __ffs(int(peers)) - 1;
  uint32_t base = 0;
  if (int(lane) == leader) base = atomicAdd(L.counts + key, uint32_t(__popc(peers)));
  base = __shfl_sync(peers, base, leader);
  const uint32_t slot = base + uint32_t(__popc(peers & ((1u << lane) - 1)));
  uint32_t* list = key >= 12 ? L.small_items[key - 12] : (key >= 4 ? L.shape_items[key - 4] : L.items[key]);
  list[slot] = bx | (by << 16);
}

// Register-resident inverse DCT: the operation sequence of Dct1D<N>::run(inverse).
template <int N>
struct RegIdct {
  static __device__ __forceinline__ void run(float (&io)[N]) {
    constexpr int h = N / 2;
    const float* sec = N == 8 ? kSecHalf8 : (N == 16 ? kSecHalf16 : kSecHalf32);
    float in0[h], in1[h];
#pragma unroll
    for (int i = 0; i < h; ++i) {
      in0[i] = io[2 * i];
      in1[i] = io[2 * i + 1];
    }
#pragma unroll
    for (int i = 1; i < h; ++i) in1[h - i] = __fadd_rn(in1[h - i], in1[h - i - 1]);
    in1[0] = __fmul_rn(in1[0], SQRT2F);
    RegIdct<h>::run(in0);
    RegIdct<h>::run(in1);
#pragma unroll
    for (int i = 0; i < h; ++i) {
      const float r = __fmul_rn(in1[i], sec[i]);
      io[i] = __fadd_rn(in0[i], r);
      io[N - i - 1] = __fsub_rn(in0[i], r);
    }
  }
};
template <>
struct RegIdct<4> {
  static __device__ __forceinline__ void run(float (&io)[4]) { dct4(io, false); }
};

// LLF of a multi-cell varblock: forward DCT of its bw x bh LF samples, rescaled
// (transform_common.rs:33-58). `llf` holds bw*bh floats, `tmp` 3*max(bw,bh).
// Shapes up to 4x4 cells, by one thread in registers: exactly the branches dct_2d_serial() takes for
// these sizes (generic/dct.rs:5-141), unrolled.
__device__ __forceinline__ void llf_fwd4(float* a, int stride) {  // forward DCT-4 on a[0], a[stride], ...
  float v[4] = {a[0], a[stride], a[2 * stride], a[3 * stride]};
  dct4(v, true);
  a[0] = v[0], a[stride] = v[1], a[2 * stride] = v[2], a[3 * stride] = v[3];
}
__device__ void compute_llf_small(const DevFrame& f, int c, uint32_t bx, uint32_t by, int bw, int bh, float* llf) {
  const float* lf = f.lf[c] + size_t(by) * f.bw + bx;
  float a[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) a[i] = 0.0f;
#pragma unroll
  for (int y = 0; y < 4; ++y)
#pragma unroll
    for (int x = 0; x < 4; ++x)
      if (y < bh && x < bw) a[y * 4 + x] = lf[size_t(y) * f.bw + x];  // a[] has row stride 4 whatever bw is
  const float mul = 0.5f;
  if (bw == 2 && bh == 1) {
    const float v0 = a[0], v1 = a[1];
    a[0] = __fmul_rn(__fadd_rn(v0, v1), mul);
    a[1] = __fmul_rn(__fsub_rn(v0, v1), mul);
  } else if (bw == 1 && bh == 2) {
    const float v0 = a[0], v1 = a[4];
    a[0] = __fmul_rn(__fadd_rn(v0, v1), mul);
    a[4] = __fmul_rn(__fsub_rn(v0, v1), mul);
  } else if (bw == 2 && bh == 2) {
    const float v00 = a[0], v01 = a[1], v10 = a[4], v11 = a[5];
    a[0] = __fmul_rn(__fmul_rn(__fadd_rn(__fadd_rn(__fadd_rn(v00, v01), v10), v11), mul), mul);
    a[1] = __fmul_rn(__fmul_rn(__fsub_rn(__fadd_rn(__fsub_rn(v00, v01), v10), v11), mul), mul);
    a[4] = __fmul_rn(__fmul_rn(__fsub_rn(__fsub_rn(__fadd_rn(v00, v01), v10), v11), mul), mul);
    a[5] = __fmul_rn(__fmul_rn(__fadd_rn(__fsub_rn(__fsub_rn(v00, v01), v10), v11), mul), mul);
  } else if (bh == 1) {  // 4 x 1
    llf_fwd4(a, 1);
  } else if (bw == 1) {  // 1 x 4
    llf_fwd4(a, 4);
  } else if (bh == 2) {  // 4 x 2: butterflies down the columns, then the two rows
#pragma unroll
    for (int x = 0; x < 4; ++x) {
      const float t0 = a[x], t1 = a[4 + x];
      a[x] = __fmul_rn(__fadd_rn(t0, t1), mul);
      a[4 + x] = __fmul_rn(__fsub_rn(t0, t1), mul);
    }
    llf_fwd4(a, 1);
    llf_fwd4(a + 4, 1);
  } else if (bw == 2) {  // 2 x 4: butterflies along the rows, then the two columns
#pragma unroll
    for (int y = 0; y < 4; ++y) {
      const float v0 = a[y * 4], v1 = a[y * 4 + 1];
      a[y * 4] = __fmul_rn(__fadd_rn(v0, v1), mul);
      a[y * 4 + 1] = __fmul_rn(__fsub_rn(v0, v1), mul);
    }
    llf_fwd4(a, 4);
    llf_fwd4(a + 1, 4);
  } else {  // 4 x 4: rows, then columns
#pragma unroll
    for (int y = 0; y < 4; ++y) llf_fwd4(a + y * 4, 1);
#pragma unroll
    for (int x = 0; x < 4; ++x) llf_fwd4(a + x, 4);
  }
  const int logbw = 31 - __clz(bw), logbh = 31 - __clz(bh);
#pragma unroll
  for (int y = 0; y < 4; ++y)
#pragma unroll
    for (int x = 0; x < 4; ++x)
      if (y < bh && x < bw)
        llf[y * bw + x] = __fdiv_rn(a[y * 4 + x], __fmul_rn(kScaleF[y << (5 - logbh)], kScaleF[x << (5 - logbw)]));
}

// The nine "special" 8x8 transforms (generic/transform.rs:50-240) by the 8 threads of a group:
// the same per-element operation sequences as transform_special(), with the independent 1-D
// transforms / butterflies / dot products spread over the threads. `g`: the 8x8 block (row-major,
// stride 8), `s`: 128 floats of scratch, both in shared memory; `r`: thread index in the group.
__device__ __forceinline__ void idct4_strided(float* p, int stride) {
  float v[4] = {p[0], p[stride], p[2 * stride], p[3 * stride]};
  dct4(v, false);
  p[0] = v[0], p[stride] = v[1], p[2 * stride] = v[2], p[3 * stride] = v[3];
}
__device__ __forceinline__ void idct8_contig(float* p) {
  float v[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) v[i] = p[i];
  RegIdct<8>::run(v);
#pragma unroll
  for (int i = 0; i < 8; ++i) p[i] = v[i];
}

__device__ void transform_special_coop(float* g, int type, float* s, int r, uint32_t gmask) {
  auto aux_idct2_coop = [&](int size) {  // aux_idct2
    const int n = size / 2;
    for (int it = r; it < n * n; it += 8) {
      const int y = it / n, x = it % n;
      const float c00 = g[y * 8 + x], c01 = g[y * 8 + x + n], c10 = g[(y + n) * 8 + x], c11 = g[(y + n) * 8 + x + n];
      s[(2 * y) * size + 2 * x] = __fadd_rn(__fadd_rn(__fadd_rn(c00, c01), c10), c11);
      s[(2 * y) * size + 2 * x + 1] = __fsub_rn(__fsub_rn(__fadd_rn(c00, c01), c10), c11);
      s[(2 * y + 1) * size + 2 * x] = __fsub_rn(__fadd_rn(__fsub_rn(c00, c01), c10), c11);
      s[(2 * y + 1) * size + 2 * x + 1] = __fadd_rn(__fsub_rn(__fsub_rn(c00, c01), c10), c11);
    }
    __syncwarp(gmask);
    for (int idx = r; idx < size * size; idx += 8) g[(idx / size) * 8 + idx % size] = s[idx];
    __syncwarp(gmask);
  };
  if (type == 2) {  // Dct2
    aux_idct2_coop(2);
    aux_idct2_coop(4);
    aux_idct2_coop(8);
  } else if (type == 3 || type == 1) {  // Dct4 / Hornuss: four 4x4 sub-blocks of interleaved samples
    aux_idct2_coop(2);
    for (int e = r; e < 64; e += 8) {  // s[(y*2+x)*16 + iy*4 + ix] <- (Dct4: transposed) sample (x + 2ix, y + 2iy)
      const int sub = e >> 4, iy = (e >> 2) & 3, ix = e & 3, y = sub >> 1, x = sub & 1;
      const float v = g[(y + iy * 2) * 8 + x + ix * 2];
      if (type == 3) s[sub * 16 + ix * 4 + iy] = v;
      else s[sub * 16 + iy * 4 + ix] = v;
    }
    __syncwarp(gmask);
    if (type == 3) {
      for (int it = r; it < 16; it += 8) idct4_strided(s + (it >> 2) * 16 + (it & 3) * 4, 1);  // rows
      __syncwarp(gmask);
      for (int it = r; it < 16; it += 8) idct4_strided(s + (it >> 2) * 16 + (it & 3), 4);      // columns
    } else if (r < 4) {
      float* q = s + r * 16;
      float residual_sum = 0.0f;
      for (int i = 1; i < 16; ++i) residual_sum = __fadd_rn(residual_sum, q[i]);
      const float avg = __fsub_rn(q[0], __fdiv_rn(residual_sum, 16.0f));
      q[0] = q[5];
      q[5] = 0.0f;
      for (int i = 0; i < 16; ++i) q[i] = __fadd_rn(q[i], avg);
    }
    __syncwarp(gmask);
    for (int e = r; e < 64; e += 8) {
      const int sub = e >> 4, iy = (e >> 2) & 3, ix = e & 3, y = sub >> 1, x = sub & 1;
      g[(y * 4 + iy) * 8 + x * 4 + ix] = s[sub * 16 + iy * 4 + ix];
    }
    __syncwarp(gmask);
  } else if (type == 12 || type == 13) {  // Dct4x8 / Dct8x4
    if (r == 0) {
      const float coeff0 = g[0], coeff1 = g[8];
      g[0] = __fadd_rn(coeff0, coeff1);
      g[8] = __fsub_rn(coeff0, coeff1);
    }
    __syncwarp(gmask);
    for (int e = r; e < 64; e += 8) {  // s[idx*32 + iy*8 + ix] <- sample (ix, 2iy + idx)
      const int idx = e >> 5, iy = (e >> 3) & 3, ix = e & 7;
      s[e] = g[(iy * 2 + idx) * 8 + ix];
    }
    __syncwarp(gmask);
    idct8_contig(s + r * 8);  // 2 x 4 rows of 8
    __syncwarp(gmask);
    for (int it = r; it < 16; it += 8) idct4_strided(s + (it >> 3) * 32 + (it & 7), 8);  // 2 x 8 columns of 4
    __syncwarp(gmask);
    for (int e = r; e < 64; e += 8) {
      const int y = e >> 3, x = e & 7;
      if (type == 13) g[x * 8 + y] = s[e];
      else g[e] = s[e];
    }
    __syncwarp(gmask);
  } else {  // Afv0..3
    const int n = type - 14;
    const int flip_x = n % 2, flip_y = n / 2;
    float* coeff_afv = s;         // 16
    float* samples_afv = s + 16;  // 16
    float* s4x4 = s + 32;         // 16
    float* s4x8 = s + 48;         // 32
    for (int e = r; e < 64; e += 8) {
      if (e < 16) {
        coeff_afv[e] = e == 0 ? __fmul_rn(__fadd_rn(__fadd_rn(g[0], g[1]), g[8]), 4.0f) : g[(2 * (e / 4)) * 8 + 2 * (e % 4)];
      } else if (e < 32) {
        const int k = e - 16, iy = k >> 2, ix = k & 3;  // s4x4[ix*4 + iy] <- (2ix+1, 2iy)
        s4x4[ix * 4 + iy] = (ix | iy) == 0 ? __fadd_rn(__fsub_rn(g[0], g[1]), g[8]) : g[(2 * iy) * 8 + 2 * ix + 1];
      } else {
        const int k = e - 32, iy = k >> 3, ix = k & 7;  // s4x8[iy*8 + ix] <- (ix, 2iy+1)
        s4x8[k] = (ix | iy) == 0 ? __fsub_rn(g[0], g[8]) : g[(2 * iy + 1) * 8 + ix];
      }
    }
    __syncwarp(gmask);
    for (int j = r; j < 16; j += 8) {
      float acc = 0.0f;
#pragma unroll
      for (int i = 0; i < 16; ++i) acc = __fmaf_rn(coeff_afv[i], kAfvBasis[i][j], acc);
      samples_afv[j] = acc;
    }
    if (r < 4) idct4_strided(s4x4 + r * 4, 1);  // 4x4 rows
    else idct8_contig(s4x8 + (r - 4) * 8);      // 4x8 rows
    __syncwarp(gmask);
    idct4_strided(s4x8 + r, 8);                 // 4x8 columns
    if (r < 4) idct4_strided(s4x4 + r, 4);      // 4x4 columns
    __syncwarp(gmask);
    for (int e = r; e < 64; e += 8) {
      const int y = e >> 3, x = e & 7;
      const int qx = x >> 2, qy = y >> 2, ix = x & 3, iy = y & 3;
      float v;
      if (qy == flip_y) {
        if (qx == flip_x) v = samples_afv[(flip_y == 0 ? iy : 3 - iy) * 4 + (flip_x == 0 ? ix : 3 - ix)];
        else v = s4x4[iy * 4 + ix];
      } else {
        v = s4x8[iy * 8 + x];
      }
      g[e] = v;
    }
    __syncwarp(gmask);
  }
}

// dequant_hf_varblock_grouped + chroma_from_luma_hf_grouped (vardct/mod.rs:442-542, 570-603) folded into the load
// stage of the inverse transforms: per varblock, the three channels are dequantised together (chroma from luma needs
// the dequantised Y coefficient at the same position), then transformed. Same operations in the same order as
// hf_dequant_cfl_kernel, so the result is bit-identical to the two-pass form.
struct DeqBlock {
  float mul[3];         // 65536 / (global_scale * hf_mul) * qm_scale[c]
  const float* mat[3];  // the block's weight matrices (normal or transposed), row stride = block width
};
__device__ __forceinline__ DeqBlock deq_block(const DevFrame& f, const DevDequantParams& p, int32_t t, uint32_t bx, uint32_t by) {
  DeqBlock d;
  const uint32_t set = kDevTransformInfo[t][2], tr = kDevTransformInfo[t][4];
  const float hf_mul = float(f.blk_mul[size_t(by) * f.bw + bx]);
  const float base = __fdiv_rn(65536.0f, __fmul_rn(p.global_scale, hf_mul));
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    d.mul[c] = __fmul_rn(base, p.qm_scale[c]);
    d.mat[c] = p.matrices + p.matrix_offset[(set * 3 + c) * 2 + tr];
  }
  return d;
}
__device__ __forceinline__ float deq_one(uint32_t raw, float m, float mul, float qb, float qbn) {
  // Most coefficients are zero: 0 * quant_bias is a signed zero that the positive matrix weight (validated by the
  // parser) and multiplier leave as it is, so the zero case needs one multiplication, and the division below stays off
  // the common path.
  if (raw == 0) return __fmul_rn(0.0f, qb);
  float q = float(int32_t(raw));
  if (fabsf(q) <= 1.0f) q = __fmul_rn(q, qb);
  else q = __fsub_rn(q, __fdiv_rn(qbn, q));
  q = __fmul_rn(q, m);
  return __fmul_rn(q, mul);
}
// chroma-from-luma factors of the 64x64 tile that holds coefficient position (x, y) (frame coordinates)
__device__ __forceinline__ void cfl_factors(const DevFrame& f, const DevDequantParams& p, uint32_t x, uint32_t y, float& kx, float& kb) {
  const size_t ti = size_t(y >> 6) * f.w64 + (x >> 6);
  kx = __fadd_rn(p.base_correlation_x, __fdiv_rn(float(f.x_from_y[ti]), p.colour_factor));
  kb = __fadd_rn(p.base_correlation_b, __fdiv_rn(float(f.b_from_y[ti]), p.colour_factor));
}

// Measured: idct_small requesting the three channels' rows of a block together costs registers and a third of its warps;
// idct_medium trips of 8 rows beat 4 and 16.
constexpr int kMediumTrip = 8;      // idct_medium: tile rows whose loads are in flight together
constexpr int kSmallMinBlocks = 3;  // idct_small: resident CTAs per SM asked of the register allocator
constexpr int kSmallGroups = 32;    // 8-thread groups per CTA
template <bool DEQ>
__global__ void __launch_bounds__(kSmallGroups * 8, kSmallMinBlocks) idct_small_kernel(DevFrame f, DevDequantParams dq, TransformLists lists) {
  __shared__ float s_tile[kSmallGroups][72];      // 8 x 9
  __shared__ float s_special[kSmallGroups][192];  // 8 x 8 copy + 128 scratch
  const uint32_t group = threadIdx.x >> 3, r = threadIdx.x & 7;
  const uint32_t gmask = 0xffu << (8 * ((threadIdx.x & 31) >> 3));
  // DEQ: one work item per varblock (the three channels together: Y first, its dequantised row feeds the chroma
  // channels); else one per (varblock, channel)
  float* tile = s_tile[group];
#pragma unroll 1
  for (int list = 0; list < kSmallTypes; ++list) {
  const uint32_t* __restrict__ items = lists.small_items[list];
  const uint32_t total = DEQ ? lists.counts[12 + list] : lists.counts[12 + list] * 3;
  for (uint32_t work = blockIdx.x * kSmallGroups + group; work < total; work += gridDim.x * kSmallGroups) {
    const uint32_t item = items[DEQ ? work : work / 3];
    const uint32_t sbx = item & 0xffff, sby = item >> 16;
    const int32_t t = f.blk_type[size_t(sby) * f.bw + sbx];
    DeqBlock db;
    float kx = 0.0f, kb = 0.0f, vy[8];
    if (DEQ) {
      db = deq_block(f, dq, t, sbx, sby);
      cfl_factors(f, dq, sbx * 8, sby * 8, kx, kb);
    }
#pragma unroll 1
    for (int ci = 0; ci < (DEQ ? 3 : 1); ++ci) {
      const uint32_t c = DEQ ? (ci == 0 ? 1u : (ci == 1 ? 0u : 2u)) : work % 3;
      uint32_t bx, by;  // where channel c keeps this block
      if (!channel_block(f, c, sbx, sby, bx, by)) continue;
      float* row = reinterpret_cast<float*>(f.coeff[c]) + (size_t(by) * 8 + r) * f.cw + size_t(bx) * 8;
      const float4 lo = *reinterpret_cast<const float4*>(row), hi = *reinterpret_cast<const float4*>(row + 4);
      float v[8] = {lo.x, lo.y, lo.z, lo.w, hi.x, hi.y, hi.z, hi.w};
      if (DEQ) {
        const float4 m0 = __ldg(reinterpret_cast<const float4*>(db.mat[c] + r * 8));
        const float4 m1 = __ldg(reinterpret_cast<const float4*>(db.mat[c] + r * 8 + 4));
        const float m[8] = {m0.x, m0.y, m0.z, m0.w, m1.x, m1.y, m1.z, m1.w};
        const float k = c == 0 ? kx : kb;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const float q = deq_one(__float_as_uint(v[i]), m[i], db.mul[c], dq.quant_bias[c], dq.quant_bias_numerator);
          if (c == 1) vy[i] = v[i] = q;
          else v[i] = __fadd_rn(q, __fmul_rn(k, vy[i]));
        }
      }
      if (r == 0) v[0] = f.lf[c][size_t(by) * f.bw + bx];
      if (t == 0) {
        RegIdct<8>::run(v);
#pragma unroll
        for (int i = 0; i < 8; ++i) tile[r * 9 + i] = v[i];
        __syncwarp(gmask);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = tile[i * 9 + r];
        RegIdct<8>::run(v);
        __syncwarp(gmask);
#pragma unroll
        for (int i = 0; i < 8; ++i) tile[i * 9 + r] = v[i];
        __syncwarp(gmask);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = tile[r * 9 + i];
      } else {
        float* g = s_special[group];
#pragma unroll
        for (int i = 0; i < 8; ++i) g[r * 8 + i] = v[i];
        __syncwarp(gmask);
        transform_special_coop(g, t, g + 64, int(r), gmask);
#pragma unroll
        for (int i = 0; i < 8; ++i) v[i] = g[r * 8 + i];
      }
      __syncwarp(gmask);
      *reinterpret_cast<float4*>(row) = make_float4(v[0], v[1], v[2], v[3]);
      *reinterpret_cast<float4*>(row + 4) = make_float4(v[4], v[5], v[6], v[7]);
    }
  }
  }
}

// not inlined: the row pass and the column pass of the medium kernel share one copy of each size's code
template <int N>
__device__ __noinline__ void idct_line_smem(float* p, int stride) {
  float v[N];
#pragma unroll
  for (int i = 0; i < N; ++i) v[i] = p[i * stride];
  RegIdct<N>::run(v);
#pragma unroll
  for (int i = 0; i < N; ++i) p[i * stride] = v[i];
}

__device__ __forceinline__ void idct_line_dispatch(float* p, int stride, int n) {
  if (n == 8) idct_line_smem<8>(p, stride);
  else if (n == 16) idct_line_smem<16>(p, stride);
  else idct_line_smem<32>(p, stride);
}

constexpr int kMediumWarps = 4;
// One varblock of a warp's 32 x 32 tile (idct_medium_kernel).
struct MediumSub {
  uint32_t bx[3], by[3];  // where channel c keeps the block (8x8 cells); by == 0xffffffff: the channel skips it
};
// Varblocks of 16x8 ... 32x32 samples of frames whose coefficients are already dequantised, one warp per 32 x 32 TILE of
// them: a tile holds (32 / w) x (32 / h) blocks of the shape being walked (8 of 16x8, 4 of 16x16, 1 of 32x32), so the row
// pass (lane = tile row) and the column pass (lane = tile column) keep all 32 lanes busy whatever the shape; with one
// block per warp a 16x8 block used 8 and 16 lanes of 32. Per block nothing changes: same loads, same operation order in
// the line transforms. `dq` is unused: the launch passes the same arguments to every transform kernel.
__global__ void __launch_bounds__(kMediumWarps * 32) idct_medium_kernel(DevFrame f, DevDequantParams dq, TransformLists lists) {
  __shared__ float s_tile[kMediumWarps][32 * 33];
  __shared__ float s_llf[kMediumWarps][8][16];
  __shared__ MediumSub s_sub[kMediumWarps][8];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* tile = s_tile[warp];
  MediumSub* sub = s_sub[warp];
#pragma unroll 1
  for (int shape = 0; shape < kMediumShapes; ++shape) {
    const uint32_t* __restrict__ items = lists.shape_items[shape];
    const uint32_t total = lists.counts[4 + shape];
    if (total == 0) continue;
    // every entry of a shape's list has the same transform type
    const uint32_t item0 = items[0];
    const int32_t t = f.blk_type[size_t(item0 >> 16) * f.bw + (item0 & 0xffff)];
    const int bw = kDevTransformInfo[t][0], bh = kDevTransformInfo[t][1];
    const int w = bw * 8, h = bh * 8;
    const int logw = 31 - __clz(w), logh = 31 - __clz(h);
    const int lognx = 5 - logw, logny = 5 - logh, logp = lognx + logny;  // blocks across, down, per tile
    const int ny = 1 << logny;
    // this lane's tile column: block column sx, sample column x inside the block
    const int sx = int(lane) >> logw, x = int(lane) & (w - 1);
#pragma unroll 1
    for (uint32_t group = blockIdx.x * kMediumWarps + warp; (group << logp) < total; group += gridDim.x * kMediumWarps) {
      const uint32_t first = group << logp;
      const int nb = int(min(uint32_t(1) << logp, total - first));
      __syncwarp();
      if (int(lane) < nb) {  // lane s describes block s of the tile
        MediumSub m;
        const uint32_t item = items[first + lane];
        const uint32_t sbx = item & 0xffff, sby = item >> 16;
#pragma unroll
        for (uint32_t c = 0; c < 3; ++c) {
          uint32_t bx, by;
          const bool has = channel_block(f, c, sbx, sby, bx, by);
          m.bx[c] = bx;
          m.by[c] = has ? by : 0xffffffffu;
        }
        sub[lane] = m;
      }
      __syncwarp();
#pragma unroll 1
      for (int ci = 0; ci < 3; ++ci) {
        const uint32_t c = uint32_t(ci);
        // the (up to 4) blocks of this lane's tile column
        float* col[4];
#pragma unroll
        for (int sy = 0; sy < 4; ++sy) {
          const int s = (sy << lognx) + sx;
          col[sy] = nullptr;
          if (sy < ny && s < nb && sub[s].by[c] != 0xffffffffu)
            col[sy] = reinterpret_cast<float*>(f.coeff[c]) + size_t(sub[s].by[c]) * 8 * f.cw + size_t(sub[s].bx[c]) * 8 + x;
        }
        // 32 tile rows, kMediumTrip per trip, all loads of a trip issued before the first use
#pragma unroll 1
        for (int y0 = 0; y0 < 32; y0 += kMediumTrip) {
          float raw[kMediumTrip];
#pragma unroll
          for (int j = 0; j < kMediumTrip; ++j) {
            const int Y = y0 + j, sy = Y >> logh, y = Y & (h - 1);
            const float* src = sy == 0 ? col[0] : (sy == 1 ? col[1] : (sy == 2 ? col[2] : col[3]));
            raw[j] = src ? src[size_t(y) * f.cw] : 0.0f;
          }
#pragma unroll
          for (int j = 0; j < kMediumTrip; ++j) tile[(y0 + j) * 33 + int(lane)] = raw[j];
        }
        // lowest frequencies from the LF image: lane s for block s, then 16 lanes place the (at most) 16 values of the tile
        if (int(lane) < nb && sub[lane].by[c] != 0xffffffffu) compute_llf_small(f, int(c), sub[lane].bx[c], sub[lane].by[c], bw, bh, s_llf[warp][lane]);
        __syncwarp();
        if (lane < 16) {
          const int cells_log = (logw - 3) + (logh - 3);  // LLF values per block
          const int s = int(lane) >> cells_log, local = int(lane) & ((1 << cells_log) - 1);
          if (s < nb && sub[s].by[c] != 0xffffffffu) {
            const int ly = local >> (logw - 3), lx = local & (bw - 1);
            tile[(((s >> lognx) << logh) + ly) * 33 + ((s & ((1 << lognx) - 1)) << logw) + lx] = s_llf[warp][s][local];
          }
        }
        __syncwarp();
        {  // rows: lane = tile row, the row's blocks one after the other
          const int sy = int(lane) >> logh;
          for (int bxi = 0; bxi < (1 << lognx); ++bxi)
            if ((sy << lognx) + bxi < nb) idct_line_dispatch(tile + lane * 33 + (bxi << logw), 1, w);
        }
        __syncwarp();
        for (int sy = 0; sy < ny; ++sy)  // columns: lane = tile column
          if ((sy << lognx) + sx < nb) idct_line_dispatch(tile + (sy << logh) * 33 + lane, 33, h);
        __syncwarp();
#pragma unroll 1
        for (int y0 = 0; y0 < 32; y0 += 4) {
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int Y = y0 + j, sy = Y >> logh, y = Y & (h - 1);
            float* dst = sy == 0 ? col[0] : (sy == 1 ? col[1] : (sy == 2 ? col[2] : col[3]));
            if (dst) dst[size_t(y) * f.cw] = tile[Y * 33 + int(lane)];
          }
        }
        __syncwarp();
      }
    }
  }
}

// ---- medium varblocks, dequantising form, one instantiation per shape --------------------------------------------------
// Same tiling as idct_medium_kernel (one warp per 32 x 32 tile of equally shaped blocks, lane = tile column in the load /
// column / store passes, lane = tile row in the row pass) and the same per-sample operations in the same order, but the
// shape is a template parameter: block-row / row loops are static, so the per-sample pointer selection, shifts and table
// look-ups of the generic body (which spent several times more instructions on indexing than on arithmetic) fold into
// immediates. The shapes are walked one after the other by all CTAs in step, so one instantiation's code is hot at a time,
// and the line transforms are the shared idct_line_smem<N>.
// medium_walk unrolls the block rows and 8-row batches of a tile: as loops they take less than half the instructions, but
// were measured slower.
constexpr int kMediumOuterUnroll = 32;
struct MediumBlk {
  uint32_t bx, by;     // block position in 8x8 cells (dequantising frames are never subsampled: the same for all channels)
  float mul[3];        // DeqBlock::mul
  float kx[4], kb[4];  // chroma-from-luma factors of the 2 x 2 64x64 tiles at (tx0, ty0)
  int xsplit, ysplit;  // first sample column / row of the block that lies in the right / lower 64x64 tile (>= w / h: none)
};

template <int LOGW, int LOGH>
__device__ __forceinline__ void medium_walk(const DevFrame& f, const DevDequantParams& dq, const uint32_t* __restrict__ items,
                                            uint32_t total, float* tile, float* ytile, float (*llf)[16], MediumBlk* sub,
                                            uint32_t first_group, uint32_t group_stride, uint32_t lane) {
  constexpr int W = 1 << LOGW, H = 1 << LOGH, NX = 32 / W, NY = 32 / H, LOGP = (5 - LOGW) + (5 - LOGH), NB = 1 << LOGP;
  constexpr int BW = W / 8, BH = H / 8;
  const uint32_t item0 = items[0];
  const int32_t t = f.blk_type[size_t(item0 >> 16) * f.bw + (item0 & 0xffff)];  // one transform type per shape list
  const uint32_t set = kDevTransformInfo[t][2], tr = kDevTransformInfo[t][4];
  const int sx = int(lane) >> LOGW, x = int(lane) & (W - 1);
#pragma unroll 1
  for (uint32_t group = first_group; (group << LOGP) < total; group += group_stride) {
    const uint32_t first = group << LOGP;
    const int nb = int(min(uint32_t(NB), total - first));
    __syncwarp();
    if (int(lane) < nb) {  // lane s describes block s of the tile
      MediumBlk m;
      const uint32_t item = items[first + lane];
      m.bx = item & 0xffff, m.by = item >> 16;
      const DeqBlock db = deq_block(f, dq, t, m.bx, m.by);
      const uint32_t tx0 = (m.bx * 8) >> 6, ty0 = (m.by * 8) >> 6;
#pragma unroll
      for (int c = 0; c < 3; ++c) m.mul[c] = db.mul[c];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const uint32_t tx = min(tx0 + uint32_t(i & 1), f.w64 - 1), ty = min(ty0 + uint32_t(i >> 1), (f.ch + 63) / 64 - 1);
        cfl_factors(f, dq, tx << 6, ty << 6, m.kx[i], m.kb[i]);
      }
      m.xsplit = int((tx0 + 1) * 64 - m.bx * 8);
      m.ysplit = int((ty0 + 1) * 64 - m.by * 8);
      sub[lane] = m;
    }
    __syncwarp();
#pragma unroll 1
    for (int ci = 0; ci < 3; ++ci) {
      const uint32_t c = ci == 0 ? 1u : (ci == 1 ? 0u : 2u);  // Y first: its dequantised samples feed the chroma channels
      // (requesting the chroma rows into L2 while Y is transformed was measured slower, with more DRAM reads: the tile's three
      // channels already overlap across the SM's warps)
      const float* __restrict__ matc = dq.matrices + dq.matrix_offset[(set * 3 + c) * 2 + tr] + x;
      const float qb = dq.quant_bias[c], qbn = dq.quant_bias_numerator;
      float* const plane = reinterpret_cast<float*>(f.coeff[c]);
#pragma unroll kMediumOuterUnroll
      for (int sy = 0; sy < NY; ++sy) {
        const int s = sy * NX + sx;
        const bool have = s < nb;
        const MediumBlk& m = sub[have ? s : 0];
        const float* src = plane + size_t(m.by) * 8 * f.cw + size_t(m.bx) * 8 + x;
        const float mulc = m.mul[c];
        const int xt = x >= m.xsplit ? 1 : 0;
        const float k_top = c == 0 ? m.kx[xt] : m.kb[xt], k_bottom = c == 0 ? m.kx[xt + 2] : m.kb[xt + 2];
        const int ysplit = m.ysplit;
#pragma unroll kMediumOuterUnroll
        for (int y0 = 0; y0 < H; y0 += 8) {
          float raw[8], mt[8];
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            raw[j] = have ? src[size_t(y0 + j) * f.cw] : 0.0f;
            mt[j] = __ldg(matc + (y0 + j) * W);
          }
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            const int y = y0 + j, Y = sy * H + y;
            const float q = deq_one(__float_as_uint(raw[j]), mt[j], mulc, qb, qbn);
            float v = q;
            if (c == 1) ytile[Y * 33 + int(lane)] = q;
            else v = __fadd_rn(q, __fmul_rn(y >= ysplit ? k_bottom : k_top, ytile[Y * 33 + int(lane)]));
            tile[Y * 33 + int(lane)] = v;
          }
        }
      }
      // lowest frequencies from the LF image: lane s for block s, then 16 lanes place the (at most) 16 values of the tile
      if (int(lane) < nb) compute_llf_small(f, int(c), sub[lane].bx, sub[lane].by, BW, BH, llf[lane]);
      __syncwarp();
      if (lane < 16) {
        constexpr int cells_log = (LOGW - 3) + (LOGH - 3);  // LLF values per block
        const int s = int(lane) >> cells_log, local = int(lane) & ((1 << cells_log) - 1);
        if (s < nb) {
          const int ly = local >> (LOGW - 3), lx = local & (BW - 1);
          tile[(((s >> (5 - LOGW)) << LOGH) + ly) * 33 + ((s & (NX - 1)) << LOGW) + lx] = llf[s][local];
        }
      }
      __syncwarp();
      {  // rows: lane = tile row, the row's blocks one after the other
        const int sy = int(lane) >> LOGH;
#pragma unroll
        for (int bxi = 0; bxi < NX; ++bxi)
          if (sy * NX + bxi < nb) idct_line_smem<W>(tile + lane * 33 + bxi * W, 1);
      }
      __syncwarp();
#pragma unroll
      for (int sy = 0; sy < NY; ++sy)  // columns: lane = tile column
        if (sy * NX + sx < nb) idct_line_smem<H>(tile + sy * H * 33 + lane, 33);
      __syncwarp();
#pragma unroll kMediumOuterUnroll
      for (int sy = 0; sy < NY; ++sy) {
        const int s = sy * NX + sx;
        if (s < nb) {
          const MediumBlk& m = sub[s];
          float* dst = plane + size_t(m.by) * 8 * f.cw + size_t(m.bx) * 8 + x;
#pragma unroll 8
          for (int y = 0; y < H; ++y) dst[size_t(y) * f.cw] = tile[(sy * H + y) * 33 + int(lane)];
        }
      }
      __syncwarp();
    }
  }
}

constexpr int kMediumMinBlocks = 5;  // the fastest of 4 / 5 / 6 when measured; not re-measured on the H100
__global__ void __launch_bounds__(kMediumWarps * 32, kMediumMinBlocks) idct_medium_deq_kernel(DevFrame f, DevDequantParams dq, TransformLists lists) {
  __shared__ float s_tile[kMediumWarps][32 * 33];
  __shared__ float s_ytile[kMediumWarps][32 * 33];  // dequantised Y coefficients (chroma from luma)
  __shared__ float s_llf[kMediumWarps][8][16];
  __shared__ MediumBlk s_sub[kMediumWarps][8];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t g0 = blockIdx.x * kMediumWarps + warp, gs = gridDim.x * kMediumWarps;
#pragma unroll 1
  for (int shape = 0; shape < kMediumShapes; ++shape) {
    const uint32_t* __restrict__ items = lists.shape_items[shape];
    const uint32_t total = lists.counts[4 + shape];
    if (total == 0) continue;
    float* tile = s_tile[warp];
    float* yt = s_ytile[warp];
    switch (shape) {  // medium_shape(): 0: 16x8, 1: 8x16, 2: 16x16, 3: 32x8, 4: 8x32, 5: 32x16, 6: 16x32, 7: 32x32 (w x h samples)
      case 0: medium_walk<4, 3>(f, dq, items, total, tile, yt, s_llf[warp], s_sub[warp], g0, gs, lane); break;
      case 1: medium_walk<3, 4>(f, dq, items, total, tile, yt, s_llf[warp], s_sub[warp], g0, gs, lane); break;
      case 2: medium_walk<4, 4>(f, dq, items, total, tile, yt, s_llf[warp], s_sub[warp], g0, gs, lane); break;
      case 3: medium_walk<5, 3>(f, dq, items, total, tile, yt, s_llf[warp], s_sub[warp], g0, gs, lane); break;
      case 4: medium_walk<3, 5>(f, dq, items, total, tile, yt, s_llf[warp], s_sub[warp], g0, gs, lane); break;
      case 5: medium_walk<5, 4>(f, dq, items, total, tile, yt, s_llf[warp], s_sub[warp], g0, gs, lane); break;
      case 6: medium_walk<4, 5>(f, dq, items, total, tile, yt, s_llf[warp], s_sub[warp], g0, gs, lane); break;
      default: medium_walk<5, 5>(f, dq, items, total, tile, yt, s_llf[warp], s_sub[warp], g0, gs, lane); break;
    }
  }
}

// dct_2d (general path: both dimensions >= 4) by a CTA; every thread owns 2*nmax floats of `lines`.
__device__ void dct_2d_coop(float* p, size_t stride, int width, int height, bool forward, float* lines, int nmax) {
  float* line = lines + size_t(threadIdx.x) * (2 * nmax + 1);  // odd stride: conflict-free banks
  float* scratch = line + nmax;
  for (int y = int(threadIdx.x); y < height; y += int(blockDim.x)) {
    float* row = p + size_t(y) * stride;
    for (int x = 0; x < width; ++x) line[x] = row[x];
    dct1d(line, scratch, width, forward);
    for (int x = 0; x < width; ++x) row[x] = line[x];
  }
  __syncthreads();
  for (int x = int(threadIdx.x); x < width; x += int(blockDim.x)) {
    float* col = p + x;
    for (int y = 0; y < height; ++y) line[y] = col[size_t(y) * stride];
    dct1d(line, scratch, height, forward);
    for (int y = 0; y < height; ++y) col[size_t(y) * stride] = line[y];
  }
  __syncthreads();
}

constexpr int kLargeThreads = 64;
template <bool DEQ>
__global__ void __launch_bounds__(kLargeThreads) idct_large_kernel(DevFrame f, DevDequantParams dq,
                                                                   const uint32_t* __restrict__ items,
                                                                   const uint32_t* __restrict__ count_ptr, int nmax) {
  extern __shared__ float s_large[];  // llf (32 x 32) | per-thread line buffers (2 * nmax each)
  float* llf = s_large;
  float* lines = s_large + 1024;
  const uint32_t total = DEQ ? *count_ptr : *count_ptr * 3;
  for (uint32_t work = blockIdx.x; work < total; work += gridDim.x) {
    const uint32_t item = items[DEQ ? work : work / 3];
    const uint32_t sbx = item & 0xffff, sby = item >> 16;
    const int32_t t = f.blk_type[size_t(sby) * f.bw + sbx];
    const int bw = kDevTransformInfo[t][0], bh = kDevTransformInfo[t][1];
    const int w = bw * 8, h = bh * 8;
    if (DEQ) {  // dequantise the three channels in place (L2-resident block), then transform them one by one
      const DeqBlock db = deq_block(f, dq, t, sbx, sby);
      const int logw = 31 - __clz(w);
      __shared__ float s_k[2][25];  // chroma-from-luma factors of the up to 5 x 5 64x64 tiles the block touches
      const uint32_t tx0 = (sbx * 8) >> 6, ty0 = (sby * 8) >> 6;
      if (threadIdx.x < 25) {
        const uint32_t tx = min(tx0 + threadIdx.x % 5, f.w64 - 1), ty = min(ty0 + threadIdx.x / 5, (f.ch + 63) / 64 - 1);
        cfl_factors(f, dq, tx << 6, ty << 6, s_k[0][threadIdx.x], s_k[1][threadIdx.x]);
      }
      __syncthreads();
      // w * h >= 4096: four elements per thread and trip, their twelve coefficient loads in flight together
      for (int idx0 = int(threadIdx.x); idx0 < w * h; idx0 += 4 * kLargeThreads) {
        uint32_t raw[4][3];
        float mat[4][3];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int idx = idx0 + j * kLargeThreads, x = idx & (w - 1), y = idx >> logw;
          const size_t gi = (size_t(sby) * 8 + y) * f.cw + size_t(sbx) * 8 + x;
#pragma unroll
          for (int c = 0; c < 3; ++c) {
            raw[j][c] = f.coeff[c][gi];
            mat[j][c] = __ldg(db.mat[c] + idx);
          }
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int idx = idx0 + j * kLargeThreads, x = idx & (w - 1), y = idx >> logw;
          const size_t gi = (size_t(sby) * 8 + y) * f.cw + size_t(sbx) * 8 + x;
          float v[3];
#pragma unroll
          for (int c = 0; c < 3; ++c) v[c] = deq_one(raw[j][c], mat[j][c], db.mul[c], dq.quant_bias[c], dq.quant_bias_numerator);
          const int ti = int(((sbx * 8 + uint32_t(x)) >> 6) - tx0) + 5 * int(((sby * 8 + uint32_t(y)) >> 6) - ty0);
          const float kx = s_k[0][ti], kb = s_k[1][ti];
          v[0] = __fadd_rn(v[0], __fmul_rn(kx, v[1]));
          v[2] = __fadd_rn(v[2], __fmul_rn(kb, v[1]));
#pragma unroll
          for (int c = 0; c < 3; ++c) f.coeff[c][gi] = __float_as_uint(v[c]);
        }
      }
      __syncthreads();
    }
#pragma unroll 1
    for (int ci = 0; ci < (DEQ ? 3 : 1); ++ci) {
      const uint32_t c = DEQ ? uint32_t(ci) : work % 3;
      uint32_t bx, by;
      if (!channel_block(f, c, sbx, sby, bx, by)) continue;
      float* block = reinterpret_cast<float*>(f.coeff[c]) + size_t(by) * 8 * f.cw + size_t(bx) * 8;
      const float* lf = f.lf[c];
      for (int i = int(threadIdx.x); i < bw * bh; i += kLargeThreads)
        llf[i] = lf[size_t(by + i / bw) * f.bw + bx + i % bw];
      __syncthreads();
      dct_2d_coop(llf, size_t(bw), bw, bh, true, lines, nmax);
      const int logbw = 31 - __clz(bw), logbh = 31 - __clz(bh);
      for (int i = int(threadIdx.x); i < bw * bh; i += kLargeThreads) {
        const int x = i % bw, y = i / bw;
        block[size_t(y) * f.cw + x] = __fdiv_rn(llf[i], __fmul_rn(kScaleF[y << (5 - logbh)], kScaleF[x << (5 - logbw)]));
      }
      __syncthreads();
      dct_2d_coop(block, f.cw, w, h, false, lines, nmax);
    }
  }
}


// ---- 64-sample varblocks (64x64, 64x32, 32x64), dequantising form: the block is staged in shared memory ---------------------
// idct_large_kernel dequantises the three channels in place in global memory and then lets every thread walk a row, later a
// column, of the block in global memory (one 4-byte request per sample, a warp's requests 64 rows apart). Here a CTA
// keeps one channel of the block in a 64 x 65 shared tile: coefficients arrive with coalesced loads and are dequantised
// on the way in (the dequantised Y copy stays in a second tile for chroma from luma), rows are transformed in place,
// columns likewise (l64_idct_pass), and the samples leave with coalesced stores - one read and one write
// of HBM per sample. Per sample the operations and their order are those of idct_large_kernel.
// One 1-D inverse-DCT pass over the lines of the shared tile by 128 threads. A 64-point line is split between two threads
// the way Dct1D<64>::run(inverse) splits it (generic/dct.rs:239-293): even-indexed and odd-indexed samples go through
// independent 32-point transforms (register-resident RegIdct<32>, the same operation sequence as Dct1D<32>), the
// odd half after its neighbour additions and the sqrt(2), and is scaled by sec before the final butterfly. Thread
// (line, half) = (tid & 63, tid >> 6): a warp works on 32 lines of the same half, so its shared accesses hit 32 banks.
__device__ __forceinline__ void l64_idct_pass(float* tile, int nlines, int len, int line_stride, int elem_stride, int tid) {
  const int line = tid & 63, half = tid >> 6;
  const bool act = line < nlines;
  float* p = tile + line * line_stride;
  float v[32];
  if (len == 64) {
    if (act) {
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = p[(2 * i + half) * elem_stride];
      if (half) {
#pragma unroll
        for (int i = 31; i >= 1; --i) v[i] = __fadd_rn(v[i], v[i - 1]);  // in1[j] += in1[j - 1], highest j first
        v[0] = __fmul_rn(v[0], SQRT2F);
      }
      RegIdct<32>::run(v);
      if (half) {
#pragma unroll
        for (int i = 0; i < 32; ++i) v[i] = __fmul_rn(v[i], kSecLarge[i]);
      }
    }
    __syncthreads();  // every sample of the tile has been read
    if (act) {
#pragma unroll
      for (int i = 0; i < 32; ++i) p[(half * 32 + i) * elem_stride] = v[i];
    }
    __syncthreads();
    float o[32];
    if (act) {
#pragma unroll
      for (int i = 0; i < 32; ++i) o[i] = p[((1 - half) * 32 + i) * elem_stride];  // the other half's results
    }
    __syncthreads();
    if (act) {
      if (!half) {
#pragma unroll
        for (int i = 0; i < 32; ++i) p[i * elem_stride] = __fadd_rn(v[i], o[i]);
      } else {
#pragma unroll
        for (int i = 0; i < 32; ++i) p[(63 - i) * elem_stride] = __fsub_rn(o[i], v[i]);
      }
    }
  } else {  // 32-point lines: one thread each
    if (act && half == 0) {
#pragma unroll
      for (int i = 0; i < 32; ++i) v[i] = p[i * elem_stride];
      RegIdct<32>::run(v);
#pragma unroll
      for (int i = 0; i < 32; ++i) p[i * elem_stride] = v[i];
    }
  }
  __syncthreads();
}

constexpr int kL64Threads = 128, kL64Pitch = 65, kL64Line = 2 * 8 + 1;  // line buffers: the forward DCT of the <= 8 x 8 LF samples only
constexpr int kL64SmemFloats = 2 * 64 * kL64Pitch + 64 + 8 * kL64Line;
__global__ void __launch_bounds__(kL64Threads, 3) idct_large64_deq_kernel(DevFrame f, DevDequantParams dq, const uint32_t* __restrict__ items,
                                                                       const uint32_t* __restrict__ count_ptr) {
  extern __shared__ float s_l64[];
  float* tile = s_l64;                      // the channel being transformed
  float* ytile = tile + 64 * kL64Pitch;     // dequantised Y
  float* llf = ytile + 64 * kL64Pitch;      // <= 8 x 8 LF samples
  float* lines = llf + 64;                  // 8 per-thread line + scratch buffers for the LF samples' forward DCT
  __shared__ float s_k[2][25];
  const int tid = int(threadIdx.x);
  const uint32_t total = *count_ptr;
  for (uint32_t work = blockIdx.x; work < total; work += gridDim.x) {
    const uint32_t item = items[work];
    const uint32_t sbx = item & 0xffff, sby = item >> 16;
    const int32_t t = f.blk_type[size_t(sby) * f.bw + sbx];
    const int bw = kDevTransformInfo[t][0], bh = kDevTransformInfo[t][1];
    const int w = bw * 8, h = bh * 8;
    const int logw = 31 - __clz(w);
    const DeqBlock db = deq_block(f, dq, t, sbx, sby);
    const uint32_t tx0 = (sbx * 8) >> 6, ty0 = (sby * 8) >> 6;
    if (tid < 25) {
      const uint32_t tx = min(tx0 + uint32_t(tid) % 5, f.w64 - 1), ty = min(ty0 + uint32_t(tid) / 5, (f.ch + 63) / 64 - 1);
      cfl_factors(f, dq, tx << 6, ty << 6, s_k[0][tid], s_k[1][tid]);
    }
    __syncthreads();
#pragma unroll 1
    for (int ci = 0; ci < 3; ++ci) {
      const uint32_t c = ci == 0 ? 1u : (ci == 1 ? 0u : 2u);
      float* const block = reinterpret_cast<float*>(f.coeff[c]) + size_t(sby) * 8 * f.cw + size_t(sbx) * 8;
      const float* __restrict__ matc = db.mat[c];
      const float mulc = db.mul[c], qb = dq.quant_bias[c], qbn = dq.quant_bias_numerator;
      // w * h >= 2048: eight samples per thread and trip, their loads in flight together
      for (int idx0 = tid; idx0 < w * h; idx0 += 8 * kL64Threads) {
        float raw[8], mt[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int idx = idx0 + j * kL64Threads, x = idx & (w - 1), y = idx >> logw;
          raw[j] = block[size_t(y) * f.cw + x];
          mt[j] = __ldg(matc + idx);
        }
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int idx = idx0 + j * kL64Threads, x = idx & (w - 1), y = idx >> logw;
          const float q = deq_one(__float_as_uint(raw[j]), mt[j], mulc, qb, qbn);
          float v = q;
          if (c == 1) {
            ytile[y * kL64Pitch + x] = q;
          } else {
            const int ti = int(((sbx * 8 + uint32_t(x)) >> 6) - tx0) + 5 * int(((sby * 8 + uint32_t(y)) >> 6) - ty0);
            v = __fadd_rn(q, __fmul_rn(s_k[c == 0 ? 0 : 1][ti], ytile[y * kL64Pitch + x]));
          }
          tile[y * kL64Pitch + x] = v;
        }
      }
      // lowest frequencies: forward DCT of the block's LF samples, rescaled (transform_common.rs:33-58)
      const float* lf = f.lf[c];
      for (int i = tid; i < bw * bh; i += kL64Threads) llf[i] = lf[size_t(sby + i / bw) * f.bw + sbx + i % bw];
      __syncthreads();
      {
        float* line = lines + size_t(tid) * kL64Line;
        if (tid < bh) {
          float* row = llf + tid * bw;
          for (int x = 0; x < bw; ++x) line[x] = row[x];
          dct1d(line, line + 8, bw, true);
          for (int x = 0; x < bw; ++x) row[x] = line[x];
        }
        __syncthreads();
        if (tid < bw) {
          for (int y = 0; y < bh; ++y) line[y] = llf[y * bw + tid];
          dct1d(line, line + 8, bh, true);
          for (int y = 0; y < bh; ++y) llf[y * bw + tid] = line[y];
        }
        __syncthreads();
      }
      const int logbw = 31 - __clz(bw), logbh = 31 - __clz(bh);
      for (int i = tid; i < bw * bh; i += kL64Threads) {
        const int x = i % bw, y = i / bw;
        tile[y * kL64Pitch + x] = __fdiv_rn(llf[i], __fmul_rn(kScaleF[y << (5 - logbh)], kScaleF[x << (5 - logbw)]));
      }
      __syncthreads();
      // inverse DCT: rows, then columns (generic/dct.rs:93-140)
      l64_idct_pass(tile, h, w, kL64Pitch, 1, tid);
      l64_idct_pass(tile, w, h, 1, kL64Pitch, tid);
      for (int idx = tid; idx < w * h; idx += kL64Threads) {
        const int x = idx & (w - 1), y = idx >> logw;
        block[size_t(y) * f.cw + x] = tile[y * kL64Pitch + x];
      }
      __syncthreads();
    }
  }
}

}  // namespace

void launch_lf_dequant(DevFrame f, const DevLfDequantJob* jobs, int num_jobs, cudaStream_t stream) {
  if (num_jobs <= 0) return;
  dim3 grid(2, 256, num_jobs);  // LF groups are at most 256 x 256 blocks
  lf_dequant_kernel<<<grid, 128, 0, stream>>>(f, jobs);
}

void launch_lf_cfl(DevFrame f, float kx, float kb, cudaStream_t stream) {
  size_t n = size_t(f.bw) * f.bh;
  lf_cfl_kernel<<<unsigned((n + 255) / 256), 256, 0, stream>>>(f, kx, kb);
}

void launch_lf_smooth(DevFrame f, float* tmp[3], float lf_x, float lf_y, float lf_b, cudaStream_t stream) {
  dim3 grid((f.bw + 127) / 128, f.bh);
  lf_smooth_kernel<<<grid, 128, 0, stream>>>(f, tmp[0], tmp[1], tmp[2], lf_x, lf_y, lf_b);
}

void launch_hf_dequant_cfl(DevFrame f, DevDequantParams p, cudaStream_t stream) {
  dim3 block(64, 4);
  dim3 grid((f.cw + 63) / 64, (f.ch + 3) / 4);
  if (f.subsampled) {
    for (int c = 0; c < 3; ++c) hf_dequant_channel_kernel<<<grid, block, 0, stream>>>(f, p, c);
    return;
  }
  hf_dequant_cfl_kernel<<<grid, block, 0, stream>>>(f, p);
}

size_t hf_transform_scratch_bytes(uint32_t bw, uint32_t bh) {
  const size_t cells = size_t(bw) * bh;
  // counters | small | (former medium list) | large | huge | the eight medium shapes (cells/2 x 2, /4 x 3, /8 x 2, /16)
  // ... | the ten small types (cells each)
  return 256 + (cells + cells / 2 + 2 * (cells / 32 + 1) + 64) * 4 + (cells * 9 / 4 + 64) * 4 + size_t(kSmallTypes) * (cells + 1) * 4;
}

namespace {
template <bool DEQ>
void launch_idcts(DevFrame f, const DevDequantParams& dq, const TransformLists& L, size_t cells, int num_sms, cudaStream_t stream) {
  const size_t per = DEQ ? 1 : 3;  // work items per varblock
  const int small_grid = int(std::min<size_t>((cells * per + kSmallGroups - 1) / kSmallGroups, size_t(num_sms) * 8));
  idct_small_kernel<DEQ><<<small_grid, kSmallGroups * 8, 0, stream>>>(f, dq, L);
  const int medium_grid = int(std::min<size_t>((cells / 2 * per + kMediumWarps) / kMediumWarps, size_t(num_sms) * 8));
  if (DEQ) idct_medium_deq_kernel<<<medium_grid, kMediumWarps * 32, 0, stream>>>(f, dq, L);
  else idct_medium_kernel<<<medium_grid, kMediumWarps * 32, 0, stream>>>(f, dq, L);
  const int large_grid = int(std::min<size_t>((cells / 32 + 1) * per, size_t(num_sms) * 4));
  if (DEQ) idct_large64_deq_kernel<<<large_grid, kL64Threads, kL64SmemFloats * 4, stream>>>(f, dq, L.items[2], L.counts + 2);
  else idct_large_kernel<DEQ><<<large_grid, kLargeThreads, (1024 + kLargeThreads * (2 * 64 + 1)) * 4, stream>>>(f, dq, L.items[2], L.counts + 2, 64);
  const int huge_grid = int(std::min<size_t>((cells / 128 + 1) * per, size_t(num_sms)));
  idct_large_kernel<DEQ><<<huge_grid, kLargeThreads, (1024 + kLargeThreads * (2 * 256 + 1)) * 4, stream>>>(f, dq, L.items[3], L.counts + 3, 256);
}
}  // namespace

// `dq` non-null: the coefficient planes still hold quantised integers; dequantisation and chroma from luma run in the
// transforms' load stage (one HBM round trip less than hf_dequant_cfl_kernel + transforms). Not for subsampled frames.
void launch_hf_transform(DevFrame f, void* scratch, const DevDequantParams* dq, cudaStream_t stream) {
  const size_t cells = size_t(f.bw) * f.bh;
  TransformLists L;
  L.counts = static_cast<uint32_t*>(scratch);
  uint32_t* base = L.counts + 64;
  L.items[0] = base;                                   // <= cells
  L.items[1] = L.items[0] + cells;                     // <= cells / 2
  L.items[2] = L.items[1] + cells / 2 + 1;             // <= cells / 32
  L.items[3] = L.items[2] + cells / 32 + 1;            // <= cells / 128
  {  // a shape's list holds at most cells / (cells per block of that shape) entries
    static const int kShapeCells[kMediumShapes] = {2, 2, 4, 4, 4, 8, 8, 16};
    uint32_t* q = L.items[3] + cells / 128 + 1;
    for (int sh = 0; sh < kMediumShapes; ++sh) {
      L.shape_items[sh] = q;
      q += cells / kShapeCells[sh] + 1;
    }
    for (int k = 0; k < kSmallTypes; ++k) {
      L.small_items[k] = q;
      q += cells + 1;
    }
  }
  cudaMemsetAsync(L.counts, 0, 128, stream);
  dim3 cb(32, 8), cg((f.bw + 31) / 32, (f.bh + 7) / 8);
  classify_varblocks_kernel<<<cg, cb, 0, stream>>>(f, L);
  // initialised once, thread-safely (function-local static): no worker thread launches before the limits are set
  static const int num_sms = [] {
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    cudaFuncSetAttribute(idct_large_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 140 * 1024);
    cudaFuncSetAttribute(idct_large_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 140 * 1024);
    cudaFuncSetAttribute(idct_large64_deq_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kL64SmemFloats * 4);
    return n;
  }();
  if (dq && !f.subsampled) {
    launch_idcts<true>(f, *dq, L, cells, num_sms, stream);
  } else {
    DevDequantParams none;
    memset(&none, 0, sizeof(none));
    launch_idcts<false>(f, none, L, cells, num_sms, stream);
  }
}

}  // namespace jxlb
