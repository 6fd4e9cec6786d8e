// Modular sub-codec on the device, the data-parallel part: inverse Squeeze, inverse RCT, simple
// palette, sample conversions (the entropy-coded channel decode lives in modular_stream.cu).
// Integer arithmetic is bit-exact with crates/jxl-modular/src/{image.rs,predictor.rs,
// transform/{squeeze,rct,palette}.rs} (i32 samples, wrapping).
#include "kernels.h"

#include <cstring>

namespace jxlb {

namespace {

__device__ __forceinline__ int32_t wadd(int32_t a, int32_t b) { return int32_t(uint32_t(a) + uint32_t(b)); }
__device__ __forceinline__ int32_t wsub(int32_t a, int32_t b) { return int32_t(uint32_t(a) - uint32_t(b)); }
__device__ __forceinline__ int32_t wmul(int32_t a, int32_t b) { return int32_t(uint32_t(a) * uint32_t(b)); }

__device__ __forceinline__ int32_t tendency(int32_t a, int32_t b, int32_t c) {  // squeeze.rs:1104-1137
  if (a >= b && b >= c) {
    int32_t x = wadd(wsub(wsub(wmul(4, a), wmul(3, c)), b), 6) / 12;
    if (wsub(x, x & 1) > wmul(2, wsub(a, b))) x = wadd(wmul(2, wsub(a, b)), 1);
    if (wadd(x, x & 1) > wmul(2, wsub(b, c))) x = wmul(2, wsub(b, c));
    return x;
  } else if (a <= b && b <= c) {
    int32_t x = wsub(wsub(wsub(wmul(4, a), wmul(3, c)), b), 6) / 12;
    if (wadd(x, x & 1) < wmul(2, wsub(a, b))) x = wsub(wmul(2, wsub(a, b)), 1);
    if (wsub(x, x & 1) < wmul(2, wsub(b, c))) x = wmul(2, wsub(b, c));
    return x;
  }
  return 0;
}

// Horizontal inverse Squeeze (squeeze.rs:59-120). The recurrence along a row is serial (`left = second`), rows are
// independent: one lane per row, a warp per band of 32 rows. A lane walking its own row straight in global memory
// would touch 32 different cache lines per warp access, so the band is processed in chunks of 32 pairs staged through
// shared memory: the warp loads the averages / residuals of the chunk row by row (128-byte coalesced reads), every
// lane then runs its row's recurrence on the shared tile (pitch 33 / 65: conflict-free), and the 64 output columns go
// back row by row as two coalesced 128-byte writes. `left` and the current average carry over between chunks in registers.
constexpr int kSqWarps = 2;
struct SqueezeBatch {  // up to four channels of one Squeeze step, blockIdx.y selects the channel
  DevView avg[4], res[4], out[4];
};
__global__ void __launch_bounds__(kSqWarps * 32) squeeze_h_kernel(SqueezeBatch b) {
  const DevView avg = b.avg[blockIdx.y], res = b.res[blockIdx.y], out = b.out[blockIdx.y];
  if (!out.w || !out.h) return;
  __shared__ int32_t s_avg[kSqWarps][32][33], s_res[kSqWarps][32][33], s_out[kSqWarps][32][65];
  const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t y0 = (blockIdx.x * kSqWarps + warp) * 32;
  if (y0 >= out.h) return;
  const uint32_t rows = min(32u, out.h - y0);
  const int32_t* ab = static_cast<const int32_t*>(avg.ptr) + size_t(y0) * avg.stride;
  const int32_t* rb = static_cast<const int32_t*>(res.ptr) + size_t(y0) * res.stride;
  int32_t* ob = static_cast<int32_t*>(out.ptr) + size_t(y0) * out.stride;
  int32_t(*ta)[33] = s_avg[warp];
  int32_t(*tr)[33] = s_res[warp];
  int32_t(*to)[65] = s_out[warp];
  int32_t a = 0, left = 0;
  if (lane < rows) a = left = ab[size_t(lane) * avg.stride];
  for (uint32_t x0 = 0; x0 < res.w; x0 += 32) {
    const uint32_t n = min(32u, res.w - x0);  // pairs in this chunk
    for (uint32_t r = 0; r < rows; ++r) {
      // average x0 + 1 + lane (the "next average" of pair x0 + lane) and residual x0 + lane of row r
      const uint32_t ax = x0 + 1 + lane;
      ta[r][lane] = ax < avg.w ? ab[size_t(r) * avg.stride + ax] : 0;
      tr[r][lane] = lane < n ? rb[size_t(r) * res.stride + x0 + lane] : 0;
    }
    __syncwarp();
    if (lane < rows) {
      for (uint32_t k = 0; k < n; ++k) {
        const int32_t next_avg = (x0 + k + 1 < avg.w) ? ta[lane][k] : a;
        const int32_t diff = wadd(tr[lane][k], tendency(left, a, next_avg));
        const int32_t first = wadd(a, diff / 2);
        const int32_t second = wsub(first, diff);
        to[lane][2 * k] = first;
        to[lane][2 * k + 1] = second;
        a = next_avg;
        left = second;
      }
    }
    __syncwarp();
    for (uint32_t r = 0; r < rows; ++r) {
      int32_t* o = ob + size_t(r) * out.stride + 2 * x0;
      if (lane < 2 * n) o[lane] = to[r][lane];
      if (lane + 32 < 2 * n) o[lane + 32] = to[r][lane + 32];
    }
    __syncwarp();
  }
  if ((out.w & 1) && lane < rows) ob[size_t(lane) * out.stride + out.w - 1] = ab[size_t(lane) * avg.stride + avg.w - 1];
}

// Vertical inverse Squeeze (squeeze.rs:803-862): one thread per column (adjacent lanes read adjacent columns: every row
// access of a warp is one 128-byte line), the recurrence runs down the column. The loads of a step do not depend on the
// recurrence, so four rows of averages / residuals are fetched before the four dependent steps that use them: one
// global-memory latency per four output row pairs instead of per pair. blockIdx.y selects the channel of a batch.
__global__ void __launch_bounds__(64) squeeze_v_kernel(SqueezeBatch b) {
  const DevView avg = b.avg[blockIdx.y], res = b.res[blockIdx.y], out = b.out[blockIdx.y];
  uint32_t x = blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= out.w || !out.h) return;
  const int32_t* ap = static_cast<const int32_t*>(avg.ptr) + x;
  const int32_t* rp = static_cast<const int32_t*>(res.ptr) + x;
  int32_t* o = static_cast<int32_t*>(out.ptr) + x;
  int32_t a = ap[0], top = a;
  uint32_t y = 0;
  for (; y + 4 <= res.h; y += 4) {
    int32_t na[4], r[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      r[j] = rp[size_t(y + j) * res.stride];
      na[j] = (y + j + 1 < avg.h) ? ap[size_t(y + j + 1) * avg.stride] : 0;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int32_t next_avg = (y + j + 1 < avg.h) ? na[j] : a;
      const int32_t diff = wadd(r[j], tendency(top, a, next_avg));
      const int32_t first = wadd(a, diff / 2);
      const int32_t second = wsub(first, diff);
      o[size_t(2 * (y + j)) * out.stride] = first;
      o[size_t(2 * (y + j) + 1) * out.stride] = second;
      a = next_avg;
      top = second;
    }
  }
  for (; y < res.h; ++y) {
    int32_t next_avg = (y + 1 < avg.h) ? ap[size_t(y + 1) * avg.stride] : a;
    int32_t diff = wadd(rp[size_t(y) * res.stride], tendency(top, a, next_avg));
    int32_t first = wadd(a, diff / 2);
    int32_t second = wsub(first, diff);
    o[size_t(2 * y) * out.stride] = first;
    o[size_t(2 * y + 1) * out.stride] = second;
    a = next_avg;
    top = second;
  }
  if (out.h & 1) o[size_t(out.h - 1) * out.stride] = ap[size_t(avg.h - 1) * avg.stride];
}

__global__ void rct_kernel(DevView va, DevView vb, DevView vc, uint32_t rct_type) {  // rct.rs:154-256
  uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= va.w) return;
  int32_t* pa = static_cast<int32_t*>(va.ptr) + size_t(y) * va.stride + x;
  int32_t* pb = static_cast<int32_t*>(vb.ptr) + size_t(y) * vb.stride + x;
  int32_t* pc = static_cast<int32_t*>(vc.ptr) + size_t(y) * vc.stride + x;
  uint32_t permutation = rct_type / 7, ty = rct_type % 7;
  int32_t a = *pa, b = *pb, c = *pc, d, e, f;
  if (ty == 6) {
    int32_t tmp = wsub(a, c >> 1);
    e = wadd(c, tmp);
    f = wsub(tmp, b >> 1);
    d = wadd(f, b);
  } else {
    d = a;
    f = (ty & 1) ? wadd(c, a) : c;
    if ((ty >> 1) == 1) e = wadd(b, a);
    else if ((ty >> 1) == 2) e = wadd(b, wadd(a, f) >> 1);
    else e = b;
  }
  switch (permutation) {
    case 1: *pa = f, *pb = d, *pc = e; break;
    case 2: *pa = e, *pb = f, *pc = d; break;
    case 3: *pa = d, *pb = f, *pc = e; break;
    case 4: *pa = e, *pb = d, *pc = f; break;
    case 5: *pa = f, *pb = e, *pc = d; break;
    default: *pa = d, *pb = e, *pc = f; break;
  }
}

struct PaletteTargets {
  DevView v[kMaxPaletteChannels];
};
__constant__ int16_t kDeltaPalette[72][3] = {
#include "../host/delta_palette.inc"
};

// First pass of the inverse palette (palette.rs:26-118): explicit colours, the implicit colour cube for indices >=
// nb_colours, delta entries for negative indices. Samples whose index is < nb_deltas still need the prediction added
// (second pass, palette_delta_kernel): they are marked in `mask` and counted in `status`.
__global__ void palette_kernel(DevView pal, PaletteTargets t, int num_c, int nb_colours, int bit_depth, int nb_deltas,
                               uint8_t* mask, int* status) {
  uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= t.v[0].w) return;
  int32_t index = static_cast<int32_t*>(t.v[0].ptr)[size_t(y) * t.v[0].stride + x];
  const bool delta = index < nb_deltas;
  mask[size_t(y) * t.v[0].w + x] = delta ? 1 : 0;
  if (delta) atomicAdd(status, 1);
  for (int c = 0; c < num_c; ++c) {
    int32_t sample;
    if (index < 0) {
      if (c >= 3) {
        sample = 0;
      } else {
        const uint32_t ii = uint32_t((-(index + 1)) % 143);
        sample = kDeltaPalette[(ii + 1) >> 1][c];
        if ((ii & 1) == 0) sample = -sample;
        if (bit_depth > 8) sample <<= min(bit_depth, 24) - 8;
      }
    } else if (index < nb_colours) {
      sample = static_cast<const int32_t*>(pal.ptr)[size_t(c) * pal.stride + index];
    } else {
      int32_t idx = index - nb_colours;
      if (idx < 64) {
        sample = ((idx >> (2 * c)) % 4) * ((1 << bit_depth) - 1) / 4 + (1 << (bit_depth > 3 ? bit_depth - 3 : 0));
      } else {
        int32_t k = idx - 64;
        for (int q = 0; q < c; ++q) k /= 5;
        sample = (k % 5) * ((1 << bit_depth) - 1) / 4;
      }
    }
    static_cast<int32_t*>(t.v[c].ptr)[size_t(y) * t.v[c].stride + x] = sample;
  }
}

__global__ void int_to_float_kernel(DevView v, uint32_t bits, uint32_t exp_bits, int float_sample) {
  uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= v.w) return;
  uint32_t* p = static_cast<uint32_t*>(v.ptr) + size_t(y) * v.stride + x;
  int32_t s = int32_t(*p);
  float f;
  if (!float_sample) {
    int32_t div = int32_t((1u << bits) - 1);
    f = __fdiv_rn(float(s), float(div));
  } else {  // jxl-image/src/lib.rs:464-488
    uint32_t sample = uint32_t(s);
    uint32_t mantissa_bits = bits - exp_bits - 1;
    uint32_t mantissa_mask = (1u << mantissa_bits) - 1;
    uint32_t exp_mask = ((1u << (bits - 1)) - 1) ^ mantissa_mask;
    uint32_t sign = (sample >> (bits - 1)) & 1;
    uint32_t mantissa = sample & mantissa_mask;
    int32_t exp = int32_t((sample & exp_mask) >> mantissa_bits) - ((1 << (exp_bits - 1)) - 1);
    if (mantissa_bits < 23) mantissa <<= (23 - mantissa_bits);
    else if (mantissa_bits > 23) mantissa >>= (mantissa_bits - 23);
    f = __uint_as_float((sign << 31) | (uint32_t(exp + 127) << 23) | mantissa);
  }
  *p = __float_as_uint(f);
}

__global__ void modular_xyb_kernel(DevView vy, DevView vx, DevView vb, float mx, float my, float mb) {
  uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= vy.w) return;
  uint32_t* py = static_cast<uint32_t*>(vy.ptr) + size_t(y) * vy.stride + x;
  uint32_t* px = static_cast<uint32_t*>(vx.ptr) + size_t(y) * vx.stride + x;
  uint32_t* pb = static_cast<uint32_t*>(vb.ptr) + size_t(y) * vb.stride + x;
  int64_t bsum = int64_t(int32_t(*pb)) + int64_t(int32_t(*py));
  int32_t bi = int32_t(bsum < INT32_MIN ? INT32_MIN : (bsum > INT32_MAX ? INT32_MAX : bsum));
  float fy = float(int32_t(*py)), fx = float(int32_t(*px)), fb = float(bi);
  *py = __float_as_uint(__fmul_rn(fx, mx));
  *px = __float_as_uint(__fmul_rn(fy, my));
  *pb = __float_as_uint(__fmul_rn(fb, mb));
}

__global__ void fill_kernel(uint32_t* p, size_t n, uint32_t v) {
  size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
  size_t stride = size_t(gridDim.x) * blockDim.x;
  for (; i < n; i += stride) p[i] = v;
}

__global__ void copy_rect_kernel(DevView src, DevView dst) {
  uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= src.w) return;
  static_cast<uint32_t*>(dst.ptr)[size_t(y) * dst.stride + x] = static_cast<const uint32_t*>(src.ptr)[size_t(y) * src.stride + x];
}

inline dim3 grid2d(uint32_t w, uint32_t h, uint32_t bx = 128) { return dim3((w + bx - 1) / bx, h, 1); }

}  // namespace

void launch_squeeze_inverse_batch(const DevView* avg, const DevView* res, const DevView* out, int n, bool horizontal,
                                  cudaStream_t stream) {
  for (int i0 = 0; i0 < n; i0 += 4) {
    SqueezeBatch b;
    memset(&b, 0, sizeof(b));
    const int m = n - i0 < 4 ? n - i0 : 4;
    uint32_t max_w = 0, max_h = 0;
    for (int i = 0; i < m; ++i) {
      b.avg[i] = avg[i0 + i], b.res[i] = res[i0 + i], b.out[i] = out[i0 + i];
      max_w = max_w > out[i0 + i].w ? max_w : out[i0 + i].w;
      max_h = max_h > out[i0 + i].h ? max_h : out[i0 + i].h;
    }
    if (!max_w || !max_h) continue;
    if (horizontal) squeeze_h_kernel<<<dim3((max_h + kSqWarps * 32 - 1) / (kSqWarps * 32), m), kSqWarps * 32, 0, stream>>>(b);
    else squeeze_v_kernel<<<dim3((max_w + 63) / 64, m), 64, 0, stream>>>(b);
  }
}

void launch_squeeze_inverse(DevView avg, DevView res, DevView out, bool horizontal, cudaStream_t stream) {
  if (!out.w || !out.h) return;
  launch_squeeze_inverse_batch(&avg, &res, &out, 1, horizontal, stream);
}

void launch_rct_inverse(DevView a, DevView b, DevView c, uint32_t rct_type, cudaStream_t stream) {
  if (!a.w || !a.h) return;
  rct_kernel<<<grid2d(a.w, a.h), 128, 0, stream>>>(a, b, c, rct_type);
}

void launch_palette_inverse(DevView palette, const DevView* targets, int num_c, int nb_colours, int bit_depth, int nb_deltas,
                            uint8_t* mask, int* status, cudaStream_t stream) {
  PaletteTargets t;
  for (int i = 0; i < num_c && i < kMaxPaletteChannels; ++i) t.v[i] = targets[i];
  if (!t.v[0].w || !t.v[0].h) return;
  palette_kernel<<<grid2d(t.v[0].w, t.v[0].h), 128, 0, stream>>>(palette, t, num_c, nb_colours, bit_depth, nb_deltas, mask, status);
}

void launch_int_to_float(DevView v, uint32_t bits, uint32_t exp_bits, bool float_sample, cudaStream_t stream) {
  if (!v.w || !v.h) return;
  int_to_float_kernel<<<grid2d(v.w, v.h), 128, 0, stream>>>(v, bits, exp_bits, float_sample ? 1 : 0);
}

void launch_modular_xyb(DevView y, DevView x, DevView b, float mx, float my, float mb, cudaStream_t stream) {
  if (!y.w || !y.h) return;
  modular_xyb_kernel<<<grid2d(y.w, y.h), 128, 0, stream>>>(y, x, b, mx, my, mb);
}

void launch_fill_u32(uint32_t* p, size_t n, uint32_t value, cudaStream_t stream) {
  if (!n) return;
  size_t blocks = (n + 1023) / 1024;
  if (blocks > 132 * 16) blocks = 132 * 16;  // grid cap for the grid-stride loop (16 x the H100's 132 SMs)
  fill_kernel<<<unsigned(blocks), 256, 0, stream>>>(p, n, value);
}

void launch_copy_rect(DevView src, DevView dst, cudaStream_t stream) {
  if (!src.w || !src.h) return;
  copy_rect_kernel<<<grid2d(src.w, src.h), 128, 0, stream>>>(src, dst);
}

}  // namespace jxlb
