// Restoration filters and colour as stand-alone stages: Gaborish 3x3, edge-preserving filter (steps 0/1/2), XYB -> RGB
// (the per-pixel formulas: pixel_math.cuh), and the render features (upsampling, patches, splines, noise, JPEG chroma
// upsampling, YCbCr, packing). Float op order follows the reference's generic path. Compiled with -fmad=false; fused
// multiply-add only where the reference uses mul_add.
#include "kernels.h"
#include "pixel_math.cuh"

namespace jxlb {

namespace {

// impls/generic/gabor.rs, one thread per pixel
__global__ void gaborish_kernel(DevView in, DevView out, float w0, float w1) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  const int width = int(in.w), height = int(in.h);
  if (x >= width) return;
  const float* base = static_cast<const float*>(in.ptr);
  auto at = [&](int dx, int dy) { return base[size_t(y + dy) * in.stride + x + dx]; };
  const float res = gaborish_px(at, x, y, width, height, w0, w1, gaborish_norm(w0, w1));
  static_cast<float*>(out.ptr)[size_t(y) * out.stride + x] = res;
}

__device__ __forceinline__ int mirror(int offset, int len) {  // util.rs:376-386
  for (;;) {
    if (offset < 0) offset = -(offset + 1);
    else if (offset >= len) offset = 2 * len - (offset + 1);
    else return offset;
  }
}

struct View3 {
  DevView v[3];
};

// epf_row<STEP> (impls/generic/epf.rs:3-204): one thread per pixel, all three channels.
template <int STEP>
__global__ void epf_kernel(View3 in, View3 out, const float* __restrict__ sigma, uint32_t sigma_stride, DevEpfParams p) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  const int width = int(in.v[0].w), height = int(in.v[0].h);
  if (x >= width || y >= height) return;
  const float* ch[3] = {static_cast<const float*>(in.v[0].ptr), static_cast<const float*>(in.v[1].ptr),
                        static_cast<const float*>(in.v[2].ptr)};
  const size_t stride[3] = {in.v[0].stride, in.v[1].stride, in.v[2].stride};
  const float sigma_val = sigma ? sigma[size_t(y >> 3) * sigma_stride + (x >> 3)] : p.sigma_for_modular;
  float o[3];
  if (sigma_val < 0.3f) {
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = ch[c][size_t(y) * stride[c] + x];
  } else {
    const float neg_inv_sigma = fmul(epf_inv_sigma(sigma_val), epf_step_mul(p, STEP, epf_row_border(y) || epf_col_border(x)));
    float sum_weights = 1.0f;
    float sum_channels[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) sum_channels[c] = ch[c][size_t(y) * stride[c] + x];
#pragma unroll
    for (int k = 0; k < epf_neighbours(STEP); ++k) {
      const int kx = x + epf_nb_x(STEP, k), ky = y + epf_nb_y(STEP, k);
      float dist = 0.0f;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float acc = 0.0f;
#pragma unroll
        for (int i = 0; i < epf_plus_size(STEP); ++i) {
          const int ox = epf_plus_x(STEP, i), oy = epf_plus_y(STEP, i);
          const int ay = mirror(ky + oy, height), ax = mirror(kx + ox, width);
          const int by = mirror(y + oy, height), bx = mirror(x + ox, width);
          acc = fadd(acc, absdiff(ch[c][size_t(ay) * stride[c] + ax], ch[c][size_t(by) * stride[c] + bx]));
        }
        dist = fadd(dist, fmul(p.channel_scale[c], acc));
      }
      const float weight = epf_weight(dist, neg_inv_sigma);
      sum_weights = fadd(sum_weights, weight);
      const int my = mirror(ky, height), mx = mirror(kx, width);
#pragma unroll
      for (int c = 0; c < 3; ++c) sum_channels[c] = fadd(sum_channels[c], fmul(weight, ch[c][size_t(my) * stride[c] + mx]));
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = fdiv(sum_channels[c], sum_weights);
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) static_cast<float*>(out.v[c].ptr)[size_t(y) * out.v[c].stride + x] = o[c];
}

// apply_jpeg_upsampling_single (jxl-render/src/filter/ycbcr.rs:6-78): the horizontal pass, then the vertical pass over
// its output, both computed per output sample (edges replicate).
__device__ __forceinline__ float jpeg_hsample(const float* row, int x, int in_w, int horizontal) {
  if (!horizontal) return row[x];
  const int i = x >> 1;
  const float cur = row[i];
  if (x & 1) return fadd(fmul(0.75f, cur), fmul(0.25f, row[min(i + 1, in_w - 1)]));
  return fadd(fmul(0.25f, row[max(i - 1, 0)]), fmul(0.75f, cur));
}

__global__ void upsample_jpeg_kernel(DevView in, DevView out, int horizontal, int vertical) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= int(out.w)) return;
  const float* src = static_cast<const float*>(in.ptr);
  const int in_w = int(in.w), in_h = int(in.h);
  float v;
  if (!vertical) {
    v = jpeg_hsample(src + size_t(y) * in.stride, x, in_w, horizontal);
  } else {
    const int r = y >> 1;
    const float cur = jpeg_hsample(src + size_t(r) * in.stride, x, in_w, horizontal);
    if (y & 1) {
      const float below = jpeg_hsample(src + size_t(min(r + 1, in_h - 1)) * in.stride, x, in_w, horizontal);
      v = fadd(fmul(0.25f, below), fmul(0.75f, cur));
    } else {
      const float above = jpeg_hsample(src + size_t(max(r - 1, 0)) * in.stride, x, in_w, horizontal);
      v = fadd(fmul(0.75f, cur), fmul(0.25f, above));
    }
  }
  static_cast<float*>(out.ptr)[size_t(y) * out.stride + x] = v;
}

__global__ void ycbcr_to_rgb_kernel(DevView vcb, DevView vy, DevView vcr, DevYcbcrParams p) {
  const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= vy.w) return;
  float* pcb = static_cast<float*>(vcb.ptr) + size_t(y) * vcb.stride + x;
  float* py = static_cast<float*>(vy.ptr) + size_t(y) * vy.stride + x;
  float* pcr = static_cast<float*>(vcr.ptr) + size_t(y) * vcr.stride + x;
  const float cb = *pcb, yy = fadd(*py, p.y_offset), cr = *pcr;
  *pcb = ffma(cr, p.cr_to_r, yy);
  *py = ffma(cb, p.cb_to_g, ffma(cr, p.cr_to_g, yy));
  *pcr = ffma(cb, p.cb_to_b, yy);
}

__global__ void xyb_to_rgb_kernel(DevView vx, DevView vy, DevView vb, DevColorParams p) {
  const uint32_t x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y;
  if (x >= vx.w) return;
  float* px = static_cast<float*>(vx.ptr) + size_t(y) * vx.stride + x;
  float* py = static_cast<float*>(vy.ptr) + size_t(y) * vy.stride + x;
  float* pb = static_cast<float*>(vb.ptr) + size_t(y) * vb.stride + x;
  float o[3] = {*px, *py, *pb};
  xyb_to_linear(o, p);
  if (p.second_stage) second_colour_stage(o, p);
  if (p.pq_intensity_target > 0.0f) {
    const float y_mult = fdiv(p.pq_intensity_target, 10000.0f);
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = pq_tf(o[c], y_mult);
  } else if (p.gamma > 0.0f) {
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = gamma_tf(o[c], p.gamma);
  } else {
    encode_tf(o, colour_tf(p), kSrgbPow);
  }
  *px = o[0];
  *py = o[1];
  *pb = o[2];
}

// upsample_inner<K, NW> (features/upsampling.rs:45-132): one thread per output sample; the 5x5
// neighbourhood is read with mirrored coordinates (== the reference's mirror-padded copy).
__global__ void upsample_kernel(DevView in, DevView out, int k, const float* __restrict__ quarter) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= int(out.w) || y >= int(out.h)) return;
  const int gw = int(in.w), gh = int(in.h), mat_n = k / 2;
  const int ref_x = x / k, ref_y = y / k, px = x % k, py = y % k;
  const int mat_x = min(px, k - px - 1), mat_y = min(py, k - py - 1);
  const bool flip_h = px >= mat_n, flip_v = py >= mat_n;
  const float* kernel = quarter + (mat_y * mat_n + mat_x) * 25;
  const float* src = static_cast<const float*>(in.ptr);
  float sum = 0.0f, mn = INFINITY, mx = -INFINITY;
#pragma unroll
  for (int iy = 0; iy < 5; ++iy) {
    const int ky = flip_v ? 4 - iy : iy;
    // One-sample-wide / -high images: the reference fills its padding in place (util.rs:423-454), which leaves
    // zeros two samples to the left and right of a single column and two rows above a single row.
    const int sy = gh == 1 ? 0 : mirror(ref_y + iy - 2, gh);
    const bool zero_row = gh == 1 && iy == 0;
#pragma unroll
    for (int ix = 0; ix < 5; ++ix) {
      const int kx = flip_h ? 4 - ix : ix;
      const int sx = gw == 1 ? 0 : mirror(ref_x + ix - 2, gw);
      const bool zero = zero_row || (gw == 1 && (ix == 0 || ix == 4));
      const float sample = zero ? 0.0f : src[size_t(sy) * in.stride + sx];
      sum = fadd(sum, fmul(__ldg(kernel + ky * 5 + kx), sample));
      mn = fminf(mn, sample);
      mx = fmaxf(mx, sample);
    }
  }
  float r;
  if (!isfinite(mn)) r = __int_as_float(0x7fc00000);
  else r = sum < mn ? mn : (sum > mx ? mx : sum);
  static_cast<float*>(out.ptr)[size_t(y) * out.stride + x] = r;
}

// ---------------------------------------------------------------------------------------------
// Patches without alpha (blend.rs:550-606). Jobs of one launch may overlap in `dst` only if the bitstream
// makes patches overlap; they are then applied in job order by launching overlapping batches separately
// (the host splits the list), so inside a launch every destination sample has one writer.
__global__ void blend_patches_kernel(const DevPatchJob* __restrict__ jobs) {
  const DevPatchJob j = jobs[blockIdx.x];
  for (uint32_t i = threadIdx.x; i < j.w * j.h; i += blockDim.x) {
    const uint32_t x = i % j.w, y = i / j.w;
    float v = j.src[size_t(y) * j.src_stride + x];
    float* d = j.dst + size_t(y) * j.dst_stride + x;
    const float base = *d;
    float r;
    if (j.mode == 1) {
      r = v;
    } else if (j.mode == 2) {
      r = fadd(base, v);
    } else if (j.mode == 3) {
      if (j.clamp) v = v < 0.0f ? 0.0f : (v > 1.0f ? 1.0f : v);
      r = fmul(base, v);
    } else if (j.mode == 4) {
      const float frame_alpha = j.base_alpha ? j.base_alpha[size_t(y) * j.base_alpha_stride + x] : 0.0f;
      const float patch_alpha = j.new_alpha ? j.new_alpha[size_t(y) * j.new_alpha_stride + x] : 0.0f;
      const float base_sample = j.swapped ? v : base, new_sample = j.swapped ? base : v;
      const float base_alpha = j.swapped ? patch_alpha : frame_alpha;
      float new_alpha = j.swapped ? frame_alpha : patch_alpha;
      if (j.clamp) new_alpha = new_alpha < 0.0f ? 0.0f : (new_alpha > 1.0f ? 1.0f : new_alpha);
      if (j.premultiplied) {
        r = fadd(new_sample, fmul(base_sample, fsub(1.0f, new_alpha)));
      } else {
        const float base_alpha_rev = fsub(1.0f, base_alpha), new_alpha_rev = fsub(1.0f, new_alpha);
        const float mixed_alpha = fsub(1.0f, fmul(new_alpha_rev, base_alpha_rev));
        const float mixed_alpha_recip = mixed_alpha > 0.0f ? fdiv(1.0f, mixed_alpha) : 0.0f;
        r = fmul(fadd(fmul(new_alpha, new_sample), fmul(fmul(base_alpha, base_sample), new_alpha_rev)), mixed_alpha_recip);
      }
    } else if (j.mode == 5) {
      const float base_sample = j.swapped ? v : base, new_sample = j.swapped ? base : v;
      float new_alpha;
      if (j.swapped) new_alpha = j.base_alpha ? j.base_alpha[size_t(y) * j.base_alpha_stride + x] : 0.0f;
      else new_alpha = j.new_alpha ? j.new_alpha[size_t(y) * j.new_alpha_stride + x] : 0.0f;
      if (j.clamp) new_alpha = new_alpha < 0.0f ? 0.0f : (new_alpha > 1.0f ? 1.0f : new_alpha);
      r = fadd(base_sample, fmul(new_alpha, new_sample));
    } else {
      const float b0 = j.swapped ? v : base;
      float n0 = j.swapped ? base : v;
      if (j.clamp) n0 = n0 < 0.0f ? 0.0f : (n0 > 1.0f ? 1.0f : n0);
      r = fadd(b0, fmul(n0, fsub(1.0f, b0)));
    }
    *d = r;
  }
}

// ---------------------------------------------------------------------------------------------
// Splines (features/spline.rs:218-252, erf :314-331)
__device__ __forceinline__ float spline_erf(float x) {
  const float ax = fabsf(x);
  const float denom1 = fadd(fmul(ax, 7.77394369e-02f), 2.05260015e-04f);
  const float denom2 = fadd(fmul(denom1, ax), 2.32120216e-01f);
  const float denom3 = fadd(fmul(denom2, ax), 2.77820801e-01f);
  const float denom4 = fadd(fmul(denom3, ax), 1.0f);
  const float denom5 = fmul(denom4, denom4);
  const float inv_denom5 = fdiv(1.0f, denom5);
  const float result = fadd(fmul(-inv_denom5, inv_denom5), 1.0f);
  return x < 0.0f ? -result : result;
}

// One thread per pixel, 32x8 tiles. The arc list is walked in chunks of 256: every thread tests one arc's bounding box
// against the tile and the hits are compacted IN LIST ORDER into shared memory (float addition order is part of the
// result), then every pixel accumulates the surviving arcs.
__global__ void __launch_bounds__(256) splat_splines_kernel(DevView v0, DevView v1, DevView v2, const DevSplineArc* __restrict__ arcs,
                                                            int num_arcs) {
  __shared__ DevSplineArc hit[256];
  __shared__ int warp_count[8];
  const int tid = threadIdx.y * 32 + threadIdx.x, lane = threadIdx.x, warp = threadIdx.y;
  const int tx0 = blockIdx.x * 32, ty0 = blockIdx.y * 8;
  const int x = tx0 + lane, y = ty0 + warp;
  const bool inside = x < int(v0.w) && y < int(v0.h);
  float* p[3] = {static_cast<float*>(v0.ptr) + size_t(y) * v0.stride + x, static_cast<float*>(v1.ptr) + size_t(y) * v1.stride + x,
                 static_cast<float*>(v2.ptr) + size_t(y) * v2.stride + x};
  float acc[3] = {0.0f, 0.0f, 0.0f};
  if (inside) acc[0] = *p[0], acc[1] = *p[1], acc[2] = *p[2];
  bool touched = false;
  for (int base = 0; base < num_arcs; base += 256) {
    DevSplineArc a;
    bool h = false;
    if (base + tid < num_arcs) {
      a = arcs[base + tid];
      h = a.xbegin < tx0 + 32 && a.xend > tx0 && a.ybegin < ty0 + 8 && a.yend > ty0;
    }
    const unsigned m = __ballot_sync(0xffffffffu, h);
    if (lane == 0) warp_count[warp] = __popc(m);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < 8; ++w) {
      if (w < warp) before += warp_count[w];
      total += warp_count[w];
    }
    if (h) hit[before + __popc(m & ((1u << lane) - 1u))] = a;
    __syncthreads();
    if (inside)
      for (int i = 0; i < total; ++i) {
        const DevSplineArc& q = hit[i];
        if (x < q.xbegin || x >= q.xend || y < q.ybegin || y >= q.yend) continue;
        const float dx = fsub(float(x), q.x), dy = fsub(float(y), q.y);
        const float distance = fsqrt(fadd(fmul(dx, dx), fmul(dy, dy)));
        const float factor = fsub(spline_erf(fmul(fadd(fmul(0.5f, distance), 0.35355338f), q.inv_sigma)),
                                  spline_erf(fmul(fsub(fmul(0.5f, distance), 0.35355338f), q.inv_sigma)));
#pragma unroll
        for (int c = 0; c < 3; ++c) acc[c] = fadd(acc[c], fmul(fmul(fmul(fmul(0.25f, q.value[c]), q.sigma), factor), factor));
        touched = true;
      }
    __syncthreads();
  }
  if (touched) {
    *p[0] = acc[0];
    *p[1] = acc[1];
    *p[2] = acc[2];
  }
}

// ---------------------------------------------------------------------------------------------
// Noise synthesis (features/noise.rs)
__device__ __forceinline__ unsigned long long split_mix_64(unsigned long long z) {  // noise.rs:454-458
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  return z ^ (z >> 31);
}

// The reference's generator is eight independent xorshift128+ streams (noise.rs:405-451) whose outputs are
// interleaved into batches of 16 floats; one thread per (group, stream) walks its stream through the
// group's three channels and stores the two floats each step contributes.
__global__ void noise_field_kernel(float* f0, float* f1, float* f2, uint32_t width, uint32_t height, uint32_t group_dim,
                                   unsigned long long seed0) {
  const uint32_t gpr = (width + group_dim - 1) / group_dim, gpc = (height + group_dim - 1) / group_dim;
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t g = t >> 3, lane = t & 7;
  if (g >= gpr * gpc) return;
  const uint32_t x0 = (g % gpr) * group_dim, y0 = (g / gpr) * group_dim;
  const uint32_t gw = min(group_dim, width - x0), gh = min(group_dim, height - y0);
  const unsigned long long seed1 = ((unsigned long long)(x0) << 32) + (unsigned long long)(y0);
  unsigned long long s0 = split_mix_64(seed0 + 0x9E3779B97F4A7C15ull), s1 = split_mix_64(seed1 + 0x9E3779B97F4A7C15ull);
  for (uint32_t i = 0; i < lane; ++i) {
    s0 = split_mix_64(s0);
    s1 = split_mix_64(s1);
  }
  const uint32_t width_n2 = (gw + 15) / 16;
  float* planes[3] = {f0, f1, f2};
  for (int c = 0; c < 3; ++c) {
    float* dst = planes[c];
    for (uint32_t row = 0; row < gh; ++row)
      for (uint32_t cb = 0; cb < width_n2; ++cb) {
        unsigned long long a = s0;
        const unsigned long long b = s1;
        const unsigned long long ret = a + b;
        s0 = b;
        a ^= a << 23;
        s1 = a ^ (b ^ (a >> 18) ^ (b >> 5));
        const uint32_t x = cb * 16 + 2 * lane;
        float* o = dst + size_t(y0 + row) * width + x0 + x;
        if (x < gw) o[0] = __uint_as_float((uint32_t(ret) >> 9) | 0x3f800000u);
        if (x + 1 < gw) o[1] = __uint_as_float((uint32_t(ret >> 32) >> 9) | 0x3f800000u);
      }
  }
}

// 5x5 high-pass of the width x height field (rows added in the order of the reference's 5-row ring buffer, which
// depends on the row's position inside its group: noise.rs:297-320; mirrored at the field's edges) and application to
// the XYB planes (noise.rs:45-83), whose view is the field's top-left corner (noise.rs:21-33).
__global__ void noise_apply_kernel(DevView vx, DevView vy, DevView vb, const float* __restrict__ f0,
                                   const float* __restrict__ f1, const float* __restrict__ f2, int width, int height,
                                   DevNoiseParams p) {
  const int x = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y * blockDim.y + threadIdx.y;
  if (x >= int(vx.w) || y >= int(vx.h)) return;
  const int ly = y % int(p.group_dim);
  const float* fields[3] = {f0, f1, f2};
  float n[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) {
    const float* f = fields[c];
    float sum = 0.0f;
#pragma unroll
    for (int s = 0; s < 5; ++s) {
      const int r = ly - 2 + (((s - ly) % 5) + 5) % 5;  // local row held by ring slot s
      const int sy = mirror(y - ly + r, height);
#pragma unroll
      for (int dx = 0; dx < 5; ++dx) {
        const int sx = mirror(x + dx - 2, width);
        sum = fadd(sum, fmul(f[size_t(sy) * width + sx], 0.16f));
      }
    }
    n[c] = fsub(sum, fmul(f[size_t(y) * width + x], 4.0f));
  }
  float* px = static_cast<float*>(vx.ptr) + size_t(y) * vx.stride + x;
  float* py = static_cast<float*>(vy.ptr) + size_t(y) * vy.stride + x;
  float* pb = static_cast<float*>(vb.ptr) + size_t(y) * vb.stride + x;
  const float grid_x = *px, grid_y = *py;
  const float in_x = fadd(grid_x, grid_y), in_y = fsub(grid_y, grid_x);
  const float in_scaled_x = fmaxf(0.0f, fmul(in_x, 3.0f)), in_scaled_y = fmaxf(0.0f, fmul(in_y, 3.0f));
  // `as usize` saturates (and maps NaN to 0) before the min with 7
  const uint32_t in_x_int = min(uint32_t(__float2uint_rz(in_scaled_x)), 7u), in_y_int = min(uint32_t(__float2uint_rz(in_scaled_y)), 7u);
  const float in_x_frac = fsub(in_scaled_x, float(in_x_int)), in_y_frac = fsub(in_scaled_y, float(in_y_int));
  const float sx = fadd(fmul(fsub(p.lut[in_x_int + 1], p.lut[in_x_int]), in_x_frac), p.lut[in_x_int]);
  const float sy = fadd(fmul(fsub(p.lut[in_y_int + 1], p.lut[in_y_int]), in_y_frac), p.lut[in_y_int]);
  const float nx = fmul(fmul(0.22f, sx), fadd(fmul(0.0078125f, n[0]), fmul(0.9921875f, n[2])));
  const float ny = fmul(fmul(0.22f, sy), fadd(fmul(0.0078125f, n[1]), fmul(0.9921875f, n[2])));
  const float nsum = fadd(nx, ny);
  *px = fadd(*px, fsub(fadd(fmul(p.corr_x, nsum), nx), ny));
  *py = fadd(*py, nsum);
  *pb = fadd(*pb, fmul(p.corr_b, nsum));
}

}  // namespace

void launch_blend_patches(const DevPatchJob* jobs, int num_jobs, cudaStream_t stream) {
  if (num_jobs <= 0) return;
  blend_patches_kernel<<<num_jobs, 128, 0, stream>>>(jobs);
}

void launch_splat_splines(const DevView v[3], const DevSplineArc* arcs, int num_arcs, cudaStream_t stream) {
  if (num_arcs <= 0 || !v[0].w || !v[0].h) return;
  dim3 block(32, 8);
  dim3 grid((v[0].w + 31) / 32, (v[0].h + 7) / 8);
  splat_splines_kernel<<<grid, block, 0, stream>>>(v[0], v[1], v[2], arcs, num_arcs);
}

void launch_add_noise(const DevView v[3], float* const field[3], uint32_t field_w, uint32_t field_h, DevNoiseParams p,
                      cudaStream_t stream) {
  if (!v[0].w || !v[0].h) return;
  const uint32_t groups = ((field_w + p.group_dim - 1) / p.group_dim) * ((field_h + p.group_dim - 1) / p.group_dim);
  noise_field_kernel<<<(groups * 8 + 63) / 64, 64, 0, stream>>>(field[0], field[1], field[2], field_w, field_h, p.group_dim, p.seed0);
  dim3 block(32, 8);
  dim3 grid((v[0].w + 31) / 32, (v[0].h + 7) / 8);
  noise_apply_kernel<<<grid, block, 0, stream>>>(v[0], v[1], v[2], field[0], field[1], field[2], int(field_w), int(field_h), p);
}

void launch_upsample(DevView in, DevView out, int k, const float* quarter, cudaStream_t stream) {
  if (!out.w || !out.h) return;
  dim3 block(32, 8);
  dim3 grid((out.w + 31) / 32, (out.h + 7) / 8);
  upsample_kernel<<<grid, block, 0, stream>>>(in, out, k, quarter);
}

void launch_gaborish(DevView in, DevView out, float w0, float w1, cudaStream_t stream) {
  if (!in.w || !in.h) return;
  dim3 grid((in.w + 127) / 128, in.h);
  gaborish_kernel<<<grid, 128, 0, stream>>>(in, out, w0, w1);
}

void launch_epf_step(const DevView in[3], const DevView out[3], const float* sigma, uint32_t sigma_stride, DevEpfParams p,
                     int step, cudaStream_t stream) {
  View3 vi, vo;
  for (int c = 0; c < 3; ++c) {
    vi.v[c] = in[c];
    vo.v[c] = out[c];
  }
  if (!vi.v[0].w || !vi.v[0].h) return;
  dim3 block(32, 8);
  dim3 grid((vi.v[0].w + 31) / 32, (vi.v[0].h + 7) / 8);
  if (step == 0) epf_kernel<0><<<grid, block, 0, stream>>>(vi, vo, sigma, sigma_stride, p);
  else if (step == 1) epf_kernel<1><<<grid, block, 0, stream>>>(vi, vo, sigma, sigma_stride, p);
  else epf_kernel<2><<<grid, block, 0, stream>>>(vi, vo, sigma, sigma_stride, p);
}

void launch_upsample_jpeg(DevView in, DevView out, int horizontal, int vertical, cudaStream_t stream) {
  if (!out.w || !out.h) return;
  dim3 grid((out.w + 127) / 128, out.h);
  upsample_jpeg_kernel<<<grid, 128, 0, stream>>>(in, out, horizontal, vertical);
}

void launch_ycbcr_to_rgb(DevView cb, DevView y, DevView cr, DevYcbcrParams p, cudaStream_t stream) {
  if (!y.w || !y.h) return;
  dim3 grid((y.w + 127) / 128, y.h);
  ycbcr_to_rgb_kernel<<<grid, 128, 0, stream>>>(cb, y, cr, p);
}

void launch_xyb_to_rgb(DevView x, DevView y, DevView b, DevColorParams p, cudaStream_t stream) {
  if (!x.w || !x.h) return;
  dim3 grid((x.w + 127) / 128, x.h);
  xyb_to_rgb_kernel<<<grid, 128, 0, stream>>>(x, y, b, p);
}

}  // namespace jxlb
