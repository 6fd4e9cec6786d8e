// Fused restoration-filter chain: Gaborish -> EPF step 0/1/2 -> XYB->RGB in ONE kernel.
//
// Unfused, every stage is an HBM->HBM pass over three f32 planes (24 B/px each: up to 120 B/px
// for Gaborish + 3 EPF steps + colour). Here a CTA owns a 32x32 output tile, loads the tile plus
// the halo the enabled stages need (<= 7 px) into shared memory once, runs the stages ping-pong
// between two shared buffers and writes the final pixels: 12 B/px read (+halo, served by L2) and
// 12 B/px written.
//
// EPF in two half-stages per step. The reference computes, per pixel p and neighbour k, the patch distance
//   dist_k(p) = sum_c scale_c * sum_{o in plus} |a_c[p+k+o] - a_c[p+o]|        (epf.rs:3-210)
// i.e. 12 x 15 (step 0) / 4 x 15 (step 1) / 4 x 3 (step 2) absolute differences. But |x - y| == |y - x| bit for bit, and
// the sums run over the same o and c in the same order, so dist_{-d}(p) == dist_d(p - d) EXACTLY: opposite neighbours
// share one distance map. Half-stage 1 evaluates the 6 / 2 / 2 maps of the "positive" directions once per pixel into
// shared memory; half-stage 2 reads two values per direction pair and forms weights and weighted sums in the
// reference's neighbour order. Same values, same rounding, half the arithmetic and a third of the shared-memory reads.
//
// The per-pixel formulas are those of every filter kernel (pixel_math.cuh, the reference's generic path). Border semantics:
// Gaborish uses its own edge formulas on the image border (gabor.rs:119-167); EPF mirrors coordinates (util.rs:376-386) --
// after each stage the part of the halo that lies outside the image is filled by mirroring, so the stencils index plainly.
#include "filter_strip.cuh"
#include "kernels.h"

#include <cuda.h>  // CUtensorMap (types only: the encoder entry point is fetched from the driver at run time)

#include <cstdlib>
#include <cstring>
#include <type_traits>

namespace jxlb {

namespace {

constexpr int kT = 32;  // output tile
// Shared-memory planes are kS x kS cells with a margin of (kS - kT) / 2 around the tile: 48 (margin 8 >= stencil radius 7) when
// the frame runs EPF step 0, 40 (margin 4 = Gaborish 1 + step 1's 2 + step 2's 1) otherwise - 8 planes of 40 x 40 are
// 51 KB, so four CTAs share an SM instead of three. Every device function below is a template on kS.
__host__ __device__ constexpr int window_size(int nmaps) { return nmaps == 6 ? 48 : 40; }

struct Rect {  // in shared-memory cell coordinates, half-open
  int x0, y0, x1, y1;
};

__device__ __forceinline__ int mirror1(int v, int len) {  // single reflection (|overhang| <= 7 < len)
  return v < 0 ? -v - 1 : (v >= len ? 2 * len - v - 1 : v);
}

// "Positive" directions of each step; the other half of the neighbour list is their negation.
//   step 0: (0,2) (1,1) (0,1) (-1,1) (2,0) (1,0)        steps 1, 2: (0,1) (1,0)
__device__ __forceinline__ constexpr int dplus_x(int step, int m) {
  return step == 0 ? (m == 0 ? 0 : m == 1 ? 1 : m == 2 ? 0 : m == 3 ? -1 : m == 4 ? 2 : 1) : (m == 0 ? 0 : 1);
}
__device__ __forceinline__ constexpr int dplus_y(int step, int m) {
  return step == 0 ? (m == 0 ? 2 : m == 1 ? 1 : m == 2 ? 1 : m == 3 ? 1 : 0) : (m == 0 ? 1 : 0);
}

// Half-stage 1: the distance maps of one EPF step at cell q. `a` points at q in channel 0 of the input buffer, `d` at q in
// map 0 (maps kPlane apart). dist_d(q) = sum_c scale_c * sum_o |a_c[q+d+o] - a_c[q+o]|, accumulated exactly like
// epf.rs (acc starts at 0.0, so the first addition is exact; likewise dist).
template <int STEP, int kS>
__device__ __forceinline__ void epf_dist(const float* __restrict__ a, float* __restrict__ d, const DevEpfParams& p) {
  constexpr int kPlane = kS * kS;
  constexpr int NM = STEP == 0 ? 6 : 2;
  constexpr int ND = epf_plus_size(STEP);
  float dist[NM];  // all maps first, stores last: a store between them would make the compiler reload every sample
#pragma unroll
  for (int m = 0; m < NM; ++m) {
    const int dx = dplus_x(STEP, m), dy = dplus_y(STEP, m);
    dist[m] = 0.0f;
    // epf.rs starts both sums at 0.0; 0.0 + t == t bit for bit for the non-negative t added first, so the first term is
    // taken as it is
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      float acc = 0.0f;
#pragma unroll
      for (int i = 0; i < ND; ++i) {
        const int ox = epf_plus_x(STEP, i), oy = epf_plus_y(STEP, i);
        const float t = absdiff(a[c * kPlane + (dy + oy) * kS + dx + ox], a[c * kPlane + oy * kS + ox]);
        acc = i == 0 ? t : fadd(acc, t);
      }
      const float term = fmul(p.channel_scale[c], acc);
      dist[m] = c == 0 ? term : fadd(dist[m], term);
    }
  }
#pragma unroll
  for (int m = 0; m < NM; ++m) d[m * kPlane] = dist[m];
}

// Half-stage 2: weights and weighted sums at pixel p in the reference's neighbour order; `a` points at p in channel 0 of
// the input buffer, `d` at p in distance map 0, `inv_sigma` is epf_inv_sigma of p's 8x8 block.
template <int STEP, int kS>
__device__ __forceinline__ void epf_apply(const float* a, const float* d, int x, int y, float sigma_val, float inv_sigma,
                                          const DevEpfParams& p, float o[3]) {
  constexpr int kPlane = kS * kS;
  if (sigma_val < 0.3f) {
#pragma unroll
    for (int c = 0; c < 3; ++c) o[c] = a[c * kPlane];
    return;
  }
  const float neg_inv_sigma = fmul(inv_sigma, epf_step_mul(p, STEP, epf_row_border(y) || epf_col_border(x)));
  float sum_weights = 1.0f;
  float sum_channels[3];
#pragma unroll
  for (int c = 0; c < 3; ++c) sum_channels[c] = a[c * kPlane];
  constexpr int NM = STEP == 0 ? 6 : 2;
#pragma unroll
  for (int k = 0; k < epf_neighbours(STEP); ++k) {
    const int kx = epf_nb_x(STEP, k), ky = epf_nb_y(STEP, k);
    // which map holds this neighbour's distance, and at which cell
    float dist = 0.0f;
#pragma unroll
    for (int m = 0; m < NM; ++m) {
      const int dx = dplus_x(STEP, m), dy = dplus_y(STEP, m);
      if (dx == kx && dy == ky) dist = d[m * kPlane];                      // positive direction: dist_d(p)
      if (dx == -kx && dy == -ky) dist = d[m * kPlane + ky * kS + kx];     // its negation: dist_d(p - d) = dist_d(p + k)
    }
    const float weight = epf_weight(dist, neg_inv_sigma);
    sum_weights = fadd(sum_weights, weight);
#pragma unroll
    for (int c = 0; c < 3; ++c) sum_channels[c] = fadd(sum_channels[c], fmul(weight, a[c * kPlane + ky * kS + kx]));
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) o[c] = fdiv(sum_channels[c], sum_weights);
}

// Visits every cell of `r` once with all 256 threads busy: the cells are numbered row by row and thread t takes cells
// t, t + 256, ... (a 35 x 35 region walked as 32-wide column strips would leave the second strip 3 lanes wide). One
// integer division per call; afterwards (x, y) advance incrementally.
__device__ __constant__ const uint32_t kRecip16[49] = {
    0,     65536, 32768, 21846, 16384, 13108, 10923, 9363, 8192, 7282, 6554, 5958, 5462, 5042, 4682, 4370, 4096,
    3856,  3641,  3450,  3277,  3121,  2979,  2850,  2731, 2622, 2521, 2428, 2341, 2260, 2185, 2115, 2048, 1986,
    1928,  1873,  1821,  1772,  1725,  1681,  1639,  1599, 1561, 1525, 1490, 1457, 1425, 1395, 1366};
template <typename F>
__device__ __forceinline__ void for_region(const Rect& r, F&& f) {
  const int w = r.x1 - r.x0, h = r.y1 - r.y0;
  if (w <= 0 || h <= 0) return;
  const int n = w * h;
  const int tid = int(threadIdx.y) * 32 + int(threadIdx.x);
  // tid / w and 256 / w without a division: ceil(2^16 / w) * t >> 16 == t / w for t <= 256, w <= 48
  const uint32_t rcp = kRecip16[w];
  int ly = int((uint32_t(tid) * rcp) >> 16), lx = tid - ly * w;
  const int dy = int((256u * rcp) >> 16), dx = 256 - dy * w;
  for (int i = tid; i < n; i += 256) {
    f(r.x0 + lx, r.y0 + ly);
    lx += dx;
    ly += dy;
    if (lx >= w) {
      lx -= w;
      ++ly;
    }
  }
}

struct FusedViews {
  const float* in[3];
  float* out[3];
  uint32_t in_stride[3], out_stride[3];
  int width, height;
  int use_tma;  // the three input planes are described by `maps` (row pitch a multiple of 16 bytes)
  // border_only: the launch is a 1-D grid over the tiles outside [1, bx_last] x [1, by_last] (the strip kernel covers those)
  int border_only, bx_last, by_last, nbx, nby;
};

// Tile of a border-only launch (fstrip::border_tile_index, shared with the host-side check in tests/emu).
__device__ __forceinline__ void border_tile_of(const FusedViews& v, int i, int& tx, int& ty) {
  fstrip::border_tile_index(v.nbx, v.nby, v.bx_last, v.by_last, i, tx, ty);
}

// TMA descriptors of the three input planes (encode_plane_maps).
struct FusedMaps {
  CUtensorMap map[3];
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }

// Window load by TMA: the elected thread arms the mbarrier `mbar` with the byte count and issues three bulk tensor copies,
// one box per plane with its corner at image pixel (gx0, gy0), into dst[c * kPlane]; the copies of the three planes are in
// flight together, and no thread spends registers or address arithmetic on them. Cells outside the image arrive as zeros.
template <int kPlane>
__device__ __forceinline__ void window_load_issue(uint32_t mbar, float* dst, const FusedMaps& maps, int gx0, int gy0) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mbar));
  asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(uint32_t(3 * kPlane * sizeof(float))) : "memory");
#pragma unroll
  for (int c = 0; c < 3; ++c)
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
            smem_u32(dst + c * kPlane)),
        "l"(reinterpret_cast<uint64_t>(&maps.map[c])), "r"(gx0), "r"(gy0), "r"(mbar)
        : "memory");
}

// Every thread waits on the barrier's phase; the barrier must be initialised (a __syncthreads after the issue) before.
__device__ __forceinline__ void window_load_wait(uint32_t mbar) {
  uint32_t done = 0;
  for (uint32_t spin = 0; !done && spin < (1u << 24); ++spin)
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(mbar), "r"(0u)
        : "memory");
}

// Cells of `need` that lie outside the image take the value of their mirrored in-image cell.
template <int kS>
__device__ __forceinline__ void mirror_fill(float* buf, Rect need, int gx0, int gy0, int width, int height) {
  constexpr int kPlane = kS * kS;
  for (int ly = need.y0 + int(threadIdx.y); ly < need.y1; ly += int(blockDim.y))
    for (int lx = need.x0 + int(threadIdx.x); lx < need.x1; lx += int(blockDim.x)) {
      const int gx = gx0 + lx, gy = gy0 + ly;
      if (gx >= 0 && gx < width && gy >= 0 && gy < height) continue;
      const int sx = mirror1(gx, width) - gx0, sy = mirror1(gy, height) - gy0;
      // cells further outside than the remaining stencil reach mirror to sources left of / above
      // the computed region; no stage reads them
      if (sx < need.x0 || sy < need.y0) continue;
#pragma unroll
      for (int c = 0; c < 3; ++c) buf[c * kPlane + ly * kS + lx] = buf[c * kPlane + sy * kS + sx];
    }
}

// NMAPS: distance maps kept in shared memory (6 when the frame runs EPF step 0, else 2; 0 without EPF).
template <int NMAPS>
__global__ void __launch_bounds__(256) fused_filter_kernel(FusedViews v, DevFusedFilterParams p, const __grid_constant__ FusedMaps maps) {
  constexpr int kS = window_size(NMAPS), kPlane = kS * kS, kHM = (kS - kT) / 2;
  extern __shared__ __align__(128) float s_buf[];
  __shared__ __align__(8) unsigned long long s_mbar;
  __shared__ float s_sigma[49], s_inv_sigma[49];  // per 8x8 block under the window (at most 7 x 7 of them)
  float* cur = s_buf;               // [3][kS][kS]
  float* alt = s_buf + 3 * kPlane;
  float* dmap = s_buf + 6 * kPlane;  // [NMAPS][kS][kS]
  const int width = v.width, height = v.height;
  // shared cell (lx, ly) <-> image pixel (gx0 + lx, gy0 + ly)
  int tile_x = int(blockIdx.x), tile_y = int(blockIdx.y);
  if (v.border_only) border_tile_of(v, int(blockIdx.x), tile_x, tile_y);
  const int gx0 = tile_x * kT - kHM, gy0 = tile_y * kT - kHM;
  const bool border_tile = gx0 < 0 || gy0 < 0 || gx0 + kS > width || gy0 + kS > height;
  const int r_gab = p.gab_enabled ? 1 : 0;
  const int r0 = p.epf_iters == 3 ? 3 : 0, r1 = p.epf_iters >= 1 ? 2 : 0, r2 = p.epf_iters >= 2 ? 1 : 0;
  int halo = r_gab + r0 + r1 + r2;
  auto rect = [&](int h) { return Rect{kHM - h, kHM - h, kHM + kT + h, kHM + kT + h}; };
  auto clip = [&](Rect r) {  // to the image
    r.x0 = max(r.x0, -gx0), r.y0 = max(r.y0, -gy0);
    r.x1 = min(r.x1, width - gx0), r.y1 = min(r.y1, height - gy0);
    return r;
  };

  // sigma and the division it feeds, once per 8x8 block under the window instead of once per pixel and step (same operands,
  // same result: epf.rs computes 6.6 * (1/sqrt(2) - 1) / sigma for every pixel of the block)
  const int bx_first = max(gx0, 0) >> 3, by_first = max(gy0, 0) >> 3;
  if (NMAPS > 0 && p.epf_iters > 0) {
    const int t = int(threadIdx.y) * 32 + int(threadIdx.x);
    if (t < 49) {
      const int bx = bx_first + t % 7, by = by_first + t / 7;
      float sg = p.epf.sigma_for_modular;
      if (p.sigma) sg = (bx < ((width + 7) >> 3) && by < ((height + 7) >> 3)) ? __ldg(p.sigma + size_t(by) * p.sigma_stride + bx) : 1.0f;
      s_sigma[t] = sg;
      s_inv_sigma[t] = epf_inv_sigma(sg);
    }
  }

  if (v.use_tma) {
    // tile + halo: the whole kS x kS window of each plane (cells outside the image are never read before mirror_fill
    // overwrites them)
    const uint32_t mbar = smem_u32(&s_mbar);
    if (threadIdx.x == 0 && threadIdx.y == 0) window_load_issue<kPlane>(mbar, cur, maps, gx0, gy0);
    __syncthreads();  // the barrier is initialised before anybody polls it
    window_load_wait(mbar);
  } else {  // load the input region (planes whose pitch TMA cannot address)
    const Rect r = clip(rect(halo));
    for_region(r, [&](int lx, int ly) {
#pragma unroll
      for (int c = 0; c < 3; ++c) cur[c * kPlane + ly * kS + lx] = v.in[c][size_t(gy0 + ly) * v.in_stride[c] + gx0 + lx];
    });
  }
  __syncthreads();

  if (p.gab_enabled) {
    halo -= 1;
    const Rect r = clip(rect(halo));
    float gw[3];
#pragma unroll
    for (int c = 0; c < 3; ++c) gw[c] = gaborish_norm(p.gab_w[c][0], p.gab_w[c][1]);
    if (!border_tile) {  // no pixel of the window lies on the image border: the 3x3 formula without the edge cases
      for_region(r, [&](int lx, int ly) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float* a = cur + c * kPlane + ly * kS + lx;
          alt[c * kPlane + ly * kS + lx] = gaborish_3x3(a[-kS - 1], a[-kS], a[-kS + 1], a[-1], a[0], a[1], a[kS - 1], a[kS], a[kS + 1],
                                                        p.gab_w[c][0], p.gab_w[c][1], gw[c]);
        }
      });
    } else {
      for_region(r, [&](int lx, int ly) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const float* a = cur + c * kPlane + ly * kS + lx;
          alt[c * kPlane + ly * kS + lx] = gaborish_px([a](int dx, int dy) { return a[dy * kS + dx]; }, gx0 + lx, gy0 + ly, width,
                                                       height, p.gab_w[c][0], p.gab_w[c][1], gw[c]);
        }
      });
    }
    float* t = cur;
    cur = alt;
    alt = t;
    __syncthreads();
  }
  if (p.epf_iters > 0 && border_tile) {  // EPF reads mirrored pixels beyond the image border
    mirror_fill<kS>(cur, rect(halo), gx0, gy0, width, height);
    __syncthreads();
  }

  auto epf_stage = [&](auto step_tag, int radius, bool last) {
    constexpr int STEP = decltype(step_tag)::value;
    if constexpr (NMAPS >= (STEP == 0 ? 6 : 2)) {
      halo -= radius;
      const Rect out = rect(halo);
      {  // half-stage 1: distance maps wherever a pixel of `out` or its negative-direction neighbour looks them up
         // (cells beyond the image included: they stand for mirrored pixels)
        constexpr int ex = STEP == 0 ? 2 : 1;  // reach of the negated directions: x - 2 .. x + 1 (step 0), x - 1 .. x
        const Rect q{out.x0 - ex, out.y0 - ex, out.x1 + (STEP == 0 ? 1 : 0), out.y1};
        for_region(q, [&](int lx, int ly) { epf_dist<STEP, kS>(cur + ly * kS + lx, dmap + ly * kS + lx, p.epf); });
      }
      __syncthreads();
      const Rect r = clip(out);
      for_region(r, [&](int lx, int ly) {
        const int x = gx0 + lx, y = gy0 + ly;
        const int bi = ((y >> 3) - by_first) * 7 + ((x >> 3) - bx_first);
        float o[3];
        epf_apply<STEP, kS>(cur + ly * kS + lx, dmap + ly * kS + lx, x, y, s_sigma[bi], s_inv_sigma[bi], p.epf, o);
        if (last) {
          if (p.colour) xyb_to_rgb_px(o, p.col, colour_tf(p.col), kSrgbPow);
#pragma unroll
          for (int c = 0; c < 3; ++c) v.out[c][size_t(y) * v.out_stride[c] + x] = o[c];
        } else {
#pragma unroll
          for (int c = 0; c < 3; ++c) alt[c * kPlane + ly * kS + lx] = o[c];
        }
      });
      if (!last) {
        float* t = cur;
        cur = alt;
        alt = t;
        __syncthreads();
        if (border_tile) {
          mirror_fill<kS>(cur, rect(halo), gx0, gy0, width, height);
          __syncthreads();
        }
      }
    }
  };
  if (p.epf_iters == 3) epf_stage(std::integral_constant<int, 0>{}, 3, false);
  if (p.epf_iters >= 1) epf_stage(std::integral_constant<int, 1>{}, 2, p.epf_iters == 1);
  if (p.epf_iters >= 2) epf_stage(std::integral_constant<int, 2>{}, 1, true);

  if (p.epf_iters == 0) {  // Gaborish (or nothing) followed by colour only
    const Rect r = clip(rect(0));
    for_region(r, [&](int lx, int ly) {
      float o[3];
#pragma unroll
      for (int c = 0; c < 3; ++c) o[c] = cur[c * kPlane + ly * kS + lx];
      if (p.colour) xyb_to_rgb_px(o, p.col, colour_tf(p.col), kSrgbPow);
      const int x = gx0 + lx, y = gy0 + ly;
#pragma unroll
      for (int c = 0; c < 3; ++c) v.out[c][size_t(y) * v.out_stride[c] + x] = o[c];
    });
  }
}


// Interior of the frame for the default filter chain (Gaborish, EPF steps 1 and 2, colour): kernels/filter_strip.cuh.
template <int ITERS, int TF>
__global__ void __launch_bounds__(fstrip::kThreads, 3)
strip_filter_kernel(FusedViews v, DevFusedFilterParams p, const __grid_constant__ FusedMaps maps, fstrip::StripRect r, float gw0,
                    float gw1, float gw2) {
  using namespace fstrip;
  extern __shared__ __align__(128) float s_buf[];
  __shared__ __align__(8) unsigned long long s_mbar;
  const int tid = int(threadIdx.x);
  const StripGeom g = strip_geom(v.width, v.height, r.x0, r.y0, r.x1, r.y1, int(blockIdx.x), int(blockIdx.y));
  const uint32_t mbar = smem_u32(&s_mbar);
  if (tid == 0) window_load_issue<kPlane>(mbar, s_buf, maps, g.gx0, g.gy0);
  phase_sigma(tid, s_buf, g, p);
  __syncthreads();  // the barrier is initialised before anybody polls it; sigma table complete
  window_load_wait(mbar);
  const float gw[3] = {gw0, gw1, gw2};
  phase_gab(tid, s_buf, p, gw);
  __syncthreads();
  phase_dist1(tid, s_buf, p);
  __syncthreads();
  if (ITERS == 1) {
    phase_apply1<true, TF>(tid, s_buf, g, p, v.out, v.out_stride);
  } else {
    phase_apply1<false, TF>(tid, s_buf, g, p, v.out, v.out_stride);
    __syncthreads();
    phase_apply2<TF>(tid, s_buf, g, p, v.out, v.out_stride);
  }
}

}  // namespace

bool fused_filters_supported(uint32_t width, uint32_t height) { return width >= 16 && height >= 16; }

namespace {
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn tensor_map_encoder() {
  static EncodeTiledFn fn = [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess)
      p = nullptr;
    return reinterpret_cast<EncodeTiledFn>(p);
  }();
  return fn;
}

// TMA descriptors of the three input planes for a box_w x box_h window (2-D, f32, out-of-bounds cells read as zero). False,
// with `maps` zeroed, when the driver has no encoder or a plane's base or row pitch is not 16-byte aligned.
bool encode_plane_maps(const FusedViews& v, int box_w, int box_h, FusedMaps& maps) {
  std::memset(&maps, 0, sizeof(maps));
  const EncodeTiledFn enc = tensor_map_encoder();
  if (!enc) return false;
  for (int c = 0; c < 3; ++c) {
    if ((reinterpret_cast<uintptr_t>(v.in[c]) & 15) != 0 || (size_t(v.in_stride[c]) * 4) % 16 != 0) return false;
    const cuuint64_t dims[2] = {cuuint64_t(v.width), cuuint64_t(v.height)};
    const cuuint64_t strides[1] = {cuuint64_t(v.in_stride[c]) * 4};
    const cuuint32_t box[2] = {cuuint32_t(box_w), cuuint32_t(box_h)};
    const cuuint32_t estr[2] = {1, 1};
    if (enc(&maps.map[c], CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(v.in[c]), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
      return false;
  }
  return true;
}
}  // namespace

void launch_filters_fused(const DevView in[3], const DevView out[3], DevFusedFilterParams p, cudaStream_t stream) {
  FusedViews v;
  for (int c = 0; c < 3; ++c) {
    v.in[c] = static_cast<const float*>(in[c].ptr);
    v.out[c] = static_cast<float*>(out[c].ptr);
    v.in_stride[c] = in[c].stride;
    v.out_stride[c] = out[c].stride;
  }
  v.width = int(in[0].w);
  v.height = int(in[0].h);
  if (!v.width || !v.height) return;
  const int nmaps = p.epf_iters == 3 ? 6 : (p.epf_iters > 0 ? 2 : 0);
  const int ks = window_size(nmaps);
  const size_t plane_bytes = size_t(ks) * ks * sizeof(float);
  FusedMaps maps;
  v.use_tma = encode_plane_maps(v, ks, ks, maps) ? 1 : 0;
  // C++ function-local statics are initialised once, thread-safely: no worker thread launches before the limits are set
  static const bool attr_set = [] {
    cudaFuncSetAttribute(fused_filter_kernel<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, 6 * window_size(0) * window_size(0) * 4);
    cudaFuncSetAttribute(fused_filter_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, 8 * window_size(2) * window_size(2) * 4);
    cudaFuncSetAttribute(fused_filter_kernel<6>, cudaFuncAttributeMaxDynamicSharedMemorySize, 12 * window_size(6) * window_size(6) * 4);
    cudaFuncSetAttribute(strip_filter_kernel<1, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, fstrip::kSmemFloats * 4);
    cudaFuncSetAttribute(strip_filter_kernel<1, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, fstrip::kSmemFloats * 4);
    cudaFuncSetAttribute(strip_filter_kernel<1, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, fstrip::kSmemFloats * 4);
    cudaFuncSetAttribute(strip_filter_kernel<2, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, fstrip::kSmemFloats * 4);
    cudaFuncSetAttribute(strip_filter_kernel<2, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, fstrip::kSmemFloats * 4);
    cudaFuncSetAttribute(strip_filter_kernel<2, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, fstrip::kSmemFloats * 4);
    return true;
  }();
  (void)attr_set;
  dim3 block(32, 8);
  dim3 grid((v.width + kT - 1) / kT, (v.height + kT - 1) / kT);
  v.border_only = 0, v.bx_last = v.by_last = 0, v.nbx = int(grid.x), v.nby = int(grid.y);

  // The default chains (Gaborish + EPF step 1, or steps 1 and 2) run the interior of the frame in the column-strip kernel and only the
  // tiles that touch the image border (mirroring, Gaborish edge formulas) in the general one.
  const fstrip::StripRect r = fstrip::strip_rect(v.width, v.height);
  // The strip kernel's window origins are 28 + 56 * tx and, for the pulled-back last column of tiles, width - 64: TMA wants the
  // box to start on a 16-byte boundary in the innermost dimension (cp.async.bulk.tensor with an origin of 325 floats ends in
  // "illegal instruction"), so frames whose width is not a multiple of four samples stay in the general kernel, whose origins
  // are multiples of four by construction.
  const bool origins_aligned = (v.width & 3) == 0;
  if (v.use_tma && origins_aligned && p.gab_enabled && (p.epf_iters == 1 || p.epf_iters == 2) && r.x1 > r.x0 && r.y1 > r.y0) {
    FusedMaps smaps;
    if (encode_plane_maps(v, fstrip::kWX, fstrip::kWY, smaps)) {
      float gw[3];
      fstrip::strip_gab_norm(p, gw);
      dim3 sgrid((r.x1 - r.x0 + fstrip::kTX - 1) / fstrip::kTX, (r.y1 - r.y0 + fstrip::kTY - 1) / fstrip::kTY);
      const int tf = fstrip::strip_tf_of(p);
      const size_t sm = fstrip::kSmemFloats * 4;
#define JXLB_STRIP_LAUNCH(I, T) strip_filter_kernel<I, T><<<sgrid, fstrip::kThreads, sm, stream>>>(v, p, smaps, r, gw[0], gw[1], gw[2])
      if (p.epf_iters == 1) {
        if (tf == 1) JXLB_STRIP_LAUNCH(1, 1);
        else if (tf == 2) JXLB_STRIP_LAUNCH(1, 2);
        else JXLB_STRIP_LAUNCH(1, 0);
      } else {
        if (tf == 1) JXLB_STRIP_LAUNCH(2, 1);
        else if (tf == 2) JXLB_STRIP_LAUNCH(2, 2);
        else JXLB_STRIP_LAUNCH(2, 0);
      }
#undef JXLB_STRIP_LAUNCH
      v.border_only = 1;
      v.bx_last = r.x1 / 32 - 1, v.by_last = r.y1 / 32 - 1;
      const int n_border = v.nbx * v.nby - v.bx_last * v.by_last;
      fused_filter_kernel<2><<<dim3(n_border), block, 8 * plane_bytes, stream>>>(v, p, maps);
      return;
    }
  }
  if (p.epf_iters == 3) fused_filter_kernel<6><<<grid, block, 12 * plane_bytes, stream>>>(v, p, maps);
  else if (p.epf_iters > 0) fused_filter_kernel<2><<<grid, block, 8 * plane_bytes, stream>>>(v, p, maps);
  else fused_filter_kernel<0><<<grid, block, 6 * plane_bytes, stream>>>(v, p, maps);
}

}  // namespace jxlb
