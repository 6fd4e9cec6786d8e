// Varblock placement of one LF group (HfMetadata post-processing, jxl-vardct/src/hf_metadata.rs:99-230), one warp.
//
// The reference places the (dct_select, hf_mul) list serially: each varblock goes to the first free 8x8 cell in raster
// order. That scan is serial as written but not by nature. Placing a varblock only occupies cells at or after its own
// position in the current row, plus cells in later rows, so the varblocks that start in cell row y tile that row's free
// cells from left to right, in list order. The warp therefore fills one row at a time, 32 records per step:
//   * the inclusive prefix sum of the records' widths gives each record its free-cell rank in the row;
//   * record i starts at the rank-th set bit of the row's free mask, and it is valid iff its ranks are consecutive cells
//     (no occupied cell and no group edge inside), it does not cross a 32-cell boundary, and sel / hf_mul are in range;
//   * the row ends when the ranks reach the row's free count; the records' heights are ORed into the rows below.
// Varblocks never cross a 32-row boundary, so the occupancy of the current 32-row band is all that is kept (1 KiB).
// Every placed varblock is then expanded into blk_type / blk_mul / epf_sigma, all lanes over the step's cells.
//
// The result equals the serial scan's, including which record fails first: a record is examined only if the records
// before it were placed and a free cell is left for it; records after a full group are ignored.
//
// The per-lane steps are plain functions of (lane, shared state), run by a `Warp` policy that calls a step for every
// lane between two barriers (PlaceWarp below on the device; a loop over 32 lanes in tests/emu/placement_emu.cc). The
// code between steps is uniform: every lane computes the same values from shared state.
#pragma once
#include "kernels.h"

namespace jxlb {
namespace {

#ifdef __CUDACC__
struct PlaceWarp {
  uint32_t lane;
  template <class F>
  __device__ __forceinline__ void each(F f) const {
    __syncwarp();  // every lane is done reading what the step writes
    f(lane);
    __syncwarp();
  }
  __device__ __forceinline__ void or_shared(uint32_t* p, uint32_t v) const { atomicOr(p, v); }
};
#endif

__device__ __constant__ const uint8_t kPlaceBlkSize[27][2] = {
    {1, 1}, {1, 1}, {1, 1}, {1, 1}, {2, 2}, {4, 4}, {1, 2}, {2, 1}, {1, 4}, {4, 1}, {2, 4}, {4, 2}, {1, 1}, {1, 1},
    {1, 1}, {1, 1}, {1, 1}, {1, 1}, {8, 8}, {4, 8}, {8, 4}, {16, 16}, {8, 16}, {16, 8}, {32, 32}, {16, 32}, {32, 16}};

__device__ __forceinline__ uint32_t place_popc(uint32_t v) {
#ifdef __CUDA_ARCH__
  return uint32_t(__popc(v));
#else
  return uint32_t(__builtin_popcount(v));
#endif
}

// Bit index of the k-th (0-based) set bit of v; k < popc(v).
__device__ __forceinline__ uint32_t place_select32(uint32_t v, uint32_t k) {
  uint32_t pos = 0, c;
  c = place_popc(v & 0xffffu);
  if (k >= c) k -= c, v >>= 16, pos += 16;
  c = place_popc(v & 0xffu);
  if (k >= c) k -= c, v >>= 8, pos += 8;
  c = place_popc(v & 0xfu);
  if (k >= c) k -= c, v >>= 4, pos += 4;
  c = place_popc(v & 0x3u);
  if (k >= c) k -= c, v >>= 2, pos += 2;
  if (k >= (v & 1u)) pos += 1;
  return pos;
}

__device__ __forceinline__ float place_div(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
__device__ __forceinline__ float place_mul(float a, float b) {
#ifdef __CUDA_ARCH__
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}

struct PlaceShared {
  uint32_t occ[32][8];   // occupancy of the current 32-row band, row y at [y & 31]
  uint32_t free_w[8];    // free cells of the current row
  uint32_t w[32], h[32];      // this step's records: size in cells (1 x 1 for an invalid dct_select)
  int32_t sel[32], mul[32];   // dct_select, hf_mul
  uint32_t end_rank[32];      // free-cell rank after the record (row ranks consumed before the step included)
  uint32_t x[32];             // column the record starts at
  uint32_t state[32];         // 0: not in this row, 1: placed, 2: invalid
  uint32_t cells_end[32];     // inclusive prefix sum of w * h over the step's placed records
  uint32_t bad_sharpness;
};
static_assert(sizeof(PlaceShared) <= kPlaceSharedBytes, "kPlaceSharedBytes is what a Modular launch reserves for the placement");
constexpr uint32_t kPlaceInRow = 1, kPlaceBad = 2;

// Position of free-cell rank r of the row (r < the row's free count).
__device__ __forceinline__ uint32_t place_select_row(const PlaceShared& s, uint32_t words, uint32_t r) {
  for (uint32_t wi = 0; wi < words; ++wi) {
    const uint32_t c = place_popc(s.free_w[wi]);
    if (r < c) return wi * 32 + place_select32(s.free_w[wi], r);
    r -= c;
  }
  return 0xffffffffu;
}

// Step: lane loads record `base + lane` (n records in the step).
__device__ __forceinline__ void place_load(uint32_t lane, PlaceShared& s, const DevPlacement& p, uint32_t base, uint32_t n) {
  if (lane >= n) return;
  const int32_t sel = p.raw[base + lane];
  const int32_t mul = int32_t(uint32_t(p.raw[p.raw_stride + base + lane]) + 1u);
  s.sel[lane] = sel;
  s.mul[lane] = mul;
  const bool ok = sel >= 0 && sel < 27;
  s.w[lane] = ok ? kPlaceBlkSize[sel][0] : 1u;
  s.h[lane] = ok ? kPlaceBlkSize[sel][1] : 1u;
}

// Step: the lane's record's rank range in the row, and whether it is placed in this row and valid there.
__device__ __forceinline__ void place_rank(uint32_t lane, PlaceShared& s, const DevPlacement& p, uint32_t n, uint32_t y,
                                           uint32_t words, uint32_t consumed, uint32_t num_free) {
  if (lane >= n) return;
  uint32_t end = consumed;
  for (uint32_t i = 0; i <= lane; ++i) end += s.w[i];
  const uint32_t w = s.w[lane], h = s.h[lane], start = end - w;
  s.end_rank[lane] = end;
  if (start >= num_free) {  // starts in a later row
    s.state[lane] = 0;
    return;
  }
  const uint32_t x = place_select_row(s, words, start);
  s.x[lane] = x;
  const int32_t sel = s.sel[lane], mul = s.mul[lane];
  bool ok = sel >= 0 && sel < 27 && mul > 0 && mul < (1 << 24);
  ok = ok && (x & 31) + w <= 32 && (y & 31) + h <= 32 && x + w <= p.bw && y + h <= p.bh;
  // no occupied cell inside: the last rank is in the row and w - 1 cells to the right of the first
  ok = ok && end <= num_free && place_select_row(s, words, end - 1) == x + w - 1;
  s.state[lane] = ok ? kPlaceInRow : kPlaceBad;
}

// Step: a placed record marks the rows below it in the band.
template <class W>
__device__ __forceinline__ void place_mark(const W& warp, uint32_t lane, PlaceShared& s, uint32_t k, uint32_t y) {
  if (lane >= k) return;
  const uint32_t w = s.w[lane], x = s.x[lane];
  const uint32_t mask = (w >= 32 ? 0xffffffffu : ((1u << w) - 1)) << (x & 31);
  for (uint32_t dy = 1; dy < s.h[lane]; ++dy) warp.or_shared(&s.occ[(y + dy) & 31][x >> 5], mask);
}

// Step: cells t = lane, lane + 32, ... of the step's k placed records (cells_end filled).
__device__ __forceinline__ void place_expand(uint32_t lane, PlaceShared& s, const DevPlacement& p, uint32_t k, uint32_t y) {
  const uint32_t total = k ? s.cells_end[k - 1] : 0;
  for (uint32_t t = lane; t < total; t += 32) {
    uint32_t i = 0, hi = k - 1;  // the first record with cells_end > t
    while (i < hi) {
      const uint32_t mid = (i + hi) >> 1;
      if (s.cells_end[mid] > t) hi = mid;
      else i = mid + 1;
    }
    const uint32_t c = t - (i ? s.cells_end[i - 1] : 0);
    const uint32_t w = s.w[i];
    const uint32_t lw = w == 1 ? 0 : w == 2 ? 1 : w == 4 ? 2 : w == 8 ? 3 : w == 16 ? 4 : 5;
    const uint32_t dx = c & (w - 1), dy = c >> lw;
    const size_t gi = size_t(y + dy) * p.grid_stride + s.x[i] + dx;
    const int32_t mul = s.mul[i];
    p.blk_type[gi] = (dx == 0 && dy == 0) ? s.sel[i] : -int32_t(1 + dx + 32 * dy);
    p.blk_mul[gi] = mul;
    if (p.has_epf) {
      const int32_t sh = p.sharpness[gi];
      if (sh < 0 || sh >= 8) {
        s.bad_sharpness = 1;
        continue;
      }
      p.epf_sigma[gi] = place_mul(place_div(p.quant_mul_base, float(mul)), p.sharp_lut[sh]);
    }
  }
}

// The placement of one LF group. Returns kDevOk or kDevBadLayout (the same in every lane).
template <class W>
__device__ __forceinline__ int place_varblocks(const W& warp, PlaceShared& s, const DevPlacement& p) {
  const uint32_t words = (p.bw + 31) / 32;
  warp.each([&](uint32_t lane) {
    for (uint32_t i = lane; i < 32 * 8; i += 32) (&s.occ[0][0])[i] = 0;
    if (lane == 0) s.bad_sharpness = 0;
  });
  uint32_t data_idx = 0;
  for (uint32_t y = 0; y < p.bh; ++y) {
    warp.each([&](uint32_t lane) {
      if (lane < 8) {
        const uint32_t valid = lane + 1 < words ? 0xffffffffu : lane + 1 == words ? ((p.bw & 31) ? (1u << (p.bw & 31)) - 1 : 0xffffffffu) : 0u;
        s.free_w[lane] = ~s.occ[y & 31][lane] & valid;
      }
    });
    uint32_t num_free = 0;
    for (uint32_t wi = 0; wi < words; ++wi) num_free += place_popc(s.free_w[wi]);
    uint32_t consumed = 0;
    while (consumed < num_free) {
      if (data_idx >= p.nb_blocks) return kDevBadLayout;  // cells left but no varblock to put there
      const uint32_t n = min(32u, p.nb_blocks - data_idx);
      warp.each([&](uint32_t lane) { place_load(lane, s, p, data_idx, n); });
      warp.each([&](uint32_t lane) { place_rank(lane, s, p, n, y, words, consumed, num_free); });
      uint32_t k = 0;  // records placed in this step: the ones in this row, up to the first invalid one
      while (k < n && s.state[k] == kPlaceInRow) ++k;
      const bool bad = k < n && s.state[k] == kPlaceBad;
      warp.each([&](uint32_t lane) {
        if (lane < k) {
          uint32_t c = 0;
          for (uint32_t i = 0; i <= lane; ++i) c += s.w[i] * s.h[i];
          s.cells_end[lane] = c;
        }
        place_mark(warp, lane, s, k, y);
      });
      warp.each([&](uint32_t lane) { place_expand(lane, s, p, k, y); });
      if (bad) return kDevBadLayout;
      data_idx += k;
      consumed = s.end_rank[k - 1];
    }
    warp.each([&](uint32_t lane) {
      if (lane < 8) s.occ[y & 31][lane] = 0;  // the row is done: the ring slot becomes row y + 32
    });
  }
  return s.bad_sharpness ? kDevBadLayout : kDevOk;
}

}  // namespace
}  // namespace jxlb
