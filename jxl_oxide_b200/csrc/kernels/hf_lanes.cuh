// HF coefficient decode, one *thread* per stream (jxl-vardct/src/hf_coeff.rs:21-252).
//
// decode_hf_warp_kernel (entropy.cu) walks every stream from a single lane of its warp; with 510 streams
// per 8K frame and 24 frames in flight the SM schedulers saturate on one-lane warps (DESIGN.md section 4).
// Here a warp carries 32 independent streams. The chain of one stream is written as a flat state machine --
// every trip of the loop decodes exactly one symbol (a block's non-zero count or one coefficient) -- so the
// lanes of a warp re-converge on the expensive part (alias-table ANS step + hybrid-uint read) no matter
// where in their groups they are; only the short bookkeeping before / after the symbol diverges.
//
// The per-stream code below is plain integer C++ with no cross-lane traffic, so it also compiles for the
// host: tests/emu/ runs it stream by stream on real frames and compares the coefficients with the oracle
// (test infrastructure; the product only ever runs it on the device).
#pragma once
#include "kernels.h"
#include "stream_common.cuh"

// Hook for the host emulation's SIMT model (tests/emu: which kind of symbol each loop trip decodes); nothing on the device.
#ifndef JXLB_LANE_TRIP
#define JXLB_LANE_TRIP(is_coefficient)
#endif

namespace jxlb {
namespace {

#define JXLB_TABLE_QUAL __device__ __constant__ const
namespace hftab {
#include "../host/jxl_tables.inc"
}
#undef JXLB_TABLE_QUAL

// per transform type: width / height in 8x8 blocks, dequant set, coefficient order id, transposed
__device__ __constant__ const uint8_t kTInfo[27][5] = {
    {1, 1, 0, 0, 1},  {1, 1, 1, 1, 0},  {1, 1, 2, 1, 0},   {1, 1, 3, 1, 0},    {2, 2, 4, 2, 1},   {4, 4, 5, 3, 1},
    {1, 2, 6, 4, 1},  {2, 1, 6, 4, 0},  {1, 4, 7, 5, 1},   {4, 1, 7, 5, 0},    {2, 4, 8, 6, 1},   {4, 2, 8, 6, 0},
    {1, 1, 9, 1, 0},  {1, 1, 9, 1, 0},  {1, 1, 10, 1, 0},  {1, 1, 10, 1, 0},   {1, 1, 10, 1, 0},  {1, 1, 10, 1, 0},
    {8, 8, 11, 7, 1}, {4, 8, 12, 8, 1}, {8, 4, 12, 8, 0},  {16, 16, 13, 9, 1}, {8, 16, 14, 10, 1}, {16, 8, 14, 10, 0},
    {32, 32, 15, 11, 1}, {16, 32, 16, 12, 1}, {32, 16, 16, 12, 0},
};

// Tables one CTA shares (shared memory on the device, plain host memory under emulation).
struct HfLaneTables {
  // Lanes index these with their own block's transform type / channel: from constant memory (kTInfo, the kernel
  // parameter bank) such a lookup costs one replay per distinct address, from shared memory it is one access.
  const uint32_t* tinfo;         // [27] hf_pack_tinfo(): width | blocks << 8 | order id << 16 | transposed << 24
  const uint32_t* order_offset;  // [13 * 3] copy of DevHfParams::order_offset
  const uint8_t* ctx;        // [0..63): coefficient frequency context, [64..127): non-zero-count context
  const uint32_t* cfg;       // packed HybridUintConfig per cluster
  const uint8_t* bctx;       // block context map
  const uint8_t* cmap;       // cluster maps of all HF presets, `cmap_stride` bytes apart
  uint32_t cmap_stride;
  CodeView cv;
};

// Per-stream scratch: predicted non-zero counts of the row above, 3 channels x 32 block columns, one byte
// each (a count is at most 63). `nz[(c * 32 + x) * nz_stride]`: on the device the lanes of a CTA interleave
// (nz_stride = blockDim.x) so that a warp's accesses to one (c, x) fall into consecutive bytes.
__device__ __forceinline__ uint32_t hf_umin(uint32_t a, uint32_t b) { return a < b ? a : b; }
__device__ __forceinline__ uint32_t hf_pack_tinfo(uint32_t t) {
  return uint32_t(kTInfo[t][0]) | (uint32_t(kTInfo[t][0]) * kTInfo[t][1]) << 8 | uint32_t(kTInfo[t][3]) << 16 |
         uint32_t(kTInfo[t][4]) << 24;
}

// Pre-pass, one thread per 8x8 cell (hf_coeff.rs:100-127): everything a stream needs to know about a varblock before
// its first symbol -- transform type and the block's context offset `hf_idx * lf_idx_mul + lf_idx` from the quantised
// LF values and the HF multiplier -- packed as `type | offset << 8`; 0xffffffff for cells that are not a varblock's
// top-left corner. Keeps the threshold loops and five dependent loads out of the streams' serial walk.
constexpr uint32_t kHfNoBlock = 0xffffffffu;
template <bool SUB>
__device__ __forceinline__ uint32_t hf_block_ctx_cell(const DevFrame& f, const DevHfParams& p, uint32_t bx, uint32_t by) {
  const size_t gi = size_t(by) * f.bw + bx;
  const int32_t t = f.blk_type[gi];
  if (t < 0) return kHfNoBlock;
  const int32_t qf = f.blk_mul[gi];
  const int32_t* thr = p.lf_thresholds;
  uint32_t lf_idx = 0;
  if (p.has_lf_quant) {
    const int32_t* thr_base[3] = {thr, thr + p.num_lf_thr[0], thr + p.num_lf_thr[0] + p.num_lf_thr[1]};
    for (int kk = 0; kk < 3; ++kk) {
      const int cc = kk == 0 ? 0 : (kk == 1 ? 2 : 1);
      lf_idx *= p.num_lf_thr[cc] + 1;
      if (p.num_lf_thr[cc]) {
        const int32_t q = SUB ? f.lf_quant[cc][size_t(by >> f.vshift[cc]) * f.bw + (bx >> f.hshift[cc])] : f.lf_quant[cc][gi];
#pragma unroll 1
        for (uint32_t i = 0; i < p.num_lf_thr[cc]; ++i)
          if (q > thr_base[cc][i]) ++lf_idx;
      }
    }
  }
  uint32_t hf_idx = 0;
#pragma unroll 1
  for (uint32_t i = 0; i < p.num_qf_thr; ++i)
    if (qf > int32_t(p.qf_thresholds[i])) ++hf_idx;
  const uint32_t lf_idx_mul = (p.num_lf_thr[0] + 1) * (p.num_lf_thr[1] + 1) * (p.num_lf_thr[2] + 1);
  return uint32_t(t) | (hf_idx * lf_idx_mul + lf_idx) << 8;
}

template <bool SUB>
__device__ __forceinline__ void hf_lane_decode(const uint8_t* __restrict__ cs, const DevFrame& f, const DevHfParams& p,
                                               const HfLaneTables& T, const uint32_t* __restrict__ blk_ctx,
                                               const DevHfJob& job, uint8_t* nz, uint32_t nz_stride, int first_pass,
                                               uint64_t* end_bit, int* status) {
  DevBitReader br;
  int err = kDevOk;
  br.init(cs, job.bit_pos, job.bit_limit);
  uint32_t hfp_bits = 0;
  while ((1u << hfp_bits) < p.num_hf_presets) ++hfp_bits;
  uint32_t hfp = br.read(hfp_bits);
  if (hfp >= p.num_hf_presets) {
    err = kDevInvalid;
    hfp = 0;
  }
  const uint32_t nbc = p.num_block_clusters;
  const uint8_t* cluster_map = T.cmap + size_t(T.cmap_stride) * hfp;
  const uint32_t lf_idx_mul = (p.num_lf_thr[0] + 1) * (p.num_lf_thr[1] + 1) * (p.num_lf_thr[2] + 1);
  const uint32_t hf_idx_mul = p.num_qf_thr + 1;
  uint32_t ans_state = p.code.use_prefix ? 0x130000u : br.read(32);

  const uint32_t gx = job.group_idx % p.groups_per_row, gy = job.group_idx / p.groups_per_row;
  const uint32_t gb = p.group_dim_blocks;
  const uint32_t bx0 = gx * gb, by0 = gy * gb;
  const uint32_t width = hf_umin(gb, f.bw - bx0), height = hf_umin(gb, f.bh - by0);
  for (uint32_t i = 0; i < 96; ++i) nz[i * nz_stride] = 0;
  // Hard stop for corrupt streams: the reader's look-ahead pointer is never more than 3 words past the consumed
  // position, so once it is more than 4 words past the section's last word the stream has certainly consumed bits
  // beyond `bit_limit` (no false positives), and no load ever lands more than 32 bytes behind the section -- inside
  // the zero padding of the device copy. (The per-channel pos() check below reports the same error, only later.)
  const uint32_t* const stop_word = br.origin + ((job.bit_limit + 31) >> 5) + 4;

  // ---- block cursor ----
  uint32_t x = 0, y = 0;     // the varblock being decoded (its top-left cell)
  uint32_t ci = 3;           // next channel slot of that block (Y, X, B); 3: move to the next block
  uint32_t w8 = 1, num_blocks = 1, num_blocks_log = 0, order_id = 0, transpose = 0, blk_ctx_idx = 0;
  bool first_block = true;
  // ---- coefficient cursor (valid while in_coeffs) ----
  bool in_coeffs = false;
  uint32_t k = 0, size = 0, non_zeros = 0, prev_nonzero = 0, nzc_ctx = 0, block_ctx = 0;
  int c = 0;
  uint32_t sx = 0;
  const uint8_t* cmap = cluster_map;
  const uint32_t* order = p.orders;
  uint32_t* dst_base = f.coeff[0];

  while (err == kDevOk) {
    uint32_t cl;
    if (!in_coeffs) {
      // Walk to the next (block, channel) that carries a non-zero count.
      bool found = false, done = false;
      while (!found) {
        if (ci >= 3) {
          // next varblock origin in raster order
          if (first_block) first_block = false;
          else ++x;
          uint32_t info = kHfNoBlock;
          for (;;) {
            if (x >= width) {
              x = 0;
              ++y;
            }
            if (y >= height) {
              done = true;
              break;
            }
            info = __ldg(blk_ctx + size_t(by0 + y) * f.bw + bx0 + x);
            if (info != kHfNoBlock) break;
            ++x;
          }
          if (done) break;
          const uint32_t ti = T.tinfo[info & 0xff];
          w8 = ti & 0xff;
          num_blocks = (ti >> 8) & 0xff;
          order_id = (ti >> 16) & 0xff;
          transpose = ti >> 24;
          num_blocks_log = 31u - uint32_t(__clz(int(num_blocks)));
          blk_ctx_idx = info >> 8;
          ci = 0;
        }
        // channel slot ci of the current block
        const uint32_t slot = ci++;
        c = slot == 0 ? 1 : (slot == 1 ? 0 : 2);
        sx = x;
        uint32_t sy = y, sbx0 = bx0, sby0 = by0;
        if (SUB) {  // hf_coeff.rs:143-155: only blocks aligned to the channel's grid, at the shifted position
          const uint32_t hs = f.hshift[c], vs = f.vshift[c];
          sx = x >> hs, sy = y >> vs, sbx0 = bx0 >> hs, sby0 = by0 >> vs;
          if (hs | vs) {
            if ((sx << hs) != x || (sy << vs) != y) continue;
            if (f.blk_type[size_t(by0 + sy) * f.bw + bx0 + sx] < 0) continue;
            if (num_blocks != 1) {
              err = kDevUnsupported;
              break;
            }
          }
        }
        const uint32_t idx = ((slot * 13 + order_id) * hf_idx_mul) * lf_idx_mul + blk_ctx_idx;
        block_ctx = T.bctx[idx];
        const uint32_t nz_here = nz[(uint32_t(c) * 32 + sx) * nz_stride];
        const uint32_t nz_left = sx ? nz[(uint32_t(c) * 32 + sx - 1) * nz_stride] : 0;
        uint32_t predicted;
        if (sy == 0) predicted = sx == 0 ? 32 : nz_left;
        else if (sx == 0) predicted = nz_here;
        else predicted = (nz_here + nz_left + 1) >> 1;
        const uint32_t pidx = predicted >= 8 ? 4 + predicted / 2 : predicted;
        cl = cluster_map[block_ctx + pidx * nbc];
        dst_base = f.coeff[c] + (size_t(sby0 + sy) * 8) * f.cw + size_t(sbx0 + sx) * 8;
        found = true;
      }
      if (!found) break;  // end of the group, or an error
    } else {
      const uint32_t cctx = (nzc_ctx + uint32_t(T.ctx[(k - num_blocks) >> num_blocks_log])) * 2 + prev_nonzero;
      if (cctx >= 458) {
        err = kDevInvalid;
        break;
      }
      cl = cmap[cctx];
    }

    // ---- the part every lane executes together: one entropy-coded integer ----
    JXLB_LANE_TRIP(in_coeffs);
    const uint32_t value = cv_read_uint(br, T.cfg[cl], cv_read_symbol(T.cv, ans_state, br, cl));
    if (br.next_word > stop_word) {
      err = kDevOverrun;
      break;
    }

    if (!in_coeffs) {
      if (value > (63u << num_blocks_log)) {
        err = kDevInvalid;
        break;
      }
      const uint32_t nz_val = (value + num_blocks - 1) >> num_blocks_log;
      for (uint32_t dx = 0; dx < w8; ++dx) nz[(uint32_t(c) * 32 + sx + dx) * nz_stride] = uint8_t(nz_val);
      if (value == 0) continue;
      non_zeros = value;
      prev_nonzero = (non_zeros <= num_blocks * 4) ? 1 : 0;
      order = p.orders + T.order_offset[order_id * 3 + c];
      size = num_blocks * 64;
      cmap = cluster_map + block_ctx * 458 + 37 * nbc;
      nzc_ctx = T.ctx[64 + ((non_zeros - 1) >> num_blocks_log)];
      k = num_blocks;
      in_coeffs = k < size;  // always true (size = 64 * num_blocks)
    } else {
      bool channel_done = false;
      if (value == 0) {
        prev_nonzero = 0;
      } else {
        // the coefficient's position feeds only the store, never the decode chain
        const uint32_t o = __ldg(order + k);
        const uint32_t cvv = uint32_t(dev_unpack_signed(value)) << p.coeff_shift;
        uint32_t dx = o & 0xffff, dy = o >> 16;
        if (transpose) {
          const uint32_t tmp = dx;
          dx = dy;
          dy = tmp;
        }
        uint32_t* dst = dst_base + size_t(dy) * f.cw + dx;
        if (first_pass) *dst = cvv;
        else *dst += cvv;
        prev_nonzero = 1;
        if (--non_zeros == 0) channel_done = true;
        else nzc_ctx = T.ctx[64 + ((non_zeros - 1) >> num_blocks_log)];
      }
      if (!channel_done && ++k >= size) channel_done = true;
      if (channel_done) {
        in_coeffs = false;
        if (br.pos() > job.bit_limit) err = kDevOverrun;
      }
    }
  }
  if (err == kDevOk && !p.code.use_prefix && ans_state != 0x130000u) err = kDevBadStream;
  if (err == kDevOk && br.pos() > job.bit_limit) err = kDevOverrun;
  *end_bit = br.pos();
  *status = err;
}

}  // namespace
}  // namespace jxlb
