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
// host: tests/emu/ runs it stream by stream on real frames, through hf_lane_decode() at the end of this file, and
// compares the coefficients with the oracle (test infrastructure; the product only ever runs it on the device).
// Shared-memory tables are read through an accessor policy `Mem`: 32-bit shared-window addresses and LDS on the device
// (HfLds below), plain host addresses in the emulation (HfHostMem).
#pragma once
#include "kernels.h"
#include "stream_common.cuh"
#ifndef __CUDACC__
#include <cstring>
#include <vector>
#endif

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

#ifdef __CUDACC__
// Device accessor policy: 32-bit shared-window addresses, LDS / STS.
struct HfLds {
  using Addr = uint32_t;
  static __device__ __forceinline__ Addr addr(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }
  static __device__ __forceinline__ uint32_t u8(Addr a) {
    uint32_t v;
    asm("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
  }
  static __device__ __forceinline__ uint32_t u32(Addr a) {
    uint32_t v;
    asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
    return v;
  }
  static __device__ __forceinline__ uint2 u64(Addr a) {
    uint2 v;
    asm("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
    return v;
  }
  static __device__ __forceinline__ void st8(Addr a, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" ::"r"(a), "r"(v)); }
};
#endif

// LSB-first reader, 64-bit buffer + one word in flight, word-indexed. Unlike DevBitReader it never refills inside a
// read: the caller tops it up to >= 32 bits once per symbol (enough for the ANS 16-bit refill or a prefix-code peek) and
// once more before a hybrid-uint tail. Loads stop two words after the section, like DevBitReader's, so both readers
// see the same bits.
struct HfBits {
  const uint32_t* base;
  uint32_t widx, stop_idx;
  uint64_t buf;
  uint32_t ahead;
  int nbits;
  __device__ __forceinline__ void init(const uint8_t* d, uint64_t bit_pos, uint64_t bit_limit) {
    base = reinterpret_cast<const uint32_t*>(d);
    const uint32_t w = uint32_t(bit_pos >> 5), skip = uint32_t(bit_pos & 31);
    stop_idx = uint32_t((bit_limit + 31) >> 5) + 2;
    buf = uint64_t(__ldg(base + w)) >> skip;
    nbits = 32 - int(skip);
    buf |= uint64_t(__ldg(base + w + 1)) << nbits;
    nbits += 32;
    ahead = __ldg(base + w + 2);
    widx = w + 3;
  }
  __device__ __forceinline__ void refill() {  // nbits <= 32 -> nbits > 32
    buf |= uint64_t(ahead) << nbits;
    nbits += 32;
    ahead = widx <= stop_idx ? __ldg(base + widx) : 0u;
    ++widx;
  }
  __device__ __forceinline__ void top_up() {
    if (nbits < 32) refill();
  }
  __device__ __forceinline__ uint32_t take(uint32_t n) {  // n <= 32 bits that are known to be buffered
    const uint32_t v = uint32_t(buf) & (n >= 32 ? 0xffffffffu : ((1u << n) - 1));
    buf >>= n;
    nbits -= int(n);
    return v;
  }
  __device__ __forceinline__ uint64_t pos() const { return uint64_t(widx - 1) * 32 - uint64_t(nbits); }
  // pos() > 32 * (k - 1), without 64-bit arithmetic
  __device__ __forceinline__ bool past_word(uint32_t k) const { return widx > k + (uint32_t(nbits) >> 5); }
};

template <class Mem>
struct HfTables {  // addresses through `Mem` (ans: only when ANS_SMEM) + global fall-backs
  typename Mem::Addr cfg, ans;
  const uint64_t* ans_g;
  const uint32_t* prefix;
  const uint32_t* prefix_meta;
  uint32_t log_alphabet_size, log_bucket, use_prefix;
};

// One symbol of cluster `cl` -> hybrid-uint value. Requires >= 32 buffered bits on entry. PREFIX: the code may be a
// prefix code (decided by T.use_prefix at run time); without it the code is ANS. With TRACK, `*past` is set when a
// read of this symbol starts at a position past bit 32 * (past_k - 1) (HfBits::past_word).
template <class Mem, bool ANS_SMEM, bool PREFIX = true, bool TRACK = false>
__device__ __forceinline__ uint32_t hf_read_value(const HfTables<Mem>& T, HfBits& br, uint32_t& ans_state, uint32_t cl,
                                                  uint32_t past_k = 0, bool* past = nullptr) {
  const uint32_t cfg = Mem::u32(T.cfg + cl * 4);
  uint32_t token;
  if (PREFIX && T.use_prefix) {  // prefix.rs:335-357
    const uint32_t off = __ldg(T.prefix_meta + cl * 2), root_bits = __ldg(T.prefix_meta + cl * 2 + 1);
    const uint32_t peeked = uint32_t(br.buf) & 0x7fffu;
    uint32_t e = __ldg(T.prefix + off + (peeked & ((1u << root_bits) - 1)));
    if (e & 0x80000000u) {
      const uint32_t sb = (e >> 16) & 0xff;
      e = __ldg(T.prefix + off + (1u << root_bits) + (e & 0xffff) + ((peeked >> root_bits) & ((1u << sb) - 1)));
    }
    br.take((e >> 16) & 0xff);
    token = e & 0xffff;
  } else {  // ans.rs:276-330
    const uint32_t state = ans_state;
    const uint32_t idx = state & 0xfff;
    const uint32_t i = idx >> T.log_bucket;
    const uint32_t pos = idx & ((1u << T.log_bucket) - 1);
    uint2 b;
    if (ANS_SMEM) {
      b = Mem::u64(T.ans + (((cl << T.log_alphabet_size) + i) << 3));
    } else {
      const uint64_t g = __ldg(T.ans_g + ((size_t(cl) << T.log_alphabet_size) + i));
      b = make_uint2(uint32_t(g), uint32_t(g >> 32));
    }
    const bool map_to_alias = pos >= ((b.x >> 8) & 0xff);
    const uint32_t hi = map_to_alias ? b.y : 0u;
    const uint32_t offset = (hi & 0xffff) + pos;
    const uint32_t dist = (b.x >> 16) ^ (hi >> 16);
    token = map_to_alias ? (b.x & 0xff) : i;
    uint32_t next = (state >> 12) * dist + offset;
    if (next < (1u << 16)) {
      if (TRACK) *past |= br.past_word(past_k);
      next = (next << 16) | br.take(16);
    }
    ans_state = next;
  }
  // hybrid uint (lib.rs:572-605)
  const uint32_t split_exponent = cfg & 0xff;
  const uint32_t split = 1u << split_exponent;
  if (token < split) return token;
  const uint32_t msb = (cfg >> 8) & 0xff, lsb = (cfg >> 16) & 0xff;
  const uint32_t in_token = msb + lsb;
  const uint32_t n = (split_exponent - in_token + ((token - split) >> in_token)) & 31;
  if (TRACK) *past |= br.past_word(past_k);
  br.top_up();
  const uint32_t rest = br.take(n);
  const uint32_t low = token & ((1u << lsb) - 1);
  uint32_t t = (token >> lsb) & ((1u << msb) - 1);
  t |= 1u << msb;
  return uint32_t((((uint64_t(t) << n) | rest) << lsb) | low);
}

// Shared-memory layout of a thread-per-stream CTA of `nthreads` streams: context LUTs, transform-type info and order
// offsets, hybrid-uint configs, block-context map, the cluster maps of every HF preset (unless they exceed
// kLaneCmapSmemBytes), 96 bytes of non-zero-count row per stream and the ANS alias tables (up to kHfAnsSmemBytes).
struct HfLaneSmem {
  uint32_t ctxlut, small, configs, bctx, cmap, cmap_stride, nz, ans, total;
};
__host__ __device__ inline HfLaneSmem hf_lane_layout(const DevHfParams& p, uint32_t nthreads) {
  HfLaneSmem L;
  uint32_t off = 0;
  auto take = [&](uint32_t bytes) {
    uint32_t o = off;
    off += (bytes + 15) & ~15u;
    return o;
  };
  L.ctxlut = take(128);
  L.small = take((27 + 39) * 4);
  L.configs = take(p.code.num_clusters * 4);
  L.bctx = take(p.block_ctx_map_size);
  L.cmap_stride = 495 * p.num_block_clusters;
  const uint32_t cmap_bytes = L.cmap_stride * p.num_hf_presets;
  L.cmap = cmap_bytes <= kLaneCmapSmemBytes ? take(cmap_bytes) : 0xffffffffu;
  L.nz = take(96 * nthreads);
  uint32_t ab = p.code.use_prefix ? 0 : (p.code.num_clusters << p.code.log_alphabet_size) * 8;
  L.ans = (!p.code.use_prefix && ab <= kHfAnsSmemBytes) ? take(ab) : 0xffffffffu;
  L.total = off;
  return L;
}
// The staged variant of hf_lane_decode: an ANS code whose alias tables and cluster maps are both in shared memory.
__host__ __device__ inline bool hf_lane_staged(const DevHfParams& p, const HfLaneSmem& L) {
  return !p.code.use_prefix && L.ans != 0xffffffffu && L.cmap != 0xffffffffu;
}

// Tables one CTA shares, read through `Mem`. Always in shared memory: tinfo, order_offset, ctx, cfg, bctx, nz. The staged variant reads
// the cluster maps and ANS tables through `code` / `cmap`; the general one through `cv` / `cmap_ptr`, which may point
// to global memory.
template <class Mem>
struct HfLaneView {
  using Addr = typename Mem::Addr;
  // Lanes index these with their own block's transform type / channel: from constant memory (kTInfo, the kernel
  // parameter bank) such a lookup costs one replay per distinct address, from shared memory it is one access.
  Addr tinfo;         // [27] hf_pack_tinfo(): width | log2(blocks) << 8 | order id << 16 | transposed << 24
  Addr order_offset;  // [13 * 3] copy of DevHfParams::order_offset
  Addr ctx;           // [0..63): coefficient frequency context, [64..127): non-zero-count context
  Addr bctx;          // block context map
  // Per-stream scratch: predicted non-zero counts of the row above, 3 channels x 32 block columns, one byte each (a
  // count is at most 63) at `nz + (c * 32 + x) * nz_stride`: on the device the lanes of a CTA interleave
  // (nz_stride = blockDim.x) so that a warp's accesses to one (c, x) fall into consecutive bytes.
  Addr nz;
  uint32_t nz_stride;
  Addr cmap;               // staged variant: cluster maps of all HF presets, `cmap_stride` bytes apart
  HfTables<Mem> code;      // staged variant: configs and ANS tables
  const uint8_t* cmap_ptr;  // general variant
  CodeView cv;              // general variant
  uint32_t cmap_stride;
};

__device__ __forceinline__ uint32_t hf_umin(uint32_t a, uint32_t b) { return a < b ? a : b; }
// One transform type's record in `tinfo`: width in blocks | log2(number of blocks) << 8 | order id << 16 | transposed << 24.
// The block count is stored as its logarithm (every varblock is a power of two of 8x8 blocks): DCT256 covers 1024 blocks,
// which does not fit a byte.
__device__ __forceinline__ uint32_t hf_pack_tinfo(uint32_t t) {
  const uint32_t blocks_log = 31u - uint32_t(__clz(int(uint32_t(kTInfo[t][0]) * kTInfo[t][1])));
  return uint32_t(kTInfo[t][0]) | blocks_log << 8 | uint32_t(kTInfo[t][3]) << 16 | uint32_t(kTInfo[t][4]) << 24;
}
struct HfTinfo {
  uint32_t w8, num_blocks_log, order_id, transpose;
};
__device__ __forceinline__ HfTinfo hf_unpack_tinfo(uint32_t ti) {
  return HfTinfo{ti & 0xff, (ti >> 8) & 0xff, (ti >> 16) & 0xff, ti >> 24};
}

// Block context of one 8x8 cell (hf_coeff.rs:100-127): everything a stream needs to know about a varblock before its
// first symbol -- transform type and the block's context offset `hf_idx * lf_idx_mul + lf_idx` from the quantised LF
// values and the HF multiplier -- packed as `type | offset << 8`; kHfNoBlock for cells that are not a varblock's
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

// Varblock list of a group: the group's varblock origins in raster order (row by row, left to right), one record each
// -- {type | context offset << 8 (hf_block_ctx_cell), x | y << 16 within the group} -- at a fixed stride of
// group_dim_blocks^2 records per group, with a count per group (hf_block_list_kernel on the device, the emulation's
// serial loop on the host). `i` is the cell's raster index within the group.
struct HfGroupRect {
  uint32_t bx0, by0, width, height;
};
__device__ __forceinline__ HfGroupRect hf_group_rect(const DevFrame& f, const DevHfParams& p, uint32_t group_idx) {
  const uint32_t gb = p.group_dim_blocks;
  HfGroupRect r;
  r.bx0 = group_idx % p.groups_per_row * gb;
  r.by0 = group_idx / p.groups_per_row * gb;
  r.width = hf_umin(gb, f.bw - r.bx0);
  r.height = hf_umin(gb, f.bh - r.by0);
  return r;
}
__device__ __forceinline__ uint2 hf_block_rec(uint32_t info, uint32_t x, uint32_t y) { return make_uint2(info, x | y << 16); }
template <bool SUB>
__device__ __forceinline__ bool hf_block_record(const DevFrame& f, const DevHfParams& p, const HfGroupRect& r, uint32_t i,
                                                uint2& rec) {
  const uint32_t x = i % r.width, y = i / r.width;
  const uint32_t info = hf_block_ctx_cell<SUB>(f, p, r.bx0 + x, r.by0 + y);
  rec = hf_block_rec(info, x, y);
  return info != kHfNoBlock;
}

// One stream. STAGED (hf_lane_staged): every table access goes through `Mem`, the bit reader is topped up once per
// trip and the symbol path has no prefix-code or global-table branch; otherwise the general reader and tables.
// `list` / `count`: this stream's group's varblock records.
template <bool SUB, bool STAGED, class Mem>
__device__ __forceinline__ void hf_lane_stream(const uint8_t* __restrict__ cs, const DevFrame& f, const DevHfParams& p,
                                               const HfLaneView<Mem>& T, const uint2* __restrict__ list, uint32_t count,
                                               const DevHfJob& job, int first_pass, uint64_t* end_bit, int* status) {
  using Addr = typename Mem::Addr;
  DevBitReader br;  // general variant
  HfBits hb;        // staged variant
  int err = kDevOk;
  uint32_t hfp_bits = 0;
  while ((1u << hfp_bits) < p.num_hf_presets) ++hfp_bits;
  uint32_t hfp, ans_state;
  // Hard stop for corrupt streams: once the reader has started a read more than two words past the section's last
  // word, the stream has certainly consumed bits beyond `bit_limit`. (The per-channel pos() check below reports the
  // same error, only later.) The general reader tracks this through its look-ahead pointer, which is never more than
  // 3 words past the position where its last read started; the staged variant tests those positions directly.
  const uint32_t last_word = uint32_t((job.bit_limit + 31) >> 5);
  const uint32_t* stop_word = nullptr;
  bool past = false;
  if (STAGED) {
    hb.init(cs, job.bit_pos, job.bit_limit);
    hfp = hb.take(hfp_bits);
    hb.top_up();
    ans_state = hb.take(32);
    past = (job.bit_pos >> 5) > last_word + 1 || job.bit_pos + hfp_bits > uint64_t(last_word + 2) * 32;
  } else {
    br.init(cs, job.bit_pos, job.bit_limit);
    hfp = br.read(hfp_bits);
    ans_state = p.code.use_prefix ? 0x130000u : br.read(32);
    stop_word = br.origin + last_word + 4;
  }
  if (hfp >= p.num_hf_presets) {
    err = kDevInvalid;
    hfp = 0;
  }
  const uint32_t nbc = p.num_block_clusters;
  const Addr a_cmap = T.cmap + T.cmap_stride * hfp;  // staged variant
  const uint8_t* cluster_map = STAGED ? nullptr : T.cmap_ptr + size_t(T.cmap_stride) * hfp;
  const uint32_t lf_idx_mul = (p.num_lf_thr[0] + 1) * (p.num_lf_thr[1] + 1) * (p.num_lf_thr[2] + 1);
  const uint32_t hf_idx_mul = p.num_qf_thr + 1;

  const HfGroupRect r = hf_group_rect(f, p, job.group_idx);
  const uint32_t bx0 = r.bx0, by0 = r.by0;
  for (uint32_t i = 0; i < 96; ++i) Mem::st8(T.nz + i * T.nz_stride, 0);

  // ---- block cursor: the current record and the next one, loaded a block ahead ----
  uint32_t x = 0, y = 0;  // the varblock being decoded (its top-left cell)
  uint32_t ci = 3;        // next channel slot of that block (Y, X, B); 3: move to the next record
  uint32_t w8 = 1, num_blocks = 1, num_blocks_log = 0, order_id = 0, transpose = 0, blk_ctx_idx = 0;
  uint32_t left = count;  // records not yet taken
  uint2 next = count ? __ldg(list) : make_uint2(0, 0);
  ++list;
  // ---- coefficient cursor (valid while in_coeffs) ----
  bool in_coeffs = false;
  uint32_t k = 0, size = 0, non_zeros = 0, prev_nonzero = 0, nzc_ctx = 0, block_ctx = 0;
  int c = 0;
  uint32_t sx = 0;
  Addr a_blk = a_cmap;                    // staged variant
  const uint8_t* cmap = cluster_map;      // general variant
  const uint32_t* order = p.orders;
  uint32_t* dst_base = f.coeff[0];

  while (err == kDevOk) {
    uint32_t cl;
    if (!in_coeffs) {
      // Move to the next (block, channel) that carries a non-zero count.
      bool found = false;
      while (!found) {
        if (ci >= 3) {
          if (left == 0) break;  // end of the group
          const uint2 rec = next;
          if (--left) next = __ldg(list++);
          x = rec.y & 0xffff;
          y = rec.y >> 16;
          const HfTinfo ti = hf_unpack_tinfo(Mem::u32(T.tinfo + (rec.x & 0xff) * 4));
          w8 = ti.w8;
          num_blocks_log = ti.num_blocks_log;
          num_blocks = 1u << num_blocks_log;
          order_id = ti.order_id;
          transpose = ti.transpose;
          blk_ctx_idx = rec.x >> 8;
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
        block_ctx = Mem::u8(T.bctx + idx);
        const uint32_t nz_here = Mem::u8(T.nz + (uint32_t(c) * 32 + sx) * T.nz_stride);
        const uint32_t nz_left = sx ? Mem::u8(T.nz + (uint32_t(c) * 32 + sx - 1) * T.nz_stride) : 0;
        uint32_t predicted;
        if (sy == 0) predicted = sx == 0 ? 32 : nz_left;
        else if (sx == 0) predicted = nz_here;
        else predicted = (nz_here + nz_left + 1) >> 1;
        const uint32_t pidx = predicted >= 8 ? 4 + predicted / 2 : predicted;
        cl = STAGED ? Mem::u8(a_cmap + block_ctx + pidx * nbc) : cluster_map[block_ctx + pidx * nbc];
        dst_base = f.coeff[c] + (size_t(sby0 + sy) * 8) * f.cw + size_t(sbx0 + sx) * 8;
        found = true;
      }
      if (!found) break;  // end of the group, or an error
    } else {
      const uint32_t cctx = (nzc_ctx + Mem::u8(T.ctx + ((k - num_blocks) >> num_blocks_log))) * 2 + prev_nonzero;
      if (cctx >= 458) {
        err = kDevInvalid;
        break;
      }
      cl = STAGED ? Mem::u8(a_blk + cctx) : cmap[cctx];
    }

    // ---- the part every lane executes together: one entropy-coded integer ----
    JXLB_LANE_TRIP(in_coeffs);
    uint32_t value;
    if (STAGED) {
      hb.top_up();
      value = hf_read_value<Mem, true, false, true>(T.code, hb, ans_state, cl, last_word + 3, &past);
    } else {
      value = cv_read_uint(br, Mem::u32(T.code.cfg + cl * 4), cv_read_symbol(T.cv, ans_state, br, cl));
      past = br.next_word > stop_word;
    }
    if (past) {
      err = kDevOverrun;
      break;
    }

    if (!in_coeffs) {
      if (value > (63u << num_blocks_log)) {
        err = kDevInvalid;
        break;
      }
      const uint32_t nz_val = (value + num_blocks - 1) >> num_blocks_log;
      for (uint32_t dx = 0; dx < w8; ++dx) Mem::st8(T.nz + (uint32_t(c) * 32 + sx + dx) * T.nz_stride, nz_val);
      if (value == 0) continue;
      non_zeros = value;
      prev_nonzero = (non_zeros <= num_blocks * 4) ? 1 : 0;
      order = p.orders + Mem::u32(T.order_offset + (order_id * 3 + c) * 4);
      size = num_blocks * 64;
      if (STAGED) a_blk = a_cmap + block_ctx * 458 + 37 * nbc;
      else cmap = cluster_map + block_ctx * 458 + 37 * nbc;
      nzc_ctx = Mem::u8(T.ctx + 64 + ((non_zeros - 1) >> num_blocks_log));
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
        else nzc_ctx = Mem::u8(T.ctx + 64 + ((non_zeros - 1) >> num_blocks_log));
      }
      if (!channel_done && ++k >= size) channel_done = true;
      if (channel_done) {
        in_coeffs = false;
        if ((STAGED ? hb.pos() : br.pos()) > job.bit_limit) err = kDevOverrun;
      }
    }
  }
  const uint64_t end = STAGED ? hb.pos() : br.pos();
  if (err == kDevOk && !p.code.use_prefix && ans_state != 0x130000u) err = kDevBadStream;
  if (err == kDevOk && end > job.bit_limit) err = kDevOverrun;
  *end_bit = end;
  *status = err;
}

#ifndef __CUDACC__
// ---- host emulation (tests/emu/) ----
// Host accessor policy: "shared memory" is plain host memory.
struct HfHostMem {
  using Addr = uintptr_t;
  static Addr addr(const void* p) { return reinterpret_cast<uintptr_t>(p); }
  static uint32_t u8(Addr a) { return *reinterpret_cast<const uint8_t*>(a); }
  static uint32_t u32(Addr a) {
    uint32_t v;
    std::memcpy(&v, reinterpret_cast<const void*>(a), 4);
    return v;
  }
  static uint2 u64(Addr a) {
    uint2 v;
    std::memcpy(&v, reinterpret_cast<const void*>(a), 8);
    return v;
  }
  static void st8(Addr a, uint32_t v) { *reinterpret_cast<uint8_t*>(a) = uint8_t(v); }
};

// One CTA's tables in host memory, as the emulation lays them out.
struct HfLaneTables {
  const uint32_t* tinfo;         // [27] hf_pack_tinfo()
  const uint32_t* order_offset;  // [13 * 3]
  const uint8_t* ctx;            // [0..63): coefficient frequency context, [64..127): non-zero-count context
  const uint32_t* cfg;           // packed HybridUintConfig per cluster
  const uint8_t* bctx;           // block context map
  const uint8_t* cmap;           // cluster maps of all HF presets, `cmap_stride` bytes apart
  uint32_t cmap_stride;
  CodeView cv;
};

// One stream on the host: `blk_ctx` holds hf_block_ctx_cell() of every cell of the frame (bw x bh); the stream's group
// list is compacted from it in raster order, and the stream runs the variant the device launcher would pick for `p`.
template <bool SUB>
inline void hf_lane_decode(const uint8_t* cs, const DevFrame& f, const DevHfParams& p, const HfLaneTables& T,
                           const uint32_t* blk_ctx, const DevHfJob& job, uint8_t* nz, uint32_t nz_stride, int first_pass,
                           uint64_t* end_bit, int* status) {
  const HfGroupRect r = hf_group_rect(f, p, job.group_idx);
  std::vector<uint2> list;
  for (uint32_t y = 0; y < r.height; ++y)
    for (uint32_t x = 0; x < r.width; ++x) {
      const uint32_t info = blk_ctx[size_t(r.by0 + y) * f.bw + r.bx0 + x];
      if (info != kHfNoBlock) list.push_back(hf_block_rec(info, x, y));
    }
  HfLaneView<HfHostMem> V;
  V.tinfo = HfHostMem::addr(T.tinfo);
  V.order_offset = HfHostMem::addr(T.order_offset);
  V.ctx = HfHostMem::addr(T.ctx);
  V.bctx = HfHostMem::addr(T.bctx);
  V.nz = HfHostMem::addr(nz);
  V.nz_stride = nz_stride;
  V.cmap = HfHostMem::addr(T.cmap);
  V.cmap_ptr = T.cmap;
  V.cmap_stride = T.cmap_stride;
  V.code.cfg = HfHostMem::addr(T.cfg);
  V.code.ans = HfHostMem::addr(T.cv.ans);
  V.code.ans_g = T.cv.ans;
  V.code.prefix = T.cv.prefix;
  V.code.prefix_meta = T.cv.prefix_meta;
  V.code.log_alphabet_size = T.cv.log_alphabet_size;
  V.code.log_bucket = 12 - T.cv.log_alphabet_size;
  V.code.use_prefix = T.cv.use_prefix;
  V.cv = T.cv;
  const uint2* recs = list.data();
  const uint32_t n = uint32_t(list.size());
  if (hf_lane_staged(p, hf_lane_layout(p, nz_stride)))
    hf_lane_stream<SUB, true>(cs, f, p, V, recs, n, job, first_pass, end_bit, status);
  else
    hf_lane_stream<SUB, false>(cs, f, p, V, recs, n, job, first_pass, end_bit, status);
}
#endif

}  // namespace
}  // namespace jxlb
