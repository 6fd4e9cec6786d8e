// Per-block work of the JPEG scan encoder (jxl-jbr/src/reconstruct/scan.rs:133-194, 408-530 and the integer
// chroma-from-luma of reconstruct.rs:316-393), written as plain functions of a block index so that the same code runs
// in the kernels of jpeg.cu and, compiled for the host, in tests/emu/jpeg_emu.cc.
//
// Planes are the decoder's full-frame planes: i32 coefficients (bw*8 x bh*8) and i32 quantised LF (bw x bh) per X/Y/B
// channel, a subsampled channel in the top-left part. Block (x, y) of a channel is at (8x, 8y) / (x, y), so the
// reference's group-local addressing (x & group mask within the group of the MCU) is the identity here.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define JPEG_HD __host__ __device__ __forceinline__
#else
#define JPEG_HD inline
#endif

namespace jxlb {

constexpr int kJpegMaxSlots = 16;  // blocks per MCU: up to 4 components x 2 x 2

// DCT8_NATURAL_ORDER (jxl-vardct/src/hf_pass.rs:123): zigzag index -> x | y << 3
struct JpegZigzag {
  uint8_t xy[64];
};

struct DevJpegScan {
  const int32_t* coeff[3];  // X, Y, B
  const int32_t* lfq[3];
  const int32_t* cfl[2];    // x_from_y, b_from_y
  uint32_t coeff_stride, lfq_stride, cfl_stride;
  int32_t quant_ratio[2][64];  // (1 << 11) * q_y / q_x, (1 << 11) * q_y / q_b
  uint32_t do_cfl;
  uint32_t w8;              // MCUs per row
  uint32_t restart_mcus;    // MCUs per restart interval (all of them without DRI)
  uint32_t blocks_per_mcu, num_blocks, num_intervals;
  uint32_t num_ezr;         // extra zero runs, sorted by block
  uint32_t num_comps;
  uint32_t comp_channel[4];    // X/Y/B plane of a scan component
  int32_t comp_dc_offset[4];
  uint32_t comp_hs[4], comp_vs[4];
  uint32_t comp_dc_table[4], comp_ac_table[4];  // 0-3 DC, 4-7 AC
  uint8_t slot_comp[kJpegMaxSlots], slot_dx[kJpegMaxSlots], slot_dy[kJpegMaxSlots];
  // previous block of the same component: slot in this MCU, or 0x80 | slot in the previous MCU
  uint8_t slot_prev[kJpegMaxSlots];
  uint64_t pad_avail_bits;  // padding bits in the jbrd box; 0 = none signalled (pad with 1s)
  uint64_t pad_base;        // padding bits consumed by earlier scans
  JpegZigzag zz;
};

enum : uint32_t { kJpegErrHuffman = 1u, kJpegErrPadding = 2u };

// A Huffman table entry: (length << 16) | code, code right-aligned; 0 = the symbol has no code.
JPEG_HD uint32_t jpeg_huff_entry(uint32_t len, uint32_t code) { return (len << 16) | code; }

JPEG_HD uint32_t jpeg_bitlen16(uint32_t v) {  // 16 - u16::leading_zeros
  uint32_t n = 0;
  while (v >> n) ++n;
  return n;
}

JPEG_HD int32_t jpeg_dc(const DevJpegScan& p, uint32_t c, uint32_t x, uint32_t y, int32_t off) {
  int32_t v = p.lfq[c][size_t(y) * p.lfq_stride + x] - off;
  v = v < -2047 ? -2047 : (v > 2047 ? 2047 : v);
  return v;
}

// Position of block `b` in its channel (block units) and its slot in the MCU.
JPEG_HD void jpeg_block_pos(const DevJpegScan& p, uint32_t b, uint32_t* mcu, uint32_t* slot, uint32_t* bx, uint32_t* by) {
  *mcu = b / p.blocks_per_mcu;
  *slot = b - *mcu * p.blocks_per_mcu;
  const uint32_t k = p.slot_comp[*slot];
  const uint32_t x8 = *mcu % p.w8, y8 = *mcu / p.w8;
  *bx = x8 * p.comp_hs[k] + p.slot_dx[*slot];
  *by = y8 * p.comp_vs[k] + p.slot_dy[*slot];
}

// The block's DC and its DC prediction (previous block of the component, 0 at the start of a restart interval).
JPEG_HD void jpeg_block_dc(const DevJpegScan& p, uint32_t b, int32_t* dc, int32_t* pred) {
  uint32_t mcu, slot, bx, by;
  jpeg_block_pos(p, b, &mcu, &slot, &bx, &by);
  const uint32_t k = p.slot_comp[slot];
  *dc = jpeg_dc(p, p.comp_channel[k], bx, by, p.comp_dc_offset[k]);
  const uint32_t prev = p.slot_prev[slot];
  *pred = 0;
  if (!(prev & 0x80)) {
    jpeg_block_pos(p, mcu * p.blocks_per_mcu + prev, &mcu, &slot, &bx, &by);
    *pred = jpeg_dc(p, p.comp_channel[k], bx, by, p.comp_dc_offset[k]);
  } else if (mcu % p.restart_mcus != 0) {
    jpeg_block_pos(p, (mcu - 1) * p.blocks_per_mcu + (prev & 0x7f), &mcu, &slot, &bx, &by);
    *pred = jpeg_dc(p, p.comp_channel[k], bx, by, p.comp_dc_offset[k]);
  }
}

// The 63 AC coefficients of block `b` in zigzag order, after the integer chroma-from-luma (reconstruct.rs:366-387).
JPEG_HD void jpeg_block_ac(const DevJpegScan& p, uint32_t b, int16_t ac[63]) {
  uint32_t mcu, slot, bx, by;
  jpeg_block_pos(p, b, &mcu, &slot, &bx, &by);
  const uint32_t c = p.comp_channel[p.slot_comp[slot]];
  const int32_t* base = p.coeff[c] + size_t(by) * 8 * p.coeff_stride + size_t(bx) * 8;
  const bool cfl = p.do_cfl && c != 1;
  const int32_t* ybase = p.coeff[1] + size_t(by) * 8 * p.coeff_stride + size_t(bx) * 8;
  const int32_t factor = cfl ? p.cfl[c >> 1][size_t(by / 8) * p.cfl_stride + bx / 8] : 0;
  const int32_t scale_factor = factor * (1 << 11) / 84;
  const int32_t* ratio = p.quant_ratio[c >> 1];
  for (int i = 1; i < 64; ++i) {
    const uint32_t x = p.zz.xy[i] & 7, y = p.zz.xy[i] >> 3;
    int32_t v = base[size_t(y) * p.coeff_stride + x];
    if (cfl) {
      const int32_t q_scale = (ratio[y + 8 * x] * scale_factor + 1024) >> 11;
      v += (ybase[size_t(y) * p.coeff_stride + x] * q_scale + 1024) >> 11;
    }
    ac[i - 1] = int16_t(v);
  }
}

// Extra zero runs signalled for block `b` (0 when none): the list is sorted by block, later entries win.
JPEG_HD uint32_t jpeg_block_ezr(const DevJpegScan& p, const uint32_t* ezr_block, const uint32_t* ezr_count, uint32_t b,
                                bool* present) {
  uint32_t lo = 0, hi = p.num_ezr;  // first entry > b
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (ezr_block[mid] <= b) lo = mid + 1;
    else hi = mid;
  }
  *present = lo > 0 && ezr_block[lo - 1] == b;
  return *present ? ezr_count[lo - 1] : 0;
}

// process_sequential (scan.rs:133-194) for one block: calls put(code, len) for every Huffman code and raw field in
// stream order (len <= 16). Returns false when a symbol has no code in its table.
template <class Put>
JPEG_HD bool jpeg_encode_block(const DevJpegScan& p, const uint32_t* huff, const uint32_t* ezr_block, const uint32_t* ezr_count,
                               uint32_t b, Put& put) {
  const uint32_t slot = b % p.blocks_per_mcu;
  const uint32_t k = p.slot_comp[slot];
  const uint32_t* dct = huff + 256 * p.comp_dc_table[k];
  const uint32_t* act = huff + 256 * p.comp_ac_table[k];
  int32_t dc, pred;
  jpeg_block_dc(p, b, &dc, &pred);
  const int16_t diff = int16_t(dc - pred);
  const uint32_t mag = uint32_t(diff < 0 ? -diff : diff);
  const uint32_t dlen = jpeg_bitlen16(mag);
  const uint32_t draw = uint32_t(diff < 0 ? -int32_t(mag) - 1 : int32_t(mag));
  uint32_t e = dct[dlen & 0xff];
  if (!e) return false;
  put(e & 0xffff, e >> 16);
  if (dlen) put(draw & ((1u << dlen) - 1), dlen);

  int16_t ac[63];
  jpeg_block_ac(p, b, ac);
  uint32_t run = 0;
  int last = -1;
  for (int i = 0; i < 63; ++i) {
    const int32_t v = ac[i];
    if (v == 0) {
      ++run;
      continue;
    }
    while (run >= 16) {
      e = act[0xf0];
      if (!e) return false;
      put(e & 0xffff, e >> 16);
      run -= 16;
    }
    const uint32_t m = v < 0 ? uint32_t(uint16_t(-v)) : uint32_t(v);
    const uint32_t len = jpeg_bitlen16(m);
    const uint32_t raw = v < 0 ? (~m & 0xffffu) : m;
    e = act[uint8_t((run << 4) | len)];
    if (!e) return false;
    put(e & 0xffff, e >> 16);
    put(raw & ((1u << len) - 1), len);
    run = 0;
    last = i;
  }
  int32_t num_zeros = 62 - last;
  bool has_ezr;
  const uint32_t ezr = jpeg_block_ezr(p, ezr_block, ezr_count, b, &has_ezr);
  if (has_ezr) {
    e = act[0xf0];
    if (!e) return false;
    for (uint32_t i = 0; i < ezr; ++i) put(e & 0xffff, e >> 16);
    num_zeros -= int32_t(ezr) * 16;
  }
  if (num_zeros > 0) {
    e = act[0];
    if (!e) return false;
    put(e & 0xffff, e >> 16);
  }
  return true;
}

struct JpegBitCounter {
  uint32_t bits = 0;
  JPEG_HD void operator()(uint32_t, uint32_t len) { bits += len; }
};

// MSB-first writer into a zeroed buffer of big-endian-ordered 32-bit words (bit 31 of word w is bit 32w of the scan).
// A block owns every word it fills completely except its first; that one and its last, partial word may be shared
// with the neighbouring blocks and are ORed in.
struct JpegBitWriter {
  uint32_t* words;
  uint64_t first_word, wi;
  uint32_t bo, cur;
  JPEG_HD JpegBitWriter(uint32_t* w, uint64_t bit) : words(w), first_word(bit >> 5), wi(bit >> 5), bo(uint32_t(bit & 31)), cur(0) {}
  JPEG_HD static void or_word(uint32_t* p, uint32_t v) {
#if defined(__CUDA_ARCH__)
    atomicOr(p, v);
#else
    *p |= v;
#endif
  }
  JPEG_HD void flush_full() {
    if (wi == first_word) or_word(words + wi, cur);
    else words[wi] = cur;
    ++wi;
    cur = 0;
    bo = 0;
  }
  JPEG_HD void operator()(uint32_t v, uint32_t n) {  // n <= 32
    if (!n) return;
    const uint32_t space = 32 - bo;
    if (n < space) {
      cur |= v << (space - n);
      bo += n;
    } else {
      const uint32_t rem = n - space;
      cur |= v >> rem;
      flush_full();
      if (rem) {
        cur = v << (32 - rem);
        bo = rem;
      }
    }
  }
  JPEG_HD void finish() {
    if (bo) or_word(words + wi, cur);
  }
};

// Padding bits of an interval (scan.rs:89-115): `n` bits of the jbrd padding stream from `offset`, read LSB first and
// written MSB first, or n 1-bits when the box has none.
JPEG_HD uint32_t jpeg_padding_value(const DevJpegScan& p, const uint8_t* pad, uint64_t offset, uint32_t n) {
  if (!p.pad_avail_bits) return (1u << n) - 1;
  uint32_t v = 0;
  for (uint32_t i = 0; i < n; ++i) {
    const uint64_t o = offset + i;
    v |= uint32_t((pad[o >> 3] >> (o & 7)) & 1) << i;
  }
  return v;
}

// Byte i of the unstuffed scan (big-endian word order).
JPEG_HD uint8_t jpeg_scan_byte(const uint32_t* words, uint64_t i) { return uint8_t(words[i >> 2] >> (24 - 8 * (i & 3))); }

}  // namespace jxlb
