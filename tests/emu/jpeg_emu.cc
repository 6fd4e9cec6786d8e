// TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT.
//
// Host emulation of the JPEG scan encoder kernels (kernels/jpeg.cu): the per-block functions of jpeg_blocks.cuh, compiled
// for the host, run in the order and with the data flow of the device launches - a bit counter per block, exclusive
// sums, per-interval padding, every block writing its bits at its own offset into a zeroed word buffer (blocks in
// reverse order, so nothing depends on a serial order), then the 0xFF count, its sum and the stuffing scatter with the
// RST markers. The planes come from the oracle's decode (oracle/oracle_jbr.cc); tests/test_jbrd.py compares the file
// with the oracle's scalar encoder.
#include <cstdlib>
#include <cstring>

#include "../../jxl_oxide_b200/csrc/kernels/jpeg_blocks.cuh"
#include "../../oracle/oracle_jbr.h"

namespace {
template <typename T>
std::vector<T> exclusive_sum(const std::vector<T>& in) {
  std::vector<T> out(in.size());
  T acc = 0;
  for (size_t i = 0; i < in.size(); ++i) {
    out[i] = acc;
    acc += in[i];
  }
  return out;
}

jxlo::JpegScanEncoderFactory emulated_scan_encoder() {
  return [](jxlo::JpegHostPlanes& hp, const jxlb::JpegHeader& header) -> jxlb::ScanEncoder {
    const std::vector<uint8_t>* padding = &header.padding;
    return [&hp, padding](const jxlb::JpegScanPlan& plan, uint64_t, std::vector<uint8_t>* out) -> uint64_t {
      jxlb::DevJpegScan p = plan.dev;
      for (int c = 0; c < 3; ++c) {
        p.coeff[c] = hp.coeff[c].data();
        p.lfq[c] = hp.lfq[c].data();
      }
      p.cfl[0] = hp.cfl[0].data();
      p.cfl[1] = hp.cfl[1].data();
      p.coeff_stride = hp.coeff_stride;
      p.lfq_stride = hp.lfq_stride;
      p.cfl_stride = hp.cfl_stride;
      const uint32_t* huff = &plan.huff[0][0];
      const uint32_t nb = p.num_blocks, ni = p.num_intervals;
      auto fail_huffman = [] { jxlb::fail(jxlb::kErrBitstream, "a JPEG symbol has no code in its Huffman table"); };
      // jpeg_lengths_kernel
      std::vector<uint64_t> lens(nb + 1, 0);
      for (uint32_t b = 0; b < nb; ++b) {
        jxlb::JpegBitCounter c;
        if (!jxlb::jpeg_encode_block(p, huff, plan.ezr_block.data(), plan.ezr_count.data(), b, c)) fail_huffman();
        lens[b] = c.bits;
      }
      const std::vector<uint64_t> boff = exclusive_sum(lens);
      // jpeg_intervals_kernel
      const uint64_t per = uint64_t(p.restart_mcus) * p.blocks_per_mcu;
      std::vector<uint64_t> ib(ni + 1, 0), ip(ni + 1, 0);
      for (uint32_t k = 0; k < ni; ++k) {
        const uint64_t fb = k * per, eb = std::min<uint64_t>(fb + per, nb);
        const uint64_t bits = boff[eb] - boff[fb], pad = (8 - bits % 8) % 8;
        ib[k] = (bits + pad) / 8;
        ip[k] = pad;
      }
      const std::vector<uint64_t> ibx = exclusive_sum(ib), ipx = exclusive_sum(ip);
      const uint64_t total = ibx[ni];
      const uint32_t nw = uint32_t((total + 3) / 4);
      // jpeg_emit_kernel
      std::vector<uint32_t> words(size_t(nw) + 1, 0);
      for (uint32_t b = nb; b-- > 0;) {
        const uint32_t k = b / p.blocks_per_mcu / p.restart_mcus;
        const uint64_t fb = k * per, eb = std::min<uint64_t>(fb + per, nb);
        const uint64_t start = ibx[k] * 8;
        jxlb::JpegBitWriter w(words.data(), start + (boff[b] - boff[fb]));
        if (!jxlb::jpeg_encode_block(p, huff, plan.ezr_block.data(), plan.ezr_count.data(), b, w)) fail_huffman();
        w.finish();
        if (b + 1 == eb) {
          const uint64_t bits = boff[eb] - boff[fb];
          const uint32_t n = uint32_t((8 - bits % 8) % 8);
          if (!n) continue;
          const uint64_t off = p.pad_base + ipx[k];
          JXLB_CHECK(!p.pad_avail_bits || off + n <= p.pad_avail_bits, jxlb::kErrBitstream,
                     "the jbrd box has fewer padding bits than the scans need");
          jxlb::JpegBitWriter pw(words.data(), start + bits);
          pw(jxlb::jpeg_padding_value(p, padding->data(), off, n), n);
          pw.finish();
        }
      }
      // jpeg_ff_count_kernel + sum + jpeg_stuff_kernel
      std::vector<uint32_t> cnt(size_t(nw) + 1, 0);
      for (uint32_t w = 0; w < nw; ++w)
        for (uint32_t j = 0; j < 4; ++j) cnt[w] += uint64_t(w) * 4 + j < total && jxlb::jpeg_scan_byte(words.data(), uint64_t(w) * 4 + j) == 0xff;
      const std::vector<uint32_t> ffoff = exclusive_sum(cnt);
      const size_t n = size_t(total) + ffoff[nw] + 2 * (size_t(ni) - 1), at = out->size();
      out->resize(at + n);
      uint8_t* o = out->data() + at;
      for (uint32_t w = 0; w < nw; ++w) {
        uint64_t stuffed = ffoff[w];
        for (uint32_t j = 0; j < 4; ++j) {
          const uint64_t i = uint64_t(w) * 4 + j;
          if (i >= total) break;
          uint32_t lo = 0, hi = ni;
          while (hi - lo > 1) {
            const uint32_t mid = (lo + hi) >> 1;
            if (ibx[mid] <= i) lo = mid;
            else hi = mid;
          }
          const uint64_t pos = i + stuffed + 2 * uint64_t(lo);
          if (lo > 0 && ibx[lo] == i) {
            o[pos - 2] = 0xff;
            o[pos - 1] = uint8_t(0xd0 + ((lo - 1) & 7));
          }
          const uint8_t v = jxlb::jpeg_scan_byte(words.data(), i);
          o[pos] = v;
          if (v == 0xff) {
            o[pos + 1] = 0;
            ++stuffed;
          }
        }
      }
      return p.pad_avail_bits ? ipx[ni] : 0;
    };
  };
}
}  // namespace

extern "C" int jxle_reconstruct_jpeg(const uint8_t* data, size_t size, uint8_t** out, size_t* out_size, char* err, size_t errlen) {
  try {
    const std::vector<uint8_t> jpeg = jxlo::reconstruct_jpeg(data, size, emulated_scan_encoder());
    *out = static_cast<uint8_t*>(std::malloc(std::max<size_t>(jpeg.size(), 1)));
    std::memcpy(*out, jpeg.data(), jpeg.size());
    *out_size = jpeg.size();
    return 0;
  } catch (const jxlb::Error& e) {
    if (err && errlen) std::snprintf(err, errlen, "%s", e.what());
    return e.code;
  }
}
