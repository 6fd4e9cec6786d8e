// TEST INFRASTRUCTURE — JPEG bitstream reconstruction on the oracle's own decode: a scalar, line-by-line restatement
// of the sequential scan encoder of crates/jxl-jbr/src/reconstruct/scan.rs (process_scan, process_sequential,
// ScanState::restart / flush_bit_writer), bit_writer.rs (64-bit buffer, byte stuffing) and the integer chroma-from-luma
// of reconstruct.rs:316-393, over the oracle's quantised LF and HF coefficients. Box parsing, Huffman table building and
// the markers around the scans are the shared host code (csrc/host/jbrd.cc).
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>

#include "../jxl_oxide_b200/csrc/host/jbrd.h"
#include "../jxl_oxide_b200/csrc/host/planner.h"
#include "oracle_backend.h"
#include "oracle_jbr.h"

namespace jxlo {

namespace {

// The frame's planes at the point the reference reconstructs from, copied to host memory.
class CaptureBackend : public OracleBackend {
 public:
  CaptureBackend(jxlb::JpegJob* job, const JpegScanEncoderFactory& factory) : OracleBackend(1), job_(job), factory_(factory) {}
  void vardct_coefficients(const jxlb::VarDctState& st) override {
    JpegHostPlanes hp;
    auto grab = [&](int plane, uint32_t w, uint32_t h, std::vector<int32_t>* out) {
      out->resize(size_t(w) * h);
      download_rect(jxlb::View{plane, 0, 0, w, h}, out->data());
    };
    hp.coeff_stride = st.bw * 8;
    hp.lfq_stride = st.bw;
    hp.cfl_stride = (st.width + 63) / 64;
    for (int c = 0; c < 3; ++c) {
      grab(st.coeff[c], st.bw * 8, st.bh * 8, &hp.coeff[c]);
      grab(st.lf_quant[c], st.bw, st.bh, &hp.lfq[c]);
    }
    grab(st.x_from_y, hp.cfl_stride, (st.height + 63) / 64, &hp.cfl[0]);
    grab(st.b_from_y, hp.cfl_stride, (st.height + 63) / 64, &hp.cfl[1]);
    jxlb::assemble_jpeg(*job_, st, factory_(hp, job_->header));
    throw jxlb::JpegDone();
  }

 private:
  jxlb::JpegJob* job_;
  JpegScanEncoderFactory factory_;
};

// bit_writer.rs:1-83
class BitWriter {
 public:
  void write_huffman(uint64_t bits, uint32_t len) {
    buf_ |= bits >> valid_;
    valid_ += len;
    if (valid_ >= 64) {
      const uint32_t extra = valid_ - 64;
      flush_buf(len - extra < 64 ? bits << (len - extra) : 0);
    }
  }
  void write_raw(uint64_t bits, uint32_t len) {
    if (len == 0) return;
    write_huffman(bits << (64 - len), len);
  }
  uint32_t padding_bits() const { return (8 - valid_ % 8) % 8; }
  void finalize(std::vector<uint8_t>* out) {
    const uint32_t valid_bytes = (valid_ + 7) / 8;
    for (uint32_t i = 0; i < valid_bytes; ++i) emit_byte(out_, uint8_t(buf_ >> (56 - 8 * i)));
    out->insert(out->end(), out_.begin(), out_.end());
    out_.clear();
    buf_ = 0;
    valid_ = 0;
  }

 private:
  static void emit_byte(std::vector<uint8_t>& o, uint8_t b) {
    o.push_back(b);
    if (b == 0xff) o.push_back(0);
  }
  void flush_buf(uint64_t next) {
    const uint64_t o = buf_;
    valid_ -= 64;
    buf_ = next;
    for (int i = 0; i < 8; ++i) emit_byte(out_, uint8_t(o >> (56 - 8 * i)));
  }
  std::vector<uint8_t> out_;
  uint64_t buf_ = 0;
  uint32_t valid_ = 0;
};

struct Lookup {  // BuiltHuffmanTable::lookup: (len, code aligned to bit 63)
  const uint32_t* t;
  void get(uint32_t sym, uint32_t* len, uint64_t* bits) const {
    const uint32_t e = t[sym & 0xff];
    if (!e) jxlb::fail(jxlb::kErrBitstream, "a JPEG symbol has no code in its Huffman table");
    *len = e >> 16;
    *bits = uint64_t(e & 0xffff) << (64 - *len);
  }
};

uint32_t bitlen16(uint32_t v) {
  uint32_t n = 0;
  while (v >> n) ++n;
  return n;
}

// process_sequential (scan.rs:133-194)
void process_sequential(BitWriter& w, int16_t* dc_pred, size_t comp, const Lookup& dc_table, const Lookup& ac_table, int16_t dc,
                        const int16_t ac[63], bool has_ezr, uint32_t ezr) {
  const int16_t diff = int16_t(dc - dc_pred[comp]);
  dc_pred[comp] = dc;
  const bool is_neg = diff < 0;
  const int16_t bits = is_neg ? int16_t(-diff) : diff;
  const uint32_t bitlen = bitlen16(uint16_t(bits));
  const int16_t raw_bits = is_neg ? int16_t(-bits - 1) : bits;
  uint32_t len;
  uint64_t code;
  dc_table.get(bitlen, &len, &code);
  w.write_huffman(code, len);
  w.write_raw(uint64_t(int64_t(raw_bits)), bitlen);

  int pos = 0;
  for (;;) {
    int nonzero = -1;
    for (int i = pos; i < 63; ++i)
      if (ac[i] != 0) {
        nonzero = i - pos;
        break;
      }
    if (nonzero < 0) break;
    const int16_t coeff = ac[pos + nonzero];
    pos += nonzero + 1;
    while (nonzero >= 16) {
      ac_table.get(0xf0, &len, &code);
      w.write_huffman(code, len);
      nonzero -= 16;
    }
    uint16_t raw;
    uint32_t n;
    if (coeff < 0) {
      const uint16_t m = uint16_t(-int32_t(coeff));
      raw = uint16_t(~m);
      n = bitlen16(m);
    } else {
      raw = uint16_t(coeff);
      n = bitlen16(raw);
    }
    ac_table.get(uint8_t((nonzero << 4) | n), &len, &code);
    w.write_huffman(code, len);
    w.write_raw(raw, n);
  }
  int32_t num_zeros = 63 - pos;
  if (has_ezr) {
    ac_table.get(0xf0, &len, &code);
    for (uint32_t i = 0; i < ezr; ++i) w.write_huffman(code, len);
    num_zeros -= int32_t(ezr) * 16;
  }
  if (num_zeros > 0) {
    ac_table.get(0, &len, &code);
    w.write_huffman(code, len);
  }
}

// ScanState::flush_bit_writer (scan.rs:89-115)
void flush(BitWriter& w, jxlb::BitReader* padding, std::vector<uint8_t>* out, uint64_t* pad_used) {
  const uint32_t n = w.padding_bits();
  if (n) {
    uint32_t bits = 0xffffffffu;
    if (padding) {
      bits = padding->read(n);
      JXLB_CHECK(!padding->overrun(), jxlb::kErrBitstream, "the jbrd box has fewer padding bits than the scans need");
      *pad_used += n;
    }
    w.write_raw(bits, n);
  }
  w.finalize(out);
}

}  // namespace

std::vector<uint8_t> reconstruct_jpeg(const uint8_t* data, size_t size, const JpegScanEncoderFactory& factory) {
  jxlb::JpegJob job = jxlb::prepare_jpeg_job(data, size);
  const std::vector<uint8_t> cs = jxlb::extract_codestream(data, size);
  CaptureBackend be(&job, factory);
  jxlb::DecodeOptions o;
  o.max_frames = 1;
  bool done = false;
  try {
    jxlb::DecodeResult res = jxlb::decode_codestream(be, cs.data(), cs.size(), o);
    for (jxlb::DecodedFrame& f : res.frames)
      for (jxlb::View& v : f.channels) be.free_plane(v.plane);
  } catch (const jxlb::JpegDone&) {
    done = true;
  }
  JXLB_CHECK(done, jxlb::kErrBitstream, "the first frame is not a VarDCT frame: its JPEG reconstruction data is invalid");
  return job.out;
}

// The scalar encoder: process_scan::<0> (scan.rs:378-535) over the captured planes.
JpegScanEncoderFactory scalar_scan_encoder() {
  return [](JpegHostPlanes& hp, const jxlb::JpegHeader& header) -> jxlb::ScanEncoder {
    auto cfl_done = std::make_shared<bool>(false);
    auto padding = std::make_shared<jxlb::BitReader>(header.padding.data(), header.padding.size());
    const bool has_padding = header.has_padding;
    return [&hp, cfl_done, padding, has_padding](const jxlb::JpegScanPlan& plan, uint64_t, std::vector<uint8_t>* out) -> uint64_t {
      const jxlb::DevJpegScan& p = plan.dev;
      if (p.do_cfl && !*cfl_done) {  // integer_cfl (reconstruct.rs:316-393) on the whole X and B planes, once
        const uint32_t w = hp.coeff_stride, h = uint32_t(hp.coeff[1].size() / w);
        for (int k = 0; k < 2; ++k) {
          std::vector<int32_t>& coeff = hp.coeff[k == 0 ? 0 : 2];
          for (uint32_t y = 0; y < h; ++y)
            for (uint32_t x = 0; x < w; ++x) {
              const int32_t factor = hp.cfl[k][size_t(y / 64) * hp.cfl_stride + x / 64];
              const int32_t coeff_y = hp.coeff[1][size_t(y) * w + x];
              const int32_t q = p.quant_ratio[k][(y % 8) + 8 * (x % 8)];
              const int32_t scale_factor = factor * (1 << 11) / 84;
              const int32_t q_scale = (q * scale_factor + (1 << 10)) >> 11;
              coeff[size_t(y) * w + x] += (coeff_y * q_scale + (1 << 10)) >> 11;
            }
        }
        *cfl_done = true;
      }
      std::map<uint32_t, uint32_t> ezr;
      for (size_t i = 0; i < plan.ezr_block.size(); ++i) ezr[plan.ezr_block[i]] = plan.ezr_count[i];
      BitWriter w;
      int16_t dc_pred[4] = {0, 0, 0, 0};
      uint32_t rst_m = 0, block_idx = 0;
      uint64_t pad_used = 0;
      jxlb::BitReader* pad = has_padding ? padding.get() : nullptr;
      const uint32_t h8 = uint32_t((uint64_t(p.num_blocks) / p.blocks_per_mcu) / p.w8);
      for (uint32_t y8 = 0; y8 < h8; ++y8)
        for (uint32_t x8 = 0; x8 < p.w8; ++x8) {
          const uint32_t mcu_idx = x8 + p.w8 * y8;
          if (p.restart_mcus && mcu_idx != 0 && mcu_idx % p.restart_mcus == 0) {  // ScanState::restart
            std::memset(dc_pred, 0, sizeof(dc_pred));
            flush(w, pad, out, &pad_used);
            out->push_back(0xff);
            out->push_back(uint8_t(0xd0 + rst_m));
            rst_m = (rst_m + 1) % 8;
          }
          for (uint32_t ci = 0; ci < p.num_comps; ++ci) {
            const Lookup dc_table{plan.huff[p.comp_dc_table[ci]]}, ac_table{plan.huff[p.comp_ac_table[ci]]};
            const uint32_t c = p.comp_channel[ci], hs = p.comp_hs[ci], vs = p.comp_vs[ci];
            for (uint32_t dy8 = 0; dy8 < vs; ++dy8) {
              const uint32_t y_dc = y8 * vs + dy8;
              for (uint32_t dx8 = 0; dx8 < hs; ++dx8) {
                const uint32_t x_dc = x8 * hs + dx8;
                int32_t dc = hp.lfq[c][size_t(y_dc) * hp.lfq_stride + x_dc] - p.comp_dc_offset[ci];
                dc = dc < -2047 ? -2047 : (dc > 2047 ? 2047 : dc);
                int16_t ac[63];
                for (int i = 1; i < 64; ++i) {
                  const uint32_t x = p.zz.xy[i] & 7, y = p.zz.xy[i] >> 3;
                  ac[i - 1] = int16_t(hp.coeff[c][size_t(y_dc * 8 + y) * hp.coeff_stride + x_dc * 8 + x]);
                }
                auto it = ezr.find(block_idx);
                process_sequential(w, dc_pred, ci, dc_table, ac_table, int16_t(dc), ac, it != ezr.end(),
                                   it != ezr.end() ? it->second : 0);
                ++block_idx;
              }
            }
          }
        }
      flush(w, pad, out, &pad_used);
      return pad_used;
    };
  };
}

}  // namespace jxlo

extern "C" {

// 0 on success with *out (malloc'd, free with jxlo_free_bytes) holding the file; otherwise the error code.
int jxlo_reconstruct_jpeg(const uint8_t* data, size_t size, uint8_t** out, size_t* out_size, char* err, size_t errlen) {
  try {
    const std::vector<uint8_t> jpeg = jxlo::reconstruct_jpeg(data, size, jxlo::scalar_scan_encoder());
    *out = static_cast<uint8_t*>(std::malloc(std::max<size_t>(jpeg.size(), 1)));
    std::memcpy(*out, jpeg.data(), jpeg.size());
    *out_size = jpeg.size();
    return 0;
  } catch (const jxlb::Error& e) {
    if (err && errlen) std::snprintf(err, errlen, "%s", e.what());
    return e.code;
  }
}

void jxlo_free_bytes(uint8_t* p) { std::free(p); }

int jxlo_jpeg_reconstruction_status(const uint8_t* data, size_t size) {
  try {
    return jxlb::jpeg_reconstruction_status(data, size);
  } catch (const jxlb::Error&) {
    return 2;
  }
}

}  // extern "C"
