// JPEG bitstream reconstruction, host side: see jbrd.h. Follows crates/jxl-jbr/src/{lib.rs,huffman.rs,reconstruct.rs}
// and the box handling of crates/jxl-oxide/src/{aux_box.rs,lib.rs:797-904}.
#include "jbrd.h"

#include <dlfcn.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <mutex>

#include "planner.h"

namespace jxlb {

namespace {
const uint8_t kHeaderIcc[] = {'I', 'C', 'C', '_', 'P', 'R', 'O', 'F', 'I', 'L', 'E', 0};
const uint8_t kHeaderExif[] = {'E', 'x', 'i', 'f', 0, 0};
const char kHeaderXmp[] = "http://ns.adobe.com/xap/1.0/";  // + its NUL: 29 bytes

// BrotliDecoderDecompress (brotli/decode.h): 0 error, 1 success, 2 needs more input, 3 needs more output
typedef int (*BrotliDecompressFn)(size_t encoded_size, const uint8_t* encoded, size_t* decoded_size, uint8_t* decoded);
BrotliDecompressFn brotli_fn() {
  static std::once_flag once;
  static BrotliDecompressFn fn = nullptr;
  std::call_once(once, [] {
    void* h = dlopen("libbrotlidec.so.1", RTLD_NOW | RTLD_LOCAL);
    if (h) fn = reinterpret_cast<BrotliDecompressFn>(dlsym(h, "BrotliDecoderDecompress"));
  });
  return fn;
}

uint32_t be32(const uint8_t* p) { return (uint32_t(p[0]) << 24) | (uint32_t(p[1]) << 16) | (uint32_t(p[2]) << 8) | p[3]; }
void put16(std::vector<uint8_t>& o, uint32_t v) {
  o.push_back(uint8_t(v >> 8));
  o.push_back(uint8_t(v));
}
}  // namespace

std::vector<uint8_t> brotli_decompress(const uint8_t* data, size_t size, size_t max_out) {
  BrotliDecompressFn fn = brotli_fn();
  JXLB_CHECK(fn, kErrUnsupported, "libbrotlidec.so.1 is not available: Brotli-compressed JPEG reconstruction data cannot be read");
  size_t cap = std::min<size_t>(max_out, std::max<size_t>(size * 4, 4096));
  for (;;) {
    std::vector<uint8_t> out(cap + 1);
    size_t n = out.size();
    const int r = fn(size, data, &n, out.data());
    if (r == 1 && n <= max_out) {
      out.resize(n);
      return out;
    }
    JXLB_CHECK(r == 3 || r == 1, kErrBitstream, "corrupt Brotli stream");
    JXLB_CHECK(cap < max_out, kErrBitstream, "Brotli stream decodes to more bytes than expected");
    cap = std::min<size_t>(max_out, cap * 4);
  }
}

ContainerBoxes collect_boxes(const uint8_t* data, size_t size) {
  static const uint8_t kSig[12] = {0, 0, 0, 0x0c, 'J', 'X', 'L', ' ', 0x0d, 0x0a, 0x87, 0x0a};
  ContainerBoxes b;
  if (size < 12 || std::memcmp(data, kSig, 12) != 0) return b;  // a bare codestream has no boxes
  size_t pos = 0;
  while (pos + 8 <= size) {
    uint64_t box_size = be32(data + pos);
    const uint8_t* ty = data + pos + 4;
    size_t header = 8;
    if (box_size == 1) {
      JXLB_CHECK(pos + 16 <= size, kErrEof, "truncated container box");
      box_size = 0;
      for (int i = 0; i < 8; ++i) box_size = (box_size << 8) | data[pos + 8 + i];
      header = 16;
    }
    const size_t end = box_size == 0 ? size : pos + size_t(box_size);
    JXLB_CHECK(end <= size && end >= pos + header, kErrEof, "truncated container box");
    const uint8_t* body = data + pos + header;
    size_t body_len = end - pos - header;
    std::vector<uint8_t> unwrapped;
    if (std::memcmp(ty, "brob", 4) == 0) {  // Brotli-compressed box: inner type, then the stream
      JXLB_CHECK(body_len >= 4, kErrBitstream, "invalid brob box");
      ty = body;
      const bool wanted = std::memcmp(ty, "jbrd", 4) == 0 || (std::memcmp(ty, "Exif", 4) == 0 && !b.has_exif) ||
                          (std::memcmp(ty, "xml ", 4) == 0 && !b.has_xml);
      if (wanted) unwrapped = brotli_decompress(body + 4, body_len - 4, size_t(1) << 30);
      body = unwrapped.data();
      body_len = unwrapped.size();
    }
    if (std::memcmp(ty, "jbrd", 4) == 0 && !b.has_jbrd) {
      b.has_jbrd = true;
      b.jbrd.assign(body, body + body_len);
    } else if (std::memcmp(ty, "Exif", 4) == 0 && !b.has_exif) {
      b.has_exif = true;
      b.exif.assign(body, body + body_len);
    } else if (std::memcmp(ty, "xml ", 4) == 0 && !b.has_xml) {
      b.has_xml = true;
      b.xml.assign(body, body + body_len);
    }
    pos = end;
  }
  return b;
}

size_t JpegHeader::expected_icc_len() const {  // lib.rs:266-288
  size_t n = 0;
  for (const App& a : app)
    if (a.type == 1) n += a.length - 5 - sizeof(kHeaderIcc);
  return n;
}
size_t JpegHeader::expected_exif_len() const {
  for (const App& a : app)
    if (a.type == 2) return a.length - 3 - sizeof(kHeaderExif);
  return 0;
}
size_t JpegHeader::expected_xmp_len() const {
  for (const App& a : app)
    if (a.type == 3) return a.length - 3 - sizeof(kHeaderXmp);
  return 0;
}

namespace {
// JpegBitstreamHeader::parse (lib.rs:143-238) and its bundles (lib.rs:297-492, huffman.rs:62-93)
JpegHeader parse_header(BitReader& br) {
  auto eof = [&] { JXLB_CHECK(!br.overrun(), kErrEof, "truncated jbrd box"); };
  JpegHeader h;
  h.is_gray = br.read_bool();
  size_t num_app = 0, num_com = 0, num_scans = 0, num_inter = 0;
  bool has_dri = false;
  while (h.markers.empty() || h.markers.back() != 0xd9) {
    const uint8_t m = uint8_t(br.read(6) + 0xc0);
    eof();
    if (m >= 0xe0 && m <= 0xef) ++num_app;
    else if (m == 0xfe) ++num_com;
    else if (m == 0xda) ++num_scans;
    else if (m == 0xff) ++num_inter;
    else if (m == 0xdd) has_dri = true;
    h.markers.push_back(m);
  }
  for (size_t i = 0; i < num_app; ++i) {
    JpegHeader::App a;
    a.type = br.read_u32({0, 0}, {1, 0}, {2, 1}, {4, 2});
    a.length = br.read(16) + 1;
    eof();
    JXLB_CHECK(a.type <= 3, kErrBitstream, "unknown APP marker type in jbrd box");
    JXLB_CHECK(a.type != 1 || a.length >= 5 + sizeof(kHeaderIcc), kErrBitstream, "ICC APP marker too short");
    JXLB_CHECK(a.type != 2 || a.length >= 3 + sizeof(kHeaderExif), kErrBitstream, "Exif APP marker too short");
    JXLB_CHECK(a.type != 3 || a.length >= 3 + sizeof(kHeaderXmp), kErrBitstream, "XMP APP marker too short");
    h.app.push_back(a);
  }
  for (size_t i = 0; i < num_com; ++i) h.com_lengths.push_back(br.read(16) + 1);
  const uint32_t num_quant = br.read(2) + 1;
  for (uint32_t i = 0; i < num_quant; ++i) {
    JpegHeader::Quant q;
    q.precision = uint8_t(br.read(1));
    q.index = uint8_t(br.read(2));
    q.is_last = br.read_bool();
    h.quant.push_back(q);
  }
  const uint32_t comp_type = br.read(2);
  std::vector<uint8_t> ids;
  if (comp_type == 0) ids = {1};
  else if (comp_type == 1) ids = {1, 2, 3};
  else if (comp_type == 2) ids = {'R', 'G', 'B'};
  else {
    const uint32_t n = br.read(2) + 1;
    for (uint32_t i = 0; i < n; ++i) ids.push_back(uint8_t(br.read(8)));
  }
  for (uint8_t id : ids) h.comps.push_back({id, uint8_t(br.read(2))});
  const uint32_t num_huff = br.read_u32({4, 0}, {2, 3}, {10, 4}, {26, 6});
  for (uint32_t i = 0; i < num_huff; ++i) {
    JpegHuffmanCode hc;
    hc.is_ac = br.read_bool();
    hc.id = uint8_t(br.read(2));
    hc.is_last = br.read_bool();
    uint32_t sum = 0;
    for (uint8_t& c : hc.counts) {
      const uint32_t x = br.read_u32({0, 0}, {1, 0}, {2, 3}, {0, 8});
      sum += x;
      c = uint8_t(x);
    }
    eof();
    for (uint32_t k = 0; k < sum; ++k) hc.values.push_back(uint8_t(br.read_u32({0, 2}, {4, 2}, {8, 4}, {1, 8})));
    eof();
    h.huffman.push_back(std::move(hc));
  }
  for (size_t i = 0; i < num_scans; ++i) {
    JpegScanInfo s;
    const uint32_t nc = br.read(2) + 1;
    s.ss = uint8_t(br.read(6));
    s.se = uint8_t(br.read(6));
    s.al = uint8_t(br.read(4));
    s.ah = uint8_t(br.read(4));
    for (uint32_t c = 0; c < nc; ++c) {
      JpegScanInfo::Comp sc;
      sc.comp_idx = uint8_t(br.read(2));
      sc.ac_tbl = uint8_t(br.read(2));
      sc.dc_tbl = uint8_t(br.read(2));
      s.comps.push_back(sc);
    }
    br.read_u32({0, 0}, {1, 0}, {2, 0}, {3, 3});  // last_needed_pass
    h.scans.push_back(std::move(s));
  }
  if (has_dri) h.restart_interval = br.read(16);
  for (JpegScanInfo& s : h.scans) {  // ScanMoreInfo (lib.rs:399-453)
    const uint32_t num_reset = br.read_u32({0, 0}, {1, 2}, {4, 4}, {20, 16});
    bool have_last = false;
    uint32_t last = 0;
    for (uint32_t i = 0; i < num_reset; ++i) {
      const uint32_t diff = br.read_u32({0, 0}, {1, 3}, {9, 5}, {41, 28});
      eof();
      const uint64_t idx = have_last ? std::min<uint64_t>(uint64_t(last) + diff + 1, 0xffffffffu) : diff;
      JXLB_CHECK(idx <= (3u << 26), kErrBitstream, "reset_points too large");
      last = uint32_t(idx);
      have_last = true;
      s.reset_points.push_back(last);
    }
    const uint32_t num_ezr = br.read_u32({0, 0}, {1, 2}, {4, 4}, {20, 16});
    have_last = false;
    for (uint32_t i = 0; i < num_ezr; ++i) {
      const uint32_t num_runs = br.read_u32({1, 0}, {2, 2}, {5, 4}, {20, 8});
      const uint32_t run_length = br.read_u32({0, 0}, {1, 3}, {9, 5}, {41, 28});
      eof();
      const uint64_t idx = have_last ? std::min<uint64_t>(uint64_t(last) + run_length + 1, 0xffffffffu) : run_length;
      JXLB_CHECK(idx <= (3u << 26), kErrBitstream, "extra_zero_runs.block_idx too large");
      last = uint32_t(idx);
      have_last = true;
      s.extra_zero_runs.push_back({last, num_runs});
    }
  }
  for (size_t i = 0; i < num_inter; ++i) h.intermarker_lengths.push_back(br.read(16));
  h.tail_data_length = br.read_u32({0, 0}, {1, 8}, {257, 16}, {65793, 22});
  h.has_padding = br.read_bool();
  if (h.has_padding) {
    const uint32_t num_bits = br.read(24);
    JXLB_CHECK(br.pos() + num_bits <= br.size_bits(), kErrEof, "truncated jbrd box");
    for (uint32_t i = 0; i < num_bits / 8; ++i) h.padding.push_back(uint8_t(br.read(8)));
    h.padding.push_back(uint8_t(br.read(num_bits % 8)));
  }
  eof();
  return h;
}

size_t expected_data_len(const JpegHeader& h) {  // lib.rs:241-264
  size_t n = h.tail_data_length;
  for (const JpegHeader::App& a : h.app)
    if (a.type == 0) n += a.length;
  for (uint32_t l : h.com_lengths) n += l;
  for (uint32_t l : h.intermarker_lengths) n += l;
  return n;
}

// Image header + ICC stream + first frame header of a bare codestream.
void first_frame_header(const std::vector<uint8_t>& cs, ImageHeader* ih, FrameHeader* fh) {
  BitReader br(cs.data(), cs.size());
  *ih = parse_image_header(br);
  if (ih->colour_encoding.want_icc) skip_icc_profile(br);
  br.zero_pad_to_byte();
  BitReader fr(cs.data(), cs.size(), skip_preview_frame(cs.data(), cs.size(), *ih, br.pos() / 8) * 8);
  *fh = parse_frame_header(fr, *ih);
  fr.check();
}

bool normal_frame(const FrameHeader& fh) {
  return fh.frame_type == FrameType::kRegular || fh.frame_type == FrameType::kSkipProgressive;
}
}  // namespace

JpegHeader parse_jbrd(const std::vector<uint8_t>& box) {
  BitReader br(box.data(), box.size());
  JpegHeader h = parse_header(br);
  br.zero_pad_to_byte();
  const size_t at = br.pos() / 8, expected = expected_data_len(h);
  if (at < box.size()) h.data = brotli_decompress(box.data() + at, box.size() - at, expected);
  JXLB_CHECK(h.data.size() == expected, kErrBitstream, "data section length of the jbrd box does not match the header");
  return h;
}

int32_t jpeg_reconstruction_status(const uint8_t* data, size_t size) {
  const ContainerBoxes boxes = collect_boxes(data, size);
  if (!boxes.has_jbrd) return 0;
  try {
    BitReader br(boxes.jbrd.data(), boxes.jbrd.size());
    const JpegHeader h = parse_header(br);
    ImageHeader ih;
    FrameHeader fh;
    first_frame_header(extract_codestream(data, size), &ih, &fh);
    if (fh.encoding != Encoding::kVarDct || !normal_frame(fh)) return 2;
    if (h.expected_icc_len() > 0 && !ih.colour_encoding.want_icc) return 2;
    if (h.expected_exif_len() > 0 && (!boxes.has_exif || boxes.exif.size() < 4)) return 2;
    if (h.expected_xmp_len() > 0 && !boxes.has_xml) return 2;
    return 1;
  } catch (const Error&) {
    return 2;
  }
}

JpegJob prepare_jpeg_job(const uint8_t* data, size_t size) {
  ContainerBoxes boxes = collect_boxes(data, size);
  JXLB_CHECK(boxes.has_jbrd, kErrUnsupported, "JPEG reconstruction unavailable: the file has no jbrd box");
  JpegJob job;
  job.header = parse_jbrd(boxes.jbrd);
  if (job.header.expected_exif_len() > 0 && boxes.has_exif) {  // aux_box/exif.rs:14-42
    JXLB_CHECK(boxes.exif.size() >= 4, kErrBitstream, "Exif box too short");
    const uint32_t tiff_offset = be32(boxes.exif.data());
    JXLB_CHECK(tiff_offset < boxes.exif.size() - 4, kErrBitstream, "tiff_header_offset of Exif box is too large");
    job.exif.assign(boxes.exif.begin() + 4, boxes.exif.end());
  }
  if (job.header.expected_xmp_len() > 0) job.xmp = boxes.xml;
  return job;
}

namespace {
// HuffmanCode::build (huffman.rs:18-59) as (length << 16) | code entries
void build_huffman(const JpegHuffmanCode& hc, uint32_t out[256]) {
  std::memset(out, 0, 256 * sizeof(uint32_t));
  JXLB_CHECK(hc.values.size() >= 2, kErrBitstream, "empty JPEG Huffman table");
  std::vector<uint32_t> lengths;
  for (uint32_t len = 0; len < 17; ++len)
    for (uint32_t k = 0; k < hc.counts[len]; ++k) lengths.push_back(len);
  lengths.pop_back();
  uint32_t code = 0, prev = lengths[0];
  for (size_t i = 0; i < lengths.size(); ++i) {
    const uint32_t len = lengths[i];
    if (len != prev) {
      code <<= (len - prev);
      prev = len;
    }
    out[hc.values[i]] = len ? jpeg_huff_entry(len, code & ((1u << len) - 1)) : 0;
    ++code;
  }
}
}  // namespace

// JpegBitstreamReconstructor::new + write + process_next (reconstruct.rs:55-790)
void assemble_jpeg(JpegJob& job, const VarDctState& st, const ScanEncoder& encode_scan) {
  const JpegHeader& h = job.header;
  const FrameHeader& fh = *st.fh;
  const ImageHeader& ih = *st.ih;
  auto incompatible = [](bool ok) { JXLB_CHECK(ok, kErrBitstream, "the frame is incompatible with its JPEG reconstruction data"); };
  JXLB_CHECK(h.expected_icc_len() == 0 || h.expected_icc_len() == ih.icc_profile.size(), kErrBitstream,
             "ICC profile length does not match the jbrd box");
  JXLB_CHECK(h.expected_exif_len() == 0 || h.expected_exif_len() == job.exif.size(), kErrBitstream,
             "Exif metadata length does not match the jbrd box");
  JXLB_CHECK(h.expected_xmp_len() == 0 || h.expected_xmp_len() == job.xmp.size(), kErrBitstream,
             "XMP metadata length does not match the jbrd box");
  incompatible(!ih.xyb_encoded && fh.encoding == Encoding::kVarDct && normal_frame(fh));
  incompatible(!fh.use_lf_frame() && fh.skip_adaptive_lf_smoothing());
  if (!st.subsampled)
    incompatible(st.lfg->colour_factor == 84 && st.lfg->base_correlation_x == 0.0f && st.lfg->base_correlation_b == 0.0f);
  const std::vector<int32_t>* jq = st.hfg->dequant->jpeg;
  for (int c = 0; c < 3; ++c) incompatible(jq[c].size() == 64);
  const bool do_cfl = !h.is_gray && !st.subsampled;
  // the jpeg_upsampling of Y, Cb, Cr (the frame header lists Cb, Y, Cr)
  const uint32_t ju[3] = {fh.jpeg_upsampling[1], fh.jpeg_upsampling[0], fh.jpeg_upsampling[2]};

  JpegZigzag zz;
  const std::vector<uint32_t> nat = natural_order(0);
  for (int i = 0; i < 64; ++i) zz.xy[i] = uint8_t((nat[i] & 0xffff) | ((nat[i] >> 16) << 3));

  std::vector<uint8_t>& o = job.out;
  o = {0xff, 0xd8};
  uint32_t huff[8][256];
  std::memset(huff, 0, sizeof(huff));
  size_t app_ptr = 0, com_ptr = 0, inter_ptr = 0, huff_ptr = 0, quant_ptr = 0, scan_ptr = 0, icc_marker = 0, icc_offset = 0;
  size_t num_icc = 0;
  for (const JpegHeader::App& a : h.app) num_icc += a.type == 1;
  size_t app_data = 0, com_data = 0, inter_data = 0;
  for (const JpegHeader::App& a : h.app)
    if (a.type == 0) com_data += a.length;
  inter_data = com_data;
  for (uint32_t l : h.com_lengths) inter_data += l;
  size_t tail_data = inter_data;
  for (uint32_t l : h.intermarker_lengths) tail_data += l;
  bool have_quant = false, progressive = false;
  uint8_t last_quant[64] = {};
  uint16_t last_quant16[64] = {};
  uint32_t restart = 0;
  uint64_t pad_used = 0;
  for (uint8_t m : h.markers) {
    if (m == 0xc0 || m == 0xc1 || m == 0xc2 || m == 0xc9 || m == 0xca) {  // SOF
      progressive = m == 0xc2 || m == 0xca;
      JXLB_CHECK(!progressive, kErrUnsupported, "progressive JPEG reconstruction is not implemented");
      const size_t nc = h.comps.size();
      o.insert(o.end(), {0xff, m});
      put16(o, uint32_t(8 + nc * 3));
      o.push_back(8);
      put16(o, ih.height & 0xffff);
      put16(o, ih.width & 0xffff);
      o.push_back(uint8_t(nc));
      static const uint8_t kSampling[4] = {0x11, 0x22, 0x21, 0x12};
      for (size_t i = 0; i < nc; ++i) o.insert(o.end(), {h.comps[i].id, i < 3 ? kSampling[ju[i]] : uint8_t(0x11), h.comps[i].q_idx});
    } else if (m == 0xc4) {  // DHT
      size_t n = huff_ptr;
      while (n < h.huffman.size() && !h.huffman[n].is_last) ++n;
      JXLB_CHECK(n < h.huffman.size(), kErrBitstream, "DHT without a last table");
      size_t len = 2;
      for (size_t i = huff_ptr; i <= n; ++i) len += 16 + h.huffman[i].values.size();
      o.insert(o.end(), {0xff, 0xc4});
      put16(o, uint32_t(len));
      for (; huff_ptr <= n; ++huff_ptr) {
        const JpegHuffmanCode& hc = h.huffman[huff_ptr];
        JXLB_CHECK(!hc.values.empty(), kErrBitstream, "empty JPEG Huffman table");
        uint8_t counts[16];
        std::memcpy(counts, hc.counts + 1, 16);
        for (int k = 15; k >= 0; --k)
          if (counts[k]) {
            --counts[k];
            break;
          }
        o.push_back(uint8_t(hc.id | (hc.is_ac ? 0x10 : 0)));
        o.insert(o.end(), counts, counts + 16);
        o.insert(o.end(), hc.values.begin(), hc.values.end() - 1);
        build_huffman(hc, huff[hc.id + (hc.is_ac ? 4 : 0)]);
      }
    } else if (m >= 0xd0 && m <= 0xd7) {  // RSTn
      o.insert(o.end(), {0xff, m});
    } else if (m == 0xd9) {  // EOI
      o.insert(o.end(), {0xff, 0xd9});
      o.insert(o.end(), h.data.begin() + tail_data, h.data.end());
    } else if (m == 0xda) {  // SOS
      JXLB_CHECK(scan_ptr < h.scans.size(), kErrBitstream, "more SOS markers than scans");
      const JpegScanInfo& si = h.scans[scan_ptr++];
      const uint32_t nc = uint32_t(si.comps.size());
      JpegScanPlan plan;
      std::memset(&plan.dev, 0, sizeof(plan.dev));
      std::vector<uint8_t>& sos = plan.sos;
      sos = {0xff, 0xda};
      put16(sos, 6 + 2 * nc);
      sos.push_back(uint8_t(nc));
      for (const JpegScanInfo::Comp& c : si.comps) {
        JXLB_CHECK(c.comp_idx < h.comps.size() && c.comp_idx < 3, kErrBitstream, "scan component out of range");
        sos.push_back(h.comps[c.comp_idx].id);
        sos.push_back(uint8_t((c.dc_tbl << 4) | c.ac_tbl));
      }
      sos.insert(sos.end(), {si.ss, si.se, uint8_t((si.ah << 4) | si.al)});
      JXLB_CHECK(si.ss == 0 && si.se == 63 && si.al == 0 && si.ah == 0, kErrUnsupported,
                 "JPEG scans other than sequential (ss 0, se 63, no successive approximation) are not implemented");
      // ScanParams (reconstruct.rs:548-594)
      uint32_t hs[4], vs[4], max_hs = 1, max_vs = 1;
      for (uint32_t i = 0; i < nc; ++i) {
        static const uint32_t kH[4] = {1, 2, 2, 1}, kV[4] = {1, 2, 1, 2};
        hs[i] = kH[ju[si.comps[i].comp_idx]];
        vs[i] = kV[ju[si.comps[i].comp_idx]];
        max_hs = std::max(max_hs, hs[i]);
        max_vs = std::max(max_vs, vs[i]);
      }
      uint32_t mh = max_hs == 2, mv = max_vs == 2;
      const uint32_t full_w8 = (fh.width + 7) / 8, full_h8 = (fh.height + 7) / 8;
      uint32_t w8 = (full_w8 + mh) >> mh, h8 = (full_h8 + mv) >> mv;
      if (nc == 1) {
        if ((1u << mh) == hs[0]) w8 = full_w8;
        if ((1u << mv) == vs[0]) h8 = full_h8;
        hs[0] = vs[0] = 1;
      }
      DevJpegScan& d = plan.dev;
      d.zz = zz;
      d.do_cfl = do_cfl;
      if (do_cfl)
        for (int i = 0; i < 64; ++i) {
          JXLB_CHECK(jq[0][i] != 0 && jq[2][i] != 0, kErrBitstream, "zero JPEG quantisation value");
          d.quant_ratio[0][i] = (1 << 11) * jq[1][i] / jq[0][i];
          d.quant_ratio[1][i] = (1 << 11) * jq[1][i] / jq[2][i];
        }
      d.w8 = w8;
      const uint64_t mcus = uint64_t(w8) * h8;
      d.restart_mcus = restart ? restart : uint32_t(std::max<uint64_t>(mcus, 1));
      d.num_intervals = uint32_t((mcus + d.restart_mcus - 1) / d.restart_mcus);
      d.num_comps = nc;
      uint32_t slots = 0;
      for (uint32_t i = 0; i < nc; ++i) {
        const uint32_t ci = si.comps[i].comp_idx;
        const uint32_t c = fh.do_ycbcr ? (ci == 0 ? 1 : (ci == 1 ? 0 : 2)) : ci;
        d.comp_channel[i] = c;
        if (!fh.do_ycbcr) {
          JXLB_CHECK(jq[c][0] != 0, kErrBitstream, "zero JPEG quantisation value");
          d.comp_dc_offset[i] = int16_t(1024 / jq[c][0]);
        }
        d.comp_hs[i] = hs[i];
        d.comp_vs[i] = vs[i];
        d.comp_dc_table[i] = si.comps[i].dc_tbl;
        d.comp_ac_table[i] = 4 + si.comps[i].ac_tbl;
        const uint32_t first = slots;
        for (uint32_t dy = 0; dy < vs[i]; ++dy)
          for (uint32_t dx = 0; dx < hs[i]; ++dx) {
            d.slot_comp[slots] = uint8_t(i);
            d.slot_dx[slots] = uint8_t(dx);
            d.slot_dy[slots] = uint8_t(dy);
            d.slot_prev[slots] = slots == first ? uint8_t(0x80 | (first + hs[i] * vs[i] - 1)) : uint8_t(slots - 1);
            ++slots;
          }
      }
      d.blocks_per_mcu = slots;
      JXLB_CHECK(mcus * slots < (uint64_t(1) << 31), kErrUnsupported, "JPEG scan too large");
      d.num_blocks = uint32_t(mcus * slots);
      // the scan must stay inside the planes (a malformed box could ask for more blocks than the frame has)
      for (uint32_t i = 0; i < nc; ++i) {
        const uint32_t c = d.comp_channel[i];
        JXLB_CHECK(w8 * hs[i] <= (st.bw >> st.hshift[c]) && h8 * vs[i] <= (st.bh >> st.vshift[c]), kErrBitstream,
                   "JPEG scan larger than the frame");
      }
      for (const auto& e : si.extra_zero_runs) {
        plan.ezr_block.push_back(e.first);
        plan.ezr_count.push_back(e.second);
      }
      d.num_ezr = uint32_t(plan.ezr_block.size());
      d.pad_avail_bits = h.has_padding ? uint64_t(h.padding.size()) * 8 : 0;
      d.pad_base = pad_used;
      std::memcpy(plan.huff, huff, sizeof(huff));
      o.insert(o.end(), sos.begin(), sos.end());
      pad_used += encode_scan(plan, pad_used, &o);
    } else if (m == 0xdb) {  // DQT
      size_t n = quant_ptr;
      while (n < h.quant.size() && !h.quant[n].is_last) ++n;
      JXLB_CHECK(n < h.quant.size(), kErrBitstream, "DQT without a last table");
      size_t len = 2;
      for (size_t i = quant_ptr; i <= n; ++i) len += 65 + (h.quant[i].precision ? 64 : 0);
      o.insert(o.end(), {0xff, 0xdb});
      put16(o, uint32_t(len));
      for (; quant_ptr <= n; ++quant_ptr) {
        const JpegHeader::Quant& qt = h.quant[quant_ptr];
        for (size_t ch = 0; ch < h.comps.size(); ++ch) {
          if (h.comps[ch].q_idx != qt.index) continue;
          size_t channel = ch;
          if (fh.do_ycbcr && channel <= 1) channel ^= 1;
          if (channel < 3) {
            for (int i = 0; i < 64; ++i) {  // transposed for DCT8
              const uint32_t y = zz.xy[i] & 7, x = zz.xy[i] >> 3;
              last_quant16[i] = uint16_t(jq[channel][x + 8 * y]);
              last_quant[i] = uint8_t(last_quant16[i]);
            }
            have_quant = true;
          }
          break;
        }
        JXLB_CHECK(have_quant, kErrBitstream, "DQT without quantisation values");
        if (qt.precision == 0) {
          o.push_back(qt.index);
          o.insert(o.end(), last_quant, last_quant + 64);
        } else {
          o.push_back(uint8_t(qt.index | (qt.precision << 4)));
          for (int i = 0; i < 64; ++i) put16(o, last_quant16[i]);
        }
      }
    } else if (m == 0xdd) {  // DRI
      o.insert(o.end(), {0xff, 0xdd, 0, 4});
      put16(o, h.restart_interval & 0xffff);
      restart = h.restart_interval;
    } else if (m >= 0xe0 && m <= 0xef) {  // APPn
      JXLB_CHECK(app_ptr < h.app.size(), kErrBitstream, "more APP markers than entries");
      const JpegHeader::App& a = h.app[app_ptr++];
      const uint32_t enc_len = (a.length - 1) & 0xffff;
      if (a.type == 0) {
        o.push_back(0xff);
        o.insert(o.end(), h.data.begin() + app_data, h.data.begin() + app_data + a.length);
        app_data += a.length;
      } else if (a.type == 1) {
        o.insert(o.end(), {0xff, 0xe2});
        put16(o, enc_len);
        o.insert(o.end(), kHeaderIcc, kHeaderIcc + sizeof(kHeaderIcc));
        o.insert(o.end(), {uint8_t(icc_marker + 1), uint8_t(num_icc)});
        const size_t len = a.length - 5 - sizeof(kHeaderIcc);
        o.insert(o.end(), ih.icc_profile.begin() + icc_offset, ih.icc_profile.begin() + icc_offset + len);
        ++icc_marker;
        icc_offset += len;
      } else if (a.type == 2) {
        o.insert(o.end(), {0xff, 0xe1});
        put16(o, enc_len);
        o.insert(o.end(), kHeaderExif, kHeaderExif + sizeof(kHeaderExif));
        o.insert(o.end(), job.exif.begin(), job.exif.end());
      } else {
        o.insert(o.end(), {0xff, 0xe1});
        put16(o, enc_len);
        o.insert(o.end(), kHeaderXmp, kHeaderXmp + sizeof(kHeaderXmp));
        o.insert(o.end(), job.xmp.begin(), job.xmp.end());
      }
    } else if (m == 0xfe) {  // COM
      const uint32_t len = h.com_lengths.at(com_ptr++);
      o.insert(o.end(), {0xff, 0xfe});
      o.insert(o.end(), h.data.begin() + com_data, h.data.begin() + com_data + len);
      com_data += len;
    } else if (m == 0xff) {  // unrecognised: bytes kept verbatim
      const uint32_t len = h.intermarker_lengths.at(inter_ptr++);
      o.insert(o.end(), h.data.begin() + inter_data, h.data.begin() + inter_data + len);
      inter_data += len;
    } else {
      fail(kErrBitstream, "unknown JPEG marker in jbrd box");
    }
  }
}

}  // namespace jxlb
