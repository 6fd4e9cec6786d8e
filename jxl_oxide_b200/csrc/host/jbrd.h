// JPEG bitstream reconstruction, host side (crates/jxl-jbr): the container boxes that carry the reconstruction data,
// the `jbrd` header, the per-scan plan the scan encoders work from, and the marker assembly around the encoded scans.
// Shared by the CUDA backend (csrc/kernels/jpeg.cu encodes the scans), the test oracle (oracle_jbr.cc) and the host
// emulation of the kernels (tests/emu/jpeg_emu.cc).
#pragma once
#include <cstdint>
#include <functional>
#include <string>
#include <utility>
#include <vector>

#include "../kernels/jpeg_blocks.cuh"
#include "backend.h"
#include "bitreader.h"
#include "frame_syntax.h"
#include "headers.h"

namespace jxlb {

// `jbrd`, first `Exif` and first `xml ` box payloads, `brob`-wrapped ones decompressed (jxl-oxide/src/aux_box.rs).
struct ContainerBoxes {
  bool has_jbrd = false, has_exif = false, has_xml = false;
  std::vector<uint8_t> jbrd, exif, xml;
};
ContainerBoxes collect_boxes(const uint8_t* data, size_t size);

// One-shot Brotli decompression through the system libbrotlidec.so.1, loaded on first use (the library is not linked:
// libjxlb200.so loads without it). Throws kErrUnsupported when the library is missing, kErrBitstream on a corrupt
// stream or when the output would exceed `max_out` bytes.
std::vector<uint8_t> brotli_decompress(const uint8_t* data, size_t size, size_t max_out);

struct JpegHuffmanCode {  // jxl-jbr/src/huffman.rs:5-11
  bool is_ac = false, is_last = false;
  uint8_t id = 0;
  uint8_t counts[17] = {};
  std::vector<uint8_t> values;
};

struct JpegScanInfo {  // lib.rs:333-453
  uint8_t ss = 0, se = 0, al = 0, ah = 0;
  struct Comp {
    uint8_t comp_idx, ac_tbl, dc_tbl;
  };
  std::vector<Comp> comps;
  std::vector<uint32_t> reset_points;
  std::vector<std::pair<uint32_t, uint32_t>> extra_zero_runs;  // (block index, number of ZRL symbols), block order
};

// JpegBitstreamHeader (lib.rs:123-238) plus the decompressed data section.
struct JpegHeader {
  bool is_gray = false;
  std::vector<uint8_t> markers;
  struct App {
    uint32_t type, length;
  };
  std::vector<App> app;
  std::vector<uint32_t> com_lengths;
  struct Quant {
    uint8_t precision, index;
    bool is_last;
  };
  std::vector<Quant> quant;
  struct Comp {
    uint8_t id, q_idx;
  };
  std::vector<Comp> comps;
  std::vector<JpegHuffmanCode> huffman;
  std::vector<JpegScanInfo> scans;
  uint32_t restart_interval = 0;
  std::vector<uint32_t> intermarker_lengths;
  uint32_t tail_data_length = 0;
  bool has_padding = false;
  std::vector<uint8_t> padding;  // padding bits, read LSB first like any JPEG XL bitstream
  std::vector<uint8_t> data;     // APP0, COM, intermarker and tail data
  size_t expected_icc_len() const;
  size_t expected_exif_len() const;
  size_t expected_xmp_len() const;
};
// Parses the box and decompresses its data section. Throws kErrEof on a truncated box.
JpegHeader parse_jbrd(const std::vector<uint8_t>& box);

// 0 unavailable (no jbrd box), 1 available, 2 invalid (jxl-oxide/src/lib.rs:797-850, for a complete file). Host only.
int32_t jpeg_reconstruction_status(const uint8_t* data, size_t size);

// Everything one decode needs to turn frame 0 into a JPEG file: the parsed box and the metadata the APP markers hold.
struct JpegJob {
  JpegHeader header;
  std::vector<uint8_t> exif, xmp;
  std::vector<uint8_t> out;  // the reconstructed file
};
// Reads boxes, the jbrd header and its data section. Throws (kErrUnsupported "unavailable" without a jbrd box).
JpegJob prepare_jpeg_job(const uint8_t* data, size_t size);

// One scan as the block encoders see it: a DevJpegScan without plane pointers, plus what the host keeps.
struct JpegScanPlan {
  DevJpegScan dev;           // plane pointers left null
  uint32_t huff[8][256];     // DC tables 0-3, AC tables 4-7 (jpeg_huff_entry)
  std::vector<uint32_t> ezr_block, ezr_count;
  std::vector<uint8_t> sos;  // the SOS marker segment
};
// Thrown by a backend's vardct_coefficients() hook once the JPEG is built: the rest of the decode is not needed.
struct JpegDone {};

// Builds the file around the scans: `encode_scan(plan, pad_offset, &bytes)` must append the scan's final bytes
// (stuffed, with RST markers) and return the number of padding bits it consumed. Validates the frame
// (reconstruct.rs:95-131) and rejects progressive scans with kErrUnsupported.
using ScanEncoder = std::function<uint64_t(const JpegScanPlan& plan, uint64_t pad_offset, std::vector<uint8_t>* out)>;
void assemble_jpeg(JpegJob& job, const VarDctState& st, const ScanEncoder& encode_scan);

}  // namespace jxlb
