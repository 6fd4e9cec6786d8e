// TEST INFRASTRUCTURE — JPEG reconstruction on the oracle's decode (oracle_jbr.cc); tests/emu/jpeg_emu.cc plugs the
// host build of the device scan encoder in through the same entry point.
#pragma once
#include <cstdint>
#include <functional>
#include <vector>

#include "../jxl_oxide_b200/csrc/host/jbrd.h"

namespace jxlo {

// The frame's quantised planes in host memory (full-frame layout, see kernels/jpeg_blocks.cuh).
struct JpegHostPlanes {
  std::vector<int32_t> coeff[3], lfq[3], cfl[2];
  uint32_t coeff_stride = 0, lfq_stride = 0, cfl_stride = 0;
};
// Makes the scan encoder of one reconstruction from the captured planes (which it may modify) and the jbrd header.
using JpegScanEncoderFactory = std::function<jxlb::ScanEncoder(JpegHostPlanes& planes, const jxlb::JpegHeader& header)>;

// Decodes frame 0 of `data` with the oracle up to its coefficients and rebuilds the JPEG file with `factory`'s encoder.
std::vector<uint8_t> reconstruct_jpeg(const uint8_t* data, size_t size, const JpegScanEncoderFactory& factory);
// The scalar restatement of scan.rs / bit_writer.rs.
JpegScanEncoderFactory scalar_scan_encoder();

}  // namespace jxlo
