// JPEG scan encoding on the device (the serial encoder of crates/jxl-jbr/src/reconstruct/scan.rs and bit_writer.rs as
// a length pass, prefix sums and a scatter). The per-block work is in jpeg_blocks.cuh, shared with the host emulation.
//
//   jpeg_lengths_kernel    one thread per block: gather + chroma-from-luma + encode into a bit counter
//   (exclusive sum)        block bit offsets, relative to the scan
//   jpeg_intervals_kernel  one thread per restart interval: its bits, its padding, its byte length
//   (exclusive sums)       interval byte offsets and padding-bit offsets
//   jpeg_emit_kernel       one thread per block: encode again, writing MSB first at the block's offset; the interval's last
//                          block appends the padding bits
//   jpeg_ff_count_kernel   one thread per 32-bit word: 0xFF bytes in it
//   (exclusive sum)        stuffed bytes before each word
//   jpeg_stuff_kernel      one thread per word: scatter the bytes, a 0x00 after every 0xFF, RSTn before each interval
#include <cub/device/device_scan.cuh>

#include "jpeg_blocks.cuh"
#include "kernels.h"

#define CUDA_CHECK(expr)                                         \
  do {                                                           \
    const cudaError_t e_ = (expr);                               \
    if (e_ != cudaSuccess) fail(kErrCuda, cudaGetErrorString(e_)); \
  } while (0)

namespace jxlb {

namespace {

constexpr int kJpegThreads = 256;

// The eight Huffman tables (8 KB) staged in shared memory: each block looks up about 2 + 2 * (non-zero AC) codes.
__device__ __forceinline__ void stage_huff(uint32_t* s, const uint32_t* __restrict__ g) {
  for (int i = threadIdx.x; i < 8 * 256; i += blockDim.x) s[i] = g[i];
  __syncthreads();
}

__global__ void __launch_bounds__(kJpegThreads) jpeg_lengths_kernel(DevJpegScan p, const uint32_t* __restrict__ huff,
                                                                   const uint32_t* __restrict__ ezr_block,
                                                                   const uint32_t* __restrict__ ezr_count,
                                                                   uint64_t* __restrict__ lens, uint32_t* __restrict__ err) {
  __shared__ uint32_t s_huff[8 * 256];
  stage_huff(s_huff, huff);
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b > p.num_blocks) return;
  if (b == p.num_blocks) {  // the exclusive sum's total
    lens[b] = 0;
    return;
  }
  JpegBitCounter c;
  if (!jpeg_encode_block(p, s_huff, ezr_block, ezr_count, b, c)) {
    atomicOr(err, kJpegErrHuffman);
    c.bits = 0;
  }
  lens[b] = c.bits;
}

__device__ __forceinline__ void interval_blocks(const DevJpegScan& p, uint32_t k, uint32_t* fb, uint32_t* eb) {
  const uint64_t per = uint64_t(p.restart_mcus) * p.blocks_per_mcu;
  *fb = uint32_t(k * per);
  *eb = uint32_t(min(uint64_t(*fb) + per, uint64_t(p.num_blocks)));
}

__global__ void jpeg_intervals_kernel(DevJpegScan p, const uint64_t* __restrict__ boff, uint64_t* __restrict__ ibytes,
                                      uint64_t* __restrict__ ipad) {
  const uint32_t k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k > p.num_intervals) return;
  if (k == p.num_intervals) {
    ibytes[k] = ipad[k] = 0;
    return;
  }
  uint32_t fb, eb;
  interval_blocks(p, k, &fb, &eb);
  const uint64_t bits = boff[eb] - boff[fb];
  const uint64_t pad = (8 - bits % 8) % 8;
  ibytes[k] = (bits + pad) / 8;
  ipad[k] = pad;
}

__global__ void __launch_bounds__(kJpegThreads) jpeg_emit_kernel(DevJpegScan p, const uint32_t* __restrict__ huff,
                                                                const uint32_t* __restrict__ ezr_block,
                                                                const uint32_t* __restrict__ ezr_count,
                                                                const uint64_t* __restrict__ boff, const uint64_t* __restrict__ ibx,
                                                                const uint64_t* __restrict__ ipx, const uint8_t* __restrict__ pad,
                                                                uint32_t* __restrict__ words, uint32_t* __restrict__ err) {
  __shared__ uint32_t s_huff[8 * 256];
  stage_huff(s_huff, huff);
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= p.num_blocks) return;
  const uint32_t k = b / p.blocks_per_mcu / p.restart_mcus;
  uint32_t fb, eb;
  interval_blocks(p, k, &fb, &eb);
  const uint64_t start = ibx[k] * 8;
  JpegBitWriter w(words, start + (boff[b] - boff[fb]));
  if (!jpeg_encode_block(p, s_huff, ezr_block, ezr_count, b, w)) {
    atomicOr(err, kJpegErrHuffman);
    return;
  }
  w.finish();
  if (b + 1 == eb) {  // flush_bit_writer (scan.rs:89-115): pad the interval to a whole byte
    const uint64_t bits = boff[eb] - boff[fb];
    const uint32_t n = uint32_t((8 - bits % 8) % 8);
    if (!n) return;
    const uint64_t off = p.pad_base + ipx[k];
    if (p.pad_avail_bits && off + n > p.pad_avail_bits) {
      atomicOr(err, kJpegErrPadding);
      return;
    }
    JpegBitWriter pw(words, start + bits);
    pw(jpeg_padding_value(p, pad, off, n), n);
    pw.finish();
  }
}

__global__ void jpeg_ff_count_kernel(const uint32_t* __restrict__ words, uint64_t total_bytes, uint32_t nw, uint32_t* __restrict__ cnt) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w > nw) return;
  uint32_t n = 0;
  if (w < nw)
    for (uint32_t j = 0; j < 4; ++j) {
      const uint64_t i = uint64_t(w) * 4 + j;
      n += i < total_bytes && jpeg_scan_byte(words, i) == 0xff;
    }
  cnt[w] = n;
}

__global__ void jpeg_stuff_kernel(const uint32_t* __restrict__ words, uint64_t total_bytes, uint32_t nw,
                                  const uint32_t* __restrict__ ffoff, const uint64_t* __restrict__ ibx, uint32_t nint,
                                  uint8_t* __restrict__ out) {
  const uint32_t w = blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= nw) return;
  uint64_t stuffed = ffoff[w];
  for (uint32_t j = 0; j < 4; ++j) {
    const uint64_t i = uint64_t(w) * 4 + j;
    if (i >= total_bytes) return;
    uint32_t lo = 0, hi = nint;  // the interval holding byte i: last k with ibx[k] <= i
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (ibx[mid] <= i) lo = mid;
      else hi = mid;
    }
    const uint64_t pos = i + stuffed + 2 * uint64_t(lo);
    if (lo > 0 && ibx[lo] == i) {  // restart(): RSTn between intervals, n counting from 0 in every scan
      out[pos - 2] = 0xff;
      out[pos - 1] = uint8_t(0xd0 + ((lo - 1) & 7));
    }
    const uint8_t v = jpeg_scan_byte(words, i);
    out[pos] = v;
    if (v == 0xff) {
      out[pos + 1] = 0;
      ++stuffed;
    }
  }
}

template <typename T>
void exclusive_sum(const T* in, T* out, uint32_t n, void* temp, size_t temp_bytes, cudaStream_t s) {
  size_t bytes = temp_bytes;
  CUDA_CHECK(cub::DeviceScan::ExclusiveSum(temp, bytes, in, out, int(n), s));
}

unsigned grid(uint64_t n, int threads) { return unsigned((n + threads - 1) / threads); }

}  // namespace

size_t jpeg_scan_temp_bytes(uint32_t max_items) {
  size_t a = 0, b = 0;
  CUDA_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, a, static_cast<const uint64_t*>(nullptr), static_cast<uint64_t*>(nullptr), int(max_items)));
  CUDA_CHECK(cub::DeviceScan::ExclusiveSum(nullptr, b, static_cast<const uint32_t*>(nullptr), static_cast<uint32_t*>(nullptr), int(max_items)));
  return std::max(a, b);
}

void launch_jpeg_lengths(const DevJpegScan& p, const uint32_t* huff, const uint32_t* ezr_block, const uint32_t* ezr_count,
                         uint64_t* lens, uint32_t* err, cudaStream_t s) {
  jpeg_lengths_kernel<<<grid(uint64_t(p.num_blocks) + 1, kJpegThreads), kJpegThreads, 0, s>>>(p, huff, ezr_block, ezr_count, lens, err);
  CUDA_CHECK(cudaGetLastError());
}

void launch_jpeg_scan_u64(const uint64_t* in, uint64_t* out, uint32_t n, void* temp, size_t temp_bytes, cudaStream_t s) {
  exclusive_sum(in, out, n, temp, temp_bytes, s);
}

void launch_jpeg_scan_u32(const uint32_t* in, uint32_t* out, uint32_t n, void* temp, size_t temp_bytes, cudaStream_t s) {
  exclusive_sum(in, out, n, temp, temp_bytes, s);
}

void launch_jpeg_intervals(const DevJpegScan& p, const uint64_t* boff, uint64_t* ibytes, uint64_t* ipad, cudaStream_t s) {
  jpeg_intervals_kernel<<<grid(uint64_t(p.num_intervals) + 1, 128), 128, 0, s>>>(p, boff, ibytes, ipad);
  CUDA_CHECK(cudaGetLastError());
}

void launch_jpeg_emit(const DevJpegScan& p, const uint32_t* huff, const uint32_t* ezr_block, const uint32_t* ezr_count,
                      const uint64_t* boff, const uint64_t* ibx, const uint64_t* ipx, const uint8_t* pad, uint32_t* words,
                      uint32_t* err, cudaStream_t s) {
  if (!p.num_blocks) return;
  jpeg_emit_kernel<<<grid(p.num_blocks, kJpegThreads), kJpegThreads, 0, s>>>(p, huff, ezr_block, ezr_count, boff, ibx, ipx, pad, words, err);
  CUDA_CHECK(cudaGetLastError());
}

void launch_jpeg_ff_count(const uint32_t* words, uint64_t total_bytes, uint32_t nw, uint32_t* cnt, cudaStream_t s) {
  jpeg_ff_count_kernel<<<grid(uint64_t(nw) + 1, kJpegThreads), kJpegThreads, 0, s>>>(words, total_bytes, nw, cnt);
  CUDA_CHECK(cudaGetLastError());
}

void launch_jpeg_stuff(const uint32_t* words, uint64_t total_bytes, uint32_t nw, const uint32_t* ffoff, const uint64_t* ibx,
                       uint32_t nint, uint8_t* out, cudaStream_t s) {
  if (!nw) return;
  jpeg_stuff_kernel<<<grid(nw, kJpegThreads), kJpegThreads, 0, s>>>(words, total_bytes, nw, ffoff, ibx, nint, out);
  CUDA_CHECK(cudaGetLastError());
}

}  // namespace jxlb
