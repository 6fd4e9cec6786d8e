// Device-side bit reader and entropy decoder (ANS / prefix / hybrid-uint / LZ77) shared by the
// Modular and HF-coefficient stream kernels. Table layouts are the ones built by
// host/entropy.cc; decoding semantics follow crates/jxl-coding/src/{lib.rs,ans.rs,prefix.rs}.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace jxlb {

enum DevStatus : int {
  kDevOk = 0,
  kDevBadStream = 1,   // ANS final state mismatch / invalid symbol
  kDevOverrun = 2,     // read past the end of the section
  kDevInvalid = 3,     // semantic validation failed (e.g. non_zeros too large)
  kDevUnsupported = 4, // valid syntax outside the implemented set
  kDevBadLayout = 5,   // HfMetadata: the varblocks do not tile their LF group (placement.cuh)
};

struct DevEntropyCode {
  const uint8_t* cluster_map;
  const uint32_t* configs;      // packed HybridUintConfig per cluster
  const uint64_t* ans;          // num_clusters << log_alphabet_size buckets
  const uint32_t* prefix;       // concatenated LUTs
  const uint32_t* prefix_meta;  // per cluster: table_offset, root_bits
  uint32_t log_alphabet_size;
  uint32_t use_prefix;
  uint32_t num_clusters, cluster_map_size, prefix_table_size;
  uint32_t lz77_enabled, lz77_min_symbol, lz77_min_length, lz_len_conf, lz_dist_cluster;
};

// LSB-first bit reader over the (zero-padded) codestream in global memory. 64-bit buffer fed in
// aligned 32-bit words; the NEXT word is always already in flight (`ahead`), so the global-load
// latency of a refill is hidden behind the symbols decoded from the current buffer.
struct DevBitReader {
  const uint32_t* next_word;  // word after `ahead`
  const uint32_t* origin;     // first word of the codestream
  const uint32_t* stop;       // last word a refill may load; beyond it the stream reads as zeros (like the
                              // reference's reader past the end of its slice, bitstream.rs:133-141)
  uint64_t buf;
  uint32_t ahead;
  int nbits;

  // `bit_limit`: absolute end of the enclosing section. A corrupt stream can ask for up to ~47 bits per symbol for
  // as many symbols as its geometry holds (65536 in a DCT256 block); the loads stop two words after the section, so
  // nothing outside the zero-padded codestream copy is ever touched and the overrun is reported from pos().
  __device__ __forceinline__ void init(const uint8_t* d, uint64_t bit_pos, uint64_t bit_limit = ~uint64_t(0)) {
    origin = reinterpret_cast<const uint32_t*>(d);
    stop = bit_limit == ~uint64_t(0) ? reinterpret_cast<const uint32_t*>(~uintptr_t(0)) : origin + ((bit_limit + 31) >> 5) + 2;
    const uint32_t* w = origin + (bit_pos >> 5);
    const uint32_t skip = uint32_t(bit_pos & 31);
    buf = uint64_t(__ldg(w)) >> skip;
    nbits = 32 - int(skip);
    buf |= uint64_t(__ldg(w + 1)) << nbits;
    nbits += 32;
    ahead = __ldg(w + 2);
    next_word = w + 3;
  }
  __device__ __forceinline__ void refill() {  // requires nbits <= 32; afterwards nbits > 32
    buf |= uint64_t(ahead) << nbits;
    nbits += 32;
    ahead = next_word <= stop ? __ldg(next_word) : 0u;
    ++next_word;
  }
  __device__ __forceinline__ uint32_t peek(uint32_t n) {  // n <= 32
    if (nbits < 32) refill();
    return uint32_t(buf) & (n >= 32 ? 0xffffffffu : ((1u << n) - 1));
  }
  __device__ __forceinline__ void consume(uint32_t n) {
    buf >>= n;
    nbits -= int(n);
  }
  // absolute bit offset of the next unread bit: the buffer ends where `ahead` begins
  __device__ __forceinline__ uint64_t pos() const { return uint64_t(next_word - 1 - origin) * 32 - uint64_t(nbits); }
  __device__ __forceinline__ uint32_t read(uint32_t n) {
    uint32_t v = peek(n);
    consume(n);
    return v;
  }
};

// Same reader with a 32-bit word index instead of 64-bit pointers: a refill costs one 32-bit compare and one
// IMAD.WIDE address instead of 64-bit pointer arithmetic and compares (the stream kernels execute one refill per ~2-4
// symbols on a single lane, so every instruction of it is on the serial path).
struct WordBitReader {
  const uint32_t* base;
  uint32_t widx, stop_idx;
  uint64_t buf;
  uint32_t ahead;
  int nbits;
  __device__ __forceinline__ void init(const uint8_t* d, uint64_t bit_pos, uint64_t bit_limit = ~uint64_t(0)) {
    base = reinterpret_cast<const uint32_t*>(d);
    const uint32_t w = uint32_t(bit_pos >> 5), skip = uint32_t(bit_pos & 31);
    stop_idx = bit_limit == ~uint64_t(0) ? 0xffffffffu : uint32_t((bit_limit + 31) >> 5) + 2;
    buf = uint64_t(__ldg(base + w)) >> skip;
    nbits = 32 - int(skip);
    buf |= uint64_t(__ldg(base + w + 1)) << nbits;
    nbits += 32;
    ahead = __ldg(base + w + 2);
    widx = w + 3;
  }
  __device__ __forceinline__ void refill() {  // requires nbits <= 32; afterwards nbits > 32
    buf |= uint64_t(ahead) << nbits;
    nbits += 32;
    ahead = widx <= stop_idx ? __ldg(base + widx) : 0u;
    ++widx;
  }
  __device__ __forceinline__ uint32_t peek(uint32_t n) {  // n <= 32
    if (nbits < 32) refill();
    return uint32_t(buf) & (n >= 32 ? 0xffffffffu : ((1u << n) - 1));
  }
  __device__ __forceinline__ void consume(uint32_t n) {
    buf >>= n;
    nbits -= int(n);
  }
  __device__ __forceinline__ uint64_t pos() const { return uint64_t(widx - 1) * 32 - uint64_t(nbits); }
  __device__ __forceinline__ uint32_t read(uint32_t n) {
    uint32_t v = peek(n);
    consume(n);
    return v;
  }
};

__device__ __constant__ const int8_t kDevSpecialDistances[120][2] = {
    {0, 1},  {1, 0},  {1, 1},  {-1, 1}, {0, 2},  {2, 0},  {1, 2},  {-1, 2}, {2, 1},  {-2, 1},
    {2, 2},  {-2, 2}, {0, 3},  {3, 0},  {1, 3},  {-1, 3}, {3, 1},  {-3, 1}, {2, 3},  {-2, 3},
    {3, 2},  {-3, 2}, {0, 4},  {4, 0},  {1, 4},  {-1, 4}, {4, 1},  {-4, 1}, {3, 3},  {-3, 3},
    {2, 4},  {-2, 4}, {4, 2},  {-4, 2}, {0, 5},  {3, 4},  {-3, 4}, {4, 3},  {-4, 3}, {5, 0},
    {1, 5},  {-1, 5}, {5, 1},  {-5, 1}, {2, 5},  {-2, 5}, {5, 2},  {-5, 2}, {4, 4},  {-4, 4},
    {3, 5},  {-3, 5}, {5, 3},  {-5, 3}, {0, 6},  {6, 0},  {1, 6},  {-1, 6}, {6, 1},  {-6, 1},
    {2, 6},  {-2, 6}, {6, 2},  {-6, 2}, {4, 5},  {-4, 5}, {5, 4},  {-5, 4}, {3, 6},  {-3, 6},
    {6, 3},  {-6, 3}, {0, 7},  {7, 0},  {1, 7},  {-1, 7}, {5, 5},  {-5, 5}, {7, 1},  {-7, 1},
    {4, 6},  {-4, 6}, {6, 4},  {-6, 4}, {2, 7},  {-2, 7}, {7, 2},  {-7, 2}, {3, 7},  {-3, 7},
    {7, 3},  {-7, 3}, {5, 6},  {-5, 6}, {6, 5},  {-6, 5}, {8, 0},  {4, 7},  {-4, 7}, {7, 4},
    {-7, 4}, {8, 1},  {8, 2},  {6, 6},  {-6, 6}, {8, 3},  {5, 7},  {-5, 7}, {7, 5},  {-7, 5},
    {8, 4},  {6, 7},  {-6, 7}, {7, 6},  {-7, 6}, {8, 5},  {7, 7},  {-7, 7}, {8, 6},  {8, 7},
};

__device__ __forceinline__ int32_t dev_unpack_signed(uint32_t x) { return int32_t((x >> 1) ^ (0u - (x & 1))); }

}  // namespace jxlb
