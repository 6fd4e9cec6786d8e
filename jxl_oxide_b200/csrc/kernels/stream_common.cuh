// Helpers shared by the two entropy-stream kernels (modular_stream.cu, entropy.cu): wrapping
// integer arithmetic, the shared-memory view of an entropy code, the symbol / hybrid-uint
// readers (crates/jxl-coding/src/{lib.rs:572-605, ans.rs:276-330, prefix.rs:335-357}) and the
// LZ77 step (lib.rs:476-569).
#pragma once
#include "common.cuh"
#ifndef __CUDACC__
#include <cstdio>
#include <cstdlib>
#endif

namespace jxlb {
namespace {

__device__ __forceinline__ int32_t wadd(int32_t a, int32_t b) { return int32_t(uint32_t(a) + uint32_t(b)); }
__device__ __forceinline__ int32_t wsub(int32_t a, int32_t b) { return int32_t(uint32_t(a) - uint32_t(b)); }
__device__ __forceinline__ int32_t wmul(int32_t a, int32_t b) { return int32_t(uint32_t(a) * uint32_t(b)); }
__device__ __forceinline__ uint32_t abs_diff(int32_t a, int32_t b) {
  return a > b ? uint32_t(a) - uint32_t(b) : uint32_t(b) - uint32_t(a);
}
__device__ __forceinline__ int32_t grad_clamped(int32_t n, int32_t w, int32_t nw) {
  int32_t hi = max(n, w), lo = min(n, w);
  int64_t v = int64_t(lo) + int64_t(hi) - int64_t(nw);
  return int32_t(v < lo ? int64_t(lo) : (v > hi ? int64_t(hi) : v));
}
__device__ __forceinline__ uint32_t ilog2_u32(uint32_t v) { return 31u - uint32_t(__clz(int(v))); }
__device__ __forceinline__ int64_t abs64(int64_t v) { return v < 0 ? -v : v; }

// Shared-memory view of an entropy code; pointers may alias global memory when a table is too
// large to stage.
struct CodeView {
  const uint32_t* configs;
  const uint64_t* ans;
  const uint32_t* prefix;
  const uint32_t* prefix_meta;
  uint32_t log_alphabet_size, use_prefix;
};

// ANS symbol (ans.rs:276-330): alias-table lookup, state update, 16-bit refill.
template <typename BR>
__device__ __forceinline__ uint32_t cv_read_symbol_ans(const CodeView& c, uint32_t& ans_state, BR& br, uint32_t cluster) {
  const uint32_t log_bucket = 12 - c.log_alphabet_size;
  uint32_t state = ans_state;
  uint32_t idx = state & 0xfff;
  uint32_t i = idx >> log_bucket;
  uint32_t pos = idx & ((1u << log_bucket) - 1);
  uint64_t b = c.ans[(size_t(cluster) << c.log_alphabet_size) + i];
  uint32_t lo = uint32_t(b), hi32 = uint32_t(b >> 32);
  uint32_t alias_symbol = lo & 0xff;
  uint32_t alias_cutoff = (lo >> 8) & 0xff;
  uint32_t dist = lo >> 16;
  bool map_to_alias = pos >= alias_cutoff;
  uint32_t hi = map_to_alias ? hi32 : 0u;
  uint32_t offset = (hi & 0xffff) + pos;
  dist ^= hi >> 16;
  uint32_t symbol = map_to_alias ? alias_symbol : i;
  uint32_t next = (state >> 12) * dist + offset;
  if (next < (1u << 16)) next = (next << 16) | br.read(16);
  ans_state = next;
  return symbol;
}

template <typename BR>
__device__ __forceinline__ uint32_t cv_read_symbol(const CodeView& c, uint32_t& ans_state, BR& br, uint32_t cluster) {
  if (c.use_prefix) {  // prefix.rs:335-357
    uint32_t off = c.prefix_meta[cluster * 2], root_bits = c.prefix_meta[cluster * 2 + 1];
    uint32_t peeked = br.peek(15);
    uint32_t e = c.prefix[off + (peeked & ((1u << root_bits) - 1))];
    if (e & 0x80000000u) {
      uint32_t sb = (e >> 16) & 0xff;
      e = c.prefix[off + (1u << root_bits) + (e & 0xffff) + ((peeked >> root_bits) & ((1u << sb) - 1))];
    }
    br.consume((e >> 16) & 0xff);
    return e & 0xffff;
  }
  return cv_read_symbol_ans(c, ans_state, br, cluster);
}

template <typename BR>
__device__ __forceinline__ uint32_t cv_read_uint(BR& br, uint32_t cfg, uint32_t token) {
  uint32_t split_exponent = cfg & 0xff;
  uint32_t split = 1u << split_exponent;
  if (token < split) return token;
  uint32_t msb = (cfg >> 8) & 0xff, lsb = (cfg >> 16) & 0xff;
  uint32_t in_token = msb + lsb;
  uint32_t n = (split_exponent - in_token + ((token - split) >> in_token)) & 31;
  uint32_t rest = br.read(n);
  uint32_t low = token & ((1u << lsb) - 1);
  uint32_t t = (token >> lsb) & ((1u << msb) - 1);
  t |= 1u << msb;
  return uint32_t((((uint64_t(t) << n) | rest) << lsb) | low);
}

// LZ77 state of one stream (lib.rs:346-352): the window of decoded values, the copy in progress and how many values the
// stream has produced. The window is indexed with `& 0xfffff` like the reference's 2^20-entry ring; a smaller window is
// enough for a stream that produces fewer values than it has entries (the index never wraps then). Host builds (the
// emulations in tests/emu/) check every index against `window_len` when the owner set it (lz77_init) and count the
// values taken from copies.
struct Lz77State {
  uint32_t* window;
  uint32_t lz_to_copy, lz_copy_pos, lz_decoded;
#ifndef __CUDACC__
  size_t window_len = ~size_t(0);
  uint64_t copied = 0;
#endif
};
__device__ __forceinline__ void lz77_init(Lz77State& lz, uint32_t* window, size_t window_len) {
  lz.window = window;
  lz.lz_to_copy = lz.lz_copy_pos = lz.lz_decoded = 0;
#ifndef __CUDACC__
  lz.window_len = window_len;
  lz.copied = 0;
#else
  (void)window_len;
#endif
}
__device__ __forceinline__ uint32_t lz77_slot(const Lz77State& lz, uint32_t pos) {
  const uint32_t i = pos & 0xfffff;
#ifndef __CUDACC__
  if (i >= lz.window_len) {
    std::fprintf(stderr, "LZ77 window index %u outside a window of %zu entries\n", i, lz.window_len);
    std::abort();
  }
#endif
  return i;
}

// One value of read_varint_with_multiplier_clustered (lib.rs:476-569) for a code with LZ77 enabled: the next value of a
// copy in progress, or a symbol of `cluster` -- a literal, or a length token that starts a copy (its distance follows in
// the code's distance cluster). Sets `err` to kDevBadStream and returns 0 for a copy before any value or a length that
// overflows (InvalidLz77Symbol); the caller stops the stream then.
template <typename BR>
__device__ __forceinline__ uint32_t lz77_read_value(const CodeView& cv, const DevEntropyCode& code, Lz77State& lz,
                                                    uint32_t& ans_state, BR& br, uint32_t cluster, uint32_t dist_multiplier,
                                                    int& err) {
  uint32_t value;
  if (lz.lz_to_copy > 0) {
    value = lz.window[lz77_slot(lz, lz.lz_copy_pos)];
    ++lz.lz_copy_pos;
    --lz.lz_to_copy;
#ifndef __CUDACC__
    ++lz.copied;
#endif
  } else {
    const uint32_t token = cv_read_symbol(cv, ans_state, br, cluster);
    if (token >= code.lz77_min_symbol) {
      if (lz.lz_decoded == 0) {
        err = kDevBadStream;
        return 0;
      }
      const uint32_t nc = cv_read_uint(br, code.lz_len_conf, token - code.lz77_min_symbol);
      if (nc > 0xffffffffu - code.lz77_min_length) {
        err = kDevBadStream;
        return 0;
      }
      lz.lz_to_copy = nc + code.lz77_min_length;
      const uint32_t dtoken = cv_read_symbol(cv, ans_state, br, code.lz_dist_cluster);
      uint32_t distance = cv_read_uint(br, cv.configs[code.lz_dist_cluster], dtoken);
      if (dist_multiplier == 0) {
      } else if (distance < 120) {
        const int32_t dd = int32_t(kDevSpecialDistances[distance][0]) +
                           int32_t(dist_multiplier) * int32_t(kDevSpecialDistances[distance][1]);
        distance = uint32_t(max(dd - 1, 0));
      } else {
        distance -= 120;
      }
      distance = min(min((1u << 20) - 1, distance) + 1, lz.lz_decoded);
      lz.lz_copy_pos = lz.lz_decoded - distance;
      value = lz.window[lz77_slot(lz, lz.lz_copy_pos)];
      ++lz.lz_copy_pos;
      --lz.lz_to_copy;
#ifndef __CUDACC__
      ++lz.copied;
#endif
    } else {
      value = cv_read_uint(br, cv.configs[cluster], token);
    }
  }
  lz.window[lz77_slot(lz, lz.lz_decoded)] = value;
  ++lz.lz_decoded;
  return value;
}

// cooperative copy global -> shared by the 32 lanes of a warp (word granularity)
__device__ __forceinline__ void warp_copy_words(uint32_t* dst, const uint32_t* src, uint32_t nwords, uint32_t lane) {
  for (uint32_t i = lane; i < nwords; i += 32) dst[i] = __ldg(src + i);
}

}  // namespace
}  // namespace jxlb
