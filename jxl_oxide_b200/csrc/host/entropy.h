// Entropy-code *syntax* parsing (histograms, cluster maps, hybrid-uint configs, LZ77
// parameters) into flat, device-uploadable tables, plus a host-side symbol reader that
// the syntax parser itself needs (MA trees, cluster maps, permutations and the TOC are
// entropy coded).
//
// Follows crates/jxl-coding/src/{lib.rs,ans.rs,prefix.rs,permutation.rs} of the reference.
// Table layouts are this project's own (designed for 64-bit / 32-bit device loads).
#pragma once
#include <cstdint>
#include <vector>

#include "bitreader.h"

namespace jxlb {

#ifdef JXLB_ENTROPY_TRACE
// Built only into tools/hf_restream.cc: every stream start (the bit position before its ANS state), every value read
// with its cluster and the bit position after it, and the bit span of each HF pass code (frame_syntax.cc).
struct EntropyCode;
void entropy_trace_begin(const void* reader, size_t pos_bits);
void entropy_trace_value(const void* reader, uint32_t cluster, uint32_t value, size_t pos_bits);
void entropy_trace_hf_code(uint32_t pass, size_t begin_bits, size_t end_bits, const EntropyCode& code);
#endif

// Hybrid-uint config, packed for the device: split_exponent | msb<<8 | lsb<<16.
struct HybridUintConfig {
  uint32_t split_exponent = 0, msb_in_token = 0, lsb_in_token = 0;
  uint32_t split() const { return 1u << split_exponent; }
  uint32_t packed() const { return split_exponent | (msb_in_token << 8) | (lsb_in_token << 16); }
};

// ANS alias-table bucket, 8 bytes. Field meaning as in ans.rs:17-24:
//   bits  0.. 7 alias_symbol, 8..15 alias_cutoff, 16..31 dist,
//   bits 32..47 alias_offset, 48..63 alias_dist_xor
inline uint64_t pack_ans_bucket(uint32_t alias_symbol, uint32_t alias_cutoff, uint32_t dist,
                                uint32_t alias_offset, uint32_t alias_dist_xor) {
  return uint64_t(alias_symbol & 0xff) | (uint64_t(alias_cutoff & 0xff) << 8) |
         (uint64_t(dist & 0xffff) << 16) | (uint64_t(alias_offset & 0xffff) << 32) |
         (uint64_t(alias_dist_xor & 0xffff) << 48);
}

// Prefix-code LUT entry (u32): bits 0..15 symbol (leaf) or sub-table offset (nested),
// bits 16..23 code length to consume (leaf) or sub-table index bits (nested), bit 31 nested.
constexpr uint32_t kPrefixNested = 0x80000000u;
constexpr uint32_t kPrefixRootBits = 10;  // MAX_TOPLEVEL_BITS, prefix.rs:7

struct PrefixMeta {
  uint32_t table_offset;  // into EntropyCode::prefix_table
  uint32_t root_bits;
};

struct EntropyCode {
  // LZ77 (lib.rs:321-343)
  bool lz77_enabled = false;
  uint32_t lz77_min_symbol = 0, lz77_min_length = 0;
  HybridUintConfig lz_len_conf;
  // clustering (lib.rs:688-749); size = num_dist (+1 when LZ77 is enabled)
  std::vector<uint8_t> cluster_map;
  uint32_t num_clusters = 0;
  bool use_prefix = false;
  uint32_t log_alphabet_size = 0;  // ANS only: 5..8
  std::vector<HybridUintConfig> configs;  // per cluster
  std::vector<int32_t> single_symbol;     // per cluster, -1 if the cluster has >1 symbol
  // ANS: num_clusters << log_alphabet_size buckets
  std::vector<uint64_t> ans_table;
  // prefix: concatenated per-cluster [root table | sub tables]
  std::vector<uint32_t> prefix_table;
  std::vector<PrefixMeta> prefix_meta;

  uint8_t lz_dist_cluster() const { return cluster_map.back(); }
  // lib.rs:460-464 (`single_token`): token known without reading any bit.
  int32_t single_token(uint32_t cluster) const {
    if (lz77_enabled) return -1;
    int32_t s = single_symbol[cluster];
    if (s < 0) return -1;
    return (uint32_t(s) < configs[cluster].split()) ? s : -1;
  }
};

// Decoder::parse (lib.rs:32-42). `num_dist` excludes the LZ77 distance context.
EntropyCode parse_entropy_code(BitReader& br, uint32_t num_dist);
// read_clusters (lib.rs:688-749)
void read_clusters(BitReader& br, uint32_t num_dist, std::vector<uint8_t>* map, uint32_t* num_clusters);

// Host symbol reader. One instance per entropy-coded stream.
class EntropyReader {
 public:
  explicit EntropyReader(const EntropyCode* code) : code_(code) {}
  // Decoder::begin (lib.rs:162-164): reads the 32-bit ANS state.
  void begin(BitReader& br) {
#ifdef JXLB_ENTROPY_TRACE
    entropy_trace_begin(this, br.pos());
#endif
    if (!code_->use_prefix) {
      state_ = br.read(32);
      initial_ = false;
    }
  }
  // Decoder::finalize (lib.rs:171-173)
  bool finalize_ok() const { return code_->use_prefix || state_ == 0x130000u; }
  uint32_t read_symbol(BitReader& br, uint32_t cluster);
  // read_uint_prefilled (lib.rs:572-605)
  static inline uint32_t read_uint(BitReader& br, const HybridUintConfig& c, uint32_t token) {
    uint32_t split = c.split();
    if (token < split) return token;
    uint32_t in_token = c.msb_in_token + c.lsb_in_token;
    uint32_t n = (c.split_exponent - in_token + ((token - split) >> in_token)) & 31;
    uint64_t rest = br.peek(n);
    br.consume(n);
    uint64_t low = token & ((1u << c.lsb_in_token) - 1);
    uint64_t t = token >> c.lsb_in_token;
    t &= (1u << c.msb_in_token) - 1;
    t |= 1u << c.msb_in_token;
    return uint32_t((((t << n) | rest) << c.lsb_in_token) | low);
  }
  // read_varint_with_multiplier_clustered (lib.rs:80-106), incl. LZ77 (lib.rs:476-569)
  uint32_t read_varint_clustered(BitReader& br, uint32_t cluster, uint32_t dist_multiplier) {
    const uint32_t v = read_varint_clustered_untraced(br, cluster, dist_multiplier);
#ifdef JXLB_ENTROPY_TRACE
    entropy_trace_value(this, cluster, v, br.pos());
#endif
    return v;
  }
  uint32_t read_varint(BitReader& br, uint32_t ctx, uint32_t dist_multiplier = 0) {
    return read_varint_clustered(br, code_->cluster_map[ctx], dist_multiplier);
  }
  const EntropyCode& code() const { return *code_; }

 private:
  uint32_t read_varint_clustered_untraced(BitReader& br, uint32_t cluster, uint32_t dist_multiplier);
  const EntropyCode* code_;
  uint32_t state_ = 0;
  bool initial_ = true;
  // LZ77 state (lib.rs:346-352)
  std::vector<uint32_t> window_;
  uint32_t num_to_copy_ = 0, copy_pos_ = 0, num_decoded_ = 0;
};

// read_permutation (permutation.rs:4-43)
std::vector<uint32_t> read_permutation(BitReader& br, EntropyReader& dec, uint32_t size, uint32_t skip);

extern const int8_t kLz77SpecialDistances[120][2];

}  // namespace jxlb
