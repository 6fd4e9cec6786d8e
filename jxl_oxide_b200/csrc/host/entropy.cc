// See entropy.h. Reference: crates/jxl-coding/src/{lib.rs,ans.rs,prefix.rs,permutation.rs}.
#include "entropy.h"

#include <algorithm>
#include <array>

namespace jxlb {

const int8_t kLz77SpecialDistances[120][2] = {  // lib.rs:485-498
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

namespace {

uint32_t add_log2_ceil(uint32_t x) {  // lib.rs:679-685
  if (x >= 0x80000000u) return 32;
  return ceil_log2_nonzero(x + 1);
}

HybridUintConfig parse_uint_config(BitReader& br, uint32_t log_alphabet_size) {  // lib.rs:378-414
  HybridUintConfig c;
  c.split_exponent = br.read(add_log2_ceil(log_alphabet_size));
  if (c.split_exponent != log_alphabet_size) {
    c.msb_in_token = br.read(add_log2_ceil(c.split_exponent));
    JXLB_CHECK(c.msb_in_token <= c.split_exponent, kErrBitstream, "invalid hybrid uint config");
    c.lsb_in_token = br.read(add_log2_ceil(c.split_exponent - c.msb_in_token));
  }
  JXLB_CHECK(c.lsb_in_token + c.msb_in_token <= c.split_exponent, kErrBitstream,
             "invalid hybrid uint config");
  JXLB_CHECK(c.split_exponent < 32, kErrBitstream, "invalid hybrid uint config");
  return c;
}

uint32_t ans_read_u8(BitReader& br) {  // ans.rs:264-271
  if (br.read_bool()) {
    uint32_t n = br.read(3);
    return ((1u << n) + br.read(n)) & 0xff;
  }
  return 0;
}

uint16_t ans_read_logcount(BitReader& br) {  // ans.rs:338-369
  switch (br.read(3)) {
    case 0: return 10;
    case 1:
      for (uint16_t v : {4, 0, 11, 13})
        if (br.read_bool()) return v;
      return 12;
    case 2: return 7;
    case 3: return br.read_bool() ? 1 : 3;
    case 4: return 6;
    case 5: return 8;
    case 6: return 9;
    default: return br.read_bool() ? 2 : 5;
  }
}

// ans.rs:31-262. Appends (1 << log_alphabet_size) buckets to `out`; returns single symbol or -1.
int32_t parse_ans_histogram(BitReader& br, uint32_t log_alphabet_size, std::vector<uint64_t>* out) {
  const uint32_t table_size = 1u << log_alphabet_size;
  const uint32_t log_bucket_size = 12 - log_alphabet_size;
  const uint16_t bucket_size = uint16_t(1u << log_bucket_size);
  std::vector<uint16_t> dist(table_size, 0);
  uint32_t alphabet_size;
  if (br.read_bool()) {
    if (br.read_bool()) {  // binary
      uint32_t v0 = ans_read_u8(br), v1 = ans_read_u8(br);
      JXLB_CHECK(v0 != v1, kErrBitstream, "invalid ANS histogram");
      alphabet_size = std::max(v0, v1) + 1;
      JXLB_CHECK(alphabet_size <= table_size, kErrBitstream, "invalid ANS histogram");
      uint16_t prob = uint16_t(br.read(12));
      dist[v0] = prob;
      dist[v1] = uint16_t((1u << 12) - prob);
    } else {  // unary
      uint32_t val = ans_read_u8(br);
      alphabet_size = val + 1;
      JXLB_CHECK(alphabet_size <= table_size, kErrBitstream, "invalid ANS histogram");
      dist[val] = 1u << 12;
    }
  } else if (br.read_bool()) {  // evenly distributed
    alphabet_size = ans_read_u8(br) + 1;
    JXLB_CHECK(alphabet_size <= table_size, kErrBitstream, "invalid ANS histogram");
    uint32_t base = (1u << 12) / alphabet_size, leftover = (1u << 12) % alphabet_size;
    for (uint32_t i = 0; i < alphabet_size; ++i) dist[i] = uint16_t(i < leftover ? base + 1 : base);
  } else {  // compressed distribution
    uint32_t len = 0;
    while (len < 3 && br.read_bool()) ++len;
    int32_t shift = int32_t(br.read(len) + (1u << len) - 1);
    JXLB_CHECK(shift <= 13, kErrBitstream, "invalid ANS histogram");
    alphabet_size = ans_read_u8(br) + 3;
    JXLB_CHECK(alphabet_size <= table_size, kErrBitstream, "invalid ANS histogram");
    std::vector<std::pair<uint32_t, uint32_t>> repeat_ranges;
    bool have_omit = false;
    uint16_t omit_log = 0;
    uint32_t omit_pos = 0;
    uint32_t idx = 0;
    while (idx < alphabet_size) {
      dist[idx] = ans_read_logcount(br);
      if (dist[idx] == 13) {
        uint32_t repeat_count = ans_read_u8(br) + 4;
        JXLB_CHECK(idx + repeat_count <= alphabet_size, kErrBitstream, "invalid ANS histogram");
        repeat_ranges.push_back({idx, idx + repeat_count});
        idx += repeat_count;
        continue;
      }
      if (have_omit) {
        if (dist[idx] > omit_log) {
          omit_log = dist[idx];
          omit_pos = idx;
        }
      } else {
        have_omit = true;
        omit_log = dist[idx];
        omit_pos = idx;
      }
      ++idx;
      JXLB_CHECK(!br.overrun(), kErrEof, "unexpected end of bitstream");
    }
    JXLB_CHECK(have_omit, kErrBitstream, "invalid ANS histogram");
    JXLB_CHECK(!(omit_pos + 1 < table_size && dist[omit_pos + 1] == 13), kErrBitstream,
               "invalid ANS histogram");
    size_t rr = 0;
    uint32_t acc = 0;
    uint16_t prev_dist = 0;
    for (uint32_t i = 0; i < table_size; ++i) {
      uint16_t& code = dist[i];
      if (rr < repeat_ranges.size() && repeat_ranges[rr].first <= i) {
        if (repeat_ranges[rr].second == i) {
          ++rr;
        } else {
          code = prev_dist;
          acc += code;
          JXLB_CHECK(acc <= (1u << 12), kErrBitstream, "invalid ANS histogram");
          continue;
        }
      }
      if (code == 0) {
        prev_dist = 0;
        continue;
      }
      if (i == omit_pos) {
        prev_dist = 0;
        continue;
      }
      if (code > 1) {
        int32_t zeros = int32_t(code) - 1;
        int32_t bitcount = std::min(std::max(shift - ((12 - zeros) >> 1), 0), zeros);
        code = uint16_t((1u << zeros) + (br.read(uint32_t(bitcount)) << (zeros - bitcount)));
      }
      prev_dist = code;
      acc += code;
      JXLB_CHECK(acc <= (1u << 12), kErrBitstream, "invalid ANS histogram");
    }
    dist[omit_pos] = uint16_t((1u << 12) - acc);
  }
  JXLB_CHECK(!br.overrun(), kErrEof, "unexpected end of bitstream");

  // Single-symbol distribution (ans.rs:170-190)
  for (uint32_t s = 0; s < table_size; ++s) {
    if (dist[s] == (1u << 12)) {
      for (uint32_t i = 0; i < table_size; ++i)
        out->push_back(pack_ans_bucket(s, 0, dist[i], bucket_size * i, dist[i] ^ (1u << 12)));
      return int32_t(s);
    }
  }

  // Alias table (ans.rs:192-254); stack order of under/overfull pairing matters.
  struct Working {
    uint16_t dist, alias_symbol, alias_offset, alias_cutoff;
  };
  std::vector<Working> b(table_size);
  std::vector<uint32_t> underfull, overfull;
  for (uint32_t i = 0; i < table_size; ++i) {
    b[i] = {dist[i], uint16_t(i < alphabet_size ? i : 0), 0, dist[i]};
    if (dist[i] < bucket_size) underfull.push_back(i);
    else if (dist[i] > bucket_size) overfull.push_back(i);
  }
  while (!overfull.empty() && !underfull.empty()) {
    uint32_t o = overfull.back(), u = underfull.back();
    overfull.pop_back();
    underfull.pop_back();
    uint16_t by = uint16_t(bucket_size - b[u].alias_cutoff);
    b[o].alias_cutoff = uint16_t(b[o].alias_cutoff - by);
    b[u].alias_symbol = uint16_t(o);
    b[u].alias_offset = b[o].alias_cutoff;
    if (b[o].alias_cutoff < bucket_size) underfull.push_back(o);
    else if (b[o].alias_cutoff > bucket_size) overfull.push_back(o);
  }
  for (uint32_t i = 0; i < table_size; ++i) {
    if (b[i].alias_cutoff == bucket_size) {
      out->push_back(pack_ans_bucket(i, 0, b[i].dist, 0, 0));
    } else {
      out->push_back(pack_ans_bucket(b[i].alias_symbol, b[i].alias_cutoff, b[i].dist,
                                     uint16_t(b[i].alias_offset - b[i].alias_cutoff),
                                     b[i].dist ^ b[b[i].alias_symbol].dist));
    }
  }
  return -1;
}

// Builds a two-level LUT from canonical (Brotli) code lengths; equivalent in decoded symbols to
// prefix.rs:28-116. Entries are bit-reversed because codes are read LSB-first.
struct PrefixBuild {
  std::vector<uint32_t> table;
  uint32_t root_bits = 0;
  int32_t single = -1;
};

PrefixBuild prefix_single(uint32_t symbol) {
  PrefixBuild p;
  p.root_bits = 0;
  p.table = {symbol & 0xffff};  // len 0
  p.single = int32_t(symbol);
  return p;
}

uint32_t bit_reverse(uint32_t v, uint32_t n) {
  uint32_t r = 0;
  for (uint32_t i = 0; i < n; ++i) r |= ((v >> i) & 1) << (n - 1 - i);
  return r;
}

PrefixBuild prefix_from_lengths(const std::vector<uint8_t>& lengths) {
  uint32_t max_len = 0;
  std::array<uint32_t, 16> count{};
  for (uint8_t l : lengths) {
    JXLB_CHECK(l <= 15, kErrBitstream, "invalid prefix code");
    if (l) {
      ++count[l];
      max_len = std::max<uint32_t>(max_len, l);
    }
  }
  JXLB_CHECK(max_len > 0, kErrBitstream, "invalid prefix code");
  uint64_t kraft = 0;
  for (uint32_t l = 1; l <= 15; ++l) kraft += uint64_t(count[l]) << (15 - l);
  JXLB_CHECK(kraft == (1u << 15), kErrBitstream, "invalid prefix code (not complete)");
  // canonical codes
  std::array<uint32_t, 17> next_code{};
  uint32_t code = 0;
  for (uint32_t l = 1; l <= 15; ++l) {
    code = (code + count[l - 1]) << 1;
    next_code[l] = code;
  }
  PrefixBuild p;
  p.root_bits = std::min(max_len, kPrefixRootBits);
  const uint32_t root_size = 1u << p.root_bits;
  p.table.assign(root_size, 0);
  // first pass: per-root-prefix maximum length for long codes
  struct Sym {
    uint32_t sym, len, rev;
  };
  std::vector<Sym> syms;
  for (uint32_t s = 0; s < lengths.size(); ++s) {
    uint32_t l = lengths[s];
    if (!l) continue;
    uint32_t c = next_code[l]++;
    syms.push_back({s, l, bit_reverse(c, l)});
  }
  std::vector<uint32_t> sub_bits(root_size, 0);
  for (const Sym& s : syms)
    if (s.len > p.root_bits) {
      uint32_t r = s.rev & (root_size - 1);
      sub_bits[r] = std::max(sub_bits[r], s.len - p.root_bits);
    }
  std::vector<uint32_t> sub_offset(root_size, 0);
  uint32_t total = root_size;
  for (uint32_t r = 0; r < root_size; ++r)
    if (sub_bits[r]) {
      sub_offset[r] = total - root_size;
      JXLB_CHECK(sub_offset[r] <= 0xffff, kErrBitstream, "prefix table too large");
      p.table[r] = kPrefixNested | (sub_bits[r] << 16) | sub_offset[r];
      total += 1u << sub_bits[r];
    }
  p.table.resize(total, 0);
  for (const Sym& s : syms) {
    uint32_t entry = (s.len << 16) | s.sym;
    if (s.len <= p.root_bits) {
      for (uint32_t i = s.rev; i < root_size; i += 1u << s.len) p.table[i] = entry;
    } else {
      uint32_t r = s.rev & (root_size - 1);
      uint32_t hi = s.rev >> p.root_bits, hl = s.len - p.root_bits;
      uint32_t base = root_size + sub_offset[r];
      for (uint32_t i = hi; i < (1u << sub_bits[r]); i += 1u << hl) p.table[base + i] = entry;
    }
  }
  return p;
}

inline uint32_t prefix_lookup(const uint32_t* table, uint32_t root_bits, BitReader& br) {
  uint32_t peeked = br.peek(15);
  uint32_t e = table[peeked & ((1u << root_bits) - 1)];
  if (e & kPrefixNested) {
    uint32_t sb = (e >> 16) & 0xff;
    e = table[(1u << root_bits) + (e & 0xffff) + ((peeked >> root_bits) & ((1u << sb) - 1))];
  }
  br.consume((e >> 16) & 0xff);
  return e & 0xffff;
}

PrefixBuild parse_prefix_simple(BitReader& br, uint32_t alphabet_size) {  // prefix.rs:150-207
  uint32_t alphabet_bits = ceil_log2_nonzero(alphabet_size);
  uint32_t nsym = br.read(2) + 1;
  uint32_t syms[4] = {0, 0, 0, 0};
  uint8_t lens[4] = {0, 0, 0, 0};
  if (nsym == 1) {
    uint32_t sym = br.read(alphabet_bits);
    JXLB_CHECK(sym < alphabet_size, kErrBitstream, "invalid prefix code");
    return prefix_single(sym);
  } else if (nsym == 2) {
    syms[2] = br.read(alphabet_bits);
    syms[3] = br.read(alphabet_bits);
    lens[2] = lens[3] = 1;
  } else if (nsym == 3) {
    for (int i = 1; i < 4; ++i) syms[i] = br.read(alphabet_bits);
    lens[1] = 1;
    lens[2] = lens[3] = 2;
  } else {
    for (int i = 0; i < 4; ++i) syms[i] = br.read(alphabet_bits);
    if (br.read_bool()) {
      lens[0] = 1, lens[1] = 2, lens[2] = 3, lens[3] = 3;
    } else {
      lens[0] = lens[1] = lens[2] = lens[3] = 2;
    }
  }
  std::vector<uint8_t> code_lengths(alphabet_size, 0);
  for (int i = 0; i < 4; ++i) {
    JXLB_CHECK(syms[i] < alphabet_size, kErrBitstream, "invalid prefix code");
    code_lengths[syms[i]] = lens[i];
  }
  return prefix_from_lengths(code_lengths);
}

PrefixBuild parse_prefix_complex(BitReader& br, uint32_t alphabet_size, uint32_t hskip) {  // prefix.rs:209-329
  static const uint32_t kOrder[18] = {1, 2, 3, 4, 0, 5, 17, 6, 16, 7, 8, 9, 10, 11, 12, 13, 14, 15};
  std::vector<uint8_t> clcl(18, 0);
  uint32_t bitacc = 0, nonzero_count = 0, nonzero_sym = 0;
  for (uint32_t k = hskip; k < 18; ++k) {
    uint32_t idx = kOrder[k];
    uint32_t base = br.read_u32({0, 0}, {4, 0}, {3, 0}, {8, 0});
    uint32_t len = base;
    if (base == 8) len = br.read_bool() ? (br.read_bool() ? 5 : 1) : 2;
    clcl[idx] = uint8_t(len);
    if (len != 0) {
      ++nonzero_count;
      nonzero_sym = idx;
      bitacc += 32u >> len;
      if (bitacc == 32) break;
      JXLB_CHECK(bitacc < 32, kErrBitstream, "invalid prefix code");
    }
  }
  PrefixBuild cl;
  if (nonzero_count == 1) {
    cl = prefix_single(nonzero_sym);
  } else {
    JXLB_CHECK(bitacc == 32, kErrBitstream, "invalid prefix code");
    // with_code_lengths over the 18-symbol alphabet (max len 5): scale Kraft check to 15 bits
    cl = prefix_from_lengths(clcl);
  }
  std::vector<uint8_t> code_lengths(alphabet_size, 0);
  uint32_t acc = 0;
  uint32_t prev_sym = 8, last_nonzero_sym = 8;
  size_t last_repeat_count = 0, repeat_count = 0;
  uint8_t repeat_sym = 0;
  for (uint32_t i = 0; i < alphabet_size; ++i) {
    uint8_t& len = code_lengths[i];
    if (repeat_count > 0) {
      len = repeat_sym;
      --repeat_count;
    } else {
      uint32_t sym = prefix_lookup(cl.table.data(), cl.root_bits, br);
      if (sym == 0) {
      } else if (sym <= 15) {
        len = uint8_t(sym);
        last_nonzero_sym = sym;
      } else if (sym == 16) {
        repeat_count = br.read(2) + 3;
        if (prev_sym == 16) {
          repeat_count += last_repeat_count * 3 - 8;
          last_repeat_count += repeat_count;
        } else {
          last_repeat_count = repeat_count;
        }
        repeat_sym = uint8_t(last_nonzero_sym);
        len = repeat_sym;
        --repeat_count;
      } else {
        repeat_count = br.read(3) + 3;
        if (prev_sym == 17) {
          repeat_count += last_repeat_count * 7 - 16;
          last_repeat_count += repeat_count;
        } else {
          last_repeat_count = repeat_count;
        }
        repeat_sym = 0;
        len = 0;
        --repeat_count;
      }
      prev_sym = sym;
      JXLB_CHECK(!br.overrun(), kErrEof, "unexpected end of bitstream");
    }
    if (len != 0) {
      acc += 1u << (15 - len);
      JXLB_CHECK(acc <= (1u << 15), kErrBitstream, "invalid prefix code");
      if (acc == (1u << 15) && repeat_count == 0) break;
    }
  }
  JXLB_CHECK(acc == (1u << 15) && repeat_count == 0, kErrBitstream, "invalid prefix code");
  return prefix_from_lengths(code_lengths);
}

PrefixBuild parse_prefix_histogram(BitReader& br, uint32_t alphabet_size) {  // prefix.rs:134-148
  if (alphabet_size == 1) return prefix_single(0);
  JXLB_CHECK(alphabet_size <= (1u << 15), kErrBitstream, "prefix alphabet too large");
  uint32_t hskip = br.read(2);
  if (hskip == 1) return parse_prefix_simple(br, alphabet_size);
  return parse_prefix_complex(br, alphabet_size, hskip);
}

EntropyCode parse_inner(BitReader& br, uint32_t num_dist, EntropyCode code) {  // lib.rs:424-470
  read_clusters(br, num_dist, &code.cluster_map, &code.num_clusters);
  code.use_prefix = br.read_bool();
  code.log_alphabet_size = code.use_prefix ? 15 : br.read(2) + 5;
  for (uint32_t i = 0; i < code.num_clusters; ++i)
    code.configs.push_back(parse_uint_config(br, code.log_alphabet_size));
  code.single_symbol.assign(code.num_clusters, -1);
  if (code.use_prefix) {
    std::vector<uint32_t> counts(code.num_clusters);
    for (uint32_t i = 0; i < code.num_clusters; ++i) {
      uint32_t count = 1;
      if (br.read_bool()) {
        uint32_t n = br.read(4);
        count = 1 + (1u << n) + br.read(n);
      }
      JXLB_CHECK(count <= (1u << 15), kErrBitstream, "invalid prefix histogram");
      counts[i] = count;
    }
    for (uint32_t i = 0; i < code.num_clusters; ++i) {
      PrefixBuild p = parse_prefix_histogram(br, counts[i]);
      code.prefix_meta.push_back({uint32_t(code.prefix_table.size()), p.root_bits});
      code.prefix_table.insert(code.prefix_table.end(), p.table.begin(), p.table.end());
      code.single_symbol[i] = p.single;
      JXLB_CHECK(!br.overrun(), kErrEof, "unexpected end of bitstream");
    }
  } else {
    for (uint32_t i = 0; i < code.num_clusters; ++i) {
      code.single_symbol[i] = parse_ans_histogram(br, code.log_alphabet_size, &code.ans_table);
    }
  }
  JXLB_CHECK(!br.overrun(), kErrEof, "unexpected end of bitstream");
  return code;
}

}  // namespace

EntropyCode parse_entropy_code(BitReader& br, uint32_t num_dist) {
  EntropyCode code;
  code.lz77_enabled = br.read_bool();
  if (code.lz77_enabled) {  // lib.rs:321-343
    code.lz77_min_symbol = br.read_u32({224, 0}, {512, 0}, {4096, 0}, {8, 15});
    code.lz77_min_length = br.read_u32({3, 0}, {4, 0}, {5, 2}, {9, 8});
    code.lz_len_conf = parse_uint_config(br, 8);
    num_dist += 1;
  }
  return parse_inner(br, num_dist, std::move(code));
}

void read_clusters(BitReader& br, uint32_t num_dist, std::vector<uint8_t>* map, uint32_t* num_clusters) {
  map->clear();
  if (num_dist == 1) {
    map->push_back(0);
    *num_clusters = 1;
    return;
  }
  if (br.read_bool()) {  // simple
    uint32_t nbits = br.read(2);
    for (uint32_t i = 0; i < num_dist; ++i) map->push_back(uint8_t(br.read(nbits)));
  } else {
    bool use_mtf = br.read_bool();
    EntropyCode nested;
    if (num_dist <= 2) {  // parse_assume_no_lz77 (lib.rs:44-55)
      JXLB_CHECK(!br.read_bool(), kErrBitstream, "LZ77 not allowed here");
      nested = parse_inner(br, 1, EntropyCode());
    } else {
      nested = parse_entropy_code(br, 1);
    }
    EntropyReader dec(&nested);
    dec.begin(br);
    for (uint32_t i = 0; i < num_dist; ++i) {
      uint32_t b = dec.read_varint(br, 0);
      JXLB_CHECK(b < 256, kErrBitstream, "invalid cluster index");
      map->push_back(uint8_t(b));
      JXLB_CHECK(!br.overrun(), kErrEof, "unexpected end of bitstream");
    }
    JXLB_CHECK(dec.finalize_ok(), kErrBitstream, "invalid ANS stream (cluster map)");
    if (use_mtf) {
      uint8_t mtf[256];
      for (int i = 0; i < 256; ++i) mtf[i] = uint8_t(i);
      for (uint8_t& c : *map) {
        uint32_t idx = c;
        c = mtf[idx];
        for (uint32_t k = idx; k > 0; --k) mtf[k] = mtf[k - 1];
        mtf[0] = c;
      }
    }
  }
  JXLB_CHECK(!br.overrun(), kErrEof, "unexpected end of bitstream");
  uint32_t maxc = 0;
  bool seen[256] = {};
  for (uint8_t c : *map) {
    maxc = std::max<uint32_t>(maxc, c);
    seen[c] = true;
  }
  for (uint32_t c = 0; c <= maxc; ++c)
    JXLB_CHECK(seen[c], kErrBitstream, "distribution cluster map has a hole");
  *num_clusters = maxc + 1;
}

uint32_t EntropyReader::read_symbol(BitReader& br, uint32_t cluster) {
  const EntropyCode& c = *code_;
  if (c.use_prefix) {
    const PrefixMeta& m = c.prefix_meta[cluster];
    return prefix_lookup(c.prefix_table.data() + m.table_offset, m.root_bits, br);
  }
  if (initial_) {  // lazy init (lib.rs:636-639)
    state_ = br.read(32);
    initial_ = false;
  }
  // ans.rs:276-330
  const uint32_t log_bucket = 12 - c.log_alphabet_size;
  uint32_t idx = state_ & 0xfff;
  uint32_t i = idx >> log_bucket;
  uint32_t pos = idx & ((1u << log_bucket) - 1);
  uint64_t b = c.ans_table[(size_t(cluster) << c.log_alphabet_size) + i];
  uint32_t alias_symbol = uint32_t(b & 0xff);
  uint32_t alias_cutoff = uint32_t((b >> 8) & 0xff);
  uint32_t dist = uint32_t((b >> 16) & 0xffff);
  bool map_to_alias = pos >= alias_cutoff;
  uint64_t cond = map_to_alias ? b : 0;
  uint32_t offset = uint32_t(cond >> 32) & 0xffff;
  uint32_t dist_xor = uint32_t(cond >> 48);
  dist ^= dist_xor;
  uint32_t symbol = map_to_alias ? alias_symbol : i;
  offset += pos;
  uint32_t next = (state_ >> 12) * dist + offset;
  if (next < (1u << 16)) {
    next = (next << 16) | br.peek(16);
    br.consume(16);
  }
  state_ = next;
  return symbol;
}

uint32_t EntropyReader::read_varint_clustered_untraced(BitReader& br, uint32_t cluster, uint32_t dist_multiplier) {
  const EntropyCode& c = *code_;
  if (!c.lz77_enabled) {
    uint32_t token = read_symbol(br, cluster);
    return read_uint(br, c.configs[cluster], token);
  }
  uint32_t r;
  if (num_to_copy_ > 0) {
    r = window_[copy_pos_ & 0xfffff];
    ++copy_pos_;
    --num_to_copy_;
  } else {
    uint32_t token = read_symbol(br, cluster);
    if (token >= c.lz77_min_symbol) {
      JXLB_CHECK(num_decoded_ != 0, kErrBitstream, "LZ77 repeat before any symbol");
      uint32_t lz_cluster = c.lz_dist_cluster();
      uint32_t n = read_uint(br, c.lz_len_conf, token - c.lz77_min_symbol);
      JXLB_CHECK(n <= 0xffffffffu - c.lz77_min_length, kErrBitstream, "invalid LZ77 symbol");
      num_to_copy_ = n + c.lz77_min_length;
      uint32_t dtoken = read_symbol(br, lz_cluster);
      uint32_t distance = read_uint(br, c.configs[lz_cluster], dtoken);
      if (dist_multiplier == 0) {
      } else if (distance < 120) {
        int32_t off = kLz77SpecialDistances[distance][0], d = kLz77SpecialDistances[distance][1];
        int32_t dd = off + int32_t(dist_multiplier) * d;
        distance = uint32_t(std::max(dd - 1, 0));
      } else {
        distance -= 120;
      }
      distance = std::min(std::min<uint32_t>((1u << 20) - 1, distance) + 1, num_decoded_);
      copy_pos_ = num_decoded_ - distance;
      r = window_[copy_pos_ & 0xfffff];
      ++copy_pos_;
      --num_to_copy_;
    } else {
      r = read_uint(br, c.configs[cluster], token);
    }
  }
  size_t off = num_decoded_ & 0xfffff;
  if (window_.size() <= off) window_.push_back(r);
  else window_[off] = r;
  ++num_decoded_;
  return r;
}

std::vector<uint32_t> read_permutation(BitReader& br, EntropyReader& dec, uint32_t size, uint32_t skip) {
  auto ctx = [](uint32_t x) { return std::min<uint32_t>(add_log2_ceil(x), 7); };
  uint32_t end = dec.read_varint(br, ctx(size));
  JXLB_CHECK(end <= size - skip, kErrBitstream, "invalid permutation");
  std::vector<uint32_t> lehmer(end);
  uint32_t prev = 0;
  for (uint32_t i = 0; i < end; ++i) {
    lehmer[i] = dec.read_varint(br, ctx(prev));
    JXLB_CHECK(lehmer[i] < size - skip - i, kErrBitstream, "invalid permutation");
    prev = lehmer[i];
    JXLB_CHECK(!br.overrun(), kErrEof, "unexpected end of bitstream");
  }
  std::vector<uint32_t> temp;
  for (uint32_t i = skip; i < size; ++i) temp.push_back(i);
  std::vector<uint32_t> perm;
  perm.reserve(size);
  for (uint32_t i = 0; i < skip; ++i) perm.push_back(i);
  for (uint32_t l : lehmer) {
    perm.push_back(temp[l]);
    temp.erase(temp.begin() + l);
  }
  perm.insert(perm.end(), temp.begin(), temp.end());
  return perm;
}

}  // namespace jxlb
