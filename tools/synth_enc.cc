// tools/synth_enc — minimal JPEG XL *bitstream writer* for synthetic VarDCT benchmark frames.
//
// Neither the reference (a decoder) nor this environment has a JPEG XL encoder, so bench.py's
// "7680x4320 VarDCT d1.0" workload is produced here: a seeded generator draws a varblock layout,
// quantised LF values, per-block multipliers / sharpness / chroma-from-luma factors and sparse
// Laplacian HF coefficients with the statistics of a libjxl d1.0 stream (~0.9 bit/px, quantiser
// global_scale 5111 / quant_lf 17 as in decode/benchmark-data/starrail.d1-e6.jxl), and writes them
// with the codestream syntax the decoder parses: all-default image metadata (XYB, sRGB), all-default
// frame header (VarDCT, Gaborish on, EPF 2 iterations), multi-section TOC, global MA tree, LF
// groups (weighted-predictor coded LF like libjxl, or --lf-gradient), default dequant matrices and
// coefficient orders, one HF preset, ANS everywhere.
// The entropy-code headers it writes are read back with the product's own parser to derive the
// exact alias tables, so encoder and decoder cannot disagree about symbol mapping.
// For tests, --all-types puts every one of the 27 transform types into the frame (the largest ones also in the partial
// groups at the right / bottom edges and next to LF-group boundaries), --only-type T tiles the frame with one type, and
// --dump-blocks FILE writes the varblock layout; without these flags the output does not change. A VarDCT frame of one
// group (at most 256 x 256, down to 1 x 1) is written with a single TOC entry. --no-gaborish turns Gaborish off;
// --modular-filters SIGMA gives a --modular frame Gaborish and --epf-iters EPF iterations with constant sigma SIGMA.
// --sharpness-cell N makes the sharpness map (and so the EPF sigma grid) change every N blocks instead of 16.
// --hf-lz77 rle|match codes the HF passes with LZ77 (HfLz77 below); everything else is written as without it, and the
// number of values the decoder takes from copies goes to stderr. --extra TYPE:BITS:DIM_SHIFT:EC_UPSAMPLING (repeatable)
// adds extra channels at their coded sizes to a VarDCT or --modular frame; --ycbcr and --upsampling make --modular frames
// with chroma-subsampled Cb, Y, Cr or a reduced colour resolution (encode_channels). --ycbcr also makes a VarDCT frame
// laid out like a JPEG transcode: Cb, Y, Cr with jpeg_upsampling, DCT8 in every cell, no chroma from luma,
// skip_adaptive_lf_smoothing, each channel's LF and HF at its shifted grid; it combines with --hf-lz77, and
// --dump-coeffs FILE writes the HF coefficients of any VarDCT frame. --upsampling K also codes a VarDCT
// frame at ceil(W / K) x ceil(H / K), and --noise / --noise-zero, --splines N and --dangling-patch give a VarDCT frame
// those LfGlobal features (write_features). --code FORM writes every entropy code of the file in one form of the
// entropy-code syntax (prefix, ans-forms, configs, clusters; see g_code) and reports the branches it reached.
//
// Not part of the product; not a general-purpose encoder (it does not transform an input image).
#include <algorithm>
#include <array>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <random>
#include <string>
#include <vector>

#include "../jxl_oxide_b200/csrc/host/entropy.h"
#include "../jxl_oxide_b200/csrc/host/frame_syntax.h"

using namespace jxlb;

namespace {

struct BitWriter {
  std::vector<uint8_t> bytes;
  uint64_t acc = 0;
  int nbits = 0;
  size_t total_bits = 0;
  void write(int n, uint64_t v) {
    while (n > 0) {
      int take = std::min(n, 32);
      acc |= (v & ((1ull << take) - 1)) << nbits;
      nbits += take;
      total_bits += take;
      v >>= take;
      n -= take;
      while (nbits >= 8) {
        bytes.push_back(uint8_t(acc));
        acc >>= 8;
        nbits -= 8;
      }
    }
  }
  void pad() {
    if (nbits) write(8 - nbits, 0);
  }
  void append(const BitWriter& o) {  // o must be byte aligned, and so must we
    bytes.insert(bytes.end(), o.bytes.begin(), o.bytes.end());
    total_bits += o.total_bits;
  }
  void append_bits(const BitWriter& o) {  // any alignment on either side
    for (uint8_t b : o.bytes) write(8, b);
    if (o.nbits) write(o.nbits, o.acc);
  }
};

// binary16 of a normal value (restoration-filter parameters)
uint16_t to_f16(float f) {
  int e;
  const float m = std::frexp(std::fabs(f), &e);  // |f| = m * 2^e, m in [0.5, 1)
  int E = e - 1 + 15;
  uint32_t frac = uint32_t(std::lround((m * 2.0f - 1.0f) * 1024.0f));
  if (frac == 1024) frac = 0, ++E;
  if (f == 0.0f || E < 1 || E > 30) fprintf(stderr, "%g is not a normal binary16 value\n", f), exit(2);
  return uint16_t((f < 0 ? 0x8000u : 0u) | uint32_t(E) << 10 | frac);
}

// U32 with explicit selector
void write_u32(BitWriter& w, int sel, int bits, uint32_t v) {
  w.write(2, uint64_t(sel));
  if (bits) w.write(bits, v);
}

struct Token {
  uint32_t ctx, value;
};

// A symbol as the entropy coder writes it: its context, its token and the extra bits of its hybrid-uint tail.
struct Sym {
  uint32_t ctx, tok, nbits, bits;
};

struct UintConfig {
  uint32_t split_exp, msb, lsb;
};
// HybridUintConfig (4, 2, 0): the configuration libjxl uses for these streams
const uint32_t kSplitExp = 4, kMsb = 2, kLsb = 0;
void tokenize_with(const UintConfig& c, uint32_t v, uint32_t* token, uint32_t* nbits, uint32_t* bits) {
  const uint32_t split = 1u << c.split_exp;
  if (v < split) {
    *token = v;
    *nbits = 0;
    *bits = 0;
    return;
  }
  uint32_t n = 31 - uint32_t(__builtin_clz(v));
  uint32_t m = v - (1u << n);
  *token = split + ((n - c.split_exp) << (c.msb + c.lsb)) + ((m >> (n - c.msb)) << c.lsb) + (m & ((1u << c.lsb) - 1));
  *nbits = n - c.msb - c.lsb;
  *bits = (m >> c.lsb) & ((1u << *nbits) - 1);
}
void tokenize(uint32_t v, uint32_t* token, uint32_t* nbits, uint32_t* bits) {
  tokenize_with({kSplitExp, kMsb, kLsb}, v, token, nbits, bits);
}
std::vector<Sym> to_syms(const std::vector<Token>& tokens) {
  std::vector<Sym> s(tokens.size());
  for (size_t i = 0; i < tokens.size(); ++i) {
    s[i].ctx = tokens[i].ctx;
    tokenize(tokens[i].value, &s[i].tok, &s[i].nbits, &s[i].bits);
  }
  return s;
}

// LZ77 parameters of an entropy code (lib.rs:321-343) with the U32 selectors they are written with.
struct Lz77Header {
  uint32_t min_symbol, min_length;
  int symbol_sel, length_sel;  // min_symbol: 224, 512, 4096, 8 + u(15); min_length: 3, 4, 5 + u(2), 9 + u(8)
  UintConfig len_cfg;
};

uint32_t add_log2_ceil(uint32_t x) { return ceil_log2_nonzero(x + 1); }

void write_u8(BitWriter& w, uint32_t v) {  // inverse of ans.rs read_u8
  if (v == 0) {
    w.write(1, 0);
    return;
  }
  w.write(1, 1);
  uint32_t n = 31 - uint32_t(__builtin_clz(v));
  w.write(3, n);
  w.write(int(n), v - (1u << n));
}

void write_logcount(BitWriter& w, uint32_t l) {  // inverse of ans.rs read_prefix
  switch (l) {
    case 10: w.write(3, 0); break;
    case 4: w.write(3, 1), w.write(1, 1); break;
    case 0: w.write(3, 1), w.write(1, 0), w.write(1, 1); break;
    case 11: w.write(3, 1), w.write(2, 0), w.write(1, 1); break;
    case 13: w.write(3, 1), w.write(3, 0), w.write(1, 1); break;
    case 12: w.write(3, 1), w.write(4, 0); break;
    case 7: w.write(3, 2); break;
    case 1: w.write(3, 3), w.write(1, 1); break;
    case 3: w.write(3, 3), w.write(1, 0); break;
    case 6: w.write(3, 4); break;
    case 8: w.write(3, 5); break;
    case 9: w.write(3, 6); break;
    case 2: w.write(3, 7), w.write(1, 1); break;
    case 5: w.write(3, 7), w.write(1, 0); break;
    default: fprintf(stderr, "bad logcount %u\n", l), exit(1);
  }
}

std::vector<uint32_t> normalize(const std::vector<uint64_t>& freq) {
  uint64_t total = 0;
  for (uint64_t f : freq) total += f;
  std::vector<uint32_t> c(freq.size(), 0);
  if (total == 0) {
    c[0] = 4096;
    return c;
  }
  int64_t sum = 0;
  size_t largest = 0;
  for (size_t i = 0; i < freq.size(); ++i) {
    if (!freq[i]) continue;
    c[i] = uint32_t(std::max<uint64_t>(1, (freq[i] * 4096 + total / 2) / total));
    sum += c[i];
    if (c[i] > c[largest]) largest = i;
  }
  // fix the sum on the largest entry (keeping it >= 1)
  int64_t diff = 4096 - sum;
  while (diff != 0) {
    // spread over the biggest entries
    size_t best = 0;
    for (size_t i = 0; i < c.size(); ++i)
      if (c[i] > c[best]) best = i;
    int64_t d = diff > 0 ? diff : std::max<int64_t>(diff, -int64_t(c[best] - 1));
    if (d == 0) break;
    c[best] = uint32_t(int64_t(c[best]) + d);
    diff -= d;
  }
  return c;
}

void write_ans_histogram(BitWriter& w, const std::vector<uint32_t>& counts) {
  int nz = 0, last = 0, only = 0;
  for (size_t i = 0; i < counts.size(); ++i)
    if (counts[i]) {
      ++nz;
      last = int(i);
      only = int(i);
    }
  if (nz == 1) {
    w.write(1, 1);  // simple
    w.write(1, 0);  // unary
    write_u8(w, uint32_t(only));
    return;
  }
  w.write(1, 0);
  w.write(1, 0);        // not evenly distributed
  w.write(3, 7);        // len = 3 (three ones, loop stops)
  w.write(3, 6);        // shift = 6 + 8 - 1 = 13
  uint32_t alphabet_size = std::max(3, last + 1);
  write_u8(w, alphabet_size - 3);
  std::vector<uint32_t> logc(alphabet_size, 0);
  uint32_t max_log = 0;
  int omit = -1;
  for (uint32_t i = 0; i < alphabet_size; ++i) {
    uint32_t c = i < counts.size() ? counts[i] : 0;
    logc[i] = c ? (32 - uint32_t(__builtin_clz(c))) : 0;
    if (logc[i] > max_log) {
      max_log = logc[i];
      omit = int(i);
    }
  }
  for (uint32_t i = 0; i < alphabet_size; ++i) write_logcount(w, logc[i]);
  for (uint32_t i = 0; i < alphabet_size; ++i) {
    if (int(i) == omit || logc[i] <= 1) continue;
    uint32_t zeros = logc[i] - 1;
    int bitcount = std::min<int>(std::max<int>(13 - int((12 - zeros) >> 1), 0), int(zeros));
    w.write(bitcount, (counts[i] - (1u << zeros)) >> (zeros - uint32_t(bitcount)));
  }
}

// ---- --code FORM: every entropy code of the file (MA tree, cluster maps, Modular channels, LF and HF) is written in
// one form of the entropy-code syntax, from the spec semantics of jxl-coding (ans.rs, prefix.rs, lib.rs):
//   prefix     prefix codes: length-limited (15) Huffman; clusters with at most 4 symbols in the simple form (NSYM 1-4,
//              both tree_select values), the others in the complex form (hskip 0, 2 and 3 in turn, repeat codes 16 and
//              17); in each code the cluster with the most symbols (16 or more) gets a chain-shaped code up to 15 bits.
//   ans-forms  ANS at log alphabet 6, 7, 8 in turn; clusters of one or two symbols in the simple forms, the others
//              flat, RLE-coded (logcount 13) or in the general form with shift 0..13 in turn.
//   configs    ANS at log alphabet 8; each cluster takes the next hybrid-uint config of kFormConfigs that can code its
//              values within the alphabet.
//   clusters   ANS at log alphabet 8; context i goes to cluster i mod K: K of 65 to 256 in a complex cluster map (with
//              and without move-to-front) where there are that many contexts, otherwise a simple map with nbits 0..3.
// The writer builds its own tables and checks that parse_entropy_code reads back exactly what was written (exit 1
// otherwise); FormReport lists the branches reached and goes to stderr as one "code-form:" line.
std::string g_code;
// --corrupt KIND: one invalid stream or code in the file, the rest as without it (tests of rejected streams):
//   ans-state        the last Modular group's stream, or the first HF group's, is encoded from end state 0x130001: every
//                    value decodes as written, but the stream does not end in state 0x130000 (lib.rs:176-180)
//   truncate         the last section is cut to half its size, the TOC saying so: its stream ends early (with --code
//                    prefix, nothing but the end of the data tells)
//   oversub-clcl     the first complex prefix code's code-length code has its last length one shorter: over-subscribed
//                    (prefix.rs:246-258)
//   oversub-lengths  the first complex prefix code's last code length is one shorter: over-subscribed (prefix.rs:317-329)
//   ans-sum          the first ANS histogram of a --code form is written with explicit counts summing past 4096
//                    (ans.rs:172-175)
std::string g_corrupt;
bool g_corrupt_done = false;  // applied (once per file)
bool g_flip_state = false;    // ans-state: set just before the stream to corrupt is written
uint32_t g_code_seed = 0;  // --seed
uint32_t g_code_turn = 0;  // advances with every choice the forms cycle through

const UintConfig kFormConfigs[] = {{0, 0, 0}, {1, 0, 1}, {2, 1, 1}, {3, 0, 3}, {4, 2, 2}, {5, 1, 3}, {6, 3, 3},
                                   {7, 0, 7}, {8, 0, 0}, {1, 1, 0}, {4, 2, 0}, {5, 0, 0}, {3, 1, 0}, {6, 0, 1}};

struct FormReport {
  uint64_t codes = 0, prefix_codes = 0, prefix_clusters = 0, single_symbol = 0, nsym[5] = {}, tree_select[2] = {},
           hskip[4] = {}, repeat16 = 0, repeat17 = 0, long_codes = 0;
  uint32_t max_prefix_len = 0, max_clusters = 0, max_ans_table_bytes = 0;
  uint64_t ans_forms[5] = {};  // unary, binary, flat, general, rle
  uint32_t shifts = 0, log_alphas = 0, map_nbits = 0, map_mtf = 0, configs = 0;  // bit sets
  uint32_t rejected_by_parser = 0;  // codes made invalid by --corrupt that parse_entropy_code refused
  void print() const {
    fprintf(stderr,
            "code-form: codes=%llu prefix_codes=%llu prefix_clusters=%llu single_symbol=%llu nsym=%llu,%llu,%llu,%llu "
            "tree_select=%llu,%llu hskip0=%llu hskip2=%llu hskip3=%llu repeat16=%llu repeat17=%llu max_prefix_len=%u "
            "root_bits=%u long_codes=%llu ans_unary=%llu ans_binary=%llu ans_flat=%llu ans_general=%llu ans_rle=%llu "
            "shifts=0x%x log_alphas=0x%x max_clusters=%u map_nbits=0x%x map_mtf=0x%x configs=0x%x "
            "max_ans_table_bytes=%u rejected_by_parser=%u\n",
            (unsigned long long)codes, (unsigned long long)prefix_codes, (unsigned long long)prefix_clusters,
            (unsigned long long)single_symbol, (unsigned long long)nsym[1], (unsigned long long)nsym[2],
            (unsigned long long)nsym[3], (unsigned long long)nsym[4], (unsigned long long)tree_select[0],
            (unsigned long long)tree_select[1], (unsigned long long)hskip[0], (unsigned long long)hskip[2],
            (unsigned long long)hskip[3], (unsigned long long)repeat16, (unsigned long long)repeat17, max_prefix_len,
            kPrefixRootBits, (unsigned long long)long_codes, (unsigned long long)ans_forms[0], (unsigned long long)ans_forms[1],
            (unsigned long long)ans_forms[2], (unsigned long long)ans_forms[3], (unsigned long long)ans_forms[4], shifts,
            log_alphas, max_clusters, map_nbits, map_mtf, configs, max_ans_table_bytes, rejected_by_parser);
  }
} g_report;

[[noreturn]] void form_fail(const char* what, uint32_t cluster) {
  fprintf(stderr, "--code %s: %s (cluster %u)\n", g_code.c_str(), what, cluster);
  exit(1);
}

// Code lengths of min_len to max_len bits for the symbols with freq > 0 (a complete code when at least two symbols are
// used and 2^min_len at most): Huffman, then lengths clamped and the Kraft sum brought back to exactly 1.
std::vector<uint8_t> limited_lengths(const std::vector<double>& freq, uint32_t max_len, uint32_t min_len = 1) {
  std::vector<uint8_t> len(freq.size(), 0);
  struct Node {
    double w;
    int a, b;
  };
  std::vector<Node> nodes;
  std::vector<std::pair<double, int>> heap;
  for (size_t i = 0; i < freq.size(); ++i)
    if (freq[i] > 0) nodes.push_back({freq[i], -1 - int(i), 0}), heap.push_back({-freq[i], int(nodes.size()) - 1});
  if (nodes.size() < 2) {
    for (const Node& n : nodes) len[size_t(-1 - n.a)] = 1;
    return len;
  }
  std::make_heap(heap.begin(), heap.end());
  while (heap.size() > 1) {
    std::pop_heap(heap.begin(), heap.end());
    const auto x = heap.back();
    heap.pop_back();
    std::pop_heap(heap.begin(), heap.end());
    const auto y = heap.back();
    heap.pop_back();
    nodes.push_back({-x.first - y.first, x.second, y.second});
    heap.push_back({x.first + y.first, int(nodes.size()) - 1});
    std::push_heap(heap.begin(), heap.end());
  }
  std::function<void(int, uint32_t)> walk = [&](int n, uint32_t d) {
    if (nodes[size_t(n)].a < 0) {
      len[size_t(-1 - nodes[size_t(n)].a)] = uint8_t(std::min(std::max(d, min_len), max_len));
      return;
    }
    walk(nodes[size_t(n)].a, d + 1);
    walk(nodes[size_t(n)].b, d + 1);
  };
  walk(heap[0].second, 0);
  const uint64_t full = 1ull << max_len;
  auto kraft = [&]() {
    uint64_t k = 0;
    for (uint8_t l : len)
      if (l) k += full >> l;
    return k;
  };
  for (uint64_t k = kraft(); k != full; k = kraft()) {
    int pick = -1;  // over-full: lengthen the longest code below max_len; short: shorten the longest code
    for (size_t i = 0; i < len.size(); ++i)
      if (len[i] && (k > full ? len[i] < max_len : len[i] > min_len) && (pick < 0 || len[i] > len[size_t(pick)])) pick = int(i);
    if (pick < 0) form_fail("no complete code", 0);
    len[size_t(pick)] = uint8_t(len[size_t(pick)] + (k > full ? 1 : -1));
  }
  return len;
}

// Canonical (Brotli) codes of `len`, bit-reversed because the stream is read LSB first.
std::vector<uint32_t> canonical_codes(const std::vector<uint8_t>& len) {
  uint32_t count[17] = {}, next[17] = {};
  for (uint8_t l : len)
    if (l) ++count[l];
  for (uint32_t l = 1, code = 0; l <= 16; ++l) next[l] = code = (code + count[l - 1]) << 1;
  std::vector<uint32_t> out(len.size(), 0);
  for (size_t s = 0; s < len.size(); ++s) {
    if (!len[s]) continue;
    const uint32_t c = next[len[s]]++;
    for (uint32_t i = 0; i < len[s]; ++i) out[s] |= ((c >> i) & 1) << (len[s] - 1 - i);
  }
  return out;
}

// ans.rs:180-254: the alias table of `dist`, packed as parse_entropy_code packs it (pack_ans_bucket).
std::vector<uint64_t> alias_table(const std::vector<uint32_t>& dist, uint32_t log_alpha, uint32_t alphabet_size) {
  const uint32_t table_size = 1u << log_alpha, bucket_size = 1u << (12 - log_alpha);
  std::vector<uint64_t> out;
  for (uint32_t s = 0; s < table_size; ++s)
    if (dist[s] == 4096) {
      for (uint32_t i = 0; i < table_size; ++i) out.push_back(pack_ans_bucket(s, 0, dist[i], bucket_size * i, dist[i] ^ 4096));
      return out;
    }
  struct B {
    uint32_t dist, sym, offset, cutoff;
  };
  std::vector<B> b(table_size);
  std::vector<uint32_t> under, over;
  for (uint32_t i = 0; i < table_size; ++i) {
    b[i] = {dist[i], i < alphabet_size ? i : 0, 0, dist[i]};
    if (dist[i] < bucket_size) under.push_back(i);
    else if (dist[i] > bucket_size) over.push_back(i);
  }
  while (!over.empty() && !under.empty()) {
    const uint32_t o = over.back(), u = under.back();
    over.pop_back(), under.pop_back();
    b[o].cutoff -= bucket_size - b[u].cutoff;
    b[u].sym = o;
    b[u].offset = b[o].cutoff;
    if (b[o].cutoff < bucket_size) under.push_back(o);
    else if (b[o].cutoff > bucket_size) over.push_back(o);
  }
  for (uint32_t i = 0; i < table_size; ++i)
    out.push_back(b[i].cutoff == bucket_size ? pack_ans_bucket(i, 0, b[i].dist, 0, 0)
                                             : pack_ans_bucket(b[i].sym, b[i].cutoff, b[i].dist, b[i].offset - b[i].cutoff,
                                                               b[i].dist ^ b[b[i].sym].dist));
  return out;
}

void write_shift(BitWriter& w, uint32_t shift) {  // inverse of ans.rs:87-95
  uint32_t len = 0;
  while (len < 3 && (1u << (len + 1)) - 1 <= shift) ++len;
  for (uint32_t i = 0; i < len; ++i) w.write(1, 1);
  if (len < 3) w.write(1, 0);
  w.write(int(len), shift + 1 - (1u << len));
}

// Counts (summing to 4096) in the general form with `shift`: each count but the omitted one (the first of the largest
// logcount) rounded down to what the shift can represent, the omitted one taking the rest. Writes the histogram.
std::vector<uint32_t> write_general(BitWriter& w, std::vector<uint32_t> c, uint32_t shift, bool rle) {
  c.resize(std::max<size_t>(c.size(), 3), 0);
  auto logc = [](uint32_t v) { return v ? 32 - uint32_t(__builtin_clz(v)) : 0u; };
  uint32_t omit = 0;
  for (uint32_t i = 0; i < c.size(); ++i)
    if (logc(c[i]) > logc(c[omit])) omit = i;
  uint32_t sum = 0;
  for (uint32_t i = 0; i < c.size(); ++i) {
    if (i == omit || c[i] <= 1) {
      sum += i == omit ? 0 : c[i];
      continue;
    }
    const int zeros = int(logc(c[i])) - 1, bitcount = std::min(std::max(int(shift) - ((12 - zeros) >> 1), 0), zeros);
    c[i] &= ~((1u << (zeros - bitcount)) - 1);
    sum += c[i];
  }
  c[omit] = 4096 - sum;
  w.write(1, 0);
  w.write(1, 0);
  write_shift(w, shift);
  write_u8(w, uint32_t(c.size()) - 3);
  // logcounts; with `rle`, runs of four or more counts equal to the one before as logcount 13 and a repeat count
  // (ans.rs:107-116, 138-155: not right after the omitted count, whose place repeats as 0, nor over it)
  std::vector<bool> repeated(c.size(), false);
  for (uint32_t i = 0; i < c.size();) {
    uint32_t r = 0;
    if (rle && i > 0 && i - 1 != omit)
      while (i + r < c.size() && i + r != omit && c[i + r] == c[i - 1]) ++r;
    if (r >= 4) {
      write_logcount(w, 13);
      write_u8(w, std::min<uint32_t>(r, 259) - 4);
      for (uint32_t k = i; k < i + std::min<uint32_t>(r, 259); ++k) repeated[k] = true;
      i += std::min<uint32_t>(r, 259);
      ++g_report.ans_forms[4];
      continue;
    }
    write_logcount(w, logc(c[i]));
    ++i;
  }
  for (uint32_t i = 0; i < c.size(); ++i) {
    if (repeated[i] || i == omit || c[i] <= 1) continue;
    const int zeros = int(logc(c[i])) - 1, bitcount = std::min(std::max(int(shift) - ((12 - zeros) >> 1), 0), zeros);
    w.write(bitcount, (c[i] - (1u << zeros)) >> (zeros - bitcount));
  }
  return c;
}

// Writes the entropy-code header for `tokens` (clustered by `cluster_of_ctx`) and then the ANS
// stream itself (32-bit initial state first). With `lz` set the code has LZ77 enabled: the symbols then hold
// literals, length tokens (min_symbol and up) and distances, and the last context of the map is the distance context.
struct EntropyEncoder {
  uint32_t num_ctx = 0, num_clusters = 0, log_alpha = 0;
  std::vector<uint8_t> cluster_of_ctx;
  std::vector<std::vector<uint32_t>> counts;     // per cluster, normalised
  std::vector<std::vector<std::vector<uint16_t>>> inv;  // cluster -> symbol -> offset -> idx
  const Lz77Header* lz = nullptr;
  // --code only: per-cluster hybrid-uint configs, and the prefix code (lengths and bit-reversed codes) of each cluster
  std::vector<UintConfig> cfg;
  std::vector<std::vector<uint8_t>> plen;
  std::vector<std::vector<uint32_t>> pcode;
  std::vector<int32_t> psingle;  // the symbol of a 0-bit prefix code, -1 otherwise
  bool broken = false;           // --corrupt made this code invalid: its streams are not written

  std::vector<Sym> syms_of(const std::vector<Token>& tokens) const {
    if (cfg.empty()) return to_syms(tokens);
    std::vector<Sym> s(tokens.size());
    for (size_t i = 0; i < tokens.size(); ++i) {
      s[i].ctx = tokens[i].ctx;
      tokenize_with(cfg[cluster_of_ctx[tokens[i].ctx]], tokens[i].value, &s[i].tok, &s[i].nbits, &s[i].bits);
    }
    return s;
  }
  void write_header(BitWriter& w, const std::vector<Token>& tokens, uint32_t num_ctx_, const std::vector<uint8_t>& map) {
    if (!g_code.empty() && g_code != "lz77" && !lz) return write_header_form(w, tokens, num_ctx_, map);
    write_header_syms(w, to_syms(tokens), num_ctx_, map);
  }

  // --code: the cluster map, the configs and the tokens are chosen here (see the comment above g_code).
  void write_header_form(BitWriter& w, const std::vector<Token>& tokens, uint32_t num_ctx_, std::vector<uint8_t> map) {
    const std::string& f = g_code;
    num_ctx = num_ctx_;
    const uint32_t turn = g_code_turn++;
    BitWriter hw;
    hw.write(1, 0);  // no LZ77
    // ---- cluster map ----
    bool simple_map = true, mtf = false;
    uint32_t nbits = 0;
    if (f == "clusters" && num_ctx > 1) {
      uint32_t K;
      if (num_ctx >= 65) {
        static uint32_t complex_maps = 0;  // K and move-to-front in turn
        const uint32_t ks[3] = {65, 256, 131};
        K = std::min(ks[complex_maps % 3], num_ctx);
        simple_map = false;
        mtf = complex_maps++ % 2;
      } else {
        static uint32_t simple_maps = 0;  // nbits 0..3 in turn, starting from the frame's seed
        nbits = (simple_maps++ + g_code_seed) % 4;
        K = std::min(1u << nbits, num_ctx);
      }
      map.resize(num_ctx);
      for (uint32_t i = 0; i < num_ctx; ++i) map[i] = uint8_t(i % K);
    } else if (num_ctx > 1) {
      uint32_t n = 0;
      for (uint8_t c : map) n = std::max<uint32_t>(n, c + 1u);
      if (n > 8) simple_map = false;
      else nbits = n <= 1 ? 0 : ceil_log2_nonzero(n);
    }
    cluster_of_ctx = map;
    num_clusters = 0;
    for (uint8_t c : map) num_clusters = std::max<uint32_t>(num_clusters, c + 1u);
    if (num_ctx > 1) {
      if (simple_map) {
        hw.write(1, 1);
        hw.write(2, nbits);
        for (uint32_t i = 0; i < num_ctx; ++i) hw.write(int(nbits), map[i]);
        g_report.map_nbits |= 1u << nbits;
      } else {
        hw.write(1, 0);
        hw.write(1, mtf ? 1 : 0);
        std::vector<Token> mt;
        uint8_t order[256];
        for (int i = 0; i < 256; ++i) order[i] = uint8_t(i);
        for (uint32_t i = 0; i < num_ctx; ++i) {
          uint32_t v = map[i];
          if (mtf) {  // lib.rs:714-725 inverted: the position of the cluster in the list, which then moves to the front
            uint32_t k = 0;
            while (order[k] != map[i]) ++k;
            std::memmove(order + 1, order, k);
            order[0] = map[i];
            v = k;
          }
          mt.push_back({0, v});
        }
        EntropyEncoder nested;
        nested.write_header(hw, mt, 1, std::vector<uint8_t>(1, 0));
        nested.write_tokens(hw, mt);
        g_report.map_mtf |= 1u << (mtf ? 1 : 0);
      }
    }
    // ---- configs and tokens ----
    const bool prefix = f == "prefix";
    cfg.assign(num_clusters, UintConfig{kSplitExp, kMsb, kLsb});
    if (f == "ans-forms") log_alpha = 6 + turn % 3;
    else log_alpha = 8;
    if (f == "configs") {
      std::vector<uint32_t> maxv(num_clusters, 0);
      for (const Token& t : tokens) maxv[map[t.ctx]] = std::max(maxv[map[t.ctx]], t.value);
      const uint32_t ncfg = sizeof(kFormConfigs) / sizeof(kFormConfigs[0]);
      for (uint32_t c = 0; c < num_clusters; ++c)
        for (uint32_t k = 0; k < ncfg; ++k) {
          const uint32_t i = (g_code_turn + k) % ncfg;
          uint32_t tok, nb, bits;
          tokenize_with(kFormConfigs[i], maxv[c], &tok, &nb, &bits);
          if (tok < (1u << log_alpha)) {
            cfg[c] = kFormConfigs[i];
            g_report.configs |= 1u << i;
            ++g_code_turn;
            break;
          }
        }
    }
    const std::vector<Sym> syms = syms_of(tokens);
    std::vector<std::vector<uint64_t>> freq(num_clusters);
    for (const Sym& s : syms) {
      auto& fr = freq[map[s.ctx]];
      if (fr.size() <= s.tok) fr.resize(s.tok + 1, 0);
      ++fr[s.tok];
    }
    for (uint32_t c = 0; c < num_clusters; ++c)
      if (!prefix && freq[c].size() > (1u << log_alpha)) form_fail("token alphabet too large", c);
    hw.write(1, prefix ? 1 : 0);
    if (!prefix) hw.write(2, log_alpha - 5);
    const uint32_t la = prefix ? 15 : log_alpha;
    for (uint32_t c = 0; c < num_clusters; ++c) {  // lib.rs:378-412
      hw.write(int(add_log2_ceil(la)), cfg[c].split_exp);
      if (cfg[c].split_exp != la) {
        hw.write(int(add_log2_ceil(cfg[c].split_exp)), cfg[c].msb);
        hw.write(int(add_log2_ceil(cfg[c].split_exp - cfg[c].msb)), cfg[c].lsb);
      }
    }
    std::vector<std::vector<uint64_t>> tables;  // ANS: the alias table of each cluster
    if (prefix) write_prefix_codes(hw, freq);
    else tables = write_ans_codes(hw, freq, f == "ans-forms");
    // ---- read back with the product's parser; everything must be what was written ----
    const size_t written_bits = hw.total_bits;
    hw.pad();
    if (g_corrupt_done && (g_corrupt == "oversub-clcl" || g_corrupt == "oversub-lengths" || g_corrupt == "ans-sum") &&
        !g_report.rejected_by_parser) {
      try {
        BitReader br(hw.bytes.data(), hw.bytes.size());
        parse_entropy_code(br, num_ctx);
      } catch (const Error&) {
        ++g_report.rejected_by_parser;
      }
      BitReader cp(hw.bytes.data(), hw.bytes.size());
      for (size_t b = written_bits; b;) {
        const uint32_t n = uint32_t(std::min<size_t>(b, 32));
        w.write(int(n), cp.read(n));
        b -= n;
      }
      broken = true;  // the streams that follow are never read
      return;
    }
    BitReader br(hw.bytes.data(), hw.bytes.size());
    EntropyCode code = parse_entropy_code(br, num_ctx);
    if (code.num_clusters != num_clusters || code.cluster_map != map || code.use_prefix != prefix ||
        (!prefix && code.log_alphabet_size != log_alpha))
      form_fail("cluster map or code kind read back differently", 0);
    for (uint32_t c = 0; c < num_clusters; ++c) {
      const HybridUintConfig& h = code.configs[c];
      if (h.split_exponent != cfg[c].split_exp || h.msb_in_token != cfg[c].msb || h.lsb_in_token != cfg[c].lsb)
        form_fail("hybrid-uint config read back differently", c);
      if (prefix) check_prefix_table(code, c);
      else
        for (size_t i = 0; i < tables[c].size(); ++i)
          if (code.ans_table[(size_t(c) << log_alpha) + i] != tables[c][i]) form_fail("ANS alias table differs", c);
    }
    if (!prefix) build_inverse(tables);
    ++g_report.codes;
    g_report.max_clusters = std::max(g_report.max_clusters, num_clusters);
    if (!prefix) {
      g_report.log_alphas |= 1u << log_alpha;
      g_report.max_ans_table_bytes = std::max(g_report.max_ans_table_bytes, (num_clusters << log_alpha) * 8);
    }
    size_t hbits = br.pos();
    BitReader cp(hw.bytes.data(), hw.bytes.size());
    for (; hbits;) {
      const uint32_t n = uint32_t(std::min<size_t>(hbits, 32));
      w.write(int(n), cp.read(n));
      hbits -= n;
    }
  }

  // lib.rs:433-452 and prefix.rs: the alphabet size of each cluster, then its code.
  void write_prefix_codes(BitWriter& hw, const std::vector<std::vector<uint64_t>>& freq) {
    ++g_report.prefix_codes;
    plen.assign(num_clusters, {});
    pcode.assign(num_clusters, {});
    psingle.assign(num_clusters, -1);
    uint32_t deep = 0, deep_n = 0;  // the cluster with the most symbols gets the chain-shaped code
    for (uint32_t c = 0; c < num_clusters; ++c) {
      uint32_t n = 0;
      for (uint64_t x : freq[c]) n += x != 0;
      if (n > deep_n) deep = c, deep_n = n;
    }
    for (uint32_t c = 0; c < num_clusters; ++c) {
      const uint32_t count = std::max<uint32_t>(1, uint32_t(freq[c].size()));
      if (count == 1) {
        hw.write(1, 0);
      } else {
        hw.write(1, 1);
        const uint32_t n = 31 - uint32_t(__builtin_clz(count - 1));
        hw.write(4, n);
        hw.write(int(n), count - 1 - (1u << n));
      }
    }
    for (uint32_t c = 0; c < num_clusters; ++c) {
      ++g_report.prefix_clusters;
      const uint32_t count = std::max<uint32_t>(1, uint32_t(freq[c].size()));
      std::vector<uint32_t> used;  // by falling frequency
      for (uint32_t s = 0; s < freq[c].size(); ++s)
        if (freq[c][s]) used.push_back(s);
      std::stable_sort(used.begin(), used.end(), [&](uint32_t a, uint32_t b) { return freq[c][a] > freq[c][b]; });
      std::vector<uint8_t>& len = plen[c];
      len.assign(count, 0);
      if (used.size() <= 1) {  // 0 bits per symbol
        ++g_report.single_symbol;
        psingle[c] = used.empty() ? 0 : int32_t(used[0]);
        if (count > 1) {
          hw.write(2, 1), hw.write(2, 0), hw.write(int(ceil_log2_nonzero(count)), used[0]);
          ++g_report.nsym[1];
        }
        pcode[c].assign(count, 0);
        continue;
      }
      if (used.size() <= 4) {  // prefix.rs:149-207
        const uint32_t abits = ceil_log2_nonzero(count), n = uint32_t(used.size());
        hw.write(2, 1);
        hw.write(2, n - 1);
        bool tree_select = false;
        if (n == 4) tree_select = (g_code_turn++ % 2) == 1, ++g_report.tree_select[tree_select];
        const uint8_t lens[5][4] = {{}, {}, {1, 1}, {1, 2, 2}, {2, 2, 2, 2}};
        for (uint32_t i = 0; i < n; ++i) {
          hw.write(int(abits), used[i]);
          len[used[i]] = tree_select ? uint8_t(std::min<uint32_t>(i + 1, 3)) : lens[n][i];
        }
        if (n == 4) hw.write(1, tree_select);
        ++g_report.nsym[n];
      } else {
        // hskip 2 and 3 leave out the code-length symbols 1, 2 (and 3): codes of at least 3 (4) bits where they fit
        const uint32_t kSkips[3] = {0, 2, 3};
        const bool chain = c == deep && used.size() >= 16;
        const uint32_t hskip = chain ? 0 : kSkips[g_code_turn++ % 3];
        const uint32_t min_len = hskip == 3 && used.size() >= 16 ? 4 : hskip && used.size() >= 8 ? 3 : 1;
        std::vector<double> wt(count, 0.0);
        for (uint32_t i = 0; i < used.size(); ++i) wt[used[i]] = chain ? std::ldexp(1.0, -int(i)) : double(freq[c][used[i]]);
        len = limited_lengths(wt, 15, min_len);
        write_complex(hw, len, hskip);
      }
      pcode[c] = canonical_codes(len);
      for (uint8_t l : len) {
        g_report.max_prefix_len = std::max<uint32_t>(g_report.max_prefix_len, l);
        g_report.long_codes += l > kPrefixRootBits;
      }
    }
  }

  // prefix.rs:209-332: the code-length code, then the code lengths with repeat codes 16 and 17.
  void write_complex(BitWriter& hw, const std::vector<uint8_t>& len, uint32_t hskip) {
    struct Item {
      uint32_t sym, nbits, bits;
    };
    std::vector<Item> items;
    size_t last = len.size();
    while (last > 0 && !len[last - 1]) --last;
    uint32_t last_nz = 8, prev = 0xff;
    for (size_t i = 0; i < last;) {
      size_t r = 0;
      while (i + r < last && len[i + r] == len[i]) ++r;
      if (len[i] == 0 && r >= 3 && prev != 17) {
        const uint32_t k = uint32_t(std::min<size_t>(r, 10));
        items.push_back({17, 3, k - 3}), prev = 17, i += k;
        ++g_report.repeat17;
      } else if (len[i] != 0 && len[i] == last_nz && r >= 3 && prev != 16) {
        const uint32_t k = uint32_t(std::min<size_t>(r, 6));
        items.push_back({16, 2, k - 3}), prev = 16, i += k;
        ++g_report.repeat16;
      } else {
        items.push_back({len[i], 0, 0}), prev = len[i];
        if (len[i]) last_nz = len[i];
        ++i;
      }
    }
    if (g_corrupt == "oversub-lengths" && !g_corrupt_done && items.back().sym >= 2 && items.back().sym <= 15)
      --items.back().sym, g_corrupt_done = true;
    std::vector<double> cf(18, 0.0);
    for (const Item& it : items) cf[it.sym] += 1.0;
    std::vector<uint8_t> cl = limited_lengths(cf, 5);
    uint32_t nz = 0;
    for (uint8_t l : cl) nz += l != 0;
    static const uint32_t kOrder[18] = {1, 2, 3, 4, 0, 5, 17, 6, 16, 7, 8, 9, 10, 11, 12, 13, 14, 15};
    while (hskip && (cl[1] || cl[2] || (hskip == 3 && cl[3]))) hskip = hskip == 3 ? 2 : 0;
    ++g_report.hskip[hskip];
    hw.write(2, hskip);
    uint32_t acc = 0, last_k = 0;
    for (uint32_t k = hskip; k < 18 && (nz == 1 || acc < 32); ++k) {
      if (cl[kOrder[k]]) acc += 32u >> cl[kOrder[k]], last_k = k;
    }
    const bool bad_clcl = g_corrupt == "oversub-clcl" && !g_corrupt_done && nz > 1 && cl[kOrder[last_k]] >= 2;
    if (bad_clcl) g_corrupt_done = true;
    acc = 0;
    for (uint32_t k = hskip; k < 18 && (nz == 1 || acc < 32); ++k) {
      const uint32_t l = cl[kOrder[k]] - (bad_clcl && k == last_k ? 1 : 0);
      if (l == 0) hw.write(2, 0);
      else if (l == 4) hw.write(2, 1);
      else if (l == 3) hw.write(2, 2);
      else if (l == 2) hw.write(2, 3), hw.write(1, 0);
      else if (l == 1) hw.write(2, 3), hw.write(1, 1), hw.write(1, 0);
      else hw.write(2, 3), hw.write(1, 1), hw.write(1, 1);
      if (l) acc += 32u >> l;
      if (bad_clcl && k == last_k) return;  // the parser stops here
    }
    const std::vector<uint32_t> cc = canonical_codes(cl);
    for (const Item& it : items) {
      if (nz > 1) hw.write(cl[it.sym], cc[it.sym]);
      if (it.nbits) hw.write(int(it.nbits), it.bits);
    }
  }

  // Every symbol's code looked up in the parser's table (entropy.h: kPrefixNested, kPrefixRootBits) gives it back.
  void check_prefix_table(const EntropyCode& code, uint32_t c) const {
    const PrefixMeta& m = code.prefix_meta[c];
    const uint32_t* t = code.prefix_table.data() + m.table_offset;
    uint32_t nused = 0;
    for (uint32_t s = 0; s < plen[c].size(); ++s) {
      if (!plen[c][s]) continue;
      ++nused;
      uint32_t e = t[pcode[c][s] & ((1u << m.root_bits) - 1)];
      if (e & kPrefixNested) {
        if (m.root_bits != kPrefixRootBits) form_fail("nested entry below the root bits", c);
        const uint32_t sb = (e >> 16) & 0xff;
        e = t[(1u << m.root_bits) + (e & 0xffff) + ((pcode[c][s] >> m.root_bits) & ((1u << sb) - 1))];
      }
      if ((e & 0xffff) != s || ((e >> 16) & 0xff) != plen[c][s]) form_fail("prefix code read back differently", c);
    }
    if (nused == 0 && code.single_symbol[c] != psingle[c]) form_fail("single-symbol prefix code read back differently", c);
  }

  // ANS histograms (ans.rs:31-178) in the form chosen for each cluster; returns each cluster's alias table.
  std::vector<std::vector<uint64_t>> write_ans_codes(BitWriter& hw, const std::vector<std::vector<uint64_t>>& freq,
                                                     bool forms) {
    std::vector<std::vector<uint64_t>> tables;
    counts.clear();
    for (uint32_t c = 0; c < num_clusters; ++c) {
      std::vector<uint64_t> fr = freq[c].empty() ? std::vector<uint64_t>(1, 0) : freq[c];
      std::vector<uint32_t> used;
      for (uint32_t s = 0; s < fr.size(); ++s)
        if (fr[s]) used.push_back(s);
      std::vector<uint32_t> dist(size_t(1) << log_alpha, 0);
      uint32_t alphabet;  // the alphabet size the histogram declares (ans.rs:46-102)
      if (g_corrupt == "ans-sum" && !g_corrupt_done) {  // counts 2048 (omitted), 4095, 4095: explicit ones sum to 8190
        g_corrupt_done = true;
        hw.write(1, 0), hw.write(1, 0), write_shift(hw, 13), write_u8(hw, 0);
        for (int i = 0; i < 3; ++i) write_logcount(hw, 12);
        hw.write(11, 2047), hw.write(11, 2047);
        counts.push_back(dist);
        tables.push_back({});
        continue;
      }
      if (used.size() > 2 || (!forms && used.size() == 2)) {
        const uint32_t kind = forms ? g_code_turn++ % 4 : 3;  // 0 flat, 1 rle, 2-3 general
        std::vector<uint32_t> nc = normalize(fr);
        if (kind == 0) {  // evenly distributed over [0, last]
          const uint32_t n = uint32_t(fr.size());
          hw.write(1, 0), hw.write(1, 1), write_u8(hw, n - 1);
          for (uint32_t i = 0; i < n; ++i) nc[i] = 4096 / n + (i < 4096 % n ? 1 : 0);
          ++g_report.ans_forms[2];
        } else if (kind == 1) {  // equal counts, the rest on symbol 0
          const uint32_t n = uint32_t(fr.size()), base = std::max<uint32_t>(1, 2048 / n);
          for (uint32_t i = 0; i < n; ++i) nc[i] = base;
          nc[0] = 4096 - (n - 1) * base;
          nc = write_general(hw, nc, 13, true);
        } else {
          const uint32_t shift = forms ? g_report.ans_forms[3] % 14 : 13;
          nc = write_general(hw, nc, shift, false);
          g_report.shifts |= 1u << shift;
          ++g_report.ans_forms[3];
        }
        for (uint32_t i = 0; i < nc.size(); ++i) dist[i] = nc[i];
        alphabet = kind == 0 ? uint32_t(fr.size()) : uint32_t(nc.size());
      } else if (used.size() == 2) {
        std::vector<uint32_t> nc = normalize(fr);
        hw.write(1, 1), hw.write(1, 1);
        write_u8(hw, used[0]), write_u8(hw, used[1]);
        hw.write(12, nc[used[0]]);
        dist[used[0]] = nc[used[0]], dist[used[1]] = 4096 - nc[used[0]];
        alphabet = used[1] + 1;
        ++g_report.ans_forms[1];
      } else {
        const uint32_t s = used.empty() ? 0 : used[0];
        hw.write(1, 1), hw.write(1, 0), write_u8(hw, s);
        dist[s] = 4096;
        alphabet = s + 1;
        ++g_report.ans_forms[0];
      }
      for (uint32_t s : used)
        if (!dist[s]) form_fail("a used symbol has no probability", c);
      counts.push_back(dist);
      tables.push_back(alias_table(dist, log_alpha, alphabet));
    }
    return tables;
  }

  // The encoder's inverse of the alias tables: symbol and offset -> table index (ans.rs:264-290, read_symbol).
  void build_inverse(const std::vector<std::vector<uint64_t>>& tables) {
    inv.assign(num_clusters, {});
    const uint32_t log_bucket = 12 - log_alpha;
    for (uint32_t c = 0; c < num_clusters; ++c) {
      inv[c].resize(size_t(1) << log_alpha);
      for (size_t s = 0; s < counts[c].size(); ++s) inv[c][s].assign(counts[c][s], 0xffff);
      for (uint32_t idx = 0; idx < 4096; ++idx) {
        const uint32_t i = idx >> log_bucket, pos = idx & ((1u << log_bucket) - 1);
        const uint64_t b = tables[c][i];
        const uint32_t alias_symbol = uint32_t(b & 0xff), cutoff = uint32_t((b >> 8) & 0xff);
        const bool alias = pos >= cutoff;
        const uint32_t offset = (alias ? uint32_t((b >> 32) & 0xffff) : 0) + pos, sym = alias ? alias_symbol : i;
        if (sym >= inv[c].size() || offset >= inv[c][sym].size()) form_fail("alias table inconsistent", c);
        inv[c][sym][offset] = uint16_t(idx);
      }
    }
  }

  // `num_ctx_` counts the distance context of an LZ77 code.
  void write_header_syms(BitWriter& w, const std::vector<Sym>& syms, uint32_t num_ctx_, const std::vector<uint8_t>& map) {
    num_ctx = num_ctx_;
    cluster_of_ctx = map;
    num_clusters = 0;
    for (uint8_t c : map) num_clusters = std::max<uint32_t>(num_clusters, c + 1u);
    std::vector<std::vector<uint64_t>> freq(num_clusters);
    uint32_t max_tok = 0;
    for (const Sym& s : syms) {
      auto& f = freq[map[s.ctx]];
      if (f.size() <= s.tok) f.resize(s.tok + 1, 0);
      ++f[s.tok];
      max_tok = std::max(max_tok, s.tok);
    }
    log_alpha = 5;
    while ((1u << log_alpha) <= max_tok) ++log_alpha;
    if (log_alpha > 8) fprintf(stderr, "token alphabet too large\n"), exit(1);
    BitWriter hw;
    hw.write(1, lz ? 1 : 0);  // lz77
    if (lz) {  // lib.rs:321-343
      const uint32_t sym_bits[4] = {0, 0, 0, 15}, sym_base[4] = {224, 512, 4096, 8};
      const uint32_t len_bits[4] = {0, 0, 2, 8}, len_base[4] = {3, 4, 5, 9};
      write_u32(hw, lz->symbol_sel, int(sym_bits[lz->symbol_sel]), lz->min_symbol - sym_base[lz->symbol_sel]);
      write_u32(hw, lz->length_sel, int(len_bits[lz->length_sel]), lz->min_length - len_base[lz->length_sel]);
      hw.write(int(add_log2_ceil(8)), lz->len_cfg.split_exp);  // IntegerConfig with log_alphabet_size 8
      if (lz->len_cfg.split_exp != 8) {
        hw.write(int(add_log2_ceil(lz->len_cfg.split_exp)), lz->len_cfg.msb);
        hw.write(int(add_log2_ceil(lz->len_cfg.split_exp - lz->len_cfg.msb)), lz->len_cfg.lsb);
      }
    }
    // cluster map (lib.rs:688-749)
    if (num_ctx > 1) {
      if (num_clusters <= 8) {
        uint32_t nb = num_clusters <= 1 ? 0 : ceil_log2_nonzero(num_clusters);
        hw.write(1, 1);
        hw.write(2, nb);
        for (uint32_t i = 0; i < num_ctx; ++i) hw.write(int(nb), map[i]);
      } else {
        hw.write(1, 0);  // not simple
        hw.write(1, 0);  // no move-to-front
        std::vector<Token> mt;
        for (uint32_t i = 0; i < num_ctx; ++i) mt.push_back({0, map[i]});
        EntropyEncoder nested;
        nested.write_header(hw, mt, 1, std::vector<uint8_t>(1, 0));
        nested.write_tokens(hw, mt);
      }
    }
    hw.write(1, 0);  // ANS, not prefix
    hw.write(2, log_alpha - 5);
    for (uint32_t c = 0; c < num_clusters; ++c) {  // IntegerConfig (lib.rs:378-414)
      hw.write(int(add_log2_ceil(log_alpha)), kSplitExp);
      hw.write(int(add_log2_ceil(kSplitExp)), kMsb);
      hw.write(int(add_log2_ceil(kSplitExp - kMsb)), kLsb);
    }
    counts.clear();
    for (uint32_t c = 0; c < num_clusters; ++c) {
      if (freq[c].empty()) freq[c].assign(1, 0);
      counts.push_back(normalize(freq[c]));
      write_ans_histogram(hw, counts.back());
    }
    hw.pad();
    // read it back with the decoder's parser to get the exact alias tables
    BitReader br(hw.bytes.data(), hw.bytes.size());
    EntropyCode code = parse_entropy_code(br, num_ctx - (lz ? 1 : 0));
    if (code.num_clusters != num_clusters || code.log_alphabet_size != log_alpha) fprintf(stderr, "header readback mismatch\n"), exit(1);
    if (lz && (!code.lz77_enabled || code.lz77_min_symbol != lz->min_symbol || code.lz77_min_length != lz->min_length ||
               code.lz_len_conf.split_exponent != lz->len_cfg.split_exp || code.lz_len_conf.msb_in_token != lz->len_cfg.msb ||
               code.lz_len_conf.lsb_in_token != lz->len_cfg.lsb || code.lz_dist_cluster() != map.back()))
      fprintf(stderr, "LZ77 header readback mismatch\n"), exit(1);
    inv.assign(num_clusters, {});
    const uint32_t log_bucket = 12 - log_alpha;
    for (uint32_t c = 0; c < num_clusters; ++c) {
      inv[c].resize(size_t(1) << log_alpha);
      for (size_t s = 0; s < counts[c].size(); ++s) inv[c][s].assign(counts[c][s], 0);
      for (uint32_t idx = 0; idx < 4096; ++idx) {
        uint32_t i = idx >> log_bucket, pos = idx & ((1u << log_bucket) - 1);
        uint64_t b = code.ans_table[(size_t(c) << log_alpha) + i];
        uint32_t alias_symbol = uint32_t(b & 0xff), cutoff = uint32_t((b >> 8) & 0xff);
        bool alias = pos >= cutoff;
        uint32_t offset = (alias ? uint32_t((b >> 32) & 0xffff) : 0) + pos;
        uint32_t sym = alias ? alias_symbol : i;
        if (sym >= inv[c].size() || offset >= inv[c][sym].size()) fprintf(stderr, "alias table inconsistent (c=%u sym=%u off=%u)\n", c, sym, offset), exit(1);
        inv[c][sym][offset] = uint16_t(idx);
      }
    }
    // copy the header bits (minus padding) into the real stream
    size_t hbits = br.pos();
    BitReader cp(hw.bytes.data(), hw.bytes.size());
    while (hbits) {
      uint32_t n = uint32_t(std::min<size_t>(hbits, 32));
      w.write(int(n), cp.read(n));
      hbits -= n;
    }
  }

  void write_tokens(BitWriter& w, const std::vector<Token>& tokens) const { write_syms(w, syms_of(tokens)); }
  void write_syms(BitWriter& w, const std::vector<Sym>& syms) const {
    if (broken) return;
    if (!plen.empty()) {  // prefix codes: no state, each symbol's code and then its extra bits
      for (const Sym& s : syms) {
        const uint32_t c = cluster_of_ctx[s.ctx];
        if (plen[c][s.tok]) w.write(plen[c][s.tok], pcode[c][s.tok]);
        if (s.nbits) w.write(int(s.nbits), s.bits);
      }
      return;
    }
    struct Out {
      uint16_t ans_bits;
      uint8_t has_ans;
      uint8_t nbits;
      uint32_t bits;
    };
    std::vector<Out> outs(syms.size());
    uint32_t state = g_flip_state ? 0x130001 : 0x130000;  // ans-state: every value decodes, the end state is wrong
    for (size_t k = syms.size(); k-- > 0;) {
      const uint32_t tok = syms[k].tok;
      uint32_t c = cluster_of_ctx[syms[k].ctx];
      uint32_t f = counts[c][tok];
      Out& o = outs[k];
      o.nbits = uint8_t(syms[k].nbits);
      o.bits = syms[k].bits;
      o.has_ans = 0;
      if ((state >> 20) >= f) {
        o.has_ans = 1;
        o.ans_bits = uint16_t(state & 0xffff);
        state >>= 16;
      }
      state = ((state / f) << 12) + inv[c][tok][state % f];
    }
    w.write(32, state);
    g_flip_state = false;
    for (const Out& o : outs) {
      if (o.has_ans) w.write(16, o.ans_bits);
      if (o.nbits) w.write(o.nbits, o.bits);
    }
  }
};

// --hf-lz77: the LZ77 codes of the HF passes and how one HF stream is parsed into literals and copies. The decoder reads
// every value of an HF stream -- non-zero counts and coefficients alike -- through read_varint_with_multiplier_clustered
// with distance multiplier 0 (hf_coeff.rs:181-222): a length token is coded in the context of the first value it
// replaces, its distance value D in the distance context, and the copy starts min(min(2^20 - 1, D) + 1, values so far)
// values back. Copies run through whatever the values mean: block, channel and non-zero-count boundaries.
//   rle:   libjxl's RLE form: min_symbol 224, min_length 3, distance value 0 (repeat the previous value).
//   match: greedy matches at any distance (hash chains over four values), overlapping ones included; min_symbol
//          8 + u(15) = 128, min_length 4. A match from the stream's first value is written with a distance beyond the
//          values decoded so far, which the decoder clamps; the stream's last copy runs past its end (a copy still
//          pending when the stream ends is ignored).
//   bad-first / bad-length: `match`, with group 0's stream made invalid -- it starts with a copy, or its first copy has
//          a length whose value plus min_length does not fit 32 bits.
//   modular (--code lz77): `match` over a Modular stream, with the U32 selectors of min_symbol (224 or 8 + u(15) = 128)
//          and min_length (3, 4, 5 + u(2) = 6, 9 + u(8) = 10) taken from `sel`. The decoder scales the special distance
//          codes 0..119 by the stream's widest channel (image.rs:460, lib.rs:530-545): a copy from dy rows up and dx
//          columns over is written with such a code where one fits, any other distance as 120 + distance - 1.
//          Matches stay within the 2^20-value window; copies run across channel boundaries, and none is pending at
//          the end of the stream.
struct HfLz77 {
  std::string mode;  // empty: no LZ77
  uint32_t sel = 0;  // modular: min_length selector in bits 0-1, min_symbol 8 + u(15) in bit 2
  Lz77Header header() const {
    if (mode == "rle") return {224, 3, 0, 0, {0, 0, 0}};
    if (mode == "modular") {
      const uint32_t len_min[4] = {3, 4, 6, 10};
      if (sel & 4) return {128, len_min[sel & 3], 3, int(sel & 3), {kSplitExp, kMsb, kLsb}};
      return {224, len_min[sel & 3], 0, int(sel & 3), {0, 0, 0}};
    }
    return {128, 4, 3, 1, {kSplitExp, kMsb, kLsb}};
  }
};
struct Lz77Counts {
  uint64_t copied = 0, from_start = 0;
  uint64_t special = 0, far = 0, cross_channel = 0, past_window = 0;  // modular: copies of each kind
};

// `mult`: the stream's distance multiplier (0 in HF streams); `chan_start`: where each channel's values begin.
std::vector<Sym> lz77_parse(const std::vector<Token>& toks, const HfLz77& opt, uint32_t dist_ctx, bool corrupt,
                            Lz77Counts* counts, uint32_t mult = 0, const std::vector<size_t>& chan_start = {}) {
  const Lz77Header h = opt.header();
  const size_t n = toks.size(), kWindow = size_t(1) << 20;
  struct Item {
    size_t pos;
    bool copy;
    uint32_t len_value, dist_value;  // copy: length - min_length, D
  };
  std::vector<Item> items;
  auto v = [&](size_t i) { return toks[i].value; };
  uint64_t copied = 0, from_start = 0;
  if (opt.mode == "rle") {
    for (size_t i = 0; i < n;) {
      size_t r = 0;
      if (i > 0)
        while (i + r < n && v(i + r) == v(i - 1)) ++r;
      if (r >= h.min_length) {
        items.push_back({i, true, uint32_t(r - h.min_length), 0});
        copied += r;
        i += r;
      } else {
        items.push_back({i, false, 0, 0});
        ++i;
      }
    }
  } else {
    const uint32_t kHashBits = 16;
    std::vector<int32_t> head(size_t(1) << kHashBits, -1), prev(n, -1);
    auto hash = [&](size_t i) {
      const uint32_t x = v(i) * 0x9E3779B1u ^ v(i + 1) * 0x85EBCA77u ^ v(i + 2) * 0xC2B2AE3Du ^ v(i + 3) * 0x27D4EB2Fu;
      return (x * 0x9E3779B1u) >> (32 - kHashBits);
    };
    auto insert = [&](size_t i) {
      if (i + 4 > n) return;
      const uint32_t k = hash(i);
      prev[i] = head[k];
      head[k] = int32_t(i);
    };
    auto match_len = [&](size_t j, size_t i) {
      size_t l = 0;
      while (i + l < n && l < 65536 && v(j + l) == v(i + l)) ++l;
      return l;
    };
    auto special = [&](size_t dist) {  // the special distance code of `dist`, or -1
      for (int k = 0; k < 120; ++k)
        if (int64_t(kLz77SpecialDistances[k][0]) + int64_t(mult) * kLz77SpecialDistances[k][1] == int64_t(dist)) return k;
      return -1;
    };
    auto chan_of = [&](size_t i) { return std::upper_bound(chan_start.begin(), chan_start.end(), i) - chan_start.begin(); };
    for (size_t i = 0; i < n;) {
      size_t best = 0, best_j = 0;
      if (i > 0 && i + 4 <= n) {
        if (mult)
          for (int k = 0; k < 120; ++k) {
            const int64_t dd = int64_t(kLz77SpecialDistances[k][0]) + int64_t(mult) * kLz77SpecialDistances[k][1];
            if (dd < 1 || dd > int64_t(i)) continue;
            const size_t l = match_len(i - size_t(dd), i);
            if (l > best) best = l, best_j = i - size_t(dd);
          }
        int tries = 0;
        for (int32_t j = head[hash(i)]; j >= 0 && tries < 32; j = prev[size_t(j)], ++tries) {
          if (i - size_t(j) > kWindow) break;
          const size_t l = match_len(size_t(j), i);
          if (l > best) best = l, best_j = size_t(j);
        }
        const size_t l0 = i < kWindow ? match_len(0, i) : 0;  // ties go to the stream's first value
        if (l0 >= best && l0 > 0) best = l0, best_j = 0;
      }
      if (best >= h.min_length) {
        uint32_t d = uint32_t(i - best_j - 1);
        const int k = mult && best_j ? special(i - best_j) : -1;
        if (best_j == 0) d = (from_start++ & 1) ? uint32_t(i) + 1000 : (1u << 20) + 17;  // clamped to i by the decoder
        if (mult) {
          d = k >= 0 ? uint32_t(k) : d + 120;
          counts->special += k >= 0;
          counts->far += k < 0;
          counts->past_window += i >= kWindow;
          if (!chan_start.empty()) counts->cross_channel += chan_of(best_j) != chan_of(i) || chan_of(i + best - 1) != chan_of(i);
        }
        items.push_back({i, true, uint32_t(best - h.min_length), d});
        copied += best;
        for (size_t k = i; k < i + best; ++k) insert(k);
        i += best;
      } else {
        items.push_back({i, false, 0, 0});
        insert(i);
        ++i;
      }
    }
    // the last copy runs past the end of the stream
    if (mult) {
    } else if (!items.empty() && items.back().copy) {
      items.back().len_value += 5;
    } else if (n >= 2) {
      for (size_t j = n - 1; j-- > 0;)
        if (v(j) == v(n - 1)) {
          items.back() = {n - 1, true, 2, uint32_t(n - 2 - j)};
          ++copied;
          break;
        }
    }
    if (corrupt && opt.mode == "bad-first") items.insert(items.begin(), Item{0, true, 0, 0});
    if (corrupt && opt.mode == "bad-length" && n >= 2)
      items.insert(items.begin() + 1, Item{items[1].pos, true, 0xffffffffu - h.min_length + 1, 0});
  }
  std::vector<Sym> out;
  for (const Item& it : items) {
    Sym s{toks[it.pos].ctx, 0, 0, 0};
    if (!it.copy) {
      tokenize(v(it.pos), &s.tok, &s.nbits, &s.bits);
      if (s.tok >= h.min_symbol) fprintf(stderr, "a literal token reaches min_symbol\n"), exit(1);
      out.push_back(s);
      continue;
    }
    tokenize_with(h.len_cfg, it.len_value, &s.tok, &s.nbits, &s.bits);
    s.tok += h.min_symbol;
    out.push_back(s);
    Sym d{dist_ctx, 0, 0, 0};
    tokenize(it.dist_value, &d.tok, &d.nbits, &d.bits);
    out.push_back(d);
  }
  counts->copied += copied;
  counts->from_start += from_start;
  return out;
}

uint32_t pack_signed(int32_t v) { return v >= 0 ? uint32_t(v) << 1 : ((uint32_t(-(v + 1)) << 1) | 1); }

// ---- weighted predictor (same arithmetic as the decoder; crates/jxl-modular/src/predictor.rs:279-441)
struct Wp {
  uint32_t width = 0, x = 0, y = 0;
  std::vector<int32_t> te_row;
  std::vector<uint32_t> se_row;
  int32_t te_w = 0, te_nw = 0, te_n = 0, te_ne = 0;
  uint32_t a[4] = {}, b[4] = {}, c[4] = {};
  int64_t prediction = 0, sub[4] = {};
  int32_t max_error = 0;
  void reset(uint32_t w) {
    *this = Wp();
    width = w;
    te_row.assign(w, 0);
    se_row.assign(size_t(w) * 4, 0);
  }
  static uint32_t ilog2(uint64_t v) {
    uint32_t r = 0;
    while (v >>= 1) ++r;
    return r;
  }
  void predict(int32_t n, int32_t nw, int32_t ne, int32_t w, int32_t nn) {
    const int64_t p1 = 16, p2 = 10, p3a = 7, p3b = 7, p3c = 7, p3d = 0, p3e = 0;
    const uint32_t mw[4] = {13, 12, 12, 12};
    int64_t tew = te_w, tenw = te_nw, ten = te_n, tene = te_ne;
    int64_t n3 = int64_t(n) << 3, nw3 = int64_t(nw) << 3, ne3 = int64_t(ne) << 3, w3 = int64_t(w) << 3, nn3 = int64_t(nn) << 3;
    sub[0] = w3 + ne3 - n3;
    sub[1] = n3 - (((tew + ten + tene) * p1) >> 5);
    sub[2] = w3 - (((tew + ten + tenw) * p2) >> 5);
    sub[3] = n3 - ((tenw * p3a + ten * p3b + tene * p3c + (nn3 - n3) * p3d + (nw3 - w3) * p3e) >> 5);
    uint32_t wt[4];
    for (int i = 0; i < 4; ++i) {
      uint32_t es = a[i] + b[i] + c[i];
      uint64_t t = (uint64_t(es) + 1) >> 5;
      uint32_t sh = t ? ilog2(t) : 0;
      wt[i] = 4 + ((mw[i] * ((1u << 24) / ((es >> sh) + 1))) >> sh);
    }
    uint32_t sw = wt[0] + wt[1] + wt[2] + wt[3];
    uint32_t lw = ilog2(uint64_t(sw) >> 4);
    for (auto& v : wt) v >>= lw;
    sw = wt[0] + wt[1] + wt[2] + wt[3];
    int64_t s = (int64_t(sw) >> 1) - 1;
    for (int i = 0; i < 4; ++i) s += sub[i] * int64_t(wt[i]);
    int64_t pred = (s * int64_t((1u << 24) / sw)) >> 24;
    if (((ten ^ tew) | (ten ^ tenw)) <= 0) {
      int64_t mn = std::min(std::min(n3, w3), ne3), mx = std::max(std::max(n3, w3), ne3);
      pred = std::min(std::max(pred, mn), mx);
    }
    int64_t me = tew;
    for (int64_t e : {ten, tenw, tene})
      if (std::llabs(e) > std::llabs(me)) me = e;
    prediction = pred;
    max_error = int32_t(me);
  }
  void record(int32_t sample_) {
    int64_t s8 = int64_t(sample_) << 3;
    int64_t true_err = prediction - s8;
    uint32_t e[4];
    for (int i = 0; i < 4; ++i) e[i] = uint32_t((uint64_t(std::llabs(sub[i] - s8)) + 3) >> 3);
    te_row[x] = int32_t(true_err);
    for (int i = 0; i < 4; ++i) se_row[size_t(x) * 4 + i] = e[i];
    ++x;
    if (x >= width) {
      ++y;
      x = 0;
      te_w = 0;
      te_n = te_row[0];
      te_nw = te_n;
      for (int i = 0; i < 4; ++i) b[i] = a[i] = se_row[i];
      if (width <= 1) {
        te_ne = te_n;
        for (int i = 0; i < 4; ++i) c[i] = b[i];
      } else {
        te_ne = te_row[1];
        for (int i = 0; i < 4; ++i) c[i] = se_row[4 + i];
      }
    } else {
      te_w = int32_t(true_err);
      te_nw = te_n;
      te_n = te_ne;
      for (int i = 0; i < 4; ++i) {
        a[i] = b[i];
        b[i] = c[i] + e[i];
      }
      if (x + 1 >= width) {
        te_ne = te_n;
        for (int i = 0; i < 4; ++i) c[i] = b[i];
      } else if (y != 0) {
        te_ne = te_row[x + 1];
        for (int i = 0; i < 4; ++i) c[i] = se_row[size_t(x + 1) * 4 + i];
      }
    }
  }
};

// ---- the global MA tree ----------------------------------------------------------------------
// [0] stream > S (HfMetadata streams) ? [1] : [2]
// [1] channel > 1 ? [3] : leaf(ctx, Zero)        (x_from_y / b_from_y)
// [3] channel > 2 ? leaf(West) : leaf(Zero)       (sharpness / block info)
// [2] LF coefficients: chain on property 15 (WP max error) with WP leaves, or one Gradient leaf
struct TreeNode {
  int property;
  int32_t value;
  int left, right;  // children (property > value -> left)
  uint32_t predictor;
};
const int32_t kWpThresholds[] = {400, 160, 64, 24, 8, 0, -8, -24, -64, -160, -400};  // descending

std::vector<TreeNode> build_tree(uint32_t hfmeta_stream_threshold, bool lf_wp) {
  std::vector<TreeNode> bfs;
  // constructed directly in BFS order (children indices are implied: next free pair)
  struct Q {
    int kind;  // 0 root, 1 meta, 3 meta2, 2 lf chain (arg = threshold index), 10.. leaves
    int arg;
  };
  std::vector<Q> queue = {{0, 0}};
  for (size_t i = 0; i < queue.size(); ++i) {
    Q q = queue[i];
    auto decision = [&](int prop, int32_t val, Q l, Q r) {
      bfs.push_back({prop, val, int(queue.size()), int(queue.size()) + 1, 0});
      queue.push_back(l);
      queue.push_back(r);
    };
    auto leaf = [&](uint32_t pred) { bfs.push_back({-1, 0, 0, 0, pred}); };
    switch (q.kind) {
      case 0: decision(1, int32_t(hfmeta_stream_threshold), {1, 0}, {2, 0}); break;
      case 1: decision(0, 1, {3, 0}, {10, 0}); break;
      case 3: decision(0, 2, {11, 0}, {10, 0}); break;
      case 2:
        if (!lf_wp) leaf(5);
        else if (q.arg < int(sizeof(kWpThresholds) / sizeof(kWpThresholds[0]))) decision(15, kWpThresholds[q.arg], {12, 0}, {2, q.arg + 1});
        else leaf(6);
        break;
      case 10: leaf(0); break;
      case 11: leaf(1); break;
      case 12: leaf(6); break;
    }
  }
  return bfs;
}

// leaf index (= context) of a tree for given property values; leaves are numbered in BFS order
struct TreeEval {
  std::vector<TreeNode> nodes;
  std::vector<int> leaf_ctx;
  explicit TreeEval(std::vector<TreeNode> n) : nodes(std::move(n)) {
    int c = 0;
    for (auto& nd : nodes) leaf_ctx.push_back(nd.property < 0 ? c++ : -1);
  }
  int num_leaves() const {
    int c = 0;
    for (int v : leaf_ctx) c += v >= 0;
    return c;
  }
  const TreeNode& walk(int32_t channel, int32_t stream, int32_t p15, int* ctx) const {
    int i = 0;
    while (nodes[i].property >= 0) {
      int32_t v = nodes[i].property == 0 ? channel : (nodes[i].property == 1 ? stream : p15);
      i = v > nodes[i].value ? nodes[i].left : nodes[i].right;
    }
    *ctx = leaf_ctx[i];
    return nodes[i];
  }
};

void write_tree(BitWriter& w, const TreeEval& te) {  // ma.rs:68-226
  std::vector<Token> toks;
  for (const TreeNode& n : te.nodes) {
    if (n.property >= 0) {
      toks.push_back({1, uint32_t(n.property + 1)});
      toks.push_back({0, pack_signed(n.value)});
    } else {
      toks.push_back({1, 0});
      toks.push_back({2, n.predictor});
      toks.push_back({3, 0});  // offset
      toks.push_back({4, 0});  // mul_log
      toks.push_back({5, 0});  // mul_bits
    }
  }
  EntropyEncoder enc;
  std::vector<uint8_t> map = {0, 1, 2, 3, 4, 5};
  enc.write_header(w, toks, 6, map);
  enc.write_tokens(w, toks);
}

// Tokens of one Modular stream with channels coded in order; `stream` is MA property 1.
struct Plane2D {
  uint32_t w = 0, h = 0;
  std::vector<int32_t> v;
  int32_t at(uint32_t x, uint32_t y) const { return v[size_t(y) * w + x]; }
};

void modular_tokens(const TreeEval& te, const std::vector<Plane2D>& channels, int32_t stream, std::vector<Token>* out) {
  Wp wp;
  for (size_t ci = 0; ci < channels.size(); ++ci) {
    const Plane2D& p = channels[ci];
    if (!p.w || !p.h) continue;
    wp.reset(p.w);
    for (uint32_t y = 0; y < p.h; ++y)
      for (uint32_t x = 0; x < p.w; ++x) {
        int32_t w_, n, nw;
        if (y == 0) {
          w_ = x ? p.at(x - 1, 0) : 0;
          n = w_, nw = w_;
        } else if (x == 0) {
          n = p.at(0, y - 1);
          w_ = n, nw = n;
        } else {
          w_ = p.at(x - 1, y), n = p.at(x, y - 1), nw = p.at(x - 1, y - 1);
        }
        int32_t ne = (y == 0 || x + 1 >= p.w) ? n : p.at(x + 1, y - 1);
        int32_t nn = y >= 2 ? p.at(x, y - 2) : n;
        wp.predict(n, nw, ne, w_, nn);
        int ctx;
        const TreeNode& leaf = te.walk(int32_t(ci), stream, wp.max_error, &ctx);
        int32_t pred;
        switch (leaf.predictor) {
          case 0: pred = 0; break;
          case 1: pred = w_; break;
          case 5: {
            int64_t g = int64_t(n) + w_ - nw, lo = std::min(n, w_), hi = std::max(n, w_);
            pred = int32_t(std::min(std::max(g, lo), hi));
            break;
          }
          default: pred = int32_t((wp.prediction + 3) >> 3); break;
        }
        int32_t value = p.at(x, y);
        out->push_back({uint32_t(ctx), pack_signed(value - pred)});
        wp.record(value);
      }
  }
}

void write_modular_header(BitWriter& w) {  // lib.rs:117-125: global tree, default WP, no transforms
  w.write(1, 1);
  w.write(1, 1);
  w.write(2, 0);
}

// ---- HF coefficient context model (jxl-vardct/src/hf_coeff.rs) ---------------------------------
const uint8_t kFreqCtx[63] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 11, 12, 13, 14, 15, 15, 16, 16, 17, 17, 18, 18, 19, 19, 20, 20, 21, 21, 22, 22, 23,
                              23, 23, 23, 24, 24, 24, 24, 25, 25, 25, 25, 26, 26, 26, 26, 27, 27, 27, 27, 28, 28, 28, 28, 29, 29, 29, 29, 30, 30, 30, 30};
const uint8_t kNzCtx[63] = {0, 31, 62, 62, 93, 93, 93, 93, 123, 123, 123, 123, 152, 152, 152, 152, 152, 152, 152, 152, 180, 180, 180, 180, 180, 180, 180, 180, 180, 180, 180, 180,
                            206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206};
const uint8_t kDefaultBlockCtxMap[39] = {0, 1, 2, 2, 3, 3, 4, 5, 6, 6, 6, 6, 6, 7, 8, 9, 9, 10, 11, 12, 13, 14, 14, 14, 14, 14, 7, 8, 9, 9, 10, 11, 12, 13, 14, 14, 14, 14, 14};

struct Block {
  uint16_t x, y;  // cell position in the frame
  uint8_t type;
  int32_t hf_mul;
};

struct Args {
  uint32_t width = 7680, height = 4320;
  uint32_t seed = 1;
  double distance = 1.0;
  bool lf_wp = true;
  std::string out = "synth.jxl";
  uint32_t passes = 1;    // HF coefficients split over this many passes (progressive; pass p carries shift passes-1-p)
  std::string colour;     // "" = all-default metadata (sRGB); p3 | rec2020-gamma | gray | dci | custom: an enum colour encoding
  bool lf_frame = false;  // put the LF image into a separate Modular LF frame (frame type 1, lf_level 1)
  uint32_t epf_iters = 2; // edge-preserving filter iterations (0..3); 2 = the all-default restoration filter
  bool gaborish = true;   // --no-gaborish: a VarDCT frame without Gaborish (or a Modular one with --modular-filters)
  float modular_sigma = 0; // --modular-filters S: Gaborish + `epf_iters` EPF iterations on a Modular frame, sigma S (f16)
  uint32_t sharpness_cell = 16;  // the sharpness map is constant over cells of this many 8x8 blocks (EPF sigma 0 in the first)
  uint32_t hf_presets = 1;// HF presets (hf_pass.rs): group g uses preset g % N, each preset has its own (rotated) cluster map
  std::string dump_raw;    // --modular: also write the source image (3 planes, int32 little endian) for lossless checks;
                           // with --ycbcr / --upsampling / --extra the coded Modular channels instead (dump_channels)
  bool modular = false;    // a Modular lossless frame (RGB 8 bit, RCT + default Squeeze, weighted predictor) instead of VarDCT
  bool all_types = false;  // every one of the 27 transform types in the frame (forced_layout), the rest drawn from all 27
  int only_type = -1;      // tile every group with this transform type wherever it fits, DCT8 elsewhere
  std::string dump_blocks; // write the varblock layout as text lines "x y type" (8x8 cells) in the order HfMetadata codes them
  HfLz77 hf_lz77;          // --hf-lz77 rle | match | bad-first | bad-length: LZ77 in the HF pass codes (see HfLz77)
  // Channels coded below the frame's resolution: a --modular frame with any of these is written without transforms,
  // from seeded integer samples at each channel's coded size (encode_channels); --extra also goes with VarDCT frames
  std::string ycbcr;       // --ycbcr 444 | 420 | 422 | 440: Cb, Y, Cr colour channels with that chroma subsampling; a
                           // VarDCT frame is then laid out like a JPEG transcode (ycbcr_shifts)
  std::string dump_coeffs; // --dump-coeffs FILE: a VarDCT frame's HF coefficients as the decoder accumulates them over
                           // the passes: per channel (X / Cb, Y, B / Cr) a plane of its blocks * 8 samples, int32
  uint32_t upsampling = 1; // --upsampling 1 | 2 | 4 | 8: the frame's colour upsampling (a VarDCT frame is coded at
                           // ceil(W / k) x ceil(H / k))
  // LfGlobal features of a VarDCT frame, drawn from generators of their own (the frame's other draws stay as without them)
  enum { kNoNoise, kSeededNoise, kZeroNoise } noise = kNoNoise;  // --noise / --noise-zero: noise parameters, seeded or all-zero LUT
  uint32_t splines = 0;    // --splines N: N seeded splines in frame coordinates (write_features)
  bool dangling_patch = false;  // --dangling-patch: one patch from reference slot 0, which no frame fills (a frame a
                                // decoder refuses, for tests of which check refuses it first)
  struct Extra {
    uint32_t type, bits, dim_shift, ec_upsampling;  // type: 0 alpha, 2 spot colour, 16 optional (unknown to renderers)
  };
  std::vector<Extra> extras;  // --extra TYPE:BITS:DIM_SHIFT:EC_UPSAMPLING, repeatable
  bool shifted() const { return !ycbcr.empty() || upsampling != 1 || !extras.empty(); }
  // modular_16bit_buffers promises that every sample fits int16: not so with 16-bit extra channels
  bool wide_samples() const {
    for (const Extra& e : extras)
      if (e.bits > 15) return true;
    return false;
  }
};

// The LfGlobal feature fields a VarDCT frame has before its LF dequantisation (lf_global.rs:60-105): splines, then noise.
// Spline i starts at a seeded point of the W x H frame: every even one in its top-left eighth (inside the coded-size
// planes of an upsampled frame, whatever its factor), every odd one in its right half (past them). Each has 1-3 further
// control points inside the frame. The splines depend on the
// seed and the frame size only. Their colour DCTs have a few low-frequency coefficients, their sigma DCT a positive DC of
// 3-10 quantised units.
void write_features(BitWriter& w, const Args& a, uint32_t W, uint32_t H) {
  if (a.dangling_patch) {  // Patches::parse (jxl-frame/src/data/patch.rs): an 8x8 patch at (0, 0), Replace
    const std::vector<Token> t = {{0, 1}, {1, 0}, {3, 0}, {3, 0}, {2, 7}, {2, 7}, {7, 0}, {4, 0}, {4, 0}, {5, 1}};
    EntropyEncoder enc;
    enc.write_header(w, t, 10, std::vector<uint8_t>(10, 0));
    enc.write_tokens(w, t);
  }
  if (a.splines) {  // Splines::parse + QuantSpline::parse (jxl-frame/src/data/spline.rs:18-66, 155-224)
    std::mt19937 srng(a.seed ^ 0x51ed27a5u);
    auto pick = [&](uint32_t lo, uint32_t hi) { return int64_t(lo + srng() % (hi - lo)); };  // [lo, hi)
    std::vector<std::vector<std::pair<int64_t, int64_t>>> pts(a.splines);
    for (uint32_t i = 0; i < a.splines; ++i) {
      if (i & 1) pts[i].push_back({W > 1 ? pick((W + 1) / 2, W) : 0, pick(0, H)});
      else pts[i].push_back({pick(0, (W + 7) / 8), pick(0, (H + 7) / 8)});
      const uint32_t n = 1 + srng() % 3;
      while (pts[i].size() <= n) {
        const std::pair<int64_t, int64_t> p{pick(0, W), pick(0, H)};
        if (p != pts[i].back()) pts[i].push_back(p);
        else if (W * H == 1) break;  // a 1 x 1 frame has no second point
      }
    }
    std::vector<Token> t;
    t.push_back({2, a.splines - 1});
    t.push_back({1, uint32_t(pts[0][0].first)});
    t.push_back({1, uint32_t(pts[0][0].second)});
    for (uint32_t i = 1; i < a.splines; ++i) {
      t.push_back({1, pack_signed(int32_t(pts[i][0].first - pts[i - 1][0].first))});
      t.push_back({1, pack_signed(int32_t(pts[i][0].second - pts[i - 1][0].second))});
    }
    t.push_back({0, pack_signed(int32_t(srng() % 5) - 2)});  // quant_adjust
    for (uint32_t i = 0; i < a.splines; ++i) {
      t.push_back({3, uint32_t(pts[i].size() - 1)});
      int64_t dx = 0, dy = 0;  // the points are coded as second differences
      for (size_t k = 1; k < pts[i].size(); ++k) {
        const int64_t nx = pts[i][k].first - pts[i][k - 1].first, ny = pts[i][k].second - pts[i][k - 1].second;
        t.push_back({4, pack_signed(int32_t(nx - dx))});
        t.push_back({4, pack_signed(int32_t(ny - dy))});
        dx = nx, dy = ny;
      }
      for (int c = 0; c < 3; ++c)  // X, Y, B
        for (int k = 0; k < 32; ++k) {
          const int32_t range[3] = {40, 12, 12};
          t.push_back({5, pack_signed(k < 4 ? int32_t(srng() % (2 * range[c] + 1)) - range[c] : 0)});
        }
      for (int k = 0; k < 32; ++k) t.push_back({5, pack_signed(k == 0 ? 3 + int32_t(srng() % 8) : (k < 3 ? int32_t(srng() % 3) - 1 : 0))});
    }
    EntropyEncoder enc;
    enc.write_header(w, t, 6, std::vector<uint8_t>(6, 0));
    enc.write_tokens(w, t);
  }
  if (a.noise != Args::kNoNoise) {  // NoiseParameters (jxl-frame/src/data/noise.rs): eight u(10) LUT entries / 1024
    std::mt19937 nrng(a.seed ^ 0x6e015e00u);
    for (int i = 0; i < 8; ++i) w.write(10, a.noise == Args::kZeroNoise ? 0 : 64 + nrng() % 512);
  }
}

// Varblocks placed before the random layout is drawn (--all-types / --only-type): the transform type at each block's
// top-left cell, -1 elsewhere. Groups are 32 x 32 cells.
std::vector<int8_t> forced_layout(const Args& a, uint32_t bw, uint32_t bh) {
  std::vector<int8_t> forced(size_t(bw) * bh, -1);
  std::vector<int8_t> covered(size_t(bw) * bh, 0);
  const uint32_t gcols = (bw + 31) / 32, grows = (bh + 31) / 32;
  auto place = [&](int t, uint32_t x, uint32_t y) {
    const uint32_t w = kTransformInfo[t].w8, h = kTransformInfo[t].h8;
    if (x / 32 != (x + w - 1) / 32 || y / 32 != (y + h - 1) / 32 || x + w > bw || y + h > bh)
      fprintf(stderr, "forced varblock %d at (%u, %u) does not fit its group\n", t, x, y), exit(2);
    for (uint32_t dy = 0; dy < h; ++dy)
      for (uint32_t dx = 0; dx < w; ++dx) {
        if (covered[size_t(y + dy) * bw + x + dx]) fprintf(stderr, "forced varblocks overlap at (%u, %u)\n", x + dx, y + dy), exit(2);
        covered[size_t(y + dy) * bw + x + dx] = 1;
      }
    forced[size_t(y) * bw + x] = int8_t(t);
  };
  auto group_size = [&](uint32_t gx, uint32_t gy, uint32_t* w, uint32_t* h) {
    *w = std::min(32u, bw - gx * 32), *h = std::min(32u, bh - gy * 32);
  };
  if (a.only_type >= 0) {
    const uint32_t w = kTransformInfo[a.only_type].w8, h = kTransformInfo[a.only_type].h8;
    for (uint32_t gy = 0; gy < grows; ++gy)
      for (uint32_t gx = 0; gx < gcols; ++gx) {
        uint32_t gw, gh;
        group_size(gx, gy, &gw, &gh);
        for (uint32_t y = 0; y + h <= gh; y += h)
          for (uint32_t x = 0; x + w <= gw; x += w) place(a.only_type, gx * 32 + x, gy * 32 + y);
      }
    return forced;
  }
  // The first three full groups hold a catalogue of all 27 types: DCT256 | DCT256x128, DCT128, DCT128x64, DCT64x32,
  // DCT32x64 | DCT128x256, DCT64x128, DCT64 and a row of the 18 types of at most 32 x 32 samples.
  std::vector<uint32_t> full;
  for (uint32_t gy = 0; gy < grows && full.size() < 3; ++gy)
    for (uint32_t gx = 0; gx < gcols && full.size() < 3; ++gx) {
      uint32_t gw, gh;
      group_size(gx, gy, &gw, &gh);
      if (gw == 32 && gh == 32) full.push_back(gy * gcols + gx);
    }
  if (full.size() < 3) fprintf(stderr, "--all-types needs a frame with at least three full 256 x 256 groups\n"), exit(2);
  auto origin = [&](uint32_t g, uint32_t* x, uint32_t* y) { *x = g % gcols * 32, *y = g / gcols * 32; };
  uint32_t x0, y0;
  origin(full[0], &x0, &y0);
  place(kDct256, x0, y0);
  origin(full[1], &x0, &y0);
  place(kDct256x128, x0, y0);
  place(kDct128, x0 + 16, y0);
  place(kDct128x64, x0 + 16, y0 + 16);
  place(kDct64x32, x0 + 24, y0 + 16);
  place(kDct32x64, x0 + 24, y0 + 24);
  origin(full[2], &x0, &y0);
  place(kDct128x256, x0, y0);
  place(kDct64x128, x0, y0 + 16);
  place(kDct64, x0 + 16, y0 + 16);
  const int small[] = {kDct32, kDct32x16, kDct16x32, kDct32x8, kDct8x32, kDct16, kDct16x8, kDct8x16, kDct8, kHornuss, kDct2,
                       kDct4, kDct4x8, kDct8x4, kAfv0, kAfv1, kAfv2, kAfv3};
  uint32_t sx = x0;
  for (int t : small) place(t, sx, y0 + 24), sx += kTransformInfo[t].w8;
  // Partial groups at the right / bottom edges and the groups on either side of an LF-group boundary (every 8 groups)
  // get the largest type of at least 64 x 64 samples that fits at their origin.
  const int big[] = {kDct256, kDct256x128, kDct128x256, kDct128, kDct128x64, kDct64x128, kDct64, kDct64x32, kDct32x64};
  for (uint32_t gy = 0; gy < grows; ++gy)
    for (uint32_t gx = 0; gx < gcols; ++gx) {
      const uint32_t g = gy * gcols + gx;
      if (std::find(full.begin(), full.end(), g) != full.end()) continue;
      uint32_t gw, gh;
      group_size(gx, gy, &gw, &gh);
      const bool lf_edge = gx % 8 == 7 || (gx % 8 == 0 && gx) || gy % 8 == 7 || (gy % 8 == 0 && gy);
      if (gw == 32 && gh == 32 && !lf_edge) continue;
      for (int t : big)
        if (kTransformInfo[t].w8 <= gw && kTransformInfo[t].h8 <= gh) {
          place(t, gx * 32, gy * 32);
          break;
        }
    }
  return forced;
}

// ---- Modular lossless frame (BASELINE config #4): forward RCT (YCoCg, type 6), forward Squeeze with the default
// parameter schedule (jxl-modular/src/transform.rs:285-341), channels split into the global / LF-group / pass-group
// streams the decoder expects (jxl-modular/src/image.rs:187-345), every stream coded with the weighted predictor under a
// WP-error context chain. Lossless by construction: the decoder's inverse transforms undo these exactly.
struct MChan {
  Plane2D p;
  int hshift = 0, vshift = 0;
};

int32_t sq_tendency(int32_t a, int32_t b, int32_t c) {  // squeeze.rs:1104-1137
  if (a >= b && b >= c) {
    int32_t x = (4 * a - 3 * c - b + 6) / 12;
    if (x - (x & 1) > 2 * (a - b)) x = 2 * (a - b) + 1;
    if (x + (x & 1) > 2 * (b - c)) x = 2 * (b - c);
    return x;
  } else if (a <= b && b <= c) {
    int32_t x = (4 * a - 3 * c - b - 6) / 12;
    if (x + (x & 1) < 2 * (a - b)) x = 2 * (a - b) - 1;
    if (x - (x & 1) < 2 * (b - c)) x = 2 * (b - c);
    return x;
  }
  return 0;
}

// Forward of inverse_h / inverse_v (squeeze.rs:59-120, 803-862): avg = first - diff / 2 (truncating), residual =
// diff - tendency(previous second, avg, next avg).
void forward_squeeze(const MChan& in, bool horizontal, MChan* avg, MChan* res) {
  const uint32_t w = in.p.w, h = in.p.h;
  *avg = in;
  *res = in;
  if (horizontal) {
    avg->p.w = (w + 1) / 2, res->p.w = w / 2;
    avg->hshift = res->hshift = in.hshift + 1;
  } else {
    avg->p.h = (h + 1) / 2, res->p.h = h / 2;
    avg->vshift = res->vshift = in.vshift + 1;
  }
  avg->p.v.assign(size_t(avg->p.w) * avg->p.h, 0);
  res->p.v.assign(size_t(res->p.w) * res->p.h, 0);
  const uint32_t lines = horizontal ? h : w, len = horizontal ? w : h;
  const uint32_t alen = (len + 1) / 2, rlen = len / 2;
  std::vector<int32_t> line(len), av(alen);
  for (uint32_t l = 0; l < lines; ++l) {
    for (uint32_t i = 0; i < len; ++i) line[i] = horizontal ? in.p.at(i, l) : in.p.at(l, i);
    for (uint32_t i = 0; i < rlen; ++i) {
      const int32_t diff = line[2 * i] - line[2 * i + 1];
      av[i] = line[2 * i] - diff / 2;
    }
    if (len & 1) av[alen - 1] = line[len - 1];
    for (uint32_t i = 0; i < alen; ++i) (horizontal ? avg->p.v[size_t(l) * alen + i] : avg->p.v[size_t(i) * avg->p.w + l]) = av[i];
    int32_t left = av[0];
    for (uint32_t i = 0; i < rlen; ++i) {
      const int32_t next_avg = i + 1 < alen ? av[i + 1] : av[i];
      const int32_t diff = line[2 * i] - line[2 * i + 1];
      const int32_t r = diff - sq_tendency(left, av[i], next_avg);
      (horizontal ? res->p.v[size_t(l) * rlen + i] : res->p.v[size_t(i) * res->p.w + l]) = r;
      left = line[2 * i + 1];
    }
  }
}

struct SqStep {
  bool horizontal, in_place;
  uint32_t begin_c, num_c;
};

int write_modular_frame(const Args& a, const std::vector<MChan>& ch, uint32_t cw, uint32_t chh);

// jpeg_upsampling of the frame header for --ycbcr (Cb, Y, Cr): 1 leaves a channel at full size in both directions, 2 and 3
// in the vertical / horizontal one; 0 subsamples it wherever another channel asks for it (param.rs:105-122)
std::array<uint32_t, 3> jpeg_upsampling(const Args& a) {
  const uint32_t y = a.ycbcr == "420" ? 1 : a.ycbcr == "422" ? 2 : a.ycbcr == "440" ? 3 : 0;
  return {0, y, 0};
}

// The channel shifts of --ycbcr (ChannelShift::from_jpeg_upsampling, as host/planner.cc derives them): channel c (Cb, Y,
// Cr) keeps one sample (or 8x8 block) per (1 << hs[c]) x (1 << vs[c]) luma ones. All zero without --ycbcr.
void ycbcr_shifts(const Args& a, uint32_t hs[3], uint32_t vs[3]) {
  const std::array<uint32_t, 3> ju = jpeg_upsampling(a);
  bool h_any = false, v_any = false;
  for (uint32_t j : ju) h_any |= j == 1 || j == 2, v_any |= j == 1 || j == 3;
  for (int c = 0; c < 3; ++c) {
    hs[c] = h_any && (ju[c] == 0 || ju[c] == 3);
    vs[c] = v_any && (ju[c] == 0 || ju[c] == 2);
  }
}

// num_extra and one ExtraChannelInfo per --extra (jxl-image/src/lib.rs:303-345)
void write_extra_channels(BitWriter& w, const Args& a) {
  const uint32_t n = uint32_t(a.extras.size());
  if (n < 2) write_u32(w, int(n), 0, 0);
  else write_u32(w, 2, 4, n - 2);
  for (const Args::Extra& e : a.extras) {
    w.write(1, 0);  // not the default alpha channel
    if (e.type < 2) write_u32(w, int(e.type), 0, 0);
    else if (e.type < 18) write_u32(w, 2, 4, e.type - 2);
    else write_u32(w, 3, 6, e.type - 18);
    w.write(1, 0);  // integer samples
    if (e.bits == 8 || e.bits == 10 || e.bits == 12) write_u32(w, int((e.bits - 8) / 2), 0, 0);
    else write_u32(w, 3, 6, e.bits - 1);
    if (e.dim_shift == 0) write_u32(w, 0, 0, 0);
    else if (e.dim_shift == 3) write_u32(w, 1, 0, 0);
    else if (e.dim_shift == 4) write_u32(w, 2, 0, 0);
    else write_u32(w, 3, 3, e.dim_shift - 1);
    write_u32(w, 0, 0, 0);  // empty name
    if (e.type == 0) w.write(1, 0);  // alpha not premultiplied
    if (e.type == 2)
      for (float f : {0.75f, 0.5f, 0.25f, 0.625f}) w.write(16, to_f16(f));  // spot colour RGB and solidity
  }
}

// The channels of a frame-level Modular image split into streams (image.rs:187-345): the global prefix of channels
// that fit one group, then every other channel cut by its shift into LF groups (shift >= 3) or pass groups.
struct ModularStreams {
  std::vector<Plane2D> global;
  std::vector<std::vector<Plane2D>> lf, pg;
};
ModularStreams split_streams(const std::vector<MChan>& ch, uint32_t cw, uint32_t chh) {
  const uint32_t gd = 256;
  const uint32_t gcols = (cw + gd - 1) / gd, grows = (chh + gd - 1) / gd;
  const uint32_t lcols = (cw + 2047) / 2048, lrows = (chh + 2047) / 2048;
  ModularStreams st;
  st.lf.resize(size_t(lcols) * lrows);
  st.pg.resize(size_t(gcols) * grows);
  size_t nglobal = 0;
  while (nglobal < ch.size() && ch[nglobal].p.w <= gd && ch[nglobal].p.h <= gd) st.global.push_back(ch[nglobal++].p);
  auto crop = [](const Plane2D& p, uint32_t x0, uint32_t y0, uint32_t w, uint32_t h) {
    Plane2D o;
    o.w = w, o.h = h;
    o.v.resize(size_t(w) * h);
    for (uint32_t y = 0; y < h; ++y)
      for (uint32_t x = 0; x < w; ++x) o.v[size_t(y) * w + x] = p.at(x0 + x, y0 + y);
    return o;
  };
  for (size_t i = nglobal; i < ch.size(); ++i) {
    const MChan& c = ch[i];
    const bool lf = c.hshift >= 3 && c.vshift >= 3;
    const uint32_t gw = lf ? gd >> (c.hshift - 3) : gd >> c.hshift, gh = lf ? gd >> (c.vshift - 3) : gd >> c.vshift;
    if (!gw || !gh) fprintf(stderr, "channel shift too large\n"), exit(1);
    const uint32_t nx = lf ? lcols : gcols, ny = lf ? lrows : grows;
    for (uint32_t gy = 0; gy < ny; ++gy)
      for (uint32_t gx = 0; gx < nx; ++gx) {
        const uint32_t x0 = gx * gw, y0 = gy * gh;
        if (x0 >= c.p.w || y0 >= c.p.h) continue;
        Plane2D part = crop(c.p, x0, y0, std::min(gw, c.p.w - x0), std::min(gh, c.p.h - y0));
        (lf ? st.lf[gy * nx + gx] : st.pg[gy * nx + gx]).push_back(std::move(part));
      }
  }
  return st;
}

// A channel of seeded samples in [lo, hi]: a smooth ramp plus noise
MChan draw_channel(std::mt19937& rng, uint32_t w, uint32_t h, int hs, int vs, int32_t lo, int32_t hi) {
  MChan c;
  c.p.w = w, c.p.h = h, c.hshift = hs, c.vshift = vs;
  c.p.v.resize(size_t(w) * h);
  const double range = double(hi - lo), fx = 0.5 + double(rng() % 1000) / 500.0, fy = 0.5 + double(rng() % 1000) / 500.0;
  for (uint32_t y = 0; y < h; ++y)
    for (uint32_t x = 0; x < w; ++x) {
      const double s = 0.5 + 0.35 * std::sin(fx * x / 7.0 + fy * y / 11.0) + double(int(rng() % 17) - 8) / 160.0;
      c.p.v[size_t(y) * w + x] = lo + int32_t(std::min(range, std::max(0.0, std::floor(s * range + 0.5))));
    }
  return c;
}

// The --extra channels at their coded sizes over a cw x chh colour grid (lf_global.rs:270-290); a shift below zero is
// refused by the header rules, so such a channel is drawn at the colour size
void draw_extras(const Args& a, uint32_t cw, uint32_t chh, std::mt19937& rng, std::vector<MChan>* ch) {
  for (const Args::Extra& e : a.extras) {
    const int s = std::max(0, int(ceil_log2_nonzero(e.ec_upsampling) + e.dim_shift) - int(ceil_log2_nonzero(a.upsampling)));
    const uint32_t add = (1u << s) - 1;
    ch->push_back(draw_channel(rng, (cw + add) >> s, (chh + add) >> s, s, s, 0, int32_t((1u << e.bits) - 1)));
  }
}

// --dump-raw of channels coded without transforms: every channel in coding order, int32 little endian
int dump_channels(const Args& a, const std::vector<MChan>& ch) {
  if (a.dump_raw.empty()) return 0;
  FILE* rf = fopen(a.dump_raw.c_str(), "wb");
  if (!rf) return perror("fopen"), 1;
  for (const MChan& c : ch) fwrite(c.p.v.data(), 4, c.p.v.size(), rf);
  fclose(rf);
  return 0;
}

// --ycbcr / --upsampling / --extra: every channel drawn at its coded size (a smooth ramp plus noise over the sample
// range), coded without transforms. --dump-raw writes the coded channels in coding order, int32 little endian.
int encode_channels(const Args& a) {
  const uint32_t up = a.upsampling, cw = (a.width + up - 1) / up, chh = (a.height + up - 1) / up;
  std::mt19937 rng(a.seed);
  std::vector<MChan> ch;
  if (!a.ycbcr.empty()) {  // shift_size (param.rs:142-165), as host/frame_syntax.cc lays the channels out
    const std::array<uint32_t, 3> ju = jpeg_upsampling(a);
    bool h_any = false, v_any = false;
    for (uint32_t j : ju) h_any |= j == 1 || j == 2, v_any |= j == 1 || j == 3;
    for (uint32_t j : ju) {
      const bool hs = h_any && (j == 0 || j == 3), vs = v_any && (j == 0 || j == 2);
      const uint32_t w = h_any ? (hs ? (cw + 1) / 2 : (cw + 1) / 2 * 2) : cw;
      const uint32_t h = v_any ? (vs ? (chh + 1) / 2 : (chh + 1) / 2 * 2) : chh;
      ch.push_back(draw_channel(rng, w, h, hs, vs, -128, 127));  // Y is stored less 128/255 (ycbcr.rs), Cb and Cr centred on 0
    }
  } else {
    for (int c = 0; c < 3; ++c) ch.push_back(draw_channel(rng, cw, chh, 0, 0, 0, 255));
  }
  draw_extras(a, cw, chh, rng, &ch);
  if (int r = dump_channels(a, ch)) return r;
  return write_modular_frame(a, ch, cw, chh);
}

int encode_modular(const Args& a) {
  const uint32_t W = a.width, H = a.height, gd = 256;
  const uint32_t gcols = (W + gd - 1) / gd, grows = (H + gd - 1) / gd, num_groups = gcols * grows;
  if (num_groups == 1) fprintf(stderr, "single-group frames are not produced by this tool\n"), exit(2);
  std::mt19937 rng(a.seed);
  auto uni = [&](double lo, double hi) { return lo + (hi - lo) * (double(rng()) / 4294967296.0); };
  // ---- content: smooth colour fields, a few hard edges and sensor-like noise, 8 bit ----
  std::vector<MChan> ch(3);
  {
    const double fx = uni(0.002, 0.006), fy = uni(0.002, 0.006), gx = uni(0.03, 0.08), gy = uni(0.03, 0.08), ph = uni(0, 6.28);
    for (int c = 0; c < 3; ++c) ch[c].p.w = W, ch[c].p.h = H, ch[c].p.v.resize(size_t(W) * H);
    for (uint32_t y = 0; y < H; ++y)
      for (uint32_t x = 0; x < W; ++x) {
        const double base = 0.5 + 0.3 * sin(fx * x + ph) * cos(fy * y) + 0.08 * sin(gx * x + gy * y);
        const bool edge = ((x / 160 + y / 120) % 5) == 0;
        const double n = (double(rng() & 0xffff) / 65536.0 - 0.5) * 6.0;
        const double r = base * 255.0 + (edge ? 40.0 : 0.0) + n;
        const double g = (0.9 * base + 0.05 * cos(gx * x * 0.5)) * 255.0 + n * 0.8;
        const double b = (0.7 * base + 0.2 * sin(fy * y * 3.0 + 1.0)) * 255.0 - (edge ? 25.0 : 0.0) + n * 1.1;
        auto clamp8 = [](double v) { return int32_t(std::min(255.0, std::max(0.0, std::floor(v + 0.5)))); };
        ch[0].p.v[size_t(y) * W + x] = clamp8(r);
        ch[1].p.v[size_t(y) * W + x] = clamp8(g);
        ch[2].p.v[size_t(y) * W + x] = clamp8(b);
      }
  }
  if (!a.dump_raw.empty()) {
    FILE* rf = fopen(a.dump_raw.c_str(), "wb");
    if (!rf) return perror("fopen"), 1;
    for (int c = 0; c < 3; ++c) fwrite(ch[c].p.v.data(), 4, ch[c].p.v.size(), rf);
    fclose(rf);
  }
  // ---- forward RCT type 6 (rct.rs:87-140 inverse: tmp = Y - (Cg >> 1); G = Cg + tmp; B = tmp - (Co >> 1); R = B + Co) ----
  for (size_t i = 0; i < size_t(W) * H; ++i) {
    const int32_t r = ch[0].p.v[i], g = ch[1].p.v[i], b = ch[2].p.v[i];
    const int32_t co = r - b, tmp = b + (co >> 1), cg = g - tmp, yy = tmp + (cg >> 1);
    ch[0].p.v[i] = yy, ch[1].p.v[i] = co, ch[2].p.v[i] = cg;
  }
  // ---- forward Squeeze, default parameters (transform.rs:285-341) ----
  std::vector<SqStep> steps;
  {
    uint32_t w = W, h = H;
    steps.push_back({true, false, 1, 2});
    steps.push_back({false, false, 1, 2});
    if (h >= w && h > 8) {
      steps.push_back({false, true, 0, 3});
      h = (h + 1) / 2;
    }
    while (w > 8 || h > 8) {
      if (w > 8) steps.push_back({true, true, 0, 3}), w = (w + 1) / 2;
      if (h > 8) steps.push_back({false, true, 0, 3}), h = (h + 1) / 2;
    }
  }
  for (const SqStep& sp : steps) {
    std::vector<MChan> residu;
    for (uint32_t c = sp.begin_c; c < sp.begin_c + sp.num_c; ++c) {
      MChan avg, res;
      forward_squeeze(ch[c], sp.horizontal, &avg, &res);
      ch[c] = std::move(avg);
      residu.push_back(std::move(res));
    }
    if (sp.in_place) ch.insert(ch.begin() + sp.begin_c + sp.num_c, residu.begin(), residu.end());
    else ch.insert(ch.end(), residu.begin(), residu.end());
  }
  return write_modular_frame(a, ch, W, H);
}

// Writes a Modular frame of coded channels `ch` over a cw x ch_ colour sample grid: with a.shifted() without
// transforms and with the header fields of encode_channels, otherwise with RCT + default Squeeze.
int write_modular_frame(const Args& a, const std::vector<MChan>& ch, uint32_t cw, uint32_t chh) {
  const uint32_t W = a.width, H = a.height, gd = 256;
  const uint32_t gcols = (cw + gd - 1) / gd, grows = (chh + gd - 1) / gd, num_groups = gcols * grows;
  const uint32_t lcols = (cw + 2047) / 2048, lrows = (chh + 2047) / 2048, num_lf = lcols * lrows;
  const ModularStreams st = split_streams(ch, cw, chh);
  const size_t nglobal = st.global.size();
  const std::vector<std::vector<Plane2D>>& lf_streams = st.lf;
  const std::vector<std::vector<Plane2D>>& pg_streams = st.pg;
  // ---- tree: chain on the weighted predictor's max error, WP leaves; tokens of every stream ----
  std::vector<TreeNode> nodes;
  {
    const int nthr = int(sizeof(kWpThresholds) / sizeof(kWpThresholds[0]));
    for (int i = 0; i < nthr; ++i) nodes.push_back({15, kWpThresholds[i], 2 * i + 1, 2 * i + 2, 0}), nodes.push_back({-1, 0, 0, 0, 6});
    // BFS order: node 2i is the decision, 2i+1 its "greater" leaf, 2i+2 the next decision; the chain ends in a leaf
    nodes.push_back({-1, 0, 0, 0, 6});
    // rebuild in BFS order: decision i at index 2i, leaf at 2i+1, next decision at 2i+2
    std::vector<TreeNode> bfs;
    for (int i = 0; i < nthr; ++i) {
      bfs.push_back({15, kWpThresholds[i], 2 * i + 1, 2 * i + 2, 0});
      bfs.push_back({-1, 0, 0, 0, 6});
    }
    bfs.push_back({-1, 0, 0, 0, 6});
    nodes = bfs;
  }
  TreeEval tree(nodes);
  std::vector<Token> all;
  std::vector<Token> global_tokens;
  std::vector<std::vector<Token>> lf_tokens(num_lf), pg_tokens(num_groups);
  {
    std::vector<Plane2D> g;
    for (size_t i = 0; i < nglobal; ++i) g.push_back(ch[i].p);
    modular_tokens(tree, g, 0, &global_tokens);
    all.insert(all.end(), global_tokens.begin(), global_tokens.end());
  }
  for (uint32_t g = 0; g < num_lf; ++g) {
    modular_tokens(tree, lf_streams[g], int32_t(1 + num_lf + g), &lf_tokens[g]);
    all.insert(all.end(), lf_tokens[g].begin(), lf_tokens[g].end());
  }
  for (uint32_t g = 0; g < num_groups; ++g) {
    modular_tokens(tree, pg_streams[g], int32_t(1 + 3 * num_lf + 17 + g), &pg_tokens[g]);
    all.insert(all.end(), pg_tokens[g].begin(), pg_tokens[g].end());
  }
  // ---- --code lz77: each stream's values parsed into literals and copies (HfLz77 "modular") ----
  const bool lz77 = g_code == "lz77";
  HfLz77 lzopt{"modular", a.seed % 8};
  const Lz77Header lzh = lzopt.header();
  Lz77Counts lzc;
  std::vector<Sym> lz_global;
  std::vector<std::vector<Sym>> lz_lf(num_lf), lz_pg(num_groups);
  if (lz77) {
    const uint32_t dist_ctx = uint32_t(tree.num_leaves());
    auto parse = [&](const std::vector<Plane2D>& planes, const std::vector<Token>& toks, std::vector<Sym>* out) {
      uint32_t mult = 0;  // the widest channel of the stream
      std::vector<size_t> starts;
      size_t at = 0;
      for (const Plane2D& p : planes) {
        mult = std::max(mult, p.w);
        starts.push_back(at);
        at += size_t(p.w) * p.h;
      }
      *out = lz77_parse(toks, lzopt, dist_ctx, false, &lzc, mult, starts);
    };
    std::vector<Plane2D> g;
    for (size_t i = 0; i < nglobal; ++i) g.push_back(ch[i].p);
    parse(g, global_tokens, &lz_global);
    for (uint32_t i = 0; i < num_lf; ++i) parse(lf_streams[i], lf_tokens[i], &lz_lf[i]);
    for (uint32_t i = 0; i < num_groups; ++i) parse(pg_streams[i], pg_tokens[i], &lz_pg[i]);
  }
  // ---- sections ----
  std::vector<BitWriter> sections(1 + num_lf + 1 + num_groups);
  EntropyEncoder enc;
  auto write_stream = [&](BitWriter& w, const std::vector<Token>& toks, const std::vector<Sym>& syms) {
    if (lz77) enc.write_syms(w, syms);
    else enc.write_tokens(w, toks);
  };
  {
    BitWriter& w = sections[0];
    w.write(1, 1);  // LfChannelDequantization all_default
    w.write(1, 1);  // global MA tree present
    write_tree(w, tree);
    std::vector<uint8_t> map(size_t(tree.num_leaves()));
    for (size_t i = 0; i < map.size(); ++i) map[i] = uint8_t(i);
    if (lz77) {
      std::vector<Sym> syms = lz_global;
      for (const auto& v : lz_lf) syms.insert(syms.end(), v.begin(), v.end());
      for (const auto& v : lz_pg) syms.insert(syms.end(), v.begin(), v.end());
      map.push_back(uint8_t(map.size()));  // the distance context gets a cluster of its own
      enc.lz = &lzh;
      enc.write_header_syms(w, syms, uint32_t(map.size()), map);
      fprintf(stderr, "lz77-modular: min_symbol=%u min_length=%u symbol_sel=%d length_sel=%d copies_values=%llu "
                      "special=%llu far=%llu from_start=%llu cross_channel=%llu past_window=%llu\n",
              lzh.min_symbol, lzh.min_length, lzh.symbol_sel, lzh.length_sel, (unsigned long long)lzc.copied,
              (unsigned long long)lzc.special, (unsigned long long)lzc.far, (unsigned long long)lzc.from_start,
              (unsigned long long)lzc.cross_channel, (unsigned long long)lzc.past_window);
    } else {
      enc.write_header(w, all, uint32_t(map.size()), map);
    }
    if (a.shifted()) {
      write_modular_header(w);
    } else {  // GlobalModular header (lib.rs:117-125): global tree, default WP, two transforms
      w.write(1, 1);
      w.write(1, 1);
      write_u32(w, 2, 4, 0);  // nb_transforms = 2
      w.write(2, 0);          // RCT
      write_u32(w, 0, 3, 0);  //   begin_c = 0
      write_u32(w, 0, 0, 0);  //   rct_type = 6
      w.write(2, 2);          // Squeeze
      write_u32(w, 0, 0, 0);  //   num_sq = 0: default parameters
    }
    write_stream(w, global_tokens, lz_global);
    w.pad();
  }
  for (uint32_t g = 0; g < num_lf; ++g) {
    if (lf_streams[g].empty()) continue;
    BitWriter& w = sections[1 + g];
    write_modular_header(w);
    write_stream(w, lf_tokens[g], lz_lf[g]);
    w.pad();
  }
  for (uint32_t g = 0; g < num_groups; ++g) {
    if (pg_streams[g].empty()) continue;
    BitWriter& w = sections[2 + num_lf + g];
    write_modular_header(w);
    g_flip_state = g_corrupt == "ans-state" && g + 1 == num_groups;
    write_stream(w, pg_tokens[g], lz_pg[g]);
    w.pad();
  }
  // ---- codestream ----
  BitWriter cs;
  cs.write(16, 0x0aff);
  cs.write(1, 0);
  auto write_dim = [&](uint32_t v) {
    if (v <= 512) write_u32(cs, 0, 9, v - 1);
    else if (v <= 8192) write_u32(cs, 1, 13, v - 1);
    else write_u32(cs, 2, 18, v - 1);
  };
  write_dim(H);
  cs.write(3, 0);
  write_dim(W);
  cs.write(1, 0);  // ImageMetadata all_default = 0
  cs.write(1, 0);  // extra_fields
  cs.write(1, 0);  // integer samples
  cs.write(2, 0);  // 8 bits
  cs.write(1, a.wide_samples() ? 0 : 1);  // modular_16bit_buffers
  write_extra_channels(cs, a);
  cs.write(1, 0);  // xyb_encoded = 0
  cs.write(1, 1);  // ColourEncoding all_default (sRGB)
  cs.write(2, 0);  // extensions
  cs.write(1, 1);  // default_m
  cs.pad();
  // frame header (header.rs:9-134): Regular, Modular, no filters
  cs.write(1, 0);      // all_default
  cs.write(2, 0);      // Regular
  cs.write(1, 1);      // Modular
  cs.write(2, 0);      // flags = 0
  cs.write(1, a.ycbcr.empty() ? 0 : 1);  // do_ycbcr
  if (!a.ycbcr.empty())
    for (uint32_t j : jpeg_upsampling(a)) cs.write(2, j);
  cs.write(2, ceil_log2_nonzero(a.upsampling));  // upsampling: U32 selector k is 2^k
  for (const Args::Extra& e : a.extras) cs.write(2, ceil_log2_nonzero(e.ec_upsampling));
  cs.write(2, 1);      // group_size_shift = 1 (256)
  cs.write(2, 0);      // num_passes = 1
  cs.write(1, 0);      // have_crop
  cs.write(2, 0);      // blend mode Replace
  for (size_t i = 0; i < a.extras.size(); ++i) cs.write(2, 0);  // extra channels: Replace as well
  cs.write(1, 1);      // is_last
  cs.write(2, 0);      // name: empty
  cs.write(1, 0);      // restoration filter: not all_default
  if (a.modular_sigma > 0.0f) {  // filter.rs:18-166, Modular: no sharpness LUT, constant sigma sigma_for_modular
    cs.write(1, a.gaborish ? 1 : 0);  // gab_enabled
    if (a.gaborish) cs.write(1, 0);   // gab_custom
    cs.write(2, a.epf_iters & 3);
    if (a.epf_iters & 3) {
      cs.write(1, 0);   //   epf_weight_custom
      cs.write(1, 0);   //   epf_sigma_custom
      cs.write(16, to_f16(a.modular_sigma));
    }
  } else {
    cs.write(1, 0);    //   gab_enabled = 0
    cs.write(2, 0);    //   epf iters = 0
  }
  cs.write(2, 0);      //   extensions
  cs.write(2, 0);      // frame extensions
  cs.write(1, 0);      // TOC not permuted
  cs.pad();
  // one group: a single TOC entry; every channel fits the global stream, so LfGlobal is all there is
  if (num_groups == 1) sections.resize(1);
  if (g_corrupt == "truncate") sections.back().bytes.resize(sections.back().bytes.size() / 2);
  for (const BitWriter& sct : sections) {
    const uint32_t sz = uint32_t(sct.bytes.size());
    if (sz < 1024) write_u32(cs, 0, 10, sz);
    else if (sz < 17408) write_u32(cs, 1, 14, sz - 1024);
    else if (sz < 4211712) write_u32(cs, 2, 22, sz - 17408);
    else write_u32(cs, 3, 30, sz - 4211712);
  }
  cs.pad();
  for (const BitWriter& sct : sections) cs.append(sct);
  FILE* f = fopen(a.out.c_str(), "wb");
  if (!f) return perror("fopen"), 1;
  fwrite(cs.bytes.data(), 1, cs.bytes.size(), f);
  fclose(f);
  fprintf(stderr, "%s: %ux%u Modular lossless, %zu bytes (%.3f bit/px), %zu channels after Squeeze (%zu global), groups %u, LF groups %u\n",
          a.out.c_str(), W, H, cs.bytes.size(), 8.0 * cs.bytes.size() / (double(W) * H), ch.size(), nglobal, num_groups, num_lf);
  return 0;
}

}  // namespace

#ifndef SYNTH_ENC_NO_MAIN  // tools/hf_restream.cc includes this file for its entropy writer
int main(int argc, char** argv) {
  Args a;
  for (int i = 1; i < argc; ++i) {
    std::string s = argv[i];
    auto next = [&]() -> std::string { return i + 1 < argc ? argv[++i] : ""; };
    if (s == "--width") a.width = uint32_t(atoi(next().c_str()));
    else if (s == "--height") a.height = uint32_t(atoi(next().c_str()));
    else if (s == "--seed") a.seed = uint32_t(atoi(next().c_str()));
    else if (s == "--distance") a.distance = atof(next().c_str());
    else if (s == "--lf-gradient") a.lf_wp = false;
    else if (s == "--lf-frame") a.lf_frame = true;
    else if (s == "--passes") a.passes = uint32_t(atoi(next().c_str()));
    else if (s == "--colour") a.colour = next();
    else if (s == "--epf-iters") a.epf_iters = uint32_t(atoi(next().c_str()));
    else if (s == "--no-gaborish") a.gaborish = false;
    else if (s == "--sharpness-cell") a.sharpness_cell = uint32_t(std::max(1, atoi(next().c_str())));
    else if (s == "--modular-filters") a.modular_sigma = float(atof(next().c_str()));
    else if (s == "--hf-presets") a.hf_presets = std::max(1, atoi(next().c_str()));
    else if (s == "--modular") a.modular = true;
    else if (s == "--dump-raw") a.dump_raw = next();
    else if (s == "--all-types") a.all_types = true;
    else if (s == "--only-type") a.only_type = atoi(next().c_str());
    else if (s == "--dump-blocks") a.dump_blocks = next();
    else if (s == "--hf-lz77") a.hf_lz77.mode = next();
    else if (s == "--code") g_code = next();
    else if (s == "--corrupt") g_corrupt = next();
    else if (s == "-o") a.out = next();
    else if (s == "--ycbcr") a.ycbcr = next();
    else if (s == "--dump-coeffs") a.dump_coeffs = next();
    else if (s == "--upsampling") a.upsampling = uint32_t(atoi(next().c_str()));
    else if (s == "--noise") a.noise = Args::kSeededNoise;
    else if (s == "--dangling-patch") a.dangling_patch = true;
    else if (s == "--noise-zero") a.noise = Args::kZeroNoise;
    else if (s == "--splines") a.splines = uint32_t(std::max(1, atoi(next().c_str())));
    else if (s == "--extra") {
      const std::string spec = next();
      const size_t c1 = spec.find(':');
      const std::string type = spec.substr(0, c1);
      Args::Extra e{type == "alpha" ? 0u : type == "spot" ? 2u : 16u, 8, 0, 1};
      if (c1 == std::string::npos || (type != "alpha" && type != "spot" && type != "unknown") ||
          sscanf(spec.c_str() + c1 + 1, "%u:%u:%u", &e.bits, &e.dim_shift, &e.ec_upsampling) != 3 || e.bits < 1 ||
          e.bits > 16 || e.dim_shift > 8 || (e.ec_upsampling != 1 && e.ec_upsampling != 2 && e.ec_upsampling != 4 && e.ec_upsampling != 8))
        fprintf(stderr, "--extra takes alpha|spot|unknown:BITS(1..16):DIM_SHIFT(0..8):EC_UPSAMPLING(1|2|4|8)\n"), exit(2);
      a.extras.push_back(e);
    }
    else fprintf(stderr, "unknown arg %s\n", s.c_str()), exit(2);
  }
  if (!a.ycbcr.empty() && a.ycbcr != "444" && a.ycbcr != "420" && a.ycbcr != "422" && a.ycbcr != "440")
    fprintf(stderr, "--ycbcr takes 444, 420, 422 or 440\n"), exit(2);
  if (a.upsampling != 1 && a.upsampling != 2 && a.upsampling != 4 && a.upsampling != 8)
    fprintf(stderr, "--upsampling takes 1, 2, 4 or 8\n"), exit(2);
  if (!a.ycbcr.empty() && !a.modular &&
      (a.lf_frame || a.all_types || a.only_type >= 0 || !a.colour.empty() || a.upsampling != 1 || !a.extras.empty() ||
       a.noise != Args::kNoNoise || a.splines || a.dangling_patch))
    fprintf(stderr, "--ycbcr of a VarDCT frame is not written with --lf-frame, --all-types, --only-type, --colour, "
                    "--upsampling, --extra or LfGlobal features\n"), exit(2);
  if (!a.dump_coeffs.empty() && a.modular) fprintf(stderr, "--dump-coeffs goes with VarDCT frames\n"), exit(2);
  if ((a.noise != Args::kNoNoise || a.splines || a.dangling_patch) && a.modular)
    fprintf(stderr, "--noise, --splines and --dangling-patch go with VarDCT frames\n"), exit(2);
  if (a.upsampling != 1 && !a.modular && (a.lf_frame || !a.extras.empty()))
    fprintf(stderr, "--upsampling of a VarDCT frame is not written with --lf-frame or --extra\n"), exit(2);
  if (!a.extras.empty() && a.lf_frame) fprintf(stderr, "--extra is not written with --lf-frame\n"), exit(2);
  if (!g_code.empty() && g_code != "prefix" && g_code != "ans-forms" && g_code != "configs" && g_code != "clusters" &&
      g_code != "lz77")
    fprintf(stderr, "--code takes prefix, ans-forms, configs, clusters or lz77 (--modular)\n"), exit(2);
  if (g_code == "lz77" && !a.modular) fprintf(stderr, "--code lz77 goes with --modular frames\n"), exit(2);
  if (!g_corrupt.empty() && g_corrupt != "ans-state" && g_corrupt != "truncate" && g_corrupt != "oversub-clcl" &&
      g_corrupt != "oversub-lengths" && g_corrupt != "ans-sum")
    fprintf(stderr, "--corrupt takes ans-state, truncate, oversub-clcl, oversub-lengths or ans-sum\n"), exit(2);
  if ((g_corrupt == "oversub-clcl" || g_corrupt == "oversub-lengths") && g_code != "prefix")
    fprintf(stderr, "--corrupt %s goes with --code prefix\n", g_corrupt.c_str()), exit(2);
  if (g_corrupt == "ans-sum" && (g_code.empty() || g_code == "prefix" || g_code == "lz77"))
    fprintf(stderr, "--corrupt ans-sum goes with --code ans-forms, configs or clusters\n"), exit(2);
  if (!g_code.empty() && !a.hf_lz77.mode.empty()) fprintf(stderr, "--code is not written with --hf-lz77\n"), exit(2);
  if (!g_code.empty()) atexit([] { g_report.print(); });
  g_code_seed = a.seed;
  if (a.modular && a.shifted()) return encode_channels(a);
  const std::string& lzm = a.hf_lz77.mode;
  if (!lzm.empty() && (a.modular || (lzm != "rle" && lzm != "match" && lzm != "bad-first" && lzm != "bad-length")))
    fprintf(stderr, "--hf-lz77 takes rle, match, bad-first or bad-length (VarDCT frames only)\n"), exit(2);
  if (a.modular) return encode_modular(a);
  if (a.only_type >= int(kNumTransformTypes) || (a.only_type >= 0 && a.all_types))
    fprintf(stderr, "--only-type takes a transform type 0..26 (not with --all-types)\n"), exit(2);
  const bool ycbcr = !a.ycbcr.empty();
  if (ycbcr) a.only_type = kDct8;  // a JPEG transcode codes DCT8 in every cell
  uint32_t hs[3], vs[3];
  ycbcr_shifts(a, hs, vs);
  std::mt19937 rng(a.seed);
  auto uni = [&](double lo, double hi) { return lo + (hi - lo) * (double(rng()) / 4294967296.0); };
  // the frame's content at its coded size; the image (and frame) size is width x height
  const uint32_t up = a.upsampling, W = (a.width + up - 1) / up, H = (a.height + up - 1) / up;
  // in a subsampled direction the block grid is rounded up to an even size (whole chroma blocks), as the decoder lays
  // it out (blocks_w in host/planner.cc); the rounding never adds a group
  const bool h_sub = hs[0] | hs[1] | hs[2], v_sub = vs[0] | vs[1] | vs[2];
  const uint32_t bw = h_sub ? ((W + 7) / 8 + 1) / 2 * 2 : (W + 7) / 8, bh = v_sub ? ((H + 7) / 8 + 1) / 2 * 2 : (H + 7) / 8;
  const uint32_t gcols = (W + 255) / 256, grows = (H + 255) / 256, num_groups = gcols * grows;
  const uint32_t lcols = (W + 2047) / 2048, lrows = (H + 2047) / 2048, num_lf = lcols * lrows;
  if (a.passes < 1 || a.passes > 3 || (a.passes > 1 && a.lf_frame)) fprintf(stderr, "--passes takes 1..3 (not with --lf-frame)\n"), exit(2);
  const uint32_t P = a.passes;
  // one group and one pass: a single TOC entry holds LfGlobal, the LF group, HfGlobal and the pass group back to back,
  // without padding between them (toc.rs; host/frame_syntax.cc reads them from one bit position on)
  const bool single = num_groups == 1 && P == 1;
  auto end_section = [&](BitWriter& w) {
    if (!single) w.pad();
  };

  // ---- content ----
  // varblock layout: raster scan per LF group (the order HfMetadata stores blocks in)
  // mix roughly like a libjxl d1 photo: mostly 8x8, a fair share of 16x8/8x16/16x16, some 32x32/64x64
  const int mix_types[] = {kDct8, kDct8, kDct8, kDct16x8, kDct8x16, kDct16, kDct16, kDct32x16, kDct16x32, kDct32, kDct4x8, kDct8x4,
                           kAfv0, kDct4, kDct2, kHornuss, kDct64, kDct32x8, kDct8x32, kAfv3};
  std::vector<int8_t> occ(size_t(bw) * bh, 0);
  std::vector<int8_t> forced;
  if (a.all_types || a.only_type >= 0) {
    forced = forced_layout(a, bw, bh);
    for (uint32_t y = 0; y < bh; ++y)
      for (uint32_t x = 0; x < bw; ++x) {
        const int t = forced[size_t(y) * bw + x];
        if (t < 0) continue;
        for (uint32_t dy = 0; dy < kTransformInfo[t].h8; ++dy)
          for (uint32_t dx = 0; dx < kTransformInfo[t].w8; ++dx) occ[size_t(y + dy) * bw + x + dx] = 1;
      }
  }
  std::vector<std::vector<Block>> lf_blocks(num_lf);
  std::vector<int32_t> blk_type(size_t(bw) * bh, -1), blk_mul(size_t(bw) * bh, 0);
  for (uint32_t lg = 0; lg < num_lf; ++lg) {
    uint32_t lx0 = (lg % lcols) * 256, ly0 = (lg / lcols) * 256;
    uint32_t lw = std::min(256u, bw - lx0), lh = std::min(256u, bh - ly0);
    for (uint32_t y = 0; y < lh; ++y)
      for (uint32_t x = 0; x < lw; ++x) {
        const int forced_type = forced.empty() ? -1 : forced[size_t(ly0 + y) * bw + lx0 + x];
        if (forced_type < 0 && occ[size_t(ly0 + y) * bw + lx0 + x]) continue;
        int type = forced_type < 0 ? kDct8 : forced_type;
        for (int attempt = 0; forced_type < 0 && a.only_type < 0 && attempt < 4; ++attempt) {
          int t = a.all_types ? int(rng() % kNumTransformTypes) : mix_types[rng() % (sizeof(mix_types) / sizeof(int))];
          uint32_t dw = kTransformInfo[t].w8, dh = kTransformInfo[t].h8;
          bool ok = (x % 32) + dw <= 32 && (y % 32) + dh <= 32 && x + dw <= lw && y + dh <= lh;
          for (uint32_t dy = 0; ok && dy < dh; ++dy)
            for (uint32_t dx = 0; ok && dx < dw; ++dx) ok = !occ[size_t(ly0 + y + dy) * bw + lx0 + x + dx];
          if (ok) {
            type = t;
            break;
          }
        }
        uint32_t dw = kTransformInfo[type].w8, dh = kTransformInfo[type].h8;
        for (uint32_t dy = 0; dy < dh; ++dy)
          for (uint32_t dx = 0; dx < dw; ++dx) occ[size_t(ly0 + y + dy) * bw + lx0 + x + dx] = 1;
        int32_t hf_mul = 3 + int32_t(rng() % 8);
        lf_blocks[lg].push_back({uint16_t(lx0 + x), uint16_t(ly0 + y), uint8_t(type), hf_mul});
        blk_type[size_t(ly0 + y) * bw + lx0 + x] = type;
        blk_mul[size_t(ly0 + y) * bw + lx0 + x] = hf_mul;
      }
  }
  if (!a.dump_blocks.empty()) {
    FILE* bf = fopen(a.dump_blocks.c_str(), "w");
    if (!bf) return perror("fopen"), 1;
    for (const auto& blocks : lf_blocks)
      for (const Block& b : blocks) fprintf(bf, "%u %u %u\n", unsigned(b.x), unsigned(b.y), unsigned(b.type));
    fclose(bf);
  }
  // LF quantised values: smooth field + small noise (Y large range, X/B small)
  std::vector<int32_t> lfq[3];
  {
    double fx1 = uni(0.004, 0.012), fy1 = uni(0.004, 0.012), fx2 = uni(0.02, 0.05), fy2 = uni(0.02, 0.05), ph = uni(0, 6.28);
    for (int c = 0; c < 3; ++c) lfq[c].resize(size_t(bw) * bh);
    for (uint32_t y = 0; y < bh; ++y)
      for (uint32_t x = 0; x < bw; ++x) {
        double base = 0.5 + 0.35 * sin(fx1 * x + ph) * cos(fy1 * y) + 0.1 * sin(fx2 * x + fy2 * y);
        // Y: LF quant step = m_y_lf*2^9/(gs*qlf) = 0.25*512/86887 = 1.47e-3 -> Y in [0,0.8] ~ 0..540
        lfq[1][size_t(y) * bw + x] = int32_t(base * 500.0 + uni(-2, 2));
        lfq[0][size_t(y) * bw + x] = int32_t(12.0 * sin(fx2 * x * 0.7 + 1.0) * cos(fy2 * y * 0.9) + uni(-1.5, 1.5));
        lfq[2][size_t(y) * bw + x] = int32_t(base * 180.0 + 20.0 * cos(fx1 * x * 1.3) + uni(-2, 2));
      }
  }

  // ---- global tree + per-stream Modular tokens ----
  TreeEval tree(build_tree(2 * num_lf, a.lf_wp));
  std::vector<Token> lf_tokens_all;                 // histogram over every Modular stream
  std::vector<std::vector<Token>> lfcoeff_tokens(num_lf), hfmeta_tokens(num_lf);
  std::vector<uint32_t> nb_blocks(num_lf);
  for (uint32_t lg = 0; lg < num_lf; ++lg) {
    uint32_t lx0 = (lg % lcols) * 256, ly0 = (lg / lcols) * 256;
    uint32_t lw = std::min(256u, bw - lx0), lh = std::min(256u, bh - ly0);
    std::vector<Plane2D> ch(3);
    const int order[3] = {1, 0, 2};  // modular channels are Y, X, B
    for (int k = 0; k < 3; ++k) {  // each channel at its shifted grid, taken from the top-left part of lfq
      const int c = order[k];
      const uint32_t sw = (lw + (1u << hs[c]) - 1) >> hs[c], sh = (lh + (1u << vs[c]) - 1) >> vs[c];
      const uint32_t sx0 = lx0 >> hs[c], sy0 = ly0 >> vs[c];
      ch[k].w = sw, ch[k].h = sh;
      ch[k].v.resize(size_t(sw) * sh);
      for (uint32_t y = 0; y < sh; ++y)
        for (uint32_t x = 0; x < sw; ++x) ch[k].v[size_t(y) * sw + x] = lfq[c][size_t(sy0 + y) * bw + sx0 + x];
    }
    modular_tokens(tree, ch, int32_t(1 + lg), &lfcoeff_tokens[lg]);
    // HfMetadata: x_from_y, b_from_y (lw/8 x lh/8), block info (nb x 2), sharpness (lw x lh)
    std::vector<Plane2D> hm(4);
    uint32_t w64 = (lw + 7) / 8, h64 = (lh + 7) / 8;
    for (int k = 0; k < 2; ++k) {
      hm[k].w = w64, hm[k].h = h64;
      hm[k].v.resize(size_t(w64) * h64);
      for (auto& v : hm[k].v) v = ycbcr ? 0 : int32_t(rng() % 33) - 16;  // no chroma from luma in a JPEG transcode
    }
    const auto& blocks = lf_blocks[lg];
    nb_blocks[lg] = uint32_t(blocks.size());
    hm[2].w = uint32_t(blocks.size()), hm[2].h = 2;
    hm[2].v.resize(blocks.size() * 2);
    for (size_t i = 0; i < blocks.size(); ++i) {
      hm[2].v[i] = blocks[i].type;
      hm[2].v[blocks.size() + i] = blocks[i].hf_mul - 1;
    }
    hm[3].w = lw, hm[3].h = lh;
    hm[3].v.resize(size_t(lw) * lh);
    {  // piecewise-constant sharpness over cells of sharpness_cell x sharpness_cell blocks
      const uint32_t sc = a.sharpness_cell;
      for (uint32_t y = 0; y < lh; ++y)
        for (uint32_t x = 0; x < lw; ++x) hm[3].v[size_t(y) * lw + x] = int32_t(((x / sc) * 7 + (y / sc) * 3 + lg) % 8);
    }
    modular_tokens(tree, hm, int32_t(1 + 2 * num_lf + lg), &hfmeta_tokens[lg]);
    if (!a.lf_frame) lf_tokens_all.insert(lf_tokens_all.end(), lfcoeff_tokens[lg].begin(), lfcoeff_tokens[lg].end());
    lf_tokens_all.insert(lf_tokens_all.end(), hfmeta_tokens[lg].begin(), hfmeta_tokens[lg].end());
  }

  // ---- --extra: the extra channels' streams of the frame's Modular image (GlobalModular, LF groups, and pass groups
  // of the last pass, after its HF data), coded with the global tree like the other Modular streams ----
  std::vector<Token> ex_global_tokens;
  std::vector<std::vector<Token>> ex_lf_tokens(num_lf), ex_pg_tokens(num_groups);
  if (!a.extras.empty()) {
    std::mt19937 erng(a.seed ^ 0x9e3779b9u);  // apart from the frame's own draws, which stay as without --extra
    std::vector<MChan> ech;
    draw_extras(a, W, H, erng, &ech);
    if (int r = dump_channels(a, ech)) return r;
    const ModularStreams st = split_streams(ech, W, H);
    modular_tokens(tree, st.global, 0, &ex_global_tokens);
    lf_tokens_all.insert(lf_tokens_all.end(), ex_global_tokens.begin(), ex_global_tokens.end());
    for (uint32_t lg = 0; lg < num_lf; ++lg) {
      modular_tokens(tree, st.lf[lg], int32_t(1 + num_lf + lg), &ex_lf_tokens[lg]);
      lf_tokens_all.insert(lf_tokens_all.end(), ex_lf_tokens[lg].begin(), ex_lf_tokens[lg].end());
    }
    for (uint32_t g = 0; g < num_groups; ++g) {
      modular_tokens(tree, st.pg[g], int32_t(1 + 3 * num_lf + 17 + (P - 1) * num_groups + g), &ex_pg_tokens[g]);
      lf_tokens_all.insert(lf_tokens_all.end(), ex_pg_tokens[g].begin(), ex_pg_tokens[g].end());
    }
  }

  // ---- HF tokens per group ----
  const uint32_t nbc = 15;
  const double kScale = 1.0 / std::max(0.25, a.distance);  // coefficient magnitude scale
  std::vector<std::vector<uint32_t>> orders(13);
  for (uint32_t id = 0; id < 13; ++id) orders[id] = natural_order(id);
  // hf_tokens[pass * num_groups + group]; a coefficient c is sent as sum over passes of (part_p << shift_p), with
  // part_p = remainder / 2^shift_p truncated toward zero
  std::vector<std::vector<Token>> hf_tokens(size_t(P) * num_groups);
  std::exponential_distribution<double> expo(1.0);
  std::vector<int32_t> dump[3];  // --dump-coeffs: channel c's plane is dump_w[c] samples wide
  uint32_t dump_w[3];
  for (int c = 0; c < 3; ++c) {
    dump_w[c] = ((bw + (1u << hs[c]) - 1) >> hs[c]) * 8;
    if (!a.dump_coeffs.empty()) dump[c].assign(size_t(dump_w[c]) * (((bh + (1u << vs[c]) - 1) >> vs[c]) * 8), 0);
  }
  for (uint32_t g = 0; g < num_groups; ++g) {
    uint32_t bx0 = (g % gcols) * 32, by0 = (g / gcols) * 32;
    uint32_t gw = std::min(32u, bw - bx0), gh = std::min(32u, bh - by0);
    std::vector<uint32_t> nz_rows[3][3];
    for (auto& pr : nz_rows)
      for (auto& v : pr) v.assign(gw, 0);
    std::vector<int32_t> coeffs, full;
    for (uint32_t y = 0; y < gh; ++y)
      for (uint32_t x = 0; x < gw; ++x) {
        int32_t t = blk_type[size_t(by0 + y) * bw + bx0 + x];
        if (t < 0) continue;
        const TransformTypeInfo& ti = kTransformInfo[t];
        uint32_t num_blocks = uint32_t(ti.w8) * ti.h8, nb_log = ceil_log2_nonzero(num_blocks), size = num_blocks * 64;
        for (int ci = 0; ci < 3; ++ci) {
          int c = ci == 0 ? 1 : (ci == 1 ? 0 : 2);
          // a subsampled channel codes only the blocks aligned to its grid, at the shifted position (hf_coeff.rs:143-155)
          const uint32_t sx = x >> hs[c], sy = y >> vs[c];
          if ((sx << hs[c]) != x || (sy << vs[c]) != y) continue;
          uint32_t block_ctx = kDefaultBlockCtxMap[ci * 13 + ti.order_id];
          // synthesise coefficients along the scan order: Laplacian with decaying scale
          full.assign(size, 0);
          double chan_scale = (c == 1 ? 1.0 : (c == 0 ? 0.35 : 0.55)) * kScale * uni(0.4, 1.6);
          for (uint32_t k = num_blocks; k < size; ++k) {
            double pos = double(k) / num_blocks;  // 1..64
            double b = chan_scale * 2.6 / (1.0 + pos * 0.55);
            double mag = expo(rng) * b;
            int32_t q = int32_t(mag + 0.35);
            if (q) full[k] = (rng() & 1) ? q : -q;
          }
          if (!a.dump_coeffs.empty())
            for (uint32_t k = num_blocks; k < size; ++k) {
              uint32_t dx = orders[ti.order_id][k] & 0xffff, dy = orders[ti.order_id][k] >> 16;
              if (ti.transpose) std::swap(dx, dy);
              const size_t px = size_t((bx0 >> hs[c]) + sx) * 8 + dx, py = size_t((by0 >> vs[c]) + sy) * 8 + dy;
              dump[c][py * dump_w[c] + px] = full[k];
            }
          for (uint32_t pass = 0; pass < P; ++pass) {
          const uint32_t shift = P - 1 - pass;
          std::vector<Token>& toks = hf_tokens[size_t(pass) * num_groups + g];
          std::vector<uint32_t>* nz_row = nz_rows[pass];
          coeffs.assign(size, 0);
          uint32_t non_zeros = 0;
          for (uint32_t k = num_blocks; k < size; ++k) {
            coeffs[k] = full[k] / (int32_t(1) << shift);
            full[k] -= coeffs[k] * (int32_t(1) << shift);
            if (coeffs[k]) ++non_zeros;
          }
          uint32_t predicted;
          if (sy == 0) predicted = sx == 0 ? 32 : nz_row[c][sx - 1];
          else if (sx == 0) predicted = nz_row[c][sx];
          else predicted = (nz_row[c][sx] + nz_row[c][sx - 1] + 1) >> 1;
          uint32_t pidx = predicted >= 8 ? 4 + predicted / 2 : predicted;
          toks.push_back({block_ctx + pidx * nbc, non_zeros});
          uint32_t nz_val = (non_zeros + num_blocks - 1) >> nb_log;
          for (uint32_t dx = 0; dx < ti.w8; ++dx) nz_row[c][sx + dx] = nz_val;
          if (!non_zeros) continue;
          uint32_t prev = non_zeros <= num_blocks * 4 ? 1 : 0;
          uint32_t base = block_ctx * 458 + 37 * nbc;
          uint32_t remaining = non_zeros;
          for (uint32_t k = num_blocks, i = 0; k < size; ++k, ++i) {
            uint32_t nzc = (remaining - 1) >> nb_log, fi = i >> nb_log;
            uint32_t cctx = (uint32_t(kNzCtx[nzc]) + kFreqCtx[fi]) * 2 + prev;
            int32_t v = coeffs[k];
            toks.push_back({base + cctx, pack_signed(v)});
            if (!v) {
              prev = 0;
              continue;
            }
            prev = 1;
            if (--remaining == 0) break;
          }
          }
        }
      }
  }
  if (!a.dump_coeffs.empty()) {
    FILE* df = fopen(a.dump_coeffs.c_str(), "wb");
    if (!df) return perror("fopen"), 1;
    for (const auto& d : dump) fwrite(d.data(), 4, d.size(), df);
    fclose(df);
  }
  // context clustering for the HF code (495 * nbc contexts -> 28 clusters)
  std::vector<uint8_t> hf_map(495 * nbc, 0);
  for (uint32_t ctx = 0; ctx < 495 * nbc; ++ctx) {
    if (ctx < 37 * nbc) {
      uint32_t block_ctx = ctx % nbc, pidx = ctx / nbc;
      hf_map[ctx] = uint8_t((block_ctx >= 7 ? 2 : 0) + (pidx >= 8 ? 1 : 0));
    } else {
      uint32_t r = ctx - 37 * nbc;
      uint32_t block_ctx = r / 458, cc = r % 458;
      uint32_t chan = block_ctx >= 7 ? 1 : 0;
      uint32_t half = cc >> 1, prev = cc & 1;
      uint32_t bucket = std::min<uint32_t>(5, half / 40);
      hf_map[ctx] = uint8_t(4 + chan * 12 + bucket * 2 + prev);
    }
  }
  // HF presets: preset p owns contexts [p * 495 * nbc, (p + 1) * 495 * nbc) of the pass code; its cluster map is the
  // base map rotated by p clusters, so a decoder that picks the wrong preset's slice reads the stream with other
  // distributions. Group g selects preset g % NP (written at the start of its stream).
  const uint32_t NP = std::min<uint32_t>(a.hf_presets, num_groups);
  if (NP > 1) {
    const uint32_t ncl = 28, per = 495 * nbc;
    std::vector<uint8_t> all(size_t(per) * NP);
    for (uint32_t pr = 0; pr < NP; ++pr)
      for (uint32_t ctx = 0; ctx < per; ++ctx) all[size_t(pr) * per + ctx] = uint8_t((hf_map[ctx] + pr) % ncl);
    hf_map.swap(all);
    for (uint32_t pass = 0; pass < P; ++pass)
      for (uint32_t g = 0; g < num_groups; ++g)
        for (Token& t : hf_tokens[size_t(pass) * num_groups + g]) t.ctx += (g % NP) * per;
  }
  std::vector<std::vector<Token>> hf_all(P);
  for (uint32_t pass = 0; pass < P; ++pass)
    for (uint32_t g = 0; g < num_groups; ++g) {
      const auto& t = hf_tokens[size_t(pass) * num_groups + g];
      hf_all[pass].insert(hf_all[pass].end(), t.begin(), t.end());
    }
  // --hf-lz77: the same values, parsed into literals and copies; the distance context gets a cluster of its own
  const Lz77Header lz_header = a.hf_lz77.header();
  const uint32_t hf_num_ctx = 495 * nbc * NP;
  std::vector<std::vector<Sym>> hf_syms(a.hf_lz77.mode.empty() ? 0 : size_t(P) * num_groups), hf_syms_all(P);
  if (!a.hf_lz77.mode.empty()) {
    Lz77Counts lzc;
    for (uint32_t pass = 0; pass < P; ++pass)
      for (uint32_t g = 0; g < num_groups; ++g) {
        std::vector<Sym>& s = hf_syms[size_t(pass) * num_groups + g];
        s = lz77_parse(hf_tokens[size_t(pass) * num_groups + g], a.hf_lz77, hf_num_ctx, pass == 0 && g == 0, &lzc);
        hf_syms_all[pass].insert(hf_syms_all[pass].end(), s.begin(), s.end());
      }
    hf_map.push_back(uint8_t(*std::max_element(hf_map.begin(), hf_map.end()) + 1));
    fprintf(stderr, "hf-lz77 %s: %llu values copied, %llu copies from the first value\n", a.hf_lz77.mode.c_str(),
            (unsigned long long)lzc.copied, (unsigned long long)lzc.from_start);
  }

  // ---- sections ----
  const uint32_t global_scale = uint32_t(std::lround(5111.0 / std::max(0.1, a.distance))), quant_lf = 17;
  std::vector<BitWriter> sections(1 + num_lf + 1 + size_t(P) * num_groups);
  EntropyEncoder lf_enc;
  std::vector<EntropyEncoder> hf_enc(P);
  {  // LfGlobal
    BitWriter& w = sections[0];
    write_features(w, a, a.width, a.height);
    w.write(1, 1);  // LfChannelDequantization all_default
    // Quantizer: global_scale U32(1+u11, 2049+u11, 4097+u12, 8193+u16), quant_lf U32(16, 1+u5, 1+u8, 1+u16)
    if (global_scale <= 2048) write_u32(w, 0, 11, global_scale - 1);
    else if (global_scale <= 4096) write_u32(w, 1, 11, global_scale - 2049);
    else if (global_scale <= 8192) write_u32(w, 2, 12, global_scale - 4097);
    else write_u32(w, 3, 16, global_scale - 8193);
    write_u32(w, 1, 5, quant_lf - 1);
    w.write(1, 1);  // HfBlockContext default
    if (ycbcr) {    // LfChannelCorrelation of a JPEG transcode: no chroma from luma (base correlations 0)
      w.write(1, 0);
      write_u32(w, 0, 0, 0);  // colour_factor 84
      w.write(16, 0);         // base_correlation_x = 0.0 (f16)
      w.write(16, 0);         // base_correlation_b = 0.0 (f16)
      w.write(8, 128);        // x_factor_lf
      w.write(8, 128);        // b_factor_lf
    } else {
      w.write(1, 1);  // LfChannelCorrelation all_default
    }
    w.write(1, 1);  // global MA tree present
    write_tree(w, tree);
    std::vector<uint8_t> map(size_t(tree.num_leaves()));
    for (size_t i = 0; i < map.size(); ++i) map[i] = uint8_t(i);
    lf_enc.write_header(w, lf_tokens_all, uint32_t(map.size()), map);
    if (!a.extras.empty()) {  // GlobalModular stream
      write_modular_header(w);
      lf_enc.write_tokens(w, ex_global_tokens);
    }
    end_section(w);
  }
  for (uint32_t lg = 0; lg < num_lf; ++lg) {
    BitWriter& w = sections[1 + lg];
    uint32_t lx0 = (lg % lcols) * 256, ly0 = (lg / lcols) * 256;
    uint32_t lw = std::min(256u, bw - lx0), lh = std::min(256u, bh - ly0);
    if (!a.lf_frame) {
      w.write(2, 0);  // extra_precision
      write_modular_header(w);
      lf_enc.write_tokens(w, lfcoeff_tokens[lg]);
    }
    if (!ex_lf_tokens[lg].empty()) {  // Modular LF-group channels, between LfCoeff and HfMetadata
      write_modular_header(w);
      lf_enc.write_tokens(w, ex_lf_tokens[lg]);
    }
    w.write(int(ceil_log2_nonzero(lw * lh)), nb_blocks[lg] - 1);
    write_modular_header(w);
    lf_enc.write_tokens(w, hfmeta_tokens[lg]);
    end_section(w);
  }
  {  // HfGlobal
    BitWriter& w = sections[1 + num_lf];
    w.write(1, 1);                                   // default dequant matrices
    w.write(int(ceil_log2_nonzero(num_groups)), NP - 1);  // num_hf_presets - 1
    for (uint32_t pass = 0; pass < P; ++pass) {
      write_u32(w, 2, 0, 0);  // used_orders = 0
      if (a.hf_lz77.mode.empty()) {
        hf_enc[pass].write_header(w, hf_all[pass], hf_num_ctx, hf_map);
      } else {
        hf_enc[pass].lz = &lz_header;
        hf_enc[pass].write_header_syms(w, hf_syms_all[pass], hf_num_ctx + 1, hf_map);
      }
    }
    end_section(w);
  }
  for (uint32_t pass = 0; pass < P; ++pass)
    for (uint32_t g = 0; g < num_groups; ++g) {
      BitWriter& w = sections[2 + num_lf + size_t(pass) * num_groups + g];
      w.write(int(ceil_log2_nonzero(NP)), g % NP);  // hfp: 0 bits with a single preset
      g_flip_state = g_corrupt == "ans-state" && pass == 0 && g == 0;
      if (a.hf_lz77.mode.empty()) hf_enc[pass].write_tokens(w, hf_tokens[size_t(pass) * num_groups + g]);
      else hf_enc[pass].write_syms(w, hf_syms[size_t(pass) * num_groups + g]);
      if (pass + 1 == P && !ex_pg_tokens[g].empty()) {  // Modular pass-group channels, after the HF data
        write_modular_header(w);
        lf_enc.write_tokens(w, ex_pg_tokens[g]);
      }
      end_section(w);
    }

  // ---- codestream ----
  BitWriter cs;
  cs.write(16, 0x0aff);
  // SizeHeader (jxl-image/src/lib.rs:98-113): explicit sizes
  cs.write(1, 0);
  auto write_dim = [&](uint32_t v) {
    if (v <= 512) write_u32(cs, 0, 9, v - 1);
    else if (v <= 8192) write_u32(cs, 1, 13, v - 1);
    else write_u32(cs, 2, 18, v - 1);
  };
  write_dim(a.height);
  cs.write(3, 0);  // ratio
  write_dim(a.width);
  if (a.colour.empty() && a.extras.empty() && !ycbcr) {
    cs.write(1, 1);  // ImageMetadata all_default
  } else {  // ImageMetadata with extra channels and / or an enum ColourEncoding (jxl-image/src/lib.rs:229-287, color.rs:21-58)
    const bool pq = a.colour == "pq";
    cs.write(1, 0);  // all_default
    cs.write(1, pq ? 1 : 0);  // extra_fields
    if (pq) {
      cs.write(3, 0);  // orientation 1
      cs.write(1, 0);  // have_intrinsic_size
      cs.write(1, 0);  // have_preview
      cs.write(1, 0);  // have_animation
    }
    cs.write(1, 0);  // integer samples
    cs.write(2, 0);  // 8 bits
    cs.write(1, a.wide_samples() ? 0 : 1);  // modular_16bit_buffers
    write_extra_channels(cs, a);
    cs.write(1, ycbcr ? 0 : 1);  // xyb_encoded
    cs.write(1, a.colour.empty() ? 1 : 0);  // ColourEncoding all_default (sRGB)
  }
  if (!a.colour.empty()) {
    const bool pq = a.colour == "pq";
    auto write_enum = [&](uint32_t v) {
      if (v == 0) write_u32(cs, 0, 0, 0);
      else if (v == 1) write_u32(cs, 1, 0, 0);
      else if (v < 18) write_u32(cs, 2, 4, v - 2);
      else write_u32(cs, 3, 6, v - 18);
    };
    auto write_xy = [&](double x, double y) {
      for (double c : {x, y}) {
        const uint32_t u = pack_signed(int32_t(std::lround(c * 1e6)));
        if (u < 524288) write_u32(cs, 0, 19, u);
        else if (u < 1048576) write_u32(cs, 1, 19, u - 524288);
        else if (u < 2097152) write_u32(cs, 2, 20, u - 1048576);
        else write_u32(cs, 3, 21, u - 2097152);
      }
    };
    cs.write(1, 0);  // want_icc
    const bool grey = a.colour == "gray";
    write_enum(grey ? 1 : 0);  // colour space: RGB / Grey
    if (a.colour == "dci") write_enum(11);  // white point: DCI
    else if (a.colour == "custom") write_enum(2), write_xy(0.3457, 0.3585);  // custom (D50-like)
    else write_enum(1);  // D65
    if (!grey) {
      if (a.colour == "p3" || a.colour == "dci") write_enum(11);
      else if (a.colour == "rec2020-gamma" || pq) write_enum(9);
      else if (a.colour == "custom") write_enum(2), write_xy(0.64, 0.33), write_xy(0.21, 0.71), write_xy(0.15, 0.06);  // Adobe RGB-like
      else fprintf(stderr, "unknown --colour %s\n", a.colour.c_str()), exit(2);
    }
    if (a.colour == "rec2020-gamma" || a.colour == "custom") {
      cs.write(1, 1);  // has_gamma
      cs.write(24, a.colour == "custom" ? 4545455 : 4166667);  // 1/2.2, 1/2.4
    } else {
      cs.write(1, 0);
      write_enum(a.colour == "dci" ? 17 : (pq ? 16 : 13));  // DCI / PQ / sRGB
    }
    write_enum(1);   // rendering intent: relative
    if (pq) {  // ToneMapping (color.rs:312-319): 1000 nits
      cs.write(1, 0);        // all_default
      cs.write(16, 0x63d0);  // intensity_target = 1000.0 (f16)
      cs.write(16, 0);       // min_nits
      cs.write(1, 0);        // relative_to_max_display
      cs.write(16, 0);       // linear_below
    }
  }
  if (!a.colour.empty() || !a.extras.empty() || ycbcr) cs.write(2, 0);  // extensions
  cs.write(1, 1);  // default_m
  cs.pad();
  auto write_u64_small = [&](uint32_t v) {  // U64 (jxl-bitstream): 0 | 1 + u(4) | 17 + u(8)
    if (v == 0) cs.write(2, 0);
    else if (v <= 16) cs.write(2, 1), cs.write(4, v - 1);
    else cs.write(2, 2), cs.write(8, v - 17);
  };
  auto write_section_size = [&](uint32_t sz) {
    if (sz < 1024) write_u32(cs, 0, 10, sz);
    else if (sz < 17408) write_u32(cs, 1, 14, sz - 1024);
    else if (sz < 4211712) write_u32(cs, 2, 22, sz - 17408);
    else write_u32(cs, 3, 30, sz - 4211712);
  };
  if (a.lf_frame) {
    // ---- the LF frame: Modular, XYB, ceil(W/8) x ceil(H/8), one group, one TOC entry ----
    if (bw > 256 || bh > 256) fprintf(stderr, "--lf-frame needs an image of at most 2048x2048\n"), exit(2);
    // integer XYB samples: Y, X, B - Y with X = x * m_x_lf/128 etc. (defaults 1/32, 1/4, 1/2;
    // jxl-render/src/image.rs:148-189); the smooth field of the LF quant values, rescaled
    std::vector<Plane2D> ch(3);
    for (auto& c : ch) c.w = bw, c.h = bh, c.v.resize(size_t(bw) * bh);
    for (size_t i = 0; i < size_t(bw) * bh; ++i) {
      const int32_t iy = lfq[1][i] / 2, ix = lfq[0][i] * 2, ib = lfq[2][i] / 2;
      ch[0].v[i] = iy;       // Y = iy / 512       (0 .. ~0.45)
      ch[1].v[i] = ix;       // X = ix / 4096
      ch[2].v[i] = ib - iy;  // B = (ib) / 256
    }
    TreeEval lf_tree(build_tree(1000000, a.lf_wp));
    std::vector<Token> toks;
    modular_tokens(lf_tree, ch, 0, &toks);
    BitWriter sec;
    sec.write(1, 1);  // LfChannelDequantization all_default
    sec.write(1, 1);  // global MA tree present
    write_tree(sec, lf_tree);
    std::vector<uint8_t> map(size_t(lf_tree.num_leaves()));
    for (size_t i = 0; i < map.size(); ++i) map[i] = uint8_t(i);
    EntropyEncoder enc;
    enc.write_header(sec, toks, uint32_t(map.size()), map);
    write_modular_header(sec);
    enc.write_tokens(sec, toks);
    sec.pad();
    // frame header (jxl-frame/src/header.rs:9-134)
    cs.write(1, 0);      // all_default
    cs.write(2, 1);      // frame_type = LfFrame
    cs.write(1, 1);      // encoding = Modular
    write_u64_small(0);  // flags
    cs.write(2, 0);      // upsampling = 1
    cs.write(2, 1);      // group_size_shift = 1 (256)
    cs.write(2, 0);      // num_passes = 1
    cs.write(2, 0);      // lf_level - 1
    cs.write(2, 0);      // name: empty
    cs.write(1, 0);      // restoration filter: not all_default
    cs.write(1, 0);      //   gab_enabled = 0
    cs.write(2, 0);      //   epf iters = 0
    write_u64_small(0);  //   extensions
    write_u64_small(0);  // frame extensions
    cs.write(1, 0);      // TOC not permuted
    cs.pad();
    write_section_size(uint32_t(sec.bytes.size()));
    cs.pad();
    cs.append(sec);
    // ---- main frame header: VarDCT with use_lf_frame ----
    cs.write(1, 0);         // all_default
    cs.write(2, 0);         // Regular
    cs.write(1, 0);         // VarDCT
    write_u64_small(0x20);  // flags: use_lf_frame
    cs.write(3, 3);         // x_qm_scale
    cs.write(3, 2);         // b_qm_scale
    cs.write(2, 0);         // num_passes = 1
    cs.write(1, 0);         // have_crop
    cs.write(2, 0);         // blend mode Replace
    cs.write(1, 1);         // is_last
    cs.write(2, 0);         // name: empty
    cs.write(1, 1);         // restoration filter all_default
    write_u64_small(0);     // frame extensions
  } else if (P > 1 || a.epf_iters != 2 || !a.gaborish || !a.extras.empty() || up != 1 || a.noise != Args::kNoNoise || a.splines || a.dangling_patch ||
             ycbcr) {
    cs.write(1, 0);         // all_default
    cs.write(2, 0);         // Regular
    cs.write(1, 0);         // VarDCT
    // flags: noise, patches, splines, skip_adaptive_lf_smoothing (set in every JPEG transcode)
    write_u64_small((a.noise != Args::kNoNoise ? 0x1 : 0) | (a.dangling_patch ? 0x2 : 0) | (a.splines ? 0x10 : 0) | (ycbcr ? 0x80 : 0));
    if (ycbcr) {
      cs.write(1, 1);  // do_ycbcr
      for (uint32_t j : jpeg_upsampling(a)) cs.write(2, j);
    }
    cs.write(2, ceil_log2_nonzero(up));  // upsampling: U32 selector k is 2^k
    for (const Args::Extra& e : a.extras) cs.write(2, ceil_log2_nonzero(e.ec_upsampling));  // U32 selector k is 2^k
    if (!ycbcr) {
      cs.write(3, 3);       // x_qm_scale
      cs.write(3, 2);       // b_qm_scale
    }
    cs.write(2, P - 1);     // num_passes (1, 2 or 3)
    if (P > 1) {
      cs.write(2, 0);       // num_ds = 0
      for (uint32_t pass = 0; pass + 1 < P; ++pass) cs.write(2, P - 1 - pass);  // shift
    }
    cs.write(1, 0);         // have_crop
    cs.write(2, 0);         // blend mode Replace
    for (size_t i = 0; i < a.extras.size(); ++i) cs.write(2, 0);  // extra channels: Replace as well
    cs.write(1, 1);         // is_last
    cs.write(2, 0);         // name: empty
    if (a.epf_iters == 2 && a.gaborish) {
      cs.write(1, 1);       // restoration filter all_default
    } else {                // filter.rs: Gaborish with default weights or off, `epf_iters` EPF iterations, default parameters
      cs.write(1, 0);
      cs.write(1, a.gaborish ? 1 : 0);  //   gab_enabled
      if (a.gaborish) cs.write(1, 0);   //   gab_custom
      cs.write(2, a.epf_iters & 3);
      if (a.epf_iters & 3) {
        cs.write(1, 0);     //   epf_sharp_custom
        cs.write(1, 0);     //   epf_weight_custom
        cs.write(1, 0);     //   epf_sigma_custom
      }
      write_u64_small(0);   //   extensions
    }
    write_u64_small(0);     // frame extensions
  } else {
    cs.write(1, 1);  // FrameHeader all_default
  }
  cs.write(1, 0);  // TOC not permuted
  cs.pad();
  if (single) {
    BitWriter one;
    for (const BitWriter& s : sections) one.append_bits(s);
    one.pad();
    sections.assign(1, one);
  }
  for (const BitWriter& s : sections) {
    uint32_t sz = uint32_t(s.bytes.size());
    if (sz < 1024) write_u32(cs, 0, 10, sz);
    else if (sz < 17408) write_u32(cs, 1, 14, sz - 1024);
    else if (sz < 4211712) write_u32(cs, 2, 22, sz - 17408);
    else write_u32(cs, 3, 30, sz - 4211712);
  }
  cs.pad();
  size_t lf_bytes = 0, hf_bytes = 0;
  for (size_t i = 0; i < sections.size(); ++i) {
    cs.append(sections[i]);
    if (i >= 1 && i < 1 + num_lf) lf_bytes += sections[i].bytes.size();
    if (i >= 2 + num_lf) hf_bytes += sections[i].bytes.size();
  }
  FILE* f = fopen(a.out.c_str(), "wb");
  if (!f) return perror("fopen"), 1;
  fwrite(cs.bytes.data(), 1, cs.bytes.size(), f);
  fclose(f);
  fprintf(stderr, "%s: %ux%u, %zu bytes (%.3f bit/px), LF sections %zu B, HF sections %zu B, groups %u, LF groups %u\n", a.out.c_str(), W,
          H, cs.bytes.size(), 8.0 * cs.bytes.size() / (double(W) * H), lf_bytes, hf_bytes, num_groups, num_lf);
  return 0;
}
#endif
