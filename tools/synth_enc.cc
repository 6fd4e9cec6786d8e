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
//
// Not part of the product; not a general-purpose encoder (it does not transform an input image).
#include <algorithm>
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

// HybridUintConfig (4, 2, 0): the configuration libjxl uses for these streams
const uint32_t kSplitExp = 4, kMsb = 2, kLsb = 0;
void tokenize(uint32_t v, uint32_t* token, uint32_t* nbits, uint32_t* bits) {
  const uint32_t split = 1u << kSplitExp;
  if (v < split) {
    *token = v;
    *nbits = 0;
    *bits = 0;
    return;
  }
  uint32_t n = 31 - uint32_t(__builtin_clz(v));
  uint32_t m = v - (1u << n);
  *token = split + ((n - kSplitExp) << (kMsb + kLsb)) + ((m >> (n - kMsb)) << kLsb) + (m & ((1u << kLsb) - 1));
  *nbits = n - kMsb - kLsb;
  *bits = (m >> kLsb) & ((1u << *nbits) - 1);
}

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

// Writes the entropy-code header for `tokens` (clustered by `cluster_of_ctx`) and then the ANS
// stream itself (32-bit initial state first).
struct EntropyEncoder {
  uint32_t num_ctx = 0, num_clusters = 0, log_alpha = 0;
  std::vector<uint8_t> cluster_of_ctx;
  std::vector<std::vector<uint32_t>> counts;     // per cluster, normalised
  std::vector<std::vector<std::vector<uint16_t>>> inv;  // cluster -> symbol -> offset -> idx

  void write_header(BitWriter& w, const std::vector<Token>& tokens, uint32_t num_ctx_, const std::vector<uint8_t>& map) {
    num_ctx = num_ctx_;
    cluster_of_ctx = map;
    num_clusters = 0;
    for (uint8_t c : map) num_clusters = std::max<uint32_t>(num_clusters, c + 1u);
    std::vector<std::vector<uint64_t>> freq(num_clusters);
    uint32_t max_tok = 0;
    for (const Token& t : tokens) {
      uint32_t tok, nb, b;
      tokenize(t.value, &tok, &nb, &b);
      auto& f = freq[map[t.ctx]];
      if (f.size() <= tok) f.resize(tok + 1, 0);
      ++f[tok];
      max_tok = std::max(max_tok, tok);
    }
    log_alpha = 5;
    while ((1u << log_alpha) <= max_tok) ++log_alpha;
    if (log_alpha > 8) fprintf(stderr, "token alphabet too large\n"), exit(1);
    BitWriter hw;
    hw.write(1, 0);  // lz77 disabled
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
    EntropyCode code = parse_entropy_code(br, num_ctx);
    if (code.num_clusters != num_clusters || code.log_alphabet_size != log_alpha) fprintf(stderr, "header readback mismatch\n"), exit(1);
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

  void write_tokens(BitWriter& w, const std::vector<Token>& tokens) const {
    struct Out {
      uint16_t ans_bits;
      uint8_t has_ans;
      uint8_t nbits;
      uint32_t bits;
    };
    std::vector<Out> outs(tokens.size());
    uint32_t state = 0x130000;
    for (size_t k = tokens.size(); k-- > 0;) {
      uint32_t tok, nb, b;
      tokenize(tokens[k].value, &tok, &nb, &b);
      uint32_t c = cluster_of_ctx[tokens[k].ctx];
      uint32_t f = counts[c][tok];
      Out& o = outs[k];
      o.nbits = uint8_t(nb);
      o.bits = b;
      o.has_ans = 0;
      if ((state >> 20) >= f) {
        o.has_ans = 1;
        o.ans_bits = uint16_t(state & 0xffff);
        state >>= 16;
      }
      state = ((state / f) << 12) + inv[c][tok][state % f];
    }
    w.write(32, state);
    for (const Out& o : outs) {
      if (o.has_ans) w.write(16, o.ans_bits);
      if (o.nbits) w.write(o.nbits, o.bits);
    }
  }
};

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
  std::string dump_raw;    // --modular: also write the source image (3 planes, int32 little endian) for lossless checks
  bool modular = false;    // a Modular lossless frame (RGB 8 bit, RCT + default Squeeze, weighted predictor) instead of VarDCT
  bool all_types = false;  // every one of the 27 transform types in the frame (forced_layout), the rest drawn from all 27
  int only_type = -1;      // tile every group with this transform type wherever it fits, DCT8 elsewhere
  std::string dump_blocks; // write the varblock layout as text lines "x y type" (8x8 cells) in the order HfMetadata codes them
};

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

int encode_modular(const Args& a) {
  const uint32_t W = a.width, H = a.height, gd = 256;
  const uint32_t gcols = (W + gd - 1) / gd, grows = (H + gd - 1) / gd, num_groups = gcols * grows;
  const uint32_t lcols = (W + 2047) / 2048, lrows = (H + 2047) / 2048, num_lf = lcols * lrows;
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
  // ---- streams (image.rs:187-345): global prefix, then by shift into LF groups (shift >= 3) or pass groups ----
  size_t nglobal = 0;
  while (nglobal < ch.size() && ch[nglobal].p.w <= gd && ch[nglobal].p.h <= gd) ++nglobal;
  std::vector<std::vector<Plane2D>> lf_streams(num_lf), pg_streams(num_groups);
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
        (lf ? lf_streams[gy * nx + gx] : pg_streams[gy * nx + gx]).push_back(std::move(part));
      }
  }
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
  // ---- sections ----
  std::vector<BitWriter> sections(1 + num_lf + 1 + num_groups);
  EntropyEncoder enc;
  {
    BitWriter& w = sections[0];
    w.write(1, 1);  // LfChannelDequantization all_default
    w.write(1, 1);  // global MA tree present
    write_tree(w, tree);
    std::vector<uint8_t> map(size_t(tree.num_leaves()));
    for (size_t i = 0; i < map.size(); ++i) map[i] = uint8_t(i);
    enc.write_header(w, all, uint32_t(map.size()), map);
    // GlobalModular header (lib.rs:117-125): global tree, default WP, two transforms
    w.write(1, 1);
    w.write(1, 1);
    write_u32(w, 2, 4, 0);  // nb_transforms = 2
    w.write(2, 0);          // RCT
    write_u32(w, 0, 3, 0);  //   begin_c = 0
    write_u32(w, 0, 0, 0);  //   rct_type = 6
    w.write(2, 2);          // Squeeze
    write_u32(w, 0, 0, 0);  //   num_sq = 0: default parameters
    enc.write_tokens(w, global_tokens);
    w.pad();
  }
  for (uint32_t g = 0; g < num_lf; ++g) {
    if (lf_streams[g].empty()) continue;
    BitWriter& w = sections[1 + g];
    write_modular_header(w);
    enc.write_tokens(w, lf_tokens[g]);
    w.pad();
  }
  for (uint32_t g = 0; g < num_groups; ++g) {
    if (pg_streams[g].empty()) continue;
    BitWriter& w = sections[2 + num_lf + g];
    write_modular_header(w);
    enc.write_tokens(w, pg_tokens[g]);
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
  cs.write(1, 1);  // modular_16bit_buffers
  cs.write(2, 0);  // no extra channels
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
  cs.write(1, 0);      // do_ycbcr
  cs.write(2, 0);      // upsampling = 1
  cs.write(2, 1);      // group_size_shift = 1 (256)
  cs.write(2, 0);      // num_passes = 1
  cs.write(1, 0);      // have_crop
  cs.write(2, 0);      // blend mode Replace
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
    else if (s == "-o") a.out = next();
    else fprintf(stderr, "unknown arg %s\n", s.c_str()), exit(2);
  }
  if (a.modular) return encode_modular(a);
  if (a.only_type >= int(kNumTransformTypes) || (a.only_type >= 0 && a.all_types))
    fprintf(stderr, "--only-type takes a transform type 0..26 (not with --all-types)\n"), exit(2);
  std::mt19937 rng(a.seed);
  auto uni = [&](double lo, double hi) { return lo + (hi - lo) * (double(rng()) / 4294967296.0); };
  const uint32_t W = a.width, H = a.height;
  const uint32_t bw = (W + 7) / 8, bh = (H + 7) / 8;
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
    for (int k = 0; k < 3; ++k) {
      ch[k].w = lw, ch[k].h = lh;
      ch[k].v.resize(size_t(lw) * lh);
      for (uint32_t y = 0; y < lh; ++y)
        for (uint32_t x = 0; x < lw; ++x) ch[k].v[size_t(y) * lw + x] = lfq[order[k]][size_t(ly0 + y) * bw + lx0 + x];
    }
    modular_tokens(tree, ch, int32_t(1 + lg), &lfcoeff_tokens[lg]);
    // HfMetadata: x_from_y, b_from_y (lw/8 x lh/8), block info (nb x 2), sharpness (lw x lh)
    std::vector<Plane2D> hm(4);
    uint32_t w64 = (lw + 7) / 8, h64 = (lh + 7) / 8;
    for (int k = 0; k < 2; ++k) {
      hm[k].w = w64, hm[k].h = h64;
      hm[k].v.resize(size_t(w64) * h64);
      for (auto& v : hm[k].v) v = int32_t(rng() % 33) - 16;
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

  // ---- HF tokens per group ----
  const uint32_t nbc = 15;
  const double kScale = 1.0 / std::max(0.25, a.distance);  // coefficient magnitude scale
  std::vector<std::vector<uint32_t>> orders(13);
  for (uint32_t id = 0; id < 13; ++id) orders[id] = natural_order(id);
  // hf_tokens[pass * num_groups + group]; a coefficient c is sent as sum over passes of (part_p << shift_p), with
  // part_p = remainder / 2^shift_p truncated toward zero
  std::vector<std::vector<Token>> hf_tokens(size_t(P) * num_groups);
  std::exponential_distribution<double> expo(1.0);
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
          if (y == 0) predicted = x == 0 ? 32 : nz_row[c][x - 1];
          else if (x == 0) predicted = nz_row[c][x];
          else predicted = (nz_row[c][x] + nz_row[c][x - 1] + 1) >> 1;
          uint32_t pidx = predicted >= 8 ? 4 + predicted / 2 : predicted;
          toks.push_back({block_ctx + pidx * nbc, non_zeros});
          uint32_t nz_val = (non_zeros + num_blocks - 1) >> nb_log;
          for (uint32_t dx = 0; dx < ti.w8; ++dx) nz_row[c][x + dx] = nz_val;
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

  // ---- sections ----
  const uint32_t global_scale = uint32_t(std::lround(5111.0 / std::max(0.1, a.distance))), quant_lf = 17;
  std::vector<BitWriter> sections(1 + num_lf + 1 + size_t(P) * num_groups);
  EntropyEncoder lf_enc;
  std::vector<EntropyEncoder> hf_enc(P);
  {  // LfGlobal
    BitWriter& w = sections[0];
    w.write(1, 1);  // LfChannelDequantization all_default
    // Quantizer: global_scale U32(1+u11, 2049+u11, 4097+u12, 8193+u16), quant_lf U32(16, 1+u5, 1+u8, 1+u16)
    if (global_scale <= 2048) write_u32(w, 0, 11, global_scale - 1);
    else if (global_scale <= 4096) write_u32(w, 1, 11, global_scale - 2049);
    else if (global_scale <= 8192) write_u32(w, 2, 12, global_scale - 4097);
    else write_u32(w, 3, 16, global_scale - 8193);
    write_u32(w, 1, 5, quant_lf - 1);
    w.write(1, 1);  // HfBlockContext default
    w.write(1, 1);  // LfChannelCorrelation all_default
    w.write(1, 1);  // global MA tree present
    write_tree(w, tree);
    std::vector<uint8_t> map(size_t(tree.num_leaves()));
    for (size_t i = 0; i < map.size(); ++i) map[i] = uint8_t(i);
    lf_enc.write_header(w, lf_tokens_all, uint32_t(map.size()), map);
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
      hf_enc[pass].write_header(w, hf_all[pass], 495 * nbc * NP, hf_map);
    }
    end_section(w);
  }
  for (uint32_t pass = 0; pass < P; ++pass)
    for (uint32_t g = 0; g < num_groups; ++g) {
      BitWriter& w = sections[2 + num_lf + size_t(pass) * num_groups + g];
      w.write(int(ceil_log2_nonzero(NP)), g % NP);  // hfp: 0 bits with a single preset
      hf_enc[pass].write_tokens(w, hf_tokens[size_t(pass) * num_groups + g]);
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
  write_dim(H);
  cs.write(3, 0);  // ratio
  write_dim(W);
  if (a.colour.empty()) {
    cs.write(1, 1);  // ImageMetadata all_default
  } else {  // ImageMetadata with an enum ColourEncoding (jxl-image/src/lib.rs:229-287, color.rs:21-58)
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
    cs.write(1, 1);  // modular_16bit_buffers
    cs.write(2, 0);  // no extra channels
    cs.write(1, 1);  // xyb_encoded
    cs.write(1, 0);  // ColourEncoding all_default
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
    cs.write(2, 0);  // extensions
  }
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
  } else if (P > 1 || a.epf_iters != 2 || !a.gaborish) {
    cs.write(1, 0);         // all_default
    cs.write(2, 0);         // Regular
    cs.write(1, 0);         // VarDCT
    write_u64_small(0);     // flags
    cs.write(2, 0);         // upsampling = 1
    cs.write(3, 3);         // x_qm_scale
    cs.write(3, 2);         // b_qm_scale
    cs.write(2, P - 1);     // num_passes (1, 2 or 3)
    if (P > 1) {
      cs.write(2, 0);       // num_ds = 0
      for (uint32_t pass = 0; pass + 1 < P; ++pass) cs.write(2, P - 1 - pass);  // shift
    }
    cs.write(1, 0);         // have_crop
    cs.write(2, 0);         // blend mode Replace
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
