// Modular stream decode: one warp per entropy-coded Modular stream (LfCoeff, ModularLfGroup,
// HfMetadata, GlobalModular, pass-group modular data).
//
// A stream is strictly serial (one ANS state; each sample's context depends on already decoded
// neighbours), so the kernel is built around the shortest dependent-instruction chain per sample:
//   * all 32 lanes stage the stream's tables into shared memory (host-compacted per-channel MA
//     subtrees or their flattened LUT, ANS alias buckets / prefix LUTs, hybrid-uint configs, the
//     weighted predictor's error rows and reciprocal table); lane 0 then walks the chain with every
//     dependent load hitting shared memory;
//   * neighbour samples are carried in registers, previous-row samples are prefetched three
//     iterations ahead, the predictor's previous-row error terms one iteration ahead;
//   * the weighted predictor runs in 32-bit arithmetic while a sticky range flag proves that the
//     reference's i64 arithmetic cannot differ (|sample| < 2^18, |true_err| < 2^21); the first
//     sample outside the range switches the rest of the channel to the i64 path;
//   * when a channel's subtree tests a single property, that property is evaluated branch-free as a
//     linear form of the neighbours and indexes a leaf LUT.
// Integer semantics are those of crates/jxl-modular/src/{image.rs:456-593,1169-1260, predictor.rs,
// ma.rs} (bit-exact, wrapping i32).
#include "kernels.h"
#include "stream_common.cuh"

#include <type_traits>

namespace jxlb {

namespace {

constexpr uint32_t kSmemTreeBytes = 64 * 1024;
constexpr uint32_t kSmemAnsBytes = 48 * 1024;
constexpr uint32_t kSmemPrefixBytes = 24 * 1024;
constexpr uint32_t kSmemLutBytes = 8 * 1024;
constexpr uint32_t kSmemWpMaxWidth = 1024;

struct SmemLayout {
  uint32_t tree, ans, prefix, prefix_meta, configs, luts, wp, div, total;
};

__host__ __device__ inline SmemLayout modular_layout(uint32_t num_nodes, const DevEntropyCode& code, uint32_t lut_total,
                                                      uint32_t use_wp, uint32_t max_w) {
  SmemLayout L;
  uint32_t off = 0;
  auto take = [&](uint32_t bytes) {
    uint32_t o = off;
    off += (bytes + 15) & ~15u;
    return o;
  };
  L.div = take(65 * 4);
  uint32_t tree_bytes = num_nodes * 16;
  L.tree = tree_bytes <= kSmemTreeBytes ? take(tree_bytes) : 0xffffffffu;
  L.configs = take(code.num_clusters * 4);
  if (code.use_prefix) {
    L.ans = 0xffffffffu;
    uint32_t pb = code.prefix_table_size * 4;
    L.prefix = pb <= kSmemPrefixBytes ? take(pb) : 0xffffffffu;
    L.prefix_meta = take(code.num_clusters * 8);
  } else {
    uint32_t ab = (code.num_clusters << code.log_alphabet_size) * 8;
    L.ans = (ab <= kSmemAnsBytes) ? take(ab) : 0xffffffffu;
    L.prefix = 0xffffffffu;
    L.prefix_meta = 0xffffffffu;
  }
  uint32_t lb = lut_total * 2;
  L.luts = lb <= kSmemLutBytes ? take(lb + 4) : 0xffffffffu;
  L.wp = (use_wp && max_w <= kSmemWpMaxWidth) ? take(max_w * 5 * 4) : 0xffffffffu;
  L.total = off;
  return L;
}

// SelfCorrectingPredictor (predictor.rs:279-441) with row state in shared (or global) memory.
//
// Fast mode bounds (M = 2^18 samples, T = 2^21 true errors, parameters p* <= 31, w* <= 15):
//   sub-prediction numerators  <= 31 * (3T + 2 * 16M) < 2^29, sub-predictions < 2^24.1,
//   weighted sum               <  2^24.1 * 31 < 2^30 (normalised weights sum to < 32),
//   recorded sub-errors        <  2^22, their three-term sums < 2^25
// so every intermediate fits an i32/u32 and equals the reference's i64 value.
struct FastWp {
  uint32_t width, wm1, x, y;
  int32_t* true_err_row;
  uint32_t* sub_err_row;
  const uint32_t* div;  // DIV_LOOKUP (predictor.rs:150-160)
  int32_t p1, p2, p3a, p3b, p3c, p3d, p3e;
  uint32_t w0, w1, w2, w3;
  int32_t te_w, te_nw, te_n, te_ne;
  uint32_t a0, a1, a2, a3;  // subpred_err_nw_ww
  uint32_t b0, b1, b2, b3;  // subpred_err_n_w
  uint32_t c0, c1, c2, c3;  // subpred_err_ne
  uint4 q_next;             // previous-row sub-errors at x+2 (prefetched)
  int32_t te_next;          // previous-row true error at x+2 (prefetched)
  bool slow;                // sticky: a sample or error left the proven range
  int32_t f0, f1, f2, f3, fpred;
  int64_t s0, s1, s2, s3, prediction;
  int32_t max_error;

  __device__ __forceinline__ void reset(uint32_t width_, int32_t* rows, const uint32_t* hdr, const uint32_t* div_) {
    width = width_;
    wm1 = width_ - 1;
    x = y = 0;
    sub_err_row = reinterpret_cast<uint32_t*>(rows);  // 16-byte aligned: accessed as uint4
    true_err_row = rows + size_t(width_) * 4;
    div = div_;
    for (uint32_t i = 0; i < width_ * 5; ++i) rows[i] = 0;
    p1 = int32_t(hdr[0]), p2 = int32_t(hdr[1]), p3a = int32_t(hdr[2]), p3b = int32_t(hdr[3]), p3c = int32_t(hdr[4]);
    p3d = int32_t(hdr[5]), p3e = int32_t(hdr[6]);
    w0 = hdr[7], w1 = hdr[8], w2 = hdr[9], w3 = hdr[10];
    te_w = te_nw = te_n = te_ne = 0;
    a0 = a1 = a2 = a3 = b0 = b1 = b2 = b3 = c0 = c1 = c2 = c3 = 0;
    slow = false;
    f0 = f1 = f2 = f3 = fpred = 0;
    s0 = s1 = s2 = s3 = prediction = 0;
    max_error = 0;
    q_next = make_uint4(0, 0, 0, 0);
    te_next = 0;
  }
  // error rows of the previous image row at x+2 (the NE position of the NEXT sample): independent
  // of the sample being decoded, and not yet overwritten by the current row
  __device__ __forceinline__ void prefetch() {
    const uint32_t xn = min(x + 2, wm1);
    te_next = true_err_row[xn];
    q_next = *reinterpret_cast<const uint4*>(sub_err_row + size_t(xn) * 4);
  }
  __device__ __forceinline__ uint32_t weight32(uint32_t err_sum, uint32_t maxweight) const {
    const uint32_t t = (err_sum + 1) >> 5;
    const uint32_t shift = 31u - uint32_t(__clz(int(t | 1u)));
    return 4 + ((maxweight * div[(err_sum >> shift) + 1]) >> shift);
  }
  __device__ __forceinline__ uint32_t weight64(uint32_t err_sum, uint32_t maxweight) const {
    uint32_t t = uint32_t((uint64_t(err_sum) + 1) >> 5);
    uint32_t shift = t ? ilog2_u32(t) : 0;
    return 4 + ((maxweight * div[(err_sum >> shift) + 1]) >> shift);
  }
  __device__ __forceinline__ void predict(int32_t n, int32_t nw, int32_t ne, int32_t wv, int32_t nn) {
    if (!slow) {
      const int32_t n3 = n << 3, nw3 = nw << 3, ne3 = ne << 3, w3_ = wv << 3, nn3 = nn << 3;
      f0 = w3_ + ne3 - n3;
      f1 = n3 - (((te_w + te_n + te_ne) * p1) >> 5);
      f2 = w3_ - (((te_w + te_n + te_nw) * p2) >> 5);
      f3 = n3 - ((te_nw * p3a + te_n * p3b + te_ne * p3c + (nn3 - n3) * p3d + (nw3 - w3_) * p3e) >> 5);
      uint32_t g0 = weight32(a0 + b0 + c0, w0), g1 = weight32(a1 + b1 + c1, w1), g2 = weight32(a2 + b2 + c2, w2),
               g3 = weight32(a3 + b3 + c3, w3);
      uint32_t sum_weights = g0 + g1 + g2 + g3;
      const uint32_t log_weight = ilog2_u32(sum_weights >> 4);
      g0 >>= log_weight, g1 >>= log_weight, g2 >>= log_weight, g3 >>= log_weight;
      sum_weights = g0 + g1 + g2 + g3;
      const int32_t s = int32_t(sum_weights >> 1) - 1 + f0 * int32_t(g0) + f1 * int32_t(g1) + f2 * int32_t(g2) + f3 * int32_t(g3);
      int32_t pred = int32_t((int64_t(s) * int64_t(div[sum_weights])) >> 24);
      if (((te_n ^ te_w) | (te_n ^ te_nw)) <= 0) {
        const int32_t mn = min(min(n3, w3_), ne3), mx = max(max(n3, w3_), ne3);
        pred = min(max(pred, mn), mx);
      }
      int32_t me = te_w;
      if (abs(te_n) > abs(me)) me = te_n;
      if (abs(te_nw) > abs(me)) me = te_nw;
      if (abs(te_ne) > abs(me)) me = te_ne;
      fpred = pred;
      max_error = me;
      return;
    }
    int64_t tew = te_w, tenw = te_nw, ten = te_n, tene = te_ne;
    int64_t n3 = int64_t(n) << 3, nw3 = int64_t(nw) << 3, ne3 = int64_t(ne) << 3, w3_ = int64_t(wv) << 3,
            nn3 = int64_t(nn) << 3;
    s0 = w3_ + ne3 - n3;
    s1 = n3 - (((tew + ten + tene) * int64_t(p1)) >> 5);
    s2 = w3_ - (((tew + ten + tenw) * int64_t(p2)) >> 5);
    s3 = n3 - ((tenw * int64_t(p3a) + ten * int64_t(p3b) + tene * int64_t(p3c) + (nn3 - n3) * int64_t(p3d) +
                (nw3 - w3_) * int64_t(p3e)) >> 5);
    uint32_t g0 = weight64(a0 + b0 + c0, w0), g1 = weight64(a1 + b1 + c1, w1), g2 = weight64(a2 + b2 + c2, w2),
             g3 = weight64(a3 + b3 + c3, w3);
    uint32_t sum_weights = g0 + g1 + g2 + g3;
    uint32_t log_weight = ilog2_u32(sum_weights >> 4);
    g0 >>= log_weight, g1 >>= log_weight, g2 >>= log_weight, g3 >>= log_weight;
    sum_weights = g0 + g1 + g2 + g3;
    int64_t s = (int64_t(sum_weights) >> 1) - 1;
    s += s0 * int64_t(g0) + s1 * int64_t(g1) + s2 * int64_t(g2) + s3 * int64_t(g3);
    int64_t pred = (s * int64_t(div[sum_weights])) >> 24;
    if (((ten ^ tew) | (ten ^ tenw)) <= 0) {
      int64_t mn = min(min(n3, w3_), ne3), mx = max(max(n3, w3_), ne3);
      pred = min(max(pred, mn), mx);
    }
    int64_t me = tew;
    if (abs64(ten) > abs64(me)) me = ten;
    if (abs64(tenw) > abs64(me)) me = tenw;
    if (abs64(tene) > abs64(me)) me = tene;
    prediction = pred;
    max_error = int32_t(me);
  }
  // Predictor::SelfCorrecting value (predictor.rs:100-106)
  __device__ __forceinline__ int32_t predicted_sample() const {
    return slow ? int32_t((prediction + 3) >> 3) : ((fpred + 3) >> 3);
  }
  __device__ __forceinline__ void record(int32_t sample_) {
    uint32_t e0, e1, e2, e3;
    int32_t te;
    if (!slow && (uint32_t(sample_ + 0x40000) >> 19) != 0) {  // sample outside [-2^18, 2^18): finish in i64
      slow = true;
      s0 = f0, s1 = f1, s2 = f2, s3 = f3, prediction = fpred;
    }
    if (!slow) {
      const int32_t s8 = sample_ << 3;
      te = fpred - s8;
      e0 = uint32_t(abs(f0 - s8) + 3) >> 3, e1 = uint32_t(abs(f1 - s8) + 3) >> 3;
      e2 = uint32_t(abs(f2 - s8) + 3) >> 3, e3 = uint32_t(abs(f3 - s8) + 3) >> 3;
      if ((uint32_t(te + 0x200000) >> 22) != 0) slow = true;  // |true_err| >= 2^21: next predict() in i64
    } else {
      const int64_t s8 = int64_t(sample_) << 3;
      te = int32_t(prediction - s8);
      e0 = uint32_t((uint64_t(abs64(s0 - s8)) + 3) >> 3), e1 = uint32_t((uint64_t(abs64(s1 - s8)) + 3) >> 3);
      e2 = uint32_t((uint64_t(abs64(s2 - s8)) + 3) >> 3), e3 = uint32_t((uint64_t(abs64(s3 - s8)) + 3) >> 3);
    }
    true_err_row[x] = te;
    *reinterpret_cast<uint4*>(sub_err_row + size_t(x) * 4) = make_uint4(e0, e1, e2, e3);
    ++x;
    if (x >= width) {
      ++y;
      x = 0;
      te_w = 0;
      te_n = true_err_row[0];
      te_nw = te_n;
      uint4 r = *reinterpret_cast<const uint4*>(sub_err_row);
      b0 = a0 = r.x, b1 = a1 = r.y, b2 = a2 = r.z, b3 = a3 = r.w;
      if (width <= 1) {
        te_ne = te_n;
        c0 = b0, c1 = b1, c2 = b2, c3 = b3;
      } else {
        te_ne = true_err_row[1];
        uint4 q = *reinterpret_cast<const uint4*>(sub_err_row + 4);
        c0 = q.x, c1 = q.y, c2 = q.z, c3 = q.w;
      }
    } else {
      te_w = te;
      te_nw = te_n;
      te_n = te_ne;
      a0 = b0, a1 = b1, a2 = b2, a3 = b3;
      b0 = c0 + e0, b1 = c1 + e1, b2 = c2 + e2, b3 = c3 + e3;
      if (x + 1 >= width) {
        te_ne = te_n;
        c0 = b0, c1 = b1, c2 = b2, c3 = b3;
      } else {
        // rows are zero until written, so during the first image row this reads zeros (the
        // reference leaves the NE terms untouched there, predictor.rs:426-437)
        te_ne = te_next;
        c0 = q_next.x, c1 = q_next.y, c2 = q_next.z, c3 = q_next.w;
      }
    }
  }
};

constexpr int kMaxPrev = 16;

struct StreamState {
  WordBitReader br;
  uint32_t ans_state;
  uint32_t* window;  // LZ77 state (lib.rs:346-352)
  uint32_t lz_to_copy, lz_copy_pos, lz_decoded;
  int err;
};

// read_varint_with_multiplier_clustered (lib.rs:476-569). FAST: the stream is ANS-coded without LZ77
// (what libjxl emits for LF / HfMetadata), decided once per stream instead of per sample.
template <bool FAST>
__device__ __forceinline__ uint32_t read_token_value(const CodeView& cv, const DevEntropyCode& code, StreamState& s,
                                                     uint32_t cluster, bool lz77, uint32_t dist_multiplier) {
  if (FAST) {
    const uint32_t token = cv_read_symbol_ans(cv, s.ans_state, s.br, cluster);
    return cv_read_uint(s.br, cv.configs[cluster], token);
  }
  if (!lz77) {
    const uint32_t token = cv_read_symbol(cv, s.ans_state, s.br, cluster);
    return cv_read_uint(s.br, cv.configs[cluster], token);
  }
  uint32_t token_value;
  if (s.lz_to_copy > 0) {
    token_value = s.window[s.lz_copy_pos & 0xfffff];
    ++s.lz_copy_pos;
    --s.lz_to_copy;
  } else {
    const uint32_t token = cv_read_symbol(cv, s.ans_state, s.br, cluster);
    if (token >= code.lz77_min_symbol) {
      if (s.lz_decoded == 0) {
        s.err = kDevBadStream;
        return 0;
      }
      const uint32_t nc = cv_read_uint(s.br, code.lz_len_conf, token - code.lz77_min_symbol);
      s.lz_to_copy = nc + code.lz77_min_length;
      const uint32_t dtoken = cv_read_symbol(cv, s.ans_state, s.br, code.lz_dist_cluster);
      uint32_t distance = cv_read_uint(s.br, cv.configs[code.lz_dist_cluster], dtoken);
      if (dist_multiplier == 0) {
      } else if (distance < 120) {
        const int32_t dd = int32_t(kDevSpecialDistances[distance][0]) +
                           int32_t(dist_multiplier) * int32_t(kDevSpecialDistances[distance][1]);
        distance = uint32_t(max(dd - 1, 0));
      } else {
        distance -= 120;
      }
      distance = min(min((1u << 20) - 1, distance) + 1, s.lz_decoded);
      s.lz_copy_pos = s.lz_decoded - distance;
      token_value = s.window[s.lz_copy_pos & 0xfffff];
      ++s.lz_copy_pos;
      --s.lz_to_copy;
    } else {
      token_value = cv_read_uint(s.br, cv.configs[cluster], token);
    }
  }
  s.window[s.lz_decoded & 0xfffff] = token_value;
  ++s.lz_decoded;
  return token_value;
}

// Predictors other than Gradient / SelfCorrecting / Zero (predictor.rs:74-126)
__device__ __noinline__ int32_t rare_predictor(uint32_t predictor, int32_t wv, int32_t n, int32_t nw, int32_t ne,
                                               int32_t nn, int32_t wwv, int32_t nee) {
  switch (predictor) {
    case 1: return wv;
    case 2: return n;
    case 3: return int32_t((int64_t(wv) + int64_t(n)) / 2);
    case 4: return abs_diff(n, nw) < abs_diff(wv, nw) ? wv : n;
    case 7: return ne;
    case 8: return nw;
    case 9: return wwv;
    case 10: return int32_t((int64_t(wv) + int64_t(nw)) / 2);
    case 11: return int32_t((int64_t(n) + int64_t(nw)) / 2);
    case 12: return int32_t((int64_t(n) + int64_t(ne)) / 2);
    default:
      return int32_t((6 * int64_t(n) - 2 * int64_t(nn) + 7 * int64_t(wv) + int64_t(wwv) + int64_t(nee) + 3 * int64_t(ne) + 8) / 16);
  }
}

// Property of a previous channel (predictor.rs:495-528)
__device__ __noinline__ int32_t prev_channel_property(const DevChannel* prev, int nprev, uint32_t e, uint32_t x, uint32_t y) {
  const uint32_t pidx = e >> 2, k = e & 3;
  if (int(pidx) >= nprev) return 0;
  const DevChannel& pc = prev[pidx];
  const int32_t* pr = pc.ptr + size_t(y) * pc.stride;
  const int32_t c = pr[x];
  if (k == 0) return c < 0 ? int32_t(0u - uint32_t(c)) : c;
  if (k == 1) return c;
  int32_t g;
  if (x == 0 && y == 0) g = 0;
  else if (x == 0) g = pr[-ptrdiff_t(pc.stride)];
  else if (y == 0) g = pr[x - 1];
  else g = grad_clamped(pr[ptrdiff_t(x) - ptrdiff_t(pc.stride)], pr[x - 1], pr[ptrdiff_t(x) - 1 - ptrdiff_t(pc.stride)]);
  return (k == 2) ? int32_t(abs_diff(c, g)) : wsub(c, g);
}

// One channel of a stream. WP: the stream's tree uses the weighted predictor (property 15 or
// predictor 6); LUT: 0 = tree walk, 1 = the channel's subtree tests one property (leaf LUT over a
// linear form), 2 = that property is the weighted predictor's max_error (libjxl's fixed LF tree).
template <bool WP, int LUT, bool FAST>
__device__ __forceinline__ void decode_channel(const DevModularJob& job, const DevEntropyCode& code, const CodeView& cv,
                                               const MaNode* tree, const uint16_t* lut, const DevChannelPlan plan,
                                               const DevChannel out, const DevChannel* prev, int nprev, uint32_t ci,
                                               int32_t* wp_rows, const uint32_t* s_div, FastWp& wp, StreamState& s,
                                               const bool lz77) {
  const uint32_t width = out.w, wm1 = width - 1;
  const uint32_t dist_multiplier = job.dist_multiplier;
  // the LUT property as a linear form of the (edge-adjusted) neighbours: v = c . (w n nw ne nn ww
  // prev_grad x y max_error), optionally |v|  (property list: predictor.rs:453-490)
  int32_t cw = 0, cn = 0, cnw = 0, cne = 0, cnn = 0, cww = 0, cpg = 0, cx = 0, cy = 0, cme = 0;
  bool use_abs = false;
  if (LUT == 1) {
    switch (plan.lut_prop) {
      case 2: cy = 1; break;
      case 3: cx = 1; break;
      case 4: cn = 1, use_abs = true; break;
      case 5: cw = 1, use_abs = true; break;
      case 6: cn = 1; break;
      case 7: cw = 1; break;
      case 8: cw = 1, cpg = -1; break;
      case 9: cw = 1, cn = 1, cnw = -1; break;
      case 10: cw = 1, cnw = -1; break;
      case 11: cnw = 1, cn = -1; break;
      case 12: cn = 1, cne = -1; break;
      case 13: cn = 1, cnn = -1; break;
      case 14: cw = 1, cww = -1; break;
      default: cme = WP ? 1 : 0; break;
    }
  }
  const int32_t lut_base = plan.lut_base;
  const uint32_t lut_last = plan.lut_len - 1;
  if (WP) wp.reset(width, wp_rows, job.wp, s_div);

  for (uint32_t y = 0; y < out.h && s.err == kDevOk; ++y) {
    int32_t* row = out.ptr + size_t(y) * out.stride;
    const int32_t* rn = y ? row - out.stride : row;
    const bool has_nn = y >= 2;
    const int32_t* rnn = has_nn ? row - 2 * size_t(out.stride) : rn;
    // West of the first sample is N (0 on the first row); NW likewise (predictor.rs:554-564)
    int32_t r_0 = y ? rn[0] : 0;
    int32_t r_1 = y ? rn[min(1u, wm1)] : 0, r_2 = y ? rn[min(2u, wm1)] : 0;
    int32_t r_m1 = r_0, w = r_0, ww = r_0;
    int32_t nn_cur = has_nn ? rnn[0] : 0;
    int32_t prev_grad = 0;
    const int32_t cyy = cy * int32_t(y);

    auto sample = [&](auto top_tag, const uint32_t x) {
      constexpr bool TOP = decltype(top_tag)::value;
      const int32_t wv = w;
      int32_t n, nw, ne, nee, nn, r_3 = 0, nn_next = 0;
      if (TOP) {
        n = nw = ne = nee = nn = wv;
      } else {
        n = r_0;
        nw = r_m1;
        ne = x + 1 < width ? r_1 : n;
        nee = x + 2 < width ? r_2 : ne;
        nn = has_nn ? nn_cur : n;
        // previous rows three / one samples ahead (independent of the value being decoded)
        r_3 = rn[min(x + 3, wm1)];
        nn_next = rnn[min(x + 1, wm1)];
      }
      const int32_t wwv = x >= 2 ? ww : wv;
      if (WP) {
        wp.prefetch();
        wp.predict(n, nw, ne, wv, nn);
      }
      const int32_t w_nw = wsub(wv, nw);
      const int32_t grad = wadd(w_nw, n);
      // ---- leaf selection ----
      uint32_t node_idx;
      if (LUT == 2) {
        const int32_t v = wp.max_error;
        const uint32_t li = v < lut_base ? 0u : min(uint32_t(v) - uint32_t(lut_base), lut_last);
        node_idx = lut[li];
      } else if (LUT == 1) {
        const int32_t pre = cn * n + cnw * nw + cne * ne + cnn * nn + cx * int32_t(x) + cyy;
        int32_t v = pre + cw * wv + cww * wwv + cpg * prev_grad + (WP ? cme * wp.max_error : 0);
        if (use_abs) v = v < 0 ? int32_t(0u - uint32_t(v)) : v;
        const uint32_t li = v < lut_base ? 0u : min(uint32_t(v) - uint32_t(lut_base), lut_last);
        node_idx = lut[li];
      } else {
        node_idx = plan.root;
        for (;;) {
          const MaNode nd = tree[node_idx];
          if (nd.property < 0) break;
          int32_t v;
          switch (nd.property) {
            case 0: v = int32_t(ci); break;
            case 1: v = int32_t(job.stream_index); break;
            case 2: v = int32_t(y); break;
            case 3: v = int32_t(x); break;
            case 4: v = int32_t(n < 0 ? 0u - uint32_t(n) : uint32_t(n)); break;
            case 5: v = int32_t(wv < 0 ? 0u - uint32_t(wv) : uint32_t(wv)); break;
            case 6: v = n; break;
            case 7: v = wv; break;
            case 8: v = wsub(wv, prev_grad); break;
            case 9: v = grad; break;
            case 10: v = w_nw; break;
            case 11: v = wsub(nw, n); break;
            case 12: v = wsub(n, ne); break;
            case 13: v = wsub(n, nn); break;
            case 14: v = wsub(wv, wwv); break;
            case 15: v = WP ? wp.max_error : 0; break;
            default: v = prev_channel_property(prev, nprev, uint32_t(nd.property - 16), x, y); break;
          }
          node_idx = v > nd.value ? nd.a : nd.b;
        }
      }
      const MaNode leaf = tree[node_idx];
      const uint32_t predictor = leaf.a & 0xff, cluster = leaf.a >> 8;
      // ---- entropy decode (lib.rs:476-605) ----
      const uint32_t token_value = read_token_value<FAST>(cv, code, s, cluster, lz77, dist_multiplier);
      const int32_t diff = wadd(wmul(dev_unpack_signed(token_value), int32_t(leaf.b)), leaf.value);
      int32_t pred;
      if (WP && predictor == 6) {
        pred = wp.predicted_sample();
      } else if (predictor == 5) {
        // clamped gradient: outside (lo, hi) the clamp decides, inside it n + w - nw cannot wrap
        const int32_t hi = max(n, wv), lo = min(n, wv);
        pred = nw >= hi ? lo : (nw <= lo ? hi : wsub(wadd(lo, hi), nw));
      } else if (predictor == 0) {
        pred = 0;
      } else if (predictor == 6) {
        pred = 0;  // a tree without the weighted predictor cannot name it (tree_uses_wp); unreachable
      } else {
        pred = rare_predictor(predictor, wv, n, nw, ne, nn, wwv, nee);
      }
      const int32_t value = wadd(diff, pred);
      row[x] = value;
      if (WP) wp.record(value);
      prev_grad = grad;
      ww = wv;
      w = value;
      if (!TOP) {
        r_m1 = r_0;
        r_0 = r_1;
        r_1 = r_2;
        r_2 = r_3;
        nn_cur = nn_next;
      }
    };

    if (y == 0) {
      w = 0, ww = 0;
      for (uint32_t x = 0; x < width && s.err == kDevOk; ++x) sample(std::true_type{}, x);
    } else {
      for (uint32_t x = 0; x < width && s.err == kDevOk; ++x) sample(std::false_type{}, x);
    }
    if (s.br.pos() > job.bit_limit) s.err = kDevOverrun;
  }
}

// ALLSM: every table of every job of the launch fits its shared-memory budget (what libjxl's LF / HfMetadata streams
// need: a few KB). All table pointers then derive from the shared array unconditionally, so the compiler emits LDS with
// 32-bit addresses instead of generic loads for the tree nodes, alias buckets, leaf LUT and predictor rows.
template <bool ALLSM>
__device__ __forceinline__ void modular_stream_body(uint8_t* smem, const uint8_t* __restrict__ cs,
                                                    const DevModularJob* __restrict__ jobs,
                                                    const DevChannel* __restrict__ channels,
                                                    const DevChannelPlan* __restrict__ plans,
                                                    uint64_t* __restrict__ end_bits, int* __restrict__ status,
                                                    const int job_idx, unsigned long long* __restrict__ trace) {
  const uint32_t lane = threadIdx.x;
  const DevModularJob& job = jobs[job_idx];
  const DevEntropyCode& code = job.code;
  const DevChannel* chans = channels + job.first_channel;
  const DevChannelPlan* chplans = plans + job.first_channel;
  uint32_t max_w = 0;
  for (uint32_t ci = 0; ci < job.num_channels; ++ci) max_w = max(max_w, chans[ci].w);
  const SmemLayout L = modular_layout(job.num_tree_nodes, code, job.lut_total, job.use_wp, max_w);

  // ---- stage tables ----
  uint32_t* s_div = reinterpret_cast<uint32_t*>(smem + L.div);
  for (uint32_t i = lane; i < 65; i += 32) s_div[i] = i ? (1u << 24) / i : 0;
  const MaNode* tree = job.tree;
  if (ALLSM || L.tree != 0xffffffffu) {
    warp_copy_words(reinterpret_cast<uint32_t*>(smem + L.tree), reinterpret_cast<const uint32_t*>(job.tree),
                    job.num_tree_nodes * 4, lane);
    tree = reinterpret_cast<const MaNode*>(smem + L.tree);
  }
  CodeView cv;
  cv.log_alphabet_size = code.log_alphabet_size;
  cv.use_prefix = code.use_prefix;
  warp_copy_words(reinterpret_cast<uint32_t*>(smem + L.configs), code.configs, code.num_clusters, lane);
  cv.configs = reinterpret_cast<const uint32_t*>(smem + L.configs);
  cv.ans = code.ans;
  cv.prefix = code.prefix;
  cv.prefix_meta = code.prefix_meta;
  if (code.use_prefix) {
    warp_copy_words(reinterpret_cast<uint32_t*>(smem + L.prefix_meta), code.prefix_meta, code.num_clusters * 2, lane);
    cv.prefix_meta = reinterpret_cast<const uint32_t*>(smem + L.prefix_meta);
    if (ALLSM || L.prefix != 0xffffffffu) {
      warp_copy_words(reinterpret_cast<uint32_t*>(smem + L.prefix), code.prefix, code.prefix_table_size, lane);
      cv.prefix = reinterpret_cast<const uint32_t*>(smem + L.prefix);
    }
  } else if (ALLSM || L.ans != 0xffffffffu) {
    warp_copy_words(reinterpret_cast<uint32_t*>(smem + L.ans), reinterpret_cast<const uint32_t*>(code.ans),
                    (code.num_clusters << code.log_alphabet_size) * 2, lane);
    cv.ans = reinterpret_cast<const uint64_t*>(smem + L.ans);
  }
  if (ALLSM) {  // unconditionally shared pointers (the unused ones are never dereferenced)
    cv.ans = reinterpret_cast<const uint64_t*>(smem + (L.ans & 0xffffffu));
    cv.prefix = reinterpret_cast<const uint32_t*>(smem + (L.prefix & 0xffffffu));
    cv.prefix_meta = reinterpret_cast<const uint32_t*>(smem + (L.prefix_meta & 0xffffffu));
  }
  const uint16_t* luts = job.luts;
  if (ALLSM || L.luts != 0xffffffffu) {
    warp_copy_words(reinterpret_cast<uint32_t*>(smem + L.luts), reinterpret_cast<const uint32_t*>(job.luts),
                    (job.lut_total + 1) / 2, lane);
    luts = reinterpret_cast<const uint16_t*>(smem + L.luts);
  }
  int32_t* wp_rows = (ALLSM || L.wp != 0xffffffffu) ? reinterpret_cast<int32_t*>(smem + L.wp) : job.wp_scratch;
  __syncwarp();
  if (lane != 0) return;
  if (trace) {  // tracing aid: device clock (ns) when this stream starts / ends decoding
    unsigned long long now;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
    trace[2 * job_idx] = now;
  }

  // ---- serial decode (lane 0) ----
  StreamState s;
  s.br.init(cs, job.bit_pos, job.bit_limit);
  s.ans_state = code.use_prefix ? 0x130000u : s.br.read(32);
  s.window = job.lz_window;
  s.lz_to_copy = s.lz_copy_pos = s.lz_decoded = 0;
  s.err = kDevOk;
  const bool lz77 = code.lz77_enabled != 0;
  const bool use_wp = job.use_wp != 0;
  FastWp wp;

  for (uint32_t ci = 0; ci < job.num_channels && s.err == kDevOk; ++ci) {
    const DevChannel out = chans[ci];
    if (!out.w || !out.h) continue;
    const DevChannelPlan plan = chplans[ci];
    DevChannel prev[kMaxPrev];
    int nprev = 0;
    for (int pj = int(ci) - 1; pj >= 0 && nprev < kMaxPrev; --pj) {
      const DevChannel p = chans[pj];
      if (p.w == out.w && p.h == out.h && p.hshift == out.hshift && p.vshift == out.vshift && p.w && p.h) prev[nprev++] = p;
    }
    const uint16_t* lut = luts + plan.lut_offset;
    const int lut_kind = plan.lut_prop < 0 ? 0 : ((use_wp && plan.lut_prop == 15) ? 2 : 1);
    const bool fast = !lz77 && !code.use_prefix;
#define JXLB_DECODE_CHANNEL(WP_, LUT_, FAST_) \
  decode_channel<WP_, LUT_, FAST_>(job, code, cv, tree, lut, plan, out, prev, nprev, ci, wp_rows, s_div, wp, s, lz77)
    if (use_wp) {
      if (lut_kind == 2) {
        if (fast) JXLB_DECODE_CHANNEL(true, 2, true);
        else JXLB_DECODE_CHANNEL(true, 2, false);
      } else if (lut_kind == 1) {
        if (fast) JXLB_DECODE_CHANNEL(true, 1, true);
        else JXLB_DECODE_CHANNEL(true, 1, false);
      } else {
        if (fast) JXLB_DECODE_CHANNEL(true, 0, true);
        else JXLB_DECODE_CHANNEL(true, 0, false);
      }
    } else {
      if (lut_kind == 1) {
        if (fast) JXLB_DECODE_CHANNEL(false, 1, true);
        else JXLB_DECODE_CHANNEL(false, 1, false);
      } else {
        if (fast) JXLB_DECODE_CHANNEL(false, 0, true);
        else JXLB_DECODE_CHANNEL(false, 0, false);
      }
    }
#undef JXLB_DECODE_CHANNEL
  }
  if (s.err == kDevOk && !code.use_prefix && s.ans_state != 0x130000u) s.err = kDevBadStream;
  if (s.err == kDevOk && s.br.pos() > job.bit_limit) s.err = kDevOverrun;
  end_bits[job_idx] = s.br.pos();
  status[job_idx] = s.err;
  if (trace) {
    unsigned long long now;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
    trace[2 * job_idx + 1] = now;
  }
}

template <bool ALLSM>
__global__ void __launch_bounds__(32) modular_stream_kernel(const uint8_t* __restrict__ cs,
                                                            const DevModularJob* __restrict__ jobs,
                                                            const DevChannel* __restrict__ channels,
                                                            const DevChannelPlan* __restrict__ plans,
                                                            uint64_t* __restrict__ end_bits, int* __restrict__ status,
                                                            int num_jobs, unsigned long long* __restrict__ trace) {
  extern __shared__ __align__(16) uint8_t smem[];
  if (int(blockIdx.x) >= num_jobs) return;
  modular_stream_body<ALLSM>(smem, cs, jobs, channels, plans, end_bits, status, int(blockIdx.x), trace);
}

// The same streams for several frames in ONE launch (csrc/pipeline.cu, LF batch service): CTA i decodes job
// `refs[i].job` of the frame whose tables `refs[i]` points to. A frame's LF stage is two long kernels (tens of milliseconds) of
// a dozen one-lane warps; launched per frame they pin one CUDA stream (= one of the device's 32 hardware queues) for
// the whole time, which caps the frames in flight. Batched, a handful of streams carry every frame's LF stage.
template <bool ALLSM>
__global__ void __launch_bounds__(32) modular_stream_batch_kernel(const DevModularBatchRef* __restrict__ refs, int total) {
  extern __shared__ __align__(16) uint8_t smem[];
  if (int(blockIdx.x) >= total) return;
  const DevModularBatchRef r = refs[blockIdx.x];
  modular_stream_body<ALLSM>(smem, r.cs, r.jobs, r.channels, r.plans, r.end_bits, r.status, int(r.job), nullptr);
  if (r.counter) {
    // this frame's streams are done when its last one is: samples and result words first, then the count, then the word
    // the frame's host thread is woken by (the rest of the launch belongs to other frames and may run for much longer)
    __threadfence_system();
    __syncwarp();
    if ((threadIdx.x & 31) == 0 && atomicAdd(r.counter, 1u) == r.num_jobs - 1) {
      __threadfence_system();
      *reinterpret_cast<volatile uint32_t*>(r.done_flag) = r.done_seq;
    }
  }
}

// Delta-palette prediction pass (palette.rs:120-152): one CTA per channel, thread 0 walks the channel in raster order
// (every prediction reads the already corrected W / N / NW / NE ... neighbours, a serial recurrence).
__global__ void __launch_bounds__(32) palette_delta_kernel(DevPaletteDeltaParams p) {
  __shared__ uint32_t s_div[65];
  for (uint32_t i = threadIdx.x; i < 65; i += 32) s_div[i] = i ? (1u << 24) / i : 0;
  __syncthreads();
  if (threadIdx.x != 0) return;
  const DevView v = p.target[blockIdx.x];
  const uint32_t width = v.w, height = v.h;
  int32_t* base = static_cast<int32_t*>(v.ptr);
  const bool use_wp = p.d_pred == 6;
  FastWp wp;
  if (use_wp) wp.reset(width, p.wp_rows + size_t(blockIdx.x) * ((5 * size_t(width) + 3) & ~size_t(3)), p.wp, s_div);  // 16-byte aligned slices
  for (uint32_t y = 0; y < height; ++y) {
    int32_t* row = base + size_t(y) * v.stride;
    const int32_t* rn = y ? row - v.stride : nullptr;
    const int32_t* rnn = y >= 2 ? row - 2 * size_t(v.stride) : nullptr;
    const uint8_t* mrow = p.mask + size_t(y) * width;
    for (uint32_t x = 0; x < width; ++x) {
      int32_t wv, n, nw;
      if (y == 0) {
        wv = x ? row[x - 1] : 0;
        n = wv, nw = wv;
      } else if (x == 0) {
        n = rn[0];
        wv = n, nw = n;
      } else {
        wv = row[x - 1], n = rn[x], nw = rn[x - 1];
      }
      const int32_t ne = (!rn || x + 1 >= width) ? n : rn[x + 1];
      const int32_t nn = rnn ? rnn[x] : n;
      if (use_wp) {
        wp.prefetch();
        wp.predict(n, nw, ne, wv, nn);
      }
      int32_t value = row[x];
      if (mrow[x]) {
        int32_t pred;
        if (p.d_pred == 0) {
          pred = 0;
        } else if (p.d_pred == 5) {
          pred = grad_clamped(n, wv, nw);
        } else if (p.d_pred == 6) {
          pred = wp.predicted_sample();
        } else {
          const int32_t nee = (!rn || x + 2 >= width) ? ne : rn[x + 2];
          const int32_t wwv = x >= 2 ? row[x - 2] : wv;
          pred = rare_predictor(p.d_pred, wv, n, nw, ne, nn, wwv, nee);
        }
        value = wadd(value, pred);
        row[x] = value;
      }
      if (use_wp) wp.record(value);
    }
  }
}

// Completion word for CudaBackend::sync(): written to mapped host memory once everything before it on the stream is done.
__global__ void signal_word_kernel(uint32_t* word, uint32_t value) {
  *reinterpret_cast<volatile uint32_t*>(word) = value;
  __threadfence_system();
}

__global__ void read_globaltimer_kernel(unsigned long long* out) {
  unsigned long long now;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
  *out = now;
}

}  // namespace

void launch_palette_delta(DevPaletteDeltaParams p, int num_c, cudaStream_t stream) {
  if (num_c <= 0 || !p.target[0].w || !p.target[0].h) return;
  palette_delta_kernel<<<num_c, 32, 0, stream>>>(p);
}

size_t modular_job_smem_bytes(const DevModularJob& job, uint32_t max_width) {
  return modular_layout(job.num_tree_nodes, job.code, job.lut_total, job.use_wp, max_width).total;
}

void launch_modular_decode(const uint8_t* cs, const DevModularJob* jobs, const DevChannel* channels,
                           const DevChannelPlan* plans, uint64_t* end_bits, int* status, int num_jobs, size_t smem_bytes,
                           bool all_tables_staged, cudaStream_t stream, unsigned long long* trace) {
  if (num_jobs <= 0) return;
  // C++ function-local statics are initialised once, thread-safely: no worker thread launches before the limits are set
  static const bool attr_set = [] {
    cudaFuncSetAttribute(modular_stream_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(modular_stream_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    return true;
  }();
  (void)attr_set;
  if (all_tables_staged)
    modular_stream_kernel<true><<<num_jobs, 32, smem_bytes, stream>>>(cs, jobs, channels, plans, end_bits, status, num_jobs, trace);
  else
    modular_stream_kernel<false><<<num_jobs, 32, smem_bytes, stream>>>(cs, jobs, channels, plans, end_bits, status, num_jobs, trace);
}

void launch_modular_decode_batch(const DevModularBatchRef* refs, int total, size_t smem_bytes, bool all_tables_staged,
                                 cudaStream_t stream) {
  if (total <= 0) return;
  // C++ function-local statics are initialised once, thread-safely: no worker thread launches before the limits are set
  static const bool attr_set = [] {
    cudaFuncSetAttribute(modular_stream_batch_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(modular_stream_batch_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    return true;
  }();
  (void)attr_set;
  if (all_tables_staged) modular_stream_batch_kernel<true><<<total, 32, smem_bytes, stream>>>(refs, total);
  else modular_stream_batch_kernel<false><<<total, 32, smem_bytes, stream>>>(refs, total);
}

// Whether modular_stream_kernel stages every table of this job (tree, entropy tables, leaf LUTs, predictor rows).
bool modular_job_all_staged(const DevModularJob& job, uint32_t max_width) {
  const SmemLayout L = modular_layout(job.num_tree_nodes, job.code, job.lut_total, job.use_wp, max_width);
  if (L.tree == 0xffffffffu || L.luts == 0xffffffffu) return false;
  if (job.code.use_prefix ? L.prefix == 0xffffffffu : L.ans == 0xffffffffu) return false;
  if (job.use_wp && L.wp == 0xffffffffu) return false;
  return !job.code.lz77_enabled;
}

void launch_signal_word(uint32_t* host_mapped_word, uint32_t value, cudaStream_t stream) {
  signal_word_kernel<<<1, 1, 0, stream>>>(host_mapped_word, value);
}

void launch_read_globaltimer(unsigned long long* out, cudaStream_t stream) { read_globaltimer_kernel<<<1, 1, 0, stream>>>(out); }

}  // namespace jxlb
