// Per-stream code of the Modular stream kernel (modular_stream.cu): the weighted predictor, the per-channel decode
// loops and the channel dispatch of one stream. Plain integer C++ over pointers, with the warp's collectives behind a
// `Warp` policy, so that tests/emu/ compiles the same code for the host and checks it against the oracle.
// Integer semantics are those of crates/jxl-modular/src/{image.rs:456-593,1169-1260, predictor.rs, ma.rs}.
#pragma once
#include <cstdlib>
#include <type_traits>

#include "kernels.h"
#include "modular_plan.cuh"
#include "stream_common.cuh"

// Test hooks of the host emulation (tests/emu/modular_emu.cc); no-ops in the kernel.
#ifndef JXLB_MODULAR_EVENT
#define JXLB_MODULAR_EVENT(k)
#endif
#ifndef JXLB_WP_FAST_FORCE_TRIP
#define JXLB_WP_FAST_FORCE_TRIP(samples) 0u
#endif

namespace jxlb {
namespace {

__device__ __forceinline__ uint32_t wp_weight32(const uint32_t* div, uint32_t err_sum, uint32_t maxweight) {
  const uint32_t t = (err_sum + 1) >> 5;
  const uint32_t shift = 31u - uint32_t(__clz(int(t | 1u)));
  return 4 + ((maxweight * div[(err_sum >> shift) + 1]) >> shift);
}

// Weighted mix of the four sub-predictions in fast mode (predictor.rs:360-395), before the clamp.
__device__ __forceinline__ int32_t wp_mix32(const uint32_t* div, int32_t f0, int32_t f1, int32_t f2, int32_t f3, uint32_t es0,
                                            uint32_t es1, uint32_t es2, uint32_t es3, uint32_t w0, uint32_t w1, uint32_t w2,
                                            uint32_t w3) {
  uint32_t g0 = wp_weight32(div, es0, w0), g1 = wp_weight32(div, es1, w1), g2 = wp_weight32(div, es2, w2),
           g3 = wp_weight32(div, es3, w3);
  uint32_t sum_weights = g0 + g1 + g2 + g3;
  const uint32_t log_weight = ilog2_u32(sum_weights >> 4);
  g0 >>= log_weight, g1 >>= log_weight, g2 >>= log_weight, g3 >>= log_weight;
  sum_weights = g0 + g1 + g2 + g3;
  const int32_t s = int32_t(sum_weights >> 1) - 1 + f0 * int32_t(g0) + f1 * int32_t(g1) + f2 * int32_t(g2) + f3 * int32_t(g3);
  return int32_t((int64_t(s) * int64_t(div[sum_weights])) >> 24);
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
      int32_t pred = wp_mix32(div, f0, f1, f2, f3, a0 + b0 + c0, a1 + b1 + c1, a2 + b2 + c2, a3 + b3 + c3, w0, w1, w2, w3);
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
                                               const bool lz77, const uint32_t y_begin, const uint32_t y_end) {
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
  if (WP && y_begin == 0) wp.reset(width, wp_rows, job.wp, s_div);

  for (uint32_t y = y_begin; y < y_end && s.err == kDevOk; ++y) {
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

// A channel whose subtree is a single leaf with the Zero (0), West (1) or Gradient (5) predictor, in an ANS stream
// without LZ77 (every HfMetadata channel libjxl writes, and all of the bench frames' HfMetadata): context, hybrid-uint
// config, multiplier and offset are fixed for the channel, so a sample is one ANS symbol, one hybrid uint, the
// prediction and the store. Same results as decode_channel<false, 1, true>.
template <int PRED>
__device__ __forceinline__ void decode_channel_const_leaf(const DevModularJob& job, const CodeView& cv, const MaNode leaf,
                                                          const DevChannel out, StreamState& s) {
  const uint32_t cluster = leaf.a >> 8, cfg = cv.configs[cluster];
  const int32_t mult = int32_t(leaf.b), offset = leaf.value;
  for (uint32_t y = 0; y < out.h; ++y) {
    int32_t* row = out.ptr + size_t(y) * out.stride;
    const int32_t* rn = y ? row - out.stride : row;
    // West of the first sample is N (0 on the first row); on the first row N = NW = W (predictor.rs:554-564)
    int32_t w = y ? rn[0] : 0;
    for (uint32_t x = 0; x < out.w; ++x) {
      const uint32_t token_value = cv_read_uint(s.br, cfg, cv_read_symbol_ans(cv, s.ans_state, s.br, cluster));
      int32_t pred = 0;
      if (PRED == 1) {
        pred = w;
      } else if (PRED == 5) {
        const int32_t n = y ? rn[x] : w, nw = y ? rn[x ? x - 1 : 0] : w;
        const int32_t hi = max(n, w), lo = min(n, w);
        pred = nw >= hi ? lo : (nw <= lo ? hi : wsub(wadd(lo, hi), nw));
      }
      w = wadd(wadd(wmul(dev_unpack_signed(token_value), mult), offset), pred);
      row[x] = w;
    }
    if (s.br.pos() > job.bit_limit) {
      s.err = kDevOverrun;
      return;
    }
  }
}

// Scratch of the weighted-predictor fast loop (shared memory on the device); pro == nullptr: not available.
struct WpFastScratch {
  int4* pro;        // kFastChunk x 4 int4: the row prologue
  uint4* leaves;    // kFastMaxLeaves packed leaves
  int32_t* rows_b;  // 5 * width words: the second pair of error rows
};

// Fixed parameters of the fast loop for one channel.
struct WpFastParams {
  int32_t p1, p2, p3a, p3b, p3c, p3d, p3e;
  uint32_t mw0, mw1, mw2, mw3;
  int32_t lut_base;
  uint32_t lut_last;
};

// Previous-row terms of column x of row y >= 1 (see wp_fast_rows) into slot i of the prologue.
__device__ __forceinline__ void wp_prologue_column(const WpFastParams& P, const uint32_t x, const uint32_t width,
                                                   const int32_t* rn, const int32_t* rnn, const int32_t* rows_prev,
                                                   int4* pro, const uint32_t i) {
  const uint32_t wm1 = width - 1, xm = x ? x - 1 : 0, xp = min(x + 1, wm1);
  const uint4* Up = reinterpret_cast<const uint4*>(rows_prev);
  const int32_t* Tp = rows_prev + size_t(width) * 4;
  const int32_t n = rn[x], nw = rn[xm], ne = rn[xp], nn = rnn ? rnn[x] : n;
  const int32_t n3 = int32_t(uint32_t(n) << 3), nw3 = int32_t(uint32_t(nw) << 3), ne3 = int32_t(uint32_t(ne) << 3),
                nn3 = int32_t(uint32_t(nn) << 3);
  const int32_t ten = Tp[x], tenw = Tp[xm], tene = Tp[xp];
  const uint4 um = Up[xm], u0 = Up[x], up = Up[xp];
  int32_t Pm = ten;
  if (abs(tenw) > abs(Pm)) Pm = tenw;
  if (abs(tene) > abs(Pm)) Pm = tene;
  const int32_t f3num = wadd(wadd(wadd(wmul(tenw, P.p3a), wmul(ten, P.p3b)), wadd(wmul(tene, P.p3c), wmul(wsub(nn3, n3), P.p3d))),
                             wmul(nw3, P.p3e));
  pro[i] = make_int4(n3, wsub(ne3, n3), min(n3, ne3), max(n3, ne3));
  pro[kFastChunk + i] = make_int4(wadd(ten, tene), wadd(ten, tenw), f3num, Pm);
  pro[2 * kFastChunk + i] = make_int4(int32_t(um.x + u0.x + up.x), int32_t(um.y + u0.y + up.y), int32_t(um.z + u0.z + up.z),
                                      int32_t(um.w + u0.w + up.w));
  pro[3 * kFastChunk + i] = make_int4(ten, ten ^ tenw, abs(Pm), 0);
}

// West-side state lane 0 carries through a row of the fast loop.
struct WpFastLane {
  int32_t w, te_w;
  uint32_t e1_0, e1_1, e1_2, e1_3, e2_0, e2_1, e2_2, e2_3;
  uint32_t trip;
};

// One sample at column x (prologue slot i). LAST: the channel's last column, where e(x-1) counts twice.
template <bool LAST>
__device__ __forceinline__ void wp_fast_step(WpFastLane& S, const WpFastParams& P, const CodeView& cv, WordBitReader& br,
                                             uint32_t& ans_state, const uint4* leaves, const int4* pro, const uint32_t i,
                                             const uint32_t x, int32_t* row, uint4* Uc, int32_t* Tc, const uint32_t* div) {
  const int4 A = pro[i], B = pro[kFastChunk + i], C = pro[2 * kFastChunk + i], D = pro[3 * kFastChunk + i];
  const int32_t w3 = int32_t(uint32_t(S.w) << 3);
  const int32_t f0 = wadd(w3, A.y);
  const int32_t f1 = wsub(A.x, wmul(wadd(S.te_w, B.x), P.p1) >> 5);
  const int32_t f2 = wsub(w3, wmul(wadd(S.te_w, B.y), P.p2) >> 5);
  const int32_t f3 = wsub(A.x, wsub(B.z, wmul(w3, P.p3e)) >> 5);
  const uint32_t es0 = uint32_t(C.x) + S.e1_0 + S.e2_0 + (LAST ? S.e1_0 : 0u);
  const uint32_t es1 = uint32_t(C.y) + S.e1_1 + S.e2_1 + (LAST ? S.e1_1 : 0u);
  const uint32_t es2 = uint32_t(C.z) + S.e1_2 + S.e2_2 + (LAST ? S.e1_2 : 0u);
  const uint32_t es3 = uint32_t(C.w) + S.e1_3 + S.e2_3 + (LAST ? S.e1_3 : 0u);
  int32_t pred = wp_mix32(div, f0, f1, f2, f3, es0, es1, es2, es3, P.mw0, P.mw1, P.mw2, P.mw3);
  if (((D.x ^ S.te_w) | D.y) <= 0) pred = min(max(pred, min(A.z, w3)), max(A.w, w3));
  const int32_t me = D.z > abs(S.te_w) ? B.w : S.te_w;
  const uint32_t li = me < P.lut_base ? 0u : min(uint32_t(me) - uint32_t(P.lut_base), P.lut_last);
  const uint4 leaf = leaves[li];
  const uint32_t token_value = cv_read_uint(br, leaf.y, cv_read_symbol_ans(cv, ans_state, br, leaf.x));
  const int32_t value = wadd(wadd(wmul(dev_unpack_signed(token_value), int32_t(leaf.z)), int32_t(leaf.w)), (pred + 3) >> 3);
  row[x] = value;
  const int32_t s8 = int32_t(uint32_t(value) << 3);
  const int32_t te = wsub(pred, s8);
  S.trip |= ((uint32_t(value) + 0x40000u) >> 19) | ((uint32_t(te) + 0x200000u) >> 22);
  S.e2_0 = S.e1_0, S.e2_1 = S.e1_1, S.e2_2 = S.e1_2, S.e2_3 = S.e1_3;
  S.e1_0 = uint32_t(abs(f0 - s8) + 3) >> 3, S.e1_1 = uint32_t(abs(f1 - s8) + 3) >> 3;
  S.e1_2 = uint32_t(abs(f2 - s8) + 3) >> 3, S.e1_3 = uint32_t(abs(f3 - s8) + 3) >> 3;
  Tc[x] = te;
  Uc[x] = make_uint4(S.e1_0, S.e1_1, S.e1_2, S.e1_3);
  S.te_w = te;
  S.w = value;
}

// Weighted-predictor fast loop: rows 1 .. h-1 of a channel whose subtree tests only max_error (property 15) and whose
// leaves all use the weighted predictor (libjxl's LfCoeff tree) in an ANS stream without LZ77, in fast mode; row 0 and
// the predictor state at the start of row 1 come from decode_channel<true, 2, true>.
//
// Everything of a sample that depends only on rows y-1 and y-2 is computed by the 32 lanes ahead of lane 0, kFastChunk
// columns at a time, into `pro` (4 x int4 per column):
//   A = { n3, ne3 - n3, min(n3, ne3), max(n3, ne3) }                           (n3 = n << 3, edge-adjusted neighbours)
//   B = { te_n + te_ne, te_n + te_nw, f3 numerator without its -w3 * p3e term, P }
//   C = { R_0 .. R_3 }:  R_i(x) = U_i(x-1) + U_i(x) + U_i(x+1), U = the previous row's sub-errors (clamped at the edges)
//   D = { te_n, te_n ^ te_nw, |P| }
// where P is the first of te_n, te_nw, te_ne with the largest |.|, so max_error = |P| > |te_w| ? P : te_w (the
// reference's order). The error sum of sub-predictor i is R_i(x) + e_i(x-1) + e_i(x-2), with e(-1) = e(-2) = 0 at the row
// start; in the last column record() copies b into c, so e_i(x-1) counts twice there (the LAST step).
// The reassociated sums are exact: wrapping adds and multiplies are associative and commutative modulo 2^32, and in
// fast mode no i32 intermediate of the reference's formulas overflows (FastWp), so the wrapped result is the value.
// Lane 0 carries only the west-side state: w, te_w, e(x-1), e(x-2), the ANS state and the bit reader. Leaves are
// packed as { cluster, hybrid-uint config, multiplier, offset }, one shared load from max_error. The current row's
// errors go to the other pair of error rows (the previous row's must stay readable for the next chunk's prologue).
//
// A sample or true error outside the fast-mode range does not switch to i64 here: the function returns false on every
// lane and the caller decodes the whole channel again in decode_channel from a snapshot of the stream state (so such a
// channel costs up to twice its time; lossy LF never leaves the range).
// `Warp` is the execution policy: a warp of 32 lanes on the device, one lane that does every column on the host.
template <class Warp>
__device__ __forceinline__ bool wp_fast_rows(const Warp& warp, const DevModularJob& job, const CodeView& cv,
                                             const DevChannelPlan& plan, const uint4* leaves, const DevChannel out,
                                             int32_t* rows_prev, int32_t* rows_cur, int4* pro, const uint32_t* div,
                                             StreamState& stream) {
  const uint32_t width = out.w, wm1 = width - 1;
  WpFastParams P;
  P.p1 = int32_t(job.wp[0]), P.p2 = int32_t(job.wp[1]), P.p3a = int32_t(job.wp[2]), P.p3b = int32_t(job.wp[3]);
  P.p3c = int32_t(job.wp[4]), P.p3d = int32_t(job.wp[5]), P.p3e = int32_t(job.wp[6]);
  P.mw0 = job.wp[7], P.mw1 = job.wp[8], P.mw2 = job.wp[9], P.mw3 = job.wp[10];
  P.lut_base = plan.lut_base;
  P.lut_last = plan.lut_len - 1;
  WordBitReader br = stream.br;  // registers for the loop, written back on return
  uint32_t ans_state = stream.ans_state;
  int err = stream.err;
  for (uint32_t y = 1; y < out.h; ++y) {
    if (warp.bcast(err) != kDevOk) break;
    int32_t* row = out.ptr + size_t(y) * out.stride;
    const int32_t* rn = row - out.stride;
    const int32_t* rnn = y >= 2 ? rn - out.stride : nullptr;
    uint4* Uc = reinterpret_cast<uint4*>(rows_cur);
    int32_t* Tc = rows_cur + size_t(width) * 4;
    WpFastLane S = {rn[0], 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
    for (uint32_t x0 = 0; x0 < width; x0 += kFastChunk) {
      const uint32_t x1 = min(x0 + kFastChunk, width);
      warp.sync();  // lane 0 is done with the previous chunk's prologue (and has written row y-1)
      for (uint32_t x = x0 + warp.lane; x < x1; x += Warp::kLanes) wp_prologue_column(P, x, width, rn, rnn, rows_prev, pro, x - x0);
      warp.sync();
      if (warp.lane == 0) {
        const uint32_t xe = min(x1, wm1);
#pragma unroll 2
        for (uint32_t x = x0; x < xe; ++x) wp_fast_step<false>(S, P, cv, br, ans_state, leaves, pro, x - x0, x, row, Uc, Tc, div);
        if (x1 == width) wp_fast_step<true>(S, P, cv, br, ans_state, leaves, pro, wm1 - x0, wm1, row, Uc, Tc, div);
      }
    }
    S.trip |= JXLB_WP_FAST_FORCE_TRIP(uint64_t(y + 1) * width);
    if (warp.bcast(S.trip)) return false;
    if (br.pos() > job.bit_limit) err = kDevOverrun;
    int32_t* t = rows_prev;
    rows_prev = rows_cur;
    rows_cur = t;
  }
  if (warp.lane == 0) {
    stream.br = br;
    stream.ans_state = ans_state;
    stream.err = err;
  }
  return true;
}

// The channels of one stream, decoded into `chans` (lane 0 walks the serial chain; the other lanes take part only in
// the fast loop's row prologues). `fs.pro == nullptr` disables the weighted-predictor fast loop.
template <class Warp>
__device__ __forceinline__ void decode_stream_channels(const Warp& warp, const DevModularJob& job, const CodeView& cv,
                                                       const MaNode* tree, const uint16_t* luts, const DevChannel* chans,
                                                       const DevChannelPlan* chplans, int32_t* wp_rows,
                                                       const uint32_t* s_div, const WpFastScratch fs, StreamState& s) {
  const DevEntropyCode& code = job.code;
  const bool lz77 = code.lz77_enabled != 0;
  const bool use_wp = job.use_wp != 0;
  FastWp wp;
  wp.slow = false;
  for (uint32_t ci = 0; ci < job.num_channels; ++ci) {
    if (warp.bcast(s.err) != kDevOk) break;
    const DevChannel out = chans[ci];
    if (!out.w || !out.h) continue;
    const DevChannelPlan plan = chplans[ci];
    const uint16_t* lut = luts + plan.lut_offset;
    const int lut_kind = plan.lut_prop < 0 ? 0 : ((use_wp && plan.lut_prop == 15) ? 2 : 1);
    const bool fast = !lz77 && !code.use_prefix;
    if (fast && lut_kind == 1 && plan.lut_len == 1) {  // a single leaf
      const MaNode leaf = tree[lut[0]];
      const uint32_t predictor = leaf.a & 0xff;
      if (predictor == 0 || predictor == 1 || predictor == 5) {
        JXLB_MODULAR_EVENT(3);
        if (warp.lane == 0) {
          if (predictor == 0) decode_channel_const_leaf<0>(job, cv, leaf, out, s);
          else if (predictor == 1) decode_channel_const_leaf<1>(job, cv, leaf, out, s);
          else decode_channel_const_leaf<5>(job, cv, leaf, out, s);
        }
        continue;
      }
    }
    DevChannel prev[kMaxPrev];
    int nprev = 0;
    for (int pj = int(ci) - 1; pj >= 0 && nprev < kMaxPrev; --pj) {
      const DevChannel p = chans[pj];
      if (p.w == out.w && p.h == out.h && p.hshift == out.hshift && p.vshift == out.vshift && p.w && p.h) prev[nprev++] = p;
    }
#define JXLB_DECODE_CHANNEL_ROWS(WP_, LUT_, FAST_, Y0_, Y1_) \
  decode_channel<WP_, LUT_, FAST_>(job, code, cv, tree, lut, plan, out, prev, nprev, ci, wp_rows, s_div, wp, s, lz77, Y0_, Y1_)
#define JXLB_DECODE_CHANNEL(WP_, LUT_, FAST_) JXLB_DECODE_CHANNEL_ROWS(WP_, LUT_, FAST_, 0, out.h)
    if (fs.pro && fast && lut_kind == 2 && plan.lut_len <= kFastMaxLeaves) {
      bool all_wp = true;
      for (uint32_t i = warp.lane; i < plan.lut_len; i += Warp::kLanes) {
        const MaNode nd = tree[lut[i]];
        all_wp = all_wp && (nd.a & 0xff) == 6;
        fs.leaves[i] = make_uint4(nd.a >> 8, cv.configs[nd.a >> 8], nd.b, uint32_t(nd.value));
      }
      if (warp.all(all_wp)) {
        JXLB_MODULAR_EVENT(1);
        const StreamState s0 = s;
        int go = 0;
        if (warp.lane == 0) {
          JXLB_DECODE_CHANNEL_ROWS(true, 2, true, 0, 1);
          go = s.err == kDevOk && !wp.slow;
        }
        if (warp.bcast(go)) {
          if (!wp_fast_rows(warp, job, cv, plan, fs.leaves, out, wp_rows, fs.rows_b, fs.pro, s_div, s) && warp.lane == 0) {
            JXLB_MODULAR_EVENT(2);
            s = s0;
            JXLB_DECODE_CHANNEL(true, 2, true);
          }
        } else if (warp.lane == 0) {
          JXLB_DECODE_CHANNEL_ROWS(true, 2, true, 1, out.h);
        }
        continue;
      }
    }
    if (warp.lane != 0) continue;
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
#undef JXLB_DECODE_CHANNEL_ROWS
  }
  if (warp.lane == 0) {
    if (s.err == kDevOk && !code.use_prefix && s.ans_state != 0x130000u) s.err = kDevBadStream;
    if (s.err == kDevOk && s.br.pos() > job.bit_limit) s.err = kDevOverrun;
  }
}

}  // namespace
}  // namespace jxlb
