// Optimised entropy-stream kernels: Modular channel decode and HF coefficient decode.
//
// Both are strictly serial per stream (ANS state / context chain), so the design goal is the
// shortest dependent-instruction chain per symbol:
//   * one warp per stream; all 32 lanes stage the stream's tables (MA tree or its flattened LUT,
//     ANS alias tables / prefix LUTs, hybrid-uint configs, cluster maps, WP error rows) into shared
//     memory, then lane 0 walks the chain with every dependent load hitting shared memory;
//   * neighbour samples are carried in registers and the next row positions are prefetched one
//     iteration ahead (they do not depend on the decoded value);
//   * the weighted predictor divides through the 65-entry reciprocal table of the reference.
// Integer semantics are those of crates/jxl-modular/src/{image.rs,predictor.rs,ma.rs} and
// crates/jxl-vardct/src/hf_coeff.rs (bit-exact, wrapping i32).
#include "kernels.h"

#include <cstdlib>
#include "stream_common.cuh"
#include "hf_lanes.cuh"

namespace jxlb {

namespace {

// ---------------------------------------------------------------------------------------------
// HF coefficients (jxl-vardct/src/hf_coeff.rs:21-252); hftab / kTInfo live in hf_lanes.cuh
constexpr int kHfWarpsPerCta = 4;
constexpr uint32_t kHfAnsSmemBytes = 128 * 1024;
constexpr uint32_t kLaneCmapSmemBytes = 32 * 1024;  // all presets' cluster maps are staged once per CTA up to this size

// Shared-memory layout of one CTA (W streams, one warp each): everything a coefficient symbol touches is staged --
// the two context LUTs, hybrid-uint configs, the block-context map, the cluster map (SHARED_CMAP: every preset's, once
// per CTA; otherwise each warp's own preset slice), and the ANS alias tables (up to 128 KB; real libjxl d1 frames
// need ~86 KB). The tables dominate: a CTA that carries more streams holds more streams per SM for the same bytes.
struct HfSmem {
  uint32_t ctxlut, configs, bctx, cmap, cmap_stride, ans, total;
};
__host__ __device__ inline HfSmem hf_layout(const DevHfParams& p, uint32_t warps = kHfWarpsPerCta, bool shared_cmap = false) {
  HfSmem L;
  uint32_t off = 0;
  auto take = [&](uint32_t bytes) {
    uint32_t o = off;
    off += (bytes + 15) & ~15u;
    return o;
  };
  L.ctxlut = take(128);
  L.configs = take(p.code.num_clusters * 4);
  L.bctx = take(p.block_ctx_map_size);
  L.cmap_stride = shared_cmap ? 495 * p.num_block_clusters : (495 * p.num_block_clusters + 15) & ~15u;
  L.cmap = take(L.cmap_stride * (shared_cmap ? p.num_hf_presets : warps));
  uint32_t ab = p.code.use_prefix ? 0 : (p.code.num_clusters << p.code.log_alphabet_size) * 8;
  L.ans = (!p.code.use_prefix && ab <= min(kHfAnsSmemBytes, p.ans_smem_limit)) ? take(ab) : 0xffffffffu;
  L.total = off;
  return L;
}

// SUB: the frame is chroma-subsampled (JPEG transcodes), channels sit at shifted block positions. W: streams (warps)
// per CTA. SHARED_CMAP: see HfSmem.
template <bool SUB, int W = kHfWarpsPerCta, bool SHARED_CMAP = false>
__global__ void __launch_bounds__(W * 32) decode_hf_fast_kernel(const uint8_t* __restrict__ cs, DevFrame f, DevHfParams p,
                                                                const DevHfJob* __restrict__ jobs,
                                                                uint64_t* __restrict__ end_bits, int* __restrict__ status,
                                                                int num_jobs, int first_pass) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ uint32_t s_nz[W][3][32];
  const HfSmem L = hf_layout(p, W, SHARED_CMAP);
  const uint32_t tid = threadIdx.x, nthreads = blockDim.x, lane = tid & 31, warp = tid >> 5;
  // ---- stage tables (whole CTA) ----
  uint8_t* s_ctx = smem + L.ctxlut;  // [0..63): freq ctx, [64..127): nonzero ctx
  for (uint32_t i = tid; i < 63; i += nthreads) {
    s_ctx[i] = hftab::kCoeffFreqContext[i];
    s_ctx[64 + i] = hftab::kCoeffNumNonzeroContext[i];
  }
  uint32_t* s_cfg = reinterpret_cast<uint32_t*>(smem + L.configs);
  for (uint32_t i = tid; i < p.code.num_clusters; i += nthreads) s_cfg[i] = __ldg(p.code.configs + i);
  uint8_t* s_bctx = smem + L.bctx;
  for (uint32_t i = tid; i < p.block_ctx_map_size; i += nthreads) s_bctx[i] = __ldg(p.block_ctx_map + i);
  CodeView cv;
  cv.log_alphabet_size = p.code.log_alphabet_size;
  cv.use_prefix = p.code.use_prefix;
  cv.configs = s_cfg;
  cv.ans = p.code.ans;
  cv.prefix = p.code.prefix;
  cv.prefix_meta = p.code.prefix_meta;
  if (L.ans != 0xffffffffu) {
    uint4* s_ans = reinterpret_cast<uint4*>(smem + L.ans);
    const uint32_t quads = (p.code.num_clusters << p.code.log_alphabet_size) / 2;  // 2 buckets per 16 bytes
    const uint4* src = reinterpret_cast<const uint4*>(p.code.ans);
    for (uint32_t i = tid; i < quads; i += nthreads) s_ans[i] = __ldg(src + i);
    cv.ans = reinterpret_cast<const uint64_t*>(s_ans);
  }
  // ---- per-warp: stream header (HF preset) and that preset's cluster-map slice ----
  const int job_idx = blockIdx.x * W + int(warp);
  const bool active = job_idx < num_jobs;
  if (SHARED_CMAP) {
    uint8_t* dst = smem + L.cmap;
    const uint32_t n = L.cmap_stride * p.num_hf_presets;
    for (uint32_t i = tid; i < n; i += nthreads) dst[i] = __ldg(p.code.cluster_map + i);
  }
  const uint32_t nbc = p.num_block_clusters;
  DevBitReader br;
  int err = kDevOk;
  uint32_t hfp = 0;
  DevHfJob job;
  job.bit_pos = 0, job.bit_limit = 0, job.group_idx = 0;
  if (active) {
    job = jobs[job_idx];
    br.init(cs, job.bit_pos, job.bit_limit);
    uint32_t hfp_bits = 0;
    while ((1u << hfp_bits) < p.num_hf_presets) ++hfp_bits;
    hfp = br.read(hfp_bits);  // every lane reads the same bits
    if (hfp >= p.num_hf_presets) {
      err = kDevInvalid;
      hfp = 0;
    }
    if (!SHARED_CMAP) {
      uint8_t* dst = smem + L.cmap + warp * L.cmap_stride;
      const uint8_t* src = p.code.cluster_map + size_t(495) * nbc * hfp;
      for (uint32_t i = lane; i < 495 * nbc; i += 32) dst[i] = __ldg(src + i);
    }
  }
  __syncthreads();
  if (!active || lane != 0) return;

  const uint8_t* cluster_map = smem + L.cmap + (SHARED_CMAP ? hfp : warp) * L.cmap_stride;
  const uint32_t lf_idx_mul = (p.num_lf_thr[0] + 1) * (p.num_lf_thr[1] + 1) * (p.num_lf_thr[2] + 1);
  const uint32_t hf_idx_mul = p.num_qf_thr + 1;
  uint32_t ans_state = p.code.use_prefix ? 0x130000u : br.read(32);

  const uint32_t gx = job.group_idx % p.groups_per_row, gy = job.group_idx / p.groups_per_row;
  const uint32_t gb = p.group_dim_blocks;
  const uint32_t bx0 = gx * gb, by0 = gy * gb;
  const uint32_t width = min(gb, f.bw - bx0), height = min(gb, f.bh - by0);
  // (variants only, so that the measured default keeps its code) hard stop for corrupt streams, see hf_lanes.cuh
  const uint32_t* const stop_word = br.origin + ((job.bit_limit + 31) >> 5) + 4;
  uint32_t(*nz_row)[32] = s_nz[warp];
  for (int c = 0; c < 3; ++c)
    for (int i = 0; i < 32; ++i) nz_row[c][i] = 0;
  const int32_t* thr_base[3] = {p.lf_thresholds, p.lf_thresholds + p.num_lf_thr[0],
                                p.lf_thresholds + p.num_lf_thr[0] + p.num_lf_thr[1]};

  for (uint32_t y = 0; y < height && err == kDevOk; ++y)
    for (uint32_t x = 0; x < width && err == kDevOk; ++x) {
      const size_t gi = size_t(by0 + y) * f.bw + bx0 + x;
      const int32_t t = f.blk_type[gi];
      if (t < 0) continue;
      const int32_t qf = f.blk_mul[gi];
      const uint32_t w8 = kTInfo[t][0], h8 = kTInfo[t][1];
      const uint32_t order_id = kTInfo[t][3];
      const bool transpose = kTInfo[t][4] != 0;
      const uint32_t num_blocks = w8 * h8;
      const uint32_t num_blocks_log = 31u - uint32_t(__clz(int(num_blocks)));
      uint32_t lf_idx = 0;
      if (p.has_lf_quant) {
        const int cs3[3] = {0, 2, 1};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const int c = cs3[k];
          lf_idx *= p.num_lf_thr[c] + 1;
          if (p.num_lf_thr[c]) {
            const int32_t q = SUB ? f.lf_quant[c][size_t((by0 + y) >> f.vshift[c]) * f.bw + ((bx0 + x) >> f.hshift[c])] : f.lf_quant[c][gi];
            for (uint32_t i = 0; i < p.num_lf_thr[c]; ++i)
              if (q > thr_base[c][i]) ++lf_idx;
          }
        }
      }
      uint32_t hf_idx = 0;
      for (uint32_t i = 0; i < p.num_qf_thr; ++i)
        if (qf > int32_t(p.qf_thresholds[i])) ++hf_idx;
#pragma unroll 1
      for (int ci = 0; ci < 3 && err == kDevOk; ++ci) {
        const uint32_t ch_idx = uint32_t(ci) * 13 + order_id;
        const int c = (ci == 0) ? 1 : (ci == 1 ? 0 : 2);
        uint32_t sx = x, sy = y, sbx0 = bx0, sby0 = by0;
        if (SUB) {  // hf_coeff.rs:143-155: only blocks aligned to the channel's grid, at the shifted position
          const uint32_t hs = f.hshift[c], vs = f.vshift[c];
          sx = x >> hs, sy = y >> vs, sbx0 = bx0 >> hs, sby0 = by0 >> vs;
          if (hs | vs) {
            if ((sx << hs) != x || (sy << vs) != y) continue;
            if (f.blk_type[size_t(by0 + sy) * f.bw + bx0 + sx] < 0) continue;
            if (num_blocks != 1) {
              err = kDevUnsupported;
              break;
            }
          }
        }
        const uint32_t idx = (ch_idx * hf_idx_mul + hf_idx) * lf_idx_mul + lf_idx;
        const uint32_t block_ctx = s_bctx[idx];
        uint32_t predicted;
        const uint32_t nz_here = nz_row[c][sx];
        const uint32_t nz_left = sx ? nz_row[c][sx - 1] : 0;
        if (sy == 0) predicted = sx == 0 ? 32 : nz_left;
        else if (sx == 0) predicted = nz_here;
        else predicted = (nz_here + nz_left + 1) >> 1;
        const uint32_t pidx = predicted >= 8 ? 4 + predicted / 2 : predicted;
        const uint32_t nz_ctx = block_ctx + pidx * nbc;
        uint32_t cl = cluster_map[nz_ctx];
        uint32_t non_zeros = cv_read_uint(br, s_cfg[cl], cv_read_symbol(cv, ans_state, br, cl));
        if (SHARED_CMAP && br.next_word > stop_word) {
          err = kDevOverrun;
          break;
        }
        if (non_zeros > (63u << num_blocks_log)) {
          err = kDevInvalid;
          break;
        }
        const uint32_t nz_val = (non_zeros + num_blocks - 1) >> num_blocks_log;
        for (uint32_t dx = 0; dx < w8; ++dx) nz_row[c][sx + dx] = nz_val;
        if (non_zeros == 0) continue;
        uint32_t prev_nonzero = (non_zeros <= num_blocks * 4) ? 1 : 0;
        const uint32_t* order = p.orders + p.order_offset[order_id * 3 + c];
        const uint32_t size = num_blocks * 64;
        const uint8_t* cmap = cluster_map + block_ctx * 458 + 37 * nbc;
        uint32_t* plane = f.coeff[c];
        const size_t base = (size_t(sby0 + sy) * 8) * f.cw + size_t(sbx0 + sx) * 8;
        // context term of the remaining-non-zeros count; changes only after a non-zero coefficient
        uint32_t nzc_ctx = s_ctx[64 + ((non_zeros - 1) >> num_blocks_log)];
        for (uint32_t k = num_blocks, i = 0; k < size; ++k, ++i) {
          const uint32_t cctx = (nzc_ctx + uint32_t(s_ctx[i >> num_blocks_log])) * 2 + prev_nonzero;
          if (cctx >= 458) {
            err = kDevInvalid;
            break;
          }
          cl = cmap[cctx];
          const uint32_t ucoeff = cv_read_uint(br, s_cfg[cl], cv_read_symbol(cv, ans_state, br, cl));
          if (SHARED_CMAP && br.next_word > stop_word) {
            err = kDevOverrun;
            break;
          }
          if (ucoeff == 0) {
            prev_nonzero = 0;
            continue;
          }
          // the coefficient's position feeds only the store, never the decode chain
          const uint32_t o = __ldg(order + k);
          const uint32_t cvv = uint32_t(dev_unpack_signed(ucoeff)) << p.coeff_shift;
          uint32_t dx = o & 0xffff, dy = o >> 16;
          if (transpose) {
            const uint32_t tmp = dx;
            dx = dy;
            dy = tmp;
          }
          uint32_t* dst = plane + base + size_t(dy) * f.cw + dx;
          if (first_pass) *dst = cvv;
          else *dst += cvv;
          prev_nonzero = 1;
          if (--non_zeros == 0) break;
          nzc_ctx = s_ctx[64 + ((non_zeros - 1) >> num_blocks_log)];
        }
        if (br.pos() > job.bit_limit) err = kDevOverrun;
      }
    }
  if (err == kDevOk && !p.code.use_prefix && ans_state != 0x130000u) err = kDevBadStream;
  if (err == kDevOk && br.pos() > job.bit_limit) err = kDevOverrun;
  end_bits[job_idx] = br.pos();
  status[job_idx] = err;
}


// ---------------------------------------------------------------------------------------------
// Production schedule: W streams (one warp each) per CTA sharing ONE staged table set (context LUTs, hybrid-uint
// configs, block-context map, every preset's cluster map, ANS alias tables), so that an SM carries 32 streams
// (2 CTAs of 16 or 1 of 32) instead of 8. At that residency the SM's issue slots, not the per-stream latency, bound the
// stage, so the per-symbol path is written for instruction count:
//   * every table access is an LDS through a 32-bit shared address computed once per block (no generic loads, no
//     per-symbol address re-derivation);
//   * the bit reader keeps a 32-bit word index (one 32-bit compare per refill) and is topped up to >= 32 bits once per
//     symbol, which covers the ANS 16-bit refill and a prefix-code peek; only the rare long hybrid-uint tail checks again;
//   * loads never pass the section's end (stop index), so corrupt streams are caught by the position check per channel.
// Semantics: jxl-vardct/src/hf_coeff.rs:21-252, jxl-coding/src/{ans.rs:276-330, prefix.rs:335-357, lib.rs:572-605}.
__device__ __forceinline__ uint32_t sm_addr(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ uint32_t lds8(uint32_t a) {
  uint32_t v;
  asm("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ uint32_t lds32(uint32_t a) {
  uint32_t v;
  asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
__device__ __forceinline__ uint2 lds64(uint32_t a) {
  uint2 v;
  asm("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a));
  return v;
}

struct HfBits {  // LSB-first reader, 64-bit buffer + one word in flight, word-indexed
  const uint32_t* base;
  uint32_t widx, stop_idx;
  uint64_t buf;
  uint32_t ahead;
  int nbits;
  __device__ __forceinline__ void init(const uint8_t* d, uint64_t bit_pos, uint64_t bit_limit) {
    base = reinterpret_cast<const uint32_t*>(d);
    const uint32_t w = uint32_t(bit_pos >> 5), skip = uint32_t(bit_pos & 31);
    stop_idx = uint32_t((bit_limit + 31) >> 5) + 2;
    buf = uint64_t(__ldg(base + w)) >> skip;
    nbits = 32 - int(skip);
    buf |= uint64_t(__ldg(base + w + 1)) << nbits;
    nbits += 32;
    ahead = __ldg(base + w + 2);
    widx = w + 3;
  }
  __device__ __forceinline__ void refill() {  // nbits <= 32 -> nbits > 32
    buf |= uint64_t(ahead) << nbits;
    nbits += 32;
    ahead = widx <= stop_idx ? __ldg(base + widx) : 0u;
    ++widx;
  }
  __device__ __forceinline__ void top_up() {
    if (nbits < 32) refill();
  }
  __device__ __forceinline__ uint32_t take(uint32_t n) {  // n <= 32 bits that are known to be buffered
    const uint32_t v = uint32_t(buf) & (n >= 32 ? 0xffffffffu : ((1u << n) - 1));
    buf >>= n;
    nbits -= int(n);
    return v;
  }
  __device__ __forceinline__ uint64_t pos() const { return uint64_t(widx - 1) * 32 - uint64_t(nbits); }
};

struct HfTables {  // 32-bit shared addresses (ans: only when ANS_SMEM) + global fall-backs
  uint32_t cfg, ans;
  const uint64_t* ans_g;
  const uint32_t* prefix;
  const uint32_t* prefix_meta;
  uint32_t log_alphabet_size, log_bucket, use_prefix;
};

// One symbol of cluster `cl` -> hybrid-uint value. Requires >= 32 buffered bits on entry.
template <bool ANS_SMEM>
__device__ __forceinline__ uint32_t hf_read_value(const HfTables& T, HfBits& br, uint32_t& ans_state, uint32_t cl) {
  const uint32_t cfg = lds32(T.cfg + cl * 4);
  uint32_t token;
  if (T.use_prefix) {  // prefix.rs:335-357
    const uint32_t off = __ldg(T.prefix_meta + cl * 2), root_bits = __ldg(T.prefix_meta + cl * 2 + 1);
    const uint32_t peeked = uint32_t(br.buf) & 0x7fffu;
    uint32_t e = __ldg(T.prefix + off + (peeked & ((1u << root_bits) - 1)));
    if (e & 0x80000000u) {
      const uint32_t sb = (e >> 16) & 0xff;
      e = __ldg(T.prefix + off + (1u << root_bits) + (e & 0xffff) + ((peeked >> root_bits) & ((1u << sb) - 1)));
    }
    br.take((e >> 16) & 0xff);
    token = e & 0xffff;
  } else {  // ans.rs:276-330
    const uint32_t state = ans_state;
    const uint32_t idx = state & 0xfff;
    const uint32_t i = idx >> T.log_bucket;
    const uint32_t pos = idx & ((1u << T.log_bucket) - 1);
    uint2 b;
    if (ANS_SMEM) {
      b = lds64(T.ans + (((cl << T.log_alphabet_size) + i) << 3));
    } else {
      const uint64_t g = __ldg(T.ans_g + ((size_t(cl) << T.log_alphabet_size) + i));
      b = make_uint2(uint32_t(g), uint32_t(g >> 32));
    }
    const bool map_to_alias = pos >= ((b.x >> 8) & 0xff);
    const uint32_t hi = map_to_alias ? b.y : 0u;
    const uint32_t offset = (hi & 0xffff) + pos;
    const uint32_t dist = (b.x >> 16) ^ (hi >> 16);
    token = map_to_alias ? (b.x & 0xff) : i;
    uint32_t next = (state >> 12) * dist + offset;
    if (next < (1u << 16)) next = (next << 16) | br.take(16);
    ans_state = next;
  }
  // hybrid uint (lib.rs:572-605)
  const uint32_t split_exponent = cfg & 0xff;
  const uint32_t split = 1u << split_exponent;
  if (token < split) return token;
  const uint32_t msb = (cfg >> 8) & 0xff, lsb = (cfg >> 16) & 0xff;
  const uint32_t in_token = msb + lsb;
  const uint32_t n = (split_exponent - in_token + ((token - split) >> in_token)) & 31;
  br.top_up();
  const uint32_t rest = br.take(n);
  const uint32_t low = token & ((1u << lsb) - 1);
  uint32_t t = (token >> lsb) & ((1u << msb) - 1);
  t |= 1u << msb;
  return uint32_t((((uint64_t(t) << n) | rest) << lsb) | low);
}

template <bool SUB, int W, bool ANS_SMEM>
__global__ void __launch_bounds__(W * 32) decode_hf_warp_kernel(const uint8_t* __restrict__ cs, DevFrame f, DevHfParams p,
                                                                const DevHfJob* __restrict__ jobs,
                                                                uint64_t* __restrict__ end_bits, int* __restrict__ status,
                                                                int num_jobs, int first_pass) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ uint32_t s_nz[W][3][32];
  const HfSmem L = hf_layout(p, W, true);
  const uint32_t tid = threadIdx.x, nthreads = blockDim.x, lane = tid & 31, warp = tid >> 5;
  // ---- stage tables (whole CTA) ----
  uint8_t* s_ctx = smem + L.ctxlut;  // [0..63): freq ctx, [64..127): nonzero ctx
  for (uint32_t i = tid; i < 63; i += nthreads) {
    s_ctx[i] = hftab::kCoeffFreqContext[i];
    s_ctx[64 + i] = hftab::kCoeffNumNonzeroContext[i];
  }
  uint32_t* s_cfg = reinterpret_cast<uint32_t*>(smem + L.configs);
  for (uint32_t i = tid; i < p.code.num_clusters; i += nthreads) s_cfg[i] = __ldg(p.code.configs + i);
  uint8_t* s_bctx = smem + L.bctx;
  for (uint32_t i = tid; i < p.block_ctx_map_size; i += nthreads) s_bctx[i] = __ldg(p.block_ctx_map + i);
  {
    uint8_t* dst = smem + L.cmap;
    const uint32_t n = L.cmap_stride * p.num_hf_presets;
    for (uint32_t i = tid; i < n; i += nthreads) dst[i] = __ldg(p.code.cluster_map + i);
  }
  if (ANS_SMEM) {
    uint4* s_ans = reinterpret_cast<uint4*>(smem + L.ans);
    const uint32_t quads = (p.code.num_clusters << p.code.log_alphabet_size) / 2;  // 2 buckets per 16 bytes
    const uint4* src = reinterpret_cast<const uint4*>(p.code.ans);
    for (uint32_t i = tid; i < quads; i += nthreads) s_ans[i] = __ldg(src + i);
  }
  __syncthreads();
  const int job_idx = blockIdx.x * W + int(warp);
  if (job_idx >= num_jobs || lane != 0) return;

  HfTables T;
  T.cfg = sm_addr(s_cfg);
  T.ans = ANS_SMEM ? sm_addr(smem + L.ans) : 0;
  T.ans_g = p.code.ans;
  T.prefix = p.code.prefix;
  T.prefix_meta = p.code.prefix_meta;
  T.log_alphabet_size = p.code.log_alphabet_size;
  T.log_bucket = 12 - p.code.log_alphabet_size;
  T.use_prefix = p.code.use_prefix;
  const uint32_t a_ctx = sm_addr(s_ctx), a_bctx = sm_addr(s_bctx);

  const DevHfJob job = jobs[job_idx];
  HfBits br;
  br.init(cs, job.bit_pos, job.bit_limit);
  int err = kDevOk;
  uint32_t hfp_bits = 0;
  while ((1u << hfp_bits) < p.num_hf_presets) ++hfp_bits;
  uint32_t hfp = br.take(hfp_bits);
  if (hfp >= p.num_hf_presets) {
    err = kDevInvalid;
    hfp = 0;
  }
  const uint32_t nbc = p.num_block_clusters;
  const uint32_t a_cmap = sm_addr(smem + L.cmap) + hfp * L.cmap_stride;
  const uint32_t lf_idx_mul = (p.num_lf_thr[0] + 1) * (p.num_lf_thr[1] + 1) * (p.num_lf_thr[2] + 1);
  const uint32_t hf_idx_mul = p.num_qf_thr + 1;
  br.top_up();
  uint32_t ans_state = p.code.use_prefix ? 0x130000u : br.take(32);

  const uint32_t gx = job.group_idx % p.groups_per_row, gy = job.group_idx / p.groups_per_row;
  const uint32_t gb = p.group_dim_blocks;
  const uint32_t bx0 = gx * gb, by0 = gy * gb;
  const uint32_t width = min(gb, f.bw - bx0), height = min(gb, f.bh - by0);
  uint32_t(*nz_row)[32] = s_nz[warp];
  for (int c = 0; c < 3; ++c)
    for (int i = 0; i < 32; ++i) nz_row[c][i] = 0;
  const int32_t* thr_base[3] = {p.lf_thresholds, p.lf_thresholds + p.num_lf_thr[0],
                                p.lf_thresholds + p.num_lf_thr[0] + p.num_lf_thr[1]};

  for (uint32_t y = 0; y < height && err == kDevOk; ++y)
    for (uint32_t x = 0; x < width && err == kDevOk; ++x) {
      const size_t gi = size_t(by0 + y) * f.bw + bx0 + x;
      const int32_t t = f.blk_type[gi];
      if (t < 0) continue;
      const int32_t qf = f.blk_mul[gi];
      const uint32_t w8 = kTInfo[t][0], h8 = kTInfo[t][1];
      const uint32_t order_id = kTInfo[t][3];
      const bool transpose = kTInfo[t][4] != 0;
      const uint32_t num_blocks = w8 * h8;
      const uint32_t num_blocks_log = 31u - uint32_t(__clz(int(num_blocks)));
      uint32_t lf_idx = 0;
      if (p.has_lf_quant) {
        const int cs3[3] = {0, 2, 1};
#pragma unroll
        for (int k = 0; k < 3; ++k) {
          const int c = cs3[k];
          lf_idx *= p.num_lf_thr[c] + 1;
          if (p.num_lf_thr[c]) {
            const int32_t q = SUB ? f.lf_quant[c][size_t((by0 + y) >> f.vshift[c]) * f.bw + ((bx0 + x) >> f.hshift[c])] : f.lf_quant[c][gi];
            for (uint32_t i = 0; i < p.num_lf_thr[c]; ++i)
              if (q > thr_base[c][i]) ++lf_idx;
          }
        }
      }
      uint32_t hf_idx = 0;
      for (uint32_t i = 0; i < p.num_qf_thr; ++i)
        if (qf > int32_t(p.qf_thresholds[i])) ++hf_idx;
#pragma unroll 1
      for (int ci = 0; ci < 3 && err == kDevOk; ++ci) {
        const uint32_t ch_idx = uint32_t(ci) * 13 + order_id;
        const int c = (ci == 0) ? 1 : (ci == 1 ? 0 : 2);
        uint32_t sx = x, sy = y, sbx0 = bx0, sby0 = by0;
        if (SUB) {  // hf_coeff.rs:143-155: only blocks aligned to the channel's grid, at the shifted position
          const uint32_t hs = f.hshift[c], vs = f.vshift[c];
          sx = x >> hs, sy = y >> vs, sbx0 = bx0 >> hs, sby0 = by0 >> vs;
          if (hs | vs) {
            if ((sx << hs) != x || (sy << vs) != y) continue;
            if (f.blk_type[size_t(by0 + sy) * f.bw + bx0 + sx] < 0) continue;
            if (num_blocks != 1) {
              err = kDevUnsupported;
              break;
            }
          }
        }
        const uint32_t idx = (ch_idx * hf_idx_mul + hf_idx) * lf_idx_mul + lf_idx;
        const uint32_t block_ctx = lds8(a_bctx + idx);
        uint32_t predicted;
        const uint32_t nz_here = nz_row[c][sx];
        const uint32_t nz_left = sx ? nz_row[c][sx - 1] : 0;
        if (sy == 0) predicted = sx == 0 ? 32 : nz_left;
        else if (sx == 0) predicted = nz_here;
        else predicted = (nz_here + nz_left + 1) >> 1;
        const uint32_t pidx = predicted >= 8 ? 4 + predicted / 2 : predicted;
        br.top_up();
        uint32_t non_zeros = hf_read_value<ANS_SMEM>(T, br, ans_state, lds8(a_cmap + block_ctx + pidx * nbc));
        if (non_zeros > (63u << num_blocks_log)) {
          err = kDevInvalid;
          break;
        }
        const uint32_t nz_val = (non_zeros + num_blocks - 1) >> num_blocks_log;
        for (uint32_t dx = 0; dx < w8; ++dx) nz_row[c][sx + dx] = nz_val;
        if (non_zeros == 0) continue;
        uint32_t prev_nonzero = (non_zeros <= num_blocks * 4) ? 1 : 0;
        const uint32_t* order = p.orders + p.order_offset[order_id * 3 + c];
        const uint32_t size = num_blocks * 64;
        const uint32_t a_blk = a_cmap + block_ctx * 458 + 37 * nbc;  // this block context's coefficient clusters
        uint32_t* plane = f.coeff[c];
        const size_t base = (size_t(sby0 + sy) * 8) * f.cw + size_t(sbx0 + sx) * 8;
        // context term of the remaining-non-zeros count; changes only after a non-zero coefficient
        uint32_t nzc2 = lds8(a_ctx + 64 + ((non_zeros - 1) >> num_blocks_log)) * 2;
        for (uint32_t k = num_blocks, i = 0; k < size; ++k, ++i) {
          const uint32_t cctx = nzc2 + lds8(a_ctx + (i >> num_blocks_log)) * 2 + prev_nonzero;
          if (cctx >= 458) {
            err = kDevInvalid;
            break;
          }
          br.top_up();
          const uint32_t ucoeff = hf_read_value<ANS_SMEM>(T, br, ans_state, lds8(a_blk + cctx));
          if (ucoeff == 0) {
            prev_nonzero = 0;
            continue;
          }
          // the coefficient's position feeds only the store, never the decode chain
          const uint32_t o = __ldg(order + k);
          const uint32_t cvv = uint32_t(dev_unpack_signed(ucoeff)) << p.coeff_shift;
          uint32_t dx = o & 0xffff, dy = o >> 16;
          if (transpose) {
            const uint32_t tmp = dx;
            dx = dy;
            dy = tmp;
          }
          uint32_t* dst = plane + base + size_t(dy) * f.cw + dx;
          if (first_pass) *dst = cvv;
          else *dst += cvv;
          prev_nonzero = 1;
          if (--non_zeros == 0) break;
          nzc2 = lds8(a_ctx + 64 + ((non_zeros - 1) >> num_blocks_log)) * 2;
        }
        if (br.pos() > job.bit_limit) err = kDevOverrun;
      }
    }
  if (err == kDevOk && !p.code.use_prefix && ans_state != 0x130000u) err = kDevBadStream;
  if (err == kDevOk && br.pos() > job.bit_limit) err = kDevOverrun;
  end_bits[job_idx] = br.pos();
  status[job_idx] = err;
}

// ---------------------------------------------------------------------------------------------
// One thread per stream (hf_lanes.cuh). A CTA of `blockDim.x` threads carries blockDim.x streams and
// stages, once: context LUTs, hybrid-uint configs, block-context map, the cluster maps of every HF preset
// (global memory when they exceed kLaneCmapSmemBytes), the ANS alias tables (same rule as above) and 96
// bytes of non-zero-count row per stream.
struct HfLaneSmem {
  uint32_t ctxlut, small, configs, bctx, cmap, cmap_stride, nz, ans, total;
};
__host__ __device__ inline HfLaneSmem hf_lane_layout(const DevHfParams& p, uint32_t nthreads) {
  HfLaneSmem L;
  uint32_t off = 0;
  auto take = [&](uint32_t bytes) {
    uint32_t o = off;
    off += (bytes + 15) & ~15u;
    return o;
  };
  L.ctxlut = take(128);
  L.small = take((27 + 39) * 4);
  L.configs = take(p.code.num_clusters * 4);
  L.bctx = take(p.block_ctx_map_size);
  L.cmap_stride = 495 * p.num_block_clusters;
  const uint32_t cmap_bytes = L.cmap_stride * p.num_hf_presets;
  L.cmap = cmap_bytes <= kLaneCmapSmemBytes ? take(cmap_bytes) : 0xffffffffu;
  L.nz = take(96 * nthreads);
  uint32_t ab = p.code.use_prefix ? 0 : (p.code.num_clusters << p.code.log_alphabet_size) * 8;
  L.ans = (!p.code.use_prefix && ab <= min(kHfAnsSmemBytes, p.ans_smem_limit)) ? take(ab) : 0xffffffffu;
  L.total = off;
  return L;
}

template <bool SUB>
__global__ void __launch_bounds__(256) hf_block_ctx_kernel(DevFrame f, DevHfParams p, uint32_t* __restrict__ out) {
  const uint32_t bx = blockIdx.x * 32 + (threadIdx.x & 31), by = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (bx < f.bw && by < f.bh) out[size_t(by) * f.bw + bx] = hf_block_ctx_cell<SUB>(f, p, bx, by);
}

template <bool SUB>
__global__ void __launch_bounds__(128) decode_hf_lanes_kernel(const uint8_t* __restrict__ cs, DevFrame f, DevHfParams p,
                                                              const uint32_t* __restrict__ blk_ctx,
                                                              const DevHfJob* __restrict__ jobs,
                                                              uint64_t* __restrict__ end_bits, int* __restrict__ status,
                                                              int num_jobs, int first_pass, uint32_t lane_stride) {
  extern __shared__ __align__(16) uint8_t smem[];
  const uint32_t tid = threadIdx.x, nthreads = blockDim.x;
  const HfLaneSmem L = hf_lane_layout(p, nthreads);
  uint8_t* s_ctx = smem + L.ctxlut;
  for (uint32_t i = tid; i < 63; i += nthreads) {
    s_ctx[i] = hftab::kCoeffFreqContext[i];
    s_ctx[64 + i] = hftab::kCoeffNumNonzeroContext[i];
  }
  uint32_t* s_cfg = reinterpret_cast<uint32_t*>(smem + L.configs);
  for (uint32_t i = tid; i < p.code.num_clusters; i += nthreads) s_cfg[i] = __ldg(p.code.configs + i);
  uint8_t* s_bctx = smem + L.bctx;
  for (uint32_t i = tid; i < p.block_ctx_map_size; i += nthreads) s_bctx[i] = __ldg(p.block_ctx_map + i);
  uint32_t* s_small = reinterpret_cast<uint32_t*>(smem + L.small);
  for (uint32_t i = tid; i < 27; i += nthreads) s_small[i] = hf_pack_tinfo(i);
  for (uint32_t i = tid; i < 39; i += nthreads) s_small[27 + i] = p.order_offset[i];
  HfLaneTables T;
  T.tinfo = s_small;
  T.order_offset = s_small + 27;
  T.ctx = s_ctx;
  T.cfg = s_cfg;
  T.bctx = s_bctx;
  T.cmap = p.code.cluster_map;
  T.cmap_stride = L.cmap_stride;
  if (L.cmap != 0xffffffffu) {
    uint8_t* s_cmap = smem + L.cmap;
    const uint32_t n = L.cmap_stride * p.num_hf_presets;
    for (uint32_t i = tid; i < n; i += nthreads) s_cmap[i] = __ldg(p.code.cluster_map + i);
    T.cmap = s_cmap;
  }
  T.cv.log_alphabet_size = p.code.log_alphabet_size;
  T.cv.use_prefix = p.code.use_prefix;
  T.cv.configs = s_cfg;
  T.cv.ans = p.code.ans;
  T.cv.prefix = p.code.prefix;
  T.cv.prefix_meta = p.code.prefix_meta;
  if (L.ans != 0xffffffffu) {
    uint4* s_ans = reinterpret_cast<uint4*>(smem + L.ans);
    const uint32_t quads = (p.code.num_clusters << p.code.log_alphabet_size) / 2;  // 2 buckets per 16 bytes
    const uint4* src = reinterpret_cast<const uint4*>(p.code.ans);
    for (uint32_t i = tid; i < quads; i += nthreads) s_ans[i] = __ldg(src + i);
    T.cv.ans = reinterpret_cast<const uint64_t*>(s_ans);
  }
  __syncthreads();
  // lane_stride > 1: only every lane_stride-th lane carries a stream (32 / lane_stride streams per warp). Fewer streams
  // per warp diverge and collide less, so a stream finishes sooner; more of them per warp cost fewer issue slots.
  if (tid % lane_stride) return;
  const int job_idx = blockIdx.x * int(nthreads / lane_stride) + int(tid / lane_stride);
  if (job_idx >= num_jobs) return;
  const DevHfJob job = jobs[job_idx];
  hf_lane_decode<SUB>(cs, f, p, T, blk_ctx, job, smem + L.nz + tid, nthreads, first_pass, end_bits + job_idx,
                      status + job_idx);
}

}  // namespace

void launch_hf_block_ctx(DevFrame f, DevHfParams p, uint32_t* out, cudaStream_t stream) {
  const dim3 grid((f.bw + 31) / 32, (f.bh + 7) / 8);
  if (f.subsampled) hf_block_ctx_kernel<true><<<grid, 256, 0, stream>>>(f, p, out);
  else hf_block_ctx_kernel<false><<<grid, 256, 0, stream>>>(f, p, out);
}

void launch_decode_hf_lanes(const uint8_t* cs, DevFrame f, DevHfParams p, const uint32_t* blk_ctx, const DevHfJob* jobs,
                            uint64_t* end_bits, int* status, int num_jobs, int first_pass, int streams_per_cta,
                            cudaStream_t stream) {
  if (num_jobs <= 0) return;
  // C++ function-local statics are initialised once, thread-safely: no worker thread launches before the limits are set
  static const bool attr_set = [] {
    cudaFuncSetAttribute(decode_hf_lanes_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(decode_hf_lanes_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    return true;
  }();
  (void)attr_set;
  static const uint32_t env_stride = [] {
    const char* e = std::getenv("JXLB_HF_LANE_STRIDE");
    const int v = e ? std::atoi(e) : 0;
    return uint32_t(v == 1 || v == 2 || v == 4 || v == 8 || v == 16 ? v : 0);
  }();
  const uint32_t stride = env_stride ? env_stride : 1;
  const int nthreads = streams_per_cta <= 32 ? 32 : (streams_per_cta <= 64 ? 64 : 128);
  const HfLaneSmem L = hf_lane_layout(p, uint32_t(nthreads));
  const int per_cta = nthreads / int(stride);
  const int ctas = (num_jobs + per_cta - 1) / per_cta;
  if (f.subsampled)
    decode_hf_lanes_kernel<true><<<ctas, nthreads, L.total, stream>>>(cs, f, p, blk_ctx, jobs, end_bits, status, num_jobs, first_pass, stride);
  else
    decode_hf_lanes_kernel<false><<<ctas, nthreads, L.total, stream>>>(cs, f, p, blk_ctx, jobs, end_bits, status, num_jobs, first_pass, stride);
}

namespace {
template <int W, bool SHARED_CMAP>
void launch_hf_warps(const uint8_t* cs, DevFrame f, DevHfParams p, const DevHfJob* jobs, uint64_t* end_bits, int* status,
                     int num_jobs, int first_pass, cudaStream_t stream) {
  // C++ function-local statics are initialised once, thread-safely: no worker thread launches before the limits are set
  static const bool attr_set = [] {
    cudaFuncSetAttribute(decode_hf_fast_kernel<false, W, SHARED_CMAP>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(decode_hf_fast_kernel<true, W, SHARED_CMAP>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    return true;
  }();
  (void)attr_set;
  const HfSmem L = hf_layout(p, W, SHARED_CMAP);
  const int ctas = (num_jobs + W - 1) / W;
  if (f.subsampled)
    decode_hf_fast_kernel<true, W, SHARED_CMAP><<<ctas, W * 32, L.total, stream>>>(cs, f, p, jobs, end_bits, status, num_jobs, first_pass);
  else
    decode_hf_fast_kernel<false, W, SHARED_CMAP><<<ctas, W * 32, L.total, stream>>>(cs, f, p, jobs, end_bits, status, num_jobs, first_pass);
}
}  // namespace

namespace {
template <int W, bool ANS_SMEM>
void launch_hf_warp(const uint8_t* cs, DevFrame f, DevHfParams p, const DevHfJob* jobs, uint64_t* end_bits, int* status,
                    int num_jobs, int first_pass, cudaStream_t stream) {
  // C++ function-local statics are initialised once, thread-safely: no worker thread launches before the limits are set
  static const bool attr_set = [] {
    cudaFuncSetAttribute(decode_hf_warp_kernel<false, W, ANS_SMEM>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    cudaFuncSetAttribute(decode_hf_warp_kernel<true, W, ANS_SMEM>, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024);
    return true;
  }();
  (void)attr_set;
  const HfSmem L = hf_layout(p, W, true);
  const int ctas = (num_jobs + W - 1) / W;
  if (f.subsampled)
    decode_hf_warp_kernel<true, W, ANS_SMEM><<<ctas, W * 32, L.total, stream>>>(cs, f, p, jobs, end_bits, status, num_jobs, first_pass);
  else
    decode_hf_warp_kernel<false, W, ANS_SMEM><<<ctas, W * 32, L.total, stream>>>(cs, f, p, jobs, end_bits, status, num_jobs, first_pass);
}
}  // namespace

// `warps_per_cta`: streams (one warp each) per CTA sharing one staged table set: 8, 16 (default) or 32. 4 selects the
// round-1 kernel (a cluster-map slice per warp), which is also the fall-back when the cluster maps of all HF presets
// exceed kLaneCmapSmemBytes.
void launch_decode_hf(const uint8_t* cs, DevFrame f, DevHfParams p, const DevHfJob* jobs, uint64_t* end_bits, int* status,
                      int num_jobs, int first_pass, int warps_per_cta, cudaStream_t stream) {
  if (num_jobs <= 0) return;
  const bool fits = 495u * p.num_block_clusters * p.num_hf_presets <= kLaneCmapSmemBytes;
  if (!fits || warps_per_cta == 4) {
    launch_hf_warps<kHfWarpsPerCta, false>(cs, f, p, jobs, end_bits, status, num_jobs, first_pass, stream);
    return;
  }
  const bool ans_smem = hf_layout(p, 16, true).ans != 0xffffffffu;  // the layout's ANS decision does not depend on W
  const int w = warps_per_cta >= 32 ? 32 : (warps_per_cta >= 16 ? 16 : 8);
#define JXLB_HF(W_)                                                                                          \
  do {                                                                                                       \
    if (ans_smem) launch_hf_warp<W_, true>(cs, f, p, jobs, end_bits, status, num_jobs, first_pass, stream);  \
    else launch_hf_warp<W_, false>(cs, f, p, jobs, end_bits, status, num_jobs, first_pass, stream);          \
  } while (0)
  if (w == 32) JXLB_HF(32);
  else if (w == 16) JXLB_HF(16);
  else JXLB_HF(8);
#undef JXLB_HF
}

}  // namespace jxlb
