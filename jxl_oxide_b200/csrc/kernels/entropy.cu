// HF coefficient decode kernels (jxl-vardct/src/hf_coeff.rs:21-252): one warp per stream (decode_hf_warp_kernel) and
// one thread per stream (decode_hf_lanes_kernel, per-stream code in hf_lanes.cuh). hf_schedule() in launch_tables.cc
// picks one. Both are strictly serial per stream (ANS state / context chain), so every table a symbol touches is staged
// in shared memory. Integer semantics are bit-exact (wrapping i32).
#include "kernels.h"

#include "stream_common.cuh"
#include "hf_lanes.cuh"

namespace jxlb {

namespace {

// ---------------------------------------------------------------------------------------------
// HF coefficients; hftab / kTInfo live in hf_lanes.cuh

// Shared-memory layout of one CTA (W streams, one warp each): everything a coefficient symbol touches is staged --
// the two context LUTs, hybrid-uint configs, the block-context map, every preset's cluster map, and the ANS alias
// tables (up to kHfAnsSmemBytes; real libjxl d1 frames need ~86 KB). The layout does not depend on W. The tables
// dominate: a CTA that carries more streams holds more streams per SM for the same bytes.
struct HfSmem {
  uint32_t ctxlut, configs, bctx, cmap, cmap_stride, ans, total;
};
__host__ __device__ inline HfSmem hf_layout(const DevHfParams& p) {
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
  L.cmap_stride = 495 * p.num_block_clusters;
  L.cmap = take(L.cmap_stride * p.num_hf_presets);
  uint32_t ab = p.code.use_prefix ? 0 : (p.code.num_clusters << p.code.log_alphabet_size) * 8;
  L.ans = (!p.code.use_prefix && ab <= kHfAnsSmemBytes) ? take(ab) : 0xffffffffu;
  L.total = off;
  return L;
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
template <bool SUB, int W, bool ANS_SMEM>
__global__ void __launch_bounds__(W * 32) decode_hf_warp_kernel(const uint8_t* __restrict__ cs, DevFrame f, DevHfParams p,
                                                                const DevHfJob* __restrict__ jobs,
                                                                uint64_t* __restrict__ end_bits, int* __restrict__ status,
                                                                int num_jobs, int first_pass) {
  extern __shared__ __align__(16) uint8_t smem[];
  __shared__ uint32_t s_nz[W][3][32];
  const HfSmem L = hf_layout(p);
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

  HfTables<HfLds> T;
  T.cfg = HfLds::addr(s_cfg);
  T.ans = ANS_SMEM ? HfLds::addr(smem + L.ans) : 0;
  T.ans_g = p.code.ans;
  T.prefix = p.code.prefix;
  T.prefix_meta = p.code.prefix_meta;
  T.log_alphabet_size = p.code.log_alphabet_size;
  T.log_bucket = 12 - p.code.log_alphabet_size;
  T.use_prefix = p.code.use_prefix;
  const uint32_t a_ctx = HfLds::addr(s_ctx), a_bctx = HfLds::addr(s_bctx);

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
  const uint32_t a_cmap = HfLds::addr(smem + L.cmap) + hfp * L.cmap_stride;
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
        const uint32_t block_ctx = HfLds::u8(a_bctx + idx);
        uint32_t predicted;
        const uint32_t nz_here = nz_row[c][sx];
        const uint32_t nz_left = sx ? nz_row[c][sx - 1] : 0;
        if (sy == 0) predicted = sx == 0 ? 32 : nz_left;
        else if (sx == 0) predicted = nz_here;
        else predicted = (nz_here + nz_left + 1) >> 1;
        const uint32_t pidx = predicted >= 8 ? 4 + predicted / 2 : predicted;
        br.top_up();
        uint32_t non_zeros = hf_read_value<HfLds, ANS_SMEM>(T, br, ans_state, HfLds::u8(a_cmap + block_ctx + pidx * nbc));
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
        uint32_t nzc2 = HfLds::u8(a_ctx + 64 + ((non_zeros - 1) >> num_blocks_log)) * 2;
        for (uint32_t k = num_blocks, i = 0; k < size; ++k, ++i) {
          const uint32_t cctx = nzc2 + HfLds::u8(a_ctx + (i >> num_blocks_log)) * 2 + prev_nonzero;
          if (cctx >= 458) {
            err = kDevInvalid;
            break;
          }
          br.top_up();
          const uint32_t ucoeff = hf_read_value<HfLds, ANS_SMEM>(T, br, ans_state, HfLds::u8(a_blk + cctx));
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
          nzc2 = HfLds::u8(a_ctx + 64 + ((non_zeros - 1) >> num_blocks_log)) * 2;
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
// One thread per stream (hf_lanes.cuh). A CTA carries `per_cta` streams and stages, once, the tables of
// hf_lane_layout(per_cta); its THREADS = per_cta * 32 / K threads all stage, and lane l < K of warp w then runs stream
// slot w * K + l. Fewer streams per warp (K < 32) give each scheduler more warps that diverge across fewer streams,
// for the same CTA count and shared memory. Its streams start from their groups' varblock lists (hf_block_list_kernel).

// One CTA per group: the group's cells in raster order, 256 at a time, compacted with a ballot and a prefix over warps.
template <bool SUB>
__global__ void __launch_bounds__(256) hf_block_list_kernel(DevFrame f, DevHfParams p, uint2* __restrict__ list,
                                                            uint32_t* __restrict__ counts) {
  __shared__ uint32_t s_warp[8];
  const uint32_t g = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const HfGroupRect r = hf_group_rect(f, p, g);
  const uint32_t n = r.width * r.height;
  uint2* out = list + size_t(g) * p.group_dim_blocks * p.group_dim_blocks;
  uint32_t base = 0;
  for (uint32_t i0 = 0; i0 < n; i0 += 256) {
    uint2 rec;
    const bool has = i0 + tid < n && hf_block_record<SUB>(f, p, r, i0 + tid, rec);
    const uint32_t ballot = __ballot_sync(0xffffffffu, has);
    if (lane == 0) s_warp[warp] = __popc(ballot);
    __syncthreads();
    uint32_t before = base, total = 0;
    for (uint32_t w = 0; w < 8; ++w) {
      before += w < warp ? s_warp[w] : 0;
      total += s_warp[w];
    }
    if (has) out[before + __popc(ballot & ((1u << lane) - 1))] = rec;
    base += total;
    __syncthreads();
  }
  if (tid == 0) counts[g] = base;
}

// LZ77: stream `job_idx` keeps its values in lz_windows[job_idx * lz_window_len ...] (unused otherwise).
// The minimum-blocks hint caps every instantiation at 64 registers (65536 / 1024), as many as a 1024-thread CTA can
// have: a CTA of more threads carries no more streams, so it should not take more of the SM's register file than it must.
template <bool SUB, bool STAGED, bool LZ77, int THREADS>
__global__ void __launch_bounds__(THREADS, 1024 / THREADS) decode_hf_lanes_kernel(const uint8_t* __restrict__ cs, DevFrame f, DevHfParams p,
                                                                  const uint2* __restrict__ list,
                                                                  const uint32_t* __restrict__ counts,
                                                                  const DevHfJob* __restrict__ jobs,
                                                                  uint64_t* __restrict__ end_bits, int* __restrict__ status,
                                                                  int num_jobs, int first_pass, uint32_t per_cta,
                                                                  uint32_t* lz_windows, uint32_t lz_window_len) {
  extern __shared__ __align__(16) uint8_t smem[];
  const uint32_t tid = threadIdx.x, nthreads = blockDim.x;
  const HfLaneSmem L = hf_lane_layout(p, per_cta);
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
  HfLaneView<HfLds> T;
  T.tinfo = HfLds::addr(s_small);
  T.order_offset = HfLds::addr(s_small + 27);
  T.ctx = HfLds::addr(s_ctx);
  T.bctx = HfLds::addr(s_bctx);
  const uint32_t k = per_cta * 32 / THREADS, lane = tid & 31;
  const uint32_t slot = (tid >> 5) * k + lane;  // this thread's stream in the CTA, if lane < k
  T.nz = HfLds::addr(smem + L.nz + slot);
  T.nz_stride = per_cta;
  T.cmap_stride = L.cmap_stride;
  T.cmap = 0;
  T.cmap_ptr = p.code.cluster_map;
  if (L.cmap != 0xffffffffu) {
    uint8_t* s_cmap = smem + L.cmap;
    const uint32_t n = L.cmap_stride * p.num_hf_presets;
    for (uint32_t i = tid; i < n; i += nthreads) s_cmap[i] = __ldg(p.code.cluster_map + i);
    T.cmap = HfLds::addr(s_cmap);
    T.cmap_ptr = s_cmap;
  }
  T.code.cfg = HfLds::addr(s_cfg);
  T.code.ans = 0;
  T.code.ans_g = p.code.ans;
  T.code.prefix = p.code.prefix;
  T.code.prefix_meta = p.code.prefix_meta;
  T.code.log_alphabet_size = p.code.log_alphabet_size;
  T.code.log_bucket = 12 - p.code.log_alphabet_size;
  T.code.use_prefix = p.code.use_prefix;
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
    T.code.ans = HfLds::addr(s_ans);
    T.cv.ans = reinterpret_cast<const uint64_t*>(s_ans);
  }
  __syncthreads();
  const int job_idx = blockIdx.x * int(per_cta) + int(slot);
  if (lane >= k || job_idx >= num_jobs) return;
  const DevHfJob job = jobs[job_idx];
  const uint32_t gb = p.group_dim_blocks;
  if constexpr (LZ77) {
    Lz77State lz;
    lz77_init(lz, lz_windows + size_t(job_idx) * lz_window_len, lz_window_len);
    hf_lane_stream<SUB, STAGED, true>(cs, f, p, T, list + size_t(job.group_idx) * gb * gb, __ldg(counts + job.group_idx),
                                      job, first_pass, &lz, end_bits + job_idx, status + job_idx);
  } else {
    hf_lane_stream<SUB, STAGED, false>(cs, f, p, T, list + size_t(job.group_idx) * gb * gb, __ldg(counts + job.group_idx),
                                       job, first_pass, nullptr, end_bits + job_idx, status + job_idx);
  }
}

}  // namespace

size_t hf_block_list_count(DevFrame f, DevHfParams p) {
  const uint32_t gb = p.group_dim_blocks;
  return size_t((f.bh + gb - 1) / gb) * p.groups_per_row;
}

void launch_hf_block_list(DevFrame f, DevHfParams p, uint2* list, uint32_t* counts, cudaStream_t stream) {
  const uint32_t groups = uint32_t(hf_block_list_count(f, p));
  if (f.subsampled) hf_block_list_kernel<true><<<groups, 256, 0, stream>>>(f, p, list, counts);
  else hf_block_list_kernel<false><<<groups, 256, 0, stream>>>(f, p, list, counts);
}

namespace {
template <int THREADS>
void launch_hf_lanes(const uint8_t* cs, DevFrame f, DevHfParams p, const uint2* list, const uint32_t* counts,
                     const DevHfJob* jobs, uint64_t* end_bits, int* status, int num_jobs, int first_pass, uint32_t per_cta,
                     cudaStream_t stream, uint32_t* lz_windows, uint32_t lz_window_len) {
  // C++ function-local statics are initialised once, thread-safely: no worker thread launches before the limits are set
  static const bool attr_set = [] {
    const int bytes = 200 * 1024;
    cudaFuncSetAttribute(decode_hf_lanes_kernel<false, false, false, THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    cudaFuncSetAttribute(decode_hf_lanes_kernel<true, false, false, THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    cudaFuncSetAttribute(decode_hf_lanes_kernel<false, true, false, THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    cudaFuncSetAttribute(decode_hf_lanes_kernel<true, true, false, THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    cudaFuncSetAttribute(decode_hf_lanes_kernel<false, false, true, THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    cudaFuncSetAttribute(decode_hf_lanes_kernel<true, false, true, THREADS>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    return true;
  }();
  (void)attr_set;
  const HfLaneSmem L = hf_lane_layout(p, per_cta);
  const int ctas = (num_jobs + int(per_cta) - 1) / int(per_cta);
#define JXLB_HF_LANES(SUB_, STAGED_, LZ77_)                                                                        \
  decode_hf_lanes_kernel<SUB_, STAGED_, LZ77_, THREADS><<<ctas, THREADS, L.total, stream>>>(                       \
      cs, f, p, list, counts, jobs, end_bits, status, num_jobs, first_pass, per_cta, lz_windows, lz_window_len)
  if (p.code.lz77_enabled) {
    if (f.subsampled) JXLB_HF_LANES(true, false, true);
    else JXLB_HF_LANES(false, false, true);
  } else if (hf_lane_staged(p, L)) {
    if (f.subsampled) JXLB_HF_LANES(true, true, false);
    else JXLB_HF_LANES(false, true, false);
  } else {
    if (f.subsampled) JXLB_HF_LANES(true, false, false);
    else JXLB_HF_LANES(false, false, false);
  }
#undef JXLB_HF_LANES
}
}  // namespace

void launch_decode_hf_lanes(const uint8_t* cs, DevFrame f, DevHfParams p, const uint2* list, const uint32_t* counts,
                            const DevHfJob* jobs, uint64_t* end_bits, int* status, int num_jobs, int first_pass,
                            int streams_per_cta, int streams_per_warp, cudaStream_t stream, uint32_t* lz_windows,
                            uint32_t lz_window_len) {
  if (num_jobs <= 0) return;
  const uint32_t per_cta = streams_per_cta <= 64 ? 64 : 128;
  const uint32_t k = streams_per_warp <= 4 ? 4 : (streams_per_warp <= 8 ? 8 : (streams_per_warp <= 16 ? 16 : 32));
#define JXLB_HF_LANES_T(T_) \
  launch_hf_lanes<T_>(cs, f, p, list, counts, jobs, end_bits, status, num_jobs, first_pass, per_cta, stream, lz_windows, lz_window_len)
  switch (per_cta * 32 / k) {
    case 64: JXLB_HF_LANES_T(64); break;
    case 128: JXLB_HF_LANES_T(128); break;
    case 256: JXLB_HF_LANES_T(256); break;
    case 512: JXLB_HF_LANES_T(512); break;
    default: JXLB_HF_LANES_T(1024); break;
  }
#undef JXLB_HF_LANES_T
}

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
  const HfSmem L = hf_layout(p);
  const int ctas = (num_jobs + W - 1) / W;
  if (f.subsampled)
    decode_hf_warp_kernel<true, W, ANS_SMEM><<<ctas, W * 32, L.total, stream>>>(cs, f, p, jobs, end_bits, status, num_jobs, first_pass);
  else
    decode_hf_warp_kernel<false, W, ANS_SMEM><<<ctas, W * 32, L.total, stream>>>(cs, f, p, jobs, end_bits, status, num_jobs, first_pass);
}
}  // namespace

void launch_decode_hf(const uint8_t* cs, DevFrame f, DevHfParams p, const DevHfJob* jobs, uint64_t* end_bits, int* status,
                      int num_jobs, int first_pass, int warps_per_cta, cudaStream_t stream) {
  if (num_jobs <= 0) return;
  const bool ans_smem = hf_layout(p).ans != 0xffffffffu;
#define JXLB_HF(W_)                                                                                          \
  do {                                                                                                       \
    if (ans_smem) launch_hf_warp<W_, true>(cs, f, p, jobs, end_bits, status, num_jobs, first_pass, stream);  \
    else launch_hf_warp<W_, false>(cs, f, p, jobs, end_bits, status, num_jobs, first_pass, stream);          \
  } while (0)
  if (warps_per_cta == 32) JXLB_HF(32);
  else if (warps_per_cta == 16) JXLB_HF(16);
  else JXLB_HF(8);
#undef JXLB_HF
}

}  // namespace jxlb
