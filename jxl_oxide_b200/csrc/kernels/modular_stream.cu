// Modular stream decode: one warp per entropy-coded Modular stream (LfCoeff, ModularLfGroup,
// HfMetadata, GlobalModular, pass-group modular data). After an HfMetadata stream the same warp places the LF group's
// varblocks (placement.cuh), so the placement rides whatever launch or batch the stream rides.
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
#include "modular_lanes.cuh"
#include "placement.cuh"

namespace jxlb {

namespace {

// The execution policy of decode_stream_channels on the device: the 32 lanes of the stream's warp.
struct DeviceWarp {
  static constexpr uint32_t kLanes = 32;
  uint32_t lane;
  __device__ __forceinline__ void sync() const { __syncwarp(); }
  template <typename T>
  __device__ __forceinline__ T bcast(T v) const { return __shfl_sync(0xffffffffu, v, 0); }
  __device__ __forceinline__ bool all(bool p) const { return __all_sync(0xffffffffu, p); }
};

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
  if (trace && lane == 0) {  // tracing aid: device clock (ns) when this stream starts / ends decoding
    unsigned long long now;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(now));
    trace[2 * job_idx] = now;
  }

  // ---- serial decode (lane 0; the whole warp computes the row prologues of the weighted-predictor fast loop) ----
  StreamState s;
  s.br.init(cs, job.bit_pos, job.bit_limit);
  s.ans_state = code.use_prefix ? 0x130000u : s.br.read(32);
  s.window = job.lz_window;
  s.lz_to_copy = s.lz_copy_pos = s.lz_decoded = 0;
  s.err = kDevOk;
  WpFastScratch fs = {nullptr, nullptr, nullptr};
  if (ALLSM && job.use_wp) {
    fs.pro = reinterpret_cast<int4*>(smem + L.fast_pro);
    fs.leaves = reinterpret_cast<uint4*>(smem + L.fast_leaves);
    fs.rows_b = reinterpret_cast<int32_t*>(smem + L.fast_rows);
  }
  decode_stream_channels(DeviceWarp{lane}, job, cv, tree, luts, chans, chplans, wp_rows, s_div, fs, s);
  int err = __shfl_sync(0xffffffffu, s.err, 0);
  if (job.place.raw && err == kDevOk) {
    // HfMetadata: the warp places the LF group's varblocks in the shared memory the tables were staged in (the launch
    // reserves at least sizeof(PlaceShared)); the raw list and the sharpness rectangle are what lane 0 just wrote
    __syncwarp();
    err = place_varblocks(PlaceWarp{lane}, *reinterpret_cast<PlaceShared*>(smem), job.place);
  }
  if (lane != 0) return;
  end_bits[job_idx] = s.br.pos();
  status[job_idx] = err;
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

void launch_signal_word(uint32_t* host_mapped_word, uint32_t value, cudaStream_t stream) {
  signal_word_kernel<<<1, 1, 0, stream>>>(host_mapped_word, value);
}

void launch_read_globaltimer(unsigned long long* out, cudaStream_t stream) { read_globaltimer_kernel<<<1, 1, 0, stream>>>(out); }

}  // namespace jxlb
