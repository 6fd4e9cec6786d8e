// CUDA (sm_90a) implementation of the planner's Backend seam: every sample-level stage runs as
// a kernel on one stream; planes live in HBM for the whole frame. There is no CPU fallback: any
// CUDA failure raises Error(kErrCuda).
#pragma once
#include <cuda_runtime.h>

#include <functional>
#include <map>
#include <string>
#include <vector>

#include "host/backend.h"
#include "host/jbrd.h"
#include "kernels/kernels.h"
#include "launch_tables.h"

namespace jxlb {

// One Modular launch handed to a pipeline's LF batch service (csrc/pipeline.cu): copies to make before the kernel, the
// frame's job tables, copies to make after it. run() blocks the calling (frame) thread until the batch has run.
struct LfBatchItem {
  struct Copy {
    void* dst;
    const void* src;
    size_t bytes;
  };
  Copy up[2];    // host (pinned) -> device
  int num_up = 0;
  DevModularBatchRef ref{};  // .job is filled per CTA by the service
  int num_jobs = 0;
  size_t smem_bytes = 0;
  bool all_staged = false;
  Copy down[2];  // device -> host (pinned)
  int num_down = 0;
  // set when ref.counter / ref.done_flag are: the item is complete as soon as *done_flag == ref.done_seq
  volatile uint32_t* done_flag = nullptr;
  bool want_timing = false;
  float elapsed_ms = 0.0f;  // device time of the batch kernel this item rode in
};
class LfBatchService {
 public:
  virtual ~LfBatchService() {}
  virtual void run(LfBatchItem& item) = 0;  // throws jxlb::Error on a CUDA failure
};

struct StopDecode {};  // thrown by stage_marker() when a stage entry point has what it asked for

class CudaBackend : public Backend, private TableSink {
 public:
  // own_stream = false: a pipeline decoder. It borrows the stream of a heavy slot (on_heavy_stage -> set_stream) and
  // runs its LF stage through `lf_service` without any stream.
  explicit CudaBackend(int device, bool own_stream = true);
  ~CudaBackend() override;

  void set_codestream(const uint8_t* data, size_t size) override;
  void new_frame() override;
  int alloc_plane(uint32_t w, uint32_t h, bool zero) override;
  void free_plane(int id) override;
  void download_rect(const View& v, void* dst) override;
  void copy_rect(const View& src, const View& dst) override;
  void decode_modular(std::vector<ModularStreamJob>& jobs) override;
  int squeeze_inverse(const View& avg, const View& residual, bool horizontal) override;
  std::vector<int> squeeze_inverse_many(const std::vector<std::pair<View, View>>& avg_res, bool horizontal) override;
  void rct_inverse(const View v[3], uint32_t rct_type) override;
  void palette_inverse(const View& palette, const std::vector<View>& targets, const Transform& t, const WpHeader& wp,
                       uint32_t bit_depth) override;
  void int_to_float(const View& v, const BitDepth& depth) override;
  void modular_xyb_to_float(const View yxb[3], const float m_lf_unscaled[3]) override;
  void build_block_info(VarDctState& st, const std::vector<BlockInfoJob>& jobs) override;
  void decode_hf(VarDctState& st, std::vector<HfGroupJob>& jobs) override;
  void lf_dequant(VarDctState& st, const std::vector<LfDequantJob>& jobs) override;
  void lf_chroma_from_luma(VarDctState& st) override;
  void lf_adaptive_smoothing(VarDctState& st) override;
  void hf_dequant_cfl(VarDctState& st) override;
  void hf_transform(VarDctState& st) override;
  void gaborish(const View v[3], const float weights[3][2]) override;
  void epf(const View v[3], const View& sigma, const EpfParams& p, bool sigma_is_constant) override;
  int upsample(const View& v, uint32_t factor_log2, const ImageHeader& ih) override;
  int upsample_jpeg(const View& v, bool horizontal, bool vertical, uint32_t out_w, uint32_t out_h) override;
  void blend_patches(const std::vector<PatchJob>& jobs) override;
  void blend_raw(const DevPatchJob& job);  // one rectangle on caller-owned device memory (jxlb_blend)
  void splat_splines(const View v[3], const std::vector<SplineArc>& arcs) override;
  void add_noise(const View v[3], const float lut[8], uint32_t group_dim, uint64_t seed0, float corr_x, float corr_b) override;
  void add_noise_in_frame(const View v[3], uint32_t field_w, uint32_t field_h, const float lut[8], uint32_t group_dim,
                          uint64_t seed0, float corr_x, float corr_b) override;
  void xyb_to_rgb(const View v[3], const ColorParams& p) override;
  void ycbcr_to_rgb(const View v[3], const YcbcrParams& p) override;
  bool filters_colour_fused(const View v[3], const RestorationFilter& rf, const View& sigma, bool sigma_is_constant,
                            const ColorParams* colour) override;
  void stage_marker(const char* name, const View* views, int n) override;
  void phase_mark(const char* name) override;
  // JPEG reconstruction (jxlb_reconstruct_jpeg): with a job set, the frame's coefficients are encoded as the job's JPEG
  // scans (kernels/jpeg.cu) and the decode ends with JpegDone.
  void vardct_coefficients(const VarDctState& st) override;
  JpegJob* jpeg_job = nullptr;

  // Heavy stage of a frame (everything that needs full-resolution planes): the planner announces it with the bytes it
  // is about to allocate; a pipeline (csrc/pipeline.cu) hooks in here to bound the number of frames past this point
  // and to hand the backend a pre-allocated slab the big planes are carved from (no allocator calls per frame).
  void begin_heavy_stage(size_t bytes_hint) override;
  std::function<void(size_t)> on_heavy_stage;  // called once per frame, before the first big allocation
  std::function<void()> on_need_stream;        // a stream-less (pipeline) decoder needs its stream now: must set_stream()
  void set_arena(void* base, size_t bytes) {
    arena_base_ = static_cast<uint8_t*>(base);
    arena_cap_ = bytes;
    arena_off_ = 0;
  }
  // The slab goes back to its owner: nothing of this backend may point into it afterwards.
  void end_arena();
  // allocation budget (0 = none): pool allocations and slab carvings count until freed
  void set_mem_limit(uint64_t bytes) { mem_limit_ = bytes; }
  uint64_t mem_in_use() const { return mem_in_use_; }
  size_t arena_peak() const { return arena_peak_; }
  size_t arena_spill() const { return arena_spill_; }  // bytes that did not fit the slab (allocated from the pool)

  cudaStream_t stream() { return S(); }
  void set_stream(cudaStream_t s) { stream_ = s; }
  bool has_stream() const { return stream_ != nullptr; }
  void end_lease();  // a pipeline decoder gives its borrowed stream back (everything queued on it has run)
  LfBatchService* lf_service = nullptr;
  // "inputs resident in HBM": upload once, then point the next decode at the device copy
  uint8_t* upload_resident(const uint8_t* data, size_t size);
  void use_resident_once(const uint8_t* dptr) { resident_next_ = dptr; }
  void sync();
  void* plane_ptr(int id) const { return id < 0 ? nullptr : planes_.at(id).ptr; }
  // device pointer + stride (elements) of a view's top-left element
  DevView dev_view(const View& v) const;

  // stage entry points: decode up to `stop_stage`, copy its planes to `stop_dst` (device, row pitch `stop_stride` words)
  std::string stop_stage;
  std::vector<void*> stop_dst;
  uint32_t stop_stride = 0;
  std::vector<std::pair<uint32_t, uint32_t>> stop_dims;  // out: width, height of every plane of the stage
  // test hook: when on, stage_marker() snapshots planes to host memory
  bool capture = false;
  std::map<std::string, std::vector<std::vector<uint32_t>>> stages;
  std::map<std::string, std::vector<std::pair<uint32_t, uint32_t>>> stage_dims;
  // launch accounting for bench.py ("gpu_launches")
  uint64_t launches = 0;
  // per-kernel device timing (CUDA events on the launching stream), for bench.py's roofline
  // Any layout (launch_pack): the tables go with the launch; `dst` is host memory of `bytes`, or device memory of this
  // decoder's GPU (the packed frame then stays in HBM, e.g. for an NCCL gather). Returns after the samples are in `dst`.
  void pack(const DevPackSpec& p, const std::vector<DevPackChannel>& channels, const std::vector<DevPackSpot>& spots, void* dst,
            size_t bytes, bool dst_on_device);
  bool fuse_filters = true;  // single-kernel Gaborish+EPF+colour (off: stage-by-stage, for stage parity tests)
  // HF coefficient streams per CTA (jxlb_set_hf_streams_per_cta, hf_schedule). Initialised from JXLB_HF_LANES.
  int hf_streams_per_cta = 0;
  // streams per warp of the thread-per-stream HF kernel (jxlb_set_hf_streams_per_warp, hf_schedule); 0: the default
  int hf_streams_per_warp = 0;
  bool profile = false;
  bool host_phases = false;  // wall clock per planner phase only (no CUDA events): where a frame's latency goes under load
  bool trace_device = false;  // modular streams stamp the device clock; host launch/return times are logged
  double phase_t0_ = -1.0;  // wall clock (ms) of the previous phase_mark
  std::map<std::string, std::pair<uint64_t, double>> profile_acc;  // name -> (launches, total ms)
  void resolve_profile();

 private:
  struct PlaneRec {
    void* ptr;
    uint32_t w, h;
  };
  void* dmalloc(size_t bytes);
  void dfree(void* p);
  // Host tables for the next launch. They are gathered in a pinned staging block that mirrors a device block of the
  // same size byte for byte, so the device address is known at once and ONE asynchronous copy per launch (flush_uploads,
  // called by begin_k) moves everything: a stage used to cost ~10 cudaMallocAsync + pageable cudaMemcpyAsync + cudaFreeAsync
  // calls, each taking the driver's context lock that every other decoder thread of the process wants too. The block is
  // recycled at every sync(). Oversized requests fall back to a pool allocation + direct copy (freed by release_temps).
  void* upload_temp(const void* src, size_t bytes);
  const void* put(const void* src, size_t bytes) override { return upload_temp(src, bytes); }  // launch tables
  void* stage_scratch(size_t bytes);  // device scratch from the same block (no host data), zeroed by nobody
  void flush_uploads();
  void release_temps();
  // results of a stage (end positions, status words): device -> pinned host, readable after the next sync()
  void* fetch_result(const void* dsrc, size_t bytes);
  DevFrame dev_frame(const VarDctState& st) const {
    return make_dev_frame(st, [this](int id) { return plane_ptr(id); });
  }
  void ensure_static_tables();
  uint64_t encode_jpeg_scan(const VarDctState& st, const JpegScanPlan& plan, std::vector<uint8_t>* out);
  void begin_k(const char* name);
  void end_k();
  struct PendingTiming {
    const char* name;
    cudaEvent_t e0, e1;
  };
  std::vector<PendingTiming> pending_;

 public:
  // Profiling timeline: every kernel launch and host phase with start/end in ms since a
  // process-wide reference point (device events and host clock are aligned at that point).
  struct TimelineEntry {
    std::string name;
    double t0_ms, t1_ms;
  };
  std::vector<TimelineEntry> timeline;

 private:

  cudaStream_t S();  // the decoder's stream, leased on first use when it has none of its own
  void* lf_arena_alloc(size_t bytes);
  bool in_lf_arena(const void* p) const {
    return lf_arena_ && p >= static_cast<const void*>(lf_arena_) && p < static_cast<const void*>(lf_arena_ + kLfArenaBytes);
  }
  int device_;
  bool own_stream_ = true;
  static constexpr size_t kLfArenaBytes = size_t(64) << 20;
  uint8_t* lf_arena_ = nullptr;  // device block of kLfArenaBytes the LF-stage planes of a pipeline decoder are carved from
  size_t lf_arena_off_ = 0;
  size_t pending_cs_bytes_ = 0;        // encoded bytes staged in h_input_, not yet copied to d_codestream_
  std::vector<void*> deferred_free_;   // pool pointers released while the decoder had no stream
  uint8_t* h_stage_ = nullptr;   // pinned
  uint8_t* d_stage_ = nullptr;
  size_t stage_cap_ = 0, stage_off_ = 0, stage_flushed_ = 0;
  uint8_t* h_result_ = nullptr;  // pinned
  size_t result_cap_ = 0, result_off_ = 0;
  uint8_t* h_input_ = nullptr;   // pinned staging of the encoded bytes
  size_t input_cap_ = 0;
  volatile uint32_t* h_flag_ = nullptr;  // mapped pinned word the stream writes its sync sequence number to
  uint32_t sync_seq_ = 0, item_seq_ = 0;
  uint8_t* arena_base_ = nullptr;
  size_t arena_cap_ = 0, arena_off_ = 0, arena_peak_ = 0, arena_spill_ = 0;
  bool heavy_announced_ = false;
  uint64_t mem_limit_ = 0, mem_in_use_ = 0;
  std::map<void*, size_t> alloc_sizes_;  // pool allocations (for the budget)
  cudaStream_t stream_ = nullptr;
  cudaEvent_t sync_event_ = nullptr;
  cudaMemPool_t pool_ = nullptr;  // this decoder's own stream-ordered pool (no cross-stream reuse dependencies)
  uint8_t* d_codestream_ = nullptr;
  const uint8_t* active_cs_ = nullptr;
  const uint8_t* resident_next_ = nullptr;
  size_t codestream_cap_ = 0;
  std::map<int, PlaneRec> planes_;
  int next_id_ = 0;
  std::vector<void*> temps_;
  // static tables
  uint32_t* d_natural_orders_ = nullptr;
  uint32_t natural_order_offset_[13];
  bool sec_uploaded_ = false;
  // per-frame caches
  const HfGlobalSyntax* cached_hfg_ = nullptr;
  float* d_dequant_ = nullptr;
  float* d_dequant_default_ = nullptr;  // all-default matrix set, uploaded once per decoder
  DevDequantParams dequant_default_params_;
  DevDequantParams dequant_params_;
  DevDequantParams pending_dequant_;  // handed from hf_dequant_cfl() to hf_transform() when the two are fused
  bool have_pending_dequant_ = false;
};

}  // namespace jxlb
