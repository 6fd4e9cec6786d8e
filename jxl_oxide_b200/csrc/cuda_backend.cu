// See cuda_backend.h.
#include "cuda_backend.h"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <atomic>
#include <thread>

namespace jxlb {

void upload_sec_large(const float* host224);  // kernels/vardct.cu

#define CUDA_CHECK(expr)                                                                              \
  do {                                                                                                \
    cudaError_t err__ = (expr);                                                                       \
    if (err__ != cudaSuccess)                                                                         \
      fail(kErrCuda, std::string("CUDA error: ") + cudaGetErrorString(err__) + " at " #expr);        \
  } while (0)

CudaBackend::CudaBackend(int device, bool own_stream) : device_(device), own_stream_(own_stream) {
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0)
    fail(kErrCuda, "no CUDA device available: the jxl_oxide_b200 hot path has no CPU fallback");
  CUDA_CHECK(cudaSetDevice(device_));
  if (own_stream_) CUDA_CHECK(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
  CUDA_CHECK(cudaEventCreateWithFlags(&sync_event_, cudaEventBlockingSync | cudaEventDisableTiming));
  stage_cap_ = size_t(2) << 20;
  CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&h_stage_), stage_cap_, cudaHostAllocDefault));
  CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&d_stage_), stage_cap_));
  result_cap_ = size_t(256) << 10;
  CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&h_result_), result_cap_, cudaHostAllocMapped));  // batched LF streams write here
  {
    void* f = nullptr;
    CUDA_CHECK(cudaHostAlloc(&f, 128, cudaHostAllocMapped));
    h_flag_ = static_cast<volatile uint32_t*>(f);
    h_flag_[0] = 0;
    h_flag_[16] = 0;  // second word (own cache line): completion of this decoder's item in a batched LF launch
  }
  ensure_static_tables();
  // A private stream-ordered pool per decoder: freed planes are reused by this decoder's next frame
  // (release threshold = never trim), and an allocation never has to wait on another decoder's
  // stream the way reuse inside the shared default pool can.
  cudaMemPoolProps props;
  std::memset(&props, 0, sizeof(props));
  props.allocType = cudaMemAllocationTypePinned;
  props.handleTypes = cudaMemHandleTypeNone;
  props.location.type = cudaMemLocationTypeDevice;
  props.location.id = device_;
  CUDA_CHECK(cudaMemPoolCreate(&pool_, &props));
  uint64_t keep = UINT64_MAX;
  CUDA_CHECK(cudaMemPoolSetAttribute(pool_, cudaMemPoolAttrReleaseThreshold, &keep));
  // All kernels of the library ask for the same (maximum shared memory) L1/shared split: an SM only
  // changes its split when idle, so kernels with different splits cannot share an SM, and the
  // long-running one-warp entropy CTAs would otherwise fence other streams' kernels off their SMs.
  CUDA_CHECK(cudaDeviceSetCacheConfig(cudaFuncCachePreferShared));
  if (const char* lanes = std::getenv("JXLB_HF_LANES")) {
    const int n = std::atoi(lanes);
    hf_streams_per_cta = n <= 0 ? 0 : (n <= 4 ? 4 : (n <= 8 ? 8 : (n <= 16 ? 16 : (n <= 32 ? 32 : (n <= 64 ? 64 : 128)))));
  }
}

CudaBackend::~CudaBackend() {
  cudaSetDevice(device_);
  if (stream_) cudaStreamSynchronize(stream_);
  for (auto& kv : planes_)
    if (!(arena_base_ && kv.second.ptr >= static_cast<void*>(arena_base_) && kv.second.ptr < static_cast<void*>(arena_base_ + arena_cap_)) &&
        !in_lf_arena(kv.second.ptr))
      cudaFree(kv.second.ptr);
  for (void* p : temps_)
    if (!in_lf_arena(p)) cudaFree(p);
  for (void* p : deferred_free_) cudaFree(p);
  if (d_codestream_ && !in_lf_arena(d_codestream_) && stream_) cudaFreeAsync(d_codestream_, stream_);
  if (d_natural_orders_) cudaFree(d_natural_orders_);
  if (d_dequant_) cudaFree(d_dequant_);
  if (d_dequant_default_) cudaFree(d_dequant_default_);
  if (sync_event_) cudaEventDestroy(sync_event_);
  if (h_stage_) cudaFreeHost(h_stage_);
  if (d_stage_) cudaFree(d_stage_);
  if (h_result_) cudaFreeHost(h_result_);
  if (h_input_) cudaFreeHost(h_input_);
  if (h_flag_) cudaFreeHost(const_cast<uint32_t*>(h_flag_));
  if (stream_ && own_stream_) cudaStreamDestroy(stream_);
  if (lf_arena_) cudaFree(lf_arena_);
  if (pool_) cudaMemPoolDestroy(pool_);
}

cudaStream_t CudaBackend::S() {
  if (!stream_) {
    // A pipeline decoder has no stream of its own: the LF stage runs through the batch service, everything else on the
    // stream of a heavy slot. Whatever needs a stream before the planner announces the heavy stage takes the slot now.
    JXLB_CHECK(bool(on_need_stream), kErrCuda, "decoder has no CUDA stream");
    on_need_stream();
    JXLB_CHECK(stream_ != nullptr, kErrCuda, "no CUDA stream was leased to the decoder");
    if (pending_cs_bytes_) {  // encoded bytes staged for a batch that never came
      CUDA_CHECK(cudaMemcpyAsync(d_codestream_, h_input_, pending_cs_bytes_, cudaMemcpyHostToDevice, stream_));
      pending_cs_bytes_ = 0;
    }
    for (void* p : deferred_free_) CUDA_CHECK(cudaFreeAsync(p, stream_));
    deferred_free_.clear();
  }
  return stream_;
}

void CudaBackend::end_lease() {
  if (!stream_ || own_stream_) return;
  release_temps();
  if (d_dequant_) {
    dfree(d_dequant_);
    d_dequant_ = nullptr;
    cached_hfg_ = nullptr;
  }
  if (d_codestream_ && !in_lf_arena(d_codestream_)) {
    CUDA_CHECK(cudaFreeAsync(d_codestream_, stream_));
    d_codestream_ = nullptr;
    codestream_cap_ = 0;
  }
  stream_ = nullptr;
}

void* CudaBackend::lf_arena_alloc(size_t bytes) {
  if (!lf_arena_) {
    CUDA_CHECK(cudaSetDevice(device_));
    CUDA_CHECK(cudaMalloc(reinterpret_cast<void**>(&lf_arena_), kLfArenaBytes));
  }
  const size_t need = (bytes + 255) & ~size_t(255);
  if (lf_arena_off_ + need > kLfArenaBytes) return nullptr;
  void* p = lf_arena_ + lf_arena_off_;
  lf_arena_off_ += need;
  return p;
}

void CudaBackend::begin_heavy_stage(size_t bytes_hint) {
  if (heavy_announced_) return;
  heavy_announced_ = true;
  if (on_heavy_stage) on_heavy_stage(bytes_hint);
}

void CudaBackend::end_arena() {
  if (!arena_base_) return;
  auto inside = [&](const void* p) { return p >= static_cast<void*>(arena_base_) && p < static_cast<void*>(arena_base_ + arena_cap_); };
  std::vector<void*> keep;
  for (void* p : temps_)
    if (!inside(p)) keep.push_back(p);
  temps_.swap(keep);
  if (d_dequant_ && inside(d_dequant_)) {
    d_dequant_ = nullptr;
    cached_hfg_ = nullptr;
  }
  for (auto it = planes_.begin(); it != planes_.end();)  // planes a failed decode left behind
    it = inside(it->second.ptr) ? planes_.erase(it) : std::next(it);
  arena_base_ = nullptr;
  arena_cap_ = arena_off_ = 0;
}

void* CudaBackend::dmalloc(size_t bytes) {
  void* p = nullptr;
  if (mem_limit_ && mem_in_use_ + bytes > mem_limit_)
    fail(kErrOutOfMemory, "allocation budget exceeded: " + std::to_string(mem_in_use_ + bytes) + " > " + std::to_string(mem_limit_) + " bytes");
  if (arena_base_ && bytes >= (256u << 10)) {  // big planes: carved from the frame slab, released with it
    const size_t need = (bytes + 511) & ~size_t(511);
    if (arena_off_ + need <= arena_cap_) {
      p = arena_base_ + arena_off_;
      arena_off_ += need;
      arena_peak_ = std::max(arena_peak_, arena_off_);
      if (mem_limit_) mem_in_use_ += need;  // released with the slab
      return p;
    }
    arena_spill_ += need;
  }
  if (!stream_ && lf_service) {  // a pipeline decoder without a stream yet: LF-stage planes come from its own LF arena
    if (void* q = lf_arena_alloc(std::max<size_t>(bytes, 16))) return q;
  }
  CUDA_CHECK(cudaSetDevice(device_));
  CUDA_CHECK(cudaMallocFromPoolAsync(&p, std::max<size_t>(bytes, 16), pool_, S()));
  if (mem_limit_) {
    mem_in_use_ += bytes;
    alloc_sizes_[p] = bytes;
  }
  return p;
}
void CudaBackend::dfree(void* p) {
  if (!p) return;
  if (in_lf_arena(p)) return;  // recycled as a whole at the next decode call
  if (!stream_ && lf_service) {  // a pool allocation of the previous frame released before this frame has a stream
    deferred_free_.push_back(p);
    return;
  }
  if (arena_base_ && p >= arena_base_ && p < arena_base_ + arena_cap_) return;  // the slab is reset as a whole
  if (mem_limit_) {
    auto it = alloc_sizes_.find(p);
    if (it != alloc_sizes_.end()) {
      mem_in_use_ -= std::min<uint64_t>(mem_in_use_, it->second);
      alloc_sizes_.erase(it);
    }
  }
  CUDA_CHECK(cudaFreeAsync(p, S()));
}
void* CudaBackend::upload_temp(const void* src, size_t bytes) {
  const size_t off = (stage_off_ + 15) & ~size_t(15);
  if (off + bytes <= stage_cap_) {
    if (bytes) std::memcpy(h_stage_ + off, src, bytes);
    stage_off_ = off + bytes;
    return d_stage_ + off;
  }
  void* p = dmalloc(bytes);  // does not fit the staging block
  temps_.push_back(p);
  if (bytes) CUDA_CHECK(cudaMemcpyAsync(p, src, bytes, cudaMemcpyHostToDevice, S()));
  return p;
}
void* CudaBackend::stage_scratch(size_t bytes) {
  if (stream_) flush_uploads();  // the range handed out must not be part of a later host -> device copy
  const size_t off = (stage_off_ + 15) & ~size_t(15);
  if (off + bytes <= stage_cap_) {
    stage_off_ = off + bytes;
    if (stream_) stage_flushed_ = stage_off_;  // stream-less: the batch copies the whole block before its kernel
    return d_stage_ + off;
  }
  void* p = dmalloc(bytes);
  temps_.push_back(p);
  return p;
}
void CudaBackend::flush_uploads() {
  if (!stream_ && lf_service) return;  // stream-less LF stage: the batch service copies the block
  if (stage_off_ > stage_flushed_)
    CUDA_CHECK(cudaMemcpyAsync(d_stage_ + stage_flushed_, h_stage_ + stage_flushed_, stage_off_ - stage_flushed_, cudaMemcpyHostToDevice, S()));
  stage_flushed_ = stage_off_;
}
void* CudaBackend::fetch_result(const void* dsrc, size_t bytes) {
  const size_t off = (result_off_ + 15) & ~size_t(15);
  JXLB_CHECK(off + bytes <= result_cap_, kErrUnsupported, "too many stream jobs in one launch for the result buffer");
  CUDA_CHECK(cudaMemcpyAsync(h_result_ + off, dsrc, bytes, cudaMemcpyDeviceToHost, S()));
  result_off_ = off + bytes;
  return h_result_ + off;
}
void CudaBackend::release_temps() {
  for (void* p : temps_) dfree(p);
  temps_.clear();
}
void CudaBackend::sync() {
  if (!stream_) return;  // a pipeline decoder between leases: nothing of it is queued anywhere
  // The stream writes a sequence number into a mapped host word and the host thread polls it (short spin, then
  // 50 us naps). Waiting inside the driver instead (cudaEventSynchronize, or the implicit wait of a pageable
  // cudaMemcpyAsync) was measured to return many milliseconds late once dozens of decoder threads wait at the same time:
  // the waits serialise on the driver. Here a waiting thread never enters the driver.
  flush_uploads();
  const uint32_t seq = ++sync_seq_;
  launch_signal_word(const_cast<uint32_t*>(h_flag_), seq, S());
  ++launches;
  uint32_t spins = 0;
  const auto t_begin = std::chrono::steady_clock::now();
  auto t0 = t_begin;
  while (*h_flag_ != seq) {
    if (++spins < 2000) {
#if defined(__x86_64__)
      __builtin_ia32_pause();
#endif
      continue;
    }
    // naps grow with the time already waited (1/8 of it, 20..200 us): a short kernel is noticed within microseconds, a
    // 15 ms one costs its thread ~100 wake-ups instead of 300
    const auto waited = std::chrono::steady_clock::now() - t_begin;
    const long nap_us = std::min<long>(200, std::max<long>(20, std::chrono::duration_cast<std::chrono::microseconds>(waited).count() / 8));
    std::this_thread::sleep_for(std::chrono::microseconds(nap_us));
    if ((spins & 255) == 0 && std::chrono::steady_clock::now() - t0 > std::chrono::milliseconds(200)) {
      // a faulting kernel never writes the word: ask the driver from time to time
      cudaError_t e = cudaStreamQuery(S());
      if (e == cudaSuccess) break;
      if (e != cudaErrorNotReady) fail(kErrCuda, std::string("CUDA error: ") + cudaGetErrorString(e) + " while waiting for the stream");
      t0 = std::chrono::steady_clock::now();
    }
  }
  std::atomic_thread_fence(std::memory_order_acquire);
  stage_off_ = stage_flushed_ = 0;  // everything queued so far has run: the staging block is free again
  result_off_ = 0;
  resolve_profile();
}

namespace {
// Process-wide time origin shared by all decoders: a device event and the host clock sampled
// together after a device synchronisation.
struct TimeOrigin {
  cudaEvent_t ev = nullptr;
  double host_ms = 0.0;
  unsigned long long dev_ns = 0;  // %globaltimer at the origin
};
double host_now_ms() {
  return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}
TimeOrigin& time_origin() {
  static TimeOrigin o = [] {
    TimeOrigin t;
    cudaEventCreate(&t.ev);
    cudaDeviceSynchronize();
    cudaEventRecord(t.ev, 0);
    cudaEventSynchronize(t.ev);
    unsigned long long* d = nullptr;
    cudaMalloc(&d, 8);
    launch_read_globaltimer(d, 0);
    cudaMemcpy(&t.dev_ns, d, 8, cudaMemcpyDeviceToHost);
    cudaFree(d);
    t.host_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
    return t;
  }();
  return o;
}
}  // namespace

void CudaBackend::begin_k(const char* name) {
  S();  // a pipeline decoder takes its stream here at the latest
  flush_uploads();
  ++launches;
  if (!profile) return;
  time_origin();
  PendingTiming t;
  t.name = name;
  CUDA_CHECK(cudaEventCreate(&t.e0));
  CUDA_CHECK(cudaEventCreate(&t.e1));
  CUDA_CHECK(cudaEventRecord(t.e0, S()));
  pending_.push_back(t);
}

void CudaBackend::end_k() {
  if (!profile || pending_.empty()) return;
  CUDA_CHECK(cudaEventRecord(pending_.back().e1, S()));
}

void CudaBackend::resolve_profile() {
  for (PendingTiming& t : pending_) {
    float ms = 0.0f;
    if (cudaEventElapsedTime(&ms, t.e0, t.e1) == cudaSuccess) {
      auto& acc = profile_acc[t.name];
      acc.first += 1;
      acc.second += double(ms);
      float since = 0.0f;
      if (cudaEventElapsedTime(&since, time_origin().ev, t.e0) == cudaSuccess)
        timeline.push_back({t.name, double(since), double(since) + double(ms)});
    }
    cudaEventDestroy(t.e0);
    cudaEventDestroy(t.e1);
  }
  pending_.clear();
}

uint8_t* CudaBackend::upload_resident(const uint8_t* data, size_t size) {
  CUDA_CHECK(cudaSetDevice(device_));
  size_t need = ((size + 7) & ~size_t(7)) + 64;
  uint8_t* p = nullptr;
  CUDA_CHECK(cudaMalloc(&p, need));
  CUDA_CHECK(cudaMemset(p, 0, need));
  CUDA_CHECK(cudaMemcpy(p, data, size, cudaMemcpyHostToDevice));
  return p;
}

void CudaBackend::set_codestream(const uint8_t* data, size_t size) {
  CUDA_CHECK(cudaSetDevice(device_));
  stages.clear();  // stage snapshots belong to one decode call
  stage_dims.clear();
  if (!stream_) {  // a new decode call of a pipeline decoder: its LF arena starts empty again
    lf_arena_off_ = 0;
    if (in_lf_arena(d_codestream_)) d_codestream_ = nullptr, codestream_cap_ = 0;
    pending_cs_bytes_ = 0;
  }
  if (resident_next_) {  // encoded bytes already live in HBM (jxlb_preload)
    active_cs_ = resident_next_;
    resident_next_ = nullptr;
    ensure_static_tables();
    return;
  }
  size_t need = ((size + 7) & ~size_t(7)) + 64;  // zero padding for the 64-bit bit reader
  // through pinned memory: a pageable source makes cudaMemcpyAsync stage and wait inside the driver, and with dozens of
  // decoder threads those copies serialise on the driver
  if (need > input_cap_) {
    if (h_input_) CUDA_CHECK(cudaFreeHost(h_input_));
    h_input_ = nullptr;
    input_cap_ = std::max<size_t>(need + need / 2, size_t(1) << 20);
    CUDA_CHECK(cudaHostAlloc(reinterpret_cast<void**>(&h_input_), input_cap_, cudaHostAllocDefault));
  }
  std::memcpy(h_input_, data, size);
  std::memset(h_input_ + size, 0, need - size);
  if (!stream_ && lf_service) {
    // pipeline decoder: the device copy lives in the LF arena and is made by the first LF batch of the frame (or when
    // the decoder gets its stream, whichever comes first)
    if (void* q = lf_arena_alloc(need)) {
      d_codestream_ = static_cast<uint8_t*>(q);
      codestream_cap_ = need;
      pending_cs_bytes_ = need;
      active_cs_ = d_codestream_;
      ensure_static_tables();
      return;
    }
  }
  if (need > codestream_cap_ || in_lf_arena(d_codestream_)) {
    // Stream-ordered (re)allocation with headroom: cudaFree / cudaMalloc wait for the whole device - with dozens of
    // decoders whose frames differ by a few bytes that was hundreds of device-wide stalls per run.
    if (d_codestream_ && !in_lf_arena(d_codestream_)) CUDA_CHECK(cudaFreeAsync(d_codestream_, S()));
    d_codestream_ = nullptr;
    codestream_cap_ = std::max<size_t>(need + need / 2, size_t(1) << 20);
    CUDA_CHECK(cudaMallocFromPoolAsync(reinterpret_cast<void**>(&d_codestream_), codestream_cap_, pool_, S()));
  }
  CUDA_CHECK(cudaMemcpyAsync(d_codestream_, h_input_, need, cudaMemcpyHostToDevice, S()));
  active_cs_ = d_codestream_;
  ensure_static_tables();
}

void CudaBackend::new_frame() {
  heavy_announced_ = false;
  cached_hfg_ = nullptr;
  if (d_dequant_) {
    dfree(d_dequant_);
    d_dequant_ = nullptr;
  }
}

void CudaBackend::ensure_static_tables() {
  if (!d_natural_orders_) {
    const std::vector<uint32_t> all = natural_order_table(natural_order_offset_);
    CUDA_CHECK(cudaMalloc(&d_natural_orders_, all.size() * 4));
    CUDA_CHECK(cudaMemcpy(d_natural_orders_, all.data(), all.size() * 4, cudaMemcpyHostToDevice));
  }
  if (!sec_uploaded_) {
    // sec_half for n = 64, 128, 256 (dct_common.rs:57-67): f32 arithmetic with libm cosf
    float tab[224];
    size_t off = 0;
    for (int i = 0; i < 3; ++i) {
      size_t n = size_t(64) << i;
      for (size_t k = 0; k < n / 2; ++k) {
        float theta = float(2 * k + 1) / float(2 * n) * 3.14159265358979323846f;
        tab[off + k] = (1.0f / cosf(theta)) / 2.0f;
      }
      off += n / 2;
    }
    upload_sec_large(tab);
    sec_uploaded_ = true;
  }
}

int CudaBackend::alloc_plane(uint32_t w, uint32_t h, bool zero) {
  PlaneRec r;
  r.w = w;
  r.h = h;
  size_t bytes = size_t(w) * h * 4;
  r.ptr = dmalloc(bytes);
  if (zero) CUDA_CHECK(cudaMemsetAsync(r.ptr, 0, bytes, S()));
  int id = next_id_++;
  planes_[id] = r;
  return id;
}

void CudaBackend::free_plane(int id) {
  auto it = planes_.find(id);
  if (it == planes_.end()) return;
  dfree(it->second.ptr);
  planes_.erase(it);
}

DevView CudaBackend::dev_view(const View& v) const {
  DevView d;
  d.ptr = nullptr;
  d.stride = 0;
  d.w = v.w;
  d.h = v.h;
  if (v.plane >= 0) {
    const PlaneRec& p = planes_.at(v.plane);
    d.ptr = static_cast<uint32_t*>(p.ptr) + size_t(v.y0) * p.w + v.x0;
    d.stride = p.w;
  }
  return d;
}

void CudaBackend::download_rect(const View& v, void* dst) {
  if (!v.w || !v.h) return;
  DevView d = dev_view(v);
  if (d.stride == v.w)  // contiguous: one linear DMA
    CUDA_CHECK(cudaMemcpyAsync(dst, d.ptr, size_t(v.w) * v.h * 4, cudaMemcpyDeviceToHost, S()));
  else
    CUDA_CHECK(cudaMemcpy2DAsync(dst, size_t(v.w) * 4, d.ptr, size_t(d.stride) * 4, size_t(v.w) * 4, v.h,
                                 cudaMemcpyDeviceToHost, S()));
  sync();
}

void CudaBackend::copy_rect(const View& src, const View& dst) {
  begin_k("copy_rect");
  launch_copy_rect(dev_view(src), dev_view(dst), S());
  end_k();
}

void CudaBackend::phase_mark(const char* name) {
  if (!profile && !host_phases) return;
  const double now = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
  if (name && phase_t0_ >= 0.0) {
    auto& acc = profile_acc[std::string("host:") + name];
    acc.first += 1;
    acc.second += now - phase_t0_;
    if (profile) timeline.push_back({std::string("host:") + name, phase_t0_ - time_origin().host_ms, now - time_origin().host_ms});
  }
  phase_t0_ = now;
}

void CudaBackend::stage_marker(const char* name, const View* views, int n) {
  if (!stop_stage.empty() && stop_stage == name) {
    // stage entry points (jxlb_decode_hf_groups, jxlb_dequant_idct, jxlb_modular_decode_groups): hand the stage's planes
    // to the caller's device buffers and end the decode here
    stop_dims.clear();
    for (int i = 0; i < n; ++i) {
      stop_dims.push_back({views[i].w, views[i].h});
      if (size_t(i) < stop_dst.size() && stop_dst[size_t(i)] && views[i].w && views[i].h) {
        JXLB_CHECK(stop_stride >= views[i].w, kErrInvalidArg, "destination stride smaller than the stage's planes");
        const DevView d = dev_view(views[i]);
        CUDA_CHECK(cudaMemcpy2DAsync(stop_dst[size_t(i)], size_t(stop_stride) * 4, d.ptr, size_t(d.stride) * 4, size_t(views[i].w) * 4,
                                     views[i].h, cudaMemcpyDeviceToDevice, S()));
      }
    }
    sync();
    throw StopDecode();
  }
  if (!capture) return;
  auto& out = stages[name];
  auto& dims = stage_dims[name];
  out.clear();
  dims.clear();
  for (int i = 0; i < n; ++i) {
    std::vector<uint32_t> buf(size_t(views[i].w) * views[i].h);
    download_rect(views[i], buf.data());
    out.push_back(std::move(buf));
    dims.push_back({views[i].w, views[i].h});
  }
}

namespace {
const char* dev_status_message(int s) {
  switch (s) {
    case kDevBadStream: return "invalid entropy-coded stream (ANS final state / LZ77)";
    case kDevOverrun: return "entropy-coded stream reads past the end of its section";
    case kDevInvalid: return "semantic validation of a decoded stream failed";
    case kDevUnsupported: return "chroma subsampling with varblocks larger than 8x8 is not supported";
    default: return "unknown device decode error";
  }
}
}  // namespace

void CudaBackend::decode_modular(std::vector<ModularStreamJob>& jobs) {
  if (jobs.empty()) return;
  ModularLaunch L = build_modular_launch(jobs, [this](const View& v) { return dev_view(v); }, *this);
  for (size_t i = 0; i < jobs.size(); ++i) {
    const ModularLaunch::JobNeeds& n = L.needs[i];
    if (n.wp_scratch_bytes) temps_.push_back(L.jobs[i].wp_scratch = static_cast<int32_t*>(dmalloc(n.wp_scratch_bytes)));
    if (n.lz_window_bytes) temps_.push_back(L.jobs[i].lz_window = static_cast<uint32_t*>(dmalloc(n.lz_window_bytes)));
  }
  const DevModularJob* d_jobs = static_cast<const DevModularJob*>(upload_temp(L.jobs.data(), L.jobs.size() * sizeof(DevModularJob)));
  const DevChannel* d_chans = static_cast<const DevChannel*>(upload_temp(L.channels.data(), L.channels.size() * sizeof(DevChannel)));
  uint64_t* d_end = static_cast<uint64_t*>(stage_scratch(jobs.size() * 8));
  int* d_status = static_cast<int*>(stage_scratch(jobs.size() * 4));
  const DevChannelPlan* d_plans = static_cast<const DevChannelPlan*>(upload_temp(L.plans.data(), L.plans.size() * sizeof(DevChannelPlan)));
  unsigned long long* d_trace = nullptr;
  double host_launch = 0.0;
  if (trace_device) {
    time_origin();
    d_trace = static_cast<unsigned long long*>(dmalloc(jobs.size() * 16));
    temps_.push_back(d_trace);
    host_launch = host_now_ms();
  }
  const uint64_t* end;
  const int* status;
  if (!stream_ && lf_service && !d_trace && jobs.size() <= 2048) {
    // LF stage of a pipeline decoder: the launch joins the batch service's next kernel (several frames' streams in one
    // launch on one of a few batch streams); this thread sleeps until that batch has run. No CUDA stream is held.
    LfBatchItem item;
    if (pending_cs_bytes_) {
      item.up[item.num_up++] = {d_codestream_, h_input_, pending_cs_bytes_};
      pending_cs_bytes_ = 0;
    }
    item.up[item.num_up++] = {d_stage_, h_stage_, stage_off_};
    item.ref.cs = active_cs_;
    item.ref.jobs = d_jobs;
    item.ref.channels = d_chans;
    item.ref.plans = d_plans;
    item.ref.end_bits = d_end;
    item.ref.status = d_status;
    item.num_jobs = int(jobs.size());
    item.smem_bytes = L.smem_bytes;
    item.all_staged = L.all_staged;
    uint8_t* h_end = h_result_;
    uint8_t* h_status = h_result_ + ((jobs.size() * 8 + 15) & ~size_t(15));
    JXLB_CHECK(size_t(h_status - h_result_) + jobs.size() * 4 <= result_cap_, kErrUnsupported, "too many stream jobs in one launch for the result buffer");
    if (profile || ((stage_off_ + 15) & ~size_t(15)) + 4 > stage_cap_) {  // timing wanted (or no room for the counter):
      // results come back after the whole launch, with its event times
      item.down[item.num_down++] = {h_end, d_end, jobs.size() * 8};
      item.down[item.num_down++] = {h_status, d_status, jobs.size() * 4};
    } else {  // the streams write their results straight into the mapped block and count themselves off
      const uint32_t zero = 0;
      item.ref.counter = static_cast<uint32_t*>(upload_temp(&zero, 4));
      item.up[item.num_up - 1].bytes = stage_off_;
      item.ref.end_bits = reinterpret_cast<uint64_t*>(h_end);
      item.ref.status = reinterpret_cast<int*>(h_status);
      item.ref.num_jobs = uint32_t(jobs.size());
      item.ref.done_flag = const_cast<uint32_t*>(h_flag_ + 16);
      item.ref.done_seq = ++item_seq_;
      item.done_flag = h_flag_ + 16;
    }
    item.want_timing = profile;
    lf_service->run(item);
    ++launches;
    if (profile) {
      auto& acc = profile_acc["modular_decode"];
      acc.first += 1;
      acc.second += double(item.elapsed_ms);
    }
    stage_off_ = stage_flushed_ = 0;
    result_off_ = 0;
    end = reinterpret_cast<const uint64_t*>(h_end);
    status = reinterpret_cast<const int*>(h_status);
  } else {
    begin_k("modular_decode");
    launch_modular_decode(active_cs_, d_jobs, d_chans, d_plans, d_end, d_status, int(jobs.size()), L.smem_bytes, L.all_staged, S(), d_trace);
    end_k();
    end = static_cast<const uint64_t*>(fetch_result(d_end, jobs.size() * 8));
    status = static_cast<const int*>(fetch_result(d_status, jobs.size() * 4));
    const unsigned long long* trace = d_trace ? static_cast<const unsigned long long*>(fetch_result(d_trace, jobs.size() * 16)) : nullptr;
    sync();
    if (d_trace) {
      const TimeOrigin& o = time_origin();
      unsigned long long first = ~0ull, last = 0;
      for (size_t i = 0; i < jobs.size(); ++i) {
        first = std::min<unsigned long long>(first, trace[2 * i]);
        last = std::max<unsigned long long>(last, trace[2 * i + 1]);
      }
      timeline.push_back({"host:launch_to_return modular", host_launch - o.host_ms, host_now_ms() - o.host_ms});
      timeline.push_back({"dev:modular_decode", (double(first) - double(o.dev_ns)) * 1e-6, (double(last) - double(o.dev_ns)) * 1e-6});
    }
    CUDA_CHECK(cudaGetLastError());
  }
  release_temps();
  for (size_t i = 0; i < jobs.size(); ++i) {
    if (status[i] != kDevOk)
      fail(status[i] == kDevOverrun ? kErrEof : kErrDeviceDecode,
           std::string("modular stream ") + std::to_string(jobs[i].stream_index) + ": " + dev_status_message(status[i]));
    jobs[i].end_bit = size_t(end[i]);
  }
}

int CudaBackend::squeeze_inverse(const View& avg, const View& res, bool horizontal) {
  uint32_t ow = horizontal ? avg.w + res.w : avg.w;
  uint32_t oh = horizontal ? avg.h : avg.h + res.h;
  JXLB_CHECK(horizontal ? (res.h == avg.h || res.w == 0) : (res.w == avg.w || res.h == 0), kErrBitstream,
             "squeeze residual size mismatch");
  int id = alloc_plane(std::max(ow, 1u), std::max(oh, 1u), false);
  if (!ow || !oh) return id;
  View ov{id, 0, 0, ow, oh};
  begin_k("squeeze_inverse");
  launch_squeeze_inverse(dev_view(avg), dev_view(res), dev_view(ov), horizontal, S());
  end_k();
  return id;
}

std::vector<int> CudaBackend::squeeze_inverse_many(const std::vector<std::pair<View, View>>& avg_res, bool horizontal) {
  std::vector<int> ids;
  std::vector<DevView> a, r, o;
  for (const auto& p : avg_res) {
    const View& avg = p.first;
    const View& res = p.second;
    const uint32_t ow = horizontal ? avg.w + res.w : avg.w, oh = horizontal ? avg.h : avg.h + res.h;
    JXLB_CHECK(horizontal ? (res.h == avg.h || res.w == 0) : (res.w == avg.w || res.h == 0), kErrBitstream,
               "squeeze residual size mismatch");
    const int id = alloc_plane(std::max(ow, 1u), std::max(oh, 1u), false);
    ids.push_back(id);
    if (!ow || !oh) continue;
    a.push_back(dev_view(avg));
    r.push_back(dev_view(res));
    o.push_back(dev_view(View{id, 0, 0, ow, oh}));
  }
  if (!o.empty()) {
    begin_k("squeeze_inverse");
    launch_squeeze_inverse_batch(a.data(), r.data(), o.data(), int(o.size()), horizontal, S());
    end_k();
  }
  return ids;
}

void CudaBackend::rct_inverse(const View v[3], uint32_t rct_type) {
  begin_k("rct_inverse");
  launch_rct_inverse(dev_view(v[0]), dev_view(v[1]), dev_view(v[2]), rct_type, S());
  end_k();
}

void CudaBackend::palette_inverse(const View& palette, const std::vector<View>& targets, const Transform& t,
                                  const WpHeader& wph, uint32_t bit_depth) {
  JXLB_CHECK(targets.size() <= size_t(kMaxPaletteChannels), kErrUnsupported, "palettes with more than 16 channels are not implemented on the device");
  DevView tv[kMaxPaletteChannels];
  for (size_t i = 0; i < targets.size(); ++i) tv[i] = dev_view(targets[i]);
  const uint32_t w = targets[0].w, h = targets[0].h;
  int* d_status = static_cast<int*>(dmalloc(4));
  uint8_t* d_mask = static_cast<uint8_t*>(dmalloc(size_t(w) * h));
  CUDA_CHECK(cudaMemsetAsync(d_status, 0, 4, S()));
  DevView pal{};
  if (palette.plane >= 0) pal = dev_view(palette);  // absent when nb_colours == 0
  begin_k("palette_inverse");
  launch_palette_inverse(pal, tv, int(targets.size()), int(t.nb_colours), int(bit_depth), int(t.nb_deltas), d_mask, d_status, S());
  end_k();
  const int* num_delta_p = static_cast<const int*>(fetch_result(d_status, 4));
  sync();
  const int num_delta = *num_delta_p;
  if (num_delta > 0) {  // palette.rs:114-152
    JXLB_CHECK(t.d_pred <= 13, kErrBitstream, "invalid delta-palette predictor");
    DevPaletteDeltaParams p;
    std::memset(&p, 0, sizeof(p));
    for (size_t i = 0; i < targets.size(); ++i) p.target[i] = tv[i];
    p.mask = d_mask;
    p.d_pred = t.d_pred;
    pack_wp(wph, p.wp);
    int32_t* rows = nullptr;
    if (t.d_pred == 6) rows = static_cast<int32_t*>(dmalloc(targets.size() * ((5 * size_t(w) + 3) & ~size_t(3)) * 4));
    p.wp_rows = rows;
    begin_k("palette_delta");
    launch_palette_delta(p, int(targets.size()), S());
    end_k();
    sync();
    if (rows) dfree(rows);
  }
  dfree(d_status);
  dfree(d_mask);
}

void CudaBackend::int_to_float(const View& v, const BitDepth& d) {
  begin_k("int_to_float");
  launch_int_to_float(dev_view(v), d.bits_per_sample, d.exp_bits, d.float_sample, S());
  end_k();
}

void CudaBackend::modular_xyb_to_float(const View yxb[3], const float m[3]) {
  begin_k("modular_xyb");
  launch_modular_xyb(dev_view(yxb[0]), dev_view(yxb[1]), dev_view(yxb[2]), m[0], m[1], m[2], S());
  end_k();
}

void CudaBackend::build_block_info(VarDctState& st, const std::vector<BlockInfoJob>& jobs) {
  if (jobs.empty()) return;
  std::vector<DevBlockInfoJob> dj;
  for (const BlockInfoJob& j : jobs) {
    const PlaneRec& raw = planes_.at(j.raw_plane);
    dj.push_back({{j.rect.bx0, j.rect.by0, j.rect.bw, j.rect.bh}, static_cast<const int32_t*>(raw.ptr), raw.w, j.nb_blocks});
  }
  const EpfParams& epf = st.fh->restoration_filter.epf;
  const DevBlockInfoJob* d_jobs = static_cast<const DevBlockInfoJob*>(upload_temp(dj.data(), dj.size() * sizeof(DevBlockInfoJob)));
  const float* d_lut = static_cast<const float*>(upload_temp(epf.sharp_lut, sizeof(epf.sharp_lut)));
  int* d_status = static_cast<int*>(stage_scratch(jobs.size() * 4));
  float quant_mul_base = epf.quant_mul * 65536.0f / float(st.lfg->global_scale);
  begin_k("build_block_info");
  void* scratch = dmalloc(build_block_info_scratch_bytes(int(jobs.size())));
  temps_.push_back(scratch);
  launch_build_block_info(dev_frame(st), d_jobs, int(jobs.size()), quant_mul_base, d_lut, epf.iters > 0 ? 1 : 0, d_status,
                          scratch, S());
  end_k();
  const int* status = static_cast<const int*>(fetch_result(d_status, jobs.size() * 4));
  sync();
  CUDA_CHECK(cudaGetLastError());
  release_temps();
  for (size_t i = 0; i < jobs.size(); ++i) JXLB_CHECK(status[i] == kDevOk, kErrBitstream, "invalid HfMetadata block layout");
}

void CudaBackend::decode_hf(VarDctState& st, std::vector<HfGroupJob>& jobs) {
  if (jobs.empty()) return;
  const uint32_t pass = jobs[0].pass_idx;
  const HfPassSyntax& hp = st.hfg->passes[pass];
  // The coefficient kernels read plain hybrid-uint tokens; an LZ77-enabled HF code (legal, hf_coeff.rs:181-222 goes
  // through read_varint_with_multiplier_clustered, but no known encoder emits it) would decode silently wrong.
  const bool hf_lz77 = hp.code.lz77_enabled;  // reported after the launch: a stream that is invalid anyway keeps its own error
  const DevHfParams p = build_hf_params(st, pass, *this, d_natural_orders_, natural_order_offset_);
  const HfSchedule sched = hf_schedule(p, hf_streams_per_cta);
  const std::vector<uint32_t> perm = hf_launch_order(jobs, sched.lanes);  // launch order -> `jobs`
  std::vector<DevHfJob> dj;
  for (uint32_t i : perm) dj.push_back({jobs[i].bit_pos, jobs[i].bit_limit, jobs[i].group_idx});
  const DevHfJob* d_jobs = static_cast<const DevHfJob*>(upload_temp(dj.data(), dj.size() * sizeof(DevHfJob)));
  uint64_t* d_end = static_cast<uint64_t*>(stage_scratch(jobs.size() * 8));
  int* d_status = static_cast<int*>(stage_scratch(jobs.size() * 4));
  uint32_t* d_blk_ctx = nullptr;
  if (sched.lanes) {
    d_blk_ctx = static_cast<uint32_t*>(dmalloc(size_t(st.bw) * st.bh * 4));
    temps_.push_back(d_blk_ctx);
    begin_k("hf_block_ctx");
    launch_hf_block_ctx(dev_frame(st), p, d_blk_ctx, S());
    end_k();
  }
  begin_k("decode_hf");
  if (sched.lanes)
    launch_decode_hf_lanes(active_cs_, dev_frame(st), p, d_blk_ctx, d_jobs, d_end, d_status, int(jobs.size()), pass == 0 ? 1 : 0,
                           sched.per_cta, S());
  else
    launch_decode_hf(active_cs_, dev_frame(st), p, d_jobs, d_end, d_status, int(jobs.size()), pass == 0 ? 1 : 0,
                     sched.per_cta, S());
  end_k();
  const uint64_t* end = static_cast<const uint64_t*>(fetch_result(d_end, jobs.size() * 8));
  const int* status = static_cast<const int*>(fetch_result(d_status, jobs.size() * 4));
  sync();
  CUDA_CHECK(cudaGetLastError());
  release_temps();
  for (size_t i = 0; i < jobs.size(); ++i) {
    HfGroupJob& job = jobs[perm[i]];
    if (status[i] != kDevOk)
      fail(status[i] == kDevOverrun ? kErrEof : (status[i] == kDevUnsupported ? kErrUnsupported : kErrDeviceDecode),
           std::string("HF group ") + std::to_string(job.group_idx) + ": " + dev_status_message(status[i]));
    job.end_bit = size_t(end[i]);
  }
  JXLB_CHECK(!hf_lz77, kErrUnsupported, "LZ77 in the HF coefficient streams is not supported on the device");
}

void CudaBackend::lf_dequant(VarDctState& st, const std::vector<LfDequantJob>& jobs) {
  std::vector<DevLfDequantJob> dj;
  for (const LfDequantJob& j : jobs)
    dj.push_back({{j.rect.bx0, j.rect.by0, j.rect.bw, j.rect.bh}, {j.scale[0], j.scale[1], j.scale[2]}});
  const DevLfDequantJob* d = static_cast<const DevLfDequantJob*>(upload_temp(dj.data(), dj.size() * sizeof(DevLfDequantJob)));
  begin_k("lf_dequant");
  launch_lf_dequant(dev_frame(st), d, int(dj.size()), S());
  end_k();
}

void CudaBackend::lf_chroma_from_luma(VarDctState& st) {
  const LfGlobalSyntax& g = *st.lfg;
  int32_t x_factor = int32_t(g.x_factor_lf) - 128, b_factor = int32_t(g.b_factor_lf) - 128;
  float kx = g.base_correlation_x + (float(x_factor) / float(g.colour_factor));
  float kb = g.base_correlation_b + (float(b_factor) / float(g.colour_factor));
  begin_k("lf_cfl");
  launch_lf_cfl(dev_frame(st), kx, kb, S());
  end_k();
}

void CudaBackend::lf_adaptive_smoothing(VarDctState& st) {
  const LfGlobalSyntax& g = *st.lfg;
  uint64_t scale_inv = uint64_t(g.global_scale) * g.quant_lf;
  float lf_x = float(512.0 * double(g.m_x_lf) / double(scale_inv));
  float lf_y = float(512.0 * double(g.m_y_lf) / double(scale_inv));
  float lf_b = float(512.0 * double(g.m_b_lf) / double(scale_inv));
  float* tmp[3];
  for (int c = 0; c < 3; ++c) tmp[c] = static_cast<float*>(dmalloc(size_t(st.bw) * st.bh * 4));
  begin_k("lf_smooth");
  launch_lf_smooth(dev_frame(st), tmp, lf_x, lf_y, lf_b, S());
  end_k();
  for (int c = 0; c < 3; ++c) {  // swap the smoothed planes in
    PlaneRec& r = planes_.at(st.lf[c]);
    dfree(r.ptr);
    r.ptr = tmp[c];
  }
}

void CudaBackend::hf_dequant_cfl(VarDctState& st) {
  const bool use_default = st.hfg->dequant_all_default;
  if (use_default ? d_dequant_default_ == nullptr : cached_hfg_ != st.hfg) {
    std::vector<float> all;
    DevDequantParams& dp = use_default ? dequant_default_params_ : dequant_params_;
    std::memset(&dp, 0, sizeof(dp));
    for (int set = 0; set < 17; ++set)
      for (int c = 0; c < 3; ++c)
        for (int tr = 0; tr < 2; ++tr) {
          const std::vector<float>& m = tr ? st.hfg->dequant->matrices_tr[set][c] : st.hfg->dequant->matrices[set][c];
          dp.matrix_offset[(set * 3 + c) * 2 + tr] = uint32_t(all.size());
          all.insert(all.end(), m.begin(), m.end());
        }
    if (use_default) {
      CUDA_CHECK(cudaMalloc(&d_dequant_default_, all.size() * 4));
      CUDA_CHECK(cudaMemcpyAsync(d_dequant_default_, all.data(), all.size() * 4, cudaMemcpyHostToDevice, S()));
      CUDA_CHECK(cudaStreamSynchronize(S()));
    } else {
      if (d_dequant_) dfree(d_dequant_);
      d_dequant_ = static_cast<float*>(dmalloc(all.size() * 4));
      CUDA_CHECK(cudaMemcpyAsync(d_dequant_, all.data(), all.size() * 4, cudaMemcpyHostToDevice, S()));
      cached_hfg_ = st.hfg;
    }
  }
  DevDequantParams p = use_default ? dequant_default_params_ : dequant_params_;
  p.matrices = use_default ? d_dequant_default_ : d_dequant_;
  const OpsinInverseMatrix& oim = st.ih->opsin_inverse_matrix;
  for (int c = 0; c < 3; ++c) p.quant_bias[c] = oim.quant_bias[c];
  p.quant_bias_numerator = oim.quant_bias_numerator;
  p.qm_scale[0] = powi_f32(0.8f, int32_t(st.fh->x_qm_scale) - 2);
  p.qm_scale[1] = 1.0f;
  p.qm_scale[2] = powi_f32(0.8f, int32_t(st.fh->b_qm_scale) - 2);
  p.global_scale = float(st.lfg->global_scale);
  p.base_correlation_x = st.lfg->base_correlation_x;
  p.base_correlation_b = st.lfg->base_correlation_b;
  p.colour_factor = float(st.lfg->colour_factor);
  // Production path: dequantisation + chroma from luma run inside the inverse transforms' load stage (hf_transform), which
  // saves one HBM round trip of the three coefficient planes. The separate kernel remains for stage snapshots (tests
  // compare the "hf_dequant" planes) and for chroma-subsampled frames (per-channel grids, no chroma from luma).
  if (!capture && !st.subsampled && fuse_dequant) {
    pending_dequant_ = p;
    have_pending_dequant_ = true;
    return;
  }
  begin_k("hf_dequant_cfl");
  launch_hf_dequant_cfl(dev_frame(st), p, S());
  end_k();
}

void CudaBackend::hf_transform(VarDctState& st) {
  void* scratch = dmalloc(hf_transform_scratch_bytes(st.bw, st.bh));
  begin_k("hf_transform");
  launch_hf_transform(dev_frame(st), scratch, have_pending_dequant_ ? &pending_dequant_ : nullptr, S());
  end_k();
  have_pending_dequant_ = false;
  dfree(scratch);
}

void CudaBackend::gaborish(const View v[3], const float weights[3][2]) {
  for (int c = 0; c < 3; ++c) {
    PlaneRec& r = planes_.at(v[c].plane);
    JXLB_CHECK(v[c].x0 == 0 && v[c].y0 == 0, kErrInvalidArg, "gaborish expects a top-left anchored view");
    void* out = dmalloc(size_t(r.w) * r.h * 4);
    DevView in = dev_view(v[c]);
    DevView ov = in;
    ov.ptr = out;
    begin_k("gaborish");
    launch_gaborish(in, ov, weights[c][0], weights[c][1], S());
    end_k();
    dfree(r.ptr);
    r.ptr = out;
  }
}

void CudaBackend::epf(const View v[3], const View& sigma, const EpfParams& p, bool sigma_is_constant) {
  DevView cur[3], alt[3];
  void* alt_ptr[3];
  for (int c = 0; c < 3; ++c) {
    PlaneRec& r = planes_.at(v[c].plane);
    JXLB_CHECK(v[c].x0 == 0 && v[c].y0 == 0, kErrInvalidArg, "epf expects a top-left anchored view");
    alt_ptr[c] = dmalloc(size_t(r.w) * r.h * 4);
    cur[c] = dev_view(v[c]);
    alt[c] = cur[c];
    alt[c].ptr = alt_ptr[c];
  }
  const float* d_sigma = nullptr;
  uint32_t sigma_stride = 0;
  if (!sigma_is_constant) {
    const PlaneRec& s = planes_.at(sigma.plane);
    d_sigma = static_cast<const float*>(s.ptr);
    sigma_stride = s.w;
  }
  DevEpfParams dp;
  for (int c = 0; c < 3; ++c) dp.channel_scale[c] = p.channel_scale[c];
  dp.pass0_sigma_scale = p.pass0_sigma_scale;
  dp.pass2_sigma_scale = p.pass2_sigma_scale;
  dp.border_sad_mul = p.border_sad_mul;
  dp.sigma_for_modular = p.sigma_for_modular;
  bool in_alt = false;
  auto run = [&](int step) {
    begin_k("epf_step");
    launch_epf_step(in_alt ? alt : cur, in_alt ? cur : alt, d_sigma, sigma_stride, dp, step, S());
    end_k();
    in_alt = !in_alt;
  };
  if (p.iters == 3) run(0);
  run(1);
  if (p.iters >= 2) run(2);
  for (int c = 0; c < 3; ++c) {
    PlaneRec& r = planes_.at(v[c].plane);
    if (in_alt) {
      dfree(r.ptr);
      r.ptr = alt_ptr[c];
    } else {
      dfree(alt_ptr[c]);
    }
  }
}

bool CudaBackend::filters_colour_fused(const View v[3], const RestorationFilter& rf, const View& sigma,
                                       bool sigma_is_constant, const ColorParams* colour) {
  if (!fuse_filters || !fused_filters_supported(v[0].w, v[0].h)) return false;
  DevView in[3], out[3];
  void* out_ptr[3];
  for (int c = 0; c < 3; ++c) {
    PlaneRec& r = planes_.at(v[c].plane);
    JXLB_CHECK(v[c].x0 == 0 && v[c].y0 == 0, kErrInvalidArg, "filters expect top-left anchored views");
    out_ptr[c] = dmalloc(size_t(r.w) * r.h * 4);
    in[c] = dev_view(v[c]);
    out[c] = in[c];
    out[c].ptr = out_ptr[c];
  }
  const float* d_sigma = nullptr;
  uint32_t sigma_stride = 0;
  if (!sigma_is_constant && rf.epf.iters > 0) {
    const PlaneRec& s = planes_.at(sigma.plane);
    d_sigma = static_cast<const float*>(s.ptr);
    sigma_stride = s.w;
  }
  JXLB_CHECK(!colour || (!colour->second_stage && colour->gamma == 0.0f), kErrInvalidArg,
             "the fused filter kernel converts to sRGB-gamut targets only");
  const DevFusedFilterParams p = fused_filter_params(rf, d_sigma, sigma_stride, colour);
  begin_k("filters_fused");
  launch_filters_fused(in, out, p, S());
  end_k();
  for (int c = 0; c < 3; ++c) {
    PlaneRec& r = planes_.at(v[c].plane);
    dfree(r.ptr);
    r.ptr = out_ptr[c];
  }
  return true;
}

void CudaBackend::blend_patches(const std::vector<PatchJob>& jobs) {
  // Patches may overlap; samples must then be updated in list order. Jobs are cut into launches such that
  // no two jobs of one launch touch the same plane rectangle.
  std::vector<DevPatchJob> batch;
  std::vector<const PatchJob*> members;
  auto flush = [&] {
    if (batch.empty()) return;
    const DevPatchJob* d = static_cast<const DevPatchJob*>(upload_temp(batch.data(), batch.size() * sizeof(DevPatchJob)));
    begin_k("blend_patches");
    launch_blend_patches(d, int(batch.size()), S());
    end_k();
    batch.clear();
    members.clear();
  };
  auto overlaps = [](const View& a, const View& b) {
    return a.plane == b.plane && a.x0 < b.x0 + b.w && b.x0 < a.x0 + a.w && a.y0 < b.y0 + b.h && b.y0 < a.y0 + a.h;
  };
  for (const PatchJob& j : jobs) {
    if (!j.dst.w || !j.dst.h) continue;
    bool clash = false;
    for (const PatchJob* m : members)
      if (overlaps(m->dst, j.dst) || (j.base_alpha.plane >= 0 && overlaps(m->dst, j.base_alpha)) ||
          (j.new_alpha.plane >= 0 && overlaps(m->dst, j.new_alpha)) ||
          (m->base_alpha.plane >= 0 && overlaps(j.dst, m->base_alpha)) ||
          (m->new_alpha.plane >= 0 && overlaps(j.dst, m->new_alpha))) {
        clash = true;
        break;
      }
    if (clash || batch.size() >= 4096) flush();
    DevView s = dev_view(j.src), d = dev_view(j.dst), ba = dev_view(j.base_alpha), na = dev_view(j.new_alpha);
    batch.push_back({static_cast<const float*>(s.ptr), static_cast<float*>(d.ptr), static_cast<const float*>(ba.ptr),
                     static_cast<const float*>(na.ptr), s.stride, d.stride, ba.stride, na.stride, j.dst.w, j.dst.h, j.mode,
                     j.clamp ? 1u : 0u, j.premultiplied ? 1u : 0u, j.swapped ? 1u : 0u});
    members.push_back(&j);
  }
  flush();
}

void CudaBackend::blend_raw(const DevPatchJob& job) {
  const DevPatchJob* d = static_cast<const DevPatchJob*>(upload_temp(&job, sizeof(job)));
  begin_k("blend_patches");
  launch_blend_patches(d, 1, S());
  end_k();
  sync();
  release_temps();
}

void CudaBackend::splat_splines(const View v[3], const std::vector<SplineArc>& arcs) {
  if (arcs.empty()) return;
  static_assert(sizeof(SplineArc) == sizeof(DevSplineArc), "arc layouts must agree");
  DevView dv[3] = {dev_view(v[0]), dev_view(v[1]), dev_view(v[2])};
  const DevSplineArc* d = static_cast<const DevSplineArc*>(upload_temp(arcs.data(), arcs.size() * sizeof(SplineArc)));
  begin_k("splat_splines");
  launch_splat_splines(dv, d, int(arcs.size()), S());
  end_k();
}

void CudaBackend::add_noise(const View v[3], const float lut[8], uint32_t group_dim, uint64_t seed0, float corr_x,
                            float corr_b) {
  JXLB_CHECK(v[0].w >= 2 && v[0].h >= 2, kErrUnsupported, "noise on frames narrower than 2 samples is not supported");
  DevView dv[3];
  float* field[3];
  for (int c = 0; c < 3; ++c) {
    JXLB_CHECK(v[c].w == v[0].w && v[c].h == v[0].h, kErrInvalidArg, "noise needs three equally sized planes");
    dv[c] = dev_view(v[c]);
    field[c] = static_cast<float*>(dmalloc(size_t(v[0].w) * v[0].h * 4));
  }
  DevNoiseParams p;
  for (int i = 0; i < 8; ++i) p.lut[i] = lut[i];
  p.lut[8] = lut[7];
  p.corr_x = corr_x;
  p.corr_b = corr_b;
  p.group_dim = group_dim;
  p.seed0 = seed0;
  begin_k("add_noise");
  launch_add_noise(dv, field, p, S());
  end_k();
  for (int c = 0; c < 3; ++c) dfree(field[c]);
}

void CudaBackend::pack_to_host(const DevPackParams& p, void* dst, size_t bytes) {
  void* d = dmalloc(bytes);
  begin_k("pack_interleaved");
  launch_pack_interleaved(p, d, S());
  end_k();
  CUDA_CHECK(cudaMemcpyAsync(dst, d, bytes, cudaMemcpyDeviceToHost, S()));
  sync();
  dfree(d);
}

void CudaBackend::pack_to_device(const DevPackParams& p, void* d_dst) {
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, d_dst) != cudaSuccess || attr.type != cudaMemoryTypeDevice || attr.device != device_) {
    cudaGetLastError();
    fail(kErrInvalidArg, "destination is not device memory of this decoder's GPU");
  }
  begin_k("pack_interleaved");
  launch_pack_interleaved(p, d_dst, S());
  end_k();
  sync();  // the caller may hand the buffer to any stream (NCCL's, torch's) afterwards
}

int CudaBackend::upsample(const View& v, uint32_t factor_log2, const ImageHeader& ih) {
  DevView cur = dev_view(v);
  void* cur_owned = nullptr;
  uint32_t w = v.w, h = v.h;
  auto pass = [&](uint32_t k, const std::vector<float>& weights) {
    // per-phase 5x5 kernels from the symmetric weight list (upsampling.rs:66-92)
    const uint32_t mat_n = k / 2;
    std::vector<float> quarter(size_t(k) * k / 4 * 25, 0.0f);
    size_t weight_idx = 0;
    for (uint32_t y = 0; y < 5 * mat_n; ++y) {
      const uint32_t mat_y = y / 5, ky = y % 5;
      for (uint32_t x = y; x < 5 * mat_n; ++x) {
        const uint32_t mat_x = x / 5, kx = x % 5;
        const float wv = weights[weight_idx++];
        quarter[size_t(mat_y * mat_n + mat_x) * 25 + ky * 5 + kx] = wv;
        quarter[size_t(mat_x * mat_n + mat_y) * 25 + kx * 5 + ky] = wv;
      }
    }
    const float* d_quarter = static_cast<const float*>(upload_temp(quarter.data(), quarter.size() * 4));
    DevView out;
    out.w = w * k;
    out.h = h * k;
    out.stride = out.w;
    out.ptr = dmalloc(size_t(out.w) * out.h * 4);
    begin_k("upsample");
    launch_upsample(cur, out, int(k), d_quarter, S());
    end_k();
    if (cur_owned) dfree(cur_owned);
    cur = out;
    cur_owned = out.ptr;
    w *= k;
    h *= k;
  };
  for (uint32_t i = 0; i < factor_log2 / 3; ++i) pass(8, ih.up8_weight);
  if (factor_log2 % 3 == 1) pass(2, ih.up2_weight);
  if (factor_log2 % 3 == 2) pass(4, ih.up4_weight);
  JXLB_CHECK(cur_owned != nullptr, kErrInvalidArg, "upsample called with factor 1");
  PlaneRec r;
  r.w = w;
  r.h = h;
  r.ptr = cur_owned;
  int id = next_id_++;
  planes_[id] = r;
  return id;
}

int CudaBackend::upsample_jpeg(const View& v, bool horizontal, bool vertical, uint32_t out_w, uint32_t out_h) {
  const int id = alloc_plane(out_w, out_h, false);
  begin_k("upsample_jpeg");
  launch_upsample_jpeg(dev_view(v), dev_view(View{id, 0, 0, out_w, out_h}), horizontal ? 1 : 0, vertical ? 1 : 0, S());
  end_k();
  return id;
}

void CudaBackend::ycbcr_to_rgb(const View v[3], const YcbcrParams& p) {
  const DevYcbcrParams d{p.y_offset, p.cr_to_r, p.cb_to_g, p.cr_to_g, p.cb_to_b};
  begin_k("ycbcr_to_rgb");
  launch_ycbcr_to_rgb(dev_view(v[0]), dev_view(v[1]), dev_view(v[2]), d, S());
  end_k();
}

void CudaBackend::xyb_to_rgb(const View v[3], const ColorParams& p) {
  DevColorParams d{};
  for (int i = 0; i < 3; ++i) {
    d.opsin_bias[i] = p.opsin_bias[i];
    d.cbrt_opsin_bias[i] = p.cbrt_opsin_bias[i];
  }
  d.itscale = p.itscale;
  for (int i = 0; i < 9; ++i) d.matrix[i] = p.matrix[i];
  d.apply_srgb_tf = p.apply_srgb_tf ? 1 : 0;
  d.apply_bt709_tf = p.apply_bt709_tf ? 1 : 0;
  d.second_stage = p.second_stage ? 1 : 0;
  d.to_luma = p.to_luma ? 1 : 0;
  for (int i = 0; i < 3; ++i) d.luminances[i] = p.luminances[i];
  for (int i = 0; i < 9; ++i) d.matrix2[i] = p.matrix2[i];
  d.gamma = p.gamma;
  d.pq_intensity_target = p.pq_intensity_target;
  begin_k("xyb_to_rgb");
  launch_xyb_to_rgb(dev_view(v[0]), dev_view(v[1]), dev_view(v[2]), d, S());
  end_k();
}

}  // namespace jxlb
