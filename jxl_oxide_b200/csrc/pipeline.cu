// Frame pipeline: N decoder contexts (one CUDA stream + one host thread each) fed from one queue, the in-library
// counterpart of the reference's frame-level concurrency (jxl-oxide-cli renders keyframes with rayon's par_iter,
// crates/jxl-oxide-cli/src/decode.rs:285-320; jxl-render spawns reference / LF frames eagerly, lib.rs:496-509).
//
// Why it lives below the C ABI: a JPEG XL frame spends most of its latency in a handful of strictly serial entropy
// streams (LfCoeff + HfMetadata of every 2048x2048 LF group, ~0.1 s for an 8K frame) that occupy a few warps, and
// only a few milliseconds in kernels that fill the GPU. Throughput therefore needs many frames in flight, but a
// frame past its LF stage holds ~25 bytes per pixel of planes. The pipeline separates the two: `workers` frames may be
// anywhere, at most `heavy_frames` of them past Backend::begin_heavy_stage(); each heavy slot owns a pre-allocated
// slab the full-resolution planes are carved from, so a frame costs no allocator call. HBM use grows with both counts:
// heavy_frames x slab, and per worker its LF arena and the memory pool of its decoder (which keeps what it held). Frames flow without barriers, so the contexts de-phase by themselves and
// the GPU-filling stages of some frames overlap the latency-bound stages of others.
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <deque>
#include <fstream>
#include <mutex>
#include <sstream>
#include <thread>

#include <pthread.h>
#include <sched.h>

#include "capi_internal.h"

using namespace jxlb;

namespace {

struct Job {
  const uint8_t* data = nullptr;  // host bytes (caller keeps them alive until the job is reported done) or
  size_t size = 0;
  int32_t slot = -1;              // a preloaded slot
  int32_t out_mode = 0;
  void* dst = nullptr;
  size_t dst_bytes = 0;
  uint64_t tag = 0;
};

struct Done {
  uint64_t tag;
  int32_t status;
  std::string error;
  void* out = nullptr;  // pipeline-owned pinned buffer (jobs submitted with dst == NULL), else the job's dst
  size_t out_bytes = 0;
};

struct HostBuf {  // pinned staging owned by the pipeline: allocated by a worker thread (NUMA-local to the GPU)
  void* p = nullptr;
  size_t bytes = 0;
  bool busy = false;
};

struct Resident {
  std::vector<uint8_t> codestream;
  uint8_t* dptr = nullptr;
};

struct Slab {  // a heavy slot: HBM for a frame's full-resolution planes + the CUDA stream its kernels run on
  void* base = nullptr;
  size_t bytes = 0;
  bool busy = false;
  cudaStream_t stream = nullptr;
};

// LF batch service: the Modular launches of every frame's LF stage (LfCoeff, HfMetadata: long kernels of a dozen one-lane
// warps) ride in shared kernels on a few batch streams. A frame in its LF stage therefore holds no CUDA stream
// and any number of frames can be in flight; the device's 32 hardware queues are left to the batch streams and the heavy
// slots. One service thread: it launches whatever is pending whenever a batch stream is free (so batches grow by
// themselves under load), polls the mapped completion words of the batches in flight and wakes the frames' threads.
class BatchService : public LfBatchService {
 public:
  BatchService(int device, int num_streams) : device_(device) {
    cudaSetDevice(device_);
    for (int i = 0; i < num_streams; ++i) {
      Batch b;
      cudaStreamCreateWithFlags(&b.stream, cudaStreamNonBlocking);
      cudaHostAlloc(reinterpret_cast<void**>(&b.h_refs), kMaxRefs * sizeof(DevModularBatchRef), cudaHostAllocDefault);
      cudaMalloc(reinterpret_cast<void**>(&b.d_refs), kMaxRefs * sizeof(DevModularBatchRef));
      void* f = nullptr;
      cudaHostAlloc(&f, 64, cudaHostAllocMapped);
      b.flag = static_cast<volatile uint32_t*>(f);
      *b.flag = 0;
      cudaEventCreate(&b.e0);
      cudaEventCreate(&b.e1);
      batches_.push_back(b);
    }
    thread_ = std::thread([this] { loop(); });
  }
  ~BatchService() override {
    {
      std::lock_guard<std::mutex> lk(mu_);
      stop_ = true;
    }
    cv_pending_.notify_all();
    thread_.join();
    cudaSetDevice(device_);
    for (Batch& b : batches_) {
      cudaStreamSynchronize(b.stream);
      cudaStreamDestroy(b.stream);
      cudaFreeHost(b.h_refs);
      cudaFree(b.d_refs);
      cudaFreeHost(const_cast<uint32_t*>(b.flag));
      cudaEventDestroy(b.e0);
      cudaEventDestroy(b.e1);
    }
  }
  void run(LfBatchItem& item) override {
    Waiter w;
    w.item = &item;
    {
      std::lock_guard<std::mutex> lk(mu_);
      pending_.push_back(&w);
    }
    cv_pending_.notify_one();
    std::unique_lock<std::mutex> lk(mu_);
    w.cv.wait(lk, [&] { return w.done; });
    if (w.error != cudaSuccess) fail(kErrCuda, std::string("CUDA error in the LF batch: ") + cudaGetErrorString(w.error));
  }
  uint64_t launches() const { return launches_; }
  uint64_t items() const { return items_; }

 private:
  static constexpr int kMaxRefs = 4096;
  struct Waiter {
    LfBatchItem* item = nullptr;
    bool done = false;
    cudaError_t error = cudaSuccess;
    std::condition_variable cv;
  };
  struct Batch {
    cudaStream_t stream = nullptr;
    DevModularBatchRef* h_refs = nullptr;
    DevModularBatchRef* d_refs = nullptr;
    volatile uint32_t* flag = nullptr;
    uint32_t seq = 0;
    bool busy = false;
    bool timed = false;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    std::vector<Waiter*> riders;
    std::chrono::steady_clock::time_point t0, t_launch;
  };

  void finish(Batch& b, cudaError_t err) {
    float ms = 0.0f;
    if (b.timed && err == cudaSuccess) cudaEventElapsedTime(&ms, b.e0, b.e1);
    {
      std::lock_guard<std::mutex> lk(mu_);
      for (Waiter* w : b.riders) {  // those not woken by their own completion word
        w->item->elapsed_ms = ms;
        w->error = err;
        w->done = true;
        w->cv.notify_one();
      }
    }
    b.riders.clear();
    b.busy = false;
  }
  // Riders whose own streams have all finished leave without waiting for the rest of the launch.
  void wake_finished(Batch& b) {
    size_t keep = 0;
    for (size_t i = 0; i < b.riders.size(); ++i) {
      Waiter* w = b.riders[i];
      const LfBatchItem& it = *w->item;
      if (it.done_flag && *it.done_flag == it.ref.done_seq) {
        std::atomic_thread_fence(std::memory_order_acquire);
        std::lock_guard<std::mutex> lk(mu_);
        w->done = true;
        w->cv.notify_one();  // `w` lives on its thread's stack: not touched after this
      } else {
        b.riders[keep++] = w;
      }
    }
    b.riders.resize(keep);
  }

  void launch(Batch& b, std::vector<Waiter*>& take) {
    cudaError_t err = cudaSuccess;
    auto chk = [&](cudaError_t e) {
      if (err == cudaSuccess && e != cudaSuccess) err = e;
    };
    int total = 0;
    size_t smem = 0;
    bool all_staged = true, timed = false;
    for (Waiter* w : take) {
      LfBatchItem& it = *w->item;
      for (int i = 0; i < it.num_up; ++i)
        if (it.up[i].bytes) chk(cudaMemcpyAsync(it.up[i].dst, it.up[i].src, it.up[i].bytes, cudaMemcpyHostToDevice, b.stream));
      for (int j = 0; j < it.num_jobs; ++j) {
        DevModularBatchRef r = it.ref;
        r.job = uint32_t(j);
        b.h_refs[total++] = r;
      }
      smem = std::max(smem, it.smem_bytes);
      all_staged = all_staged && it.all_staged;
      timed = timed || it.want_timing;
    }
    chk(cudaMemcpyAsync(b.d_refs, b.h_refs, size_t(total) * sizeof(DevModularBatchRef), cudaMemcpyHostToDevice, b.stream));
    if (timed) chk(cudaEventRecord(b.e0, b.stream));
    launch_modular_decode_batch(b.d_refs, total, smem, all_staged, b.stream);
    chk(cudaGetLastError());
    if (timed) chk(cudaEventRecord(b.e1, b.stream));
    for (Waiter* w : take) {
      LfBatchItem& it = *w->item;
      for (int i = 0; i < it.num_down; ++i)
        if (it.down[i].bytes) chk(cudaMemcpyAsync(it.down[i].dst, it.down[i].src, it.down[i].bytes, cudaMemcpyDeviceToHost, b.stream));
    }
    b.seq += 1;
    launch_signal_word(const_cast<uint32_t*>(b.flag), b.seq, b.stream);
    chk(cudaGetLastError());
    b.riders = take;
    b.busy = true;
    b.timed = timed;
    b.t0 = b.t_launch = std::chrono::steady_clock::now();
    ++launches_;
    items_ += take.size();
    if (err != cudaSuccess) {  // nothing useful is in flight: report to the riders right away
      cudaStreamSynchronize(b.stream);
      finish(b, err);
    }
  }

  void loop() {
    cudaSetDevice(device_);
    for (;;) {
      // completions
      bool any_busy = false;
      for (Batch& b : batches_) {
        if (!b.busy) continue;
        wake_finished(b);
        if (*b.flag == b.seq) {
          std::atomic_thread_fence(std::memory_order_acquire);
          const double ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - b.t_launch).count();
          ema_batch_ms_ = ema_batch_ms_ == 0.0 ? ms : 0.8 * ema_batch_ms_ + 0.2 * ms;
          finish(b, cudaSuccess);
        } else if (std::chrono::steady_clock::now() - b.t0 > std::chrono::milliseconds(500)) {
          cudaError_t e = cudaStreamQuery(b.stream);  // a faulting kernel never writes the word
          if (e != cudaErrorNotReady && e != cudaSuccess) finish(b, e);
          else if (e == cudaSuccess && *b.flag == b.seq) finish(b, cudaSuccess);
          else b.t0 = std::chrono::steady_clock::now();
        }
        any_busy = any_busy || b.busy;
      }
      // launches: everything pending goes into the next free batch stream
      std::vector<Waiter*> take;
      Batch* free_batch = nullptr;
      for (Batch& b : batches_)
        if (!b.busy) {
          free_batch = &b;
          break;
        }
      // Pacing: with every batch stream free at once, the first arrival would take one stream, the next arrival the next
      // one ... and everything after that waits a whole (long) kernel for the streams to free up - again all together.
      // Launches are therefore spaced a stream's share of the typical batch duration apart: the streams stay staggered
      // and a frame waits that share at most (half of it on average) for its ride.
      const auto now = std::chrono::steady_clock::now();
      const double since_ms = std::chrono::duration<double, std::milli>(now - last_launch_).count();
      const double gap_ms = std::min(30.0, std::max(0.5, ema_batch_ms_ / double(batches_.size())));
      if (any_busy && since_ms < gap_ms) free_batch = nullptr;
      {
        std::unique_lock<std::mutex> lk(mu_);
        if (stop_ && pending_.empty() && !any_busy) return;
        if (free_batch && !pending_.empty()) {
          int refs = 0;
          while (!pending_.empty() && refs + pending_.front()->item->num_jobs <= kMaxRefs) {
            refs += pending_.front()->item->num_jobs;
            take.push_back(pending_.front());
            pending_.pop_front();
          }
        } else if (!any_busy) {
          cv_pending_.wait(lk, [&] { return stop_ || !pending_.empty(); });
          continue;
        }
      }
      if (!take.empty()) {
        launch(*free_batch, take);
        last_launch_ = std::chrono::steady_clock::now();
        continue;
      }
      std::this_thread::sleep_for(std::chrono::microseconds(60));
    }
  }

  int device_;
  std::vector<Batch> batches_;
  std::thread thread_;
  std::mutex mu_;
  std::condition_variable cv_pending_;
  std::deque<Waiter*> pending_;
  bool stop_ = false;
  uint64_t launches_ = 0, items_ = 0;
  std::chrono::steady_clock::time_point last_launch_{};
  double ema_batch_ms_ = 0.0;  // host clock, launch to completion word
};

// CPUs local to the GPU's PCIe root (sysfs), so that worker threads - and whatever they first-touch - sit on the NUMA
// node the device DMAs to. Empty when the topology cannot be read (containers without sysfs): affinity is left alone.
std::vector<int> device_local_cpus(int device) {
  std::vector<int> cpus;
  char busid[32] = {0};
  if (cudaDeviceGetPCIBusId(busid, sizeof(busid), device) != cudaSuccess) return cpus;
  for (char* c = busid; *c; ++c) *c = char(tolower(*c));
  std::ifstream f(std::string("/sys/bus/pci/devices/") + busid + "/local_cpulist");
  std::string list;
  if (!f || !std::getline(f, list)) return cpus;
  std::stringstream ss(list);
  std::string part;
  while (std::getline(ss, part, ',')) {
    int a = 0, b = 0;
    if (std::sscanf(part.c_str(), "%d-%d", &a, &b) == 2) {
      for (int i = a; i <= b; ++i) cpus.push_back(i);
    } else if (std::sscanf(part.c_str(), "%d", &a) == 1) {
      cpus.push_back(a);
    }
  }
  return cpus;
}

}  // namespace

struct jxlb_pipeline {
  int device = 0;
  int heavy_frames = 0;
  std::vector<jxlb_decoder*> decoders;
  std::vector<std::thread> threads;
  std::mutex mu;
  std::condition_variable cv_job, cv_done, cv_slab;
  std::deque<Job> queue;
  std::deque<Done> done;
  uint64_t submitted = 0, reported = 0;
  bool stopping = false;
  std::map<int32_t, Resident> resident;
  std::vector<Slab> slabs;
  std::unique_ptr<BatchService> batcher;
  std::vector<HostBuf> hostbufs;
  size_t host_bytes = 0;  // size every buffer of the output ring has
  std::condition_variable cv_host;
  std::mutex copy_mu;  // one frame's output crosses the host link at a time
  std::string error;
  std::vector<int> cpus;

  size_t max_hint = 0;  // largest heavy-stage request seen: slabs are (re)allocated to it
  int acquire_slab(size_t bytes_hint) {
    std::unique_lock<std::mutex> lk(mu);
    max_hint = std::max(max_hint, bytes_hint);
    bytes_hint = max_hint;
    int idx = -1;
    cv_slab.wait(lk, [&] {
      for (size_t i = 0; i < slabs.size(); ++i)
        if (!slabs[i].busy) {
          idx = int(i);
          return true;
        }
      return false;
    });
    Slab& s = slabs[size_t(idx)];
    s.busy = true;
    if (s.bytes < bytes_hint) {  // first frame of this size: (re)allocate the slab; never shrinks
      lk.unlock();
      cudaSetDevice(device);
      if (s.base) cudaFree(s.base);
      s.base = nullptr;
      s.bytes = 0;
      void* p = nullptr;
      if (cudaMalloc(&p, bytes_hint) == cudaSuccess) {
        s.base = p;
        s.bytes = bytes_hint;
      } else {
        cudaGetLastError();  // out of memory: the frame falls back to the stream-ordered pool
      }
    }
    return idx;
  }
  // The output ring is allocated in one go the first time a frame asks for `bytes` (and again if a larger frame comes):
  // cudaHostAlloc of a few hundred MB takes tens of milliseconds during which no other thread gets a CUDA call through,
  // so it must not trickle into steady state buffer by buffer.
  void* acquire_host(size_t bytes) {
    std::unique_lock<std::mutex> lk(mu);
    if (bytes > host_bytes) {
      cv_host.wait(lk, [&] {  // every buffer back in the ring before it is rebuilt
        for (const HostBuf& b : hostbufs)
          if (b.busy) return false;
        return true;
      });
      if (bytes > host_bytes) {
        for (HostBuf& b : hostbufs) {
          if (b.p) cudaFreeHost(b.p);
          b.p = nullptr;
          b.bytes = 0;
          void* q = nullptr;
          if (cudaHostAlloc(&q, bytes, cudaHostAllocDefault) == cudaSuccess) {
            std::memset(q, 0, bytes);  // first touch by a (GPU-local) worker thread
            b.p = q;
            b.bytes = bytes;
          } else {
            cudaGetLastError();
          }
        }
        host_bytes = bytes;
      }
    }
    int idx = -1;
    cv_host.wait(lk, [&] {
      for (size_t i = 0; i < hostbufs.size(); ++i)
        if (!hostbufs[i].busy && hostbufs[i].p) {
          idx = int(i);
          return true;
        }
      for (const HostBuf& b : hostbufs)
        if (b.p) return false;  // all busy: wait
      idx = -2;                  // nothing could be allocated at all
      return true;
    });
    if (idx < 0) return nullptr;
    hostbufs[size_t(idx)].busy = true;
    return hostbufs[size_t(idx)].p;
  }
  bool release_host(void* ptr) {
    bool found = false;
    {
      std::lock_guard<std::mutex> lk(mu);
      for (HostBuf& b : hostbufs)
        if (b.p == ptr && b.busy) {
          b.busy = false;
          found = true;
        }
    }
    if (found) cv_host.notify_all();
    return found;
  }
  void release_slab(int idx) {
    {
      std::lock_guard<std::mutex> lk(mu);
      slabs[size_t(idx)].busy = false;
    }
    cv_slab.notify_one();
  }

  void worker(size_t wi) {
    cudaSetDevice(device);
    if (!cpus.empty()) {
      cpu_set_t set;
      CPU_ZERO(&set);
      for (int c : cpus) CPU_SET(c, &set);
      pthread_setaffinity_np(pthread_self(), sizeof(set), &set);
    }
    jxlb_decoder* dec = decoders[wi];
    int held = -1;
    // A heavy slot = slab + stream. The planner's begin_heavy_stage() takes the slot for its memory; the stream is handed
    // to the decoder only when it first needs one (a Modular frame decodes all its streams through the batch service
    // and wants the stream for the inverse transforms only).
    dec->be->on_heavy_stage = [&](size_t hint) {
      if (held >= 0) return;  // a later frame of the same image: it shares the slot (overflow goes to the pool)
      held = acquire_slab(hint);
      dec->be->set_arena(slabs[size_t(held)].base, slabs[size_t(held)].bytes);
    };
    dec->be->on_need_stream = [&] {
      if (held < 0) {
        held = acquire_slab(0);
        dec->be->set_arena(slabs[size_t(held)].base, slabs[size_t(held)].bytes);
      }
      dec->be->set_stream(slabs[size_t(held)].stream);
    };
    dec->be->lf_service = batcher.get();
    for (;;) {
      Job job;
      {
        std::unique_lock<std::mutex> lk(mu);
        cv_job.wait(lk, [&] { return stopping || !queue.empty(); });
        if (queue.empty()) return;
        job = queue.front();
        queue.pop_front();
      }
      Done d{job.tag, JXLB_OK, std::string()};
      int32_t rc;
      if (job.data) {
        rc = jxlb_decode(dec, job.data, job.size, nullptr);
      } else {
        const Resident* r = nullptr;
        {
          std::lock_guard<std::mutex> lk(mu);
          auto it = resident.find(job.slot);
          if (it != resident.end()) r = &it->second;
        }
        if (!r) {
          rc = JXLB_ERR_INVALID_ARG;
          dec->error = "unknown preload slot";
        } else {
          rc = decode_resident(dec, r->codestream.data(), r->codestream.size(), r->dptr, nullptr);
        }
      }
      if (rc == JXLB_OK && (job.out_mode == 4 || job.out_mode == 5)) {
        // packed straight into the caller's device buffer (input of an NCCL gather): no host link involved
        rc = jxlb_frame_write_to_device(dec, 0, job.out_mode - 4, 0, job.dst, job.dst_bytes);
        d.out = job.dst;
        d.out_bytes = job.dst_bytes;
      } else if (rc == JXLB_OK && job.out_mode != 0) {
        void* dst = job.dst;
        size_t dst_bytes = job.dst_bytes;
        if (!dst) {  // library-owned pinned staging, sized from the decoded frame
          jxlb_frame_info fi;
          jxlb_frame_get_info(dec, 0, &fi);
          if (job.out_mode == 1) {
            dst_bytes = 0;
            for (const View& v : dec->res.frames[0].channels) dst_bytes += size_t(v.w) * v.h * 4;
          } else {
            dst_bytes = size_t(fi.width) * fi.height * size_t(jxlb_frame_stream_channels(dec, 0)) * (job.out_mode == 2 ? 1 : 2);
          }
          dst = acquire_host(dst_bytes);
          if (!dst) {
            rc = JXLB_ERR_CUDA;
            dec->error = "cannot allocate pinned host memory for the frame output";
          }
        }
        if (rc == JXLB_OK) {
          // Device -> host copies of different streams share the copy engines chunk by chunk; a dozen 400 MB copies
          // in flight together were measured slower in total than one at a time. The decode work of the
          // other frames goes on meanwhile; only the copies queue up.
          rc = jxlb_sync(dec);
          std::lock_guard<std::mutex> copy_lock(copy_mu);
          if (rc != JXLB_OK) {
          } else if (job.out_mode == 1) rc = frame_planar_to_host(dec, 0, static_cast<float*>(dst), dst_bytes);
          else rc = jxlb_frame_write_to_buffer(dec, 0, job.out_mode - 2, 0, dst, dst_bytes);
          d.out = dst;
          d.out_bytes = dst_bytes;
          if (rc != JXLB_OK && !job.dst) {
            release_host(dst);
            d.out = nullptr;
          }
        }
      } else if (rc == JXLB_OK) {
        rc = jxlb_sync(dec);
      }
      if (rc != JXLB_OK) {
        d.status = rc;
        d.error = dec->error;
        jxlb_sync(dec);
      }
      jxlb_release_frames(dec);
      if (held >= 0) {
        dec->be->end_arena();
        try {
          dec->be->end_lease();
        } catch (const Error&) {
        }
        release_slab(held);
        held = -1;
      }
      {
        std::lock_guard<std::mutex> lk(mu);
        done.push_back(std::move(d));
      }
      cv_done.notify_all();
    }
  }
};

extern "C" {

int32_t jxlb_pipeline_create(int32_t device, const jxlb_pipeline_config* cfg, jxlb_pipeline** out) {
  if (!out) return JXLB_ERR_INVALID_ARG;
  *out = nullptr;
  const int workers = cfg && cfg->workers > 0 ? cfg->workers : 64;
  const int heavy = cfg && cfg->heavy_frames > 0 ? cfg->heavy_frames : 16;
  auto p = std::make_unique<jxlb_pipeline>();
  p->device = device;
  p->heavy_frames = heavy;
  p->slabs.resize(size_t(heavy));
  if (cudaSetDevice(device) != cudaSuccess) return JXLB_ERR_CUDA;
  // A pipeline owns its device's decode work: L2 fetches 32-byte sectors instead of whole 128-byte lines. The inverse
  // transforms read 32-byte row segments of varblocks whose line neighbours belong to another size class, i.e. to another
  // kernel at another time, so 32-byte fetches read less DRAM for the same kernel times. A stand-alone decoder leaves the
  // limit alone.
  cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 32);
  for (Slab& sl : p->slabs)
    if (cudaStreamCreateWithFlags(&sl.stream, cudaStreamNonBlocking) != cudaSuccess) return JXLB_ERR_CUDA;
  p->batcher.reset(new BatchService(device, cfg && cfg->batch_streams > 0 ? cfg->batch_streams : 6));
  p->hostbufs.resize(6);  // outputs cross the host link one at a time; a few buffers cover the consumer's turnaround
  for (int i = 0; i < workers; ++i) {
    int32_t rc = JXLB_OK;
    jxlb_decoder* d = create_decoder_internal(device, 0, false, &rc);
    if (rc != JXLB_OK) {
      for (jxlb_decoder* q : p->decoders) jxlb_decoder_destroy(q);
      return rc;
    }
    // many frames in flight: one thread per HF stream (16 warps per 8K frame instead of 510 one-lane warps), see bench.py
    jxlb_set_hf_streams_per_cta(d, cfg && cfg->hf_streams_per_cta > 0 ? cfg->hf_streams_per_cta : 128);
    p->decoders.push_back(d);
  }
  if (!(cfg && cfg->no_affinity)) p->cpus = device_local_cpus(device);
  for (int i = 0; i < workers; ++i) p->threads.emplace_back([q = p.get(), i] { q->worker(size_t(i)); });
  *out = p.release();
  return JXLB_OK;
}

void jxlb_pipeline_destroy(jxlb_pipeline* p) {
  if (!p) return;
  {
    std::lock_guard<std::mutex> lk(p->mu);
    p->stopping = true;
    p->queue.clear();
  }
  p->cv_job.notify_all();
  for (std::thread& t : p->threads) t.join();
  for (jxlb_decoder* d : p->decoders) jxlb_decoder_destroy(d);
  cudaSetDevice(p->device);
  p->batcher.reset();
  for (Slab& s : p->slabs) {
    if (s.base) cudaFree(s.base);
    if (s.stream) cudaStreamDestroy(s.stream);
  }
  for (auto& kv : p->resident)
    if (kv.second.dptr) cudaFree(kv.second.dptr);
  for (HostBuf& b : p->hostbufs)
    if (b.p) cudaFreeHost(b.p);
  delete p;
}

const char* jxlb_pipeline_last_error(const jxlb_pipeline* p) { return p ? p->error.c_str() : "null pipeline"; }

int32_t jxlb_pipeline_preload(jxlb_pipeline* p, int32_t slot, const uint8_t* data, size_t size) {
  if (!p || !data) return JXLB_ERR_INVALID_ARG;
  try {
    Resident r;
    r.codestream = extract_codestream(data, size);
    r.dptr = p->decoders[0]->be->upload_resident(r.codestream.data(), r.codestream.size());
    std::lock_guard<std::mutex> lk(p->mu);
    Resident& dst = p->resident[slot];
    if (dst.dptr) cudaFree(dst.dptr);
    dst = std::move(r);
    return JXLB_OK;
  } catch (const Error& e) {
    p->error = e.what();
    return e.code;
  }
}

int32_t jxlb_pipeline_submit(jxlb_pipeline* p, const uint8_t* data, size_t size, int32_t slot, int32_t out_mode, void* dst,
                             size_t dst_bytes, uint64_t tag) {
  if (!p || out_mode < 0 || out_mode > 5 || (!data && slot < 0) || (out_mode >= 4 && !dst)) return JXLB_ERR_INVALID_ARG;
  Job j;
  j.data = data;
  j.size = size;
  j.slot = slot;
  j.out_mode = out_mode;
  j.dst = dst;
  j.dst_bytes = dst_bytes;
  j.tag = tag;
  {
    std::lock_guard<std::mutex> lk(p->mu);
    if (p->stopping) return JXLB_ERR_INVALID_ARG;
    p->queue.push_back(j);
    ++p->submitted;
  }
  p->cv_job.notify_one();
  return JXLB_OK;
}

int32_t jxlb_pipeline_wait(jxlb_pipeline* p, uint64_t* tag, int32_t* status, void** out, size_t* out_bytes, char* err,
                           size_t err_cap) {
  if (!p || !tag || !status) return JXLB_ERR_INVALID_ARG;
  std::unique_lock<std::mutex> lk(p->mu);
  if (p->reported == p->submitted) return JXLB_ERR_INVALID_ARG;  // nothing in flight
  p->cv_done.wait(lk, [&] { return !p->done.empty(); });
  Done d = std::move(p->done.front());
  p->done.pop_front();
  ++p->reported;
  *tag = d.tag;
  *status = d.status;
  if (out) *out = d.out;
  if (out_bytes) *out_bytes = d.out_bytes;
  if (err && err_cap) std::snprintf(err, err_cap, "%s", d.error.c_str());
  return JXLB_OK;
}

int32_t jxlb_pipeline_release_output(jxlb_pipeline* p, void* out) {
  if (!p || !out) return JXLB_ERR_INVALID_ARG;
  return p->release_host(out) ? JXLB_OK : JXLB_ERR_INVALID_ARG;
}

uint64_t jxlb_pipeline_launch_count(const jxlb_pipeline* p) {
  uint64_t n = 0;
  if (p)
    for (const jxlb_decoder* d : p->decoders) n += d->be->launches;
  return n;
}

int32_t jxlb_pipeline_workers(const jxlb_pipeline* p) { return p ? int32_t(p->decoders.size()) : 0; }

jxlb_decoder* jxlb_pipeline_decoder(jxlb_pipeline* p, int32_t index) {
  return (p && index >= 0 && size_t(index) < p->decoders.size()) ? p->decoders[size_t(index)] : nullptr;
}

}  // extern "C"
