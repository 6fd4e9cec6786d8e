// How a frame's host syntax becomes the parameter blocks and tables of the stream and filter kernels. Plain C++ with no
// CUDA runtime calls: the CUDA backend puts the tables into its staging block, the host emulations in tests/emu/ into host
// memory, and both build them with the same code.
#pragma once
#include <cstddef>
#include <cstdint>
#include <functional>
#include <vector>

#include "host/backend.h"
#include "kernels/kernels.h"

namespace jxlb {

// Where tables go: copies `bytes` bytes from `src` and returns the address the kernel reads them at.
struct TableSink {
  virtual const void* put(const void* src, size_t bytes) = 0;
};

DevEntropyCode make_dev_code(const EntropyCode& c, TableSink& sink);
void pack_wp(const WpHeader& w, uint32_t out[11]);  // p1 p2 p3a p3b p3c p3d p3e w0..w3

// Channel subtrees with more nodes than this are not copied per job: the job walks the frame's whole tree instead.
constexpr size_t kMaxChannelTreeNodes = 60000;

// One Modular launch. The jobs' global scratch (wp_scratch, lz_window) is left null for the caller to fill. A job with a
// varblock placement carries it (DevModularJob::place), and the launch reserves kPlaceSharedBytes per CTA at least.
struct ModularLaunch {
  struct JobNeeds {
    size_t wp_scratch_bytes = 0, lz_window_bytes = 0;
    bool whole_tree = false;  // the job's channels walk the frame's whole tree (a subtree exceeded the node limit)
  };
  std::vector<DevModularJob> jobs;
  std::vector<DevChannel> channels;
  std::vector<DevChannelPlan> plans;
  std::vector<JobNeeds> needs;  // per job
  size_t smem_bytes = 0;        // per CTA: the largest job's
  bool all_staged = true;       // every job stages every table (the kernel's shared-memory-only variant)
};
// Per job: the entropy code and the MA subtree each channel can reach, pruned, renumbered and shared by channels and
// jobs with identical content (the whole-tree plans of kernels/modular_plan.cuh when a subtree is too large).
ModularLaunch build_modular_launch(const std::vector<ModularStreamJob>& jobs,
                                   const std::function<DevView(const View&)>& view_to_dev, TableSink& sink,
                                   size_t max_channel_tree_nodes = kMaxChannelTreeNodes);

// The device form of a varblock placement (kernels/placement.cuh).
DevPlacement make_dev_placement(const VarblockPlacement& p, const std::function<DevView(const View&)>& view_to_dev);

// The 13 natural coefficient orders back to back; offset[id] is where order `id` starts.
std::vector<uint32_t> natural_order_table(uint32_t offset[13]);
// Parameters of one HF pass. `natural_orders` is natural_order_table() where the kernel can read it, used unless the pass
// carries a custom order.
DevHfParams build_hf_params(const VarDctState& st, uint32_t pass, TableSink& sink, const uint32_t* natural_orders,
                            const uint32_t natural_offset[13]);
// Which kernel decodes the HF streams of one pass, and how many streams share a CTA: one thread per stream
// (launch_decode_hf_lanes, `per_cta` 64 or 128, `per_warp` of them in each warp) or one warp per stream
// (launch_decode_hf, `per_cta` 8, 16 or 32, `per_warp` 1).
struct HfSchedule {
  bool lanes;
  int per_cta;
  int per_warp;
};
// Streams per warp of the thread-per-stream kernel unless the decoder sets it (jxlb_set_hf_streams_per_warp).
constexpr int kHfStreamsPerWarpDefault = 8;
// `streams_per_cta` is the decoder's setting (jxlb_set_hf_streams_per_cta): 0 (one warp per stream, 16 per CTA), 4 (the
// same as 8), 8, 16, 32, 64 or 128. Cluster maps larger than kLaneCmapSmemBytes and codes with LZ77 always run one thread
// per stream, 128 per CTA. `streams_per_warp` (jxlb_set_hf_streams_per_warp): 0 (kHfStreamsPerWarpDefault), 4, 8, 16 or
// 32, for every thread-per-stream schedule.
HfSchedule hf_schedule(const DevHfParams& p, int streams_per_cta, int streams_per_warp);
// Entries of one HF stream's LZ77 window for groups of `group_dim` pixels: min(2^20, 3 * group_dim^2). A stream reads one
// value per varblock channel (its non-zero count) plus at most 63 coefficients per 8x8 block of it, so at most
// group_dim^2 values per channel; below 2^20 entries the window's `& 0xfffff` index never wraps, and at group_dim 1024
// the window is the reference's 2^20-entry ring.
size_t hf_lz77_window_entries(uint32_t group_dim);
// Launch order of the HF streams as indices into `jobs`. longest_first (the thread-per-stream kernel): longest section
// first, so that streams of similar length share a warp.
std::vector<uint32_t> hf_launch_order(const std::vector<HfGroupJob>& jobs, bool longest_first);
DevFrame make_dev_frame(const VarDctState& st, const std::function<void*(int)>& plane_ptr);

// `sigma`: the per-block sigma grid, or nullptr for the constant sigma_for_modular.
DevFusedFilterParams fused_filter_params(const RestorationFilter& rf, const float* sigma, uint32_t sigma_stride,
                                         const ColorParams* colour);

}  // namespace jxlb
