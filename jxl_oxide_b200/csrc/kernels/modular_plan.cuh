// What the host has to know about the Modular stream kernel (modular_stream.cu) to build its launch tables
// (launch_tables.cc): the shared-memory layout of a job, whether a launch stages every table, and the per-channel plans
// for a frame's whole MA tree (the fallback when a channel's reachable subtree is too large to compact).
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

#include "kernels.h"

namespace jxlb {

constexpr uint32_t kFastChunk = 128;       // columns per warp-computed row prologue of the weighted-predictor fast loop
constexpr uint32_t kFastMaxLeaves = 1024;  // a LUT spans at most 1024 property values (launch_tables.cc)

constexpr uint32_t kSmemTreeBytes = 64 * 1024;
constexpr uint32_t kSmemAnsBytes = 48 * 1024;
constexpr uint32_t kSmemPrefixBytes = 24 * 1024;
constexpr uint32_t kSmemLutBytes = 8 * 1024;
constexpr uint32_t kSmemWpMaxWidth = 1024;

struct SmemLayout {
  uint32_t tree, ans, prefix, prefix_meta, configs, luts, wp, div, fast_pro, fast_leaves, fast_rows, total;
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
  // weighted-predictor fast loop: row prologue (4 x int4 per column), packed leaves, second pair of error rows
  L.fast_pro = L.fast_leaves = L.fast_rows = 0xffffffffu;
  if (L.wp != 0xffffffffu) {
    L.fast_pro = take(kFastChunk * 64);
    L.fast_leaves = take((lut_total < kFastMaxLeaves ? lut_total : kFastMaxLeaves) * 16);
    L.fast_rows = take(max_w * 5 * 4);
  }
  L.total = off;
  return L;
}

// bytes of dynamic shared memory a job wants for its tree / entropy tables / WP rows / LUTs
inline size_t modular_job_smem_bytes(const DevModularJob& job, uint32_t max_width) {
  return modular_layout(job.num_tree_nodes, job.code, job.lut_total, job.use_wp, max_width).total;
}

// Whether modular_stream_kernel stages every table of this job (tree, entropy tables, leaf LUTs, predictor rows).
inline bool modular_job_all_staged(const DevModularJob& job, uint32_t max_width) {
  const SmemLayout L = modular_layout(job.num_tree_nodes, job.code, job.lut_total, job.use_wp, max_width);
  if (L.tree == 0xffffffffu || L.luts == 0xffffffffu) return false;
  if (job.code.use_prefix ? L.prefix == 0xffffffffu : L.ans == 0xffffffffu) return false;
  if (job.use_wp && L.wp == 0xffffffffu) return false;
  return !job.code.lz77_enabled;
}

// Resolves the MA-tree nodes that test properties which are constant for a whole channel
// (channel index, stream index, previous channels that do not exist), like
// MaTreeNode::next_decision_node (crates/jxl-modular/src/ma.rs:424-470). Sets *stream_dependent when
// a stream-index test was taken.
inline uint32_t resolve_static(const MaTree& t, uint32_t idx, uint32_t ci, uint32_t stream, int nprev,
                               bool* stream_dependent = nullptr) {
  for (;;) {
    const MaNode& n = t.nodes[idx];
    if (n.property < 0) return idx;
    int32_t v;
    if (n.property == 0) v = int32_t(ci);
    else if (n.property == 1) {
      v = int32_t(stream);
      if (stream_dependent) *stream_dependent = true;
    } else if (n.property >= 16 && (n.property - 16) / 4 >= nprev) v = 0;
    else return idx;
    idx = v > n.value ? n.a : n.b;
  }
}

inline DevChannelPlan build_channel_plan(const MaTree& t, uint32_t ci, uint32_t stream, int nprev, std::vector<uint16_t>* luts) {
  DevChannelPlan plan;
  plan.root = resolve_static(t, 0, ci, stream, nprev);
  plan.lut_prop = -1;
  plan.lut_base = 0;
  plan.lut_len = 0;
  plan.lut_offset = uint32_t(luts->size());
  if (t.nodes.size() >= 65536) return plan;
  // which sample-dependent properties does the reachable subtree test?
  int prop = -1;
  bool single = true;
  int64_t lower = INT64_MAX, upper = INT64_MIN;
  std::vector<uint32_t> stack = {plan.root};
  size_t visited = 0;
  while (!stack.empty() && single) {
    uint32_t idx = resolve_static(t, stack.back(), ci, stream, nprev);
    stack.pop_back();
    if (++visited > 4096) {
      single = false;
      break;
    }
    const MaNode& n = t.nodes[idx];
    if (n.property < 0) continue;
    if (n.property >= 16 || (prop >= 0 && prop != n.property)) {
      single = false;
      break;
    }
    prop = n.property;
    lower = std::min<int64_t>(lower, n.value);
    upper = std::max<int64_t>(upper, n.value);
    stack.push_back(n.a);
    stack.push_back(n.b);
  }
  if (!single) return plan;
  if (prop < 0) {  // the channel has a single leaf
    plan.lut_prop = 6;
    plan.lut_base = 0;
    plan.lut_len = 1;
    luts->push_back(uint16_t(plan.root));
    return plan;
  }
  if (upper - lower > 1022) return plan;
  plan.lut_prop = prop;
  plan.lut_base = int32_t(lower);
  plan.lut_len = uint32_t(upper - lower + 2);
  for (int64_t v = lower; v <= upper + 1; ++v) {
    uint32_t idx = plan.root;
    for (;;) {
      idx = resolve_static(t, idx, ci, stream, nprev);
      const MaNode& n = t.nodes[idx];
      if (n.property < 0) break;
      idx = v > n.value ? n.a : n.b;
    }
    luts->push_back(uint16_t(idx));
  }
  return plan;
}


inline bool tree_uses_wp(const MaTree& t) {
  for (const MaNode& n : t.nodes) {
    if (n.property == 15) return true;
    if (n.property < 0 && (n.a & 0xff) == 6) return true;
  }
  return false;
}

}  // namespace jxlb
