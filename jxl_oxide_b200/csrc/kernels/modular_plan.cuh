// Host-built per-channel plans of the Modular stream kernel (modular_stream.cu) for a frame's whole MA tree: the
// fallback when a channel's reachable subtree is too large to compact (cuda_backend.cu), and the plans the host
// emulation in tests/emu/ runs the kernel's per-stream code with.
#pragma once
#include <algorithm>
#include <cstdint>
#include <vector>

#include "kernels.h"

namespace jxlb {

// Resolves the MA-tree nodes that test properties which are constant for a whole channel
// (channel index, stream index, previous channels that do not exist), like
// MaTreeNode::next_decision_node (crates/jxl-modular/src/ma.rs:424-470).
inline uint32_t resolve_static(const MaTree& t, uint32_t idx, uint32_t ci, uint32_t stream, int nprev) {
  for (;;) {
    const MaNode& n = t.nodes[idx];
    if (n.property < 0) return idx;
    int32_t v;
    if (n.property == 0) v = int32_t(ci);
    else if (n.property == 1) v = int32_t(stream);
    else if (n.property >= 16 && (n.property - 16) / 4 >= nprev) v = 0;
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
