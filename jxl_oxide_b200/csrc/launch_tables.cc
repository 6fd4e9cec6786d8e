// See launch_tables.h.
#include "launch_tables.h"

#include <algorithm>
#include <climits>
#include <cstring>
#include <map>
#include <memory>
#include <tuple>

#include "kernels/modular_plan.cuh"

namespace jxlb {

DevEntropyCode make_dev_code(const EntropyCode& c, TableSink& sink) {
  DevEntropyCode d;
  std::memset(&d, 0, sizeof(d));
  d.cluster_map = static_cast<const uint8_t*>(sink.put(c.cluster_map.data(), c.cluster_map.size()));
  std::vector<uint32_t> cfg;
  for (const HybridUintConfig& h : c.configs) cfg.push_back(h.packed());
  d.configs = static_cast<const uint32_t*>(sink.put(cfg.data(), cfg.size() * 4));
  d.log_alphabet_size = c.log_alphabet_size;
  d.use_prefix = c.use_prefix ? 1 : 0;
  d.num_clusters = c.num_clusters;
  d.cluster_map_size = uint32_t(c.cluster_map.size());
  d.prefix_table_size = uint32_t(c.prefix_table.size());
  if (c.use_prefix) {
    d.prefix = static_cast<const uint32_t*>(sink.put(c.prefix_table.data(), c.prefix_table.size() * 4));
    std::vector<uint32_t> meta;
    for (const PrefixMeta& m : c.prefix_meta) {
      meta.push_back(m.table_offset);
      meta.push_back(m.root_bits);
    }
    d.prefix_meta = static_cast<const uint32_t*>(sink.put(meta.data(), meta.size() * 4));
  } else {
    d.ans = static_cast<const uint64_t*>(sink.put(c.ans_table.data(), c.ans_table.size() * 8));
  }
  d.lz77_enabled = c.lz77_enabled ? 1 : 0;
  d.lz77_min_symbol = c.lz77_min_symbol;
  d.lz77_min_length = c.lz77_min_length;
  d.lz_len_conf = c.lz_len_conf.packed();
  d.lz_dist_cluster = c.cluster_map.empty() ? 0 : c.cluster_map.back();
  return d;
}

void pack_wp(const WpHeader& w, uint32_t out[11]) {
  const uint32_t v[11] = {w.p1, w.p2, w.p3a, w.p3b, w.p3c, w.p3d, w.p3e, w.w[0], w.w[1], w.w[2], w.w[3]};
  std::memcpy(out, v, sizeof(v));
}

namespace {
// The part of an MA tree one channel of one stream can reach, with static decisions resolved and
// node indices renumbered from 0 (the reference prunes the same way when it flattens a tree for a
// channel, crates/jxl-modular/src/ma.rs:579-645). Small enough to live in shared memory even when
// the frame's global tree has thousands of nodes.
struct ChannelTree {
  std::vector<MaNode> nodes;  // nodes[0] is the root
  int32_t lut_prop = -1, lut_base = 0;
  std::vector<uint16_t> lut;  // leaf indices into `nodes`
  bool stream_dependent = false;
};

bool build_channel_tree(const MaTree& t, uint32_t ci, uint32_t stream, int nprev, size_t max_nodes, ChannelTree* out) {
  auto resolve = [&](uint32_t idx) { return resolve_static(t, idx, ci, stream, nprev, &out->stream_dependent); };
  out->nodes.clear();
  out->nodes.push_back(t.nodes[resolve(0)]);
  std::vector<uint32_t> stack = {0};
  while (!stack.empty()) {
    const uint32_t cur = stack.back();
    stack.pop_back();
    if (out->nodes[cur].property < 0) continue;
    if (out->nodes.size() + 2 > max_nodes) return false;
    const uint32_t a = resolve(out->nodes[cur].a), b = resolve(out->nodes[cur].b);
    const uint32_t na = uint32_t(out->nodes.size());
    out->nodes.push_back(t.nodes[a]);
    out->nodes.push_back(t.nodes[b]);
    out->nodes[cur].a = na;
    out->nodes[cur].b = na + 1;
    stack.push_back(na);
    stack.push_back(na + 1);
  }
  // single-property subtree -> leaf LUT over [lower, upper + 1] (ma.rs:241-330)
  int prop = -1;
  int64_t lower = INT64_MAX, upper = INT64_MIN;
  for (const MaNode& n : out->nodes) {
    if (n.property < 0) continue;
    if (n.property >= 16 || (prop >= 0 && prop != n.property)) return true;  // general walk
    prop = n.property;
    lower = std::min<int64_t>(lower, n.value);
    upper = std::max<int64_t>(upper, n.value);
  }
  if (prop < 0) {  // single leaf
    out->lut_prop = 6;
    out->lut_base = 0;
    out->lut.assign(1, 0);
    return true;
  }
  if (upper - lower > 1022) return true;
  out->lut_prop = prop;
  out->lut_base = int32_t(lower);
  for (int64_t v = lower; v <= upper + 1; ++v) {
    uint32_t idx = 0;
    while (out->nodes[idx].property >= 0) idx = v > out->nodes[idx].value ? out->nodes[idx].a : out->nodes[idx].b;
    out->lut.push_back(uint16_t(idx));
  }
  return true;
}
}  // namespace

ModularLaunch build_modular_launch(const std::vector<ModularStreamJob>& jobs,
                                   const std::function<DevView(const View&)>& view_to_dev, TableSink& sink,
                                   size_t max_channel_tree_nodes) {
  struct TreeDev {
    const MaNode* nodes = nullptr;  // full tree, put only for the uncompacted fallback
    DevEntropyCode code;
    bool wp = false;
  };
  struct JobTables {  // tables shared by every job with the same per-channel subtrees
    const MaNode* nodes;
    uint32_t num_nodes;
    const uint16_t* luts;
    uint32_t lut_total;
    std::vector<DevChannelPlan> plans;
    bool wp;
  };
  std::map<const MaTree*, TreeDev> trees;
  std::map<std::tuple<const MaTree*, uint32_t, int, int64_t>, std::unique_ptr<ChannelTree>> channel_trees;
  std::map<std::vector<const ChannelTree*>, JobTables> job_tables;
  ModularLaunch L;
  L.jobs.resize(jobs.size());
  L.needs.resize(jobs.size());
  for (size_t i = 0; i < jobs.size(); ++i) {
    const ModularStreamJob& j = jobs[i];
    auto it = trees.find(j.tree);
    if (it == trees.end()) {
      TreeDev td;
      td.code = make_dev_code(j.tree->code, sink);
      it = trees.emplace(j.tree, td).first;
    }
    DevModularJob& d = L.jobs[i];
    std::memset(&d, 0, sizeof(d));
    d.bit_pos = j.bit_pos;
    d.bit_limit = j.bit_limit;
    d.code = it->second.code;
    pack_wp(j.wp, d.wp);
    d.stream_index = j.stream_index;
    d.first_channel = uint32_t(L.channels.size());
    d.num_channels = uint32_t(j.channels.size());
    uint32_t max_w = 0;
    uint64_t samples = 0;
    for (const ModularChannelTarget& c : j.channels) {
      DevView v = view_to_dev(c.view);
      L.channels.push_back({static_cast<int32_t*>(v.ptr), v.stride, c.view.w, c.view.h, c.hshift, c.vshift});
      max_w = std::max(max_w, c.view.w);
      samples += uint64_t(c.view.w) * c.view.h;
    }
    d.dist_multiplier = max_w;
    // per-channel subtrees (cached across the jobs of this call when they do not depend on the stream index)
    std::vector<const ChannelTree*> key;
    bool compact = true;
    std::vector<int> nprevs(j.channels.size());
    for (size_t ci = 0; ci < j.channels.size(); ++ci) {
      const ModularChannelTarget& c = j.channels[ci];
      int nprev = 0;
      for (size_t pj = 0; pj < ci; ++pj) {
        const ModularChannelTarget& q = j.channels[pj];
        if (q.view.w && q.view.h && q.view.w == c.view.w && q.view.h == c.view.h && q.hshift == c.hshift && q.vshift == c.vshift) ++nprev;
      }
      nprevs[ci] = nprev = std::min(nprev, 16);
      if (!compact) continue;
      auto any = channel_trees.find({j.tree, uint32_t(ci), nprev, -1});
      if (any == channel_trees.end()) any = channel_trees.find({j.tree, uint32_t(ci), nprev, int64_t(j.stream_index)});
      if (any == channel_trees.end()) {
        auto ct = std::make_unique<ChannelTree>();
        if (!build_channel_tree(*j.tree, uint32_t(ci), j.stream_index, nprev, max_channel_tree_nodes, ct.get())) {
          compact = false;
          continue;
        }
        const int64_t skey = ct->stream_dependent ? int64_t(j.stream_index) : -1;
        any = channel_trees.emplace(std::make_tuple(j.tree, uint32_t(ci), nprev, skey), std::move(ct)).first;
      }
      // Channels whose reachable subtrees are identical node for node (a tree that never tests the channel index, e.g.
      // a Squeeze image's 36 global channels under one weighted-predictor chain) share one staged copy: the first
      // channel tree with that content stands for all of them.
      const ChannelTree* canon = any->second.get();
      for (const ChannelTree* prev : key)
        if (prev != canon && prev->lut_prop == canon->lut_prop && prev->lut_base == canon->lut_base && prev->lut == canon->lut &&
            prev->nodes.size() == canon->nodes.size() &&
            std::memcmp(prev->nodes.data(), canon->nodes.data(), canon->nodes.size() * sizeof(MaNode)) == 0) {
          canon = prev;
          break;
        }
      key.push_back(canon);
    }
    if (compact) {
      auto jt = job_tables.find(key);
      if (jt == job_tables.end()) {
        JobTables t;
        std::vector<MaNode> nodes;
        std::vector<uint16_t> luts;
        t.wp = false;
        std::map<const ChannelTree*, DevChannelPlan> seen;  // channels that reach the same subtree share its copy
        for (const ChannelTree* ct : key) {
          auto dup = seen.find(ct);
          if (dup != seen.end()) {
            t.plans.push_back(dup->second);
            continue;
          }
          const uint32_t base = uint32_t(nodes.size());
          DevChannelPlan plan;
          plan.root = base;
          plan.lut_prop = -1;
          plan.lut_base = 0;
          plan.lut_len = 0;
          plan.lut_offset = uint32_t(luts.size());
          for (MaNode n : ct->nodes) {
            if (n.property >= 0) {
              n.a += base;
              n.b += base;
              if (n.property == 15) t.wp = true;
            } else if ((n.a & 0xff) == 6) {
              t.wp = true;
            }
            nodes.push_back(n);
          }
          if (ct->lut_prop >= 0 && nodes.size() <= 65536) {
            plan.lut_prop = ct->lut_prop;
            plan.lut_base = ct->lut_base;
            plan.lut_len = uint32_t(ct->lut.size());
            for (uint16_t l : ct->lut) luts.push_back(uint16_t(l + base));
          }
          t.plans.push_back(plan);
          seen.emplace(ct, plan);
        }
        t.num_nodes = uint32_t(nodes.size());
        t.lut_total = uint32_t(luts.size());
        luts.push_back(0);
        luts.push_back(0);
        t.nodes = static_cast<const MaNode*>(sink.put(nodes.data(), nodes.size() * sizeof(MaNode)));
        t.luts = static_cast<const uint16_t*>(sink.put(luts.data(), luts.size() * 2));
        jt = job_tables.emplace(key, std::move(t)).first;
      }
      const JobTables& t = jt->second;
      d.tree = t.nodes;
      d.num_tree_nodes = t.num_nodes;
      d.luts = t.luts;
      d.lut_total = t.lut_total;
      d.use_wp = t.wp ? 1 : 0;
      L.plans.insert(L.plans.end(), t.plans.begin(), t.plans.end());
    } else {  // a channel's subtree is too large to copy per job: walk the frame's tree in global memory
      TreeDev& td = it->second;
      if (!td.nodes) {
        td.nodes = static_cast<const MaNode*>(sink.put(j.tree->nodes.data(), j.tree->nodes.size() * sizeof(MaNode)));
        td.wp = tree_uses_wp(*j.tree);
      }
      d.tree = td.nodes;
      d.num_tree_nodes = uint32_t(j.tree->nodes.size());
      d.use_wp = td.wp ? 1 : 0;
      std::vector<uint16_t> luts;
      for (size_t ci = 0; ci < j.channels.size(); ++ci)
        L.plans.push_back(build_channel_plan(*j.tree, uint32_t(ci), j.stream_index, nprevs[ci], &luts));
      d.lut_total = uint32_t(luts.size());
      luts.push_back(0);
      luts.push_back(0);
      d.luts = static_cast<const uint16_t*>(sink.put(luts.data(), luts.size() * 2));
      L.needs[i].whole_tree = true;
    }
    L.smem_bytes = std::max(L.smem_bytes, modular_job_smem_bytes(d, max_w));
    if (j.placement.group.nb_blocks) {
      d.place = make_dev_placement(j.placement, view_to_dev);
      L.smem_bytes = std::max(L.smem_bytes, kPlaceSharedBytes);
    }
    L.all_staged = L.all_staged && modular_job_all_staged(d, max_w);
    if (d.use_wp && max_w) L.needs[i].wp_scratch_bytes = size_t(max_w) * 5 * 4;
    if (d.code.lz77_enabled) L.needs[i].lz_window_bytes = size_t(std::min<uint64_t>(1u << 20, std::max<uint64_t>(samples, 1))) * 4;
  }
  return L;
}

DevPlacement make_dev_placement(const VarblockPlacement& p, const std::function<DevView(const View&)>& view_to_dev) {
  const BlockInfoJob& g = p.group;
  DevPlacement d;
  std::memset(&d, 0, sizeof(d));
  const DevView raw = view_to_dev(View{g.raw_plane, 0, 0, g.nb_blocks, 2});
  d.raw = static_cast<const int32_t*>(raw.ptr);
  d.raw_stride = raw.stride;
  d.nb_blocks = g.nb_blocks;
  d.bw = g.rect.bw;
  d.bh = g.rect.bh;
  auto grid = [&](int plane) { return view_to_dev(View{plane, g.rect.bx0, g.rect.by0, g.rect.bw, g.rect.bh}); };
  const DevView type = grid(p.blk_type);
  d.grid_stride = type.stride;
  d.blk_type = static_cast<int32_t*>(type.ptr);
  d.blk_mul = static_cast<int32_t*>(grid(p.blk_mul).ptr);
  d.epf_sigma = static_cast<float*>(grid(p.epf_sigma).ptr);
  d.sharpness = static_cast<const int32_t*>(grid(p.sharpness).ptr);
  d.quant_mul_base = p.quant_mul_base;
  for (int i = 0; i < 8; ++i) d.sharp_lut[i] = p.sharp_lut[i];
  d.has_epf = p.has_epf ? 1 : 0;
  return d;
}

std::vector<uint32_t> natural_order_table(uint32_t offset[13]) {
  std::vector<uint32_t> all;
  for (uint32_t id = 0; id < 13; ++id) {
    offset[id] = uint32_t(all.size());
    std::vector<uint32_t> o = natural_order(id);
    all.insert(all.end(), o.begin(), o.end());
  }
  return all;
}

DevHfParams build_hf_params(const VarDctState& st, uint32_t pass, TableSink& sink, const uint32_t* natural_orders,
                            const uint32_t natural_offset[13]) {
  const HfBlockContext& hbc = st.lfg->hf_block_ctx;
  const HfPassSyntax& hp = st.hfg->passes[pass];
  DevHfParams p;
  std::memset(&p, 0, sizeof(p));
  p.code = make_dev_code(hp.code, sink);
  // orders: natural (static) unless the pass carries a custom permutation
  std::vector<uint32_t> custom;
  bool any_custom = false;
  for (int id = 0; id < 13; ++id)
    for (int c = 0; c < 3; ++c) any_custom |= !hp.order[id][c].empty();
  if (!any_custom) {
    p.orders = natural_orders;
    for (int id = 0; id < 13; ++id)
      for (int c = 0; c < 3; ++c) p.order_offset[id * 3 + c] = natural_offset[id];
  } else {
    for (int id = 0; id < 13; ++id)
      for (int c = 0; c < 3; ++c) {
        p.order_offset[id * 3 + c] = uint32_t(custom.size());
        if (hp.order[id][c].empty()) {
          std::vector<uint32_t> o = natural_order(uint32_t(id));
          custom.insert(custom.end(), o.begin(), o.end());
        } else {
          custom.insert(custom.end(), hp.order[id][c].begin(), hp.order[id][c].end());
        }
      }
    p.orders = static_cast<const uint32_t*>(sink.put(custom.data(), custom.size() * 4));
  }
  p.block_ctx_map = static_cast<const uint8_t*>(sink.put(hbc.block_ctx_map.data(), hbc.block_ctx_map.size()));
  p.block_ctx_map_size = uint32_t(hbc.block_ctx_map.size());
  std::vector<int32_t> thr;
  for (int c = 0; c < 3; ++c) {
    p.num_lf_thr[c] = uint32_t(hbc.lf_thresholds[c].size());
    thr.insert(thr.end(), hbc.lf_thresholds[c].begin(), hbc.lf_thresholds[c].end());
  }
  thr.push_back(0);
  p.lf_thresholds = static_cast<const int32_t*>(sink.put(thr.data(), thr.size() * 4));
  p.has_lf_quant = st.use_lf_frame ? 0 : 1;
  std::vector<uint32_t> qf = hbc.qf_thresholds;
  p.num_qf_thr = uint32_t(qf.size());
  qf.push_back(0);
  p.qf_thresholds = static_cast<const uint32_t*>(sink.put(qf.data(), qf.size() * 4));
  p.num_block_clusters = hbc.num_block_clusters;
  p.num_hf_presets = st.hfg->num_hf_presets;
  p.coeff_shift = pass < st.fh->passes.shift.size() ? st.fh->passes.shift[pass] : 0;
  p.group_dim_blocks = st.group_dim / 8;
  p.groups_per_row = st.groups_per_row;
  return p;
}

HfSchedule hf_schedule(const DevHfParams& p, int streams_per_cta, int streams_per_warp) {
  const int per_warp = streams_per_warp > 0 ? streams_per_warp : kHfStreamsPerWarpDefault;
  const bool cmaps_fit = 495u * p.num_block_clusters * p.num_hf_presets <= kLaneCmapSmemBytes;
  if (p.code.lz77_enabled || !cmaps_fit || streams_per_cta > 64) return {true, 128, per_warp};
  if (streams_per_cta == 64) return {true, 64, per_warp};
  if (streams_per_cta >= 32) return {false, 32, 1};
  if (streams_per_cta >= 16 || streams_per_cta == 0) return {false, 16, 1};
  return {false, 8, 1};
}

size_t hf_lz77_window_entries(uint32_t group_dim) {
  return size_t(std::min<uint64_t>(uint64_t(1) << 20, 3 * uint64_t(group_dim) * group_dim));
}

std::vector<uint32_t> hf_launch_order(const std::vector<HfGroupJob>& jobs, bool longest_first) {
  std::vector<uint32_t> perm(jobs.size());
  for (size_t i = 0; i < jobs.size(); ++i) perm[i] = uint32_t(i);
  if (longest_first) std::stable_sort(perm.begin(), perm.end(), [&](uint32_t a, uint32_t b) {
    return jobs[a].bit_limit - jobs[a].bit_pos > jobs[b].bit_limit - jobs[b].bit_pos;
  });
  return perm;
}

DevFrame make_dev_frame(const VarDctState& st, const std::function<void*(int)>& plane_ptr) {
  DevFrame f;
  f.width = st.width;
  f.height = st.height;
  f.bw = st.bw;
  f.bh = st.bh;
  f.cw = st.bw * 8;
  f.ch = st.bh * 8;
  f.w64 = (st.width + 63) / 64;
  for (int c = 0; c < 3; ++c) {
    f.lf_quant[c] = static_cast<int32_t*>(plane_ptr(st.lf_quant[c]));
    f.lf[c] = static_cast<float*>(plane_ptr(st.lf[c]));
    f.coeff[c] = static_cast<uint32_t*>(plane_ptr(st.coeff[c]));
  }
  f.x_from_y = static_cast<int32_t*>(plane_ptr(st.x_from_y));
  f.b_from_y = static_cast<int32_t*>(plane_ptr(st.b_from_y));
  f.sharpness = static_cast<int32_t*>(plane_ptr(st.sharpness));
  f.blk_type = static_cast<int32_t*>(plane_ptr(st.blk_type));
  f.blk_mul = static_cast<int32_t*>(plane_ptr(st.blk_mul));
  f.epf_sigma = static_cast<float*>(plane_ptr(st.epf_sigma));
  f.group_blocks = st.group_dim / 8;
  for (int c = 0; c < 3; ++c) f.hshift[c] = uint8_t(st.hshift[c]), f.vshift[c] = uint8_t(st.vshift[c]);
  f.subsampled = st.subsampled ? 1 : 0;
  return f;
}

DevFusedFilterParams fused_filter_params(const RestorationFilter& rf, const float* sigma, uint32_t sigma_stride,
                                         const ColorParams* colour) {
  DevFusedFilterParams p;
  std::memset(&p, 0, sizeof(p));
  p.gab_enabled = rf.gab_enabled ? 1 : 0;
  for (int c = 0; c < 3; ++c) {
    p.gab_w[c][0] = rf.gab_weights[c][0];
    p.gab_w[c][1] = rf.gab_weights[c][1];
    p.epf.channel_scale[c] = rf.epf.channel_scale[c];
  }
  p.epf_iters = int(rf.epf.iters);
  p.epf.pass0_sigma_scale = rf.epf.pass0_sigma_scale;
  p.epf.pass2_sigma_scale = rf.epf.pass2_sigma_scale;
  p.epf.border_sad_mul = rf.epf.border_sad_mul;
  p.epf.sigma_for_modular = rf.epf.sigma_for_modular;
  p.sigma = sigma;
  p.sigma_stride = sigma_stride;
  if (colour) {  // sRGB-gamut targets only: second_stage, gamma and PQ stay off
    p.colour = 1;
    for (int i = 0; i < 3; ++i) {
      p.col.opsin_bias[i] = colour->opsin_bias[i];
      p.col.cbrt_opsin_bias[i] = colour->cbrt_opsin_bias[i];
    }
    p.col.itscale = colour->itscale;
    for (int i = 0; i < 9; ++i) p.col.matrix[i] = colour->matrix[i];
    p.col.apply_srgb_tf = colour->apply_srgb_tf ? 1 : 0;
    p.col.apply_bt709_tf = colour->apply_bt709_tf ? 1 : 0;
  }
  return p;
}

}  // namespace jxlb
