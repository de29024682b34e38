// C ABI of the Modular-frame path (jxg_modular_*, include/jxg.h): batches of Modular frames whose ModularHF
// sections are decoded on the GPU (modular_kernels.cu). Host work: the front end (modular_frame.cc) and the staging
// of tables, sections and the host-decoded small channels into one pinned blob.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <functional>
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <utility>
#include <vector>

#include "../../../include/jxg.h"
#include "../host/lf_frame.h"
#include "../host/modular_frame.h"
#include "../host/modular_region.h"
#include "batch_common.h"
#include "modular_device.h"

using namespace jxgpu;
using namespace jxgpu::detail;

namespace {

struct MFrame {
  jxg::ModularFrameState* ms = nullptr;
  jxg::LfFrameState* lf = nullptr;  // a thumbnail of a VarDCT frame (jxg_modular_batch_add_lf); ms is null then
  void* out;
  size_t out_stride;
  bool out_is_device;
  bool region = false;             // a region of the frame (jxg_modular_batch_add_region)
  size_t out_row_bytes = 0, out_rows = 0;  // the output's rows as the store writes them
  size_t store_index = 0;          // its job in store_jobs, or in lf_store_jobs for a thumbnail
  jxg::ModularRegionPlan plan;     // the cone: per buffer the rectangle the arena holds, the streams decoded
  uint64_t arena_base = 0;         // element offset of this frame's planes
  std::vector<uint64_t> buf_off;   // per plan buffer, element offset in the arena of its arena rectangle's top-left
  uint64_t host_planes_blob = 0;   // blob offset of the packed host-decoded planes
  uint64_t host_planes_elems = 0;
  size_t dev_out_off = 0;
};

// Non-empty group-stream rects by the channel walk the decode kernel takes for them: the generic tree walk, the table
// walk without a property (a single leaf) or over property p (2..15); of the table rects, those whose stream uses WP.
struct WalkStats {
  uint32_t generic = 0, single = 0, by_prop[16] = {}, table_wp = 0;
};

// Device buffers: the context's pools; tables: in its pinned blob. A steady-state loop of batches allocates nothing.
struct ModularBatch : BatchCore {
  std::vector<MFrame> frames;
  std::vector<MStreamDev> streams;
  std::vector<uint32_t> order, rct_streams;
  std::vector<MRectDev> rects;
  std::vector<CodeDev> codes;
  std::vector<MRctDev> rcts;
  std::vector<uint32_t> refs;
  std::vector<std::vector<MJobDev>> levels;  // jobs grouped by plan step index
  std::vector<jxg::ModularJobKind> level_kind;
  std::vector<MJobDev> store_jobs;
  std::vector<MJobDev> lf_dequant_jobs, lf_smooth_jobs, lf_store_jobs;  // thumbnails: one job per LF stream / frame
  uint64_t arena_elems = 0, wp_bytes = 0, out_bytes = 0;
  uint64_t lz_window_elems = 0;             // symbol windows of the LZ77 streams, one per stream
  uint32_t lz77_streams = 0, rle_streams = 0;  // streams with LZ77; of those, streams whose copies all have distance 1
  uint32_t num_plain = 0;                   // streams without LZ77: the first ones of `order`
  WalkStats walks;                          // routes of the non-empty group-stream rects (jxg_modular_batch_walk_stats)
  uint32_t lanes_per_warp = 1;
  cudaEvent_t ev_decode = nullptr;
  struct {  // byte offsets of the batch tables in the blob
    uint64_t streams = 0, order = 0, rct_streams = 0, rects = 0, codes = 0, rcts = 0, refs = 0, jobs = 0;
  } tab;
};

uint64_t blob_append(ModularBatch* b, const void* p, size_t bytes, size_t align = 16, size_t tail = 0) {
  int64_t o = b->ctx->blob.append(p, bytes, align, tail);
  if (o < 0) throw jxg::Error(JXG_ERR_CUDA, "pinned staging allocation failed");
  return uint64_t(o);
}

uint32_t add_code(ModularBatch* b, const jxg::EntropyCode& c) {
  CodeDev d;
  memset(&d, 0, sizeof(d));
  if (c.lz77_enabled) {
    d.lz_enabled = 1;
    d.lz_min_symbol = c.lz77_min_symbol;
    d.lz_min_length = c.lz77_min_length;
    d.lz_len_cfg = c.lz77_length_uint.packed();
    d.lz_dist_cluster = c.lz_dist_cluster;
  }
  d.use_prefix = c.use_prefix;
  d.log_alpha = c.log_alpha_size;
  d.num_clusters = c.num_clusters;
  d.cmap_off = blob_append(b, c.context_map.data(), c.context_map.size());
  std::vector<uint32_t> cfg;
  for (const auto& u : c.uint_configs) cfg.push_back(u.packed());
  d.cfg_off = blob_append(b, cfg.data(), cfg.size() * 4);
  if (c.use_prefix) {
    d.huff_off = blob_append(b, c.huff_entries.data(), c.huff_entries.size() * 4);
    d.huff_offset_off = blob_append(b, c.huff_offset.data(), c.huff_offset.size() * 4);
  } else {
    d.ans_off = blob_append(b, c.ans_buckets.data(), c.ans_buckets.size() * 8);
  }
  b->codes.push_back(d);
  return uint32_t(b->codes.size() - 1);
}

uint64_t add_tree(ModularBatch* b, const jxg::ModularTree& t) {
  std::vector<int32_t> nodes(t.nodes.size() * 4);
  for (size_t i = 0; i < t.nodes.size(); i++) {
    const jxg::TreeNode& n = t.nodes[i];
    nodes[i * 4 + 0] = n.property;
    nodes[i * 4 + 1] = n.val;
    if (n.property >= 0) {
      nodes[i * 4 + 2] = int32_t(n.left);
      nodes[i * 4 + 3] = 0;
    } else {
      if (n.ctx >= (1u << 27)) throw jxg::Error(JXG_ERR_UNSUPPORTED, "MA tree too large for the device encoding");  // check_tree
      nodes[i * 4 + 2] = int32_t(n.left | (n.ctx << 4));  // predictor | ctx << 4
      nodes[i * 4 + 3] = int32_t(n.right);                // multiplier
    }
  }
  return blob_append(b, nodes.data(), nodes.size() * 4, 16);
}

// Table form of a channel's tree walk (see modular_device.h). Returns false when the channel needs the generic walk.
// `root`: first node whose decision is not on the channel index / stream id. Keys of the cache: (tree, root).
struct WalkKey {
  uint64_t tree_off;
  uint32_t root, ci;
  uint64_t stream_id;
  bool operator<(const WalkKey& o) const {
    return std::tie(tree_off, root, ci, stream_id) < std::tie(o.tree_off, o.root, o.ci, o.stream_id);
  }
};

// Does the tree decide on the channel index / stream id (properties 0 / 1) below a split on another property?
bool has_inner_static(const jxg::ModularTree& t) {
  std::vector<std::pair<uint32_t, bool>> stack{{0u, false}};
  while (!stack.empty()) {
    auto [n, below] = stack.back();
    stack.pop_back();
    const jxg::TreeNode& nd = t.nodes[n];
    if (nd.property < 0) continue;
    const bool is_static = nd.property == 0 || nd.property == 1;
    if (is_static && below) return true;
    stack.push_back({nd.left, below || !is_static});
    stack.push_back({nd.right, below || !is_static});
  }
  return false;
}
struct WalkInfo {
  uint32_t walk;
  uint64_t lut_off;
};

uint32_t static_root(const jxg::ModularTree& t, uint32_t ci, uint64_t stream_id) {
  uint32_t n = 0;
  while (t.nodes[n].property == 0 || t.nodes[n].property == 1) {
    const int64_t v = t.nodes[n].property == 0 ? int64_t(ci) : int64_t(int32_t(uint32_t(stream_id)));
    n = v > int64_t(t.nodes[n].val) ? t.nodes[n].left : t.nodes[n].right;
  }
  return n;
}

bool build_walk_table(const jxg::ModularTree& t, uint32_t root, uint32_t ci, uint64_t stream_id, std::vector<uint32_t>& lut,
                      uint32_t& prop, uint32_t& single) {
  struct Item {
    int32_t lo, hi;  // [lo, hi)
    uint32_t node;
  };
  auto entry = [&](uint32_t node, uint32_t& e) {
    const jxg::TreeNode& n = t.nodes[node];
    if (node >= (1u << 16) || n.ctx >= t.code.context_map.size()) return false;
    const uint32_t cluster = t.code.context_map[n.ctx];
    const bool plain = n.val == 0 && n.right == 1;
    e = (n.left & 15u) | (cluster << 4) | (plain ? 1u << 12 : 0u) | (node << 16);
    return true;
  };
  prop = kLutNoProperty;
  lut.assign(kLutSize, 0);
  std::vector<Item> stack{Item{kLutMin, kLutMin + kLutSize, root}};
  bool any_split = false;
  while (!stack.empty()) {
    Item it = stack.back();
    stack.pop_back();
    uint32_t node = it.node;
    // decisions on the channel / stream below other splits are still constant
    while (t.nodes[node].property == 0 || t.nodes[node].property == 1) {
      const int64_t v = t.nodes[node].property == 0 ? int64_t(ci) : int64_t(int32_t(uint32_t(stream_id)));
      node = v > int64_t(t.nodes[node].val) ? t.nodes[node].left : t.nodes[node].right;
    }
    const jxg::TreeNode& n = t.nodes[node];
    if (n.property < 0) {
      uint32_t e;
      if (!entry(node, e)) return false;
      for (int32_t v = it.lo; v < it.hi; v++) lut[size_t(v - kLutMin)] = e;
      single = e;
      continue;
    }
    if (n.property < 2 || n.property > 15) return false;  // properties of previous channels: generic walk
    if (prop == kLutNoProperty) prop = uint32_t(n.property);
    else if (prop != uint32_t(n.property)) return false;
    // values beyond the table are clamped to its ends: the decision must not change there
    if (n.val < kLutMin || n.val > kLutMin + kLutSize - 2) return false;
    any_split = true;
    const int32_t first_left = n.val + 1;  // v > val -> left child
    if (first_left < it.hi) stack.push_back(Item{std::max(first_left, it.lo), it.hi, n.left});
    if (first_left > it.lo) stack.push_back(Item{it.lo, std::min(first_left, it.hi), n.right});
  }
  if (!any_split) prop = kLutNoProperty;
  return true;
}

// Everything add_frame appends to, so that a refused frame leaves the batch as it was (jxg_modular_batch_add).
struct BatchMark {
  size_t frames, streams, rct_streams, rects, codes, rcts, refs, levels, store_jobs, lf_dequant_jobs, lf_smooth_jobs,
      lf_store_jobs, blob, blob_pending;
  std::vector<size_t> level_jobs;
  uint64_t arena_elems, wp_bytes, out_bytes, lz_window_elems;
  uint32_t lz77_streams, rle_streams;
  WalkStats walks;

  explicit BatchMark(const ModularBatch* b)
      : frames(b->frames.size()), streams(b->streams.size()), rct_streams(b->rct_streams.size()), rects(b->rects.size()),
        codes(b->codes.size()), rcts(b->rcts.size()), refs(b->refs.size()), levels(b->levels.size()),
        store_jobs(b->store_jobs.size()), lf_dequant_jobs(b->lf_dequant_jobs.size()),
        lf_smooth_jobs(b->lf_smooth_jobs.size()), lf_store_jobs(b->lf_store_jobs.size()), blob(b->ctx->blob.size), blob_pending(b->ctx->blob.pending.size()),
        arena_elems(b->arena_elems), wp_bytes(b->wp_bytes), out_bytes(b->out_bytes), lz_window_elems(b->lz_window_elems),
        lz77_streams(b->lz77_streams), rle_streams(b->rle_streams), walks(b->walks) {
    for (const auto& l : b->levels) level_jobs.push_back(l.size());
  }
  void restore(ModularBatch* b) const {
    b->frames.resize(frames);
    b->streams.resize(streams);
    b->rct_streams.resize(rct_streams);
    b->rects.resize(rects);
    b->codes.resize(codes);
    b->rcts.resize(rcts);
    b->refs.resize(refs);
    b->levels.resize(levels);
    b->level_kind.resize(levels);
    for (size_t l = 0; l < levels; l++) b->levels[l].resize(level_jobs[l]);
    b->store_jobs.resize(store_jobs);
    b->lf_dequant_jobs.resize(lf_dequant_jobs);
    b->lf_smooth_jobs.resize(lf_smooth_jobs);
    b->lf_store_jobs.resize(lf_store_jobs);
    b->ctx->blob.size = blob;
    b->ctx->blob.pending.resize(blob_pending);
    b->arena_elems = arena_elems;
    b->wp_bytes = wp_bytes;
    b->out_bytes = out_bytes;
    b->lz_window_elems = lz_window_elems;
    b->lz77_streams = lz77_streams;
    b->rle_streams = rle_streams;
    b->walks = walks;
  }
};

// Element index of pixel (x, y) of plan buffer i: its arena rectangle starts at buf_off[i], rows of the rectangle's width.
uint32_t buf_stride(const MFrame& f, size_t i) { return f.plan.arena[i].w(); }
int64_t buf_origin(const MFrame& f, size_t i) {  // the index of pixel (0, 0), outside the rectangle unless it starts there
  const jxg::PlaneRect& r = f.plan.arena[i];
  return int64_t(f.buf_off[i]) - int64_t(r.y0) * r.w() - int64_t(r.x0);
}
uint64_t buf_index(const MFrame& f, size_t i, uint32_t x, uint32_t y) { return uint64_t(buf_origin(f, i) + int64_t(y) * buf_stride(f, i) + x); }

// Plane arena: per plan buffer its arena rectangle (the whole plane for a whole frame); host-decoded coded channels first
// (one contiguous copy from the blob of their rectangles), then the rest.
void add_arena(ModularBatch* b, MFrame& f) {
  const jxg::ModularFrameState* ms = f.ms;
  const std::vector<jxg::PlaneRect>& ar = f.plan.arena;
  f.arena_base = b->arena_elems;
  f.buf_off.assign(ms->bufs.size(), 0);
  uint64_t cursor = f.arena_base;
  for (size_t c = 0; c < ms->coded.size(); c++)
    if (ms->host_decoded[c]) {
      f.buf_off[c] = cursor;
      cursor += uint64_t(ar[c].w()) * ar[c].h();
    }
  f.host_planes_elems = cursor - f.arena_base;
  for (size_t i = 0; i < ms->bufs.size(); i++)
    if (i >= ms->coded.size() || !ms->host_decoded[i]) {
      cursor = (cursor + 3) & ~uint64_t(3);
      f.buf_off[i] = cursor;
      cursor += uint64_t(ar[i].w()) * ar[i].h();
    }
  b->arena_elems = (cursor + 63) & ~uint64_t(63);
  if (f.host_planes_elems) {
    f.host_planes_blob = blob_append(b, nullptr, 0, 16);
    for (size_t c = 0; c < ms->coded.size(); c++) {
      const jxg::ModularChannel& ch = ms->coded[c];
      if (!ms->host_decoded[c] || ar[c].empty() || ch.data.empty()) continue;
      if (ar[c].w() == ch.w) {
        blob_append(b, ch.row(ar[c].y0), size_t(ch.w) * ar[c].h() * 4, 4);
      } else {
        for (uint32_t y = ar[c].y0; y < ar[c].y1; y++) blob_append(b, ch.row(y) + ar[c].x0, size_t(ar[c].w()) * 4, 4);
      }
    }
  }
}

// What jxg_modular_batch_add refuses in any group stream, whether or not a region decodes it.
void check_tree(const jxg::ModularTree& t) {
  for (const jxg::TreeNode& n : t.nodes)
    if (n.property < 0 && n.ctx >= (1u << 27)) throw jxg::Error(JXG_ERR_UNSUPPORTED, "MA tree too large for the device encoding");
}
void check_streams(const std::vector<jxg::ModularGroupStream>& hf, const jxg::ModularTree& global_tree) {
  for (const jxg::ModularGroupStream& st : hf) {
    if (st.empty) continue;
    check_tree(st.local_tree ? *st.local_tree : global_tree);
    for (const jxg::ModularTransform& t : st.header.transforms) {
      if (t.id != 0) throw jxg::Error(JXG_ERR_UNSUPPORTED, "only RCT is implemented as a group-local transform on the device path");
      if (t.begin_channel + 3 > st.rects.size()) throw jxg::Error(jxg::kErrBitstream, "RCT channel range");
      const jxg::ModularRect &r0 = st.rects[t.begin_channel], &r1 = st.rects[t.begin_channel + 1], &r2 = st.rects[t.begin_channel + 2];
      if (r0.w != r1.w || r0.w != r2.w || r0.h != r1.h || r0.h != r2.h) throw jxg::Error(jxg::kErrBitstream, "RCT on channels of different size");
    }
  }
}

// The group streams of one frame of the batch: its section bytes, its channels (their shifts decide which rects are
// reference channels), the global tree, the streams decoded (null: all) and where a rect lives in the plane arena.
struct StreamSource {
  const uint8_t* codestream;
  const std::vector<jxg::ModularGroupStream>& hf;
  const std::vector<jxg::ModularChannel>& coded;
  const jxg::ModularTree& global_tree;
  const std::vector<uint8_t>* selected;
  std::function<void(const jxg::ModularRect&, uint32_t& stride, uint64_t& base)> addr;
};

// Codes / trees, and per selected group stream its MStreamDev, rects, reference channels, local RCTs and LZ77 window.
// The stream keeps its index in src.hf (the whole-frame group index).
void add_streams(ModularBatch* b, const StreamSource& src) {
  uint32_t global_code = 0;
  uint64_t global_tree = 0;
  bool have_global = false;
  std::map<WalkKey, WalkInfo> walk_cache;
  std::map<uint64_t, bool> inner_static;
  for (size_t g = 0; g < src.hf.size(); g++) {
    const jxg::ModularGroupStream& st = src.hf[g];
    if (src.selected && !(*src.selected)[g]) continue;
    const jxg::ModularTree* tree = st.local_tree ? st.local_tree.get() : &src.global_tree;
    MStreamDev d;
    memset(&d, 0, sizeof(d));
    if (st.local_tree) {
      d.code = add_code(b, tree->code);
      d.tree_off = add_tree(b, *tree);
    } else {
      if (!have_global) {
        global_code = add_code(b, tree->code);
        global_tree = add_tree(b, *tree);
        have_global = true;
      }
      d.code = global_code;
      d.tree_off = global_tree;
    }
    d.frame = uint32_t(b->frames.size());
    d.group = st.group;
    d.sec_off = blob_append(b, src.codestream + st.sec_off, st.sec_len, 8, 24);
    d.sec_len = st.sec_len;
    d.data_bitpos = uint32_t(st.data_bitpos);
    d.stream_id = uint32_t(st.stream_id);
    d.uses_wp = tree->uses_wp;
    const jxg::WeightedHeader& wp = st.header.wp;
    const uint32_t wpp[11] = {wp.p1c, wp.p2c, wp.p3ca, wp.p3cb, wp.p3cc, wp.p3cd, wp.p3ce, wp.w[0], wp.w[1], wp.w[2], wp.w[3]};
    memcpy(d.wp_params, wpp, sizeof(wpp));
    d.first_rect = uint32_t(b->rects.size());
    d.num_rects = uint32_t(st.rects.size());
    uint32_t max_w = 0;
    for (size_t ri = 0; ri < st.rects.size(); ri++) {
      const jxg::ModularRect& r = st.rects[ri];
      MRectDev rd;
      src.addr(r, rd.stride, rd.base);
      rd.w = r.w;
      rd.h = r.h;
      rd.walk = kWalkGeneric;
      rd.lut_off = 0;
      if (r.w && r.h) {
        const uint32_t root = static_root(*tree, uint32_t(ri), st.stream_id);
        // channel / stream decisions below another split make the table specific to this channel of this stream
        auto is_it = inner_static.find(d.tree_off);
        if (is_it == inner_static.end()) is_it = inner_static.emplace(d.tree_off, has_inner_static(*tree)).first;
        const WalkKey key{d.tree_off, root, is_it->second ? uint32_t(ri) : ~0u, is_it->second ? st.stream_id : ~uint64_t(0)};
        auto it = walk_cache.find(key);
        if (it == walk_cache.end()) {
          std::vector<uint32_t> lut;
          uint32_t prop = kLutNoProperty, single = 0;
          WalkInfo wi{kWalkGeneric, 0};
          if (build_walk_table(*tree, root, uint32_t(ri), st.stream_id, lut, prop, single)) {
            wi.walk = kWalkLut | (prop << 8);
            wi.lut_off = prop == kLutNoProperty ? uint64_t(single) : blob_append(b, lut.data(), lut.size() * 4, 16);
          }
          it = walk_cache.emplace(key, wi).first;
        }
        rd.walk = it->second.walk;
        rd.lut_off = it->second.lut_off;
        if ((rd.walk & 0xff) != kWalkLut) {
          b->walks.generic++;
        } else {
          if ((rd.walk >> 8) == kLutNoProperty) b->walks.single++;
          else b->walks.by_prop[(rd.walk >> 8) & 15]++;
          if (d.uses_wp) b->walks.table_wp++;
        }
      }
      // reference channels: earlier channels of the stream with the same shape, nearest first (common.rs:52-60)
      rd.ref_first = uint32_t(b->refs.size());
      if (tree->num_properties > 16)
        for (size_t k = ri; k-- > 0;) {
          const jxg::ModularRect& q = st.rects[k];
          if (q.w == r.w && q.h == r.h && src.coded[q.chan].hshift == src.coded[r.chan].hshift &&
              src.coded[q.chan].vshift == src.coded[r.chan].vshift)
            b->refs.push_back(d.first_rect + uint32_t(k));
        }
      rd.ref_count = uint32_t(b->refs.size()) - rd.ref_first;
      b->rects.push_back(rd);
      max_w = std::max(max_w, r.w);
    }
    if (d.uses_wp) {
      d.wp_scratch_off = b->wp_bytes;
      b->wp_bytes += (size_t(max_w + 1) * (8 + 2) * 4 + 63) & ~size_t(63);
    }
    d.first_rct = uint32_t(b->rcts.size());
    for (const jxg::ModularTransform& t : st.header.transforms) b->rcts.push_back(MRctDev{t.begin_channel, t.rct_type});  // check_streams
    d.num_rct = uint32_t(b->rcts.size()) - d.first_rct;
    if (d.num_rct) b->rct_streams.push_back(uint32_t(b->streams.size()));
    if (tree->code.lz77_enabled) {
      uint64_t pixels = 0;
      for (const jxg::ModularRect& r : st.rects) pixels += uint64_t(r.w) * r.h;
      d.dist_multiplier = st.dist_multiplier;
      d.lz_window_off = b->lz_window_elems;
      b->lz_window_elems += std::min<uint64_t>(pixels, uint64_t(1) << 20);  // one symbol per pixel
      b->lz77_streams++;
      if (tree->code.is_rle()) b->rle_streams++;
    }
    b->streams.push_back(d);
  }
}

void set_rect(MJobDev& j, const jxg::PlaneRect& r) {
  j.x0 = r.x0;
  j.y0 = r.y0;
  j.x1 = r.x1;
  j.y1 = r.y1;
}

// Global inverse plan -> jobs per level, each on the rectangle the cone gives its step; a step the region does not
// need has no job. A frame with fewer steps than the batch has levels has no jobs in the last ones; levels are launched
// in order and the store runs after all of them, so only the kinds of the common steps must agree, whatever the order
// of adding.
void add_plan(ModularBatch* b, const MFrame& f) {
  const jxg::ModularFrameState* ms = f.ms;
  for (size_t si = 0; si < ms->steps.size(); si++) {
    const jxg::ModularStep& s = ms->steps[si];
    if (b->levels.size() <= si) {
      b->levels.emplace_back();
      b->level_kind.push_back(s.kind);
    }
    if (b->level_kind[si] != s.kind)
      throw jxg::Error(JXG_ERR_UNSUPPORTED, "frames of one Modular batch must share the global transform structure");
    MJobDev j;
    memset(&j, 0, sizeof(j));
    j.a = buf_origin(f, s.a);
    j.b = buf_origin(f, s.b);
    j.c = buf_origin(f, s.c);
    j.sa = buf_stride(f, s.a);
    j.sb = buf_stride(f, s.b);
    j.sc = buf_stride(f, s.c);
    j.w = ms->bufs[s.a].w;
    j.h = ms->bufs[s.a].h;
    j.rw = s.kind == jxg::kJobHSqueeze ? ms->bufs[s.b].w : (s.kind == jxg::kJobVSqueeze ? ms->bufs[s.b].h : 0);
    j.op = s.rct_op;
    if (s.kind == jxg::kJobPalette) {  // one job per colour channel: a index plane, b palette plane (row c = component c), c output
      if (ms->bufs[s.b].h < s.n || ms->bufs[s.b].w < s.num_colors) throw jxg::Error(jxg::kErrBitstream, "palette channel smaller than its header says");
      for (uint32_t c = 0; c < s.n; c++) {
        if (f.plan.need[s.c + c].empty()) continue;
        j.c = buf_origin(f, s.c + c);
        j.sc = buf_stride(f, s.c + c);
        set_rect(j, f.plan.need[s.c + c]);
        j.rw = s.num_colors;
        j.op = c;
        b->levels[si].push_back(j);
      }
      continue;
    }
    if (f.plan.step[si].empty()) continue;
    set_rect(j, f.plan.step[si]);
    b->levels[si].push_back(j);
  }
}

// Store job: the coded window of the final colour planes -> the u8 output, in the file's orientation (render/save.rs).
void add_store(ModularBatch* b, MFrame& f) {
  const jxg::ModularFrameState* ms = f.ms;
  const uint32_t W = ms->header.xsize(), H = ms->header.ysize();
  MJobDev sj;
  memset(&sj, 0, sizeof(sj));
  const uint32_t nc = ms->num_color_channels;
  const uint32_t ob[3] = {ms->out_buf[0], ms->out_buf[nc > 1 ? 1 : 0], ms->out_buf[nc > 2 ? 2 : 0]};
  sj.a = buf_origin(f, ob[0]);
  sj.b = buf_origin(f, ob[1]);
  sj.c = buf_origin(f, ob[2]);
  sj.sa = buf_stride(f, ob[0]);
  sj.sb = buf_stride(f, ob[1]);
  sj.sc = buf_stride(f, ob[2]);
  set_rect(sj, f.plan.coded);
  sj.w = W;
  sj.h = H;
  sj.op = ms->file.orientation;
  sj.out_x = f.plan.out_x;
  sj.out_y = f.plan.out_y;
  f.out_row_bytes = size_t(f.plan.out_w) * 3;
  f.out_rows = f.plan.out_h;
  if (!f.out_is_device) {
    f.dev_out_off = b->out_bytes;
    b->out_bytes += (f.out_row_bytes * f.out_rows + 255) & ~size_t(255);
  }
  f.store_index = b->store_jobs.size();
  b->store_jobs.push_back(sj);
}

// The frame checks of jxg_modular_batch_add, for the whole frame and for any region of it alike.
void check_frame(const jxg::ModularFrameState* ms) {
  if (!ms->device_plan_ok)
    throw jxg::Error(JXG_ERR_UNSUPPORTED, "palette transforms with delta entries or a predictor are not implemented on the device path");
  if (ms->toc.offsets.size() == 1 && !ms->hf[0].empty)
    throw jxg::Error(JXG_ERR_UNSUPPORTED, "single-section Modular frames with a coded group are not on the device path");
}
void check_plan(const jxg::ModularFrameState* ms) {
  check_streams(ms->hf, ms->global_tree);
  for (const jxg::ModularStep& s : ms->steps)
    if (s.kind == jxg::kJobPalette && (ms->bufs[s.b].h < s.n || ms->bufs[s.b].w < s.num_colors))
      throw jxg::Error(jxg::kErrBitstream, "palette channel smaller than its header says");
  const uint32_t W = ms->header.xsize(), H = ms->header.ysize();
  for (uint32_t c = 0; c < ms->num_color_channels; c++)
    if (ms->bufs[ms->out_buf[c]].w != W || ms->bufs[ms->out_buf[c]].h != H)
      throw jxg::Error(jxg::kErrBitstream, "unexpected output channel size");
}

// The cone of `region` (nullptr: the whole frame), after the frame checks; throws what jxg_modular_batch_add refuses.
void plan_frame(const jxg::ModularFrameState* ms, const JxgRegion* region, jxg::ModularRegionPlan& plan) {
  const char* why = "";
  if (int r = jxg::plan_modular_region(*ms, region, plan, &why)) throw jxg::Error(r, why);
  check_frame(ms);
}

void add_frame(ModularBatch* b, jxg::ModularFrameState* ms, const JxgRegion* region, void* out, size_t stride, bool is_device) {
  MFrame f;
  plan_frame(ms, region, f.plan);
  if (stride < size_t(f.plan.out_w) * 3) throw jxg::Error(JXG_ERR_INVALID_OUTPUT, "output row stride too small");
  check_plan(ms);
  f.ms = ms;
  f.region = region != nullptr;
  f.out = out;
  f.out_stride = stride;
  f.out_is_device = is_device;
  add_arena(b, f);
  add_streams(b, StreamSource{ms->codestream.data(), ms->hf, ms->coded, ms->global_tree, &f.plan.selected,
                              [&f](const jxg::ModularRect& r, uint32_t& stride, uint64_t& base) {
                                stride = buf_stride(f, r.chan);
                                base = buf_index(f, r.chan, r.x0, r.y0);
                              }});
  add_plan(b, f);
  add_store(b, f);
  b->frames.push_back(std::move(f));
}

// A thumbnail: the frame's LF streams decode into three i32 planes of xb x yb (Y, X, B); each stream's dequantisation
// job writes its rectangle of the f32 planes X, Y, B; the smoothing (when the frame applies it) writes them to a second
// f32 plane set; the store reads the last set.
void add_lf(ModularBatch* b, jxg::LfFrameState* lp, uint32_t format, void* out, size_t stride, bool is_device) {
  jxg::FrameState& fs = lp->fs;
  const size_t bpp = format_bpp(format);
  if (!bpp) throw jxg::Error(JXG_ERR_ARGUMENT, "unknown output format");
  const uint32_t w = fs.xb, h = fs.yb;
  const bool planar = format == JXG_FORMAT_XYB_F32_PLANAR;
  const uint32_t orientation = planar || fs.file.orientation == 0 ? 1u : fs.file.orientation;
  const uint32_t disp_w = orientation >= 5 ? h : w, disp_h = orientation >= 5 ? w : h;
  if (int r = check_output(bpp, disp_w, stride, out, is_device)) throw jxg::Error(r, g_error);
  check_streams(lp->streams, fs.global_tree);
  MFrame f;
  f.lf = lp;
  f.out = out;
  f.out_stride = stride;
  f.out_is_device = is_device;
  f.out_row_bytes = size_t(disp_w) * bpp;
  f.out_rows = planar ? size_t(3) * h : disp_h;
  const uint64_t plane = uint64_t(w) * h;
  const bool smooth = fs.header.adaptive_lf_smoothing();
  f.arena_base = b->arena_elems;
  const uint64_t q = f.arena_base, dq = q + 3 * plane, sm = dq + 3 * plane;
  b->arena_elems = (f.arena_base + (smooth ? 9 : 6) * plane + 63) & ~uint64_t(63);
  add_streams(b, StreamSource{fs.codestream.data(), lp->streams, lp->coded, fs.global_tree, nullptr,
                              [&](const jxg::ModularRect& r, uint32_t& s, uint64_t& base) {
                                s = w;
                                base = q + r.chan * plane + uint64_t(r.y0) * w + r.x0;
                              }});
  MJobDev j;
  memset(&j, 0, sizeof(j));
  j.sa = w;
  j.w = w;
  j.h = h;
  j.a = int64_t(q);
  j.c = int64_t(dq);
  for (size_t k = 0; k < lp->streams.size(); k++) {
    const jxg::LfDequantFactors lf = jxg::lf_dequant_factors(fs, lp->mul[k]);
    const MLfDequantDev p{{lf.fac[0], lf.fac[1], lf.fac[2]}, lf.cfl_x, lf.cfl_b};
    j.params = blob_append(b, &p, sizeof(p));
    const jxg::ModularRect& r = lp->streams[k].rects[0];
    set_rect(j, jxg::PlaneRect{r.x0, r.y0, r.x0 + r.w, r.y0 + r.h});
    b->lf_dequant_jobs.push_back(j);
  }
  MLfFrameDev p;
  memset(&p, 0, sizeof(p));
  jxg::lf_smoothing_factors(fs, p.lf_factors);
  JxgFrameDesc d;
  fs.fill_desc(&d, format);
  set_output_colour(p, &d);
  j.params = blob_append(b, &p, sizeof(p));
  set_rect(j, jxg::PlaneRect{0, 0, w, h});
  if (smooth) {
    j.a = int64_t(dq);
    j.c = int64_t(sm);
    b->lf_smooth_jobs.push_back(j);
  }
  j.a = int64_t(smooth ? sm : dq);
  j.c = 0;
  j.op = orientation;
  if (!is_device) {
    f.dev_out_off = b->out_bytes;
    b->out_bytes += (f.out_row_bytes * f.out_rows + 255) & ~size_t(255);
  }
  f.store_index = b->lf_store_jobs.size();
  b->lf_store_jobs.push_back(j);
  b->frames.push_back(std::move(f));
}

int launch_all(ModularBatch* b, cudaStream_t s, bool copy_to_host) {
  Context* cx = b->ctx;
  MBatchDev B;
  memset(&B, 0, sizeof(B));
  B.blob = static_cast<const uint8_t*>(cx->d_blob.p);
  B.streams = reinterpret_cast<const MStreamDev*>(B.blob + b->tab.streams);
  B.order = reinterpret_cast<const uint32_t*>(B.blob + b->tab.order);
  B.rct_streams = reinterpret_cast<const uint32_t*>(B.blob + b->tab.rct_streams);
  B.rects = reinterpret_cast<const MRectDev*>(B.blob + b->tab.rects);
  B.codes = reinterpret_cast<const CodeDev*>(B.blob + b->tab.codes);
  B.rcts = reinterpret_cast<const MRctDev*>(B.blob + b->tab.rcts);
  B.refs = reinterpret_cast<const uint32_t*>(B.blob + b->tab.refs);
  B.planes = static_cast<int32_t*>(cx->d_planes_a.p);
  B.wp_scratch = static_cast<uint8_t*>(cx->d_modular_wp.p);
  B.status = static_cast<int32_t*>(cx->d_status.p);
  B.queue = reinterpret_cast<uint32_t*>(B.status + b->streams.size());
  B.num_streams = uint32_t(b->streams.size());
  B.lz_window = static_cast<uint32_t*>(cx->d_modular_lzwin.p);
  // host-decoded planes: blob -> arena (device to device)
  for (const MFrame& f : b->frames)
    if (f.host_planes_elems)
      CUDA_TRY(cudaMemcpyAsync(B.planes + f.arena_base, B.blob + f.host_planes_blob, f.host_planes_elems * 4,
                               cudaMemcpyDeviceToDevice, s));
  b->launches = uint64_t(
      launch_modular_decode(B, b->num_plain, b->lanes_per_warp, uint32_t(b->rct_streams.size()), schedule_sms(cx), s));
  CUDA_TRY(cudaEventRecord(b->ev_decode, s));
  const MJobDev* jobs = reinterpret_cast<const MJobDev*>(B.blob + b->tab.jobs);  // the levels in order, then the stores
  auto launch_jobs = [&](jxg::ModularJobKind kind, const std::vector<MJobDev>& level) {
    uint32_t mw = 0, mh = 0;
    for (const MJobDev& j : level) {
      mw = std::max(mw, j.x1 - j.x0);
      mh = std::max(mh, j.y1 - j.y0);
    }
    launch_modular_jobs(kind, jobs, uint32_t(level.size()), mw, mh, B.planes, B.blob, schedule_sms(cx), s);
    jobs += level.size();
    b->launches++;
  };
  for (size_t l = 0; l < b->levels.size(); l++) launch_jobs(b->level_kind[l], b->levels[l]);
  // the jobs of the Modular frames' stores, then the thumbnails' jobs in stage order (each kind waits for the one before)
  const std::pair<jxg::ModularJobKind, const std::vector<MJobDev>*> tail[4] = {
      {jxg::kJobStore, &b->store_jobs}, {jxg::kJobLfDequant, &b->lf_dequant_jobs},
      {jxg::kJobLfSmooth, &b->lf_smooth_jobs}, {jxg::kJobLfStore, &b->lf_store_jobs}};
  for (const auto& [kind, list] : tail)
    if (!list->empty()) launch_jobs(kind, *list);
  if (copy_to_host) {
    for (const MFrame& f : b->frames)
      if (!f.out_is_device) {
        CUDA_TRY(cudaMemcpy2DAsync(f.out, f.out_stride, static_cast<uint8_t*>(cx->d_out.p) + f.dev_out_off, f.out_row_bytes,
                                   f.out_row_bytes, f.out_rows, cudaMemcpyDeviceToHost, s));
        b->d2h += f.out_row_bytes * f.out_rows;
      }
  }
  CUDA_TRY(cudaMemcpyAsync(b->status_host, cx->d_status.p, b->status_n * 4, cudaMemcpyDeviceToHost, s));
  CUDA_TRY(cudaGetLastError());
  return 0;
}

}  // namespace

extern "C" {

int jxg_modular_parse_file(const uint8_t* data, size_t size, void** parsed, JxgImageInfo* info) {
  if (!data || !parsed) return JXG_ERR_ARGUMENT;
  try {
    auto ms = jxg::parse_modular_file(data, size);
    if (info) {  // the Modular path takes one-pass frames only (parse_modular_file)
      uint64_t hf = 0;
      for (const auto& st : ms->hf) hf += st.sec_len;
      jxg::fill_image_info(ms->file, ms->header, hf, info);
    }
    *parsed = ms.release();
    return JXG_OK;
  } catch (jxg::Error& e) {
    return set_error(e.code, e.what());
  }
}

void jxg_modular_parsed_free(void* parsed) { delete static_cast<jxg::ModularFrameState*>(parsed); }

int jxg_modular_batch_begin(void* c, void** out_batch) {
  if (!c || !out_batch) return JXG_ERR_ARGUMENT;
  auto b = std::make_unique<ModularBatch>();
  if (int r = batch_begin(*b, static_cast<Context*>(c), &b->ev_decode)) return r;
  *out_batch = b.release();
  return JXG_OK;
}

int jxg_modular_batch_add(void* bp, void* parsed, void* out, size_t out_row_stride, int out_is_device) {
  ModularBatch* b = static_cast<ModularBatch*>(bp);
  if (!b || !parsed || !out) return JXG_ERR_ARGUMENT;
  if (b->uploaded) return set_error(JXG_ERR_ARGUMENT, "batch already submitted");
  const BatchMark mark(b);
  try {
    add_frame(b, static_cast<jxg::ModularFrameState*>(parsed), nullptr, out, out_row_stride, out_is_device != 0);
    return JXG_OK;
  } catch (jxg::Error& e) {
    mark.restore(b);  // a refused frame leaves nothing behind: no streams decode for it, no stats count it
    return set_error(e.code, e.what());
  }
}

int jxg_modular_batch_add_region(void* bp, void* parsed, const JxgRegion* region, void* out, size_t out_row_stride,
                                 int out_is_device) {
  ModularBatch* b = static_cast<ModularBatch*>(bp);
  if (!b || !parsed || !region || !out) return JXG_ERR_ARGUMENT;
  if (b->uploaded) return set_error(JXG_ERR_ARGUMENT, "batch already submitted");
  const BatchMark mark(b);
  try {
    add_frame(b, static_cast<jxg::ModularFrameState*>(parsed), region, out, out_row_stride, out_is_device != 0);
    return JXG_OK;
  } catch (jxg::Error& e) {
    mark.restore(b);
    return set_error(e.code, e.what());
  }
}

int jxg_modular_batch_add_lf(void* bp, void* parsed, uint32_t output_format, void* out, size_t out_row_stride,
                             int out_is_device) {
  ModularBatch* b = static_cast<ModularBatch*>(bp);
  if (!b || !parsed || !out) return JXG_ERR_ARGUMENT;
  if (b->uploaded) return set_error(JXG_ERR_ARGUMENT, "batch already submitted");
  const BatchMark mark(b);
  try {
    add_lf(b, static_cast<jxg::LfFrameState*>(parsed), output_format, out, out_row_stride, out_is_device != 0);
    return JXG_OK;
  } catch (jxg::Error& e) {
    mark.restore(b);
    return set_error(e.code, e.what());
  }
}

int jxg_lf_parse_file(const uint8_t* data, size_t size, void** parsed, JxgImageInfo* info) {
  if (!data || !parsed) return JXG_ERR_ARGUMENT;
  try {
    std::unique_ptr<jxg::LfFrameState> lp = jxg::parse_vardct_lf_file(data, size);
    if (info) jxg::fill_image_info(lp->fs.file, lp->fs.header, lp->hf_bytes, info);
    *parsed = lp.release();
    return JXG_OK;
  } catch (jxg::Error& e) {
    return set_error(e.code, e.what());
  } catch (std::exception& e) {
    return set_error(JXG_ERR_BITSTREAM, e.what());
  }
}

void jxg_lf_parsed_free(void* parsed) { delete static_cast<jxg::LfFrameState*>(parsed); }

int jxg_modular_parsed_region_plan(void* parsed, const JxgRegion* region, uint32_t* groups, uint32_t max_groups,
                                   uint32_t* n_groups, uint32_t* rects, uint32_t max_buffers, uint32_t* n_buffers) {
  if (!parsed || !region || !n_groups || !n_buffers) return JXG_ERR_ARGUMENT;
  const jxg::ModularFrameState* ms = static_cast<const jxg::ModularFrameState*>(parsed);
  try {
    jxg::ModularRegionPlan plan;
    plan_frame(ms, region, plan);
    check_plan(ms);
    std::vector<uint32_t> sel;
    for (size_t g = 0; g < plan.selected.size(); g++)
      if (plan.selected[g]) sel.push_back(ms->hf[g].group);
    *n_groups = uint32_t(sel.size());
    *n_buffers = uint32_t(plan.need.size());
    if ((groups && max_groups < sel.size()) || (rects && max_buffers < plan.need.size()))
      return set_error(JXG_ERR_ARGUMENT, "region plan: output arrays too small");
    if (groups) std::copy(sel.begin(), sel.end(), groups);
    if (rects)
      for (size_t i = 0; i < plan.need.size(); i++) {
        const jxg::PlaneRect &a = plan.arena[i], &n = plan.need[i];
        const uint32_t v[8] = {a.x0, a.y0, a.x1, a.y1, n.x0, n.y0, n.x1, n.y1};
        std::copy(v, v + 8, rects + i * 8);
      }
    return JXG_OK;
  } catch (jxg::Error& e) {
    return set_error(e.code, e.what());
  }
}

int jxg_modular_batch_set_lanes(void* bp, int lanes_per_warp) {
  ModularBatch* b = static_cast<ModularBatch*>(bp);
  if (!b || lanes_per_warp < 1) return JXG_ERR_ARGUMENT;
  b->lanes_per_warp = uint32_t(lanes_per_warp);
  return JXG_OK;
}

int jxg_modular_batch_run(void* bp, void* cuda_stream) {
  ModularBatch* b = static_cast<ModularBatch*>(bp);
  if (!b || b->frames.empty()) return JXG_ERR_ARGUMENT;
  Context* cx = b->ctx;
  CUDA_TRY(cudaSetDevice(cx->device));
  cudaStream_t s = batch_stream(*b, cuda_stream);
  b->h2d = b->d2h = 0;
  // streams without LZ77, then those with it (each group has its own decode launch); longest section first within
  // each (the decode kernel's queue is a longest-processing-time schedule)
  b->order.resize(b->streams.size());
  for (uint32_t i = 0; i < b->order.size(); i++) b->order[i] = i;
  auto lz = [&](uint32_t i) { return b->codes[b->streams[i].code].lz_enabled != 0; };
  std::stable_sort(b->order.begin(), b->order.end(), [&](uint32_t x, uint32_t y) {
    return lz(x) != lz(y) ? lz(y) : b->streams[x].sec_len > b->streams[y].sec_len;
  });
  b->num_plain = uint32_t(b->streams.size()) - b->lz77_streams;
  if (int r = cx->d_planes_a.ensure(std::max<size_t>(b->arena_elems * 4, 16))) return r;
  if (int r = cx->d_status.ensure((b->streams.size() + 8) * 4)) return r;
  if (int r = cx->d_out.ensure(std::max<size_t>(b->out_bytes, 16))) return r;
  if (int r = cx->d_modular_wp.ensure(std::max<size_t>(b->wp_bytes, 16))) return r;
  if (b->lz_window_elems && cx->d_modular_lzwin.ensure(b->lz_window_elems * 4)) {
    cudaGetLastError();
    return set_error(JXG_ERR_UNSUPPORTED, "no device memory for the LZ77 windows of the batch (" +
                                              std::to_string(b->lz_window_elems * 4) + " bytes)");
  }
  for (MFrame& f : b->frames) {
    MJobDev& j = f.lf ? b->lf_store_jobs[f.store_index] : b->store_jobs[f.store_index];
    j.out = f.out_is_device ? f.out : static_cast<uint8_t*>(cx->d_out.p) + f.dev_out_off;
    j.out_stride = f.out_is_device ? f.out_stride : f.out_row_bytes;
  }
  if (int r = batch_status(*b, b->streams.size())) return r;
  std::vector<MJobDev> all_jobs;  // the launch order of launch_all
  for (auto& l : b->levels) all_jobs.insert(all_jobs.end(), l.begin(), l.end());
  for (const auto* l : {&b->store_jobs, &b->lf_dequant_jobs, &b->lf_smooth_jobs, &b->lf_store_jobs})
    all_jobs.insert(all_jobs.end(), l->begin(), l->end());
  PinnedArena& blob = cx->blob;
  if (!batch_table(blob, b->streams, b->tab.streams) || !batch_table(blob, b->order, b->tab.order) ||
      !batch_table(blob, b->rct_streams, b->tab.rct_streams) || !batch_table(blob, b->rects, b->tab.rects) ||
      !batch_table(blob, b->codes, b->tab.codes) || !batch_table(blob, b->rcts, b->tab.rcts) ||
      !batch_table(blob, b->refs, b->tab.refs) || !batch_table(blob, all_jobs, b->tab.jobs))
    return set_error(JXG_ERR_CUDA, "pinned staging allocation failed");
  if (int r = cx->d_blob.ensure(blob.size + 64)) return r;
  if (int r = fill_pools(cx, s, true)) return r;
  CUDA_TRY(cudaEventRecord(b->ev0, s));
  CUDA_TRY(cudaMemcpyAsync(cx->d_blob.p, blob.p, blob.size, cudaMemcpyHostToDevice, s));
  b->h2d += blob.size;
  b->uploaded = true;
  if (int r = launch_all(b, s, true)) return r;
  CUDA_TRY(cudaEventRecord(b->ev1, s));
  return JXG_OK;
}

int jxg_modular_batch_rerun_device(void* bp, void* cuda_stream) {
  ModularBatch* b = static_cast<ModularBatch*>(bp);
  if (!b || !b->uploaded) return set_error(JXG_ERR_ARGUMENT, "batch was never submitted");
  CUDA_TRY(cudaSetDevice(b->ctx->device));
  cudaStream_t s = batch_stream(*b, cuda_stream);
  CUDA_TRY(cudaStreamWaitEvent(s, b->ev1, 0));  // the previous run of this batch still owns its device buffers
  if (int r = fill_pools(b->ctx, s, false)) return r;
  CUDA_TRY(cudaEventRecord(b->ev0, s));
  if (int r = launch_all(b, s, false)) return r;
  CUDA_TRY(cudaEventRecord(b->ev1, s));
  return JXG_OK;
}

int jxg_modular_batch_wait(void* bp, uint32_t* bad_frame, uint32_t* bad_group) {
  ModularBatch* b = static_cast<ModularBatch*>(bp);
  if (!b || !b->uploaded) return JXG_ERR_ARGUMENT;
  if (int r = batch_wait_last_run(*b)) return r;
  CUDA_TRY(cudaGetLastError());
  return batch_first_failure(*b, b->streams, "Modular group stream failed: frame ", bad_frame, bad_group);
}

// Parity tap: the final colour planes (3 x H x W i32, before the u8 conversion) of frame f.
int jxg_modular_batch_read_planes(void* bp, uint32_t f, int32_t* out, size_t out_len) {
  ModularBatch* b = static_cast<ModularBatch*>(bp);
  if (!b || !b->uploaded || f >= b->frames.size() || !out) return JXG_ERR_ARGUMENT;
  if (b->frames[f].region) return set_error(JXG_ERR_ARGUMENT, "read_planes: a region frame holds no whole planes");
  if (b->frames[f].lf) return set_error(JXG_ERR_ARGUMENT, "read_planes: a thumbnail holds no Modular colour planes");
  if (int r = batch_wait_last_run(*b)) return r;
  const MJobDev& j = b->store_jobs[b->frames[f].store_index];  // a whole frame: the planes are whole, rows of width w
  const size_t n = size_t(j.w) * j.h;
  if (out_len < 3 * n) return set_error(JXG_ERR_ARGUMENT, "plane buffer too small");
  const int32_t* planes = static_cast<const int32_t*>(b->ctx->d_planes_a.p);
  CUDA_TRY(cudaMemcpy(out, planes + j.a, n * 4, cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemcpy(out + n, planes + j.b, n * 4, cudaMemcpyDeviceToHost));
  CUDA_TRY(cudaMemcpy(out + 2 * n, planes + j.c, n * 4, cudaMemcpyDeviceToHost));
  return JXG_OK;
}

// ms[0] = whole batch on the device, ms[1] = the group-stream decode kernel (+ local RCTs) alone.
int jxg_modular_batch_stats(void* bp, uint64_t* h2d, uint64_t* d2h, uint64_t* launches, float* ms) {
  ModularBatch* b = static_cast<ModularBatch*>(bp);
  if (!b || !b->uploaded) return JXG_ERR_ARGUMENT;
  if (int r = batch_wait_last_run(*b)) return r;
  if (h2d) *h2d = b->h2d;
  if (d2h) *d2h = b->d2h;
  if (launches) *launches = b->launches;
  if (ms) {
    ms[0] = ms[1] = 0;
    cudaEventElapsedTime(&ms[0], b->ev0, b->ev1);
    cudaEventElapsedTime(&ms[1], b->ev0, b->ev_decode);
    cudaGetLastError();
  }
  return JXG_OK;
}

int jxg_modular_batch_lz77_stats(void* bp, uint32_t* lz77_streams, uint32_t* rle_streams, uint64_t* window_bytes) {
  ModularBatch* b = static_cast<ModularBatch*>(bp);
  if (!b) return JXG_ERR_ARGUMENT;
  if (lz77_streams) *lz77_streams = b->lz77_streams;
  if (rle_streams) *rle_streams = b->rle_streams;
  if (window_bytes) *window_bytes = b->lz_window_elems * 4;
  return JXG_OK;
}

int jxg_modular_batch_walk_stats(void* bp, uint32_t* generic, uint32_t* single_leaf, uint32_t* by_property,
                                 uint32_t* table_wp) {
  ModularBatch* b = static_cast<ModularBatch*>(bp);
  if (!b) return JXG_ERR_ARGUMENT;
  if (generic) *generic = b->walks.generic;
  if (single_leaf) *single_leaf = b->walks.single;
  if (by_property) memcpy(by_property, b->walks.by_prop, sizeof(b->walks.by_prop));
  if (table_wp) *table_wp = b->walks.table_wp;
  return JXG_OK;
}

int jxg_modular_walk_table(const int32_t* nodes, uint32_t n_nodes, const uint8_t* context_map, uint32_t n_contexts,
                           uint32_t channel, uint32_t stream_id, uint32_t* lut_out, uint32_t* property) {
  if (!nodes || !n_nodes || !context_map || !lut_out || !property) return JXG_ERR_ARGUMENT;
  jxg::ModularTree t;
  t.nodes.resize(n_nodes);
  for (uint32_t i = 0; i < n_nodes; i++) {
    jxg::TreeNode& n = t.nodes[i];
    n.property = nodes[i * 5];
    n.val = nodes[i * 5 + 1];
    n.left = uint32_t(nodes[i * 5 + 2]);
    n.right = uint32_t(nodes[i * 5 + 3]);
    n.ctx = uint32_t(nodes[i * 5 + 4]);
    // children must lie behind their parent (no cycles) and inside the array
    if (n.property >= 0 && (n.left <= i || n.right <= i || n.left >= n_nodes || n.right >= n_nodes)) return JXG_ERR_ARGUMENT;
    if (n.property < 0 && n.ctx >= n_contexts) return JXG_ERR_ARGUMENT;
  }
  t.code.context_map.assign(context_map, context_map + n_contexts);
  std::vector<uint32_t> lut;
  uint32_t prop = kLutNoProperty, single = 0;
  const uint32_t root = static_root(t, channel, stream_id);
  if (!build_walk_table(t, root, channel, stream_id, lut, prop, single)) return 0;
  *property = prop;
  for (int i = 0; i < kLutSize; i++) lut_out[i] = prop == kLutNoProperty ? single : lut[size_t(i)];
  return 1;
}

void jxg_modular_batch_end(void* bp) {
  ModularBatch* b = static_cast<ModularBatch*>(bp);
  if (!b) return;
  batch_end(*b);
  cudaEventDestroy(b->ev_decode);
  delete b;
}

}  // extern "C"
