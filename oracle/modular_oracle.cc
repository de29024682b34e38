// CPU checker for Modular frames (BASELINE config 5; SURVEY §8 rows a18 / a19). TEST INFRASTRUCTURE, like oracle.cc:
// only tests/, __graft_entry__.smoke() and bench.py's CPU legs may call it.
//
// The per-pixel MA-tree decode, the predictors, the weighted predictor and the inverse RCT / palette / Squeeze are
// the scalar restatement in jxl_rs_b200/csrc/host/modular.cc (decode_channel <- modular/decode/channel.rs:220,
// tree.rs:189-280, predict.rs:148-527, squeeze.rs:144-195, rct.rs:9-40) that the host front-end already uses for the
// LF image and the HF metadata of VarDCT frames; here it runs over every ModularHF section and the global inverse
// transforms (decode_modular_frame_cpu below), followed by ConvertI32ToU8 (render/stages/convert.rs:642). The device
// path re-implements exactly these pieces as CUDA kernels and never calls this file.
// Pinning: lossless round trips of the synthetic Modular writer (decoded == source image, bit-exact) and the
// reference's Modular fixtures decoding with every ANS stream ending in its checksum state.
#include <algorithm>
#include <cstring>
#include <string>

#include "../jxl_rs_b200/csrc/host/modular_frame.h"
#include "oracle.h"

extern std::string g_jxo_modular_error;
std::string g_jxo_modular_error;

namespace {

// Every ModularHF section through the scalar sub-bitstream decoder (bitstream.rs:134), results stored at the group
// rects of the full-size coded channels (mod.rs:150), then the global inverse transforms (mod.rs:820 run_transforms).
std::vector<jxg::ModularChannel> decode_modular_frame_cpu(jxg::ModularFrameState& ms) {
  for (jxg::ModularGroupStream& st : ms.hf) {
    if (st.empty) continue;
    std::vector<jxg::ModularChannel> ch;
    for (const jxg::ModularRect& r : st.rects) ch.emplace_back(r.w, r.h, ms.coded[r.chan].hshift, ms.coded[r.chan].vshift);
    jxg::BitReader br(ms.codestream.data() + st.sec_off, st.sec_len);
    br.skip_bits(st.header_bitpos);  // non-zero only in single-section frames
    jxg::decode_modular_subbitstream(ch, size_t(st.stream_id), ms.has_global_tree ? &ms.global_tree : nullptr, br);
    for (size_t i = 0; i < st.rects.size(); i++) {
      const jxg::ModularRect& r = st.rects[i];
      if (!r.w || !r.h) continue;
      jxg::ModularChannel& dst = ms.coded[r.chan];
      if (dst.data.empty()) dst.data.assign(size_t(dst.w) * dst.h, 0);
      for (uint32_t y = 0; y < r.h; y++) memcpy(dst.row(r.y0 + y) + r.x0, ch[i].row(y), size_t(r.w) * 4);
    }
  }
  std::vector<jxg::ModularChannel> full = ms.coded;
  for (auto& c : full)
    if (c.data.empty()) c.data.assign(size_t(c.w) * c.h, 0);
  jxg::undo_transforms(full, ms.global_header, ms.file.bit_depth.bits_per_sample);
  full.resize(std::min<size_t>(full.size(), ms.num_color_channels));
  return full;
}

}  // namespace

extern "C" {

const char* jxo_modular_last_error(void) { return g_jxo_modular_error.c_str(); }

int jxo_modular_info(const uint8_t* data, size_t size, uint32_t* width, uint32_t* height, uint32_t* channels,
                     uint32_t* num_groups) {
  try {
    auto ms = jxg::parse_modular_file(data, size);
    const bool tr = ms->file.orientation >= 5;  // display size (render/save.rs)
    *width = tr ? ms->header.ysize() : ms->header.xsize();
    *height = tr ? ms->header.xsize() : ms->header.ysize();
    *channels = ms->num_color_channels;
    *num_groups = ms->header.num_groups();
    return 0;
  } catch (jxg::Error& e) {
    g_jxo_modular_error = e.what();
    return e.code;
  }
}

// ImageMetadata.orientation of the file (1..8), or 1 when it does not parse.
int jxo_modular_orientation(const uint8_t* data, size_t size) {
  try {
    return int(jxg::parse_modular_file(data, size)->file.orientation);
  } catch (jxg::Error&) {
    return 1;
  }
}

// What the trees and headers of a Modular file use, as one JSON object (test report of the features a file reaches):
// predictors and split properties of every tree (global and HF-group local), leaves with an offset / a multiplier,
// global and local transforms, non-default WeightedHeaders, local trees, prefix / LZ77 codes, geometry.
// Returns the length of the text (written when it fits in cap), or a negative error code.
int64_t jxo_modular_features(const uint8_t* data, size_t size, char* out, size_t cap) {
  try {
    auto ms = jxg::parse_modular_file(data, size);
    std::vector<int> preds(14, 0), props(256, 0);
    size_t offset_leaves = 0, mul_leaves = 0, local_trees = 0, custom_wp = 0, local_tr = 0;
    bool prefix = false, lz77 = false;
    auto scan = [&](const jxg::ModularTree& t) {
      for (const jxg::TreeNode& n : t.nodes) {
        if (n.property >= 0) {
          props[size_t(n.property)] = 1;
        } else {
          preds[n.left] = 1;
          offset_leaves += n.val != 0;
          mul_leaves += n.right != 1;
        }
      }
      prefix |= t.code.use_prefix;
      lz77 |= t.code.lz77_enabled;
    };
    auto is_default_wp = [](const jxg::WeightedHeader& w) {
      const jxg::WeightedHeader d;
      return std::memcmp(&w, &d, sizeof(d)) == 0;
    };
    auto transforms = [](const jxg::GroupHeader& g) {
      std::string s;
      for (const jxg::ModularTransform& t : g.transforms) {
        if (!s.empty()) s += ",";
        if (t.id == 0) s += "\"rct" + std::to_string(t.rct_type) + "\"";
        else if (t.id == 1)
          s += "\"palette(c=" + std::to_string(t.num_channels) + ",colors=" + std::to_string(t.num_colors) +
               ",deltas=" + std::to_string(t.num_deltas) + ",pred=" + std::to_string(t.predictor_id) + ")\"";
        else s += "\"squeeze(" + std::to_string(t.squeezes.size()) + " steps)\"";
      }
      return "[" + s + "]";
    };
    if (ms->has_global_tree) scan(ms->global_tree);
    custom_wp += !is_default_wp(ms->global_header.wp);
    for (const jxg::ModularGroupStream& st : ms->hf) {
      if (st.empty) continue;
      if (st.local_tree) {
        local_trees++;
        scan(*st.local_tree);
      }
      custom_wp += !is_default_wp(st.header.wp);
      local_tr += st.header.transforms.size();
    }
    auto list = [](const std::vector<int>& v) {
      std::string s;
      for (size_t i = 0; i < v.size(); i++)
        if (v[i]) s += (s.empty() ? "" : ",") + std::to_string(i);
      return "[" + s + "]";
    };
    const std::string j = "{\"predictors\":" + list(preds) + ",\"split_properties\":" + list(props) +
                          ",\"offset_leaves\":" + std::to_string(offset_leaves) + ",\"multiplier_leaves\":" +
                          std::to_string(mul_leaves) + ",\"global_transforms\":" + transforms(ms->global_header) +
                          ",\"local_transforms\":" + std::to_string(local_tr) + ",\"custom_wp_headers\":" +
                          std::to_string(custom_wp) + ",\"local_trees\":" + std::to_string(local_trees) +
                          ",\"prefix\":" + (prefix ? "true" : "false") + ",\"lz77\":" + (lz77 ? "true" : "false") +
                          ",\"group_dim\":" + std::to_string(ms->header.group_dim()) + ",\"groups\":" +
                          std::to_string(ms->header.num_groups()) + ",\"grey\":" +
                          (ms->num_color_channels == 1 ? "true" : "false") + ",\"orientation\":" +
                          std::to_string(ms->file.orientation) + "}";
    if (j.size() < cap) std::memcpy(out, j.c_str(), j.size() + 1);
    return int64_t(j.size());
  } catch (jxg::Error& e) {
    g_jxo_modular_error = e.what();
    return e.code;
  }
}

// out: interleaved RGB u8 (grey is replicated); planes (optional): 3 full-size i32 planes before the u8 conversion.
int jxo_decode_modular_file(const uint8_t* data, size_t size, uint8_t* out, size_t out_row_stride, int32_t* planes) {
  try {
    auto ms = jxg::parse_modular_file(data, size);
    std::vector<jxg::ModularChannel> ch = decode_modular_frame_cpu(*ms);
    const uint32_t w = ms->header.xsize(), h = ms->header.ysize();
    const uint32_t orientation = ms->file.orientation;
    std::vector<uint8_t> staging;
    uint8_t* const user_out = out;
    const size_t user_stride = out_row_stride;
    if (orientation != 1) {
      staging.resize(size_t(w) * h * 3);
      out = staging.data();
      out_row_stride = size_t(w) * 3;
    }
    for (uint32_t c = 0; c < 3; c++) {
      const jxg::ModularChannel& src = ch[std::min<size_t>(c, ch.size() - 1)];
      if (src.w != w || src.h != h) throw jxg::Error(jxg::kErrBitstream, "unexpected output channel size");
      if (planes) memcpy(planes + size_t(c) * w * h, src.data.data(), size_t(w) * h * 4);
      for (uint32_t y = 0; y < h; y++) {
        const int32_t* r = src.row(y);
        uint8_t* o = out + size_t(y) * out_row_stride + c;
        for (uint32_t x = 0; x < w; x++) o[size_t(x) * 3] = uint8_t(std::min(std::max(r[x], 0), 255));  // convert.rs:675-680
      }
    }
    if (orientation != 1) jxo_orient_image(staging.data(), w, h, 3, orientation, user_out, user_stride);
    return 0;
  } catch (jxg::Error& e) {
    g_jxo_modular_error = e.what();
    return e.code;
  }
}

}  // extern "C"
