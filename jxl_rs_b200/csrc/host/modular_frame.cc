// See modular_frame.h.
#include "modular_frame.h"

#include <algorithm>
#include <cstring>

namespace jxg {

namespace {

constexpr uint32_t kNumQuantTablesIds = 17;  // NUM_QUANT_TABLES in the stream-id formula (common.rs:29-35)

bool is_meta(const ModularChannel& c) { return c.hshift < 0 || c.vshift < 0; }
bool meta_or_small(const ModularChannel& c, uint32_t group_dim) {  // mod.rs:74
  return is_meta(c) || (c.w <= group_dim && c.h <= group_dim);
}
int min_shift(const ModularChannel& c) { return std::min(c.hshift, c.vshift); }

// mod.rs:150-190 with buffer grid kind None (one full-size plane per channel)
ModularRect grid_rect(const ModularChannel& c, uint32_t chan, uint32_t dim, uint32_t gx, uint32_t gy) {
  ModularRect r{chan, 0, 0, 0, 0};
  const uint32_t gw = dim >> c.hshift, gh = dim >> c.vshift;
  const uint64_t bx = uint64_t(gx) * gw, by = uint64_t(gy) * gh;
  if (gw == 0 || gh == 0 || bx >= c.w || by >= c.h) return r;
  r.x0 = uint32_t(bx);
  r.y0 = uint32_t(by);
  r.w = std::min<uint32_t>(c.w - r.x0, gw);
  r.h = std::min<uint32_t>(c.h - r.y0, gh);
  return r;
}

std::vector<ModularChannel> rect_channels(const ModularFrameState& ms, const std::vector<ModularRect>& rects) {
  std::vector<ModularChannel> out;
  for (const ModularRect& r : rects) out.emplace_back(r.w, r.h, ms.coded[r.chan].hshift, ms.coded[r.chan].vshift);
  return out;
}

void store_rects(ModularFrameState& ms, const std::vector<ModularRect>& rects, const std::vector<ModularChannel>& ch) {
  for (size_t i = 0; i < rects.size(); i++) {
    const ModularRect& r = rects[i];
    if (!r.w || !r.h) continue;
    ModularChannel& dst = ms.coded[r.chan];
    if (dst.data.empty()) dst.data.assign(size_t(dst.w) * dst.h, 0);
    for (uint32_t y = 0; y < r.h; y++) memcpy(dst.row(r.y0 + y) + r.x0, ch[i].row(y), size_t(r.w) * 4);
  }
}

// frame/decode.rs:307-397 for a Modular frame, then modular/mod.rs:258-490.
void decode_lf_global_modular(ModularFrameState& ms, BitReader& br) {
  const FrameHeader& h = ms.header;
  if (h.has_patches()) fail("patches are outside the hot-path scope", kErrUnsupported);
  if (h.has_splines()) fail("splines are outside the hot-path scope", kErrUnsupported);
  if (h.has_noise()) fail("noise synthesis is outside the hot-path scope", kErrUnsupported);
  read_lf_quant_factors(br, ms.lf_quant);  // used by XYB frames only
  if (br.read_bool()) {
    size_t limit = std::min<size_t>(1024 + size_t(h.width) * h.height * ms.num_color_channels / 16, size_t(1) << 22);
    ms.global_tree = ModularTree::read(br, limit);
    ms.has_global_tree = true;
  }
  // FullModularImage::read (mod.rs:258)
  for (uint32_t c = 0; c < ms.num_color_channels; c++) {
    ModularChannel ch;
    ch.w = h.xsize();
    ch.h = h.ysize();
    ms.coded.push_back(ch);
  }
  ms.global_header = GroupHeader::read(br);
  ms.nb_meta = 0;
  meta_apply_transforms(ms.coded, ms.nb_meta, ms.global_header, /*allocate=*/false);
  // section 0: the leading "meta or small" channels (mod.rs:353-365)
  size_t n0 = 0;
  while (n0 < ms.coded.size() && meta_or_small(ms.coded[n0], h.group_dim())) n0++;
  ms.host_decoded.assign(ms.coded.size(), 0);
  bool empty = true;
  for (size_t i = 0; i < n0; i++) {
    ms.host_decoded[i] = 1;
    ms.coded[i].data.assign(size_t(ms.coded[i].w) * ms.coded[i].h, 0);
    if (ms.coded[i].w && ms.coded[i].h) empty = false;
  }
  if (!empty) {  // bitstream.rs:134 with the header given
    ModularTree local;
    const ModularTree* tree = &ms.global_tree;
    if (!ms.global_header.use_global_tree) {
      size_t samples = 0;
      for (size_t i = 0; i < n0; i++) samples += size_t(ms.coded[i].w) * ms.coded[i].h;
      local = ModularTree::read(br, std::min<size_t>(1024 + samples, size_t(1) << 20));
      tree = &local;
    } else if (!ms.has_global_tree) {
      fail("no global MA tree");
    }
    std::vector<ModularChannel*> ptrs;
    for (size_t i = 0; i < n0; i++) ptrs.push_back(&ms.coded[i]);
    decode_modular_channels(ptrs, 0, ms.global_header, *tree, br);
  }
  br.check();
  // channel -> section assignment of the rest (mod.rs:367-400), single pass: HF groups take shifts [0, 2]
  const uint32_t xg = h.xsize_groups(), ng = h.num_groups();
  ms.hf.assign(ng, ModularGroupStream());
  for (uint32_t g = 0; g < ng; g++) {
    ModularGroupStream& st = ms.hf[g];
    st.group = g;
    st.stream_id = 1 + 3 * uint64_t(h.num_lf_groups()) + kNumQuantTablesIds + g;
    for (size_t c = n0; c < ms.coded.size(); c++) {
      if (is_meta(ms.coded[c]) || min_shift(ms.coded[c]) > 2) continue;
      ModularRect r = grid_rect(ms.coded[c], uint32_t(c), h.group_dim(), g % xg, g / xg);
      st.rects.push_back(r);
      if (r.w && r.h) st.empty = false;
    }
  }
}

void decode_lf_group_modular(ModularFrameState& ms, uint32_t g, BitReader& br) {
  const FrameHeader& h = ms.header;
  size_t n0 = 0;
  while (n0 < ms.coded.size() && ms.host_decoded[n0]) n0++;
  std::vector<ModularRect> rects;
  const uint32_t xlg = h.xsize_lf_groups();
  for (size_t c = n0; c < ms.coded.size(); c++) {
    if (is_meta(ms.coded[c]) || min_shift(ms.coded[c]) < 3) continue;
    rects.push_back(grid_rect(ms.coded[c], uint32_t(c), h.group_dim() * 8, g % xlg, g / xlg));
  }
  std::vector<ModularChannel> ch = rect_channels(ms, rects);
  decode_modular_subbitstream(ch, 1 + size_t(h.num_lf_groups()) + g, ms.has_global_tree ? &ms.global_tree : nullptr, br);
  store_rects(ms, rects, ch);
  br.check();
}

void parse_hf_stream_header(ModularFrameState& ms, ModularGroupStream& st, BitReader& br) {
  read_group_stream_header(st, ms.coded, ms.has_global_tree, br);
}

// Symbolic undo_transforms (modular.cc) over buffer ids.
void build_inverse_plan(ModularFrameState& ms) {
  ms.bufs.clear();
  ms.steps.clear();
  std::vector<uint32_t> cur;
  for (const ModularChannel& c : ms.coded) {
    cur.push_back(uint32_t(ms.bufs.size()));
    ms.bufs.push_back(ModularBuf{c.w, c.h});
  }
  const GroupHeader& header = ms.global_header;
  for (size_t ti = header.transforms.size(); ti-- > 0;) {
    const ModularTransform& t = header.transforms[ti];
    if (t.id == 0) {
      const uint32_t perm = t.rct_type / 7, b = t.begin_channel;
      ModularStep s;
      s.kind = kJobRct;
      s.a = cur[b];
      s.b = cur[b + 1];
      s.c = cur[b + 2];
      s.rct_op = t.rct_type % 7;
      ms.steps.push_back(s);
      uint32_t ids[3] = {cur[b], cur[b + 1], cur[b + 2]};
      cur[b + perm % 3] = ids[0];
      cur[b + (perm + 1 + perm / 3) % 3] = ids[1];
      cur[b + (perm + 2 - perm / 3) % 3] = ids[2];
    } else if (t.id == 1) {
      // transforms/palette.rs:165-199 (num_deltas == 0 and the Zero predictor: a per-pixel look-up). Delta entries predict
      // from already reconstructed neighbours, a raster-order chain over the whole image: no device form.
      const size_t bi = size_t(t.begin_channel) + 1;
      if (t.num_deltas != 0 || t.predictor_id != 0 || bi >= cur.size() || t.num_channels == 0) {
        ms.device_plan_ok = false;
        return;
      }
      ModularStep s;
      s.kind = kJobPalette;
      s.a = cur[bi];
      s.b = cur[0];
      s.c = uint32_t(ms.bufs.size());
      s.n = t.num_channels;
      s.num_colors = t.num_colors;
      for (uint32_t c = 0; c < t.num_channels; c++) ms.bufs.push_back(ModularBuf{ms.bufs[s.a].w, ms.bufs[s.a].h});
      ms.steps.push_back(s);
      cur.erase(cur.begin() + bi);
      for (uint32_t c = 0; c < t.num_channels; c++) cur.insert(cur.begin() + bi + c, s.c + c);
      cur.erase(cur.begin());
    } else {
      for (size_t si = t.squeezes.size(); si-- > 0;) {
        const SqueezeParams& sq = t.squeezes[si];
        const size_t b = sq.begin_channel, e = b + sq.num_channels;
        const size_t offset = sq.in_place ? e : cur.size() - sq.num_channels;
        for (size_t c = b; c < e; c++) {
          const uint32_t avg = cur[c], res = cur[offset + (c - b)];
          ModularStep s;
          s.kind = sq.horizontal ? kJobHSqueeze : kJobVSqueeze;
          s.a = avg;
          s.b = res;
          s.c = uint32_t(ms.bufs.size());
          if (sq.horizontal) ms.bufs.push_back(ModularBuf{ms.bufs[avg].w + ms.bufs[res].w, ms.bufs[avg].h});
          else ms.bufs.push_back(ModularBuf{ms.bufs[avg].w, ms.bufs[avg].h + ms.bufs[res].h});
          ms.steps.push_back(s);
          cur[c] = s.c;
        }
        cur.erase(cur.begin() + offset, cur.begin() + offset + sq.num_channels);
      }
    }
  }
  for (uint32_t c = 0; c < ms.num_color_channels && c < cur.size(); c++) ms.out_buf[c] = cur[c];
}

}  // namespace

void read_group_stream_header(ModularGroupStream& st, const std::vector<ModularChannel>& coded, bool has_global_tree,
                              BitReader& br) {
  if (st.empty) return;
  st.header_bitpos = br.total_bits_read();
  st.header = GroupHeader::read(br);
  std::vector<ModularChannel> shapes;
  for (const ModularRect& r : st.rects) {
    ModularChannel c;
    c.w = r.w;
    c.h = r.h;
    c.hshift = coded[r.chan].hshift;
    c.vshift = coded[r.chan].vshift;
    shapes.push_back(c);
  }
  uint32_t nb_meta = 0;
  meta_apply_transforms(shapes, nb_meta, st.header, /*allocate=*/false);
  if (!st.header.use_global_tree) {
    size_t samples = 0;
    for (auto& c : shapes) samples += size_t(c.w) * c.h;
    st.local_tree = std::make_shared<ModularTree>(ModularTree::read(br, std::min<size_t>(1024 + samples, size_t(1) << 20)));
  } else if (!has_global_tree) {
    fail("no global MA tree");
  }
  st.data_bitpos = br.total_bits_read();
  for (const ModularChannel& c : shapes) st.dist_multiplier = std::max(st.dist_multiplier, c.w);
  br.check();
}

std::unique_ptr<ModularFrameState> parse_modular_file(const uint8_t* data, size_t size) {
  auto msp = std::make_unique<ModularFrameState>();
  ModularFrameState& ms = *msp;
  ms.codestream = extract_codestream(data, size);
  BitReader br(ms.codestream.data(), ms.codestream.size());
  ms.file = read_file_header(br);
  if (ms.file.have_preview) fail("preview frames are outside the hot-path scope", kErrUnsupported);
  ms.header = read_frame_header(br, ms.file);
  FrameHeader& h = ms.header;
  if (h.encoding != 1) fail("not a Modular frame", kErrUnsupported);
  if (h.frame_type != 0) fail("only regular frames are in scope", kErrUnsupported);
  ms.xyb = ms.file.xyb_encoded;
  if (h.do_ycbcr) fail("YCbCr Modular frames are outside the scope", kErrUnsupported);
  if (h.num_extra_channels) fail("extra channels are outside the hot-path scope", kErrUnsupported);
  if (h.upsampling != 1) fail("upsampling is outside the hot-path scope", kErrUnsupported);
  if (h.has_lf_frame()) fail("LF frames are outside the hot-path scope", kErrUnsupported);
  if (h.have_crop || h.blending.mode != 0) fail("cropped/blended frames are outside the hot-path scope", kErrUnsupported);
  if (h.passes.num_passes != 1) fail("multi-pass Modular frames are outside the scope", kErrUnsupported);
  check_single_still_frame(ms.file, h);
  if (ms.xyb) {
    // The reference filters a Modular XYB frame with a constant EPF sigma of its own; the device path has no such stage.
    if (h.rf.gab || h.rf.epf_iters > 0) fail("XYB Modular frames with Gaborish or EPF are outside the scope", kErrUnsupported);
    resolve_output_colour(ms.file);  // refuses the colour encodings the output stage cannot reproduce
  } else if (ms.file.bit_depth.floating_point || ms.file.bit_depth.bits_per_sample != 8) {
    fail("only 8-bit integer samples are in scope", kErrUnsupported);
  }
  // frame/decode.rs:167-170: an XYB frame codes three colour channels whatever the colour encoding
  ms.num_color_channels = !ms.xyb && ms.file.color_encoding.color_space == ColorSpace::Gray ? 1 : 3;
  ms.toc = read_toc(br, h.num_toc_entries());
  ms.sections_base = br.byte_pos();
  const uint8_t* base = ms.codestream.data() + ms.sections_base;
  const size_t avail = ms.codestream.size() - ms.sections_base;
  for (size_t i = 0; i < ms.toc.offsets.size(); i++)
    if (ms.toc.offsets[i] + ms.toc.lengths[i] > avail) fail("truncated file: section beyond end", kErrOutOfBounds);

  if (ms.toc.offsets.size() == 1) {
    // All sections share one bit stream (frame_info.rs:414-450): LfGlobal, LfGroup 0, (empty) HfGlobal, HF group 0.
    BitReader sbr(base + ms.toc.offsets[0], ms.toc.lengths[0]);
    decode_lf_global_modular(ms, sbr);
    decode_lf_group_modular(ms, 0, sbr);
    ModularGroupStream& st = ms.hf[0];
    st.sec_off = ms.sections_base + ms.toc.offsets[0];
    st.sec_len = ms.toc.lengths[0];
    parse_hf_stream_header(ms, st, sbr);
  } else {
    {
      BitReader sbr(base + ms.toc.offsets[0], ms.toc.lengths[0]);
      decode_lf_global_modular(ms, sbr);
    }
    for (uint32_t g = 0; g < h.num_lf_groups(); g++) {
      BitReader sbr(base + ms.toc.offsets[1 + g], ms.toc.lengths[1 + g]);
      decode_lf_group_modular(ms, g, sbr);
    }
    for (uint32_t g = 0; g < h.num_groups(); g++) {
      const size_t s = 2 + size_t(h.num_lf_groups()) + g;
      ModularGroupStream& st = ms.hf[g];
      st.sec_off = ms.sections_base + ms.toc.offsets[s];
      st.sec_len = ms.toc.lengths[s];
      BitReader sbr(base + ms.toc.offsets[s], ms.toc.lengths[s]);
      parse_hf_stream_header(ms, st, sbr);
    }
  }
  // channels with shift >= 3 were filled by the ModularLF streams
  for (size_t c = 0; c < ms.coded.size(); c++)
    if (!ms.host_decoded[c] && !is_meta(ms.coded[c]) && min_shift(ms.coded[c]) > 2) {
      ms.host_decoded[c] = 1;
      if (ms.coded[c].data.empty()) ms.coded[c].data.assign(size_t(ms.coded[c].w) * ms.coded[c].h, 0);
    }
  build_inverse_plan(ms);
  return msp;
}

}  // namespace jxg
