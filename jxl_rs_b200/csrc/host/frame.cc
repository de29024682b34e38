// See frame.h.
#include "frame.h"

#include <immintrin.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <atomic>
#include <mutex>
#include <thread>

#include "quant.h"

namespace jxg {

static std::atomic<bool> g_pair_lf_groups{true};

namespace {

// Re-packs the bits of `data` starting at bit `bit_pos` into a fresh byte
// vector (only needed for single-section frames, frame_info.rs:414-450, where
// the HF group follows HfGlobal without byte alignment).
std::vector<uint8_t> repack_bits(const uint8_t* data, size_t size, size_t bit_pos) {
  std::vector<uint8_t> out;
  size_t byte = bit_pos / 8, sh = bit_pos % 8;
  if (sh == 0) return std::vector<uint8_t>(data + std::min(byte, size), data + size);
  for (size_t i = byte; i < size; i++) {
    uint32_t lo = data[i] >> sh;
    uint32_t hi = i + 1 < size ? uint32_t(data[i + 1]) << (8 - sh) : 0;
    out.push_back(uint8_t(lo | hi));
  }
  return out;
}

bool ec_is_meta(const ModularChannel& c) { return c.hshift < 0 || c.vshift < 0; }

// The part of coded channel `c` one (LF) group of side `dim` carries (modular/mod.rs:150-190).
ModularChannel ec_group_rect(const ModularChannel& c, uint32_t dim, uint32_t gx, uint32_t gy) {
  const uint32_t gw = dim >> c.hshift, gh = dim >> c.vshift;
  const uint64_t bx = uint64_t(gx) * gw, by = uint64_t(gy) * gh;
  if (gw == 0 || gh == 0 || bx >= c.w || by >= c.h) return ModularChannel(0, 0, c.hshift, c.vshift);
  return ModularChannel(std::min<uint32_t>(c.w - uint32_t(bx), gw), std::min<uint32_t>(c.h - uint32_t(by), gh), c.hshift,
                        c.vshift);
}

// FullModularImage::read + read_section0 (modular/mod.rs:258-365, 405-470) for the extra channels of a VarDCT frame:
// decoded and dropped (see FrameState::ec). Needed in full because a single-section frame has LfGroup / HfGlobal /
// the HF group right behind this data in the same bit stream.
void skip_extra_channels_global(FrameState& fs, BitReader& br) {
  const FrameHeader& h = fs.header;
  for (uint32_t i = 0; i < h.num_extra_channels; i++) {
    const uint32_t ecups = h.ec_upsampling[i];
    if (ecups == 0 || (ecups & (ecups - 1))) fail("invalid extra-channel upsampling");
    const int32_t shift = int32_t(floor_log2(ecups));  // colour upsampling is 1 here (checked by the caller)
    ModularChannel c;
    c.w = (h.width + ecups - 1) / ecups;
    c.h = (h.height + ecups - 1) / ecups;
    c.hshift = c.vshift = shift;
    fs.ec.coded.push_back(c);
  }
  fs.ec.header = GroupHeader::read(br);
  fs.ec.nb_meta = 0;
  meta_apply_transforms(fs.ec.coded, fs.ec.nb_meta, fs.ec.header, /*allocate=*/false);
  const uint32_t gd = h.group_dim();
  size_t n0 = 0;
  while (n0 < fs.ec.coded.size() &&
         (ec_is_meta(fs.ec.coded[n0]) || (fs.ec.coded[n0].w <= gd && fs.ec.coded[n0].h <= gd)))
    n0++;
  fs.ec.n0 = n0;
  std::vector<ModularChannel> scratch;
  bool empty = true;
  for (size_t i = 0; i < n0; i++) {
    const ModularChannel& c = fs.ec.coded[i];
    scratch.emplace_back(c.w, c.h, c.hshift, c.vshift);
    if (c.w && c.h) empty = false;
  }
  if (empty) return;
  ModularTree local;
  const ModularTree* tree = &fs.global_tree;
  if (!fs.ec.header.use_global_tree) {
    size_t samples = 0;
    for (const ModularChannel& c : scratch) samples += size_t(c.w) * c.h;
    local = ModularTree::read(br, std::min<size_t>(1024 + samples, size_t(1) << 20));
    tree = &local;
  } else if (!fs.has_global_tree) {
    fail("no global MA tree");
  }
  std::vector<ModularChannel*> ptrs;
  for (ModularChannel& c : scratch) ptrs.push_back(&c);
  decode_modular_channels(ptrs, 0, fs.ec.header, *tree, br);
}

// The ModularLF stream of LF group `g` (modular/mod.rs:367-400: channels with min(hshift, vshift) >= 3): decoded and
// dropped. Empty for full-resolution extra channels without Squeeze.
void skip_extra_channels_lf_group(FrameState& fs, uint32_t g, BitReader& br) {
  const FrameHeader& h = fs.header;
  std::vector<ModularChannel> ch;
  const uint32_t xlg = h.xsize_lf_groups();
  for (size_t c = fs.ec.n0; c < fs.ec.coded.size(); c++) {
    const ModularChannel& cc = fs.ec.coded[c];
    if (ec_is_meta(cc) || std::min(cc.hshift, cc.vshift) < 3) continue;
    ch.push_back(ec_group_rect(cc, h.group_dim() * 8, g % xlg, g / xlg));
  }
  decode_modular_subbitstream(ch, 1 + size_t(h.num_lf_groups()) + g, fs.has_global_tree ? &fs.global_tree : nullptr, br);
}

}  // namespace

// frame/decode.rs:307-427
void decode_lf_global(FrameState& fs, BitReader& br) {
  const FrameHeader& h = fs.header;
  if (h.has_patches()) fail("patches are outside the hot-path scope", kErrUnsupported);
  if (h.has_splines()) fail("splines are outside the hot-path scope", kErrUnsupported);
  // features/noise.rs:14 + render/stages/noise.rs: noise synthesis is not rendered by this path, and dropping it would
  // silently differ from the reference's pixels, so the frame is refused.
  if (h.has_noise()) fail("noise synthesis is outside the hot-path scope", kErrUnsupported);
  // LfQuantFactors (quantizer.rs:28-52)
  if (!br.read_bool()) {
    for (float& q : fs.lf_quant) {
      q = read_f16(br) / 128.0f;
      if (q < 1e-8f) fail("LF quant factor too small");
    }
  }
  // QuantizerParams (quantizer.rs:60-77)
  switch (br.read(2)) {
    case 0: fs.global_scale = uint32_t(br.read(11)) + 1; break;
    case 1: fs.global_scale = uint32_t(br.read(11)) + 2049; break;
    case 2: fs.global_scale = uint32_t(br.read(12)) + 4097; break;
    default: fs.global_scale = uint32_t(br.read(16)) + 8193;
  }
  switch (br.read(2)) {
    case 0: fs.quant_lf = 16; break;
    case 1: fs.quant_lf = uint32_t(br.read(5)) + 1; break;
    case 2: fs.quant_lf = uint32_t(br.read(8)) + 1; break;
    default: fs.quant_lf = uint32_t(br.read(16)) + 1;
  }
  // BlockContextMap (block_context_map.rs:61-126)
  if (br.read_bool()) {
    static const uint8_t kDefault[39] = {0, 1, 2, 2, 3,  3,  4,  5,  6,  6,  6,  6,  6,  7, 8, 9, 9, 10, 11, 12,
                                         13, 14, 14, 14, 14, 14, 7, 8, 9, 9, 10, 11, 12, 13, 14, 14, 14, 14, 14};
    fs.block_ctx_map.assign(kDefault, kDefault + 39);
    fs.num_lf_contexts = 1;
    fs.num_block_contexts = 15;
  } else {
    fs.num_lf_contexts = 1;
    for (auto& thr : fs.lf_thresholds) {
      size_t n = size_t(br.read(4));
      thr.resize(n);
      for (auto& v : thr) {
        uint64_t u;
        switch (br.read(2)) {
          case 0: u = br.read(4); break;
          case 1: u = br.read(8) + 16; break;
          case 2: u = br.read(16) + 272; break;
          default: u = br.read(32) + 65808;
        }
        v = unpack_signed(uint32_t(u));
      }
      fs.num_lf_contexts *= uint32_t(n + 1);
    }
    size_t nq = size_t(br.read(4));
    fs.qf_thresholds.resize(nq);
    for (auto& v : fs.qf_thresholds) {
      switch (br.read(2)) {
        case 0: v = uint32_t(br.read(2)); break;
        case 1: v = uint32_t(br.read(3)) + 4; break;
        case 2: v = uint32_t(br.read(5)) + 12; break;
        default: v = uint32_t(br.read(8)) + 44;
      }
      v += 1;
    }
    if (fs.num_lf_contexts * (nq + 1) > 64) fail("block context map too big");
    fs.block_ctx_map = decode_context_map(3 * kNumOrders * fs.num_lf_contexts * (nq + 1), br);
    fs.num_block_contexts = uint32_t(*std::max_element(fs.block_ctx_map.begin(), fs.block_ctx_map.end())) + 1;
    if (fs.num_block_contexts > 16) fail("too many block contexts");
  }
  // ColorCorrelationParams (color_correlation_map.rs:43-75)
  if (!br.read_bool()) {
    switch (br.read(2)) {
      case 0: fs.color_factor = 84; break;
      case 1: fs.color_factor = 256; break;
      case 2: fs.color_factor = uint32_t(br.read(8)) + 2; break;
      default: fs.color_factor = uint32_t(br.read(16)) + 258;
    }
    fs.base_correlation_x = read_f16(br);
    fs.base_correlation_b = read_f16(br);
    if (fs.base_correlation_x > 4.0f || fs.base_correlation_b > 4.0f) fail("base colour correlation out of range");
    fs.ytox_lf = int32_t(br.read(8)) - 128;
    fs.ytob_lf = int32_t(br.read(8)) - 128;
  }
  // global MA tree (frame/decode.rs:380-391)
  if (br.read_bool()) {
    size_t limit = std::min<size_t>(1024 + size_t(h.width) * h.height * (3 + h.num_extra_channels) / 16, size_t(1) << 22);
    fs.global_tree = ModularTree::read(br, limit);
    fs.has_global_tree = true;
  }
  // FullModularImage::read: zero channels for VarDCT without extra channels (modular/mod.rs:303-321).
  if (h.num_extra_channels) skip_extra_channels_global(fs, br);
  br.check();
}

LfDequantFactors lf_dequant_factors(const FrameState& fs, float mul) {
  const float inv_quant_lf = 65536.0f / (float(fs.global_scale) * float(fs.quant_lf));
  LfDequantFactors f;
  for (int c = 0; c < 3; c++) f.fac[c] = fs.lf_quant[c] * inv_quant_lf * mul;
  f.cfl_x = fs.base_correlation_x + float(fs.ytox_lf) / float(fs.color_factor);
  f.cfl_b = fs.base_correlation_b + float(fs.ytob_lf) / float(fs.color_factor);
  return f;
}

// modular/mod.rs:837-929 dequant_lf for a 4:4:4 frame: quantised LF integers of a w x h rect (row stride qstride) ->
// dequantised X / Y / B LF samples with the LF chroma-from-luma, and the LF context bucket of every block, written at
// element offset `o0` (row stride fs.xb) of fs.lf[] / fs.quant_lf_map.
void dequant_lf_rect(FrameState& fs, const int32_t* qy_p, const int32_t* qx_p, const int32_t* qb_p, size_t qstride, uint32_t w,
                     uint32_t hh, float mul, size_t o0) {
  const LfDequantFactors f = lf_dequant_factors(fs, mul);
  const float fac_x = f.fac[0], fac_y = f.fac[1], fac_b = f.fac[2], cfl_x = f.cfl_x, cfl_b = f.cfl_b;
  for (uint32_t y = 0; y < hh; y++) {
    const int32_t *qy = qy_p + size_t(y) * qstride, *qx = qx_p + size_t(y) * qstride, *qb = qb_p + size_t(y) * qstride;
    size_t o = o0 + size_t(y) * fs.xb;
    for (uint32_t x = 0; x < w; x++) {
      float in_x = float(qx[x]) * fac_x, in_y = float(qy[x]) * fac_y, in_b = float(qb[x]) * fac_b;
      fs.lf[1][o + x] = in_y;
      fs.lf[0][o + x] = in_y * cfl_x + in_x;
      fs.lf[2][o + x] = in_y * cfl_b + in_b;
    }
    if (fs.num_lf_contexts > 1) {
      for (uint32_t x = 0; x < w; x++) {
        auto bucket = [](const std::vector<int32_t>& thr, int32_t v) {
          uint32_t n = 0;
          for (int32_t t : thr) n += v > t;
          return n;
        };
        uint32_t b = bucket(fs.lf_thresholds[0], qx[x]);
        b = b * uint32_t(fs.lf_thresholds[2].size() + 1) + bucket(fs.lf_thresholds[2], qb[x]);
        b = b * uint32_t(fs.lf_thresholds[1].size() + 1) + bucket(fs.lf_thresholds[1], qy[x]);
        fs.quant_lf_map[o + x] = uint8_t(b);
      }
    }
  }
}

// Varblocks of one LF group's rect (w x hh blocks, maps with row stride `stride`, every entry 27 = INVALID_TRANSFORM on
// entry) in raster order at the first uncovered block (modular/mod.rs:1040-1075): block `num` of the HF-metadata channel
// {raw_transforms, raw_quants} lands there; its first block carries bit 7.
void place_varblocks(uint32_t w, uint32_t hh, size_t stride, uint32_t count, const int32_t* raw_transforms, const int32_t* raw_quants,
                     uint8_t* transform_map, int32_t* raw_quant_map) {
  uint32_t num = 0;
  for (uint32_t y = 0; y < hh; y++) {
    uint8_t* tm = transform_map + size_t(y) * stride;
    int32_t* rq = raw_quant_map + size_t(y) * stride;
    const uint32_t ngy = std::min(hh, (y / 32 + 1) * 32);
    for (uint32_t x = 0; x < w;) {
      if (tm[x] != 27) {  // already covered by an earlier varblock
        x++;
        continue;
      }
      if (num >= count) fail("invalid VarDCT transform map");
      const int32_t raw_transform = raw_transforms[num];
      const int32_t raw_quant = 1 + std::clamp(raw_quants[num], 0, 255);
      if (raw_transform < 0 || raw_transform >= 27) fail("invalid VarDCT transform");
      const uint32_t cx = kCoveredBlocksX[raw_transform], cy = kCoveredBlocksY[raw_transform];
      const uint32_t ngx = std::min(w, (x / 32 + 1) * 32);
      if (x + cx > ngx || y + cy > ngy) fail("HF block out of bounds");
      num++;
      if ((cx | cy) == 1) {  // the 8x8-class transforms (most varblocks): no loops with data-dependent trip counts
        tm[x] = uint8_t(raw_transform) | 128;
        rq[x] = raw_quant;
        x++;
        continue;
      }
      for (uint32_t iy = 0; iy < cy; iy++) {
        uint8_t* t = tm + size_t(iy) * stride + x;
        int32_t* q = rq + size_t(iy) * stride + x;
        for (uint32_t ix = 0; ix < cx; ix++) {  // a block covered earlier is overwritten, like mod.rs:1066-1075
          t[ix] = uint8_t(raw_transform);
          q[ix] = raw_quant;
        }
      }
      tm[x] |= 128;  // first block of the varblock
      x += cx;
    }
  }
}

namespace {
// modular/mod.rs:837-1080: one LF group (LF image, ModularLF stream of extra channels, HF metadata), in phases so
// that two groups can run their Modular sub-bitstreams in lockstep (decode_substreams_paired):
//   begin_lf -> [LF image channels] -> finish_lf_begin_meta -> [HF metadata channels] -> finish_meta
struct LfGroupJob {
  FrameState& fs;
  const uint32_t g;
  BitReader br;
  uint32_t x0, y0, w, hh;
  float mul = 1.0f;
  uint32_t count = 0, cw = 0, chh = 0;
  std::vector<ModularChannel> ch;
  std::unique_ptr<SubStream> ss;

  LfGroupJob(FrameState& f, uint32_t group, const uint8_t* data, size_t size) : fs(f), g(group), br(data, size) {
    const FrameHeader& h = fs.header;
    const uint32_t gd = h.group_dim();  // LF group = group_dim blocks
    const uint32_t gx = g % h.xsize_lf_groups(), gy = g / h.xsize_lf_groups();
    x0 = gx * gd;
    y0 = gy * gd;
    w = std::min(gd, fs.xb - x0);
    hh = std::min(gd, fs.yb - y0);
  }
  const ModularTree* global_tree() const { return fs.has_global_tree ? &fs.global_tree : nullptr; }

  // ---- LF coefficients (decode_vardct_lf) ----
  void begin_lf() {
    const uint32_t extra_precision = uint32_t(br.read(2));
    mul = 1.0f / float(1u << extra_precision);
    for (int c = 0; c < 3; c++) ch.emplace_back(w, hh);
    ss = std::make_unique<SubStream>();
    substream_begin(*ss, ch, 1 + g, global_tree(), br);
  }

  // call after the LF sub-bitstream has been finished
  void finish_lf_begin_meta() {
    const FrameHeader& h = fs.header;
    // dequant_lf (444): channel 0 = Y, 1 = X, 2 = B
    dequant_lf_rect(fs, ch[0].row(0), ch[1].row(0), ch[2].row(0), ch[0].w, w, hh, mul, size_t(y0) * fs.xb + x0);
    ss.reset();
    ch.clear();
    // ModularLF stream: no channels in a VarDCT frame without extra channels.
    if (h.num_extra_channels) skip_extra_channels_lf_group(fs, g, br);
    // ---- HF metadata (decode_hf_metadata) ----
    count = uint32_t(br.read(ceil_log2(uint64_t(w) * hh))) + 1;
    cw = (w + 7) / 8;
    chh = (hh + 7) / 8;
    ch.emplace_back(cw, chh, 3, 3);
    ch.emplace_back(cw, chh, 3, 3);
    ch.emplace_back(count, 2);
    ch.emplace_back(w, hh);
    ss = std::make_unique<SubStream>();
    substream_begin(*ss, ch, 1 + 2 * size_t(h.num_lf_groups()) + g, global_tree(), br);
  }

  // call after the HF-metadata sub-bitstream has been finished
  void finish_meta() {
    {
      uint32_t cxb = (fs.xb + 7) / 8;
      for (uint32_t y = 0; y < chh; y++)
        for (uint32_t x = 0; x < cw; x++) {
          size_t o = size_t(y0 / 8 + y) * cxb + x0 / 8 + x;
          fs.ytox_map[o] = int8_t(std::clamp(ch[0].row(y)[x], -128, 127));
          fs.ytob_map[o] = int8_t(std::clamp(ch[1].row(y)[x], -128, 127));
        }
      // EPF sharpness: one pass per row (range check folded into an OR so that the loop vectorises)
      for (uint32_t y = 0; y < hh; y++) {
        const int32_t* e = ch[3].row(y);
        uint8_t* eo = &fs.epf_map[size_t(y0 + y) * fs.xb + x0];
        int32_t seen = 0;
        for (uint32_t x = 0; x < w; x++) {
          seen |= e[x];
          eo[x] = uint8_t(e[x]);
        }
        if (seen & ~7) fail("invalid EPF sharpness value");
      }
      place_varblocks(w, hh, fs.xb, count, ch[2].row(0), ch[2].row(1), &fs.transform_map[size_t(y0) * fs.xb + x0],
                      &fs.raw_quant_map[size_t(y0) * fs.xb + x0]);
    }
    ss.reset();
    br.check();
  }
};

// One LF group on its own.
void decode_lf_group(FrameState& fs, uint32_t g, const uint8_t* data, size_t size) {
  LfGroupJob job(fs, g, data, size);
  job.begin_lf();
  substream_finish(*job.ss);
  job.finish_lf_begin_meta();
  substream_finish(*job.ss);
  job.finish_meta();
}

// Two LF groups with their sub-bitstreams in lockstep (same results as two decode_lf_group calls).
void decode_lf_group_pair(FrameState& fs, uint32_t ga, const uint8_t* da, size_t sa, uint32_t gb, const uint8_t* db,
                          size_t sb) {
  LfGroupJob a(fs, ga, da, sa), b(fs, gb, db, sb);
  a.begin_lf();
  b.begin_lf();
  decode_substreams_paired(*a.ss, *b.ss);
  a.finish_lf_begin_meta();
  b.finish_lf_begin_meta();
  decode_substreams_paired(*a.ss, *b.ss);
  a.finish_meta();
  b.finish_meta();
}

// frame/decode.rs:506-566
void decode_hf_global(FrameState& fs, BitReader& br) {
  const FrameHeader& h = fs.header;
  const ModularTree* gt = fs.has_global_tree ? &fs.global_tree : nullptr;
  if (!br.read_bool()) {  // DequantMatrices::decode, quant_weights.rs:1088-1120
    for (int i = 0; i < kNumQuantTables; i++) {
      QuantEncoding e = read_quant_encoding(i, br, h, gt);
      if (e.mode != QuantEncoding::kLibrary) fs.custom_dequant[i] = compute_dequant_table(e, i);
    }
  }
  fs.num_histograms = uint32_t(br.read(ceil_log2(h.num_groups()))) + 1;
  fs.passes.resize(h.passes.num_passes);
  for (uint32_t p = 0; p < h.passes.num_passes; p++) {
    PassState& ps = fs.passes[p];
    uint32_t used_orders;
    switch (br.read(2)) {
      case 0: used_orders = 0x5f; break;
      case 1: used_orders = 0x13; break;
      case 2: used_orders = 0; break;
      default: used_orders = uint32_t(br.read(kNumOrders));
    }
    if (used_orders) {  // coeff_order.rs:122-152
      ps.custom_orders = true;
      // all 39 orders concatenated (the layout the device consumes), natural ones copied from the process-wide
      // cache, the coded ones composed with their permutation in place
      size_t total = 0;
      for (int o = 0; o < 3 * kNumOrders; o++) {
        ps.coeff_order_offset[o] = uint32_t(total);
        total += natural_coeff_order_cached(o / 3).size();
      }
      ps.coeff_order.resize(total);
      for (int o = 0; o < 3 * kNumOrders; o++) {
        const std::vector<uint32_t>& nat = natural_coeff_order_cached(o / 3);
        memcpy(&ps.coeff_order[ps.coeff_order_offset[o]], nat.data(), nat.size() * sizeof(uint32_t));
      }
      EntropyCode code = EntropyCode::decode(8, br, true);
      SymbolReader reader(code, br, 0);
      for (int ord = 0; ord < kNumOrders; ord++) {
        if (!(used_orders & (1u << ord))) continue;
        int t = kOrderTransform[ord];
        uint32_t num_blocks = uint32_t(kCoveredBlocksX[t]) * kCoveredBlocksY[t];
        const std::vector<uint32_t>& nat = natural_coeff_order_cached(ord);
        for (int c = 0; c < 3; c++) {
          std::vector<uint32_t> perm = decode_permutation(num_blocks * 64, num_blocks, code, br, reader);
          uint32_t* o = &ps.coeff_order[ps.coeff_order_offset[3 * ord + c]];
          for (size_t i = 0; i < nat.size(); i++) o[i] = nat[perm[i]];  // Permutation::compose
        }
      }
      reader.check_final_state(br);
    }
    size_t num_contexts = size_t(fs.num_histograms) * fs.num_ac_contexts();
    ps.code = EntropyCode::decode(num_contexts, br, true);
    // frame/decode.rs:536-538: pad so that zero-density contexts never index past the map.
    ps.code.context_map.resize(ps.code.context_map.size() + 16, 0);
    for (auto& u : ps.code.uint_configs) ps.uint_configs_packed.push_back(u.packed());
  }
  br.check();
}

}  // namespace

// frame/adaptive_lf_smoothing.rs:44-125. The reference is scalar Rust (no fused multiply-add), so the function is
// compiled without floating-point contraction and the AVX2 body does, lane by lane, the same operations in the same
// order as compute_pixel_channel (:20-41): results are bit-identical to the scalar definition.
#pragma GCC push_options
#pragma GCC optimize("fp-contract=off")
void lf_smoothing_factors(const FrameState& fs, float out[3]) {
  const float inv_quant_lf = (65536.0f / float(fs.global_scale)) / float(fs.quant_lf);
  for (int c = 0; c < 3; c++) out[c] = inv_quant_lf * fs.lf_quant[c];
}

// Rows [y_begin, y_end) of the smoothing, in place. `top0[c]` is the original row y_begin - 1 and `bot_last[c]` the
// original row y_end (both saved by the caller before any band runs, because neighbouring bands overwrite them).
static void smooth_band(FrameState& fs, size_t y_begin, size_t y_end, const float* const top0[3],
                        const float* const bot_last[3]) {
  const size_t xs = fs.xb;
  float lf_factors[3];
  lf_smoothing_factors(fs, lf_factors);
  const float kSide = 0.20345139757231578f, kCorner = 0.0334829185968739f;
  const float kCenter = 1.0f - 4.0f * (kSide + kCorner);
  // In place: row y of the output only needs the original rows y-1, y, y+1, so two saved original rows per channel
  // (the previous one and the current one) replace the reference's second image; border samples stay unchanged
  // (:80-85).
  std::vector<float> saved(6 * xs);
  float* prev[3];
  float* cur[3];
  for (int c = 0; c < 3; c++) {
    prev[c] = &saved[size_t(2 * c) * xs];
    cur[c] = &saved[size_t(2 * c + 1) * xs];
    memcpy(prev[c], top0[c], xs * sizeof(float));
  }
  const __m256 vside = _mm256_set1_ps(kSide), vcorner = _mm256_set1_ps(kCorner), vcenter = _mm256_set1_ps(kCenter);
  const __m256 vabs = _mm256_castsi256_ps(_mm256_set1_epi32(0x7fffffff));
  for (size_t y = y_begin; y < y_end; y++) {
    float* outp[3];
    const float* bot[3];
    for (int c = 0; c < 3; c++) {
      outp[c] = &fs.lf[c][y * xs];
      bot[c] = y + 1 == y_end ? bot_last[c] : &fs.lf[c][(y + 1) * xs];
      memcpy(cur[c], outp[c], xs * sizeof(float));
    }
    size_t x = 1;
    for (; x + 8 <= xs - 1; x += 8) {
      __m256 gap = _mm256_set1_ps(0.5f), mc[3], sm[3];
      for (int c = 0; c < 3; c++) {
        const float* t = prev[c] + x;
        const float* m = cur[c] + x;
        const float* b = bot[c] + x;
        const __m256 corner = _mm256_add_ps(
            _mm256_add_ps(_mm256_add_ps(_mm256_loadu_ps(t - 1), _mm256_loadu_ps(t + 1)), _mm256_loadu_ps(b - 1)),
            _mm256_loadu_ps(b + 1));
        const __m256 side = _mm256_add_ps(
            _mm256_add_ps(_mm256_add_ps(_mm256_loadu_ps(m - 1), _mm256_loadu_ps(m + 1)), _mm256_loadu_ps(t)),
            _mm256_loadu_ps(b));
        mc[c] = _mm256_loadu_ps(m);
        sm[c] = _mm256_add_ps(_mm256_add_ps(_mm256_mul_ps(corner, vcorner), _mm256_mul_ps(side, vside)),
                              _mm256_mul_ps(mc[c], vcenter));
        const __m256 d = _mm256_div_ps(_mm256_sub_ps(mc[c], sm[c]), _mm256_set1_ps(lf_factors[c]));
        gap = _mm256_max_ps(_mm256_and_ps(d, vabs), gap);  // operand order: keeps gap if d is NaN, like f32::max
      }
      const __m256 factor =
          _mm256_max_ps(_mm256_sub_ps(_mm256_set1_ps(3.0f), _mm256_mul_ps(_mm256_set1_ps(4.0f), gap)), _mm256_setzero_ps());
      for (int c = 0; c < 3; c++)
        _mm256_storeu_ps(outp[c] + x, _mm256_add_ps(_mm256_mul_ps(_mm256_sub_ps(sm[c], mc[c]), factor), mc[c]));
    }
    for (; x + 1 < xs; x++) {
      float gap = 0.5f, mc[3], sm[3];
      for (int c = 0; c < 3; c++) {
        const float *t = prev[c], *m = cur[c], *b = bot[c];
        float corner = t[x - 1] + t[x + 1] + b[x - 1] + b[x + 1];
        float side = m[x - 1] + m[x + 1] + t[x] + b[x];
        mc[c] = m[x];
        sm[c] = corner * kCorner + side * kSide + mc[c] * kCenter;
        gap = std::max(gap, std::fabs((mc[c] - sm[c]) / lf_factors[c]));
      }
      float factor = std::max(3.0f - 4.0f * gap, 0.0f);
      for (int c = 0; c < 3; c++) outp[c][x] = (sm[c] - mc[c]) * factor + mc[c];
    }
    for (int c = 0; c < 3; c++) std::swap(prev[c], cur[c]);
  }
}

void adaptive_lf_smoothing(FrameState& fs, int threads) {
  const size_t xs = fs.xb, ys = fs.yb;
  if (xs <= 2 || ys <= 2) return;
  // rows 1 .. ys-2 in bands of whole rows, one per thread (at least 64 rows each)
  const size_t rows = ys - 2;
  const size_t nb = std::max<size_t>(1, std::min<size_t>(size_t(std::max(1, threads)), rows / 64));
  std::vector<float> edge(nb * 6 * xs);  // per band: original rows (begin - 1) and (end), 3 channels each
  std::vector<size_t> begin(nb + 1);
  for (size_t b = 0; b <= nb; b++) begin[b] = 1 + rows * b / nb;
  for (size_t b = 0; b < nb; b++)
    for (int c = 0; c < 3; c++) {
      memcpy(&edge[(b * 6 + c) * xs], &fs.lf[c][(begin[b] - 1) * xs], xs * sizeof(float));
      memcpy(&edge[(b * 6 + 3 + c) * xs], &fs.lf[c][begin[b + 1] * xs], xs * sizeof(float));
    }
  auto run = [&](size_t b) {
    const float* top0[3];
    const float* bot_last[3];
    for (int c = 0; c < 3; c++) {
      top0[c] = &edge[(b * 6 + c) * xs];
      bot_last[c] = &edge[(b * 6 + 3 + c) * xs];
    }
    smooth_band(fs, begin[b], begin[b + 1], top0, bot_last);
  };
  std::vector<std::thread> pool;
  for (size_t b = 1; b < nb; b++) pool.emplace_back(run, b);
  run(0);
  for (auto& t : pool) t.join();
}
#pragma GCC pop_options

void set_pair_lf_groups(bool on) { g_pair_lf_groups.store(on); }

namespace {

// Pool of the large FrameState buffers (see recycle_frame_state in frame.h).
struct BigBuffers {
  std::vector<uint8_t> codestream, transform_map, epf_map, quant_lf_map;
  std::vector<float> lf[3];
  std::vector<int32_t> raw_quant_map;
  size_t bytes() const {
    return codestream.capacity() + transform_map.capacity() + epf_map.capacity() + quant_lf_map.capacity() +
           4 * (lf[0].capacity() + lf[1].capacity() + lf[2].capacity() + raw_quant_map.capacity());
  }
};
constexpr size_t kPoolMaxEntries = 512, kPoolMaxBytes = size_t(2) << 30;
std::mutex g_pool_mutex;
std::vector<BigBuffers> g_pool;
size_t g_pool_bytes = 0;

void take_buffers(FrameState& fs) {
  std::lock_guard<std::mutex> lock(g_pool_mutex);
  if (g_pool.empty()) return;
  BigBuffers b = std::move(g_pool.back());
  g_pool.pop_back();
  g_pool_bytes -= b.bytes();
  fs.codestream = std::move(b.codestream);
  fs.transform_map = std::move(b.transform_map);
  fs.epf_map = std::move(b.epf_map);
  fs.quant_lf_map = std::move(b.quant_lf_map);
  fs.raw_quant_map = std::move(b.raw_quant_map);
  for (int c = 0; c < 3; c++) fs.lf[c] = std::move(b.lf[c]);
}

}  // namespace

void recycle_frame_state(FrameState* fs) {
  if (!fs) return;
  BigBuffers b;
  b.codestream = std::move(fs->codestream);
  b.transform_map = std::move(fs->transform_map);
  b.epf_map = std::move(fs->epf_map);
  b.quant_lf_map = std::move(fs->quant_lf_map);
  b.raw_quant_map = std::move(fs->raw_quant_map);
  for (int c = 0; c < 3; c++) b.lf[c] = std::move(fs->lf[c]);
  delete fs;
  const size_t n = b.bytes();
  std::lock_guard<std::mutex> lock(g_pool_mutex);
  if (g_pool.size() < kPoolMaxEntries && g_pool_bytes + n <= kPoolMaxBytes) {
    g_pool_bytes += n;
    g_pool.push_back(std::move(b));
  }  // else: b is freed on return
}

void fill_image_info(const FileHeader& file, const FrameHeader& h, uint64_t hf_bytes, JxgImageInfo* info) {
  memset(info, 0, sizeof(*info));
  info->coded_width = h.xsize();
  info->coded_height = h.ysize();
  info->orientation = file.orientation;
  info->width = file.orientation >= 5 ? info->coded_height : info->coded_width;
  info->height = file.orientation >= 5 ? info->coded_width : info->coded_height;
  info->num_groups = h.num_groups();
  info->num_passes = h.passes.num_passes;
  info->encoding = h.encoding;
  info->hf_bytes = hf_bytes;
}

void read_vardct_headers(FrameState& fs, const uint8_t* data, size_t size, bool lf_sections_only) {
  extract_codestream(data, size, fs.codestream);
  BitReader br(fs.codestream.data(), fs.codestream.size());
  fs.file = read_file_header(br);
  if (fs.file.have_preview) fail("preview frames are outside the hot-path scope", kErrUnsupported);
  fs.header = read_frame_header(br, fs.file);
  FrameHeader& h = fs.header;
  if (h.encoding != 0) fail("not a VarDCT frame (Modular frames use the Modular path)", kErrUnsupported);
  if (h.frame_type != 0) fail("only regular frames are in scope", kErrUnsupported);
  if (!fs.file.xyb_encoded || h.do_ycbcr) fail("non-XYB VarDCT (JPEG recompression) is outside the scope", kErrUnsupported);
  if (h.upsampling != 1) fail("upsampling is outside the hot-path scope", kErrUnsupported);
  if (h.has_lf_frame()) fail("LF frames are outside the hot-path scope", kErrUnsupported);
  if (h.have_crop || h.blending.mode != 0) fail("cropped/blended frames are outside the hot-path scope", kErrUnsupported);
  check_single_still_frame(fs.file, h);
  resolve_output_colour(fs.file);  // refuses the colour encodings this path cannot reproduce
  fs.toc = read_toc(br, h.num_toc_entries());
  fs.sections_base = br.byte_pos();
  const size_t avail = fs.codestream.size() - fs.sections_base;
  const size_t n = fs.toc.offsets.size(), whole = lf_sections_only && n > 1 ? 1 + size_t(h.num_lf_groups()) : n;
  for (size_t i = 0; i < whole; i++)
    if (fs.toc.offsets[i] + fs.toc.lengths[i] > avail) fail("truncated file: section beyond end", kErrOutOfBounds);
  fs.xb = h.xsize_blocks();
  fs.yb = h.ysize_blocks();
}

std::unique_ptr<FrameState> parse_vardct_file(const uint8_t* data, size_t size, int threads) {
  auto fsp = std::make_unique<FrameState>();
  FrameState& fs = *fsp;
  take_buffers(fs);
  read_vardct_headers(fs, data, size, false);
  const FrameHeader& h = fs.header;
  const uint8_t* base = fs.codestream.data() + fs.sections_base;
  size_t nb = size_t(fs.xb) * fs.yb;
  // LF samples, raw quant and EPF sharpness of every block are written by its LF group (a stream that leaves a block
  // uncovered is rejected below), so pooled buffers are only resized; the transform map is the coverage marker.
  for (auto& p : fs.lf) p.resize(nb);
  fs.transform_map.assign(nb, 27);
  fs.raw_quant_map.resize(nb);
  fs.epf_map.resize(nb);
  fs.quant_lf_map.assign(nb, 0);
  size_t ncm = size_t((fs.xb + 7) / 8) * ((fs.yb + 7) / 8);
  fs.ytox_map.assign(ncm, 0);
  fs.ytob_map.assign(ncm, 0);

  const uint32_t num_groups = h.num_groups(), num_passes = h.passes.num_passes;
  fs.hf_off.assign(size_t(num_groups) * num_passes, 0);
  fs.hf_len.assign(size_t(num_groups) * num_passes, 0);

  if (fs.toc.offsets.size() == 1) {
    BitReader sbr(base + fs.toc.offsets[0], fs.toc.lengths[0]);
    decode_lf_global(fs, sbr);
    // single-section frames (frame_info.rs:414-450) share one bit stream: the LF group continues where LfGlobal
    // stopped and HfGlobal continues where the LF group stops
    {
      LfGroupJob job(fs, 0, base + fs.toc.offsets[0], fs.toc.lengths[0]);
      job.br.skip_bits(sbr.total_bits_read());
      job.begin_lf();
      substream_finish(*job.ss);
      job.finish_lf_begin_meta();
      substream_finish(*job.ss);
      job.finish_meta();
      sbr.skip_bits(job.br.total_bits_read() - sbr.total_bits_read());
    }
    decode_hf_global(fs, sbr);
    // The single HF group follows without alignment: re-pack it byte aligned at the end of the codestream buffer.
    std::vector<uint8_t> packed = repack_bits(base + fs.toc.offsets[0], fs.toc.lengths[0], sbr.total_bits_read());
    fs.hf_off[0] = fs.codestream.size();
    fs.hf_len[0] = uint32_t(packed.size());
    fs.codestream.insert(fs.codestream.end(), packed.begin(), packed.end());
  } else {
    {
      BitReader sbr(base + fs.toc.offsets[0], fs.toc.lengths[0]);
      decode_lf_global(fs, sbr);
    }
    const uint32_t nlf = h.num_lf_groups();
    const uint32_t nthreads = std::min<uint32_t>(nlf, uint32_t(std::max(1, threads)));
    if (nthreads <= 1) {
      // two groups at a time: their Modular sub-bitstreams advance in lockstep (decode_substreams_paired)
      uint32_t g = 0;
      for (; g + 1 < nlf && g_pair_lf_groups.load(std::memory_order_relaxed); g += 2)
        decode_lf_group_pair(fs, g, base + fs.toc.offsets[1 + g], fs.toc.lengths[1 + g], g + 1,
                             base + fs.toc.offsets[2 + g], fs.toc.lengths[2 + g]);
      for (; g < nlf; g++) decode_lf_group(fs, g, base + fs.toc.offsets[1 + g], fs.toc.lengths[1 + g]);
    } else {
      // LF groups are independent sections writing disjoint rectangles of the planes; the error of the lowest
      // failing group is reported, like the serial loop would.
      std::atomic<uint32_t> next{0};
      std::mutex err_mutex;
      uint32_t err_group = UINT32_MAX;
      std::unique_ptr<Error> err;
      auto work = [&] {
        const bool pair = g_pair_lf_groups.load(std::memory_order_relaxed) && nlf >= 4 * nthreads;
        for (;;) {
          const uint32_t g = next.fetch_add(pair ? 2 : 1);
          if (g >= nlf) return;
          try {
            if (pair && g + 1 < nlf)
              decode_lf_group_pair(fs, g, base + fs.toc.offsets[1 + g], fs.toc.lengths[1 + g], g + 1,
                                   base + fs.toc.offsets[2 + g], fs.toc.lengths[2 + g]);
            else
              decode_lf_group(fs, g, base + fs.toc.offsets[1 + g], fs.toc.lengths[1 + g]);
          } catch (Error& e) {
            std::lock_guard<std::mutex> lock(err_mutex);
            if (g < err_group) {
              err_group = g;
              err = std::make_unique<Error>(e);
            }
          } catch (std::exception& e) {
            std::lock_guard<std::mutex> lock(err_mutex);
            if (g < err_group) {
              err_group = g;
              err = std::make_unique<Error>(kErrBitstream, e.what());
            }
          }
        }
      };
      std::vector<std::thread> pool;
      for (uint32_t t = 1; t < nthreads; t++) pool.emplace_back(work);
      work();
      for (auto& t : pool) t.join();
      if (err) throw *err;
    }
    {
      size_t s = 1 + h.num_lf_groups();
      BitReader sbr(base + fs.toc.offsets[s], fs.toc.lengths[s]);
      decode_hf_global(fs, sbr);
    }
    for (uint32_t p = 0; p < num_passes; p++)
      for (uint32_t g = 0; g < num_groups; g++) {
        size_t s = 2 + h.num_lf_groups() + size_t(num_groups) * p + g;
        fs.hf_off[size_t(p) * num_groups + g] = fs.sections_base + fs.toc.offsets[s];
        fs.hf_len[size_t(p) * num_groups + g] = fs.toc.lengths[s];
      }
  }
  for (uint8_t t : fs.transform_map)
    if (t == 27) fail("VarDCT transform map has uncovered blocks");
  if (h.adaptive_lf_smoothing()) adaptive_lf_smoothing(fs, threads);
  return fsp;
}

void FrameState::fill_desc(JxgFrameDesc* d, uint32_t output_format) {
  memset(d, 0, sizeof(*d));
  d->abi_version = JXG_ABI_VERSION;
  d->width = header.xsize();
  d->height = header.ysize();
  d->global_scale = global_scale;
  d->x_qm_scale = header.x_qm_scale;
  d->b_qm_scale = header.b_qm_scale;
  memcpy(d->quant_biases, file.opsin.quant_biases, sizeof(d->quant_biases));
  d->base_correlation_x = base_correlation_x;
  d->base_correlation_b = base_correlation_b;
  d->color_factor = color_factor;
  d->num_qf_thresholds = uint32_t(qf_thresholds.size());
  for (size_t i = 0; i < qf_thresholds.size(); i++) d->qf_thresholds[i] = qf_thresholds[i];
  d->num_lf_contexts = num_lf_contexts;
  d->num_block_contexts = num_block_contexts;
  d->block_ctx_map_len = uint32_t(block_ctx_map.size());
  d->block_ctx_map = block_ctx_map.data();
  d->num_histograms = num_histograms;
  d->num_passes = uint32_t(passes.size());
  pass_descs.assign(passes.size(), JxgPassDesc{});
  for (size_t p = 0; p < passes.size(); p++) {
    PassState& ps = passes[p];
    JxgPassDesc& pd = pass_descs[p];
    pd.shift = p < header.passes.shift.size() ? header.passes.shift[p] : 0;
    pd.use_prefix = ps.code.use_prefix;
    pd.log_alpha_size = ps.code.log_alpha_size;
    pd.num_clusters = ps.code.num_clusters;
    pd.num_contexts = uint32_t(ps.code.context_map.size());
    pd.lz77_enabled = ps.code.lz77_enabled;
    pd.lz77_min_symbol = ps.code.lz77_min_symbol;
    pd.lz77_min_length = ps.code.lz77_min_length;
    pd.lz77_length_uint = ps.code.lz77_length_uint.packed();
    pd.lz_dist_cluster = ps.code.lz_dist_cluster;
    pd.context_map = ps.code.context_map.data();
    pd.uint_configs = ps.uint_configs_packed.data();
    pd.ans_buckets = reinterpret_cast<const uint64_t*>(ps.code.ans_buckets.data());
    pd.huff_entries = ps.code.huff_entries.data();
    pd.huff_offset = ps.code.huff_offset.data();
    pd.huff_entries_len = uint32_t(ps.code.huff_entries.size());
    if (ps.custom_orders) {
      pd.coeff_order = ps.coeff_order.data();
      memcpy(pd.coeff_order_offset, ps.coeff_order_offset, sizeof(pd.coeff_order_offset));
      pd.coeff_order_len = uint32_t(ps.coeff_order.size());
    }
  }
  d->passes = pass_descs.data();
  for (int i = 0; i < kNumQuantTables; i++) d->dequant_tables[i] = custom_dequant[i].empty() ? nullptr : custom_dequant[i].data();
  for (int c = 0; c < 3; c++) d->lf[c] = lf[c].data();
  d->transform_map = transform_map.data();
  d->raw_quant_map = raw_quant_map.data();
  d->epf_map = epf_map.data();
  d->quant_lf = quant_lf_map.data();
  d->ytox_map = ytox_map.data();
  d->ytob_map = ytob_map.data();
  const RestorationFilter& rf = header.rf;
  d->gab = rf.gab;
  memcpy(d->gab_w1, rf.gab_w1, sizeof(d->gab_w1));
  memcpy(d->gab_w2, rf.gab_w2, sizeof(d->gab_w2));
  d->epf_iters = rf.epf_iters;
  memcpy(d->epf_sharp_lut, rf.epf_sharp_lut, sizeof(d->epf_sharp_lut));
  memcpy(d->epf_channel_scale, rf.epf_channel_scale, sizeof(d->epf_channel_scale));
  d->epf_quant_mul = rf.epf_quant_mul;
  d->epf_pass0_sigma_scale = rf.epf_pass0_sigma_scale;
  d->epf_pass2_sigma_scale = rf.epf_pass2_sigma_scale;
  d->epf_border_sad_mul = rf.epf_border_sad_mul;
  memcpy(d->opsin_biases, file.opsin.opsin_biases, sizeof(d->opsin_biases));
  d->intensity_target = file.intensity_target;
  d->output_format = output_format;
  d->orientation = file.orientation;
  // api/inner/codestream_parser/image_info.rs:204-237 + render/stages/xyb.rs:65-140: a non-ICC embedded encoding is the
  // output encoding for every sample format; an ICC profile cannot be output to, so integer formats get sRGB and
  // float formats linear sRGB.
  const bool is_float = output_format == JXG_FORMAT_RGB_F32 || output_format == JXG_FORMAT_XYB_F32_PLANAR;
  const OutputColour oc = resolve_output_colour(file);
  d->output_tf = oc.from_icc ? uint32_t(is_float ? JXG_TF_LINEAR : JXG_TF_SRGB) : oc.tf;
  d->output_gamma = oc.gamma;
  memcpy(d->output_luminances, oc.luminances, sizeof(d->output_luminances));
  memcpy(d->opsin_inverse_matrix, oc.matrix, sizeof(d->opsin_inverse_matrix));
}

}  // namespace jxg
