// Synthetic *Modular* (lossless, 8-bit RGB) JPEG XL writer: test-data tooling for BASELINE config 5, like
// encoder.cc is for the VarDCT configs (the reference has no encoder). It emits: non-XYB image metadata (or, in the XYB
// mode, XYB-encoded metadata and the procedural picture quantised to Y, X, B channels: a lossy Modular frame), a Modular
// frame header (group size 256, no restoration filter), LfGlobal with a global MA tree + one clustered ANS code,
// global transforms RCT (YCoCg) and/or Squeeze (default parameters), and one sub-bitstream per section following
// the channel -> section rules of modular/mod.rs:353-400. Forward RCT / forward Squeeze are derived here from the
// decoder definitions (rct.rs:9-40, squeeze.rs:144-195); the round trip "decode == source" is part of the tests.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <deque>
#include <stdexcept>
#include <string>

#include "../jxl_rs_b200/csrc/host/headers.h"
#include "../jxl_rs_b200/csrc/host/modular.h"
#include "entropy_writer.h"

namespace jxs {

void make_image_u8(uint32_t width, uint32_t height, uint64_t seed, std::vector<uint8_t>& rgb);
void make_xyb_image(uint32_t width, uint32_t height, uint64_t seed, std::vector<float> (&xyb)[3]);
void write_xyb_image_metadata(BitWriter& out, uint32_t orientation, uint32_t colour);

// XYB mode of encode_modular. lf_quant_f16: the LfQuantFactors as written (f16 values, the factors times 128; all zero:
// the default factors); colour / orientation: as the VarDCT writer's; gab / epf_iters: the restoration filter flags.
struct ModularXyb {
  bool on = false;
  float lf_quant_f16[3] = {0.0f, 0.0f, 0.0f};
  uint32_t colour = 0, orientation = 1, gab = 0, epf_iters = 0;
};

namespace {

using jxg::ModularChannel;

struct MNode {  // MA tree node in BFS order
  int property = -1;  // -1: leaf
  int32_t splitval = 0;
  uint32_t left = 0, right = 0;
  uint32_t predictor = 5, ctx = 0;
};

// Nested description -> BFS order (tree.rs:284-340 assigns children at the end of the pending queue).
struct TDesc {
  int property;
  int32_t splitval;
  uint32_t predictor;
  int left, right;  // indices into the description vector, -1 for leaves
};
std::vector<MNode> flatten(const std::vector<TDesc>& d) {
  std::vector<MNode> out;
  std::deque<int> q{0};
  while (!q.empty()) {
    const int i = q.front();
    q.pop_front();
    MNode n;
    if (d[i].property >= 0) {
      n.property = d[i].property;
      n.splitval = d[i].splitval;
      n.left = uint32_t(out.size() + q.size() + 1);
      n.right = n.left + 1;
      q.push_back(d[i].left);
      q.push_back(d[i].right);
    } else {
      n.predictor = d[i].predictor;
    }
    out.push_back(n);
  }
  uint32_t leaf = 0;
  for (auto& n : out)
    if (n.property < 0) n.ctx = leaf++;
  return out;
}

std::vector<MNode> make_tree(uint32_t kind) {
  std::vector<TDesc> d;
  auto leaf = [&](uint32_t pred) {
    d.push_back(TDesc{-1, 0, pred, -1, -1});
    return int(d.size() - 1);
  };
  auto split = [&](int prop, int32_t val, int l, int r) {
    d.push_back(TDesc{prop, val, 0, l, r});
    return int(d.size() - 1);
  };
  int root;
  if (kind == 0) {
    d.push_back(TDesc{-1, 0, 5, -1, -1});  // one Gradient leaf
    return flatten(d);
  } else if (kind == 1) {
    // channel split, then splits on |N - NN|-like local activity (property 13) and on W - NW (property 10)
    int a = leaf(5), b = leaf(5), c = leaf(1), e = leaf(5), f = leaf(4), g = leaf(5);
    int lumaA = split(13, 6, a, split(13, -7, b, c));
    int chroma = split(10, 3, e, split(10, -4, f, g));
    root = split(0, 0, chroma, lumaA);
  } else if (kind == 3) {
    // properties of the previous channel (decode/common.rs:40-83): 17 = its value, 19 = its gradient residual
    int a = leaf(5), b = leaf(5), c = leaf(1), e = leaf(5), f = leaf(5), g = leaf(0), h = leaf(5);
    int luma = split(13, 6, a, split(13, -7, b, c));
    int chroma = split(19, 4, e, split(19, -5, f, split(17, 100, g, h)));
    root = split(0, 0, chroma, luma);
  } else {
    // weighted predictor with contexts from its max-error property (15), plus a Gradient branch for channel > 0
    int a = leaf(6), b = leaf(6), c = leaf(6), e = leaf(5), f = leaf(6);
    int lum = split(15, 12, a, split(15, -13, b, c));
    int chr = split(15, 5, e, f);
    root = split(0, 0, chr, lum);
  }
  // move the root to index 0
  std::vector<TDesc> r;
  std::vector<int> map(d.size(), -1);
  std::deque<int> q{root};
  while (!q.empty()) {  // re-index so that the root is first (any order works for flatten)
    int i = q.front();
    q.pop_front();
    map[i] = int(r.size());
    r.push_back(d[i]);
    if (d[i].property >= 0) {
      q.push_back(d[i].left);
      q.push_back(d[i].right);
    }
  }
  for (auto& n : r)
    if (n.property >= 0) {
      n.left = map[n.left];
      n.right = map[n.right];
    }
  return flatten(r);
}

inline int32_t wadd(int32_t a, int32_t b) { return int32_t(uint32_t(a) + uint32_t(b)); }
inline int32_t wsub(int32_t a, int32_t b) { return int32_t(uint32_t(a) - uint32_t(b)); }
inline int32_t wabs(int32_t a) { return a < 0 ? int32_t(0u - uint32_t(a)) : a; }
inline int64_t clamped_gradient(int64_t l, int64_t t, int64_t tl) {
  int64_t mn = std::min(l, t), mx = std::max(l, t), g = l + t - tl;
  return tl < mn ? mx : (tl > mx ? mn : g);
}

// Tokenises one sub-bitstream (list of channels) with the tree; mirrors decode/channel.rs:220 from the encoder side.
void tokenize(const std::vector<ModularChannel>& chans, uint64_t stream_id, const std::vector<MNode>& tree, bool uses_wp,
              std::vector<Token>& out) {
  const jxg::WeightedHeader wph;
  for (size_t ci = 0; ci < chans.size(); ci++) {
    const ModularChannel& ch = chans[ci];
    if (!ch.w || !ch.h) continue;
    jxg::WpState wp(wph, uses_wp ? ch.w : 0);
    int32_t props[16 + 8] = {0};
    // up to two reference channels (previous channels of the same shape, nearest first), decode/common.rs:40-83
    const ModularChannel* refs[2] = {nullptr, nullptr};
    for (size_t i = 0, n = 0; i < ci && n < 2; i++) {
      const ModularChannel& rc = chans[ci - 1 - i];
      if (rc.w == ch.w && rc.h == ch.h && rc.hshift == ch.hshift && rc.vshift == ch.vshift) refs[n++] = &rc;
    }
    props[0] = int32_t(ci);
    props[1] = int32_t(stream_id);
    for (uint32_t y = 0; y < ch.h; y++) {
      const int32_t* row = ch.row(y);
      const int32_t* top = y ? ch.row(y - 1) : row;
      const int32_t* toptop = y > 1 ? ch.row(y - 2) : top;
      props[9] = 0;
      props[2] = int32_t(y);
      for (uint32_t x = 0; x < ch.w; x++) {
        const int32_t left = x ? row[x - 1] : (y ? top[0] : 0);
        const int32_t n = y ? top[x] : left;
        const int32_t nw = (x && y) ? top[x - 1] : left;
        const int32_t ne = (x + 1 < ch.w && y) ? top[x + 1] : n;
        const int32_t ww = x > 1 ? row[x - 2] : left;
        const int32_t nn = y > 1 ? toptop[x] : n;
        props[3] = int32_t(x);
        props[4] = wabs(n);
        props[5] = wabs(left);
        props[6] = n;
        props[7] = left;
        props[8] = wsub(left, props[9]);
        props[9] = wsub(wadd(left, n), nw);
        props[10] = wsub(left, nw);
        props[11] = wsub(nw, n);
        props[12] = wsub(n, ne);
        props[13] = wsub(n, nn);
        props[14] = wsub(left, ww);
        int64_t wp_pred = 0;
        int32_t wp_prop = 0;
        if (uses_wp) wp.predict(x, y, n, left, ne, nw, nn, wp_pred, wp_prop);
        props[15] = wp_prop;
        for (int ri = 0; ri < 2; ri++) {
          int32_t* rp = props + 16 + 4 * ri;
          rp[0] = rp[1] = rp[2] = rp[3] = 0;
          if (!refs[ri]) continue;
          const int32_t* rrow = refs[ri]->row(y);
          const int32_t* rprev = refs[ri]->row(y ? y - 1 : 0);
          const int32_t v = rrow[x];
          const int32_t vleft = x ? rrow[x - 1] : 0, vtop = y ? rprev[x] : vleft, vtl = (x && y) ? rprev[x - 1] : vleft;
          const int64_t d = int64_t(v) - clamped_gradient(vleft, vtop, vtl);
          rp[0] = wabs(v);
          rp[1] = v;
          rp[2] = int32_t(d < 0 ? -d : d);
          rp[3] = int32_t(d);
        }
        const MNode* nd = &tree[0];
        while (nd->property >= 0) nd = &tree[props[nd->property] > nd->splitval ? nd->left : nd->right];
        int64_t guess;
        switch (nd->predictor) {
          case 0: guess = 0; break;
          case 1: guess = left; break;
          case 2: guess = n; break;
          case 4: {
            int64_t pp = int64_t(left) + n - nw;
            guess = std::llabs(pp - left) < std::llabs(pp - n) ? left : n;
            break;
          }
          case 6: guess = wp_pred; break;
          default: guess = clamped_gradient(left, n, nw);
        }
        out.push_back(Token{nd->ctx, pack_signed(int32_t(int64_t(row[x]) - guess))});
        if (uses_wp) wp.update(row[x], x, y);
      }
    }
  }
}

// squeeze.rs:144-170
int64_t smooth_tendency(int64_t b, int64_t a, int64_t n) {
  int64_t diff = 0;
  if (b >= a && a >= n) {
    diff = (4 * b - 3 * n - a + 6) / 12;
    if (diff - (diff & 1) > 2 * (b - a)) diff = 2 * (b - a) + 1;
    if (diff + (diff & 1) > 2 * (a - n)) diff = 2 * (a - n);
  } else if (b <= a && a <= n) {
    diff = (4 * b - 3 * n - a - 6) / 12;
    if (diff + (diff & 1) < 2 * (b - a)) diff = 2 * (b - a) - 1;
    if (diff - (diff & 1) < 2 * (a - n)) diff = 2 * (a - n);
  }
  return diff;
}

// Forward horizontal squeeze: out (w) -> avg ((w+1)/2), residual (w/2); inverse of squeeze.rs:390 (unsqueeze).
void fwd_hsqueeze(const ModularChannel& in, ModularChannel& avg, ModularChannel& res) {
  const uint32_t aw = (in.w + 1) / 2, rw = in.w - aw;
  avg = ModularChannel(aw, in.h, in.hshift + 1, in.vshift);
  res = ModularChannel(rw, in.h, in.hshift + 1, in.vshift);
  for (uint32_t y = 0; y < in.h; y++) {
    const int32_t* o = in.row(y);
    int32_t* a = avg.row(y);
    for (uint32_t x = 0; x < rw; x++) a[x] = int32_t(int64_t(o[2 * x]) - (int64_t(o[2 * x]) - o[2 * x + 1]) / 2);
    if (in.w & 1) a[aw - 1] = o[in.w - 1];
    int32_t* r = rw ? res.row(y) : nullptr;
    for (uint32_t x = 0; x < rw; x++) {
      const int64_t av = a[x], next_avg = x + 1 < aw ? a[x + 1] : av, left = x ? o[2 * x - 1] : av;
      r[x] = int32_t(int64_t(o[2 * x]) - o[2 * x + 1] - smooth_tendency(left, av, next_avg));
    }
  }
}
void fwd_vsqueeze(const ModularChannel& in, ModularChannel& avg, ModularChannel& res) {
  const uint32_t ah = (in.h + 1) / 2, rh = in.h - ah;
  avg = ModularChannel(in.w, ah, in.hshift, in.vshift + 1);
  res = ModularChannel(in.w, rh, in.hshift, in.vshift + 1);
  for (uint32_t y = 0; y < rh; y++)
    for (uint32_t x = 0; x < in.w; x++)
      avg.row(y)[x] = int32_t(int64_t(in.row(2 * y)[x]) - (int64_t(in.row(2 * y)[x]) - in.row(2 * y + 1)[x]) / 2);
  if (in.h & 1) memcpy(avg.row(ah - 1), in.row(in.h - 1), size_t(in.w) * 4);
  for (uint32_t y = 0; y < rh; y++) {
    const int32_t* a = avg.row(y);
    const int32_t* an = y + 1 < ah ? avg.row(y + 1) : a;
    const int32_t* op = y ? in.row(2 * y - 1) : a;
    for (uint32_t x = 0; x < in.w; x++)
      res.row(y)[x] = int32_t(int64_t(in.row(2 * y)[x]) - in.row(2 * y + 1)[x] - smooth_tendency(op[x], a[x], an[x]));
  }
}

void write_group_header(BitWriter& bw, const std::vector<jxg::ModularTransform>& tr) {
  bw.write(1, 1);  // use_global_tree
  bw.write(1, 1);  // WeightedHeader all_default
  if (tr.empty()) bw.write(0, 2);
  else if (tr.size() == 1) bw.write(1, 2);
  else {
    bw.write(2, 2);
    bw.write(tr.size() - 2, 4);
  }
  for (const auto& t : tr) {
    bw.write(t.id, 2);
    if (t.id == 0) {
      bw.write(0, 2);  // begin_channel selector 0: 3 bits
      bw.write(t.begin_channel, 3);
      if (t.rct_type == 6) bw.write(0, 2);
      else if (t.rct_type < 4) { bw.write(1, 2); bw.write(t.rct_type, 2); }
      else if (t.rct_type < 18) { bw.write(2, 2); bw.write(t.rct_type - 2, 4); }
      else { bw.write(3, 2); bw.write(t.rct_type - 10, 6); }
    } else if (t.id == 1) {  // headers/modular.rs:85-117
      bw.write(0, 2);  // begin_channel selector 0: 3 bits
      bw.write(t.begin_channel, 3);
      if (t.num_channels == 1) bw.write(0, 2);
      else if (t.num_channels == 3) bw.write(1, 2);
      else if (t.num_channels == 4) bw.write(2, 2);
      else { bw.write(3, 2); bw.write(t.num_channels - 1, 13); }
      if (t.num_colors < 256) { bw.write(0, 2); bw.write(t.num_colors, 8); }
      else if (t.num_colors < 1280) { bw.write(1, 2); bw.write(t.num_colors - 256, 10); }
      else if (t.num_colors < 5376) { bw.write(2, 2); bw.write(t.num_colors - 1280, 12); }
      else { bw.write(3, 2); bw.write(t.num_colors - 5376, 16); }
      if (t.num_deltas != 0) throw std::runtime_error("the synthetic writer has no delta palettes");
      bw.write(0, 2);  // num_deltas = 0
      bw.write(t.predictor_id, 4);
    } else {
      bw.write(0, 2);  // Squeeze with default parameters (num_sq = 0)
    }
  }
}

void append_bits(BitWriter& dst, BitWriter& src) {
  size_t total = src.total;
  BitWriter copy = src;
  std::vector<uint8_t> bytes = copy.finish();
  size_t full = total / 8;
  for (size_t i = 0; i < full; i++) dst.write(bytes[i], 8);
  if (total % 8) dst.write(bytes[full], unsigned(total % 8));
}
void write_toc_entry(BitWriter& bw, uint32_t v) {  // toc.rs:28
  if (v < 1024) bw.u2s_sel(0, v, 10);
  else if (v < 17408) bw.u2s_sel(1, v - 1024, 14);
  else if (v < 4211712) bw.u2s_sel(2, v - 17408, 22);
  else bw.u2s_sel(3, v - 4211712, 30);
}

bool is_meta(const ModularChannel& c) { return c.hshift < 0 || c.vshift < 0; }

}  // namespace

// ---- LZ77 copies in Modular streams ----------------------------------------------------------------------------------
// A Modular stream reads its copy distances with a multiplier, the widest channel of the stream (bitstream.rs:193-202):
// a distance symbol k < 120 is the special offset (dx, dy) of entropy_coding/decode.rs:87-101, distance
// multiplier * dy + dx (at least 1), and k >= 120 the plain distance k - 119. Either is capped at 2^20 and then at the
// number of symbols decoded so far (decode.rs:107-124). The writer states the rule for the four offsets it uses.
struct LzCensus {  // what the LZ77 modes wrote (the last encode of this thread): the tests assert reach with it
  uint64_t copies = 0, special = 0, plain = 0, cross_channel = 0, clamped = 0, max_distance = 0, max_stream = 0;
};
thread_local LzCensus g_lz_census;

namespace {

struct SpecialDist {
  uint32_t sym;
  int32_t dx, dy;
};
constexpr SpecialDist kSpecialUsed[] = {{0, 0, 1}, {1, 1, 0}, {2, 1, 1}, {3, -1, 1}};  // above, left, up-left, up-right
constexpr uint32_t kWindow = 1u << 20;

struct LzParams {
  Lz77 lz;
  HybridCfg cfg, len_cfg{0, 0, 0}, dist_cfg;
};

Sym literal_sym(const Token& t, const LzParams& P) {
  Sym s{t.ctx, 0, 0, 0};
  P.cfg.encode(t.value, s.tok, s.nbits, s.bits);
  if (s.tok >= P.lz.min_symbol) throw std::runtime_error("literal token collides with the LZ77 range");
  return s;
}

// One stream's tokens -> coded symbols with copies. mode 0: literals only; 1: run-length (every copy repeats the
// previous symbol: special symbol 1, the only symbol of the distance cluster); 2: general (the special offsets above,
// plain distances 2, 3, 4, 8, 64 and 2^20, copies whose distance the decoder clamps). chan_end: the symbol index where
// each channel ends. fault 1: the stream starts with a copy; 2: its first copy has a length that overflows u32.
std::vector<Sym> modular_lz77(const std::vector<Token>& t, const std::vector<size_t>& chan_end, uint32_t mult, uint32_t mode,
                              const LzParams& P, uint32_t dist_ctx, uint32_t fault, LzCensus& cs) {
  struct Cand {
    uint32_t sym, distance;  // distance symbol, distance before the clamp to the decoded count
    bool special;
  };
  std::vector<Cand> cands;
  if (mode == 1) cands.push_back(Cand{1, 1, true});
  if (mode == 2) {
    for (const SpecialDist& sd : kSpecialUsed) {
      const int64_t d = std::max<int64_t>(int64_t(mult) * sd.dy + sd.dx, 1);
      cands.push_back(Cand{sd.sym, uint32_t(std::min<int64_t>(d, kWindow)), true});
    }
    for (uint32_t d : {2u, 3u, 4u, 8u, 64u, kWindow}) cands.push_back(Cand{120 + d - 1, d, false});
  }
  const size_t max_len = mode == 1 ? (size_t(1) << 24) : 4096;
  const size_t min_len = std::max<size_t>(P.lz.min_length, mode == 1 ? 1 : 4);
  auto copy = [&](std::vector<Sym>& out, uint32_t ctx, uint64_t len, uint32_t dsym) {
    Sym l{ctx, 0, 0, 0};
    P.len_cfg.encode(uint32_t(len - P.lz.min_length), l.tok, l.nbits, l.bits);
    l.tok += P.lz.min_symbol;
    out.push_back(l);
    Sym d{dist_ctx, 0, 0, 0};
    P.dist_cfg.encode(dsym, d.tok, d.nbits, d.bits);
    out.push_back(d);
  };
  std::vector<Sym> out;
  out.reserve(t.size());
  cs.max_stream = std::max<uint64_t>(cs.max_stream, t.size());
  if (fault == 1 && !t.empty()) copy(out, t[0].ctx, P.lz.min_length, 1);
  for (size_t i = 0; i < t.size();) {
    size_t best_len = 0;
    const Cand* best = nullptr;
    for (const Cand& c : cands) {
      const size_t e = std::min<size_t>(c.distance, i);
      if (e == 0) continue;
      size_t l = 0;
      while (i + l < t.size() && l < max_len && t[i + l].value == t[i + l - e].value) l++;
      if (l > best_len) best_len = l, best = &c;
    }
    if (best && best_len >= min_len) {
      if (fault == 2) {  // the first copy gets a length the decoder must refuse (decode.rs:300-317)
        fault = 0;
        Sym l{t[i].ctx, 0, 0, 0};
        P.len_cfg.encode(0xffffffffu, l.tok, l.nbits, l.bits);
        l.tok += P.lz.min_symbol;
        out.push_back(l);
      }
      copy(out, t[i].ctx, best_len, best->sym);
      const size_t e = std::min<size_t>(best->distance, i);
      cs.copies++;
      (best->special ? cs.special : cs.plain)++;
      cs.clamped += best->distance > i;
      cs.max_distance = std::max<uint64_t>(cs.max_distance, e);
      const size_t c0 = std::upper_bound(chan_end.begin(), chan_end.end(), i) - chan_end.begin();
      const size_t c1 = std::upper_bound(chan_end.begin(), chan_end.end(), i + best_len - 1) - chan_end.begin();
      cs.cross_channel += c0 != c1;
      i += best_len;
    } else {
      out.push_back(literal_sym(t[i], P));
      i++;
    }
  }
  return out;
}

// The code of LZ77 streams: contexts [0, nctx) clustered by cmap into nc clusters, then the distance context alone in
// cluster nc with its own hybrid-uint configuration.
AnsCode lz_code(std::vector<uint8_t> cmap, uint32_t nc, const std::vector<const std::vector<Sym>*>& streams, bool prefix,
                const LzParams& P) {
  if (nc >= 256) throw std::runtime_error("too many clusters for an LZ77 code");
  cmap.push_back(uint8_t(nc));
  AnsCode c = build_code_lz77(cmap.size(), cmap, nc + 1, streams, P.lz, prefix);
  c.cfg = P.cfg;
  c.lz_len_cfg = P.len_cfg;
  c.lz_dist_own_cfg = true;
  c.lz_dist_cfg = P.dist_cfg;
  return c;
}

}  // namespace

// Snaps the picture to colours a palette transform without delta entries can carry three ways: the left quarter to the
// implicit 4x4x4 cube (levels 32, 95, 159, 223), the rest to the levels of the implicit 5x5x5 cube (0, 63, 127, 191, 255).
void snap_to_palette_colours(uint32_t W, uint32_t H, std::vector<uint8_t>& rgb) {
  for (uint32_t y = 0; y < H; y++)
    for (uint32_t x = 0; x < W; x++)
      for (int c = 0; c < 3; c++) {
        uint8_t& v = rgb[(size_t(y) * W + x) * 3 + c];
        if (x < W / 4) v = uint8_t((((uint32_t(v) * 4) >> 8) * 255u >> 2) + 32);
        else v = uint8_t((((uint32_t(v) * 5) >> 8) * 255u) >> 2);
      }
}

// f16 bits of a finite value that f16 represents exactly (headers/encodings.rs:59-74 reads it back unchanged).
uint16_t f16_bits_exact(float v) {
  if (v == 0.0f) return 0;
  int e = 0;
  const float m = std::frexp(std::fabs(v), &e);  // |v| = m * 2^e, m in [0.5, 1)
  const float mant = (m * 2.0f - 1.0f) * 1024.0f;
  if (e - 1 < -14 || e - 1 > 15 || mant != std::floor(mant)) throw std::runtime_error("value not exact in f16");
  return uint16_t((v < 0 ? 0x8000u : 0u) | (uint32_t(e - 1 + 15) << 10) | uint32_t(mant));
}

// The XYB mode's coded colour channels Y, X, B: the procedural picture in XYB quantised so that the decoder's
// X = x s_x, Y = y s_y, B = (b + y) s_b (render/stages/convert.rs:278-343) gives it back to within half a step.
void xyb_channels(uint32_t W, uint32_t H, uint64_t seed, const ModularXyb& xyb, std::vector<ModularChannel>& ch) {
  float lf_quant[3] = {1.0f / 4096.0f, 1.0f / 512.0f, 1.0f / 256.0f};  // quant_weights::LF_QUANT
  if (xyb.lf_quant_f16[0] != 0.0f || xyb.lf_quant_f16[1] != 0.0f || xyb.lf_quant_f16[2] != 0.0f)
    for (int c = 0; c < 3; c++) lf_quant[c] = jxg::f16_bits_to_float(f16_bits_exact(xyb.lf_quant_f16[c])) / 128.0f;
  std::vector<float> img[3];
  make_xyb_image(W, H, seed, img);
  ch.clear();
  for (int c = 0; c < 3; c++) ch.emplace_back(W, H, 0, 0);
  for (size_t i = 0; i < size_t(W) * H; i++) {
    const int32_t y = int32_t(std::lround(img[1][i] / lf_quant[1]));
    ch[0].data[i] = y;
    ch[1].data[i] = int32_t(std::lround(img[0][i] / lf_quant[0]));
    ch[2].data[i] = int32_t(std::lround(img[2][i] / lf_quant[2])) - y;
  }
}

std::vector<uint8_t> encode_modular(uint32_t W, uint32_t H, uint64_t seed, uint32_t rct_type, uint32_t squeeze,
                                    uint32_t tree_kind, const uint8_t* source_rgb, uint32_t palette, uint32_t lz77,
                                    const ModularXyb& xyb = ModularXyb()) {
  if (xyb.on && (source_rgb || palette)) throw std::runtime_error("the XYB mode takes no source image and no palette");
  std::vector<uint8_t> rgb;
  if (source_rgb) rgb.assign(source_rgb, source_rgb + size_t(W) * H * 3);
  else if (!xyb.on) make_image_u8(W, H, seed, rgb);
  if (palette && !source_rgb) snap_to_palette_colours(W, H, rgb);
  const uint32_t group_dim = 256;
  const uint32_t xg = (W + group_dim - 1) / group_dim, yg = (H + group_dim - 1) / group_dim, num_groups = xg * yg;
  const uint32_t lf_dim = group_dim * 8;
  const uint32_t xlg = (W + lf_dim - 1) / lf_dim, ylg = (H + lf_dim - 1) / lf_dim, num_lf_groups = xlg * ylg;

  // ---- channels + forward transforms ----
  std::vector<ModularChannel> ch;
  const bool custom_quant = xyb.lf_quant_f16[0] != 0.0f || xyb.lf_quant_f16[1] != 0.0f || xyb.lf_quant_f16[2] != 0.0f;
  if (xyb.on) {
    xyb_channels(W, H, seed, xyb, ch);
  } else {
    for (int c = 0; c < 3; c++) {
      ch.emplace_back(W, H, 0, 0);
      for (size_t i = 0; i < size_t(W) * H; i++) ch[c].data[i] = rgb[i * 3 + c];
    }
  }
  jxg::GroupHeader gh;
  gh.use_global_tree = true;
  if (palette) {
    // Forward palette over the three colour channels (meta_apply.rs:181-230 / palette.rs:165-199 inverted), no delta
    // entries, Zero predictor. Colours on the 5x5x5 cube with an odd level sum and all colours on the 4x4x4 cube use
    // the implicit entries behind the explicit ones; everything else gets an explicit entry.
    if (rct_type || squeeze) throw std::runtime_error("the synthetic palette variant takes no other global transform");
    auto cube5 = [](int32_t v) { return v == 0 ? 0 : v == 63 ? 1 : v == 127 ? 2 : v == 191 ? 3 : v == 255 ? 4 : -1; };
    auto cube4 = [](int32_t v) { return v == 32 ? 0 : v == 95 ? 1 : v == 159 ? 2 : v == 223 ? 3 : -1; };
    std::vector<uint32_t> colours;  // explicit entries, first appearance order
    std::vector<int32_t> entry_of(1u << 24, -1);
    std::vector<int32_t> pending(size_t(W) * H, 0);
    for (size_t i = 0; i < size_t(W) * H; i++) {
      const int32_t r = ch[0].data[i], g = ch[1].data[i], b = ch[2].data[i];
      const int a5 = cube5(r), b5 = cube5(g), c5 = cube5(b), a4 = cube4(r), b4 = cube4(g), c4 = cube4(b);
      if (a4 >= 0 && b4 >= 0 && c4 >= 0) pending[i] = -1 - (a4 | (b4 << 2) | (c4 << 4));            // small cube
      else if (a5 >= 0 && b5 >= 0 && c5 >= 0 && ((a5 + b5 + c5) & 1)) pending[i] = -100 - (a5 + 5 * b5 + 25 * c5);  // large cube
      else {
        const uint32_t key = uint32_t(r) | (uint32_t(g) << 8) | (uint32_t(b) << 16);
        if (entry_of[key] < 0) {
          entry_of[key] = int32_t(colours.size());
          colours.push_back(key);
        }
        pending[i] = entry_of[key];
      }
    }
    if (colours.empty()) colours.push_back(0);
    if (colours.size() > 5376) throw std::runtime_error("too many colours for the synthetic palette variant");
    const uint32_t N = uint32_t(colours.size());
    for (size_t i = 0; i < size_t(W) * H; i++) {
      const int32_t p = pending[i];
      ch[0].data[i] = p >= 0 ? p : (p > -100 ? int32_t(N) + (-1 - p) : int32_t(N) + 64 + (-100 - p));
    }
    ch.erase(ch.begin() + 1, ch.begin() + 3);
    ModularChannel pal(N, 3, -1, -1);
    for (uint32_t i = 0; i < N; i++)
      for (int c = 0; c < 3; c++) pal.row(uint32_t(c))[i] = int32_t((colours[i] >> (8 * c)) & 0xff);
    ch.insert(ch.begin(), std::move(pal));
    jxg::ModularTransform t;
    t.id = 1;
    t.begin_channel = 0;
    t.num_channels = 3;
    t.num_colors = N;
    t.num_deltas = 0;
    t.predictor_id = 0;
    gh.transforms.push_back(t);
  }
  if (rct_type) {
    if (rct_type != 6) throw std::runtime_error("the synthetic writer only has the forward YCoCg RCT (type 6)");
    jxg::ModularTransform t;
    t.id = 0;
    t.begin_channel = 0;
    t.rct_type = 6;
    gh.transforms.push_back(t);
    for (size_t i = 0; i < size_t(W) * H; i++) {  // inverse of rct.rs:27-37
      const int32_t r = ch[0].data[i], g = ch[1].data[i], b = ch[2].data[i];
      const int32_t co = r - b, tmp = b + (co >> 1), cg = g - tmp, y = tmp + (cg >> 1);
      ch[0].data[i] = y;
      ch[1].data[i] = co;
      ch[2].data[i] = cg;
    }
  }
  if (squeeze) {
    jxg::ModularTransform t;
    t.id = 2;
    gh.transforms.push_back(t);
    // derive the default parameter list exactly as the decoder will (squeeze.rs:39-105) on shape-only channels
    std::vector<ModularChannel> shapes;
    for (auto& c : ch) {
      ModularChannel s;
      s.w = c.w;
      s.h = c.h;
      shapes.push_back(s);
    }
    jxg::GroupHeader tmp;
    tmp.transforms.push_back(t);
    uint32_t nb_meta = 0;
    jxg::meta_apply_transforms(shapes, nb_meta, tmp, false);
    for (const auto& sq : tmp.transforms[0].squeezes) {
      const size_t b = sq.begin_channel, e = b + sq.num_channels;
      const size_t offset = sq.in_place ? e : ch.size();
      for (size_t c = b; c < e; c++) {
        ModularChannel avg, res;
        if (sq.horizontal) fwd_hsqueeze(ch[c], avg, res);
        else fwd_vsqueeze(ch[c], avg, res);
        ch[c] = std::move(avg);
        ch.insert(ch.begin() + offset + (c - b), std::move(res));
      }
    }
    for (size_t i = 0; i < ch.size(); i++)
      if (ch[i].w != shapes[i].w || ch[i].h != shapes[i].h) throw std::runtime_error("squeeze shape mismatch");
  }

  // ---- channel -> section assignment (modular/mod.rs:353-400, single pass) ----
  const std::vector<MNode> tree = make_tree(tree_kind);
  bool uses_wp = false;
  for (auto& n : tree)
    if ((n.property < 0 && n.predictor == 6) || n.property == 15) uses_wp = true;
  size_t n0 = 0;
  while (n0 < ch.size() && (is_meta(ch[n0]) || (ch[n0].w <= group_dim && ch[n0].h <= group_dim))) n0++;
  auto rect_of = [&](const ModularChannel& c, uint32_t dim, uint32_t gx, uint32_t gy) {
    ModularChannel r;
    const uint32_t gw = dim >> c.hshift, ghh = dim >> c.vshift;
    const uint64_t bx = uint64_t(gx) * gw, by = uint64_t(gy) * ghh;
    r.hshift = c.hshift;
    r.vshift = c.vshift;
    if (!gw || !ghh || bx >= c.w || by >= c.h) return r;
    r = ModularChannel(std::min<uint32_t>(c.w - uint32_t(bx), gw), std::min<uint32_t>(c.h - uint32_t(by), ghh), c.hshift, c.vshift);
    for (uint32_t y = 0; y < r.h; y++) memcpy(r.row(y), c.row(uint32_t(by) + y) + bx, size_t(r.w) * 4);
    return r;
  };
  std::vector<Token> tok0;
  std::vector<std::vector<Token>> tok_lf(num_lf_groups), tok_hf(num_groups);
  std::vector<std::vector<size_t>> hf_chan_end(num_groups);
  std::vector<uint32_t> hf_mult(num_groups, 0);
  {
    std::vector<ModularChannel> c0(ch.begin(), ch.begin() + n0);
    tokenize(c0, 0, tree, uses_wp, tok0);
  }
  for (uint32_t g = 0; g < num_lf_groups; g++) {
    std::vector<ModularChannel> cs;
    for (size_t c = n0; c < ch.size(); c++)
      if (std::min(ch[c].hshift, ch[c].vshift) >= 3) cs.push_back(rect_of(ch[c], lf_dim, g % xlg, g / xlg));
    tokenize(cs, 1 + num_lf_groups + g, tree, uses_wp, tok_lf[g]);
  }
  for (uint32_t g = 0; g < num_groups; g++) {
    std::vector<ModularChannel> cs;
    for (size_t c = n0; c < ch.size(); c++)
      if (std::min(ch[c].hshift, ch[c].vshift) <= 2) cs.push_back(rect_of(ch[c], group_dim, g % xg, g / xg));
    tokenize(cs, 1 + 3 * uint64_t(num_lf_groups) + 17 + g, tree, uses_wp, tok_hf[g]);
    size_t end = 0;
    for (const ModularChannel& c : cs) {
      hf_mult[g] = std::max(hf_mult[g], c.w);
      end += size_t(c.w) * c.h;
      hf_chan_end[g].push_back(end);
    }
  }

  // ---- entropy code over all streams ----
  size_t num_ctx = 0;
  for (auto& n : tree)
    if (n.property < 0) num_ctx++;
  std::vector<const std::vector<Token>*> all{&tok0};
  for (auto& t : tok_lf) all.push_back(&t);
  for (auto& t : tok_hf) all.push_back(&t);
  uint32_t nc;
  HybridCfg cfg;
  std::vector<uint8_t> cmap = cluster_contexts(num_ctx, all, 8, nc, cfg);
  AnsCode code;
  // lz77 != 0: the group streams carry copies (section 0 and the LF groups only literals, read with the same code)
  std::vector<Sym> sym0;
  std::vector<std::vector<Sym>> sym_lf(num_lf_groups), sym_hf(num_groups);
  if (lz77) {
    if (lz77 > 2) throw std::runtime_error("lz77 must be 0, 1 or 2");
    LzParams P;
    P.lz.enabled = true;
    P.cfg = cfg;
    P.dist_cfg = lz77 == 1 ? HybridCfg{0, 0, 0} : cfg;  // run-length: split exponent 0 (Histograms::is_rle)
    g_lz_census = LzCensus();
    const uint32_t dctx = uint32_t(num_ctx);
    sym0 = modular_lz77(tok0, {tok0.size()}, 0, 0, P, dctx, 0, g_lz_census);
    for (uint32_t g = 0; g < num_lf_groups; g++) sym_lf[g] = modular_lz77(tok_lf[g], {tok_lf[g].size()}, 0, 0, P, dctx, 0, g_lz_census);
    for (uint32_t g = 0; g < num_groups; g++)
      sym_hf[g] = modular_lz77(tok_hf[g], hf_chan_end[g], hf_mult[g], lz77, P, dctx, 0, g_lz_census);
    std::vector<const std::vector<Sym>*> ptrs{&sym0};
    for (auto& v : sym_lf) ptrs.push_back(&v);
    for (auto& v : sym_hf) ptrs.push_back(&v);
    code = lz_code(cmap, nc, ptrs, false, P);
  } else {
    code = build_code(num_ctx, cmap, nc, all);
  }
  auto write_stream = [&](BitWriter& bw, const std::vector<Token>& toks, const std::vector<Sym>& syms) {
    if (lz77) write_symbols(bw, code, syms);
    else write_tokens(bw, code, toks);
  };

  // ---- sections ----
  BitWriter lf_global;
  lf_global.write(custom_quant ? 0 : 1, 1);  // LfQuantFactors all_default
  if (custom_quant)
    for (int c = 0; c < 3; c++) lf_global.write(f16_bits_exact(xyb.lf_quant_f16[c]), 16);
  lf_global.write(1, 1);  // global tree present
  {
    std::vector<Token> tt;  // tree.rs:284-340: contexts 0 splitval, 1 property+1, 2 predictor, 3 offset, 4 mul_log, 5 mul_bits
    for (const MNode& n : tree) {
      if (n.property >= 0) {
        tt.push_back(Token{1, uint32_t(n.property + 1)});
        tt.push_back(Token{0, pack_signed(n.splitval)});
      } else {
        tt.push_back(Token{1, 0});
        tt.push_back(Token{2, n.predictor});
        tt.push_back(Token{3, 0});
        tt.push_back(Token{4, 0});
        tt.push_back(Token{5, 0});
      }
    }
    uint32_t tnc;
    HybridCfg tcfg;
    std::vector<uint8_t> tmap = cluster_contexts(6, {&tt}, 8, tnc, tcfg);
    AnsCode tcode = build_code(6, tmap, tnc, {&tt});
    write_code(lf_global, tcode);
    write_tokens(lf_global, tcode, tt);
  }
  write_code(lf_global, code);
  write_group_header(lf_global, gh.transforms);
  if (!tok0.empty()) write_stream(lf_global, tok0, sym0);
  std::vector<BitWriter> lf_groups(num_lf_groups), hf_groups(num_groups);
  for (uint32_t g = 0; g < num_lf_groups; g++)
    if (!tok_lf[g].empty()) {
      write_group_header(lf_groups[g], {});
      write_stream(lf_groups[g], tok_lf[g], sym_lf[g]);
    }
  for (uint32_t g = 0; g < num_groups; g++)
    if (!tok_hf[g].empty()) {
      write_group_header(hf_groups[g], {});
      write_stream(hf_groups[g], tok_hf[g], sym_hf[g]);
    }
  BitWriter hf_global;  // empty for Modular frames

  // ---- file assembly ----
  BitWriter out;
  out.write(0xff, 8);
  out.write(0x0a, 8);
  auto write_dim = [&](uint32_t v) {
    uint32_t m = v - 1;
    if (m < (1u << 9)) out.u2s_sel(0, m, 9);
    else if (m < (1u << 13)) out.u2s_sel(1, m, 13);
    else if (m < (1u << 18)) out.u2s_sel(2, m, 18);
    else out.u2s_sel(3, m, 30);
  };
  out.write(0, 1);  // small = false
  write_dim(H);
  out.write(0, 3);  // ratio 0
  write_dim(W);
  // ImageMetadata (image_metadata.rs:197-236)
  if (xyb.on) {
    write_xyb_image_metadata(out, xyb.orientation, xyb.colour);
  } else {
    out.write(0, 1);   // all_default
    out.write(0, 1);   // extra_fields
    out.write(0, 1);   // bit depth: integer samples
    out.write(0, 2);   // 8 bits
    out.write(1, 1);   // modular_16bit_buffers
    out.write(0, 2);   // no extra channels
    out.write(0, 1);   // xyb_encoded = false
    out.write(1, 1);   // ColorEncoding all_default (sRGB)
    out.write_u64(0);  // extensions
  }
  out.write(1, 1);   // CustomTransformData all_default
  out.zero_pad_to_byte();
  // FrameHeader (frame_header.rs:267-444)
  out.write(0, 1);   // all_default
  out.write(0, 2);   // RegularFrame
  out.write(1, 1);   // Modular
  out.write_u64(0);  // flags
  if (!xyb.on) out.write(0, 1);  // do_ycbcr (absent for XYB images)
  out.write(0, 2);   // upsampling 1
  out.write(1, 2);   // group_size_shift 1 (256)
  out.write(0, 2);   // one pass
  out.write(0, 1);   // have_crop
  out.write(0, 2);   // blending Replace
  out.write(1, 1);   // is_last
  out.write(0, 2);   // name length 0
  out.write(0, 1);   // RestorationFilter all_default = 0
  out.write(xyb.gab, 1);
  if (xyb.gab) out.write(0, 1);  // default Gaborish weights
  out.write(xyb.epf_iters, 2);
  if (xyb.epf_iters) {  // frame_header.rs:185-227 for a Modular frame: default weights and sigmas, then the EPF sigma
    out.write(0, 1);
    out.write(0, 1);
    out.write(f16_bits_exact(1.0f), 16);
  }
  out.write_u64(0);  // restoration filter extensions
  out.write_u64(0);  // frame header extensions
  std::vector<std::vector<uint8_t>> sections;
  if (num_groups == 1) {
    BitWriter all_bits;
    append_bits(all_bits, lf_global);
    append_bits(all_bits, lf_groups[0]);
    append_bits(all_bits, hf_global);
    append_bits(all_bits, hf_groups[0]);
    sections.push_back(all_bits.finish());
  } else {
    sections.push_back(lf_global.finish());
    for (auto& b : lf_groups) sections.push_back(b.finish());
    sections.push_back(hf_global.finish());
    for (auto& b : hf_groups) sections.push_back(b.finish());
  }
  out.write(0, 1);  // TOC not permuted
  out.zero_pad_to_byte();
  for (auto& s : sections) write_toc_entry(out, uint32_t(s.size()));
  out.zero_pad_to_byte();
  std::vector<uint8_t> bytes = out.finish();
  for (auto& s : sections) bytes.insert(bytes.end(), s.begin(), s.end());
  return bytes;
}

// ---------------------------------------------------------------------------------------------------------------------
// Token-level Modular writer: serialises a frame whose trees, transforms, group headers and symbols were all chosen by
// the caller (tests/modular_ref.py decodes forward and records what a decoder must read). It predicts nothing and
// validates nothing, so frames a decoder must refuse can be written too. Flat u32 description, in this order:
//   width, height, group_size_shift (0..3), grey, orientation (1..8), prefix codes, hybrid-uint split_exponent, msb,
//   lsb, the global tree, the number of sections (1 + LF groups + HF groups, in TOC order without HfGlobal), then
//   per section: kind (0: no bytes, 1: group header only, 2: group header + local tree + symbols), and for kind > 0:
//   use_global_tree, WeightedHeader default flag and its 11 fields (p1c p2c p3ca..p3ce w0..w3), the transforms, then
//   for kind 2: the local tree (empty when use_global_tree) and the symbols as count, (context, value) pairs.
// A tree is its node count followed by 5 words per node in BFS order: a split is {property + 1, split value, 0, 0, 0},
// a leaf {0, predictor, offset, mul_log, mul_bits}. Transforms are a count, then per transform its id followed by
// RCT: begin, type; palette: begin, num_c, num_colors, num_deltas, predictor; Squeeze: count, then per step
// horizontal, in_place, begin, num_c.
namespace {

struct WordReader {
  const uint32_t* w;
  size_t n, i = 0;
  uint32_t next() {
    if (i >= n) throw std::runtime_error("token description ends early");
    return w[i++];
  }
};

struct TokTree {
  std::vector<uint32_t> words;  // 5 per node
  size_t leaves = 0;
};

TokTree read_tok_tree(WordReader& r) {
  TokTree t;
  const uint32_t n = r.next();
  for (uint32_t i = 0; i < 5 * n; i++) t.words.push_back(r.next());
  for (uint32_t i = 0; i < n; i++) t.leaves += t.words[5 * i] == 0;
  return t;
}

// u2S field (headers/encodings.rs:76-98) with the four (bits, offset) distributions: the first one that holds v.
void write_u2s(BitWriter& bw, uint32_t v, const uint32_t (&d)[4][2]) {
  for (uint32_t s = 0; s < 4; s++) {
    const uint32_t bits = d[s][0], off = d[s][1];
    if (v < off) continue;
    if (bits == 0 ? v == off : uint64_t(v - off) < (uint64_t(1) << bits)) {
      bw.u2s_sel(s, v - off, bits);
      return;
    }
  }
  throw std::runtime_error("value not representable in its u2S field");
}

void copy_transforms(WordReader& r, BitWriter& bw) {  // GroupHeader transforms (headers/modular.rs:62-140)
  static const uint32_t kBegin[4][2] = {{3, 0}, {6, 8}, {10, 72}, {13, 1096}};
  const uint32_t nt = r.next();
  write_u2s(bw, nt, {{0, 0}, {0, 1}, {4, 2}, {8, 18}});
  for (uint32_t i = 0; i < nt; i++) {
    const uint32_t id = r.next();
    bw.write(id, 2);
    if (id == 0) {
      write_u2s(bw, r.next(), kBegin);
      write_u2s(bw, r.next(), {{0, 6}, {2, 0}, {4, 2}, {6, 10}});
    } else if (id == 1) {
      write_u2s(bw, r.next(), kBegin);
      write_u2s(bw, r.next(), {{0, 1}, {0, 3}, {0, 4}, {13, 1}});
      write_u2s(bw, r.next(), {{8, 0}, {10, 256}, {12, 1280}, {16, 5376}});
      write_u2s(bw, r.next(), {{0, 0}, {8, 1}, {10, 257}, {16, 1281}});
      bw.write(r.next(), 4);
    } else if (id == 2) {
      const uint32_t ns = r.next();
      write_u2s(bw, ns, {{0, 0}, {4, 1}, {6, 9}, {8, 41}});
      for (uint32_t s = 0; s < ns; s++) {
        bw.write(r.next(), 1);
        bw.write(r.next(), 1);
        write_u2s(bw, r.next(), kBegin);
        write_u2s(bw, r.next(), {{0, 1}, {0, 2}, {0, 3}, {4, 4}});
      }
    } else {
      throw std::runtime_error("transform id must be 0, 1 or 2");
    }
  }
}

// Tree symbols (tree.rs:284-351) under their own six-context code, then nothing else: the caller writes the code of
// the tree's leaves.
void write_tok_tree(BitWriter& bw, const TokTree& t) {
  std::vector<Token> tt;
  for (size_t i = 0; i < t.words.size(); i += 5) {
    const uint32_t* n = &t.words[i];
    tt.push_back(Token{1, n[0]});
    if (n[0]) {
      tt.push_back(Token{0, pack_signed(int32_t(n[1]))});
    } else {
      tt.push_back(Token{2, n[1]});
      tt.push_back(Token{3, pack_signed(int32_t(n[2]))});
      tt.push_back(Token{4, n[3]});
      tt.push_back(Token{5, n[4]});
    }
  }
  uint32_t tnc;
  HybridCfg tcfg;
  std::vector<uint8_t> tmap = cluster_contexts(6, {&tt}, 8, tnc, tcfg);
  AnsCode tcode = build_code(6, tmap, tnc, {&tt});
  write_code(bw, tcode);
  write_tokens(bw, tcode, tt);
}

// One cluster per leaf (up to 255 leaves), so that a decoder which takes another leaf reads another histogram.
AnsCode leaf_code(size_t leaves, const std::vector<const std::vector<Token>*>& streams, bool prefix, const HybridCfg& cfg) {
  const size_t nctx = std::max<size_t>(leaves, 1);
  uint32_t nc = 0;
  std::vector<uint8_t> cmap;
  if (nctx <= 255) {
    for (size_t i = 0; i < nctx; i++) cmap.push_back(uint8_t(i));
    nc = uint32_t(nctx);
  } else {
    cmap = cluster_contexts(nctx, streams, 16, nc, cfg);
  }
  for (auto* s : streams)
    for (const Token& t : *s)
      if (t.ctx >= nctx) throw std::runtime_error("symbol context beyond the tree's leaves");
  return build_code(nctx, cmap, nc, streams, 5, prefix, cfg);
}

}  // namespace

std::vector<uint8_t> encode_modular_tokens(const uint32_t* words, size_t nwords) {
  WordReader r{words, nwords};
  const uint32_t W = r.next(), H = r.next(), gshift = r.next(), grey = r.next(), orientation = r.next();
  const bool prefix = r.next() != 0;
  HybridCfg cfg;
  cfg.split_exponent = r.next();
  cfg.msb = r.next();
  cfg.lsb = r.next();
  if (gshift > 3 || orientation < 1 || orientation > 8 || !W || !H) throw std::runtime_error("bad frame geometry");
  const TokTree global = read_tok_tree(r);
  struct Section {
    uint32_t kind = 0;
    BitWriter header;  // group header (+ local tree when not using the global one) is written once the codes exist
    TokTree local;
    bool use_global = true;
    std::vector<Token> toks;
  };
  const uint32_t nsec = r.next();
  std::vector<Section> secs(nsec);
  for (Section& s : secs) {
    s.kind = r.next();
    if (s.kind == 0) continue;
    s.use_global = r.next() != 0;
    s.header.write(s.use_global, 1);
    const uint32_t wp_default = r.next();
    uint32_t wp[11];
    for (uint32_t& v : wp) v = r.next();
    s.header.write(wp_default, 1);
    if (!wp_default) {
      for (int i = 0; i < 7; i++) s.header.write(wp[i], 5);
      for (int i = 7; i < 11; i++) s.header.write(wp[i], 4);
    }
    copy_transforms(r, s.header);
    if (s.kind < 2) continue;
    s.local = read_tok_tree(r);
    const uint32_t nt = r.next();
    for (uint32_t i = 0; i < nt; i++) {
      const uint32_t ctx = r.next();
      s.toks.push_back(Token{ctx, r.next()});
    }
  }
  // optional LZ77 block: min_symbol, min_length, length hybrid config (3 words), mode, fault kind, fault section, then
  // one distance multiplier per section
  const bool lz = r.i != r.n;
  LzParams P;
  uint32_t lz_mode = 0, fault = 0, fault_sec = 0;
  std::vector<uint32_t> mult(nsec, 0);
  if (lz) {
    P.lz.enabled = true;
    P.lz.min_symbol = r.next();
    P.lz.min_length = r.next();
    P.len_cfg.split_exponent = r.next();
    P.len_cfg.msb = r.next();
    P.len_cfg.lsb = r.next();
    lz_mode = r.next();
    fault = r.next();
    fault_sec = r.next();
    for (uint32_t& m : mult) m = r.next();
    if (lz_mode < 1 || lz_mode > 2) throw std::runtime_error("lz77 mode must be 1 or 2");
    P.cfg = cfg;
    P.dist_cfg = lz_mode == 1 ? HybridCfg{0, 0, 0} : cfg;
  }
  if (r.i != r.n) throw std::runtime_error("token description has trailing words");
  // leaf contexts one cluster each, the distance context after them
  std::vector<std::vector<Sym>> syms(nsec);
  auto leaf_map = [](size_t leaves) {
    if (leaves > 255) throw std::runtime_error("an LZ77 code takes at most 255 leaves");
    std::vector<uint8_t> m(std::max<size_t>(leaves, 1));
    for (size_t i = 0; i < m.size(); i++) m[i] = uint8_t(i);
    return m;
  };
  if (lz) {
    g_lz_census = LzCensus();
    for (uint32_t i = 0; i < nsec; i++) {
      if (secs[i].kind != 2) continue;
      const size_t dctx = std::max<size_t>(secs[i].use_global ? global.leaves : secs[i].local.leaves, 1);
      syms[i] = modular_lz77(secs[i].toks, {secs[i].toks.size()}, mult[i], lz_mode, P, uint32_t(dctx),
                             fault && i == fault_sec ? fault : 0, g_lz_census);
    }
  }

  // the global code covers every section that uses the global tree
  std::vector<const std::vector<Token>*> gstreams;
  std::vector<const std::vector<Sym>*> gsyms;
  for (uint32_t i = 0; i < nsec; i++)
    if (secs[i].kind == 2 && secs[i].use_global) {
      gstreams.push_back(&secs[i].toks);
      gsyms.push_back(&syms[i]);
    }
  const AnsCode gcode = lz ? lz_code(leaf_map(global.leaves), uint32_t(leaf_map(global.leaves).size()), gsyms, prefix, P)
                           : leaf_code(global.leaves, gstreams, prefix, cfg);
  auto section_bits = [&](uint32_t i, BitWriter& out) {
    Section& s = secs[i];
    if (s.kind == 0) return;
    append_bits(out, s.header);
    if (s.kind < 2) return;
    if (s.use_global) {
      if (lz) write_symbols(out, gcode, syms[i]);
      else write_tokens(out, gcode, s.toks);
    } else {
      write_tok_tree(out, s.local);
      if (lz) {
        const AnsCode lcode = lz_code(leaf_map(s.local.leaves), uint32_t(leaf_map(s.local.leaves).size()), {&syms[i]}, prefix, P);
        write_code(out, lcode);
        write_symbols(out, lcode, syms[i]);
        return;
      }
      const AnsCode lcode = leaf_code(s.local.leaves, {&s.toks}, prefix, cfg);
      write_code(out, lcode);
      write_tokens(out, lcode, s.toks);
    }
  };

  const uint32_t group_dim = 128u << gshift;
  const uint32_t xg = (W + group_dim - 1) / group_dim, yg = (H + group_dim - 1) / group_dim, num_groups = xg * yg;
  const uint32_t lf_dim = group_dim * 8;
  const uint32_t num_lf_groups = ((W + lf_dim - 1) / lf_dim) * ((H + lf_dim - 1) / lf_dim);
  if (nsec != 1 + num_lf_groups + num_groups) throw std::runtime_error("section count does not match the geometry");

  BitWriter lf_global;
  lf_global.write(1, 1);  // LfQuantFactors all_default
  lf_global.write(1, 1);  // global tree present
  write_tok_tree(lf_global, global);
  write_code(lf_global, gcode);
  section_bits(0, lf_global);
  std::vector<BitWriter> groups(nsec - 1);
  for (uint32_t i = 1; i < nsec; i++) section_bits(i, groups[i - 1]);

  BitWriter out;
  out.write(0xff, 8);
  out.write(0x0a, 8);
  auto write_dim = [&](uint32_t v) {
    uint32_t m = v - 1;
    if (m < (1u << 9)) out.u2s_sel(0, m, 9);
    else if (m < (1u << 13)) out.u2s_sel(1, m, 13);
    else if (m < (1u << 18)) out.u2s_sel(2, m, 18);
    else out.u2s_sel(3, m, 30);
  };
  out.write(0, 1);  // small = false
  write_dim(H);
  out.write(0, 3);  // ratio 0
  write_dim(W);
  // ImageMetadata (image_metadata.rs:197-236)
  out.write(0, 1);                // all_default
  out.write(1, 1);                // extra_fields
  out.write(orientation - 1, 3);
  out.write(0, 1);                // have_intrinsic_size
  out.write(0, 1);                // have_preview
  out.write(0, 1);                // have_animation
  out.write(0, 1);                // bit depth: integer samples
  out.u2s_sel(0);                 //            8 bits
  out.write(1, 1);                // modular_16bit_buffers
  out.u2s_sel(0);                 // no extra channels
  out.write(0, 1);                // xyb_encoded = false
  if (!grey) {
    out.write(1, 1);              // ColorEncoding all_default (sRGB)
  } else {                        // color_encoding.rs:166-196: grey, D65, sRGB curve, relative intent
    out.write(0, 1);
    out.write(0, 1);              // want_icc
    out.u2s_sel(1);               // colour space Gray
    out.u2s_sel(1);               // white point D65
    out.write(0, 1);              // have_gamma
    out.u2s_sel(2, 13 - 2, 4);    // transfer function sRGB (13)
    out.u2s_sel(1);               // rendering intent relative
  }
  out.write(1, 1);                // ToneMapping all_default
  out.write_u64(0);               // extensions
  out.write(1, 1);                // CustomTransformData all_default
  out.zero_pad_to_byte();
  // FrameHeader (frame_header.rs:267-444)
  out.write(0, 1);   // all_default
  out.write(0, 2);   // RegularFrame
  out.write(1, 1);   // Modular
  out.write_u64(0);  // flags
  out.write(0, 1);   // do_ycbcr
  out.write(0, 2);   // upsampling 1
  out.write(gshift, 2);
  out.write(0, 2);   // one pass
  out.write(0, 1);   // have_crop
  out.write(0, 2);   // blending Replace
  out.write(1, 1);   // is_last
  out.write(0, 2);   // name length 0
  out.write(0, 1);   // RestorationFilter all_default = 0
  out.write(0, 1);   // gab off
  out.write(0, 2);   // epf off
  out.write_u64(0);  // restoration filter extensions
  out.write_u64(0);  // frame header extensions
  std::vector<std::vector<uint8_t>> sections;
  BitWriter hf_global;  // empty for Modular frames
  if (num_groups == 1) {
    BitWriter all_bits;
    append_bits(all_bits, lf_global);
    append_bits(all_bits, groups[0]);
    append_bits(all_bits, hf_global);
    append_bits(all_bits, groups[1]);
    sections.push_back(all_bits.finish());
  } else {
    sections.push_back(lf_global.finish());
    for (uint32_t g = 0; g < num_lf_groups; g++) sections.push_back(groups[g].finish());
    sections.push_back(hf_global.finish());
    for (uint32_t g = 0; g < num_groups; g++) sections.push_back(groups[num_lf_groups + g].finish());
  }
  out.write(0, 1);  // TOC not permuted
  out.zero_pad_to_byte();
  for (auto& s : sections) write_toc_entry(out, uint32_t(s.size()));
  out.zero_pad_to_byte();
  std::vector<uint8_t> bytes = out.finish();
  for (auto& s : sections) bytes.insert(bytes.end(), s.begin(), s.end());
  return bytes;
}

}  // namespace jxs

extern "C" {

static thread_local std::string g_merr;
const char* jxs_modular_last_error() { return g_merr.c_str(); }

// The 8-bit RGB source image of seed `seed` (interleaved), what a lossless decode must reproduce.
int jxs_modular_source_ex(uint32_t width, uint32_t height, uint64_t seed, uint32_t palette, uint8_t* out_rgb) {
  try {
    std::vector<uint8_t> rgb;
    jxs::make_image_u8(width, height, seed, rgb);
    if (palette) jxs::snap_to_palette_colours(width, height, rgb);
    memcpy(out_rgb, rgb.data(), rgb.size());
    return 0;
  } catch (std::exception& e) {
    g_merr = e.what();
    return -1;
  }
}

int jxs_modular_source(uint32_t width, uint32_t height, uint64_t seed, uint8_t* out_rgb) {
  try {
    std::vector<uint8_t> rgb;
    jxs::make_image_u8(width, height, seed, rgb);
    memcpy(out_rgb, rgb.data(), rgb.size());
    return 0;
  } catch (std::exception& e) {
    g_merr = e.what();
    return -1;
  }
}

// rct: 0 = none, 6 = YCoCg; squeeze: 0/1 (default parameters); tree_kind: 0 one Gradient leaf, 1 property tree
// without the weighted predictor, 2 weighted-predictor tree. source_rgb: optional caller-supplied image.
int64_t jxs_encode_modular(uint32_t width, uint32_t height, uint64_t seed, uint32_t rct, uint32_t squeeze,
                           uint32_t tree_kind, const uint8_t* source_rgb, uint8_t* out, size_t cap) {
  try {
    std::vector<uint8_t> b = jxs::encode_modular(width, height, seed, rct, squeeze, tree_kind, source_rgb, 0, 0);
    if (b.size() <= cap && out) memcpy(out, b.data(), b.size());
    return int64_t(b.size());
  } catch (std::exception& e) {
    g_merr = e.what();
    return -1;
  }
}

// palette: 1 = forward palette over the three colour channels (no delta entries); the picture is first snapped to
// colours of the implicit cubes / a few hundred explicit entries (jxs_modular_source_ex returns that picture).
int64_t jxs_encode_modular_ex(uint32_t width, uint32_t height, uint64_t seed, uint32_t rct, uint32_t squeeze,
                              uint32_t tree_kind, uint32_t palette, const uint8_t* source_rgb, uint8_t* out, size_t cap) {
  try {
    std::vector<uint8_t> b = jxs::encode_modular(width, height, seed, rct, squeeze, tree_kind, source_rgb, palette, 0);
    if (b.size() <= cap && out) memcpy(out, b.data(), b.size());
    return int64_t(b.size());
  } catch (std::exception& e) {
    g_merr = e.what();
    return -1;
  }
}

// lz77: 1 = run-length copies (distance 1 only, the distance cluster a single symbol), 2 = general copies.
int64_t jxs_encode_modular_lz77(uint32_t width, uint32_t height, uint64_t seed, uint32_t rct, uint32_t squeeze,
                                uint32_t tree_kind, uint32_t palette, uint32_t lz77, const uint8_t* source_rgb, uint8_t* out,
                                size_t cap) {
  try {
    std::vector<uint8_t> b = jxs::encode_modular(width, height, seed, rct, squeeze, tree_kind, source_rgb, palette, lz77);
    if (b.size() <= cap && out) memcpy(out, b.data(), b.size());
    return int64_t(b.size());
  } catch (std::exception& e) {
    g_merr = e.what();
    return -1;
  }
}

// The census of the last LZ77 encode of this thread: copies, special distances, plain distances, copies crossing a
// channel boundary, copies the decoder clamps, the longest distance, the longest stream (symbols).
void jxs_modular_lz77_census(uint64_t* out) {
  const jxs::LzCensus& c = jxs::g_lz_census;
  const uint64_t v[7] = {c.copies, c.special, c.plain, c.cross_channel, c.clamped, c.max_distance, c.max_stream};
  memcpy(out, v, sizeof(v));
}

// The token-level writer (encode_modular_tokens above): `words` is the flat frame description.
// The coded channels Y, X, B (3 x height x width i32) of the XYB mode's frame of `seed` and factors q_f16.
int jxs_modular_xyb_source(uint32_t width, uint32_t height, uint64_t seed, const float* q_f16, int32_t* out) {
  try {
    jxs::ModularXyb x;
    for (int c = 0; c < 3; c++) x.lf_quant_f16[c] = q_f16 ? q_f16[c] : 0.0f;
    std::vector<jxg::ModularChannel> ch;
    jxs::xyb_channels(width, height, seed, x, ch);
    for (int c = 0; c < 3; c++) memcpy(out + size_t(c) * width * height, ch[c].data.data(), size_t(width) * height * 4);
    return 0;
  } catch (std::exception& e) {
    g_merr = e.what();
    return -1;
  }
}

// The XYB mode (ModularXyb): q_f16 the three LfQuantFactors as written (NULL or all zero: the defaults).
int64_t jxs_encode_modular_xyb(uint32_t width, uint32_t height, uint64_t seed, uint32_t rct, uint32_t squeeze,
                               uint32_t tree_kind, const float* q_f16, uint32_t colour, uint32_t orientation, uint32_t gab,
                               uint32_t epf_iters, uint8_t* out, size_t cap) {
  try {
    if (orientation < 1 || orientation > 8 || colour > 7 || gab > 1 || epf_iters > 3)
      throw std::runtime_error("XYB mode: orientation 1..8, colour 0..7, gab 0/1, epf_iters 0..3");
    jxs::ModularXyb x;
    x.on = true;
    for (int c = 0; c < 3; c++) x.lf_quant_f16[c] = q_f16 ? q_f16[c] : 0.0f;
    x.colour = colour;
    x.orientation = orientation;
    x.gab = gab;
    x.epf_iters = epf_iters;
    std::vector<uint8_t> b = jxs::encode_modular(width, height, seed, rct, squeeze, tree_kind, nullptr, 0, 0, x);
    if (b.size() <= cap) memcpy(out, b.data(), b.size());
    return int64_t(b.size());
  } catch (std::exception& e) {
    g_merr = e.what();
    return -1;
  }
}

int64_t jxs_encode_modular_tokens(const uint32_t* words, size_t nwords, uint8_t* out, size_t cap) {
  try {
    std::vector<uint8_t> b = jxs::encode_modular_tokens(words, nwords);
    if (b.size() <= cap && out) memcpy(out, b.data(), b.size());
    return int64_t(b.size());
  } catch (std::exception& e) {
    g_merr = e.what();
    return -1;
  }
}
}
