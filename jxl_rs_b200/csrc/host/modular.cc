// See modular.h.
#include "modular.h"

#include <immintrin.h>

#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <type_traits>

namespace jxg {

namespace {
struct ChannelBufferPool {
  static constexpr size_t kMaxBuffers = 16, kMinSamples = 4096, kMaxSamples = size_t(4) << 20;
  std::vector<std::vector<int32_t>> free_list;
};
thread_local ChannelBufferPool tl_channel_pool;
}  // namespace

std::vector<int32_t> take_channel_buffer(size_t n) {
  auto& fl = tl_channel_pool.free_list;
  if (n >= ChannelBufferPool::kMinSamples && !fl.empty()) {
    // best fit among the (few) pooled buffers: the smallest capacity that holds n, else the largest
    size_t best = 0;
    for (size_t i = 1; i < fl.size(); i++) {
      const size_t ci = fl[i].capacity(), cb = fl[best].capacity();
      if ((ci >= n && (cb < n || ci < cb)) || (ci < n && cb < n && ci > cb)) best = i;
    }
    std::vector<int32_t> v = std::move(fl[best]);
    fl.erase(fl.begin() + best);
    v.assign(n, 0);
    return v;
  }
  return std::vector<int32_t>(n, 0);
}

void give_channel_buffer(std::vector<int32_t>&& buf) {
  const size_t cap = buf.capacity();
  auto& fl = tl_channel_pool.free_list;
  if (cap >= ChannelBufferPool::kMinSamples && cap <= ChannelBufferPool::kMaxSamples &&
      fl.size() < ChannelBufferPool::kMaxBuffers) {
    fl.push_back(std::move(buf));
  } else {
    std::vector<int32_t>().swap(buf);
  }
}

namespace {

struct U32D {
  uint32_t bits, off;
};
inline uint32_t u2s(BitReader& br, U32D a, U32D b, U32D c, U32D d) {
  const U32D ds[4] = {a, b, c, d};
  const U32D& s = ds[br.read(2)];
  return uint32_t(br.read(s.bits)) + s.off;
}
constexpr U32D V(uint32_t v) { return U32D{0, v}; }
constexpr U32D B(uint32_t n, uint32_t off = 0) { return U32D{n, off}; }

inline int32_t wadd(int32_t a, int32_t b) { return int32_t(uint32_t(a) + uint32_t(b)); }
inline int32_t wsub(int32_t a, int32_t b) { return int32_t(uint32_t(a) - uint32_t(b)); }
inline int32_t wabs(int32_t a) { return a < 0 ? int32_t(0u - uint32_t(a)) : a; }

enum Predictor : uint32_t {
  kZero = 0, kWest, kNorth, kAvgWN, kSelect, kGradient, kWeighted, kNorthEast, kNorthWest, kWestWest, kAvgWNW,
  kAvgNNW, kAvgNNE, kAvgAll, kNumPredictors
};

// predict.rs:137-143
inline int64_t clamped_gradient(int64_t left, int64_t top, int64_t topleft) {
  int64_t mn = std::min(left, top), mx = std::max(left, top);
  int64_t grad = left + top - topleft;
  int64_t g = topleft < mn ? mx : grad;
  return topleft > mx ? mn : g;
}

struct Neigh {
  int32_t left, top, toptop, topleft, topright, leftleft, toprightright;
};

// predict.rs:64-103 (get_rows)
inline Neigh get_neigh(const int32_t* row, const int32_t* top_row, const int32_t* toptop_row, size_t x, size_t y,
                       size_t w) {
  Neigh n;
  n.left = x > 0 ? row[x - 1] : (y > 0 ? top_row[0] : 0);
  n.top = y > 0 ? top_row[x] : n.left;
  n.topleft = (x > 0 && y > 0) ? top_row[x - 1] : n.left;
  n.topright = (x + 1 < w && y > 0) ? top_row[x + 1] : n.top;
  n.leftleft = x > 1 ? row[x - 2] : n.left;
  n.toptop = y > 1 ? toptop_row[x] : n.top;
  n.toprightright = (x + 2 < w && y > 0) ? top_row[x + 2] : n.topright;
  return n;
}

// get_neigh for 2 <= x < w - 2, y >= 2: every neighbour exists
inline Neigh get_neigh_interior(const int32_t* row, const int32_t* top_row, const int32_t* toptop_row, size_t x) {
  Neigh n;
  n.left = row[x - 1];
  n.top = top_row[x];
  n.topleft = top_row[x - 1];
  n.topright = top_row[x + 1];
  n.leftleft = row[x - 2];
  n.toptop = toptop_row[x];
  n.toprightright = top_row[x + 2];
  return n;
}

// predict.rs:148-194
inline int64_t predict_one(uint32_t p, const Neigh& n, int64_t wp_pred) {
  int64_t left = n.left, top = n.top, topleft = n.topleft, topright = n.topright;
  switch (p) {
    case kZero: return 0;
    case kWest: return left;
    case kNorth: return top;
    case kSelect: {
      int64_t pp = left + top - topleft;
      return std::llabs(pp - left) < std::llabs(pp - top) ? left : top;
    }
    case kGradient: return clamped_gradient(left, top, topleft);
    case kWeighted: return wp_pred;
    case kWestWest: return n.leftleft;
    case kNorthEast: return topright;
    case kNorthWest: return topleft;
    case kAvgWN: return (top + left) / 2;
    case kAvgWNW: return (left + topleft) / 2;
    case kAvgNNW: return (top + topleft) / 2;
    case kAvgNNE: return (top + topright) / 2;
    case kAvgAll:
      return (6 * top - 2 * int64_t(n.toptop) + 7 * left + int64_t(n.leftleft) + int64_t(n.toprightright) +
              3 * topright + 8) / 16;
  }
  return 0;
}

// c ? a : b without a branch
inline int64_t bsel(bool c, int64_t a, int64_t b) { return b ^ ((a ^ b) & (int64_t(0) - int64_t(c))); }

const uint32_t kDivLookup[64] = {
    16777216, 8388608, 5592405, 4194304, 3355443, 2796202, 2396745, 2097152, 1864135, 1677721, 1525201,
    1398101,  1290555, 1198372, 1118481, 1048576, 986895,  932067,  883011,  838860,  798915,  762600,
    729444,   699050,  671088,  645277,  621378,  599186,  578524,  559240,  541200,  524288,  508400,
    493447,   479349,  466033,  453438,  441505,  430185,  419430,  409200,  399457,  390167,  381300,
    372827,   364722,  356962,  349525,  342392,  335544,  328965,  322638,  316551,  310689,  305040,
    299593,   294337,  289262,  284359,  279620,  275036,  270600,  266305,  262144,
};

}  // namespace

// ---------------------------------------------------------------------------
// Weighted predictor
// ---------------------------------------------------------------------------

WpState::WpState(const WeightedHeader& h, size_t xs) : xsize(xs), hdr(h) {
  size_t n = (xs + 1) * 2;
  pred_errors.assign(n * 4, 0);
  error.assign(n, 0);
}

// Force-inlined bodies: the per-pixel loops call these directly (a call per pixel with nine arguments and results
// through memory costs ~15 % of the weighted-predictor path); WpState::predict / update are the out-of-line entry points.
__attribute__((always_inline)) static inline void wp_predict(WpState& S, size_t x, size_t y, int32_t top, int32_t left,
                                                             int32_t topright, int32_t topleft, int32_t toptop,
                                                             int64_t& pred_out, int32_t& prop_out) {
  const size_t xsize = S.xsize;
  const WeightedHeader& hdr = S.hdr;
  const uint32_t* pred_errors = S.pred_errors.data();
  const int32_t* error = S.error.data();
  size_t cur_row = (y & 1) ? 0 : xsize + 1, prev_row = (y & 1) ? xsize + 1 : 0;
  size_t pos_ne = x + 1 < xsize ? x + 1 : x;
  size_t pos_nw = x > 0 ? x - 1 : 0;
  const uint32_t* en = &pred_errors[(prev_row + x) * 4];
  const uint32_t* ene = &pred_errors[(prev_row + pos_ne) * 4];
  const uint32_t* enw = &pred_errors[(prev_row + pos_nw) * 4];
  uint32_t wv[4];
  for (int i = 0; i < 4; i++) {
    uint32_t err = en[i] + ene[i] + enw[i];
    uint32_t l2 = floor_log2(uint64_t(err) + 1);
    uint32_t shift = l2 > 5 ? l2 - 5 : 0;
    uint32_t div = kDivLookup[err >> shift];
    wv[i] = 4u + ((hdr.w[i] * div) >> shift);
  }
  int64_t te_w = error[cur_row + x];
  int64_t te_n = error[prev_row + 1 + x];
  int64_t te_nw = error[prev_row + 1 + pos_nw];
  int64_t sum_wn = te_n + te_w;
  int64_t te_ne = error[prev_row + 1 + pos_ne];
  // the property is the neighbouring error of largest magnitude; which one that is depends on the data, so the
  // selections are written as masks (mispredicted branches otherwise)
  int64_t p = te_w;
  p = bsel(std::llabs(te_n) > std::llabs(p), te_n, p);
  p = bsel(std::llabs(te_nw) > std::llabs(p), te_nw, p);
  p = bsel(std::llabs(te_ne) > std::llabs(p), te_ne, p);
  // add_bits (predict.rs): value * 8 (a multiplication: << on a negative value is undefined before C++20)
  int64_t n = int64_t(top) * 8, w = int64_t(left) * 8, ne = int64_t(topright) * 8, nw = int64_t(topleft) * 8,
          nn = int64_t(toptop) * 8;
  int64_t p0 = w + ne - n;
  int64_t p1 = n - (((sum_wn + te_ne) * int64_t(hdr.p1c)) >> 5);
  int64_t p2 = w - (((sum_wn + te_nw) * int64_t(hdr.p2c)) >> 5);
  int64_t p3 = n - ((te_nw * int64_t(hdr.p3ca) + te_n * int64_t(hdr.p3cb) + te_ne * int64_t(hdr.p3cc) +
                     (nn - n) * int64_t(hdr.p3cd) + (nw - w) * int64_t(hdr.p3ce)) >> 5);
  uint32_t log_weight = floor_log2(uint64_t(wv[0]) + wv[1] + wv[2] + wv[3]);
  int64_t w0 = int64_t(wv[0]) >> (log_weight - 4), w1 = int64_t(wv[1]) >> (log_weight - 4),
          w2 = int64_t(wv[2]) >> (log_weight - 4), w3 = int64_t(wv[3]) >> (log_weight - 4);
  int64_t weight_sum = w0 + w1 + w2 + w3;
  int64_t sum = (weight_sum >> 1) - 1 + w0 * p0 + w1 * p1 + w2 * p2 + w3 * p3;
  int64_t pr = (sum * int64_t(kDivLookup[weight_sum - 1])) >> 24;
  {
    const int64_t mx = bsel(w > ne, w, ne), mx3 = bsel(mx > n, mx, n);
    const int64_t mn = bsel(w < ne, w, ne), mn3 = bsel(mn < n, mn, n);
    const int64_t lo = bsel(mx3 < pr, mx3, pr);          // min(mx, pr)
    const int64_t clamped = bsel(mn3 > lo, mn3, lo);     // max(mn, min(mx, pr))
    pr = bsel(((te_n ^ te_w) | (te_n ^ te_nw)) <= 0, clamped, pr);
  }
  S.prediction[0] = p0;
  S.prediction[1] = p1;
  S.prediction[2] = p2;
  S.prediction[3] = p3;
  S.pred = pr;
  pred_out = (pr + 3) >> 3;
  prop_out = int32_t(p);
}

__attribute__((always_inline)) static inline void wp_update(WpState& S, int32_t val, size_t x, size_t y) {
  const size_t xsize = S.xsize;
  uint32_t* pred_errors = S.pred_errors.data();
  int32_t* error = S.error.data();
  const int64_t pred = S.pred;
  const int64_t* prediction = S.prediction;
  size_t cur_row = (y & 1) ? 0 : xsize + 1, prev_row = (y & 1) ? xsize + 1 : 0;
  int64_t v = int64_t(val) * 8;
  error[cur_row + x + 1] = int32_t(pred - v);
  uint32_t* cur = &pred_errors[(cur_row + x) * 4];
  uint32_t* prev = &pred_errors[(prev_row + x + 1) * 4];
  for (int i = 0; i < 4; i++) {
    uint32_t e = uint32_t((std::llabs(prediction[i] - v) + 3) >> 3);
    cur[i] = e;
    prev[i] += e;
  }
}

void WpState::predict(size_t x, size_t y, int32_t top, int32_t left, int32_t topright, int32_t topleft,
                      int32_t toptop, int64_t& pred_out, int32_t& prop_out) {
  wp_predict(*this, x, y, top, left, topright, topleft, toptop, pred_out, prop_out);
}

void WpState::update(int32_t val, size_t x, size_t y) { wp_update(*this, val, x, y); }

// ---------------------------------------------------------------------------
// Headers / tree
// ---------------------------------------------------------------------------

GroupHeader GroupHeader::read(BitReader& br) {
  GroupHeader g;
  g.use_global_tree = br.read_bool();
  if (!br.read_bool()) {  // WeightedHeader all_default
    WeightedHeader& w = g.wp;
    w.p1c = uint32_t(br.read(5));
    w.p2c = uint32_t(br.read(5));
    w.p3ca = uint32_t(br.read(5));
    w.p3cb = uint32_t(br.read(5));
    w.p3cc = uint32_t(br.read(5));
    w.p3cd = uint32_t(br.read(5));
    w.p3ce = uint32_t(br.read(5));
    for (auto& x : w.w) x = uint32_t(br.read(4));
  }
  uint32_t nt = u2s(br, V(0), V(1), B(4, 2), B(8, 18));
  g.transforms.resize(nt);
  for (auto& t : g.transforms) {
    t.id = uint32_t(br.read(2));
    if (t.id == 3) fail("invalid modular transform");
    if (t.id == 0 || t.id == 1) t.begin_channel = u2s(br, B(3), B(6, 8), B(10, 72), B(13, 1096));
    if (t.id == 0) {
      t.rct_type = u2s(br, V(6), B(2), B(4, 2), B(6, 10));
      if (t.rct_type >= 42) fail("invalid RCT type");
    }
    if (t.id == 1) {
      t.num_channels = u2s(br, V(1), V(3), V(4), B(13, 1));
      t.num_colors = u2s(br, B(8), B(10, 256), B(12, 1280), B(16, 5376));
      t.num_deltas = u2s(br, V(0), B(8, 1), B(10, 257), B(16, 1281));
      t.predictor_id = uint32_t(br.read(4));
      if (t.predictor_id >= kNumPredictors) fail("invalid predictor");
    }
    if (t.id == 2) {
      uint32_t ns = u2s(br, V(0), B(4, 1), B(6, 9), B(8, 41));
      t.squeezes.resize(ns);
      for (auto& s : t.squeezes) {
        s.horizontal = br.read_bool();
        s.in_place = br.read_bool();
        s.begin_channel = u2s(br, B(3), B(6, 8), B(10, 72), B(13, 1096));
        s.num_channels = u2s(br, V(1), V(2), V(3), B(4, 4));
      }
    }
  }
  br.check();
  return g;
}

// tree.rs:39-155 (validate_tree): every split must divide the range its ancestors leave for its property
// (left child: property > val, right child: property <= val), and no node may lie deeper than 2048. Depth first with
// the ranges of the current root-to-node path only; each frame restores the range its parent narrowed.
static void validate_tree(const std::vector<TreeNode>& nodes, uint32_t num_properties) {
  constexpr uint32_t kHeightLimit = 2048;
  std::vector<std::pair<int32_t, int32_t>> range(num_properties, {INT32_MIN, INT32_MAX});
  struct Frame {
    uint32_t node, depth, stage;  // stage 0: enter, 1: left child done, 2: both done
    int32_t restore_prop;         // < 0: nothing to restore (root)
    std::pair<int32_t, int32_t> restore;
  };
  std::vector<Frame> stack{Frame{0, 0, 0, -1, {0, 0}}};
  while (!stack.empty()) {
    Frame f = stack.back();
    stack.pop_back();
    if (f.depth > kHeightLimit) fail("MA tree too tall");
    const TreeNode& n = nodes[f.node];
    if (n.property < 0 || f.stage == 2) {
      if (f.restore_prop >= 0) range[size_t(f.restore_prop)] = f.restore;
      continue;
    }
    const size_t p = size_t(n.property);
    const auto [lo, hi] = range[p];
    if (lo > n.val || hi <= n.val) fail("MA tree split on an empty range");
    f.stage++;
    stack.push_back(f);
    stack.push_back(Frame{f.stage == 1 ? n.left : n.right, f.depth + 1, 0, n.property, range[p]});
    range[p] = f.stage == 1 ? std::pair<int32_t, int32_t>{n.val + 1, hi} : std::pair<int32_t, int32_t>{lo, n.val};
  }
}

ModularTree ModularTree::read(BitReader& br, size_t size_limit) {
  // tree.rs:284-358; contexts: 0 splitval, 1 property, 2 predictor, 3 offset, 4 mul_log, 5 mul_bits
  ModularTree t;
  EntropyCode tc = EntropyCode::decode(6, br, true);
  SymbolReader r(tc, br, 0);
  size_t to_decode = 1;
  uint32_t leaf_id = 0, max_property = 0;
  while (to_decode > 0) {
    if (t.nodes.size() > size_limit) fail("MA tree too large");
    to_decode--;
    uint32_t property = r.read_unsigned(br, 1);
    if (property > 0) {
      property -= 1;
      if (property > 255) fail("invalid MA tree property");
      max_property = std::max(max_property, property);
      int32_t splitval = r.read_signed(br, 0);
      uint32_t left = uint32_t(t.nodes.size() + to_decode + 1);
      t.nodes.push_back(TreeNode{int32_t(property), splitval, left, left + 1, 0});
      to_decode += 2;
      if (property == 15) t.uses_wp = true;
    } else {
      uint32_t predictor = r.read_unsigned(br, 2);
      if (predictor >= kNumPredictors) fail("invalid predictor");
      int32_t offset = r.read_signed(br, 3);
      uint32_t mul_log = r.read_unsigned(br, 4);
      if (mul_log >= 31) fail("MA tree multiplier too large");
      uint32_t mul_bits = r.read_unsigned(br, 5);
      uint64_t mul = (uint64_t(mul_bits) + 1) << mul_log;
      if (mul > 0xffffffffull) fail("MA tree multiplier too large");
      t.nodes.push_back(TreeNode{-1, offset, predictor, uint32_t(mul), leaf_id++});
      if (predictor == kWeighted) t.uses_wp = true;
    }
    br.check();
  }
  r.check_final_state(br);
  t.num_properties = max_property + 1;
  validate_tree(t.nodes, t.num_properties);
  t.code = EntropyCode::decode((t.nodes.size() + 1) / 2, br, true);
  return t;
}

// ---------------------------------------------------------------------------
// Channel decode (decode/channel.rs FullTree path; the reference's specialised
// trees are performance variants of the same semantics)
// ---------------------------------------------------------------------------

// Reader adapters for the specialised walks below: `read_clustered(cluster)` returns one whole symbol.
struct SlowReader {  // LZ77 streams: the member-state reader
  SymbolReader* r;
  BitReader* br;
  inline bool room(size_t) const { return false; }
  template <bool kUnchecked = false>
  inline uint32_t read_clustered(uint32_t cluster) { return r->read_clustered(*br, cluster); }
};

// Single-cluster ANS reader for big static-leaf channels. The per-symbol loop is bound by instruction issue, not
// by latency, so everything that is constant for one cluster is tabulated:
//  * the alias table of the cluster is expanded into a direct 4096-entry table
//    (symbol | offset << 8 | (freq - 1) << 20, 16 KB): no alias compare / selects (ans.rs:356-393);
//  * the hybrid-uint configuration becomes a per-token table {number of extra bits, value without them}
//    (hybrid_uint.rs:87-102): value = base | extra_bits << lsb;
//  * the bit window is re-loaded from a bit position every symbol (one unaligned 8-byte load gives >= 57 bits,
//    enough for the 16 refill bits + <= 31 extra bits), so consuming is one addition.
// Same arithmetic, entry by entry, as SymbolReader::read_token + HybridUint::read.
struct DirectReader {
  const uint8_t* data;
  size_t size;  // bytes
  size_t bitpos;
  uint32_t state;
  const uint32_t* tab;
  const uint64_t* tok_tab;  // base << 8 | nbits
  uint32_t lsb;
  // `nsym` more symbols of <= 47 bits can be read with unchecked 8-byte loads.
  inline bool room(size_t nsym) const { return (bitpos >> 3) + nsym * 6 + 16 <= size; }
  template <bool kUnchecked = false>
  __attribute__((always_inline)) inline uint32_t read_clustered(uint32_t /*cluster*/) {
    uint64_t w;
    const size_t byte = bitpos >> 3;
    if (kUnchecked || byte + 8 <= size) {
      memcpy(&w, data + byte, 8);
    } else {  // tail of the section: zero bits past the end (bit_reader.rs:109 reports the over-read afterwards)
      w = 0;
      for (size_t i = 0; i < 8 && byte + i < size; i++) w |= uint64_t(data[byte + i]) << (8 * i);
    }
    w >>= bitpos & 7;
    const uint32_t e = tab[state & 0xfff];
    const uint32_t next = (state >> kAnsLogSumProbs) * ((e >> 20) + 1) + ((e >> 8) & 0xfff);
    const uint32_t sh = uint32_t(next < (1u << 16)) << 4;
    state = (next << sh) | uint32_t(_bzhi_u64(w, sh));
    w >>= sh;
    const uint64_t t = tok_tab[e & 0xff];
    const uint32_t nbits = uint32_t(t & 0xff);
    bitpos += sh + nbits;
    return uint32_t(t >> 8) | (uint32_t(_bzhi_u64(w, nbits)) << lsb);
  }
};

static void build_direct_tables(const EntropyCode& code, uint32_t cluster, uint32_t* tab, uint64_t* tok_tab) {
  const uint32_t log_bucket = kAnsLogSumProbs - code.log_alpha_size;
  const AnsBucket* buckets = code.ans_buckets.data() + (size_t(cluster) << code.log_alpha_size);
  // per bucket: positions below the cut-off keep the bucket's own symbol, the rest go to its alias; inside each run
  // only the offset changes (by one per position), so both runs are plain counting loops.
  // build_alias_map guarantees 1 <= dist <= 4096 and offset < dist for every slot.
  const uint32_t bucket_size = 1u << log_bucket;
  for (uint32_t i = 0; i < (1u << code.log_alpha_size); i++) {
    const AnsBucket& b = buckets[i];
    uint32_t* t = tab + (size_t(i) << log_bucket);
    const uint32_t cutoff = std::min<uint32_t>(b.alias_cutoff, bucket_size);
    const uint32_t own = (i & 0xff) | (((uint32_t(b.dist) - 1) & 0xfff) << 20);
    for (uint32_t pos = 0; pos < cutoff; pos++) t[pos] = own | ((pos & 0xfff) << 8);
    const uint32_t alias_dist = uint32_t(b.dist) ^ uint32_t(b.alias_dist_xor);
    const uint32_t alias = uint32_t(b.alias_symbol) | (((alias_dist - 1) & 0xfff) << 20);
    for (uint32_t pos = cutoff; pos < bucket_size; pos++) t[pos] = alias | (((uint32_t(b.alias_offset) + pos) & 0xfff) << 8);
  }
  const HybridUint& u = code.uint_configs[cluster];
  for (uint32_t tok = 0; tok < 256; tok++) {
    if (tok < u.split_token()) {
      tok_tab[tok] = uint64_t(tok) << 8;
      continue;
    }
    const uint32_t bits_in_token = u.lsb + u.msb;
    const uint32_t nbits = (u.split_exponent - bits_in_token + ((tok - u.split_token()) >> bits_in_token)) & 31;
    const uint32_t low = tok & ((1u << u.lsb) - 1);
    const uint32_t hi = ((tok >> u.lsb) & ((1u << u.msb) - 1)) | (1u << u.msb);
    const uint32_t base = ((hi << nbits) << u.lsb) | low;
    tok_tab[tok] = uint64_t(base) << 8 | nbits;
  }
}

// Row segments shared by the single-stream and the paired static-leaf decoders. `kU`: refills without the
// end-of-data test (the caller checked room() for the segment).
struct GradState {
  __m128i left, topleft;
};

// Gradient predictor, y > 0, columns [x0, x1) of one row; same arithmetic as decode_static_leaf's gradient_row.
template <bool kU, class R>
__attribute__((always_inline)) inline void grad_segment(R& rd, uint32_t cluster, uint32_t uoff, uint32_t umul,
                                                        int32_t* row, const int32_t* top_row, size_t x0, size_t x1,
                                                        GradState& s) {
  for (size_t x = x0; x < x1; x++) {
    const __m128i top = _mm_cvtsi32_si128(top_row[x]);
    const uint32_t res = uint32_t(unpack_signed(rd.template read_clustered<kU>(cluster)));
    const __m128i add = _mm_cvtsi32_si128(int32_t(uoff + umul * res));
    const __m128i mn = _mm_min_epi32(s.left, top), mx = _mm_max_epi32(s.left, top);
    __m128i g = _mm_sub_epi32(_mm_add_epi32(s.left, top), s.topleft);
    g = _mm_blendv_epi8(g, mx, _mm_cmpgt_epi32(mn, s.topleft));
    g = _mm_blendv_epi8(g, mn, _mm_cmpgt_epi32(s.topleft, mx));
    s.left = _mm_add_epi32(g, add);
    row[x] = _mm_cvtsi128_si32(s.left);
    s.topleft = top;
  }
}

// Zero / West predictor (and Gradient on the first row): value = (left & keep) + offset + mul * residual.
template <bool kU, class R>
__attribute__((always_inline)) inline void west_segment(R& rd, uint32_t cluster, uint32_t uoff, uint32_t umul,
                                                        uint32_t keep, int32_t* row, size_t x0, size_t x1,
                                                        uint32_t& left) {
  for (size_t x = x0; x < x1; x++) {
    left = (left & keep) + uoff + umul * uint32_t(unpack_signed(rd.template read_clustered<kU>(cluster)));
    row[x] = int32_t(left);
  }
}

constexpr size_t kRowChunk = 512;  // room() is decided per chunk of columns, so long rows need no whole-row slack

// Only channel / stream id are tested by the tree: one leaf (predictor, offset, multiplier, cluster) for the
// whole channel, so the symbol chain is independent of the sample values.
template <class R>
static void decode_static_leaf(ModularChannel& ch, const TreeNode* nd, uint32_t cluster, R& io) {
  R rd = io;  // a true local (its address never escapes), so the reader state lives in registers
  const size_t w = ch.w, h = ch.h;
  const uint32_t pred = nd->left;
  const int64_t offset = nd->val, mul = nd->right;
  const uint32_t uoff = uint32_t(offset), umul = uint32_t(mul);
  auto next_signed = [&]() { return int64_t(unpack_signed(rd.read_clustered(cluster))); };
  for (size_t y = 0; y < h; y++) {
    int32_t* row = ch.row(uint32_t(y));
    const int32_t* top_row = y > 0 ? ch.row(uint32_t(y - 1)) : row;
    const int32_t* toptop_row = y > 1 ? ch.row(uint32_t(y - 2)) : top_row;
    if (pred == kZero || pred == kWest || (pred == kGradient && y == 0)) {
      // predictors that only look at the left neighbour (West; Gradient on the first row, where top = topleft =
      // left, predict.rs:64-103) or at nothing (Zero)
      const uint32_t keep = pred == kZero ? 0u : ~0u;
      uint32_t left = y > 0 ? uint32_t(top_row[0]) : 0u;  // x = 0: left = top_row[0], or 0 at the origin
      for (size_t c0 = 0; c0 < w; c0 += kRowChunk) {
        const size_t c1 = std::min(w, c0 + kRowChunk);
        if (rd.room(c1 - c0)) west_segment<true>(rd, cluster, uoff, umul, keep, row, c0, c1, left);
        else west_segment<false>(rd, cluster, uoff, umul, keep, row, c0, c1, left);
      }
    } else if (pred == kGradient) {
      // clamped_gradient on xmm scalars: its selects depend only on i32 comparisons of left / top / topleft, and
      // left + top - topleft is exact in wrapping i32 whenever it is the selected value (it then lies between left
      // and top): the serial left -> left chain has no (unpredictable) branches and stays out of the general-purpose
      // registers the symbol reader needs.
      GradState gs;
      gs.left = gs.topleft = _mm_cvtsi32_si128(top_row[0]);  // x = 0: left = topleft = top_row[0]
      for (size_t c0 = 0; c0 < w; c0 += kRowChunk) {
        const size_t c1 = std::min(w, c0 + kRowChunk);
        if (rd.room(c1 - c0)) grad_segment<true>(rd, cluster, uoff, umul, row, top_row, c0, c1, gs);
        else grad_segment<false>(rd, cluster, uoff, umul, row, top_row, c0, c1, gs);
      }
    } else {
      for (size_t x = 0; x < w; x++) {
        Neigh n = get_neigh(row, top_row, toptop_row, x, y, w);
        const int64_t guess = predict_one(pred, n, 0) + offset;
        row[x] = int32_t(guess + mul * next_signed());
      }
    }
  }
  io = rd;
}

// No weighted predictor, no reference-channel properties: evaluate only the properties the walk visits.
template <bool kWp, class R>
static void decode_lazy_props(ModularChannel& ch, size_t ci, size_t stream_id, const TreeNode* nodes,
                              const TreeNode* root, const uint8_t* cmap, const WeightedHeader& wph, R& io) {
  R rd = io;
  const size_t w = ch.w, h = ch.h;
  WpState wp(wph, kWp ? w : 0);
  for (size_t y = 0; y < h; y++) {
    int32_t* row = ch.row(uint32_t(y));
    const int32_t* top_row = y > 0 ? ch.row(uint32_t(y - 1)) : row;
    const int32_t* toptop_row = y > 1 ? ch.row(uint32_t(y - 2)) : top_row;
    int32_t prev_p9 = 0;
    for (size_t x = 0; x < w; x++) {
      const Neigh n = get_neigh(row, top_row, toptop_row, x, y, w);
      const int32_t p9 = wsub(wadd(n.left, n.top), n.topleft);
      int64_t wp_pred = 0;
      int32_t wp_prop = 0;
      if (kWp) wp_predict(wp, x, y, n.top, n.left, n.topright, n.topleft, n.toptop, wp_pred, wp_prop);
      const TreeNode* nd = root;
      while (nd->property >= 0) {
        int32_t v;
        switch (nd->property) {
          case 0: v = int32_t(ci); break;
          case 1: v = int32_t(stream_id); break;
          case 2: v = int32_t(y); break;
          case 3: v = int32_t(x); break;
          case 4: v = wabs(n.top); break;
          case 5: v = wabs(n.left); break;
          case 6: v = n.top; break;
          case 7: v = n.left; break;
          case 8: v = wsub(n.left, prev_p9); break;
          case 9: v = p9; break;
          case 10: v = wsub(n.left, n.topleft); break;
          case 11: v = wsub(n.topleft, n.top); break;
          case 12: v = wsub(n.top, n.topright); break;
          case 13: v = wsub(n.top, n.toptop); break;
          case 14: v = wsub(n.left, n.leftleft); break;
          default: v = wp_prop; break;  // property 15; 0 without the weighted predictor
        }
        nd = nodes + (v > nd->val ? nd->left : nd->right);
      }
      prev_p9 = p9;
      const int64_t guess = predict_one(nd->left, n, wp_pred) + int64_t(nd->val);
      const int32_t val =
          int32_t(guess + int64_t(nd->right) * int64_t(unpack_signed(rd.read_clustered(cmap[nd->ctx]))));
      if (kWp) wp_update(wp, val, x, y);
      row[x] = val;
    }
  }
  io = rd;
}

// Subtrees whose decision nodes all test the same property p (libjxl's LF trees: only the weighted-predictor
// property 15) become a table from clamp(value, -1024, 1023) to the leaf, like make_lut in
// decode/specialized_trees.rs:197-249: one load instead of a chain of data-dependent branches. Returns false if a
// split value lies outside the range the clamp preserves (or outside the range of its own subtree).
constexpr int32_t kLutMin = -1024, kLutMax = 1023;
static bool make_prop_lut(const TreeNode* nodes, const TreeNode* root, std::vector<uint32_t>& lut) {
  struct Item {
    int32_t lo, hi;  // values lo .. hi - 1 reach `node`
    const TreeNode* node;
  };
  lut.assign(size_t(kLutMax - kLutMin + 1), 0);
  std::vector<Item> stack{Item{kLutMin, kLutMax + 1, root}};
  while (!stack.empty()) {
    const Item it = stack.back();
    stack.pop_back();
    if (it.node->property >= 0) {
      const int64_t first_left = int64_t(it.node->val) + 1;  // v > val goes left
      if (first_left >= it.hi || first_left <= it.lo) return false;
      stack.push_back(Item{int32_t(first_left), it.hi, nodes + it.node->left});
      stack.push_back(Item{it.lo, int32_t(first_left), nodes + it.node->right});
    } else {
      for (int32_t v = it.lo; v < it.hi; v++) lut[size_t(v - kLutMin)] = uint32_t(it.node - nodes);
    }
  }
  return true;
}

// kProp15: the table is over the weighted-predictor property (the libjxl LF case), which removes the property switch.
template <bool kWp, bool kProp15, class R>
static void decode_prop_lut(ModularChannel& ch, const TreeNode* nodes, int prop, const uint32_t* lut,
                            const uint8_t* cmap, const WeightedHeader& wph, R& io) {
  R rd = io;
  const size_t w = ch.w, h = ch.h;
  WpState wp(wph, kWp ? w : 0);
  for (size_t y = 0; y < h; y++) {
    int32_t* row = ch.row(uint32_t(y));
    const int32_t* top_row = y > 0 ? ch.row(uint32_t(y - 1)) : row;
    const int32_t* toptop_row = y > 1 ? ch.row(uint32_t(y - 2)) : top_row;
    int32_t prev_p9 = 0;
    const size_t interior_end = (y >= 2 && w > 4) ? w - 2 : 0;  // 2 <= x < w - 2: every neighbour exists
    // one loop body (a single copy of the predictor + reader code keeps its state in registers)
    for (size_t x = 0; x < w; x++) {
      const Neigh n = (x >= 2 && x < interior_end) ? get_neigh_interior(row, top_row, toptop_row, x)
                                                   : get_neigh(row, top_row, toptop_row, x, y, w);
      int64_t wp_pred = 0;
      int32_t wp_prop = 0;
      if (kWp) wp_predict(wp, x, y, n.top, n.left, n.topright, n.topleft, n.toptop, wp_pred, wp_prop);
      int32_t v;
      if (kProp15) {
        v = wp_prop;
      } else {
        const int32_t p9 = wsub(wadd(n.left, n.top), n.topleft);
        switch (prop) {  // loop invariant
          case 2: v = int32_t(y); break;
          case 3: v = int32_t(x); break;
          case 4: v = wabs(n.top); break;
          case 5: v = wabs(n.left); break;
          case 6: v = n.top; break;
          case 7: v = n.left; break;
          case 8: v = wsub(n.left, prev_p9); break;
          case 9: v = p9; break;
          case 10: v = wsub(n.left, n.topleft); break;
          case 11: v = wsub(n.topleft, n.top); break;
          case 12: v = wsub(n.top, n.topright); break;
          case 13: v = wsub(n.top, n.toptop); break;
          case 14: v = wsub(n.left, n.leftleft); break;
          default: v = wp_prop; break;
        }
        prev_p9 = p9;
      }
      const int32_t clamped = v < kLutMin ? kLutMin : (v > kLutMax ? kLutMax : v);
      const TreeNode* nd = nodes + lut[size_t(clamped - kLutMin)];
      const int64_t guess =
          (kWp && nd->left == kWeighted ? wp_pred : predict_one(nd->left, n, wp_pred)) + int64_t(nd->val);
      const int32_t val =
          int32_t(guess + int64_t(nd->right) * int64_t(unpack_signed(rd.read_clustered(cmap[nd->ctx]))));
      if (kWp) wp_update(wp, val, x, y);
      row[x] = val;
    }
  }
  io = rd;
}

// Runs `f(reader)` with the register-resident reader when the code allows it (no LZ77), else with the member one.
template <class F>
static void with_reader(SymbolReader& reader, BitReader& br, F&& f) {
  if (!reader.can_localise()) {
    SlowReader s{&reader, &br};
    f(s);
  } else if (reader.uses_prefix()) {
    auto l = reader.local<true>(br);
    f(l);
    reader.commit(l, br);
  } else {
    auto l = reader.local<false>(br);
    f(l);
    reader.commit(l, br);
  }
}

static std::atomic<bool> g_force_generic_walk{false};
void set_force_generic_walk(bool on) { g_force_generic_walk.store(on); }

// Where the per-pixel walk of one channel starts and what it needs.
struct ChannelPlan {
  const TreeNode* root;
  uint32_t used_mask;  // properties 0..15 tested below root
  bool wide_props, sub_wp;
};
static ChannelPlan plan_channel(const ModularTree& tree, size_t ci, size_t stream_id) {
  const TreeNode* nodes = tree.nodes.data();
  // Static prefix: nodes that split on the channel index / stream id have one outcome for the whole channel
  // (libjxl's global trees start with such a chain), so the walk can start below them.
  const TreeNode* root = nodes;
  while (root->property == 0 || root->property == 1) {
    const int32_t v = root->property == 0 ? int32_t(ci) : int32_t(stream_id);
    root = nodes + (v > root->val ? root->left : root->right);
  }
  // Which properties and predictors does the subtree under `root` use?
  ChannelPlan p{root, 0, false, false};
  std::vector<const TreeNode*> stack{root};
  while (!stack.empty()) {
    const TreeNode* nd = stack.back();
    stack.pop_back();
    if (nd->property < 0) {
      if (nd->left == kWeighted) p.sub_wp = true;
      continue;
    }
    if (nd->property < 16) p.used_mask |= 1u << nd->property;
    else p.wide_props = true;
    if (nd->property == 15) p.sub_wp = true;
    stack.push_back(nodes + nd->left);
    stack.push_back(nodes + nd->right);
  }
  return p;
}

// A channel the direct-table reader takes: one leaf, one ANS cluster, big enough to pay for the table.
static bool direct_eligible(const ChannelPlan& plan, const SymbolReader& reader, const ModularChannel& ch) {
  return !g_force_generic_walk.load(std::memory_order_relaxed) && plan.root->property < 0 && !plan.sub_wp &&
         reader.can_localise() && !reader.uses_prefix() && size_t(ch.w) * ch.h >= 8192;
}

static void decode_channel(std::vector<ModularChannel*>& chans, size_t ci, size_t stream_id, const GroupHeader& header,
                           const ModularTree& tree, SymbolReader& reader, BitReader& br) {
  ModularChannel& ch = *chans[ci];
  const size_t w = ch.w, h = ch.h;
  size_t num_ref_props = tree.num_properties > 16 ? ((tree.num_properties - 16 + 3) / 4) * 4 : 0;
  std::vector<int32_t> refs(num_ref_props * w, 0);
  int32_t props[16 + 256] = {0};
  props[0] = int32_t(ci);
  props[1] = int32_t(stream_id);
  const bool use_wp = tree.uses_wp;
  const TreeNode* nodes = tree.nodes.data();
  // ---- specialised walks (same semantics as the generic loop below; the reference keeps a family of these in
  // decode/specialized_trees.rs).
  const ChannelPlan plan = plan_channel(tree, ci, stream_id);
  const TreeNode* root = plan.root;
  const uint32_t used_mask = plan.used_mask;
  const bool wide_props = plan.wide_props, sub_wp = plan.sub_wp;
  const bool specialise = !g_force_generic_walk.load(std::memory_order_relaxed);
  if (specialise && root->property < 0 && !sub_wp) {
    const TreeNode* nd = root;
    const uint32_t cluster = tree.code.context_map[nd->ctx];  // one leaf -> one cluster for the whole channel
    if (direct_eligible(plan, reader, ch)) {
      // big channel, one ANS cluster: direct table (its 4096-entry build is < 1 % of the channel)
      uint32_t tab[4096];
      uint64_t tok_tab[256];
      build_direct_tables(tree.code, cluster, tab, tok_tab);
      DirectReader d{br.data(), br.size_bytes(), br.bit_pos(), reader.ans_state(), tab, tok_tab,
                     tree.code.uint_configs[cluster].lsb};
      decode_static_leaf(ch, nd, cluster, d);
      reader.set_ans_state(d.state);
      br.seek_bits(d.bitpos);
    } else {
      with_reader(reader, br, [&](auto& rd) { decode_static_leaf(ch, nd, cluster, rd); });
    }
    br.check();
    return;
  }
  if (specialise && !wide_props) {
    // Properties 0..15 evaluated on demand; the weighted predictor runs only if the subtree uses it (as property
    // 15 or as a leaf predictor).
    const uint8_t* cmap = tree.code.context_map.data();
    // one dynamic property only -> table walk
    int single_prop = -1;
    std::vector<uint32_t> lut;
    const uint32_t dyn_mask = used_mask & ~3u;
    if (w * h >= 1024 && dyn_mask != 0 && (dyn_mask & (dyn_mask - 1)) == 0 && (used_mask & 3u) == 0) {
      single_prop = __builtin_ctz(dyn_mask);
      if (!make_prop_lut(nodes, root, lut)) single_prop = -1;
    }
    with_reader(reader, br, [&](auto& rd) {
      if (single_prop == 15) {
        decode_prop_lut<true, true>(ch, nodes, single_prop, lut.data(), cmap, header.wp, rd);
      } else if (single_prop >= 0) {
        if (sub_wp) decode_prop_lut<true, false>(ch, nodes, single_prop, lut.data(), cmap, header.wp, rd);
        else decode_prop_lut<false, false>(ch, nodes, single_prop, lut.data(), cmap, header.wp, rd);
      } else if (sub_wp) {
        decode_lazy_props<true>(ch, ci, stream_id, nodes, root, cmap, header.wp, rd);
      } else {
        decode_lazy_props<false>(ch, ci, stream_id, nodes, root, cmap, header.wp, rd);
      }
    });
    br.check();
    return;
  }
  WpState wp(header.wp, use_wp ? w : 0);
  for (size_t y = 0; y < h; y++) {
    int32_t* row = ch.row(uint32_t(y));
    const int32_t* top_row = y > 0 ? ch.row(uint32_t(y - 1)) : row;
    const int32_t* toptop_row = y > 1 ? ch.row(uint32_t(y - 2)) : top_row;
    if (num_ref_props) {  // decode/common.rs:42-83
      std::fill(refs.begin(), refs.end(), 0);
      size_t offset = 0;
      for (size_t i = 0; i < ci && offset < num_ref_props; i++) {
        const ModularChannel& rc = *chans[ci - i - 1];
        if (rc.w != ch.w || rc.h != ch.h || rc.hshift != ch.hshift || rc.vshift != ch.vshift) continue;
        const int32_t* rrow = rc.row(uint32_t(y));
        const int32_t* rprev = rc.row(uint32_t(y > 0 ? y - 1 : 0));
        for (size_t x = 0; x < w; x++) {
          int32_t* rp = &refs[x * num_ref_props + offset];
          int32_t v = rrow[x];
          rp[0] = wabs(v);
          rp[1] = v;
          int32_t vleft = x > 0 ? rrow[x - 1] : 0;
          int32_t vtop = y > 0 ? rprev[x] : vleft;
          int32_t vtopleft = (x > 0 && y > 0) ? rprev[x - 1] : vleft;
          int64_t vpred = clamped_gradient(vleft, vtop, vtopleft);
          int64_t d = int64_t(v) - vpred;
          rp[2] = int32_t(d < 0 ? -d : d);
          rp[3] = int32_t(d);
        }
        offset += 4;
      }
    }
    props[9] = 0;
    props[2] = int32_t(y);
    for (size_t x = 0; x < w; x++) {
      Neigh n = get_neigh(row, top_row, toptop_row, x, y, w);
      // tree.rs:189-240
      props[3] = int32_t(x);
      props[4] = wabs(n.top);
      props[5] = wabs(n.left);
      props[6] = n.top;
      props[7] = n.left;
      props[8] = wsub(n.left, props[9]);
      props[9] = wsub(wadd(n.left, n.top), n.topleft);
      props[10] = wsub(n.left, n.topleft);
      props[11] = wsub(n.topleft, n.top);
      props[12] = wsub(n.top, n.topright);
      props[13] = wsub(n.top, n.toptop);
      props[14] = wsub(n.left, n.leftleft);
      int64_t wp_pred = 0;
      int32_t wp_prop = 0;
      if (use_wp) wp.predict(x, y, n.top, n.left, n.topright, n.topleft, n.toptop, wp_pred, wp_prop);
      props[15] = wp_prop;
      for (size_t i = 0; i < num_ref_props; i++) props[16 + i] = refs[x * num_ref_props + i];
      const TreeNode* nd = nodes;
      while (nd->property >= 0) nd = nodes + (props[nd->property] > nd->val ? nd->left : nd->right);
      int64_t guess = predict_one(nd->left, n, wp_pred) + int64_t(nd->val);
      int32_t dec = reader.read_signed(br, nd->ctx);
      int32_t val = int32_t(guess + int64_t(nd->right) * int64_t(dec));  // decode/common.rs:85
      if (use_wp) wp.update(val, x, y);
      row[x] = val;
    }
  }
  br.check();
}

// ---------------------------------------------------------------------------
// Two static-leaf channels of two independent sub-bitstreams in lockstep
// ---------------------------------------------------------------------------

namespace {

struct LeafChannel {  // one static-leaf channel being decoded by decode_static_leaf_pair
  ModularChannel* ch;
  uint32_t pred, uoff, umul;
  // row kind: 0 = west-like (Zero, West, Gradient on row 0), 1 = Gradient with a row above
  int kind(size_t y) const { return (pred == kGradient && y > 0) ? 1 : 0; }
  uint32_t keep() const { return pred == kZero ? 0u : ~0u; }
};

}  // namespace

// Both channels are direct-table channels with predictor Zero, West or Gradient. Rows advance in lockstep; where both
// rows are of the same kind and far enough from the end of their sections for unchecked refills, the two symbol
// chains share one loop body (the second stream costs ~6 instead of ~19 cycles per symbol); everything else — row
// tails, rows of different kinds, the last rows of a section — takes the single-stream segments.
__attribute__((noinline)) static void decode_static_leaf_pair(const LeafChannel& A, DirectReader& ioA, const LeafChannel& B,
                                                            DirectReader& ioB) {
  DirectReader ra = ioA, rb = ioB;  // true locals: both readers stay in registers
  const size_t wA = A.ch->w, hA = A.ch->h, wB = B.ch->w, hB = B.ch->h;
  auto single_row = [&](const LeafChannel& L, DirectReader& rd, size_t y) __attribute__((always_inline)) {
    const size_t w = L.ch->w;
    int32_t* row = L.ch->row(uint32_t(y));
    const int32_t* top_row = y > 0 ? L.ch->row(uint32_t(y - 1)) : row;
    GradState s;
    s.left = s.topleft = _mm_cvtsi32_si128(top_row[0]);
    uint32_t left = y > 0 ? uint32_t(top_row[0]) : 0u;
    for (size_t c0 = 0; c0 < w; c0 += kRowChunk) {
      const size_t c1 = std::min(w, c0 + kRowChunk);
      const bool fast = rd.room(c1 - c0);
      if (L.kind(y) == 1) {
        if (fast) grad_segment<true>(rd, 0, L.uoff, L.umul, row, top_row, c0, c1, s);
        else grad_segment<false>(rd, 0, L.uoff, L.umul, row, top_row, c0, c1, s);
      } else {
        if (fast) west_segment<true>(rd, 0, L.uoff, L.umul, L.keep(), row, c0, c1, left);
        else west_segment<false>(rd, 0, L.uoff, L.umul, L.keep(), row, c0, c1, left);
      }
    }
  };
  // Rows are walked in chunks of kChunk columns: "enough input left for unchecked refills" is decided per chunk, so a
  // very long row (the 2 x count channel of the HF metadata) does not need its whole length of slack.
  constexpr size_t kChunk = kRowChunk;
  const size_t hmax = std::max(hA, hB);
  for (size_t y = 0; y < hmax; y++) {
    const bool inA = y < hA, inB = y < hB;
    if (inA && inB && A.kind(y) == B.kind(y)) {
      int32_t* rowA = A.ch->row(uint32_t(y));
      int32_t* rowB = B.ch->row(uint32_t(y));
      const int32_t* topA = y > 0 ? A.ch->row(uint32_t(y - 1)) : rowA;
      const int32_t* topB = y > 0 ? B.ch->row(uint32_t(y - 1)) : rowB;
      const size_t n = std::min(wA, wB);
      const bool grad = A.kind(y) == 1;
      GradState sa, sb;
      sa.left = sa.topleft = _mm_cvtsi32_si128(topA[0]);
      sb.left = sb.topleft = _mm_cvtsi32_si128(topB[0]);
      uint32_t la = y > 0 ? uint32_t(topA[0]) : 0u, lb = y > 0 ? uint32_t(topB[0]) : 0u;
      const uint32_t ka = A.keep(), kb = B.keep();
      // columns [x0, x1) of stream L alone
      auto alone = [&](const LeafChannel& L, DirectReader& rd, int32_t* row, const int32_t* top, size_t x0, size_t x1,
                       GradState& gs, uint32_t& left, uint32_t keep) __attribute__((always_inline)) {
        for (size_t c0 = x0; c0 < x1; c0 += kChunk) {
          const size_t c1 = std::min(x1, c0 + kChunk);
          const bool fast = rd.room(c1 - c0);
          if (grad) {
            if (fast) grad_segment<true>(rd, 0, L.uoff, L.umul, row, top, c0, c1, gs);
            else grad_segment<false>(rd, 0, L.uoff, L.umul, row, top, c0, c1, gs);
          } else {
            if (fast) west_segment<true>(rd, 0, L.uoff, L.umul, keep, row, c0, c1, left);
            else west_segment<false>(rd, 0, L.uoff, L.umul, keep, row, c0, c1, left);
          }
        }
      };
      for (size_t c0 = 0; c0 < n; c0 += kChunk) {
        const size_t c1 = std::min(n, c0 + kChunk);
        if (ra.room(c1 - c0) && rb.room(c1 - c0)) {
          if (grad) {
            for (size_t x = c0; x < c1; x++) {  // one body, two independent chains
              grad_segment<true>(ra, 0, A.uoff, A.umul, rowA, topA, x, x + 1, sa);
              grad_segment<true>(rb, 0, B.uoff, B.umul, rowB, topB, x, x + 1, sb);
            }
          } else {
            for (size_t x = c0; x < c1; x++) {
              west_segment<true>(ra, 0, A.uoff, A.umul, ka, rowA, x, x + 1, la);
              west_segment<true>(rb, 0, B.uoff, B.umul, kb, rowB, x, x + 1, lb);
            }
          }
        } else {
          alone(A, ra, rowA, topA, c0, c1, sa, la, ka);
          alone(B, rb, rowB, topB, c0, c1, sb, lb, kb);
        }
      }
      alone(A, ra, rowA, topA, n, wA, sa, la, ka);
      alone(B, rb, rowB, topB, n, wB, sb, lb, kb);
    } else {
      if (inA) single_row(A, ra, y);
      if (inB) single_row(B, rb, y);
    }
  }
  ioA = ra;
  ioB = rb;
}

SubStream::~SubStream() { delete reader; }

void substream_begin(SubStream& s, std::vector<ModularChannel>& channels, size_t stream_id,
                     const ModularTree* global_tree, BitReader& br) {
  s.channels = &channels;
  s.stream_id = stream_id;
  s.br = &br;
  s.empty = true;
  for (auto& c : channels)
    if (c.w && c.h) s.empty = false;
  if (s.empty) return;
  s.header = GroupHeader::read(br);
  uint32_t nb_meta = 0;
  meta_apply_transforms(channels, nb_meta, s.header);
  s.tree = global_tree;
  if (!s.header.use_global_tree) {
    size_t samples = 0;
    for (auto& c : channels) samples += size_t(c.w) * c.h;
    s.local = ModularTree::read(br, std::min<size_t>(1024 + samples, 1u << 20));
    s.tree = &s.local;
  } else if (!global_tree) {
    fail("no global MA tree");
  }
  for (auto& c : channels) s.ptrs.push_back(&c);
  size_t image_width = 0;
  for (auto* c : s.ptrs) image_width = std::max<size_t>(image_width, c->w);
  s.reader = new SymbolReader(s.tree->code, br, image_width);
  s.next = 0;
}

// Skips empty channels; false when none is left.
static bool substream_has_channel(SubStream& s) {
  if (s.empty) return false;
  while (s.next < s.ptrs.size() && (s.ptrs[s.next]->w == 0 || s.ptrs[s.next]->h == 0)) s.next++;
  return s.next < s.ptrs.size();
}

static void substream_decode_next(SubStream& s) {
  decode_channel(s.ptrs, s.next, s.stream_id, s.header, *s.tree, *s.reader, *s.br);
  s.next++;
}

void substream_finish(SubStream& s) {
  if (s.empty) return;
  while (substream_has_channel(s)) substream_decode_next(s);
  s.reader->check_final_state(*s.br);
  undo_transforms(*s.channels, s.header, 8);
}

void decode_substreams_paired(SubStream& a, SubStream& b) {
  for (;;) {
    const bool ha = substream_has_channel(a), hb = substream_has_channel(b);
    if (!ha || !hb) break;
    ModularChannel& ca = *a.ptrs[a.next];
    ModularChannel& cb = *b.ptrs[b.next];
    const ChannelPlan pa = plan_channel(*a.tree, a.next, a.stream_id), pb = plan_channel(*b.tree, b.next, b.stream_id);
    auto pairable = [](const ChannelPlan& p, const SymbolReader& r, const ModularChannel& c) {
      return direct_eligible(p, r, c) && (p.root->left == kZero || p.root->left == kWest || p.root->left == kGradient);
    };
    const bool ea = pairable(pa, *a.reader, ca), eb = pairable(pb, *b.reader, cb);
    if (ea && eb) {
      uint32_t tab_a[4096], tab_b[4096];
      uint64_t tok_a[256], tok_b[256];
      const uint32_t cla = a.tree->code.context_map[pa.root->ctx], clb = b.tree->code.context_map[pb.root->ctx];
      build_direct_tables(a.tree->code, cla, tab_a, tok_a);
      build_direct_tables(b.tree->code, clb, tab_b, tok_b);
      DirectReader da{a.br->data(), a.br->size_bytes(), a.br->bit_pos(), a.reader->ans_state(), tab_a, tok_a,
                      a.tree->code.uint_configs[cla].lsb};
      DirectReader db{b.br->data(), b.br->size_bytes(), b.br->bit_pos(), b.reader->ans_state(), tab_b, tok_b,
                      b.tree->code.uint_configs[clb].lsb};
      const LeafChannel la{&ca, pa.root->left, uint32_t(pa.root->val), pa.root->right};
      const LeafChannel lb{&cb, pb.root->left, uint32_t(pb.root->val), pb.root->right};
      decode_static_leaf_pair(la, da, lb, db);
      a.reader->set_ans_state(da.state);
      a.br->seek_bits(da.bitpos);
      b.reader->set_ans_state(db.state);
      b.br->seek_bits(db.bitpos);
      a.br->check();
      b.br->check();
      a.next++;
      b.next++;
    } else {
      // not a pair: let the stream(s) with an ordinary channel catch up, then look again
      if (!ea) substream_decode_next(a);
      if (!eb) substream_decode_next(b);
    }
  }
  substream_finish(a);
  substream_finish(b);
}

void decode_modular_channels(std::vector<ModularChannel*>& channels, size_t stream_id, const GroupHeader& header,
                             const ModularTree& tree, BitReader& br) {
  size_t image_width = 0;
  for (auto* c : channels) image_width = std::max<size_t>(image_width, c->w);
  SymbolReader reader(tree.code, br, image_width);
  for (size_t i = 0; i < channels.size(); i++) {
    if (channels[i]->w == 0 || channels[i]->h == 0) continue;
    decode_channel(channels, i, stream_id, header, tree, reader, br);
  }
  reader.check_final_state(br);
}

// ---------------------------------------------------------------------------
// Transforms
// ---------------------------------------------------------------------------

// squeeze.rs:39-105
static std::vector<SqueezeParams> default_squeeze(const std::vector<ModularChannel>& ch, uint32_t nb_meta) {
  std::vector<SqueezeParams> params;
  size_t first = nb_meta;
  uint32_t w = ch[first].w, h = ch[first].h;
  size_t nc = ch.size() - first;
  if (nc > 2 && ch[first + 1].w == w && ch[first + 1].h == h) {
    SqueezeParams sp{true, false, uint32_t(first + 1), 2};
    if (w > 1) params.push_back(sp);
    if (h > 1) {
      sp.horizontal = false;
      params.push_back(sp);
    }
  }
  const uint32_t kMax = 8;
  SqueezeParams sp{false, true, uint32_t(first), uint32_t(nc)};
  if (w <= h && h > kMax) {
    sp.horizontal = false;
    params.push_back(sp);
    h = (h + 1) / 2;
  }
  while (w > kMax || h > kMax) {
    if (w > kMax) {
      sp.horizontal = true;
      params.push_back(sp);
      w = (w + 1) / 2;
    }
    if (h > kMax) {
      sp.horizontal = false;
      params.push_back(sp);
      h = (h + 1) / 2;
    }
  }
  return params;
}

void meta_apply_transforms(std::vector<ModularChannel>& ch, uint32_t& nb_meta, GroupHeader& header, bool allocate) {
  auto make = [&](uint32_t w, uint32_t h, int32_t hs, int32_t vs) {
    if (allocate) return ModularChannel(w, h, hs, vs);
    ModularChannel c;
    c.w = w;
    c.h = h;
    c.hshift = hs;
    c.vshift = vs;
    return c;
  };
  for (auto& t : header.transforms) {
    if (t.id == 0) {  // RCT: channel list unchanged (meta_apply.rs RCT arm checks equal sizes)
      if (t.begin_channel + 3 > ch.size()) fail("RCT channel range");
      for (int i = 1; i < 3; i++)
        if (ch[t.begin_channel + i].w != ch[t.begin_channel].w || ch[t.begin_channel + i].h != ch[t.begin_channel].h)
          fail("RCT on channels of different size");
    } else if (t.id == 1) {  // palette, meta_apply.rs:181-230
      size_t b = t.begin_channel, n = t.num_channels;
      if (b + n > ch.size()) fail("palette channel range");
      for (size_t i = 1; i < n; i++)
        if (ch[b + i].w != ch[b].w || ch[b + i].h != ch[b].h) fail("palette on channels of different size");
      if (b < nb_meta) {
        if (b + n > nb_meta) fail("palette mixes meta and non-meta channels");
        nb_meta += 2 - uint32_t(n);
      } else {
        nb_meta += 1;
      }
      ch.erase(ch.begin() + b + 1, ch.begin() + b + n);
      ch.insert(ch.begin(), make(t.num_colors + t.num_deltas, uint32_t(n), -1, -1));
    } else {  // squeeze, meta_apply.rs squeeze arm / squeeze.rs:17-37
      if (t.squeezes.empty()) t.squeezes = default_squeeze(ch, nb_meta);
      for (const auto& s : t.squeezes) {
        size_t b = s.begin_channel, e = b + s.num_channels;
        if (e > ch.size() || s.num_channels == 0) fail("squeeze channel range");
        bool meta_b = b < nb_meta, meta_e = (e - 1) < nb_meta;
        if (meta_b != meta_e) fail("squeeze mixes meta and non-meta channels");
        if (meta_b && !s.in_place) fail("meta squeeze must be in place");
        if (meta_b) nb_meta += s.num_channels;
        size_t offset = s.in_place ? e : ch.size();
        for (size_t c = b; c < e; c++) {
          ModularChannel& in = ch[c];
          ModularChannel res;
          // meta_apply.rs:111-113: a channel shifted by more than 30 in either direction takes no further squeeze
          if (in.hshift > 30 || in.vshift > 30) fail("too many squeezes");
          if (s.horizontal) {
            uint32_t w = in.w;
            in.w = (w + 1) / 2;
            if (in.hshift >= 0) in.hshift++;
            res = make(w - in.w, in.h, in.hshift, in.vshift);
          } else {
            uint32_t h = in.h;
            in.h = (h + 1) / 2;
            if (in.vshift >= 0) in.vshift++;
            res = make(in.w, h - in.h, in.hshift, in.vshift);
          }
          if (allocate) in.data.assign(size_t(in.w) * in.h, 0);
          else in.data.clear();
          ch.insert(ch.begin() + offset + (c - b), std::move(res));
        }
      }
    }
  }
}

// squeeze.rs:144-170 (scalar definition)
static inline int64_t smooth_tendency(int64_t b, int64_t a, int64_t n) {
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

static void inv_hsqueeze(const ModularChannel& avg, const ModularChannel& res, ModularChannel& out) {
  out = ModularChannel(avg.w + res.w, avg.h, avg.hshift > 0 ? avg.hshift - 1 : avg.hshift, avg.vshift);
  for (uint32_t y = 0; y < out.h; y++) {
    const int32_t* a = avg.row(y);
    const int32_t* r = res.w ? res.row(y) : nullptr;
    int32_t* o = out.row(y);
    for (uint32_t x = 0; x < res.w; x++) {
      int64_t av = a[x];
      int64_t next_avg = x + 1 < avg.w ? a[x + 1] : av;
      int64_t left = x ? o[2 * x - 1] : av;
      int64_t diff = int64_t(r[x]) + smooth_tendency(left, av, next_avg);
      int64_t A = av + diff / 2;
      o[2 * x] = int32_t(A);
      o[2 * x + 1] = int32_t(A - diff);
    }
    if (out.w & 1) o[out.w - 1] = a[avg.w - 1];
  }
}

static void inv_vsqueeze(const ModularChannel& avg, const ModularChannel& res, ModularChannel& out) {
  out = ModularChannel(avg.w, avg.h + res.h, avg.hshift, avg.vshift > 0 ? avg.vshift - 1 : avg.vshift);
  for (uint32_t y = 0; y < res.h; y++) {
    const int32_t* a = avg.row(y);
    const int32_t* an = y + 1 < avg.h ? avg.row(y + 1) : a;
    const int32_t* r = res.row(y);
    int32_t* o0 = out.row(2 * y);
    int32_t* o1 = out.row(2 * y + 1);
    const int32_t* op = y ? out.row(2 * y - 1) : a;
    for (uint32_t x = 0; x < out.w; x++) {
      int64_t av = a[x];
      int64_t diff = int64_t(r[x]) + smooth_tendency(op[x], av, an[x]);
      int64_t A = av + diff / 2;
      o0[x] = int32_t(A);
      o1[x] = int32_t(A - diff);
    }
  }
  if (out.h & 1) std::copy(avg.row(avg.h - 1), avg.row(avg.h - 1) + avg.w, out.row(out.h - 1));
}

// rct.rs:9-40 + do_rct_step permutation
static void inv_rct(std::vector<ModularChannel>& ch, size_t b, uint32_t rct_type) {
  uint32_t perm = rct_type / 7, op = rct_type % 7;
  ModularChannel &c0 = ch[b], &c1 = ch[b + 1], &c2 = ch[b + 2];
  size_t n = c0.data.size();
  int32_t *p0 = c0.data.data(), *p1 = c1.data.data(), *p2 = c2.data.data();
  for (size_t i = 0; i < n; i++) {
    int32_t v0 = p0[i], v1 = p1[i], v2 = p2[i];
    switch (op) {
      case 1: v2 = wadd(v2, v0); break;
      case 2: v1 = wadd(v1, v0); break;
      case 3: v1 = wadd(v1, v0); v2 = wadd(v2, v0); break;
      case 4: v1 = wadd(v1, wadd(v0, v2) >> 1); break;
      case 5: v2 = wadd(v0, v2); v1 = wadd(v1, wadd(v0, v2) >> 1); break;
      case 6: {
        int32_t y = v0, co = v1, cg = v2;
        y = wsub(y, cg >> 1);
        int32_t g = wadd(cg, y);
        y = wsub(y, co >> 1);
        int32_t r = wadd(y, co);
        v0 = r; v1 = g; v2 = y;
        break;
      }
      default: break;
    }
    p0[i] = v0; p1[i] = v1; p2[i] = v2;
  }
  // out[perm % 3] = first, out[(perm + 1 + perm / 3) % 3] = second, out[(perm + 2 - perm / 3) % 3] = third
  std::vector<int32_t> d[3] = {std::move(c0.data), std::move(c1.data), std::move(c2.data)};
  ch[b + perm % 3].data = std::move(d[0]);
  ch[b + (perm + 1 + perm / 3) % 3].data = std::move(d[1]);
  ch[b + (perm + 2 - perm / 3) % 3].data = std::move(d[2]);
}

// palette.rs:17-138
static int32_t palette_value(const ModularChannel& pal, int64_t index, size_t c, size_t palette_size,
                             size_t bit_depth) {
  static const int16_t kDelta[72][3] = {
      {0, 0, 0},       {4, 4, 4},       {11, 0, 0},      {0, 0, -13},     {0, -12, 0},     {-10, -10, -10},
      {-18, -18, -18}, {-27, -27, -27}, {-18, -18, 0},   {0, 0, -32},     {-32, 0, 0},     {-37, -37, -37},
      {0, -32, -32},   {24, 24, 45},    {50, 50, 50},    {-45, -24, -24}, {-24, -45, -45}, {0, -24, -24},
      {-34, -34, 0},   {-24, 0, -24},   {-45, -45, -24}, {64, 64, 64},    {-32, 0, -32},   {0, -32, 0},
      {-32, 0, 32},    {-24, -45, -24}, {45, 24, 45},    {24, -24, -45},  {-45, -24, 24},  {80, 80, 80},
      {64, 0, 0},      {0, 0, -64},     {0, -64, -64},   {-24, -24, 45},  {96, 96, 96},    {64, 64, 0},
      {45, -24, -24},  {34, -34, 0},    {112, 112, 112}, {24, -45, -45},  {45, 45, -24},   {0, -32, 32},
      {24, -24, 45},   {0, 96, 96},     {45, -24, 24},   {24, -45, -24},  {-24, -45, 24},  {0, -64, 0},
      {96, 0, 0},      {128, 128, 128}, {64, 0, 64},     {144, 144, 144}, {96, 96, 0},     {-36, -36, 36},
      {45, -24, -45},  {45, -45, -24},  {0, 0, -96},     {0, 128, 128},   {0, 96, 0},      {45, 24, -45},
      {-128, 0, 0},    {24, -45, 24},   {-45, 24, -45},  {64, 0, -64},    {64, -64, -64},  {96, 0, 96},
      {45, -45, 24},   {24, 45, -45},   {64, 64, -64},   {128, 128, 0},   {0, 0, -128},    {-24, 45, -45},
  };
  if (index < 0) {
    if (c >= 3) return 0;
    size_t idx = size_t(-(index + 1));
    idx %= 1 + 2 * (72 - 1);
    int32_t result = kDelta[(idx + 1) >> 1][c] * ((idx & 1) ? 1 : -1);
    if (bit_depth > 8) result *= 1 << (bit_depth - 8);
    return result;
  }
  size_t idx = size_t(index);
  auto scale = [&](size_t value) { return int32_t((value * ((size_t(1) << bit_depth) - 1)) >> 2); };
  if (palette_size <= idx && idx < palette_size + 64) {
    if (c >= 3) return 0;
    idx -= palette_size;
    idx >>= c * 2;
    return scale(idx % 4) + (1 << std::max<int>(0, int(bit_depth) - 3));
  } else if (palette_size + 64 <= idx) {
    if (c >= 3) return 0;
    idx -= palette_size + 64;
    if (c == 1) idx /= 5;
    if (c == 2) idx /= 25;
    return scale(idx % 5);
  }
  return pal.row(uint32_t(c))[idx];
}

static void inv_palette(std::vector<ModularChannel>& ch, const ModularTransform& t, const WeightedHeader& wph,
                        uint32_t bit_depth_in) {
  // channel 0 is the palette, channel begin+1 the index channel.
  size_t b = t.begin_channel + 1, n = t.num_channels;
  ModularChannel pal = std::move(ch[0]);
  ModularChannel index = std::move(ch[b]);
  size_t bit_depth = std::min<uint32_t>(bit_depth_in, 24);
  std::vector<ModularChannel> outs;
  size_t w = index.w, h = index.h;
  for (size_t c = 0; c < n; c++) {
    ModularChannel out(index.w, index.h, index.hshift, index.vshift);
    if (w == 0) {
    } else if (t.num_deltas == 0 && t.predictor_id == kZero) {
      for (size_t y = 0; y < h; y++)
        for (size_t x = 0; x < w; x++)
          out.row(uint32_t(y))[x] = palette_value(pal, index.row(uint32_t(y))[x], c, t.num_colors, bit_depth);
    } else {
      bool weighted = t.predictor_id == kWeighted;
      WpState wp(wph, weighted ? w : 0);
      for (size_t y = 0; y < h; y++) {
        int32_t* row = out.row(uint32_t(y));
        const int32_t* top_row = y > 0 ? out.row(uint32_t(y - 1)) : row;
        const int32_t* toptop_row = y > 1 ? out.row(uint32_t(y - 2)) : top_row;
        for (size_t x = 0; x < w; x++) {
          int32_t idx = index.row(uint32_t(y))[x];
          int32_t entry = palette_value(pal, idx, c, t.num_colors + t.num_deltas, bit_depth);
          Neigh nb = get_neigh(row, top_row, toptop_row, x, y, w);
          int64_t wp_pred = 0;
          int32_t wp_prop;
          if (weighted) wp.predict(x, y, nb.top, nb.left, nb.topright, nb.topleft, nb.toptop, wp_pred, wp_prop);
          int32_t val = entry;
          if (idx < int32_t(t.num_deltas)) val = int32_t(predict_one(t.predictor_id, nb, wp_pred) + entry);
          row[x] = val;
          if (weighted) wp.update(val, x, y);
        }
      }
    }
    outs.push_back(std::move(out));
  }
  ch.erase(ch.begin() + b);
  for (size_t c = 0; c < n; c++) ch.insert(ch.begin() + b + c, std::move(outs[c]));
  ch.erase(ch.begin());
}

void undo_transforms(std::vector<ModularChannel>& ch, const GroupHeader& header, uint32_t bit_depth) {
  for (size_t ti = header.transforms.size(); ti-- > 0;) {
    const ModularTransform& t = header.transforms[ti];
    if (t.id == 0) {
      inv_rct(ch, t.begin_channel, t.rct_type);
    } else if (t.id == 1) {
      inv_palette(ch, t, header.wp, bit_depth);
    } else {
      for (size_t si = t.squeezes.size(); si-- > 0;) {
        const SqueezeParams& s = t.squeezes[si];
        size_t b = s.begin_channel, e = b + s.num_channels;
        size_t offset = s.in_place ? e : ch.size() - s.num_channels;
        for (size_t c = b; c < e; c++) {
          ModularChannel out;
          if (s.horizontal) inv_hsqueeze(ch[c], ch[offset + (c - b)], out);
          else inv_vsqueeze(ch[c], ch[offset + (c - b)], out);
          ch[c] = std::move(out);
        }
        ch.erase(ch.begin() + offset, ch.begin() + offset + s.num_channels);
      }
    }
  }
}

void decode_modular_subbitstream(std::vector<ModularChannel>& channels, size_t stream_id,
                                 const ModularTree* global_tree, BitReader& br) {
  SubStream s;
  substream_begin(s, channels, stream_id, global_tree, br);
  substream_finish(s);
}

}  // namespace jxg
