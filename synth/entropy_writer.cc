// See entropy_writer.h.
#include "entropy_writer.h"

#include <numeric>

namespace jxs {

namespace {

constexpr uint32_t kLogSum = 12, kSum = 1u << kLogSum;

// (symbol -> code bits, length) of the fixed log-count prefix code (ans.rs:325-349).
struct LogCountCode {
  uint8_t bits[14], len[14];
  LogCountCode() {
    static const uint8_t lens[14] = {5, 4, 4, 4, 4, 4, 3, 3, 3, 3, 3, 6, 7, 7};
    // canonical patterns recovered from the decoder LUT: index i -> (symbol, nbits)
    static const uint8_t kTable[128][2] = {
        {10, 3}, {12, 7}, {7, 3}, {3, 4}, {6, 3}, {8, 3}, {9, 3}, {5, 4}, {10, 3}, {4, 4}, {7, 3}, {1, 4}, {6, 3},
        {8, 3},  {9, 3},  {2, 4}, {10, 3}, {0, 5}, {7, 3}, {3, 4}, {6, 3}, {8, 3}, {9, 3}, {5, 4}, {10, 3}, {4, 4},
        {7, 3},  {1, 4},  {6, 3}, {8, 3}, {9, 3}, {2, 4}, {10, 3}, {11, 6}, {7, 3}, {3, 4}, {6, 3}, {8, 3}, {9, 3},
        {5, 4},  {10, 3}, {4, 4}, {7, 3}, {1, 4}, {6, 3}, {8, 3}, {9, 3}, {2, 4}, {10, 3}, {0, 5}, {7, 3}, {3, 4},
        {6, 3},  {8, 3},  {9, 3}, {5, 4}, {10, 3}, {4, 4}, {7, 3}, {1, 4}, {6, 3}, {8, 3}, {9, 3}, {2, 4}, {10, 3},
        {13, 7}, {7, 3},  {3, 4}, {6, 3}, {8, 3}, {9, 3}, {5, 4}, {10, 3}, {4, 4}, {7, 3}, {1, 4}, {6, 3}, {8, 3},
        {9, 3},  {2, 4},  {10, 3}, {0, 5}, {7, 3}, {3, 4}, {6, 3}, {8, 3}, {9, 3}, {5, 4}, {10, 3}, {4, 4}, {7, 3},
        {1, 4},  {6, 3},  {8, 3}, {9, 3}, {2, 4}, {10, 3}, {11, 6}, {7, 3}, {3, 4}, {6, 3}, {8, 3}, {9, 3}, {5, 4},
        {10, 3}, {4, 4},  {7, 3}, {1, 4}, {6, 3}, {8, 3}, {9, 3}, {2, 4}, {10, 3}, {0, 5}, {7, 3}, {3, 4}, {6, 3},
        {8, 3},  {9, 3},  {5, 4}, {10, 3}, {4, 4}, {7, 3}, {1, 4}, {6, 3}, {8, 3}, {9, 3}, {2, 4},
    };
    (void)lens;
    for (int s = 0; s < 14; s++) len[s] = 0;
    for (int i = 0; i < 128; i++) {
      int s = kTable[i][0];
      if (!len[s]) {
        len[s] = kTable[i][1];
        bits[s] = uint8_t(i & ((1 << kTable[i][1]) - 1));
      }
    }
  }
};
const LogCountCode kLogCountCode;

void write_u8(BitWriter& bw, uint32_t v) {  // inverse of ans.rs read_u8
  if (v == 0) {
    bw.write(0, 1);
    return;
  }
  bw.write(1, 1);
  uint32_t n = floor_log2(v);
  bw.write(n, 3);
  bw.write(v - (1u << n), n);
}

void write_hybrid_cfg(BitWriter& bw, const HybridCfg& c, uint32_t log_alpha) {  // hybrid_uint.rs:27-57
  bw.write(c.split_exponent, ceil_log2(log_alpha + 1));
  if (c.split_exponent != log_alpha) {
    bw.write(c.msb, ceil_log2(c.split_exponent + 1));
    bw.write(c.lsb, ceil_log2(c.split_exponent - c.msb + 1));
  }
}

// decoder-side alias mapping idx -> (symbol, offset), following ans.rs:197-266 / :356-393
void alias_lookup_table(const std::vector<uint16_t>& dist_in, uint32_t log_alpha, std::vector<uint16_t>& sym_of,
                        std::vector<uint16_t>& off_of) {
  const size_t table_size = size_t(1) << log_alpha;
  const uint32_t log_bucket = kLogSum - log_alpha;
  const uint16_t bucket_size = uint16_t(1u << log_bucket);
  std::vector<uint16_t> dist(table_size, 0);
  std::copy(dist_in.begin(), dist_in.end(), dist.begin());
  size_t alphabet_size = dist_in.size();
  struct W {
    uint16_t dist, alias_symbol, alias_offset, alias_cutoff;
  };
  int single = -1;
  for (size_t i = 0; i < table_size; i++)
    if (dist[i] == kSum) single = int(i);
  sym_of.assign(kSum, 0);
  off_of.assign(kSum, 0);
  if (single >= 0) {
    for (uint32_t idx = 0; idx < kSum; idx++) {
      sym_of[idx] = uint16_t(single);
      off_of[idx] = uint16_t(idx);
    }
    return;
  }
  std::vector<W> b(table_size);
  for (size_t i = 0; i < table_size; i++) b[i] = {dist[i], uint16_t(i < alphabet_size ? i : 0), 0, dist[i]};
  std::vector<size_t> underfull, overfull;
  for (size_t i = 0; i < table_size; i++) {
    if (dist[i] < bucket_size) underfull.push_back(i);
    else if (dist[i] > bucket_size) overfull.push_back(i);
  }
  while (!overfull.empty() && !underfull.empty()) {
    size_t o = overfull.back();
    overfull.pop_back();
    size_t u = underfull.back();
    underfull.pop_back();
    uint16_t by = uint16_t(bucket_size - b[u].alias_cutoff);
    b[o].alias_cutoff = uint16_t(b[o].alias_cutoff - by);
    b[u].alias_symbol = uint16_t(o);
    b[u].alias_offset = b[o].alias_cutoff;
    if (b[o].alias_cutoff < bucket_size) underfull.push_back(o);
    else if (b[o].alias_cutoff > bucket_size) overfull.push_back(o);
  }
  if (!overfull.empty() || !underfull.empty()) throw std::runtime_error("alias table construction failed");
  for (uint32_t idx = 0; idx < kSum; idx++) {
    uint32_t i = idx >> log_bucket, pos = idx & (bucket_size - 1u);
    if (b[i].alias_cutoff == bucket_size || pos < b[i].alias_cutoff) {
      sym_of[idx] = uint16_t(i);
      off_of[idx] = uint16_t(pos);
    } else {
      sym_of[idx] = b[i].alias_symbol;
      off_of[idx] = uint16_t(b[i].alias_offset - b[i].alias_cutoff + pos);
    }
  }
}

void write_histogram(BitWriter& bw, const std::vector<uint16_t>& freq, uint32_t log_alpha) {
  // freq sums to 4096 (or is empty -> treated as single symbol 0)
  size_t used = 0, last = 0;
  for (size_t i = 0; i < freq.size(); i++)
    if (freq[i]) {
      used++;
      last = i;
    }
  if (used <= 1) {  // single symbol: bits 1,0 + symbol (ans.rs:53-66)
    bw.write(1, 1);
    bw.write(0, 1);
    write_u8(bw, uint32_t(used ? last : 0));
    return;
  }
  bw.write(0, 1);
  bw.write(0, 1);
  // shift = 13: unary "111", then value 6 in 3 bits (ans.rs:101-112)
  bw.write(1, 1);
  bw.write(1, 1);
  bw.write(1, 1);
  bw.write(6, 3);
  size_t alphabet = std::max<size_t>(last + 1, 3);
  if (alphabet > (size_t(1) << log_alpha)) throw std::runtime_error("alphabet exceeds ANS table");
  write_u8(bw, uint32_t(alphabet - 3));
  std::vector<uint32_t> logc(alphabet, 0);
  uint32_t max_log = 0;
  for (size_t i = 0; i < alphabet; i++) {
    uint32_t c = i < freq.size() ? freq[i] : 0;
    logc[i] = c ? floor_log2(c) + 1 : 0;
    max_log = std::max(max_log, logc[i]);
  }
  size_t omit = 0;
  while (logc[omit] != max_log) omit++;
  for (size_t i = 0; i < alphabet; i++) bw.write(kLogCountCode.bits[logc[i]], kLogCountCode.len[logc[i]]);
  for (size_t i = 0; i < alphabet; i++) {
    if (i == omit || logc[i] <= 1) continue;
    uint32_t zeros = logc[i] - 1;
    int bitcount = std::min<int>(std::max<int>(13 - int((kLogSum - zeros) >> 1), 0), int(zeros));
    uint32_t c = freq[i];
    bw.write((c - (1u << zeros)) >> (zeros - bitcount), unsigned(bitcount));
    if (((c - (1u << zeros)) & ((1u << (zeros - bitcount)) - 1)) != 0) throw std::runtime_error("histogram precision loss");
  }
}

// ---- prefix codes (entropy_coding/huffman.rs) ----

// Huffman code lengths limited to `limit` bits: plain Huffman, and while the tree is too deep the small counts are
// raised (flattening the distribution) and the tree rebuilt. >= 2 used symbols.
std::vector<uint8_t> limited_code_lengths(std::vector<uint64_t> counts, unsigned limit) {
  const size_t n = counts.size();
  std::vector<uint8_t> len(n, 0);
  for (uint64_t floor = 1;; floor *= 2) {
    struct Node {
      uint64_t w;
      int l, r;
    };
    std::vector<Node> nodes;
    std::vector<int> live;
    for (size_t i = 0; i < n; i++)
      if (counts[i]) {
        nodes.push_back(Node{std::max(counts[i], floor), -1 - int(i), 0});
        live.push_back(int(nodes.size()) - 1);
      }
    while (live.size() > 1) {
      std::sort(live.begin(), live.end(), [&](int a, int b) { return nodes[a].w > nodes[b].w || (nodes[a].w == nodes[b].w && a > b); });
      int a = live.back();
      live.pop_back();
      int b = live.back();
      live.pop_back();
      nodes.push_back(Node{nodes[a].w + nodes[b].w, a, b});
      live.push_back(int(nodes.size()) - 1);
    }
    std::fill(len.begin(), len.end(), 0);
    unsigned deepest = 0;
    std::vector<std::pair<int, unsigned>> stack{{live[0], 0}};
    while (!stack.empty()) {
      auto [id, d] = stack.back();
      stack.pop_back();
      if (nodes[id].l < 0) {
        len[size_t(-1 - nodes[id].l)] = uint8_t(std::max(d, 1u));
        deepest = std::max(deepest, d);
      } else {
        stack.push_back({nodes[id].l, d + 1});
        stack.push_back({nodes[id].r, d + 1});
      }
    }
    if (deepest <= limit) return len;
  }
}

// Canonical codes in the decoder's order (huffman.rs:276-400): symbols sorted by (length, symbol) take consecutive
// codes; the table is indexed by the bit-reversed code, i.e. the pattern is written LSB first.
std::vector<uint16_t> canonical_bits(const std::vector<uint8_t>& len) {
  std::vector<uint16_t> bits(len.size(), 0);
  uint32_t code = 0;
  for (unsigned l = 1; l <= 15; l++) {
    for (size_t s = 0; s < len.size(); s++)
      if (len[s] == l) {
        uint32_t rev = 0;
        for (unsigned b = 0; b < l; b++)
          if (code & (1u << b)) rev |= 1u << (l - 1 - b);
        bits[s] = uint16_t(rev);
        code++;
      }
    code <<= 1;
  }
  return bits;
}

void write_varint16(BitWriter& bw, uint32_t v) {  // inverse of decode.rs:18-29
  if (v == 0) {
    bw.write(0, 1);
    return;
  }
  bw.write(1, 1);
  uint32_t n = floor_log2(v);
  bw.write(n, 4);
  bw.write(v - (1u << n), n);
}

// One prefix code in the format Table::decode reads (huffman.rs:404-443). `len` covers the announced alphabet.
void write_prefix_code(BitWriter& bw, const std::vector<uint8_t>& len) {
  const size_t al = len.size();
  if (al == 1) return;
  std::vector<uint32_t> used;
  for (size_t i = 0; i < al; i++)
    if (len[i]) used.push_back(uint32_t(i));
  const unsigned max_bits = ceil_log2(al);
  if (used.size() <= 2) {  // simple code (huffman.rs:73-205): 1 symbol (0 bits) or 2 symbols (1 bit each)
    bw.write(1, 2);
    bw.write(uint32_t(used.size()) - 1, 2);
    for (uint32_t sym : used) bw.write(sym, max_bits);
    return;
  }
  bw.write(0, 2);  // complex code, no skipped code-length-code entries
  // the lengths are sent literally (no repeat codes 16 / 17) up to the last used symbol: the decoder stops when the
  // Kraft sum is complete (huffman.rs:222)
  std::vector<uint64_t> cl_counts(18, 0);
  for (size_t i = 0; i <= used.back(); i++) cl_counts[len[i]]++;
  size_t distinct = 0;
  for (auto c : cl_counts) distinct += c != 0;
  static const uint8_t kOrder[18] = {1, 2, 3, 4, 0, 5, 17, 6, 16, 7, 8, 9, 10, 11, 12, 13, 14, 15};
  static const uint8_t kStaticBits[6] = {0b00, 0b0111, 0b011, 0b10, 0b01, 0b1111};  // value -> pattern (LSB first)
  static const uint8_t kStaticLen[6] = {2, 4, 3, 2, 2, 4};
  std::vector<uint8_t> cl_len(18, 0);
  if (distinct == 1) {  // a single code-length symbol: zero bits per length (num_codes == 1 is accepted, huffman.rs:430)
    for (int i = 0; i < 18; i++)
      if (cl_counts[i]) cl_len[i] = 1;
  } else {
    cl_len = limited_code_lengths(cl_counts, 5);
  }
  int space = 32;
  for (int i = 0; i < 18 && space > 0; i++) {
    const uint8_t v = cl_len[kOrder[i]];
    bw.write(kStaticBits[v], kStaticLen[v]);
    if (v) space -= 32 >> v;
  }
  if (distinct != 1 && space != 0) throw std::runtime_error("code-length code is not complete");
  if (distinct == 1) return;  // every length costs zero bits
  // the code-length code itself is canonical over symbols 0..17 with a 5-bit root table (huffman.rs:213)
  const std::vector<uint16_t> cl_bits = canonical_bits(cl_len);
  for (size_t i = 0; i <= used.back(); i++) bw.write(cl_bits[len[i]], cl_len[len[i]]);
}

}  // namespace

std::vector<uint16_t> normalize_counts(const std::vector<uint64_t>& counts, size_t alphabet) {
  std::vector<uint16_t> f(alphabet, 0);
  uint64_t total = 0;
  for (size_t i = 0; i < alphabet; i++) total += counts[i];
  if (total == 0) return f;
  size_t used = 0, argmax = 0;
  for (size_t i = 0; i < alphabet; i++) {
    if (counts[i]) used++;
    if (counts[i] > counts[argmax]) argmax = i;
  }
  if (used == 1) {
    f[argmax] = uint16_t(kSum);
    return f;
  }
  int64_t sum = 0;
  for (size_t i = 0; i < alphabet; i++) {
    if (!counts[i]) continue;
    uint64_t v = (counts[i] * kSum + total / 2) / total;
    if (v == 0) v = 1;
    if (v >= kSum) v = kSum - 1;
    f[i] = uint16_t(v);
    sum += int64_t(v);
  }
  // fix up the sum on the largest entries
  int64_t diff = int64_t(kSum) - sum;
  while (diff != 0) {
    size_t best = alphabet;
    for (size_t i = 0; i < alphabet; i++) {
      if (!f[i]) continue;
      if (diff < 0 && f[i] <= 1) continue;
      if (best == alphabet || f[i] > f[best]) best = i;
    }
    int64_t step = diff > 0 ? std::min<int64_t>(diff, int64_t(kSum - 1) - f[best]) : -std::min<int64_t>(-diff, f[best] - 1);
    if (step == 0) throw std::runtime_error("cannot normalise histogram");
    f[best] = uint16_t(int64_t(f[best]) + step);
    diff -= step;
  }
  return f;
}

std::vector<uint8_t> cluster_contexts(size_t num_contexts, const std::vector<const std::vector<Token>*>& streams,
                                      uint32_t max_clusters, uint32_t& num_clusters, const HybridCfg& cfg) {
  std::vector<uint8_t> map(num_contexts, 0);
  if (num_contexts <= max_clusters) {
    for (size_t i = 0; i < num_contexts; i++) map[i] = uint8_t(i);
    num_clusters = uint32_t(num_contexts);
    return map;
  }
  // mean token per context; contexts ordered by mean and cut into equal-population buckets
  std::vector<double> sum(num_contexts, 0.0);
  std::vector<uint64_t> cnt(num_contexts, 0);
  for (auto* s : streams)
    for (const Token& t : *s) {
      uint32_t tok, nb, bits;
      cfg.encode(t.value, tok, nb, bits);
      sum[t.ctx] += tok;
      cnt[t.ctx]++;
    }
  std::vector<uint32_t> used;
  uint64_t total = 0;
  for (size_t i = 0; i < num_contexts; i++)
    if (cnt[i]) {
      used.push_back(uint32_t(i));
      total += cnt[i];
    }
  std::sort(used.begin(), used.end(), [&](uint32_t a, uint32_t b) {
    double ma = sum[a] / double(cnt[a]), mb = sum[b] / double(cnt[b]);
    return ma < mb || (ma == mb && a < b);
  });
  uint32_t k = std::min<uint32_t>(max_clusters, std::max<uint32_t>(1, uint32_t(used.size())));
  uint64_t acc = 0;
  uint32_t cur = 0;
  uint32_t max_used = 0;
  for (uint32_t c : used) {
    uint32_t bucket = std::min<uint32_t>(k - 1, uint32_t(acc * k / std::max<uint64_t>(total, 1)));
    cur = std::max(cur, bucket);
    map[c] = uint8_t(cur);
    max_used = std::max(max_used, cur);
    acc += cnt[c];
  }
  // compact ids so that there are no holes (context_map.rs:31-41)
  std::vector<int> remap(256, -1);
  uint32_t next = 0;
  remap[0] = int(next++);  // unused contexts share cluster 0
  for (size_t i = 0; i < num_contexts; i++) {
    if (remap[map[i]] < 0) remap[map[i]] = int(next++);
  }
  for (auto& m : map) m = uint8_t(remap[m]);
  num_clusters = next;
  return map;
}

static std::vector<Sym> plain_symbols(const std::vector<Token>& tokens, const HybridCfg& cfg) {
  std::vector<Sym> out;
  out.reserve(tokens.size());
  for (const Token& t : tokens) {
    Sym s{t.ctx, 0, 0, 0};
    cfg.encode(t.value, s.tok, s.nbits, s.bits);
    out.push_back(s);
  }
  return out;
}
// Each token with the configuration of its context's cluster.
static std::vector<Sym> plain_symbols(const std::vector<Token>& tokens, const std::vector<uint8_t>& cluster_of_ctx,
                                      const std::vector<HybridCfg>& cfgs) {
  std::vector<Sym> out;
  out.reserve(tokens.size());
  for (const Token& t : tokens) {
    Sym s{t.ctx, 0, 0, 0};
    cfgs.at(cluster_of_ctx.at(t.ctx)).encode(t.value, s.tok, s.nbits, s.bits);
    out.push_back(s);
  }
  return out;
}

std::vector<Sym> lz77_symbols(const std::vector<Token>& tokens, const HybridCfg& cfg, const Lz77& lz, const HybridCfg& len_cfg,
                              uint32_t dist_ctx) {
  std::vector<Sym> out;
  out.reserve(tokens.size());
  static const uint32_t kDist[6] = {1, 2, 3, 4, 8, 64};
  for (size_t i = 0; i < tokens.size();) {
    size_t best_len = 0, best_dist = 0;
    for (uint32_t d : kDist) {
      if (d > i) break;
      size_t l = 0;
      while (i + l < tokens.size() && l < 4000 && tokens[i + l].value == tokens[i + l - d].value) l++;
      if (l > best_len) best_len = l, best_dist = d;
    }
    if (best_len >= std::max<size_t>(lz.min_length, 4)) {
      Sym len{tokens[i].ctx, 0, 0, 0};  // the copy is announced in the context of the symbol it replaces
      len_cfg.encode(uint32_t(best_len - lz.min_length), len.tok, len.nbits, len.bits);
      len.tok += lz.min_symbol;
      out.push_back(len);
      Sym dist{dist_ctx, 0, 0, 0};
      cfg.encode(uint32_t(best_dist - 1), dist.tok, dist.nbits, dist.bits);
      out.push_back(dist);
      i += best_len;
    } else {
      Sym s{tokens[i].ctx, 0, 0, 0};
      cfg.encode(tokens[i].value, s.tok, s.nbits, s.bits);
      if (s.tok >= lz.min_symbol) throw std::runtime_error("literal token collides with the LZ77 range");
      out.push_back(s);
      i++;
    }
  }
  return out;
}

static AnsCode build_code_syms(size_t num_contexts, const std::vector<uint8_t>& cluster_of_ctx, uint32_t num_clusters,
                               const std::vector<const std::vector<Sym>*>& streams, uint32_t min_log_alpha, bool use_prefix);

AnsCode build_code(size_t num_contexts, const std::vector<uint8_t>& cluster_of_ctx, uint32_t num_clusters,
                   const std::vector<const std::vector<Token>*>& streams, uint32_t min_log_alpha, bool use_prefix,
                   const HybridCfg& cfg) {
  std::vector<std::vector<Sym>> syms;
  for (auto* s : streams) syms.push_back(plain_symbols(*s, cfg));
  std::vector<const std::vector<Sym>*> ptrs;
  for (auto& v : syms) ptrs.push_back(&v);
  AnsCode code = build_code_syms(num_contexts, cluster_of_ctx, num_clusters, ptrs, min_log_alpha, use_prefix);
  code.cfg = cfg;
  return code;
}

AnsCode build_code_cfgs(size_t num_contexts, const std::vector<uint8_t>& cluster_of_ctx, uint32_t num_clusters,
                        const std::vector<const std::vector<Token>*>& streams, uint32_t min_log_alpha, bool use_prefix,
                        const std::vector<HybridCfg>& cfgs) {
  if (cfgs.size() != num_clusters) throw std::runtime_error("one hybrid-uint configuration per cluster expected");
  std::vector<std::vector<Sym>> syms;
  for (auto* s : streams) syms.push_back(plain_symbols(*s, cluster_of_ctx, cfgs));
  std::vector<const std::vector<Sym>*> ptrs;
  for (auto& v : syms) ptrs.push_back(&v);
  AnsCode code = build_code_syms(num_contexts, cluster_of_ctx, num_clusters, ptrs, min_log_alpha, use_prefix);
  code.cfg = cfgs[0];
  code.cluster_cfgs = cfgs;
  return code;
}

AnsCode build_code_lz77(size_t num_contexts, const std::vector<uint8_t>& cluster_of_ctx, uint32_t num_clusters,
                        const std::vector<const std::vector<Sym>*>& streams, const Lz77& lz, bool use_prefix) {
  AnsCode code = build_code_syms(num_contexts, cluster_of_ctx, num_clusters, streams, 8, use_prefix);
  code.lz = lz;
  return code;
}

static AnsCode build_code_syms(size_t num_contexts, const std::vector<uint8_t>& cluster_of_ctx, uint32_t num_clusters,
                               const std::vector<const std::vector<Sym>*>& streams, uint32_t min_log_alpha, bool use_prefix) {
  AnsCode code;
  code.use_prefix = use_prefix;
  code.num_contexts = uint32_t(num_contexts);
  code.context_map = cluster_of_ctx;
  code.num_clusters = num_clusters;
  std::vector<std::vector<uint64_t>> counts(num_clusters, std::vector<uint64_t>(256, 0));
  uint32_t max_token = 0;
  for (auto* s : streams)
    for (const Sym& t : *s) {
      const uint32_t tok = t.tok;
      if (tok >= 256) throw std::runtime_error("token too large for ANS alphabet");
      counts[cluster_of_ctx[t.ctx]][tok]++;
      max_token = std::max(max_token, tok);
    }
  if (use_prefix) {
    code.log_alpha_size = 15;  // HUFFMAN_MAX_BITS (decode.rs:509-513): only sizes the hybrid-uint configuration
    code.plen.resize(num_clusters);
    code.pbits.resize(num_clusters);
    for (uint32_t c = 0; c < num_clusters; c++) {
      size_t used = 0, last = 0;
      for (size_t i = 0; i < 256; i++)
        if (counts[c][i]) {
          used++;
          last = i;
        }
      std::vector<uint64_t> cc(counts[c].begin(), counts[c].begin() + last + 1);
      if (used == 0) cc[0] = 1, used = 1;  // unused cluster: one symbol, zero bits
      std::vector<uint8_t> len(cc.size(), 0);
      if (used == 1) len[last] = 0;  // single symbol: simple code, 0 bits (the decoder's table reads nothing)
      else if (used == 2) {
        for (size_t i = 0; i < cc.size(); i++)
          if (cc[i]) len[i] = 1;
      } else {
        len = limited_code_lengths(cc, 15);
      }
      if (used == 1) {
        code.plen[c].assign(cc.size(), 0);
        code.pbits[c].assign(cc.size(), 0);
        code.plen[c][last] = 0;
      } else {
        code.plen[c] = len;
        code.pbits[c] = canonical_bits(len);
      }
    }
    return code;
  }
  code.log_alpha_size = std::max<uint32_t>(min_log_alpha, std::max<uint32_t>(5, ceil_log2(uint64_t(max_token) + 1)));
  if (code.log_alpha_size > 8) throw std::runtime_error("alphabet too large");
  // split_exponent must be <= log_alpha_size; 4 always is.
  size_t alphabet = size_t(1) << code.log_alpha_size;
  code.freqs.resize(num_clusters);
  code.inv.resize(num_clusters);
  code.slots.resize(num_clusters);
  for (uint32_t c = 0; c < num_clusters; c++) {
    code.freqs[c] = normalize_counts(counts[c], alphabet);
    std::vector<uint16_t> dist = code.freqs[c];
    bool empty = std::all_of(dist.begin(), dist.end(), [](uint16_t v) { return v == 0; });
    if (empty) {
      dist[0] = uint16_t(kSum);
      code.freqs[c][0] = uint16_t(kSum);
    }
    // trim to the alphabet size the serialiser will announce, as the decoder builds its alias table from that
    size_t last = 0;
    for (size_t i = 0; i < dist.size(); i++)
      if (dist[i]) last = i;
    size_t used = 0;
    for (auto v : dist) used += v != 0;
    size_t asz = used <= 1 ? last + 1 : std::max<size_t>(last + 1, 3);
    dist.resize(asz);
    std::vector<uint16_t> sym_of, off_of;
    alias_lookup_table(dist, code.log_alpha_size, sym_of, off_of);
    std::vector<uint16_t>& start = code.inv[c];
    start.assign(alphabet + 1, 0);
    for (size_t s = 0; s < alphabet; s++) start[s + 1] = uint16_t(start[s] + code.freqs[c][s]);
    code.slots[c].assign(kSum, 0);
    for (uint32_t idx = 0; idx < kSum; idx++) code.slots[c][start[sym_of[idx]] + off_of[idx]] = uint16_t(idx);
  }
  return code;
}

static const HybridCfg& cluster_cfg(const AnsCode& code, uint32_t c) {
  if (!code.cluster_cfgs.empty()) return code.cluster_cfgs[c];
  return code.lz.enabled && code.lz_dist_own_cfg && c == code.context_map.back() ? code.lz_dist_cfg : code.cfg;
}

void write_context_map(BitWriter& bw, const std::vector<uint8_t>& map, uint32_t num_clusters) {
  // context map (context_map.rs:43-76)
  uint32_t bits_needed = ceil_log2(num_clusters);
  if (bits_needed <= 3 && uint32_t(map.size()) * bits_needed < 2048) {
    bw.write(1, 1);  // is_simple
    bw.write(bits_needed, 2);
    if (bits_needed)
      for (uint8_t m : map) bw.write(m, bits_needed);
  } else {
    bw.write(0, 1);  // not simple
    bw.write(0, 1);  // no MTF
    std::vector<Token> toks;
    toks.reserve(map.size());
    for (uint8_t m : map) toks.push_back(Token{0, m});
    std::vector<uint8_t> one(1, 0);
    AnsCode sub = build_code(1, one, 1, {&toks});
    write_code(bw, sub);
    write_tokens(bw, sub, toks);
  }
}

void write_code(BitWriter& bw, const AnsCode& code) {
  if (code.lz.enabled) {  // decode.rs:36-44 + :489-498
    bw.write(1, 1);
    const uint32_t ms = code.lz.min_symbol, ml = code.lz.min_length;
    if (ms == 224) bw.u2s_sel(0);
    else if (ms == 512) bw.u2s_sel(1);
    else if (ms == 4096) bw.u2s_sel(2);
    else if (ms >= 8 && ms < 8 + (1u << 15)) bw.u2s_sel(3, ms - 8, 15);
    else throw std::runtime_error("LZ77 min_symbol out of range");
    if (ml == 3) bw.u2s_sel(0);
    else if (ml == 4) bw.u2s_sel(1);
    else if (ml >= 5 && ml < 9) bw.u2s_sel(2, ml - 5, 2);
    else if (ml >= 9 && ml < 9 + 256) bw.u2s_sel(3, ml - 9, 8);
    else throw std::runtime_error("LZ77 min_length out of range");
    write_hybrid_cfg(bw, code.lz_len_cfg, 8);
  } else {
    bw.write(0, 1);
  }
  if (code.num_contexts > 1) write_context_map(bw, code.context_map, code.num_clusters);
  if (code.use_prefix) {  // decode.rs:509-524, huffman.rs:466-480
    bw.write(1, 1);
    for (uint32_t c = 0; c < code.num_clusters; c++) write_hybrid_cfg(bw, cluster_cfg(code, c), 15);
    for (uint32_t c = 0; c < code.num_clusters; c++) write_varint16(bw, uint32_t(code.plen[c].size()) - 1);
    for (uint32_t c = 0; c < code.num_clusters; c++) {
      // a one-symbol code whose symbol is not 0 still needs the simple-code header; plen alone cannot say which
      // symbol, so that case is written here
      size_t used = 0, last = 0;
      for (size_t i = 0; i < code.plen[c].size(); i++)
        if (code.plen[c][i]) used++, last = i;
      if (used == 0 && code.plen[c].size() > 1) {  // single symbol = the last of the announced alphabet
        bw.write(1, 2);
        bw.write(0, 2);
        bw.write(uint32_t(code.plen[c].size() - 1), ceil_log2(code.plen[c].size()));
        continue;
      }
      (void)last;
      write_prefix_code(bw, code.plen[c]);
    }
    return;
  }
  bw.write(0, 1);  // use_prefix_code = 0
  bw.write(code.log_alpha_size - 5, 2);
  for (uint32_t c = 0; c < code.num_clusters; c++) write_hybrid_cfg(bw, cluster_cfg(code, c), code.log_alpha_size);
  for (uint32_t c = 0; c < code.num_clusters; c++) write_histogram(bw, code.freqs[c], code.log_alpha_size);
}

void write_tokens(BitWriter& bw, const AnsCode& code, const std::vector<Token>& tokens) {
  if (!code.cluster_cfgs.empty()) return write_symbols(bw, code, plain_symbols(tokens, code.context_map, code.cluster_cfgs));
  write_symbols(bw, code, plain_symbols(tokens, code.cfg));
}

void write_symbols(BitWriter& bw, const AnsCode& code, const std::vector<Sym>& tokens) {
  if (code.use_prefix) {  // no initial state; token pattern then the hybrid-uint extra bits (decode.rs:286-330)
    for (const Sym& t : tokens) {
      const uint32_t c = code.context_map[t.ctx];
      if (t.tok >= code.plen[c].size()) throw std::runtime_error("token outside the prefix alphabet");
      bw.write(code.pbits[c][t.tok], code.plen[c][t.tok]);
      bw.write(t.bits, t.nbits);
    }
    return;
  }
  const size_t n = tokens.size();
  std::vector<uint8_t> has_chunk(n, 0);
  std::vector<uint16_t> chunk(n, 0);
  uint32_t state = 0x130000;
  for (size_t i = n; i-- > 0;) {
    const Sym& t = tokens[i];
    const uint32_t tok = t.tok;
    uint32_t c = code.context_map[t.ctx];
    uint32_t f = code.freqs[c][tok];
    if (f == 0) throw std::runtime_error("token with zero frequency");
    if ((state >> 20) >= f) {
      has_chunk[i] = 1;
      chunk[i] = uint16_t(state & 0xffff);
      state >>= 16;
    }
    uint32_t q = state / f, r = state % f;
    state = (q << kLogSum) + code.slots[c][code.inv[c][tok] + r];
  }
  bw.write(state, 32);
  for (size_t i = 0; i < n; i++) {
    if (has_chunk[i]) bw.write(chunk[i], 16);
    bw.write(tokens[i].bits, tokens[i].nbits);
  }
}

}  // namespace jxs
