// Entropy *encoder* for synthetic JPEG XL streams: bit writer, hybrid-uint
// tokenisation, context clustering, ANS histogram normalisation + serialisation
// in the format jxl/src/entropy_coding/ans.rs:98-314 parses, and the reverse
// rANS pass that makes a decoder end in state 0x130000 (ans.rs:425).
//
// Test-data tooling (the reference has no encoder: jxl_cli/src/enc/ only holds
// PNG/PPM/NPY writers); not part of the product path.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <vector>

namespace jxs {

struct BitWriter {
  std::vector<uint8_t> bytes;
  uint64_t acc = 0;
  unsigned nbits = 0;
  size_t total = 0;
  void write(uint64_t v, unsigned n) {  // n <= 32
    if (n == 0) return;
    acc |= (v & ((uint64_t(1) << n) - 1)) << nbits;
    nbits += n;
    total += n;
    while (nbits >= 8) {
      bytes.push_back(uint8_t(acc));
      acc >>= 8;
      nbits -= 8;
    }
  }
  void zero_pad_to_byte() {
    if (nbits) write(0, 8 - nbits);
  }
  std::vector<uint8_t> finish() {
    zero_pad_to_byte();
    return std::move(bytes);
  }
  // u2S-style helpers (headers/encodings.rs:76-98)
  void u2s_sel(unsigned sel, uint64_t v = 0, unsigned n = 0) {
    write(sel, 2);
    write(v, n);
  }
  void write_u64(uint64_t v) {  // encodings.rs:111-139
    if (v == 0) write(0, 2);
    else if (v <= 16) { write(1, 2); write(v - 1, 4); }
    else if (v <= 272) { write(2, 2); write(v - 17, 8); }
    else {
      write(3, 2);
      write(v & 0xfff, 12);
      v >>= 12;
      unsigned shift = 12;
      while (v) {
        write(1, 1);
        if (shift >= 60) { write(v & 0xf, 4); return; }
        write(v & 0xff, 8);
        v >>= 8;
        shift += 8;
      }
      write(0, 1);
    }
  }
};

inline uint32_t ceil_log2(uint64_t x) {
  uint32_t n = 0;
  while ((uint64_t(1) << n) < x) n++;
  return n;
}
inline uint32_t floor_log2(uint64_t x) {
  uint32_t n = 0;
  while (x >>= 1) n++;
  return n;
}
inline uint32_t pack_signed(int32_t v) { return v >= 0 ? uint32_t(v) << 1 : ((uint32_t(-(v + 1)) << 1) | 1); }

struct Token {
  uint32_t ctx;
  uint32_t value;
};

// hybrid_uint.rs:11-16 config and the inverse of HybridUint::read (:87-102)
struct HybridCfg {
  uint32_t split_exponent = 4, msb = 2, lsb = 0;
  void encode(uint32_t value, uint32_t& token, uint32_t& nbits, uint32_t& bits) const {
    uint32_t split_token = 1u << split_exponent;
    if (value < split_token) {
      token = value;
      nbits = 0;
      bits = 0;
      return;
    }
    uint32_t n = floor_log2(value);
    uint32_t m = value - (1u << n);
    token = split_token + ((n - split_exponent) << (msb + lsb)) + ((m >> (n - msb)) << lsb) + (m & ((1u << lsb) - 1));
    nbits = n - msb - lsb;
    bits = (value >> lsb) & ((1u << nbits) - 1);
  }
};

// LZ77 layer of a code (entropy_coding/decode.rs:36-44, 286-330): tokens >= min_symbol announce a copy of
// hybrid(length_cfg, token - min_symbol) + min_length earlier symbols, followed by the distance - 1 coded in the extra
// context behind the regular ones (dist_multiplier 0: plain distances).
struct Lz77 {
  bool enabled = false;
  uint32_t min_symbol = 224, min_length = 3;
};
// One coded symbol: context (index into the context map; the distance context is num_contexts - 1 of an LZ77 code),
// entropy-coded token, raw bits behind it.
struct Sym {
  uint32_t ctx, tok, nbits, bits;
};

// One clustered ANS code (all clusters), ready to serialise and to encode with.
struct AnsCode {
  uint32_t num_contexts = 0;
  std::vector<uint8_t> context_map;
  uint32_t num_clusters = 0;
  uint32_t log_alpha_size = 6;
  HybridCfg cfg;
  std::vector<HybridCfg> cluster_cfgs;            // empty: every cluster uses `cfg`; else one configuration per cluster
  std::vector<std::vector<uint16_t>> freqs;       // [cluster][alphabet] sums to 4096
  std::vector<std::vector<uint16_t>> inv;         // [cluster] start index per symbol into slots
  std::vector<std::vector<uint16_t>> slots;       // [cluster] concatenated idx lists per symbol (offset -> idx)
  // Prefix-code variant (entropy_coding/huffman.rs): per cluster canonical code lengths (<= 15) and the bit patterns
  // as the decoder's table expects them (first bit read = LSB).
  Lz77 lz;
  HybridCfg lz_len_cfg{0, 0, 0};  // hybrid-uint configuration of the copy lengths (8-bit alphabet form, decode.rs:493)
  // Hybrid-uint configuration of the distance cluster (the last cluster of the context map) when it differs from `cfg`.
  bool lz_dist_own_cfg = false;
  HybridCfg lz_dist_cfg{0, 0, 0};
  bool use_prefix = false;
  std::vector<std::vector<uint8_t>> plen;         // [cluster][alphabet]
  std::vector<std::vector<uint16_t>> pbits;       // [cluster][alphabet]
};

// Normalises counts to sum 4096 with every used symbol >= 1.
std::vector<uint16_t> normalize_counts(const std::vector<uint64_t>& counts, size_t alphabet);
// Builds a code from tokens: `cluster_of_ctx` (size num_contexts, values < num_clusters) given by the caller; every
// cluster uses the hybrid-uint configuration `cfg`.
AnsCode build_code(size_t num_contexts, const std::vector<uint8_t>& cluster_of_ctx, uint32_t num_clusters,
                   const std::vector<const std::vector<Token>*>& streams, uint32_t min_log_alpha = 5, bool use_prefix = false,
                   const HybridCfg& cfg = HybridCfg());
// build_code with one hybrid-uint configuration per cluster (cfgs[cluster]).
AnsCode build_code_cfgs(size_t num_contexts, const std::vector<uint8_t>& cluster_of_ctx, uint32_t num_clusters,
                        const std::vector<const std::vector<Token>*>& streams, uint32_t min_log_alpha, bool use_prefix,
                        const std::vector<HybridCfg>& cfgs);
// Convenience: one cluster per context when num_contexts <= 8, else quantile clustering into <= max_clusters.
std::vector<uint8_t> cluster_contexts(size_t num_contexts, const std::vector<const std::vector<Token>*>& streams,
                                      uint32_t max_clusters, uint32_t& num_clusters, const HybridCfg& cfg);
// Serialises a context map (context_map.rs:43-76): the simple form when it fits, else entropy coded without MTF.
void write_context_map(BitWriter& bw, const std::vector<uint8_t>& map, uint32_t num_clusters);
// Serialises the LZ77 parameters, context map, ANS flag, log_alpha, uint configs, histograms (decode.rs:487-545).
void write_code(BitWriter& bw, const AnsCode& code);
// Writes initial state + symbols so that decoding ends in 0x130000.
void write_tokens(BitWriter& bw, const AnsCode& code, const std::vector<Token>& tokens);

// LZ77 variant: tokens -> coded symbols with greedy copies (runs and short-distance repeats), then a code built from
// the symbols of all streams (num_contexts counts the distance context), and the symbol writer.
std::vector<Sym> lz77_symbols(const std::vector<Token>& tokens, const HybridCfg& cfg, const Lz77& lz, const HybridCfg& len_cfg,
                              uint32_t dist_ctx);
AnsCode build_code_lz77(size_t num_contexts, const std::vector<uint8_t>& cluster_of_ctx, uint32_t num_clusters,
                        const std::vector<const std::vector<Sym>*>& streams, const Lz77& lz, bool use_prefix);
void write_symbols(BitWriter& bw, const AnsCode& code, const std::vector<Sym>& syms);

}  // namespace jxs
