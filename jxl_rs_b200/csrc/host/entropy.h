// Entropy-code front end: parses histogram sets (ANS alias tables / prefix
// code LUTs, context maps, hybrid-uint configs, LZ77 params) into flat tables
// that both the host-side symbol reader (used for headers, trees, LF and
// HF-metadata streams) and the device kernels consume unchanged.
//
// Reference: jxl/src/entropy_coding/{decode,ans,huffman,hybrid_uint,context_map}.rs
#pragma once
#include <cstdint>
#include <vector>

#include "bitreader.h"

namespace jxg {

// hybrid_uint.rs:11-16, packed for the device as
//   split_exponent | msb_in_token << 8 | lsb_in_token << 16
struct HybridUint {
  uint32_t split_exponent = 0, msb = 0, lsb = 0;
  uint32_t split_token() const { return 1u << split_exponent; }
  uint32_t packed() const { return split_exponent | (msb << 8) | (lsb << 16); }
  static HybridUint decode(uint32_t log_alpha_size, BitReader& br);
  // hybrid_uint.rs:87-102
  inline uint32_t read(uint32_t token, BitReader& br) const {
    if (token < split_token()) return token;
    uint32_t bits_in_token = lsb + msb;
    uint32_t nbits = (split_exponent - bits_in_token + ((token - split_token()) >> bits_in_token)) & 31;
    uint32_t low = token & ((1u << lsb) - 1);
    uint32_t token_nolow = token >> lsb;
    uint32_t bits = uint32_t(br.read(nbits));
    uint32_t hi = (token_nolow & ((1u << msb) - 1)) | (1u << msb);
    return (((hi << nbits) | bits) << lsb) | low;
  }
};

constexpr uint32_t kAnsChecksum = 0x130000;  // ans.rs:425
constexpr uint32_t kAnsLogSumProbs = 12;

// ans.rs:31-39 — 8-byte alias-table bucket, same field order and widths.
struct AnsBucket {
  uint8_t alias_symbol;
  uint8_t alias_cutoff;
  uint16_t dist;
  uint16_t alias_offset;
  uint16_t alias_dist_xor;
};
static_assert(sizeof(AnsBucket) == 8, "bucket must be 8 bytes");

// huffman.rs:18-21, packed as bits | value << 16.
using HuffEntry = uint32_t;

struct EntropyCode {
  // decode.rs:36-45
  bool lz77_enabled = false;
  uint32_t lz77_min_symbol = 0, lz77_min_length = 0;
  HybridUint lz77_length_uint;
  uint32_t lz_dist_cluster = 0;

  bool use_prefix = false;
  uint32_t log_alpha_size = 0;
  std::vector<uint8_t> context_map;  // context -> cluster
  uint32_t num_clusters = 0;
  std::vector<HybridUint> uint_configs;  // per cluster
  // ANS: num_clusters << log_alpha_size buckets.
  std::vector<AnsBucket> ans_buckets;
  // Prefix: per-cluster LUT (>= 256 root entries + 2nd level), concatenated.
  std::vector<HuffEntry> huff_entries;
  std::vector<uint32_t> huff_offset;  // per cluster, into huff_entries
  std::vector<int32_t> single_symbol;  // per cluster, -1 if none

  // decode.rs:487-545
  static EntropyCode decode(size_t num_contexts, BitReader& br, bool allow_lz77);
  bool is_rle() const;
  // Pieces of decode(), exposed for the known-answer tests (ans.rs:463-485, huffman.rs:516-527).
  static int32_t decode_ans_histogram_for_test(BitReader& br, uint32_t log_alpha_size, std::vector<AnsBucket>& out);
  static EntropyCode decode_prefix_codes_for_test(size_t num_clusters, BitReader& br);
};


// decode.rs:177-405 (host copy; the VarDCT and Modular device kernels each have their own, DESIGN §9 item 6).
class SymbolReader {
 public:
  SymbolReader(const EntropyCode& code, BitReader& br, size_t dist_multiplier);
  uint32_t read_unsigned(BitReader& br, size_t ctx) { return read_clustered(br, code_.context_map[ctx]); }
  int32_t read_signed(BitReader& br, size_t ctx) { return unpack_signed(read_unsigned(br, ctx)); }
  inline uint32_t read_clustered(BitReader& br, uint32_t cluster) {
    if (!code_.lz77_enabled) return code_.uint_configs[cluster].read(read_token(br, cluster), br);
    return read_clustered_lz77(br, cluster);
  }
  // decode.rs:400: latched errors, over-read, final ANS state.
  void check_final_state(BitReader& br) const;

  // Register-resident reader for the per-pixel Modular loops (no LZ77): BitReader::Local plus the ANS state.
  // One fill() per symbol covers the 16 refill bits of the ANS step and the <= 32 extra bits of the hybrid uint
  // (48 <= 56), so the symbol chain carries no refill branch. Same arithmetic as read_token / HybridUint::read.
  template <bool kPrefix>
  struct Local {
    BitReader::Local br;
    uint32_t state;
    const EntropyCode* code;
    uint32_t log_alpha, log_bucket;
    inline uint32_t token(uint32_t cluster) {
      if (kPrefix) {
        constexpr unsigned kRootBits = 8;
        const HuffEntry* t = &code->huff_entries[code->huff_offset[cluster]];
        size_t pos = size_t(br.peek(kRootBits));
        uint32_t n_bits = t[pos] & 0xff;
        if (n_bits > kRootBits) {
          br.consume(kRootBits);
          n_bits -= kRootBits;
          pos += t[pos] >> 16;
          pos += size_t(br.peek(n_bits));
        }
        HuffEntry e = t[pos];
        br.consume(e & 0xff);
        return e >> 16;
      }
      const AnsBucket* buckets = code->ans_buckets.data() + (size_t(cluster) << log_alpha);
      const uint32_t idx = state & 0xfff;
      const uint32_t i = idx >> log_bucket;
      const uint32_t pos = idx & ((1u << log_bucket) - 1);
      const AnsBucket b = buckets[i];
      // Mask arithmetic instead of ?: — alias / refill / direct-token are data dependent and the compiler turns
      // selects into (mispredicted) branches.
      const uint32_t am = 0u - uint32_t(pos >= b.alias_cutoff);
      const uint32_t offset = (uint32_t(b.alias_offset) & am) + pos;
      const uint32_t dist = uint32_t(b.dist) ^ (uint32_t(b.alias_dist_xor) & am);
      const uint32_t symbol = i ^ ((i ^ uint32_t(b.alias_symbol)) & am);
      const uint32_t next = (state >> kAnsLogSumProbs) * dist + offset;
      const uint32_t rm = 0u - uint32_t(next < (1u << 16));
      const uint32_t sh = 16u & rm;
      state = (next << sh) | (uint32_t(br.peek(16)) & rm);
      br.consume(sh);
      return symbol;
    }
    // One whole symbol of `cluster`: fill, token, hybrid-uint extra bits.
    inline bool room(size_t nsym) const { return br.room(nsym); }
    template <bool kUnchecked = false>
    inline uint32_t read_clustered(uint32_t cluster) {
      if (kUnchecked) br.fill_unchecked();
      else br.fill();
      const uint32_t tok = token(cluster);
      const HybridUint& u = code->uint_configs[cluster];
      // Branch-free hybrid uint (hybrid_uint.rs:87-102): a direct token takes 0 extra bits and selects itself;
      // whether a residual is below the split is data dependent and mispredicts on LF-image residuals.
      const uint32_t dm = 0u - uint32_t(tok >= u.split_token());  // all ones: the token carries extra bits
      const uint32_t bits_in_token = u.lsb + u.msb;
      const uint32_t nbits =
          (u.split_exponent - bits_in_token + ((tok - u.split_token()) >> bits_in_token)) & 31 & dm;
      const uint32_t low = tok & ((1u << u.lsb) - 1);
      const uint32_t token_nolow = tok >> u.lsb;
      const uint32_t bits = uint32_t(br.peek(nbits));
      br.consume(nbits);
      const uint32_t hi = (token_nolow & ((1u << u.msb) - 1)) | (1u << u.msb);
      const uint32_t composed = (((hi << nbits) | bits) << u.lsb) | low;
      return tok ^ ((tok ^ composed) & dm);
    }
  };
  bool can_localise() const { return !code_.lz77_enabled; }
  uint32_t ans_state() const { return state_; }
  void set_ans_state(uint32_t s) { state_ = s; }
  bool uses_prefix() const { return code_.use_prefix; }
  template <bool kPrefix>
  Local<kPrefix> local(const BitReader& br) const {
    return Local<kPrefix>{br.local(), state_, &code_, code_.log_alpha_size, kAnsLogSumProbs - code_.log_alpha_size};
  }
  template <bool kPrefix>
  void commit(const Local<kPrefix>& l, BitReader& br) {
    state_ = l.state;
    br.commit(l.br);
  }

 private:
  uint32_t read_clustered_lz77(BitReader& br, uint32_t cluster);
  // ans.rs:356-393 / huffman.rs:446-457 (in the header so that the per-pixel Modular loops inline it)
  inline uint32_t read_token(BitReader& br, uint32_t cluster) {
    if (code_.use_prefix) {
      constexpr unsigned kRootBits = 8;
      const HuffEntry* t = &code_.huff_entries[code_.huff_offset[cluster]];
      size_t pos = size_t(br.peek(kRootBits));
      uint32_t n_bits = t[pos] & 0xff;
      if (n_bits > kRootBits) {
        br.consume(kRootBits);
        n_bits -= kRootBits;
        pos += t[pos] >> 16;
        pos += size_t(br.peek(n_bits));
      }
      HuffEntry e = t[pos];
      br.consume(e & 0xff);
      return e >> 16;
    }
    const uint32_t log_bucket = kAnsLogSumProbs - code_.log_alpha_size;
    uint32_t idx = state_ & 0xfff;
    uint32_t i = idx >> log_bucket;
    uint32_t pos = idx & ((1u << log_bucket) - 1);
    const AnsBucket& b = code_.ans_buckets[(size_t(cluster) << code_.log_alpha_size) + i];
    bool alias = pos >= b.alias_cutoff;
    uint32_t offset = (alias ? b.alias_offset : 0) + pos;
    uint32_t dist = uint32_t(b.dist) ^ (alias ? b.alias_dist_xor : 0);
    uint32_t symbol = alias ? b.alias_symbol : i;
    uint32_t next = (state_ >> kAnsLogSumProbs) * dist + offset;
    if (next < (1u << 16)) {
      next = (next << 16) | uint32_t(br.peek(16));
      br.consume(16);
    }
    state_ = next;
    return symbol;
  }
  const EntropyCode& code_;
  uint32_t state_ = kAnsChecksum;
  // LZ77 (decode.rs:73-147)
  std::vector<uint32_t> window_;
  uint32_t dist_multiplier_ = 0, num_to_copy_ = 0, copy_pos_ = 0, num_decoded_ = 0;
  bool err_lz77_repeat_ = false, err_overflow_ = false;
};

// context_map.rs:43
std::vector<uint8_t> decode_context_map(size_t num_contexts, BitReader& br);

// headers/permutation.rs:27-160 (Lehmer-coded permutation)
// permutation.rs:103-160: applies a Lehmer code to the tail [skip, size) of the identity permutation.
std::vector<uint32_t> apply_lehmer(const std::vector<uint32_t>& lehmer, uint32_t skip, uint32_t size);
std::vector<uint32_t> decode_permutation(uint32_t size, uint32_t skip, const EntropyCode& code, BitReader& br,
                                         SymbolReader& reader);

}  // namespace jxg
