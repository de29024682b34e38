// Modular-frame device path (BASELINE config 5; SURVEY §8 rows a18 / a19), sm_90a.
//   k_modular_decode   per-pixel MA-tree walk + predictor (+ weighted predictor) + ANS / prefix symbol decode of the
//                      ModularHF sections: one lane per (frame, group) stream, persistent lanes pulling streams
//                      (longest first) from a device queue            <- modular/decode/channel.rs:220, tree.rs:189-280,
//                      streams with LZ77 in a launch of their own        predict.rs:148-527, decode/common.rs:85,
//                                                                        entropy_coding/decode.rs:286-330
//   k_modular_local_rct  inverse RCT of a group's local transforms     <- transforms/rct.rs:9-40 (apply_local.rs)
//   k_modular_rct / k_unsqueeze_h / k_unsqueeze_v  global inverse transforms over the job rectangles (full planes for
//                                                    a whole frame, the dependency cone of a region, host/modular_region.h)
//                                                                     <- transforms/rct.rs, squeeze.rs:144-195,390,577
//   k_modular_store    i32 planes -> interleaved RGB u8                <- render/stages/convert.rs:642-690
// Integer work throughout: results are bit-exact against the CPU path (tests/test_gpu_modular.py).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../../include/jxg.h"
#include "launch.h"
#include "modular_device.h"
#include "output_stage.h"

namespace jxgpu {

namespace {

__constant__ uint32_t c_div_lookup[64] = {
    16777216, 8388608, 5592405, 4194304, 3355443, 2796202, 2396745, 2097152, 1864135, 1677721, 1525201,
    1398101,  1290555, 1198372, 1118481, 1048576, 986895,  932067,  883011,  838860,  798915,  762600,
    729444,   699050,  671088,  645277,  621378,  599186,  578524,  559240,  541200,  524288,  508400,
    493447,   479349,  466033,  453438,  441505,  430185,  419430,  409200,  399457,  390167,  381300,
    372827,   364722,  356962,  349525,  342392,  335544,  328965,  322638,  316551,  310689,  305040,
    299593,   294337,  289262,  284359,  279620,  275036,  270600,  266305,  262144,
};

struct MBr {  // bit reader over an 8-byte aligned, zero padded section copy (bit_reader.rs semantics)
  const uint32_t* words;
  uint32_t wlimit, wi;  // next word to load (clamped: a corrupt stream cannot walk out of the blob)
  uint64_t buf;         // `avail` valid bits, LSB first
  uint32_t avail;
  uint64_t bitpos;      // bits consumed
  __device__ __forceinline__ void init(const uint32_t* w, uint32_t limit, uint64_t start_bit) {
    words = w;
    wlimit = limit;
    bitpos = start_bit;
    wi = min(uint32_t(start_bit >> 5), limit);
    const uint32_t sh = uint32_t(start_bit) & 31;
    buf = (uint64_t(__ldg(words + wi)) | (uint64_t(__ldg(words + min(wi + 1, limit))) << 32)) >> sh;
    avail = 64 - sh;
    wi = min(wi + 2, limit);
  }
  __device__ __forceinline__ void refill() {  // keeps >= 32 valid bits
    if (avail <= 32) {
      buf |= uint64_t(__ldg(words + wi)) << avail;
      avail += 32;
      wi = min(wi + 1, wlimit);
    }
  }
  __device__ __forceinline__ uint32_t peek32() {
    refill();
    return uint32_t(buf);
  }
  __device__ __forceinline__ void consume(uint32_t n) {  // n <= 32, after a peek32()
    buf >>= n;
    avail -= n;
    bitpos += n;
  }
  __device__ __forceinline__ uint32_t read(uint32_t n) {  // n <= 32
    const uint32_t w = peek32();
    const uint32_t v = n == 32 ? w : (w & ((1u << n) - 1u));
    consume(n);
    return v;
  }
};

struct MSym {  // symbol reader state of one stream (decode.rs:177-405; LZ77 state in MLz)
  MBr br;
  uint32_t ans_state;
  const uint8_t* cmap;
  const uint32_t* cfg;
  const uint2* ans;
  const uint32_t* huff;
  const uint32_t* huff_offset;
  uint32_t use_prefix, log_alpha;
};

__device__ __forceinline__ uint32_t m_token(MSym& s, uint32_t cluster) {
  uint32_t token;
  if (s.use_prefix) {  // huffman.rs:446-457
    const uint32_t* t = s.huff + __ldg(s.huff_offset + cluster);
    const uint32_t w = s.br.peek32();
    uint32_t pos = w & 0xff;
    uint32_t e = __ldg(t + pos);
    uint32_t nb = e & 0xff, used = 0;
    if (nb > 8) {
      used = 8;
      nb -= 8;
      pos += (e >> 16) + ((w >> 8) & ((1u << nb) - 1u));
      e = __ldg(t + pos);
    }
    s.br.consume(used + (e & 0xff));  // <= 8 + 15 bits
    token = e >> 16;
  } else {  // ans.rs:356-393
    const uint32_t log_bucket = 12 - s.log_alpha;
    const uint32_t idx = s.ans_state & 0xfff;
    const uint32_t i = idx >> log_bucket, pos = idx & ((1u << log_bucket) - 1);
    const uint2 b = __ldg(s.ans + ((cluster << s.log_alpha) + i));
    const bool alias = pos >= ((b.x >> 8) & 0xff);
    const uint32_t dist = (b.x >> 16) ^ (alias ? (b.y >> 16) : 0u);
    const uint32_t offset = pos + (alias ? (b.y & 0xffff) : 0u);
    token = alias ? (b.x & 0xff) : i;
    uint32_t next = (s.ans_state >> 12) * dist + offset;
    if (next < (1u << 16)) next = (next << 16) | s.br.read(16);
    s.ans_state = next;
  }
  return token;
}

// hybrid_uint.rs:87-102
__device__ __forceinline__ uint32_t m_hybrid(MSym& s, uint32_t cfg, uint32_t token) {
  const uint32_t split_exponent = cfg & 0xff, msb = (cfg >> 8) & 0xff, lsb = (cfg >> 16) & 0xff;
  const uint32_t split_token = 1u << split_exponent;
  if (token < split_token) return token;
  const uint32_t bits_in_token = lsb + msb;
  const uint32_t nbits = (split_exponent - bits_in_token + ((token - split_token) >> bits_in_token)) & 31;
  const uint32_t low = token & ((1u << lsb) - 1);
  const uint32_t bits = s.br.read(nbits);
  const uint32_t hi = ((token >> lsb) & ((1u << msb) - 1)) | (1u << msb);
  return (((hi << nbits) | bits) << lsb) | low;
}

__device__ __forceinline__ uint32_t m_read_clustered(MSym& s, uint32_t cluster) {
  const uint32_t token = m_token(s, cluster);
  return m_hybrid(s, __ldg(s.cfg + cluster), token);
}

// LZ77 state of one stream (decode.rs:73-147). All channels of the stream share it: the window, the count of decoded
// symbols and a pending copy carry across channel boundaries.
constexpr uint32_t kLzMask = (1u << 20) - 1;  // WINDOW_MASK: the window is a ring of 2^20 symbols
struct MLz {
  uint32_t* win;  // min(2^20, pixels of the stream) entries: positions below 2^20 index it directly
  uint32_t decoded, to_copy, copy_pos;
  uint32_t mult, min_symbol, min_length, len_cfg, dist_cluster;
  uint32_t err;  // a copy before any symbol, or a length overflow (decode.rs:300-317)
};

__constant__ int8_t c_special_dist[120][2] = {  // SPECIAL_DISTANCES (decode.rs:87-101): (dx, dy)
    {0, 1},  {1, 0},  {1, 1},  {-1, 1}, {0, 2},  {2, 0},  {1, 2},  {-1, 2}, {2, 1},  {-2, 1}, {2, 2},  {-2, 2},
    {0, 3},  {3, 0},  {1, 3},  {-1, 3}, {3, 1},  {-3, 1}, {2, 3},  {-2, 3}, {3, 2},  {-3, 2}, {0, 4},  {4, 0},
    {1, 4},  {-1, 4}, {4, 1},  {-4, 1}, {3, 3},  {-3, 3}, {2, 4},  {-2, 4}, {4, 2},  {-4, 2}, {0, 5},  {3, 4},
    {-3, 4}, {4, 3},  {-4, 3}, {5, 0},  {1, 5},  {-1, 5}, {5, 1},  {-5, 1}, {2, 5},  {-2, 5}, {5, 2},  {-5, 2},
    {4, 4},  {-4, 4}, {3, 5},  {-3, 5}, {5, 3},  {-5, 3}, {0, 6},  {6, 0},  {1, 6},  {-1, 6}, {6, 1},  {-6, 1},
    {2, 6},  {-2, 6}, {6, 2},  {-6, 2}, {4, 5},  {-4, 5}, {5, 4},  {-5, 4}, {3, 6},  {-3, 6}, {6, 3},  {-6, 3},
    {0, 7},  {7, 0},  {1, 7},  {-1, 7}, {5, 5},  {-5, 5}, {7, 1},  {-7, 1}, {4, 6},  {-4, 6}, {6, 4},  {-6, 4},
    {2, 7},  {-2, 7}, {7, 2},  {-7, 2}, {3, 7},  {-3, 7}, {7, 3},  {-7, 3}, {5, 6},  {-5, 6}, {6, 5},  {-6, 5},
    {8, 0},  {4, 7},  {-4, 7}, {7, 4},  {-7, 4}, {8, 1},  {8, 2},  {6, 6},  {-6, 6}, {8, 3},  {5, 7},  {-5, 7},
    {7, 5},  {-7, 5}, {8, 4},  {6, 7},  {-6, 7}, {7, 6},  {-7, 6}, {8, 5},  {7, 7},  {-7, 7}, {8, 6},  {8, 7},
};

// One symbol of `cluster` (decode.rs:286-330). Without LZ77 this is m_read_clustered. With it, a pending copy comes
// before the token read and ignores the pixel's cluster; every symbol, copied or not, is pushed to the window. The
// pull reads its slot before the push writes: a copy at distance 2^20 reads the slot the push then overwrites.
template <bool LZ>
__device__ __forceinline__ uint32_t m_read(MSym& s, MLz& z, uint32_t cluster) {
  if (!LZ) return m_read_clustered(s, cluster);
  uint32_t sym;
  if (z.to_copy) {
    z.to_copy--;
    sym = z.win[z.copy_pos++ & kLzMask];
  } else {
    const uint32_t tok = m_token(s, cluster);
    if (tok < z.min_symbol) {
      sym = m_hybrid(s, __ldg(s.cfg + cluster), tok);
    } else {
      if (z.decoded == 0) {  // lz77_repeat
        z.err = 1;
        return 0;
      }
      const uint32_t n = m_hybrid(s, z.len_cfg, tok - z.min_symbol);
      if (n > 0xffffffffu - z.min_length) {
        z.err = 1;
        return 0;
      }
      const uint32_t dsym = m_read_clustered(s, z.dist_cluster);
      uint32_t d = dsym - 120;  // apply_copy (decode.rs:107-122)
      if (dsym < 120) {
        const int64_t v = int64_t(z.mult * uint32_t(c_special_dist[dsym][1])) + c_special_dist[dsym][0] - 1;
        d = (v < 0 || v > int64_t(0xffffffffu)) ? 0u : uint32_t(v);
      }
      const uint32_t distance = min(min(d, kLzMask) + 1u, z.decoded);
      z.copy_pos = z.decoded - distance;
      z.to_copy = n + z.min_length - 1;  // the first copied symbol is returned now
      sym = z.win[z.copy_pos++ & kLzMask];
    }
  }
  z.win[z.decoded++ & kLzMask] = sym;
  return sym;
}

__device__ __forceinline__ int32_t m_unpack_signed(uint32_t u) { return int32_t((u >> 1) ^ (((~u) & 1u) - 1u)); }
__device__ __forceinline__ int32_t wadd(int32_t a, int32_t b) { return int32_t(uint32_t(a) + uint32_t(b)); }
__device__ __forceinline__ int32_t wsub(int32_t a, int32_t b) { return int32_t(uint32_t(a) - uint32_t(b)); }
__device__ __forceinline__ int32_t wabs(int32_t a) { return a < 0 ? int32_t(0u - uint32_t(a)) : a; }
__device__ __forceinline__ int64_t labs64(int64_t a) { return a < 0 ? -a : a; }
__device__ __forceinline__ uint32_t floor_log2_u64(uint64_t v) { return 63 - __clzll(v); }

// predict.rs:137-143
__device__ __forceinline__ int64_t clamped_gradient(int64_t left, int64_t top, int64_t topleft) {
  const int64_t mn = min(left, top), mx = max(left, top);
  const int64_t grad = left + top - topleft;
  const int64_t g = topleft < mn ? mx : grad;
  return topleft > mx ? mn : g;
}

// Weighted predictor (predict.rs:221-527); state rows live in per-stream global scratch.
struct MWp {
  uint32_t* perr;  // [(xsize + 1) * 2][4]
  int32_t* err;    // [(xsize + 1) * 2]
  uint32_t xsize;
  uint32_t p1c, p2c, p3ca, p3cb, p3cc, p3cd, p3ce, w[4];
  int64_t prediction[4];
  int64_t pred;
  __device__ __forceinline__ void predict(uint32_t x, uint32_t y, int32_t top, int32_t left, int32_t topright,
                                          int32_t topleft, int32_t toptop, int64_t& pred_out, int32_t& prop_out) {
    const uint32_t cur_row = (y & 1) ? 0 : xsize + 1, prev_row = (y & 1) ? xsize + 1 : 0;
    const uint32_t pos_ne = x + 1 < xsize ? x + 1 : x;
    const uint32_t pos_nw = x > 0 ? x - 1 : 0;
    const uint4 en = *reinterpret_cast<const uint4*>(perr + (prev_row + x) * 4);
    const uint4 ene = *reinterpret_cast<const uint4*>(perr + (prev_row + pos_ne) * 4);
    const uint4 enw = *reinterpret_cast<const uint4*>(perr + (prev_row + pos_nw) * 4);
    const uint32_t es[4] = {en.x + ene.x + enw.x, en.y + ene.y + enw.y, en.z + ene.z + enw.z, en.w + ene.w + enw.w};
    uint32_t wv[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const uint32_t e = es[i];
      const uint32_t l2 = floor_log2_u64(uint64_t(e) + 1);
      const uint32_t shift = l2 > 5 ? l2 - 5 : 0;
      wv[i] = 4u + ((w[i] * c_div_lookup[e >> shift]) >> shift);
    }
    const int64_t te_w = err[cur_row + x];
    const int64_t te_n = err[prev_row + 1 + x];
    const int64_t te_nw = err[prev_row + 1 + pos_nw];
    const int64_t sum_wn = te_n + te_w;
    const int64_t te_ne = err[prev_row + 1 + pos_ne];
    int64_t p = te_w;
    if (labs64(te_n) > labs64(p)) p = te_n;
    if (labs64(te_nw) > labs64(p)) p = te_nw;
    if (labs64(te_ne) > labs64(p)) p = te_ne;
    const int64_t n = int64_t(top) << 3, wv_ = int64_t(left) << 3, ne = int64_t(topright) << 3,
                  nw = int64_t(topleft) << 3, nn = int64_t(toptop) << 3;
    const int64_t p0 = wv_ + ne - n;
    const int64_t p1 = n - (((sum_wn + te_ne) * int64_t(p1c)) >> 5);
    const int64_t p2 = wv_ - (((sum_wn + te_nw) * int64_t(p2c)) >> 5);
    const int64_t p3 = n - ((te_nw * int64_t(p3ca) + te_n * int64_t(p3cb) + te_ne * int64_t(p3cc) +
                             (nn - n) * int64_t(p3cd) + (nw - wv_) * int64_t(p3ce)) >> 5);
    const uint32_t log_weight = floor_log2_u64(uint64_t(wv[0]) + wv[1] + wv[2] + wv[3]);
    const int64_t w0 = int64_t(wv[0]) >> (log_weight - 4), w1 = int64_t(wv[1]) >> (log_weight - 4),
                  w2 = int64_t(wv[2]) >> (log_weight - 4), w3 = int64_t(wv[3]) >> (log_weight - 4);
    const int64_t weight_sum = w0 + w1 + w2 + w3;
    const int64_t sum = (weight_sum >> 1) - 1 + w0 * p0 + w1 * p1 + w2 * p2 + w3 * p3;
    int64_t pr = (sum * int64_t(c_div_lookup[weight_sum - 1])) >> 24;
    if (((te_n ^ te_w) | (te_n ^ te_nw)) <= 0) {
      const int64_t mx = max(wv_, max(ne, n)), mn = min(wv_, min(ne, n));
      pr = max(mn, min(mx, pr));
    }
    prediction[0] = p0;
    prediction[1] = p1;
    prediction[2] = p2;
    prediction[3] = p3;
    pred = pr;
    pred_out = (pr + 3) >> 3;
    prop_out = int32_t(p);
  }
  __device__ __forceinline__ void update(int32_t val, uint32_t x, uint32_t y) {
    const uint32_t cur_row = (y & 1) ? 0 : xsize + 1, prev_row = (y & 1) ? xsize + 1 : 0;
    const int64_t v = int64_t(val) << 3;
    err[cur_row + x + 1] = int32_t(pred - v);
    uint32_t* cur = perr + (cur_row + x) * 4;
    uint32_t* prev = perr + (prev_row + x + 1) * 4;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      const uint32_t e = uint32_t((labs64(prediction[i] - v) + 3) >> 3);
      cur[i] = e;
      prev[i] += e;
    }
  }
};

// predict.rs:148-194 in wrapping 32-bit arithmetic. The pixel is (guess + offset + multiplier * dec) truncated to i32
// (decode/common.rs:85), so only the low 32 bits of the guess matter; the comparisons of Select and of the clamped
// gradient are made on exact values (a difference of two i32 fits a u32; the clamped gradient lies between left and top).
__device__ __forceinline__ int32_t m_predict32(uint32_t predictor, int32_t L, int32_t T, int32_t TL, int32_t TR, int32_t ww,
                                               int32_t nn, int32_t nee, int64_t wp_pred) {
  switch (predictor) {
    case 0: return 0;
    case 1: return L;
    case 2: return T;
    case 4: {
      const uint32_t dl = T > TL ? uint32_t(T) - uint32_t(TL) : uint32_t(TL) - uint32_t(T);  // |pp - L| = |T - TL|
      const uint32_t dt = L > TL ? uint32_t(L) - uint32_t(TL) : uint32_t(TL) - uint32_t(L);  // |pp - T| = |L - TL|
      return dl < dt ? L : T;
    }
    case 5: {
      const int32_t mn = min(L, T), mx = max(L, T);
      const int32_t grad = wsub(wadd(L, T), TL);  // exact whenever it is the result (then mn <= grad <= mx)
      return TL < mn ? mx : (TL > mx ? mn : grad);
    }
    case 6: return int32_t(wp_pred);
    case 7: return TR;
    case 8: return TL;
    case 9: return ww;
    case 3: return int32_t((int64_t(T) + L) / 2);
    case 10: return int32_t((int64_t(L) + TL) / 2);
    case 11: return int32_t((int64_t(T) + TL) / 2);
    case 12: return int32_t((int64_t(T) + TR) / 2);
    default: return int32_t((6 * int64_t(T) - 2 * int64_t(nn) + 7 * int64_t(L) + int64_t(ww) + int64_t(nee) + 3 * int64_t(TR) + 8) / 16);
  }
}

// One channel whose tree walk is a table over one property (MRectDev::walk == kWalkLut): per pixel the property, one
// table load (predictor, cluster, leaf), the predictor and the symbol. specialized_trees.rs:197-372 is the CPU form.
// PROP: the property (2..15), -1 = single leaf, -2 = read from the rect at run time. Pixels with all neighbours inside
// the channel (y >= 2, 2 <= x < w - 2) skip the edge rules of predict.rs:64-103. LZ: the stream's code uses LZ77.
template <bool WP, int PROP, bool LZ>
__device__ __forceinline__ void m_channel_lut(const MBatchDev& B, const MRectDev& rc, MSym& sym, MLz& lz, MWp& wp,
                                              const int4* nodes) {
  const uint32_t w = rc.w, h = rc.h;
  const int prop_rt = int(rc.walk >> 8);
  int32_t* const base = B.planes + rc.base;
  const uint32_t* const lut = reinterpret_cast<const uint32_t*>(B.blob + rc.lut_off);
  const uint32_t single = uint32_t(rc.lut_off);
  for (uint32_t y = 0; y < h; y++) {
    int32_t* const row = base + size_t(y) * rc.stride;
    const int32_t* const top = y > 0 ? row - rc.stride : row;
    const int32_t* const toptop = y > 1 ? top - rc.stride : top;
    int32_t prev_p9 = 0;
    // one pixel: neighbours in, value out (and stored)
    auto pixel = [&](uint32_t x, int32_t left, int32_t n, int32_t nw, int32_t ne, int32_t ww, int32_t nn, int32_t nee) -> int32_t {
      int64_t wp_pred = 0;
      int32_t wp_prop = 0;
      if (WP) wp.predict(x, y, n, left, ne, nw, nn, wp_pred, wp_prop);
      const int32_t p9 = wsub(wadd(left, n), nw);
      uint32_t e = single;
      const int p = PROP == -2 ? (prop_rt == int(kLutNoProperty) ? -1 : prop_rt) : PROP;
      if (p >= 0) {
        int32_t v;
        switch (p) {  // tree.rs:189-280
          case 2: v = int32_t(y); break;
          case 3: v = int32_t(x); break;
          case 4: v = wabs(n); break;
          case 5: v = wabs(left); break;
          case 6: v = n; break;
          case 7: v = left; break;
          case 8: v = wsub(left, prev_p9); break;
          case 9: v = p9; break;
          case 10: v = wsub(left, nw); break;
          case 11: v = wsub(nw, n); break;
          case 12: v = wsub(n, ne); break;
          case 13: v = wsub(n, nn); break;
          case 14: v = wsub(left, ww); break;
          default: v = wp_prop; break;
        }
        e = __ldg(lut + uint32_t(min(max(v, kLutMin), kLutMin + kLutSize - 1) - kLutMin));
      }
      prev_p9 = p9;
      const int32_t guess = m_predict32(e & 15u, left, n, nw, ne, ww, nn, nee, wp_pred);
      const int32_t dec = m_unpack_signed(m_read<LZ>(sym, lz, (e >> 4) & 255u));
      int32_t val;
      if (e & (1u << 12)) {
        val = wadd(guess, dec);
      } else {
        const int4 leaf = __ldg(nodes + (e >> 16));
        val = int32_t(uint32_t(guess) + uint32_t(leaf.y) + uint32_t(leaf.w) * uint32_t(dec));  // decode/common.rs:85, low 32 bits
      }
      if (WP) wp.update(val, x, y);
      row[x] = val;
      return val;
    };
    // neighbours with the edge rules (predict.rs:64-103); v1 / v2: the two pixels to the left in this row
    auto edge_pixel = [&](uint32_t x, int32_t v1, int32_t v2) -> int32_t {
      const bool has_top = y > 0, has_tt = y > 1;
      const int32_t left = x > 0 ? v1 : (has_top ? top[0] : 0);
      const int32_t n = has_top ? top[x] : left;
      const int32_t nw = (x > 0 && has_top) ? top[x - 1] : left;
      const int32_t ne = (x + 1 < w && has_top) ? top[x + 1] : n;
      const int32_t ww = x > 1 ? v2 : left;
      const int32_t nn = has_tt ? toptop[x] : n;
      const int32_t nee = (x + 2 < w && has_top) ? top[x + 2] : ne;
      return pixel(x, left, n, nw, ne, ww, nn, nee);
    };
    int32_t v1 = 0, v2 = 0;  // row[x - 1], row[x - 2]
    uint32_t x = 0;
    const uint32_t x_in0 = min(2u, w), x_in1 = (y >= 2 && w > 4) ? w - 2 : x_in0;
    for (; x < x_in0; x++) {
      const int32_t v = edge_pixel(x, v1, v2);
      v2 = v1;
      v1 = v;
    }
    if (x_in1 > x_in0) {
      // interior: sliding window over the two rows above, loaded ahead of their use
      int32_t t_prev = top[x - 1], t_cur = top[x], t_next = top[x + 1], tt_cur = toptop[x];
      for (; x < x_in1; x++) {
        const int32_t t_next2 = top[x + 2];
        const int32_t tt_next = toptop[x + 1];
        const int32_t v = pixel(x, v1, t_cur, t_prev, t_next, v2, tt_cur, t_next2);
        v2 = v1;
        v1 = v;
        t_prev = t_cur;
        t_cur = t_next;
        t_next = t_next2;
        tt_cur = tt_next;
      }
    }
    for (; x < w; x++) {
      const int32_t v = edge_pixel(x, v1, v2);
      v2 = v1;
      v1 = v;
    }
  }
}

}  // namespace

// One lane per stream; lanes >= S of a warp idle. Persistent: finished lanes pull the next stream from B.queue.
// LZ: every stream of the launch uses LZ77 (the others run without the window code).
template <int S, bool LZ>
__global__ void __launch_bounds__(128) k_modular_decode(const MBatchDev B, const uint32_t total_lanes) {
  const uint32_t warp = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (lane >= S) return;
  for (uint32_t sidx = warp * S + lane; sidx < B.num_streams; sidx = atomicAdd(B.queue, 1u) + total_lanes) {
    const MStreamDev& st = B.streams[B.order[sidx]];
    const CodeDev& code = B.codes[st.code];
    MSym sym;
    sym.br.init(reinterpret_cast<const uint32_t*>(B.blob + st.sec_off), (st.sec_len >> 2) + 1, st.data_bitpos);
    sym.cmap = B.blob + code.cmap_off;
    sym.cfg = reinterpret_cast<const uint32_t*>(B.blob + code.cfg_off);
    sym.ans = reinterpret_cast<const uint2*>(B.blob + code.ans_off);
    sym.huff = reinterpret_cast<const uint32_t*>(B.blob + code.huff_off);
    sym.huff_offset = reinterpret_cast<const uint32_t*>(B.blob + code.huff_offset_off);
    sym.use_prefix = code.use_prefix;
    sym.log_alpha = code.log_alpha;
    sym.ans_state = 0x130000u;
    if (!code.use_prefix) sym.ans_state = sym.br.read(32);  // ans.rs:431
    MLz lz;
    if (LZ) {
      lz.win = B.lz_window + st.lz_window_off;
      lz.decoded = lz.to_copy = lz.copy_pos = lz.err = 0;
      lz.mult = st.dist_multiplier;
      lz.min_symbol = code.lz_min_symbol;
      lz.min_length = code.lz_min_length;
      lz.len_cfg = code.lz_len_cfg;
      lz.dist_cluster = code.lz_dist_cluster;
    }
    const int4* const nodes = reinterpret_cast<const int4*>(B.blob + st.tree_off);
    const int4 root = __ldg(nodes);
    MWp wp;
    const bool use_wp = st.uses_wp != 0;
    if (use_wp) {
      wp.p1c = st.wp_params[0];
      wp.p2c = st.wp_params[1];
      wp.p3ca = st.wp_params[2];
      wp.p3cb = st.wp_params[3];
      wp.p3cc = st.wp_params[4];
      wp.p3cd = st.wp_params[5];
      wp.p3ce = st.wp_params[6];
      for (int i = 0; i < 4; i++) wp.w[i] = st.wp_params[7 + i];
    }
    for (uint32_t ci = 0; ci < st.num_rects; ci++) {
      const MRectDev rc = B.rects[st.first_rect + ci];
      if (rc.w == 0 || rc.h == 0) continue;  // channel numbering stays stable (bitstream.rs:203-206)
      const uint32_t w = rc.w, h = rc.h;
      int32_t* const base = B.planes + rc.base;
      // Decision nodes on the channel index / stream id are constant for the whole channel: resolve them once.
      int4 chan_root = root;
      while (chan_root.x == 0 || chan_root.x == 1) {
        const int32_t v = chan_root.x == 0 ? int32_t(ci) : int32_t(st.stream_id);
        chan_root = __ldg(nodes + (v > chan_root.y ? chan_root.z : chan_root.z + 1));
      }
      if (use_wp) {  // fresh state per channel (channel.rs:236)
        wp.xsize = w;
        wp.perr = reinterpret_cast<uint32_t*>(B.wp_scratch + st.wp_scratch_off);
        wp.err = reinterpret_cast<int32_t*>(wp.perr + size_t(w + 1) * 8);
        for (uint32_t i = 0; i < (w + 1) * 8; i++) wp.perr[i] = 0;
        for (uint32_t i = 0; i < (w + 1) * 2; i++) wp.err[i] = 0;
      }
      if ((rc.walk & 0xff) == kWalkLut) {
        if (use_wp) {
          m_channel_lut<true, -2, LZ>(B, rc, sym, lz, wp, nodes);
        } else {
          switch (rc.walk >> 8) {  // the property is a compile-time constant of the channel loop
            case 9: m_channel_lut<false, 9, LZ>(B, rc, sym, lz, wp, nodes); break;
            case 10: m_channel_lut<false, 10, LZ>(B, rc, sym, lz, wp, nodes); break;
            case 13: m_channel_lut<false, 13, LZ>(B, rc, sym, lz, wp, nodes); break;
            case kLutNoProperty: m_channel_lut<false, -1, LZ>(B, rc, sym, lz, wp, nodes); break;
            default: m_channel_lut<false, -2, LZ>(B, rc, sym, lz, wp, nodes); break;
          }
        }
        continue;
      }
      for (uint32_t y = 0; y < h; y++) {
        int32_t* const row = base + size_t(y) * rc.stride;
        const int32_t* const top = y > 0 ? row - rc.stride : row;
        const int32_t* const toptop = y > 1 ? top - rc.stride : top;
        int32_t prev_p9 = 0;
        int4 row_root = chan_root;  // ... and the ones on y once per row
        while (row_root.x >= 0 && row_root.x <= 2) {
          const int32_t v = row_root.x == 0 ? int32_t(ci) : (row_root.x == 1 ? int32_t(st.stream_id) : int32_t(y));
          row_root = __ldg(nodes + (v > row_root.y ? row_root.z : row_root.z + 1));
        }
        // Sliding neighbour window (predict.rs:64-103): the pixels of this row stay in registers (no store -> load
        // round trip on the dependent chain), the rows above are loaded one pixel ahead of their use.
        const bool has_top = y > 0, has_tt = y > 1;
        int32_t v_prev = 0, v_prev2 = 0;                 // row[x-1], row[x-2]
        int32_t t_prev = 0;                              // top[x-1]
        int32_t t_cur = has_top ? top[0] : 0;            // top[x]
        int32_t t_next = (has_top && w > 1) ? top[1] : 0;  // top[x+1]
        int32_t tt_cur = has_tt ? toptop[0] : 0;         // toptop[x]
        const int32_t top0 = t_cur;
        for (uint32_t x = 0; x < w; x++) {
          const int32_t t_next2 = (has_top && x + 2 < w) ? top[x + 2] : 0;    // used as top[x+1] next iteration
          const int32_t tt_next = (has_tt && x + 1 < w) ? toptop[x + 1] : 0;  // toptop[x+1]
          const int32_t left = x > 0 ? v_prev : (has_top ? top0 : 0);
          const int32_t n = has_top ? t_cur : left;
          const int32_t nw = (x > 0 && has_top) ? t_prev : left;
          const int32_t ne = (x + 1 < w && has_top) ? t_next : n;
          const int32_t ww = x > 1 ? v_prev2 : left;
          const int32_t nn = has_tt ? tt_cur : n;
          int64_t wp_pred = 0;
          int32_t wp_prop = 0;
          if (use_wp) wp.predict(x, y, n, left, ne, nw, nn, wp_pred, wp_prop);
          const int32_t p9 = wsub(wadd(left, n), nw);
          // tree.rs:189-280 + flat walk (tree.rs:360-390)
          int4 nd = row_root;
          while (nd.x >= 0) {
            int32_t v;
            switch (nd.x) {
              case 0: v = int32_t(ci); break;
              case 1: v = int32_t(st.stream_id); break;
              case 2: v = int32_t(y); break;
              case 3: v = int32_t(x); break;
              case 4: v = wabs(n); break;
              case 5: v = wabs(left); break;
              case 6: v = n; break;
              case 7: v = left; break;
              case 8: v = wsub(left, prev_p9); break;
              case 9: v = p9; break;
              case 10: v = wsub(left, nw); break;
              case 11: v = wsub(nw, n); break;
              case 12: v = wsub(n, ne); break;
              case 13: v = wsub(n, nn); break;
              case 14: v = wsub(left, ww); break;
              case 15: v = wp_prop; break;
              default: {  // properties of previous channels of the same shape (decode/common.rs:40-83)
                const uint32_t j = uint32_t(nd.x) - 16u, slot = j >> 2;
                v = 0;
                if (slot < rc.ref_count) {
                  const MRectDev rr = B.rects[B.refs[rc.ref_first + slot]];
                  const int32_t* rrow = B.planes + rr.base + size_t(y) * rr.stride;
                  const int32_t* rprev = y > 0 ? rrow - rr.stride : rrow;
                  const int32_t rv = rrow[x];
                  if ((j & 3) == 0) v = wabs(rv);
                  else if ((j & 3) == 1) v = rv;
                  else {
                    const int32_t vleft = x > 0 ? rrow[x - 1] : 0;
                    const int32_t vtop = y > 0 ? rprev[x] : vleft;
                    const int32_t vtl = (x > 0 && y > 0) ? rprev[x - 1] : vleft;
                    const int64_t d = int64_t(rv) - clamped_gradient(vleft, vtop, vtl);
                    v = (j & 3) == 2 ? int32_t(d < 0 ? -d : d) : int32_t(d);
                  }
                }
                break;
              }
            }
            nd = __ldg(nodes + (v > nd.y ? nd.z : nd.z + 1));
          }
          prev_p9 = p9;
          const uint32_t predictor = uint32_t(nd.z) & 15u, ctx = uint32_t(nd.z) >> 4;
          int64_t guess;
          const int64_t L = left, T = n, TL = nw, TR = ne;
          switch (predictor) {  // predict.rs:148-194
            case 0: guess = 0; break;
            case 1: guess = L; break;
            case 2: guess = T; break;
            case 3: guess = (T + L) / 2; break;
            case 4: {
              const int64_t pp = L + T - TL;
              guess = labs64(pp - L) < labs64(pp - T) ? L : T;
              break;
            }
            case 5: guess = clamped_gradient(L, T, TL); break;
            case 6: guess = wp_pred; break;
            case 7: guess = TR; break;
            case 8: guess = TL; break;
            case 9: guess = ww; break;
            case 10: guess = (L + TL) / 2; break;
            case 11: guess = (T + TL) / 2; break;
            case 12: guess = (T + TR) / 2; break;
            default: {
              const int32_t nee = (x + 2 < w && has_top) ? t_next2 : ne;
              guess = (6 * T - 2 * int64_t(nn) + 7 * L + int64_t(ww) + int64_t(nee) + 3 * TR + 8) / 16;
            }
          }
          guess += int64_t(nd.y);
          const int32_t dec = m_unpack_signed(m_read<LZ>(sym, lz, __ldg(sym.cmap + ctx)));
          const int32_t val = int32_t(guess + int64_t(uint32_t(nd.w)) * int64_t(dec));  // decode/common.rs:85
          if (use_wp) wp.update(val, x, y);
          row[x] = val;
          v_prev2 = v_prev;
          v_prev = val;
          t_prev = t_cur;
          t_cur = t_next;
          t_next = t_next2;
          tt_cur = tt_next;
        }
      }
    }
    int err = 0;
    if (LZ && lz.err) err = JXG_ERR_LZ77;
    else if (sym.br.bitpos > uint64_t(st.sec_len) * 8u) err = JXG_ERR_OUT_OF_BOUNDS;
    else if (!code.use_prefix && sym.ans_state != 0x130000u) err = JXG_ERR_ANS_CHECKSUM;
    B.status[B.order[sidx]] = err;
  }
}

// rct.rs:9-40 on one triple of values; returns in (v0, v1, v2) before the permutation.
__device__ __forceinline__ void inv_rct_op(uint32_t op, int32_t& v0, int32_t& v1, int32_t& v2) {
  switch (op) {
    case 1: v2 = wadd(v2, v0); break;
    case 2: v1 = wadd(v1, v0); break;
    case 3: v1 = wadd(v1, v0); v2 = wadd(v2, v0); break;
    case 4: v1 = wadd(v1, wadd(v0, v2) >> 1); break;
    case 5: v2 = wadd(v0, v2); v1 = wadd(v1, wadd(v0, v2) >> 1); break;
    case 6: {
      int32_t y = v0;
      const int32_t co = v1, cg = v2;
      y = wsub(y, cg >> 1);
      const int32_t g = wadd(cg, y);
      y = wsub(y, co >> 1);
      const int32_t r = wadd(y, co);
      v0 = r;
      v1 = g;
      v2 = y;
      break;
    }
    default: break;
  }
}

// Local (per group) RCTs, applied in reverse order; one CTA per stream that has any.
__global__ void __launch_bounds__(256) k_modular_local_rct(const MBatchDev B) {
  const MStreamDev& st = B.streams[B.rct_streams[blockIdx.x]];
  for (uint32_t ti = st.num_rct; ti-- > 0;) {
    const MRctDev t = B.rcts[st.first_rct + ti];
    const uint32_t perm = t.type / 7, op = t.type % 7;
    const MRectDev r0 = B.rects[st.first_rect + t.begin], r1 = B.rects[st.first_rect + t.begin + 1],
                   r2 = B.rects[st.first_rect + t.begin + 2];
    const MRectDev ro[3] = {r0, r1, r2};
    const MRectDev& d0 = ro[perm % 3];
    const MRectDev& d1 = ro[(perm + 1 + perm / 3) % 3];
    const MRectDev& d2 = ro[(perm + 2 - perm / 3) % 3];
    for (uint32_t i = threadIdx.x; i < r0.w * r0.h; i += blockDim.x) {
      const uint32_t y = i / r0.w, x = i - y * r0.w;
      int32_t v0 = B.planes[r0.base + size_t(y) * r0.stride + x], v1 = B.planes[r1.base + size_t(y) * r1.stride + x],
              v2 = B.planes[r2.base + size_t(y) * r2.stride + x];
      inv_rct_op(op, v0, v1, v2);
      B.planes[d0.base + size_t(y) * d0.stride + x] = v0;
      B.planes[d1.base + size_t(y) * d1.stride + x] = v1;
      B.planes[d2.base + size_t(y) * d2.stride + x] = v2;
    }
    __syncthreads();
  }
}

// Global RCT over the job rectangle, in place (the permutation is applied by the host to the buffer ids): rows
// grid-strided over the CTAs, columns over the threads.
__global__ void __launch_bounds__(256) k_modular_rct(const MJobDev* jobs, int32_t* planes) {
  const MJobDev j = jobs[blockIdx.y];
  for (uint32_t y = j.y0 + blockIdx.x; y < j.y1; y += gridDim.x) {
    int32_t* const pa = planes + (j.a + int64_t(y) * j.sa);
    int32_t* const pb = planes + (j.b + int64_t(y) * j.sb);
    int32_t* const pc = planes + (j.c + int64_t(y) * j.sc);
    for (uint32_t x = j.x0 + threadIdx.x; x < j.x1; x += blockDim.x) {
      int32_t v0 = pa[x], v1 = pb[x], v2 = pc[x];
      inv_rct_op(j.op, v0, v1, v2);
      pa[x] = v0;
      pb[x] = v1;
      pc[x] = v2;
    }
  }
}

// squeeze.rs:144-170
__device__ __forceinline__ int64_t smooth_tendency(int64_t b, int64_t a, int64_t n) {
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

// Horizontal unsqueeze (squeeze.rs:390): one thread per output row, serial along x (each output depends on the one
// to its left). job: a = avg (w x h), b = residual (rw x h), c = out ((w + rw) x h); rows [y0, y1), output columns
// [0, x1): x1 / 2 pairs from column 0, then the tail column (the last average) when x1 is odd (x1 = w + rw).
__global__ void __launch_bounds__(128) k_unsqueeze_h(const MJobDev* jobs, int32_t* planes) {
  const MJobDev j = jobs[blockIdx.y];
  const uint32_t y = j.y0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (y >= j.y1) return;
  const uint32_t aw = j.w, pairs = j.x1 >> 1;
  const int32_t* a = planes + (j.a + int64_t(y) * j.sa);
  const int32_t* r = planes + (j.b + int64_t(y) * j.sb);
  int32_t* o = planes + (j.c + int64_t(y) * j.sc);
  int64_t av = aw ? a[0] : 0, left = av;
  for (uint32_t x = 0; x < pairs; x++) {
    const int64_t next_avg = x + 1 < aw ? a[x + 1] : av;
    const int64_t diff = int64_t(r[x]) + smooth_tendency(left, av, next_avg);
    const int64_t A = av + diff / 2;
    o[2 * x] = int32_t(A);
    left = A - diff;
    o[2 * x + 1] = int32_t(left);
    left = int32_t(left);
    av = next_avg;
  }
  if (j.x1 & 1) o[j.x1 - 1] = a[aw - 1];
}

// Vertical unsqueeze (squeeze.rs:577): one thread per column, serial along y, coalesced across x.
// job: a = avg (w x h), b = residual (w x rh), c = out (w x (h + rh)); rw holds rh. Columns [x0, x1), output rows
// [0, y1): y1 / 2 pairs from row 0, then the tail row when y1 is odd (y1 = h + rh).
__global__ void __launch_bounds__(128) k_unsqueeze_v(const MJobDev* jobs, int32_t* planes) {
  const MJobDev j = jobs[blockIdx.y];
  const uint32_t x = j.x0 + blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= j.x1) return;
  const uint32_t ah = j.h, pairs = j.y1 >> 1;
  const size_t sa = j.sa, sb = j.sb, sc = j.sc;
  const int32_t* a = planes + (j.a + x);
  const int32_t* r = planes + (j.b + x);
  int32_t* o = planes + (j.c + x);
  int64_t av = ah ? a[0] : 0, up = av;
  for (uint32_t y = 0; y < pairs; y++) {
    const int64_t next_avg = y + 1 < ah ? a[(y + 1) * sa] : av;
    const int64_t diff = int64_t(r[y * sb]) + smooth_tendency(up, av, next_avg);
    const int64_t A = av + diff / 2;
    o[(2 * y) * sc] = int32_t(A);
    up = int32_t(A - diff);
    o[(2 * y + 1) * sc] = int32_t(up);
    av = next_avg;
  }
  if (j.y1 & 1) o[(j.y1 - 1) * sc] = a[(ah - 1) * sa];
}

// ImageMetadata.orientation (headers/image_metadata.rs:85-96 display_pixel): coded pixel (x, y) of a w x h image -> its
// display position; 1 = identity.
__device__ __forceinline__ void display_pixel(uint32_t orientation, uint32_t w, uint32_t h, uint32_t x, uint32_t y,
                                              uint32_t& dx, uint32_t& dy) {
  dx = x;
  dy = y;
  switch (orientation) {
    case 2: dx = w - 1 - x; break;
    case 3: dx = w - 1 - x; dy = h - 1 - y; break;
    case 4: dy = h - 1 - y; break;
    case 5: dx = y; dy = x; break;
    case 6: dx = h - 1 - y; dy = x; break;
    case 7: dx = h - 1 - y; dy = w - 1 - x; break;
    case 8: dx = y; dy = w - 1 - x; break;
    default: break;
  }
}

// i32 planes -> interleaved RGB u8, clamped (convert.rs:675-680). job: a, b, c = R, G, B planes (w x h, the coded
// frame), op = orientation; the coded window [x0, x1) x [y0, y1) goes to the output whose top-left pixel is display
// pixel (out_x, out_y). Rows grid-strided over the CTAs, columns over the threads.
__global__ void __launch_bounds__(256) k_modular_store(const MJobDev* jobs, const int32_t* planes) {
  const MJobDev j = jobs[blockIdx.y];
  for (uint32_t y = j.y0 + blockIdx.x; y < j.y1; y += gridDim.x) {
    for (uint32_t x = j.x0 + threadIdx.x; x < j.x1; x += blockDim.x) {
      uint32_t dx, dy;
      display_pixel(j.op, j.w, j.h, x, y, dx, dy);
      uint8_t* d = static_cast<uint8_t*>(j.out) + size_t(dy - j.out_y) * j.out_stride + size_t(dx - j.out_x) * 3;
      d[0] = uint8_t(min(max(planes[j.a + int64_t(y) * j.sa + x], 0), 255));
      d[1] = uint8_t(min(max(planes[j.b + int64_t(y) * j.sb + x], 0), 255));
      d[2] = uint8_t(min(max(planes[j.c + int64_t(y) * j.sc + x], 0), 255));
    }
  }
}

// ---------------------------------------------------------------------------
// host-side launchers
// ---------------------------------------------------------------------------
template <bool LZ>
void launch_decode(const MBatchDev& B, uint32_t lanes_per_warp, uint32_t sms, cudaStream_t stream) {
  const uint32_t S = lanes_per_warp <= 1 ? 1 : (lanes_per_warp <= 2 ? 2 : 4);
  const uint32_t warps = (B.num_streams + S - 1) / S;
  const uint32_t grid = min((warps + 3) / 4, sms * 8u);
  const uint32_t total_lanes = grid * 4 * S;
  if (S == 1) k_modular_decode<1, LZ><<<grid, 128, 0, stream>>>(B, total_lanes);
  else if (S == 2) k_modular_decode<2, LZ><<<grid, 128, 0, stream>>>(B, total_lanes);
  else k_modular_decode<4, LZ><<<grid, 128, 0, stream>>>(B, total_lanes);
}

int launch_modular_decode(const MBatchDev& B, uint32_t num_plain, uint32_t lanes_per_warp, uint32_t num_rct_streams,
                          uint32_t sms, cudaStream_t stream) {
  int launches = 0;
  if (B.num_streams) cudaMemsetAsync(B.queue, 0, 2 * sizeof(uint32_t), stream);
  if (num_plain) {
    MBatchDev P = B;
    P.num_streams = num_plain;
    launch_decode<false>(P, lanes_per_warp, sms, stream);
    launches++;
  }
  if (B.num_streams > num_plain) {  // longest first among the LZ77 streams too, with their own queue counter
    MBatchDev L = B;
    L.order = B.order + num_plain;
    L.num_streams = B.num_streams - num_plain;
    L.queue = B.queue + 1;
    launch_decode<true>(L, lanes_per_warp, sms, stream);
    launches++;
  }
  if (num_rct_streams) {
    k_modular_local_rct<<<num_rct_streams, 256, 0, stream>>>(B);
    launches++;
  }
  return launches;
}

// transforms/palette.rs:17-163 get_palette_value for 8-bit samples: explicit entries, the implicit 4x4x4 and 5x5x5
// colour cubes behind them, the 72-entry delta table for negative indices.
__constant__ int16_t c_palette_delta[72][3] = {
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

__device__ __forceinline__ int32_t palette_value8(const int32_t* pal, uint32_t pal_stride, int32_t index, uint32_t c, uint32_t palette_size) {
  if (index < 0) {
    if (c >= 3) return 0;
    uint32_t idx = uint32_t(-(int64_t(index) + 1));
    idx %= 1 + 2 * (72 - 1);
    const int32_t d = c_palette_delta[(idx + 1) >> 1][c];
    return (idx & 1) ? d : -d;
  }
  uint32_t idx = uint32_t(index);
  if (idx >= palette_size && idx < palette_size + 64) {  // small cube
    if (c >= 3) return 0;
    idx -= palette_size;
    idx >>= c * 2;
    return int32_t(((idx % 4) * 255u) >> 2) + 32;
  }
  if (idx >= palette_size + 64) {  // large cube
    if (c >= 3) return 0;
    idx -= palette_size + 64;
    if (c == 1) idx /= 5;
    if (c == 2) idx /= 25;
    return int32_t(((idx % 5) * 255u) >> 2);
  }
  return pal[size_t(c) * pal_stride + idx];
}

// Inverse palette without delta entries (palette.rs:165-199): out[c][p] = palette_value(index[p], c) over the job
// rectangle. One job per colour channel (blockIdx.y); rows grid-strided over the CTAs, columns over the threads. The
// palette plane b is held whole: row c = component c.
__global__ void __launch_bounds__(256) k_modular_palette(const MJobDev* jobs, int32_t* planes) {
  const MJobDev j = jobs[blockIdx.y];
  const int32_t* pal = planes + j.b;
  for (uint32_t y = j.y0 + blockIdx.x; y < j.y1; y += gridDim.x) {
    const int32_t* index = planes + (j.a + int64_t(y) * j.sa);
    int32_t* out = planes + (j.c + int64_t(y) * j.sc);
    for (uint32_t x = j.x0 + threadIdx.x; x < j.x1; x += blockDim.x) out[x] = palette_value8(pal, j.sb, index[x], j.op, j.rw);
  }
}

// ---------------------------------------------------------------------------
// Thumbnail jobs: the LF image of a VarDCT frame (modular/mod.rs:837-982, adaptive_lf_smoothing.rs:44-125) and its
// store. The host computes the same values with scalar float code compiled without contraction: every operation here
// is the correctly rounded one of the host, in the host's order.
// ---------------------------------------------------------------------------

// dequant_lf_rect (frame.cc) on one LF group's rectangle: quantised Y, X, B at a -> X, Y, B at c.
__global__ void __launch_bounds__(256) k_lf_dequant(const MJobDev* jobs, int32_t* planes, const uint8_t* blob) {
  const MJobDev j = jobs[blockIdx.y];
  const MLfDequantDev p = *reinterpret_cast<const MLfDequantDev*>(blob + j.params);
  const size_t plane = size_t(j.sa) * j.h;
  const int32_t* qy = planes + j.a;
  const int32_t* qx = qy + plane;
  const int32_t* qb = qx + plane;
  float* out = reinterpret_cast<float*>(planes + j.c);
  for (uint32_t y = j.y0 + blockIdx.x; y < j.y1; y += gridDim.x) {
    for (uint32_t x = j.x0 + threadIdx.x; x < j.x1; x += blockDim.x) {
      const size_t i = size_t(y) * j.sa + x;
      const float in_x = __fmul_rn(float(qx[i]), p.fac[0]), in_y = __fmul_rn(float(qy[i]), p.fac[1]),
                  in_b = __fmul_rn(float(qb[i]), p.fac[2]);
      out[i] = __fadd_rn(__fmul_rn(in_y, p.cfl_x), in_x);
      out[plane + i] = in_y;
      out[2 * plane + i] = __fadd_rn(__fmul_rn(in_y, p.cfl_b), in_b);
    }
  }
}

// adaptive_lf_smoothing (frame.cc smooth_band's scalar loop) of the whole LF image, X, Y, B at a -> c; border samples
// and images of at most two rows or columns are copied.
__global__ void __launch_bounds__(256) k_lf_smooth(const MJobDev* jobs, int32_t* planes, const uint8_t* blob) {
  const MJobDev j = jobs[blockIdx.y];
  const MLfFrameDev& p = *reinterpret_cast<const MLfFrameDev*>(blob + j.params);
  const size_t plane = size_t(j.sa) * j.h;
  const float* in = reinterpret_cast<const float*>(planes + j.a);
  float* out = reinterpret_cast<float*>(planes + j.c);
  const float kSide = 0.20345139757231578f, kCorner = 0.0334829185968739f;
  const float kCenter = __fsub_rn(1.0f, __fmul_rn(4.0f, __fadd_rn(kSide, kCorner)));
  const bool smooth = j.w > 2 && j.h > 2;
  for (uint32_t y = blockIdx.x; y < j.h; y += gridDim.x) {
    for (uint32_t x = threadIdx.x; x < j.w; x += blockDim.x) {
      const size_t i = size_t(y) * j.sa + x;
      if (!smooth || x == 0 || y == 0 || x + 1 == j.w || y + 1 == j.h) {
        for (int c = 0; c < 3; c++) out[c * plane + i] = in[c * plane + i];
        continue;
      }
      float gap = 0.5f, mc[3], sm[3];
      for (int c = 0; c < 3; c++) {
        const float* m = in + c * plane + i;
        const float* t = m - j.sa;
        const float* b = m + j.sa;
        const float corner = __fadd_rn(__fadd_rn(__fadd_rn(t[-1], t[1]), b[-1]), b[1]);
        const float side = __fadd_rn(__fadd_rn(__fadd_rn(m[-1], m[1]), t[0]), b[0]);
        mc[c] = m[0];
        sm[c] = __fadd_rn(__fadd_rn(__fmul_rn(corner, kCorner), __fmul_rn(side, kSide)), __fmul_rn(mc[c], kCenter));
        const float d = fabsf(__fdiv_rn(__fsub_rn(mc[c], sm[c]), p.lf_factors[c]));
        gap = gap < d ? d : gap;  // std::max(gap, d)
      }
      const float f = __fsub_rn(3.0f, __fmul_rn(4.0f, gap));
      const float factor = f < 0.0f ? 0.0f : f;  // std::max(f, 0.0f)
      for (int c = 0; c < 3; c++) out[c * plane + i] = __fadd_rn(__fmul_rn(__fsub_rn(sm[c], mc[c]), factor), mc[c]);
    }
  }
}

// XYB samples -> an output through the output stage of the full decode's store (output_stage.h): the u8 dither at the
// coded coordinate of the w x h image, then the orientation (op); the coded window [x0, x1) x [y0, y1) goes to the
// output whose top-left pixel is display pixel (out_x, out_y). XYB_F32_PLANAR writes the window's planes in the coded
// orientation, plane c from row c * (y1 - y0). Rows grid-strided over the CTAs, columns over the threads. The input:
// * kModularXyb false (kJobLfStore, a thumbnail): the f32 planes X, Y, B at a, a + sa * h, a + 2 * sa * h;
// * kModularXyb true (kJobXybStore, an XYB Modular frame): the i32 channels Y at a, X at b, B at c (strides sa, sb,
//   sc), converted as ConvertModularXYBToF32Stage (render/stages/convert.rs:278-343) does with the LfQuantFactors in
//   p.lf_factors: X = x s_x, Y = y s_y, B = (b + y) s_b, each operation on f32 and correctly rounded.
template <bool kModularXyb>
__global__ void __launch_bounds__(256) k_xyb_store(const MJobDev* jobs, const int32_t* planes, const uint8_t* blob) {
  const MJobDev j = jobs[blockIdx.y];
  const MLfFrameDev& p = *reinterpret_cast<const MLfFrameDev*>(blob + j.params);
  const size_t plane = size_t(j.sa) * j.h;
  uint8_t* const out = static_cast<uint8_t*>(j.out);
  for (uint32_t y = j.y0 + blockIdx.x; y < j.y1; y += gridDim.x) {
    for (uint32_t x = j.x0 + threadIdx.x; x < j.x1; x += blockDim.x) {
      float xyb[3];
      if (kModularXyb) {
        const float qy = float(planes[j.a + int64_t(y) * j.sa + x]), qx = float(planes[j.b + int64_t(y) * j.sb + x]),
                    qb = float(planes[j.c + int64_t(y) * j.sc + x]);
        xyb[0] = __fmul_rn(qx, p.lf_factors[0]);
        xyb[1] = __fmul_rn(qy, p.lf_factors[1]);
        xyb[2] = __fmul_rn(__fadd_rn(qb, qy), p.lf_factors[2]);
      } else {
        const float* in = reinterpret_cast<const float*>(planes + j.a) + size_t(y) * j.sa + x;
        for (int c = 0; c < 3; c++) xyb[c] = in[c * plane];
      }
      if (p.output_format == JXG_FORMAT_XYB_F32_PLANAR) {
        for (int c = 0; c < 3; c++)
          reinterpret_cast<float*>(out + (size_t(c) * (j.y1 - j.y0) + (y - j.y0)) * j.out_stride)[x - j.x0] = xyb[c];
        continue;
      }
      float v[3];
      xyb_to_output(p, xyb[0], xyb[1], xyb[2], v);
      uint32_t dx, dy;
      display_pixel(j.op, j.w, j.h, x, y, dx, dy);
      dx -= j.out_x;
      uint8_t* const row = out + size_t(dy - j.out_y) * j.out_stride;
      switch (p.output_format) {
        case JXG_FORMAT_RGB_F32:
          for (int c = 0; c < 3; c++) reinterpret_cast<float*>(row)[size_t(dx) * 3 + c] = v[c];
          break;
        case JXG_FORMAT_RGB_U16:
        case JXG_FORMAT_RGB_F16:
          for (int c = 0; c < 3; c++) reinterpret_cast<uint16_t*>(row)[size_t(dx) * 3 + c] = sample16(p, v[c]);
          break;
        default: {  // RGB_U8, RGBA_U8
          const uint32_t bpp = p.output_format == JXG_FORMAT_RGBA_U8 ? 4 : 3;
          uint8_t* d = row + size_t(dx) * bpp;
          for (int c = 0; c < 3; c++) d[c] = sample8(v[c], int(x), int(y), c);
          if (bpp == 4) d[3] = 255;
        }
      }
    }
  }
}

void launch_modular_jobs(int kind, const MJobDev* jobs, uint32_t num_jobs, uint32_t max_w, uint32_t max_h, int32_t* planes,
                         const uint8_t* blob, uint32_t sms, cudaStream_t stream) {
  if (!num_jobs) return;
  const uint32_t rows = max(min(max_h, sms * 16), 1u);  // grid of the row-strided kernels
  if (kind == 0) {
    k_modular_rct<<<dim3(rows, num_jobs), 256, 0, stream>>>(jobs, planes);
  } else if (kind == 1) {  // a level can hold only empty channels (a squeeze of a zero-height residual): one idle block
    k_unsqueeze_h<<<dim3(max((max_h + 127) / 128, 1u), num_jobs), 128, 0, stream>>>(jobs, planes);
  } else if (kind == 2) {
    k_unsqueeze_v<<<dim3(max((max_w + 127) / 128, 1u), num_jobs), 128, 0, stream>>>(jobs, planes);
  } else if (kind == 4) {
    k_modular_palette<<<dim3(rows, num_jobs), 256, 0, stream>>>(jobs, planes);
  } else if (kind == 5) {
    k_lf_dequant<<<dim3(rows, num_jobs), 256, 0, stream>>>(jobs, planes, blob);
  } else if (kind == 6) {
    k_lf_smooth<<<dim3(rows, num_jobs), 256, 0, stream>>>(jobs, planes, blob);
  } else if (kind == 7) {
    k_xyb_store<false><<<dim3(rows, num_jobs), 256, 0, stream>>>(jobs, planes, blob);
  } else if (kind == 8) {
    k_xyb_store<true><<<dim3(rows, num_jobs), 256, 0, stream>>>(jobs, planes, blob);
  } else {
    k_modular_store<<<dim3(rows, num_jobs), 256, 0, stream>>>(jobs, planes);
  }
}

}  // namespace jxgpu
