// sm_90a kernels of the VarDCT hot path.
//
//   k_block_plan     K0  varblock descriptors of every (frame, group) stream, the block order of all three entropy kernels
//   k_entropy_lean   K1  decode of the AC coefficients with the JPEG XL context model (jxl/src/frame/group.rs:454-578,
//   k_entropy_fast       entropy_coding/*.rs): persistent lanes for single-pass ANS frames (lean), packed lanes for
//   k_entropy            prefix-coded or shifted single-pass frames (fast), one lane per warp for multi-pass and LZ77 frames
//   k_idct_small     K2  one CTA per group: dequant + chroma-from-luma + LLF + inverse variable-block DCT
//   k_dequant_idct       (group.rs:100-250, jxl_transforms/src/transform.rs); each kernel walks the varblocks of its
//                        transform classes in the block plan's partition
//   k_filters_store  K3-K5 fused Gaborish -> EPF 0/1/2 -> XYB -> output transfer curve -> store
//                    (render/stages/{gaborish,epf/*,xyb,from_linear,convert}.rs, color/tf.rs)
//   k_orient         orientation post-pass of frames with orientation != 1
//   k_expand_coeffs  coefficient lists -> dense layout (jxg_batch_read_coeffs)
//
// No tensor cores: there is no dense contraction on this path; everything is
// HBM / latency bound integer and f32 work.
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "../../../include/jxg.h"
#include "device_types.h"
#include "output_stage.h"
#include "../host/region.h"

namespace jxgpu {

__constant__ float c_wc[9][128];       // 1 / (2 cos((i + 0.5) pi / n)), n = 2^l
__constant__ float c_rdct_scale[6][32];  // reinterpreting-DCT output scales (6 decimals)
__constant__ uint8_t c_cov_x[27] = {1, 1, 1, 1, 2, 4, 1, 2, 1, 4, 2, 4, 1, 1, 1, 1, 1, 1, 8, 4, 8, 16, 8, 16, 32, 16, 32};
__constant__ uint8_t c_cov_y[27] = {1, 1, 1, 1, 2, 4, 2, 1, 4, 1, 4, 2, 1, 1, 1, 1, 1, 1, 8, 8, 4, 16, 16, 8, 32, 32, 16};
__constant__ uint8_t c_shape[27] = {0, 1, 1, 1, 2, 3, 4, 4, 5, 5, 6, 6, 1, 1, 1, 1, 1, 1, 7, 8, 8, 9, 10, 10, 11, 12, 12};
__constant__ uint8_t c_qtable[27] = {0, 1, 2, 3, 4, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 10, 10, 11, 12, 12, 13, 14, 14, 15, 16, 16};
// block_context_map.rs:20-31
__constant__ uint16_t c_freq_ctx[64] = {0xBAD, 0,  1,  2,  3,  4,  5,  6,  7,  8,  9,  10, 11, 12, 13, 14, 15, 15, 16, 16, 17, 17,
                                        18,    18, 19, 19, 20, 20, 21, 21, 22, 22, 23, 23, 23, 23, 24, 24, 24, 24, 25, 25, 25, 25,
                                        26,    26, 26, 26, 27, 27, 27, 27, 28, 28, 28, 28, 29, 29, 29, 29, 30, 30, 30, 30};
__constant__ uint16_t c_nz_ctx[64] = {0xBAD, 0,   31,  62,  62,  93,  93,  93,  93,  123, 123, 123, 123, 152, 152, 152,
                                      152,   152, 152, 152, 152, 180, 180, 180, 180, 180, 180, 180, 180, 180, 180, 180,
                                      180,   206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206,
                                      206,   206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206};
__constant__ float c_afv[256] = {
#include "afv_basis.inc"
};
// The dither table of output_stage.h in global memory: the vector store path indexes it with per-lane (x, y), which the
// constant cache would serialise; consecutive lanes read consecutive words here.
__device__ float g_dither[1024] = {
#include "dither_table.inc"
};

// ===========================================================================
// K1: entropy decode
// ===========================================================================

// The symbol reader of k_entropy_fast and k_entropy: bit reader, token step (ANS alias bucket or two-level prefix table)
// and hybrid uint, over the table formats of PassDev. k_entropy_lean reads the same formats with its own fused per-symbol
// step: the speculative context look-ups and the register bit window are its measured form (DESIGN §3).
struct LaneBr {  // 32-bit window bit reader (bit_reader.rs semantics: zeros past the end, checked at the end)
  const uint32_t* words;
  uint32_t nwords, bitpos, ci, lo, hi;
  __device__ __forceinline__ uint32_t ldw(uint32_t i) const { return i < nwords ? __ldg(words + i) : 0u; }
  __device__ __forceinline__ void init(const uint8_t* p, uint32_t len) {
    words = reinterpret_cast<const uint32_t*>(p);
    nwords = (len + 3) >> 2;
    bitpos = 0;
    ci = 0;
    lo = ldw(0);
    hi = ldw(1);
  }
  __device__ __forceinline__ uint32_t peek32() const { return __funnelshift_r(lo, hi, bitpos & 31); }
  __device__ __forceinline__ uint32_t peek(uint32_t n) const {  // n <= 31
    return peek32() & ((1u << n) - 1u);
  }
  __device__ __forceinline__ void skip(uint32_t n) {  // n <= 32
    const uint32_t nb = bitpos + n;
    if ((nb >> 5) != ci) {
      ci++;
      lo = hi;
      hi = ldw(ci + 1);
    }
    bitpos = nb;
  }
};

constexpr uint32_t kCfg420 = 4u | (2u << 8) | (0u << 16);  // hybrid_uint.rs:60-65

__device__ __forceinline__ uint32_t lane_hybrid(uint32_t cfg, uint32_t token, LaneBr& br) {
  if (cfg == kCfg420) {  // hybrid_uint.rs:67-80 (read_config_420)
    if (token < 16) return token;
    const uint32_t nbits = ((token >> 2) - 2) & 31;
    const uint32_t bits = br.peek(nbits);
    br.skip(nbits);
    return (((token & 3) | 4) << nbits) | bits;
  }
  const uint32_t split_exponent = cfg & 0xff, msb = (cfg >> 8) & 0xff, lsb = (cfg >> 16) & 0xff;
  const uint32_t split_token = 1u << split_exponent;
  if (token < split_token) return token;
  const uint32_t bits_in_token = lsb + msb;
  const uint32_t nbits = (split_exponent - bits_in_token + ((token - split_token) >> bits_in_token)) & 31;
  const uint32_t low = token & ((1u << lsb) - 1);
  const uint32_t token_nolow = token >> lsb;
  const uint32_t bits = br.peek(nbits);
  br.skip(nbits);
  const uint32_t hi = (token_nolow & ((1u << msb) - 1)) | (1u << msb);
  return (((hi << nbits) | bits) << lsb) | low;
}

struct PassState {
  LaneBr br;
  uint32_t ans_state;
  uint32_t hist_idx;
  // LZ77 (decode.rs:86-146): window of the symbols decoded so far (linear, see kLzWindow), pending copy
  uint32_t* lz_win;
  uint32_t lz_to_copy, lz_copy_pos, lz_decoded, lz_err;
};

struct PassTables {
  const uint8_t* context_map;
  const uint32_t* uint_configs;
  const uint2* ans;  // 8-byte buckets
  const uint32_t* huff;
  const uint32_t* huff_offset;
  uint32_t use_prefix, log_alpha_size;
  uint32_t lz_enabled, lz_min_symbol, lz_min_length, lz_len_cfg, lz_dist_cluster;
};

// ans.rs:356-393 / huffman.rs:446-457
__device__ __forceinline__ uint32_t lane_token(const PassTables& T, PassState& s, uint32_t cluster) {
  LaneBr& br = s.br;
  if (T.use_prefix) {
    const uint32_t* tb = T.huff + __ldg(T.huff_offset + cluster);
    uint32_t p = br.peek(8);
    uint32_t e = __ldg(tb + p);
    uint32_t n_bits = e & 0xff;
    if (n_bits > 8) {
      br.skip(8);
      n_bits -= 8;
      p += e >> 16;
      p += br.peek(n_bits);
      e = __ldg(tb + p);
    }
    br.skip(e & 0xff);
    return e >> 16;
  }
  const uint32_t log_bucket = 12 - T.log_alpha_size;
  const uint32_t idx = s.ans_state & 0xfff;
  const uint32_t i = idx >> log_bucket, p = idx & ((1u << log_bucket) - 1u);
  const uint2 b = __ldg(T.ans + ((cluster << T.log_alpha_size) + i));
  const bool alias = p >= ((b.x >> 8) & 0xff);
  const uint32_t dist = (b.x >> 16) ^ (alias ? (b.y >> 16) : 0u);
  const uint32_t offset = p + (alias ? (b.y & 0xffff) : 0u);
  uint32_t next = (s.ans_state >> 12) * dist + offset;
  if (next < (1u << 16)) {
    next = (next << 16) | br.peek(16);
    br.skip(16);
  }
  s.ans_state = next;
  return alias ? (b.x & 0xff) : i;
}

// One symbol of a stream without LZ77.
__device__ __forceinline__ uint32_t lane_symbol(const PassTables& T, PassState& s, uint32_t ctx) {
  const uint32_t cluster = __ldg(T.context_map + ctx);
  const uint32_t tok = lane_token(T, s, cluster);
  return lane_hybrid(__ldg(T.uint_configs + cluster), tok, s.br);
}

// decode.rs:286-330 with dist_multiplier == 0 (HF streams create their reader without an image width, group.rs:345-349).
// Inlined: behind a call the stream state would live in local memory on k_entropy's per-symbol path.
__device__ __forceinline__ uint32_t read_symbol_lz77(const PassTables& T, PassState& s, uint32_t ctx) {
  auto push = [&](uint32_t sym) {
    s.lz_win[min(s.lz_decoded, kLzWindow - 1)] = sym;
    s.lz_decoded++;
    return sym;
  };
  if (s.lz_to_copy) {  // pull_symbol
    s.lz_to_copy--;
    return push(s.lz_win[min(s.lz_copy_pos++, kLzWindow - 1)]);
  }
  const uint32_t cluster = __ldg(T.context_map + ctx);
  const uint32_t tok = lane_token(T, s, cluster);
  if (tok < T.lz_min_symbol) return push(lane_hybrid(__ldg(T.uint_configs + cluster), tok, s.br));
  if (s.lz_decoded == 0) {  // a copy before anything was decoded (errors.lz77_repeat)
    s.lz_err = 1;
    return 0;
  }
  const uint32_t n = lane_hybrid(T.lz_len_cfg, tok - T.lz_min_symbol, s.br);
  if (n > 0xffffffffu - T.lz_min_length) {
    s.lz_err = 1;
    return 0;
  }
  const uint32_t dtok = lane_token(T, s, T.lz_dist_cluster);
  const uint32_t dsym = lane_hybrid(__ldg(T.uint_configs + T.lz_dist_cluster), dtok, s.br);
  const uint32_t distance = min(min(dsym, (1u << 20) - 1u) + 1u, s.lz_decoded);  // apply_copy, decode.rs:111-124
  s.lz_copy_pos = s.lz_decoded - distance;
  s.lz_to_copy = n + T.lz_min_length - 1;  // the first copied symbol is returned right away
  return push(s.lz_win[min(s.lz_copy_pos++, kLzWindow - 1)]);
}

__device__ __forceinline__ uint32_t read_symbol(const PassTables& T, PassState& s, uint32_t ctx) {
  return T.lz_enabled ? read_symbol_lz77(T, s, ctx) : lane_symbol(T, s, ctx);
}

__device__ __forceinline__ int32_t unpack_signed(uint32_t u) { return int32_t((u >> 1) ^ (((~u) & 1u) - 1u)); }

// One coefficient list (device_types.h): base of the entries, offset words behind them.
__device__ __forceinline__ uint32_t* list_base(const BatchDev& B, uint32_t section) { return B.nzlist + size_t(section) * kListStride; }
// Writer side: the entry of coefficient value v at position pos of a varblock with 2^lnc coefficients per channel is
// stored at the cursor whatever v is; the cursor only moves for v != 0 (branch-free; a zero is overwritten by the next
// entry or stays behind the end of the channel). `ovf` collects values that do not fit the entry.
__device__ __forceinline__ void list_put(uint32_t* base, uint32_t& n, uint32_t pos, int32_t v, uint32_t lnc, uint32_t& ovf) {
  const int32_t sv = int32_t(uint32_t(v) << lnc);
  ovf |= uint32_t((sv >> lnc) ^ v);
  base[n] = pos | uint32_t(sv);
  n += v != 0 ? 1u : 0u;
}
__device__ __forceinline__ uint32_t entry_pos(uint32_t e, uint32_t lnc) { return e & ((1u << lnc) - 1u); }
__device__ __forceinline__ int32_t entry_value(uint32_t e, uint32_t lnc) { return int32_t(e) >> lnc; }

// ---- bulk asynchronous copies (TMA engine, 1-D form) + mbarrier: global -> shared without passing through registers ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t arrivals) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(arrivals) : "memory");
}
__device__ __forceinline__ void mbar_fence_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
// One thread: announce `bytes` of asynchronous traffic on the barrier, then start the copy that will deliver them.
// src, dst and bytes are multiples of 16.
__device__ __forceinline__ void bulk_load(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile("{\n.reg .pred p;\nmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\nselp.u32 %0, 1, 0, p;\n}"
                 : "=r"(done)
                 : "r"(smem_u32(bar)), "r"(parity)
                 : "memory");
  } while (!done);
}

// Prefix of a stream's pass-0 coefficient list staged in shared memory by bulk copies (k_idct_small): the offset words
// of all varblocks and the first `staged` entries; entries beyond that, and other passes, are read from global memory.
struct ListStage {
  const uint32_t* off;  // nullptr: nothing staged
  const uint32_t* ent;
  uint32_t staged;
};

// Non-zero count predicted for a channel's varblock at (bx, by) from the column bytes of the channel (group.rs:489-505).
// Varblocks are visited in raster order of their top-left corner (the block plan's order), so the last count written to
// a column is the one of the block right above the current row, and for column bx - 1 the one of the block to the left.
__device__ __forceinline__ uint32_t predict_nz(const uint8_t* col, uint32_t bx, uint32_t by) {
  if (bx == 0) return by == 0 ? 32u : col[0];
  if (by == 0) return col[bx - 1];
  return (uint32_t(col[bx]) + uint32_t(col[bx - 1]) + 1u) >> 1;
}

// One varblock (descriptor d of k_block_plan), one pass: the three channels in Y, X, B order (group.rs:509-577).
__device__ __forceinline__ int decode_block_pass(const BatchDev& B, const FrameDev& F, const PassDev& P,
                                                 const PassTables& T, PassState& s, const uint4 d,
                                                 uint8_t* nzcol /* [3][32] */, uint32_t* list, uint32_t& nlist, uint32_t bi,
                                                 uint32_t& ovf) {
  const uint32_t context_offset = s.hist_idx * F.num_block_contexts * (37 + 458);
  const uint32_t bx = d.x & 31, by = (d.x >> 5) & 31, cx = (d.x >> 10) & 63, shape = (d.x >> 22) & 15, lnb = d.x >> 26;
  const uint32_t num_blocks = 1u << lnb, num_coeffs = num_blocks * 64;
#pragma unroll 1
  for (int ci = 0; ci < 3; ci++) {
    const int c = ci == 0 ? 1 : (ci == 1 ? 0 : 2);
    uint8_t* col = nzcol + c * 32;
    const uint32_t predicted = predict_nz(col, bx, by);
    const uint32_t block_context = (d.y >> (8 * ci)) & 0xff;
    uint32_t nzc = predicted < 8 ? predicted : (predicted < 64 ? 4 + predicted / 2 : 36);
    uint32_t nonzeros = read_symbol(T, s, nzc * F.num_block_contexts + block_context + context_offset);
    if (nonzeros + num_blocks > num_coeffs) return JXG_ERR_INVALID_NUM_NONZEROS;
    const uint8_t nzv = uint8_t((nonzeros + num_blocks - 1) >> lnb);
    for (uint32_t ix = 0; ix < cx; ix++) col[bx + ix] = nzv;
    const uint32_t histo_offset = F.num_block_contexts * 37 + 458 * block_context + context_offset;
    uint32_t prev = nonzeros > num_coeffs / 16 ? 0u : 1u;
    const uint32_t* order = P.custom_orders
                                ? reinterpret_cast<const uint32_t*>(B.blob + P.order_off) + P.order_offset[shape * 3 + c]
                                : B.natural_orders + B.natural_order_off[shape];
    list[kOffBase + bi * 3 + ci] = nlist;  // first entry of channel ci (Y, X, B) of this varblock in this pass
    const uint32_t rnd = num_blocks - 1;
#pragma unroll 1
    for (uint32_t k = num_blocks; k < num_coeffs && nonzeros != 0; k++) {
      uint32_t ctx = histo_offset + (uint32_t(c_nz_ctx[((nonzeros + rnd) >> lnb) & 63]) + uint32_t(c_freq_ctx[(k >> lnb) & 63])) * 2 + prev;
      uint32_t u = read_symbol(T, s, ctx);
      int32_t coeff = int32_t(uint32_t(unpack_signed(u)) << P.shift);
      prev = coeff != 0;
      nonzeros -= prev;
      list_put(list, nlist, __ldg(order + k), coeff, lnb + 6, ovf);
    }
    if (nonzeros != 0) return JXG_ERR_RESIDUAL_NONZEROS;
  }
  return 0;
}

__device__ __forceinline__ PassTables make_tables(const BatchDev& B, const PassDev& P) {
  PassTables T;
  T.context_map = B.blob + P.code.cmap_off;
  T.uint_configs = reinterpret_cast<const uint32_t*>(B.blob + P.code.cfg_off);
  T.ans = reinterpret_cast<const uint2*>(B.blob + P.code.ans_off);
  T.huff = reinterpret_cast<const uint32_t*>(B.blob + P.code.huff_off);
  T.huff_offset = reinterpret_cast<const uint32_t*>(B.blob + P.code.huff_offset_off);
  T.use_prefix = P.code.use_prefix;
  T.log_alpha_size = P.code.log_alpha;
  T.lz_enabled = P.code.lz_enabled;
  T.lz_min_symbol = P.code.lz_min_symbol;
  T.lz_min_length = P.code.lz_min_length;
  T.lz_len_cfg = P.code.lz_len_cfg;
  T.lz_dist_cluster = P.code.lz_dist_cluster;
  return T;
}

__device__ __forceinline__ int init_pass(const BatchDev& B, const FrameDev& F, uint32_t pass, uint32_t g, PassState& s) {
  const SectionDev sec = B.sections[F.section_base + pass * F.num_groups + g];
  s.br.init(B.blob + sec.off, sec.len);
  uint32_t nb = 0;
  while ((1u << nb) < F.num_histograms) nb++;
  s.hist_idx = s.br.peek(nb);  // group.rs:333-341
  s.br.skip(nb);
  if (s.hist_idx >= F.num_histograms) return JXG_ERR_INVALID_HISTOGRAM_INDEX;
  s.ans_state = 0x130000u;
  if (!F.passes[pass].code.use_prefix) {  // ans.rs:431
    s.ans_state = s.br.peek32();
    s.br.skip(32);
  }
  s.lz_win = F.has_lz ? B.lzwin + size_t(F.lz_win_base + pass * F.num_groups + g) * kLzWindow : nullptr;
  s.lz_to_copy = s.lz_copy_pos = s.lz_decoded = s.lz_err = 0;
  return 0;
}

// check_final_state (decode.rs:400)
__device__ __forceinline__ int finish_pass(const BatchDev& B, const FrameDev& F, uint32_t pass, uint32_t g, const PassState& s) {
  const SectionDev sec = B.sections[F.section_base + pass * F.num_groups + g];
  if (s.lz_err) return JXG_ERR_LZ77;
  if (s.br.bitpos > sec.len * 8u) return JXG_ERR_OUT_OF_BOUNDS;                         // bit_reader.rs:109
  if (!F.passes[pass].code.use_prefix && s.ans_state != 0x130000u) return JXG_ERR_ANS_CHECKSUM;  // ans.rs:441
  return 0;
}

constexpr int kEntropyWarps = 4;

// K1 slow path (multi-pass and LZ77 frames): one lane per warp and stream, the varblocks of the block plan in order,
// each through all passes.
__global__ void __launch_bounds__(kEntropyWarps * 32) k_entropy(const BatchDev B) {
  // non-zero counts by column (see predict_nz), one set per pass: group.rs keeps one count per pass
  __shared__ uint8_t s_nzcol[kEntropyWarps][kMaxPasses][3 * 32];
  const uint32_t warp = threadIdx.x >> 5;
  const uint32_t slow_idx = blockIdx.x * kEntropyWarps + warp;
  if (slow_idx >= B.num_slow || (threadIdx.x & 31) != 0) return;
  const StreamDev sd = B.streams_slow[slow_idx];
  const FrameDev& F = B.frames[sd.frame];
  const uint32_t g = sd.group;
  const uint32_t stream = F.first_stream + g;
  const uint32_t nblk = B.nblk[stream];
  if (nblk == 0xffffffffu) {  // the block plan failed: invalid or overlapping varblocks
    B.status[stream] = JXG_ERR_INVALID_TRANSFORM;
    return;
  }
  const uint4* desc = B.desc + size_t(stream) * 1024;
  const uint32_t np = F.num_passes;
  int err = 0;
  // one coefficient list per pass (section = pass * num_groups + group); the transform kernels add the passes up
  PassState st[kMaxPasses];
  uint32_t nlist[kMaxPasses];
  for (uint32_t p = 0; p < np; p++) nlist[p] = 0;
  uint32_t ovf = 0;
  for (uint32_t p = 0; p < np && !err; p++) err = init_pass(B, F, p, g, st[p]);
  for (uint32_t bi = 0; bi < nblk && !err; bi++) {
    const uint4 d = __ldg(desc + bi);
    for (uint32_t p = 0; p < np && !err; p++) {
      PassState s = st[p];
      const PassTables T = make_tables(B, F.passes[p]);
      const uint32_t section = F.section_base + p * F.num_groups + g;
      uint32_t n = nlist[p];
      err = decode_block_pass(B, F, F.passes[p], T, s, d, s_nzcol[warp][p], list_base(B, section), n, bi, ovf);
      nlist[p] = n;
      st[p] = s;
    }
  }
  for (uint32_t p = 0; p < np && !err; p++) {
    list_base(B, F.section_base + p * F.num_groups + g)[kOffBase + nblk * 3] = nlist[p];
    err = finish_pass(B, F, p, g, st[p]);
  }
  if (!err && ovf) err = JXG_ERR_UNSUPPORTED;  // a coefficient beyond the entry width (device_types.h)
  B.status[stream] = err;
}

// ---------------------------------------------------------------------------
// K1 fast path (single-pass frames that are prefix coded or shifted): S streams per warp, one lane per stream,
// the decode loop written as a small state machine so that the lanes of a warp stay converged on the common
// "decode one symbol" body. A stream's symbols are strictly serial (one rANS state, contexts depend on the previous
// values), so throughput comes from packing independent streams: S is chosen by the host so that the grid is about
// one resident wave of warps.
// ---------------------------------------------------------------------------
template <int S>
__global__ void __launch_bounds__(128, 8) k_entropy_fast(const BatchDev B) {
  __shared__ uint16_t s_nz_ctx[64], s_freq_ctx[64];
  __shared__ uint8_t s_nzcol[4 * S][3 * 32];  // per lane: non-zero counts by column (see predict_nz)
  if (threadIdx.x < 64) {
    s_nz_ctx[threadIdx.x] = c_nz_ctx[threadIdx.x];
    s_freq_ctx[threadIdx.x] = c_freq_ctx[threadIdx.x];
  }
  __syncthreads();
  const uint32_t warp = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  const uint32_t sidx = warp * S + lane;
  bool done = !(lane < S && sidx < B.num_fast);
  // per-lane stream state (dummy but valid values for idle lanes)
  const StreamDev sd = done ? StreamDev{0, 0} : B.streams_fast[sidx];
  const FrameDev& F = B.frames[sd.frame];
  const uint32_t g = sd.group;
  const uint32_t gsid = F.first_stream + g;
  uint32_t* const list = list_base(B, F.section_base + g);  // single pass: list of section `group`
  uint32_t nlist = 0, ovf = 0;
  uint8_t* const nz = s_nzcol[(threadIdx.x >> 5) * S + (lane < S ? lane : 0)];
  const uint4* const desc = B.desc + size_t(gsid) * 1024;
  const uint32_t nblk = done ? 0u : B.nblk[gsid];
  const PassDev& P = F.passes[0];
  const PassTables T = make_tables(B, P);
  const uint32_t shift = P.shift;
  const uint32_t nbc = F.num_block_contexts;
  PassState s;
  uint32_t context_offset = 0;
  if (!done) {
    // nblk == 0xffffffff: the block plan failed (invalid or overlapping varblocks)
    const int err = nblk == 0xffffffffu ? JXG_ERR_INVALID_TRANSFORM : init_pass(B, F, 0, g, s);
    if (err) {
      B.status[gsid] = err;
      done = true;
    } else {
      context_offset = s.hist_idx * nbc * (37 + 458);
    }
  }
  enum { PH_BLOCK = 0, PH_NNZ = 1, PH_COEF = 2 };
  uint32_t phase = PH_BLOCK, bi = 0;
  // current block / channel
  uint32_t bx = 0, by = 0, cx = 1, shape = 0, bctx3 = 0, num_blocks = 1, num_coeffs = 64, lnb = 0;
  uint32_t ci = 0, k = 0, nonzeros = 0, prev = 0, histo_offset = 0, block_context = 0;
  const uint32_t* order = B.natural_orders;

  for (;;) {
    if (!__any_sync(0xffffffffu, !done)) break;
    if (!done && phase == PH_BLOCK) {
      if (bi == nblk) {  // stream finished
        int err = finish_pass(B, F, 0, g, s);
        if (!err && ovf) err = JXG_ERR_UNSUPPORTED;  // a coefficient beyond the entry width (device_types.h)
        B.status[gsid] = err;
        list[kOffBase + nblk * 3] = nlist;
        done = true;
      } else {
        const uint4 d = __ldg(desc + bi);
        bx = d.x & 31;
        by = (d.x >> 5) & 31;
        cx = (d.x >> 10) & 63;
        shape = (d.x >> 22) & 15;
        lnb = d.x >> 26;
        num_blocks = 1u << lnb;
        num_coeffs = num_blocks * 64;
        bctx3 = d.y;
        ci = 0;
        phase = PH_NNZ;
      }
    }
    if (done) continue;
    // ---- one symbol ----
    uint32_t ctx;
    const int c = ci == 0 ? 1 : (ci == 1 ? 0 : 2);  // Y, X, B
    if (phase == PH_NNZ) {
      const uint32_t predicted = predict_nz(nz + c * 32, bx, by);
      block_context = (bctx3 >> (8 * ci)) & 0xff;
      const uint32_t nzc = predicted < 8 ? predicted : (predicted < 64 ? 4 + predicted / 2 : 36);
      ctx = nzc * nbc + block_context + context_offset;
    } else {
      ctx = histo_offset + (uint32_t(s_nz_ctx[((nonzeros + num_blocks - 1) >> lnb) & 63]) + uint32_t(s_freq_ctx[(k >> lnb) & 63])) * 2 + prev;
    }
    const uint32_t value = lane_symbol(T, s, ctx);
    bool next_channel = false;
    if (phase == PH_NNZ) {
      nonzeros = value;
      if (nonzeros + num_blocks > num_coeffs) {
        B.status[gsid] = JXG_ERR_INVALID_NUM_NONZEROS;
        done = true;
        continue;
      }
      uint8_t* col = nz + c * 32;
      const uint8_t nzv = uint8_t((nonzeros + num_blocks - 1) >> lnb);
      for (uint32_t ix = 0; ix < cx; ix++) col[bx + ix] = nzv;
      histo_offset = nbc * 37 + 458 * block_context + context_offset;
      prev = nonzeros > num_coeffs / 16 ? 0u : 1u;
      k = num_blocks;
      order = P.custom_orders ? reinterpret_cast<const uint32_t*>(B.blob + P.order_off) + P.order_offset[shape * 3 + c]
                              : B.natural_orders + B.natural_order_off[shape];
      list[kOffBase + bi * 3 + ci] = nlist;
      if (nonzeros == 0) next_channel = true;
      else phase = PH_COEF;
    } else {
      const int32_t coeff = int32_t(uint32_t(unpack_signed(value)) << shift);
      list_put(list, nlist, __ldg(order + k), coeff, lnb + 6, ovf);
      if (coeff != 0) {
        prev = 1;
        nonzeros--;
      } else {
        prev = 0;
      }
      k++;
      if (nonzeros == 0) next_channel = true;
      else if (k >= num_coeffs) {
        B.status[gsid] = JXG_ERR_RESIDUAL_NONZEROS;  // group.rs:574
        done = true;
        continue;
      }
    }
    if (next_channel) {
      ci++;
      phase = PH_NNZ;
      if (ci == 3) {
        bi++;
        phase = PH_BLOCK;
      }
    }
  }
}

// ---------------------------------------------------------------------------
// K1 lean path: ANS-coded single-pass frames.
//  * Persistent lanes: S lanes per warp each own one (frame, group) stream at a time and pull the next one
//    from a device-wide queue (B.queue) when theirs ends. The host orders the streams longest first, so the
//    queue is a longest-processing-time schedule: the kernel ends close to max(longest stream, total / lanes)
//    instead of waiting for whichever warp drew the longest streams.
//  * The per-symbol step is branch-light and identical for the "number of non-zeros" symbol and the
//    coefficient symbols, so packed lanes stay converged; only block / channel / stream set-up diverges.
//  * Short dependent chain per symbol: the cluster of the next coefficient symbol only depends on whether the
//    current token is zero (value != 0 <=> token != 0), so both candidate context-map entries are fetched
//    before the token is known; the bit window (5 words) lives in registers and is shifted by selects.
// Section copies are 8-byte aligned and zero padded; the word index is clamped to the section so that a
// corrupt stream cannot walk out of the blob (the over-read is reported from bitpos at the end).
// ---------------------------------------------------------------------------
// ---------------------------------------------------------------------------
// K0: block plan of the entropy and transform kernels. One warp per (frame, group) stream walks the group's 32x32 transform map
// in raster order and writes, for every varblock, a 16-byte descriptor
//   x: bx | by << 5 | cx << 10 | cy << 16 | shape << 22 | log2(cx * cy) << 26
//   y: block contexts of Y, X, B (block_context_map.rs:128-150), one byte each
//   z: offset of the block's coefficients inside the group's dense decode-order array (group.rs:455; parity tap only)
//   w: transform type (HfTransformType)
// plus the block count. This is everything the serial decode lanes needed several dependent loads and a scan loop for,
// computed here fully in parallel. Then the same warp partitions the varblocks into the transform classes (kClass*,
// BatchDev::cls_n / cls_list), so that each transform kernel walks only its own varblocks.
// ---------------------------------------------------------------------------
// Bucket of each transform type in the class partition: the classes in kClass* order, and inside the register classes
// one bucket per type (lanes of a warp then mostly share a type). kNumBuckets buckets.
constexpr uint32_t kNumBuckets = 9;
__constant__ uint8_t c_bucket[27] = {0, 7, 7, 1, 6, 7, 4, 5, 7, 7, 7, 7, 2, 3, 7, 7, 7, 7, 8, 8, 8, 8, 8, 8, 8, 8, 8};
// first bucket of each class, and kNumBuckets
__constant__ uint8_t c_class_bucket[6] = {0, 4, 6, 7, 8, kNumBuckets};

__global__ void __launch_bounds__(128) k_block_plan(const BatchDev B) {
  const uint32_t sidx = blockIdx.x * 4 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (sidx >= B.num_streams) return;
  const StreamDev sd = B.streams[sidx];  // ordered by frame then group: sidx == F.first_stream + group
  const FrameDev& F = B.frames[sd.frame];
  const uint32_t g = sd.group;
  const uint32_t bx0 = (g % F.xg) * 32, by0 = (g / F.xg) * 32;
  const uint32_t gw = min(32u, F.xb - bx0), gh = min(32u, F.yb - by0);
  const size_t goff = size_t(by0) * F.xb + bx0;
  const uint8_t* tmap = B.blob + F.transform_off + goff;
  const int32_t* rq = reinterpret_cast<const int32_t*>(B.blob + F.raw_quant_off) + goff;
  const uint8_t* qlf = B.blob + F.quant_lf_off + goff;
  const uint8_t* bcm = B.blob + F.block_ctx_map_off;
  uint4* desc = B.desc + size_t(sidx) * 1024;
  uint32_t seq = 0, coeffs_offset = 0;
  bool bad = false;
  for (uint32_t by = 0; by < gh; by++) {
    const uint32_t bidx = by * F.xb + lane;
    const uint32_t raw_t = lane < gw ? tmap[bidx] : 0u;
    const bool first = raw_t >= 128;
    const uint32_t t = raw_t & 127;
    if (first && t >= 27) bad = true;
    const uint32_t tt = min(t, 26u);
    const uint32_t cx = c_cov_x[tt], cy = c_cov_y[tt], nb = first ? cx * cy : 0u;
    // exclusive prefix sums over the row: number of first blocks and of coefficients
    const uint32_t mask = __ballot_sync(0xffffffffu, first);
    const uint32_t rank = __popc(mask & ((1u << lane) - 1u));
    uint32_t incl = nb * 64;
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
      const uint32_t v = __shfl_up_sync(0xffffffffu, incl, d);
      if (int(lane) >= d) incl += v;
    }
    const uint32_t row_total = __shfl_sync(0xffffffffu, incl, 31);
    if (first && coeffs_offset + incl > kGroupCoeffs) bad = true;  // overlapping varblocks would overflow the group's area
    if (first && !bad) {
      const uint32_t off = coeffs_offset + incl - nb * 64;
      const uint32_t shape = c_shape[tt];
      const uint32_t raw_quant = uint32_t(rq[bidx]);
      uint32_t qf_idx = 0;
      for (uint32_t i = 0; i < F.num_qf_thresholds; i++) qf_idx += raw_quant > F.qf_thresholds[i];
      const uint32_t qf_lf_idx = qf_idx * F.num_lf_contexts + qlf[bidx];
      const uint32_t stride = (F.num_qf_thresholds + 1) * F.num_lf_contexts;
      // channel order of block_context(): index 0 = Y, 1 = X, 2 = B (group.rs:478-480 c < 2 ? c ^ 1 : 2)
      const uint32_t cy_ctx = bcm[(0 * 13 + shape) * stride + qf_lf_idx];
      const uint32_t cx_ctx = bcm[(1 * 13 + shape) * stride + qf_lf_idx];
      const uint32_t cb_ctx = bcm[(2 * 13 + shape) * stride + qf_lf_idx];
      uint4 d;
      d.x = lane | (by << 5) | (cx << 10) | (cy << 16) | (shape << 22) | ((31u - __clz(cx * cy)) << 26);
      d.y = cy_ctx | (cx_ctx << 8) | (cb_ctx << 16);
      d.z = off;
      d.w = tt;
      desc[seq + rank] = d;
    }
    seq += __popc(mask);
    coeffs_offset += row_total;
  }
  bad = __any_sync(0xffffffffu, bad);
  if (lane == 0) B.nblk[sidx] = bad ? 0xffffffffu : seq;

  // Class partition: a counting sort of the descriptors by bucket, read back in raster (ordinal) order. A failed plan
  // has empty classes (its stream reports the error and no transform touches it).
  uint32_t* cls_n = B.cls_n + size_t(sidx) * kClassWords;
  if (bad) {
    if (lane < kClassWords) cls_n[lane] = 0;
    return;
  }
  uint32_t* cls_list = B.cls_list + size_t(sidx) * 1024;
  const uint32_t* dw = reinterpret_cast<const uint32_t*>(desc);  // x and w words, written above by this warp
  __syncwarp();
  uint32_t cnt = 0;  // lane k < kNumBuckets: varblocks of bucket k
  for (uint32_t i0 = 0; i0 < seq; i0 += 32) {
    const uint32_t bk = i0 + lane < seq ? c_bucket[dw[size_t(i0 + lane) * 4 + 3]] : kNumBuckets;
#pragma unroll
    for (uint32_t k = 0; k < kNumBuckets; k++) {
      const uint32_t m = __ballot_sync(0xffffffffu, bk == k);
      if (lane == k) cnt += __popc(m);
    }
  }
  uint32_t start = cnt;  // exclusive prefix sum over the buckets
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const uint32_t v = __shfl_up_sync(0xffffffffu, start, d);
    if (int(lane) >= d) start += v;
  }
  start -= cnt;
  // class c covers buckets c_class_bucket[c] .. c_class_bucket[c + 1] - 1 (lane kNumBuckets holds the total); lane c < 5
  // stores its count
  const uint32_t s0 = __shfl_sync(0xffffffffu, start, c_class_bucket[min(lane, 5u)]);
  const uint32_t s1 = __shfl_sync(0xffffffffu, start, c_class_bucket[min(lane + 1, 5u)]);
  if (lane < kClassWords) cls_n[lane] = lane < 5 ? s1 - s0 : 0u;
  uint32_t fill = start;  // lane k: next slot of bucket k
  for (uint32_t i0 = 0; i0 < seq; i0 += 32) {
    const uint32_t i = i0 + lane;
    const uint32_t x = i < seq ? dw[size_t(i) * 4] : 0u, t = i < seq ? dw[size_t(i) * 4 + 3] : 0u;
    const uint32_t bk = i < seq ? c_bucket[t] : kNumBuckets;
#pragma unroll
    for (uint32_t k = 0; k < kNumBuckets; k++) {
      const uint32_t m = __ballot_sync(0xffffffffu, bk == k);
      const uint32_t at = __shfl_sync(0xffffffffu, fill, k);
      if (bk == k) cls_list[at + __popc(m & ((1u << lane) - 1u))] = cls_entry(i, x & 31, (x >> 5) & 31, t);
      if (lane == k) fill += __popc(m);
    }
  }
}

// Loads the compiler must not sink below the token computation (it would re-serialise the chain).
__device__ __forceinline__ uint32_t spec_ld_u8(const uint8_t* p) {
  uint32_t v;
  asm volatile("ld.global.nc.u8 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}
__device__ __forceinline__ uint32_t spec_ld_u32(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(v) : "l"(p));
  return v;
}

constexpr uint32_t kLeanCtxSmem = 16384;  // context maps up to this size are staged in shared memory

__device__ __forceinline__ uint32_t spec_lds_u8(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u8 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}
__device__ __forceinline__ uint32_t spec_lds_u16(uint32_t addr) {
  uint32_t v;
  asm volatile("ld.shared.u16 %0, [%1];" : "=r"(v) : "r"(addr));
  return v;
}

// CTXS: the frame's context map fits the shared-memory staging area (host decision for the whole batch).
// Launch bound 6 CTAs / SM (<= 85 registers; the compiler takes 71 - 78). A 64-register build (bound 8) was slower per
// 64-frame batch and did not buy co-residency with the filters of other batches.
template <int S, bool K420, bool CTXS>
__global__ void __launch_bounds__(128, 6) k_entropy_lean(const BatchDev B) {
  // context LUTs, pre-multiplied by 2 (block_context_map.rs:34-46), natural-order table offsets
  __shared__ uint16_t s_nz2[64], s_fr2[64];
  __shared__ uint32_t s_order_off[13];
  // Per-lane non-zero counts: one byte per block column and channel is enough. Varblocks are visited in raster order
  // of their top-left corner, so the last value written to a column is the count of the block right above the
  // current row, and (for column bx - 1) of the block to the left — the two neighbours group.rs:489-505 predicts from.
  __shared__ uint8_t s_nzcol[4 * S][3 * 32];
  extern __shared__ __align__(16) uint8_t s_ctxmap[];  // the frame's context map (CTXS)
  if (threadIdx.x < 64) {
    // entry 0 of both tables is the reference's 0xBAD marker: never used by a valid context, but the speculative
    // look-ups of the per-symbol step may touch it, so it must stay inside the context map
    s_nz2[threadIdx.x] = threadIdx.x ? uint16_t(c_nz_ctx[threadIdx.x] * 2) : uint16_t(0);
    s_fr2[threadIdx.x] = threadIdx.x ? uint16_t(c_freq_ctx[threadIdx.x] * 2) : uint16_t(0);
  }
  if (threadIdx.x < 13) s_order_off[threadIdx.x] = B.natural_order_off[threadIdx.x];
  // CTA -> frame: all lanes of a CTA work on one frame, so its context map and alias tables stay close.
  uint32_t fidx;
  {
    uint32_t lo = 0, hi = B.num_frames;
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (B.lean_cta_first[mid] <= blockIdx.x) lo = mid;
      else hi = mid;
    }
    fidx = lo;
  }
  const FrameDev& F = B.frames[fidx];
  const PassDev& P = F.passes[0];
  const uint32_t nbc = F.num_block_contexts;
  if (CTXS) {
    const uint32_t num_ctx = F.num_histograms * nbc * (37 + 458);
    const uint8_t* src = B.blob + P.code.cmap_off;  // 16-byte aligned in the blob
    for (uint32_t i = threadIdx.x * 16; i < num_ctx + 64; i += blockDim.x * 16)  // speculative look-ups run a bit past the end
      *reinterpret_cast<uint4*>(s_ctxmap + i) = __ldg(reinterpret_cast<const uint4*>(src + i));
  }
  __syncthreads();
  const uint8_t* const ctxmap_g = B.blob + P.code.cmap_off;
  // Shared-window addresses of the three look-up tables, made opaque so that they stay in registers: left to itself the
  // compiler rematerialises them inside the per-symbol loop (S2R SR_CgaCtaId + LEA + adds, ~8 of the ~92 instructions).
  uint32_t ctxmap_s = uint32_t(__cvta_generic_to_shared(s_ctxmap));
  uint32_t nz2_s = uint32_t(__cvta_generic_to_shared(s_nz2)), fr2_s = uint32_t(__cvta_generic_to_shared(s_fr2));
  asm volatile("" : "+r"(ctxmap_s), "+r"(nz2_s), "+r"(fr2_s));
  auto ctx_cluster = [&](uint32_t ctx) { return CTXS ? spec_lds_u8(ctxmap_s + ctx) : spec_ld_u8(ctxmap_g + ctx); };
  const uint32_t lane = threadIdx.x & 31;
  // Warp schedule written by the host (batch.cc schedule_lean): the first stream of this warp in the frame's
  // longest-first list and its number of lanes (<= S). The longest streams of a frame sit alone in their warp — the
  // kernel ends when the longest stream ends, and a lane that shares its warp pays for the divergent set-up paths of
  // its neighbours — the shorter ones are packed 2 or S to a warp.
  const uint2 wsched = B.lean_warp[blockIdx.x * 4 + (threadIdx.x >> 5)];
  const uint32_t frame_lanes = F.lean_lanes;
  uint32_t qpos = wsched.x + lane;  // position in this frame's (longest first) stream list
  bool done = !(lane < wsched.y && qpos < F.lean_count);
  uint8_t* const nz = s_nzcol[(threadIdx.x >> 5) * S + (lane < S ? lane : 0)];
  // ---- per-frame constants ----
  const uint32_t* const ucfg = reinterpret_cast<const uint32_t*>(B.blob + P.code.cfg_off);
  const uint2* const ans = reinterpret_cast<const uint2*>(B.blob + P.code.ans_off);
  const uint32_t log_alpha = P.code.log_alpha, log_bucket = 12 - P.code.log_alpha, bucket_mask = (1u << (12 - P.code.log_alpha)) - 1;
  // Coefficient orders: read once here, not by every channel's set-up (the stores of the loop keep the compiler from
  // hoisting the loads of P itself).
  const bool custom_orders = P.custom_orders != 0;
  const uint32_t* const order_base = custom_orders ? reinterpret_cast<const uint32_t*>(B.blob + P.order_off) : B.natural_orders;
  // ---- per-stream state (re-initialised by the set-up path when a lane takes a new stream) ----
  uint32_t gsid = 0, nblk = 0, bi = 0;
  const uint4* desc = B.desc;
  uint32_t* list = B.nzlist;  // this stream's coefficient list (pass 0), entries written so far, its section index
  uint32_t nlist = 0, ovf = 0;
  const uint32_t* words = reinterpret_cast<const uint32_t*>(B.blob);
  uint32_t sec_bits = 0, wlimit = 0;
  uint32_t bitpos = 0, ans_state = 0x130000u, context_offset = 0;
  uint32_t wi = 0, w0 = 0, w1 = 0, w2 = 0;
  // ---- per-block state ----
  uint32_t coeffs_offset = 0;
  uint32_t bx = 0, by = 0, cxy = 0x0101, shape = 0, bctx3 = 0, num_blocks = 1, num_coeffs = 64, lnb = 0;
  uint32_t ci = 3;          // 3: need a new block
  bool need_setup = true;   // channel (and maybe block / stream) set-up before the next symbol
  bool new_stream = true, failed = false;
  bool mode_nnz = true;
  uint32_t block_context = 0, cluster = 0;
  uint32_t k = 0, nonzeros = 0, histo_offset = 0;
  const uint32_t* order = B.natural_orders;

  for (;;) {
    if (!__any_sync(0xffffffffu, !done)) break;
    if (!done && need_setup) {
      // ---------- rare path: next stream, block and/or channel ----------
      while (ci == 3) {
        if (new_stream) {
          const uint32_t lidx = F.lean_first + qpos;
          const uint32_t g = B.streams_lean[lidx].group;
          gsid = F.first_stream + g;
          list = list_base(B, F.section_base + g);
          nlist = 0;
          ovf = 0;
          desc = B.desc + size_t(gsid) * 1024;
          nblk = B.nblk[gsid];
          bi = 0;
          const SectionDev sec = B.sections[F.section_base + g];
          words = reinterpret_cast<const uint32_t*>(B.blob + sec.off);
          sec_bits = sec.len * 8u;
          wlimit = (sec.len >> 2) + 1;
          uint32_t nb = 0;
          while ((1u << nb) < F.num_histograms) nb++;
          const uint32_t hist_idx = nb ? (__ldg(words) & ((1u << nb) - 1u)) : 0u;  // group.rs:333-341 (nb <= 12)
          failed = false;
          histo_offset = 0;
          if (nblk == 0xffffffffu) {
            B.status[gsid] = JXG_ERR_INVALID_TRANSFORM;
            failed = true;
            nblk = 0;
          } else if (hist_idx >= F.num_histograms) {
            B.status[gsid] = JXG_ERR_INVALID_HISTOGRAM_INDEX;
            failed = true;
            nblk = 0;
          }
          context_offset = failed ? 0u : hist_idx * nbc * (37 + 458);
          ans_state = __funnelshift_r(__ldg(words), __ldg(words + 1), nb);  // ans.rs:431
          bitpos = nb + 32;
          wi = 1;
          w0 = __ldg(words + 1);
          w1 = __ldg(words + 2);
          w2 = __ldg(words + 3);
          new_stream = false;
        }
        if (bi >= nblk) {  // stream finished: check_final_state (decode.rs:400), then take the next one
          if (!failed) {
            int err = 0;
            if (bitpos > sec_bits) err = JXG_ERR_OUT_OF_BOUNDS;
            else if (ans_state != 0x130000u) err = JXG_ERR_ANS_CHECKSUM;
            else if (ovf) err = JXG_ERR_UNSUPPORTED;  // a coefficient beyond the entry width (device_types.h)
            B.status[gsid] = err;
            list[kOffBase + nblk * 3] = nlist;  // end of the last varblock's entries
          }
          qpos = atomicAdd(B.queue + fidx, 1u) + frame_lanes;
          if (qpos >= F.lean_count) {
            done = true;
            break;
          }
          new_stream = true;
          continue;
        }
        const uint4 d = __ldg(desc + bi);
        bi++;
        bx = d.x & 31;
        by = (d.x >> 5) & 31;
        const uint32_t cx = (d.x >> 10) & 63, cy = (d.x >> 16) & 63;
        cxy = cx | (cy << 8);
        shape = (d.x >> 22) & 15;
        lnb = d.x >> 26;
        num_blocks = cx * cy;
        num_coeffs = num_blocks * 64;
        bctx3 = d.y;
        coeffs_offset = d.z;
        ci = 0;
      }
      if (!done) {
        const int c = ci == 0 ? 1 : (ci == 1 ? 0 : 2);  // Y, X, B
        const uint8_t* nzc_col = nz + c * 32;
        // both neighbours read, the prediction selected: no branches inside the (divergent) set-up path
        const uint32_t up = nzc_col[bx], left = nzc_col[bx ? bx - 1 : 0];
        const uint32_t predicted = bx == 0 ? (by == 0 ? 32u : up) : (by == 0 ? left : (up + left + 1u) >> 1);
        block_context = (bctx3 >> (8 * ci)) & 0xff;
        const uint32_t nzc = predicted < 8 ? predicted : (predicted < 64 ? 4 + predicted / 2 : 36);
        cluster = ctx_cluster(nzc * nbc + block_context + context_offset);
        mode_nnz = true;
        need_setup = false;
      }
    }
    if (done) continue;
    // ---------- common path: one symbol ----------
    // speculative: clusters of the next coefficient symbol for token == 0 (A) and token != 0 (B)
    const uint32_t w3 = spec_ld_u32(words + wi + 3), w4 = spec_ld_u32(words + wi + 4);
    const uint32_t fr_next = spec_lds_u16(fr2_s + ((((k + 1) >> lnb) & 63) << 1));
    const uint32_t nzq = nonzeros + num_blocks - 1;
    const uint32_t ctxA = histo_offset + fr_next + spec_lds_u16(nz2_s + (((nzq >> lnb) & 63) << 1));
    const uint32_t ctxB = histo_offset + fr_next + spec_lds_u16(nz2_s + ((((nzq - 1) >> lnb) & 63) << 1)) + 1u;
    const uint32_t clA = ctx_cluster(ctxA), clB = ctx_cluster(ctxB);
    // rANS step (ans.rs:356-393)
    const uint32_t idx12 = ans_state & 0xfff;
    const uint32_t bi12 = idx12 >> log_bucket, bp = idx12 & bucket_mask;
    const uint2 bk = __ldg(ans + ((cluster << log_alpha) + bi12));
    const bool alias = bp >= ((bk.x >> 8) & 0xff);
    const uint32_t dist = (bk.x >> 16) ^ (alias ? (bk.y >> 16) : 0u);
    const uint32_t offset = bp + (alias ? (bk.y & 0xffff) : 0u);
    const uint32_t token = alias ? (bk.x & 0xff) : bi12;
    const uint32_t nonzero = token != 0 ? 1u : 0u;
    const uint32_t cluster_next = nonzero ? clB : clA;
    uint32_t next = (ans_state >> 12) * dist + offset;
    const uint32_t sh = bitpos & 31;
    const bool refill = next < (1u << 16);
    const uint32_t w16 = __funnelshift_r(w0, w1, sh) & 0xffff;
    ans_state = refill ? ((next << 16) | w16) : next;
    const uint32_t sh2 = sh + (refill ? 16u : 0u);  // <= 47
    // hybrid uint (hybrid_uint.rs:87-102), branch free
    uint32_t split_exponent = 4, msb = 2, lsb = 0;
    if (!K420) {
      const uint32_t cfg = __ldg(ucfg + cluster);
      split_exponent = cfg & 0xff;
      msb = (cfg >> 8) & 0xff;
      lsb = (cfg >> 16) & 0xff;
    }
    const uint32_t split_token = 1u << split_exponent;
    const bool direct = token < split_token;
    const uint32_t bits_in_token = msb + lsb;
    const uint32_t nbits = direct ? 0u : ((split_exponent - bits_in_token + ((token - split_token) >> bits_in_token)) & 31);
    const uint32_t win = sh2 < 32 ? __funnelshift_r(w0, w1, sh2) : __funnelshift_r(w1, w2, sh2);
    const uint32_t bits = win & ((1u << nbits) - 1u);
    const uint32_t hi = ((token >> lsb) & ((1u << msb) - 1u)) | (1u << msb);
    const uint32_t composed = (((hi << nbits) | bits) << lsb) | (token & ((1u << lsb) - 1u));
    const uint32_t value = direct ? token : composed;
    bitpos += (refill ? 16u : 0u) + nbits;
    {  // advance the register window by 0..2 words
      const uint32_t nwi = min(bitpos >> 5, wlimit);
      const uint32_t adv = nwi - wi;
      wi = nwi;
      const uint32_t t0 = adv == 0 ? w0 : (adv == 1 ? w1 : w2);
      const uint32_t t1 = adv == 0 ? w1 : (adv == 1 ? w2 : w3);
      const uint32_t t2 = adv == 0 ? w2 : (adv == 1 ? w3 : w4);
      w0 = t0;
      w1 = t1;
      w2 = t2;
    }
    // ---------- post ----------
    if (mode_nnz) {
      const int c = ci == 0 ? 1 : (ci == 1 ? 0 : 2);
      nonzeros = value;
      if (nonzeros + num_blocks > num_coeffs) {
        B.status[gsid] = JXG_ERR_INVALID_NUM_NONZEROS;
        failed = true;
        bi = nblk;
        ci = 3;
        need_setup = true;
        continue;
      }
      uint8_t* nzc_col = nz + c * 32;
      const uint8_t nzv = uint8_t((nonzeros + num_blocks - 1) >> lnb);
      const uint32_t cx = cxy & 0xff;
#pragma unroll 1
      for (uint32_t ix = 0; ix < cx; ix++) nzc_col[bx + ix] = nzv;  // a rolled loop: most varblocks are one block wide
      histo_offset = nbc * 37 + 458 * block_context + context_offset;
      k = num_blocks;
      order = order_base + (custom_orders ? P.order_offset[shape * 3 + c] : s_order_off[shape]);
      list[kOffBase + (bi - 1) * 3 + ci] = nlist;  // first entry of this varblock's channel ci (Y, X, B)
      mode_nnz = false;
      if (nonzeros == 0) {
        need_setup = true;
        ci++;
      } else {
        const uint32_t prev = nonzeros > num_coeffs / 16 ? 0u : 1u;
        cluster = ctx_cluster(histo_offset + uint32_t(s_nz2[((nonzeros + num_blocks - 1) >> lnb) & 63]) +
                              uint32_t(s_fr2[(k >> lnb) & 63]) + prev);
      }
    } else {
      list_put(list, nlist, __ldg(order + k), unpack_signed(value), lnb + 6, ovf);  // lean streams have shift == 0 (host routing)
      nonzeros -= nonzero;
      cluster = cluster_next;
      k++;
      if (nonzeros == 0) {
        need_setup = true;
        ci++;
      } else if (k >= num_coeffs) {
        B.status[gsid] = JXG_ERR_RESIDUAL_NONZEROS;  // group.rs:574
        failed = true;
        bi = nblk;
        ci = 3;
        need_setup = true;
      }
    }
  }
}

// ===========================================================================
// K2: dequant + CfL + LLF + inverse DCT
// ===========================================================================

template <int N>
struct Log2 {
  static constexpr int v = 1 + Log2<N / 2>::v;
};
template <>
struct Log2<1> {
  static constexpr int v = 0;
};

// gen_idct.py:112-127 / idct_large.rs:251-310: even/odd split recursion.
template <int N>
__device__ __forceinline__ void idct1d(float* v) {
  if constexpr (N == 1) {
    return;
  } else if constexpr (N == 2) {
    float a = v[0], b = v[1];
    v[0] = a + b;
    v[1] = a - b;
  } else {
    constexpr int H = N / 2;
    float first[H], second[H];
#pragma unroll
    for (int i = 0; i < H; i++) {
      first[i] = v[2 * i];
      second[i] = v[2 * i + 1];
    }
    idct1d<H>(first);
#pragma unroll
    for (int i = H - 1; i >= 1; i--) second[i] += second[i - 1];
    second[0] *= 1.41421356237309504880f;
    idct1d<H>(second);
#pragma unroll
    for (int i = 0; i < H; i++) {
      float mul = c_wc[Log2<N>::v][i];
      v[i] = fmaf(second[i], mul, first[i]);
      v[N - 1 - i] = fmaf(-second[i], mul, first[i]);
    }
  }
}

// Large sizes: same recursion, arrays in local memory, loops not unrolled.
template <int N>
__device__ __noinline__ void idct1d_large(float* v) {
  if constexpr (N <= 32) {
    idct1d<N>(v);
  } else {
    constexpr int H = N / 2;
    float first[H], second[H];
#pragma unroll 1
    for (int i = 0; i < H; i++) {
      first[i] = v[2 * i];
      second[i] = v[2 * i + 1];
    }
    idct1d_large<H>(first);
#pragma unroll 1
    for (int i = H - 1; i >= 1; i--) second[i] += second[i - 1];
    second[0] *= 1.41421356237309504880f;
    idct1d_large<H>(second);
#pragma unroll 1
    for (int i = 0; i < H; i++) {
      float mul = c_wc[Log2<N>::v][i];
      v[i] = fmaf(second[i], mul, first[i]);
      v[N - 1 - i] = fmaf(-second[i], mul, first[i]);
    }
  }
}

// gen_reinterpreting_dct.py:47-136
template <int N>
__device__ __forceinline__ void rdct1d_rec(float* v) {
  if constexpr (N == 1) {
    return;
  } else if constexpr (N == 2) {
    float a = v[0], b = v[1];
    v[0] = a + b;
    v[1] = a - b;
  } else {
    constexpr int H = N / 2;
    float first[H], second[H];
#pragma unroll
    for (int i = 0; i < H; i++) {
      first[i] = v[i] + v[N - 1 - i];
      second[i] = v[i] - v[N - 1 - i];
    }
    rdct1d_rec<H>(first);
#pragma unroll
    for (int i = 0; i < H; i++) second[i] *= c_wc[Log2<N>::v][i];
    rdct1d_rec<H>(second);
    second[0] = fmaf(second[0], 1.41421356237309504880f, second[1]);
#pragma unroll
    for (int i = 1; i + 1 < H; i++) second[i] = second[i] + second[i + 1];
#pragma unroll
    for (int i = 0; i < H; i++) {
      v[2 * i] = first[i];
      v[2 * i + 1] = second[i];
    }
  }
}
template <int N>
__device__ __forceinline__ void rdct1d(float* v) {
  if constexpr (N > 1) {
    rdct1d_rec<N>(v);
#pragma unroll
    for (int i = 0; i < N; i++) v[i] *= c_rdct_scale[Log2<N>::v][i];
  }
}
__device__ __noinline__ void rdct1d_dyn(float* v, int n) {
  switch (n) {
    case 2: rdct1d<2>(v); break;
    case 4: rdct1d<4>(v); break;
    case 8: rdct1d<8>(v); break;
    case 16: rdct1d<16>(v); break;
    case 32: rdct1d<32>(v); break;
    default: break;
  }
}

// LLF of one channel: cy x cx LF samples -> coefficients (tests.rs:154-180).
// Serial (tiny); `put(vf, hf, value)` stores into the caller's layout.
template <typename Put>
__device__ __forceinline__ void llf_small(const float* lf, uint32_t lf_stride, int cy, int cx, Put put) {
  float tmp[16];  // cy, cx <= 4
  float line[4];
  for (int y = 0; y < cy; y++) {
    for (int x = 0; x < cx; x++) line[x] = lf[y * lf_stride + x];
    if (cx == 2) rdct1d<2>(line);
    else if (cx == 4) rdct1d<4>(line);
    for (int x = 0; x < cx; x++) tmp[y * 4 + x] = line[x];
  }
  for (int hf = 0; hf < cx; hf++) {
    for (int y = 0; y < cy; y++) line[y] = tmp[y * 4 + hf];
    if (cy == 2) rdct1d<2>(line);
    else if (cy == 4) rdct1d<4>(line);
    for (int vf = 0; vf < cy; vf++) put(vf, hf, line[vf]);
  }
}

// group.rs:85-96
__device__ __forceinline__ float adjust_quant_bias(int32_t q, float bias_c, float bias3) {
  float qf = float(q);
  return (q > -2 && q < 2) ? qf * bias_c : qf - bias3 / qf;
}

// Dequantisation constants of one varblock (group.rs:137-177).
struct DeqParams {
  const float* mat;  // dequant weights of the block's table: channel c at mat + c * ncoef
  uint32_t ncoef;
  float sx, sy, sb, x_cc, b_cc, bias0, bias1, bias2, bias3;
};

// Coefficient lists -> DEQUANTISED coefficient tile of one varblock in shared memory (three channels at stride
// `cstride` floats, element of position pos at idx(pos)). Only the non-zero entries are touched: the tile is zeroed, the
// Y entries write dy and seed X / B with cc * dy, then the X / B entries write mul_add(cc, dy, d) — exactly
// group.rs:100-133 evaluated at every position (a zero quantised value dequantises to 0, and mul_add(cc, dy, 0) is the
// rounded product), at a tenth of the arithmetic since >= 90 % of the coefficients are zero. `nl` lanes of rank r work
// together and separate the phases with sync(). Frames with several passes add the passes up as integers first
// (group.rs:556-567: the sum is the coefficient) and convert in place.
template <typename Sync, typename Idx>
__device__ __forceinline__ void gather_dequant_tile(const BatchDev& B, const FrameDev& F, uint32_t g, uint32_t seq, float* tile,
                                                    uint32_t cstride, uint32_t zero_floats, const DeqParams& D, uint32_t r, uint32_t nl,
                                                    bool valid, const ListStage& st, Sync sync, Idx idx) {
  const uint32_t lnc = 31 - __clz(D.ncoef);
  sync();  // the previous varblock of this lane group has been read completely
  for (uint32_t c = 0; c < 3; c++) {
    float4* t4 = reinterpret_cast<float4*>(tile + c * cstride);
    for (uint32_t i = r; i < zero_floats / 4; i += nl) t4[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
  }
  sync();
  if (F.num_passes == 1) {
    const uint32_t* base = list_base(B, F.section_base + g);
    const bool from_stage = st.off != nullptr;
    const uint32_t* ow = from_stage ? st.off + seq * 3 : base + kOffBase + seq * 3;
    uint32_t o0 = 0, o1 = 0, o2 = 0, o3 = 0;
    if (valid) {
      o0 = ow[0];
      o1 = ow[1];
      o2 = ow[2];
      o3 = min(ow[3], kListCap);
    }
    const uint32_t staged = from_stage ? st.staged : 0u;
    for (uint32_t i = o0 + r; i < o1; i += nl) {  // Y
      const uint32_t e = i < staged ? st.ent[i] : __ldg(base + i);
      const uint32_t pos = entry_pos(e, lnc), j = idx(pos);
      const float dy = adjust_quant_bias(entry_value(e, lnc), D.bias1, D.bias3) * (__ldg(D.mat + D.ncoef + pos) * D.sy);
      tile[cstride + j] = dy;
      tile[j] = D.x_cc * dy;
      tile[2 * cstride + j] = D.b_cc * dy;
    }
    sync();
    for (uint32_t i = o1 + r; i < o3; i += nl) {  // X, then B
      const uint32_t e = i < staged ? st.ent[i] : __ldg(base + i);
      const uint32_t pos = entry_pos(e, lnc), j = idx(pos);
      const bool is_x = i < o2;
      const uint32_t c = is_x ? 0u : 2u;
      const float d = adjust_quant_bias(entry_value(e, lnc), is_x ? D.bias0 : D.bias2, D.bias3) *
                      (__ldg(D.mat + c * D.ncoef + pos) * (is_x ? D.sx : D.sb));
      tile[c * cstride + j] = fmaf(is_x ? D.x_cc : D.b_cc, tile[cstride + j], d);
    }
    sync();
    return;
  }
  int32_t* it = reinterpret_cast<int32_t*>(tile);
  for (uint32_t p = 0; p < F.num_passes; p++) {
    const uint32_t* base = list_base(B, F.section_base + p * F.num_groups + g);
    const uint32_t* ow = base + kOffBase + seq * 3;
    if (valid) {
      const uint32_t o0 = ow[0], o1 = ow[1], o2 = ow[2], o3 = min(ow[3], kListCap);
      for (uint32_t i = o0 + r; i < o3; i += nl) {
        const uint32_t e = __ldg(base + i);
        const uint32_t c = i < o1 ? 1u : (i < o2 ? 0u : 2u);
        it[c * cstride + idx(entry_pos(e, lnc))] += entry_value(e, lnc);
      }
    }
    sync();
  }
  if (valid) {
    for (uint32_t k = r; k < D.ncoef; k += nl) {
      const uint32_t j = idx(k);
      const float dy = adjust_quant_bias(it[cstride + j], D.bias1, D.bias3) * (__ldg(D.mat + D.ncoef + k) * D.sy);
      const float dxc = adjust_quant_bias(it[j], D.bias0, D.bias3) * (__ldg(D.mat + k) * D.sx);
      const float dbc = adjust_quant_bias(it[2 * cstride + j], D.bias2, D.bias3) * (__ldg(D.mat + 2 * D.ncoef + k) * D.sb);
      tile[cstride + j] = dy;
      tile[j] = fmaf(D.x_cc, dy, dxc);
      tile[2 * cstride + j] = fmaf(D.b_cc, dy, dbc);
    }
  }
  sync();
}

struct DequantCtx {
  const int32_t* qx;
  const int32_t* qy;
  const int32_t* qb;
  const float* mat;
  uint32_t num_coeffs;
  float sx, sy, sb, x_cc, b_cc, bias0, bias1, bias2, bias3;
  __device__ __forceinline__ void get_q(uint32_t k, int32_t qxv, int32_t qyv, int32_t qbv, float& vx, float& vy, float& vb) const {
    float dy = adjust_quant_bias(qyv, bias1, bias3) * (__ldg(mat + num_coeffs + k) * sy);
    float dxc = adjust_quant_bias(qxv, bias0, bias3) * (__ldg(mat + k) * sx);
    float dbc = adjust_quant_bias(qbv, bias2, bias3) * (__ldg(mat + 2 * num_coeffs + k) * sb);
    vy = dy;
    vx = fmaf(x_cc, dy, dxc);
    vb = fmaf(b_cc, dy, dbc);
  }
  __device__ __forceinline__ void get(uint32_t k, float& vx, float& vy, float& vb) const { get_q(k, qx[k], qy[k], qb[k], vx, vy, vb); }
};

// ---- special 8x8 transforms, one lane per channel, serial (transform.rs:306-661) ----
__device__ __forceinline__ void idct2d_4x4(float* b) {  // [hf][vf] layout, in place -> [y][x]
  float t[16], line[4];
  for (int vf = 0; vf < 4; vf++) {
    for (int hf = 0; hf < 4; hf++) line[hf] = b[hf * 4 + vf];
    idct1d<4>(line);
    for (int x = 0; x < 4; x++) t[vf * 4 + x] = line[x];
  }
  for (int x = 0; x < 4; x++) {
    for (int vf = 0; vf < 4; vf++) line[vf] = t[vf * 4 + x];
    idct1d<4>(line);
    for (int y = 0; y < 4; y++) b[y * 4 + x] = line[y];
  }
}
__device__ __forceinline__ void idct2d_4x8(float* b) {  // 4 rows x 8 cols, [vf][hf] -> [y][x]
  float t[32], l8[8], l4[4];
  for (int vf = 0; vf < 4; vf++) {
    for (int hf = 0; hf < 8; hf++) l8[hf] = b[vf * 8 + hf];
    idct1d<8>(l8);
    for (int x = 0; x < 8; x++) t[vf * 8 + x] = l8[x];
  }
  for (int x = 0; x < 8; x++) {
    for (int vf = 0; vf < 4; vf++) l4[vf] = t[vf * 8 + x];
    idct1d<4>(l4);
    for (int y = 0; y < 4; y++) b[y * 8 + x] = l4[y];
  }
}
__device__ __forceinline__ void idct2d_8x4(float* b) {  // 8 rows x 4 cols, stored [hf][vf] stride 8 -> [y][x] stride 4
  float t[32], l8[8], l4[4];
  for (int vf = 0; vf < 8; vf++) {
    for (int hf = 0; hf < 4; hf++) l4[hf] = b[hf * 8 + vf];
    idct1d<4>(l4);
    for (int x = 0; x < 4; x++) t[vf * 4 + x] = l4[x];
  }
  for (int x = 0; x < 4; x++) {
    for (int vf = 0; vf < 8; vf++) l8[vf] = t[vf * 4 + x];
    idct1d<8>(l8);
    for (int y = 0; y < 8; y++) b[y * 4 + x] = l8[y];
  }
}

__device__ __noinline__ void special_transform(int t, const float* co, float* px) {
  if (t == 1) {  // IDENTITY
    float b00 = co[0], b01 = co[1], b10 = co[8], b11 = co[9];
    float dcs[4] = {b00 + b01 + b10 + b11, b00 + b01 - b10 - b11, b00 - b01 + b10 - b11, b00 - b01 - b10 + b11};
    for (int y = 0; y < 2; y++)
      for (int x = 0; x < 2; x++) {
        float residual_sum = 0.0f;
        for (int iy = 0; iy < 4; iy++)
          for (int ix = 0; ix < 4; ix++) {
            if (ix == 0 && iy == 0) continue;
            residual_sum += co[(y + iy * 2) * 8 + x + ix * 2];
          }
        float center = dcs[y * 2 + x] - residual_sum * (1.0f / 16.0f);
        px[(4 * y + 1) * 8 + 4 * x + 1] = center;
        for (int iy = 0; iy < 4; iy++)
          for (int ix = 0; ix < 4; ix++) {
            if (ix == 1 && iy == 1) continue;
            px[(y * 4 + iy) * 8 + x * 4 + ix] = co[(y + iy * 2) * 8 + x + ix * 2] + center;
          }
        px[y * 4 * 8 + x * 4] = co[(y + 2) * 8 + x + 2] + center;
      }
  } else if (t == 2) {  // DCT2X2
    float tmp[64];
    auto top = [](int s, const float* in, float* out) {
      int n = s / 2;
      for (int y = 0; y < n; y++)
        for (int x = 0; x < n; x++) {
          float c00 = in[y * 8 + x], c01 = in[y * 8 + n + x], c10 = in[(y + n) * 8 + x], c11 = in[(y + n) * 8 + n + x];
          out[y * 2 * 8 + x * 2] = c00 + c01 + c10 + c11;
          out[y * 2 * 8 + x * 2 + 1] = c00 + c01 - c10 - c11;
          out[(y * 2 + 1) * 8 + x * 2] = c00 - c01 + c10 - c11;
          out[(y * 2 + 1) * 8 + x * 2 + 1] = c00 - c01 - c10 + c11;
        }
    };
    for (int i = 0; i < 64; i++) {
      tmp[i] = co[i];
      px[i] = co[i];
    }
    top(2, tmp, px);
    top(4, px, tmp);
    top(8, tmp, px);
  } else if (t == 3) {  // DCT4X4
    float b00 = co[0], b01 = co[1], b10 = co[8], b11 = co[9];
    float dcs[4] = {b00 + b01 + b10 + b11, b00 + b01 - b10 - b11, b00 - b01 + b10 - b11, b00 - b01 - b10 + b11};
    for (int y = 0; y < 2; y++)
      for (int x = 0; x < 2; x++) {
        float block[16];
        for (int iy = 0; iy < 4; iy++)
          for (int ix = 0; ix < 4; ix++) block[iy * 4 + ix] = co[(y + iy * 2) * 8 + x + ix * 2];
        block[0] = dcs[y * 2 + x];
        idct2d_4x4(block);
        for (int iy = 0; iy < 4; iy++)
          for (int ix = 0; ix < 4; ix++) px[(y * 4 + iy) * 8 + x * 4 + ix] = block[iy * 4 + ix];
      }
  } else if (t == 12 || t == 13) {  // DCT4X8 / DCT8X4
    float dcs[2] = {co[0] + co[8], co[0] - co[8]};
    for (int h = 0; h < 2; h++) {
      float block[32];
      for (int iy = 0; iy < 4; iy++)
        for (int ix = 0; ix < 8; ix++) block[iy * 8 + ix] = (ix == 0 && iy == 0) ? dcs[h] : co[(h + iy * 2) * 8 + ix];
      if (t == 13) {
        idct2d_8x4(block);
        for (int iy = 0; iy < 8; iy++)
          for (int ix = 0; ix < 4; ix++) px[iy * 8 + h * 4 + ix] = block[iy * 4 + ix];
      } else {
        idct2d_4x8(block);
        for (int iy = 0; iy < 4; iy++)
          for (int ix = 0; ix < 8; ix++) px[(h * 4 + iy) * 8 + ix] = block[iy * 8 + ix];
      }
    }
  } else {  // AFV0..3
    int kind = t - 14;
    int afv_x = kind & 1, afv_y = kind / 2;
    float b00 = co[0], b01 = co[1], b10 = co[8];
    float dcs[3] = {(b00 + b10 + b01) * 4.0f, b00 + b10 - b01, b00 - b10};
    float coeff[16], block[32];
    for (int iy = 0; iy < 4; iy++)
      for (int ix = 0; ix < 4; ix++) coeff[iy * 4 + ix] = (ix == 0 && iy == 0) ? dcs[0] : co[iy * 2 * 8 + ix * 2];
    for (int i = 0; i < 16; i++) {
      float p = 0.0f;
      for (int j = 0; j < 16; j++) p += coeff[j] * c_afv[j * 16 + i];
      block[i] = p;
    }
    for (int iy = 0; iy < 4; iy++) {
      int by = afv_y ? 3 - iy : iy;
      for (int ix = 0; ix < 4; ix++) {
        int bx = afv_x ? 3 - ix : ix;
        px[(iy + afv_y * 4) * 8 + afv_x * 4 + ix] = block[by * 4 + bx];
      }
    }
    for (int iy = 0; iy < 4; iy++)
      for (int ix = 0; ix < 4; ix++) block[iy * 4 + ix] = (ix == 0 && iy == 0) ? dcs[1] : co[iy * 2 * 8 + ix * 2 + 1];
    idct2d_4x4(block);
    for (int iy = 0; iy < 4; iy++)
      for (int ix = 0; ix < 4; ix++) px[(iy + afv_y * 4) * 8 + (1 - afv_x) * 4 + ix] = block[iy * 4 + ix];
    for (int iy = 0; iy < 4; iy++)
      for (int ix = 0; ix < 8; ix++) block[iy * 8 + ix] = (ix == 0 && iy == 0) ? dcs[2] : co[(1 + iy * 2) * 8 + ix];
    idct2d_4x8(block);
    for (int iy = 0; iy < 4; iy++)
      for (int ix = 0; ix < 8; ix++) px[(iy + (1 - afv_y) * 4) * 8 + ix] = block[iy * 8 + ix];
  }
}

// noinline: one copy of each IDCT size in the kernel, whatever the number of call sites (instruction-cache footprint)
template <int N>
__device__ __noinline__ void warp_row_pass(float* ch, int lane_row, int stride) {
  float v[N];
#pragma unroll
  for (int i = 0; i < N; i++) v[i] = ch[lane_row * stride + i];
  idct1d<N>(v);
#pragma unroll
  for (int i = 0; i < N; i++) ch[lane_row * stride + i] = v[i];
}
template <int N>
__device__ __noinline__ void warp_col_pass(float* ch, int lane_col, int stride) {
  float v[N];
#pragma unroll
  for (int i = 0; i < N; i++) v[i] = ch[i * stride + lane_col];
  idct1d<N>(v);
#pragma unroll
  for (int i = 0; i < N; i++) ch[i * stride + lane_col] = v[i];
}

// k_dequant_idct takes the varblocks of the classes kClassWarp and kClassCta (k_block_plan). Types transformed in
// registers by k_idct_small are the 8x8-footprint transforms and plain DCTs with rows of <= 16 coefficients. Rows of 32
// (32x8 ... 32x32) unroll into ~300 KB of code and starve on instruction fetch, so they take the compact shared-memory
// path here.
constexpr int kIdctWarps = 8;   // per warp: dequantised work tiles 3 x kWarpBuf floats
constexpr size_t kLargeSmemBytes = size_t(kIdctWarps) * (3 * (32 * 33)) * sizeof(float);
constexpr int kWarpBuf = 32 * 33;  // floats per channel per warp

// Global in-place 1-D passes for varblocks with a dimension >= 64.
template <int N>
__device__ __noinline__ void big_line_pass(float* base, size_t elem_stride) {
  float v[N];
#pragma unroll 1
  for (int i = 0; i < N; i++) v[i] = base[i * elem_stride];
  idct1d_large<N>(v);
#pragma unroll 1
  for (int i = 0; i < N; i++) base[i * elem_stride] = v[i];
}
__device__ __forceinline__ void big_line_dispatch(int n, float* base, size_t elem_stride) {
  switch (n) {
    case 32: big_line_pass<32>(base, elem_stride); break;
    case 64: big_line_pass<64>(base, elem_stride); break;
    case 128: big_line_pass<128>(base, elem_stride); break;
    case 256: big_line_pass<256>(base, elem_stride); break;
    default: break;
  }
}

// Shared-memory warp path of one plain-DCT varblock with compile-time shape (index arithmetic becomes shifts).
template <int R, int C>
__device__ __forceinline__ void warp_dct_block(float* wbuf, int lane, const float* const* lfp, size_t lf_index,
                                               uint32_t lf_stride, float* const* planes, size_t px0, uint32_t plane_stride) {
  // wbuf: the three dequantised channels, coefficient (vf, hf) at [vf * (C + 1) + hf] (gather_dequant_tile)
  constexpr int stride = C + 1, cx = C / 8, cy = R / 8;
  if (lane < 3) {  // LLF (group.rs:227-236)
    float* ch = wbuf + lane * kWarpBuf;
    llf_small(lfp[lane] + lf_index, lf_stride, cy, cx, [&](int vf, int hf, float v) { ch[vf * stride + hf] = v; });
  }
  __syncwarp();
  for (int r = lane; r < 3 * R; r += 32) warp_row_pass<C>(wbuf + (r / R) * kWarpBuf, r % R, stride);
  __syncwarp();
  for (int r = lane; r < 3 * C; r += 32) warp_col_pass<R>(wbuf + (r / C) * kWarpBuf, r % C, stride);
  __syncwarp();
#pragma unroll
  for (int c = 0; c < 3; c++) {
    const float* ch = wbuf + c * kWarpBuf;
    float* pl = planes[c] + px0;
#pragma unroll 4
    for (int i = lane; i < R * C; i += 32) {
      const int y = i / C, x = i % C;
      pl[size_t(y) * plane_stride + x] = ch[y * stride + x];
    }
  }
}

__global__ void __launch_bounds__(kIdctWarps * 32) k_dequant_idct(const BatchDev B) {
  extern __shared__ float smem[];
  __shared__ uint32_t s_next;
  const uint32_t stream = blockIdx.x;
  if (B.status[stream] != 0) return;
  // this kernel's varblocks, from the block plan: the warp class, then the CTA class
  const uint32_t* cn = B.cls_n + size_t(stream) * kClassWords;
  const uint32_t nwarp = cn[kClassWarp], nbig = cn[kClassCta];
  if (nwarp + nbig == 0) return;
  const uint32_t* wlist = B.cls_list + size_t(stream) * 1024 + (cn[kClassReg8] + cn[kClassReg16_8] + cn[kClassReg16]);
  const uint32_t* blist = wlist + nwarp;
  const StreamDev sd = B.streams[stream];
  const FrameDev& F = B.frames[sd.frame];
  const uint32_t g = sd.group;
  const uint32_t gx = g % F.xg, gy = g / F.xg;
  const uint32_t bx0 = gx * 32, by0 = gy * 32;
  const int32_t* rq = reinterpret_cast<const int32_t*>(B.blob + F.raw_quant_off);
  const int8_t* ytox = reinterpret_cast<const int8_t*>(B.blob + F.ytox_off);
  const int8_t* ytob = reinterpret_cast<const int8_t*>(B.blob + F.ytob_off);
  float* planes[3] = {B.planes_a + F.plane_base, B.planes_a + F.plane_base + F.plane_size,
                      B.planes_a + F.plane_base + 2 * F.plane_size};
  const float* lfp[3] = {reinterpret_cast<const float*>(B.blob + F.lf_off[0]),
                         reinterpret_cast<const float*>(B.blob + F.lf_off[1]),
                         reinterpret_cast<const float*>(B.blob + F.lf_off[2])};
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* wbuf = smem + warp * (3 * kWarpBuf);
  if (threadIdx.x == 0) s_next = 0;
  __syncthreads();

  // everything of the dequantisation context but the coefficient pointers (set by the callers)
  auto setup = [&](uint32_t bx, uint32_t by, int t, DequantCtx& dq) {
    const size_t bidx = size_t(by0 + by) * F.xb + bx0 + bx;
    const uint32_t cx = c_cov_x[t], cy = c_cov_y[t];
    dq.num_coeffs = cx * cy * 64;
    dq.qx = dq.qy = dq.qb = nullptr;
    int qt = c_qtable[t];
    dq.mat = F.dequant_off[qt] >= 0 ? reinterpret_cast<const float*>(B.blob + F.dequant_off[qt])
                                    : B.dequant_default + B.dequant_default_off[qt];
    const size_t cidx = size_t((by0 + by) >> 3) * F.cxb + ((bx0 + bx) >> 3);
    dq.x_cc = F.base_correlation_x + float(ytox[cidx]) / float(F.color_factor);
    dq.b_cc = F.base_correlation_b + float(ytob[cidx]) / float(F.color_factor);
    dq.sy = F.inv_global_scale / float(rq[bidx]);
    dq.sx = dq.sy * F.x_dm;
    dq.sb = dq.sy * F.b_dm;
    dq.bias0 = F.quant_biases[0];
    dq.bias1 = F.quant_biases[1];
    dq.bias2 = F.quant_biases[2];
    dq.bias3 = F.quant_biases[3];
  };

  // ---- warp path: each warp grabs the next varblock of the warp class ----
  for (;;) {
    uint32_t li = 0;
    if (lane == 0) li = atomicAdd(&s_next, 1u);
    li = __shfl_sync(0xffffffffu, li, 0);
    if (li >= nwarp) break;
    const uint32_t e = wlist[li];
    const uint32_t seq = e & 1023, bx = (e >> 10) & 31, by = (e >> 15) & 31;
    const int t = int(e >> 20);
    const int cx = c_cov_x[t], cy = c_cov_y[t];
    DequantCtx dq;
    setup(bx, by, t, dq);
    const int R = 8 * cy, C = 8 * cx;
    const bool is_dct = (t == 0) || (t >= 4 && t <= 11);
    {  // the varblock's coefficients: list entries -> dequantised work tiles (wbuf, channels at stride kWarpBuf); plain DCTs
       // in [vf][hf] order with row stride C + 1, the 8x8 specials in storage order
      const uint32_t lR = 31 - __clz(uint32_t(R)), lC = 31 - __clz(uint32_t(C));
      const bool wide_l = R < C;
      const DeqParams D{dq.mat, dq.num_coeffs, dq.sx, dq.sy, dq.sb, dq.x_cc, dq.b_cc, dq.bias0, dq.bias1, dq.bias2, dq.bias3};
      const uint32_t zero_floats = is_dct ? uint32_t((R * (C + 1) + 3) & ~3) : 64u;
      gather_dequant_tile(B, F, g, seq, wbuf, uint32_t(kWarpBuf), zero_floats, D, uint32_t(lane), 32, true,
                          ListStage{nullptr, nullptr, 0}, [] { __syncwarp(); },
                          [=](uint32_t k) {
                            if (!is_dct) return k;
                            const uint32_t vf = wide_l ? k >> lC : k & (uint32_t(R) - 1), hf = wide_l ? k & (uint32_t(C) - 1) : k >> lR;
                            return vf * uint32_t(C + 1) + hf;
                          });
    }
    const size_t px0 = (size_t(by0 + by) * 8) * F.plane_stride + size_t(bx0 + bx) * 8;
    const size_t lf_index = size_t(by0 + by) * F.xb + bx0 + bx;
    if (is_dct && R == 32 && C == 32) {
      warp_dct_block<32, 32>(wbuf, lane, lfp, lf_index, F.xb, planes, px0, F.plane_stride);
    } else if (is_dct && R == 32 && C == 16) {
      warp_dct_block<32, 16>(wbuf, lane, lfp, lf_index, F.xb, planes, px0, F.plane_stride);
    } else if (is_dct && R == 16 && C == 32) {
      warp_dct_block<16, 32>(wbuf, lane, lfp, lf_index, F.xb, planes, px0, F.plane_stride);
    } else if (is_dct && R == 32 && C == 8) {
      warp_dct_block<32, 8>(wbuf, lane, lfp, lf_index, F.xb, planes, px0, F.plane_stride);
    } else if (is_dct && R == 8 && C == 32) {
      warp_dct_block<8, 32>(wbuf, lane, lfp, lf_index, F.xb, planes, px0, F.plane_stride);
    } else if (is_dct) {
      const int stride = C + 1;
      if (lane < 3) {  // LLF (group.rs:227-236, transform.rs:387-...)
        float* ch = wbuf + lane * kWarpBuf;
        const float* lf = lfp[lane] + size_t(by0 + by) * F.xb + bx0 + bx;
        if (cx == 1 && cy == 1) ch[0] = lf[0];
        else llf_small(lf, F.xb, cy, cx, [&](int vf, int hf, float v) { ch[vf * stride + hf] = v; });
      }
      __syncwarp();
      for (int r = lane; r < 3 * R; r += 32) {
        float* ch = wbuf + (r / R) * kWarpBuf;
        int row = r % R;
        if (C == 8) warp_row_pass<8>(ch, row, stride);
        else if (C == 16) warp_row_pass<16>(ch, row, stride);
        else warp_row_pass<32>(ch, row, stride);
      }
      __syncwarp();
      for (int r = lane; r < 3 * C; r += 32) {
        float* ch = wbuf + (r / C) * kWarpBuf;
        int col = r % C;
        if (R == 8) warp_col_pass<8>(ch, col, stride);
        else if (R == 16) warp_col_pass<16>(ch, col, stride);
        else warp_col_pass<32>(ch, col, stride);
      }
      __syncwarp();
      for (int c = 0; c < 3; c++) {
        const float* ch = wbuf + c * kWarpBuf;
        for (int i = lane; i < R * C; i += 32) {
          int y = i / C, x = i % C;
          planes[c][px0 + size_t(y) * F.plane_stride + x] = ch[y * stride + x];
        }
      }
    } else {
      // special transforms work on the storage layout (64 coefficients, stride 8)
      if (lane < 3) {
        float* ch = wbuf + lane * kWarpBuf;
        ch[0] = lfp[lane][size_t(by0 + by) * F.xb + bx0 + bx];
        float co[64];
        for (int i = 0; i < 64; i++) co[i] = ch[i];
        special_transform(t, co, ch + 64);
      }
      __syncwarp();
      for (int c = 0; c < 3; c++) {
        const float* ch = wbuf + c * kWarpBuf + 64;
        for (int i = lane; i < 64; i += 32) planes[c][px0 + size_t(i >> 3) * F.plane_stride + (i & 7)] = ch[i];
      }
    }
    __syncwarp();
  }
  __syncthreads();

  // ---- big varblocks (a dimension >= 64): CTA-cooperative, in place in HBM ----
  for (uint32_t bi = 0; bi < nbig; bi++) {
    const uint32_t e = blist[bi];
    const uint32_t seq = e & 1023, bx = (e >> 10) & 31, by = (e >> 15) & 31;
    const int t = int(e >> 20);
    const int cx = c_cov_x[t], cy = c_cov_y[t];
    const int R = 8 * cy, C = 8 * cx;
    DequantCtx dq;
    setup(bx, by, t, dq);
    const size_t px0 = (size_t(by0 + by) * 8) * F.plane_stride + size_t(bx0 + bx) * 8;
    const bool wide = R < C;
    // The varblock's own pixel area is its coefficient array (coefficient k at the place its dequantised value goes):
    // zero it, then write the non-zero entries dequantised — Y first (seeding X / B with cc * dy), then X and B with
    // mul_add(cc, dy, d), group.rs:100-133 at every position. Frames with several passes add the passes up as integers
    // in the same place first and convert afterwards.
    auto place = [&](uint32_t k) {
      const int vf = wide ? int(k) / C : int(k) % R, hf = wide ? int(k) % C : int(k) / R;
      return px0 + size_t(vf) * F.plane_stride + hf;
    };
    for (uint32_t k = threadIdx.x; k < dq.num_coeffs; k += blockDim.x) {
      const size_t o = place(k);
      planes[0][o] = 0.0f;
      planes[1][o] = 0.0f;
      planes[2][o] = 0.0f;
    }
    __syncthreads();
    const uint32_t lnc = 31 - __clz(dq.num_coeffs);
    if (F.num_passes == 1) {
      const uint32_t* base = list_base(B, F.section_base + g);
      const uint32_t* ow = base + kOffBase + seq * 3;
      const uint32_t o0 = __ldg(ow), o1 = __ldg(ow + 1), o2 = __ldg(ow + 2), o3 = min(__ldg(ow + 3), kListCap);
      for (uint32_t i = o0 + threadIdx.x; i < o1; i += blockDim.x) {  // Y
        const uint32_t e = __ldg(base + i), cpos = entry_pos(e, lnc);
        const size_t o = place(cpos);
        const float dy = adjust_quant_bias(entry_value(e, lnc), dq.bias1, dq.bias3) * (__ldg(dq.mat + dq.num_coeffs + cpos) * dq.sy);
        planes[1][o] = dy;
        planes[0][o] = dq.x_cc * dy;
        planes[2][o] = dq.b_cc * dy;
      }
      __syncthreads();
      for (uint32_t i = o1 + threadIdx.x; i < o3; i += blockDim.x) {  // X, then B
        const uint32_t e = __ldg(base + i), cpos = entry_pos(e, lnc);
        const size_t o = place(cpos);
        const bool is_x = i < o2;
        const uint32_t c = is_x ? 0u : 2u;
        const float d = adjust_quant_bias(entry_value(e, lnc), is_x ? dq.bias0 : dq.bias2, dq.bias3) *
                        (__ldg(dq.mat + c * dq.num_coeffs + cpos) * (is_x ? dq.sx : dq.sb));
        planes[c][o] = fmaf(is_x ? dq.x_cc : dq.b_cc, planes[1][o], d);
      }
      __syncthreads();
    } else {
      int32_t* ip[3] = {reinterpret_cast<int32_t*>(planes[0]), reinterpret_cast<int32_t*>(planes[1]), reinterpret_cast<int32_t*>(planes[2])};
      for (uint32_t p = 0; p < F.num_passes; p++) {
        const uint32_t* base = list_base(B, F.section_base + p * F.num_groups + g);
        const uint32_t* ow = base + kOffBase + seq * 3;
        const uint32_t o0 = __ldg(ow), o1 = __ldg(ow + 1), o2 = __ldg(ow + 2), o3 = min(__ldg(ow + 3), kListCap);
        for (uint32_t i = o0 + threadIdx.x; i < o3; i += blockDim.x) {
          const uint32_t e = __ldg(base + i);
          const uint32_t c = i < o1 ? 1u : (i < o2 ? 0u : 2u);  // entries come as Y, X, B
          ip[c][place(entry_pos(e, lnc))] += entry_value(e, lnc);
        }
        __syncthreads();
      }
      for (uint32_t k = threadIdx.x; k < dq.num_coeffs; k += blockDim.x) {
        const size_t o = place(k);
        float vx, vy, vb;
        dq.get_q(k, ip[0][o], ip[1][o], ip[2][o], vx, vy, vb);
        planes[0][o] = vx;
        planes[1][o] = vy;
        planes[2][o] = vb;
      }
      __syncthreads();
    }
    // LLF: rows then columns of the cy x cx LF samples, staged in shared memory.
    float* llf = smem;  // 3 * 32 * 33
    for (int r = threadIdx.x; r < 3 * cy; r += blockDim.x) {
      int c = r / cy, y = r % cy;
      float line[32];
      const float* lf = lfp[c] + size_t(by0 + by + y) * F.xb + bx0 + bx;
      for (int x = 0; x < cx; x++) line[x] = lf[x];
      rdct1d_dyn(line, cx);
      for (int x = 0; x < cx; x++) llf[c * kWarpBuf + y * 33 + x] = line[x];
    }
    __syncthreads();
    for (int r = threadIdx.x; r < 3 * cx; r += blockDim.x) {
      int c = r / cx, hf = r % cx;
      float line[32];
      for (int y = 0; y < cy; y++) line[y] = llf[c * kWarpBuf + y * 33 + hf];
      rdct1d_dyn(line, cy);
      for (int vf = 0; vf < cy; vf++) planes[c][px0 + size_t(vf) * F.plane_stride + hf] = line[vf];
    }
    __syncthreads();
    for (int r = threadIdx.x; r < 3 * R; r += blockDim.x)
      big_line_dispatch(C, planes[r / R] + px0 + size_t(r % R) * F.plane_stride, 1);
    __syncthreads();
    for (int r = threadIdx.x; r < 3 * C; r += blockDim.x)
      big_line_dispatch(R, planes[r / C] + px0 + (r % C), F.plane_stride);
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------
// K2a: register path for the 8x8-footprint transforms DCT8x8, DCT4x4, DCT4x8,
// DCT8x4 (the bulk of all varblocks). Eight threads own one block: thread i holds
// storage row i (coefficients k = 8 i .. 8 i + 7) of all three channels in
// registers; 1-D IDCTs run in registers, 8x8 transposes go through warp shuffles,
// loads and stores are 16-byte vectors. No shared-memory tile, no barriers.
// ---------------------------------------------------------------------------
__device__ __forceinline__ void transpose8(float (&v)[8], uint32_t r, uint32_t gmask) {
#pragma unroll
  for (int s = 1; s < 8; s <<= 1) {
#pragma unroll
    for (int j = 0; j < 8; j++) {
      if (j & s) continue;
      const float send = (r & s) ? v[j] : v[j | s];
      const float recv = __shfl_xor_sync(gmask, send, s);
      if (r & s) v[j] = recv;
      else v[j | s] = recv;
    }
  }
}

constexpr int kSmallThreads = 256;

template <int N>
__device__ __forceinline__ void transposeN(float* v, uint32_t r, uint32_t gmask) {
#pragma unroll
  for (int s = 1; s < N; s <<= 1) {
#pragma unroll
    for (int j = 0; j < N; j++) {
      if (j & s) continue;
      const float send = (r & s) ? v[j] : v[j | s];
      const float recv = __shfl_xor_sync(gmask, send, s);
      if (r & s) v[j] = recv;
      else v[j | s] = recv;
    }
  }
}

struct RegBlockCtx {
  const float* coeffs;  // the varblock's dequantised coefficient tile in shared memory: channel c at coeffs + c * cstride
  uint32_t cstride;
  const float* mat;       // dequant matrix of the block's table (channel 0)
  float* plane;           // plane set base (channel 0) + pixel offset of the block
  const float* lf;        // LF plane set base handled by caller
  size_t plane_size, plane_stride;
  uint32_t num_coeffs;
  float sx, sy, sb, x_cc, b_cc, bias0, bias1, bias2, bias3;
};

__device__ __forceinline__ DeqParams deq_of(const RegBlockCtx& X) {
  return DeqParams{X.mat, X.num_coeffs, X.sx, X.sy, X.sb, X.x_cc, X.b_cc, X.bias0, X.bias1, X.bias2, X.bias3};
}

// One plain-DCT varblock of min(R,C) = NT storage rows x max(R,C) = L entries, NT threads (lanes r = 0..NT-1 of
// an aligned lane group). TALL: rows >= cols, storage [hf][vf]; else storage [vf][hf] (tests.rs:123-136).
template <int NT, int L, bool TALL>
__device__ __forceinline__ void reg_dct_block(const RegBlockCtx& X, const float* const* lfp, uint32_t lf_stride, uint32_t r,
                                              uint32_t gmask, bool valid) {
  constexpr int M = L / NT;
  constexpr int CY = TALL ? L / 8 : NT / 8, CX = TALL ? NT / 8 : L / 8;  // covered blocks
#pragma unroll 1
  for (int c = 0; c < 3; c++) {
    float w[L];
    {
      const float4* tc = reinterpret_cast<const float4*>(X.coeffs + c * X.cstride + r * L);  // storage row r of channel c
#pragma unroll
      for (int j4 = 0; j4 < L / 4; j4++) {
        const float4 t = tc[j4];
        w[4 * j4] = t.x;
        w[4 * j4 + 1] = t.y;
        w[4 * j4 + 2] = t.z;
        w[4 * j4 + 3] = t.w;
      }
    }
    // LLF: rows < (TALL ? CX : CY), entries < (TALL ? CY : CX)
    if (r < uint32_t(TALL ? CX : CY)) {
      const float* lf = lfp[c];
      if (CX == 1 && CY == 1) {
        w[0] = lf[0];
      } else {
        llf_small(lf, lf_stride, CY, CX, [&](int vf, int hf, float val) {
          const int row = TALL ? hf : vf, ent = TALL ? vf : hf;
          if (uint32_t(row) == r) {
#pragma unroll
            for (int e = 0; e < 4; e++)
              if (e == ent) w[e] = val;
          }
        });
      }
    }
    idct1d<L>(w);
    float* plane = X.plane + size_t(c) * X.plane_size;
#pragma unroll
    for (int q = 0; q < M; q++) {
      float* u = w + q * NT;
      transposeN<NT>(u, r, gmask);
      idct1d<NT>(u);
      if (TALL) {  // thread r holds pixel row y = q NT + r, x = 0..NT-1
        if (valid) {
          float4* d = reinterpret_cast<float4*>(plane + size_t(q * NT + r) * X.plane_stride);
#pragma unroll
          for (int j4 = 0; j4 < NT / 4; j4++) d[j4] = make_float4(u[4 * j4], u[4 * j4 + 1], u[4 * j4 + 2], u[4 * j4 + 3]);
        }
      } else {  // thread r holds column x = q NT + r; transpose back to rows
        transposeN<NT>(u, r, gmask);
        if (valid) {
          float4* d = reinterpret_cast<float4*>(plane + size_t(r) * X.plane_stride + q * NT);
#pragma unroll
          for (int j4 = 0; j4 < NT / 4; j4++) d[j4] = make_float4(u[4 * j4], u[4 * j4 + 1], u[4 * j4 + 2], u[4 * j4 + 3]);
        }
      }
    }
  }
}

// KIND selects the coefficient-row length handled by this instantiation (register budget): 0: L = 8 (class kClassReg8:
// types 0, 3, 12, 13), 1: L = 16 (kClassReg16_8 and kClassReg16: types 6, 7, 4).

// Shared memory for the coefficient tiles of the lane groups of one CTA: every class of a KIND needs 32 x 8 lanes x 3 x NC
// words with NC = 64 / 128 coefficients per channel (the 16-lane class holds 2x the coefficients in half the groups).
template <int KIND>
__host__ __device__ constexpr size_t small_tile_bytes() {
  return size_t(kSmallThreads / 8) * 3 * (KIND == 0 ? 64 : 128) * sizeof(int32_t);
}
// Behind the tiles: the staged offset words (kOffWords) and the first kStageEntries entries of the group's list,
// delivered by two bulk copies issued by thread 0. A CTA whose group has no varblock of its KIND issues none.
constexpr uint32_t kStageEntries = 8192;
template <int KIND>
constexpr size_t small_smem_bytes() {
  return small_tile_bytes<KIND>() + size_t(kOffWords + kStageEntries) * sizeof(uint32_t);
}

template <int KIND>
__global__ void __launch_bounds__(kSmallThreads, KIND == 0 ? 3 : 2) k_idct_small(const BatchDev B) {
  extern __shared__ __align__(16) float s_tiles[];
  __shared__ __align__(8) uint64_t s_bar[2];
  const uint32_t stream = blockIdx.x;
  if (B.status[stream] != 0) return;
  // this kernel's varblocks, from the block plan: KIND 0: the 8-lane class; KIND 1: its 8-lane class, then the 16-lane one
  const uint32_t* cn = B.cls_n + size_t(stream) * kClassWords;
  const uint32_t n8 = KIND == 0 ? cn[kClassReg8] : cn[kClassReg16_8], n16 = KIND == 0 ? 0u : cn[kClassReg16];
  if (n8 + n16 == 0) return;  // before the staging copies: most groups have no varblock of one of the two kinds
  const uint32_t* list = B.cls_list + size_t(stream) * 1024 + (KIND == 0 ? 0u : cn[kClassReg8]);
  const StreamDev sd = B.streams[stream];
  const FrameDev& F = B.frames[sd.frame];
  const uint32_t g = sd.group;
  uint32_t* const s_off = reinterpret_cast<uint32_t*>(s_tiles + small_tile_bytes<KIND>() / 4);
  uint32_t* const s_ent = s_off + kOffWords;
  if (threadIdx.x == 0) {
    mbar_init(&s_bar[0], 1);
    mbar_init(&s_bar[1], 1);
    mbar_fence_init();
    // pass-0 list of this group: offset words, and the head of the entries (whatever lies behind the last entry is
    // copied too and never looked at)
    const uint32_t* base = list_base(B, F.section_base + g);
    bulk_load(s_off, base + kOffBase, kOffWords * 4, &s_bar[0]);
    bulk_load(s_ent, base, kStageEntries * 4, &s_bar[1]);
  }
  const uint32_t bx0 = (g % F.xg) * 32, by0 = (g / F.xg) * 32;
  __syncthreads();  // the barriers are initialised
  mbar_wait(&s_bar[0], 0);
  mbar_wait(&s_bar[1], 0);
  const ListStage stage{s_off, s_ent, kStageEntries};
  const int32_t* rq = reinterpret_cast<const int32_t*>(B.blob + F.raw_quant_off);
  const int8_t* ytox = reinterpret_cast<const int8_t*>(B.blob + F.ytox_off);
  const int8_t* ytob = reinterpret_cast<const int8_t*>(B.blob + F.ytob_off);
  const float bias0 = F.quant_biases[0], bias1 = F.quant_biases[1], bias2 = F.quant_biases[2], bias3 = F.quant_biases[3];

  auto setup_ctx = [&](uint32_t e, RegBlockCtx& X, const float* (&lfp)[3], int& t) {
    const uint32_t bx = (e >> 10) & 31, by = (e >> 15) & 31;
    const size_t bidx = size_t(by0 + by) * F.xb + bx0 + bx;
    t = int(e >> 20);
    const int qt = c_qtable[t];
    X.mat = F.dequant_off[qt] >= 0 ? reinterpret_cast<const float*>(B.blob + F.dequant_off[qt]) : B.dequant_default + B.dequant_default_off[qt];
    X.num_coeffs = uint32_t(c_cov_x[t]) * c_cov_y[t] * 64;
    const size_t cidx = size_t((by0 + by) >> 3) * F.cxb + ((bx0 + bx) >> 3);
    X.x_cc = F.base_correlation_x + float(ytox[cidx]) / float(F.color_factor);
    X.b_cc = F.base_correlation_b + float(ytob[cidx]) / float(F.color_factor);
    X.sy = F.inv_global_scale / float(rq[bidx]);
    X.sx = X.sy * F.x_dm;
    X.sb = X.sy * F.b_dm;
    X.bias0 = bias0; X.bias1 = bias1; X.bias2 = bias2; X.bias3 = bias3;
    X.plane = B.planes_a + F.plane_base + (size_t(by0 + by) * 8) * F.plane_stride + size_t(bx0 + bx) * 8;
    X.plane_size = F.plane_size;
    X.plane_stride = F.plane_stride;
    for (int c = 0; c < 3; c++) lfp[c] = reinterpret_cast<const float*>(B.blob + F.lf_off[c]) + bidx;
  };

  // ---------------- class 0: 8 lanes per block ----------------
  {
    const uint32_t r = threadIdx.x & 7;
    const uint32_t gmask = 0xffu << (threadIdx.x & 24);
    const uint32_t count = n8;
    const uint32_t iters = (count + kSmallThreads / 8 - 1) / (kSmallThreads / 8);
    // class-list entries are loaded one iteration ahead: the varblock's set-up loads then start at once
    uint32_t e_next = iters ? list[((threadIdx.x >> 3) < count ? (threadIdx.x >> 3) : 0u)] : 0u;
    for (uint32_t it = 0; it < iters; it++) {
      const uint32_t li = it * (kSmallThreads / 8) + (threadIdx.x >> 3);
      const bool valid = li < count;
      const uint32_t e = e_next;  // invalid lanes hold the class's first entry
      if (it + 1 < iters) e_next = list[(li + kSmallThreads / 8 < count ? li + kSmallThreads / 8 : 0u)];
      RegBlockCtx X;
      const float* lfp[3];
      int t;
      const uint32_t seq = e & 1023;
      setup_ctx(e, X, lfp, t);
      constexpr uint32_t NC = KIND == 0 ? 64 : 128;
      float* tile = s_tiles + (threadIdx.x >> 3) * 3 * NC;
      gather_dequant_tile(B, F, g, seq, tile, NC, NC, deq_of(X), r, 8, valid, stage, [&] { __syncwarp(gmask); },
                          [](uint32_t pos) { return pos; });
      X.coeffs = tile;
      X.cstride = NC;
      if constexpr (KIND == 1) {
        if (t == 6) reg_dct_block<8, 16, true>(X, lfp, F.xb, r, gmask, valid);
        else reg_dct_block<8, 16, false>(X, lfp, F.xb, r, gmask, valid);
      } else if (t == 0) {
        reg_dct_block<8, 8, true>(X, lfp, F.xb, r, gmask, valid);
      } else {
        // DCT4x4 / DCT4x8 / DCT8x4: all three channels at once (64 coefficients each)
        float v[3][8];
#pragma unroll
        for (int c = 0; c < 3; c++) {  // storage row r of the dequantised tile
          const float4* tp = reinterpret_cast<const float4*>(X.coeffs + c * X.cstride + r * 8);
          const float4 a = tp[0], b = tp[1];
          v[c][0] = a.x; v[c][1] = a.y; v[c][2] = a.z; v[c][3] = a.w;
          v[c][4] = b.x; v[c][5] = b.y; v[c][6] = b.z; v[c][7] = b.w;
        }
#pragma unroll
        for (int c = 0; c < 3; c++) {
          float (&w)[8] = v[c];
          if (r == 0) w[0] = lfp[c][0];
          float* plane = X.plane + size_t(c) * X.plane_size;
          const uint32_t base = threadIdx.x & 24;
          if (t == 12 || t == 13) {
            // DC pair (transform.rs:617-620): dcs = [c0 + c8, c0 - c8], c0 = row 0 col 0, c8 = row 1 col 0
            const float c0 = __shfl_sync(gmask, w[0], base), c8 = __shfl_sync(gmask, w[0], base + 1);
            if (r == 0) w[0] = c0 + c8;
            if (r == 1) w[0] = c0 - c8;
            idct1d<8>(w);             // t=13: over vf -> y; t=12: over hf -> x
            transposeN<8>(w, r, gmask);  // thread j holds entries i = h + 2 f (f = hf for 8x4, vf for 4x8)
            float a4[4] = {w[0], w[2], w[4], w[6]}, b4[4] = {w[1], w[3], w[5], w[7]};
            idct1d<4>(a4);
            idct1d<4>(b4);
            if (t == 13) {  // DCT8X4: thread y: half 0 -> x 0..3, half 1 -> x 4..7
              if (valid) {
                float4* d = reinterpret_cast<float4*>(plane + size_t(r) * X.plane_stride);
                d[0] = make_float4(a4[0], a4[1], a4[2], a4[3]);
                d[1] = make_float4(b4[0], b4[1], b4[2], b4[3]);
              }
            } else {  // DCT4X8: thread x holds the column: half 0 -> y 0..3, half 1 -> y 4..7
              w[0] = a4[0]; w[1] = a4[1]; w[2] = a4[2]; w[3] = a4[3];
              w[4] = b4[0]; w[5] = b4[1]; w[6] = b4[2]; w[7] = b4[3];
              transposeN<8>(w, r, gmask);
              if (valid) {
                float4* d = reinterpret_cast<float4*>(plane + size_t(r) * X.plane_stride);
                d[0] = make_float4(w[0], w[1], w[2], w[3]);
                d[1] = make_float4(w[4], w[5], w[6], w[7]);
              }
            }
          } else {  // DCT4X4 (transform.rs:579-612): thread i = qy + 2 hf holds j = qx + 2 vf
            const float c00 = __shfl_sync(gmask, w[0], base), c01 = __shfl_sync(gmask, w[1], base);
            const float c10 = __shfl_sync(gmask, w[0], base + 1), c11 = __shfl_sync(gmask, w[1], base + 1);
            if (r == 0) {
              w[0] = c00 + c01 + c10 + c11;  // quadrant (0,0)
              w[1] = c00 + c01 - c10 - c11;  // quadrant (0,1)
            }
            if (r == 1) {
              w[0] = c00 - c01 + c10 - c11;  // quadrant (1,0)
              w[1] = c00 - c01 - c10 + c11;  // quadrant (1,1)
            }
            float a4[4] = {w[0], w[2], w[4], w[6]}, b4[4] = {w[1], w[3], w[5], w[7]};  // over vf for qx = 0 / 1
            idct1d<4>(a4);
            idct1d<4>(b4);
#pragma unroll
            for (int y = 0; y < 4; y++) {
              w[2 * y] = a4[y];
              w[2 * y + 1] = b4[y];
            }
            transposeN<8>(w, r, gmask);  // thread j = qx + 2 y holds i = qy + 2 hf
            float p4[4] = {w[0], w[2], w[4], w[6]}, q4[4] = {w[1], w[3], w[5], w[7]};  // over hf for qy = 0 / 1
            idct1d<4>(p4);
            idct1d<4>(q4);
            if (valid) {
              const uint32_t qx = r & 1, y = r >> 1;
              *reinterpret_cast<float4*>(plane + size_t(y) * X.plane_stride + qx * 4) = make_float4(p4[0], p4[1], p4[2], p4[3]);
              *reinterpret_cast<float4*>(plane + size_t(4 + y) * X.plane_stride + qx * 4) = make_float4(q4[0], q4[1], q4[2], q4[3]);
            }
          }
        }
      }
    }
  }
  // ---------------- class 1: 16 lanes per block ----------------
  if constexpr (KIND == 1) {
    const uint32_t r = threadIdx.x & 15;
    const uint32_t gmask = 0xffffu << (threadIdx.x & 16);
    const uint32_t count = n16;
    const uint32_t iters = (count + kSmallThreads / 16 - 1) / (kSmallThreads / 16);
    // class-list entries are loaded one iteration ahead: the varblock's set-up loads then start at once
    uint32_t e_next = iters ? list[n8 + ((threadIdx.x >> 4) < count ? (threadIdx.x >> 4) : 0u)] : 0u;
    for (uint32_t it = 0; it < iters; it++) {
      const uint32_t li = it * (kSmallThreads / 16) + (threadIdx.x >> 4);
      const bool valid = li < count;
      const uint32_t e = e_next;  // invalid lanes hold the class's first entry
      if (it + 1 < iters) e_next = list[n8 + (li + kSmallThreads / 16 < count ? li + kSmallThreads / 16 : 0u)];
      RegBlockCtx X;
      const float* lfp[3];
      int t;
      const uint32_t seq = e & 1023;
      setup_ctx(e, X, lfp, t);
      constexpr uint32_t NC = 256;
      float* tile = s_tiles + (threadIdx.x >> 4) * 3 * NC;
      gather_dequant_tile(B, F, g, seq, tile, NC, NC, deq_of(X), r, 16, valid, stage, [&] { __syncwarp(gmask); },
                          [](uint32_t pos) { return pos; });
      X.coeffs = tile;
      X.cstride = NC;
      reg_dct_block<16, 16, true>(X, lfp, F.xb, r, gmask, valid);
    }
  }
}

// ===========================================================================
// K3-K5: loop filters and colour
// ===========================================================================

__device__ __forceinline__ int mirror(int v, int s) {  // util/mirror.rs:8
  while (v < 0 || v >= s) v = v < 0 ? -v - 1 : 2 * s - v - 1;
  return v;
}

// ===========================================================================
// K3+K4+K5 fused: Gaborish -> EPF0 -> EPF1 -> EPF2 -> XYB -> sRGB -> store, one
// shared-memory tile per CTA, templated on the frame's filter configuration.
//
// * Every window cell holds the value of its *mirrored* image pixel, and every
//   stage evaluates out-of-image cells at the mirrored coordinate, so halo
//   cells hold exactly what the reference's mirror-padded rows hold
//   (render/simple_pipeline/run_stage.rs:127-134) and stages chain in the tile.
// * EPF sums of absolute differences are built from channel-combined differences
//   D_o(c) = sum_ch scale_ch * |I_ch(c) - I_ch(c + o)| (epf0.rs:157-168 /
//   epf1.rs:98-101 evaluate the same sums per pixel). EPF stage 0 stores its six
//   difference maps in shared memory; stages 1 and 2 need only D_(1,0) and
//   D_(0,1) and recompute them from the source cells, which keeps the Gaborish +
//   EPF 2 tile at two plane buffers (69 KB) and spares each stage a barrier.
// * HBM traffic: one read of the IDCT planes (+ halo) and one write of the output.
// ===========================================================================
constexpr int kTW = 64, kTH = 32;

struct FusedTiles {
  const uint32_t* tile_prefix;  // [num_frames + 1], kTW x kTH tiles
  uint32_t num_frames;
  uint32_t tile_begin;          // first tile of this launch (frame ranges are launched separately so that the
                                // D2H copy of finished frames overlaps the filtering of the next ones)
};

template <bool GAB, int EPF>
struct FCfg {
  static constexpr int H = (GAB ? 1 : 0) + (EPF >= 3 ? 3 : 0) + (EPF >= 1 ? 2 : 0) + (EPF >= 2 ? 1 : 0);
  static constexpr int WW = kTW + 2 * H, WH = kTH + 2 * H, NC = WW * WH;
  static constexpr int NMAPS = EPF >= 3 ? 6 : 0;  // only EPF stage 0 reads stored maps; stages 1 and 2 recompute theirs
  static constexpr int SBW = WW / 8 + 2, SBH = WH / 8 + 2;  // sigma blocks covering the window
  static constexpr size_t kSmemBytes = sizeof(float) * (size_t(6 + NMAPS) * NC + SBW * SBH);
  // EPF <= 2 tiles (<= 69 KB): 384 threads at <= 56 registers, 3 CTAs per SM. At 512 threads the same 3 CTAs need <= 40
  // registers, where the vector path spills (176 B stored / 232 B loaded per thread) and filters a 4K batch 22 % slower
  // (DESIGN §7). The EPF 3 tile (172 KB) fits one CTA per SM at any size, so it keeps 512 threads: at 384 it has a
  // quarter fewer warps per SM, and config 4 then measured 8 % slower than with stored maps at 512 threads.
  static constexpr int kThreads = EPF >= 3 ? 512 : 384;
  static constexpr int kMinCtas = EPF >= 3 ? 1 : 3;
};

// The region slicer (host/region.h) selects HF groups from this tile and halo: they must agree for every configuration.
template <bool GAB, int EPF>
constexpr bool region_geometry_matches() {
  return FCfg<GAB, EPF>::H == int(jxg::filter_halo(GAB, EPF)) && kTW == int(jxg::kFilterTileW) && kTH == int(jxg::kFilterTileH);
}
static_assert(region_geometry_matches<false, 0>() && region_geometry_matches<false, 1>() && region_geometry_matches<false, 2>() &&
                  region_geometry_matches<false, 3>() && region_geometry_matches<true, 0>() && region_geometry_matches<true, 1>() &&
                  region_geometry_matches<true, 2>() && region_geometry_matches<true, 3>(),
              "host/region.h filter_halo / kFilterTileW / kFilterTileH differ from the fused filter kernel");

// Cell -> source position. INTERIOR tiles (window fully inside the image) skip every range / mirror computation.
template <bool INTERIOR, int WW>
__device__ __forceinline__ bool cell_source(int lx, int ly, int wx0, int wy0, int w, int h, int r, int& o, int& mx, int& my) {
  if (INTERIOR) {
    mx = wx0 + lx;
    my = wy0 + ly;
    o = ly * WW + lx;
    return true;
  }
  const int gx = wx0 + lx, gy = wy0 + ly;
  if (gx < -r || gx > w - 1 + r || gy < -r || gy > h - 1 + r) return false;  // never needed by a valid output
  mx = mirror(gx, w);
  my = mirror(gy, h);
  o = (my - wy0) * WW + (mx - wx0);
  return true;
}

// One EPF stage. src/dst: [3][NC]; maps: [6][NC], stage 0 only; M = margin of the output region (compile time).
template <int STAGE, int WW, int WH, int H, int SBW, int M, bool INTERIOR>
__device__ __forceinline__ void epf_stage(const FrameDev& F, const float* src, float* dst, float* maps, const float* sig,
                                          int wx0, int wy0, int sbx0, int sby0) {
  constexpr int NC = WW * WH;
  const int w = int(F.width), h = int(F.height);
  const float s0 = F.epf_channel_scale[0], s1 = F.epf_channel_scale[1], s2 = F.epf_channel_scale[2];
  // ---- phase A (stage 0): difference maps over the source-valid area ----
  if (STAGE == 0) {
    constexpr int NO = 6;
    constexpr int MP = M - 3;  // margin of valid source cells
    constexpr int ox[6] = {1, 0, 2, 0, 1, 1}, oy[6] = {0, 1, 0, 2, 1, -1};  // (1,0) (0,1) (2,0) (0,2) (1,1) (1,-1)
    constexpr int aw = WW - 2 * MP, ah = WH - 2 * MP;
    for (int idx = threadIdx.x; idx < aw * ah; idx += blockDim.x) {
      const int lx = MP + idx % aw, ly = MP + idx / aw;
      const int o = ly * WW + lx;
      const float c0 = src[o], c1 = src[NC + o], c2 = src[2 * NC + o];
#pragma unroll
      for (int k = 0; k < NO; k++) {
        const int nx = lx + ox[k], ny = ly + oy[k];
        if (nx >= WW - MP || ny >= WH - MP || ny < MP) continue;
        const int on = o + oy[k] * WW + ox[k];
        maps[k * NC + o] = fmaf(fabsf(src[on] - c0), s0, fmaf(fabsf(src[NC + on] - c1), s1, fabsf(src[2 * NC + on] - c2) * s2));
      }
    }
    __syncthreads();
  }
  // ---- phase B ----
  const float kMinSigma = -3.90524291751269967465540850526868f;
  const float sigma_scale = STAGE == 0 ? F.epf_pass0_sigma_scale : (STAGE == 1 ? 1.0f : F.epf_pass2_sigma_scale);
  const float sm = sigma_scale * 1.65f, bsm = sm * F.epf_border_sad_mul;
  constexpr int R = H - M;  // halo still needed after this stage
  constexpr int bw_ = kTW + 2 * R, bh_ = kTH + 2 * R;
  // D_(1,0) and D_(0,1) at cell c, summed as phase A sums them
  auto diff = [&](int a, int b) {
    return fmaf(fabsf(src[b] - src[a]), s0, fmaf(fabsf(src[NC + b] - src[NC + a]), s1, fabsf(src[2 * NC + b] - src[2 * NC + a]) * s2));
  };
  auto Dh = [&](int c) { return STAGE == 0 ? maps[c] : diff(c, c + 1); };
  auto Dv = [&](int c) { return STAGE == 0 ? maps[NC + c] : diff(c, c + WW); };
  for (int idx = threadIdx.x; idx < bw_ * bh_; idx += blockDim.x) {
    const int lx = M + idx % bw_, ly = M + idx / bw_;
    int o, mx, my;
    if (!cell_source<INTERIOR, WW>(lx, ly, wx0, wy0, w, h, R, o, mx, my)) continue;
    const int od = ly * WW + lx;
    const float inv_sigma_px = sig[((my >> 3) - sby0) * SBW + ((mx >> 3) - sbx0)];
    if (inv_sigma_px < kMinSigma) {
#pragma unroll
      for (int c = 0; c < 3; c++) dst[c * NC + od] = src[c * NC + o];
      continue;
    }
    const bool border = (((my + 1) & 7) < 2) || (((mx + 1) & 7) < 2);  // x or y == 0 or 7 (mod 8)
    const float inv_s = inv_sigma_px * (border ? bsm : sm);
    if (STAGE == 2) {
      // neighbours in the reference's order: up, left, right, down (epf2.rs:83)
      const float sad[4] = {Dv(o - WW), Dh(o - 1), Dh(o), Dv(o)};
      const int offs[4] = {-WW, -1, 1, WW};
      float wacc = 1.0f, acc[3] = {src[o], src[NC + o], src[2 * NC + o]};
#pragma unroll
      for (int k = 0; k < 4; k++) {
        float wt = fmaxf(fmaf(sad[k], inv_s, 1.0f), 0.0f);
        wacc += wt;
#pragma unroll
        for (int c = 0; c < 3; c++) acc[c] = fmaf(wt, src[c * NC + o + offs[k]], acc[c]);
      }
      float inv_w = 1.0f / wacc;
#pragma unroll
      for (int c = 0; c < 3; c++) dst[c * NC + od] = acc[c] * inv_w;
      continue;
    }
    auto plus_sum = [&](auto D, int base) { return D(base - WW) + D(base - 1) + D(base) + D(base + 1) + D(base + WW); };
    if (STAGE == 1) {
      const float sad[4] = {plus_sum(Dv, o - WW), plus_sum(Dh, o - 1), plus_sum(Dh, o), plus_sum(Dv, o)};
      const int offs[4] = {-WW, -1, 1, WW};
      float wts[4], wsum = 1.0f;
#pragma unroll
      for (int k = 0; k < 4; k++) {
        wts[k] = fmaxf(fmaf(sad[k], inv_s, 1.0f), 0.0f);
        wsum += wts[k];
      }
      const float inv_w = 1.0f / wsum;
#pragma unroll
      for (int c = 0; c < 3; c++) {
        const float* p = src + c * NC + o;
        float v = p[0];
#pragma unroll
        for (int k = 3; k >= 0; k--) v = fmaf(p[offs[k]], wts[k], v);
        dst[c * NC + od] = v * inv_w;
      }
      continue;
    }
    // STAGE 0: 12 neighbours (epf0.rs:182-195 order)
    auto MB = [&](int c) { return maps[2 * NC + c]; };  // (2,0)
    auto MD = [&](int c) { return maps[3 * NC + c]; };  // (0,2)
    auto ME = [&](int c) { return maps[4 * NC + c]; };  // (1,1)
    auto MF = [&](int c) { return maps[5 * NC + c]; };  // (1,-1)
    const int offs[12] = {-2 * WW, -WW - 1, -WW, -WW + 1, -2, -1, 1, 2, WW - 1, WW, WW + 1, 2 * WW};
    const float sad[12] = {
        plus_sum(MD, o - 2 * WW), plus_sum(ME, o - WW - 1), plus_sum(Dv, o - WW), plus_sum(MF, o),
        plus_sum(MB, o - 2),      plus_sum(Dh, o - 1),      plus_sum(Dh, o),      plus_sum(MB, o),
        plus_sum(MF, o + WW - 1), plus_sum(Dv, o),          plus_sum(ME, o),      plus_sum(MD, o)};
    float wts[12], wsum = 1.0f;
#pragma unroll
    for (int k = 0; k < 12; k++) {
      wts[k] = fmaxf(fmaf(sad[k], inv_s, 1.0f), 0.0f);
      wsum += wts[k];
    }
    const float inv_w = 1.0f / wsum;
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const float* p = src + c * NC + o;
      float v = p[0];
#pragma unroll
      for (int k = 11; k >= 0; k--) v = fmaf(p[offs[k]], wts[k], v);
      dst[c * NC + od] = v * inv_w;
    }
  }
  __syncthreads();
}

template <bool GAB, int EPF, bool INTERIOR>
__device__ __forceinline__ void filter_tile(const BatchDev& B, const FrameDev& F, const float* src_planes, float* smem, int x0, int y0) {
  using C = FCfg<GAB, EPF>;
  constexpr int H = C::H, WW = C::WW, WH = C::WH, NC = C::NC;
  float* bufA = smem;
  float* bufB = smem + 3 * NC;
  float* maps = smem + 6 * NC;
  float* sig = maps + C::NMAPS * NC;
  const int w = int(F.width), h = int(F.height);
  const int wx0 = x0 - H, wy0 = y0 - H;
  // ---- load, pre-mirrored; cells farther than H outside the image are never needed ----
  for (int idx = threadIdx.x; idx < NC; idx += blockDim.x) {
    const int lx = idx % WW, ly = idx / WW;
    size_t so;
    if (INTERIOR) {
      so = size_t(wy0 + ly) * F.plane_stride + (wx0 + lx);
    } else {
      const int gx = wx0 + lx, gy = wy0 + ly;
      if (gx > w - 1 + H || gy > h - 1 + H) continue;
      so = size_t(mirror(gy, h)) * F.plane_stride + mirror(gx, w);
    }
#pragma unroll
    for (int c = 0; c < 3; c++) bufA[c * NC + idx] = src_planes[F.plane_base + c * F.plane_size + so];
  }
  const int sbx0 = max(wx0, 0) >> 3, sby0 = max(wy0, 0) >> 3;
  if (EPF > 0) {  // features/epf.rs:54-79, once per 8x8 block touched by the window
    for (int idx = threadIdx.x; idx < C::SBW * C::SBH; idx += blockDim.x) {
      const int bx = sbx0 + idx % C::SBW, by = sby0 + idx / C::SBW;
      float v = 0.0f;
      if (bx < int(F.xb) && by < int(F.yb)) {
        const size_t bidx = size_t(by) * F.xb + bx;
        const int32_t raw_quant = reinterpret_cast<const int32_t*>(B.blob + F.raw_quant_off)[bidx];
        const uint32_t sharp = (B.blob + F.epf_off)[bidx];
        float sigma_quant = F.epf_quant_mul / (F.quant_scale * float(raw_quant) * -1.1715728752538099024f);
        v = 1.0f / fminf(sigma_quant * F.epf_sharp_lut[sharp], -1e-4f);
      }
      sig[idx] = v;
    }
  }
  __syncthreads();
  float* cur = bufA;
  float* nxt = bufB;
  constexpr int M_GAB = GAB ? 1 : 0;
  constexpr int M_E0 = M_GAB + (EPF >= 3 ? 3 : 0);
  constexpr int M_E1 = M_E0 + (EPF >= 1 ? 2 : 0);
  constexpr int M_E2 = M_E1 + (EPF >= 2 ? 1 : 0);
  static_assert(M_E2 == H, "margins must add up to the halo");
  if (GAB) {  // gaborish.rs:40-88
    constexpr int R = H - M_GAB;
    constexpr int rw = kTW + 2 * R, rh = kTH + 2 * R;
    for (int idx = threadIdx.x; idx < rw * rh; idx += blockDim.x) {
      const int lx = M_GAB + idx % rw, ly = M_GAB + idx / rw;
      int o, mx, my;
      if (!cell_source<INTERIOR, WW>(lx, ly, wx0, wy0, w, h, R, o, mx, my)) continue;
#pragma unroll
      for (int c = 0; c < 3; c++) {
        const float* p = cur + c * NC + o;
        float sum = p[0] * F.gab_k0[c];
        sum = fmaf(F.gab_k1[c], p[-WW] + p[-1] + p[WW] + p[1], sum);
        sum = fmaf(F.gab_k2[c], p[-WW - 1] + p[-WW + 1] + p[WW - 1] + p[WW + 1], sum);
        nxt[c * NC + ly * WW + lx] = sum;
      }
    }
    __syncthreads();
    float* t = cur; cur = nxt; nxt = t;
  }
  if (EPF >= 3) {
    epf_stage<0, WW, WH, H, C::SBW, M_E0, INTERIOR>(F, cur, nxt, maps, sig, wx0, wy0, sbx0, sby0);
    float* t = cur; cur = nxt; nxt = t;
  }
  if (EPF >= 1) {
    epf_stage<1, WW, WH, H, C::SBW, M_E1, INTERIOR>(F, cur, nxt, maps, sig, wx0, wy0, sbx0, sby0);
    float* t = cur; cur = nxt; nxt = t;
  }
  if (EPF >= 2) {
    epf_stage<2, WW, WH, H, C::SBW, M_E2, INTERIOR>(F, cur, nxt, maps, sig, wx0, wy0, sbx0, sby0);
    float* t = cur; cur = nxt; nxt = t;
  }
  // ---- colour + store of the kTW x kTH core ----
  const int tw = min(kTW, w - x0), th = min(kTH, h - y0);
  uint8_t* out_base = static_cast<uint8_t*>(F.out_ptr);
  if (F.output_format == JXG_FORMAT_XYB_F32_PLANAR) {
    for (int idx = threadIdx.x; idx < kTW * th; idx += blockDim.x) {
      const int lx = idx % kTW, ly = idx / kTW;
      if (lx >= tw) continue;
      const int o = (H + ly) * WW + H + lx;
      for (int c = 0; c < 3; c++)
        reinterpret_cast<float*>(out_base + (size_t(c) * F.height + y0 + ly) * F.out_row_stride)[x0 + lx] = cur[c * NC + o];
    }
    return;
  }
  uint8_t* stage_u8 = reinterpret_cast<uint8_t*>(nxt);  // free buffer: interleaved output staging (<= 24 KB)
  const bool fmt16 = F.output_format == JXG_FORMAT_RGB_U16 || F.output_format == JXG_FORMAT_RGB_F16;
  const int bpp = F.output_format == JXG_FORMAT_RGB_U8 ? 3 : (F.output_format == JXG_FORMAT_RGBA_U8 ? 4 : (fmt16 ? 6 : 12));
  for (int idx = threadIdx.x; idx < kTW * th; idx += blockDim.x) {
    const int lx = idx % kTW, ly = idx / kTW;
    if (lx >= tw) continue;
    const int o = (H + ly) * WW + H + lx;
    const int x = x0 + lx, y = y0 + ly;
    float v[3];
    xyb_to_output(F, cur[o], cur[NC + o], cur[2 * NC + o], v);
    if (bpp == 12) {
      float* d = reinterpret_cast<float*>(stage_u8) + (ly * kTW + lx) * 3;
      d[0] = v[0];
      d[1] = v[1];
      d[2] = v[2];
    } else if (bpp == 6) {
      uint16_t* d = reinterpret_cast<uint16_t*>(stage_u8) + (ly * kTW + lx) * 3;
#pragma unroll
      for (int c = 0; c < 3; c++) d[c] = sample16(F, v[c]);
    } else {
      uint8_t* d = stage_u8 + (ly * kTW + lx) * bpp;
#pragma unroll
      for (int c = 0; c < 3; c++) d[c] = sample8(v[c], x, y, c);
      if (bpp == 4) d[3] = 255;
    }
  }
  __syncthreads();
  // the part of the tile inside the window (the whole tile of a full frame), stored at out + (y - win_y) * stride +
  // (x - win_x) * bpp
  const int lx0 = max(int(F.win_x) - x0, 0), lx1 = min(int(F.win_x + F.win_w) - x0, tw);
  const int ly0 = max(int(F.win_y) - y0, 0), ly1 = min(int(F.win_y + F.win_h) - y0, th);
  const int row_bytes = (lx1 - lx0) * bpp;
  for (int ly = ly0 + (threadIdx.x >> 5); ly < ly1; ly += (blockDim.x >> 5)) {  // one warp per row
    uint8_t* dst = out_base + size_t(y0 + ly - int(F.win_y)) * F.out_row_stride + size_t(x0 + lx0 - int(F.win_x)) * bpp;
    const uint8_t* srow = stage_u8 + (ly * kTW + lx0) * bpp;
    const int lane = threadIdx.x & 31;
    if (((reinterpret_cast<uintptr_t>(dst) | reinterpret_cast<uintptr_t>(srow) | uintptr_t(row_bytes)) & 15) == 0) {
      for (int i = lane; i < row_bytes / 16; i += 32) reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(srow)[i];
    } else {
      for (int i = lane; i < row_bytes; i += 32) dst[i] = srow[i];
    }
  }
}

// ---------------------------------------------------------------------------
// Vectorised interior path of the default filter configuration (Gaborish + EPF iters 2, halo 4): every thread owns
// quads of 4 horizontally adjacent cells, loads rows with 16-byte shared-memory accesses, computes the EPF differences
// of its quad and their plus-shaped sums once for the four cells, and converts / stores its four pixels straight from
// registers.
// Same arithmetic as the scalar path except for the association of a few float sums and the approximate
// sqrt / divide of the sRGB curve (<= 3 ulp), both far inside the 1e-3 / 1 LSB parity tolerances.
// ---------------------------------------------------------------------------
__device__ __forceinline__ float4 ld4(const float* p) { return *reinterpret_cast<const float4*>(p); }
__device__ __forceinline__ void st4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }

__device__ __forceinline__ float linear_to_srgb_fast(float v) {  // color/tf.rs:13-44
  const float a = fabsf(v);
  const float s = a * rsqrtf(fmaxf(a, 1e-30f));
  float yp = 7.352629620e-1f, yq = 2.424867759e-2f;
  yp = fmaf(yp, s, 1.474205315f);
  yq = fmaf(yq, s, 9.258482155e-1f);
  yp = fmaf(yp, s, 3.903842876e-1f);
  yq = fmaf(yq, s, 1.340816930f);
  yp = fmaf(yp, s, 5.287254571e-3f);
  yq = fmaf(yq, s, 3.036675394e-1f);
  yp = fmaf(yp, s, -5.135152395e-4f);
  yq = fmaf(yq, s, 1.004519624e-2f);
  const float r = a < 0.0031308f ? a * 12.92f : __fdividef(yp, yq);
  return copysignf(r, v);
}

// Channel-combined EPF differences of one row segment, accumulated one channel at a time (channel 0, 1, 2, each
// term fmaf(|a - b|, scale, sum) from 0): dh[i] = D_(1,0) of cell a[i], dv[i] = D_(0,1) of cell a[i + DA] whose lower
// neighbour is b[i + DB].
template <int NH, int NV, int DA, int DB>
__device__ __forceinline__ void acc_diffs(float* dh, float* dv, const float* a, const float* b, float sc) {
#pragma unroll
  for (int i = 0; i < NH; i++) dh[i] = fmaf(fabsf(a[i] - a[i + 1]), sc, dh[i]);
#pragma unroll
  for (int i = 0; i < NV; i++) dv[i] = fmaf(fabsf(a[i + DA] - b[i + DB]), sc, dv[i]);
}

// Sigma of every 8x8 block touched by a tile's window (features/epf.rs:54-79).
template <int SBW, int SBH>
__device__ __forceinline__ void tile_sigma(const BatchDev& B, const FrameDev& F, float* sig, int sbx0, int sby0, int t0, int nt) {
  for (int idx = t0; idx < SBW * SBH; idx += nt) {
    const int bx = sbx0 + idx % SBW, by = sby0 + idx / SBW;
    float v = 0.0f;
    if (bx < int(F.xb) && by < int(F.yb)) {
      const size_t bidx = size_t(by) * F.xb + bx;
      const int32_t raw_quant = reinterpret_cast<const int32_t*>(B.blob + F.raw_quant_off)[bidx];
      const uint32_t sharp = (B.blob + F.epf_off)[bidx];
      const float sigma_quant = F.epf_quant_mul / (F.quant_scale * float(raw_quant) * -1.1715728752538099024f);
      v = 1.0f / fminf(sigma_quant * F.epf_sharp_lut[sharp], -1e-4f);
    }
    sig[idx] = v;
  }
}

// A filter tile: its frame, origin and whether the vector path takes it.
struct TileRef {
  const FrameDev* F;
  int x0, y0;
  bool mine;  // the frame has this kernel's filter configuration
  bool vec;   // interior tile with an aligned output row: vector path
};

// Gaborish + EPF iters 2 on an interior tile, four pixels per thread: bufA receives the tile's window, bufB is the
// second plane buffer. Three barriers: after the load, after Gaborish and after EPF stage 1.
__device__ __forceinline__ void filter_tile_v4(const BatchDev& B, const FrameDev& F, const float* src_planes, float* bufA,
                                               float* bufB, float* sig, int x0, int y0) {
  using C = FCfg<true, 2>;
  constexpr int H = 4, WW = C::WW, WH = C::WH, NC = C::NC, QW = WW / 4;
  static_assert(C::H == H && WW == 72 && WH == 40, "vector path is written for the halo-4 configuration");
  const int wx0 = x0 - H, wy0 = y0 - H;
  const int sbx0 = wx0 >> 3, sby0 = wy0 >> 3;
  // ---- load ----
  for (int q = threadIdx.x; q < QW * WH; q += blockDim.x) {
    const int ly = q / QW, o = ly * WW + (q % QW) * 4;
    const float* g = src_planes + F.plane_base + size_t(wy0 + ly) * F.plane_stride + wx0 + (q % QW) * 4;
#pragma unroll
    for (int c = 0; c < 3; c++) st4(bufA + c * NC + o, __ldg(reinterpret_cast<const float4*>(g + c * F.plane_size)));
  }
  tile_sigma<C::SBW, C::SBH>(B, F, sig, sbx0, sby0, threadIdx.x, blockDim.x);
  __syncthreads();
  // ---- Gaborish (gaborish.rs:40-88): rows 1..38, bufA -> bufB ----
  for (int q = threadIdx.x; q < QW * (WH - 2); q += blockDim.x) {
    const int ly = 1 + q / QW, o = ly * WW + (q % QW) * 4;
#pragma unroll
    for (int c = 0; c < 3; c++) {
      const float k0 = F.gab_k0[c], k1 = F.gab_k1[c], k2 = F.gab_k2[c];
      const float* p = bufA + c * NC + o;
      const float4 u = ld4(p - WW), m = ld4(p), d = ld4(p + WW);
      const float ml = p[-1], mr = p[4];
      const float v0 = p[-WW - 1] + p[WW - 1], v1 = u.x + d.x, v2 = u.y + d.y, v3 = u.z + d.z, v4 = u.w + d.w,
                  v5 = p[-WW + 4] + p[WW + 4];
      float4 r;
      r.x = fmaf(k2, v0 + v2, fmaf(k1, v1 + ml + m.y, m.x * k0));
      r.y = fmaf(k2, v1 + v3, fmaf(k1, v2 + m.x + m.z, m.y * k0));
      r.z = fmaf(k2, v2 + v4, fmaf(k1, v3 + m.y + m.w, m.z * k0));
      r.w = fmaf(k2, v3 + v5, fmaf(k1, v4 + m.z + mr, m.w * k0));
      st4(bufB + c * NC + o, r);
    }
  }
  __syncthreads();
  const float kMinSigma = -3.90524291751269967465540850526868f;
  // ---- EPF stage 1 (epf1.rs): bufB rows 3..36 -> bufA ----
  {
    const float sm = 1.65f, bsm = sm * F.epf_border_sad_mul;
    for (int q = threadIdx.x; q < QW * (WH - 6); q += blockDim.x) {
      const int ly = 3 + q / QW, lx = (q % QW) * 4, o = ly * WW + lx;
      const int mx = wx0 + lx, my = wy0 + ly;
      const float inv_sigma_px = sig[((my >> 3) - sby0) * C::SBW + ((mx >> 3) - sbx0)];
      if (inv_sigma_px < kMinSigma) {
#pragma unroll
        for (int c = 0; c < 3; c++) st4(bufA + c * NC + o, ld4(bufB + c * NC + o));
        continue;
      }
      const bool rowb = ((my + 1) & 7) < 2;
      const float is_n = inv_sigma_px * (rowb ? bsm : sm), is_b = inv_sigma_px * bsm;
      const bool lo4 = (mx & 4) == 0;  // quad covers columns 0..3 (border at cell 0) or 4..7 (border at cell 3)
      const float isg[4] = {lo4 ? is_b : is_n, is_n, is_n, lo4 ? is_n : is_b};
      // Plus-shaped sums of the differences of bufB: ph of Dh at columns x-1 .. x+3 (left / right SADs of the four
      // cells), pu / pd of Dv at rows y-1 (up SAD) and y (down SAD). The difference rows are taken top to bottom,
      // each folded into the sums as soon as its three channels are in, so that few stay live.
      float ph[5], pu[4], pd[4], hu[5] = {};
      auto row = [&](const float* p, float* r6) {  // cells x-1 .. x+4 of the row at p
        const float4 v = ld4(p);
        r6[0] = p[-1]; r6[1] = v.x; r6[2] = v.y; r6[3] = v.z; r6[4] = v.w; r6[5] = p[4];
      };
      {  // Dv at row y-2 (columns x .. x+3)
        float va[4] = {};
#pragma unroll
        for (int c = 0; c < 3; c++) {
          const float* p = bufB + c * NC + o;
          const float4 a = ld4(p - 2 * WW), b = ld4(p - WW);
          const float r0[4] = {a.x, a.y, a.z, a.w}, r1[4] = {b.x, b.y, b.z, b.w};
          acc_diffs<0, 4, 0, 0>(nullptr, va, r0, r1, F.epf_channel_scale[c]);
        }
#pragma unroll
        for (int i = 0; i < 4; i++) pu[i] = va[i];
      }
      {  // Dh at row y-1 (x-1 .. x+3), Dv at row y-1 (x-1 .. x+4)
        float vb[6] = {};
#pragma unroll
        for (int c = 0; c < 3; c++) {
          const float* p = bufB + c * NC + o;
          float r1[6], r2[6];
          row(p - WW, r1);
          row(p, r2);
          acc_diffs<5, 6, 0, 0>(hu, vb, r1, r2, F.epf_channel_scale[c]);
        }
#pragma unroll
        for (int i = 0; i < 4; i++) {
          pu[i] = pu[i] + vb[i] + vb[i + 1] + vb[i + 2];
          pd[i] = vb[i + 1];
        }
      }
      {  // Dh at row y (x-2 .. x+4), Dv at row y (x-1 .. x+4)
        float hm[7] = {}, vm[6] = {};
#pragma unroll
        for (int c = 0; c < 3; c++) {
          const float* p = bufB + c * NC + o;
          const float4 m = ld4(p);
          const float2 ml = *reinterpret_cast<const float2*>(p - 2), mr = *reinterpret_cast<const float2*>(p + 4);
          const float r2[8] = {ml.x, ml.y, m.x, m.y, m.z, m.w, mr.x, mr.y};
          float r3[6];
          row(p + WW, r3);
          acc_diffs<7, 6, 1, 0>(hm, vm, r2, r3, F.epf_channel_scale[c]);
        }
#pragma unroll
        for (int i = 0; i < 5; i++) ph[i] = hm[i] + hm[i + 1] + hm[i + 2] + hu[i];
#pragma unroll
        for (int i = 0; i < 4; i++) {
          pu[i] = pu[i] + vm[i + 1];
          pd[i] = pd[i] + vm[i] + vm[i + 1] + vm[i + 2];
        }
      }
      {  // Dh at row y+1 (x-1 .. x+3), Dv at row y+1 (x .. x+3)
        float hd[5] = {}, ve[4] = {};
#pragma unroll
        for (int c = 0; c < 3; c++) {
          const float* p = bufB + c * NC + o;
          float r3[6];
          row(p + WW, r3);
          const float4 e = ld4(p + 2 * WW);
          const float r4[4] = {e.x, e.y, e.z, e.w};
          acc_diffs<5, 4, 1, 0>(hd, ve, r3, r4, F.epf_channel_scale[c]);
        }
#pragma unroll
        for (int i = 0; i < 5; i++) ph[i] = ph[i] + hd[i];
#pragma unroll
        for (int i = 0; i < 4; i++) pd[i] = pd[i] + ve[i];
      }
      asm volatile("" ::: "memory");  // reload the rows below rather than keep all three channels live from above
      float wu[4], wl[4], wr[4], wd[4], iw[4];
#pragma unroll
      for (int i = 0; i < 4; i++) {
        wu[i] = fmaxf(fmaf(pu[i], isg[i], 1.0f), 0.0f);
        wl[i] = fmaxf(fmaf(ph[i], isg[i], 1.0f), 0.0f);
        wr[i] = fmaxf(fmaf(ph[i + 1], isg[i], 1.0f), 0.0f);
        wd[i] = fmaxf(fmaf(pd[i], isg[i], 1.0f), 0.0f);
        iw[i] = 1.0f / (1.0f + wu[i] + wl[i] + wr[i] + wd[i]);
      }
#pragma unroll
      for (int c = 0; c < 3; c++) {
        const float* p = bufB + c * NC + o;
        const float4 u = ld4(p - WW), m = ld4(p), d = ld4(p + WW);
        const float ml = p[-1], mr = p[4];
        float4 r;
        r.x = fmaf(u.x, wu[0], fmaf(ml, wl[0], fmaf(m.y, wr[0], fmaf(d.x, wd[0], m.x)))) * iw[0];
        r.y = fmaf(u.y, wu[1], fmaf(m.x, wl[1], fmaf(m.z, wr[1], fmaf(d.y, wd[1], m.y)))) * iw[1];
        r.z = fmaf(u.z, wu[2], fmaf(m.y, wl[2], fmaf(m.w, wr[2], fmaf(d.z, wd[2], m.z)))) * iw[2];
        r.w = fmaf(u.w, wu[3], fmaf(m.z, wl[3], fmaf(mr, wr[3], fmaf(d.w, wd[3], m.w)))) * iw[3];
        st4(bufA + c * NC + o, r);
      }
    }
  }
  __syncthreads();
  // ---- EPF stage 2 (epf2.rs) on the 64x32 core + colour + store ----
  {
    const int w = int(F.width);
    uint8_t* out_base = static_cast<uint8_t*>(F.out_ptr);
    for (int q = threadIdx.x; q < (kTW / 4) * kTH; q += blockDim.x) {
      const int ly = H + q / (kTW / 4), lx = H + (q % (kTW / 4)) * 4, o = ly * WW + lx;
      const int mx = wx0 + lx, my = wy0 + ly;
      float px[3][4];
      const float inv_sigma_px = sig[((my >> 3) - sby0) * C::SBW + ((mx >> 3) - sbx0)];
      if (inv_sigma_px < kMinSigma) {
#pragma unroll
        for (int c = 0; c < 3; c++) {
          const float4 m = ld4(bufA + c * NC + o);
          px[c][0] = m.x; px[c][1] = m.y; px[c][2] = m.z; px[c][3] = m.w;
        }
      } else {
        const float sm = F.epf_pass2_sigma_scale * 1.65f, bsm = sm * F.epf_border_sad_mul;  // read here: no register to spare
        const bool rowb = ((my + 1) & 7) < 2;
        const float is_n = inv_sigma_px * (rowb ? bsm : sm), is_b = inv_sigma_px * bsm;
        const bool lo4 = (mx & 4) == 0;
        const float isg[4] = {lo4 ? is_b : is_n, is_n, is_n, lo4 ? is_n : is_b};
        // differences of bufA: Dv at rows y-1 and y (columns x .. x+3), Dh at row y (x-1 .. x+3)
        float sup[4] = {}, shh[5] = {}, sdn[4] = {};
#pragma unroll
        for (int c = 0; c < 3; c++) {
          const float sc = F.epf_channel_scale[c];
          const float* p = bufA + c * NC + o;
          const float4 u = ld4(p - WW), m = ld4(p), d = ld4(p + WW);
          const float r0[4] = {u.x, u.y, u.z, u.w};
          const float r1[6] = {p[-1], m.x, m.y, m.z, m.w, p[4]};
          const float r2[4] = {d.x, d.y, d.z, d.w};
          acc_diffs<0, 4, 0, 1>(nullptr, sup, r0, r1, sc);
          acc_diffs<5, 4, 1, 0>(shh, sdn, r1, r2, sc);
        }
        asm volatile("" ::: "memory");  // as in EPF stage 1
        float wu[4], wl[4], wr[4], wd[4], iw[4];
#pragma unroll
        for (int i = 0; i < 4; i++) {
          wu[i] = fmaxf(fmaf(sup[i], isg[i], 1.0f), 0.0f);
          wl[i] = fmaxf(fmaf(shh[i], isg[i], 1.0f), 0.0f);
          wr[i] = fmaxf(fmaf(shh[i + 1], isg[i], 1.0f), 0.0f);
          wd[i] = fmaxf(fmaf(sdn[i], isg[i], 1.0f), 0.0f);
          iw[i] = 1.0f / (1.0f + wu[i] + wl[i] + wr[i] + wd[i]);
        }
#pragma unroll
        for (int c = 0; c < 3; c++) {
          const float* p = bufA + c * NC + o;
          const float4 u = ld4(p - WW), m = ld4(p), d = ld4(p + WW);
          const float ml = p[-1], mr = p[4];
          // accumulation order of the reference: up, left, right, down (epf2.rs:83)
          px[c][0] = fmaf(wd[0], d.x, fmaf(wr[0], m.y, fmaf(wl[0], ml, fmaf(wu[0], u.x, m.x)))) * iw[0];
          px[c][1] = fmaf(wd[1], d.y, fmaf(wr[1], m.z, fmaf(wl[1], m.x, fmaf(wu[1], u.y, m.y)))) * iw[1];
          px[c][2] = fmaf(wd[2], d.z, fmaf(wr[2], m.w, fmaf(wl[2], m.y, fmaf(wu[2], u.z, m.z)))) * iw[2];
          px[c][3] = fmaf(wd[3], d.w, fmaf(wr[3], mr, fmaf(wl[3], m.z, fmaf(wu[3], u.w, m.w)))) * iw[3];
        }
      }
      const int gx = mx, gy = my;
      if (F.output_format == JXG_FORMAT_XYB_F32_PLANAR) {
#pragma unroll
        for (int c = 0; c < 3; c++)
          st4(reinterpret_cast<float*>(out_base + (size_t(c) * F.height + gy) * F.out_row_stride) + gx,
              make_float4(px[c][0], px[c][1], px[c][2], px[c][3]));
        continue;
      }
      float rgb[4][3];
#pragma unroll
      for (int i = 0; i < 4; i++) {  // xyb.rs:197-241
        float l = px[1][i] + px[0][i] - F.bias_cbrt[0], mm = px[1][i] - px[0][i] - F.bias_cbrt[1], s = px[2][i] - F.bias_cbrt[2];
        const float l2 = l * l, m2 = mm * mm, s2 = s * s;
        l = fmaf(l2, l * F.intensity_scale, F.scaled_bias[0]);
        mm = fmaf(m2, mm * F.intensity_scale, F.scaled_bias[1]);
        s = fmaf(s2, s * F.intensity_scale, F.scaled_bias[2]);
        rgb[i][0] = fmaf(F.opsin[0], l, fmaf(F.opsin[1], mm, F.opsin[2] * s));
        rgb[i][1] = fmaf(F.opsin[3], l, fmaf(F.opsin[4], mm, F.opsin[5] * s));
        rgb[i][2] = fmaf(F.opsin[6], l, fmaf(F.opsin[7], mm, F.opsin[8] * s));
        if (F.output_tf == JXG_TF_SRGB) {
#pragma unroll
          for (int c = 0; c < 3; c++) rgb[i][c] = linear_to_srgb_fast(rgb[i][c]);
        } else if (F.output_tf != JXG_TF_LINEAR) {
          from_linear_other(F, rgb[i]);
        }
      }
      (void)w;
      // Window-relative position of the quad. A quad fully inside the window at a multiple of 4 pixels from its left
      // edge (every quad of a full frame) is stored with 16-byte / word stores; any other quad sample by sample, only
      // its pixels inside the window. Both store the same values.
      const int qx = gx - int(F.win_x), qy = gy - int(F.win_y);
      uint8_t* out_row = out_base + size_t(qy) * F.out_row_stride;
      const bool whole = (qx & 3) == 0 && qx >= 0 && qx + 4 <= int(F.win_w) && unsigned(qy) < F.win_h;
      auto inside = [&](int i) { return unsigned(qx + i) < F.win_w && unsigned(qy) < F.win_h; };
      if (F.output_format == JXG_FORMAT_RGB_F32) {
        float* d = reinterpret_cast<float*>(out_row) + ptrdiff_t(qx) * 3;
        if (whole) {
          st4(d, make_float4(rgb[0][0], rgb[0][1], rgb[0][2], rgb[1][0]));
          st4(d + 4, make_float4(rgb[1][1], rgb[1][2], rgb[2][0], rgb[2][1]));
          st4(d + 8, make_float4(rgb[2][2], rgb[3][0], rgb[3][1], rgb[3][2]));
        } else {
#pragma unroll
          for (int i = 0; i < 4; i++)
            if (inside(i))
#pragma unroll
              for (int c = 0; c < 3; c++) d[i * 3 + c] = rgb[i][c];
        }
        continue;
      }
      uint32_t b8[4][3];
#pragma unroll
      for (int i = 0; i < 4; i++)
#pragma unroll
        for (int c = 0; c < 3; c++) {  // convert.rs:574-598 (blue-noise dither)
          const float dth = g_dither[((gy + 13 * c) & 31) * 32 + ((gx + i + 23 * c) & 31)];
          b8[i][c] = uint32_t(__float2int_rn(fminf(fmaxf(fmaf(rgb[i][c], 255.0f, dth), 0.0f), 255.0f)));
        }
      if (!whole) {
        const int bpp = F.output_format == JXG_FORMAT_RGB_U8 ? 3 : 4;
#pragma unroll
        for (int i = 0; i < 4; i++)
          if (inside(i)) {
            uint8_t* d = out_row + ptrdiff_t(qx + i) * bpp;
            if (bpp == 4) *reinterpret_cast<uint32_t*>(d) = b8[i][0] | (b8[i][1] << 8) | (b8[i][2] << 16) | 0xff000000u;
            else {
              d[0] = uint8_t(b8[i][0]);
              d[1] = uint8_t(b8[i][1]);
              d[2] = uint8_t(b8[i][2]);
            }
          }
      } else if (F.output_format == JXG_FORMAT_RGB_U8) {
        uint32_t* d = reinterpret_cast<uint32_t*>(out_row + size_t(qx) * 3);
        d[0] = b8[0][0] | (b8[0][1] << 8) | (b8[0][2] << 16) | (b8[1][0] << 24);
        d[1] = b8[1][1] | (b8[1][2] << 8) | (b8[2][0] << 16) | (b8[2][1] << 24);
        d[2] = b8[2][2] | (b8[3][0] << 8) | (b8[3][1] << 16) | (b8[3][2] << 24);
      } else {
        uint4 v;
        v.x = b8[0][0] | (b8[0][1] << 8) | (b8[0][2] << 16) | 0xff000000u;
        v.y = b8[1][0] | (b8[1][1] << 8) | (b8[1][2] << 16) | 0xff000000u;
        v.z = b8[2][0] | (b8[2][1] << 8) | (b8[2][2] << 16) | 0xff000000u;
        v.w = b8[3][0] | (b8[3][1] << 8) | (b8[3][2] << 16) | 0xff000000u;
        *reinterpret_cast<uint4*>(out_row + size_t(qx) * 4) = v;
      }
    }
  }
}

template <bool GAB, int EPF>
__device__ __forceinline__ TileRef locate_tile(const BatchDev& B, const FusedTiles& T, uint32_t tile_id) {
  using C = FCfg<GAB, EPF>;
  TileRef r;
  r.F = nullptr;
  r.x0 = r.y0 = 0;
  r.mine = r.vec = false;
  uint32_t lo = 0, hi = T.num_frames;
  while (hi - lo > 1) {
    uint32_t mid = (lo + hi) >> 1;
    if (T.tile_prefix[mid] <= tile_id) lo = mid;
    else hi = mid;
  }
  const FrameDev& F = B.frames[lo];
  r.F = &F;
  if ((F.gab != 0) != GAB || int(min(F.epf_iters, 3u)) != EPF) return r;  // another instantiation handles this frame
  r.mine = true;
  const uint32_t local = tile_id - T.tile_prefix[lo];
  r.x0 = int(F.win_tx0 + local % F.win_ntx) * kTW;
  r.y0 = int(F.win_ty0 + local / F.win_ntx) * kTH;
  const bool interior = r.x0 - C::H >= 0 && r.y0 - C::H >= 0 && r.x0 + kTW + C::H <= int(F.width) && r.y0 + kTH + C::H <= int(F.height);
  // 16-byte accesses need an aligned output row (RGB8: stride and base multiples of 4, f32 / RGBA: of 16)
  const uintptr_t oa = reinterpret_cast<uintptr_t>(F.out_ptr) | uintptr_t(F.out_row_stride);
  const bool aligned = F.output_format == JXG_FORMAT_RGB_U8 ? (oa & 3) == 0 : (oa & 15) == 0;
  const bool vec_format = F.output_format <= JXG_FORMAT_XYB_F32_PLANAR;  // the 16-bit stores take the generic path
  r.vec = GAB && EPF == 2 && interior && aligned && vec_format;
  return r;
}

template <bool GAB, int EPF>
__global__ void __launch_bounds__(FCfg<GAB, EPF>::kThreads, FCfg<GAB, EPF>::kMinCtas) k_filters_store(const BatchDev B, const FusedTiles T, const float* src_planes) {
  using C = FCfg<GAB, EPF>;
  extern __shared__ float smem[];
  const TileRef r = locate_tile<GAB, EPF>(B, T, blockIdx.x + T.tile_begin);
  if (!r.mine) return;
  const FrameDev& F = *r.F;
  const bool interior = r.x0 - C::H >= 0 && r.y0 - C::H >= 0 && r.x0 + kTW + C::H <= int(F.width) && r.y0 + kTH + C::H <= int(F.height);
  if (GAB && EPF == 2 && r.vec) {
    filter_tile_v4(B, F, src_planes, smem, smem + 3 * FCfg<true, 2>::NC, smem + 6 * FCfg<true, 2>::NC, r.x0, r.y0);
  } else if (interior) {
    filter_tile<GAB, EPF, true>(B, F, src_planes, smem, r.x0, r.y0);
  } else {
    filter_tile<GAB, EPF, false>(B, F, src_planes, smem, r.x0, r.y0);
  }
}

int sm_count() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
    return 132;
  return n;
}

template <bool GAB, int EPF>
static void launch_filters(const BatchDev& B, const FusedTiles& FT, uint32_t tiles, cudaStream_t stream) {
  k_filters_store<GAB, EPF><<<tiles, FCfg<GAB, EPF>::kThreads, FCfg<GAB, EPF>::kSmemBytes, stream>>>(B, FT, B.planes_a);
}
template <bool GAB, int EPF>
static cudaError_t configure_filters() {
  return cudaFuncSetAttribute(k_filters_store<GAB, EPF>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              int(FCfg<GAB, EPF>::kSmemBytes));
}

// ---------------------------------------------------------------------------
// Orientation post-pass (headers/image_metadata.rs:85-96 display_pixel, applied by the reference's save stage,
// render/save.rs): pixel (x, y) of the coded w x h image goes to display_pixel(x, y). Only frames whose
// ImageMetadata.orientation != 1 take it: they are filtered / stored into a tight staging image first.
// One thread per pixel; threads of a warp read consecutive source pixels.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_orient(const uint8_t* src, size_t src_stride, uint8_t* dst, size_t dst_stride,
                                                uint32_t w, uint32_t h, uint32_t bpp, uint32_t orientation) {
  const uint32_t x = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
  if (x >= w || y >= h) return;
  uint32_t dx, dy;
  switch (orientation) {
    case 2: dx = w - 1 - x; dy = y; break;          // FlipHorizontal
    case 3: dx = w - 1 - x; dy = h - 1 - y; break;  // Rotate180
    case 4: dx = x; dy = h - 1 - y; break;          // FlipVertical
    case 5: dx = y; dy = x; break;                  // Transpose
    case 6: dx = h - 1 - y; dy = x; break;          // Rotate90Cw
    case 7: dx = h - 1 - y; dy = w - 1 - x; break;  // AntiTranspose
    case 8: dx = y; dy = w - 1 - x; break;          // Rotate90Ccw
    default: dx = x; dy = y; break;
  }
  const uint8_t* s = src + size_t(y) * src_stride + size_t(x) * bpp;
  uint8_t* d = dst + size_t(dy) * dst_stride + size_t(dx) * bpp;
  if ((bpp & 3) == 0) {
    for (uint32_t i = 0; i < bpp; i += 4) *reinterpret_cast<uint32_t*>(d + i) = *reinterpret_cast<const uint32_t*>(s + i);
  } else {
    for (uint32_t i = 0; i < bpp; i++) d[i] = s[i];
  }
}

// ===========================================================================
// host-callable launch wrappers (used by batch.cc through launch.h)
// ===========================================================================

}  // namespace jxgpu

#include "launch.h"

namespace jxgpu {
static_assert(kFusedTileW == kTW && kFusedTileH == kTH, "launch.h tile size differs from the fused filter kernel");

cudaError_t upload_constants(const float* wc, const float* rdct_scale) {
  cudaError_t e = cudaMemcpyToSymbol(c_wc, wc, sizeof(float) * 9 * 128);
  if (e != cudaSuccess) return e;
  return cudaMemcpyToSymbol(c_rdct_scale, rdct_scale, sizeof(float) * 6 * 32);
}

cudaError_t configure_kernels() {
  cudaError_t e;
  if ((e = configure_filters<false, 0>()) != cudaSuccess) return e;
  if ((e = configure_filters<false, 1>()) != cudaSuccess) return e;
  if ((e = configure_filters<false, 2>()) != cudaSuccess) return e;
  if ((e = configure_filters<false, 3>()) != cudaSuccess) return e;
  if ((e = configure_filters<true, 0>()) != cudaSuccess) return e;
  if ((e = configure_filters<true, 1>()) != cudaSuccess) return e;
  if ((e = configure_filters<true, 2>()) != cudaSuccess) return e;
  if ((e = configure_filters<true, 3>()) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(k_idct_small<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(small_smem_bytes<0>()))) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(k_idct_small<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(small_smem_bytes<1>()))) != cudaSuccess) return e;
  if ((e = cudaFuncSetAttribute(k_dequant_idct, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kLargeSmemBytes))) != cudaSuccess) return e;
  return cudaSuccess;
}

int launch_pipeline(const BatchDev& B, cudaStream_t stream, int debug_stop, cudaEvent_t* ev, bool lean_all_420,
                    uint32_t lean_S, uint32_t lean_ctas, bool lean_ctx_smem, uint32_t fast_S) {
  // ev (optional, kNumStages + 1 events): ev[i] is recorded before stage i, ev[i+1] after it; stages that do not
  // run record nothing (the host pairs consecutive recorded events).
  int launches = 0;
  auto mark = [&](int i) {
    if (ev) cudaEventRecord(ev[i], stream);
  };
  mark(0);  // stage 0 (memset) is empty: there is no dense coefficient array to clear
  mark(1);
  k_block_plan<<<(B.num_streams + 3) / 4, 128, 0, stream>>>(B);
  launches++;
  if (B.num_lean) {
    // Persistent lanes, scheduled per frame by the host (batch.cc schedule_lean): S = 4 or 8 lanes per warp, lean_ctas CTAs.
    cudaMemsetAsync(B.queue, 0, sizeof(uint32_t) * B.num_frames, stream);
    const uint32_t S = lean_S, grid = lean_ctas;
    const int smem = lean_ctx_smem ? int(kLeanCtxSmem) : 0;
#define JXG_LEAN(SV, KV, CV) k_entropy_lean<SV, KV, CV><<<grid, 128, smem, stream>>>(B)
#define JXG_LEAN_S(KV, CV)             \
  do {                                 \
    if (S == 8) JXG_LEAN(8, KV, CV);   \
    else JXG_LEAN(4, KV, CV);          \
  } while (0)
    if (lean_all_420) {
      if (lean_ctx_smem) JXG_LEAN_S(true, true);
      else JXG_LEAN_S(true, false);
    } else {
      if (lean_ctx_smem) JXG_LEAN_S(false, true);
      else JXG_LEAN_S(false, false);
    }
#undef JXG_LEAN_S
#undef JXG_LEAN
    launches++;
  }
  if (B.num_fast) {
    // streams per warp chosen by the host (batch.cc schedule_fast): about one resident wave of warps
    if (fast_S <= 1) k_entropy_fast<1><<<(B.num_fast + 3) / 4, 128, 0, stream>>>(B);
    else if (fast_S == 2) k_entropy_fast<2><<<(B.num_fast + 7) / 8, 128, 0, stream>>>(B);
    else if (fast_S == 4) k_entropy_fast<4><<<(B.num_fast + 15) / 16, 128, 0, stream>>>(B);
    else k_entropy_fast<8><<<(B.num_fast + 31) / 32, 128, 0, stream>>>(B);
    launches++;
  }
  if (B.num_slow) {
    k_entropy<<<(B.num_slow + kEntropyWarps - 1) / kEntropyWarps, kEntropyWarps * 32, 0, stream>>>(B);
    launches++;
  }
  mark(2);
  if (debug_stop == 1) return launches;
  k_idct_small<0><<<B.num_streams, kSmallThreads, small_smem_bytes<0>(), stream>>>(B);
  k_idct_small<1><<<B.num_streams, kSmallThreads, small_smem_bytes<1>(), stream>>>(B);
  launches += 2;
  k_dequant_idct<<<B.num_streams, kIdctWarps * 32, kLargeSmemBytes, stream>>>(B);
  launches++;
  mark(3);
  return launches;  // the fused filter + colour + store kernel is launched per frame range by the caller
}

// Parity tap: the coefficient lists of one frame expanded into the reference's dense decode-order layout
// [groups][3][65536] (group.rs:53-55), all passes added up. One CTA per group; `dense` must be zeroed by the caller.
__global__ void __launch_bounds__(256) k_expand_coeffs(const BatchDev B, uint32_t frame, int32_t* dense) {
  const FrameDev& F = B.frames[frame];
  const uint32_t g = blockIdx.x, gsid = F.first_stream + g;
  const uint32_t nblk = B.nblk[gsid];
  if (nblk == 0xffffffffu) return;
  const uint4* desc = B.desc + size_t(gsid) * 1024;
  int32_t* out = dense + size_t(g) * 3 * kGroupCoeffs;
  for (uint32_t p = 0; p < F.num_passes; p++) {
    const uint32_t section = F.section_base + p * F.num_groups + g;
    const uint32_t* base = list_base(B, section);
    const uint32_t* ow = base + kOffBase;
    for (uint32_t bi = threadIdx.x >> 5; bi < nblk; bi += blockDim.x >> 5) {  // one warp per varblock
      const uint4 d = desc[bi];
      const uint32_t lnc = (d.x >> 26) + 6;  // log2 of the varblock's coefficients per channel
      const uint32_t o0 = ow[bi * 3], o1 = ow[bi * 3 + 1], o2 = ow[bi * 3 + 2], o3 = min(ow[bi * 3 + 3], kListCap);
      for (uint32_t i = o0 + (threadIdx.x & 31); i < o3; i += 32) {
        const uint32_t e = base[i];
        const uint32_t c = i < o1 ? 1u : (i < o2 ? 0u : 2u);
        out[c * kGroupCoeffs + d.z + entry_pos(e, lnc)] += entry_value(e, lnc);
      }
    }
    __syncthreads();
  }
}

void launch_expand_coeffs(const BatchDev& B, uint32_t frame, uint32_t num_groups, int32_t* dense, cudaStream_t stream) {
  k_expand_coeffs<<<num_groups, 256, 0, stream>>>(B, frame, dense);
}

void launch_orient(const void* src, size_t src_stride, void* dst, size_t dst_stride, uint32_t w, uint32_t h, uint32_t bpp,
                   uint32_t orientation, cudaStream_t stream) {
  k_orient<<<dim3((w + 31) / 32, (h + 7) / 8), 256, 0, stream>>>(static_cast<const uint8_t*>(src), src_stride,
                                                                 static_cast<uint8_t*>(dst), dst_stride, w, h, bpp, orientation);
}

// Fused filter/colour/store kernel over tiles [tile_begin, tile_begin + tile_count): one launch per filter
// configuration present in the batch (CTAs of frames with another configuration exit at once).
int launch_filter_range(const BatchDev& B, const uint32_t* fused_prefix, uint32_t tile_begin, uint32_t tile_count,
                        uint32_t filter_cfg_mask, cudaStream_t stream) {
  int launches = 0;
  if (!tile_count) return 0;
  FusedTiles FT{fused_prefix, B.num_frames, tile_begin};
  for (int cfg = 0; cfg < 8; cfg++) {
    if (!(filter_cfg_mask & (1u << cfg))) continue;
    switch (cfg) {
      case 0: launch_filters<false, 0>(B, FT, tile_count, stream); break;
      case 1: launch_filters<false, 1>(B, FT, tile_count, stream); break;
      case 2: launch_filters<false, 2>(B, FT, tile_count, stream); break;
      case 3: launch_filters<false, 3>(B, FT, tile_count, stream); break;
      case 4: launch_filters<true, 0>(B, FT, tile_count, stream); break;
      case 5: launch_filters<true, 1>(B, FT, tile_count, stream); break;
      case 6: launch_filters<true, 2>(B, FT, tile_count, stream); break;
      default: launch_filters<true, 3>(B, FT, tile_count, stream); break;
    }
    launches++;
  }
  return launches;
}

}  // namespace jxgpu
