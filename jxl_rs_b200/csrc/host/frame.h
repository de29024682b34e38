// Host front-end of one VarDCT frame: everything jxl-rs does *before* the hot
// path (jxl/src/frame/decode.rs:307-566): LfGlobal, LfGroups (LF image + HF
// metadata through the Modular decoder), HfGlobal (dequant matrices,
// coefficient orders, per-pass histograms), LF finalisation (adaptive
// smoothing). Produces the flat frame state behind JxgFrameDesc.
#pragma once
#include <array>
#include <cstdint>
#include <memory>
#include <vector>

#include "../../../include/jxg.h"
#include "entropy.h"
#include "headers.h"
#include "modular.h"
#include "region.h"

namespace jxg {

constexpr int kNumQuantTables = 17;
constexpr int kNumOrders = 13;

// quant_weights.rs: library tables (computed once, shared) and custom tables.
const std::vector<float>& library_dequant_table(int idx);
extern const uint8_t kQuantTableRows[kNumQuantTables];  // REQUIRED_SIZE_X (rows, in blocks)
extern const uint8_t kQuantTableCols[kNumQuantTables];  // REQUIRED_SIZE_Y (cols, in blocks)
int quant_table_for_transform(int transform);           // QuantTable::for_strategy

// transform_map.rs
extern const uint8_t kCoveredBlocksX[27], kCoveredBlocksY[27], kBlockShapeId[27];
// coeff_order.rs:66
std::vector<uint32_t> natural_coeff_order(int order_idx);
const std::vector<uint32_t>& natural_coeff_order_cached(int order_idx);  // same, computed once per process
extern const uint8_t kOrderTransform[kNumOrders];  // TRANSFORM_TYPE_LUT

struct PassState {
  EntropyCode code;            // context map padded by 16 (frame/decode.rs:536-538)
  bool custom_orders = false;
  std::vector<uint32_t> coeff_order;  // 39 concatenated orders if custom_orders
  uint32_t coeff_order_offset[39] = {0};
  std::vector<uint32_t> uint_configs_packed;
};

struct FrameState {
  FileHeader file;
  FrameHeader header;
  Toc toc;
  std::vector<uint8_t> codestream;  // owns the bytes
  size_t sections_base = 0;         // byte offset of section 0 in codestream

  // LfGlobal
  float lf_quant[3] = {1.0f / 4096.0f, 1.0f / 512.0f, 1.0f / 256.0f};
  uint32_t global_scale = 0, quant_lf = 0;
  std::vector<int32_t> lf_thresholds[3];
  std::vector<uint32_t> qf_thresholds;
  std::vector<uint8_t> block_ctx_map;
  uint32_t num_lf_contexts = 1, num_block_contexts = 15;
  uint32_t color_factor = 84;
  float base_correlation_x = 0.0f, base_correlation_b = 1.0f;
  int32_t ytox_lf = 0, ytob_lf = 0;
  bool has_global_tree = false;
  ModularTree global_tree;

  // Extra channels (alpha, depth, ...) of a VarDCT frame are Modular-coded next to the colour data
  // (FullModularImage::read, modular/mod.rs:258-330). The hot path decodes the colour channels only — the
  // reference API's "extra channel not requested" case, JxlPixelFormat::extra_channel_format = None
  // (api/data_types.rs:154) — so the front-end just steps over their sub-bitstreams: the global header and the
  // "meta or small" channels in LfGlobal, the shift >= 3 channels in every LfGroup section; the ModularHF streams
  // sit behind the AC coefficients of their HF section and are never reached.
  struct ExtraChannelImage {
    std::vector<ModularChannel> coded;  // channel shapes after the global meta-apply (no sample planes)
    GroupHeader header;
    uint32_t nb_meta = 0;
    size_t n0 = 0;  // leading channels coded in LfGlobal
  } ec;

  // planes (xb x yb)
  uint32_t xb = 0, yb = 0;
  std::vector<float> lf[3];
  std::vector<uint8_t> transform_map, epf_map, quant_lf_map;
  std::vector<int32_t> raw_quant_map;
  std::vector<int8_t> ytox_map, ytob_map;

  // HfGlobal
  std::vector<float> custom_dequant[kNumQuantTables];  // empty = library
  uint32_t num_histograms = 1;
  std::vector<PassState> passes;
  std::vector<JxgPassDesc> pass_descs;

  // Section table for the HF groups (pass-major), offsets into codestream.
  std::vector<uint64_t> hf_off;
  std::vector<uint32_t> hf_len;

  // A frame parsed from a prefix of its file (parse_vardct_file with `prefix`): group_passes[g] is the number of HF
  // passes group g decodes with, the longest run of whole sections from pass 0 (frame_info.rs:548-565 check_group);
  // hf_len is 0 for the sections past it. Empty group_passes: a frame parsed from a whole file.
  bool prefix = false;
  std::vector<uint8_t> group_passes;

  // the sub-frame jxg_parsed_region_desc handed out last (its pointers stay valid until the next call)
  std::unique_ptr<RegionSlice> region_tap;

  size_t num_ac_contexts() const { return size_t(num_block_contexts) * (37 + 458); }
  void fill_desc(JxgFrameDesc* d, uint32_t output_format);
};

// modular/mod.rs:837-929 dequant_lf (4:4:4) on a w x h rect of quantised LF integers; exposed for the tests.
// HF-metadata placement of one LF group (modular/mod.rs:1040-1075), see frame.cc.
void place_varblocks(uint32_t w, uint32_t hh, size_t stride, uint32_t count, const int32_t* raw_transforms, const int32_t* raw_quants,
                     uint8_t* transform_map, int32_t* raw_quant_map);
void dequant_lf_rect(FrameState& fs, const int32_t* qy, const int32_t* qx, const int32_t* qb, size_t qstride, uint32_t w, uint32_t h,
                     float mul, size_t o0);

// The scalars of dequant_lf_rect for LF multiplier `mul` (1 / 2^extra_precision): per X / Y / B the factor of the
// quantised sample, and the LF chroma-from-luma of X and B.
struct LfDequantFactors {
  float fac[3], cfl_x, cfl_b;
};
LfDequantFactors lf_dequant_factors(const FrameState& fs, float mul);
// The per-channel divisors of the adaptive LF smoothing's gap (adaptive_lf_smoothing.rs:57-60).
void lf_smoothing_factors(const FrameState& fs, float out[3]);

// frame/adaptive_lf_smoothing.rs:44 on fs.lf (uses xb, yb, global_scale, quant_lf, lf_quant). Exposed for the tests.
void adaptive_lf_smoothing(FrameState& fs, int threads = 1);

// The output-stage fields of a JxgFrameDesc for an XYB image (opsin biases and re-targeted matrix, intensity target,
// transfer function, luminances) and its output_format / orientation; the other fields are left as they are.
void fill_output_colour(const FileHeader& file, uint32_t output_format, JxgFrameDesc* d);

// JxgImageInfo of a parsed frame (jxg_parse_file, jxg_lf_parse_file, jxg_modular_parse_file): sizes, orientation,
// groups, passes, encoding and the HF section bytes `hf_bytes`.
void fill_image_info(const FileHeader& file, const FrameHeader& h, uint64_t hf_bytes, JxgImageInfo* info);

// Which sections read_vardct_headers requires whole: every section, LfGlobal and the LF groups (a thumbnail), or those
// and HfGlobal (a prefix decode). A one-section frame always needs its section whole.
enum class WholeSections { kAll, kLf, kLfAndHfGlobal };

// Container, headers, scope checks (everything outside this path's scope is refused with kErrUnsupported), the output
// colour check and the TOC: fills fs.codestream, file, header, toc, sections_base, xb and yb. A required section that
// does not fit in the file is refused with kErrOutOfBounds.
void read_vardct_headers(FrameState& fs, const uint8_t* data, size_t size, WholeSections whole);
// frame/decode.rs:307-427: LfGlobal of a VarDCT frame (quantiser, block context map, colour correlation, global tree,
// extra-channel data).
void decode_lf_global(FrameState& fs, BitReader& br);

// Parses a complete file up to (not including) the HF groups of its first
// displayed VarDCT frame. Throws jxg::Error.
// `threads` > 1 decodes the LF groups of the frame (LF image + HF metadata, independent TOC sections,
// frame/decode.rs:429) on that many host threads: the latency path for one large image (a 16384x16384 frame has 64
// LF groups and ~45 M Modular symbols); batches of many frames keep 1 and parallelise over frames instead. The
// parsed state does not depend on `threads`.
// `prefix`: `data` may end anywhere after HfGlobal (a bare codestream; a container must be whole). Sections are used
// only when their whole byte range is inside `data` (frame_info.rs:302-328), and group g only with its passes
// 0 .. group_passes[g] - 1 (see FrameState::group_passes).
std::unique_ptr<FrameState> parse_vardct_file(const uint8_t* data, size_t size, int threads = 1, bool prefix = false);

// Upsample8x::new (render/stages/upsample.rs:21-69): the 210 weights8 expanded by symmetry into the 64 5x5 kernels,
// out[(oy * 8 + ox) * 25 + ky * 5 + kx] for output pixel (ox, oy) of an LF sample and input (x + kx - 2, y + ky - 2).
void upsample8_kernel(const std::array<float, 210>& weights, float out[64 * 25]);

// Test hook: decode the LF groups of serial parses one at a time instead of in lockstep pairs.
void set_pair_lf_groups(bool on);

// Destroys a FrameState but keeps its large buffers (codestream copy, LF planes, per-block maps; ~4 MB for a 4K
// frame) in a bounded process-wide pool that parse_vardct_file draws from: a steady-state decode loop then does no
// large malloc / free, i.e. no mmap, page-fault and munmap (TLB shoot-down) traffic between the parse threads.
void recycle_frame_state(FrameState* fs);

}  // namespace jxg
