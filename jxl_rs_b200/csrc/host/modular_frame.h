// Host front-end of one Modular-encoded frame (BASELINE config 5, SURVEY §8 rows a18/a19): everything jxl-rs does
// before the per-group pixel streams — headers, TOC, LfGlobal (global MA tree, FullModularImage header, global
// transforms, the "meta or small" channels of section 0), the ModularLF streams (channels with shift >= 3) — plus, for
// every ModularHF(group) section, its GroupHeader / local tree and the bit position where the pixel symbols start.
// The per-pixel decode of those sections and the inverse transforms are the device path (k_modular_* kernels).
//
// Reference: jxl/src/frame/decode.rs:307-427, jxl/src/frame/modular/mod.rs:258-490 (FullModularImage::read,
// read_section0, read_stream), modular/decode/bitstream.rs:134, modular/decode/common.rs:23 (stream ids).
#pragma once
#include <cstdint>
#include <memory>
#include <vector>

#include "headers.h"
#include "modular.h"

namespace jxg {

struct ModularRect {  // the part of coded channel `chan` one group stream carries (mod.rs:150 get_grid_rect)
  uint32_t chan, x0, y0, w, h;
};

struct ModularGroupStream {
  uint32_t group = 0;
  uint64_t stream_id = 0;
  uint64_t sec_off = 0;  // byte offset of the section in `codestream`
  uint32_t sec_len = 0;
  bool empty = true;           // all rects empty: nothing is coded (bitstream.rs:143-149)
  GroupHeader header;          // local header (only read when !empty)
  std::shared_ptr<ModularTree> local_tree;  // null: global tree
  uint64_t header_bitpos = 0;  // bit offset in the section of the GroupHeader (0 unless the frame has one section)
  uint64_t data_bitpos = 0;    // bit offset in the section of the first entropy-coded bit (ANS state / first symbol)
  uint32_t dist_multiplier = 0;  // widest channel after the local transforms: LZ77 special distances (bitstream.rs:193-202)
  std::vector<ModularRect> rects;  // in channel order; zero-sized ones keep their index (bitstream.rs:203-206)
};

// Symbolic inverse-transform plan over full-size i32 planes ("buffers"); buffers [0, coded.size()) are the coded
// channels, later ids are outputs of unsqueeze steps.
struct ModularBuf {
  uint32_t w = 0, h = 0;
};
// Kinds of the plan steps and of the device jobs that carry them out (the `kind` of launch_modular_jobs in
// cuda/modular_device.h): one numbering. It lives here because the front-end also builds without the CUDA headers.
enum ModularJobKind : uint32_t {
  kJobRct = 0,       // in place on a, b, c
  kJobHSqueeze = 1,  // horizontal unsqueeze: a avg, b residual -> c
  kJobVSqueeze = 2,  // vertical unsqueeze
  kJobStore = 3,     // final colour planes -> u8 output (device job only, no plan step)
  kJobPalette = 4,   // palette without delta entries: a index channel, b palette, c .. c + n - 1 the colour channels
  // Thumbnail jobs (device only), over a VarDCT LF image of three xb x yb planes at a, a + plane, a + 2 * plane:
  kJobLfDequant = 5,  // quantised Y, X, B (i32) of one LF group's rectangle -> dequantised X, Y, B (f32)
  kJobLfSmooth = 6,   // adaptive LF smoothing, X, Y, B at a -> c (out of place)
  kJobLfStore = 7,    // X, Y, B planes -> the thumbnail output
};
struct ModularStep {
  ModularJobKind kind = kJobRct;
  uint32_t a = 0, b = 0, c = 0;
  uint32_t rct_op = 0;
  uint32_t n = 0, num_colors = 0;  // palette: colour channels, explicit palette entries
};

struct ModularFrameState {
  bool device_plan_ok = true;  // false: a global transform has no device form (delta palettes): the device path refuses the frame
  FileHeader file;
  FrameHeader header;
  Toc toc;
  std::vector<uint8_t> codestream;
  size_t sections_base = 0;
  bool has_global_tree = false;
  ModularTree global_tree;
  GroupHeader global_header;
  uint32_t nb_meta = 0;
  uint32_t num_color_channels = 3;
  std::vector<ModularChannel> coded;   // channel list after the global meta-apply, full-size planes
  std::vector<uint8_t> host_decoded;   // per coded channel: 1 = filled by the host (section 0 / ModularLF)
  std::vector<ModularGroupStream> hf;  // one per group (single pass)
  // inverse plan
  std::vector<ModularBuf> bufs;
  std::vector<ModularStep> steps;
  uint32_t out_buf[3] = {0, 0, 0};  // buffers holding the final colour channels
};

// Reads what precedes the pixel symbols of one group stream (bitstream.rs:134-190): its GroupHeader and local tree, the
// bit position of its first entropy-coded bit and its LZ77 distance multiplier. `coded` gives the shifts of the channels
// the stream's rects index. Nothing is read for an empty stream.
void read_group_stream_header(ModularGroupStream& st, const std::vector<ModularChannel>& coded, bool has_global_tree,
                              BitReader& br);

// Parses a complete file holding one Modular frame. Throws jxg::Error (kErrUnsupported for features outside the
// scope of the device path).
std::unique_ptr<ModularFrameState> parse_modular_file(const uint8_t* data, size_t size);

}  // namespace jxg
