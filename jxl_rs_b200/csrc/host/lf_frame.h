// Host front end of a 1:8 thumbnail of a VarDCT frame: the headers, TOC and LfGlobal, and for every LF group the bit
// position where the symbols of its LF-coefficient stream start (decode_vardct_lf, frame/modular/mod.rs:931-982). The
// LF pixels, the ModularLF stream of extra channels, the HF metadata, HfGlobal and the HF groups are not decoded: the
// LF streams are decoded on the device (jxg_modular_batch_add_lf).
#pragma once
#include <cstdint>
#include <memory>
#include <vector>

#include "frame.h"
#include "modular_frame.h"

namespace jxg {

struct LfFrameState {
  FrameState fs;                            // headers, TOC and LfGlobal only: no planes, no HfGlobal
  std::vector<ModularChannel> coded;        // shapes of the LF image channels Y, X, B (xb x yb, no sample planes)
  std::vector<ModularGroupStream> streams;  // one per LF group: rects Y, X, B of the group, stream id VarDCTLF(g)
  std::vector<float> mul;                   // per stream 1 / 2^extra_precision (mod.rs:938)
  uint64_t hf_bytes = 0;                    // JxgImageInfo::hf_bytes as jxg_parse_file reports it
};

// Reads no byte past the end of the last LF-group section. A one-section frame (at most 256x256) is parsed in full by
// parse_vardct_file as well, because its hf_bytes is known only where HfGlobal ends: its section must be whole and its
// HF metadata and HfGlobal valid. Accepts and refuses with the header and scope checks of parse_vardct_file. Throws
// jxg::Error.
std::unique_ptr<LfFrameState> parse_vardct_lf_file(const uint8_t* data, size_t size);

}  // namespace jxg
