// See lf_frame.h.
#include "lf_frame.h"

#include <algorithm>

namespace jxg {

std::unique_ptr<LfFrameState> parse_vardct_lf_file(const uint8_t* data, size_t size) {
  auto lp = std::make_unique<LfFrameState>();
  FrameState& fs = lp->fs;
  read_vardct_headers(fs, data, size, WholeSections::kLf);
  const FrameHeader& h = fs.header;
  const uint8_t* base = fs.codestream.data() + fs.sections_base;
  for (int c = 0; c < 3; c++) {
    ModularChannel ch;
    ch.w = fs.xb;
    ch.h = fs.yb;
    lp->coded.push_back(ch);
  }
  // decode_vardct_lf up to the first symbol: extra_precision, then the sub-bitstream's GroupHeader and local tree
  auto lf_stream = [&](uint32_t g, BitReader& br, size_t sec) {
    const uint32_t gd = h.group_dim(), xlg = h.xsize_lf_groups();
    const uint32_t x0 = (g % xlg) * gd, y0 = (g / xlg) * gd;
    const uint32_t w = std::min(gd, fs.xb - x0), hh = std::min(gd, fs.yb - y0);
    ModularGroupStream st;
    st.group = g;
    st.stream_id = 1 + g;
    st.sec_off = fs.sections_base + fs.toc.offsets[sec];
    st.sec_len = fs.toc.lengths[sec];
    const uint32_t extra_precision = uint32_t(br.read(2));
    for (uint32_t c = 0; c < 3; c++) st.rects.push_back(ModularRect{c, x0, y0, w, hh});
    st.empty = false;
    read_group_stream_header(st, lp->coded, fs.has_global_tree, br);
    lp->streams.push_back(std::move(st));
    lp->mul.push_back(1.0f / float(1u << extra_precision));
  };
  if (fs.toc.offsets.size() == 1) {
    // One section holds LfGlobal, the LF group, HfGlobal and the HF group in one bit stream; the HF byte count of
    // jxg_parse_file is the size of that stream behind HfGlobal, so the (at most 256x256) frame is parsed in full for it.
    std::unique_ptr<FrameState> full = parse_vardct_file(data, size, 1);
    lp->hf_bytes = full->hf_len[0];
    recycle_frame_state(full.release());
    BitReader br(base + fs.toc.offsets[0], fs.toc.lengths[0]);
    decode_lf_global(fs, br);
    lf_stream(0, br, 0);
  } else {
    {
      BitReader br(base + fs.toc.offsets[0], fs.toc.lengths[0]);
      decode_lf_global(fs, br);
    }
    for (uint32_t g = 0; g < h.num_lf_groups(); g++) {
      BitReader br(base + fs.toc.offsets[1 + g], fs.toc.lengths[1 + g]);
      lf_stream(g, br, 1 + g);
    }
    for (size_t s = 2 + h.num_lf_groups(); s < fs.toc.lengths.size(); s++) lp->hf_bytes += fs.toc.lengths[s];
  }
  return lp;
}

}  // namespace jxg
