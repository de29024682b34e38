// Region decode of a VarDCT frame: the one place that decides which HF groups a display rectangle needs.
// A region becomes a sub-frame — a self-contained JxgFrameDesc + section list over a rectangle of whole 256x256 groups
// — and a window of that sub-frame to store. The sub-frame decode equals the full decode on the region because
// * every pixel depends only on IDCT pixels within the filter halo H (Gaborish 1, EPF 2 / +1 / +3), and the sub-frame
//   holds all of them or shares the frame edge they are mirrored at;
// * its origin is a multiple of 256, which keeps the phase of everything tied to coordinates: 8x8 blocks, 64x64 CfL
//   tiles, the 32x32 dither table and the 64x32 filter tiles;
// * with Gaborish + EPF 2 (the only configuration with a vector filter path) the halo is taken around the filter tiles
//   that meet the region, so that each of them is interior in the sub-frame exactly when it is interior in the frame and
//   takes the same path.
// A region of a prefix frame (jxg_parse_file_prefix) takes the same groups. A group there without an HF pass (k_g = 0)
// is the LF image upsampled 8x (k_upsample_lf8), whose window reads LF samples up to 2 columns and rows outside the
// group, mirrors rows at the frame's LF height and takes its column margins from the frame's LF width. Those are LF
// samples, not neighbouring HF groups, so the selection does not grow; instead the sub-frame carries the frame's LF
// geometry and an LF window (its LF blocks grown by 2, clipped to the frame), and the kernel works in frame coordinates.
#pragma once
#include <cstdint>
#include <vector>

#include "../../../include/jxg.h"

namespace jxg {

struct RegionSlice {
  JxgFrameDesc desc;                     // the sub-frame; its table pointers point into the vectors below
  std::vector<uint64_t> sec_off;         // sections of the sub-frame (pass-major, sub-frame group order)
  std::vector<uint32_t> sec_len;
  std::vector<uint32_t> real_group;      // sub-frame group -> group of the full frame
  uint32_t origin[2];                    // coded origin of the sub-frame in the frame (multiples of 256)
  uint32_t coded_win[4];                 // the region in the sub-frame's coded coordinates: x, y, width, height
  uint32_t window[2];                    // the region's top-left in the sub-frame's display-oriented output
  std::vector<float> lf[3];
  std::vector<uint8_t> transform_map, epf_map, quant_lf;
  std::vector<int32_t> raw_quant_map;
  std::vector<int8_t> ytox_map, ytob_map;
  // A region of a prefix frame: the passes of each sub-frame group (group_passes[real_group[i]]), the frame's LF size
  // (blocks across and down) and, when one of those pass counts is 0, the LF window the upsampling reads: x0, y0, x1, y1
  // (half-open) of the frame's LF image and its three planes. All zero and empty otherwise.
  std::vector<uint8_t> group_passes;
  uint32_t lf_size[2] = {0, 0};
  uint32_t lf_window[4] = {0, 0, 0, 0};
  std::vector<float> lf_win[3];
};

// Coded pixel of display pixel (dx, dy) for a coded w x h frame: the inverse of display_pixel
// (headers/image_metadata.rs:85-96, k_orient).
inline void coded_pixel(uint32_t o, uint32_t w, uint32_t h, uint32_t dx, uint32_t dy, uint32_t& x, uint32_t& y) {
  switch (o) {
    case 2: x = w - 1 - dx; y = dy; break;
    case 3: x = w - 1 - dx; y = h - 1 - dy; break;
    case 4: x = dx; y = h - 1 - dy; break;
    case 5: x = dy; y = dx; break;
    case 6: x = dy; y = h - 1 - dx; break;
    case 7: x = w - 1 - dy; y = h - 1 - dx; break;
    case 8: x = w - 1 - dy; y = dx; break;
    default: x = dx; y = dy; break;
  }
}

// display_pixel itself.
inline void display_pixel(uint32_t o, uint32_t w, uint32_t h, uint32_t x, uint32_t y, uint32_t& dx, uint32_t& dy) {
  switch (o) {
    case 2: dx = w - 1 - x; dy = y; break;
    case 3: dx = w - 1 - x; dy = h - 1 - y; break;
    case 4: dx = x; dy = h - 1 - y; break;
    case 5: dx = y; dy = x; break;
    case 6: dx = h - 1 - y; dy = x; break;
    case 7: dx = h - 1 - y; dy = w - 1 - x; break;
    case 8: dx = y; dy = w - 1 - x; break;
    default: dx = x; dy = y; break;
  }
}

// Geometry of the fused filter kernel the selection depends on: its 64x32 tile (kTW x kTH, launch.h kFusedTileW / H)
// and its halo in pixels, Gaborish 1 + EPF 2 / +1 / +3 (FCfg<GAB, EPF>::H). kernels.cu checks both against the kernel's
// own constants at compile time.
constexpr uint32_t kFilterTileW = 64, kFilterTileH = 32;
constexpr uint32_t filter_halo(bool gab, uint32_t epf_iters) {
  return (gab ? 1 : 0) + (epf_iters >= 1 ? 2 : 0) + (epf_iters >= 2 ? 1 : 0) + (epf_iters >= 3 ? 3 : 0);
}

// Slices `full` (and its n_sections sections) to the region r, given in display coordinates (the frame's orientation
// applied; XYB output has none). Returns 0, or JXG_ERR_ARGUMENT with *why set when the region is empty or leaves the
// image, or the output format is XYB_F32_PLANAR. `group_passes` (a prefix frame: the passes of each group of the frame,
// nullptr otherwise) fills the prefix fields of the slice.
int slice_region(const JxgFrameDesc& full, const uint64_t* sec_off, const uint32_t* sec_len, uint32_t n_sections,
                 const JxgRegion& r, RegionSlice* out, const char** why, const uint8_t* group_passes = nullptr);

}  // namespace jxg
