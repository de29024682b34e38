// Region decode of a Modular frame: the one place that decides which group streams a display rectangle needs and which
// rectangle of each plan buffer the inverse transforms read and write for it (the dependency cone).
//
// The inverse plan (ModularFrameState::steps) is walked backwards from the coded rectangle of the region:
// * global RCT: the three channels each need the union of the three needs (a pixel mixes the same position of all);
// * palette: the index channel needs the union of the colour channels' needs, the palette channel is needed whole;
// * horizontal unsqueeze (squeeze.rs:390, k_unsqueeze_h): each output pair depends on the output to its left, so an
//   output rectangle [x0, x1) x [y0, y1) is produced from column 0: the pairs up to the one holding x1 - 1 (and the
//   tail column when x1 reaches an odd output width) are written, which reads those residual columns and the average
//   columns up to the next average of the last pair; vertical unsqueeze is the same along columns;
// * a coded channel decoded on the device needs every ModularHF stream whose rect in it meets its need; a stream is
//   entropy-decoded whole, so it writes all of its rects in all of its channels;
// * channels decoded by the host (section 0, ModularLF) are already there: only their needed rectangle is uploaded.
// So on Squeeze frames the cone reaches the top-left corner of each level: a crop at the bottom right of a squeezed
// image needs most of its group streams. That is the dependency structure of the transform, not slack.
// Every rectangle is a bounding box; the whole frame is the case where every buffer is needed whole.
#pragma once
#include <cstdint>
#include <vector>

#include "../../../include/jxg.h"
#include "modular_frame.h"

namespace jxg {

struct PlaneRect {  // [x0, x1) x [y0, y1); empty rectangles are all zero
  uint32_t x0 = 0, y0 = 0, x1 = 0, y1 = 0;
  bool empty() const { return x0 >= x1 || y0 >= y1; }
  uint32_t w() const { return empty() ? 0 : x1 - x0; }
  uint32_t h() const { return empty() ? 0 : y1 - y0; }
  void unite(const PlaneRect& o);  // bounding box
  bool meets(const PlaneRect& o) const;
};

struct ModularRegionPlan {
  PlaneRect coded;                // the region in coded coordinates (the whole frame without a region)
  uint32_t out_x = 0, out_y = 0;  // display coordinates of the output's top-left pixel
  uint32_t out_w = 0, out_h = 0;  // output size in pixels (display orientation)
  std::vector<PlaneRect> need;    // per plan buffer: the rectangle later steps and the store read
  std::vector<PlaneRect> arena;   // per plan buffer: the rectangle the plane arena holds (need + what is written)
  std::vector<PlaneRect> step;    // per plan step: the rectangle the job writes (RCT: in place; palette: unused)
  std::vector<uint8_t> selected;  // per ModularHF stream (ms.hf): decoded for the region
};

// The cone of `region` (display coordinates, the frame's orientation applied), or of the whole frame for nullptr.
// Returns 0, or JXG_ERR_ARGUMENT with *why set for an empty region or one outside the image.
int plan_modular_region(const ModularFrameState& ms, const JxgRegion* region, ModularRegionPlan& plan, const char** why);

}  // namespace jxg
