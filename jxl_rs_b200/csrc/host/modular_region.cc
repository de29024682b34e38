#include "modular_region.h"

#include <algorithm>

#include "region.h"

namespace jxg {

void PlaneRect::unite(const PlaneRect& o) {
  if (o.empty()) return;
  if (empty()) {
    *this = o;
    return;
  }
  x0 = std::min(x0, o.x0);
  y0 = std::min(y0, o.y0);
  x1 = std::max(x1, o.x1);
  y1 = std::max(y1, o.y1);
}

bool PlaneRect::meets(const PlaneRect& o) const {
  return !empty() && !o.empty() && x0 < o.x1 && o.x0 < x1 && y0 < o.y1 && o.y0 < y1;
}

namespace {

PlaneRect whole(const ModularBuf& b) {
  PlaneRect r;
  if (b.w && b.h) r = PlaneRect{0, 0, b.w, b.h};
  return r;
}

}  // namespace

int plan_modular_region(const ModularFrameState& ms, const JxgRegion* region, ModularRegionPlan& p, const char** why) {
  const uint32_t W = ms.header.xsize(), H = ms.header.ysize(), o = ms.file.orientation;
  const uint32_t disp_w = o >= 5 ? H : W, disp_h = o >= 5 ? W : H;
  const size_t nb = ms.bufs.size();
  p.need.assign(nb, PlaneRect());
  if (region) {
    const JxgRegion& r = *region;
    if (!r.width || !r.height) {
      *why = "region: empty";
      return JXG_ERR_ARGUMENT;
    }
    if (r.x >= disp_w || r.y >= disp_h || r.width > disp_w - r.x || r.height > disp_h - r.y) {
      *why = "region: outside the image";
      return JXG_ERR_ARGUMENT;
    }
    // orientation maps rectangles to rectangles: two opposite corners fix the coded one
    uint32_t ax, ay, bx, by;
    coded_pixel(o, W, H, r.x, r.y, ax, ay);
    coded_pixel(o, W, H, r.x + r.width - 1, r.y + r.height - 1, bx, by);
    p.coded = PlaneRect{std::min(ax, bx), std::min(ay, by), std::max(ax, bx) + 1, std::max(ay, by) + 1};
    p.out_x = r.x;
    p.out_y = r.y;
    p.out_w = r.width;
    p.out_h = r.height;
    for (uint32_t c = 0; c < ms.num_color_channels; c++) p.need[ms.out_buf[c]].unite(p.coded);
  } else {
    p.coded = PlaneRect{0, 0, W, H};
    p.out_x = p.out_y = 0;
    p.out_w = disp_w;
    p.out_h = disp_h;
    for (size_t i = 0; i < nb; i++) p.need[i] = whole(ms.bufs[i]);
  }
  // backwards through the plan: what each step reads for what is needed of what it writes
  p.step.assign(ms.steps.size(), PlaneRect());
  for (size_t si = ms.steps.size(); si-- > 0;) {
    const ModularStep& s = ms.steps[si];
    if (s.kind == kJobRct) {
      PlaneRect u = p.need[s.a];
      u.unite(p.need[s.b]);
      u.unite(p.need[s.c]);
      p.need[s.a] = p.need[s.b] = p.need[s.c] = p.step[si] = u;
    } else if (s.kind == kJobPalette) {
      PlaneRect u;
      for (uint32_t c = 0; c < s.n; c++) u.unite(p.need[s.c + c]);
      p.need[s.a].unite(u);
      p.need[s.b] = whole(ms.bufs[s.b]);
      p.step[si] = u;
    } else {
      const PlaneRect out = p.need[s.c];
      if (out.empty()) continue;
      const bool hz = s.kind == kJobHSqueeze;
      const uint32_t an = hz ? ms.bufs[s.a].w : ms.bufs[s.a].h, rn = hz ? ms.bufs[s.b].w : ms.bufs[s.b].h;
      const uint32_t end = hz ? out.x1 : out.y1;  // outputs [0, end) along the squeezed axis
      const uint32_t pairs = std::min(rn, (end + 1) / 2);
      const uint32_t written = 2 * pairs + (((an + rn) & 1) && end == an + rn ? 1 : 0);
      const uint32_t avgs = std::min(pairs + 1, an);  // the next average of the last pair
      if (hz) {
        p.step[si] = PlaneRect{0, out.y0, written, out.y1};
        p.need[s.a].unite(PlaneRect{0, out.y0, avgs, out.y1});
        p.need[s.b].unite(PlaneRect{0, out.y0, pairs, out.y1});
      } else {
        p.step[si] = PlaneRect{out.x0, 0, out.x1, written};
        p.need[s.a].unite(PlaneRect{out.x0, 0, out.x1, avgs});
        p.need[s.b].unite(PlaneRect{out.x0, 0, out.x1, pairs});
      }
    }
  }
  for (PlaneRect& r : p.need)
    if (r.empty()) r = PlaneRect();
  // streams: every one with a rect that meets its channel's need, decoded whole
  p.arena = p.need;
  p.selected.assign(ms.hf.size(), 0);
  for (size_t g = 0; g < ms.hf.size(); g++) {
    const ModularGroupStream& st = ms.hf[g];
    if (st.empty) continue;
    for (const ModularRect& r : st.rects)
      if (p.need[r.chan].meets(PlaneRect{r.x0, r.y0, r.x0 + r.w, r.y0 + r.h})) p.selected[g] = 1;
    if (p.selected[g])
      for (const ModularRect& r : st.rects)
        if (r.w && r.h) p.arena[r.chan].unite(PlaneRect{r.x0, r.y0, r.x0 + r.w, r.y0 + r.h});
  }
  for (size_t si = 0; si < ms.steps.size(); si++)
    if (ms.steps[si].kind == kJobHSqueeze || ms.steps[si].kind == kJobVSqueeze) p.arena[ms.steps[si].c].unite(p.step[si]);
  return 0;
}

}  // namespace jxg
