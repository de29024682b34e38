#include "region.h"

#include <algorithm>
#include <cstring>

namespace jxg {

namespace {

constexpr uint32_t kGroup = 256, kTileW = kFilterTileW, kTileH = kFilterTileH;  // HF group; filter tile

template <typename T>
void slice_plane(const T* src, size_t src_stride, uint32_t x0, uint32_t y0, uint32_t w, uint32_t h, std::vector<T>& dst) {
  dst.resize(size_t(w) * h);
  for (uint32_t y = 0; y < h; y++) memcpy(dst.data() + size_t(y) * w, src + size_t(y0 + y) * src_stride + x0, size_t(w) * sizeof(T));
}

}  // namespace

int slice_region(const JxgFrameDesc& full, const uint64_t* sec_off, const uint32_t* sec_len, uint32_t n_sections,
                 const JxgRegion& r, RegionSlice* out, const char** why, const uint8_t* group_passes) {
  auto bad = [&](const char* w) {
    *why = w;
    return int(JXG_ERR_ARGUMENT);
  };
  if (full.output_format == JXG_FORMAT_XYB_F32_PLANAR) return bad("region: XYB_F32_PLANAR output has no region form");
  const uint32_t W = full.width, Hh = full.height;
  const uint32_t o = (full.orientation == 0) ? 1u : full.orientation;
  if (o > 8) return bad("region: orientation must be 1..8");
  const uint32_t disp_w = o >= 5 ? Hh : W, disp_h = o >= 5 ? W : Hh;
  if (!r.width || !r.height) return bad("region: empty");
  if (r.x >= disp_w || r.y >= disp_h || r.width > disp_w - r.x || r.height > disp_h - r.y) return bad("region: outside the image");
  const uint32_t xg = (W + kGroup - 1) / kGroup, yg = (Hh + kGroup - 1) / kGroup, G = xg * yg;
  if (!full.num_passes || n_sections != G * full.num_passes) return bad("region: n_sections != groups * passes");
  // coded rectangle Rc: orientation maps rectangles to rectangles, so two opposite corners fix it
  uint32_t ax, ay, bx, by;
  coded_pixel(o, W, Hh, r.x, r.y, ax, ay);
  coded_pixel(o, W, Hh, r.x + r.width - 1, r.y + r.height - 1, bx, by);
  const uint32_t cx0 = std::min(ax, bx), cy0 = std::min(ay, by), cx1 = std::max(ax, bx) + 1, cy1 = std::max(ay, by) + 1;
  // pixels the region depends on: the halo around Rc, or around the filter tiles that meet Rc (vector path, see region.h)
  uint32_t rx0 = cx0, ry0 = cy0, rx1 = cx1, ry1 = cy1;
  if (full.gab && full.epf_iters == 2) {
    rx0 = rx0 / kTileW * kTileW;
    ry0 = ry0 / kTileH * kTileH;
    rx1 = std::min(W, (rx1 + kTileW - 1) / kTileW * kTileW);
    ry1 = std::min(Hh, (ry1 + kTileH - 1) / kTileH * kTileH);
  }
  const uint32_t H = filter_halo(full.gab != 0, full.epf_iters);
  const uint32_t gx0 = (rx0 > H ? rx0 - H : 0) / kGroup, gy0 = (ry0 > H ? ry0 - H : 0) / kGroup;
  const uint32_t gx1 = (std::min(W, rx1 + H) - 1) / kGroup + 1, gy1 = (std::min(Hh, ry1 + H) - 1) / kGroup + 1;
  const uint32_t ox = gx0 * kGroup, oy = gy0 * kGroup;
  const uint32_t sw = std::min(W, gx1 * kGroup) - ox, sh = std::min(Hh, gy1 * kGroup) - oy;
  RegionSlice& s = *out;
  s.origin[0] = ox;
  s.origin[1] = oy;
  s.coded_win[0] = cx0 - ox;
  s.coded_win[1] = cy0 - oy;
  s.coded_win[2] = cx1 - cx0;
  s.coded_win[3] = cy1 - cy0;
  // the window's top-left in the sub-frame's display output: the display image of the coded window's corners
  display_pixel(o, sw, sh, s.coded_win[0], s.coded_win[1], ax, ay);
  display_pixel(o, sw, sh, s.coded_win[0] + s.coded_win[2] - 1, s.coded_win[1] + s.coded_win[3] - 1, bx, by);
  s.window[0] = std::min(ax, bx);
  s.window[1] = std::min(ay, by);
  // sections: pass-major, sub-frame group order
  s.real_group.clear();
  for (uint32_t y = gy0; y < gy1; y++)
    for (uint32_t x = gx0; x < gx1; x++) s.real_group.push_back(y * xg + x);
  s.sec_off.clear();
  s.sec_len.clear();
  for (uint32_t p = 0; p < full.num_passes; p++)
    for (uint32_t g : s.real_group) {
      s.sec_off.push_back(sec_off[p * G + g]);
      s.sec_len.push_back(sec_len[p * G + g]);
    }
  // per-block tables (block origin ox / 8 = 32 gx0) and CfL tiles (origin ox / 64)
  const uint32_t xb = (W + 7) / 8, sxb = (sw + 7) / 8, syb = (sh + 7) / 8, bx0 = ox / 8, by0 = oy / 8;
  const uint32_t cxb = (xb + 7) / 8, scxb = (sxb + 7) / 8, scyb = (syb + 7) / 8;
  for (int c = 0; c < 3; c++) slice_plane(full.lf[c], xb, bx0, by0, sxb, syb, s.lf[c]);
  slice_plane(full.transform_map, xb, bx0, by0, sxb, syb, s.transform_map);
  slice_plane(full.raw_quant_map, xb, bx0, by0, sxb, syb, s.raw_quant_map);
  slice_plane(full.epf_map, xb, bx0, by0, sxb, syb, s.epf_map);
  slice_plane(full.quant_lf, xb, bx0, by0, sxb, syb, s.quant_lf);
  slice_plane(full.ytox_map, cxb, bx0 / 8, by0 / 8, scxb, scyb, s.ytox_map);
  slice_plane(full.ytob_map, cxb, bx0 / 8, by0 / 8, scxb, scyb, s.ytob_map);
  // a prefix frame: the sub-frame's pass counts and, for its groups without a pass, the LF window of the upsampling
  const uint32_t yb = (Hh + 7) / 8;
  s.group_passes.clear();
  for (int c = 0; c < 3; c++) s.lf_win[c].clear();
  std::fill(s.lf_size, s.lf_size + 2, 0u);
  std::fill(s.lf_window, s.lf_window + 4, 0u);
  if (group_passes) {
    for (uint32_t g : s.real_group) s.group_passes.push_back(group_passes[g]);
    s.lf_size[0] = xb;
    s.lf_size[1] = yb;
    if (std::find(s.group_passes.begin(), s.group_passes.end(), uint8_t(0)) != s.group_passes.end()) {
      const uint32_t wx0 = bx0 > 2 ? bx0 - 2 : 0, wy0 = by0 > 2 ? by0 - 2 : 0;
      const uint32_t wx1 = std::min(xb, bx0 + sxb + 2), wy1 = std::min(yb, by0 + syb + 2);
      s.lf_window[0] = wx0;
      s.lf_window[1] = wy0;
      s.lf_window[2] = wx1;
      s.lf_window[3] = wy1;
      for (int c = 0; c < 3; c++) slice_plane(full.lf[c], xb, wx0, wy0, wx1 - wx0, wy1 - wy0, s.lf_win[c]);
    }
  }
  s.desc = full;
  s.desc.width = sw;
  s.desc.height = sh;
  for (int c = 0; c < 3; c++) s.desc.lf[c] = s.lf[c].data();
  s.desc.transform_map = s.transform_map.data();
  s.desc.raw_quant_map = s.raw_quant_map.data();
  s.desc.epf_map = s.epf_map.data();
  s.desc.quant_lf = s.quant_lf.data();
  s.desc.ytox_map = s.ytox_map.data();
  s.desc.ytob_map = s.ytob_map.data();
  return 0;
}

}  // namespace jxg
