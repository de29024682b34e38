// Minimal from-scratch JPEG XL VarDCT *writer* for synthetic test frames
// (SURVEY Appendix A). Produces valid single-frame codestreams: default image
// metadata (8-bit sRGB, XYB), one VarDCT frame, ANS-coded LF (Modular with
// Gradient predictor), HF metadata and AC coefficients with the full context
// model of jxl/src/frame/group.rs:454-578 mirrored on the encoder side.
//
// Test-data tooling, not part of the product path.
#include <algorithm>
#include <atomic>
#include <exception>
#include <mutex>
#include <thread>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <stdexcept>
#include <string>
#include <vector>

#include "../jxl_rs_b200/csrc/host/frame.h"  // library dequant tables, natural orders, geometry tables
#include "../jxl_rs_b200/csrc/host/quant.h"  // custom dequant tables
#include "entropy_writer.h"

namespace jxs {

struct Rng {  // splitmix64
  uint64_t s;
  explicit Rng(uint64_t seed) : s(seed * 0x9E3779B97F4A7C15ull + 0x1234567ull) {}
  uint64_t next() {
    uint64_t z = (s += 0x9E3779B97F4A7C15ull);
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
  }
  double uniform() { return double(next() >> 11) * (1.0 / 9007199254740992.0); }
  uint32_t below(uint32_t n) { return uint32_t(next() % n); }
};

struct Params {
  uint32_t width, height;
  uint64_t seed;
  float distance;      // ~ butteraugli-style quality knob: larger = coarser quantisation
  uint32_t epf_iters;  // 0..3
  uint32_t gab;        // 0/1
  uint32_t profile;    // 0 = DCT8x8 only, 1 = mixed <= 32x32 (+4x8/8x4/4x4), 2 = + 64x64 family, 3 = + 128 / 256 families
  uint32_t lf_tree;    // coding of the LF image: 0 = one Gradient leaf per channel, 1 = libjxl-like (channel prefix,
                       // then a subtree on the weighted-predictor property 15 with Weighted leaves)
  uint32_t entropy;    // AC coefficient streams: 0 = ANS, 1 = prefix codes (entropy_coding/huffman.rs)
  uint32_t orientation = 1;  // ImageMetadata.orientation 1..8
  // colour encoding written into ImageMetadata (the pixels are always produced from sRGB-primaries XYB; the variants
  // exist to exercise the decoder's output-colour derivation): 0 default sRGB, 1 linear, 2 gamma 0.45455,
  // 3 P3 / D65 / PQ at 1000 nits, 4 BT2100 / D65 / HLG at 1000 nits, 5 custom primaries / DCI white / BT709, 6 grey sRGB,
  // 7 DCI transfer function with the E white point
  uint32_t colour = 0;
  uint32_t x_qm_scale = 3, b_qm_scale = 2;  // FrameHeader, 0..7 (group.rs:395-396)
  // Custom dequantisation matrices, one entry per table index (see jxs_encode_synthetic_ex); all mode 0 = all_default
  struct DequantSpec {
    uint32_t mode = 0;                                   // quant_weights.rs:128 (0 library, 1..7)
    std::vector<std::pair<uint32_t, unsigned>> fields;   // (value, bits) after the mode, in the reader's order
    std::vector<int32_t> raw;                            // mode 7: 3 channels of 8*REQUIRED_SIZE_X columns
  };
  std::vector<DequantSpec> dequant = {};                 // empty or kNumQuantTables entries
};

// Worker threads inside one encode (jxs_set_threads): only loops whose result does not depend on the order of
// evaluation are split, so the bitstream of a (size, seed, parameters) tuple is the same for every thread count.
static std::atomic<int> g_threads{1};
template <typename F>
static void parallel_for(size_t n, F&& fn) {
  const size_t nt = std::min<size_t>(size_t(std::max(1, g_threads.load())), n);
  if (nt <= 1) {
    for (size_t i = 0; i < n; i++) fn(i);
    return;
  }
  std::atomic<size_t> next{0};
  std::exception_ptr err;
  std::mutex mu;
  auto work = [&] {
    try {
      for (;;) {
        const size_t i = next.fetch_add(1);
        if (i >= n) return;
        fn(i);
      }
    } catch (...) {
      std::lock_guard<std::mutex> lk(mu);
      err = std::current_exception();
    }
  };
  std::vector<std::thread> th;
  for (size_t t = 1; t < nt; t++) th.emplace_back(work);
  work();
  for (auto& t : th) t.join();
  if (err) std::rethrow_exception(err);
}

// ---------------------------------------------------------------------------
// synthetic source image (linear RGB in [0,1])
// ---------------------------------------------------------------------------
static void make_image(const Params& p, std::vector<float> (&rgb)[3]) {
  const uint32_t W = p.width, H = p.height;
  Rng rng(p.seed);
  for (auto& c : rgb) c.assign(size_t(W) * H, 0.0f);
  struct Wave {
    float fx, fy, ph, amp[3];
  };
  std::vector<Wave> waves(6);
  for (auto& w : waves) {
    float period = 200.0f + float(rng.uniform()) * 1300.0f;
    float ang = float(rng.uniform()) * 6.2831853f;
    w.fx = std::cos(ang) * 6.2831853f / period;
    w.fy = std::sin(ang) * 6.2831853f / period;
    w.ph = float(rng.uniform()) * 6.2831853f;
    for (float& a : w.amp) a = 0.02f + 0.08f * float(rng.uniform());
  }
  auto grid_noise = [&](uint32_t cell, float amp, int chan_corr) {
    uint32_t gw = W / cell + 2, gh = H / cell + 2;
    std::vector<float> g[3];
    for (int c = 0; c < 3; c++) {
      g[c].resize(size_t(gw) * gh);
      for (auto& v : g[c]) v = float(rng.uniform()) - 0.5f;
    }
    if (chan_corr)
      for (size_t i = 0; i < g[0].size(); i++) {
        g[1][i] = 0.8f * g[0][i] + 0.2f * g[1][i];
        g[2][i] = 0.7f * g[0][i] + 0.3f * g[2][i];
      }
    parallel_for(H, [&](size_t yi) {
      const uint32_t y = uint32_t(yi);
      uint32_t gy = y / cell;
      float fy = float(y % cell) / float(cell);
      for (uint32_t x = 0; x < W; x++) {
        uint32_t gx = x / cell;
        float fx = float(x % cell) / float(cell);
        for (int c = 0; c < 3; c++) {
          const float* q = g[c].data() + size_t(gy) * gw + gx;
          float v = (q[0] * (1 - fx) + q[1] * fx) * (1 - fy) + (q[gw] * (1 - fx) + q[gw + 1] * fx) * fy;
          rgb[c][size_t(y) * W + x] += amp * v;
        }
      }
    });
  };
  float base[3] = {0.35f + 0.2f * float(rng.uniform()), 0.35f + 0.2f * float(rng.uniform()), 0.3f + 0.2f * float(rng.uniform())};
  parallel_for(H, [&](size_t yi) {
    const uint32_t y = uint32_t(yi);
    for (uint32_t x = 0; x < W; x++) {
      for (int c = 0; c < 3; c++) {
        float v = base[c] + 0.1f * float(x) / float(W) - 0.08f * float(y) / float(H);
        for (auto& w : waves) v += w.amp[c] * std::sin(w.fx * float(x) + w.fy * float(y) + w.ph);
        rgb[c][size_t(y) * W + x] = v;
      }
    }
  });
  grid_noise(64, 0.25f, 1);
  grid_noise(16, 0.12f, 1);
  grid_noise(4, 0.09f, 1);
  grid_noise(2, 0.06f, 0);
  // shapes with hard edges
  int nshapes = 12 + int(rng.below(12));
  for (int s = 0; s < nshapes; s++) {
    float cx = float(rng.uniform()) * W, cy = float(rng.uniform()) * H;
    float rad = (0.02f + 0.1f * float(rng.uniform())) * float(std::min(W, H));
    float col[3] = {float(rng.uniform()) * 0.5f - 0.25f, float(rng.uniform()) * 0.5f - 0.25f, float(rng.uniform()) * 0.5f - 0.25f};
    bool disc = rng.below(2);
    int x0 = std::max(0, int(cx - rad)), x1 = std::min(int(W), int(cx + rad));
    int y0 = std::max(0, int(cy - rad)), y1 = std::min(int(H), int(cy + rad));
    for (int y = y0; y < y1; y++)
      for (int x = x0; x < x1; x++) {
        if (disc && (x - cx) * (x - cx) + (y - cy) * (y - cy) > rad * rad) continue;
        for (int c = 0; c < 3; c++) rgb[c][size_t(y) * W + x] += col[c];
      }
  }
  // fine per-pixel noise
  for (int c = 0; c < 3; c++)
    for (auto& v : rgb[c]) {
      v += 0.05f * (float(rng.uniform()) - 0.5f);
      v = std::min(1.0f, std::max(0.0f, v));
    }
}

// inverse of render/stages/xyb.rs:197-241 with the default opsin matrix
static void to_xyb(std::vector<float> (&rgb)[3], const jxg::OpsinInverseMatrix& op) {
  double m[9], inv[9];
  for (int i = 0; i < 9; i++) m[i] = op.inverse_matrix[i];
  double det = m[0] * (m[4] * m[8] - m[5] * m[7]) - m[1] * (m[3] * m[8] - m[5] * m[6]) + m[2] * (m[3] * m[7] - m[4] * m[6]);
  inv[0] = (m[4] * m[8] - m[5] * m[7]) / det;
  inv[1] = (m[2] * m[7] - m[1] * m[8]) / det;
  inv[2] = (m[1] * m[5] - m[2] * m[4]) / det;
  inv[3] = (m[5] * m[6] - m[3] * m[8]) / det;
  inv[4] = (m[0] * m[8] - m[2] * m[6]) / det;
  inv[5] = (m[2] * m[3] - m[0] * m[5]) / det;
  inv[6] = (m[3] * m[7] - m[4] * m[6]) / det;
  inv[7] = (m[1] * m[6] - m[0] * m[7]) / det;
  inv[8] = (m[0] * m[4] - m[1] * m[3]) / det;
  double bias[3] = {op.opsin_biases[0], op.opsin_biases[1], op.opsin_biases[2]};
  double cb[3] = {std::cbrt(bias[0]), std::cbrt(bias[1]), std::cbrt(bias[2])};
  size_t n = rgb[0].size();
  const size_t chunk = 1 << 16;
  parallel_for((n + chunk - 1) / chunk, [&](size_t ci) {
  for (size_t i = ci * chunk; i < std::min(n, (ci + 1) * chunk); i++) {
    double r = rgb[0][i], g = rgb[1][i], b = rgb[2][i];
    double l = inv[0] * r + inv[1] * g + inv[2] * b, mm = inv[3] * r + inv[4] * g + inv[5] * b, s = inv[6] * r + inv[7] * g + inv[8] * b;
    double lg = std::cbrt(l - bias[0]) + cb[0], mg = std::cbrt(mm - bias[1]) + cb[1], sg = std::cbrt(s - bias[2]) + cb[2];
    rgb[0][i] = float((lg - mg) * 0.5);
    rgb[1][i] = float((lg + mg) * 0.5);
    rgb[2][i] = float(sg);
  }
  });
}

// ---------------------------------------------------------------------------
// forward transforms (inverse of the decoder's IDCT convention:
// out[y] = in[0] + sqrt2 * sum_u in[u] cos((y+.5) u pi / N))
// ---------------------------------------------------------------------------
struct DctTables {
  std::vector<float> fwd[9];  // [log2 N][u * N + y]
  DctTables() {
    for (int l = 0; l <= 8; l++) {
      int N = 1 << l;
      fwd[l].resize(size_t(N) * N);
      for (int u = 0; u < N; u++)
        for (int y = 0; y < N; y++)
          fwd[l][size_t(u) * N + y] = float((u == 0 ? 1.0 : std::sqrt(2.0) * std::cos((y + 0.5) * u * M_PI / N)) / N);
    }
  }
};
static const DctTables kDct;
static int ilog2(int n) {
  int l = 0;
  while ((1 << l) < n) l++;
  return l;
}
// px: R x C (stride given) -> D[vf * C + hf]
static void forward_dct2d(const float* px, size_t stride, int R, int C, float* D) {
  std::vector<float> tmp(size_t(R) * C);
  const float* fc = kDct.fwd[ilog2(C)].data();
  const float* fr = kDct.fwd[ilog2(R)].data();
  for (int y = 0; y < R; y++)
    for (int hf = 0; hf < C; hf++) {
      float s = 0;
      for (int x = 0; x < C; x++) s += fc[size_t(hf) * C + x] * px[size_t(y) * stride + x];
      tmp[size_t(y) * C + hf] = s;
    }
  for (int vf = 0; vf < R; vf++)
    for (int hf = 0; hf < C; hf++) {
      float s = 0;
      for (int y = 0; y < R; y++) s += fr[size_t(vf) * R + y] * tmp[size_t(y) * C + hf];
      D[size_t(vf) * C + hf] = s;
    }
}
static void small_idct(float* v, int n) {  // decoder-convention inverse, O(n^2)
  if (n == 1) return;
  std::vector<float> out(n);
  for (int y = 0; y < n; y++) {
    double s = v[0];
    for (int u = 1; u < n; u++) s += std::sqrt(2.0) * v[u] * std::cos((y + 0.5) * u * M_PI / n);
    out[y] = float(s);
  }
  for (int y = 0; y < n; y++) v[y] = out[y];
}
static double llf_c(int i, int n) {  // tests.rs:138 scales(n)[i] / n
  return std::cos(i / (16.0 * n) * M_PI) * std::cos(i / (8.0 * n) * M_PI) * std::cos(i / (4.0 * n) * M_PI);
}

struct Varblock {
  uint16_t bx, by;  // frame block coordinates of the first block
  uint8_t t;
};

struct Frame {
  Params p;
  uint32_t xb, yb, xg, yg, num_groups, xlfg, ylfg, num_lf_groups;
  std::vector<uint8_t> transform_map;  // t | 128 first
  std::vector<uint8_t> raw_quant;      // 1..255
  std::vector<uint8_t> sharp;
  std::vector<int8_t> ytox, ytob;
  std::vector<int32_t> lfq[3];         // quantised LF ints (X, Y, B)
  std::vector<Varblock> blocks;        // raster order of first blocks
  std::vector<std::vector<int32_t>> coeffs;  // per varblock: 3 * num_coeffs quantised ints (storage layout)
  uint32_t global_scale, quant_lf;
};

using jxg::kCoveredBlocksX;
using jxg::kCoveredBlocksY;

static void plan_transforms(Frame& f) {
  Rng rng(f.p.seed ^ 0xabcdefull);
  f.transform_map.assign(size_t(f.xb) * f.yb, 255);
  auto place = [&](uint32_t bx, uint32_t by, int t) -> bool {
    uint32_t cx = kCoveredBlocksX[t], cy = kCoveredBlocksY[t];
    if (bx + cx > f.xb || by + cy > f.yb) return false;
    if ((bx / 32) != ((bx + cx - 1) / 32) || (by / 32) != ((by + cy - 1) / 32)) return false;
    for (uint32_t y = 0; y < cy; y++)
      for (uint32_t x = 0; x < cx; x++)
        if (f.transform_map[size_t(by + y) * f.xb + bx + x] != 255) return false;
    for (uint32_t y = 0; y < cy; y++)
      for (uint32_t x = 0; x < cx; x++) f.transform_map[size_t(by + y) * f.xb + bx + x] = uint8_t(t) | ((x == 0 && y == 0) ? 128 : 0);
    return true;
  };
  if (f.p.profile >= 1) {
    // profile 3 first drops the largest transforms on 32x32-block (group) and 16x16-block cells:
    // DCT256X256 (24), 256X128 (25), 128X256 (26), 128X128 (21), 128X64 (22), 64X128 (23)
    if (f.p.profile >= 3) {
      for (uint32_t by = 0; by < f.yb; by += 32)
        for (uint32_t bx = 0; bx < f.xb; bx += 32) {
          const uint32_t r = rng.below(100);
          if (r < 15 && place(bx, by, 24)) continue;
          if (r < 25 && place(bx, by, 25)) { place(bx + 16, by, 25); continue; }   // 256 rows x 128 cols, twice
          if (r < 35 && place(bx, by, 26)) { place(bx, by + 16, 26); continue; }   // 128 rows x 256 cols, twice
          for (uint32_t qy = 0; qy < 32; qy += 16)
            for (uint32_t qx = 0; qx < 32; qx += 16) {
              const uint32_t q = rng.below(100), x = bx + qx, y = by + qy;
              if (q < 25) place(x, y, 21);
              else if (q < 40) { place(x, y, 22); place(x + 8, y, 22); }           // 128 rows x 64 cols
              else if (q < 55) { place(x, y, 23); place(x, y + 8, 23); }           // 64 rows x 128 cols
            }
        }
    }
    // 4x4-block cells (32x32 px); profile 2 first drops some 8x8-block (64x64 px) transforms
    if (f.p.profile >= 2) {
      for (uint32_t by = 0; by + 8 <= f.yb; by += 8)
        for (uint32_t bx = 0; bx + 8 <= f.xb; bx += 8) {
          uint32_t r = rng.below(100);
          if (r < 6) place(bx, by, 18);                                                 // DCT64X64
          else if (r < 9) { place(bx, by, 19); place(bx + 4, by, 19); }                 // 2x DCT64X32 (8 rows x 4 cols)
          else if (r < 12) { place(bx, by, 20); place(bx, by + 4, 20); }                // 2x DCT32X64
        }
    }
    for (uint32_t by = 0; by < f.yb; by += 4)
      for (uint32_t bx = 0; bx < f.xb; bx += 4) {
        uint32_t r = rng.below(100);
        if (r < 12) place(bx, by, 5);                                                  // DCT32X32
        else if (r < 18) { place(bx, by, 10); place(bx + 2, by, 10); }                 // DCT32X16 (4 rows x 2 cols)
        else if (r < 24) { place(bx, by, 11); place(bx, by + 2, 11); }                 // DCT16X32
        else if (r < 28) { for (int i = 0; i < 4; i++) place(bx + i, by, 8); }         // DCT32X8 (4 rows x 1 col)
        else if (r < 32) { for (int i = 0; i < 4; i++) place(bx, by + i, 9); }         // DCT8X32
        else if (r < 60) {
          for (int qy = 0; qy < 2; qy++)
            for (int qx = 0; qx < 2; qx++) {
              uint32_t q = rng.below(10), x = bx + 2 * qx, y = by + 2 * qy;
              if (q < 4) place(x, y, 4);                                               // DCT16X16
              else if (q < 6) { place(x, y, 6); place(x + 1, y, 6); }                  // DCT16X8 (2 rows x 1 col)
              else if (q < 8) { place(x, y, 7); place(x, y + 1, 7); }                  // DCT8X16
            }
        }
      }
  }
  for (uint32_t by = 0; by < f.yb; by++)
    for (uint32_t bx = 0; bx < f.xb; bx++) {
      if (f.transform_map[size_t(by) * f.xb + bx] != 255) continue;
      int t = 0;
      if (f.p.profile == 4) {  // also IDENTITY, DCT2X2 and AFV0-3 (random coefficients, see random_coeff_type)
        static const int kTypes[10] = {0, 12, 13, 3, 1, 2, 14, 15, 16, 17};
        t = kTypes[rng.below(10)];
      } else if (f.p.profile >= 1) {
        uint32_t r = rng.below(100);
        t = r < 70 ? 0 : r < 80 ? 12 : r < 90 ? 13 : 3;  // DCT, DCT4X8, DCT8X4, DCT4X4
      }
      place(bx, by, t);
    }
  for (uint32_t by = 0; by < f.yb; by++)
    for (uint32_t bx = 0; bx < f.xb; bx++)
      if (f.transform_map[size_t(by) * f.xb + bx] & 128) f.blocks.push_back(Varblock{uint16_t(bx), uint16_t(by), uint8_t(f.transform_map[size_t(by) * f.xb + bx] & 127)});
}

// IDENTITY, DCT2X2 and AFV0-3 have no forward transform here: their varblocks get the block mean as LF and random
// sparse quantised coefficients, valid input for the decoder but not a picture of the source.
static bool random_coeff_type(int t) { return t == 1 || t == 2 || (t >= 14 && t <= 17); }

// Transforms one varblock of one channel: returns coefficients in *storage*
// layout plus the cy x cx LF samples.
static void forward_varblock(int t, const float* px, size_t stride, std::vector<float>& co, std::vector<float>& lf) {
  const int cx = kCoveredBlocksX[t], cy = kCoveredBlocksY[t];
  const int R = 8 * cy, C = 8 * cx;
  co.assign(size_t(R) * C, 0.0f);
  lf.assign(size_t(cx) * cy, 0.0f);
  if (t == 12 || t == 13 || t == 3 || random_coeff_type(t)) {
    float mean = 0;
    for (int y = 0; y < 8; y++)
      for (int x = 0; x < 8; x++) mean += px[size_t(y) * stride + x];
    lf[0] = mean / 64.0f;
    if (random_coeff_type(t)) return;
    if (t == 12) {  // DCT4X8: halves along y, each 4 rows x 8 cols (transform.rs:638-661)
      float D[2][32];
      for (int h = 0; h < 2; h++) forward_dct2d(px + size_t(h) * 4 * stride, stride, 4, 8, D[h]);
      for (int h = 0; h < 2; h++)
        for (int iy = 0; iy < 4; iy++)
          for (int ix = 0; ix < 8; ix++)
            if (ix || iy) co[(h + iy * 2) * 8 + ix] = D[h][iy * 8 + ix];
      co[8] = (D[0][0] - D[1][0]) * 0.5f;
    } else if (t == 13) {  // DCT8X4: halves along x, each 8 rows x 4 cols, stored [hf][vf] (transform.rs:613-637)
      float D[2][32];
      for (int h = 0; h < 2; h++) forward_dct2d(px + size_t(h) * 4, stride, 8, 4, D[h]);  // D[vf * 4 + hf]
      for (int h = 0; h < 2; h++)
        for (int hf = 0; hf < 4; hf++)
          for (int vf = 0; vf < 8; vf++)
            if (hf || vf) co[(h + hf * 2) * 8 + vf] = D[h][vf * 4 + hf];
      co[8] = (D[0][0] - D[1][0]) * 0.5f;
    } else {  // DCT4X4 (transform.rs:579-612)
      float D[4][16];
      for (int y = 0; y < 2; y++)
        for (int x = 0; x < 2; x++) forward_dct2d(px + size_t(y) * 4 * stride + x * 4, stride, 4, 4, D[y * 2 + x]);
      for (int y = 0; y < 2; y++)
        for (int x = 0; x < 2; x++)
          for (int hf = 0; hf < 4; hf++)
            for (int vf = 0; vf < 4; vf++)
              if (hf || vf) co[(y + hf * 2) * 8 + x + vf * 2] = D[y * 2 + x][vf * 4 + hf];
      float d0 = D[0][0], d1 = D[1][0], d2 = D[2][0], d3 = D[3][0];
      co[1] = (d0 + d1 - d2 - d3) * 0.25f;
      co[8] = (d0 - d1 + d2 - d3) * 0.25f;
      co[9] = (d0 - d1 - d2 + d3) * 0.25f;
    }
    co[0] = 0.0f;
    return;
  }
  std::vector<float> D(size_t(R) * C);
  forward_dct2d(px, stride, R, C, D.data());
  const bool wide = R < C;
  for (int vf = 0; vf < R; vf++)
    for (int hf = 0; hf < C; hf++) co[wide ? size_t(vf) * C + hf : size_t(hf) * R + vf] = D[size_t(vf) * C + hf];
  // LF samples from the lowest cy x cx frequencies (inverse of the reinterpreting DCT, tests.rs:138-180)
  std::vector<float> low(size_t(cx) * cy);
  for (int vf = 0; vf < cy; vf++)
    for (int hf = 0; hf < cx; hf++) low[size_t(vf) * cx + hf] = float(D[size_t(vf) * C + hf] * llf_c(vf, cy) * llf_c(hf, cx));
  std::vector<float> line(std::max(cx, cy));
  for (int vf = 0; vf < cy; vf++) {
    for (int hf = 0; hf < cx; hf++) line[hf] = low[size_t(vf) * cx + hf];
    small_idct(line.data(), cx);
    for (int x = 0; x < cx; x++) low[size_t(vf) * cx + x] = line[x];
  }
  for (int x = 0; x < cx; x++) {
    for (int vf = 0; vf < cy; vf++) line[vf] = low[size_t(vf) * cx + x];
    small_idct(line.data(), cy);
    for (int y = 0; y < cy; y++) lf[size_t(y) * cx + x] = line[y];
  }
  // LLF positions are implied by the LF image: not coded
  for (int vf = 0; vf < cy; vf++)
    for (int hf = 0; hf < cx; hf++) co[wide ? size_t(vf) * C + hf : size_t(hf) * R + vf] = 0.0f;
}

// ---------------------------------------------------------------------------
// Modular sub-bitstream writer (fixed per-channel tree, one predictor)
// ---------------------------------------------------------------------------
struct Chan {
  uint32_t w, h;
  std::vector<int32_t> d;
};
static inline int64_t clamped_gradient(int64_t l, int64_t t, int64_t tl) {
  int64_t mn = std::min(l, t), mx = std::max(l, t), g = l + t - tl;
  return tl < mn ? mx : (tl > mx ? mn : g);
}
// MA tree in the bitstream's order (tree.rs:284-340: breadth first, children appended to the pending queue).
struct TNode {
  int property = -1;  // -1: leaf
  int32_t splitval = 0;
  uint32_t left = 0, right = 0;  // property > splitval -> left
  uint32_t predictor = 5, ctx = 0;
};
struct TDesc {  // nested description; left / right index into the description vector
  int property;
  int32_t splitval;
  uint32_t predictor;
  int left, right;
};
static std::vector<TNode> flatten_tree(const std::vector<TDesc>& d, int root) {
  std::vector<TNode> out;
  std::vector<int> q{root};
  for (size_t qi = 0; qi < q.size(); qi++) {
    const TDesc& t = d[q[qi]];
    TNode n;
    if (t.property >= 0) {
      n.property = t.property;
      n.splitval = t.splitval;
      n.left = uint32_t(q.size());
      n.right = n.left + 1;
      q.push_back(t.left);
      q.push_back(t.right);
    } else {
      n.predictor = t.predictor;
    }
    out.push_back(n);
  }
  uint32_t leaf = 0;
  for (auto& n : out)
    if (n.property < 0) n.ctx = leaf++;
  return out;
}

// lf_tree: false = one leaf (`predictor`) per channel; true = libjxl-like: the same channel prefix, then per channel
// a subtree that splits on the weighted-predictor property (15) and predicts with the weighted predictor (6).
static void write_modular(BitWriter& bw, const std::vector<Chan>& ch, uint32_t predictor, bool wp_tree = false) {
  bool empty = true;
  for (auto& c : ch)
    if (c.w && c.h) empty = false;
  if (empty) return;
  bw.write(0, 1);  // use_global_tree = false
  bw.write(1, 1);  // WeightedHeader all_default
  bw.write(0, 2);  // no transforms
  const size_t n = ch.size();
  std::vector<TDesc> d;
  auto leaf = [&](uint32_t pred) {
    d.push_back(TDesc{-1, 0, pred, -1, -1});
    return int(d.size() - 1);
  };
  auto split = [&](int prop, int32_t val, int l, int r) {
    d.push_back(TDesc{prop, val, 0, l, r});
    return int(d.size() - 1);
  };
  auto channel_subtree = [&]() {
    if (!wp_tree) return leaf(predictor);
    // contexts by the signed maximum neighbouring error of the weighted predictor (in 1/8 sample units)
    static const int32_t kThr[6] = {96, 24, 5, -6, -25, -97};
    int t = leaf(6);
    for (int i = 5; i >= 0; i--) t = split(15, kThr[i], leaf(6), t);
    return t;
  };
  int root = channel_subtree();  // channel 0
  for (size_t c = 1; c < n; c++) root = split(0, int32_t(c) - 1, channel_subtree(), root);  // channel > c-1 -> c..
  const std::vector<TNode> tree = flatten_tree(d, root);
  std::vector<Token> tt;
  for (const TNode& nd : tree) {
    if (nd.property >= 0) {
      tt.push_back(Token{1, uint32_t(nd.property + 1)});
      tt.push_back(Token{0, pack_signed(nd.splitval)});
    } else {
      tt.push_back(Token{1, 0});
      tt.push_back(Token{2, nd.predictor});
      tt.push_back(Token{3, 0});
      tt.push_back(Token{4, 0});
      tt.push_back(Token{5, 0});
    }
  }
  {
    uint32_t nc;
    HybridCfg cfg;
    std::vector<uint8_t> map = cluster_contexts(6, {&tt}, 8, nc, cfg);
    AnsCode code = build_code(6, map, nc, {&tt});
    write_code(bw, code);
    write_tokens(bw, code, tt);
  }
  const size_t num_leaves = (tree.size() + 1) / 2;
  std::vector<Token> dt;
  const jxg::WeightedHeader wph;
  for (size_t c = 0; c < n; c++) {
    const Chan& k = ch[c];
    if (!k.w || !k.h) continue;
    jxg::WpState wp(wph, wp_tree ? k.w : 0);
    for (uint32_t y = 0; y < k.h; y++)
      for (uint32_t x = 0; x < k.w; x++) {
        const int32_t* row = &k.d[size_t(y) * k.w];
        const int32_t* top = y ? row - k.w : row;
        const int32_t* toptop = y > 1 ? top - k.w : top;
        const int32_t left = x ? row[x - 1] : (y ? top[0] : 0);
        const int32_t t = y ? top[x] : left;
        const int32_t tl = (x && y) ? top[x - 1] : left;
        const int32_t tr = (x + 1 < k.w && y) ? top[x + 1] : t;
        const int32_t tt2 = y > 1 ? toptop[x] : t;
        int64_t wp_pred = 0;
        int32_t wp_prop = 0;
        if (wp_tree) wp.predict(x, y, t, left, tr, tl, tt2, wp_pred, wp_prop);
        const TNode* nd = &tree[0];
        while (nd->property >= 0) {
          const int32_t v = nd->property == 0 ? int32_t(c) : wp_prop;
          nd = &tree[v > nd->splitval ? nd->left : nd->right];
        }
        const int64_t pred = nd->predictor == 6   ? wp_pred
                             : nd->predictor == 5 ? clamped_gradient(left, t, tl)
                             : nd->predictor == 1 ? int64_t(left)
                                                  : 0;
        dt.push_back(Token{nd->ctx, pack_signed(int32_t(int64_t(row[x]) - pred))});
        if (wp_tree) wp.update(row[x], x, y);
      }
  }
  uint32_t nc;
  HybridCfg cfg;
  std::vector<uint8_t> map = cluster_contexts(num_leaves, {&dt}, 8, nc, cfg);
  AnsCode code = build_code(num_leaves, map, nc, {&dt});
  write_code(bw, code);
  write_tokens(bw, code, dt);
}

static void append_bits(BitWriter& dst, BitWriter& src) {
  size_t total = src.total;
  BitWriter copy = src;
  std::vector<uint8_t> bytes = copy.finish();
  size_t full = total / 8;
  for (size_t i = 0; i < full; i++) dst.write(bytes[i], 8);
  if (total % 8) dst.write(bytes[full], unsigned(total % 8));
}

static void write_toc_entry(BitWriter& bw, uint32_t v) {  // toc.rs:28
  if (v < 1024) bw.u2s_sel(0, v, 10);
  else if (v < 17408) bw.u2s_sel(1, v - 1024, 14);
  else if (v < 4211712) bw.u2s_sel(2, v - 17408, 22);
  else bw.u2s_sel(3, v - 4211712, 30);
}

// block_context_map.rs:20-31
static const uint16_t kFreqCtx[64] = {0xBAD, 0,  1,  2,  3,  4,  5,  6,  7,  8,  9,  10, 11, 12, 13, 14, 15, 15, 16, 16, 17, 17,
                                      18,    18, 19, 19, 20, 20, 21, 21, 22, 22, 23, 23, 23, 23, 24, 24, 24, 24, 25, 25, 25, 25,
                                      26,    26, 26, 26, 27, 27, 27, 27, 28, 28, 28, 28, 29, 29, 29, 29, 30, 30, 30, 30};
static const uint16_t kNzCtx[64] = {0xBAD, 0,   31,  62,  62,  93,  93,  93,  93,  123, 123, 123, 123, 152, 152, 152,
                                    152,   152, 152, 152, 152, 180, 180, 180, 180, 180, 180, 180, 180, 180, 180, 180,
                                    180,   206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206,
                                    206,   206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206, 206};
static const uint8_t kDefaultBlockCtx[39] = {0, 1, 2, 2, 3,  3,  4,  5,  6,  6,  6,  6,  6,  7, 8, 9, 9, 10, 11, 12,
                                             13, 14, 14, 14, 14, 14, 7, 8, 9, 9, 10, 11, 12, 13, 14, 14, 14, 14, 14};

std::vector<uint8_t> encode(const Params& p) {
  Frame f;
  f.p = p;
  const uint32_t W = p.width, H = p.height;
  f.xb = (W + 7) / 8;
  f.yb = (H + 7) / 8;
  f.xg = (W + 255) / 256;
  f.yg = (H + 255) / 256;
  f.num_groups = f.xg * f.yg;
  f.xlfg = (f.xb + 255) / 256;
  f.ylfg = (f.yb + 255) / 256;
  f.num_lf_groups = f.xlfg * f.ylfg;
  const uint32_t PW = f.xb * 8, PH = f.yb * 8;

  // ---- source image -> padded XYB planes ----
  std::vector<float> img[3];
  make_image(p, img);
  jxg::OpsinInverseMatrix opsin;
  to_xyb(img, opsin);
  std::vector<float> xyb[3];
  for (int c = 0; c < 3; c++) {
    xyb[c].resize(size_t(PW) * PH);
    for (uint32_t y = 0; y < PH; y++)
      for (uint32_t x = 0; x < PW; x++) xyb[c][size_t(y) * PW + x] = img[c][size_t(std::min(y, H - 1)) * W + std::min(x, W - 1)];
    img[c].clear();
    img[c].shrink_to_fit();
  }

  // ---- quantisation parameters ----
  f.global_scale = std::max<uint32_t>(1, std::min<uint32_t>(65535, uint32_t(std::lround(4587.0 / std::max(0.05f, p.distance)))));
  f.quant_lf = 16;
  const float inv_global_scale = 65536.0f / float(f.global_scale);
  const float x_dm = std::pow(1.0f / 1.25f, float(p.x_qm_scale) - 2.0f), b_dm = std::pow(1.0f / 1.25f, float(p.b_qm_scale) - 2.0f);
  // the dequantisation tables the decoder will use, computed by the front-end from the fields as written
  std::vector<float> custom_tables[jxg::kNumQuantTables];
  const float* tables[jxg::kNumQuantTables];
  for (int i = 0; i < jxg::kNumQuantTables; i++) {
    tables[i] = jxg::library_dequant_table(i).data();
    if (p.dequant.empty() || p.dequant[i].mode == 0) continue;
    const Params::DequantSpec& s = p.dequant[i];
    try {
      jxg::QuantEncoding e;
      if (s.mode == 7) {
        e.mode = jxg::QuantEncoding::kRaw;
        e.qtable_den = jxg::f16_bits_to_float(uint16_t(s.fields.at(0).first));
        e.qtable = s.raw;
      } else {
        BitWriter w;
        w.write(s.mode, 3);
        for (auto& fb : s.fields) w.write(fb.first, fb.second);
        std::vector<uint8_t> bytes = w.finish();
        jxg::BitReader br(bytes.data(), bytes.size());
        e = jxg::read_quant_encoding(i, br, jxg::FrameHeader(), nullptr);
      }
      custom_tables[i] = jxg::compute_dequant_table(e, i);
      tables[i] = custom_tables[i].data();
    } catch (const jxg::Error&) {
      // an encoding the decoder refuses: written as given, the coefficients quantised with the library table
    }
  }
  Rng rng(p.seed ^ 0x5151ull);
  plan_transforms(f);
  const size_t nb = size_t(f.xb) * f.yb;
  f.raw_quant.assign(nb, 5);
  f.sharp.assign(nb, 4);
  {  // smooth fields for the quant field and EPF sharpness
    uint32_t cw = f.xb / 16 + 2, chh = f.yb / 16 + 2;
    std::vector<uint8_t> q(size_t(cw) * chh), s(size_t(cw) * chh);
    for (auto& v : q) v = uint8_t(3 + rng.below(6));
    for (auto& v : s) v = uint8_t(rng.below(8));
    for (const Varblock& vb : f.blocks) {
      uint32_t cx = kCoveredBlocksX[vb.t], cy = kCoveredBlocksY[vb.t];
      uint8_t rq = q[size_t(vb.by / 16) * cw + vb.bx / 16];
      for (uint32_t y = 0; y < cy; y++)
        for (uint32_t x = 0; x < cx; x++) {
          f.raw_quant[size_t(vb.by + y) * f.xb + vb.bx + x] = rq;
          f.sharp[size_t(vb.by + y) * f.xb + vb.bx + x] = s[size_t((vb.by + y) / 16) * cw + (vb.bx + x) / 16];
        }
    }
  }
  const uint32_t cxb = (f.xb + 7) / 8, cyb = (f.yb + 7) / 8;
  f.ytox.assign(size_t(cxb) * cyb, 0);
  f.ytob.assign(size_t(cxb) * cyb, 0);
  for (auto& v : f.ytox) v = int8_t(int(rng.below(9)) - 4);
  for (auto& v : f.ytob) v = int8_t(int(rng.below(17)) - 8);

  // ---- transforms + quantisation ----
  for (auto& q : f.lfq) q.assign(nb, 0);
  f.coeffs.resize(f.blocks.size());
  const float inv_quant_lf = 65536.0f / (float(f.global_scale) * float(f.quant_lf));
  const float lf_fac[3] = {(1.0f / 4096.0f) * inv_quant_lf, (1.0f / 512.0f) * inv_quant_lf, (1.0f / 256.0f) * inv_quant_lf};
  parallel_for(f.blocks.size(), [&](size_t bi) {
    std::vector<float> co[3], lf[3];
    const Varblock& vb = f.blocks[bi];
    const int t = vb.t;
    const uint32_t cx = kCoveredBlocksX[t], cy = kCoveredBlocksY[t];
    const size_t num_coeffs = size_t(cx) * cy * 64;
    for (int c = 0; c < 3; c++) forward_varblock(t, &xyb[c][size_t(vb.by) * 8 * PW + size_t(vb.bx) * 8], PW, co[c], lf[c]);
    // LF (modular/mod.rs:837-889 inverted)
    for (uint32_t y = 0; y < cy; y++)
      for (uint32_t x = 0; x < cx; x++) {
        size_t o = size_t(vb.by + y) * f.xb + vb.bx + x, i = size_t(y) * cx + x;
        int32_t qy = int32_t(std::lround(lf[1][i] / lf_fac[1]));
        float yy = float(qy) * lf_fac[1];
        f.lfq[1][o] = qy;
        f.lfq[0][o] = int32_t(std::lround((lf[0][i] - yy * 0.0f) / lf_fac[0]));
        f.lfq[2][o] = int32_t(std::lround((lf[2][i] - yy * 1.0f) / lf_fac[2]));
      }
    // HF (group.rs:100-177 inverted, without the decoder-side bias adjustment)
    const float* mat = tables[jxg::quant_table_for_transform(t)];
    const float rq = float(f.raw_quant[size_t(vb.by) * f.xb + vb.bx]);
    const float sy = inv_global_scale / rq, sx = sy * x_dm, sb = sy * b_dm;
    const size_t ci = size_t(vb.by / 8) * cxb + vb.bx / 8;
    const float x_cc = 0.0f + float(f.ytox[ci]) / 84.0f, b_cc = 1.0f + float(f.ytob[ci]) / 84.0f;
    std::vector<int32_t>& q = f.coeffs[bi];
    q.assign(3 * num_coeffs, 0);
    auto quant = [](float v) {
      float a = std::fabs(v);
      if (a < 0.58f) return int32_t(0);
      return int32_t(std::copysign(std::floor(a + 0.42f), v));
    };
    if (random_coeff_type(t)) {  // about one coefficient in four, in [-3, 3]; position 0 is the LF sample
      Rng cr(p.seed * 0x2545F4914F6CDD1Dull + bi);
      for (size_t k = 1; k < num_coeffs; k++)
        for (int c = 0; c < 3; c++)
          if (cr.below(4) == 0) q[size_t(c) * num_coeffs + k] = int32_t(cr.below(7)) - 3;
      return;
    }
    const int R = 8 * int(cy), C = 8 * int(cx);
    const bool plain_dct = !(t == 12 || t == 13 || t == 3);
    for (size_t k = 0; k < num_coeffs; k++) {
      if (plain_dct) {  // skip LLF positions
        int vf = R < C ? int(k) / C : int(k) % R, hf = R < C ? int(k) % C : int(k) / R;
        if (vf < int(cy) && hf < int(cx)) continue;
      } else if (k == 0) {
        continue;
      }
      int32_t qy = quant(co[1][k] / (mat[num_coeffs + k] * sy));
      float dy = float(qy) * mat[num_coeffs + k] * sy;
      q[num_coeffs + k] = qy;
      q[k] = quant((co[0][k] - x_cc * dy) / (mat[k] * sx));
      q[2 * num_coeffs + k] = quant((co[2][k] - b_cc * dy) / (mat[2 * num_coeffs + k] * sb));
    }
  });
  for (auto& pl : xyb) {
    pl.clear();
    pl.shrink_to_fit();
  }

  // ---- AC tokens per group (group.rs:454-578 mirrored) ----
  std::vector<std::vector<Token>> ac(f.num_groups);
  {
    std::vector<uint32_t> block_index(nb, 0);
    for (size_t bi = 0; bi < f.blocks.size(); bi++) block_index[size_t(f.blocks[bi].by) * f.xb + f.blocks[bi].bx] = uint32_t(bi);
    std::vector<std::vector<uint32_t>> orders(13);
    for (int s = 0; s < 13; s++) orders[s] = jxg::natural_coeff_order(s);
    parallel_for(f.num_groups, [&](size_t gi) {
      const uint32_t g = uint32_t(gi);
      uint32_t bx0 = (g % f.xg) * 32, by0 = (g / f.xg) * 32;
      uint32_t gw = std::min(32u, f.xb - bx0), gh = std::min(32u, f.yb - by0);
      uint32_t nz[3][1024];
      memset(nz, 0, sizeof(nz));
      std::vector<Token>& out = ac[g];
      for (uint32_t by = 0; by < gh; by++)
        for (uint32_t bx = 0; bx < gw; bx++) {
          size_t o = size_t(by0 + by) * f.xb + bx0 + bx;
          if (!(f.transform_map[o] & 128)) continue;
          int t = f.transform_map[o] & 127;
          uint32_t cx = kCoveredBlocksX[t], cy = kCoveredBlocksY[t], shape = jxg::kBlockShapeId[t];
          size_t num_blocks = size_t(cx) * cy, num_coeffs = num_blocks * 64;
          unsigned lnb = 0;
          while ((size_t(1) << lnb) < num_blocks) lnb++;
          const std::vector<int32_t>& q = f.coeffs[block_index[o]];
          for (int c : {1, 0, 2}) {
            const int32_t* qc = &q[size_t(c) * num_coeffs];
            const std::vector<uint32_t>& order = orders[shape];
            size_t nonzeros = 0;
            for (size_t k = num_blocks; k < num_coeffs; k++) nonzeros += qc[order[k]] != 0;
            size_t predicted;
            if (bx == 0) predicted = by == 0 ? 32 : nz[c][(by - 1) * 32];
            else if (by == 0) predicted = nz[c][bx - 1];
            else predicted = (nz[c][(by - 1) * 32 + bx] + nz[c][by * 32 + bx - 1] + 1) / 2;
            size_t idx = (c < 2 ? size_t(c ^ 1) : 2) * 13 + shape;
            size_t block_context = kDefaultBlockCtx[idx];
            size_t nzc = predicted < 8 ? predicted : predicted < 64 ? 4 + predicted / 2 : 36;
            out.push_back(Token{uint32_t(nzc * 15 + block_context), uint32_t(nonzeros)});
            uint32_t nzv = uint32_t((nonzeros + num_blocks - 1) >> lnb);
            for (uint32_t iy = 0; iy < cy; iy++)
              for (uint32_t ix = 0; ix < cx; ix++) nz[c][(by + iy) * 32 + bx + ix] = nzv;
            size_t histo_offset = 15 * 37 + 458 * block_context;
            size_t prev = nonzeros > num_coeffs / 16 ? 0 : 1;
            for (size_t k = num_blocks; k < num_coeffs && nonzeros; k++) {
              size_t ctx = histo_offset + (kNzCtx[((nonzeros + num_blocks - 1) >> lnb) & 63] + kFreqCtx[(k >> lnb) & 63]) * 2 + prev;
              int32_t v = qc[order[k]];
              out.push_back(Token{uint32_t(ctx), pack_signed(v)});
              prev = v != 0;
              nonzeros -= prev;
            }
          }
        }
    });
  }
  const size_t num_ac_ctx = 15 * (37 + 458);
  std::vector<const std::vector<Token>*> ac_ptrs;
  for (auto& v : ac) ac_ptrs.push_back(&v);
  uint32_t ac_clusters;
  HybridCfg cfg;
  std::vector<uint8_t> ac_map = cluster_contexts(num_ac_ctx, ac_ptrs, 48, ac_clusters, cfg);
  // entropy 0 / 1: ANS / prefix codes; 2 / 3: the same with LZ77 copies (runs of equal coefficients, mostly zeros)
  const bool use_lz = p.entropy >= 2, use_prefix = (p.entropy & 1) != 0;
  std::vector<std::vector<Sym>> ac_syms;
  AnsCode ac_code;
  if (use_lz) {
    Lz77 lz;
    lz.enabled = true;
    const HybridCfg len_cfg{0, 0, 0};
    ac_syms.resize(ac.size());
    parallel_for(ac.size(), [&](size_t g) { ac_syms[g] = lz77_symbols(ac[g], cfg, lz, len_cfg, uint32_t(num_ac_ctx)); });
    ac_map.push_back(uint8_t(ac_clusters));  // the distance context gets a cluster of its own
    std::vector<const std::vector<Sym>*> sp;
    for (auto& v : ac_syms) sp.push_back(&v);
    ac_code = build_code_lz77(num_ac_ctx + 1, ac_map, ac_clusters + 1, sp, lz, use_prefix);
    ac_code.lz_len_cfg = len_cfg;
  } else {
    ac_code = build_code(num_ac_ctx, ac_map, ac_clusters, ac_ptrs, 6, use_prefix);
  }

  // ---- sections ----
  BitWriter lf_global;
  lf_global.write(1, 1);  // LfQuantFactors default (quantizer.rs:32)
  {                       // QuantizerParams (quantizer.rs:60-77)
    uint32_t gs = f.global_scale;
    if (gs <= 2048) lf_global.u2s_sel(0, gs - 1, 11);
    else if (gs <= 4096) lf_global.u2s_sel(1, gs - 2049, 11);
    else if (gs <= 8192) lf_global.u2s_sel(2, gs - 4097, 12);
    else lf_global.u2s_sel(3, gs - 8193, 16);
    lf_global.write(0, 2);  // quant_lf = 16
  }
  lf_global.write(1, 1);  // default BlockContextMap
  lf_global.write(1, 1);  // default ColorCorrelationParams
  lf_global.write(0, 1);  // no global tree

  std::vector<BitWriter> lf_groups(f.num_lf_groups);
  for (uint32_t g = 0; g < f.num_lf_groups; g++) {
    BitWriter& bw = lf_groups[g];
    uint32_t x0 = (g % f.xlfg) * 256, y0 = (g / f.xlfg) * 256;
    uint32_t w = std::min(256u, f.xb - x0), h = std::min(256u, f.yb - y0);
    bw.write(0, 2);  // extra_precision
    std::vector<Chan> ch(3);
    const int order[3] = {1, 0, 2};  // stored Y, X, B
    for (int i = 0; i < 3; i++) {
      ch[i].w = w;
      ch[i].h = h;
      ch[i].d.resize(size_t(w) * h);
      for (uint32_t y = 0; y < h; y++)
        for (uint32_t x = 0; x < w; x++) ch[i].d[size_t(y) * w + x] = f.lfq[order[i]][size_t(y0 + y) * f.xb + x0 + x];
    }
    write_modular(bw, ch, 5, f.p.lf_tree != 0);
    // HF metadata (modular/mod.rs:984-1080)
    std::vector<int32_t> types, quants;
    for (uint32_t y = 0; y < h; y++)
      for (uint32_t x = 0; x < w; x++) {
        size_t o = size_t(y0 + y) * f.xb + x0 + x;
        if (f.transform_map[o] & 128) {
          types.push_back(f.transform_map[o] & 127);
          quants.push_back(int32_t(f.raw_quant[o]) - 1);
        }
      }
    uint32_t count = uint32_t(types.size());
    bw.write(count - 1, ceil_log2(uint64_t(w) * h));
    uint32_t cw = (w + 7) / 8, chh = (h + 7) / 8;
    std::vector<Chan> mc(4);
    mc[0].w = mc[1].w = cw;
    mc[0].h = mc[1].h = chh;
    mc[0].d.resize(size_t(cw) * chh);
    mc[1].d.resize(size_t(cw) * chh);
    for (uint32_t y = 0; y < chh; y++)
      for (uint32_t x = 0; x < cw; x++) {
        mc[0].d[size_t(y) * cw + x] = f.ytox[size_t(y0 / 8 + y) * cxb + x0 / 8 + x];
        mc[1].d[size_t(y) * cw + x] = f.ytob[size_t(y0 / 8 + y) * cxb + x0 / 8 + x];
      }
    mc[2].w = count;
    mc[2].h = 2;
    mc[2].d = types;
    mc[2].d.insert(mc[2].d.end(), quants.begin(), quants.end());
    mc[3].w = w;
    mc[3].h = h;
    mc[3].d.resize(size_t(w) * h);
    for (uint32_t y = 0; y < h; y++)
      for (uint32_t x = 0; x < w; x++) mc[3].d[size_t(y) * w + x] = f.sharp[size_t(y0 + y) * f.xb + x0 + x];
    write_modular(bw, mc, 1);
  }

  BitWriter hf_global;
  bool all_default = true;
  for (const auto& s : p.dequant) all_default &= s.mode == 0;
  hf_global.write(all_default ? 1 : 0, 1);            // DequantMatrices all_default (quant_weights.rs:1093)
  if (!all_default)
    for (int i = 0; i < jxg::kNumQuantTables; i++) {  // QuantEncoding::decode (quant_weights.rs:117-255)
      const Params::DequantSpec& s = p.dequant[i];
      hf_global.write(s.mode, 3);
      for (auto& fb : s.fields) hf_global.write(fb.first, fb.second);
      if (s.mode == 7) {  // decode_quant_table (modular/mod.rs:1083-1122): stream 1 + 3 num_lf_groups + i, local tree
        const uint32_t w = 8u * jxg::kQuantTableRows[i], h = 8u * jxg::kQuantTableCols[i];
        std::vector<Chan> ch(3);
        for (int c = 0; c < 3; c++) {
          ch[c].w = w;
          ch[c].h = h;
          ch[c].d.assign(s.raw.begin() + size_t(c) * w * h, s.raw.begin() + size_t(c + 1) * w * h);
        }
        write_modular(hf_global, ch, 5);
      }
    }
  hf_global.write(0, ceil_log2(f.num_groups));        // num_histograms - 1
  hf_global.write(2, 2);                              // used_orders selector 2 => natural orders
  write_code(hf_global, ac_code);

  std::vector<BitWriter> hf_groups(f.num_groups);
  parallel_for(f.num_groups, [&](size_t g) {
    // histogram_index: ceil_log2(num_histograms = 1) = 0 bits
    if (use_lz) write_symbols(hf_groups[g], ac_code, ac_syms[g]);
    else write_tokens(hf_groups[g], ac_code, ac[g]);
  });

  // ---- file assembly ----
  BitWriter out;
  out.write(0xff, 8);
  out.write(0x0a, 8);
  // SizeHeader (size.rs:31-47)
  auto write_dim = [&](uint32_t v) {
    uint32_t m = v - 1;
    if (m < (1u << 9)) out.u2s_sel(0, m, 9);
    else if (m < (1u << 13)) out.u2s_sel(1, m, 13);
    else if (m < (1u << 18)) out.u2s_sel(2, m, 18);
    else out.u2s_sel(3, m, 30);
  };
  out.write(0, 1);  // small = false
  write_dim(H);
  out.write(0, 3);  // ratio 0: explicit xsize
  write_dim(W);
  if (p.orientation == 1 && p.colour == 0) {
    out.write(1, 1);  // ImageMetadata all_default
  } else {  // headers/image_metadata.rs:197-236
    auto write_enum = [&](uint32_t v) {  // jxl_macros default enum coder: u2S(0, 1, Bits(4) + 2, Bits(6) + 18)
      if (v == 0) out.u2s_sel(0);
      else if (v == 1) out.u2s_sel(1);
      else if (v < 18) out.u2s_sel(2, v - 2, 4);
      else out.u2s_sel(3, v - 18, 6);
    };
    auto write_f16 = [&](float v) {  // exactly representable positive values only (headers/encodings.rs:59-74)
      int e = 0;
      float m = std::frexp(v, &e);  // v = m * 2^e, m in [0.5, 1)
      const uint32_t mant = uint32_t(std::lround((m * 2.0f - 1.0f) * 1024.0f));
      out.write(v == 0.0f ? 0u : (uint32_t(e - 1 + 15) << 10) | mant, 16);
    };
    auto write_xy = [&](double x, double y) {  // CustomXY: pack_signed(round(v * 1e6)) through u2S (color_encoding.rs:91-100)
      for (double v : {x, y}) {
        const uint32_t u = pack_signed(int32_t(std::lround(v * 1e6)));
        if (u < (1u << 19)) out.u2s_sel(0, u, 19);
        else if (u < 524288u + (1u << 19)) out.u2s_sel(1, u - 524288u, 19);
        else if (u < 1048576u + (1u << 20)) out.u2s_sel(2, u - 1048576u, 20);
        else out.u2s_sel(3, u - 2097152u, 21);
      }
    };
    out.write(0, 1);                    // all_default
    out.write(1, 1);                    // extra_fields
    out.write(p.orientation - 1, 3);
    out.write(0, 1);                    // have_intrinsic_size
    out.write(0, 1);                    // have_preview
    out.write(0, 1);                    // have_animation
    out.write(0, 1);                    // BitDepth: integer samples
    out.u2s_sel(0);                     //           8 bits
    out.write(1, 1);                    // modular_16bit_sufficient
    out.u2s_sel(0);                     // no extra channels
    out.write(1, 1);                    // xyb_encoded
    bool hdr = false;
    if (p.colour == 0) {
      out.write(1, 1);                  // ColorEncoding all_default
    } else {  // headers/color_encoding.rs:166-196
      out.write(0, 1);
      out.write(0, 1);                  // want_icc
      write_enum(p.colour == 6 ? 1 : 0);  // colour space RGB / Gray
      uint32_t wp = 1, prim = 1, tf = 13;  // D65, sRGB primaries, sRGB curve
      bool gamma = false;
      switch (p.colour) {
        case 1: tf = 8; break;
        case 2: gamma = true; break;
        case 3: prim = 11; tf = 16; hdr = true; break;
        case 4: prim = 9; tf = 18; hdr = true; break;
        case 5: wp = 11; prim = 2; tf = 1; break;
        case 6: break;
        default: wp = 10; tf = 17; break;
      }
      write_enum(wp);
      if (p.colour != 6) {
        write_enum(prim);
        if (prim == 2) {
          write_xy(0.66, 0.31);
          write_xy(0.28, 0.62);
          write_xy(0.14, 0.07);
        }
      }
      out.write(gamma ? 1 : 0, 1);      // have_gamma
      if (gamma) out.write(4545455, 24);
      else write_enum(tf);
      write_enum(1);                    // rendering intent: relative
    }
    if (hdr) {  // ToneMapping (image_metadata.rs:156-167)
      out.write(0, 1);
      write_f16(1000.0f);               // intensity_target
      write_f16(0.0f);                  // min_nits
      out.write(0, 1);                  // relative_to_max_display
      write_f16(0.0f);                  // linear_below
    } else {
      out.write(1, 1);                  // ToneMapping all_default
    }
    out.write_u64(0);                   // extensions
  }
  out.write(1, 1);  // CustomTransformData all_default
  out.zero_pad_to_byte();
  // FrameHeader (frame_header.rs:267-444)
  const bool default_header = p.epf_iters == 2 && p.gab == 1 && p.x_qm_scale == 3 && p.b_qm_scale == 2;
  if (default_header) {
    out.write(1, 1);
  } else {
    out.write(0, 1);       // all_default
    out.write(0, 2);       // RegularFrame
    out.write(0, 1);       // VarDCT
    out.write_u64(0);      // flags
    out.write(0, 2);       // upsampling = 1
    out.write(p.x_qm_scale, 3);
    out.write(p.b_qm_scale, 3);
    out.write(0, 2);       // num_passes = 1
    out.write(0, 1);       // have_crop
    out.write(0, 2);       // blending mode Replace
    out.write(1, 1);       // is_last
    out.write(0, 2);       // name length 0
    out.write(0, 1);       // RestorationFilter all_default = 0
    out.write(p.gab, 1);   // gab
    if (p.gab) out.write(0, 1);  // gab_custom
    out.write(p.epf_iters, 2);
    if (p.epf_iters > 0) {
      out.write(0, 1);  // epf_sharp_custom
      out.write(0, 1);  // epf_weight_custom
      out.write(0, 1);  // epf_sigma_custom
    }
    out.write_u64(0);  // restoration filter extensions
    out.write_u64(0);  // frame header extensions
  }
  std::vector<std::vector<uint8_t>> sections;
  if (f.num_groups == 1) {  // single TOC entry: sections concatenated bitwise (frame_info.rs:414-450)
    BitWriter all;
    append_bits(all, lf_global);
    append_bits(all, lf_groups[0]);
    append_bits(all, hf_global);
    append_bits(all, hf_groups[0]);
    sections.push_back(all.finish());
  } else {
    sections.push_back(lf_global.finish());
    for (auto& b : lf_groups) sections.push_back(b.finish());
    sections.push_back(hf_global.finish());
    for (auto& b : hf_groups) sections.push_back(b.finish());
  }
  // TOC (toc.rs:20-32)
  out.write(0, 1);  // not permuted
  out.zero_pad_to_byte();
  for (auto& s : sections) write_toc_entry(out, uint32_t(s.size()));
  out.zero_pad_to_byte();
  std::vector<uint8_t> bytes = out.finish();
  for (auto& s : sections) bytes.insert(bytes.end(), s.begin(), s.end());
  return bytes;
}

// ---------------------------------------------------------------------------
// Token-level VarDCT writer (jxs_encode_vardct_tokens): every symbol of the AC coefficient streams is given by the
// caller, together with the BlockContextMap, the LF integers, the varblocks, the coefficient orders and the entropy
// codes. Nothing is predicted or checked, so frames a decoder must refuse can be written too.
// ---------------------------------------------------------------------------
struct TokenPassSpec {
  uint32_t selector = 2, used_orders = 0;
  struct Perm {
    uint32_t ord, c;
    std::vector<uint32_t> perm;
  };
  std::vector<Perm> perms;
  std::vector<uint8_t> context_map;
  uint32_t num_clusters = 1;
  std::vector<HybridCfg> cfgs;
  uint32_t log_alpha = 5;
  bool prefix = false, lz77 = false;
  uint32_t lz_min_symbol = 224, lz_min_length = 3;
};

// coeff_order.rs / permutation.rs:27-90 inverted: the Lehmer code of perm[skip..] over the values skip..size-1, as
// tokens of the 8 permutation contexts (get_context = min(7, ceil_log2(x + 1))); trailing zero codes are not written.
static void permutation_tokens(const std::vector<uint32_t>& perm, uint32_t skip, std::vector<Token>& out) {
  const uint32_t size = uint32_t(perm.size());
  const uint32_t n = size - skip;
  std::vector<uint32_t> fen(n + 1, 0);  // Fenwick tree over the values still unused
  auto add = [&](uint32_t i, int d) {
    for (i++; i <= n; i += i & (0u - i)) fen[i] += uint32_t(d);
  };
  auto below = [&](uint32_t i) {  // unused values < i
    uint32_t s = 0;
    for (; i; i -= i & (0u - i)) s += fen[i];
    return s;
  };
  for (uint32_t i = 0; i < n; i++) add(i, 1);
  std::vector<uint32_t> lehmer(n);
  for (uint32_t i = 0; i < n; i++) {
    const uint32_t v = perm[skip + i];
    if (v < skip || v >= size) throw std::runtime_error("permutation entry outside its range");
    lehmer[i] = below(v - skip);
    add(v - skip, -1);
  }
  uint32_t end = n;
  while (end && lehmer[end - 1] == 0) end--;
  auto ctx = [](uint32_t x) { return std::min<uint32_t>(7, ceil_log2(uint64_t(x) + 1)); };
  out.push_back(Token{ctx(size), end});
  uint32_t prev = 0;
  for (uint32_t i = 0; i < end; i++) {
    out.push_back(Token{ctx(prev), lehmer[i]});
    prev = lehmer[i];
  }
}

std::vector<uint8_t> encode_vardct_tokens(const uint32_t* w, size_t len) {
  size_t pos = 0;
  auto next = [&]() -> uint32_t {
    if (pos >= len) throw std::runtime_error("VarDCT token spec too short");
    return w[pos++];
  };
  const uint32_t W = next(), H = next(), num_passes = next();
  if (!W || !H || num_passes < 1 || num_passes > 11) throw std::runtime_error("bad size or pass count");
  std::vector<uint32_t> shifts(num_passes - 1);
  for (auto& s : shifts) s = next();
  const uint32_t xb = (W + 7) / 8, yb = (H + 7) / 8, xg = (W + 255) / 256, yg = (H + 255) / 256, num_groups = xg * yg;
  const uint32_t xlfg = (xb + 255) / 256, ylfg = (yb + 255) / 256, num_lf_groups = xlfg * ylfg;
  BitWriter lf_global;
  lf_global.write(1, 1);                // LfQuantFactors default
  lf_global.u2s_sel(0, 1024 - 1, 11);   // global_scale 1024
  lf_global.write(0, 2);                // quant_lf = 16
  if (next() == 0) {
    lf_global.write(1, 1);  // default BlockContextMap
  } else {                  // block_context_map.rs:61-126
    lf_global.write(0, 1);
    for (int c = 0; c < 3; c++) {
      const uint32_t n = next();
      lf_global.write(n, 4);
      for (uint32_t i = 0; i < n; i++) {
        const uint32_t u = pack_signed(int32_t(next()));
        if (u < 16) lf_global.u2s_sel(0, u, 4);
        else if (u < 272) lf_global.u2s_sel(1, u - 16, 8);
        else if (u < 65808) lf_global.u2s_sel(2, u - 272, 16);
        else lf_global.u2s_sel(3, u - 65808, 32);
      }
    }
    const uint32_t nq = next();
    lf_global.write(nq, 4);
    for (uint32_t i = 0; i < nq; i++) {
      const uint32_t v = next() - 1;  // stored minus one
      if (v < 4) lf_global.u2s_sel(0, v, 2);
      else if (v < 12) lf_global.u2s_sel(1, v - 4, 3);
      else if (v < 44) lf_global.u2s_sel(2, v - 12, 5);
      else lf_global.u2s_sel(3, v - 44, 8);
    }
    std::vector<uint8_t> map(next());
    uint32_t nc = 0;
    for (auto& m : map) {
      m = uint8_t(next());
      nc = std::max<uint32_t>(nc, m + 1u);
    }
    write_context_map(lf_global, map, nc);
  }
  lf_global.write(1, 1);  // default ColorCorrelationParams
  lf_global.write(0, 1);  // no global tree
  // quantised LF integers, X / Y / B per block in raster order
  std::vector<int32_t> lfq[3];
  for (auto& q : lfq) q.resize(size_t(xb) * yb);
  for (size_t i = 0; i < size_t(xb) * yb; i++)
    for (int c = 0; c < 3; c++) lfq[c][i] = int32_t(next());
  // varblocks
  std::vector<uint8_t> tmap(size_t(xb) * yb, 255);
  std::vector<int32_t> rq(size_t(xb) * yb, 0);
  const uint32_t nvb = next();
  for (uint32_t i = 0; i < nvb; i++) {
    const uint32_t bx = next(), by = next(), t = next(), q = next();
    if (t >= 27) throw std::runtime_error("transform type above 26");
    const uint32_t cx = kCoveredBlocksX[t], cy = kCoveredBlocksY[t];
    if (bx + cx > xb || by + cy > yb) throw std::runtime_error("varblock outside the frame");
    for (uint32_t y = 0; y < cy; y++)
      for (uint32_t x = 0; x < cx; x++) {
        uint8_t& m = tmap[size_t(by + y) * xb + bx + x];
        if (m != 255) throw std::runtime_error("overlapping varblocks");
        m = uint8_t(t) | ((x | y) ? 0 : 128);
      }
    rq[size_t(by) * xb + bx] = int32_t(q);
  }
  for (uint8_t m : tmap)
    if (m == 255) throw std::runtime_error("block not covered by a varblock");
  std::vector<BitWriter> lf_groups(num_lf_groups);
  for (uint32_t g = 0; g < num_lf_groups; g++) {
    BitWriter& bw = lf_groups[g];
    const uint32_t x0 = (g % xlfg) * 256, y0 = (g / xlfg) * 256;
    const uint32_t gw = std::min(256u, xb - x0), gh = std::min(256u, yb - y0);
    bw.write(0, 2);  // extra_precision
    std::vector<Chan> ch(3);
    const int order[3] = {1, 0, 2};  // stored Y, X, B
    for (int i = 0; i < 3; i++) {
      ch[i].w = gw;
      ch[i].h = gh;
      for (uint32_t y = 0; y < gh; y++)
        for (uint32_t x = 0; x < gw; x++) ch[i].d.push_back(lfq[order[i]][size_t(y0 + y) * xb + x0 + x]);
    }
    write_modular(bw, ch, 5);
    std::vector<int32_t> types, quants;
    for (uint32_t y = 0; y < gh; y++)
      for (uint32_t x = 0; x < gw; x++) {
        const size_t o = size_t(y0 + y) * xb + x0 + x;
        if (tmap[o] & 128) {
          types.push_back(tmap[o] & 127);
          quants.push_back(rq[o] - 1);
        }
      }
    const uint32_t count = uint32_t(types.size());
    bw.write(count - 1, ceil_log2(uint64_t(gw) * gh));
    const uint32_t cw = (gw + 7) / 8, chh = (gh + 7) / 8;
    std::vector<Chan> mc(4);
    mc[0].w = mc[1].w = cw;
    mc[0].h = mc[1].h = chh;
    mc[0].d.assign(size_t(cw) * chh, 0);
    mc[1].d.assign(size_t(cw) * chh, 0);
    mc[2].w = count;
    mc[2].h = 2;
    mc[2].d = types;
    mc[2].d.insert(mc[2].d.end(), quants.begin(), quants.end());
    mc[3].w = gw;
    mc[3].h = gh;
    mc[3].d.assign(size_t(gw) * gh, 0);
    write_modular(bw, mc, 1);
  }
  // HfGlobal (frame/decode.rs:506-566)
  BitWriter hf_global;
  hf_global.write(1, 1);  // DequantMatrices all_default
  const uint32_t num_histograms = next();
  hf_global.write(num_histograms - 1, ceil_log2(num_groups));
  std::vector<AnsCode> codes(num_passes);
  std::vector<BitWriter> order_bits(num_passes);  // per pass: used_orders and the permutations (before its AC code)
  for (uint32_t p = 0; p < num_passes; p++) {
    TokenPassSpec ps;
    ps.selector = next();
    ps.used_orders = next();
    order_bits[p].write(ps.selector, 2);
    if (ps.selector == 3) order_bits[p].write(ps.used_orders, 13);
    const uint32_t used = ps.selector == 0 ? 0x5f : ps.selector == 1 ? 0x13 : ps.selector == 2 ? 0 : ps.used_orders;
    const uint32_t nperm = next();
    for (uint32_t i = 0; i < nperm; i++) {
      TokenPassSpec::Perm pm;
      pm.ord = next();
      pm.c = next();
      pm.perm.resize(next());
      for (auto& v : pm.perm) v = next();
      ps.perms.push_back(std::move(pm));
    }
    if (used) {  // coeff_order.rs:122-148: one stream over 8 contexts for every (used order, channel) in turn
      static const int kOrderTransform[13] = {0, 1, 4, 5, 7, 9, 11, 18, 20, 21, 23, 24, 26};  // TRANSFORM_TYPE_LUT
      std::vector<Token> toks;
      for (uint32_t ord = 0; ord < 13; ord++) {
        if (!(used & (1u << ord))) continue;
        const uint32_t nb = uint32_t(kCoveredBlocksX[kOrderTransform[ord]]) * kCoveredBlocksY[kOrderTransform[ord]];
        for (uint32_t c = 0; c < 3; c++) {
          std::vector<uint32_t> perm(nb * 64);
          for (uint32_t i = 0; i < perm.size(); i++) perm[i] = i;
          for (auto& pm : ps.perms)
            if (pm.ord == ord && pm.c == c) {
              if (pm.perm.size() != perm.size()) throw std::runtime_error("permutation of the wrong size");
              perm = pm.perm;
            }
          permutation_tokens(perm, nb, toks);
        }
      }
      std::vector<uint8_t> one(8, 0);
      AnsCode oc = build_code(8, one, 1, {&toks}, 6);
      write_code(order_bits[p], oc);
      write_tokens(order_bits[p], oc, toks);
    }
    ps.context_map.resize(next());
    for (auto& m : ps.context_map) m = uint8_t(next());
    ps.num_clusters = next();
    for (uint32_t i = 0; i < ps.num_clusters; i++) {
      HybridCfg h;
      h.split_exponent = next();
      h.msb = next();
      h.lsb = next();
      ps.cfgs.push_back(h);
    }
    ps.log_alpha = next();
    ps.prefix = next() != 0;
    ps.lz77 = next() != 0;
    ps.lz_min_symbol = next();
    ps.lz_min_length = next();
    // the sections' tokens of this pass come later in the spec; the code is built once they are read
    codes[p].num_contexts = uint32_t(ps.context_map.size());
    codes[p].context_map = ps.context_map;
    codes[p].num_clusters = ps.num_clusters;
    codes[p].cluster_cfgs = ps.cfgs;
    codes[p].log_alpha_size = ps.log_alpha;
    codes[p].use_prefix = ps.prefix;
    codes[p].lz.enabled = ps.lz77;
    codes[p].lz.min_symbol = ps.lz_min_symbol;
    codes[p].lz.min_length = ps.lz_min_length;
  }
  std::vector<uint32_t> hist(size_t(num_passes) * num_groups);
  std::vector<std::vector<Token>> toks(size_t(num_passes) * num_groups);
  for (size_t s = 0; s < toks.size(); s++) {
    hist[s] = next();
    toks[s].resize(next());
    for (auto& t : toks[s]) {
      t.ctx = next();
      t.value = next();
    }
  }
  if (pos != len) throw std::runtime_error("VarDCT token spec too long");
  std::vector<std::vector<Sym>> syms(toks.size());
  for (uint32_t p = 0; p < num_passes; p++) {
    const AnsCode spec = codes[p];
    std::vector<const std::vector<Token>*> tp;
    for (uint32_t g = 0; g < num_groups; g++) tp.push_back(&toks[size_t(p) * num_groups + g]);
    if (spec.lz.enabled) {  // one hybrid-uint configuration for the literals; the distance context gets its own cluster
      for (auto& h : spec.cluster_cfgs)
        if (h.split_exponent != spec.cluster_cfgs[0].split_exponent || h.msb != spec.cluster_cfgs[0].msb ||
            h.lsb != spec.cluster_cfgs[0].lsb)
          throw std::runtime_error("an LZ77 pass takes one hybrid-uint configuration");
      const HybridCfg len_cfg{0, 0, 0};
      std::vector<const std::vector<Sym>*> sp;
      for (uint32_t g = 0; g < num_groups; g++) {
        syms[size_t(p) * num_groups + g] = lz77_symbols(*tp[g], spec.cluster_cfgs[0], spec.lz, len_cfg, spec.num_contexts);
        sp.push_back(&syms[size_t(p) * num_groups + g]);
      }
      std::vector<uint8_t> map = spec.context_map;
      map.push_back(uint8_t(spec.num_clusters));
      codes[p] = build_code_lz77(spec.num_contexts + 1, map, spec.num_clusters + 1, sp, spec.lz, spec.use_prefix);
      codes[p].cfg = spec.cluster_cfgs[0];
      codes[p].lz_len_cfg = len_cfg;
    } else {
      codes[p] = build_code_cfgs(spec.num_contexts, spec.context_map, spec.num_clusters, tp, spec.log_alpha_size,
                                 spec.use_prefix, spec.cluster_cfgs);
    }
  }
  for (uint32_t p = 0; p < num_passes; p++) {
    append_bits(hf_global, order_bits[p]);
    write_code(hf_global, codes[p]);
  }
  std::vector<BitWriter> hf_groups(toks.size());
  for (size_t s = 0; s < toks.size(); s++) {
    hf_groups[s].write(hist[s], ceil_log2(num_histograms));  // group.rs:333-341
    const AnsCode& code = codes[s / num_groups];
    if (code.lz.enabled) write_symbols(hf_groups[s], code, syms[s]);
    else write_tokens(hf_groups[s], code, toks[s]);
  }

  BitWriter out;
  out.write(0xff, 8);
  out.write(0x0a, 8);
  auto write_dim = [&](uint32_t v) {  // size.rs:31-47
    const uint32_t m = v - 1;
    if (m < (1u << 9)) out.u2s_sel(0, m, 9);
    else if (m < (1u << 13)) out.u2s_sel(1, m, 13);
    else if (m < (1u << 18)) out.u2s_sel(2, m, 18);
    else out.u2s_sel(3, m, 30);
  };
  out.write(0, 1);  // small = false
  write_dim(H);
  out.write(0, 3);  // explicit xsize
  write_dim(W);
  out.write(1, 1);  // ImageMetadata all_default
  out.write(1, 1);  // CustomTransformData all_default
  out.zero_pad_to_byte();
  // FrameHeader (frame_header.rs:267-444) with the default filters and qm scales
  out.write(0, 1);  // all_default
  out.write(0, 2);  // RegularFrame
  out.write(0, 1);  // VarDCT
  out.write_u64(0);  // flags
  out.write(0, 2);  // upsampling = 1
  out.write(3, 3);  // x_qm_scale
  out.write(2, 3);  // b_qm_scale
  if (num_passes == 1) out.u2s_sel(0);  // Passes (frame_header.rs:46-75)
  else if (num_passes <= 3) out.u2s_sel(num_passes - 1);
  else out.u2s_sel(3, num_passes - 4, 3);
  if (num_passes != 1) {
    out.u2s_sel(0);  // num_ds = 0
    for (uint32_t s : shifts) out.write(s, 2);
  }
  out.write(0, 1);  // have_crop
  out.write(0, 2);  // blending mode Replace
  out.write(1, 1);  // is_last
  out.write(0, 2);  // name length 0
  out.write(0, 1);  // RestorationFilter all_default = 0
  out.write(1, 1);  // gab
  out.write(0, 1);  // gab_custom
  out.write(2, 2);  // epf_iters
  out.write(0, 1);  // epf_sharp_custom
  out.write(0, 1);  // epf_weight_custom
  out.write(0, 1);  // epf_sigma_custom
  out.write_u64(0);  // restoration filter extensions
  out.write_u64(0);  // frame header extensions
  std::vector<std::vector<uint8_t>> sections;
  if (num_groups == 1 && num_passes == 1) {  // single TOC entry: sections concatenated bitwise
    BitWriter all;
    append_bits(all, lf_global);
    append_bits(all, lf_groups[0]);
    append_bits(all, hf_global);
    append_bits(all, hf_groups[0]);
    sections.push_back(all.finish());
  } else {
    sections.push_back(lf_global.finish());
    for (auto& b : lf_groups) sections.push_back(b.finish());
    sections.push_back(hf_global.finish());
    for (auto& b : hf_groups) sections.push_back(b.finish());
  }
  out.write(0, 1);  // TOC not permuted
  out.zero_pad_to_byte();
  for (auto& s : sections) write_toc_entry(out, uint32_t(s.size()));
  out.zero_pad_to_byte();
  std::vector<uint8_t> bytes = out.finish();
  for (auto& s : sections) bytes.insert(bytes.end(), s.begin(), s.end());
  return bytes;
}

// 8-bit RGB rendering of the same procedural image (source of the synthetic Modular frames).
void make_image_u8(uint32_t width, uint32_t height, uint64_t seed, std::vector<uint8_t>& rgb) {
  Params p{width, height, seed, 1.0f, 0, 0, 0, 0, 0};
  std::vector<float> img[3];
  make_image(p, img);
  rgb.resize(size_t(width) * height * 3);
  for (size_t i = 0; i < size_t(width) * height; i++)
    for (int c = 0; c < 3; c++) rgb[i * 3 + c] = uint8_t(std::lround(std::min(1.0f, std::max(0.0f, img[c][i])) * 255.0f));
}

}  // namespace jxs

extern "C" {

static thread_local std::string g_err;
const char* jxs_last_error() { return g_err.c_str(); }
// Worker threads used inside each following encode (process-wide; 1 = serial). The output does not depend on it.
void jxs_set_threads(int n) { jxs::g_threads.store(n < 1 ? 1 : n); }

// Encodes one synthetic frame. Returns the number of bytes written (or the
// needed size when `cap` is too small), negative on error.
int64_t jxs_encode_synthetic(uint32_t width, uint32_t height, uint64_t seed, float distance, uint32_t epf_iters,
                             uint32_t gab, uint32_t profile, uint8_t* out, size_t cap) {
  try {
    // profile: bits 0..7 transform mix, bit 8: libjxl-like LF tree (weighted predictor), bits 9..10: AC entropy coder
    // bits 12..15: orientation - 1, bits 16..19: colour encoding variant
    jxs::Params p{width, height, seed, distance, epf_iters, gab, profile & 0xff, (profile >> 8) & 1, (profile >> 9) & 3,
                  ((profile >> 12) & 7) + 1, (profile >> 16) & 15};
    std::vector<uint8_t> b = jxs::encode(p);
    if (b.size() <= cap && out) memcpy(out, b.data(), b.size());
    return int64_t(b.size());
  } catch (std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

// jxs_encode_synthetic with the frame header's x_qm_scale / b_qm_scale and custom dequantisation matrices.
// dequant: for each of the 17 table indices in turn, the mode (0..7), then
//   modes 1..7: the number n of fields that follow the mode in the bitstream, then n (value, bits) pairs;
//   mode 7:     additionally 3 * 64 * REQUIRED_SIZE_X * REQUIRED_SIZE_Y raw entries (int32, each channel in raster
//               order, 8 * REQUIRED_SIZE_X wide), written as a Modular sub-bitstream after the fields.
// dequant_len 0: all library tables (the same bitstream as jxs_encode_synthetic).
int64_t jxs_encode_synthetic_ex(uint32_t width, uint32_t height, uint64_t seed, float distance, uint32_t epf_iters,
                                uint32_t gab, uint32_t profile, uint32_t x_qm_scale, uint32_t b_qm_scale,
                                const uint32_t* dequant, size_t dequant_len, uint8_t* out, size_t cap) {
  try {
    jxs::Params p{width, height, seed, distance, epf_iters, gab, profile & 0xff, (profile >> 8) & 1, (profile >> 9) & 3,
                  ((profile >> 12) & 7) + 1, (profile >> 16) & 15};
    if (x_qm_scale > 7 || b_qm_scale > 7) throw std::runtime_error("x_qm_scale / b_qm_scale must be 0..7");
    p.x_qm_scale = x_qm_scale;
    p.b_qm_scale = b_qm_scale;
    size_t pos = 0;
    auto next = [&]() -> uint32_t {
      if (pos >= dequant_len) throw std::runtime_error("dequant array too short");
      return dequant[pos++];
    };
    if (dequant_len) {
      p.dequant.resize(jxg::kNumQuantTables);
      for (int i = 0; i < jxg::kNumQuantTables; i++) {
        jxs::Params::DequantSpec& s = p.dequant[i];
        s.mode = next();
        if (s.mode > 7) throw std::runtime_error("dequant mode above 7");
        if (s.mode == 0) continue;
        const uint32_t n = next();
        for (uint32_t k = 0; k < n; k++) {
          const uint32_t v = next(), bits = next();
          if (bits > 32) throw std::runtime_error("dequant field wider than 32 bits");
          s.fields.emplace_back(v, bits);
        }
        if (s.mode == 7) {
          if (s.fields.size() != 1 || s.fields[0].second != 16) throw std::runtime_error("RAW takes one 16-bit field");
          s.raw.resize(size_t(3) * 64 * jxg::kQuantTableRows[i] * jxg::kQuantTableCols[i]);
          for (auto& v : s.raw) v = int32_t(next());
        }
      }
      if (pos != dequant_len) throw std::runtime_error("dequant array too long");
    }
    std::vector<uint8_t> b = jxs::encode(p);
    if (b.size() <= cap && out) memcpy(out, b.data(), b.size());
    return int64_t(b.size());
  } catch (std::exception& e) {
    g_err = e.what();
    return -1;
  }
}

// One VarDCT frame written exactly as described by `spec` (synth/__init__.py encode_vardct_tokens gives the layout).
// Returns the number of bytes written (or the needed size when `cap` is too small), negative on error.
int64_t jxs_encode_vardct_tokens(const uint32_t* spec, size_t len, uint8_t* out, size_t cap) {
  try {
    std::vector<uint8_t> b = jxs::encode_vardct_tokens(spec, len);
    if (b.size() <= cap && out) memcpy(out, b.data(), b.size());
    return int64_t(b.size());
  } catch (std::exception& e) {
    g_err = e.what();
    return -1;
  }
}
}
