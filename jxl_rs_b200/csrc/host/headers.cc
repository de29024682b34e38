// See headers.h.
#include "headers.h"

#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

#include "entropy.h"

namespace jxg {

namespace {

// encodings.rs U32Coder: one distribution = (nbits, offset); nbits==0 && value only.
struct U32D {
  uint32_t bits, off;
};
inline uint32_t u2s(BitReader& br, U32D a, U32D b, U32D c, U32D d) {
  const U32D ds[4] = {a, b, c, d};
  const U32D& s = ds[br.read(2)];
  return uint32_t(br.read(s.bits)) + s.off;
}
constexpr U32D V(uint32_t v) { return U32D{0, v}; }
constexpr U32D B(uint32_t n, uint32_t off = 0) { return U32D{n, off}; }

// jxl_macros/src/lib.rs:671-679: default enum coder
inline uint32_t read_enum(BitReader& br) { return u2s(br, V(0), V(1), B(4, 2), B(6, 18)); }

std::string read_string(BitReader& br) {  // encodings.rs:141-171
  uint32_t len = u2s(br, V(0), B(4), B(5, 16), B(10, 48));
  std::string s;
  for (uint32_t i = 0; i < len; i++) s.push_back(char(br.read(8)));
  return s;
}

BitDepth read_bit_depth(BitReader& br) {  // bit_depth.rs:13-27
  BitDepth d;
  d.floating_point = br.read_bool();
  if (d.floating_point) {
    d.bits_per_sample = u2s(br, V(32), V(16), V(24), B(6, 1));
    d.exponent_bits = uint32_t(br.read(4)) + 1;
  } else {
    d.bits_per_sample = u2s(br, V(8), V(10), V(12), B(6, 1));
  }
  return d;
}

void read_size(BitReader& br, uint32_t& xs, uint32_t& ys) {  // size.rs:31-47
  bool small = br.read_bool();
  if (small) ys = (uint32_t(br.read(5)) + 1) * 8;
  else ys = 1 + u2s(br, B(9), B(13), B(18), B(30));
  uint32_t ratio = uint32_t(br.read(3));
  if (ratio == 0) {
    if (small) xs = (uint32_t(br.read(5)) + 1) * 8;
    else xs = 1 + u2s(br, B(9), B(13), B(18), B(30));
  } else {
    static const uint32_t num[8] = {0, 1, 12, 4, 3, 16, 5, 2}, den[8] = {1, 1, 10, 3, 2, 9, 4, 1};
    xs = uint32_t(uint64_t(ys) * num[ratio] / den[ratio]);
  }
}

void read_preview(BitReader& br) {  // size.rs:49-66
  bool div8 = br.read_bool();
  if (div8) u2s(br, V(16), V(32), B(5, 1), B(9, 33));
  else u2s(br, B(6), B(8, 64), B(10, 320), B(12, 1344));
  uint32_t ratio = uint32_t(br.read(3));
  if (ratio == 0) {
    if (div8) u2s(br, V(16), V(32), B(5, 1), B(9, 33));
    else u2s(br, B(6), B(8, 64), B(10, 320), B(12, 1344));
  }
}

void read_custom_xy(BitReader& br, int32_t* xy) {  // color_encoding.rs:91-100: u2S then unpack_signed (encodings.rs:99-108)
  for (int i = 0; i < 2; i++) {
    const uint32_t u = u2s(br, B(19), B(19, 524288), B(20, 1048576), B(21, 2097152));
    xy[i] = int32_t((u >> 1) ^ (((~u) & 1u) - 1u));
  }
}

ColorEncoding read_color_encoding(BitReader& br) {  // color_encoding.rs:166-196
  ColorEncoding c;
  c.all_default = br.read_bool();
  if (c.all_default) return c;
  c.want_icc = br.read_bool();
  c.color_space = ColorSpace(read_enum(br));
  bool not_xyb = c.color_space != ColorSpace::XYB;
  if (!c.want_icc && not_xyb) {
    c.white_point = read_enum(br);
    if (c.white_point == 2) read_custom_xy(br, c.white_xy);
  }
  if (!c.want_icc && not_xyb && c.color_space != ColorSpace::Gray) {
    c.primaries = read_enum(br);
    if (c.primaries == 2)
      for (int i = 0; i < 3; i++) read_custom_xy(br, c.primaries_xy[i]);
  }
  if (!c.want_icc) {
    if (not_xyb) c.have_gamma = br.read_bool();
    if (c.have_gamma) c.gamma = uint32_t(br.read(24));
    if (!c.have_gamma && not_xyb) c.tf = TransferFunction(read_enum(br));
    c.rendering_intent = read_enum(br);
  }
  return c;
}

ExtraChannelInfo read_extra_channel(BitReader& br) {  // extra_channels.rs:36-56
  ExtraChannelInfo e;
  if (br.read_bool()) return e;
  e.type = read_enum(br);
  e.bit_depth = read_bit_depth(br);
  e.dim_shift = u2s(br, V(0), V(3), V(4), B(3, 1));
  read_string(br);
  if (e.type == 0) e.alpha_associated = br.read_bool();
  if (e.type == 2)
    for (int i = 0; i < 4; i++) read_f16(br);
  if (e.type == 5) u2s(br, V(1), B(2), B(4, 3), B(8, 19));
  if (e.dim_shift > 3) fail("dim_shift too large");
  return e;
}

void skip_icc(BitReader& br) {  // icc/mod.rs:100-190 (decoded and discarded)
  uint64_t len = read_u64(br);
  if (len > (1ull << 24)) fail("ICC too large");
  EntropyCode code = EntropyCode::decode(41, br, true);
  SymbolReader reader(code, br, 0);
  uint8_t b1 = 0, b2 = 0;
  auto is_alpha = [](uint8_t b) { return (b >= 'a' && b <= 'z') || (b >= 'A' && b <= 'Z'); };
  auto is_num = [](uint8_t b) { return (b >= '0' && b <= '9') || b == '.' || b == ','; };
  for (uint64_t i = 0; i < len; i++) {
    uint32_t ctx = 0;
    if (i > 128) {
      uint32_t p1 = is_alpha(b1) ? 0 : is_num(b1) ? 1 : b1 <= 1 ? 2 + b1 : b1 <= 15 ? 4 : (b1 >= 241 && b1 <= 254) ? 5 : b1 == 255 ? 6 : 7;
      uint32_t p2 = is_alpha(b2) ? 0 : is_num(b2) ? 1 : b2 <= 15 ? 2 : b2 >= 241 ? 3 : 4;
      ctx = 1 + p1 + 8 * p2;
    }
    uint32_t sym = reader.read_unsigned(br, ctx);
    if (sym >= 256) fail("invalid ICC symbol");
    b2 = b1;
    b1 = uint8_t(sym);
  }
  reader.check_final_state(br);
}

}  // namespace

float f16_bits_to_float(uint16_t h) {
  uint32_t sign = h >> 15, exp = (h >> 10) & 31, man = h & 1023;
  float v;
  if (exp == 0) v = std::ldexp(float(man), -24);
  else if (exp == 31) v = man ? NAN : INFINITY;
  else v = std::ldexp(float(man | 1024), int(exp) - 25);
  return sign ? -v : v;
}

float read_f16(BitReader& br) {
  float v = f16_bits_to_float(uint16_t(br.read(16)));
  if (!std::isfinite(v)) fail("NaN or Inf in header float");
  return v;
}

void read_lf_quant_factors(BitReader& br, float out[3]) {
  static const float kDefault[3] = {1.0f / 4096.0f, 1.0f / 512.0f, 1.0f / 256.0f};
  if (br.read_bool()) {
    for (int c = 0; c < 3; c++) out[c] = kDefault[c];
    return;
  }
  for (int c = 0; c < 3; c++) {
    out[c] = read_f16(br) / 128.0f;
    if (out[c] < 1e-8f) fail("LF quant factor too small");
  }
}

uint64_t read_u64(BitReader& br) {  // encodings.rs:111-139
  switch (br.read(2)) {
    case 0: return 0;
    case 1: return 1 + br.read(4);
    case 2: return 17 + br.read(8);
    default: {
      uint64_t result = br.read(12);
      unsigned shift = 12;
      while (br.read(1) == 1) {
        if (shift >= 60) return result | (br.read(4) << shift);
        result |= br.read(8) << shift;
        shift += 8;
      }
      return result;
    }
  }
}

void read_extensions(BitReader& br) {  // encodings.rs:377-407
  uint64_t selector = read_u64(br);
  uint64_t total = 0;
  for (int i = 0; i < 64; i++)
    if (selector & (1ull << i)) total += read_u64(br);
  if (total > br.size_bits()) fail("extension size overflow", kErrOutOfBounds);
  br.skip_bits(size_t(total));
}

std::vector<uint8_t> extract_codestream(const uint8_t* data, size_t size) {
  std::vector<uint8_t> out;
  extract_codestream(data, size, out);
  return out;
}

void extract_codestream(const uint8_t* data, size_t size, std::vector<uint8_t>& out) {
  out.clear();
  if (size >= 2 && data[0] == 0xff && data[1] == 0x0a) {
    out.assign(data, data + size);
    return;
  }
  static const uint8_t kSig[12] = {0, 0, 0, 0xc, 'J', 'X', 'L', ' ', 0xd, 0xa, 0x87, 0xa};
  if (size < 12 || memcmp(data, kSig, 12) != 0) fail("not a JPEG XL file");
  size_t pos = 0;
  while (pos + 8 <= size) {
    uint64_t box_size = (uint64_t(data[pos]) << 24) | (uint64_t(data[pos + 1]) << 16) | (uint64_t(data[pos + 2]) << 8) | data[pos + 3];
    const uint8_t* ty = data + pos + 4;
    size_t header = 8;
    if (box_size == 1) {
      if (pos + 16 > size) fail("truncated box header");
      box_size = 0;
      for (int i = 0; i < 8; i++) box_size = (box_size << 8) | data[pos + 8 + i];
      header = 16;
    }
    size_t end = box_size == 0 ? size : pos + size_t(box_size);
    if (end > size || end < pos + header) fail("bad box size");
    if (!memcmp(ty, "jxlc", 4)) out.insert(out.end(), data + pos + header, data + end);
    else if (!memcmp(ty, "jxlp", 4)) {
      if (end < pos + header + 4) fail("bad jxlp box");
      // in-order jxlp only (box_parser.rs handles out-of-order; test files exercising it are rejected upstream of here)
      out.insert(out.end(), data + pos + header + 4, data + end);
    }
    pos = end;
  }
  if (out.empty()) fail("no codestream box");
}

FileHeader read_file_header(BitReader& br) {
  FileHeader h;
  if (br.read(8) != 0xff || br.read(8) != 0x0a) fail("invalid signature");
  read_size(br, h.xsize, h.ysize);
  // ImageMetadata (image_metadata.rs:197-236)
  bool all_default = br.read_bool();
  bool extra_fields = false;
  if (!all_default) {
    extra_fields = br.read_bool();
    if (extra_fields) {
      h.orientation = uint32_t(br.read(3)) + 1;
      if (br.read_bool()) {  // intrinsic size
        uint32_t a, b;
        read_size(br, a, b);
      }
      h.have_preview = br.read_bool();
      if (h.have_preview) read_preview(br);
      h.have_animation = br.read_bool();
      if (h.have_animation) {
        u2s(br, V(100), V(1000), B(10, 1), B(30, 1));
        u2s(br, V(1), V(1001), B(8, 1), B(10, 1));
        u2s(br, V(0), B(3), B(16), B(32));
        h.have_timecodes = br.read_bool();
      }
    }
    h.bit_depth = read_bit_depth(br);
    h.modular_16bit_sufficient = br.read_bool();
    uint32_t num_ec = u2s(br, V(0), V(1), B(4, 2), B(12, 1));
    for (uint32_t i = 0; i < num_ec; i++) h.extra_channels.push_back(read_extra_channel(br));
    h.xyb_encoded = br.read_bool();
    h.color_encoding = read_color_encoding(br);
    if (extra_fields) {  // ToneMapping
      if (!br.read_bool()) {
        h.intensity_target = read_f16(br);
        read_f16(br);
        br.read_bool();
        read_f16(br);
        if (h.intensity_target <= 0) fail("invalid intensity target");
      }
    }
    read_extensions(br);
  }
  // CustomTransformData (transform_data.rs:322-345)
  if (!br.read_bool()) {
    if (h.xyb_encoded) {
      if (!br.read_bool()) {
        for (float& v : h.opsin.inverse_matrix) v = read_f16(br);
        for (float& v : h.opsin.opsin_biases) v = read_f16(br);
        for (float& v : h.opsin.quant_biases) v = read_f16(br);
      }
    }
    h.custom_upsampling_mask = uint32_t(br.read(3));
    if (h.custom_upsampling_mask & 1)
      for (int i = 0; i < 15; i++) read_f16(br);
    if (h.custom_upsampling_mask & 2)
      for (int i = 0; i < 55; i++) read_f16(br);
    if (h.custom_upsampling_mask & 4)
      for (float& v : h.weights8) v = read_f16(br);
  }
  if (h.color_encoding.want_icc) skip_icc(br);
  br.check();
  return h;
}

static BlendingInfo read_blending(BitReader& br, uint32_t num_ec, bool full_frame) {  // frame_header.rs:111-139
  BlendingInfo b;
  b.mode = u2s(br, V(0), V(1), V(2), B(2, 3));
  if (b.mode > 4) fail("invalid blend mode");
  bool uses_alpha = num_ec > 0 && (b.mode == 2 || b.mode == 3);
  if (uses_alpha) b.alpha_channel = u2s(br, V(0), V(1), V(2), B(3, 3));
  if (uses_alpha || b.mode == 4) b.clamp = br.read_bool();
  if (!(full_frame && b.mode == 0)) b.source = u2s(br, V(0), V(1), V(2), V(3));
  return b;
}

std::array<float, 210> FileHeader::default_weights8() {
  return {
#include "upsample8_weights.inc"
  };
}

FrameHeader read_frame_header(BitReader& br, const FileHeader& fh) {
  br.jump_to_byte_boundary();  // #[aligned], frame_header.rs:264
  FrameHeader f;
  uint32_t num_ec = uint32_t(fh.extra_channels.size());
  f.num_extra_channels = num_ec;
  f.ec_upsampling.assign(num_ec, 1);
  f.ec_blending.assign(num_ec, BlendingInfo{});
  bool all_default = br.read_bool();
  if (!all_default) {
    f.frame_type = uint32_t(br.read(2));
    f.encoding = uint32_t(br.read(1));
    f.flags = read_u64(br);
    if (!fh.xyb_encoded) f.do_ycbcr = br.read_bool();
    bool use_lf = f.has_lf_frame();
    if (f.do_ycbcr && !use_lf)
      for (auto& u : f.jpeg_upsampling) u = uint32_t(br.read(2));
    if (!use_lf) {
      f.upsampling = u2s(br, V(1), V(2), V(4), V(8));
      for (auto& u : f.ec_upsampling) u = u2s(br, V(1), V(2), V(4), V(8));
    }
    if (f.encoding == 1) f.group_size_shift = uint32_t(br.read(2));
    if (f.encoding == 0 && fh.xyb_encoded) {
      f.x_qm_scale = uint32_t(br.read(3));
      f.b_qm_scale = uint32_t(br.read(3));
    }
    if (f.frame_type != 2) {  // Passes (frame_header.rs:46-75)
      Passes& p = f.passes;
      p.num_passes = u2s(br, V(1), V(2), V(3), B(3, 4));
      if (p.num_passes != 1) {
        p.num_ds = u2s(br, V(0), V(1), V(2), B(1, 3));
        p.shift.resize(p.num_passes - 1);
        for (auto& s : p.shift) s = uint32_t(br.read(2));
        p.downsample.resize(p.num_ds);
        for (auto& s : p.downsample) s = u2s(br, V(1), V(2), V(4), V(8));
        p.last_pass.resize(p.num_ds);
        for (auto& s : p.last_pass) s = u2s(br, V(0), V(1), V(2), B(3));
      }
    }
    if (f.frame_type == 1) f.lf_level = u2s(br, V(1), V(2), V(3), V(4));
    if (f.frame_type != 1) f.have_crop = br.read_bool();
    if (f.have_crop) {
      if (f.frame_type != 2) {
        f.x0 = unpack_signed(u2s(br, B(8), B(11, 256), B(14, 2304), B(30, 18688)));
        f.y0 = unpack_signed(u2s(br, B(8), B(11, 256), B(14, 2304), B(30, 18688)));
      }
      f.frame_width = u2s(br, B(8), B(11, 256), B(14, 2304), B(30, 18688));
      f.frame_height = u2s(br, B(8), B(11, 256), B(14, 2304), B(30, 18688));
    }
    bool covers = f.x0 <= 0 && f.y0 <= 0 && int64_t(f.frame_width) + f.x0 >= int64_t(fh.xsize) &&
                  int64_t(f.frame_height) + f.y0 >= int64_t(fh.ysize);
    bool full_frame = !f.have_crop || covers;
    bool normal = f.frame_type == 0 || f.frame_type == 3;
    if (normal) {
      f.blending = read_blending(br, num_ec, full_frame);
      for (auto& b : f.ec_blending) b = read_blending(br, num_ec, full_frame);
      if (fh.have_animation) f.duration = u2s(br, V(0), V(1), B(8), B(32));
      if (fh.have_timecodes) br.read(32);
      f.is_last = br.read_bool();
    } else {
      f.is_last = false;
    }
    if (f.frame_type != 1 && !f.is_last) f.save_as_reference = uint32_t(br.read(2));
    bool can_be_referenced = !f.is_last && f.frame_type != 1 && (f.duration == 0 || f.save_as_reference != 0);
    bool sbct_def_false = can_be_referenced && f.blending.mode == 0 && full_frame && normal;
    f.save_before_ct = f.frame_type == 1;
    if (f.frame_type == 2 || sbct_def_false) f.save_before_ct = br.read_bool();
    f.name = read_string(br);
    // RestorationFilter (frame_header.rs:146-234)
    RestorationFilter& r = f.rf;
    if (!br.read_bool()) {
      r.gab = br.read_bool();
      if (r.gab && br.read_bool()) {
        for (int c = 0; c < 3; c++) {
          r.gab_w1[c] = read_f16(br);
          r.gab_w2[c] = read_f16(br);
        }
      }
      r.epf_iters = uint32_t(br.read(2));
      bool vardct = f.encoding == 0;
      if (r.epf_iters > 0 && vardct && br.read_bool())
        for (float& v : r.epf_sharp_lut) v = read_f16(br);
      if (r.epf_iters > 0 && br.read_bool()) {
        for (float& v : r.epf_channel_scale) v = read_f16(br);
        read_f16(br);  // epf_pass1_zeroflush
        read_f16(br);  // epf_pass2_zeroflush
      }
      if (r.epf_iters > 0 && br.read_bool()) {
        if (vardct) r.epf_quant_mul = read_f16(br);
        r.epf_pass0_sigma_scale = read_f16(br);
        r.epf_pass2_sigma_scale = read_f16(br);
        r.epf_border_sad_mul = read_f16(br);
      }
      if (r.epf_iters > 0 && !vardct) r.epf_sigma_for_modular = read_f16(br);
      read_extensions(br);
    }
    read_extensions(br);
  }
  f.width = f.frame_width ? f.frame_width : fh.xsize;
  f.height = f.frame_height ? f.frame_height : fh.ysize;
  // postprocess (frame_header.rs:667-677)
  if (f.upsampling > 1)
    for (uint32_t i = 0; i < num_ec; i++) f.ec_upsampling[i] <<= fh.extra_channels[i].dim_shift;
  if (f.encoding != 0 || !fh.xyb_encoded) f.x_qm_scale = 2;
  br.check();
  return f;
}

Toc read_toc(BitReader& br, uint32_t num_entries) {
  Toc toc;
  bool permuted = br.read_bool();
  std::vector<uint32_t> perm;
  if (permuted) {  // encodings.rs:173-194
    EntropyCode code = EntropyCode::decode(8, br, true);
    SymbolReader reader(code, br, 0);
    perm = decode_permutation(num_entries, 0, code, br, reader);
    reader.check_final_state(br);
  }
  br.jump_to_byte_boundary();
  toc.sizes.resize(num_entries);
  for (auto& s : toc.sizes) s = u2s(br, B(10), B(14, 1024), B(22, 17408), B(30, 4211712));
  br.jump_to_byte_boundary();
  br.check();
  // frame/decode.rs:263-285: logical section i is bitstream entry perm[i].
  std::vector<uint64_t> bs_off(num_entries);
  uint64_t off = 0;
  for (uint32_t i = 0; i < num_entries; i++) {
    bs_off[i] = off;
    off += toc.sizes[i];
  }
  toc.offsets.assign(num_entries, 0);
  toc.lengths.assign(num_entries, 0);
  for (uint32_t i = 0; i < num_entries; i++) {
    uint32_t src = permuted ? perm[i] : i;
    toc.offsets[i] = bs_off[src];
    toc.lengths[i] = toc.sizes[src];
  }
  return toc;
}

void check_single_still_frame(const FileHeader& fh, const FrameHeader& h) {
  // A few header bytes can announce 2^30 x 2^30 pixels; refuse before any plane is sized from them. JXG_MAX_PIXELS
  // (default 2^29, twice BASELINE config 4) is the knob for hosts with the memory for more.
  uint64_t max_pixels = uint64_t(1) << 29;
  if (const char* e = getenv("JXG_MAX_PIXELS")) max_pixels = std::max<uint64_t>(1, strtoull(e, nullptr, 10));
  if (uint64_t(h.xsize()) * h.ysize() > max_pixels || uint64_t(fh.xsize) * fh.ysize > max_pixels)
    fail("image larger than JXG_MAX_PIXELS", kErrUnsupported);
  if (fh.have_animation) fail("animations are outside the hot-path scope", kErrUnsupported);
  if (!h.is_last) fail("multi-frame (layered) files are outside the hot-path scope", kErrUnsupported);
  if (h.duration != 0 || h.save_as_reference != 0) fail("frames with a duration / reference slot are outside the hot-path scope", kErrUnsupported);
  if (fh.orientation < 1 || fh.orientation > 8) fail("bad orientation");
}

namespace {
// util/linalg.rs:29-110 and api/color.rs:124-275, in double precision like the reference.
struct M3 {
  double m[3][3];
};
M3 mul(const M3& a, const M3& b) {
  M3 r;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) r.m[i][j] = a.m[i][0] * b.m[0][j] + a.m[i][1] * b.m[1][j] + a.m[i][2] * b.m[2][j];
  return r;
}
void mulv(const M3& a, const double* v, double* out) {
  for (int i = 0; i < 3; i++) out[i] = a.m[i][0] * v[0] + a.m[i][1] * v[1] + a.m[i][2] * v[2];
}
M3 inverse(const M3& a) {
  const double (*m)[3] = a.m;
  const double det = m[0][0] * (m[1][1] * m[2][2] - m[2][1] * m[1][2]) - m[0][1] * (m[1][0] * m[2][2] - m[1][2] * m[2][0]) +
                     m[0][2] * (m[1][0] * m[2][1] - m[1][1] * m[2][0]);
  if (!(std::fabs(det) > 1e-10)) fail("singular colour matrix");
  const double id = 1.0 / det;
  M3 r;
  r.m[0][0] = (m[1][1] * m[2][2] - m[2][1] * m[1][2]) * id;
  r.m[0][1] = (m[0][2] * m[2][1] - m[0][1] * m[2][2]) * id;
  r.m[0][2] = (m[0][1] * m[1][2] - m[0][2] * m[1][1]) * id;
  r.m[1][0] = (m[1][2] * m[2][0] - m[1][0] * m[2][2]) * id;
  r.m[1][1] = (m[0][0] * m[2][2] - m[0][2] * m[2][0]) * id;
  r.m[1][2] = (m[1][0] * m[0][2] - m[0][0] * m[1][2]) * id;
  r.m[2][0] = (m[1][0] * m[2][1] - m[2][0] * m[1][1]) * id;
  r.m[2][1] = (m[2][0] * m[0][1] - m[0][0] * m[2][1]) * id;
  r.m[2][2] = (m[0][0] * m[1][1] - m[1][0] * m[0][1]) * id;
  return r;
}
void check_white(float wx, float wy) {
  if (!(wx >= 0.0f && wx <= 1.0f && wy > 0.0f && wy <= 1.0f)) fail("white point out of range");
}
// api/color.rs:124-190: RGB -> XYZ relative to the encoding's own white point.
M3 primaries_to_xyz(const float (*p)[2], float wx, float wy) {
  check_white(wx, wy);
  M3 pm;
  for (int i = 0; i < 3; i++) {
    pm.m[0][i] = double(p[i][0]);
    pm.m[1][i] = double(p[i][1]);
    pm.m[2][i] = 1.0 - double(p[i][0]) - double(p[i][1]);
  }
  const M3 pinv = inverse(pm);
  const double w[3] = {double(wx) / double(wy), 1.0, (1.0 - double(wx) - double(wy)) / double(wy)};
  double sv[3];
  mulv(pinv, w, sv);
  M3 sd{{{sv[0], 0, 0}, {0, sv[1], 0}, {0, 0, sv[2]}}};
  return mul(pm, sd);
}
// api/color.rs:193-252: Bradford adaptation of the white point to D50.
M3 adapt_to_xyz_d50(float wx, float wy) {
  check_white(wx, wy);
  static const M3 kBradford{{{0.8951, 0.2664, -0.1614}, {-0.7502, 1.7135, 0.0367}, {0.0389, -0.0685, 1.0296}}};
  static const M3 kBradfordInv{{{0.9869929, -0.1470543, 0.1599627}, {0.4323053, 0.5183603, 0.0492912}, {-0.0085287, 0.0400428, 0.9684867}}};
  const double w[3] = {double(wx) / double(wy), 1.0, (1.0 - double(wx) - double(wy)) / double(wy)};
  const double w50[3] = {0.96422, 1.0, 0.82521};
  double ls[3], l50[3];
  mulv(kBradford, w, ls);
  mulv(kBradford, w50, l50);
  M3 a{{{0, 0, 0}, {0, 0, 0}, {0, 0, 0}}};
  for (int i = 0; i < 3; i++) {
    if (ls[i] == 0.0) fail("white point with a zero LMS component");
    a.m[i][i] = l50[i] / ls[i];
  }
  return mul(kBradfordInv, mul(a, kBradford));
}
}  // namespace

OutputColour resolve_output_colour(const FileHeader& fh) {
  const ColorEncoding& c = fh.color_encoding;
  OutputColour oc;
  memcpy(oc.matrix, fh.opsin.inverse_matrix, sizeof(oc.matrix));
  if (c.want_icc) {
    oc.from_icc = true;
    return oc;
  }
  if (c.all_default) return oc;  // RGB, D65, sRGB primaries, sRGB curve
  if (c.color_space == ColorSpace::XYB || c.color_space == ColorSpace::Unknown)
    fail("XYB / unknown colour spaces have no simple output profile (outside the hot-path scope)", kErrUnsupported);
  // api/color.rs:319-326, 363-393 (the sRGB primaries are libjxl's rounded-through-f32 values)
  static const float kSrgbPrim[3][2] = {{0.6399987f, 0.33001015f}, {0.3000038f, 0.60000336f}, {0.15000205f, 0.059997204f}};
  static const float kBt2100Prim[3][2] = {{0.708f, 0.292f}, {0.170f, 0.797f}, {0.131f, 0.046f}};
  static const float kP3Prim[3][2] = {{0.680f, 0.320f}, {0.265f, 0.690f}, {0.150f, 0.060f}};
  float wx = 0.3127f, wy = 0.3290f;
  switch (c.white_point) {
    case 1: break;
    case 2: wx = float(c.white_xy[0]) / 1000000.0f; wy = float(c.white_xy[1]) / 1000000.0f; break;
    case 10: wx = wy = 1.0f / 3.0f; break;
    case 11: wx = 0.314f; wy = 0.351f; break;
    default: fail("unknown white point");
  }
  M3 inv;
  for (int i = 0; i < 9; i++) inv.m[i / 3][i % 3] = double(fh.opsin.inverse_matrix[i]);
  if (c.color_space == ColorSpace::Gray) {
    if (c.white_point != 1) fail("grey with a non-D65 white point needs a CMS (outside the hot-path scope)", kErrUnsupported);
    M3 lum;
    for (int i = 0; i < 3; i++)
      for (int j = 0; j < 3; j++) lum.m[i][j] = double(oc.luminances[j]);
    inv = mul(lum, inv);
  } else {
    float prim[3][2];
    switch (c.primaries) {
      case 1: memcpy(prim, kSrgbPrim, sizeof(prim)); break;
      case 2:
        for (int i = 0; i < 3; i++)
          for (int k = 0; k < 2; k++) prim[i][k] = float(c.primaries_xy[i][k]) / 1000000.0f;
        break;
      case 9: memcpy(prim, kBt2100Prim, sizeof(prim)); break;
      case 11: memcpy(prim, kP3Prim, sizeof(prim)); break;
      default: fail("unknown primaries");
    }
    if (c.primaries != 1 || c.white_point != 1) {  // xyb.rs:92-107
      const M3 srgb_to_xyzd50 = mul(adapt_to_xyz_d50(0.3127f, 0.3290f), primaries_to_xyz(kSrgbPrim, 0.3127f, 0.3290f));
      const M3 original_to_xyz = primaries_to_xyz(prim, wx, wy);
      for (int j = 0; j < 3; j++) oc.luminances[j] = float(original_to_xyz.m[1][j]);
      const M3 original_to_xyzd50 = mul(adapt_to_xyz_d50(wx, wy), original_to_xyz);
      const M3 srgb_to_original = mul(inverse(original_to_xyzd50), srgb_to_xyzd50);
      inv = mul(srgb_to_original, inv);
    }
  }
  for (int i = 0; i < 9; i++) oc.matrix[i] = float(inv.m[i / 3][i % 3]);
  if (c.have_gamma) {  // color_encoding.rs:145-158
    oc.tf = 2;
    oc.gamma = float(c.gamma) * 0.0000001f;
    if (oc.gamma > 1.0f || oc.gamma * 8192.0f < 1.0f) fail("invalid gamma");
    return oc;
  }
  switch (c.tf) {  // xyb.rs:122-133
    case TransferFunction::SRGB: oc.tf = 1; break;
    case TransferFunction::Linear: oc.tf = 0; break;  // Gamma(1.0): the reference skips the stage (frame/render.rs:761)
    case TransferFunction::BT709: oc.tf = 3; break;
    case TransferFunction::PQ: oc.tf = 4; break;
    case TransferFunction::HLG: oc.tf = 5; break;
    case TransferFunction::DCI: oc.tf = 2; oc.gamma = 1.0f / 2.6f; break;
    default: fail("unknown transfer function");
  }
  return oc;
}

}  // namespace jxg
