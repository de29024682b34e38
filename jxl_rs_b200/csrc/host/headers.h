// Codestream headers needed to reach the VarDCT hot path: signature/container,
// SizeHeader, ImageMetadata, CustomTransformData, FrameHeader, TOC.
//
// Reference: jxl/src/headers/{mod,size,image_metadata,bit_depth,color_encoding,
// extra_channels,transform_data,frame_header,toc,permutation,encodings}.rs and
// the container walk in jxl/src/api/inner/box_parser.rs.
#pragma once
#include <array>
#include <cstdint>
#include <string>
#include <vector>

#include "bitreader.h"

namespace jxg {

struct BitDepth {
  bool floating_point = false;
  uint32_t bits_per_sample = 8;
  uint32_t exponent_bits = 0;
};

struct ExtraChannelInfo {
  uint32_t type = 0;  // 0 = alpha
  BitDepth bit_depth;
  uint32_t dim_shift = 0;
  bool alpha_associated = false;
};

enum class TransferFunction : uint32_t { BT709 = 1, Unknown = 2, Linear = 8, SRGB = 13, PQ = 16, DCI = 17, HLG = 18 };
enum class ColorSpace : uint32_t { RGB = 0, Gray = 1, XYB = 2, Unknown = 3 };

struct ColorEncoding {
  bool all_default = true;
  bool want_icc = false;
  ColorSpace color_space = ColorSpace::RGB;
  uint32_t white_point = 1;  // D65 = 1, Custom = 2, E = 10, DCI = 11
  uint32_t primaries = 1;    // sRGB = 1, Custom = 2, BT2100 = 9, P3 = 11
  int32_t white_xy[2] = {0, 0};        // CustomXY, in 1e-6 units (color_encoding.rs:91-106)
  int32_t primaries_xy[3][2] = {{0, 0}, {0, 0}, {0, 0}};
  bool have_gamma = false;
  uint32_t gamma = 0;
  TransferFunction tf = TransferFunction::SRGB;
  uint32_t rendering_intent = 1;
};

struct OpsinInverseMatrix {
  // headers/transform_data.rs:19-32
  float inverse_matrix[9] = {11.031566901960783f, -9.866943921568629f, -0.16462299647058826f,
                             -3.254147380392157f, 4.418770392156863f,  -0.16462299647058826f,
                             -3.6588512862745097f, 2.7129230470588235f, 1.9459282392156863f};
  float opsin_biases[3] = {-0.0037930732552754493f, -0.0037930732552754493f, -0.0037930732552754493f};
  float quant_biases[4] = {1.0f - 0.05465007330715401f, 1.0f - 0.07005449891748593f, 1.0f - 0.049935103337343655f,
                           0.145f};
};

struct FileHeader {
  uint32_t xsize = 0, ysize = 0;
  // ImageMetadata
  uint32_t orientation = 1;
  bool have_preview = false;
  bool have_animation = false;
  bool have_timecodes = false;
  BitDepth bit_depth;
  bool modular_16bit_sufficient = true;
  std::vector<ExtraChannelInfo> extra_channels;
  bool xyb_encoded = true;
  ColorEncoding color_encoding;
  float intensity_target = 255.0f;
  OpsinInverseMatrix opsin;
  uint32_t custom_upsampling_mask = 0;
  // CustomTransformData.weights8 (transform_data.rs:343): the 8x upsampling weights, default or custom (mask bit 4)
  std::array<float, 210> weights8 = default_weights8();
  static std::array<float, 210> default_weights8();
};

struct Passes {
  uint32_t num_passes = 1;
  uint32_t num_ds = 0;
  std::vector<uint32_t> shift, downsample, last_pass;
};

struct RestorationFilter {
  // headers/frame_header.rs:146-234
  bool gab = true;
  float gab_w1[3] = {0.115169525f, 0.115169525f, 0.115169525f};  // x, y, b
  float gab_w2[3] = {0.061248592f, 0.061248592f, 0.061248592f};
  uint32_t epf_iters = 2;
  float epf_sharp_lut[8] = {0.0f, 1.0f / 7.0f, 2.0f / 7.0f, 3.0f / 7.0f, 4.0f / 7.0f, 5.0f / 7.0f, 6.0f / 7.0f, 1.0f};
  float epf_channel_scale[3] = {40.0f, 5.0f, 3.5f};
  float epf_quant_mul = 0.46f;
  float epf_pass0_sigma_scale = 0.9f;
  float epf_pass2_sigma_scale = 6.5f;
  float epf_border_sad_mul = 2.0f / 3.0f;
  float epf_sigma_for_modular = 1.0f;
};

struct BlendingInfo {
  uint32_t mode = 0, alpha_channel = 0, source = 0;
  bool clamp = false;
};

struct FrameHeader {
  uint32_t frame_type = 0;  // 0 regular, 1 LF, 2 reference-only, 3 skip-progressive
  uint32_t encoding = 0;    // 0 VarDCT, 1 Modular
  uint64_t flags = 0;
  bool do_ycbcr = false;
  uint32_t jpeg_upsampling[3] = {0, 0, 0};
  uint32_t upsampling = 1;
  std::vector<uint32_t> ec_upsampling;
  uint32_t group_size_shift = 1;
  uint32_t x_qm_scale = 3, b_qm_scale = 2;
  Passes passes;
  uint32_t lf_level = 0;
  bool have_crop = false;
  int32_t x0 = 0, y0 = 0;
  uint32_t frame_width = 0, frame_height = 0;
  BlendingInfo blending;
  std::vector<BlendingInfo> ec_blending;
  uint32_t duration = 0;
  bool is_last = true;
  uint32_t save_as_reference = 0;
  bool save_before_ct = false;
  std::string name;
  RestorationFilter rf;
  // derived
  uint32_t width = 0, height = 0;
  uint32_t num_extra_channels = 0;

  static constexpr uint64_t kNoise = 1, kPatches = 2, kSplines = 0x10, kUseLfFrame = 0x20, kSkipAdaptiveLf = 0x80;
  bool has_noise() const { return flags & kNoise; }
  bool has_patches() const { return flags & kPatches; }
  bool has_splines() const { return flags & kSplines; }
  bool has_lf_frame() const { return flags & kUseLfFrame; }
  bool adaptive_lf_smoothing() const { return !(flags & kSkipAdaptiveLf) && !has_lf_frame() && encoding == 0; }

  // geometry (frame_header.rs:448-665); 4:4:4 only (chroma subsampling is JPEG-recompression, out of scope)
  uint32_t group_dim() const { return 128u << group_size_shift; }
  uint32_t xsize() const { return (width + upsampling - 1) / upsampling; }
  uint32_t ysize() const { return (height + upsampling - 1) / upsampling; }
  uint32_t xsize_blocks() const { return (xsize() + 7) / 8; }
  uint32_t ysize_blocks() const { return (ysize() + 7) / 8; }
  uint32_t xsize_groups() const { return (xsize() + group_dim() - 1) / group_dim(); }
  uint32_t ysize_groups() const { return (ysize() + group_dim() - 1) / group_dim(); }
  uint32_t num_groups() const { return xsize_groups() * ysize_groups(); }
  uint32_t xsize_lf_groups() const { return (xsize_blocks() + group_dim() - 1) / group_dim(); }
  uint32_t ysize_lf_groups() const { return (ysize_blocks() + group_dim() - 1) / group_dim(); }
  uint32_t num_lf_groups() const { return xsize_lf_groups() * ysize_lf_groups(); }
  uint32_t num_toc_entries() const {
    if (num_groups() == 1 && passes.num_passes == 1) return 1;
    return 2 + num_lf_groups() + num_groups() * passes.num_passes;
  }
};

struct Toc {
  std::vector<uint32_t> sizes;    // in bitstream order
  std::vector<uint64_t> offsets;  // byte offsets (relative to the end of the TOC), logical section order
  std::vector<uint32_t> lengths;  // logical section order
};

// Strips the ISOBMFF container if present (box_parser.rs): returns the bare
// codestream (concatenated jxlc / jxlp payloads), or a copy of the input when
// it already starts with FF 0A.
std::vector<uint8_t> extract_codestream(const uint8_t* data, size_t size);
// Same, into a caller-owned vector (its capacity is reused).
void extract_codestream(const uint8_t* data, size_t size, std::vector<uint8_t>& out);

// Reads signature + SizeHeader + ImageMetadata + CustomTransformData (+ skips
// an ICC stream if present); leaves `br` positioned before the first frame
// header's byte alignment.
FileHeader read_file_header(BitReader& br);

FrameHeader read_frame_header(BitReader& br, const FileHeader& fh);

// toc.rs:20-32 + frame/decode.rs:263-285 (sections(): permutation applied).
Toc read_toc(BitReader& br, uint32_t num_entries);

// Scope guard shared by the VarDCT and the Modular front-ends: one still frame. Layered / animated files
// (FrameHeader.is_last == false, ImageMetadata.have_animation, a duration) would need blending of several frames
// (frame/render.rs:503); decoding only the first frame would silently differ from the reference, so these are refused
// with kErrUnsupported. (Orientation is applied by the store, as the reference's save stage does.)
void check_single_still_frame(const FileHeader& fh, const FrameHeader& h);

// Output colour of an XYB image: render/stages/xyb.rs:65-140 OutputColorInfo::from_header (opsin matrix re-targeted to
// the embedded primaries / white point, grey luminances folded in, embedded transfer function) plus the profile
// choice of api/inner/codestream_parser/image_info.rs:204-237 (an ICC-tagged image cannot be output to: integer
// samples get sRGB, float samples linear sRGB -> from_icc). Grey with a non-D65 white point and the XYB colour space
// (no simple output profile, color.rs:1287-1300) are refused with kErrUnsupported.
struct OutputColour {
  bool from_icc = false;
  uint32_t tf = 1;         // JXG_TF_* of the embedded encoding (ignored when from_icc)
  float gamma = 1.0f;      // exponent of JXG_TF_GAMMA
  float matrix[9];         // opsin inverse matrix, re-targeted
  float luminances[3] = {0.2126f, 0.7152f, 0.0722f};  // Y row of the output primaries (HLG OOTF)
};
OutputColour resolve_output_colour(const FileHeader& fh);

float f16_bits_to_float(uint16_t h);
float read_f16(BitReader& br);  // encodings.rs:59-74 (rejects NaN/Inf)
// LfQuantFactors of LfGlobal (quantizer.rs:28-52): the defaults (quant_weights::LF_QUANT), or three f16 values / 128.
void read_lf_quant_factors(BitReader& br, float out[3]);
uint64_t read_u64(BitReader& br);
void read_extensions(BitReader& br);

}  // namespace jxg
