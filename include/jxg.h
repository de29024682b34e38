/*
 * jxg.h — C ABI of libjxgpu.so: the H100 (sm_90a) replacement for the
 * per-group VarDCT decode + render hot path of libjxl/jxl-rs.
 *
 * The reference crate exposes no FFI (jxl/src/lib.rs:6 `#![deny(unsafe_code)]`);
 * the seam these entry points sit behind is internal:
 *
 *   Frame::decode_and_render_hf_groups        jxl/src/frame/render.rs:143
 *     (fan-out `parallel_runner.run(...)`     jxl/src/frame/render.rs:461-479)
 *       -> Frame::decode_hf_group             jxl/src/frame/decode.rs:790
 *       -> decode_vardct_group                jxl/src/frame/group.rs:383
 *       -> render stages Gaborish/EPF/XYB/FromLinear/Convert/Save
 *                                             jxl/src/frame/render.rs:579-620,757-905
 *
 * A Rust host keeps doing what jxl-rs does today up to that point (container,
 * headers, TOC, LfGlobal, LfGroups, HfGlobal) and hands the parsed frame state
 * plus the raw HF section bytes to `jxg_batch_add_frame`. INTEGRATION.md shows
 * the `extern "C"` block a maintainer would add.
 *
 * Conventions: every function returns 0 (JXG_OK) or a negative JXG_ERR_*.
 * All pointers in a JxgFrameDesc are HOST pointers that must stay valid until
 * jxg_batch_add_frame returns (the library copies what it needs into pinned
 * staging memory). One host thread per context; distinct contexts are
 * independent. No torch types cross this boundary.
 */
#ifndef JXG_H_
#define JXG_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define JXG_ABI_VERSION 2

/* Error codes; names mirror jxl/src/error.rs variants raised on this path. */
enum {
  JXG_OK = 0,
  JXG_ERR_BITSTREAM = -1,              /* generic malformed input (host front-end)  */
  JXG_ERR_UNSUPPORTED = -2,            /* feature outside the hot-path scope        */
  JXG_ERR_OUT_OF_BOUNDS = -3,          /* Error::OutOfBounds: section over-read     */
  JXG_ERR_INVALID_HISTOGRAM_INDEX = -4,/* Error::InvalidHistogramIndex group.rs:339 */
  JXG_ERR_INVALID_NUM_NONZEROS = -5,   /* Error::InvalidNumNonZeros   group.rs:544  */
  JXG_ERR_RESIDUAL_NONZEROS = -6,      /* Error::EndOfBlockResidualNonZeros :575    */
  JXG_ERR_ANS_CHECKSUM = -7,           /* Error::AnsChecksumMismatch  ans.rs:441    */
  JXG_ERR_INVALID_TRANSFORM = -8,      /* Error::InvalidVarDCTTransform             */
  JXG_ERR_INVALID_OUTPUT = -9,         /* Error::InvalidOutputBufferSize            */
  JXG_ERR_LZ77 = -10,                  /* UnexpectedLz77Repeat / ArithmeticOverflow */
  JXG_ERR_CUDA = -20,                  /* CUDA runtime failure                      */
  JXG_ERR_NO_DEVICE = -21,             /* no CUDA device: there is NO CPU fallback  */
  JXG_ERR_ARGUMENT = -22
};

/* Output pixel formats (JxlPixelFormat, jxl/src/api/data_types.rs:154). */
enum {
  JXG_FORMAT_RGB_U8 = 0,   /* interleaved sRGB-encoded u8, 3 B/px  (convert.rs:548) */
  JXG_FORMAT_RGBA_U8 = 1,  /* + opaque alpha 255 (fill_opaque_alpha, render.rs:858) */
  JXG_FORMAT_RGB_F32 = 2,  /* interleaved f32, 12 B/px; linear sRGB unless tf set   */
  JXG_FORMAT_XYB_F32_PLANAR = 3, /* debug/parity tap: the 3 XYB planes after filters */
  JXG_FORMAT_RGB_U16 = 4,  /* interleaved u16 (native endian), 6 B/px: clamp to [0,1], x 65535, round
                              (ConvertF32ToU16Stage, convert.rs:717-786, bit_depth 16; no dither) */
  JXG_FORMAT_RGB_F16 = 5   /* interleaved IEEE half, 6 B/px (ConvertF32ToF16Stage, convert.rs:789-857); PQ output
                              is clamped to [0,1], HLG to [-0.074, 1.1] first (frame/render.rs:746-750) */
};

/* Output transfer function (render/stages/from_linear.rs). */
enum {
  JXG_TF_LINEAR = 0, /* no curve (the reference adds no stage for a linear output, frame/render.rs:761)      */
  JXG_TF_SRGB = 1,   /* color/tf.rs:13-44                                                                     */
  JXG_TF_GAMMA = 2,  /* |v|^output_gamma, sign kept (from_linear.rs:97-109; DCI is gamma 1/2.6)               */
  JXG_TF_BT709 = 3,  /* color/tf.rs:114-150                                                                   */
  JXG_TF_PQ = 4,     /* color/tf.rs:261-304, 1.0 = intensity_target nits                                      */
  JXG_TF_HLG = 5     /* inverse OOTF with output_luminances, then the HLG OETF (color/tf.rs:458-470, 481-497) */
};

/* One entropy-coded histogram set + coefficient orders, per pass
 * (HfGlobalState.passes[i], jxl/src/frame/decode.rs:519-545). */
typedef struct JxgPassDesc {
  uint32_t shift;                 /* frame_header.passes.shift[pass] (group.rs:350) */
  uint32_t use_prefix;            /* 1: prefix codes, 0: ANS                         */
  uint32_t log_alpha_size;        /* ANS only: 5..8                                  */
  uint32_t num_clusters;
  uint32_t num_contexts;          /* length of context_map (incl. +16 padding)       */
  uint32_t lz77_enabled, lz77_min_symbol, lz77_min_length;
  uint32_t lz77_length_uint;      /* packed hybrid-uint config                       */
  uint32_t lz_dist_cluster;
  const uint8_t* context_map;     /* [num_contexts] context -> cluster (decode.rs:547)*/
  const uint32_t* uint_configs;   /* [num_clusters] split_exp | msb<<8 | lsb<<16     */
  const uint64_t* ans_buckets;    /* [num_clusters << log_alpha_size], ans.rs:31-39:
                                     alias_symbol u8 | alias_cutoff u8 <<8 | dist u16 <<16
                                     | alias_offset u16 <<32 | alias_dist_xor u16 <<48 */
  const uint32_t* huff_entries;   /* bits | value<<16, concatenated 2-level LUTs     */
  const uint32_t* huff_offset;    /* [num_clusters] start of each LUT                */
  uint32_t huff_entries_len;
  /* 13 shapes x 3 channels coefficient orders (coeff_order.rs:122). NULL = all
   * natural orders (used_orders == 0). Otherwise order i starts at
   * coeff_order_offset[i] (index = shape*3 + c). */
  const uint32_t* coeff_order;
  uint32_t coeff_order_offset[39];
  uint32_t coeff_order_len;
} JxgPassDesc;

typedef struct JxgFrameDesc {
  uint32_t abi_version;           /* JXG_ABI_VERSION                                  */
  uint32_t width, height;         /* frame_header.size() in pixels                    */
  /* ---- quantiser / CfL (LfGlobal) ---- */
  uint32_t global_scale;          /* quantizer.rs:55                                  */
  uint32_t x_qm_scale, b_qm_scale;/* group.rs:395-396                                 */
  float quant_biases[4];          /* transform_data.rs:30-31                          */
  float base_correlation_x, base_correlation_b; uint32_t color_factor; /* color_correlation_map.rs:21 */
  /* ---- block context map (block_context_map.rs:46-53) ---- */
  uint32_t num_qf_thresholds; uint32_t qf_thresholds[15];
  uint32_t num_lf_contexts;       /* product of (lf thresholds + 1)                   */
  uint32_t num_block_contexts;    /* max(ctx_map)+1, <= 16                            */
  uint32_t block_ctx_map_len;     /* 39 * (num_qf_thresholds+1) * num_lf_contexts     */
  const uint8_t* block_ctx_map;
  uint32_t num_histograms;        /* HfGlobal, frame/decode.rs:512                    */
  uint32_t num_passes;
  const JxgPassDesc* passes;      /* [num_passes]                                     */
  /* ---- dequant matrices (quant_weights.rs:1081): NULL entry = library default ---- */
  const float* dequant_tables[17];
  /* ---- per-frame planes, dimensions in 8x8 blocks: xb = ceil(width/8) ---- */
  const float* lf[3];             /* X, Y, B dequantised (and smoothed) LF, stride xb */
  const uint8_t* transform_map;   /* HfTransformType | 128 for first block of varblock*/
  const int32_t* raw_quant_map;   /* 1..256                                           */
  const uint8_t* epf_map;         /* sharpness 0..7                                   */
  const uint8_t* quant_lf;        /* LF context bucket per block (modular/mod.rs:895) */
  const int8_t* ytox_map;         /* ceil(xb/8) x ceil(yb/8)                          */
  const int8_t* ytob_map;
  /* ---- restoration filter (frame_header.rs:146-234) ---- */
  uint32_t gab;                   float gab_w1[3], gab_w2[3];   /* per X,Y,B */
  uint32_t epf_iters;
  float epf_sharp_lut[8]; float epf_channel_scale[3];
  float epf_quant_mul, epf_pass0_sigma_scale, epf_pass2_sigma_scale, epf_border_sad_mul;
  /* ---- colour (xyb.rs:145-241) ---- */
  float opsin_inverse_matrix[9]; float opsin_biases[3]; float intensity_target;
  uint32_t output_tf;             /* JXG_TF_*                                         */
  uint32_t output_format;         /* JXG_FORMAT_*                                     */
  /* ImageMetadata.orientation 1..8 (headers/image_metadata.rs:41-50), applied by the store as the reference's save stage
   * does (render/save.rs, api/options.rs:39 adjust_orientation = true): the output buffer holds the image in display
   * orientation, i.e. height x width swap for values 5..8. The XYB debug tap ignores it. */
  uint32_t orientation;
  /* Output encoding as OutputColorInfo::from_header derives it (render/stages/xyb.rs:65-140): opsin_inverse_matrix above
   * is already re-targeted to the output primaries / white point (grey: three luminance rows). */
  float output_gamma;             /* JXG_TF_GAMMA exponent                             */
  float output_luminances[3];     /* Y row of the output primaries (JXG_TF_HLG)        */
} JxgFrameDesc;

/* PCI bus id of a CUDA device in the spelling of /sys/bus/pci/devices ("0000:1b:00.0"): lets the host bind its
 * threads and pinned allocations to the GPU's NUMA node before jxg_init. buf: >= 16 bytes. */
int jxg_device_pci_bus_id(int device, char* buf, int len);

/* Context: one per device/rank. Owns streams, pinned staging and device pools. */
int jxg_init(int device, void** ctx);
void jxg_shutdown(void* ctx);

/* Test hook, off by default: with `byte` in 0..255, every later jxg_batch_run / jxg_modular_batch_run of the context
 * first writes `byte` over the whole capacity of each of the context's device pools (the intermediates of both engines
 * and the device copy of the staging blob, whose tail past the uploaded bytes keeps the pattern), on the stream that
 * carries the upload, and jxg_batch_begin / jxg_modular_batch_begin write it over the pinned staging arena on the host;
 * jxg_batch_rerun_device / jxg_modular_batch_rerun_device fill every pool but the staging blob, which the rerun reuses.
 * Output bytes must not depend on the byte: a kernel that reads device memory its batch did not write shows up as a
 * difference. Constant tables of the context, caller-owned outputs and the status readback buffer are not touched.
 * byte = -1 turns the hook off. Each begin, run and rerun uses the byte in force when it is called. JXG_ERR_ARGUMENT for a
 * NULL context or a byte outside -1..255. */
int jxg_context_set_pool_fill(void* ctx, int byte);

/* Test hook, off by default: with n >= 1 every scheduling decision of the context's later batches (VarDCT and Modular)
 * takes n in place of the device's SM count: the lean entropy kernel's lanes per warp, lanes per frame and queued
 * streams, the fast entropy kernel's streams per warp, the Modular decode grid and the grid-stride grids of the Modular
 * transforms. n = 0 restores the device's own count. Outputs do not depend on it, only which schedule produces them:
 * a small n reaches the queued streams and wide warps of very large batches with small ones. JXG_ERR_ARGUMENT for a
 * NULL context or a negative n. */
int jxg_context_set_sm_budget(void* ctx, int n);

/* Batch of frames decoded together (one kernel pipeline over all groups of
 * all frames). Replaces N calls of decode_and_render_hf_groups. */
int jxg_batch_begin(void* ctx, uint32_t n_frames_hint, void** batch);

/* hf_bytes: the frame's HF section bytes, any layout; section s (pass-major:
 * s = pass * num_groups + group, frame/mod.rs:326-338) lives at
 * hf_bytes[sec_off[s] .. sec_off[s] + sec_len[s]). n_sections = passes * groups.
 * out/out_row_stride: destination for the frame's pixels; `out_is_device` says
 * whether it is a device pointer (left in HBM) or a host pointer (D2H copy is
 * part of jxg_batch_run + jxg_batch_wait). The device stores whole samples, so
 * out_row_stride must be a multiple of the sample size: 4 bytes for RGBA_U8,
 * RGB_F32 and XYB_F32_PLANAR, 2 for RGB_U16 and RGB_F16, any for RGB_U8. A
 * device `out` must be aligned the same way. Otherwise the call returns
 * JXG_ERR_INVALID_OUTPUT. (jxg_batch_add_parsed follows the same rule.) */
int jxg_batch_add_frame(void* batch, const JxgFrameDesc* desc, const uint8_t* hf_bytes,
                        const uint64_t* sec_off, const uint32_t* sec_len, uint32_t n_sections,
                        void* out, size_t out_row_stride, int out_is_device);

/* Uploads (H2D from pinned staging), launches the kernels, queues D2H for host
 * outputs. Asynchronous on the context's stream (or `cuda_stream` if non-NULL). */
int jxg_batch_run(void* batch, void* cuda_stream);
/* Blocks until the batch finished; returns the first error (per-stream status
 * words written by the entropy kernel, check_final_state decode.rs:400). */
int jxg_batch_wait(void* batch, uint32_t* first_bad_frame, uint32_t* first_bad_group);
/* Re-run the same batch (inputs already resident in HBM): device-only timing. Ordered after the batch's own last
 * run, whichever stream that ran on. */
int jxg_batch_rerun_device(void* batch, void* cuda_stream);
void jxg_batch_end(void* batch);

/* Parity taps: copy intermediate planes of frame `f` of a batch to host, after
 * waiting for the batch's own last run on whichever stream it ran.
 * coeffs: 3 planes of i32, dense per group in decode order (group.rs:53).
 * xyb: the 3 padded XYB planes (f32) after dequant + IDCT; `stage` must be 0
 * (JXG_ERR_ARGUMENT otherwise). Meaningful after a run stopped with debug stop 2. */
int jxg_batch_read_coeffs(void* batch, uint32_t f, int32_t* out, size_t out_len);
int jxg_batch_read_xyb(void* batch, uint32_t f, int stage, float* out, size_t out_len);

/* Opt-in host-side staging speed-up: copies of the large inputs (LF planes, per-block maps, HF sections) into the
 * pinned staging blob are postponed to jxg_batch_run and spread over `threads` host threads. Every pointer passed to
 * jxg_batch_add_frame / jxg_batch_add_parsed afterwards must stay valid until jxg_batch_run returns. 0 = immediate
 * copies (default; the contract a `&[u8]`-borrowing Rust caller gets, frame/render.rs:143). */
int jxg_batch_set_deferred_copy(void* batch, int threads);

/* Debug/parity: 0 = run everything (default), 1 = stop after the entropy kernel,
 * 2 = stop after dequant+IDCT (planes readable with jxg_batch_read_xyb stage 0).
 * JXG_ERR_ARGUMENT for a NULL batch or any other stage. */
int jxg_batch_set_debug_stop(void* batch, int stage);

/* Per-stage device timing with CUDA events on the launching stream (bench.py roofline):
 * stages = memset, entropy, dequant_idct, gaborish, epf0, epf1, epf2, xyb_store. */
int jxg_batch_set_profile(void* batch, int on);
int jxg_batch_stage_times(void* batch, float* ms, int n);
/* Absolute device times (ms since a process-wide reference event set at the first call) of the 9 stage events of the
 * last run: the timeline of several batches in flight. With n >= 11, ms[9] and ms[10] are the run's first event (before
 * the H2D copy of the staging blob) and its last one (behind the D2H copies of the outputs). */
int jxg_batch_stage_marks(void* batch, float* ms, int n);

/* Counters for bench.py (kernels launched by the last run, bytes moved). */
int jxg_batch_stats(void* batch, uint64_t* kernel_launches, uint64_t* h2d_bytes, uint64_t* d2h_bytes,
                    float* last_device_ms);

/* Which entropy kernel instances the batch's streams go to: the streams of k_entropy_lean (ANS, one pass, no shift,
 * no LZ77), k_entropy_fast (prefix codes or a shifted single pass) and k_entropy (several passes or LZ77);
 * lean_all_420: the lean kernel's instance that assumes hybrid-uint configuration (4, 2, 0) in every cluster;
 * lean_ctx_smem: the instance that stages the context maps in shared memory; lean_S: lanes per warp of the lean
 * schedule (4 or 8), 0 before jxg_batch_run or without lean streams. Any pointer may be NULL. */
int jxg_batch_entropy_stats(void* batch, uint32_t* n_lean, uint32_t* n_fast, uint32_t* n_slow, int* lean_all_420,
                            int* lean_ctx_smem, uint32_t* lean_S);

/* The entropy schedule of the last jxg_batch_run. For frame f: its lean streams (lean_count), the lanes that start on
 * them (lean_lanes; the other lean_count - lean_lanes streams are queued and taken by whichever of the frame's lanes
 * ends first) and its CTAs of k_entropy_lean. With f = JXG_ALL_FRAMES: the batch's lean streams, the sum of the lanes
 * and the grid k_entropy_lean is launched with. fast_S: streams per warp of k_entropy_fast (1, 2, 4 or 8; 0 without
 * such streams). lean_pulls (waits for the last run): how often the frame's lanes pulled from its stream queue, once
 * per queued stream and once more per lane when the queue was empty, so lean_count when every queued stream was
 * taken exactly once. JXG_ERR_ARGUMENT before jxg_batch_run or for a frame out of range. Any output pointer may be
 * NULL. */
#define JXG_ALL_FRAMES 0xffffffffu
int jxg_batch_entropy_schedule(void* batch, uint32_t f, uint32_t* lean_count, uint32_t* lean_lanes, uint32_t* lean_ctas,
                               uint32_t* fast_S, uint32_t* lean_pulls);
/* The status word of each group of frame f after the last run (0, or the JXG_ERR_* its entropy stream or block plan
 * ended with; groups of a region frame are those of its sub-frame), out[0 .. num_groups). Waits for the last run.
 * JXG_ERR_ARGUMENT before jxg_batch_run, for a frame out of range or when n < the frame's group count. */
int jxg_batch_stream_status(void* batch, uint32_t f, int32_t* out, uint32_t n);

/* The transform-class partition of the block plan for each group of frame f after the last run: counts[g * 8 + c] =
 * varblocks of class c of group g, entries[g * 1024 ..] = one word per varblock, class after class: its ordinal in the
 * raster order of the group's varblocks | bx << 10 | by << 15 (its first block inside the group) | transform type << 20.
 * Classes: 0 DCT8X8 / DCT4X4 / DCT4X8 / DCT8X4, 1 DCT16X8 / DCT8X16, 2 DCT16X16, 3 the other types of at most 4 x 4
 * blocks, 4 larger varblocks; words 5..7 are 0. Classes 0..2 are grouped by transform type in the order
 * 0, 3, 12, 13 / 6, 7 / 4, raster order within a type; classes 3 and 4 are in raster order. A group whose block plan
 * failed has all counts 0. Slots of entries behind the group's varblocks are not written. Waits for the last run;
 * JXG_ERR_ARGUMENT before jxg_batch_run, for a frame out of range or when n < the frame's group count. */
int jxg_batch_read_transform_plan(void* batch, uint32_t f, uint32_t* counts, uint32_t* entries, uint32_t n);

/* ---------------- convenience front-end (host parse + batch) ----------------
 * Parses complete .jxl files (container or bare codestream) on the host with
 * the in-tree C++ front-end (the stand-in for the Rust host: headers, TOC,
 * LfGlobal, LfGroups, HfGlobal), then feeds the batch API above. Mirrors
 * JxlDecoder::process for whole files (jxl/src/api/decoder.rs:258).
 * Frames with extra channels (alpha ...) are accepted and decode to their colour channels — the output of the
 * reference when JxlPixelFormat::extra_channel_format holds None (api/data_types.rs:154); patches, splines,
 * upsampling, non-regular / blended frames and JPEG recompression return JXG_ERR_UNSUPPORTED. */
typedef struct JxgImageInfo {
  uint32_t width, height; /* size of the OUTPUT (display orientation): what the caller allocates */
  uint32_t num_groups, num_passes;
  uint32_t encoding;      /* 0 VarDCT, 1 Modular */
  uint64_t hf_bytes;      /* sum of HF section sizes */
  uint32_t coded_width, coded_height; /* frame size as coded (swapped against width/height for orientation 5..8) */
  uint32_t orientation;   /* 1..8 */
} JxgImageInfo;

int jxg_parse_file(const uint8_t* data, size_t size, void** parsed, JxgImageInfo* info);
/* Same, decoding the frame's LF groups (independent TOC sections, frame/decode.rs:429 decode_lf_group) on `threads`
 * host threads, the fan-out jxl-rs does over its parallel runner (api/inner/codestream_parser/frame_info.rs:505-520):
 * the latency path for one large image. The parsed state does not depend on `threads`. */
int jxg_parse_file_mt(const uint8_t* data, size_t size, int threads, void** parsed, JxgImageInfo* info);
void jxg_parsed_free(void* parsed);
/* Adds a parsed frame to a batch with the given output. */
int jxg_batch_add_parsed(void* batch, void* parsed, uint32_t output_format, void* out, size_t out_row_stride,
                         int out_is_device);
/* Exposes the parsed frame as the (desc, sections) tuple jxg_batch_add_frame takes;
 * pointers stay valid until jxg_parsed_free. */
int jxg_parsed_desc(void* parsed, uint32_t output_format, JxgFrameDesc* desc, const uint8_t** hf_bytes,
                    const uint64_t** sec_off, const uint32_t** sec_len, uint32_t* n_sections);

/* ---- Region decode of VarDCT frames ------------------------------------------------------------------------------
 * A region is a rectangle of the OUTPUT image (display orientation, the JxgImageInfo width x height). Its pixels are
 * defined as the pixels the whole-frame decode gives on that rectangle; the reference has no crop API. The bytes are
 * the same when both outputs take the same store path. That holds in every case but one: Gaborish + EPF 2 frames with
 * orientation 1 in RGB_U8, RGBA_U8 or RGB_F32. These filter their interior tiles with a vector path when the output
 * row is aligned: for RGB_U8 a row stride (and, for a device output, a base address) that is a multiple of 4 bytes,
 * otherwise a multiple of 16. The vector path differs from the scalar one by a few float ulps (1 LSB at most in U8).
 * So the region and whole outputs are byte-identical when both are aligned or both are not. Only the HF
 * groups the region needs are entropy-decoded, transformed and filtered: the 256x256 groups that hold a pixel the
 * region's pixels depend on through Gaborish and EPF (within 1 + 2 / 3 / 6 pixels; with Gaborish + EPF 2, of the
 * 64x32 filter tiles that meet the region), and only the region is stored. The output buffer holds region.height rows
 * of region.width pixels; stride and alignment rules are those of jxg_batch_add_frame applied to that width. The
 * region must be non-empty and inside the image, and the format must not be XYB_F32_PLANAR: JXG_ERR_ARGUMENT
 * otherwise. jxg_batch_read_coeffs / jxg_batch_read_xyb refuse a region frame (JXG_ERR_ARGUMENT); jxg_batch_wait
 * reports the group index of the whole frame. Each region is its own frame of the batch, also when regions of one
 * frame overlap. */
typedef struct JxgRegion {
  uint32_t x, y, width, height;
} JxgRegion;

/* jxg_batch_add_frame for a region: desc and the sections describe the whole frame and are checked as
 * jxg_batch_add_frame checks them. */
int jxg_batch_add_frame_region(void* batch, const JxgFrameDesc* desc, const uint8_t* hf_bytes, const uint64_t* sec_off,
                               const uint32_t* sec_len, uint32_t n_sections, const JxgRegion* region, void* out,
                               size_t out_row_stride, int out_is_device);
/* jxg_batch_add_parsed for a region. */
int jxg_batch_add_parsed_region(void* batch, void* parsed, uint32_t output_format, const JxgRegion* region, void* out,
                                size_t out_row_stride, int out_is_device);
/* Parity tap, no device needed: the sub-frame a region decodes, as a self-contained (desc, sections) tuple that
 * jxg_batch_add_frame would take. Its groups are the rectangle of whole groups the region needs (origin: the coded
 * position of its top-left pixel, multiples of 256); section s = pass * G' + group of the sub-frame (G' its group count)
 * is section pass * G + group of the frame. window: the top-left of the region inside the sub-frame's display-oriented
 * output. The pointers stay valid until the next call on `parsed` or jxg_parsed_free. */
int jxg_parsed_region_desc(void* parsed, uint32_t output_format, const JxgRegion* region, JxgFrameDesc* desc,
                           const uint8_t** hf_bytes, const uint64_t** sec_off, const uint32_t** sec_len,
                           uint32_t* n_sections, uint32_t origin[2], uint32_t window[2]);

/* ---- Modular frames (BASELINE config 5; SURVEY §8 rows a18 / a19) ------------------------------------------------
 * Seam: FullModularImage::read_stream for ModularHF sections (jxl/src/frame/modular/mod.rs:567,
 * decode/bitstream.rs:134, decode/channel.rs:220) plus the inverse transforms (transforms/{rct,squeeze}.rs) and
 * ConvertI32ToU8 (render/stages/convert.rs:642). The host front end (headers, LfGlobal incl. the global MA tree,
 * section 0, ModularLF streams, group headers / local trees) is jxg_modular_parse_file; a Rust host would hand over
 * the same state from Frame::decode_lf_global / decode_lf_group (frame/decode.rs:307-497).
 * Device scope: lossless 8-bit RGB / grey and lossy (XYB-encoded) frames, one pass, global transforms RCT and Squeeze,
 * group-local RCT, ANS or prefix codes,
 * all 14 predictors incl. the weighted one, all properties incl. those of reference channels, the global palette
 * transform without delta entries (transforms/palette.rs:165-199), LZ77 in group streams (decode.rs:286-330, the window
 * in device memory: min(2^20, pixels) x 4 bytes per LZ77 stream). Delta palettes return JXG_ERR_UNSUPPORTED (no CPU
 * fallback). A group stream that fails (ANS checksum, over-read, an LZ77 copy before any symbol or a copy length
 * overflow: JXG_ERR_LZ77) is reported by jxg_modular_batch_wait; the other streams still decode. Output of a lossless
 * frame: interleaved RGB u8 (grey replicated), ConvertI32ToU8. An XYB frame (ImageMetadata.xyb_encoded, what lossy
 * Modular encoders write) codes three channels Y, X, B whatever its colour encoding (frame/decode.rs:167-170); they are
 * converted as ConvertModularXYBToF32Stage does (render/stages/convert.rs:278-343: X = x s_x, Y = y s_y,
 * B = (b + y) s_b with the frame's LfQuantFactors) and stored through the output stage of a VarDCT frame (XYB to the
 * output colour, transfer curve, sample conversion with the u8 dither at frame coordinates, orientation), in any
 * JXG_FORMAT_* (jxg_modular_batch_add_output). An XYB frame with Gaborish or EPF enabled is refused with
 * JXG_ERR_UNSUPPORTED at the parse: those filters are not applied to Modular frames here. Frames of one batch must agree on the kind of each inverse-transform step they share: one
 * frame's step list may be a prefix of another's, in either order of adding. A frame jxg_modular_batch_add refuses
 * leaves the batch as it was (no stream of it decodes, no statistic counts it); a group-local Squeeze is refused with
 * JXG_ERR_UNSUPPORTED. A rectangle of a frame can be decoded alone (jxg_modular_batch_add_region). */
int jxg_modular_parse_file(const uint8_t* data, size_t size, void** parsed, JxgImageInfo* info);
void jxg_modular_parsed_free(void* parsed);
int jxg_modular_batch_begin(void* ctx, void** batch);
/* `parsed` must stay alive until jxg_modular_batch_end. Output RGB_U8 (an XYB frame too); the same as
 * jxg_modular_batch_add_output with JXG_FORMAT_RGB_U8 and no region. */
int jxg_modular_batch_add(void* batch, void* parsed, void* out, size_t out_row_stride, int out_is_device);
/* Adds a frame, or the region `region` of it (NULL: the whole frame; see jxg_modular_batch_add_region), in output
 * format `output_format`. An XYB frame takes every format, with the stride and alignment rules of jxg_batch_add_frame
 * applied to the frame's or region's width; XYB_F32_PLANAR writes the X, Y, B planes of the whole frame in the coded
 * orientation (3 x coded height rows of coded width f32) and has no region form (JXG_ERR_ARGUMENT). A lossless frame
 * takes RGB_U8 only, and is then exactly jxg_modular_batch_add / _add_region; any other format returns
 * JXG_ERR_UNSUPPORTED. An unknown format returns JXG_ERR_ARGUMENT. A refused frame leaves the batch as it was. */
int jxg_modular_batch_add_output(void* batch, void* parsed, uint32_t output_format, const JxgRegion* region, void* out,
                                 size_t out_row_stride, int out_is_device);
/* The colour side of a parsed Modular frame, no device needed: *xyb_encoded (1: an XYB frame), the coded colour
 * channels (3 for every XYB frame), and for an XYB frame its LfQuantFactors (lf_quant[3], X, Y, B) and in `desc` the
 * output stage a batch applies for output_format: width, height, orientation, output_format, opsin_biases,
 * intensity_target, output_tf, output_gamma, output_luminances, opsin_inverse_matrix (every other field zero). Any
 * pointer may be NULL; lf_quant and desc are not written for a lossless frame. An unknown format: JXG_ERR_ARGUMENT. */
int jxg_modular_parsed_colour(void* parsed, uint32_t output_format, int* xyb_encoded, uint32_t* colour_channels,
                              float* lf_quant, JxgFrameDesc* desc);

/* ---- Region decode of Modular frames ----------------------------------------------------------------------------
 * A region is a JxgRegion rectangle of the OUTPUT image (display orientation, the JxgImageInfo width x height of
 * jxg_modular_parse_file). Its pixels are defined as the pixels of the whole-frame decode on that rectangle, and they
 * are byte-identical to them for every orientation, host and device outputs and any valid stride: everything up to the
 * u8 store is integer arithmetic, and an XYB frame's conversion and output stage are per pixel, with the u8 dither at
 * whole-frame coordinates. The output holds region.height rows of region.width RGB u8 pixels; the stride rule
 * is that of jxg_modular_batch_add applied to the region's width (JXG_ERR_INVALID_OUTPUT). An empty region or one
 * outside the image returns JXG_ERR_ARGUMENT; a frame jxg_modular_batch_add refuses is refused with the same code, and
 * a refused region leaves the batch as it was. Only the group streams the region depends on are uploaded and decoded,
 * and the global inverse transforms and the store run only on the rectangles it depends on (the dependency cone):
 * RCT mixes the same position of its three channels, a palette look-up needs the palette whole, and an unsqueeze
 * output depends on the outputs to its left (horizontal) or above (vertical), so on Squeeze frames the cone reaches the
 * top-left corner of each squeeze level and a crop far from it needs most of the frame's streams. The plane memory of
 * the frame is sized to the cone. jxg_modular_batch_wait reports the failing group by its index in the whole frame;
 * jxg_modular_batch_read_planes refuses a region frame (JXG_ERR_ARGUMENT). Each region is its own frame of the batch,
 * also when regions of one parsed frame overlap. */
int jxg_modular_batch_add_region(void* batch, void* parsed, const JxgRegion* region, void* out, size_t out_row_stride,
                                 int out_is_device);
/* Parity tap, no device needed: the cone of a region as jxg_modular_batch_add_region computes it, after the same
 * checks. groups[0 .. *n_groups): the ModularHF groups decoded (whole-frame indices, ascending). rects: 8 words per
 * buffer of the frame's inverse plan (its coded channels first, then the outputs of the plan's steps in plan order):
 * the rectangle the frame's plane memory holds of it, then the rectangle the region needs of it, each as
 * x0, y0, x1, y1 (half-open; all zero when empty). groups and rects may be NULL; *n_groups and *n_buffers are always
 * written, and JXG_ERR_ARGUMENT is returned when max_groups or max_buffers is smaller than they say. */
int jxg_modular_parsed_region_plan(void* parsed, const JxgRegion* region, uint32_t* groups, uint32_t max_groups,
                                   uint32_t* n_groups, uint32_t* rects, uint32_t max_buffers, uint32_t* n_buffers);
/* Streams per warp of the decode kernel (1, 2 or 4; default 1). */
int jxg_modular_batch_set_lanes(void* batch, int lanes_per_warp);
int jxg_modular_batch_run(void* batch, void* cuda_stream);
int jxg_modular_batch_wait(void* batch, uint32_t* first_bad_frame, uint32_t* first_bad_group);
/* Ordered after the batch's own last run, whichever stream that ran on. */
int jxg_modular_batch_rerun_device(void* batch, void* cuda_stream);
/* Parity tap: final colour planes of frame f (3 x H x W i32, before the u8 conversion; Y, X, B of an XYB frame before
 * its conversion to XYB floats), after waiting for the
 * batch's own last run on whichever stream it ran. JXG_ERR_ARGUMENT for a region frame. */
int jxg_modular_batch_read_planes(void* batch, uint32_t f, int32_t* out, size_t out_len);
/* ms[0]: whole batch on the device, ms[1]: group-stream decode kernel (+ local RCT). */
int jxg_modular_batch_stats(void* batch, uint64_t* h2d_bytes, uint64_t* d2h_bytes, uint64_t* kernel_launches, float* ms);
/* Group streams of the frames added so far whose code uses LZ77; of those, the ones whose copies all have distance 1
 * (Histograms::is_rle, the shape of libjxl's fastest lossless mode); device bytes of their symbol windows. */
int jxg_modular_batch_lz77_stats(void* batch, uint32_t* lz77_streams, uint32_t* rle_streams, uint64_t* window_bytes);
/* Non-empty group-stream rects of the frames added so far, by the channel walk the decode kernel takes for them (the
 * walk chosen at jxg_modular_batch_add, after the channel / stream decisions of the tree): the generic tree walk; the
 * table walk of a single leaf; the table walk over property p in by_property[p] (16 entries, 2..15 used, see
 * jxg_modular_walk_table); and of the table rects, those whose stream uses the weighted predictor. Any pointer may be
 * NULL. */
int jxg_modular_batch_walk_stats(void* batch, uint32_t* generic, uint32_t* single_leaf, uint32_t* by_property,
                                 uint32_t* table_wp);
void jxg_modular_batch_end(void* batch);
/* Parity tap (no device needed): the table form of one channel's MA-tree walk as the Modular path builds it - the device
 * counterpart of the single-property specialisations of frame/modular/decode/specialized_trees.rs:197-372.
 * nodes: n_nodes x 5 ints {property (< 0: leaf), split value | offset, left child | predictor, right child | multiplier,
 * leaf context}; context_map: leaf context -> cluster. Returns 1 and fills lut[2048] (index = property value clamped to
 * [-1024, 1023] + 1024; entry = predictor | cluster << 4 | plain << 12 | leaf node << 16) and *property (0xff: single leaf,
 * every entry equal) when the tree left after the channel / stream decisions has a table form, 0 when the channel needs
 * the generic walk, JXG_ERR_ARGUMENT on malformed input. */
int jxg_modular_walk_table(const int32_t* nodes, uint32_t n_nodes, const uint8_t* context_map, uint32_t n_contexts,
                           uint32_t channel, uint32_t stream_id, uint32_t* lut, uint32_t* property);

/* ---- Thumbnail decode (1:8) of VarDCT frames --------------------------------------------------------------------
 * The LF image of a VarDCT frame (one sample per 8x8 block) is a 1:8 picture of it, coded in LfGlobal and the LfGroup
 * sections ahead of HfGlobal and the HF groups. A thumbnail has ceil(width / 8) x ceil(height / 8) pixels (JxgImageInfo
 * width and height, display orientation). Its pixel (bx, by) of the coded LF image is the reference's lf_image after
 * finalize_lf (decode_vardct_lf, frame/modular/mod.rs:931-982; dequant_lf, mod.rs:837, with extra_precision and the LF
 * chroma-from-luma; adaptive_lf_smoothing, frame/adaptive_lf_smoothing.rs:44, when the frame applies it): the planes
 * JxgFrameDesc.lf carries. These go through the output stage of the full decode (XYB -> linear with the re-targeted
 * opsin matrix, transfer function, sample format, orientation), with the u8 dither taken at the coded LF coordinate
 * (bx, by). Gaborish and EPF are full-resolution filters and are not applied: a thumbnail is not a box-downscale of the
 * full decode. The reference has no thumbnail API.
 *
 * jxg_lf_parse_file parses the headers, TOC and LfGlobal and, per LF group, the header of its LF-coefficient stream; it
 * decodes no LF pixel, no HF metadata, no HfGlobal and no HF section, and reads no byte past the end of the last LF-group
 * section, so a bare codestream cut anywhere after it parses (one cut inside an LF-group section:
 * JXG_ERR_OUT_OF_BOUNDS). A container must be whole. A frame with one section (one group, one pass, at most 256x256)
 * keeps LfGlobal, the LF group, HfGlobal and the HF group in one bit stream, and its HF byte count (JxgImageInfo.hf_bytes)
 * is known only where HfGlobal ends: such a frame is parsed in full, as jxg_parse_file parses it, so its section must be
 * whole and a one-section file whose HF metadata or HfGlobal is corrupt is refused. `info` is what jxg_parse_file returns for the same file, and the file checks are those of jxg_parse_file, with
 * the same codes. */
int jxg_lf_parse_file(const uint8_t* data, size_t size, void** parsed, JxgImageInfo* info);
void jxg_lf_parsed_free(void* parsed);
/* Adds a thumbnail of `parsed` (jxg_lf_parse_file; it must stay alive until jxg_modular_batch_end) as a frame of a
 * Modular batch: its LF streams are decoded on the device with the batch's group streams (lanes, pools, status words
 * and jxg_modular_batch_wait, which reports a failing LF stream by its LF-group index), then dequantised, smoothed and
 * stored. All six output formats; XYB_F32_PLANAR holds the three LF planes after smoothing in the coded orientation,
 * plane c from row c * height (the JxgFrameDesc.lf planes, bit for bit). Stride and alignment rules are those of
 * jxg_batch_add_frame applied to the thumbnail's width (JXG_ERR_INVALID_OUTPUT). An LF stream with a local palette or
 * Squeeze returns JXG_ERR_UNSUPPORTED (local RCT is decoded); an unknown format JXG_ERR_ARGUMENT. A refused thumbnail
 * leaves the batch as it was. jxg_modular_batch_read_planes refuses a thumbnail frame (JXG_ERR_ARGUMENT). */
int jxg_modular_batch_add_lf(void* batch, void* parsed, uint32_t output_format, void* out, size_t out_row_stride,
                             int out_is_device);

/* ---- Prefix decode of VarDCT frames (a partly received file) ---------------------------------------------------
 * The full-resolution picture of a file of which only a prefix has arrived, as the reference renders it when asked to
 * flush (api/inner/process.rs:169 flush_pixels, frame_info.rs:601 do_flush). A section counts when its whole byte range
 * (TOC offset + length, after any TOC permutation) lies in the prefix (frame_info.rs:302-328). HF group g is decoded with
 * passes 0 .. k_g - 1, k_g the longest run of arrived passes from pass 0 (frame_info.rs:548-565): a later pass that has
 * arrived is not used while an earlier one is missing, and the coefficients of the missing passes are zero. A group with
 * k_g = 0 is the frame's LF image (JxgFrameDesc.lf, after smoothing) upsampled 8x by the reference's Upsample8x
 * (frame/decode.rs:51-150 upsample_lf_group; render/stages/upsample.rs): per output pixel a 5x5 convolution whose weights
 * are the file's CustomTransformData.weights8 (default or custom), clamped to the window's min / max, with LF rows
 * mirrored at the image edges and LF columns taken from the group's row buffer as the reference fills it: where that
 * buffer is never written (the right margin of a frame one group wide; the group left of a last group column one LF
 * sample wide) the window reads 0.0. Both kinds of group then go through the full decode's Gaborish, EPF, colour
 * conversion, store and orientation.
 *
 * jxg_parse_file_prefix takes a bare codestream cut anywhere after HfGlobal; LfGlobal, every LF group and HfGlobal must be
 * whole (JXG_ERR_OUT_OF_BOUNDS otherwise: a shorter prefix has only the thumbnail, jxg_lf_parse_file). A container must
 * be whole, and so must the section of a one-section frame (one group, one pass). The handle is an ordinary parsed frame
 * for jxg_batch_add_parsed, jxg_batch_add_parsed_region, jxg_batch_read_coeffs, jxg_batch_read_xyb and jxg_parsed_free;
 * info.hf_bytes counts the bytes of the HF sections the decode uses. A complete prefix decodes exactly as
 * jxg_parse_file + jxg_batch_add_parsed, with the same kernels. jxg_parsed_desc and jxg_parsed_region_desc refuse a prefix frame with JXG_ERR_ARGUMENT (a descriptor
 * has no per-group pass counts). A decode error in a section it uses is reported by jxg_batch_wait as for a whole frame.
 *
 * A region of a prefix frame (jxg_batch_add_parsed_region): its pixels are the whole prefix decode's pixels
 * (jxg_batch_add_parsed of the same handle) on that rectangle, byte-identical under the alignment rule of region
 * decode above. The region takes the groups a region of the whole file takes, each with its k_g; only its groups with
 * k_g > 0 are entropy-decoded, and its groups with k_g = 0 are upsampled in the coordinates of the whole frame, from the
 * region's LF blocks and 2 LF samples around them (clipped to the image): rows mirror at the frame's LF edges and the
 * two 0.0 margins above fall where they fall in the whole frame. When every group of the region has all passes, the
 * region is decoded exactly as a region of the whole file, with the same kernels. jxg_batch_wait reports the group
 * index of the whole frame. Region checks and codes are those of region decode. */
int jxg_parse_file_prefix(const uint8_t* data, size_t size, void** parsed, JxgImageInfo* info);
/* k_g of each HF group of a frame of jxg_parse_file_prefix, out[0 .. num_groups). JXG_ERR_ARGUMENT for another frame or
 * when n < the frame's group count. */
int jxg_parsed_group_passes(void* parsed, uint8_t* out, uint32_t n);
/* Parity tap, no device needed: the groups a region of a frame of jxg_parse_file_prefix decodes, as
 * jxg_batch_add_parsed_region computes them. groups: their whole-frame indices in sub-frame order (row by row of the
 * rectangle of groups); passes: their k_g; lf_window: the rectangle of the frame's LF image (x0, y0, x1, y1 in LF
 * samples, half-open) uploaded for the upsampling, all zero when no group of the region has k_g = 0. *n_groups is always
 * written; groups and passes may be NULL (only the count), otherwise max_groups must be at least *n_groups, and
 * lf_window may be NULL. JXG_ERR_ARGUMENT for another frame and for a region a whole-file region refuses. */
int jxg_parsed_prefix_region_plan(void* parsed, const JxgRegion* region, uint32_t* groups, uint8_t* passes,
                                  uint32_t max_groups, uint32_t* n_groups, uint32_t lf_window[4]);

const char* jxg_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* JXG_H_ */
