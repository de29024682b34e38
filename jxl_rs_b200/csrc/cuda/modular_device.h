// Device-visible layout of a Modular-frame batch (see modular_kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "device_types.h"  // CodeDev

namespace jxgpu {

struct MStreamDev {  // one ModularHF(group) section
  uint32_t frame, group;
  uint64_t sec_off;  // byte offset of the 8-byte aligned section copy in the blob
  uint32_t sec_len;
  uint32_t data_bitpos;  // first entropy-coded bit
  uint64_t tree_off;     // int4[] nodes: {property | -1, splitval | offset, left child | predictor + (ctx << 4), multiplier}
  uint32_t code;
  uint32_t stream_id;
  uint32_t first_rect, num_rects;
  uint32_t uses_wp;
  uint32_t wp_params[11];   // p1c, p2c, p3ca..p3ce, w[4]
  uint64_t wp_scratch_off;  // bytes into wp_scratch
  uint32_t first_rct, num_rct;
  // LZ77 streams: the widest channel of the stream (the distance multiplier, bitstream.rs:193-202) and the element
  // offset of the stream's window (min(2^20, pixels) u32 entries) in MBatchDev::lz_window
  uint32_t dist_multiplier;
  uint64_t lz_window_off;
};

// Channel walk. The decisions of the MA tree on the channel index and the stream id are constant for a channel; when
// what is left of the tree splits on ONE property (or is a single leaf) the host turns it into a table over that
// property's value clamped to [-1024, 1023] - the device form of the reference's single-property specialisations
// (frame/modular/decode/specialized_trees.rs:197-372: make_lut, GradientOnly, WpOnly, SingleGradientOnly), widened to any
// of the per-pixel properties 2..15 and to arbitrary leaves.
constexpr uint32_t kWalkGeneric = 0, kWalkLut = 1;
constexpr uint32_t kLutNoProperty = 0xff;   // single leaf: `lut_off` holds the entry itself
constexpr int32_t kLutMin = -1024, kLutSize = 2048;
// Table entry: predictor | cluster << 4 | plain << 12 | leaf node index << 16 (plain: offset 0, multiplier 1).

struct MRectDev {
  uint64_t base;  // element index of the rect origin in the plane arena
  uint32_t stride, w, h;
  uint32_t ref_first;  // into MBatchDev::refs: rects usable as reference channels (same shape, nearest first)
  uint32_t ref_count;
  uint32_t walk;       // kWalkGeneric | kWalkLut | property << 8
  uint64_t lut_off;    // blob offset of u32[kLutSize] (kWalkLut with a property), or the single entry itself
};

struct MRctDev {
  uint32_t begin, type;
};

// One global transform / store job. A buffer's pixel (x, y) is planes[a + y * sa + x] (b, c alike): a is the element
// index of the buffer's pixel (0, 0), outside the arena when the buffer's arena rectangle does not start there (a region
// frame); only pixels inside that rectangle are touched. The job's rectangle [x0, x1) x [y0, y1), in the coordinates
// of the buffers it writes, is the whole frame's planes for a whole frame (see each kernel).
struct MJobDev {
  int64_t a, b, c;
  uint32_t sa, sb, sc;
  uint32_t x0, y0, x1, y1;
  uint32_t w, h, rw, op;
  void* out;
  uint64_t out_stride;
  uint32_t out_x, out_y;  // store: display coordinates of the output's top-left pixel
  uint64_t params;        // thumbnail and XYB store jobs: blob offset of their MLfDequantDev / MLfFrameDev
};

// Thumbnail jobs (kJobLf*): the LF image is three planes of w x h samples with row stride sa; a plane set at element
// index a holds X, Y, B (f32) or, as the dequantisation's input, Y, X, B (i32) at a, a + sa * h, a + 2 * sa * h.
struct MLfDequantDev {  // one LF stream: dequant_lf_rect's factors for its extra_precision (frame.h lf_dequant_factors)
  float fac[3], cfl_x, cfl_b;
};
// One thumbnail, or one XYB Modular frame: the output stage (output_stage.h, set_output_colour) and lf_factors, the
// thumbnail's smoothing divisors or the Modular frame's LfQuantFactors (X, Y, B).
struct MLfFrameDev {
  float lf_factors[3];
  float opsin[9], bias_cbrt[3], scaled_bias[3], intensity_scale;
  uint32_t output_tf, output_format;
  float tf_gamma, tf_lum[3], tf_hlg_exp, tf_pq_mul;
};

struct MBatchDev {
  const uint8_t* blob;
  const MStreamDev* streams;
  const uint32_t* order;        // stream indices, longest section first
  const uint32_t* rct_streams;  // streams with local RCTs
  const MRectDev* rects;
  const CodeDev* codes;
  const MRctDev* rcts;
  const uint32_t* refs;  // rect indices, see MRectDev::ref_first
  int32_t* planes;
  uint8_t* wp_scratch;
  int32_t* status;
  uint32_t* queue;
  uint32_t num_streams;
  uint32_t* lz_window;  // symbol windows of the LZ77 streams
};

// The first num_plain entries of B.order are streams without LZ77, the remaining B.num_streams - num_plain use it: each
// group is decoded by its own launch of k_modular_decode (B.queue[0] / B.queue[1]), then the local RCTs run. `sms`: the SMs
// the grids are sized for (schedule_sms, batch_common.h): the decode grid is capped at 8 CTAs per SM, the grid-stride
// job grids at 16.
int launch_modular_decode(const MBatchDev& B, uint32_t num_plain, uint32_t lanes_per_warp, uint32_t num_rct_streams,
                          uint32_t sms, cudaStream_t stream);
// kind: a jxg::ModularJobKind (host/modular_frame.h): 0 RCT, 1 horizontal unsqueeze, 2 vertical unsqueeze, 3 store,
// 4 palette look-up, 5-7 the thumbnail jobs, 8 the XYB store. max_w / max_h: the largest x1 - x0 / y1 - y0 of the jobs. blob: the device
// copy of the staging blob (the thumbnail jobs' parameters).
void launch_modular_jobs(int kind, const MJobDev* jobs, uint32_t num_jobs, uint32_t max_w, uint32_t max_h, int32_t* planes,
                         const uint8_t* blob, uint32_t sms, cudaStream_t stream);

}  // namespace jxgpu
