// Device-visible layout of a Modular-frame batch (see modular_kernels.cu).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace jxgpu {

struct MCodeDev {  // one EntropyCode (decode.rs:36-58), tables in the blob
  uint32_t use_prefix, log_alpha, num_clusters, pad;
  uint64_t cmap_off;         // u8[num_contexts]
  uint64_t cfg_off;          // u32[num_clusters], packed as HybridUint::packed()
  uint64_t ans_off;          // u64[num_clusters << log_alpha] alias buckets (ans.rs:31-39)
  uint64_t huff_off;         // u32[] bits | value << 16
  uint64_t huff_offset_off;  // u32[num_clusters]
  // LZ77 (decode.rs:36-45): tokens >= lz_min_symbol start a copy of hybrid(lz_len_cfg) + lz_min_length symbols, whose
  // distance is read from cluster lz_dist_cluster
  uint32_t lz_enabled, lz_min_symbol, lz_min_length, lz_len_cfg, lz_dist_cluster, lz_pad;
};

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

struct MJobDev {  // one global transform / store job (element offsets into the plane arena)
  uint64_t a, b, c;
  uint32_t w, h, rw, op;
  void* out;
  uint64_t out_stride;
};

struct MBatchDev {
  const uint8_t* blob;
  const MStreamDev* streams;
  const uint32_t* order;        // stream indices, longest section first
  const uint32_t* rct_streams;  // streams with local RCTs
  const MRectDev* rects;
  const MCodeDev* codes;
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
// group is decoded by its own launch of k_modular_decode (B.queue[0] / B.queue[1]), then the local RCTs run.
int launch_modular_decode(const MBatchDev& B, uint32_t num_plain, uint32_t lanes_per_warp, uint32_t num_rct_streams,
                          cudaStream_t stream);
// kind: 0 RCT, 1 horizontal unsqueeze, 2 vertical unsqueeze, 3 store, 4 palette look-up
void launch_modular_jobs(int kind, const MJobDev* jobs, uint32_t num_jobs, uint32_t max_w, uint32_t max_h, int32_t* planes,
                         cudaStream_t stream);

}  // namespace jxgpu
