// Host-side entry points into kernels.cu.
#pragma once
#include <cuda_runtime.h>

#include "device_types.h"

namespace jxgpu {
// Streaming multiprocessors of the current device (132 on an H100 SXM). The schedules read it through
// schedule_sms (batch_common.h), which a context's SM budget overrides.
int sm_count();
cudaError_t upload_constants(const float* wc, const float* rdct_scale);
cudaError_t configure_kernels();
// Enqueues the K1..K2 part of the pipeline on `stream`: block plan, entropy kernels, transform kernels; returns the
// number of kernel launches.
// debug_stop 1 stops after the entropy kernels, 2 after the transforms (as 0 does: the caller launches the filters).
// lean_*: the k_entropy_lean schedule (batch.cc schedule_lean); fast_S: streams per warp of k_entropy_fast (1, 2, 4, 8).
int launch_pipeline(const BatchDev& B, cudaStream_t stream, int debug_stop, cudaEvent_t* ev, bool lean_all_420,
                    uint32_t lean_S, uint32_t lean_ctas, bool lean_ctx_smem, uint32_t fast_S);
constexpr int kFusedTileW = 64, kFusedTileH = 32;
int launch_filter_range(const BatchDev& B, const uint32_t* fused_prefix, uint32_t tile_begin, uint32_t tile_count,
                        uint32_t filter_cfg_mask, cudaStream_t stream);
// Parity tap (jxg_batch_read_coeffs): lists of one frame -> dense [groups][3][65536] i32 (zeroed by the caller).
void launch_expand_coeffs(const BatchDev& B, uint32_t frame, uint32_t num_groups, int32_t* dense, cudaStream_t stream);
// Orientation post-pass of one frame: coded w x h image at `src` (row stride src_stride) -> display orientation at `dst`.
void launch_orient(const void* src, size_t src_stride, void* dst, size_t dst_stride, uint32_t w, uint32_t h, uint32_t bpp,
                   uint32_t orientation, cudaStream_t stream);
constexpr int kNumStages = 8;  // memset, entropy, dequant_idct, gaborish, epf0, epf1, epf2, xyb_store
}  // namespace jxgpu
