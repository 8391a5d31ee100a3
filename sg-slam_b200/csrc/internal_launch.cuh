// internal_launch.cuh -- launchers one translation unit of libsgs_cuda.so offers another; not part of the C ABI (hidden symbols).
#pragma once
#include <cuda_runtime.h>

#include "sgs_common.h"

namespace sgs {

// ---- lk_kernel.cu
// The padded pyramid levels of the current images of the last LK call: level l of frame f starts at I + off[l] + f * frame_bytes[l] (its
// border included; frame_bytes[l] is a multiple of 16).  A buffer of `bytes` bytes addressed the same way holds max_batch frames of every level.
struct LkPyramid {
    const uint8_t* I;
    size_t bytes;
    int max_level;
    int64_t off[4], frame_bytes[4];
};
LkPyramid lk_pyramid(const sgs_lk* k);
// sgs_lk_track_batch_device with the previous images read from d_store (laid out as lk_pyramid describes): frame f tracks into row d_row[f] of the
// store, or into its own image when d_row[f] < 0.  The current images' pyramid is built as usual.
int lk_track_from_store(sgs_lk* k, const uint8_t* d_cur, int nframes, size_t frame_stride, int pitch, const sgs_keypoint* d_kps, const int32_t* d_counts,
                        int cap, const uint8_t* d_store, const int32_t* d_row, float* d_prev_xy, cudaStream_t st);

// ---- fundamental.cu
// sgs_fundamental_batch_device's launch.  d_no_prev (may be NULL): d_no_prev[f] != 0 marks a frame without a previous frame (status 3), in place of
// d_prev_index[f] == f; the previous boxes and flag are then read from row f.
int fm_launch(const sgs_keypoint* d_kps, const float2* d_cur, const float2* d_prev, const int32_t* d_counts, int cap, int nframes,
              const sgs_rect* d_boxes, const int32_t* d_nboxes, const uint8_t* d_have_dyn, int max_boxes, const int32_t* d_prev_index,
              const uint8_t* d_no_prev, double thresh, double confidence, int max_iters, double* d_F, int32_t* d_info, uint8_t* d_mask, cudaStream_t st);

}  // namespace sgs
