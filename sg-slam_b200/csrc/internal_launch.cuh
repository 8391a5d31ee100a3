// internal_launch.cuh -- launchers one translation unit of libsgs_cuda.so offers another; not part of the C ABI (hidden symbols).
#pragma once
#include <cuda_runtime.h>

#include <vector>

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
// The arguments of fm_launch (device pointers; fill from FmArgs{} so that what is left out is NULL).  Frame f's pairs: current points
// kps[f * cap + i] (or cur[f * cap + i] when kps is NULL), previous points prev[f * cap + i], i < counts[f] (every frame has cap pairs when
// counts is NULL).
struct FmArgs {
    const sgs_keypoint* kps; const float2* cur; const float2* prev; const int32_t* counts; int cap, nframes;
    // the previous frames' person boxes [.][max_boxes], their number and the potential-dynamic flag (prev_have_dyn NULL: no pair is filtered)
    const sgs_rect* prev_boxes; const int32_t* prev_nboxes; const uint8_t* prev_have_dyn; int max_boxes;
    // At most one of the two.  prev_index[f]: the row holding frame f's previous boxes and flag, == f for a frame without a previous frame.
    // no_prev[f] != 0: frame f has no previous frame; its previous boxes and flag are in row f.  With neither, every frame has a previous frame, read from row f.
    const int32_t* prev_index; const uint8_t* no_prev;
    double thresh, confidence; int max_iters;
    double* F; int32_t* info; uint8_t* mask;     // [nframes][9], [nframes][4] (may be NULL), [nframes][cap] (may be NULL)
};
// sgs_fundamental_batch_device's launch
int fm_launch(const FmArgs& a, cudaStream_t st);

// ---- kfdb.cu
// sgs_kfdb_reloc_candidates_device in two halves, so that a caller can refuse the call before it enqueues anything of its own.  The checks on the
// host: map[f] == -1 skips row f, the other rows name distinct known maps (SGS_ERR_INVALID) of at most 16384 key frames (SGS_ERR_UNSUPPORTED); rows
// receives (row, group offset, group length, map) of every queried row, *max_len the largest group.
int kfdb_plan_query(const sgs_kfdb* db, const char* fn, int nframes, const int32_t* map, std::vector<int4>& rows, int* max_len);
int kfdb_launch_query(sgs_kfdb* db, const char* fn, const std::vector<int4>& rows, int max_len, const int32_t* d_bow_word, const double* d_bow_value,
                      const int32_t* d_bow_n, int bow_cap, const int32_t* d_covis, int32_t* d_cand, int cand_cap, int32_t* d_ncand, int32_t* d_stats,
                      cudaStream_t st);

}  // namespace sgs
