// match_dev.cuh -- launchers of the batched matchers (match.cu), the last-frame matcher's argument block and the per-point scratch of the
// projection matchers.  The other matchers read their sgs_abi.h batch struct as it is.  All pointers are DEVICE pointers; per-frame arrays
// are laid out [nframes][cap] with the given capacities.
#pragma once
#include <cuda_runtime.h>

#include "match_rules.cuh"
#include "sgs_common.h"

namespace sgs {

constexpr int kTopK = 4;          // candidates kept per map point by the optimistic scan

struct PointPre {                 // phase-2 result of one last-frame point
    uint32_t k[kTopK];            // ascending (dist << 16 | position in the sorted grid array); 0xFFFFFFFF = none
    float u, v, invz, radius;
    int16_t min_level, max_level;
    int16_t valid;
    int16_t ngated;               // candidates that passed every gate except claims (complete list iff <= kTopK)
};

struct LocalPre { uint32_t k[kTopK]; int32_t ngated; };

struct LastFrameArgs {
    sgs_camera cam;
    // current frames
    const sgs_keypoint* cur_kps; const uint8_t* cur_desc; const float* cur_uright; const int32_t* cur_n;
    int32_t cur_cap;
    // last-frame map points
    const float* last_xyz; const uint8_t* last_desc; const uint8_t* last_flags;  // bit0: has map point & !outlier, bit1: Observations()>0
    const int32_t* last_octave; const float* last_angle; const int32_t* last_n; int32_t last_cap;
    const float* tcw_cur; const float* tcw_last;   // [nframes][16]
    float th; int32_t mono, check_ori;
    // KeyFrame variant (SearchByProjection(Frame&, KeyFrame*, sAlreadyFound, th, ORBdist), src/ORBmatcher.cc:1474): window from the predicted
    // scale level, every assigned keypoint blocks, no stereo gate; orb_dist replaces TH_HIGH (100 in the last-frame variant)
    int32_t kf_mode, orb_dist; float log_sf; const float* kf_min_dist; const float* kf_max_dist;
    // in/out
    int32_t* cur_mp; const uint8_t* cur_mp_obs_in; int32_t* nmatches; unsigned long long* ncand;
    const uint8_t* frame_enable;   // optional [nframes]: frames with 0 are left untouched (the wide-window retry of Tracking.cc:927-931 runs on the frames that need it)
    // scratch [nframes][last_cap]
    PointPre* pre; int32_t* events;
};

// one block per frame of the matcher that takes these arguments; SGS_ERR_UNSUPPORTED when its frame grid does not fit in shared memory.
// The local-map matcher takes the capacities and the scratch of its sgs_matcher; the fuse search takes log_sf = logf(cam.scale_factors[1]).
int launch_matcher(const LastFrameArgs& A, int nframes, cudaStream_t st);
int launch_matcher(const sgs_localmap_batch& A, int cur_cap, LocalPre* pre, int mp_cap, int nframes, cudaStream_t st);
int launch_matcher(const sgs_fuse_batch& A, float log_sf, int nframes, cudaStream_t st);
int launch_matcher(const sgs_init_batch& A, int nframes, cudaStream_t st);

}  // namespace sgs
