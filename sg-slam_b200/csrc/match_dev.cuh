// match_dev.cuh -- argument blocks of the batched projection matchers (match.cu).  All pointers are DEVICE pointers;
// per-frame arrays are laid out [nframes][cap] with the given capacities.
#pragma once
#include <cuda_runtime.h>

#include "match_rules.cuh"
#include "sgs_common.h"

namespace sgs {

struct MatchCam {                 // Frame statics (src/Frame.cc:176-196) + the extractor's scale factors
    float min_x, min_y, max_x, max_y;
    float fx, fy, cx, cy, bf;
    int32_t nlevels;
    float scale[kMaxLevels];
};

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
    MatchCam cam;
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

struct LocalMapArgs {
    MatchCam cam;
    const sgs_keypoint* cur_kps; const uint8_t* cur_desc; const float* cur_uright; const int32_t* cur_n;
    int32_t cur_cap;
    const uint8_t* mp_inview; const float* proj_x; const float* proj_y; const float* proj_xr; const int32_t* level;
    const float* view_cos; const uint8_t* mp_desc; const uint8_t* mp_obs; const int32_t* mp_n; int32_t mp_cap;
    float th, nnratio; int32_t id_base;
    int32_t* f_mp; uint8_t* f_mp_obs; int32_t* nmatches; unsigned long long* ncand;
    LocalPre* pre;
};

struct FuseArgs {                 // search half of ORBmatcher::Fuse(KeyFrame*, vpMapPoints, th), src/ORBmatcher.cc:829-980
    MatchCam cam;
    const sgs_keypoint* kf_kps; const uint8_t* kf_desc; const float* kf_uright; const int32_t* kf_n; int32_t kf_cap;
    const float* tcw; const float* ow;            // [nframes][16], [nframes][3]
    const float* mp_xyz; const float* mp_normal; const float* mp_min_dist; const float* mp_max_dist; const uint8_t* mp_desc; const uint8_t* mp_valid;
    const int32_t* mp_n; int32_t mp_cap;
    float th, log_sf; float inv_sigma2[kMaxLevels];
    const float* xform2;          // [nframes][12]: sR21 (3x3 row major) + t21, variant 2 only
    int32_t sim3_variant;         // 2: one direction of SearchBySim3 (:1106-1330): second transform xform2, distance |p3Dc2|, no viewing-angle test;
                                  // 1: Fuse(KeyFrame*, Scw, ...) (:982-1104): pose already decomposed by the caller, invz = 1.0 / z in double, no chi-square gates
                                  // 3: SearchByProjection(KeyFrame*, Scw, ...) (:292-405): as 1 with invz = 1 / z in float; occupied features are skipped and claimed in point order
    int32_t* best_idx; int32_t* best_dist;
    int32_t* kf_matched; int32_t* nmatches;   // variant 3 (SearchByProjection(KeyFrame*, Scw, vpPoints, vpMatched, th), :292-405): vpMatched in/out [nframes][kf_cap], matches per frame
};

struct InitArgs {                 // ORBmatcher::SearchForInitialization(F1, F2, vbPrevMatched, vnMatches12, windowSize), src/ORBmatcher.cc:407-522
    MatchCam cam;                 // image bounds of F2 (its feature grid)
    const sgs_keypoint* f1_kps; const uint8_t* f1_desc; const int32_t* f1_n; int32_t f1_cap;
    const sgs_keypoint* f2_kps; const uint8_t* f2_desc; const int32_t* f2_n; int32_t f2_cap;
    float* prev_xy;               // in/out [nframes][f1_cap][2]
    int32_t window; float nnratio; int32_t check_ori;
    int32_t* match12; int32_t* nmatches;
};

// one block per frame of the matcher that takes these arguments; SGS_ERR_UNSUPPORTED when its frame grid does not fit in shared memory
int launch_matcher(const LastFrameArgs& A, int nframes, cudaStream_t st);
int launch_matcher(const LocalMapArgs& A, int nframes, cudaStream_t st);
int launch_matcher(const FuseArgs& A, int nframes, cudaStream_t st);
int launch_matcher(const InitArgs& A, int nframes, cudaStream_t st);

}  // namespace sgs
