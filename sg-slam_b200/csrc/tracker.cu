// tracker.cu -- batched front end of the tracking thread's per-frame hot path with HOST buffers at the boundary:
//   sgs_tracker_extract : Frame::ExtractORB (src/Frame.cc:274-280) for a batch of frames; keypoints go back to the host
//                         (LK + findFundamentalMat, src/Frame.cc:445-472, run on the device in sgs_tracker_track_lk and the steps);
//   sgs_tracker_track   : dyn-reject verdicts + ordered compaction (src/Frame.cc:560-604) followed by
//                         ORBmatcher::SearchByProjection(cur, last, th, mono) (src/ORBmatcher.cc:1332-1472, called from
//                         Tracking::TrackWithMotionModel, src/Tracking.cc:924), on the device-resident extraction results.
//   sgs_tracker_step / sgs_tracker_step_rgbd(_device): the whole front end with the detector on its own stream; the RGB-D step starts from the
//                         colour and raw depth frames (grab.cu) and adds UndistortKeyPoints + ComputeStereoFromRGBD (one shared body, enqueue_step).
//   sgs_tracker_step_rgbd_stream(_device): the RGB-D step for live streams, one new frame per stream slot, the previous frames kept in StreamState.
// One H2D of the frames, one H2D of the per-frame track inputs, one D2H of the compacted results + matches.
#include <cuda_runtime.h>

#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

#include "block_compact.cuh"
#include "host_stage.cuh"
#include "internal_launch.cuh"
#include "sgs_common.h"

template <class T> using Child = std::unique_ptr<T, void (*)(T*)>;      // a handle the tracker owns, released by its sgs_*_destroy

// What the RGB-D stream steps keep per stream slot (0 .. max_batch-1) between calls -- the reference's file-scope imGrayPre,
// bPreFrameHavePotentialDynamicObj and vPreFramePotentialDynamicBorder (src/Frame.cc:27-33) -- and the per-frame arrays of one call.  Allocated on the
// first stream call, apart from every buffer the batch calls write, so that those calls can neither read nor change it.
struct StreamState {
    // per slot: the last frame's padded LK levels (the geometry of sgs_lk's pyramid, LkPyramid), its boxes [max_boxes], nboxes, flag, and
    // bit 0 = the slot holds a frame, bit 1 = that frame was a first frame
    uint8_t* levels = nullptr; sgs_rect* boxes = nullptr; int32_t* nboxes = nullptr; uint8_t* have = nullptr; uint8_t* state = nullptr;
    // per frame of a call: slot, new_stream (host entry point's copies), the LK row (slot, or -1 for a first frame), the first-frame mark, and the previous
    // frame's flag (quirk Q13 applied), nboxes and boxes, gathered for findFundamentalMat
    int32_t* slot = nullptr; uint8_t* new_stream = nullptr; int32_t* row = nullptr; uint8_t* first = nullptr; uint8_t* pre_have = nullptr;
    int32_t* pre_nboxes = nullptr; sgs_rect* pre_boxes = nullptr;
    bool ready = false;
};

struct sgs_tracker {
    explicit sgs_tracker(int dev) : device(dev), res(dev) {}
    int device, max_batch = 0, cap = 0, point_cap = 0, max_boxes = 0, nfeatures = 0;
    sgs::HandleResources res;
    sgs_camera cam{};
    Child<sgs_extractor> ex{nullptr, sgs_extractor_destroy};
    Child<sgs_matcher> mt{nullptr, sgs_matcher_destroy};
    Child<sgs_lk> lk{nullptr, sgs_lk_destroy};
    int width = 0, height = 0;
    int32_t* d_pidx = nullptr;
    double* d_Fgpu = nullptr; int32_t* d_finfo = nullptr;     // findFundamentalMat on the device
    cudaStream_t st = nullptr;
    // the bulk host uploads of every host track call and step run on copy_st beside the kernels, joined by copy_ev before the rejection;
    // copy_st is not ordered after work still pending on `st` from the device entry points
    cudaStream_t copy_st = nullptr; cudaEvent_t copy_ev = nullptr;
    // device inputs of track()
    float* d_prev = nullptr; float* d_uright_in = nullptr; double* d_F = nullptr; sgs_rect* d_boxes = nullptr; int32_t* d_nboxes = nullptr;
    uint8_t* d_have = nullptr;
    float* d_lxyz = nullptr; uint8_t* d_ldesc = nullptr; uint8_t* d_lflags = nullptr; int32_t* d_loct = nullptr; float* d_lang = nullptr;
    int32_t* d_ln = nullptr; float* d_tc = nullptr; float* d_tl = nullptr;
    // device outputs
    sgs_keypoint* d_kps2 = nullptr; uint8_t* d_desc2 = nullptr; int32_t* d_cnt2 = nullptr; uint8_t* d_keep = nullptr; float* d_uright2 = nullptr;
    int32_t* d_mp = nullptr; int32_t* d_nm = nullptr; unsigned long long* d_ncand = nullptr;
    int last_nframes = 0;
    const sgs_keypoint* keys_un = nullptr;      // mvKeysUn of the last track call: d_kps2, or d_kpsun2 after an RGB-D step
    // detector inside the step (sgs_tracker_step / sgs_tracker_detect_device): RGB staging, its own stream, the join events
    uint8_t* d_rgb = nullptr; size_t d_rgb_cap = 0; int32_t* d_det_status = nullptr;
    cudaStream_t det_st = nullptr; cudaEvent_t det_ev = nullptr; cudaEvent_t ex_ev = nullptr;
    cudaEvent_t rgb_ev = nullptr;               // the colour frames of a step are on the device
    // RGB-D steps, sized on first use: raw depth staging (host entry point), float depth, mvKeysUn / mvDepth before and after the compaction
    uint8_t* d_depth_raw = nullptr; size_t d_depth_raw_cap = 0; float* d_depthf = nullptr;
    sgs_keypoint* d_kpsun = nullptr; float* d_dz = nullptr; sgs_keypoint* d_kpsun2 = nullptr; float* d_dz2 = nullptr;
    // sgs_tracker_pose_chain_device: scratch sized on first use for (max_batch, mp_cap)
    int chain_mp_cap = 0;
    Child<sgs_matcher> mt_local{nullptr, sgs_matcher_destroy};
    uint8_t* d_enable = nullptr; int32_t* d_nm2 = nullptr; uint8_t* d_obs = nullptr; uint8_t* d_seen = nullptr; int32_t* d_ninl = nullptr; int32_t* d_nml = nullptr;
    double* d_po_err = nullptr; uint8_t* d_po_level = nullptr;
    uint8_t* d_inview = nullptr; float* d_projx = nullptr; float* d_projy = nullptr; float* d_projxr = nullptr; int32_t* d_level = nullptr; float* d_viewcos = nullptr;
    unsigned long long* d_ncand2 = nullptr;
    // the local-map ids of the outliers the last pose chain's first discard dropped, [max_batch][mp_cap of that call]; sized by the pose chain only, so
    // that a sgs_tracker_refkf_chain_device call reading it as seen_in never reallocates it
    uint8_t* d_mdisc = nullptr; int mdisc_cap = 0;
    // sgs_tracker_refkf_chain_device, sized on first use: the frame's BoW (word, weight, node) and keypoint angles [B][cap], the key frame's valid flags
    // [B][point_cap], the matches [B][cap], per row the counts (keypoints, key-frame features, local-map points; 0 = no work), the BoW nmatches, the
    // run flag and the two poses
    int32_t* d_rk_word = nullptr; double* d_rk_weight = nullptr; int32_t* d_rk_node = nullptr; float* d_rk_ang = nullptr; uint8_t* d_rk_valid = nullptr;
    int32_t* d_rk_mp = nullptr; int32_t* d_rk_n = nullptr; int32_t* d_rk_kfn = nullptr; int32_t* d_rk_mpn = nullptr; int32_t* d_rk_nm = nullptr;
    uint8_t* d_rk_run = nullptr; float* d_rk_T1 = nullptr; float* d_rk_T2 = nullptr;
    // sgs_tracker_reloc_candidates_device, sized on first use: the enabled rows, their keypoint counts (0 = disabled), the per-feature BoW [B][cap] and
    // the frames' BowVectors [B][cap]
    uint8_t* d_rl_en = nullptr; int32_t* d_rl_n = nullptr; int32_t* d_rl_word = nullptr; double* d_rl_weight = nullptr; int32_t* d_rl_node = nullptr;
    int32_t* d_rl_bw = nullptr; double* d_rl_bv = nullptr; int32_t* d_rl_bn = nullptr;
    StreamState ss;                             // the RGB-D stream steps
};

namespace sgs {
constexpr int kCompactThreads = 256;
// ordered compaction of the per-keypoint side arrays (u_right; after an RGB-D step also mvKeysUn and mvDepth, kun_in / dz_in may be NULL) with the
// verdicts of the dyn-reject kernel
__global__ void compact_uright_kernel(const float* __restrict__ ur_in, const uint8_t* __restrict__ keep, const int32_t* __restrict__ n_in,
                                      const int32_t* __restrict__ n_out, int cap, float* __restrict__ ur_out, int32_t* __restrict__ mp,
                                      const sgs_keypoint* __restrict__ kun_in, sgs_keypoint* __restrict__ kun_out, const float* __restrict__ dz_in,
                                      float* __restrict__ dz_out) {
    const int f = blockIdx.x;
    const int n = min(n_in[f], cap);
    const bool restored = n_out[f] == n;   // restore-all (or nothing rejected): identity
    const int64_t base = (int64_t)f * cap;
    int kept = 0;
    for (int i0 = 0; i0 < n; i0 += kCompactThreads) {
        const int i = i0 + threadIdx.x;
        const bool ok = i < n && (restored || keep[base + i]);
        const int slot = block_ordered_slot<kCompactThreads>(ok, kept);
        if (slot >= 0) {
            const int64_t o = base + slot;
            ur_out[o] = ur_in[base + i];
            if (kun_in) { kun_out[o] = kun_in[base + i]; dz_out[o] = dz_in[base + i]; }
        }
    }
    for (int i = threadIdx.x; i < cap; i += kCompactThreads) mp[base + i] = -1;   // Tracking.cc:916 clears mvpMapPoints before the search
}
// ---- glue of sgs_tracker_pose_chain_device (Tracking::TrackWithMotionModel / TrackLocalMap between the matcher and optimiser calls) ----------
// src/Tracking.cc:927-931: fewer than 20 matches -> clear the frame's matches and search again with 2 th
__global__ void chain_retry_kernel(const int32_t* __restrict__ nm, int cap, int32_t* __restrict__ mp, uint8_t* __restrict__ enable, int32_t* __restrict__ stats) {
    const int f = blockIdx.x;
    const bool retry = nm[f] < 20;
    if (threadIdx.x == 0) { enable[f] = retry ? 1 : 0; stats[8 * f] = nm[f]; stats[8 * f + 1] = retry ? 1 : 0; }
    if (retry) for (int i = threadIdx.x; i < cap; i += blockDim.x) mp[(int64_t)f * cap + i] = -1;
}
__global__ void chain_merge_counts_kernel(const uint8_t* __restrict__ enable, const int32_t* __restrict__ nm2, int32_t* __restrict__ nm, int32_t* __restrict__ stats, int nframes) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    if (enable[f]) nm[f] = nm2[f];
    stats[8 * f + 2] = nm[f];
}
// :940-957 discard the outliers of the first PoseOptimization (TrackReferenceKeyFrame: :816-835); SearchLocalPoints' first loop (:1265-1281): every map
// point matched in the frame -- the discarded ones too, their mnLastFrameSeen was set at :951 / :831 -- is marked as seen, bad ones lose their slot
// (flags bit 2 = isBad()).  flags / local_id: [F][point_cap] of the points the ids below point_cap name.  run (NULL = every row): 0 = the row is left
// as it is.  discards (NULL: not kept): the local-map ids of the dropped outliers, for rows with nm >= 20 -- below that TrackWithMotionModel returns at
// :933 before its discard.
__global__ void __launch_bounds__(256) chain_discard_kernel(const int32_t* __restrict__ n_cur, int cap, int point_cap, const uint8_t* __restrict__ last_flags,
                                                            const int32_t* __restrict__ last_local_id, int mp_cap, int32_t* __restrict__ mp, uint8_t* __restrict__ outlier,
                                                            uint8_t* __restrict__ obs, uint8_t* __restrict__ seen, const int32_t* __restrict__ nm, int32_t* __restrict__ stats,
                                                            const uint8_t* __restrict__ run, uint8_t* __restrict__ discards) {
    __shared__ int s_drop, s_map;
    const int f = blockIdx.x;
    if (run && !run[f]) return;
    const int n = min(n_cur[f], cap);
    const bool keep_discards = discards && nm[f] >= 20;
    if (threadIdx.x == 0) { s_drop = 0; s_map = 0; }
    __syncthreads();
    int drop = 0, nmap = 0;
    for (int i = threadIdx.x; i < cap; i += blockDim.x) {
        const int64_t k = (int64_t)f * cap + i;
        int id = i < n ? mp[k] : -1;
        uint8_t ob = 0;
        if (id >= 0) {
            const uint8_t fl = last_flags[(int64_t)f * point_cap + id];
            const int lid = last_local_id ? last_local_id[(int64_t)f * point_cap + id] : -1;
            const bool local = lid >= 0 && lid < mp_cap;
            if (local) seen[(int64_t)f * mp_cap + lid] = 1;
            if (outlier[k]) {
                if (local && keep_discards) discards[(int64_t)f * mp_cap + lid] = 1;
                id = -1; outlier[k] = 0; ++drop;
            } else {
                if (fl & 2) ++nmap;
                if (fl & 4) id = -1;                       // isBad(): removed by SearchLocalPoints, after the counts of TrackWithMotionModel
                else ob = (fl >> 1) & 1;
            }
        }
        if (i < n) mp[k] = id;
        obs[k] = ob;
    }
    atomicAdd(&s_drop, drop); atomicAdd(&s_map, nmap);
    __syncthreads();
    if (threadIdx.x == 0) { stats[8 * f + 3] = nm[f] - s_drop; stats[8 * f + 4] = s_map; }
}
// SearchLocalPoints' second loop (:1286-1300): points seen in this frame (seen, or seen_in: marked before this chain, may be NULL) or bad are skipped
// before isInFrustum; nToMatch
__global__ void __launch_bounds__(256) chain_mask_kernel(const int32_t* __restrict__ mp_n, int mp_cap, const uint8_t* __restrict__ mp_valid, const uint8_t* __restrict__ seen,
                                                         const uint8_t* __restrict__ seen_in, uint8_t* __restrict__ inview, int32_t* __restrict__ stats,
                                                         const uint8_t* __restrict__ run) {
    __shared__ int s_cnt;
    const int f = blockIdx.x;
    if (run && !run[f]) return;
    const int n = min(mp_n[f], mp_cap);
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    int c = 0;
    for (int j = threadIdx.x; j < mp_cap; j += blockDim.x) {
        const int64_t k = (int64_t)f * mp_cap + j;
        const uint8_t v = (j < n && inview[k] && mp_valid[k] && !seen[k] && !(seen_in && seen_in[k])) ? 1 : 0;
        inview[k] = v; c += v;
    }
    atomicAdd(&s_cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) stats[8 * f + 5] = s_cnt;
}
// :982-996 mnMatchesInliers (mbOnlyTracking == false): map point && !outlier && Observations() > 0
__global__ void __launch_bounds__(256) chain_final_kernel(const int32_t* __restrict__ n_cur, int cap, const int32_t* __restrict__ mp, const uint8_t* __restrict__ outlier,
                                                          const uint8_t* __restrict__ obs, const int32_t* __restrict__ nml, int32_t* __restrict__ f_mp, int32_t* __restrict__ stats,
                                                          const uint8_t* __restrict__ run) {
    __shared__ int s_cnt;
    const int f = blockIdx.x;
    if (run && !run[f]) return;
    const int n = min(n_cur[f], cap);
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    int c = 0;
    for (int i = threadIdx.x; i < cap; i += blockDim.x) {
        const int64_t k = (int64_t)f * cap + i;
        const int id = i < n ? mp[k] : -1;
        f_mp[k] = id;
        if (id >= 0 && !outlier[k] && obs[k]) ++c;
    }
    atomicAdd(&s_cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) { stats[8 * f + 6] = nml[f]; stats[8 * f + 7] = s_cnt; }
}
// ---- glue of sgs_tracker_refkf_chain_device (Tracking::TrackReferenceKeyFrame, src/Tracking.cc:796-838) ------------------------------------------
// Per row before ComputeBoW: enabled (frame_enable NULL = all) rows with 0 <= kf_n <= point_cap run; the others get zero counts, so that the BoW
// transform and matcher exit at once.  A running row gets its key-frame features' SearchByBoW validity (map point present && !isBad(), :176-178 of
// src/ORBmatcher.cc) and its keypoint angles (mvKeysUn[i].angle == mvKeys[i].angle); an enabled row with kf_n out of range gets stats[0] = -1.
__global__ void __launch_bounds__(256) refkf_prep_kernel(const uint8_t* __restrict__ enable, const int32_t* __restrict__ n_cur, int cap, const int32_t* __restrict__ kf_n,
                                                         int point_cap, const uint8_t* __restrict__ kf_flags, const sgs_keypoint* __restrict__ kps,
                                                         int32_t* __restrict__ n_out, int32_t* __restrict__ kfn_out, uint8_t* __restrict__ run,
                                                         uint8_t* __restrict__ kf_valid, float* __restrict__ angle, int32_t* __restrict__ stats) {
    const int f = blockIdx.x;
    const bool en = !enable || enable[f];
    const int kn = kf_n[f];
    const bool ok = en && kn >= 0 && kn <= point_cap;
    const int n = ok ? min(n_cur[f], cap) : 0;
    if (threadIdx.x == 0) {
        n_out[f] = n; kfn_out[f] = ok ? kn : 0; run[f] = ok ? 1 : 0;
        if (en && !ok) for (int q = 0; q < 8; ++q) stats[8 * f + q] = q == 0 ? -1 : 0;
    }
    if (!ok) return;
    for (int i = threadIdx.x; i < kn; i += blockDim.x) {
        const uint8_t fl = kf_flags[(int64_t)f * point_cap + i];
        kf_valid[(int64_t)f * point_cap + i] = ((fl & 1) && !(fl & 4)) ? 1 : 0;
    }
    for (int i = threadIdx.x; i < n; i += blockDim.x) angle[(int64_t)f * cap + i] = kps[(int64_t)f * cap + i].angle;
}
// :808-809: fewer than 15 BoW matches stops the row (stats 0..1 written, the rest 0); a row that passes gets its local-map count and cleared outlier flags
// (mvbOutlier of keypoints without a map point stays false).  Rows that do not run get zero counts for the rest of the chain.
__global__ void __launch_bounds__(256) refkf_gate_kernel(const int32_t* __restrict__ nm, const int32_t* __restrict__ mp_n, int cap, int32_t* __restrict__ n_cur,
                                                         int32_t* __restrict__ mpn_out, uint8_t* __restrict__ run, uint8_t* __restrict__ outlier, int32_t* __restrict__ stats) {
    const int f = blockIdx.x;
    const bool en = run[f] != 0;
    const bool pass = en && nm[f] >= 15;
    __syncthreads();                                   // every thread has read run[f] before thread 0 rewrites it
    if (threadIdx.x == 0) {
        mpn_out[f] = pass ? mp_n[f] : 0;
        if (!pass) { n_cur[f] = 0; run[f] = 0; }
        if (en) for (int q = 0; q < 8; ++q) stats[8 * f + q] = q == 0 ? nm[f] : q == 1 ? (pass ? 1 : 0) : 0;
    }
    if (pass) for (int i = threadIdx.x; i < cap; i += blockDim.x) outlier[(int64_t)f * cap + i] = 0;
}
// the poses of the rows that ran: after the first PoseOptimization (:814) and after TrackLocalMap
__global__ void refkf_commit_kernel(const uint8_t* __restrict__ run, const float* __restrict__ T1, const float* __restrict__ T2, float* __restrict__ tcw_refkf,
                                    float* __restrict__ tcw_final) {
    const int f = blockIdx.x, q = threadIdx.x;
    if (!run[f] || q >= 16) return;
    tcw_refkf[16 * f + q] = T1[16 * f + q]; tcw_final[16 * f + q] = T2[16 * f + q];
}
// sgs_tracker_reloc_candidates_device: the keypoints of the enabled rows enter ComputeBoW, the disabled rows get none
__global__ void reloc_counts_kernel(const uint8_t* __restrict__ enable, const int32_t* __restrict__ n_cur, int32_t* __restrict__ n_out, int nframes) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f < nframes) n_out[f] = enable[f] ? n_cur[f] : 0;
}
// ---- the RGB-D stream steps (StreamState) ----------------------------------------------------------------------------------------------------
// Per frame of a call, before LK: a first frame (its slot never held a frame, or new_stream[f]) tracks into its own image and has no previous frame;
// any other frame reads its slot's stored levels, and the flag and boxes its previous frame ended with.  The flag counts as false when that frame was
// itself a first frame: the reference writes it only inside the rejection, which a first frame never runs (src/Frame.cc:154-162, quirk Q13).
__global__ void stream_resolve_kernel(int nframes, const int32_t* __restrict__ slot, const uint8_t* __restrict__ new_stream, const uint8_t* __restrict__ s_state,
                                      const uint8_t* __restrict__ s_have, const int32_t* __restrict__ s_nboxes, const sgs_rect* __restrict__ s_boxes, int max_boxes,
                                      int32_t* __restrict__ row, uint8_t* __restrict__ first, uint8_t* __restrict__ pre_have, int32_t* __restrict__ pre_nboxes,
                                      sgs_rect* __restrict__ pre_boxes) {
    const int f = blockIdx.x * blockDim.x + threadIdx.x;
    if (f >= nframes) return;
    const int s = slot[f];
    const uint8_t st = s_state[s];
    const bool fi = !(st & 1) || (new_stream && new_stream[f]);
    row[f] = fi ? -1 : s;
    first[f] = fi ? 1 : 0;
    pre_have[f] = (!fi && s_have[s] && !(st & 2)) ? 1 : 0;
    pre_nboxes[f] = fi ? 0 : s_nboxes[s];
    if (!fi) for (int b = 0; b < max_boxes; ++b) pre_boxes[(int64_t)f * max_boxes + b] = s_boxes[(int64_t)s * max_boxes + b];
}
// After LK and findFundamentalMat: frame f's padded levels (current-image pyramid, row f), boxes, flag and first-frame mark become the state of slot[f].
// Grid (x, nframes); the levels are copied in 16-byte words.
__global__ void __launch_bounds__(256) stream_commit_kernel(const LkPyramid P, uint8_t* __restrict__ s_levels, const int32_t* __restrict__ slot,
                                                            const uint8_t* __restrict__ first, const sgs_rect* __restrict__ boxes, const int32_t* __restrict__ nboxes,
                                                            const uint8_t* __restrict__ have, int max_boxes, sgs_rect* __restrict__ s_boxes,
                                                            int32_t* __restrict__ s_nboxes, uint8_t* __restrict__ s_have, uint8_t* __restrict__ s_state) {
    const int f = blockIdx.y, s = slot[f];
#pragma unroll
    for (int l = 0; l < 4; ++l) {
        const int64_t n16 = l <= P.max_level ? P.frame_bytes[l] / 16 : 0;
        const uint4* src = reinterpret_cast<const uint4*>(P.I + P.off[l] + (int64_t)f * P.frame_bytes[l]);
        uint4* dst = reinterpret_cast<uint4*>(s_levels + P.off[l] + (int64_t)s * P.frame_bytes[l]);
        for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n16; i += (int64_t)gridDim.x * blockDim.x) dst[i] = src[i];
    }
    if (blockIdx.x == 0) {
        for (int b = threadIdx.x; b < max_boxes; b += blockDim.x) s_boxes[(int64_t)s * max_boxes + b] = boxes[(int64_t)f * max_boxes + b];
        if (threadIdx.x == 0) { s_nboxes[s] = nboxes[f]; s_have[s] = have[f]; s_state[s] = 1 | (first[f] ? 2 : 0); }
    }
}
}  // namespace sgs

using namespace sgs;

namespace {
int bad(const char* fn, const char* why) { set_error("%s: %s", fn, why); return SGS_ERR_INVALID; }

// The argument checks of the entry points: each returns false after set_error("<fn>: ...") on a refusal, which the entry point returns as
// SGS_ERR_INVALID before it enqueues anything.
// nframes in [1, limit] (the frames of the last extract call, or max_batch for the calls that bring their own frames); prev_index [nframes]
// (host, NULL: none to check): each frame's previous frame is a row of the batch
bool frames_ok(const char* fn, int nframes, int limit, const int32_t* prev_index = nullptr) {
    if (nframes < 1 || nframes > limit) { set_error("%s: nframes = %d outside [1,%d]", fn, nframes, limit); return false; }
    for (int f = 0; prev_index && f < nframes; ++f)
        if (prev_index[f] < 0 || prev_index[f] >= nframes) { set_error("%s: prev_index out of range", fn); return false; }
    return true;
}

// nframes in [1, limit]; slot [nframes] (host): distinct stream slots in [0, limit)
bool slots_ok(const char* fn, int nframes, int limit, const int32_t* slot) {
    if (!frames_ok(fn, nframes, limit)) return false;
    std::vector<uint8_t> seen(limit, 0);
    for (int f = 0; f < nframes; ++f) {
        if (slot[f] < 0 || slot[f] >= limit) { set_error("%s: slot[%d] = %d outside [0,%d)", fn, f, slot[f], limit); return false; }
        if (seen[slot[f]]++) { set_error("%s: slot %d appears twice", fn, slot[f]); return false; }
    }
    return true;
}

// colour frames: interleaved 8-bit RGB, byte pitch and frame stride
bool rgb_layout_ok(const sgs_tracker* t, const char* fn, size_t rgb_stride, int rgb_pitch) {
    if (rgb_pitch >= t->width * 3 && rgb_stride >= (size_t)rgb_pitch * t->height) return true;
    set_error("%s: rgb pitch / stride too small", fn);
    return false;
}

// the depth format and layout of the RGB-D steps (byte pitch and frame stride)
bool depth_args_ok(const sgs_tracker* t, const char* fn, const sgs_rgbd_format* fmt, size_t depth_stride, int depth_pitch, const void* depth) {
    const char* why = nullptr;
    const size_t esz = fmt->depth_type == 0 ? 2 : 4;
    if (fmt->depth_type != 0 && fmt->depth_type != 1) why = "depth_type is neither 0 (uint16) nor 1 (float32)";
    else if (!std::isfinite(fmt->depth_map_factor) || !(fmt->depth_map_factor > 0.f)) why = "depth_map_factor is not a finite positive number";
    else if ((size_t)depth_pitch < esz * t->width || depth_stride < (size_t)depth_pitch * t->height) why = "depth pitch / stride too small";
    else if (depth_pitch % esz || depth_stride % esz || (uintptr_t)depth % esz) why = "depth pitch, stride or pointer not a multiple of the element size";
    if (why) set_error("%s: %s", fn, why);
    return why == nullptr;
}

// the extraction results of the last extract call, on the device: keypoints [F][cap], descriptors [F][cap][32], counts [F]
struct Extracted { const sgs_keypoint* kps; const uint8_t* desc; const int32_t* n; int cap; };
Extracted extracted(const sgs_tracker* t) {
    Extracted e{};
    sgs_extractor_results_device(t->ex.get(), &e.kps, &e.desc, &e.n, &e.cap);
    return e;
}

// The eight per-frame arrays SearchByProjection(cur, last) reads about the last frame: [F][point_cap](..) and the poses [F][16], host or device
// pointers (the last_* fields of sgs_posechain_batch and the arguments of the track calls).
struct LastFrame {
    const float* xyz = nullptr; const uint8_t* desc = nullptr; const uint8_t* flags = nullptr; const int32_t* octave = nullptr;
    const float* angle = nullptr; const int32_t* n = nullptr; const float* tcw_cur = nullptr; const float* tcw_last = nullptr;

    bool complete() const { return xyz && desc && flags && octave && angle && n && tcw_cur && tcw_last; }
};
// the tracker's device copies, filled by stage_host_inputs
LastFrame device_last(const sgs_tracker* t) {
    LastFrame l;
    l.xyz = t->d_lxyz; l.desc = t->d_ldesc; l.flags = t->d_lflags; l.octave = t->d_loct; l.angle = t->d_lang; l.n = t->d_ln; l.tcw_cur = t->d_tc; l.tcw_last = t->d_tl;
    return l;
}

// SearchByProjection(cur, last, th, mono) of the tracker's compacted current frame into its cur_mp / nmatches / ncand
sgs_lastframe_batch lastframe_search(const sgs_tracker* t, const LastFrame& l, float th, int mono, int check_orientation) {
    sgs_lastframe_batch a;
    std::memset(&a, 0, sizeof a);
    a.cam = t->cam;
    a.cur_kps = t->keys_un; a.cur_desc = t->d_desc2; a.cur_uright = t->d_uright2; a.cur_n = t->d_cnt2;
    a.last_xyz = l.xyz; a.last_desc = l.desc; a.last_flags = l.flags; a.last_octave = l.octave; a.last_angle = l.angle; a.last_n = l.n;
    a.tcw_cur = l.tcw_cur; a.tcw_last = l.tcw_last; a.th = th; a.mono = mono; a.check_orientation = check_orientation;
    a.cur_mp = t->d_mp; a.nmatches = t->d_nm; a.ncand = (uint64_t*)t->d_ncand;
    return a;
}

// The per-frame inputs of a track call.  NULL: not given -- computed on the device (u_right of an RGB-D step, F), or the tracker's own
// array as it is (boxes).  prev_xy replaces prev_index in sgs_tracker_track, which runs no LK.  slot (stream steps) replaces prev_index: the previous
// frames come from the slots' StreamState; new_stream may be NULL.
struct TrackInputs {
    LastFrame last;
    const float* u_right = nullptr;
    const int32_t* prev_index = nullptr; const float* prev_xy = nullptr; const double* F = nullptr;
    const sgs_rect* boxes = nullptr; const int32_t* nboxes = nullptr; const uint8_t* have_dyn = nullptr;
    const int32_t* slot = nullptr; const uint8_t* new_stream = nullptr;
};

// Host inputs -> the tracker's device arrays.  What LK and the F estimate read goes first, on the tracker's stream; the bulk (u_right, the
// last-frame arrays) goes on the copy stream beside those kernels, and copy_ev marks its end for the wait before the rejection.
int stage_host_inputs(sgs_tracker* t, size_t B, const TrackInputs& in) {
    const size_t K = t->cap, M = t->point_cap;
    auto h2d = [](void* dst, const void* src, size_t bytes, cudaStream_t s) { return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s); };
    const cudaStream_t st = t->st, cs = t->copy_st;
    if (in.prev_index) SGS_CUDA_TRY(h2d(t->d_pidx, in.prev_index, sizeof(int32_t) * B, st));
    if (in.prev_xy) SGS_CUDA_TRY(h2d(t->d_prev, in.prev_xy, B * K * 8, st));
    if (in.F) SGS_CUDA_TRY(h2d(t->d_F, in.F, B * 72, st));
    if (in.boxes) SGS_CUDA_TRY(h2d(t->d_boxes, in.boxes, B * t->max_boxes * sizeof(sgs_rect), st));
    if (in.nboxes) SGS_CUDA_TRY(h2d(t->d_nboxes, in.nboxes, B * 4, st));
    if (in.have_dyn) SGS_CUDA_TRY(h2d(t->d_have, in.have_dyn, B, st));
    if (in.slot) SGS_CUDA_TRY(h2d(t->ss.slot, in.slot, B * 4, st));
    if (in.new_stream) SGS_CUDA_TRY(h2d(t->ss.new_stream, in.new_stream, B, st));
    const LastFrame& l = in.last;
    if (in.u_right) SGS_CUDA_TRY(h2d(t->d_uright_in, in.u_right, B * K * 4, cs));
    SGS_CUDA_TRY(h2d(t->d_lxyz, l.xyz, B * M * 12, cs)); SGS_CUDA_TRY(h2d(t->d_ldesc, l.desc, B * M * 32, cs));
    SGS_CUDA_TRY(h2d(t->d_lflags, l.flags, B * M, cs)); SGS_CUDA_TRY(h2d(t->d_loct, l.octave, B * M * 4, cs)); SGS_CUDA_TRY(h2d(t->d_lang, l.angle, B * M * 4, cs));
    SGS_CUDA_TRY(h2d(t->d_ln, l.n, B * 4, cs)); SGS_CUDA_TRY(h2d(t->d_tc, l.tcw_cur, B * 64, cs)); SGS_CUDA_TRY(h2d(t->d_tl, l.tcw_last, B * 64, cs));
    SGS_CUDA_TRY(cudaEventRecord(t->copy_ev, cs));
    return SGS_OK;
}

// Where a host entry point's results go: the arrays of sgs_tracker_track, then the extras of the steps.  u_right and the extras may be NULL.
struct HostOutputs {
    sgs_keypoint* kps = nullptr; uint8_t* desc = nullptr; float* u_right = nullptr; int32_t* counts = nullptr; int32_t* cur_mp = nullptr;
    int32_t* nmatches = nullptr; sgs_rect* boxes = nullptr; int32_t* nboxes = nullptr; uint8_t* have = nullptr; sgs_keypoint* kps_un = nullptr; float* depth = nullptr;

    bool complete() const { return kps && desc && counts && cur_mp && nmatches; }
};

// the results, device -> host on the tracker's stream, then the one synchronisation of the call
int download_results(sgs_tracker* t, size_t B, const HostOutputs& o) {
    const size_t K = t->cap;
    const cudaStream_t st = t->st;
    auto d2h = [st](void* dst, const void* src, size_t bytes) { return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, st); };
    SGS_CUDA_TRY(d2h(o.kps, t->d_kps2, B * K * sizeof(sgs_keypoint))); SGS_CUDA_TRY(d2h(o.desc, t->d_desc2, B * K * 32)); SGS_CUDA_TRY(d2h(o.counts, t->d_cnt2, B * 4));
    if (o.u_right) SGS_CUDA_TRY(d2h(o.u_right, t->d_uright2, B * K * 4));
    SGS_CUDA_TRY(d2h(o.cur_mp, t->d_mp, B * K * 4)); SGS_CUDA_TRY(d2h(o.nmatches, t->d_nm, B * 4));
    if (o.boxes) SGS_CUDA_TRY(d2h(o.boxes, t->d_boxes, B * t->max_boxes * sizeof(sgs_rect)));
    if (o.nboxes) SGS_CUDA_TRY(d2h(o.nboxes, t->d_nboxes, B * 4));
    if (o.have) SGS_CUDA_TRY(d2h(o.have, t->d_have, B));
    if (o.kps_un) SGS_CUDA_TRY(d2h(o.kps_un, t->d_kpsun2, B * K * sizeof(sgs_keypoint)));
    if (o.depth) SGS_CUDA_TRY(d2h(o.depth, t->d_dz2, B * K * 4));
    SGS_CUDA_TRY(cudaStreamSynchronize(st));
    return SGS_OK;
}

// dyn-reject + compaction + SearchByProjection(cur, last) on `st` (body of sgs_tracker_track_device).  kun / dz (RGB-D step, else NULL): mvKeysUn and
// mvDepth of the extracted keypoints, compacted beside them; the search then runs on the compacted mvKeysUn.
int enqueue_track(sgs_tracker* t, int nframes, const float* prev_xy, const float* u_right, const double* F, const sgs_rect* boxes, const int32_t* nboxes,
                  const uint8_t* have_dyn, const LastFrame& last, float th, int mono, int check_orientation, const sgs_keypoint* kun, const float* dz,
                  cudaStream_t st) {
    const Extracted ex = extracted(t);
    int rc = sgs_dynreject_batch_device(ex.kps, ex.desc, ex.n, ex.cap, nframes, prev_xy, F, boxes, nboxes, t->max_boxes, have_dyn,
                                        t->nfeatures, t->d_kps2, t->d_desc2, t->d_cnt2, t->d_keep, st);
    if (rc != SGS_OK) return rc;
    compact_uright_kernel<<<nframes, kCompactThreads, 0, st>>>(u_right, t->d_keep, ex.n, t->d_cnt2, ex.cap, t->d_uright2, t->d_mp, kun, t->d_kpsun2, dz, t->d_dz2);
    t->keys_un = kun ? t->d_kpsun2 : t->d_kps2;
    SGS_CUDA_TRY(cudaMemsetAsync(t->d_ncand, 0, (size_t)nframes * 8, st));
    const sgs_lastframe_batch a = lastframe_search(t, last, th, mono, check_orientation);
    return sgs_match_project_lastframe_batch_device(t->mt.get(), &a, nframes, st);
}

// device buffers of the RGB-D steps, sized for max_batch frames on first use (raw_bytes: one raw depth frame, staged by the host entry point)
int ensure_rgbd_buffers(sgs_tracker* t, size_t raw_bytes) {
    HandleResources& R = t->res;
    const size_t B = t->max_batch, K = t->cap, px = (size_t)t->width * t->height;
    if (!t->d_kpsun2) {     // allocated last: a failed first attempt is repeated whole by the next call
        SGS_CUDA_TRY(R.regrow(&t->d_depthf, B * px * 4 + 16)); SGS_CUDA_TRY(R.regrow(&t->d_kpsun, B * K * sizeof(sgs_keypoint) + 16));
        SGS_CUDA_TRY(R.regrow(&t->d_dz, B * K * 4 + 16)); SGS_CUDA_TRY(R.regrow(&t->d_dz2, B * K * 4 + 16)); SGS_CUDA_TRY(R.regrow(&t->d_kpsun2, B * K * sizeof(sgs_keypoint) + 16));
    }
    SGS_CUDA_TRY(R.grow(&t->d_depth_raw, &t->d_depth_raw_cap, raw_bytes * B));
    return SGS_OK;
}

// the StreamState, allocated on the first stream call; every slot starts empty (cleared on `st`, ahead of the call's first read)
int ensure_stream_state(sgs_tracker* t, cudaStream_t st) {
    StreamState& S = t->ss;
    if (S.ready) return SGS_OK;     // set last: a failed first attempt is repeated whole by the next call
    HandleResources& R = t->res;
    const size_t B = t->max_batch, MB = t->max_boxes;
    SGS_CUDA_TRY(R.regrow(&S.levels, lk_pyramid(t->lk.get()).bytes)); SGS_CUDA_TRY(R.regrow(&S.boxes, B * MB * sizeof(sgs_rect) + 16));
    SGS_CUDA_TRY(R.regrow(&S.nboxes, B * 4 + 16)); SGS_CUDA_TRY(R.regrow(&S.have, B + 16)); SGS_CUDA_TRY(R.regrow(&S.state, B + 16));
    SGS_CUDA_TRY(R.regrow(&S.slot, B * 4 + 16)); SGS_CUDA_TRY(R.regrow(&S.new_stream, B + 16)); SGS_CUDA_TRY(R.regrow(&S.row, B * 4 + 16));
    SGS_CUDA_TRY(R.regrow(&S.first, B + 16)); SGS_CUDA_TRY(R.regrow(&S.pre_have, B + 16)); SGS_CUDA_TRY(R.regrow(&S.pre_nboxes, B * 4 + 16));
    SGS_CUDA_TRY(R.regrow(&S.pre_boxes, B * MB * sizeof(sgs_rect) + 16));
    SGS_CUDA_TRY(cudaMemsetAsync(S.state, 0, B, st));
    S.ready = true;
    return SGS_OK;
}

// B host frames of `rows` rows of row_bytes (byte pitch, frame stride) -> dense device frames on `s`: one copy when the host frames are dense too
cudaError_t upload_frames(uint8_t* dst, const void* src, size_t stride, int pitch, size_t row_bytes, int rows, size_t B, cudaStream_t s) {
    if (stride == (size_t)pitch * rows) return cudaMemcpy2DAsync(dst, row_bytes, src, pitch, row_bytes, (size_t)rows * B, cudaMemcpyHostToDevice, s);
    for (size_t f = 0; f < B; ++f)
        if (const cudaError_t e = cudaMemcpy2DAsync(dst + f * row_bytes * rows, row_bytes, (const uint8_t*)src + f * stride, pitch, row_bytes, rows,
                                                    cudaMemcpyHostToDevice, s)) return e;
    return cudaSuccess;
}

// colour frames host -> the tracker's dense staging buffer (pitch width * 3) on the detector stream
int upload_rgb(sgs_tracker* t, const uint8_t* rgb, size_t rgb_stride, int rgb_pitch, size_t B) {
    const size_t row = (size_t)t->width * 3;
    SGS_CUDA_TRY(t->res.grow(&t->d_rgb, &t->d_rgb_cap, row * t->height * t->max_batch));
    SGS_CUDA_TRY(upload_frames(t->d_rgb, rgb, rgb_stride, rgb_pitch, row, t->height, B, t->det_st));
    return SGS_OK;
}

// Where the frames of a step come from.  The colour frames are on the device (ready in the order of rgb_st).  The gray frames either come from host
// memory (sgs_tracker_step) or, with gray == NULL, are converted from the colour frames together with the raw depth (RGB-D steps).
struct StepFrames {
    const uint8_t* d_rgb; size_t rgb_stride; int rgb_pitch; cudaStream_t rgb_st;
    const uint8_t* gray = nullptr; size_t gray_stride = 0; int gray_pitch = 0;
    const void* d_depth = nullptr; size_t depth_stride = 0; int depth_pitch = 0; const sgs_rgbd_format* fmt = nullptr;
};
// the colour frames staged by upload_rgb
StepFrames staged_rgb(const sgs_tracker* t) { return {t->d_rgb, (size_t)t->width * 3 * t->height, t->width * 3, t->det_st}; }

// The stream and event choreography of every step: the detector on its own stream beside extract -> LK on `st`, joined before findFundamentalMat;
// an RGB-D step converts gray and depth on `st` and adds UndistortKeyPoints + ComputeStereoFromRGBD before the rejection.  host_inputs: `in`
// holds host pointers, staged by stage_host_inputs while the kernels run; else device pointers.
int enqueue_step(sgs_tracker* t, sgs_detector* det, const StepFrames& fr, int nframes, const TrackInputs& in, bool host_inputs, float th, int mono,
                 int check_orientation, cudaStream_t st) {
    const size_t B = nframes;
    const bool rgbd = fr.gray == nullptr;
    // ---- detector branch: network on the colour frames, boxes into the tracker's arrays
    if (fr.rgb_st != t->det_st || (rgbd && fr.rgb_st != st)) SGS_CUDA_TRY(cudaEventRecord(t->rgb_ev, fr.rgb_st));
    if (fr.rgb_st != t->det_st) SGS_CUDA_TRY(cudaStreamWaitEvent(t->det_st, t->rgb_ev, 0));
    int rc = sgs_tracker_detect_device(t, det, fr.d_rgb, (int64_t)fr.rgb_stride, fr.rgb_pitch, t->width, t->height, nframes, t->det_st);
    if (rc != SGS_OK) return rc;
    SGS_CUDA_TRY(cudaEventRecord(t->det_ev, t->det_st));
    // ---- tracking branch: gray frames into the extractor's level 0 + ORB extraction, then LK on `st`
    const uint8_t* d_frames; int pitch; size_t fstride;
    sgs_extractor_level0_device(t->ex.get(), &d_frames, &pitch, &fstride);
    const float* depth = nullptr; size_t depth_fstride = 0; int depth_pitch = 0;      // float depth, in elements
    if (!rgbd) {
        rc = sgs_extract_batch(t->ex.get(), fr.gray, nframes, fr.gray_stride, fr.gray_pitch, nullptr, nullptr, 0, nullptr);
        if (rc != SGS_OK) return rc;
        SGS_CUDA_TRY(cudaEventRecord(t->ex_ev, (cudaStream_t)sgs_extractor_stream(t->ex.get())));
        SGS_CUDA_TRY(cudaStreamWaitEvent(st, t->ex_ev, 0));
    } else {
        if (fr.rgb_st != st) SGS_CUDA_TRY(cudaStreamWaitEvent(st, t->rgb_ev, 0));
        const sgs_rgbd_format& fm = *fr.fmt;
        const bool in_place = fm.depth_type == 1 && fm.depth_map_factor == 1.0f;      // Tracking.cc:229-230 converts iff factor != 1 or not CV_32F
        const size_t wpitch = (size_t)t->width * 4;
        rc = sgs_grab_rgbd_batch_device(fr.d_rgb, fr.rgb_stride, fr.rgb_pitch, in_place ? nullptr : fr.d_depth, fr.depth_stride, fr.depth_pitch, &fm, t->width,
                                        t->height, nframes, const_cast<uint8_t*>(d_frames), fstride, pitch, in_place ? nullptr : t->d_depthf,
                                        wpitch * t->height, (int)wpitch, st);
        if (rc != SGS_OK) return rc;
        if (in_place) { depth = (const float*)fr.d_depth; depth_fstride = fr.depth_stride / 4; depth_pitch = fr.depth_pitch / 4; }
        else { depth = t->d_depthf; depth_fstride = (size_t)t->width * t->height; depth_pitch = t->width; }
        rc = sgs_extract_batch_device(t->ex.get(), d_frames, nframes, fstride, pitch, st);
        if (rc != SGS_OK) return rc;
    }
    t->last_nframes = nframes;
    const int32_t* d_pidx = in.prev_index; const int32_t* d_slot = in.slot; const uint8_t* d_new = in.new_stream;
    LastFrame last = in.last;
    if (host_inputs) {
        rc = stage_host_inputs(t, B, in);
        if (rc != SGS_OK) return rc;
        d_pidx = t->d_pidx; last = device_last(t);
        d_slot = t->ss.slot; d_new = in.new_stream ? t->ss.new_stream : nullptr;
    }
    // stream step: each frame's previous frame is the last one its slot received (StreamState), not a row of this batch
    const bool streams = in.slot != nullptr;
    const StreamState& S = t->ss;
    const Extracted ex = extracted(t);
    if (streams) {
        stream_resolve_kernel<<<(nframes + 127) / 128, 128, 0, st>>>(nframes, d_slot, d_new, S.state, S.have, S.nboxes, S.boxes, t->max_boxes, S.row, S.first,
                                                                      S.pre_have, S.pre_nboxes, S.pre_boxes);
        rc = lk_track_from_store(t->lk.get(), d_frames, nframes, fstride, pitch, ex.kps, ex.n, ex.cap, S.levels, S.row, t->d_prev, st);
    } else {
        rc = sgs_tracker_lk_device(t, d_frames, nframes, fstride, pitch, d_pidx, st);
    }
    if (rc != SGS_OK) return rc;
    SGS_CUDA_TRY(cudaStreamWaitEvent(st, t->det_ev, 0));                  // the join of src/Frame.cc:478-481: boxes of every frame of the batch are there
    if (streams) {
        // the parameters of sgs_tracker_fundamental_device; the previous boxes and flag are the gathered ones.  Then LK has read the slots' levels, and
        // the frames become their slots' state.
        FmArgs a{};
        a.kps = ex.kps; a.prev = reinterpret_cast<const float2*>(t->d_prev); a.counts = ex.n; a.cap = ex.cap; a.nframes = nframes;
        a.prev_boxes = S.pre_boxes; a.prev_nboxes = S.pre_nboxes; a.prev_have_dyn = S.pre_have; a.max_boxes = t->max_boxes; a.no_prev = S.first;
        a.thresh = 1.0; a.confidence = 0.99; a.max_iters = 1000; a.F = t->d_Fgpu; a.info = t->d_finfo;
        rc = fm_launch(a, st);
        if (rc != SGS_OK) return rc;
        const LkPyramid P = lk_pyramid(t->lk.get());
        const int gx = (int)std::max<int64_t>(1, (P.frame_bytes[0] / 16 + 2047) / 2048);
        stream_commit_kernel<<<dim3(gx, nframes), 256, 0, st>>>(P, S.levels, d_slot, S.first, t->d_boxes, t->d_nboxes, t->d_have, t->max_boxes, S.boxes,
                                                                S.nboxes, S.have, S.state);
        SGS_CUDA_TRY(cudaGetLastError());
    } else {
        rc = sgs_tracker_fundamental_device(t, nframes, nullptr, nullptr, nullptr, d_pidx, st);
    }
    if (rc != SGS_OK) return rc;
    if (rgbd) {     // Frame.cc:146-174 undistorts and looks the depth up after the rejection; both are per point, so doing them first gives the same values
        rc = sgs_undistort_batch_device(ex.kps, ex.n, ex.cap, nframes, t->cam.fx, t->cam.fy, t->cam.cx, t->cam.cy, fr.fmt->dist_coef, t->d_kpsun, st);
        if (rc != SGS_OK) return rc;
        rc = sgs_stereo_from_depth_batch_device(ex.kps, t->d_kpsun, ex.n, ex.cap, nframes, depth, depth_fstride, depth_pitch, t->cam.bf, t->d_uright_in, t->d_dz, st);
        if (rc != SGS_OK) return rc;
    }
    if (host_inputs) SGS_CUDA_TRY(cudaStreamWaitEvent(st, t->copy_ev, 0));
    return enqueue_track(t, nframes, t->d_prev, t->d_uright_in, t->d_Fgpu, t->d_boxes, t->d_nboxes, t->d_have, last, th, mono, check_orientation,
                         rgbd ? t->d_kpsun : nullptr, rgbd ? t->d_dz : nullptr, st);
}

// the chain scratch of sgs_tracker_pose_chain_device and sgs_tracker_refkf_chain_device, sized for (max_batch, mp_cap) on first use or a larger map
int ensure_chain_scratch(sgs_tracker* t, const char* fn, int mp_cap) {
    if (t->chain_mp_cap >= mp_cap) return SGS_OK;
    const size_t B = t->max_batch, K = t->cap, M = mp_cap;
    t->chain_mp_cap = 0;
    t->mt_local.reset();
    sgs_matcher* mt_local = nullptr;
    const int rc = sgs_matcher_create(t->device, t->max_batch, t->cap, mp_cap, &mt_local);
    t->mt_local.reset(mt_local);
    if (rc != SGS_OK) return rc;
    HandleResources& R = t->res;
    // 16 bytes of slack past the end of every array, as in sgs_tracker_create
    SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_enable, B + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_nm2, B * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_obs, B * K + 16));
    SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_seen, B * M + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_ninl, B * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_nml, B * 4 + 16));
    SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_po_err, B * K * 24 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_po_level, B * K + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_inview, B * M + 16));
    SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_projx, B * M * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_projy, B * M * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_projxr, B * M * 4 + 16));
    SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_level, B * M * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_viewcos, B * M * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_ncand2, B * 8 + 16));
    t->chain_mp_cap = mp_cap;
    return SGS_OK;
}

// The first PoseOptimization of both chains on the tracker's compacted frame: map point of keypoint i = points_xyz[mp[i]] (-1 none), counts n
sgs_poseopt_batch first_optimization(const sgs_tracker* t, const float* tcw_in, const int32_t* n, const int32_t* mp, const float* points_xyz,
                                     const float* inv_level_sigma2, float* tcw_out, uint8_t* outlier) {
    sgs_poseopt_batch po;
    std::memset(&po, 0, sizeof po);
    po.cam = t->cam; po.tcw_in = tcw_in; po.kps = t->keys_un; po.uright = t->d_uright2; po.n = n; po.cap = t->cap;
    po.mp_index = mp; po.points_xyz = points_xyz; po.point_cap = t->point_cap;
    for (int l = 0; l < 16; ++l) po.inv_level_sigma2[l] = inv_level_sigma2[l];
    po.tcw_out = tcw_out; po.outlier = outlier; po.ninliers = t->d_ninl; po.scratch_err = t->d_po_err; po.scratch_level = t->d_po_level;
    return po;
}

// The local map of every frame and the local search's parameters: the mp_* / th_local / nnratio_local fields both chain structs share.  mp_n: [F]
// local-map sizes (0: the row does no work).
struct LocalMap {
    const float* xyz; const float* normal; const float* min_dist; const float* max_dist; const uint8_t* desc; const uint8_t* valid; const uint8_t* obs;
    const int32_t* n; int cap; float th, nnratio;
};
template <class Batch> LocalMap local_map(const Batch* a, const int32_t* mp_n) {
    return {a->mp_xyz, a->mp_normal, a->mp_min_dist, a->mp_max_dist, a->mp_desc, a->mp_valid, a->mp_obs, mp_n, a->mp_cap, a->th_local, a->nnratio_local};
}

// The frame after the first PoseOptimization, as the TrackLocalMap half takes it, and where that half writes.
struct FirstHalf {
    const int32_t* n = nullptr;          // [F] keypoints (0: the row does no work)
    const uint8_t* run = nullptr;        // [F] NULL = every row; 0 = the row's stats and f_mp are not written
    const int32_t* nm = nullptr;         // [F] matches before the discard
    const uint8_t* flags = nullptr; const int32_t* local_id = nullptr;   // [F][point_cap] for the ids below point_cap (local_id may be NULL)
    const uint8_t* seen_in = nullptr;    // [F][mp_cap] may be NULL: local-map points already seen in the frame
    uint8_t* discards = nullptr;         // [F][mp_cap] may be NULL: receives the local-map ids of the dropped outliers (rows with nm >= 20)
    int32_t* mp = nullptr;               // [F][cap] in/out: the matches as ids
    const float* tcw_first = nullptr; float* tcw_final = nullptr; int32_t* f_mp = nullptr; int32_t* stats = nullptr;
};

// Both chains after their first PoseOptimization `po` (its outlier flags are read): discard the outliers, SearchLocalPoints (frustum test with the new pose,
// scale prediction, projection search), the second PoseOptimization, mnMatchesInliers.
int enqueue_local_half(sgs_tracker* t, const LocalMap& lm_in, const FirstHalf& h, sgs_poseopt_batch po, int F, cudaStream_t st) {
    const int cap = t->cap, M = lm_in.cap;
    SGS_CUDA_TRY(cudaMemsetAsync(t->d_seen, 0, (size_t)F * M, st));
    chain_discard_kernel<<<F, 256, 0, st>>>(h.n, cap, t->point_cap, h.flags, h.local_id, M, h.mp, po.outlier, t->d_obs, t->d_seen, h.nm, h.stats, h.run, h.discards);
    sgs_frustum_batch fr;
    std::memset(&fr, 0, sizeof fr);
    fr.cam = t->cam; fr.tcw = h.tcw_first; fr.mp_xyz = lm_in.xyz; fr.mp_normal = lm_in.normal; fr.mp_min_dist = lm_in.min_dist; fr.mp_max_dist = lm_in.max_dist;
    fr.mp_n = lm_in.n; fr.point_cap = M; fr.viewing_cos_limit = 0.5f;
    fr.mp_inview = t->d_inview; fr.proj_x = t->d_projx; fr.proj_y = t->d_projy; fr.proj_xr = t->d_projxr; fr.level = t->d_level; fr.view_cos = t->d_viewcos;
    int rc = sgs_frustum_batch_device(&fr, F, st);
    if (rc != SGS_OK) return rc;
    chain_mask_kernel<<<F, 256, 0, st>>>(lm_in.n, M, lm_in.valid, t->d_seen, h.seen_in, t->d_inview, h.stats, h.run);
    sgs_localmap_batch lm;
    std::memset(&lm, 0, sizeof lm);
    lm.cam = t->cam; lm.cur_kps = t->keys_un; lm.cur_desc = t->d_desc2; lm.cur_uright = t->d_uright2; lm.cur_n = h.n;
    lm.mp_inview = t->d_inview; lm.proj_x = t->d_projx; lm.proj_y = t->d_projy; lm.proj_xr = t->d_projxr; lm.level = t->d_level; lm.view_cos = t->d_viewcos;
    lm.mp_desc = lm_in.desc; lm.mp_obs = lm_in.obs; lm.mp_n = lm_in.n; lm.th = lm_in.th; lm.nnratio = lm_in.nnratio; lm.id_base = t->point_cap;
    lm.f_mp = h.mp; lm.f_mp_obs = t->d_obs; lm.nmatches = t->d_nml; lm.ncand = (uint64_t*)t->d_ncand2;
    rc = sgs_match_project_localmap_batch_device(t->mt_local.get(), &lm, F, st);
    if (rc != SGS_OK) return rc;
    po.tcw_in = h.tcw_first; po.tcw_out = h.tcw_final; po.points2_xyz = lm_in.xyz; po.id_base2 = t->point_cap; po.point2_cap = M;
    rc = sgs_pose_optimization_batch_device(&po, F, st);
    if (rc != SGS_OK) return rc;
    chain_final_kernel<<<F, 256, 0, st>>>(h.n, cap, h.mp, po.outlier, t->d_obs, t->d_nml, h.f_mp, h.stats, h.run);
    SGS_CUDA_TRY(cudaGetLastError());
    return SGS_OK;
}
}  // namespace

extern "C" {

SGS_API void sgs_tracker_destroy(sgs_tracker* t) { delete t; }

SGS_API int sgs_tracker_create(const sgs_orb_params* params, int width, int height, int max_batch, int point_cap, int max_boxes,
                               const sgs_camera* cam, int device, sgs_tracker** out) {
    if (!params || !cam || !out || point_cap < 1 || max_boxes < 0) return bad("sgs_tracker_create", "bad argument");
    *out = nullptr;
    auto t = std::make_unique<sgs_tracker>(device);
    t->max_batch = max_batch; t->point_cap = point_cap; t->max_boxes = max_boxes > 0 ? max_boxes : 1; t->cam = *cam;
    t->nfeatures = params->nfeatures;
    sgs_extractor* ex = nullptr;
    int rc = sgs_extractor_create(params, width, height, max_batch, device, &ex);
    t->ex.reset(ex);
    if (rc != SGS_OK) return rc;
    sgs_extractor_max_keypoints(ex, &t->cap);
    sgs_matcher* mt = nullptr;
    rc = sgs_matcher_create(device, max_batch, t->cap, point_cap, &mt);
    t->mt.reset(mt);
    if (rc != SGS_OK) return rc;
    t->width = width; t->height = height;
    sgs_lk* lk = nullptr;
    rc = sgs_lk_create(width, height, max_batch, device, &lk);
    t->lk.reset(lk);
    if (rc != SGS_OK) return rc;
    HandleResources& R = t->res;
    const char* const fn = "sgs_tracker_create";
    SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_pidx, sizeof(int32_t) * (size_t)max_batch));
    const size_t B = max_batch, K = t->cap, M = point_cap;
    SGS_CUDA_TRY_AT(fn, R.stream(&t->st)); SGS_CUDA_TRY_AT(fn, R.stream(&t->copy_st)); SGS_CUDA_TRY_AT(fn, R.event(&t->copy_ev, cudaEventDisableTiming));
    SGS_CUDA_TRY_AT(fn, R.stream(&t->det_st)); SGS_CUDA_TRY_AT(fn, R.event(&t->det_ev, cudaEventDisableTiming)); SGS_CUDA_TRY_AT(fn, R.event(&t->ex_ev, cudaEventDisableTiming));
    SGS_CUDA_TRY_AT(fn, R.event(&t->rgb_ev, cudaEventDisableTiming));
    // every array below has 16 bytes of slack past its end
    SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_prev, B * K * 8 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_uright_in, B * K * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_F, B * 72 + 16));
    SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_boxes, B * t->max_boxes * sizeof(sgs_rect) + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_nboxes, B * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_have, B + 16));
    SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_lxyz, B * M * 12 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_ldesc, B * M * 32 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_lflags, B * M + 16));
    SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_loct, B * M * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_lang, B * M * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_ln, B * 4 + 16));
    SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_tc, B * 64 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_tl, B * 64 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_kps2, B * K * sizeof(sgs_keypoint) + 16));
    SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_desc2, B * K * 32 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_cnt2, B * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_keep, B * K + 16));
    SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_uright2, B * K * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_mp, B * K * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_nm, B * 4 + 16));
    SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_ncand, B * 8 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_Fgpu, B * 72 + 16)); SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_finfo, B * 16 + 16));
    SGS_CUDA_TRY_AT(fn, R.alloc(&t->d_det_status, B * 4 + 16));
    t->keys_un = t->d_kps2;
    *out = t.release();
    return SGS_OK;
}

SGS_API int sgs_tracker_max_keypoints(const sgs_tracker* t, int* cap) {
    if (!t || !cap) return bad("sgs_tracker_max_keypoints", "NULL");
    *cap = t->cap;
    return SGS_OK;
}

SGS_API int sgs_tracker_extract(sgs_tracker* t, const uint8_t* gray, int nframes, size_t frame_stride, int pitch, sgs_keypoint* kps, uint8_t* desc,
                                int cap, int* n) {
    if (!t) return bad("sgs_tracker_extract", "NULL handle");
    int rc = sgs_extract_batch(t->ex.get(), gray, nframes, frame_stride, pitch, kps, desc, cap, n);
    if (rc == SGS_OK) t->last_nframes = nframes;
    return rc;
}

SGS_API int sgs_tracker_extract_device(sgs_tracker* t, const uint8_t* d_gray, int nframes, size_t frame_stride, int pitch, void* stream) {
    if (!t) return bad("sgs_tracker_extract_device", "NULL handle");
    int rc = sgs_extract_batch_device(t->ex.get(), d_gray, nframes, frame_stride, pitch, stream ? stream : (void*)t->st);
    if (rc == SGS_OK) t->last_nframes = nframes;
    return rc;
}

// all pointers are DEVICE pointers; enqueues dyn-reject + u_right compaction + projection matching on `stream`
SGS_API int sgs_tracker_track_device(sgs_tracker* t, int nframes, const float* prev_xy, const float* u_right, const double* F, const sgs_rect* boxes,
                                     const int32_t* nboxes, const uint8_t* have_dyn, const float* last_xyz, const uint8_t* last_desc,
                                     const uint8_t* last_flags, const int32_t* last_octave, const float* last_angle, const int32_t* last_n,
                                     const float* tcw_cur, const float* tcw_last, float th, int mono, int check_orientation, void* stream) {
    const char* const fn = "sgs_tracker_track_device";
    LastFrame last;
    last.xyz = last_xyz; last.desc = last_desc; last.flags = last_flags; last.octave = last_octave; last.angle = last_angle; last.n = last_n;
    last.tcw_cur = tcw_cur; last.tcw_last = tcw_last;
    if (!t || !last.complete()) return bad(fn, "NULL argument");
    if (!frames_ok(fn, nframes, t->last_nframes)) return SGS_ERR_INVALID;
    // NULL: the tracker's own arrays, filled by sgs_tracker_lk_device (prev_xy), sgs_tracker_stereo_device (u_right), sgs_tracker_fundamental_device
    // (F) and sgs_tracker_detect_device (boxes, nboxes, have_dyn)
    return enqueue_track(t, nframes, prev_xy ? prev_xy : t->d_prev, u_right ? u_right : t->d_uright_in, F ? F : t->d_Fgpu, boxes ? boxes : t->d_boxes,
                         nboxes ? nboxes : t->d_nboxes, have_dyn ? have_dyn : t->d_have, last, th, mono, check_orientation, nullptr, nullptr,
                         stream ? (cudaStream_t)stream : t->st);
}

// device pointers to the results of the last track call: kps [B][cap], desc, u_right, counts [B], cur_mp [B][cap], nmatches [B], ncand [B]
SGS_API int sgs_tracker_results_device(const sgs_tracker* t, const sgs_keypoint** kps, const uint8_t** desc, const float** u_right,
                                       const int32_t** counts, const int32_t** cur_mp, const int32_t** nmatches, const uint64_t** ncand) {
    if (!t) return bad("sgs_tracker_results_device", "NULL handle");
    if (kps) *kps = t->d_kps2;
    if (desc) *desc = t->d_desc2;
    if (u_right) *u_right = t->d_uright2;
    if (counts) *counts = t->d_cnt2;
    if (cur_mp) *cur_mp = t->d_mp;
    if (nmatches) *nmatches = t->d_nm;
    if (ncand) *ncand = (const uint64_t*)t->d_ncand;
    return SGS_OK;
}

SGS_API int sgs_tracker_track(sgs_tracker* t, int nframes, const float* prev_xy, const float* u_right, const double* F, const sgs_rect* boxes,
                              const int32_t* nboxes, const uint8_t* have_dyn, const float* last_xyz, const uint8_t* last_desc,
                              const uint8_t* last_flags, const int32_t* last_octave, const float* last_angle, const int32_t* last_n,
                              const float* tcw_cur, const float* tcw_last, float th, int mono, int check_orientation, sgs_keypoint* kps_out,
                              uint8_t* desc_out, float* u_right_out, int32_t* counts_out, int32_t* cur_mp_out, int32_t* nmatches_out) {
    const char* const fn = "sgs_tracker_track";
    LastFrame last;
    last.xyz = last_xyz; last.desc = last_desc; last.flags = last_flags; last.octave = last_octave; last.angle = last_angle; last.n = last_n;
    last.tcw_cur = tcw_cur; last.tcw_last = tcw_last;
    HostOutputs out;
    out.kps = kps_out; out.desc = desc_out; out.u_right = u_right_out; out.counts = counts_out; out.cur_mp = cur_mp_out; out.nmatches = nmatches_out;
    if (!t || !prev_xy || !u_right || !F || !nboxes || !have_dyn || !last.complete() || !out.complete()) return bad(fn, "NULL argument");
    if (!frames_ok(fn, nframes, t->last_nframes)) return SGS_ERR_INVALID;
    SGS_CUDA_TRY(cudaSetDevice(t->device));
    TrackInputs in{last};
    in.u_right = u_right; in.prev_xy = prev_xy; in.F = F; in.boxes = boxes; in.nboxes = nboxes; in.have_dyn = have_dyn;
    int rc = stage_host_inputs(t, nframes, in);
    if (rc != SGS_OK) return rc;
    SGS_CUDA_TRY(cudaStreamWaitEvent(t->st, t->copy_ev, 0));
    rc = enqueue_track(t, nframes, t->d_prev, t->d_uright_in, t->d_F, t->d_boxes, t->d_nboxes, t->d_have, device_last(t), th, mono, check_orientation,
                       nullptr, nullptr, t->st);
    if (rc != SGS_OK) return rc;
    return download_results(t, nframes, out);
}

SGS_API sgs_extractor* sgs_tracker_extractor(sgs_tracker* t) { return t ? t->ex.get() : nullptr; }
SGS_API sgs_lk* sgs_tracker_lk(sgs_tracker* t) { return t ? t->lk.get() : nullptr; }

SGS_API int sgs_tracker_lk_device(sgs_tracker* t, const uint8_t* d_frames, int nframes, size_t frame_stride, int pitch, const int32_t* d_prev_index,
                                  void* stream) {
    const char* const fn = "sgs_tracker_lk_device";
    if (!t || !d_frames || !d_prev_index) return bad(fn, "NULL argument");
    if (!frames_ok(fn, nframes, t->last_nframes)) return SGS_ERR_INVALID;
    const Extracted ex = extracted(t);
    return sgs_lk_track_batch_device(t->lk.get(), d_frames, nullptr, d_prev_index, nframes, frame_stride, pitch, ex.kps, ex.n, ex.cap, t->d_prev,
                                     stream ? stream : (void*)t->st);
}

SGS_API int sgs_tracker_fundamental_device(sgs_tracker* t, int nframes, const sgs_rect* d_boxes, const int32_t* d_nboxes, const uint8_t* d_have_dyn,
                                           const int32_t* d_prev_index, void* stream) {
    const char* const fn = "sgs_tracker_fundamental_device";
    if (!t || !d_prev_index) return bad(fn, "NULL argument");
    if (!frames_ok(fn, nframes, t->last_nframes)) return SGS_ERR_INVALID;
    const Extracted ex = extracted(t);
    // NULL boxes: the tracker's own arrays, filled by sgs_tracker_detect_device.  Parameters of the reference call: FM_RANSAC, 1.0, 0.99
    // (src/Frame.cc:470,472); OpenCV's default of 1000 iterations
    return sgs_fundamental_batch_device(ex.kps, t->d_prev, ex.n, ex.cap, nframes, d_boxes ? d_boxes : t->d_boxes, d_nboxes ? d_nboxes : t->d_nboxes,
                                        d_have_dyn ? d_have_dyn : t->d_have, t->max_boxes, d_prev_index, 1.0, 0.99, 1000, t->d_Fgpu, t->d_finfo,
                                        stream ? stream : (void*)t->st);
}

SGS_API int sgs_tracker_stereo_device(sgs_tracker* t, int nframes, const float* d_depth, size_t depth_frame_stride, int depth_pitch, void* stream) {
    const char* const fn = "sgs_tracker_stereo_device";
    if (!t || !d_depth) return bad(fn, "NULL argument");
    if (!frames_ok(fn, nframes, t->last_nframes)) return SGS_ERR_INVALID;
    const Extracted ex = extracted(t);
    return sgs_stereo_from_depth_batch_device(ex.kps, nullptr, ex.n, ex.cap, nframes, d_depth, depth_frame_stride, depth_pitch, t->cam.bf, t->d_uright_in, nullptr,
                                              stream ? stream : (void*)t->st);
}

SGS_API int sgs_tracker_fundamental_device_ptr(const sgs_tracker* t, const double** d_F, const int32_t** d_info) {
    if (!t) return bad("sgs_tracker_fundamental_device_ptr", "NULL");
    if (d_F) *d_F = t->d_Fgpu;
    if (d_info) *d_info = t->d_finfo;
    return SGS_OK;
}

SGS_API int sgs_tracker_prev_xy_device(const sgs_tracker* t, const float** d_prev_xy) {
    if (!t || !d_prev_xy) return bad("sgs_tracker_prev_xy_device", "NULL");
    *d_prev_xy = t->d_prev;
    return SGS_OK;
}

SGS_API int sgs_tracker_track_lk(sgs_tracker* t, int nframes, const int32_t* prev_index, const float* u_right, const double* F, const sgs_rect* boxes,
                                 const int32_t* nboxes, const uint8_t* have_dyn, const float* last_xyz, const uint8_t* last_desc,
                                 const uint8_t* last_flags, const int32_t* last_octave, const float* last_angle, const int32_t* last_n,
                                 const float* tcw_cur, const float* tcw_last, float th, int mono, int check_orientation, sgs_keypoint* kps_out,
                                 uint8_t* desc_out, float* u_right_out, int32_t* counts_out, int32_t* cur_mp_out, int32_t* nmatches_out) {
    const char* const fn = "sgs_tracker_track_lk";
    LastFrame last;
    last.xyz = last_xyz; last.desc = last_desc; last.flags = last_flags; last.octave = last_octave; last.angle = last_angle; last.n = last_n;
    last.tcw_cur = tcw_cur; last.tcw_last = tcw_last;
    HostOutputs out;
    out.kps = kps_out; out.desc = desc_out; out.u_right = u_right_out; out.counts = counts_out; out.cur_mp = cur_mp_out; out.nmatches = nmatches_out;
    if (!t || !prev_index || !u_right || !nboxes || !have_dyn || !last.complete() || !out.complete()) return bad(fn, "NULL argument");
    if (!frames_ok(fn, nframes, t->last_nframes, prev_index)) return SGS_ERR_INVALID;
    SGS_CUDA_TRY(cudaSetDevice(t->device));
    TrackInputs in{last};
    in.u_right = u_right; in.prev_index = prev_index; in.F = F; in.boxes = boxes; in.nboxes = nboxes; in.have_dyn = have_dyn;
    int rc = stage_host_inputs(t, nframes, in);
    if (rc != SGS_OK) return rc;
    const uint8_t* d_frames; int pitch; size_t fstride;
    sgs_extractor_level0_device(t->ex.get(), &d_frames, &pitch, &fstride);
    rc = sgs_tracker_lk_device(t, d_frames, nframes, fstride, pitch, t->d_pidx, t->st);
    if (rc != SGS_OK) return rc;
    if (!F) {       // F == NULL: findFundamentalMat on the device, previous-frame boxes = the boxes of row prev_index[f]
        rc = sgs_tracker_fundamental_device(t, nframes, t->d_boxes, t->d_nboxes, t->d_have, t->d_pidx, t->st);
        if (rc != SGS_OK) return rc;
    }
    SGS_CUDA_TRY(cudaStreamWaitEvent(t->st, t->copy_ev, 0));
    rc = enqueue_track(t, nframes, t->d_prev, t->d_uright_in, F ? t->d_F : t->d_Fgpu, t->d_boxes, t->d_nboxes, t->d_have, device_last(t), th, mono,
                       check_orientation, nullptr, nullptr, t->st);
    if (rc != SGS_OK) return rc;
    return download_results(t, nframes, out);
}

SGS_API int sgs_tracker_pose_chain_device(sgs_tracker* t, const sgs_posechain_batch* a, int nframes, void* stream) {
    if (!t || !a) return bad("sgs_tracker_pose_chain_device", "NULL");
    const char* const fn = "sgs_tracker_pose_chain_device";
    LastFrame last;
    last.xyz = a->last_xyz; last.desc = a->last_desc; last.flags = a->last_flags; last.octave = a->last_octave; last.angle = a->last_angle;
    last.n = a->last_n; last.tcw_cur = a->tcw_cur; last.tcw_last = a->tcw_last;
    if (!last.complete() || !a->mp_xyz || !a->mp_normal || !a->mp_min_dist || !a->mp_max_dist || !a->mp_desc || !a->mp_valid || !a->mp_obs || !a->mp_n ||
        !a->tcw_motion || !a->tcw_final || !a->f_mp || !a->outlier || !a->stats)
        return bad(fn, "NULL array");
    if (!frames_ok(fn, nframes, t->last_nframes)) return SGS_ERR_INVALID;
    if (a->mp_cap < 1) return bad(fn, "mp_cap < 1");
    SGS_CUDA_TRY(cudaSetDevice(t->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : t->st;
    int rc = ensure_chain_scratch(t, fn, a->mp_cap);
    if (rc != SGS_OK) return rc;
    if (t->mdisc_cap < a->mp_cap) {
        t->mdisc_cap = 0;
        SGS_CUDA_TRY_AT(fn, t->res.regrow(&t->d_mdisc, (size_t)t->max_batch * a->mp_cap + 16));
        t->mdisc_cap = a->mp_cap;
    }
    const int F = nframes, cap = t->cap;
    // 1. the wide-window retry of the frames with fewer than 20 matches: the search of the track call with 2 th, on those frames, into its own counts
    chain_retry_kernel<<<F, 256, 0, st>>>(t->d_nm, cap, t->d_mp, t->d_enable, a->stats);
    sgs_lastframe_batch lf = lastframe_search(t, last, 2.f * a->th, a->mono, a->check_orientation);
    lf.nmatches = t->d_nm2; lf.ncand = (uint64_t*)t->d_ncand2; lf.frame_enable = t->d_enable;
    SGS_CUDA_TRY(cudaMemsetAsync(t->d_ncand2, 0, (size_t)F * 8, st));
    SGS_CUDA_TRY(cudaMemsetAsync(t->d_nm2, 0, (size_t)F * 4, st));
    rc = sgs_match_project_lastframe_batch_device(t->mt.get(), &lf, F, st);
    if (rc != SGS_OK) return rc;
    chain_merge_counts_kernel<<<(F + 127) / 128, 128, 0, st>>>(t->d_enable, t->d_nm2, t->d_nm, a->stats, F);
    // 2. PoseOptimization on the last-frame matches
    SGS_CUDA_TRY(cudaMemsetAsync(a->outlier, 0, (size_t)F * cap, st));
    sgs_poseopt_batch po = first_optimization(t, a->tcw_cur, t->d_cnt2, t->d_mp, a->last_xyz, a->inv_level_sigma2, a->tcw_motion, a->outlier);
    rc = sgs_pose_optimization_batch_device(&po, F, st);
    if (rc != SGS_OK) return rc;
    // 3-5. discard, SearchLocalPoints, PoseOptimization, inlier count; the discarded outliers' local-map ids are kept for sgs_tracker_motion_discards_device
    SGS_CUDA_TRY(cudaMemsetAsync(t->d_mdisc, 0, (size_t)F * a->mp_cap, st));
    FirstHalf h;
    h.n = t->d_cnt2; h.nm = t->d_nm; h.flags = a->last_flags; h.local_id = a->last_local_id; h.discards = t->d_mdisc; h.mp = t->d_mp;
    h.tcw_first = a->tcw_motion; h.tcw_final = a->tcw_final; h.f_mp = a->f_mp; h.stats = a->stats;
    return enqueue_local_half(t, local_map(a, a->mp_n), h, po, F, st);
}

SGS_API int sgs_tracker_motion_discards_device(const sgs_tracker* t, const uint8_t** d_mask) {
    if (!t || !d_mask) return bad("sgs_tracker_motion_discards_device", "NULL");
    if (!t->d_mdisc) return bad("sgs_tracker_motion_discards_device", "no pose chain has run on this handle");
    *d_mask = t->d_mdisc;
    return SGS_OK;
}

SGS_API int sgs_tracker_refkf_chain_device(sgs_tracker* t, const sgs_vocabulary* voc, const sgs_refkf_batch* a, int nframes, void* stream) {
    const char* const fn = "sgs_tracker_refkf_chain_device";
    if (!t || !voc || !a) return bad(fn, "NULL");
    if (!a->kf_node || !a->kf_weight || !a->kf_desc || !a->kf_angle || !a->kf_xyz || !a->kf_flags || !a->kf_n || !a->tcw_last || !a->mp_xyz || !a->mp_normal ||
        !a->mp_min_dist || !a->mp_max_dist || !a->mp_desc || !a->mp_valid || !a->mp_obs || !a->mp_n || !a->tcw_refkf || !a->tcw_final || !a->f_mp || !a->outlier ||
        !a->stats)
        return bad(fn, "NULL array");
    if (!frames_ok(fn, nframes, t->last_nframes)) return SGS_ERR_INVALID;
    if (a->mp_cap < 1) return bad(fn, "mp_cap < 1");
    if (t->point_cap > 8192 || t->cap > 8192) { set_error("%s: SearchByBoW takes at most 8192 features per side (point_cap %d, cap %d)", fn, t->point_cap, t->cap); return SGS_ERR_UNSUPPORTED; }
    SGS_CUDA_TRY(cudaSetDevice(t->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : t->st;
    int rc = ensure_chain_scratch(t, fn, a->mp_cap);
    if (rc != SGS_OK) return rc;
    if (!t->d_rk_T2) {      // allocated last: a failed first attempt is repeated whole by the next call
        HandleResources& R = t->res;
        const size_t B = t->max_batch, K = t->cap, P = t->point_cap;
        SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rk_word, B * K * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rk_weight, B * K * 8 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rk_node, B * K * 4 + 16));
        SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rk_ang, B * K * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rk_valid, B * P + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rk_mp, B * K * 4 + 16));
        SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rk_n, B * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rk_kfn, B * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rk_mpn, B * 4 + 16));
        SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rk_nm, B * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rk_run, B + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rk_T1, B * 64 + 16));
        SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rk_T2, B * 64 + 16));
    }
    const int F = nframes, cap = t->cap, pc = t->point_cap;
    // 1. Frame::ComputeBoW (:799, levelsup 4) of the running rows
    refkf_prep_kernel<<<F, 256, 0, st>>>(a->frame_enable, t->d_cnt2, cap, a->kf_n, pc, a->kf_flags, t->keys_un, t->d_rk_n, t->d_rk_kfn, t->d_rk_run, t->d_rk_valid,
                                         t->d_rk_ang, a->stats);
    rc = sgs_bow_transform_batch_device(voc, t->d_desc2, t->d_rk_n, cap, F, 4, t->d_rk_word, t->d_rk_weight, t->d_rk_node, st);
    if (rc != SGS_OK) return rc;
    // 2. ORBmatcher(0.7, true).SearchByBoW(mpReferenceKF, mCurrentFrame, vpMapPointMatches) (:803-806)
    sgs_bow_batch bw;
    std::memset(&bw, 0, sizeof bw);
    bw.kf_node = a->kf_node; bw.kf_weight = a->kf_weight; bw.kf_valid = t->d_rk_valid; bw.kf_desc = a->kf_desc; bw.kf_angle = a->kf_angle; bw.kf_n = t->d_rk_kfn;
    bw.kf_cap = pc; bw.f_node = t->d_rk_node; bw.f_weight = t->d_rk_weight; bw.f_desc = t->d_desc2; bw.f_angle = t->d_rk_ang; bw.f_n = t->d_rk_n; bw.f_cap = cap;
    bw.nnratio = 0.7f; bw.check_orientation = 1; bw.match_f = t->d_rk_mp; bw.nmatches = t->d_rk_nm;
    rc = sgs_match_bow_batch_device(&bw, F, st);
    if (rc != SGS_OK) return rc;
    // 3. below 15 matches the row stops (:808-809)
    refkf_gate_kernel<<<F, 256, 0, st>>>(t->d_rk_nm, a->mp_n, cap, t->d_rk_n, t->d_rk_mpn, t->d_rk_run, a->outlier, a->stats);
    // 4. mvpMapPoints = the matches, SetPose(mLastFrame.mTcw), PoseOptimization (:811-814)
    sgs_poseopt_batch po = first_optimization(t, a->tcw_last, t->d_rk_n, t->d_rk_mp, a->kf_xyz, a->inv_level_sigma2, t->d_rk_T1, a->outlier);
    rc = sgs_pose_optimization_batch_device(&po, F, st);
    if (rc != SGS_OK) return rc;
    // 5-6. discard the outliers (:816-835), then TrackLocalMap as in the pose chain, with the seen_in points left out as well
    SGS_CUDA_TRY(cudaMemsetAsync(t->d_ncand2, 0, (size_t)F * 8, st));
    FirstHalf h;
    h.n = t->d_rk_n; h.run = t->d_rk_run; h.nm = t->d_rk_nm; h.flags = a->kf_flags; h.local_id = a->kf_local_id; h.seen_in = a->seen_in; h.mp = t->d_rk_mp;
    h.tcw_first = t->d_rk_T1; h.tcw_final = t->d_rk_T2; h.f_mp = a->f_mp; h.stats = a->stats;
    rc = enqueue_local_half(t, local_map(a, t->d_rk_mpn), h, po, F, st);
    if (rc != SGS_OK) return rc;
    refkf_commit_kernel<<<F, 32, 0, st>>>(t->d_rk_run, t->d_rk_T1, t->d_rk_T2, a->tcw_refkf, a->tcw_final);
    SGS_CUDA_TRY(cudaGetLastError());
    return SGS_OK;
}

SGS_API int sgs_tracker_reloc_candidates_device(sgs_tracker* t, const sgs_vocabulary* voc, sgs_kfdb* db, const sgs_reloc_batch* a, int nframes, void* stream) {
    const char* const fn = "sgs_tracker_reloc_candidates_device";
    if (!t || !voc || !db || !a) return bad(fn, "NULL");
    if (!a->map || !a->covis || !a->cand || !a->ncand || !a->stats || a->cand_cap < 1) return bad(fn, "NULL array or cand_cap < 1");
    if (!frames_ok(fn, nframes, t->last_nframes)) return SGS_ERR_INVALID;
    if (t->cap > 8192) { set_error("%s: the BowVector takes at most 8192 features (cap %d)", fn, t->cap); return SGS_ERR_UNSUPPORTED; }
    std::vector<int32_t> map(a->map, a->map + nframes);
    std::vector<uint8_t> en(nframes, 1);
    for (int f = 0; f < nframes; ++f)
        if (a->frame_enable && !a->frame_enable[f]) { en[f] = 0; map[f] = -1; }
        else if (map[f] < 0) return bad(fn, "an enabled row names no map");
    std::vector<int4> rows;
    int max_len = 0;
    int rc = kfdb_plan_query(db, fn, nframes, map.data(), rows, &max_len);
    if (rc != SGS_OK) return rc;
    SGS_CUDA_TRY(cudaSetDevice(t->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : t->st;
    if (!t->d_rl_bn) {      // allocated last: a failed first attempt is repeated whole by the next call
        HandleResources& R = t->res;
        const size_t B = t->max_batch, K = t->cap;
        SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rl_en, B + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rl_n, B * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rl_word, B * K * 4 + 16));
        SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rl_weight, B * K * 8 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rl_node, B * K * 4 + 16));
        SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rl_bw, B * K * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rl_bv, B * K * 8 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_rl_bn, B * 4 + 16));
    }
    const int F = nframes, cap = t->cap;
    // 1. Frame::ComputeBoW (:1463) of the enabled rows
    SGS_CUDA_TRY_AT(fn, cudaMemcpyAsync(t->d_rl_en, en.data(), (size_t)F, cudaMemcpyHostToDevice, st));
    reloc_counts_kernel<<<(F + 127) / 128, 128, 0, st>>>(t->d_rl_en, t->d_cnt2, t->d_rl_n, F);
    rc = sgs_bow_transform_batch_device(voc, t->d_desc2, t->d_rl_n, cap, F, 4, t->d_rl_word, t->d_rl_weight, t->d_rl_node, st);
    if (rc != SGS_OK) return rc;
    rc = sgs_bow_vector_batch_device(t->d_rl_word, t->d_rl_weight, t->d_rl_n, cap, F, t->d_rl_bw, t->d_rl_bv, t->d_rl_bn, st);
    if (rc != SGS_OK) return rc;
    // 2. mpKeyFrameDB->DetectRelocalizationCandidates(&mCurrentFrame) (:1467)
    return kfdb_launch_query(db, fn, rows, max_len, t->d_rl_bw, t->d_rl_bv, t->d_rl_bn, cap, a->covis, a->cand, a->cand_cap, a->ncand, a->stats, st);
}

// Detector2D::detect for the frames of the batch (src/Tracking.cc:288-307 hands the colour image to the detector thread; src/Frame.cc:478-500
// joins it before the rejection): the person boxes land in the tracker's own box arrays, in the layout the F estimate and the rejection take
// when called with boxes == NULL.  d_rgb: device frames (interleaved 8-bit RGB).  Enqueued on `stream` (NULL: the tracker's detector stream, which
// the next sgs_tracker_fundamental_device / _track_device call on the tracker's stream is NOT ordered after -- use sgs_tracker_step for that).
SGS_API int sgs_tracker_detect_device(sgs_tracker* t, sgs_detector* det, const uint8_t* d_rgb, int64_t frame_stride, int pitch, int width, int height, int nframes,
                                      void* stream) {
    const char* const fn = "sgs_tracker_detect_device";
    if (!t || !det || !d_rgb) return bad(fn, "NULL argument");
    if (!frames_ok(fn, nframes, t->max_batch)) return SGS_ERR_INVALID;
    return sgs_detector_detect_device(det, d_rgb, frame_stride, pitch, width, height, nframes, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, t->d_boxes, t->d_nboxes,
                                      t->d_have, t->max_boxes, t->d_det_status, stream ? stream : (void*)t->det_st);
}
SGS_API int sgs_tracker_boxes_device(const sgs_tracker* t, const sgs_rect** d_boxes, const int32_t** d_nboxes, const uint8_t** d_have_dyn) {
    if (!t) return bad("sgs_tracker_boxes_device", "NULL");
    if (d_boxes) *d_boxes = t->d_boxes;
    if (d_nboxes) *d_nboxes = t->d_nboxes;
    if (d_have_dyn) *d_have_dyn = t->d_have;
    return SGS_OK;
}

// The whole per-frame front end of the tracking thread for a batch of frames, HOST buffers in and out (src/Tracking.cc:203-307 + the Frame
// constructor src/Frame.cc:129-198 + TrackWithMotionModel's matcher call :906-924):
//   colour frames -> detector (own stream)            ------------------\
//   gray frames   -> ORB extract -> LK to the previous frame -> join -> findFundamentalMat -> dyn-reject + compaction -> SearchByProjection(cur, last)
// Uploads run on copy streams beside the kernels; one synchronisation at the end.  boxes_out / nboxes_out / have_out (may be NULL): the
// detector's person boxes for the rejection, as the Frame would hold them.
SGS_API int sgs_tracker_step(sgs_tracker* t, sgs_detector* det, const uint8_t* gray, size_t gray_stride, int gray_pitch, const uint8_t* rgb, size_t rgb_stride,
                             int rgb_pitch, int nframes, const int32_t* prev_index, const float* u_right, const float* last_xyz, const uint8_t* last_desc,
                             const uint8_t* last_flags, const int32_t* last_octave, const float* last_angle, const int32_t* last_n, const float* tcw_cur,
                             const float* tcw_last, float th, int mono, int check_orientation, sgs_keypoint* kps_out, uint8_t* desc_out, float* u_right_out,
                             int32_t* counts_out, int32_t* cur_mp_out, int32_t* nmatches_out, sgs_rect* boxes_out, int32_t* nboxes_out, uint8_t* have_out) {
    const char* const fn = "sgs_tracker_step";
    LastFrame last;
    last.xyz = last_xyz; last.desc = last_desc; last.flags = last_flags; last.octave = last_octave; last.angle = last_angle; last.n = last_n;
    last.tcw_cur = tcw_cur; last.tcw_last = tcw_last;
    HostOutputs out;
    out.kps = kps_out; out.desc = desc_out; out.u_right = u_right_out; out.counts = counts_out; out.cur_mp = cur_mp_out; out.nmatches = nmatches_out;
    out.boxes = boxes_out; out.nboxes = nboxes_out; out.have = have_out;
    if (!t || !det || !gray || !rgb || !prev_index || !u_right || !last.complete() || !out.complete()) return bad(fn, "NULL argument");
    if (!frames_ok(fn, nframes, t->max_batch, prev_index) || !rgb_layout_ok(t, fn, rgb_stride, rgb_pitch)) return SGS_ERR_INVALID;
    SGS_CUDA_TRY(cudaSetDevice(t->device));
    int rc = upload_rgb(t, rgb, rgb_stride, rgb_pitch, nframes);
    if (rc != SGS_OK) return rc;
    StepFrames fr = staged_rgb(t);
    fr.gray = gray; fr.gray_stride = gray_stride; fr.gray_pitch = gray_pitch;
    TrackInputs in{last};
    in.u_right = u_right; in.prev_index = prev_index;
    rc = enqueue_step(t, det, fr, nframes, in, true, th, mono, check_orientation, t->st);
    if (rc != SGS_OK) return rc;
    return download_results(t, nframes, out);
}

// The RGB-D front end (Tracking::GrabImageRGBD + the RGB-D Frame constructor + the first matcher call) on device frames; see sgs_abi.h.
SGS_API int sgs_tracker_step_rgbd_device(sgs_tracker* t, sgs_detector* det, const uint8_t* d_rgb, size_t rgb_stride, int rgb_pitch, const void* d_depth,
                                         size_t depth_stride, int depth_pitch, const sgs_rgbd_format* fmt, int nframes, const int32_t* d_prev_index,
                                         const float* last_xyz, const uint8_t* last_desc, const uint8_t* last_flags, const int32_t* last_octave,
                                         const float* last_angle, const int32_t* last_n, const float* tcw_cur, const float* tcw_last, float th, int mono,
                                         int check_orientation, void* stream) {
    const char* const fn = "sgs_tracker_step_rgbd_device";
    LastFrame last;
    last.xyz = last_xyz; last.desc = last_desc; last.flags = last_flags; last.octave = last_octave; last.angle = last_angle; last.n = last_n;
    last.tcw_cur = tcw_cur; last.tcw_last = tcw_last;
    if (!t || !det || !d_rgb || !d_depth || !fmt || !d_prev_index || !last.complete()) return bad(fn, "NULL argument");
    if (!frames_ok(fn, nframes, t->max_batch) || !rgb_layout_ok(t, fn, rgb_stride, rgb_pitch) ||
        !depth_args_ok(t, fn, fmt, depth_stride, depth_pitch, d_depth)) return SGS_ERR_INVALID;
    SGS_CUDA_TRY(cudaSetDevice(t->device));
    const int rc = ensure_rgbd_buffers(t, 0);
    if (rc != SGS_OK) return rc;
    cudaStream_t st = stream ? (cudaStream_t)stream : t->st;
    StepFrames fr{d_rgb, rgb_stride, rgb_pitch, st};
    fr.d_depth = d_depth; fr.depth_stride = depth_stride; fr.depth_pitch = depth_pitch; fr.fmt = fmt;
    TrackInputs in{last};
    in.prev_index = d_prev_index;
    return enqueue_step(t, det, fr, nframes, in, false, th, mono, check_orientation, st);
}

// The same from host buffers: one upload of the colour frames (detector and gray conversion read it), the raw depth as given, one synchronisation.
SGS_API int sgs_tracker_step_rgbd(sgs_tracker* t, sgs_detector* det, const uint8_t* rgb, size_t rgb_stride, int rgb_pitch, const void* depth,
                                  size_t depth_stride, int depth_pitch, const sgs_rgbd_format* fmt, int nframes, const int32_t* prev_index,
                                  const float* last_xyz, const uint8_t* last_desc, const uint8_t* last_flags, const int32_t* last_octave,
                                  const float* last_angle, const int32_t* last_n, const float* tcw_cur, const float* tcw_last, float th, int mono,
                                  int check_orientation, sgs_keypoint* kps_out, uint8_t* desc_out, float* u_right_out, int32_t* counts_out,
                                  int32_t* cur_mp_out, int32_t* nmatches_out, sgs_rect* boxes_out, int32_t* nboxes_out, uint8_t* have_out,
                                  sgs_keypoint* kps_un_out, float* depth_out) {
    const char* const fn = "sgs_tracker_step_rgbd";
    LastFrame last;
    last.xyz = last_xyz; last.desc = last_desc; last.flags = last_flags; last.octave = last_octave; last.angle = last_angle; last.n = last_n;
    last.tcw_cur = tcw_cur; last.tcw_last = tcw_last;
    HostOutputs out;
    out.kps = kps_out; out.desc = desc_out; out.u_right = u_right_out; out.counts = counts_out; out.cur_mp = cur_mp_out; out.nmatches = nmatches_out;
    out.boxes = boxes_out; out.nboxes = nboxes_out; out.have = have_out; out.kps_un = kps_un_out; out.depth = depth_out;
    if (!t || !det || !rgb || !depth || !fmt || !prev_index || !last.complete() || !out.complete()) return bad(fn, "NULL argument");
    if (!frames_ok(fn, nframes, t->max_batch, prev_index) || !rgb_layout_ok(t, fn, rgb_stride, rgb_pitch) ||
        !depth_args_ok(t, fn, fmt, depth_stride, depth_pitch, depth)) return SGS_ERR_INVALID;
    SGS_CUDA_TRY(cudaSetDevice(t->device));
    const size_t row = (size_t)t->width * (fmt->depth_type == 0 ? 2 : 4);
    int rc = ensure_rgbd_buffers(t, row * t->height);
    if (rc != SGS_OK) return rc;
    rc = upload_rgb(t, rgb, rgb_stride, rgb_pitch, nframes);
    if (rc != SGS_OK) return rc;
    SGS_CUDA_TRY(upload_frames(t->d_depth_raw, depth, depth_stride, depth_pitch, row, t->height, nframes, t->st));
    StepFrames fr = staged_rgb(t);
    fr.d_depth = t->d_depth_raw; fr.depth_stride = row * t->height; fr.depth_pitch = (int)row; fr.fmt = fmt;
    TrackInputs in{last};
    in.prev_index = prev_index;      // no u_right: the step computes it from the depth
    rc = enqueue_step(t, det, fr, nframes, in, true, th, mono, check_orientation, t->st);
    if (rc != SGS_OK) return rc;
    return download_results(t, nframes, out);
}

// The RGB-D step for live streams, one new frame per stream slot: the previous frames are the slots' (StreamState); see sgs_abi.h.
SGS_API int sgs_tracker_step_rgbd_stream_device(sgs_tracker* t, sgs_detector* det, const uint8_t* d_rgb, size_t rgb_stride, int rgb_pitch, const void* d_depth,
                                                size_t depth_stride, int depth_pitch, const sgs_rgbd_format* fmt, int nframes, const int32_t* d_slot,
                                                const uint8_t* d_new_stream, const float* last_xyz, const uint8_t* last_desc, const uint8_t* last_flags,
                                                const int32_t* last_octave, const float* last_angle, const int32_t* last_n, const float* tcw_cur,
                                                const float* tcw_last, float th, int mono, int check_orientation, void* stream) {
    const char* const fn = "sgs_tracker_step_rgbd_stream_device";
    LastFrame last;
    last.xyz = last_xyz; last.desc = last_desc; last.flags = last_flags; last.octave = last_octave; last.angle = last_angle; last.n = last_n;
    last.tcw_cur = tcw_cur; last.tcw_last = tcw_last;
    if (!t || !det || !d_rgb || !d_depth || !fmt || !d_slot || !last.complete()) return bad(fn, "NULL argument");
    if (!frames_ok(fn, nframes, t->max_batch) || !rgb_layout_ok(t, fn, rgb_stride, rgb_pitch) ||
        !depth_args_ok(t, fn, fmt, depth_stride, depth_pitch, d_depth)) return SGS_ERR_INVALID;
    SGS_CUDA_TRY(cudaSetDevice(t->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : t->st;
    int rc = ensure_rgbd_buffers(t, 0);
    if (rc != SGS_OK) return rc;
    rc = ensure_stream_state(t, st);
    if (rc != SGS_OK) return rc;
    StepFrames fr{d_rgb, rgb_stride, rgb_pitch, st};
    fr.d_depth = d_depth; fr.depth_stride = depth_stride; fr.depth_pitch = depth_pitch; fr.fmt = fmt;
    TrackInputs in{last};
    in.slot = d_slot; in.new_stream = d_new_stream;
    return enqueue_step(t, det, fr, nframes, in, false, th, mono, check_orientation, st);
}

// The same from host buffers; the slots are checked (range, duplicates) before anything runs.
SGS_API int sgs_tracker_step_rgbd_stream(sgs_tracker* t, sgs_detector* det, const uint8_t* rgb, size_t rgb_stride, int rgb_pitch, const void* depth,
                                         size_t depth_stride, int depth_pitch, const sgs_rgbd_format* fmt, int nframes, const int32_t* slot,
                                         const uint8_t* new_stream, const float* last_xyz, const uint8_t* last_desc, const uint8_t* last_flags,
                                         const int32_t* last_octave, const float* last_angle, const int32_t* last_n, const float* tcw_cur,
                                         const float* tcw_last, float th, int mono, int check_orientation, sgs_keypoint* kps_out, uint8_t* desc_out,
                                         float* u_right_out, int32_t* counts_out, int32_t* cur_mp_out, int32_t* nmatches_out, sgs_rect* boxes_out,
                                         int32_t* nboxes_out, uint8_t* have_out, sgs_keypoint* kps_un_out, float* depth_out) {
    const char* const fn = "sgs_tracker_step_rgbd_stream";
    LastFrame last;
    last.xyz = last_xyz; last.desc = last_desc; last.flags = last_flags; last.octave = last_octave; last.angle = last_angle; last.n = last_n;
    last.tcw_cur = tcw_cur; last.tcw_last = tcw_last;
    HostOutputs out;
    out.kps = kps_out; out.desc = desc_out; out.u_right = u_right_out; out.counts = counts_out; out.cur_mp = cur_mp_out; out.nmatches = nmatches_out;
    out.boxes = boxes_out; out.nboxes = nboxes_out; out.have = have_out; out.kps_un = kps_un_out; out.depth = depth_out;
    if (!t || !det || !rgb || !depth || !fmt || !slot || !last.complete() || !out.complete()) return bad(fn, "NULL argument");
    if (!slots_ok(fn, nframes, t->max_batch, slot) || !rgb_layout_ok(t, fn, rgb_stride, rgb_pitch) ||
        !depth_args_ok(t, fn, fmt, depth_stride, depth_pitch, depth)) return SGS_ERR_INVALID;
    SGS_CUDA_TRY(cudaSetDevice(t->device));
    const size_t row = (size_t)t->width * (fmt->depth_type == 0 ? 2 : 4);
    int rc = ensure_rgbd_buffers(t, row * t->height);
    if (rc != SGS_OK) return rc;
    rc = ensure_stream_state(t, t->st);
    if (rc != SGS_OK) return rc;
    rc = upload_rgb(t, rgb, rgb_stride, rgb_pitch, nframes);
    if (rc != SGS_OK) return rc;
    SGS_CUDA_TRY(upload_frames(t->d_depth_raw, depth, depth_stride, depth_pitch, row, t->height, nframes, t->st));
    StepFrames fr = staged_rgb(t);
    fr.d_depth = t->d_depth_raw; fr.depth_stride = row * t->height; fr.depth_pitch = (int)row; fr.fmt = fmt;
    TrackInputs in{last};
    in.slot = slot; in.new_stream = new_stream;
    rc = enqueue_step(t, det, fr, nframes, in, true, th, mono, check_orientation, t->st);
    if (rc != SGS_OK) return rc;
    return download_results(t, nframes, out);
}

SGS_API int sgs_tracker_frame_device(const sgs_tracker* t, const sgs_keypoint** d_kps_un, const float** d_depth) {
    if (!t) return bad("sgs_tracker_frame_device", "NULL handle");
    if (!t->d_kpsun2) return bad("sgs_tracker_frame_device", "no RGB-D step has run on this handle");
    if (d_kps_un) *d_kps_un = t->d_kpsun2;
    if (d_depth) *d_depth = t->d_dz2;
    return SGS_OK;
}

}  // extern "C"
