// tracker.cu -- batched front end of the tracking thread's per-frame hot path with HOST buffers at the boundary:
//   sgs_tracker_extract : Frame::ExtractORB (src/Frame.cc:274-280) for a batch of frames; keypoints go back to the host
//                         (the host runs LK + findFundamentalMat on them, src/Frame.cc:445-472 -- not on the GPU yet);
//   sgs_tracker_track   : dyn-reject verdicts + ordered compaction (src/Frame.cc:560-604) followed by
//                         ORBmatcher::SearchByProjection(cur, last, th, mono) (src/ORBmatcher.cc:1332-1472, called from
//                         Tracking::TrackWithMotionModel, src/Tracking.cc:924), on the device-resident extraction results.
// One H2D of the frames, one H2D of the per-frame track inputs, one D2H of the compacted results + matches.
#include <cuda_runtime.h>

#include <cstring>
#include <memory>
#include <vector>

#include "host_stage.cuh"
#include "sgs_common.h"

template <class T> using Child = std::unique_ptr<T, void (*)(T*)>;      // a handle the tracker owns, released by its sgs_*_destroy

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
    cudaStream_t copy_st = nullptr; cudaEvent_t copy_ev = nullptr;      // input uploads of sgs_tracker_track_lk run beside the LK kernels
    // device inputs of track()
    float* d_prev = nullptr; float* d_uright_in = nullptr; double* d_F = nullptr; sgs_rect* d_boxes = nullptr; int32_t* d_nboxes = nullptr;
    uint8_t* d_have = nullptr;
    float* d_lxyz = nullptr; uint8_t* d_ldesc = nullptr; uint8_t* d_lflags = nullptr; int32_t* d_loct = nullptr; float* d_lang = nullptr;
    int32_t* d_ln = nullptr; float* d_tc = nullptr; float* d_tl = nullptr;
    // device outputs
    sgs_keypoint* d_kps2 = nullptr; uint8_t* d_desc2 = nullptr; int32_t* d_cnt2 = nullptr; uint8_t* d_keep = nullptr; float* d_uright2 = nullptr;
    int32_t* d_mp = nullptr; int32_t* d_nm = nullptr; unsigned long long* d_ncand = nullptr;
    int last_nframes = 0;
    // detector inside the step (sgs_tracker_step / sgs_tracker_detect_device): RGB staging, its own stream, the join events
    uint8_t* d_rgb = nullptr; size_t d_rgb_cap = 0; int32_t* d_det_status = nullptr;
    cudaStream_t det_st = nullptr; cudaEvent_t det_ev = nullptr; cudaEvent_t ex_ev = nullptr;
    // sgs_tracker_pose_chain_device: scratch sized on first use for (max_batch, mp_cap)
    int chain_mp_cap = 0;
    Child<sgs_matcher> mt_local{nullptr, sgs_matcher_destroy};
    uint8_t* d_enable = nullptr; int32_t* d_nm2 = nullptr; uint8_t* d_obs = nullptr; uint8_t* d_seen = nullptr; int32_t* d_ninl = nullptr; int32_t* d_nml = nullptr;
    double* d_po_err = nullptr; uint8_t* d_po_level = nullptr;
    uint8_t* d_inview = nullptr; float* d_projx = nullptr; float* d_projy = nullptr; float* d_projxr = nullptr; int32_t* d_level = nullptr; float* d_viewcos = nullptr;
    unsigned long long* d_ncand2 = nullptr;
};

namespace sgs {
// ordered compaction of the per-keypoint u_right side array with the verdicts of the dyn-reject kernel
__global__ void compact_uright_kernel(const float* __restrict__ ur_in, const uint8_t* __restrict__ keep, const int32_t* __restrict__ n_in,
                                      const int32_t* __restrict__ n_out, int cap, float* __restrict__ ur_out, int32_t* __restrict__ mp) {
    __shared__ int s_warp[8];
    __shared__ int s_carry;
    const int f = blockIdx.x;
    const int n = min(n_in[f], cap);
    const bool restored = n_out[f] == n;   // restore-all (or nothing rejected): identity
    const int64_t base = (int64_t)f * cap;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i0 = 0; i0 < n; i0 += 256) {
        const int i = i0 + threadIdx.x;
        const bool ok = i < n && (restored || keep[base + i]);
        const unsigned m = __ballot_sync(0xffffffffu, ok);
        if (lane == 0) s_warp[warp] = __popc(m);
        __syncthreads();
        int off = s_carry;
        for (int w = 0; w < warp; ++w) off += s_warp[w];
        if (ok) ur_out[base + off + __popc(m & ((1u << lane) - 1))] = ur_in[base + i];
        __syncthreads();
        if (threadIdx.x == 0) { int t = 0; for (int w = 0; w < 8; ++w) t += s_warp[w]; s_carry += t; }
        __syncthreads();
    }
    for (int i = threadIdx.x; i < cap; i += 256) mp[base + i] = -1;   // Tracking.cc:916 clears mvpMapPoints before the search
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
// :940-957 discard the outliers of the first PoseOptimization; SearchLocalPoints' first loop (:1265-1281): every map point matched in the frame --
// the discarded ones too, their mnLastFrameSeen was set at :951 -- is marked as seen, bad ones lose their slot (last_flags bit 2 = isBad()).
__global__ void __launch_bounds__(256) chain_discard_kernel(const int32_t* __restrict__ n_cur, int cap, int point_cap, const uint8_t* __restrict__ last_flags,
                                                            const int32_t* __restrict__ last_local_id, int mp_cap, int32_t* __restrict__ mp, uint8_t* __restrict__ outlier,
                                                            uint8_t* __restrict__ obs, uint8_t* __restrict__ seen, const int32_t* __restrict__ nm, int32_t* __restrict__ stats) {
    __shared__ int s_drop, s_map;
    const int f = blockIdx.x;
    const int n = min(n_cur[f], cap);
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
            if (lid >= 0 && lid < mp_cap) seen[(int64_t)f * mp_cap + lid] = 1;
            if (outlier[k]) { id = -1; outlier[k] = 0; ++drop; }
            else {
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
// SearchLocalPoints' second loop (:1286-1300): points seen in this frame or bad are skipped before isInFrustum; nToMatch
__global__ void __launch_bounds__(256) chain_mask_kernel(const int32_t* __restrict__ mp_n, int mp_cap, const uint8_t* __restrict__ mp_valid, const uint8_t* __restrict__ seen,
                                                         uint8_t* __restrict__ inview, int32_t* __restrict__ stats) {
    __shared__ int s_cnt;
    const int f = blockIdx.x;
    const int n = min(mp_n[f], mp_cap);
    if (threadIdx.x == 0) s_cnt = 0;
    __syncthreads();
    int c = 0;
    for (int j = threadIdx.x; j < mp_cap; j += blockDim.x) {
        const int64_t k = (int64_t)f * mp_cap + j;
        const uint8_t v = (j < n && inview[k] && mp_valid[k] && !seen[k]) ? 1 : 0;
        inview[k] = v; c += v;
    }
    atomicAdd(&s_cnt, c);
    __syncthreads();
    if (threadIdx.x == 0) stats[8 * f + 5] = s_cnt;
}
// :982-996 mnMatchesInliers (mbOnlyTracking == false): map point && !outlier && Observations() > 0
__global__ void __launch_bounds__(256) chain_final_kernel(const int32_t* __restrict__ n_cur, int cap, const int32_t* __restrict__ mp, const uint8_t* __restrict__ outlier,
                                                          const uint8_t* __restrict__ obs, const int32_t* __restrict__ nml, int32_t* __restrict__ f_mp, int32_t* __restrict__ stats) {
    __shared__ int s_cnt;
    const int f = blockIdx.x;
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
}  // namespace sgs

using namespace sgs;

namespace {
int bad(const char* m) { set_error("%s", m); return SGS_ERR_INVALID; }

// the per-frame inputs of the last-frame search, host -> device on `s`
int upload_track_inputs(sgs_tracker* t, size_t B, const float* u_right, const float* last_xyz, const uint8_t* last_desc, const uint8_t* last_flags,
                        const int32_t* last_octave, const float* last_angle, const int32_t* last_n, const float* tcw_cur, const float* tcw_last, cudaStream_t s) {
    const size_t K = t->cap, M = t->point_cap;
    auto h2d = [s](void* dst, const void* src, size_t bytes) { return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, s); };
    SGS_CUDA_TRY(h2d(t->d_uright_in, u_right, B * K * 4)); SGS_CUDA_TRY(h2d(t->d_lxyz, last_xyz, B * M * 12)); SGS_CUDA_TRY(h2d(t->d_ldesc, last_desc, B * M * 32));
    SGS_CUDA_TRY(h2d(t->d_lflags, last_flags, B * M)); SGS_CUDA_TRY(h2d(t->d_loct, last_octave, B * M * 4)); SGS_CUDA_TRY(h2d(t->d_lang, last_angle, B * M * 4));
    SGS_CUDA_TRY(h2d(t->d_ln, last_n, B * 4)); SGS_CUDA_TRY(h2d(t->d_tc, tcw_cur, B * 64)); SGS_CUDA_TRY(h2d(t->d_tl, tcw_last, B * 64));
    return SGS_OK;
}

// the results of the last-frame search, device -> host on `s` (u_right_out may be NULL)
int download_track_results(const sgs_tracker* t, size_t B, sgs_keypoint* kps_out, uint8_t* desc_out, float* u_right_out, int32_t* counts_out,
                           int32_t* cur_mp_out, int32_t* nmatches_out, cudaStream_t s) {
    const size_t K = t->cap;
    auto d2h = [s](void* dst, const void* src, size_t bytes) { return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s); };
    SGS_CUDA_TRY(d2h(kps_out, t->d_kps2, B * K * sizeof(sgs_keypoint))); SGS_CUDA_TRY(d2h(desc_out, t->d_desc2, B * K * 32)); SGS_CUDA_TRY(d2h(counts_out, t->d_cnt2, B * 4));
    if (u_right_out) SGS_CUDA_TRY(d2h(u_right_out, t->d_uright2, B * K * 4));
    SGS_CUDA_TRY(d2h(cur_mp_out, t->d_mp, B * K * 4)); SGS_CUDA_TRY(d2h(nmatches_out, t->d_nm, B * 4));
    return SGS_OK;
}
}  // namespace

extern "C" {

SGS_API void sgs_tracker_destroy(sgs_tracker* t) { delete t; }

SGS_API int sgs_tracker_create(const sgs_orb_params* params, int width, int height, int max_batch, int point_cap, int max_boxes,
                               const sgs_camera* cam, int device, sgs_tracker** out) {
    if (!params || !cam || !out || point_cap < 1 || max_boxes < 0) return bad("sgs_tracker_create: bad argument");
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
    *out = t.release();
    return SGS_OK;
}

SGS_API int sgs_tracker_max_keypoints(const sgs_tracker* t, int* cap) {
    if (!t || !cap) return bad("sgs_tracker_max_keypoints: NULL");
    *cap = t->cap;
    return SGS_OK;
}

SGS_API int sgs_tracker_extract(sgs_tracker* t, const uint8_t* gray, int nframes, size_t frame_stride, int pitch, sgs_keypoint* kps, uint8_t* desc,
                                int cap, int* n) {
    if (!t) return bad("sgs_tracker_extract: NULL handle");
    int rc = sgs_extract_batch(t->ex.get(), gray, nframes, frame_stride, pitch, kps, desc, cap, n);
    if (rc == SGS_OK) t->last_nframes = nframes;
    return rc;
}

SGS_API int sgs_tracker_extract_device(sgs_tracker* t, const uint8_t* d_gray, int nframes, size_t frame_stride, int pitch, void* stream) {
    if (!t) return bad("sgs_tracker_extract_device: NULL handle");
    int rc = sgs_extract_batch_device(t->ex.get(), d_gray, nframes, frame_stride, pitch, stream ? stream : (void*)t->st);
    if (rc == SGS_OK) t->last_nframes = nframes;
    return rc;
}

// all pointers are DEVICE pointers; enqueues dyn-reject + u_right compaction + projection matching on `stream`
SGS_API int sgs_tracker_track_device(sgs_tracker* t, int nframes, const float* prev_xy, const float* u_right, const double* F, const sgs_rect* boxes,
                                     const int32_t* nboxes, const uint8_t* have_dyn, const float* last_xyz, const uint8_t* last_desc,
                                     const uint8_t* last_flags, const int32_t* last_octave, const float* last_angle, const int32_t* last_n,
                                     const float* tcw_cur, const float* tcw_last, float th, int mono, int check_orientation, void* stream) {
    if (!t || !last_xyz || !last_desc || !last_flags || !last_octave || !last_angle ||
        !last_n || !tcw_cur || !tcw_last) return bad("sgs_tracker_track_device: NULL argument");
    if (!nboxes) nboxes = t->d_nboxes;           // boxes / nboxes / have_dyn == NULL: the tracker's own arrays, filled by sgs_tracker_detect_device
    if (!have_dyn) have_dyn = t->d_have;
    if (!u_right) u_right = t->d_uright_in;      // filled by sgs_tracker_stereo_device
    if (!F) F = t->d_Fgpu;                  // filled by sgs_tracker_fundamental_device
    if (nframes < 1 || nframes > t->last_nframes) return bad("sgs_tracker_track_device: nframes exceeds the last extract call");
    if (!prev_xy) prev_xy = t->d_prev;      // filled by sgs_tracker_lk_device
    cudaStream_t st = stream ? (cudaStream_t)stream : t->st;
    const sgs_keypoint* d_kps; const uint8_t* d_desc; const int32_t* d_cnt; int cap = 0;
    sgs_extractor_results_device(t->ex.get(), &d_kps, &d_desc, &d_cnt, &cap);
    int rc = sgs_dynreject_batch_device(d_kps, d_desc, d_cnt, cap, nframes, prev_xy, F, boxes ? boxes : t->d_boxes, nboxes, t->max_boxes, have_dyn,
                                        t->nfeatures, t->d_kps2, t->d_desc2, t->d_cnt2, t->d_keep, st);
    if (rc != SGS_OK) return rc;
    compact_uright_kernel<<<nframes, 256, 0, st>>>(u_right, t->d_keep, d_cnt, t->d_cnt2, cap, t->d_uright2, t->d_mp);
    SGS_CUDA_TRY(cudaMemsetAsync(t->d_ncand, 0, (size_t)nframes * 8, st));
    sgs_lastframe_batch a;
    std::memset(&a, 0, sizeof a);
    a.cam = t->cam;
    a.cur_kps = t->d_kps2; a.cur_desc = t->d_desc2; a.cur_uright = t->d_uright2; a.cur_n = t->d_cnt2;
    a.last_xyz = last_xyz; a.last_desc = last_desc; a.last_flags = last_flags; a.last_octave = last_octave; a.last_angle = last_angle; a.last_n = last_n;
    a.tcw_cur = tcw_cur; a.tcw_last = tcw_last; a.th = th; a.mono = mono; a.check_orientation = check_orientation;
    a.cur_mp = t->d_mp; a.cur_mp_obs_in = nullptr; a.nmatches = t->d_nm; a.ncand = (uint64_t*)t->d_ncand;
    return sgs_match_project_lastframe_batch_device(t->mt.get(), &a, nframes, st);
}

// device pointers to the results of the last track call: kps [B][cap], desc, u_right, counts [B], cur_mp [B][cap], nmatches [B], ncand [B]
SGS_API int sgs_tracker_results_device(const sgs_tracker* t, const sgs_keypoint** kps, const uint8_t** desc, const float** u_right,
                                       const int32_t** counts, const int32_t** cur_mp, const int32_t** nmatches, const uint64_t** ncand) {
    if (!t) return bad("sgs_tracker_results_device: NULL handle");
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
    if (!t || !prev_xy || !u_right || !F || !nboxes || !have_dyn || !last_xyz || !last_desc || !last_flags || !last_octave || !last_angle ||
        !last_n || !tcw_cur || !tcw_last || !kps_out || !desc_out || !counts_out || !cur_mp_out || !nmatches_out)
        return bad("sgs_tracker_track: NULL argument");
    if (nframes < 1 || nframes > t->last_nframes) return bad("sgs_tracker_track: nframes exceeds the last sgs_tracker_extract call");
    SGS_CUDA_TRY(cudaSetDevice(t->device));
    const size_t B = nframes, K = t->cap;
    cudaStream_t st = t->st;
    SGS_CUDA_TRY(cudaMemcpyAsync(t->d_prev, prev_xy, B * K * 8, cudaMemcpyHostToDevice, st)); SGS_CUDA_TRY(cudaMemcpyAsync(t->d_F, F, B * 72, cudaMemcpyHostToDevice, st));
    if (boxes) SGS_CUDA_TRY(cudaMemcpyAsync(t->d_boxes, boxes, B * t->max_boxes * sizeof(sgs_rect), cudaMemcpyHostToDevice, st));
    SGS_CUDA_TRY(cudaMemcpyAsync(t->d_nboxes, nboxes, B * 4, cudaMemcpyHostToDevice, st)); SGS_CUDA_TRY(cudaMemcpyAsync(t->d_have, have_dyn, B, cudaMemcpyHostToDevice, st));
    int rc = upload_track_inputs(t, B, u_right, last_xyz, last_desc, last_flags, last_octave, last_angle, last_n, tcw_cur, tcw_last, st);
    if (rc != SGS_OK) return rc;
    rc = sgs_tracker_track_device(t, nframes, t->d_prev, t->d_uright_in, t->d_F, t->d_boxes, t->d_nboxes, t->d_have, t->d_lxyz, t->d_ldesc,
                                  t->d_lflags, t->d_loct, t->d_lang, t->d_ln, t->d_tc, t->d_tl, th, mono, check_orientation, st);
    if (rc != SGS_OK) return rc;
    rc = download_track_results(t, B, kps_out, desc_out, u_right_out, counts_out, cur_mp_out, nmatches_out, st);
    if (rc != SGS_OK) return rc;
    SGS_CUDA_TRY(cudaStreamSynchronize(st));
    return SGS_OK;
}

SGS_API sgs_extractor* sgs_tracker_extractor(sgs_tracker* t) { return t ? t->ex.get() : nullptr; }
SGS_API sgs_lk* sgs_tracker_lk(sgs_tracker* t) { return t ? t->lk.get() : nullptr; }

SGS_API int sgs_tracker_lk_device(sgs_tracker* t, const uint8_t* d_frames, int nframes, size_t frame_stride, int pitch, const int32_t* d_prev_index,
                                  void* stream) {
    if (!t || !d_frames || !d_prev_index) return bad("sgs_tracker_lk_device: NULL argument");
    if (nframes < 1 || nframes > t->last_nframes) return bad("sgs_tracker_lk_device: nframes exceeds the last extract call");
    const sgs_keypoint* d_kps; const uint8_t* d_desc; const int32_t* d_cnt; int cap = 0;
    sgs_extractor_results_device(t->ex.get(), &d_kps, &d_desc, &d_cnt, &cap);
    return sgs_lk_track_batch_device(t->lk.get(), d_frames, nullptr, d_prev_index, nframes, frame_stride, pitch, d_kps, d_cnt, cap, t->d_prev,
                                     stream ? stream : (void*)t->st);
}

SGS_API int sgs_tracker_fundamental_device(sgs_tracker* t, int nframes, const sgs_rect* d_boxes, const int32_t* d_nboxes, const uint8_t* d_have_dyn,
                                           const int32_t* d_prev_index, void* stream) {
    if (!t || !d_prev_index) return bad("sgs_tracker_fundamental_device: NULL argument");
    if (!d_nboxes) d_nboxes = t->d_nboxes;       // NULL: the tracker's own arrays, filled by sgs_tracker_detect_device
    if (!d_have_dyn) d_have_dyn = t->d_have;
    if (nframes < 1 || nframes > t->last_nframes) return bad("sgs_tracker_fundamental_device: nframes exceeds the last extract call");
    const sgs_keypoint* d_kps; const uint8_t* d_desc; const int32_t* d_cnt; int cap = 0;
    sgs_extractor_results_device(t->ex.get(), &d_kps, &d_desc, &d_cnt, &cap);
    // parameters of the reference call: FM_RANSAC, 1.0, 0.99 (src/Frame.cc:470,472); OpenCV's default of 1000 iterations
    return sgs_fundamental_batch_device(d_kps, t->d_prev, d_cnt, cap, nframes, d_boxes ? d_boxes : t->d_boxes, d_nboxes, d_have_dyn, t->max_boxes,
                                        d_prev_index, 1.0, 0.99, 1000, t->d_Fgpu, t->d_finfo, stream ? stream : (void*)t->st);
}

SGS_API int sgs_tracker_stereo_device(sgs_tracker* t, int nframes, const float* d_depth, size_t depth_frame_stride, int depth_pitch, void* stream) {
    if (!t || !d_depth) return bad("sgs_tracker_stereo_device: NULL argument");
    if (nframes < 1 || nframes > t->last_nframes) return bad("sgs_tracker_stereo_device: nframes exceeds the last extract call");
    const sgs_keypoint* d_kps; const uint8_t* d_desc; const int32_t* d_cnt; int cap = 0;
    sgs_extractor_results_device(t->ex.get(), &d_kps, &d_desc, &d_cnt, &cap);
    return sgs_stereo_from_depth_batch_device(d_kps, nullptr, d_cnt, cap, nframes, d_depth, depth_frame_stride, depth_pitch, t->cam.bf, t->d_uright_in, nullptr,
                                              stream ? stream : (void*)t->st);
}

SGS_API int sgs_tracker_fundamental_device_ptr(const sgs_tracker* t, const double** d_F, const int32_t** d_info) {
    if (!t) return bad("sgs_tracker_fundamental_device_ptr: NULL");
    if (d_F) *d_F = t->d_Fgpu;
    if (d_info) *d_info = t->d_finfo;
    return SGS_OK;
}

SGS_API int sgs_tracker_prev_xy_device(const sgs_tracker* t, const float** d_prev_xy) {
    if (!t || !d_prev_xy) return bad("sgs_tracker_prev_xy_device: NULL");
    *d_prev_xy = t->d_prev;
    return SGS_OK;
}

SGS_API int sgs_tracker_track_lk(sgs_tracker* t, int nframes, const int32_t* prev_index, const float* u_right, const double* F, const sgs_rect* boxes,
                                 const int32_t* nboxes, const uint8_t* have_dyn, const float* last_xyz, const uint8_t* last_desc,
                                 const uint8_t* last_flags, const int32_t* last_octave, const float* last_angle, const int32_t* last_n,
                                 const float* tcw_cur, const float* tcw_last, float th, int mono, int check_orientation, sgs_keypoint* kps_out,
                                 uint8_t* desc_out, float* u_right_out, int32_t* counts_out, int32_t* cur_mp_out, int32_t* nmatches_out) {
    if (!t || !prev_index) return bad("sgs_tracker_track_lk: NULL argument");
    if (nframes < 1 || nframes > t->last_nframes) return bad("sgs_tracker_track_lk: nframes exceeds the last sgs_tracker_extract call");
    SGS_CUDA_TRY(cudaSetDevice(t->device));
    for (int f = 0; f < nframes; ++f) if (prev_index[f] < 0 || prev_index[f] >= nframes) return bad("sgs_tracker_track_lk: prev_index out of range");
    if (!u_right || !nboxes || !have_dyn || !last_xyz || !last_desc || !last_flags || !last_octave || !last_angle || !last_n || !tcw_cur ||
        !tcw_last || !kps_out || !desc_out || !counts_out || !cur_mp_out || !nmatches_out) return bad("sgs_tracker_track_lk: NULL argument");
    const size_t B = nframes;
    cudaStream_t st = t->st;
    // what LK and the F estimate need goes first on the compute stream; the bulk of the inputs (last-frame points, u_right) is uploaded on
    // the copy stream while those kernels run
    SGS_CUDA_TRY(cudaMemcpyAsync(t->d_pidx, prev_index, sizeof(int32_t) * B, cudaMemcpyHostToDevice, st));
    if (F) SGS_CUDA_TRY(cudaMemcpyAsync(t->d_F, F, B * 72, cudaMemcpyHostToDevice, st));
    if (boxes) SGS_CUDA_TRY(cudaMemcpyAsync(t->d_boxes, boxes, B * t->max_boxes * sizeof(sgs_rect), cudaMemcpyHostToDevice, st));
    SGS_CUDA_TRY(cudaMemcpyAsync(t->d_nboxes, nboxes, B * 4, cudaMemcpyHostToDevice, st)); SGS_CUDA_TRY(cudaMemcpyAsync(t->d_have, have_dyn, B, cudaMemcpyHostToDevice, st));
    int rc = upload_track_inputs(t, B, u_right, last_xyz, last_desc, last_flags, last_octave, last_angle, last_n, tcw_cur, tcw_last, t->copy_st);
    if (rc != SGS_OK) return rc;
    SGS_CUDA_TRY(cudaEventRecord(t->copy_ev, t->copy_st));
    const uint8_t* d_frames; int pitch; size_t fstride;
    sgs_extractor_level0_device(t->ex.get(), &d_frames, &pitch, &fstride);
    rc = sgs_tracker_lk_device(t, d_frames, nframes, fstride, pitch, t->d_pidx, st);
    if (rc != SGS_OK) return rc;
    if (!F) {       // F == NULL: findFundamentalMat on the device, previous-frame boxes = the boxes of row prev_index[f]
        rc = sgs_tracker_fundamental_device(t, nframes, t->d_boxes, t->d_nboxes, t->d_have, t->d_pidx, st);
        if (rc != SGS_OK) return rc;
    }
    SGS_CUDA_TRY(cudaStreamWaitEvent(st, t->copy_ev, 0));
    rc = sgs_tracker_track_device(t, nframes, nullptr, t->d_uright_in, F ? t->d_F : nullptr, t->d_boxes, t->d_nboxes, t->d_have, t->d_lxyz, t->d_ldesc, t->d_lflags,
                                  t->d_loct, t->d_lang, t->d_ln, t->d_tc, t->d_tl, th, mono, check_orientation, st);
    if (rc != SGS_OK) return rc;
    rc = download_track_results(t, B, kps_out, desc_out, u_right_out, counts_out, cur_mp_out, nmatches_out, st);
    if (rc != SGS_OK) return rc;
    SGS_CUDA_TRY(cudaStreamSynchronize(st));
    return SGS_OK;
}

SGS_API int sgs_tracker_pose_chain_device(sgs_tracker* t, const sgs_posechain_batch* a, int nframes, void* stream) {
    if (!t || !a) return bad("sgs_tracker_pose_chain_device: NULL");
    if (!a->last_xyz || !a->last_desc || !a->last_flags || !a->last_octave || !a->last_angle || !a->last_n || !a->tcw_cur || !a->tcw_last || !a->mp_xyz || !a->mp_normal ||
        !a->mp_min_dist || !a->mp_max_dist || !a->mp_desc || !a->mp_valid || !a->mp_obs || !a->mp_n || !a->tcw_motion || !a->tcw_final || !a->f_mp || !a->outlier || !a->stats)
        return bad("sgs_tracker_pose_chain_device: NULL array");
    if (nframes < 1 || nframes > t->last_nframes) return bad("sgs_tracker_pose_chain_device: nframes exceeds the last track call");
    if (a->mp_cap < 1) return bad("sgs_tracker_pose_chain_device: mp_cap < 1");
    SGS_CUDA_TRY(cudaSetDevice(t->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : t->st;
    const size_t B = t->max_batch, K = t->cap, M = a->mp_cap;
    if (t->chain_mp_cap < a->mp_cap) {                       // scratch for this local-map capacity (first call, or a larger map)
        t->chain_mp_cap = 0;
        t->mt_local.reset();
        sgs_matcher* mt_local = nullptr;
        int rc = sgs_matcher_create(t->device, t->max_batch, t->cap, a->mp_cap, &mt_local);
        t->mt_local.reset(mt_local);
        if (rc != SGS_OK) return rc;
        HandleResources& R = t->res;
        const char* const fn = "sgs_tracker_pose_chain_device";
        // 16 bytes of slack past the end of every array, as in sgs_tracker_create
        SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_enable, B + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_nm2, B * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_obs, B * K + 16));
        SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_seen, B * M + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_ninl, B * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_nml, B * 4 + 16));
        SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_po_err, B * K * 24 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_po_level, B * K + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_inview, B * M + 16));
        SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_projx, B * M * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_projy, B * M * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_projxr, B * M * 4 + 16));
        SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_level, B * M * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_viewcos, B * M * 4 + 16)); SGS_CUDA_TRY_AT(fn, R.regrow(&t->d_ncand2, B * 8 + 16));
        t->chain_mp_cap = a->mp_cap;
    }
    const int F = nframes, cap = t->cap;
    // 1. the wide-window retry of the frames with fewer than 20 matches
    chain_retry_kernel<<<F, 256, 0, st>>>(t->d_nm, cap, t->d_mp, t->d_enable, a->stats);
    sgs_lastframe_batch lf;
    std::memset(&lf, 0, sizeof lf);
    lf.cam = t->cam;
    lf.cur_kps = t->d_kps2; lf.cur_desc = t->d_desc2; lf.cur_uright = t->d_uright2; lf.cur_n = t->d_cnt2;
    lf.last_xyz = a->last_xyz; lf.last_desc = a->last_desc; lf.last_flags = a->last_flags; lf.last_octave = a->last_octave; lf.last_angle = a->last_angle; lf.last_n = a->last_n;
    lf.tcw_cur = a->tcw_cur; lf.tcw_last = a->tcw_last; lf.th = 2.f * a->th; lf.mono = a->mono; lf.check_orientation = a->check_orientation;
    lf.cur_mp = t->d_mp; lf.nmatches = t->d_nm2; lf.ncand = (uint64_t*)t->d_ncand2; lf.frame_enable = t->d_enable;
    SGS_CUDA_TRY(cudaMemsetAsync(t->d_ncand2, 0, (size_t)F * 8, st));
    SGS_CUDA_TRY(cudaMemsetAsync(t->d_nm2, 0, (size_t)F * 4, st));
    int rc = sgs_match_project_lastframe_batch_device(t->mt.get(), &lf, F, st);
    if (rc != SGS_OK) return rc;
    chain_merge_counts_kernel<<<(F + 127) / 128, 128, 0, st>>>(t->d_enable, t->d_nm2, t->d_nm, a->stats, F);
    // 2. PoseOptimization on the last-frame matches
    SGS_CUDA_TRY(cudaMemsetAsync(a->outlier, 0, (size_t)F * cap, st));
    sgs_poseopt_batch po;
    std::memset(&po, 0, sizeof po);
    po.cam = t->cam; po.tcw_in = a->tcw_cur; po.kps = t->d_kps2; po.uright = t->d_uright2; po.n = t->d_cnt2; po.cap = cap;
    po.mp_index = t->d_mp; po.points_xyz = a->last_xyz; po.point_cap = t->point_cap;
    for (int l = 0; l < 16; ++l) po.inv_level_sigma2[l] = a->inv_level_sigma2[l];
    po.tcw_out = a->tcw_motion; po.outlier = a->outlier; po.ninliers = t->d_ninl; po.scratch_err = t->d_po_err; po.scratch_level = t->d_po_level;
    rc = sgs_pose_optimization_batch_device(&po, F, st);
    if (rc != SGS_OK) return rc;
    // 3. discard outliers, mark the map points seen in the frame
    SGS_CUDA_TRY(cudaMemsetAsync(t->d_seen, 0, (size_t)F * M, st));
    chain_discard_kernel<<<F, 256, 0, st>>>(t->d_cnt2, cap, t->point_cap, a->last_flags, a->last_local_id, a->mp_cap, t->d_mp, a->outlier, t->d_obs, t->d_seen, t->d_nm, a->stats);
    // 4. SearchLocalPoints: frustum test with the new pose, scale prediction, projection search
    sgs_frustum_batch fr;
    std::memset(&fr, 0, sizeof fr);
    fr.cam = t->cam; fr.tcw = a->tcw_motion; fr.mp_xyz = a->mp_xyz; fr.mp_normal = a->mp_normal; fr.mp_min_dist = a->mp_min_dist; fr.mp_max_dist = a->mp_max_dist;
    fr.mp_n = a->mp_n; fr.point_cap = a->mp_cap; fr.viewing_cos_limit = 0.5f;
    fr.mp_inview = t->d_inview; fr.proj_x = t->d_projx; fr.proj_y = t->d_projy; fr.proj_xr = t->d_projxr; fr.level = t->d_level; fr.view_cos = t->d_viewcos;
    rc = sgs_frustum_batch_device(&fr, F, st);
    if (rc != SGS_OK) return rc;
    chain_mask_kernel<<<F, 256, 0, st>>>(a->mp_n, a->mp_cap, a->mp_valid, t->d_seen, t->d_inview, a->stats);
    sgs_localmap_batch lm;
    std::memset(&lm, 0, sizeof lm);
    lm.cam = t->cam; lm.cur_kps = t->d_kps2; lm.cur_desc = t->d_desc2; lm.cur_uright = t->d_uright2; lm.cur_n = t->d_cnt2;
    lm.mp_inview = t->d_inview; lm.proj_x = t->d_projx; lm.proj_y = t->d_projy; lm.proj_xr = t->d_projxr; lm.level = t->d_level; lm.view_cos = t->d_viewcos;
    lm.mp_desc = a->mp_desc; lm.mp_obs = a->mp_obs; lm.mp_n = a->mp_n; lm.th = a->th_local; lm.nnratio = a->nnratio_local; lm.id_base = t->point_cap;
    lm.f_mp = t->d_mp; lm.f_mp_obs = t->d_obs; lm.nmatches = t->d_nml; lm.ncand = (uint64_t*)t->d_ncand2;
    rc = sgs_match_project_localmap_batch_device(t->mt_local.get(), &lm, F, st);
    if (rc != SGS_OK) return rc;
    // 5. PoseOptimization on last-frame + local-map matches, inlier count
    po.tcw_in = a->tcw_motion; po.tcw_out = a->tcw_final; po.points2_xyz = a->mp_xyz; po.id_base2 = t->point_cap; po.point2_cap = a->mp_cap;
    rc = sgs_pose_optimization_batch_device(&po, F, st);
    if (rc != SGS_OK) return rc;
    chain_final_kernel<<<F, 256, 0, st>>>(t->d_cnt2, cap, t->d_mp, a->outlier, t->d_obs, t->d_nml, a->f_mp, a->stats);
    SGS_CUDA_TRY(cudaGetLastError());
    return SGS_OK;
}

// Detector2D::detect for the frames of the batch (src/Tracking.cc:288-307 hands the colour image to the detector thread; src/Frame.cc:478-500
// joins it before the rejection): the person boxes land in the tracker's own box arrays, in the layout the F estimate and the rejection take
// when called with boxes == NULL.  d_rgb: device frames (interleaved 8-bit RGB).  Enqueued on `stream` (NULL: the tracker's detector stream, which
// the next sgs_tracker_fundamental_device / _track_device call on the tracker's stream is NOT ordered after -- use sgs_tracker_step for that).
SGS_API int sgs_tracker_detect_device(sgs_tracker* t, sgs_detector* det, const uint8_t* d_rgb, int64_t frame_stride, int pitch, int width, int height, int nframes,
                                      void* stream) {
    if (!t || !det || !d_rgb) return bad("sgs_tracker_detect_device: NULL argument");
    if (nframes < 1 || nframes > t->max_batch) return bad("sgs_tracker_detect_device: nframes outside [1,max_batch]");
    return sgs_detector_detect_device(det, d_rgb, frame_stride, pitch, width, height, nframes, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, t->d_boxes, t->d_nboxes,
                                      t->d_have, t->max_boxes, t->d_det_status, stream ? stream : (void*)t->det_st);
}
SGS_API int sgs_tracker_boxes_device(const sgs_tracker* t, const sgs_rect** d_boxes, const int32_t** d_nboxes, const uint8_t** d_have_dyn) {
    if (!t) return bad("sgs_tracker_boxes_device: NULL");
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
    if (!t || !det || !gray || !rgb || !prev_index || !u_right || !last_xyz || !last_desc || !last_flags || !last_octave || !last_angle || !last_n || !tcw_cur ||
        !tcw_last || !kps_out || !desc_out || !counts_out || !cur_mp_out || !nmatches_out) return bad("sgs_tracker_step: NULL argument");
    if (nframes < 1 || nframes > t->max_batch) return bad("sgs_tracker_step: nframes outside [1,max_batch]");
    if (rgb_pitch < t->width * 3 || rgb_stride < (size_t)rgb_pitch * t->height) return bad("sgs_tracker_step: rgb pitch / stride too small");
    for (int f = 0; f < nframes; ++f) if (prev_index[f] < 0 || prev_index[f] >= nframes) return bad("sgs_tracker_step: prev_index out of range");
    SGS_CUDA_TRY(cudaSetDevice(t->device));
    const size_t B = nframes;
    // ---- detector branch: colour frames up, network, boxes into the tracker's arrays
    const size_t rgb_bytes = (size_t)t->width * 3 * t->height;
    if (t->d_rgb_cap < rgb_bytes * (size_t)t->max_batch) {
        t->d_rgb_cap = 0;
        SGS_CUDA_TRY(t->res.regrow(&t->d_rgb, rgb_bytes * (size_t)t->max_batch));
        t->d_rgb_cap = rgb_bytes * (size_t)t->max_batch;
    }
    if (rgb_stride == (size_t)rgb_pitch * t->height) {
        SGS_CUDA_TRY(cudaMemcpy2DAsync(t->d_rgb, (size_t)t->width * 3, rgb, rgb_pitch, (size_t)t->width * 3, (size_t)t->height * B, cudaMemcpyHostToDevice, t->det_st));
    } else {
        for (size_t f = 0; f < B; ++f)
            SGS_CUDA_TRY(cudaMemcpy2DAsync(t->d_rgb + f * rgb_bytes, (size_t)t->width * 3, rgb + f * rgb_stride, rgb_pitch, (size_t)t->width * 3, t->height, cudaMemcpyHostToDevice, t->det_st));
    }
    int rc = sgs_tracker_detect_device(t, det, t->d_rgb, (int64_t)rgb_bytes, t->width * 3, t->width, t->height, nframes, t->det_st);
    if (rc != SGS_OK) return rc;
    SGS_CUDA_TRY(cudaEventRecord(t->det_ev, t->det_st));
    // ---- tracking branch: gray frames up + ORB extraction (the extractor's streams), then LK on the tracker's stream
    rc = sgs_extract_batch(t->ex.get(), gray, nframes, gray_stride, gray_pitch, nullptr, nullptr, 0, nullptr);
    if (rc != SGS_OK) return rc;
    t->last_nframes = nframes;
    cudaStream_t st = t->st;
    SGS_CUDA_TRY(cudaEventRecord(t->ex_ev, (cudaStream_t)sgs_extractor_stream(t->ex.get())));
    SGS_CUDA_TRY(cudaStreamWaitEvent(st, t->ex_ev, 0));
    SGS_CUDA_TRY(cudaMemcpyAsync(t->d_pidx, prev_index, sizeof(int32_t) * B, cudaMemcpyHostToDevice, st));
    rc = upload_track_inputs(t, B, u_right, last_xyz, last_desc, last_flags, last_octave, last_angle, last_n, tcw_cur, tcw_last, t->copy_st);
    if (rc != SGS_OK) return rc;
    SGS_CUDA_TRY(cudaEventRecord(t->copy_ev, t->copy_st));
    const uint8_t* d_frames; int pitch; size_t fstride;
    sgs_extractor_level0_device(t->ex.get(), &d_frames, &pitch, &fstride);
    rc = sgs_tracker_lk_device(t, d_frames, nframes, fstride, pitch, t->d_pidx, st);
    if (rc != SGS_OK) return rc;
    SGS_CUDA_TRY(cudaStreamWaitEvent(st, t->det_ev, 0));                  // the join of src/Frame.cc:478-481: boxes of every frame of the batch are there
    rc = sgs_tracker_fundamental_device(t, nframes, nullptr, nullptr, nullptr, t->d_pidx, st);
    if (rc != SGS_OK) return rc;
    SGS_CUDA_TRY(cudaStreamWaitEvent(st, t->copy_ev, 0));
    rc = sgs_tracker_track_device(t, nframes, nullptr, t->d_uright_in, nullptr, nullptr, nullptr, nullptr, t->d_lxyz, t->d_ldesc, t->d_lflags, t->d_loct, t->d_lang, t->d_ln,
                                  t->d_tc, t->d_tl, th, mono, check_orientation, st);
    if (rc != SGS_OK) return rc;
    rc = download_track_results(t, B, kps_out, desc_out, u_right_out, counts_out, cur_mp_out, nmatches_out, st);
    if (rc != SGS_OK) return rc;
    if (boxes_out) SGS_CUDA_TRY(cudaMemcpyAsync(boxes_out, t->d_boxes, B * t->max_boxes * sizeof(sgs_rect), cudaMemcpyDeviceToHost, st));
    if (nboxes_out) SGS_CUDA_TRY(cudaMemcpyAsync(nboxes_out, t->d_nboxes, B * 4, cudaMemcpyDeviceToHost, st));
    if (have_out) SGS_CUDA_TRY(cudaMemcpyAsync(have_out, t->d_have, B, cudaMemcpyDeviceToHost, st));
    SGS_CUDA_TRY(cudaStreamSynchronize(st));
    return SGS_OK;
}

}  // extern "C"
