/* =====================================================================================
 * sgs_abi.h -- C ABI of libsgs_cuda.so: the H100-native (sm_90a) replacement for the
 * SG-SLAM / ORB-SLAM2 per-frame tracking hot path.
 *
 * The reference has no FFI layer: the boundary is three C++ classes inside libsg-slam.so
 * (ORB_SLAM2::ORBextractor, ORB_SLAM2::ORBmatcher, ORB_SLAM2::Frame).  Each entry point
 * below names the reference interface it replaces (paths relative to
 * /root/reference/src/sg-slam/).  the headers under include/sgslam/ hold the header-compatible C++
 * mirror of those classes implemented on top of this ABI; INTEGRATION.md shows the
 * reference-side binding.
 *
 * Conventions
 *   - plain pointers and sizes only; no torch / OpenCV / STL types
 *   - every function returns an sgs_status (0 == SGS_OK); sgs_last_error() gives the
 *     message of the calling thread's last failure
 *   - "_device" variants take/return CUDA device pointers and enqueue on the given
 *     cudaStream_t (passed as void*, NULL == the handle's own stream) without
 *     synchronising; all other variants take HOST pointers and synchronise before return
 *   - there is NO CPU fallback: without a CUDA device every call fails with
 *     SGS_ERR_CUDA
 * ===================================================================================== */
#ifndef SGS_ABI_H_
#define SGS_ABI_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define SGS_API __attribute__((visibility("default")))
#else
#define SGS_API
#endif

#define SGS_ABI_VERSION 1

typedef enum sgs_status {
    SGS_OK = 0,
    SGS_ERR_INVALID = 1,     /* bad argument (NULL, size mismatch, unsupported geometry) */
    SGS_ERR_CUDA = 2,        /* CUDA runtime failure or no device */
    SGS_ERR_CAPACITY = 3,    /* caller-provided capacity too small; nothing was truncated silently */
    SGS_ERR_UNSUPPORTED = 4  /* configuration outside what the reference itself supports */
} sgs_status;

/* ORBextractor constructor arguments, src/ORBextractor.cc:411-413 (TUM3.yaml:41-54). */
typedef struct sgs_orb_params {
    int32_t nfeatures;
    float scale_factor;
    int32_t nlevels;
    int32_t ini_th_fast;
    int32_t min_th_fast;
} sgs_orb_params;

/* Binary layout of cv::KeyPoint (28 bytes): pt.x, pt.y, size, angle, response, octave, class_id. */
typedef struct sgs_keypoint {
    float x, y, size, angle, response;
    int32_t octave, class_id;
} sgs_keypoint;

typedef struct sgs_rect { float x, y, w, h; } sgs_rect; /* cv::Rect_<float> */

SGS_API int sgs_abi_version(void);
SGS_API const char* sgs_last_error(void);
SGS_API int sgs_device_count(int* n);

/* ------------------------------------------------------------------------------------
 * ORBextractor  (include/ORBextractor.h:45-105, src/ORBextractor.cc)
 * One handle = one extractor bound to an image geometry and a maximum batch size; device
 * buffers (pyramids, candidate lists, results) are owned by the handle.
 * ------------------------------------------------------------------------------------ */
typedef struct sgs_extractor sgs_extractor;

/* ORBextractor::ORBextractor (src/ORBextractor.cc:411-471) + buffer allocation for frames of width x height,
 * up to max_batch frames per call, on CUDA device `device`.
 * Limits (pinned by tests/test_gpu_orb_cases.py):
 *   - width and height in [1, 4096]; 4097 returns SGS_ERR_INVALID;
 *   - scale_factor exactly 2.0 returns SGS_ERR_UNSUPPORTED (cv::resize would switch to INTER_AREA);
 *   - every level must hold at least one 30-px FAST cell in each direction, and must not be portrait (quirk Q2): SGS_ERR_UNSUPPORTED;
 *   - the quadtree keeps its node arrays in shared memory: nfeatures may be at most about 1393 (the exact limit is
 *     2 * max(N, 4 * roots) + 4 * roots + 16 <= 2806 nodes for the largest level budget N; 640x480 with one level accepts 1393 and
 *     refuses 1394 with SGS_ERR_UNSUPPORTED). */
SGS_API int sgs_extractor_create(const sgs_orb_params* params, int width, int height, int max_batch, int device,
                                 sgs_extractor** out);
SGS_API void sgs_extractor_destroy(sgs_extractor* ex);

/* Getters: GetLevels/GetScaleFactors/GetInverseScaleFactors/GetScaleSigmaSquares/GetInverseScaleSigmaSquares
 * (include/ORBextractor.h:62-85); any output pointer may be NULL.  Arrays have nlevels entries. */
SGS_API int sgs_extractor_tables(const sgs_extractor* ex, float* scale, float* inv_scale, float* sigma2,
                                 float* inv_sigma2, int32_t* features_per_level);
/* Upper bound on keypoints per frame (nfeatures + 3 per level, SURVEY Appendix E.5): size output buffers with it. */
SGS_API int sgs_extractor_max_keypoints(const sgs_extractor* ex, int* cap);
/* Level geometry of mvImagePyramid[level] (include/ORBextractor.h:87): width, height and device pitch. */
SGS_API int sgs_extractor_level_info(const sgs_extractor* ex, int level, int* width, int* height, int* pitch);

/* ORBextractor::operator() (src/ORBextractor.cc:1045-1106) on ONE host image (8-bit gray, `pitch` bytes/row).
 * kps/desc are caller-allocated with room for `cap` keypoints (desc: cap x 32 bytes, row i belongs to kps[i]).
 * An empty image (gray == NULL or w*h == 0) yields *n = 0 like the reference's early return (:1048). */
SGS_API int sgs_extract(sgs_extractor* ex, const uint8_t* gray, int width, int height, int pitch, sgs_keypoint* kps,
                        uint8_t* desc, int cap, int* n);

/* Same, for `nframes` independent host images laid out `frame_stride` bytes apart.  kps: [nframes][cap],
 * desc: [nframes][cap][32] (may be NULL: keypoints only), n: [nframes].  Host<->device copies happen inside; pinned caller
 * buffers (input, and outputs with cap == sgs_extractor_max_keypoints) are used directly, without staging. */
SGS_API int sgs_extract_batch(sgs_extractor* ex, const uint8_t* gray, int nframes, size_t frame_stride, int pitch,
                              sgs_keypoint* kps, uint8_t* desc, int cap, int* n);
/* kps == desc == n == NULL: upload + kernels only, no copy back and no synchronisation -- the results stay on the device
 * (sgs_extractor_results_device); sgs_extractor_stream is the stream that work was enqueued on (for event ordering). */
SGS_API void* sgs_extractor_stream(const sgs_extractor* ex);

/* Device-resident batch: d_gray is a DEVICE pointer ([nframes] images, frame_stride/pitch bytes); results stay on the
 * device inside the handle (see sgs_extractor_results_device).  Asynchronous on `stream`. */
SGS_API int sgs_extract_batch_device(sgs_extractor* ex, const uint8_t* d_gray, int nframes, size_t frame_stride,
                                     int pitch, void* stream);
/* Device pointers to the results of the last *_device call: kps [max_batch][cap], desc [max_batch][cap][32],
 * counts [max_batch] (int32).  Valid until the next call on the handle. */
SGS_API int sgs_extractor_results_device(const sgs_extractor* ex, const sgs_keypoint** d_kps, const uint8_t** d_desc,
                                         const int32_t** d_counts, int* cap);

/* Copies the results of the last call on the handle (device-resident or not) for frames [0,nframes) to host buffers
 * kps [nframes][cap], desc [nframes][cap][32], n [nframes]; synchronises `stream` (NULL == the handle's stream). */
SGS_API int sgs_extractor_fetch(sgs_extractor* ex, int nframes, sgs_keypoint* kps, uint8_t* desc, int cap, int* n, void* stream);

/* Parity / debugging accessors (host copies of device intermediates of the LAST call, frame index `frame`). */
SGS_API int sgs_extractor_read_level(sgs_extractor* ex, int frame, int level, int blurred, uint8_t* out, int out_pitch);
/* FAST candidates of one level before the quadtree: packed as int32 triples (x, y, score) relative to (16,16),
 * in unspecified order.  Returns SGS_ERR_CAPACITY (with *n = required) when cap is too small. */
SGS_API int sgs_extractor_read_candidates(sgs_extractor* ex, int frame, int level, int32_t* xyscore, int cap, int* n);

/* ------------------------------------------------------------------------------------
 * ORBmatcher  (include/ORBmatcher.h:41-89, src/ORBmatcher.cc)
 * ------------------------------------------------------------------------------------ */

/* ORBmatcher::DescriptorDistance (src/ORBmatcher.cc:1649-1665) for n pairs of 32-byte descriptors (host). */
SGS_API int sgs_hamming_pairs(const uint8_t* a, const uint8_t* b, int n, int32_t* dist, int device);

/* Brute-force nearest / second-nearest train descriptor for every query descriptor (the inner loop shared by every
 * ORBmatcher search, src/ORBmatcher.cc:93-113, over an unrestricted candidate set; first index wins ties).
 * best_idx/best_dist/second_dist: [nq].  Host pointers. */
SGS_API int sgs_hamming_bf(const uint8_t* query, int nq, const uint8_t* train, int nt, int32_t* best_idx,
                           int32_t* best_dist, int32_t* second_dist, int device);
/* Device-resident variant (all pointers are device pointers), asynchronous on `stream`.  d_scratch (int32 elements,
 * size from sgs_hamming_bf_scratch_elems; may be NULL) lets small query sets split the train set over all SMs. */
SGS_API int sgs_hamming_bf_scratch_elems(int nq, int nt, int64_t* elems);
SGS_API int sgs_hamming_bf_device(const uint8_t* d_query, int nq, const uint8_t* d_train, int nt, int32_t* d_best_idx,
                                  int32_t* d_best_dist, int32_t* d_second_dist, int32_t* d_scratch, void* stream);
/* MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:242-307) for `npoints` map points: d_desc [P][max_obs][32] (the descriptors of the
 * point's observations, max_obs <= 64), d_counts [P]; d_best_idx [P] = index of the descriptor with the smallest median distance to the others. */
SGS_API int sgs_distinctive_descriptor_batch_device(const uint8_t* d_desc, const int32_t* d_counts, int max_obs, int npoints,
                                                    int32_t* d_best_idx, void* stream);

/* Flattened read-only view of a Frame as the matchers need it (src/Frame.cc:129-198): undistorted keypoints,
 * mvuRight, descriptors, image bounds (mnMinX..), intrinsics and the extractor's scale factors. */
typedef struct sgs_frame_view {
    int32_t n;                  /* Frame::N */
    const sgs_keypoint* keys_un;/* mvKeysUn */
    const float* u_right;       /* mvuRight */
    const uint8_t* desc;        /* mDescriptors, n x 32 */
    float min_x, min_y, max_x, max_y; /* mnMinX.. (src/Frame.cc:686-714) */
    float fx, fy, cx, cy, bf;   /* Frame::fx.., mbf */
    int32_t nlevels;
    const float* scale_factors; /* mvScaleFactors */
} sgs_frame_view;

/* ORBmatcher::SearchByProjection(Frame& Current, const Frame& Last, th, bMono) (src/ORBmatcher.cc:1332-1472).
 * The LastFrame object graph is flattened by the caller:
 *   last_has_mp[i]  LastFrame.mvpMapPoints[i] != NULL && !LastFrame.mvbOutlier[i]
 *   last_xyz        pMP->GetWorldPos() (3 floats)      last_desc    pMP->GetDescriptor() (32 bytes)
 *   last_obs[i]     pMP->Observations() > 0            last_octave  LastFrame.mvKeys[i].octave
 *   last_angle      LastFrame.mvKeysUn[i].angle
 * tcw_cur / tcw_last: 4x4 row-major float poses (Frame::mTcw).
 * cur_mp_inout[j]: index i of the last-frame point assigned to CurrentFrame.mvpMapPoints[j], -1 for NULL; on entry it
 * holds the caller's state (Tracking.cc:916 clears it), cur_mp_obs_in[j] (may be NULL == all 1) tells whether a
 * pre-existing entry has Observations()>0.  *nmatches is the reference's return value.  Host pointers. */
SGS_API int sgs_match_project_lastframe(const sgs_frame_view* cur, const float* tcw_cur, const float* tcw_last, int nlast,
                                        const uint8_t* last_has_mp, const float* last_xyz, const uint8_t* last_desc,
                                        const uint8_t* last_obs, const int32_t* last_octave, const float* last_angle,
                                        float th, int mono, int check_orientation, int32_t* cur_mp_inout,
                                        const uint8_t* cur_mp_obs_in, int* nmatches, int device);

/* ORBmatcher::SearchByProjection(Frame& F, const vector<MapPoint*>&, th) (src/ORBmatcher.cc:45-129) with the fields
 * Frame::isInFrustum (src/Frame.cc:296-352) stores in each MapPoint passed as flat arrays:
 *   mp_inview[i] (mbTrackInView && !isBad()), proj_x/proj_y/proj_xr (mTrackProjX/Y/XR), level (mnTrackScaleLevel),
 *   view_cos (mTrackViewCos), mp_desc (GetDescriptor), mp_obs (Observations()>0).
 * f_mp_inout[j] >= 0 means F.mvpMapPoints[j] is set (opaque id), f_mp_obs_inout[j] its Observations()>0 flag.  New
 * matches store id_base + i.  nnratio is ORBmatcher::mfNNratio. */
SGS_API int sgs_match_project_localmap(const sgs_frame_view* f, int nmp, const uint8_t* mp_inview, const float* proj_x,
                                       const float* proj_y, const float* proj_xr, const int32_t* level,
                                       const float* view_cos, const uint8_t* mp_desc, const uint8_t* mp_obs, float th,
                                       float nnratio, int32_t id_base, int32_t* f_mp_inout, uint8_t* f_mp_obs_inout,
                                       int* nmatches, int device);

/* ---- batched, device-resident matchers (one CUDA block per independent frame / stream) --------------------------
 * Per-frame arrays are laid out [nframes][cap]; every pointer is a DEVICE pointer.  The camera block carries the Frame
 * statics (src/Frame.cc:176-196) and the extractor's scale factors. */
typedef struct sgs_camera {
    float min_x, min_y, max_x, max_y;
    float fx, fy, cx, cy, bf;
    int32_t nlevels;
    float scale_factors[16];
} sgs_camera;

typedef struct sgs_matcher sgs_matcher;   /* owns the per-point scratch of the batched kernels */
SGS_API int sgs_matcher_create(int device, int max_frames, int cur_cap, int point_cap, sgs_matcher** out);
SGS_API void sgs_matcher_destroy(sgs_matcher* m);

typedef struct sgs_lastframe_batch {      /* SearchByProjection(Frame&, const Frame&, th, bMono), src/ORBmatcher.cc:1332 */
    sgs_camera cam;
    const sgs_keypoint* cur_kps; const uint8_t* cur_desc; const float* cur_uright; const int32_t* cur_n; /* [F][cur_cap] / [F] */
    const float* last_xyz;        /* [F][point_cap][3] */
    const uint8_t* last_desc;     /* [F][point_cap][32] */
    const uint8_t* last_flags;    /* bit0: map point present && !outlier, bit1: Observations()>0 */
    const int32_t* last_octave; const float* last_angle; const int32_t* last_n;
    const float* tcw_cur; const float* tcw_last;   /* [F][16] row-major */
    float th; int32_t mono, check_orientation;
    int32_t* cur_mp;              /* in/out [F][cur_cap]: index of the matched last-frame point or -1 */
    const uint8_t* cur_mp_obs_in; /* may be NULL */
    int32_t* nmatches;            /* out [F] */
    uint64_t* ncand;              /* out [F] (accumulated): candidates examined, for the roofline byte count */
    const uint8_t* frame_enable;  /* may be NULL; [F]: 0 = leave this frame untouched (the wide-window retry of src/Tracking.cc:927-931 only runs on the frames that need it) */
} sgs_lastframe_batch;
SGS_API int sgs_match_project_lastframe_batch_device(sgs_matcher* m, const sgs_lastframe_batch* args, int nframes, void* stream);

typedef struct sgs_keyframe_batch {       /* SearchByProjection(Frame&, KeyFrame*, sAlreadyFound, th, ORBdist), src/ORBmatcher.cc:1474 (relocalisation) */
    sgs_camera cam;
    const sgs_keypoint* cur_kps; const uint8_t* cur_desc; const float* cur_uright; const int32_t* cur_n;   /* cur_uright is not read by the search but must be valid */
    const float* kf_xyz;          /* [F][point_cap][3]  map points of the key frame, in key-frame keypoint order */
    const uint8_t* kf_desc;       /* [F][point_cap][32] MapPoint::GetDescriptor() */
    const uint8_t* kf_valid;      /* 1: map point exists, !isBad(), not in sAlreadyFound */
    const float* kf_angle;        /* pKF->mvKeysUn[i].angle */
    const float* kf_min_dist; const float* kf_max_dist;   /* mfMinDistance / mfMaxDistance (raw) */
    const int32_t* kf_n;          /* [F] */
    const float* tcw_cur;         /* [F][16] */
    float th; int32_t orb_dist, check_orientation;
    int32_t* cur_mp;              /* in/out [F][cur_cap]: >= 0 means CurrentFrame.mvpMapPoints[j] is set; new matches write the key-frame index */
    int32_t* nmatches; uint64_t* ncand;
} sgs_keyframe_batch;
SGS_API int sgs_match_project_keyframe_batch_device(sgs_matcher* m, const sgs_keyframe_batch* args, int nframes, void* stream);
SGS_API int sgs_match_project_keyframe(const sgs_frame_view* cur, const float* tcw_cur, int nkf, const uint8_t* kf_valid, const float* kf_xyz,
                                       const uint8_t* kf_desc, const float* kf_angle, const float* kf_min_dist, const float* kf_max_dist,
                                       float th, int orb_dist, int check_orientation, int32_t* cur_mp_inout, int* nmatches, int device);

typedef struct sgs_fuse_batch {           /* search half of Fuse(KeyFrame*, const vector<MapPoint*>&, th), src/ORBmatcher.cc:829-980 */
    sgs_camera cam;                       /* the key frame's intrinsics, image bounds and scale factors */
    const sgs_keypoint* kf_kps; const uint8_t* kf_desc; const float* kf_uright; const int32_t* kf_n; int32_t kf_cap;   /* mvKeysUn, mDescriptors, mvuRight */
    const float* tcw;                     /* [F][16] key-frame pose */
    const float* ow;                      /* [F][3]  pKF->GetCameraCenter() */
    const float* mp_xyz; const float* mp_normal; const float* mp_min_dist; const float* mp_max_dist;      /* [F][mp_cap](x3) */
    const uint8_t* mp_desc;               /* [F][mp_cap][32] */
    const uint8_t* mp_valid;              /* exists && !isBad() && !IsInKeyFrame(pKF) */
    const int32_t* mp_n; int32_t mp_cap;
    float th; float inv_level_sigma2[16]; /* pKF->mvInvLevelSigma2 */
    int32_t sim3_variant;                 /* 1: Fuse(KeyFrame*, cv::Mat Scw, vpPoints, th, vpReplacePoint) (src/ORBmatcher.cc:982-1104): tcw / ow hold the
                                             Rcw, tcw and Ow the caller decomposed from Scw (:988-992); no chi-square gates
                                             2: one direction of SearchBySim3(pKF1, pKF2, vpMatches12, s12, R12, t12, th) (:1106-1330): tcw = pose of the key
                                             frame that OWNS the points, xform2 = [sR21 | t21] (:1122-1124), kf_* = the other key frame; distance |p3Dc2|,
                                             no viewing-angle test (mp_normal / ow unused); the caller applies <= TH_HIGH and the mutual check (:1314-1327)
                                             3: SearchByProjection(KeyFrame*, cv::Mat Scw, vpPoints, vpMatched, th) (:292-405, loop closing): tcw / ow as in 1
                                             (decomposed from Scw by the caller, :301-305), mp_valid = !isBad() && not in spAlreadyFound; the points are
                                             matched IN ORDER -- a feature taken by an earlier point is skipped by later ones (:374) -- and bestDist <=
                                             TH_LOW is applied here; best_idx[i] = the feature point i claimed (-1: none), results in kf_matched */
    const float* xform2;                  /* [F][12] (3x3 row major + 3), variant 2 only */
    int32_t* best_idx; int32_t* best_dist;/* out [F][mp_cap]: key-frame feature to fuse with (-1 / 256 when no candidate passed the gates); the caller
                                             applies bestDist <= TH_LOW and the Replace / AddObservation side effects in order */
    int32_t* kf_matched;                  /* variant 3 only, in/out [F][kf_cap]: vpMatched -- >= 0 = occupied on entry; a feature matched by this call
                                             receives the index of the map point that claimed it */
    int32_t* nmatches;                    /* variant 3 only, out [F] (may be NULL): the function's return value */
} sgs_fuse_batch;
SGS_API int sgs_fuse_search_batch_device(const sgs_fuse_batch* args, int nframes, void* stream);
/* One key frame from host memory (same fields and variants as sgs_fuse_batch; kf = the key frame's mvKeysUn / mvuRight / mDescriptors view).
 * kf_matched_inout [kf->n] and nmatches are used by variant 3 only; xform2 [12] by variant 2 only; inv_level_sigma2 [nlevels] by variant 0 only. */
SGS_API int sgs_fuse_search(const sgs_frame_view* kf, const float* tcw, const float* ow, int nmp, const uint8_t* mp_valid, const float* mp_xyz,
                            const float* mp_normal, const float* mp_min_dist, const float* mp_max_dist, const uint8_t* mp_desc, float th,
                            const float* inv_level_sigma2, int sim3_variant, const float* xform2, int32_t* best_idx, int32_t* best_dist,
                            int32_t* kf_matched_inout, int* nmatches, int device);

typedef struct sgs_init_batch {           /* SearchForInitialization(Frame& F1, Frame& F2, vbPrevMatched, vnMatches12, windowSize), src/ORBmatcher.cc:407-522 */
    sgs_camera cam;                       /* image bounds of F2 (its feature grid); intrinsics unused */
    const sgs_keypoint* f1_kps; const uint8_t* f1_desc; const int32_t* f1_n; int32_t f1_cap;   /* reference frame: mvKeysUn, mDescriptors */
    const sgs_keypoint* f2_kps; const uint8_t* f2_desc; const int32_t* f2_n; int32_t f2_cap;   /* current frame */
    float* prev_xy;                       /* in/out [F][f1_cap][2]: vbPrevMatched (matched entries receive the matched keypoint's position) */
    int32_t window_size; float nnratio; int32_t check_orientation;                             /* 100 / 0.9 / true at src/Tracking.cc:660-661 */
    int32_t* match12;                     /* out [F][f1_cap]: vnMatches12 */
    int32_t* nmatches;                    /* out [F] */
} sgs_init_batch;
SGS_API int sgs_search_for_initialization_batch_device(const sgs_init_batch* args, int nframes, void* stream);
/* One pair from host memory (only n, keys_un, desc and the image bounds of the views are read). */
SGS_API int sgs_search_for_initialization(const sgs_frame_view* f1, const sgs_frame_view* f2, float* prev_xy_inout, int window_size, float nnratio,
                                          int check_orientation, int32_t* match12, int* nmatches, int device);

typedef struct sgs_localmap_batch {       /* SearchByProjection(Frame&, vector<MapPoint*>&, th), src/ORBmatcher.cc:45 */
    sgs_camera cam;
    const sgs_keypoint* cur_kps; const uint8_t* cur_desc; const float* cur_uright; const int32_t* cur_n;
    const uint8_t* mp_inview; const float* proj_x; const float* proj_y; const float* proj_xr; const int32_t* level;
    const float* view_cos; const uint8_t* mp_desc; const uint8_t* mp_obs; const int32_t* mp_n;
    float th, nnratio; int32_t id_base;
    int32_t* f_mp; uint8_t* f_mp_obs; int32_t* nmatches; uint64_t* ncand;
} sgs_localmap_batch;
SGS_API int sgs_match_project_localmap_batch_device(sgs_matcher* m, const sgs_localmap_batch* args, int nframes, void* stream);

/* ------------------------------------------------------------------------------------
 * Optimizer::PoseOptimization(Frame*) (src/Optimizer.cc:239-451): motion-only bundle adjustment after every matcher call, for `nframes`
 * frames (device pointers).  Map point of keypoint i: points_xyz[mp_index[i]] when mp_index is given (-1 = none; this is the cur_mp array the
 * projection matchers write), else points_xyz[i] with has_mp[i].  uright < 0 = monocular observation.  Outputs: the optimised pose, the
 * outlier flags (mvbOutlier) and nInitialCorrespondences - nBad.  Checked against a CPU restatement of the g2o algorithm, itself pinned against the
 * reference's Optimizer.cc + g2o compiled unmodified on an Eigen stand-in (tests/test_optimizer_ref.py, DESIGN.md section 2).  scratch_err: 3 doubles per keypoint, scratch_level: 1 byte per keypoint.
 * ------------------------------------------------------------------------------------ */
typedef struct sgs_poseopt_batch {
    sgs_camera cam;                       /* fx, fy, cx, cy, bf are used */
    const float* tcw_in;                  /* [F][16] pFrame->mTcw */
    const sgs_keypoint* kps; const float* uright; const int32_t* n; int32_t cap;       /* mvKeysUn, mvuRight */
    const uint8_t* has_mp; const int32_t* mp_index; const float* points_xyz; int32_t point_cap;
    float inv_level_sigma2[16];
    float* tcw_out; uint8_t* outlier; int32_t* ninliers;
    double* scratch_err; uint8_t* scratch_level;
    const float* points2_xyz; int32_t id_base2, point2_cap;   /* may be NULL: mp_index values >= id_base2 address points2_xyz[f][id - id_base2] (the ids sgs_match_project_localmap* writes with id_base) */
} sgs_poseopt_batch;
SGS_API int sgs_pose_optimization_batch_device(const sgs_poseopt_batch* args, int nframes, void* stream);
/* host-pointer variant, one frame (outlier flags of keypoints without a map point are left untouched = 0) */
SGS_API int sgs_pose_optimization(const sgs_camera* cam, const float* tcw_in, int n, const sgs_keypoint* kps_un, const float* uright,
                                  const uint8_t* has_mp, const float* xyz, const float* inv_level_sigma2, float* tcw_out, uint8_t* outlier,
                                  int* ninliers, int device);

/* ------------------------------------------------------------------------------------
 * Settings file of the reference (Examples/TUM*.yaml, OpenCV FileStorage "%YAML:1.0" with flat `key: value` lines): the keys the hot path reads
 * at src/Tracking.cc:53-147 (camera, ORB extractor, depth) and src/System.cc:160-162 (detector thresholds).  A missing key reads as 0, like an
 * empty cv::FileNode converted to a number.  Host code, no device involved.
 * ------------------------------------------------------------------------------------ */
typedef struct sgs_settings {
    float fx, fy, cx, cy, k1, k2, p1, p2, k3, bf, fps;   /* Camera.* (Tracking.cc:54-81) */
    int32_t width, height, rgb;                            /* Camera.width / height / RGB */
    float th_depth;                                        /* mThDepth = bf * ThDepth / fx (Tracking.cc:136) */
    float depth_map_factor;                                /* mDepthMapFactor = 1 / DepthMapFactor, or 1 when |DepthMapFactor| < 1e-5 (:142-146) */
    sgs_orb_params orb;                                    /* ORBextractor.* (:113-117) */
    float detection_confidence_threshold, dynamic_detection_confidence_threshold;   /* Detector2D.* (System.cc:160-162) */
} sgs_settings;
SGS_API int sgs_settings_load(const char* path, sgs_settings* out);

/* ------------------------------------------------------------------------------------
 * Bag of words (tracking fallback, Tracking::TrackReferenceKeyFrame src/Tracking.cc:858-904):
 *   sgs_vocabulary_create       : the DBoW2 tree as flat arrays -- parent[i] of node i in node-id order (node 0 = root; DBoW2 appends children
 *                                 to their parent in that order, TemplatedVocabulary.h:1351-1420 / 1467-1508), node descriptors [nnodes][32],
 *                                 node weights (leaves: the TF-IDF word weight).  Word ids number the leaves in node-id order.
 *   sgs_bow_transform_batch_device : TemplatedVocabulary::transform(features, BowVector&, FeatureVector&, levelsup) per feature
 *                                 (Frame::ComputeBoW, src/Frame.cc:421-428, levelsup = 4): word id, word weight, node id at level L - levelsup
 *                                 (0 = root when that level is <= 0).  A feature enters the FeatureVector iff its weight is > 0.
 *   sgs_match_bow_batch_device  : ORBmatcher::SearchByBoW(KeyFrame*, Frame&, vpMapPointMatches) (src/ORBmatcher.cc:159-290) for `nframes`
 *                                 (key frame, frame) pairs: match_f[j] = key-frame feature whose map point goes to frame feature j, or -1.
 * Limits (pinned by tests/test_gpu_bow_cases.py):
 *   - at most 4096 children per vocabulary node (sgs_vocabulary_create returns SGS_ERR_UNSUPPORTED beyond);
 *   - at most 8192 features per side and frame: kf_cap and f_cap in 1 .. 8192 (SGS_ERR_UNSUPPORTED, nothing launched, beyond);
 *   - descriptor rows (vocabulary nodes, d_desc, kf_desc, f_desc) are read as uint4: every descriptor array must be 16-byte aligned;
 *   - levelsup >= L files every feature under node 0 (the root), so the matchers see one bucket;
 *   - counts above the cap are clamped to the cap; rows past a frame's count are not written by the transform, and the matcher sets
 *     every match_f row past the count (up to the cap) to -1.
 * ------------------------------------------------------------------------------------ */
typedef struct sgs_vocabulary sgs_vocabulary;
SGS_API int sgs_vocabulary_create(int device, int k, int L, int nnodes, const int32_t* parent, const uint8_t* node_desc,
                                  const double* node_weight, sgs_vocabulary** out);
/* the same with the node descriptors in DEVICE memory (e.g. the buffer an ncclBroadcast just filled): copied device to device, no host bounce */
SGS_API int sgs_vocabulary_create_device(int device, int k, int L, int nnodes, const int32_t* parent, const uint8_t* d_node_desc,
                                         const double* node_weight, sgs_vocabulary** out);
SGS_API void sgs_vocabulary_destroy(sgs_vocabulary* v);
/* Vocabulary files of the reference: ORBVocabulary::loadFromTextFile / loadFromBinaryFile (Thirdparty/DBoW2/DBoW2/TemplatedVocabulary.h:1351-1420,
 * :1467-1508); like src/System.cc:69-73 a ".txt" suffix selects the text reader.  sgs_vocabulary_parse_file fills the flat arrays sgs_vocabulary_create
 * takes (nnodes counts the implicit root = node 0; all arrays NULL = size query; SGS_ERR_CAPACITY when cap < nnodes) -- what rank 0 broadcasts in a
 * multi-GPU job; sgs_vocabulary_load = parse + create. */
SGS_API int sgs_vocabulary_parse_file(const char* path, int* k, int* L, int* nnodes, int32_t* parent, uint8_t* node_desc, double* node_weight,
                                      uint8_t* is_leaf, int cap);
SGS_API int sgs_vocabulary_load(const char* path, int device, sgs_vocabulary** out);
SGS_API int sgs_bow_transform_batch_device(const sgs_vocabulary* v, const uint8_t* d_desc, const int32_t* d_counts, int cap, int nframes,
                                           int levelsup, int32_t* d_word, double* d_weight, int32_t* d_node, void* stream);
typedef struct sgs_bow_batch {
    const int32_t* kf_node; const double* kf_weight;   /* [F][kf_cap] from sgs_bow_transform_batch_device on the key frame's descriptors */
    const uint8_t* kf_valid;                             /* map point exists && !isBad() */
    const uint8_t* kf_desc; const float* kf_angle; const int32_t* kf_n; int32_t kf_cap;
    const int32_t* f_node; const double* f_weight; const uint8_t* f_desc; const float* f_angle; const int32_t* f_n; int32_t f_cap;
    const uint8_t* f_valid;                              /* NULL for a Frame; key-frame pair: second key frame's map point exists && !isBad() */
    int32_t keyframe_pair;                               /* 1: SearchByBoW(KeyFrame*, KeyFrame*, vpMatches12) (src/ORBmatcher.cc:524-657): strict
                                                            < TH_LOW, match_f is [F][kf_cap], indexed by the FIRST key frame's features */
    float nnratio; int32_t check_orientation;            /* 0.7 / true at src/Tracking.cc:865 */
    /* keyframe_pair == 2: ORBmatcher::SearchForTriangulation(pKF1, pKF2, F12, vMatchedPairs, bOnlyStereo) (src/ORBmatcher.cc:659-827):
     * kf_valid / f_valid mean "the feature has NO map point"; no ratio test; candidates must pass the epipole gate (both sides without
     * stereo) and CheckDistEpipolarLine (:140-157); match_f is [F][kf_cap] like the key-frame pair mode. */
    const uint8_t* kf_stereo; const uint8_t* f_stereo;   /* mvuRight >= 0 */
    const float* kf_xy; const float* f_xy;               /* mvKeysUn[i].pt, [F][cap][2] */
    const int32_t* f_octave;                             /* mvKeysUn[i].octave of the second key frame */
    const float* F12;                                    /* [F][9] float, row major */
    const float* epipole;                                /* [F][2]: (ex, ey) of src/ORBmatcher.cc:667-672 */
    float level_sigma2[16], scale_factors[16];           /* pKF2->mvLevelSigma2 / mvScaleFactors */
    int32_t only_stereo;
    int32_t* match_f;                                    /* out [F][f_cap] (or [F][kf_cap], see keyframe_pair) */
    int32_t* nmatches;                                   /* out [F] */
} sgs_bow_batch;
SGS_API int sgs_match_bow_batch_device(const sgs_bow_batch* args, int nframes, void* stream);
/* host-pointer variants: one descriptor set / one (key frame, frame) pair */
SGS_API int sgs_bow_transform(const sgs_vocabulary* v, const uint8_t* desc, int n, int levelsup, int32_t* word, double* weight, int32_t* node);
SGS_API int sgs_match_bow(int nkf, const int32_t* kf_node, const double* kf_weight, const uint8_t* kf_valid, const uint8_t* kf_desc,
                          const float* kf_angle, int nf, const int32_t* f_node, const double* f_weight, const uint8_t* f_desc,
                          const float* f_angle, float nnratio, int check_orientation, int32_t* match_f, int* nmatches, int device);
/* Two key frames from host memory.  mode 1: SearchByBoW(KeyFrame*, KeyFrame*, vpMatches12) (valid = map point exists && !isBad()); mode 2:
 * SearchForTriangulation (valid = the feature has NO map point; the stereo flags, positions, second frame's octaves, F12 [9], epipole [2], the
 * second key frame's mvLevelSigma2 / mvScaleFactors [nlevels] and only_stereo are needed).  match12[i1] = feature of the second key frame or -1. */
SGS_API int sgs_match_bow_keyframes(int mode, int n1, const int32_t* node1, const double* weight1, const uint8_t* valid1, const uint8_t* desc1, const float* angle1,
                                    int n2, const int32_t* node2, const double* weight2, const uint8_t* valid2, const uint8_t* desc2, const float* angle2,
                                    float nnratio, int check_orientation, const uint8_t* stereo1, const uint8_t* stereo2, const float* xy1, const float* xy2,
                                    const int32_t* octave2, const float* F12, const float* epipole, const float* level_sigma2, const float* scale_factors, int nlevels,
                                    int only_stereo, int32_t* match12, int* nmatches, int device);

/* ------------------------------------------------------------------------------------
 * Frame geometry between the extractor and the matchers (device pointers, `nframes` frames, work enqueued on `stream`):
 *   sgs_stereo_from_depth_batch_device : Frame::ComputeStereoFromRGBD (src/Frame.cc:893-914).  d_depth: float depth images
 *       [F][h][depth_pitch] (elements; depth_frame_stride 0 shares one image); d_kps_un NULL = undistorted keypoints equal the
 *       distorted ones; outputs d_u_right [F][cap] (mvuRight, -1 without depth) and optional d_depth_out (mvDepth).
 *   sgs_frustum_batch_device           : Frame::isInFrustum (src/Frame.cc:296-352) + MapPoint::PredictScale (src/MapPoint.cc:400-418)
 *       for every local-map point: fills the per-point inputs of sgs_match_project_localmap* (mbTrackInView, mTrackProjX/Y/XR,
 *       mnTrackScaleLevel, mTrackViewCos).  mp_min_dist / mp_max_dist are mfMinDistance / mfMaxDistance (the 0.8 / 1.2 factors
 *       of Get{Min,Max}DistanceInvariance are applied inside); log(scaleFactor) is taken from cam.scale_factors[1].
 * ------------------------------------------------------------------------------------ */
typedef struct sgs_frustum_batch {
    sgs_camera cam;
    const float* tcw;             /* [F][16] row-major */
    const float* mp_xyz;          /* [F][point_cap][3]  GetWorldPos() */
    const float* mp_normal;       /* [F][point_cap][3]  GetNormal() */
    const float* mp_min_dist; const float* mp_max_dist;   /* [F][point_cap] */
    const int32_t* mp_n;          /* [F] */
    int32_t point_cap;
    float viewing_cos_limit;      /* 0.5 at src/Tracking.cc:1282 */
    uint8_t* mp_inview; float* proj_x; float* proj_y; float* proj_xr; int32_t* level; float* view_cos;   /* out [F][point_cap] */
} sgs_frustum_batch;
SGS_API int sgs_stereo_from_depth_batch_device(const sgs_keypoint* d_kps, const sgs_keypoint* d_kps_un, const int32_t* d_counts, int cap,
                                               int nframes, const float* d_depth, size_t depth_frame_stride, int depth_pitch, float bf,
                                               float* d_u_right, float* d_depth_out, void* stream);
SGS_API int sgs_frustum_batch_device(const sgs_frustum_batch* args, int nframes, void* stream);
/* Frame::UndistortKeyPoints (src/Frame.cc:654-684) = cv::undistortPoints(pts, K, distCoef, Mat(), K), distCoef = (k1, k2, p1, p2, k3);
 * k1 == 0 copies the keypoints, like the reference.  sgs_image_bounds: Frame::ComputeImageBounds (:686-714) -> min_x, min_y, max_x, max_y. */
SGS_API int sgs_undistort_batch_device(const sgs_keypoint* d_kps, const int32_t* d_counts, int cap, int nframes, float fx, float fy, float cx,
                                       float cy, const float* dist_coef5, sgs_keypoint* d_kps_un, void* stream);
SGS_API int sgs_undistort_points(const float* xy, int n, float fx, float fy, float cx, float cy, const float* dist_coef5, float* out_xy,
                                 int device);
SGS_API int sgs_image_bounds(int width, int height, float fx, float fy, float cx, float cy, const float* dist_coef5, float* bounds4,
                             int device);
/* host-pointer variant, one frame, n points (arrays of n / 3 n elements) */
SGS_API int sgs_frustum(const sgs_camera* cam, const float* tcw, int n, const float* xyz, const float* normal, const float* min_dist,
                        const float* max_dist, float viewing_cos_limit, uint8_t* inview, float* proj_x, float* proj_y, float* proj_xr,
                        int32_t* level, float* view_cos, int device);

/* ------------------------------------------------------------------------------------
 * Frame: dynamic-feature rejection, geometry half
 * Frame::RmDynamicPointWithSemanticAndGeometry "version3" loop (src/Frame.cc:560-604) +
 * CheckEpiLineDistToRmDynamicPoint (:613-627) + isInDynamicRegion (:629-652).
 *   cur_xy / prev_xy : mvKeys[i].pt and the LK-tracked previous point (2 floats each)
 *   F                : 3x3 row-major double from findFundamentalMat (NULL == empty matrix: keep all, quirk Q11)
 *   boxes            : mvPotentialDynamicBorderForRmDynamicFeature; have_dyn = mbHaveDynamicObjectForRmDynamicFeature
 *   keep[i]          : 1 iff keypoint i passes its epipolar test; dist (may be NULL): the distances (double)
 *   *nkeep           : Cur_keypoint_sum (the reference's return value)
 *   *restored        : 1 when the restore-all branch fired (:599-602): the caller keeps every keypoint
 * ------------------------------------------------------------------------------------ */
SGS_API int sgs_dynreject(const float* cur_xy, const float* prev_xy, int n, const double* F, const sgs_rect* boxes,
                          int nboxes, int have_dyn, int nfeatures, uint8_t* keep, double* dist, int* nkeep,
                          int* restored, int device);

/* Fused device-side variant used by the batched pipeline: computes the verdicts and applies them as an ORDERED compaction
 * of keypoints and descriptor rows (the erase loop :563-597) for `nframes` frames resident on the device.
 *   in : d_kps [F][cap], d_desc [F][cap][32], d_counts [F], d_prev_xy [F][cap][2], d_F [F][9] (double; a NaN in F[0] marks
 *        an empty matrix), d_boxes [F][max_boxes], d_nboxes [F], d_have_dyn [F] (uint8); a frame uses its first
 *        d_counts[f] keypoints and d_nboxes[f] boxes, each clamped to [0, cap] and [0, max_boxes]
 *   out: d_kps_out / d_desc_out / d_counts_out (same shapes; when the restore-all branch fires the frame is copied
 *        unchanged), d_keep [F][cap] (per-point verdicts, may be NULL); rows at and past d_counts_out[f] and verdicts
 *        past the clamped count are not written.  cap * 4 bytes must fit in 160 KB of shared memory, else
 *        SGS_ERR_UNSUPPORTED and nothing is enqueued. */
SGS_API int sgs_dynreject_batch_device(const sgs_keypoint* d_kps, const uint8_t* d_desc, const int32_t* d_counts, int cap,
                                       int nframes, const float* d_prev_xy, const double* d_F, const sgs_rect* d_boxes,
                                       const int32_t* d_nboxes, int max_boxes, const uint8_t* d_have_dyn, int nfeatures,
                                       sgs_keypoint* d_kps_out, uint8_t* d_desc_out, int32_t* d_counts_out, uint8_t* d_keep,
                                       void* stream);

/* ------------------------------------------------------------------------------------
 * cv::findFundamentalMat(points1, points2, cv::FM_RANSAC, 1.0, 0.99) as called at src/Frame.cc:469-472 (points1 = current
 * keypoints, points2 = their LK-tracked positions in the previous frame), including the selection in front of it
 * (src/Frame.cc:454-468: when the previous frame had dynamic boxes and more than 20 pairs have their PREVIOUS point outside
 * them, only those pairs are used).  F: 3x3 row-major double scaled to F33 = 1; a NaN in F[0] == empty matrix.
 *   All three branches of OpenCV's function are on the device: >= 15 pairs RANSAC, 8..14 pairs LMedS (300 fixed samples, smallest median
 *   error), exactly 7 pairs the 7-point solver itself (first of its stacked solutions = what the reference reads), fewer: empty matrix.
 *   info (4 x int32, may be NULL): pairs used, inliers of F, iterations run, status (0 ok, 1 fewer than 7 pairs, 2 no model found,
 *   3 no previous frame).
 *   sgs_fundamental_ransac       : host pointers, one point set, no box selection; mask [n] may be NULL.
 *   sgs_fundamental_batch_device : device pointers, `nframes` frames: d_kps [F][cap], d_prev_xy [F][cap][2], d_counts [F],
 *                                  previous-frame boxes d_prev_boxes [F][max_boxes] / d_prev_nboxes [F] / d_prev_have_dyn [F]
 *                                  (all three may be NULL); d_prev_index (may be NULL): row of the batch whose boxes are the
 *                                  previous frame's, d_prev_index[f] == f marks "no previous frame"; d_F [F][9], d_info [F][4].
 *                                  With d_prev_index the reference's file-scope state is followed: the flag of a row that is itself a
 *                                  stream's first frame counts as false (src/Frame.cc:154-162, 482-491: the first frame never runs the
 *                                  rejection, so it never records "previous frame had dynamic objects"; quirk Q13 in DESIGN.md).
 * ------------------------------------------------------------------------------------ */
SGS_API int sgs_fundamental_ransac(const float* pts1_xy, const float* pts2_xy, int n, double ransac_thresh, double confidence,
                                   int max_iters, double* F, uint8_t* mask, int32_t* info, int device);
SGS_API int sgs_fundamental_batch_device(const sgs_keypoint* d_kps, const float* d_prev_xy, const int32_t* d_counts, int cap,
                                         int nframes, const sgs_rect* d_prev_boxes, const int32_t* d_prev_nboxes,
                                         const uint8_t* d_prev_have_dyn, int max_boxes, const int32_t* d_prev_index,
                                         double ransac_thresh, double confidence, int max_iters, double* d_F, int32_t* d_info,
                                         void* stream);

/* ------------------------------------------------------------------------------------
 * Batched front end with HOST buffers: the part of Frame::Frame (RGB-D ctor, src/Frame.cc:129-198) and
 * Tracking::TrackWithMotionModel (src/Tracking.cc:906-931) that runs on the GPU, for `nframes` independent frames.
 *   sgs_tracker_extract : ExtractORB (src/Frame.cc:146).  Keypoints/descriptors also return to the host.
 *                         calcOpticalFlowPyrLK + findFundamentalMat (src/Frame.cc:445-472) run on the device in sgs_tracker_track_lk
 *                         and sgs_tracker_step; sgs_tracker_track takes their results (prev_xy, F) from the caller instead.
 *   sgs_tracker_track   : dyn-reject verdicts + ordered compaction of keypoints, descriptors and u_right
 *                         (src/Frame.cc:560-604) on the device-resident extraction results, then
 *                         SearchByProjection(cur, last, th, mono) (src/ORBmatcher.cc:1332-1472).
 * Array shapes: prev_xy [F][cap][2], u_right [F][cap] (mvuRight of the UNfiltered keypoints), F [F][9] (NaN in F[0] ==
 * empty matrix), boxes [F][max_boxes], last_* [F][point_cap](..), tcw_* [F][16]; outputs kps_out [F][cap],
 * desc_out [F][cap][32], u_right_out [F][cap] (may be NULL), counts_out [F], cur_mp_out [F][cap], nmatches_out [F].
 * Pinned host memory is copied without staging.  The host-buffer calls (sgs_tracker_track, _track_lk, _step, _step_rgbd)
 * upload u_right and the last-frame arrays on a copy stream of the tracker that is not ordered after work still pending
 * from the device-pointer calls below: synchronise their stream before a host-buffer call on the same tracker.
 * ------------------------------------------------------------------------------------ */
typedef struct sgs_tracker sgs_tracker;
SGS_API int sgs_tracker_create(const sgs_orb_params* params, int width, int height, int max_batch, int point_cap,
                               int max_boxes, const sgs_camera* cam, int device, sgs_tracker** out);
SGS_API void sgs_tracker_destroy(sgs_tracker* t);
SGS_API int sgs_tracker_max_keypoints(const sgs_tracker* t, int* cap);
SGS_API int sgs_tracker_extract(sgs_tracker* t, const uint8_t* gray, int nframes, size_t frame_stride, int pitch,
                                sgs_keypoint* kps, uint8_t* desc, int cap, int* n);
SGS_API int sgs_tracker_track(sgs_tracker* t, int nframes, const float* prev_xy, const float* u_right, const double* F,
                              const sgs_rect* boxes, const int32_t* nboxes, const uint8_t* have_dyn, const float* last_xyz,
                              const uint8_t* last_desc, const uint8_t* last_flags, const int32_t* last_octave,
                              const float* last_angle, const int32_t* last_n, const float* tcw_cur, const float* tcw_last,
                              float th, int mono, int check_orientation, sgs_keypoint* kps_out, uint8_t* desc_out,
                              float* u_right_out, int32_t* counts_out, int32_t* cur_mp_out, int32_t* nmatches_out);

/* Device-resident variants: every pointer is a DEVICE pointer, work is enqueued on `stream` without synchronising and
 * the results stay in the handle (sgs_tracker_results_device: kps [F][cap], desc, u_right, counts [F], cur_mp [F][cap],
 * nmatches [F], ncand [F] = candidates examined by the matcher, for the roofline byte count). */
SGS_API int sgs_tracker_extract_device(sgs_tracker* t, const uint8_t* d_gray, int nframes, size_t frame_stride, int pitch,
                                       void* stream);
SGS_API int sgs_tracker_track_device(sgs_tracker* t, int nframes, const float* prev_xy, const float* u_right, const double* F,
                                     const sgs_rect* boxes, const int32_t* nboxes, const uint8_t* have_dyn,
                                     const float* last_xyz, const uint8_t* last_desc, const uint8_t* last_flags,
                                     const int32_t* last_octave, const float* last_angle, const int32_t* last_n,
                                     const float* tcw_cur, const float* tcw_last, float th, int mono, int check_orientation,
                                     void* stream);
SGS_API int sgs_tracker_results_device(const sgs_tracker* t, const sgs_keypoint** kps, const uint8_t** desc,
                                       const float** u_right, const int32_t** counts, const int32_t** cur_mp,
                                       const int32_t** nmatches, const uint64_t** ncand);
SGS_API sgs_extractor* sgs_tracker_extractor(sgs_tracker* t);  /* the extractor owned by the tracker (tables, profiling) */
/* LK inside the tracker: tracks the keypoints of the last extract call into the previous image of each frame
 * (d_frames[d_prev_index[f]], the same device batch that was extracted) and keeps the result as the `prev_xy` of the next
 * sgs_tracker_track_device call made with prev_xy == NULL.  sgs_tracker_prev_xy_device returns that buffer [F][cap][2]. */
SGS_API int sgs_tracker_lk_device(sgs_tracker* t, const uint8_t* d_frames, int nframes, size_t frame_stride, int pitch,
                                  const int32_t* d_prev_index, void* stream);
SGS_API int sgs_tracker_prev_xy_device(const sgs_tracker* t, const float** d_prev_xy);
/* findFundamentalMat on the GPU for the frames of the last extract call, from the keypoints and the LK result held by the
 * tracker (sgs_tracker_lk_device must have run).  d_boxes / d_nboxes / d_have_dyn are the per-frame detector boxes of the BATCH
 * (the same arrays sgs_tracker_track_device takes); d_prev_index [F] selects, per frame, the row that is its previous frame
 * (== own row: no previous frame, F = NaN -> every keypoint is kept).  The result is used by the next
 * sgs_tracker_track_device / sgs_tracker_track_lk call made with F == NULL; sgs_tracker_fundamental_device_ptr exposes it
 * (d_F [F][9] double, d_info [F][4] int32, see sgs_fundamental_batch_device). */
SGS_API int sgs_tracker_fundamental_device(sgs_tracker* t, int nframes, const sgs_rect* d_boxes, const int32_t* d_nboxes,
                                           const uint8_t* d_have_dyn, const int32_t* d_prev_index, void* stream);
SGS_API int sgs_tracker_fundamental_device_ptr(const sgs_tracker* t, const double** d_F, const int32_t** d_info);
/* Frame::ComputeStereoFromRGBD for the frames of the last extract call (see sgs_stereo_from_depth_batch_device); the result is the
 * u_right used by the next sgs_tracker_track_device call made with u_right == NULL. */
SGS_API int sgs_tracker_stereo_device(sgs_tracker* t, int nframes, const float* d_depth, size_t depth_frame_stride, int depth_pitch,
                                      void* stream);
/* Host-buffer variant of sgs_tracker_track with the LK stage on the GPU: prev_index [F] (host) replaces prev_xy; the frames are
 * the ones uploaded by the preceding sgs_tracker_extract call (they are still resident on the device). */
SGS_API int sgs_tracker_track_lk(sgs_tracker* t, int nframes, const int32_t* prev_index, const float* u_right, const double* F,
                                 const sgs_rect* boxes, const int32_t* nboxes, const uint8_t* have_dyn, const float* last_xyz,
                                 const uint8_t* last_desc, const uint8_t* last_flags, const int32_t* last_octave,
                                 const float* last_angle, const int32_t* last_n, const float* tcw_cur, const float* tcw_last,
                                 float th, int mono, int check_orientation, sgs_keypoint* kps_out, uint8_t* desc_out,
                                 float* u_right_out, int32_t* counts_out, int32_t* cur_mp_out, int32_t* nmatches_out);
/* level 0 of the extractor's own pyramid (the frames of the last host-API extract call), for device-side consumers */
SGS_API int sgs_extractor_level0_device(const sgs_extractor* ex, const uint8_t** d_frames, int* pitch, size_t* frame_stride);

/* ------------------------------------------------------------------------------------
 * cv::calcOpticalFlowPyrLK as called at src/Frame.cc:445 (window 21x21, maxLevel 3, COUNT|EPS 30 / 0.01): tracks the CURRENT
 * frame's keypoints into the PREVIOUS gray image.  Window sums are exact integer sums, so positions equal bit for bit the exact-sum
 * restatement in tests/lk_exact.py; that restatement agrees with OpenCV to ~1e-4 px (OpenCV sums in float, in SIMD order; tolerance
 * in tests/test_gpu_lk.py).  status/err are not produced (the reference ignores them).
 *   sgs_lk_track              : one host image pair, n points (x, y) -> out (x, y)
 *   sgs_lk_track_batch_device : `nframes` device image pairs; points are the keypoints d_kps [F][cap] (counts [F]); writes
 *                               d_prev_xy [F][cap][2] -- the `prev_xy` input of the dyn-reject stage.  The previous images are
 *                               either a second array d_prev [F] or, when d_prev_index [F] is given, frames of d_cur itself
 *                               (previous image of frame f = d_cur[d_prev_index[f]]; consecutive frames of streams in one batch)
 * ------------------------------------------------------------------------------------ */
typedef struct sgs_lk sgs_lk;
SGS_API int sgs_lk_create(int width, int height, int max_batch, int device, sgs_lk** out);
SGS_API void sgs_lk_destroy(sgs_lk* k);
SGS_API int sgs_lk_track(sgs_lk* k, const uint8_t* cur, const uint8_t* prev, int pitch, const float* pts, int n, float* out);
SGS_API int sgs_lk_track_batch_device(sgs_lk* k, const uint8_t* d_cur, const uint8_t* d_prev, const int32_t* d_prev_index,
                                      int nframes, size_t frame_stride, int pitch, const sgs_keypoint* d_kps,
                                      const int32_t* d_counts, int cap, float* d_prev_xy, void* stream);
/* parity accessor: pyramid level (1..3) of frame 0 of the last call; which = 0 current image, 1 previous image */
SGS_API int sgs_lk_read_level(sgs_lk* k, int which, int level, uint8_t* out, int out_pitch);
/* parity accessor: the whole padded level (0..max_level) of batch frame `frame` as the tracker reads it, border included, after the
 * stream of the last call has finished.  img [h + 2 pad][w + 2 pad] (REFLECT_101 border); for which == 0 also, when deriv != NULL,
 * the derivative plane [h + 2 pad][w + 2 pad] as dx | dy << 16 (int16 halves, zero border); *pad (may be NULL) = the border width.
 * which = 1 (the previous images) is only built by calls given d_prev, not d_prev_index. */
SGS_API int sgs_lk_read_padded(sgs_lk* k, int which, int level, int frame, uint8_t* img, uint32_t* deriv, int* pad);
/* Stage timing with CUDA events on the launching stream, like sgs_extractor_set_profiling / _stage_times:
 * ms_total2 = accumulated {pyramid build (cv::pyrDown levels), lk_track_kernel} over *ncalls calls. */
SGS_API int sgs_lk_set_profiling(sgs_lk* k, int enable);
SGS_API int sgs_lk_stage_times(sgs_lk* k, double* ms_total2, int* ncalls);
SGS_API sgs_lk* sgs_tracker_lk(sgs_tracker* t);                 /* the LK handle owned by the tracker (profiling) */

/* harness helper: synchronous device -> host copy of a buffer returned by one of the *_device accessors */
SGS_API int sgs_memcpy_d2h(void* dst, const void* d_src, size_t bytes);

/* ---- measurement hooks (bench.py): per-stage device time of the extractor from CUDA events recorded on the launching
 * stream.  Stages: 0 pyramid, 1 FAST, 2 quadtree, 3 blur, 4 orientation+BRIEF.  ms_total5 accumulates over `ncalls`. */
SGS_API int sgs_extractor_set_profiling(sgs_extractor* ex, int enable);
SGS_API int sgs_extractor_stage_times(sgs_extractor* ex, double* ms_total5, int* ncalls);

/* ------------------------------------------------------------------------------------
 * The rest of the tracking thread's per-frame chain on the device, after sgs_tracker_track_device / sgs_tracker_track_lk / sgs_tracker_step
 * (whose SearchByProjection(cur, last, th) matches are still on the device):
 *   Tracking::TrackWithMotionModel, src/Tracking.cc:926-967 : < 20 matches -> the search again with 2 th on cleared matches (:927-931);
 *       Optimizer::PoseOptimization (:937); outliers lose their map point (:940-957); nmatches / nmatchesMap;
 *   Tracking::TrackLocalMap, :969-1000 with SearchLocalPoints, :1262-1312 : map points already matched in the frame (the discarded outliers
 *       included, their mnLastFrameSeen is the frame's id) are left out; Frame::isInFrustum(pMP, 0.5) + MapPoint::PredictScale for the rest;
 *       ORBmatcher(0.8).SearchByProjection(F, mvpLocalMapPoints, th_local); Optimizer::PoseOptimization again; mnMatchesInliers.
 * UpdateLocalMap (which key frames / points form the local map) stays with the caller: the local map arrives as arrays, one list per frame.
 * Ids written to f_mp: 0 .. point_cap-1 = the last-frame point (as after sgs_tracker_track_*), point_cap + j = local-map point j.
 * stats [F][8]: 0 nmatches of the first search, 1 retried with 2 th (0/1), 2 nmatches after the retry, 3 nmatches after discarding outliers,
 *   4 nmatchesMap, 5 nToMatch (local-map points in the frustum), 6 matches added by the local search, 7 mnMatchesInliers.
 * ------------------------------------------------------------------------------------ */
typedef struct sgs_posechain_batch {
    /* the arguments sgs_tracker_track_device took (needed for the retry and as the points of the first PoseOptimization) */
    const float* last_xyz; const uint8_t* last_desc; const uint8_t* last_flags; const int32_t* last_octave; const float* last_angle; const int32_t* last_n;
    const float* tcw_cur; const float* tcw_last; float th; int32_t mono, check_orientation;
    const int32_t* last_local_id;     /* [F][point_cap]: index of last-frame point i in this frame's local-map list, -1 = not in it (may be NULL = none is) */
    /* local map of every frame: [F][mp_cap] */
    const float* mp_xyz; const float* mp_normal; const float* mp_min_dist; const float* mp_max_dist; const uint8_t* mp_desc;
    const uint8_t* mp_valid;          /* !isBad() */
    const uint8_t* mp_obs;            /* Observations() > 0 */
    const int32_t* mp_n; int32_t mp_cap;
    float th_local, nnratio_local;    /* 3 (RGB-D; 1 otherwise; 5 after a relocalisation) and 0.8, src/Tracking.cc:1303-1310 */
    float inv_level_sigma2[16];       /* Frame::mvInvLevelSigma2 */
    /* outputs (device) */
    float* tcw_motion; float* tcw_final;      /* [F][16] pose after TrackWithMotionModel / after TrackLocalMap */
    int32_t* f_mp;                    /* [F][cap] final mvpMapPoints as ids (see above) */
    uint8_t* outlier;                 /* [F][cap] mvbOutlier after the second PoseOptimization */
    int32_t* stats;                   /* [F][8] */
} sgs_posechain_batch;
SGS_API int sgs_tracker_pose_chain_device(sgs_tracker* t, const sgs_posechain_batch* args, int nframes, void* stream);

/* ------------------------------------------------------------------------------------------------------------------------------
 * Object detector: Detector2D (src/Detector2D.cc:16-89, include/Detector2D.h:29-80) -- ncnn forward of the MobileNetV3-SSDLite graph
 * Thirdparty/ncnn_model/mobilenetv3_ssdlite_voc.{param,bin} and the reference's post-processing of the "detection_out" rows.
 * The handle reads the ncnn text graph + weight blob itself (same two files the reference loads at Detector2D.cc:25-26) and runs the
 * layers as FP32 CUDA kernels on a batch of frames.  ncnn is an unpinned, un-vendored dependency of the reference: the layer semantics
 * are restated from its published definitions (parity unpinned, see DESIGN.md).
 * ------------------------------------------------------------------------------------------------------------------------------ */
typedef struct sgs_detector sgs_detector;
typedef struct sgs_object2d {   /* Object2D, include/Detector2D.h:29-37 (name = class_names[id]) */
    int32_t id;
    float prob;
    sgs_rect rect;
} sgs_object2d;

/* Detector2D::Detector2D(detection_confidence_threshold, dynamic_detection_confidence_threshold) + load_param/load_model.
 * max_frames = largest batch one sgs_detector_detect_device call may carry.  flags: bit 0 = diagnostic mode (every layer its own kernel,
 * every intermediate blob kept, readable with sgs_detector_blob); bit 1 = plan only (parse, shapes, kernel list and activation pool are
 * built, no device is touched; the handle serves sgs_detector_info / sgs_detector_describe only).
 * The 1x1 convolutions (90 % of the MACs) run as a TMA-fed wgmma GEMM on [frame][h][w][c] activations with error-compensated TF32 operands
 * (three wgmma per 8-wide k-step, FP32 accumulate: ~1e-6 relative); there is no other GEMM path. */
SGS_API int sgs_detector_create(const char* param_path, const char* bin_path, int max_frames, float detection_confidence_threshold,
                                float dynamic_detection_confidence_threshold, int flags, int device, sgs_detector** out);
SGS_API void sgs_detector_destroy(sgs_detector* d);
/* Sizes fixed by the graph: rows_cap = DetectionOutput keep_top_k (rows per frame), input_size = 300 (Detector2D.h:70). */
SGS_API int sgs_detector_info(const sgs_detector* d, int* rows_cap, int* input_size, int* num_layers, int* num_kernels_per_batch);

/* Detector2D::detect (src/Detector2D.cc:34-89) on nframes interleaved 8-bit 3-channel frames resident in device memory (frame f starts at
 * d_rgb + f*frame_stride, rows pitch bytes apart; channel order is taken as given, Detector2D.cc:39 passes PIXEL_RGB = no swap).
 * Outputs (device pointers, any may be NULL):
 *   d_rows     [F][rows_cap][6]  detection_out rows [label, score, xmin, ymin, xmax, ymax] (normalised);  d_nrows [F]
 *   d_objects  [F][rows_cap]     every accepted row in detection order (what draw_objects sees, :66);       d_nobjects [F]
 *   d_dyn_map  [F][max_boxes]    mvPotentialDynamicBorderForMapping (:70);                                  d_ndyn_map [F]
 *   d_dyn_rm   [F][max_boxes]    mvPotentialDynamicBorderForRmDynamicFeature (:74), d_ndyn_rm [F] -- the layout sgs_dynreject_batch_device /
 *                                sgs_tracker_* take as d_boxes / d_nboxes;  d_have_dyn_rm [F] (uint8) = the flag the FRAME ends up with
 *                                (src/Frame.cc:482-491): Detector2D's mbHaveDynamicObjectForRmDynamicFeature (:73) is copied only when mvObjects2D
 *                                -- the NON-person objects -- is not empty; otherwise the Frame member is never written (include/Frame.h:112,
 *                                uninitialised in the reference; defined as false here, quirk Q12) and the previous-frame flag is false.
 * Person boxes beyond max_boxes are not written: d_ndyn_* are clamped to max_boxes and d_status[f] (may be NULL) is set to 1. */
SGS_API int sgs_detector_detect_device(sgs_detector* d, const uint8_t* d_rgb, int64_t frame_stride, int pitch, int width, int height,
                                       int nframes, float* d_rows, int32_t* d_nrows, sgs_object2d* d_objects, int32_t* d_nobjects,
                                       sgs_rect* d_dyn_map, int32_t* d_ndyn_map, sgs_rect* d_dyn_rm, int32_t* d_ndyn_rm,
                                       uint8_t* d_have_dyn_rm, int max_boxes, int32_t* d_status, void* stream);
/* One frame from host memory: objects[0..*n) = accepted rows in detection order (persons included, id 15).  SGS_ERR_CAPACITY with
 * *n = required when cap is too small. */
SGS_API int sgs_detect(sgs_detector* d, const uint8_t* rgb, int width, int height, int pitch, sgs_object2d* objects, int cap, int* n);
/* Detector inside the tracking step (src/Tracking.cc:288-307 hands the colour image to the detector thread, src/Frame.cc:478-500 joins it before the
 * rejection).  sgs_tracker_detect_device runs Detector2D::detect on device frames and leaves the person boxes in the tracker's own box arrays
 * (sgs_tracker_boxes_device), which sgs_tracker_fundamental_device / sgs_tracker_track_device use when called with boxes / nboxes / have_dyn == NULL.
 * stream == NULL: the tracker's detector stream.
 * sgs_tracker_step is the whole front end with HOST buffers: colour frames -> detector on its own stream; gray frames -> ORB extract -> LK ->
 * (join) findFundamentalMat -> dyn-reject + compaction -> SearchByProjection(cur, last); uploads overlap the kernels, one synchronisation at the end.
 * Shapes as for sgs_tracker_track_lk; rgb: interleaved 8-bit frames (rgb_pitch bytes per row); boxes_out [F][max_boxes] / nboxes_out [F] / have_out [F]
 * (may be NULL) return the boxes the rejection used. */
SGS_API int sgs_tracker_detect_device(sgs_tracker* t, sgs_detector* det, const uint8_t* d_rgb, int64_t frame_stride, int pitch, int width, int height,
                                      int nframes, void* stream);
SGS_API int sgs_tracker_boxes_device(const sgs_tracker* t, const sgs_rect** d_boxes, const int32_t** d_nboxes, const uint8_t** d_have_dyn);
SGS_API int sgs_tracker_step(sgs_tracker* t, sgs_detector* det, const uint8_t* gray, size_t gray_stride, int gray_pitch, const uint8_t* rgb,
                             size_t rgb_stride, int rgb_pitch, int nframes, const int32_t* prev_index, const float* u_right, const float* last_xyz,
                             const uint8_t* last_desc, const uint8_t* last_flags, const int32_t* last_octave, const float* last_angle,
                             const int32_t* last_n, const float* tcw_cur, const float* tcw_last, float th, int mono, int check_orientation,
                             sgs_keypoint* kps_out, uint8_t* desc_out, float* u_right_out, int32_t* counts_out, int32_t* cur_mp_out,
                             int32_t* nmatches_out, sgs_rect* boxes_out, int32_t* nboxes_out, uint8_t* have_out);

/* ------------------------------------------------------------------------------------------------------------------------------
 * RGB-D frames as the camera delivers them: Tracking::GrabImageRGBD (src/Tracking.cc:206-251) + the RGB-D Frame constructor (src/Frame.cc:129-198)
 * + TrackWithMotionModel's matcher call (src/Tracking.cc:906-924).  The format block is filled from the sgs_settings the caller loads:
 *   rgb              Camera.RGB: != 0 -> cvtColor(CV_RGB2GRAY) (byte 0 gets the R weight), 0 -> CV_BGR2GRAY.  Followed literally: a caller that
 *                    reads BGR files (imread) with a settings file saying RGB: 1 gets what the reference computes on those bytes.
 *   depth_type       0: uint16 raw depth, 1: float32 (anything else is SGS_ERR_INVALID)
 *   depth_map_factor mDepthMapFactor (sgs_settings.depth_map_factor): depth = (float)raw * depth_map_factor; finite and > 0
 *   dist_coef        k1 k2 p1 p2 k3 of Frame::UndistortKeyPoints (k1 == 0: mvKeysUn = mvKeys)
 * The intrinsics are the handle's sgs_camera (its image bounds come from sgs_image_bounds with the same coefficients).
 * ------------------------------------------------------------------------------------------------------------------------------ */
typedef struct sgs_rgbd_format {
    int32_t rgb;
    int32_t depth_type;
    float depth_map_factor;
    float dist_coef[5];
} sgs_rgbd_format;
/* The two conversions alone, on device frames (all pitches and frame strides in bytes):
 *   gray  [F] = cvtColor(rgb [F], RGB2GRAY / BGR2GRAY) of interleaved 8-bit 3-channel frames: Y = (9798 R + 19235 G + 3735 B + 2^14) >> 15
 *   depth_out [F] = raw depth [F] converted to float32 metres, (float)raw * depth_map_factor
 * d_rgb / d_gray may both be NULL (depth only), d_depth / d_depth_out may both be NULL (gray only).  One launch on `stream`. */
SGS_API int sgs_grab_rgbd_batch_device(const uint8_t* d_rgb, size_t rgb_stride, int rgb_pitch, const void* d_depth, size_t depth_stride, int depth_pitch,
                                       const sgs_rgbd_format* fmt, int width, int height, int nframes, uint8_t* d_gray, size_t gray_stride, int gray_pitch,
                                       float* d_depth_out, size_t depth_out_stride, int depth_out_pitch, void* stream);
/* The whole RGB-D front end on device frames, enqueued on `stream` (NULL: the tracker's stream) without synchronising:
 *   colour frames -> detector (the tracker's detector stream) -------------------------------------------------------------\
 *   colour + raw depth -> gray (into the extractor's level 0) + float depth -> ORB extract -> LK -> join -> findFundamentalMat ->
 *   UndistortKeyPoints -> ComputeStereoFromRGBD (depth at mvKeys, uRight from mvKeysUn.x) -> dyn-reject + ordered compaction of keypoints,
 *   descriptors, mvKeysUn, mvuRight and mvDepth -> SearchByProjection(cur, last) on mvKeysUn.
 * d_rgb: interleaved 8-bit frames, d_depth: uint16 or float32 frames (pitches / strides in bytes, multiples of the depth element size); a float32 depth
 * with factor 1 is read in place.  d_prev_index [F] (device; values in [0, nframes), not checked) and the last-frame arrays are those of
 * sgs_tracker_lk_device / sgs_tracker_track_device.  The results are those of sgs_tracker_results_device (u_right = mvuRight of the kept keypoints) and
 * sgs_tracker_frame_device; the next sgs_tracker_pose_chain_device reads mvKeysUn. */
SGS_API int sgs_tracker_step_rgbd_device(sgs_tracker* t, sgs_detector* det, const uint8_t* d_rgb, size_t rgb_stride, int rgb_pitch, const void* d_depth,
                                         size_t depth_stride, int depth_pitch, const sgs_rgbd_format* fmt, int nframes, const int32_t* d_prev_index,
                                         const float* last_xyz, const uint8_t* last_desc, const uint8_t* last_flags, const int32_t* last_octave,
                                         const float* last_angle, const int32_t* last_n, const float* tcw_cur, const float* tcw_last, float th, int mono,
                                         int check_orientation, void* stream);
/* The same step from HOST buffers: each colour frame is uploaded once (detector and gray conversion read the same copy), the raw depth as given;
 * outputs as sgs_tracker_step plus kps_un_out [F][cap] (mvKeysUn) and depth_out [F][cap] (mvDepth), each of which may be NULL.  Synchronises. */
SGS_API int sgs_tracker_step_rgbd(sgs_tracker* t, sgs_detector* det, const uint8_t* rgb, size_t rgb_stride, int rgb_pitch, const void* depth,
                                  size_t depth_stride, int depth_pitch, const sgs_rgbd_format* fmt, int nframes, const int32_t* prev_index,
                                  const float* last_xyz, const uint8_t* last_desc, const uint8_t* last_flags, const int32_t* last_octave,
                                  const float* last_angle, const int32_t* last_n, const float* tcw_cur, const float* tcw_last, float th, int mono,
                                  int check_orientation, sgs_keypoint* kps_out, uint8_t* desc_out, float* u_right_out, int32_t* counts_out,
                                  int32_t* cur_mp_out, int32_t* nmatches_out, sgs_rect* boxes_out, int32_t* nboxes_out, uint8_t* have_out,
                                  sgs_keypoint* kps_un_out, float* depth_out);
/* The RGB-D step for LIVE streams, one new frame per stream per call, the previous frames kept on the device.  The tracker has max_batch stream
 * slots, 0 .. max_batch-1.  Frame f of a call is the next frame of slot d_slot[f]; slots are distinct within a call, and any subset of them, in any order,
 * may appear.  For frame f in slot s:
 *   previous frame   the last frame any earlier stream call on this handle gave to s (a stream may skip calls);
 *   first frame      s has never held a frame, or d_new_stream[f] != 0 (d_new_stream may be NULL: all 0).  A first frame behaves as a row with
 *                    prev_index[f] == f of sgs_tracker_step_rgbd_device: LK tracks into its own image, F is NaN with info status 3, every keypoint is kept;
 *   dynamic state    the flag and person boxes the previous frame ended with filter the point pairs (src/Frame.cc:454-472); the flag counts as false when
 *                    the previous frame was itself a first frame (quirk Q13);
 *   after the call   s holds this frame's LK pyramid levels, its boxes and flag, and whether it was a first frame.
 * Every result -- sgs_tracker_results_device, the boxes, sgs_tracker_frame_device, sgs_tracker_fundamental_device_ptr, sgs_tracker_prev_xy_device -- equals
 * bit for bit what sgs_tracker_step_rgbd_device returns for a batch that holds each stream's previous frame and chains them with prev_index.  The batch
 * entry points on the same handle neither read nor change the slots; sgs_tracker_pose_chain_device after a stream call reads its mvKeysUn.  The
 * slots survive everything but the handle: the reference keeps this state at file scope through Tracking::Reset, so a caller mirroring it keeps
 * new_stream = 0 across a reset, and sets it when a different sequence starts feeding the slot.
 * d_slot [F], d_new_stream [F]: device arrays, not checked (out-of-range or duplicate slots are undefined).  The other arguments are those of
 * sgs_tracker_step_rgbd_device.  Calls on different streams must be ordered by the caller: each reads the slots the previous one wrote.
 * A call refused with SGS_ERR_INVALID changes no slot.  After SGS_ERR_CUDA the state of that call's slots is unspecified: restart them with new_stream. */
SGS_API int sgs_tracker_step_rgbd_stream_device(sgs_tracker* t, sgs_detector* det, const uint8_t* d_rgb, size_t rgb_stride, int rgb_pitch, const void* d_depth,
                                                size_t depth_stride, int depth_pitch, const sgs_rgbd_format* fmt, int nframes, const int32_t* d_slot,
                                                const uint8_t* d_new_stream, const float* last_xyz, const uint8_t* last_desc, const uint8_t* last_flags,
                                                const int32_t* last_octave, const float* last_angle, const int32_t* last_n, const float* tcw_cur,
                                                const float* tcw_last, float th, int mono, int check_orientation, void* stream);
/* The same from HOST buffers (slot [F], new_stream [F] or NULL, outputs as sgs_tracker_step_rgbd).  Refuses nframes outside [1, max_batch], a NULL slot,
 * a slot outside [0, max_batch) and a slot given twice with SGS_ERR_INVALID before anything runs.  Synchronises. */
SGS_API int sgs_tracker_step_rgbd_stream(sgs_tracker* t, sgs_detector* det, const uint8_t* rgb, size_t rgb_stride, int rgb_pitch, const void* depth,
                                         size_t depth_stride, int depth_pitch, const sgs_rgbd_format* fmt, int nframes, const int32_t* slot,
                                         const uint8_t* new_stream, const float* last_xyz, const uint8_t* last_desc, const uint8_t* last_flags,
                                         const int32_t* last_octave, const float* last_angle, const int32_t* last_n, const float* tcw_cur,
                                         const float* tcw_last, float th, int mono, int check_orientation, sgs_keypoint* kps_out, uint8_t* desc_out,
                                         float* u_right_out, int32_t* counts_out, int32_t* cur_mp_out, int32_t* nmatches_out, sgs_rect* boxes_out,
                                         int32_t* nboxes_out, uint8_t* have_out, sgs_keypoint* kps_un_out, float* depth_out);
/* Device pointers to the compacted mvKeysUn [F][cap] and mvDepth [F][cap] (-1 without depth) of the last RGB-D step; SGS_ERR_INVALID before the first. */
SGS_API int sgs_tracker_frame_device(const sgs_tracker* t, const sgs_keypoint** d_kps_un, const float** d_depth);
/* Text listing of the kernel list: one line per kernel with its fused element-wise tail and activation-pool buffers.  SGS_ERR_CAPACITY
 * with *n = bytes required (terminator included) when cap is too small. */
SGS_API int sgs_detector_describe(const sgs_detector* d, char* out, int64_t cap, int64_t* n);
/* Per-kernel timing of sgs_detector_detect_device, same contract as sgs_extractor_set_profiling: while enabled, CUDA events bracket every launch of a
 * call on the launching stream (preprocess, the kernels in the order of sgs_detector_describe, the two DetectionOutput kernels); ms_total[i] accumulates
 * over ncalls completed calls.  Costs one event per kernel: leave it off in production. */
SGS_API int sgs_detector_set_profiling(sgs_detector* d, int enable);
SGS_API int sgs_detector_kernel_times(sgs_detector* d, double* ms_total, int cap, int* nkernels, int* ncalls);
/* Diagnostics: copies blob `name` of frame `frame` of the last batch to host floats (ncnn memory order c,h,w).  Needs flags bit 0. */
SGS_API int sgs_detector_blob(sgs_detector* d, const char* name, int frame, float* out, int64_t cap, int64_t* n);

#ifdef __cplusplus
}
#endif
#endif /* SGS_ABI_H_ */
