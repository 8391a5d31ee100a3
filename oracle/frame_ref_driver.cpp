// C entry points around the reference's OWN Frame (src/Frame.cc and src/ORBextractor.cc compiled from the reference tree, unmodified, against the stand-ins of
// frame_shim/ and orbmatcher_shim/; the OpenCV algorithms they call are the oracle's cv2-pinned restatements): a stream of RGB-D frames with planted detector
// results in, what the reference's RGB-D constructor leaves in the Frame out -- extraction, RmDynamicPointWithSemanticAndGeometry (LK, the previous-frame
// box filter, findFundamentalMat, the epipolar / box test, the erase loop, the restore-all guard, the file-scope previous-frame state), UndistortKeyPoints,
// ComputeStereoFromRGBD, the grid -- plus isInFrustum and GetFeaturesInArea of the last frame.  TEST INFRASTRUCTURE (oracle/_ref/libframe_ref.so).
#include <cstdint>
#include <cstring>
#include <new>
#include <vector>

#include "Frame.h"

// file-scope state of src/Frame.cc (:27-33)
extern std::vector<cv::Point2f> Prepoint, PrepointRmDynamic, Curpoint, CurpointRmDynamic;
extern std::vector<uchar> State;
extern std::vector<float> Err;
extern cv::Mat imGrayPre;
extern bool bPreFrameHavePotentialDynamicObj;
extern std::vector<cv::Rect_<float> > vPreFramePotentialDynamicBorder;

namespace ORB_SLAM2 {
int MapPoint::PredictScale(const float& currentDist, Frame* pF) {      // src/MapPoint.cc:402-418 (`log` of a float under `using namespace std`: logf)
    float ratio = mfMaxDistance / currentDist;
    int nScale = ceil(log(ratio) / pF->mfLogScaleFactor);
    if (nScale < 0) nScale = 0; else if (nScale >= pF->mnScaleLevels) nScale = pF->mnScaleLevels - 1;
    return nScale;
}
}  // namespace ORB_SLAM2

using namespace ORB_SLAM2;

struct Kp { float x, y, size, angle, response; int32_t octave, class_id; };
void ref_arena_restart();

namespace {
ORBextractor* g_ex = nullptr;
ORBVocabulary g_voc;
Tracking g_trk;
Detector2D g_det;
alignas(64) unsigned char g_frame_mem[2][sizeof(Frame)];      // the Frame is built in ZEROED memory: the members the reference leaves uninitialised read as 0 / false (quirk Q12)
Frame* g_frame[2] = {nullptr, nullptr};
int g_cur = 0;
std::vector<cv::Rect_<float> > rects(const float* b, int n) { std::vector<cv::Rect_<float> > v; for (int i = 0; i < n; ++i) v.push_back(cv::Rect_<float>(b[4 * i], b[4 * i + 1], b[4 * i + 2], b[4 * i + 3])); return v; }
void put(const std::vector<cv::KeyPoint>& k, Kp* out, int cap) { for (int i = 0; i < (int)k.size() && i < cap; ++i) out[i] = Kp{k[i].pt.x, k[i].pt.y, k[i].size, k[i].angle, k[i].response, k[i].octave, k[i].class_id}; }
}  // namespace

#define REF_API extern "C" __attribute__((visibility("default")))

// a new stream: no previous image, previous-frame flags cleared, static calibration recomputed by the next frame
REF_API void ref_frame_reset(int nfeatures, float scale_factor, int nlevels, int ini_th, int min_th) {
    for (int i = 0; i < 2; ++i) if (g_frame[i]) { g_frame[i]->~Frame(); g_frame[i] = nullptr; }
    delete g_ex; g_ex = nullptr;
    // every heap object of the previous stream is released (not just cleared: a kept capacity would point into the arena that restarts below)
    imGrayPre = cv::Mat();
    bPreFrameHavePotentialDynamicObj = false;
    std::vector<cv::Rect_<float> >().swap(vPreFramePotentialDynamicBorder);
    std::vector<cv::Point2f>().swap(Prepoint); std::vector<cv::Point2f>().swap(PrepointRmDynamic);
    std::vector<cv::Point2f>().swap(Curpoint); std::vector<cv::Point2f>().swap(CurpointRmDynamic);
    std::vector<uchar>().swap(State); std::vector<float>().swap(Err);
    g_det = Detector2D();
    ref_arena_restart();               // addresses grow with creation order from here on (one stream must fit the arena: about 40 MB per frame of 1 GB)
    g_ex = new ORBextractor(nfeatures, scale_factor, nlevels, ini_th, min_th);
    Frame::mbInitialComputations = true;
    Frame::nNextId = 0;
    g_trk.mpDetector2d = &g_det;
}

// One frame of the stream through Frame::Frame(Tracking*, imGray, imDepth, ...).  Detector results (what Detector2D holds when Tracking builds the Frame,
// src/Detector2D.cc:52-88): the non-person objects (only their count matters to the Frame), the two flags, the two box lists.
// Outputs: the Frame's keypoints (after the rejection), undistorted keypoints, descriptors, uRight, depth; flags[0..3] = the Frame's
// mbHaveDynamicObjectForRmDynamicFeature, mbHaveDynamicObjectForMapping, then the file-scope bPreFrameHavePotentialDynamicObj and the size of
// vPreFramePotentialDynamicBorder AFTER the frame; bounds[0..5] = mnMinX, mnMaxX, mnMinY, mnMaxY, mfGridElementWidthInv, mfGridElementHeightInv.
REF_API int ref_frame_push(const uint8_t* gray, int w, int h, const float* depth, const float* K4, const float* dist5, float bf, float th_depth,
                           int nobjects, int have_rm, int have_map, const float* rm_boxes, int nrm, const float* map_boxes, int nmap,
                           Kp* keys, Kp* keys_un, uint8_t* desc, float* u_right, float* depth_out, int cap, int32_t* flags, float* bounds) {
    if (!g_ex) return -1;
    cv::Mat im(h, w, CV_8U), dm(h, w, CV_32F), K = cv::Mat::eye(3, 3, CV_32F), D(5, 1, CV_32F);
    for (int y = 0; y < h; ++y) { std::memcpy(im.ptr(y), gray + (size_t)y * w, (size_t)w); std::memcpy(dm.ptr(y), depth + (size_t)y * w, (size_t)w * 4); }
    K.at<float>(0, 0) = K4[0]; K.at<float>(1, 1) = K4[1]; K.at<float>(0, 2) = K4[2]; K.at<float>(1, 2) = K4[3];
    for (int i = 0; i < 5; ++i) D.at<float>(i) = dist5[i];
    g_det.mvObjects2D.assign(nobjects, Object2D());
    g_det.mbHaveDynamicObjectForRmDynamicFeature = have_rm != 0;
    g_det.mbHaveDynamicObjectForMapping = have_map != 0;
    g_det.mvPotentialDynamicBorderForRmDynamicFeature = rects(rm_boxes, nrm);
    g_det.mvPotentialDynamicBorderForMapping = rects(map_boxes, nmap);
    const int slot = g_cur ^ 1;
    if (g_frame[slot]) { g_frame[slot]->~Frame(); g_frame[slot] = nullptr; }
    std::memset(g_frame_mem[slot], 0, sizeof(Frame));
    Frame dummy;
    g_frame[slot] = new (g_frame_mem[slot]) Frame(&g_trk, im, dm, 0.0, g_ex, &g_voc, K, D, bf, th_depth, dummy);
    g_cur = slot;
    const Frame& F = *g_frame[slot];
    const int n = (int)F.mvKeys.size();
    put(F.mvKeys, keys, cap); put(F.mvKeysUn, keys_un, cap);
    for (int i = 0; i < n && i < cap && i < F.mDescriptors.rows; ++i) std::memcpy(desc + 32 * (size_t)i, F.mDescriptors.ptr(i), 32);
    for (int i = 0; i < (int)F.mvuRight.size() && i < cap; ++i) { u_right[i] = F.mvuRight[i]; depth_out[i] = F.mvDepth[i]; }
    flags[0] = F.mbHaveDynamicObjectForRmDynamicFeature; flags[1] = F.mbHaveDynamicObjectForMapping;
    flags[2] = bPreFrameHavePotentialDynamicObj; flags[3] = (int32_t)vPreFramePotentialDynamicBorder.size();
    flags[4] = F.mDescriptors.rows; flags[5] = F.N;
    bounds[0] = Frame::mnMinX; bounds[1] = Frame::mnMaxX; bounds[2] = Frame::mnMinY; bounds[3] = Frame::mnMaxY;
    bounds[4] = Frame::mfGridElementWidthInv; bounds[5] = Frame::mfGridElementHeightInv;
    return n;
}

// Frame::GetFeaturesInArea of the last frame
REF_API int ref_frame_features_in_area(float x, float y, float r, int min_level, int max_level, int32_t* out, int cap) {
    if (!g_frame[g_cur]) return -1;
    const std::vector<size_t> v = g_frame[g_cur]->GetFeaturesInArea(x, y, r, min_level, max_level);
    for (int i = 0; i < (int)v.size() && i < cap; ++i) out[i] = (int32_t)v[i];
    return (int)v.size();
}

// Frame::isInFrustum of the last frame with pose Tcw (4x4 row major) for n map points: xyz, normal, min / max distance (raw, before the 0.8 / 1.2 factors).
// out[i][0..5] = in view, u, v, uR, predicted level, viewCos
REF_API int ref_frame_is_in_frustum(const float* Tcw, float viewing_cos_limit, int n, const float* xyz, const float* normal, const float* min_dist, const float* max_dist, float* out) {
    if (!g_frame[g_cur]) return -1;
    Frame& F = *g_frame[g_cur];
    cv::Mat T(4, 4, CV_32F);
    for (int i = 0; i < 16; ++i) T.at<float>(i / 4, i % 4) = Tcw[i];
    F.SetPose(T);
    int cnt = 0;
    for (int i = 0; i < n; ++i) {
        MapPoint mp;
        mp.mWorldPos = cv::Mat(3, 1, CV_32F); mp.mNormalVector = cv::Mat(3, 1, CV_32F);
        for (int k = 0; k < 3; ++k) { mp.mWorldPos.at<float>(k) = xyz[3 * i + k]; mp.mNormalVector.at<float>(k) = normal[3 * i + k]; }
        mp.mfMinDistance = min_dist[i]; mp.mfMaxDistance = max_dist[i];
        const bool in = F.isInFrustum(&mp, viewing_cos_limit);
        float* o = out + 6 * (size_t)i;
        o[0] = in ? 1.f : 0.f; o[1] = mp.mTrackProjX; o[2] = mp.mTrackProjY; o[3] = mp.mTrackProjXR; o[4] = (float)mp.mnTrackScaleLevel; o[5] = mp.mTrackViewCos;
        cnt += in;
    }
    return cnt;
}

// The two per-keypoint tests of the rejection on their own: Frame::CheckEpiLineDistToRmDynamicPoint(kp, prev, F (9, row major), threshold) and
// Frame::isInDynamicRegion(kp, boxes (x, y, w, h)), the KeyPoint overloads the erase loop calls.  Neither reads the Frame's members.
REF_API int ref_frame_check_epi_line_dist(float x, float y, float px, float py, const double* F9, double threshold) {
    Frame fr;
    cv::KeyPoint kp; kp.pt = cv::Point2f(x, y);
    cv::Mat F(3, 3, CV_64F);
    for (int i = 0; i < 9; ++i) F.at<double>(i / 3, i % 3) = F9[i];
    return fr.CheckEpiLineDistToRmDynamicPoint(kp, cv::Point2f(px, py), F, threshold) ? 1 : 0;
}

REF_API int ref_frame_is_in_dynamic_region(float x, float y, const float* boxes, int nboxes) {
    Frame fr;
    cv::KeyPoint kp; kp.pt = cv::Point2f(x, y);
    return fr.isInDynamicRegion(kp, rects(boxes, nboxes)) ? 1 : 0;
}

// ---- allocation order = address order (see orbextractor_ref_driver.cpp: DistributeOctTree breaks size ties by node ADDRESS; quirk Q1) -------------------------
#include <cstdlib>
namespace {
struct Arena {
    char* base = nullptr; size_t cap = (size_t)1 << 30, off = 0;
    void* get(size_t n) {
        n = (n + 15) & ~(size_t)15;
        if (!base) base = (char*)std::malloc(cap);
        if (!base || off + n > cap) return std::malloc(n);
        void* p = base + off; off += n; return p;
    }
    bool owns(void* p) const { return base && (char*)p >= base && (char*)p < base + cap; }
};
Arena g_arena;
bool g_monotone = false;
}  // namespace
__attribute__((visibility("hidden"))) void* operator new(size_t n) { if (g_monotone) return g_arena.get(n); void* p = std::malloc(n ? n : 1); if (!p) throw std::bad_alloc(); return p; }
__attribute__((visibility("hidden"))) void operator delete(void* p) noexcept { if (!p || g_arena.owns(p)) return; std::free(p); }
__attribute__((visibility("hidden"))) void operator delete(void* p, size_t) noexcept { ::operator delete(p); }
void ref_arena_restart() { g_arena.off = 0; }
REF_API void ref_set_monotone_allocator(int on) { g_monotone = on != 0; }
