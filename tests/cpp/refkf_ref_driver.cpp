// C entry point around the reference's OWN Tracking::TrackReferenceKeyFrame + TrackLocalMap (optionally after TrackWithMotionModel), for
// tests/test_refkf_chain_ref.py, which compiles it at test time like the library oracle/Makefile builds from oracle/tracking_ref_driver.cpp: that driver is
// included whole (its object-graph helpers, OpenPoint / OpenTracking / fill_frame, and its two entry points), this file adds the reference-key-frame route.
// TEST INFRASTRUCTURE.
#include "ORBmatcher.h"

#include "tracking_ref_driver.cpp"

namespace {
struct OpenRefTracking : OpenTracking {
    using OpenTracking::OpenTracking;
    void relocalised_at(long unsigned int id) { mnLastRelocFrameId = id; }
};
}  // namespace

// Tracking::TrackReferenceKeyFrame (src/Tracking.cc:796-838) then TrackLocalMap (:969-1014), optionally after TrackWithMotionModel (:906-967) on the same frame
// (with_motion: m last-frame points as in ref_track_motion_and_local_map; its pose = tcw_cur, the last frame's = tcw_last, which must be the identity).  Reference key
// frame: kn features, kf_flags / kf_node as in ref_track_reference_keyframe.  kf_local_id[j] / last_local_id[j] >= 0: that point IS local-map point number
// kf_local_id[j] (one object); other points are objects of their own.  reloc != 0: the frame follows a relocalisation (mnLastRelocFrameId = its id - 1, th 5 in
// SearchLocalPoints).  Outputs: the motion model's return value (0 when not run); nmatches of SearchByBoW (the reference's ORBmatcher(0.7, true) on the same frame
// and key frame); TrackReferenceKeyFrame's return value, pose and per keypoint the key-frame feature it holds (-1 none); when nmatches >= 15 also TrackLocalMap's
// return value, pose, per keypoint the point id (key-frame feature, or point_cap + local index), the outlier flags and mnMatchesInliers.
REF_API void ref_track_refkf_and_local_map(const float* cam9, const float* scale_factors, const float* inv_level_sigma2, int nlevels,
                                           int n, const float* cur_xy, const int32_t* cur_octave, const float* cur_angle, const float* cur_uright, const uint8_t* cur_desc,
                                           const int32_t* cur_node,
                                           int kn, const float* kf_xyz, const uint8_t* kf_desc, const uint8_t* kf_flags, const float* kf_angle, const int32_t* kf_node,
                                           const int32_t* kf_local_id,
                                           int with_motion, int m, const float* last_xyz, const uint8_t* last_desc, const uint8_t* last_flags, const int32_t* last_octave,
                                           const float* last_angle, const int32_t* last_local_id, const float* tcw_cur, const float* tcw_last, int reloc,
                                           int L, const float* mp_xyz, const float* mp_normal, const float* mp_min, const float* mp_max, const uint8_t* mp_desc,
                                           const uint8_t* mp_valid, const uint8_t* mp_obs, int point_cap,
                                           int32_t* ok_motion, int32_t* nm_bow, int32_t* ok_ref, float* tcw_ref, int32_t* mp_ref, int32_t* ok_local, float* tcw_final,
                                           int32_t* mp_final, uint8_t* outlier, int32_t* inliers) {
    Frame::fx = cam9[0]; Frame::fy = cam9[1]; Frame::cx = cam9[2]; Frame::cy = cam9[3]; Frame::invfx = 1.0f / Frame::fx; Frame::invfy = 1.0f / Frame::fy;
    Frame::mnMinX = cam9[5]; Frame::mnMinY = cam9[6]; Frame::mnMaxX = cam9[7]; Frame::mnMaxY = cam9[8];
    Frame::mfGridElementWidthInv = static_cast<float>(FRAME_GRID_COLS) / (Frame::mnMaxX - Frame::mnMinX);
    Frame::mfGridElementHeightInv = static_cast<float>(FRAME_GRID_ROWS) / (Frame::mnMaxY - Frame::mnMinY);
    Frame::mbInitialComputations = false;
    std::map<std::string, double>& S = cv::FileStorage::values();
    S.clear();
    S["Camera.fx"] = cam9[0]; S["Camera.fy"] = cam9[1]; S["Camera.cx"] = cam9[2]; S["Camera.cy"] = cam9[3]; S["Camera.bf"] = cam9[4]; S["Camera.fps"] = 30; S["Camera.RGB"] = 1;
    S["ORBextractor.nFeatures"] = 1000; S["ORBextractor.scaleFactor"] = scale_factors[1]; S["ORBextractor.nLevels"] = nlevels; S["ORBextractor.iniThFAST"] = 20; S["ORBextractor.minThFAST"] = 7;
    S["ThDepth"] = 40; S["DepthMapFactor"] = 1;
    Map map; KeyFrameDatabase db; ORBVocabulary voc; FrameDrawer fd; MapDrawer md; System sys;
    OpenRefTracking trk(&sys, &voc, &fd, &md, &map, &db, std::string("planted"), (int)System::RGBD, boost::shared_ptr<PointCloudMapping>());

    KeyFrame ref_kf; ref_kf.Tcw = cv::Mat::eye(4, 4, CV_32F);                  // reference key frame of the last frame: identity, UpdateLastFrame keeps the given pose
    KeyFrame local_kf;                                                         // owns the local map points (UpdateLocalPoints collects them)
    std::vector<std::unique_ptr<OpenPoint> > pool;
    std::vector<MapPoint*> local(L, static_cast<MapPoint*>(NULL));
    for (int l = 0; l < L; ++l) {
        pool.emplace_back(new OpenPoint(vec3(mp_xyz + 3 * l), &ref_kf, &map));
        pool.back()->set(mp_normal + 3 * l, mp_min[l], mp_max[l], mp_desc + 32 * (size_t)l, mp_obs[l] ? 1 : 0, !mp_valid[l]);
        local[l] = pool.back().get();
    }
    local_kf.mvpMapPoints = local;
    // the reference key frame and its points
    KeyFrame kf; kf.Tcw = cv::Mat::eye(4, 4, CV_32F);
    kf.N = kn; kf.mvKeysUn.resize(kn); kf.mvKeys.resize(kn); kf.mDescriptors = cv::Mat(kn > 0 ? kn : 1, 32, CV_8U); kf.mvpMapPoints.assign(kn, static_cast<MapPoint*>(NULL));
    for (int j = 0; j < kn; ++j) {
        kf.mvKeysUn[j].angle = kf_angle[j]; kf.mvKeys[j].angle = kf_angle[j];
        std::memcpy(kf.mDescriptors.ptr(j), kf_desc + 32 * (size_t)j, 32);
        if (kf_node[j] >= 0) kf.mFeatVec[kf_node[j]].push_back(j);
        if (!(kf_flags[j] & 1)) continue;
        if (kf_local_id && kf_local_id[j] >= 0) { kf.mvpMapPoints[j] = local[kf_local_id[j]]; continue; }
        pool.emplace_back(new OpenPoint(vec3(kf_xyz + 3 * j), &kf, &map));
        pool.back()->set(NULL, 0.f, 0.f, kf_desc + 32 * (size_t)j, (kf_flags[j] & 2) ? 1 : 0, (kf_flags[j] & 4) != 0);
        kf.mvpMapPoints[j] = pool.back().get();
    }
    Frame cur, last;
    fill_frame(cur, n, cur_xy, cur_octave, cur_angle, cur_uright, cur_desc, scale_factors, inv_level_sigma2, nlevels, cam9[4], 100);
    for (int i = 0; i < n; ++i) if (cur_node[i] >= 0) cur.mFeatVec[cur_node[i]].push_back(i);
    cur.mBowVec[0] = 1.0;                                                     // not empty: Frame::ComputeBoW keeps the planted vectors
    cur.mpORBvocabulary = &voc;
    const int ml = with_motion ? m : 0;
    std::vector<float> zero2(2 * (size_t)(ml > 0 ? ml : 1), 0.f);
    std::vector<int32_t> zo(ml > 0 ? ml : 1, 0);
    fill_frame(last, ml, zero2.data(), with_motion ? last_octave : zo.data(), with_motion ? last_angle : NULL, NULL, NULL, scale_factors, inv_level_sigma2, nlevels,
               cam9[4], 99);
    last.mTcw = mat44(tcw_last); last.UpdatePoseMatrices(); last.mpReferenceKF = &ref_kf;
    for (int j = 0; j < ml; ++j) {
        if (!(last_flags[j] & 1)) continue;
        if (last_local_id[j] >= 0) { last.mvpMapPoints[j] = local[last_local_id[j]]; continue; }
        pool.emplace_back(new OpenPoint(vec3(last_xyz + 3 * j), &ref_kf, &map));
        pool.back()->set(NULL, 0.f, 0.f, last_desc + 32 * (size_t)j, (last_flags[j] & 2) ? 1 : 0, (last_flags[j] & 4) != 0);
        last.mvpMapPoints[j] = pool.back().get();
    }
    trk.state(cur, last, mat44(tcw_cur), mat44(tcw_last), &local_kf);
    if (reloc) trk.relocalised_at(99);
    *ok_motion = with_motion ? (trk.motion_model() ? 1 : 0) : 0;
    Frame& F = trk.mCurrentFrame;
    {
        ORBmatcher matcher(0.7, true);
        std::vector<MapPoint*> matches;
        *nm_bow = matcher.SearchByBoW(&kf, F, matches);
    }
    *ok_ref = trk.reference_keyframe(&kf) ? 1 : 0;
    if (F.mTcw.empty()) F.mTcw = cv::Mat::eye(4, 4, CV_32F);
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) tcw_ref[4 * i + j] = F.mTcw.at<float>(i, j);
    std::vector<MapPoint*> held(F.mvpMapPoints);
    for (int i = 0; i < n; ++i) {
        mp_ref[i] = -1;
        if (*nm_bow >= 15 && held[i]) for (int j = 0; j < kn; ++j) if (kf.mvpMapPoints[j] == held[i]) { mp_ref[i] = j; break; }
    }
    *ok_local = 0; *inliers = 0;
    if (*nm_bow < 15) return;
    *ok_local = trk.local_map() ? 1 : 0;
    for (int i = 0; i < 4; ++i) for (int j = 0; j < 4; ++j) tcw_final[4 * i + j] = F.mTcw.at<float>(i, j);
    for (int i = 0; i < n; ++i) {
        MapPoint* p = F.mvpMapPoints[i];
        mp_final[i] = -1; outlier[i] = (p && F.mvbOutlier[i]) ? 1 : 0;
        if (!p) continue;
        if (p == held[i]) { mp_final[i] = mp_ref[i]; continue; }
        for (int l = 0; l < L; ++l) if (local[l] == p) { mp_final[i] = point_cap + l; break; }
    }
    *inliers = trk.inliers();
}
