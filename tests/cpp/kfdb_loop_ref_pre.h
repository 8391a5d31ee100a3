// Minimal KeyFrame / Frame stand-ins under which the reference's OWN src/KeyFrameDatabase.cc compiles unmodified for both of its queries
// (force-included by tests/test_kfdb_loop_ref.py; it defines the real headers' include guards so that they become no-ops).  Unlike
// tests/cpp/kfdb_ref_pre.h, the connected set (GetConnectedKeyFrames) is kept apart from the 10 best neighbours, and the ordered covisible key
// frames that LoopClosing::DetectLoop scores (GetVectorCovisibleKeyFrames) are a third list.  TEST INFRASTRUCTURE.
#pragma once
#define KEYFRAME_H
#define FRAME_H
#include <set>
#include <vector>

#include "Thirdparty/DBoW2/DBoW2/BowVector.h"

namespace ORB_SLAM2 {
class KeyFrame {
public:
    long unsigned int mnId = 0;
    DBoW2::BowVector mBowVec;
    long unsigned int mnLoopQuery = 0; int mnLoopWords = 0; float mLoopScore = 0.f;
    long unsigned int mnRelocQuery = 0; int mnRelocWords = 0; float mRelocScore = 0.f;
    std::vector<KeyFrame*> neighbours;                       // GetBestCovisibilityKeyFrames order (src/KeyFrame.cc:175-183)
    std::set<KeyFrame*> connected;                           // mConnectedKeyFrameWeights' keys (:160-167)
    std::vector<KeyFrame*> covisible;                        // mvpOrderedConnectedKeyFrames (:169-173), none of them bad
    std::vector<KeyFrame*> GetBestCovisibilityKeyFrames(const int& N) {
        return (int)neighbours.size() <= N ? neighbours : std::vector<KeyFrame*>(neighbours.begin(), neighbours.begin() + N);
    }
    std::set<KeyFrame*> GetConnectedKeyFrames() { return connected; }
    std::vector<KeyFrame*> GetVectorCovisibleKeyFrames() { return covisible; }
    bool isBad() { return false; }
};
class Frame {
public:
    long unsigned int mnId = 0;
    DBoW2::BowVector mBowVec;
};
}  // namespace ORB_SLAM2
