// Minimal KeyFrame / Frame stand-ins under which the reference's OWN src/KeyFrameDatabase.cc compiles unmodified (force-included by
// tests/test_kfdb_ref.py; it defines the real headers' include guards so that they become no-ops).  Only the members KeyFrameDatabase.cc touches.
// TEST INFRASTRUCTURE.
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
    std::vector<KeyFrame*> GetBestCovisibilityKeyFrames(const int& N) {
        return (int)neighbours.size() <= N ? neighbours : std::vector<KeyFrame*>(neighbours.begin(), neighbours.begin() + N);
    }
    std::set<KeyFrame*> GetConnectedKeyFrames() { return std::set<KeyFrame*>(neighbours.begin(), neighbours.end()); }
};
class Frame {
public:
    long unsigned int mnId = 0;
    DBoW2::BowVector mBowVec;
};
}  // namespace ORB_SLAM2
