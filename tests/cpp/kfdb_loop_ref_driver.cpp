// C entry points around the reference's OWN KeyFrameDatabase (src/KeyFrameDatabase.cc, compiled unmodified with the real DBoW2 sources) for
// tests/test_kfdb_loop_ref.py: the add / erase / clear / relocalisation entry points of tests/cpp/kfdb_ref_driver.cpp, compiled here against the
// stand-ins of tests/cpp/kfdb_loop_ref_pre.h, and the loop query: LoopClosing::DetectLoop's minScore (src/LoopClosing.cc:124-138) with the
// reference vocabulary's own score, then DetectLoopCandidates.  TEST INFRASTRUCTURE.
#include "kfdb_ref_driver.cpp"

// The loop query of a new key frame against map m: slot `self` (its BowVector must be the one given) or, for self < 0, a key frame outside the pool.
// It takes a new id; conn: the slots of its connected set (ids outside the pool are left out); ncov covisible key frames with the BowVectors
// cov_ids / cov_vals [ncov][cov_cap], cov_n [ncov].  Writes the candidates' slots and returns their number; stats [4]: the key frames of the pool
// that this query listed (mnLoopQuery), their largest mnLoopWords, how many of them are above int(max * 0.8f), the candidates; *min_score.
REF_API int kdb_loop(void* h, int m, int self, int n, const int32_t* ids, const double* vals, int nconn, const int32_t* conn, int ncov, int cov_cap,
                     const int32_t* cov_n, const int32_t* cov_ids, const double* cov_vals, int32_t* cand, int32_t* stats, float* min_score) {
    Db* d = static_cast<Db*>(h);
    KeyFrame outside;
    KeyFrame* pKF = self >= 0 ? &d->kf[self] : &outside;
    pKF->mnId = d->next_frame++;
    fill(pKF->mBowVec, n, ids, vals);
    pKF->connected.clear();
    for (int i = 0; i < nconn; ++i)
        if (conn[i] >= 0 && conn[i] < (int)d->kf.size()) pKF->connected.insert(&d->kf[conn[i]]);
    std::vector<KeyFrame> cov(ncov);
    pKF->covisible.clear();
    for (int c = 0; c < ncov; ++c) {
        fill(cov[c].mBowVec, cov_n[c], cov_ids + (size_t)c * cov_cap, cov_vals + (size_t)c * cov_cap);
        pKF->covisible.push_back(&cov[c]);
    }
    // LoopClosing.cc:124-138
    const std::vector<KeyFrame*> vpConnectedKeyFrames = pKF->GetVectorCovisibleKeyFrames();
    const DBoW2::BowVector& CurrentBowVec = pKF->mBowVec;
    float minScore = 1;
    for (size_t i = 0; i < vpConnectedKeyFrames.size(); i++) {
        KeyFrame* pKFc = vpConnectedKeyFrames[i];
        if (pKFc->isBad()) continue;
        float score = d->voc->score(CurrentBowVec, pKFc->mBowVec);
        if (score < minScore) minScore = score;
    }
    const std::vector<KeyFrame*> r = d->maps[m]->DetectLoopCandidates(pKF, minScore);
    pKF->covisible.clear();
    for (size_t i = 0; i < r.size(); ++i) cand[i] = (int32_t)(r[i] - d->kf.data());
    int share = 0, maxc = 0, nscores = 0;
    for (const KeyFrame& k : d->kf)
        if (k.mnLoopQuery == pKF->mnId) { ++share; if (k.mnLoopWords > maxc) maxc = k.mnLoopWords; }
    const int minc = maxc * 0.8f;
    for (const KeyFrame& k : d->kf)
        if (k.mnLoopQuery == pKF->mnId && k.mnLoopWords > minc) ++nscores;
    stats[0] = share; stats[1] = maxc; stats[2] = nscores; stats[3] = (int32_t)r.size();
    *min_score = minScore;
    return (int)r.size();
}
