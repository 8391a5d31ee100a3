// C entry points around the reference's OWN KeyFrameDatabase (src/KeyFrameDatabase.cc, compiled unmodified with the real DBoW2 BowVector /
// ScoringObject and the real TemplatedVocabulary's L1 scoring) for tests/test_kfdb_ref.py: one database per map over a shared pool of key frames,
// driven by add / erase / clear / query.  TEST INFRASTRUCTURE.
#include <cstdint>
#include <memory>
#include <vector>

#include "KeyFrameDatabase.h"

#define REF_API extern "C" __attribute__((visibility("default")))

using namespace ORB_SLAM2;

namespace {
struct Voc : ORBVocabulary {            // the reference's vocabulary type with TF_IDF / L1_NORM; only its size and scoring object are used
    explicit Voc(int nwords) : ORBVocabulary(10, 6, DBoW2::TF_IDF, DBoW2::L1_NORM) { m_words.resize(nwords, nullptr); }
};
struct Db {
    std::unique_ptr<Voc> voc;
    std::vector<std::unique_ptr<KeyFrameDatabase>> maps;
    std::vector<KeyFrame> kf;
    long unsigned int next_frame = 1;   // every query a new frame, as in the tracking thread (frame 0 initialises)
};
void fill(DBoW2::BowVector& v, int n, const int32_t* ids, const double* vals) {
    v.clear();
    for (int i = 0; i < n; ++i) v.addWeight((DBoW2::WordId)ids[i], vals[i]);
}
}  // namespace

REF_API void* kdb_create(int nwords, int nmaps, int nslots) {
    Db* d = new Db();
    d->voc.reset(new Voc(nwords));
    for (int m = 0; m < nmaps; ++m) d->maps.emplace_back(new KeyFrameDatabase(*d->voc));
    d->kf.resize(nslots);
    for (int s = 0; s < nslots; ++s) d->kf[s].mnId = s;
    return d;
}
REF_API void kdb_free(void* h) { delete static_cast<Db*>(h); }
// the key frame of slot s (a new KeyFrame: mRelocScore 0, DESIGN.md Q16) enters map m
REF_API void kdb_add(void* h, int s, int m, int n, const int32_t* ids, const double* vals) {
    Db* d = static_cast<Db*>(h);
    KeyFrame& k = d->kf[s];
    fill(k.mBowVec, n, ids, vals);
    k.mRelocScore = 0.f;
    d->maps[m]->add(&k);
}
REF_API void kdb_erase(void* h, int s, int m) { Db* d = static_cast<Db*>(h); d->maps[m]->erase(&d->kf[s]); }
REF_API void kdb_clear(void* h, int m) { static_cast<Db*>(h)->maps[m]->clear(); }
REF_API void kdb_set_covis(void* h, int s, const int32_t* nb10) {
    Db* d = static_cast<Db*>(h);
    d->kf[s].neighbours.clear();
    for (int k = 0; k < 10; ++k) if (nb10[k] >= 0) d->kf[s].neighbours.push_back(&d->kf[nb10[k]]);
}
// DetectRelocalizationCandidates of one frame against map m: the candidates' slots, their number; every slot's mRelocScore after it
REF_API int kdb_query(void* h, int m, int n, const int32_t* ids, const double* vals, int32_t* cand, float* scores) {
    Db* d = static_cast<Db*>(h);
    Frame F;
    F.mnId = d->next_frame++;
    fill(F.mBowVec, n, ids, vals);
    const std::vector<KeyFrame*> r = d->maps[m]->DetectRelocalizationCandidates(&F);
    for (size_t i = 0; i < r.size(); ++i) cand[i] = (int32_t)(r[i] - d->kf.data());
    for (size_t s = 0; s < d->kf.size(); ++s) scores[s] = d->kf[s].mRelocScore;
    return (int)r.size();
}
