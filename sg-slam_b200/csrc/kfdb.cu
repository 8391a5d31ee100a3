// kfdb.cu -- KeyFrameDatabase (src/KeyFrameDatabase.cc:33-74) for up to max_maps independent maps in one handle, and its relocalisation query
// KeyFrameDatabase::DetectRelocalizationCandidates (:199-311) for a batch of frames, one per map.
//   The key frames' BowVectors live in a pool of max_keyframes slots.  The inverted file is not materialised: a key frame's position in
//   lKFsSharingWords is fixed by its smallest word shared with the frame and, among key frames that first meet at the same word, by the order of
//   the adds (add pushes to the back of every list of the key frame's words, erase removes from all of them), so the handle keeps a handle-wide add
//   counter per slot instead.  mRelocScore (include/KeyFrame.h:151) is device state of the slot: 0 at add, written by every query that scores it.
//   query: pair kernel   one warp per (row, key frame of the row's map): common words by binary search of each frame word in the key frame's
//                        BowVector, the first common word, and L1Scoring::score (ScoringObject.cpp:23-68) -- the terms per lane, their sum serial in
//                        ascending word order;
//          row kernel    one block per row: maxCommonWords and the 0.8 gate, mRelocScore of the scored key frames, their (first common word, add
//                        counter) sort, the covisibility accumulation, the 0.75 retention and the pBestKF dedupe in list order.
// The loop query KeyFrameDatabase::DetectLoopCandidates (:76-197), with LoopClosing::DetectLoop's minScore, runs the same pair kernel, then a prep
// kernel (the connected key frames leave the sharing set; minScore against the covisible BowVectors), then the row kernel with the loop rules.
// Floating point: the score is DBoW2's float64 sum in DBoW2's order, rounded to float once; the accumulation is float in the reference's order.
#include <cuda_runtime.h>

#include <algorithm>
#include <climits>
#include <memory>
#include <vector>

#include "block_compact.cuh"
#include "host_stage.cuh"
#include "internal_launch.cuh"
#include "sgs_common.h"

namespace {
constexpr int kMaxQueryKeyframes = 16384;        // key frames of one queried map: the row kernel sorts its scored ones in shared memory
constexpr uint64_t kSeqLimit = 1ull << 40;       // add counter: packed below the first common word's index in the sort key
constexpr int kMaxBowCap = 1 << 23;
constexpr int kRowThreads = 512;
}  // namespace

struct sgs_kfdb {
    explicit sgs_kfdb(int dev) : device(dev), res(dev) {}
    int device, max_maps = 0, max_keyframes = 0, max_words = 0;
    sgs::HandleResources res;
    // host bookkeeping: per slot its map (-1 = not live) and add counter; the live slots grouped by map (ascending within a map) and where each
    // map's group starts (max_maps + 1 entries)
    std::vector<int32_t> slot_map, group, group_off;
    std::vector<uint64_t> slot_seq;
    uint64_t next_seq = 0;
    // device: BowVectors [max_keyframes][max_words] (ids ascending, values), their lengths, add counters, mRelocScore, each slot's map (-1 = not
    // live), the groups
    int32_t* d_word = nullptr; double* d_value = nullptr; int32_t* d_n = nullptr; uint64_t* d_seq = nullptr; float* d_score = nullptr;
    int32_t* d_map = nullptr; int32_t* d_group = nullptr;
    // per-slot scratch of a query (the rows of one call name distinct maps, so each slot belongs to at most one row): common words, index of the
    // first common word in the frame's BowVector, si, the dedupe mark
    int32_t* d_cnt = nullptr; int32_t* d_first = nullptr; float* d_si = nullptr; int32_t* d_mark = nullptr;
    // add: the slots, add counters and source rows of one call; query: per row (row, group offset, group length, map)
    int32_t* d_add_slot = nullptr; uint64_t* d_add_seq = nullptr; int4* d_rows = nullptr;
    // loop query: per row (connected ids begin, end, covisible rows begin, end)
    int4* d_loop = nullptr;
};

namespace sgs {

// add: row i of the caller's BowVectors into slot slot[i]; mRelocScore = 0 (KeyFrame.cc:35 leaves it uninitialised, DESIGN.md Q16)
__global__ void kfdb_add_kernel(const int32_t* __restrict__ slot, const uint64_t* __restrict__ seq, const int32_t* __restrict__ bw, const double* __restrict__ bv,
                                const int32_t* __restrict__ bn, int bow_cap, int max_words, int32_t* __restrict__ word, double* __restrict__ value,
                                int32_t* __restrict__ n_out, uint64_t* __restrict__ seq_out, float* __restrict__ score) {
    const int i = blockIdx.x, s = slot[i];
    const int n = bn[i];
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        word[(int64_t)s * max_words + j] = bw[(int64_t)i * bow_cap + j];
        value[(int64_t)s * max_words + j] = bv[(int64_t)i * bow_cap + j];
    }
    if (threadIdx.x == 0) { n_out[s] = n; seq_out[s] = seq[i]; score[s] = 0.f; }
}

struct KfdbDev {
    const int32_t* word; const double* value; const int32_t* n; const uint64_t* seq; const int32_t* map; const int32_t* group; int max_words, max_keyframes;
    float* score; int32_t* cnt; int32_t* first; float* si; int32_t* mark;
};

// One warp: the words the frame's BowVector (fw, fv: nf words) shares with a key frame's (kw, kv: nk words), the index of the first of them in the
// frame's BowVector (-1: none), and float(L1Scoring::score(F, KF)) (ScoringObject.cpp:23-68): every frame word binary-searched in the key frame's,
// the terms per lane, their float64 sum serial in ascending word order.  Every lane returns the same values.
__device__ __forceinline__ float warp_l1_score(const int32_t* fw, const double* fv, int nf, const int32_t* __restrict__ kw, const double* __restrict__ kv,
                                               int nk, int lane, int& cnt, int& first) {
    cnt = 0; first = -1;
    double score = 0.0;
    for (int c0 = 0; c0 < nf && nk > 0; c0 += 32) {
        const int i = c0 + lane;
        int j = -1;
        double t = 0.0;
        if (i < nf) {
            const int w = fw[i];
            int lo = 0, hi = nk;
            while (lo < hi) { const int mid = (lo + hi) >> 1; if (__ldg(kw + mid) < w) lo = mid + 1; else hi = mid; }
            if (lo < nk && __ldg(kw + lo) == w) {
                j = lo;
                const double vi = fv[i], wi = __ldg(kv + j);
                t = fabs(vi - wi) - fabs(vi) - fabs(wi);
            }
        }
        unsigned m = __ballot_sync(0xffffffffu, j >= 0);
        if (m && first < 0) first = c0 + __ffs(m) - 1;
        cnt += __popc(m);
        while (m) {                                                 // the sum in ascending word order
            const int b = __ffs(m) - 1;
            score += __shfl_sync(0xffffffffu, t, b);
            m &= m - 1;
        }
    }
    return __double2float_rn(-score / 2.0);
}

// :207-222 mnRelocWords and the first common word, and :249 L1Scoring::score for every key frame of the row's map
__global__ void __launch_bounds__(256) kfdb_pair_kernel(const KfdbDev D, const int4* __restrict__ rows, const int32_t* __restrict__ fw_all,
                                                        const double* __restrict__ fv_all, const int32_t* __restrict__ fn_all, int bow_cap) {
    const int4 row = rows[blockIdx.y];
    const int p = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (p >= row.z) return;
    const int slot = D.group[row.y + p];
    const int nf = min(max(fn_all[row.x], 0), bow_cap);
    int cnt, first;
    const float si = warp_l1_score(fw_all + (int64_t)row.x * bow_cap, fv_all + (int64_t)row.x * bow_cap, nf, D.word + (int64_t)slot * D.max_words,
                                   D.value + (int64_t)slot * D.max_words, D.n[slot], lane, cnt, first);
    if (lane == 0) { D.cnt[slot] = cnt; D.first[slot] = first; D.si[slot] = si; }
}

// LoopClosing.cc:124-138 and KeyFrameDatabase.cc:78, after the pair pass, one block per row: the connected key frames (KeyFrame.cc:160-167) of the
// row's map get a common-word count of 0, so that they neither enter lKFsSharingWords nor count as sharing neighbours; minScore, from 1 the least
// score against the covisible BowVectors, one warp per BowVector.  The least (score, visiting index) is kept, so a zero minimum has the sign of the
// first zero the reference meets (DESIGN.md Q17).  loop[q] = (connected ids begin, end, covisible rows begin, end).
__global__ void __launch_bounds__(256) kfdb_loop_prep_kernel(const KfdbDev D, const int4* __restrict__ rows, const int4* __restrict__ loop,
                                                             const int32_t* __restrict__ fw_all, const double* __restrict__ fv_all,
                                                             const int32_t* __restrict__ fn_all, int bow_cap, const int32_t* __restrict__ conn,
                                                             const int32_t* __restrict__ cw, const double* __restrict__ cv, const int32_t* __restrict__ cn,
                                                             float* __restrict__ min_score) {
    __shared__ unsigned long long s_min;                                    // |score| bits << 32 | visiting index << 1 | sign
    const int4 row = rows[blockIdx.x], lr = loop[blockIdx.x];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) s_min = (unsigned long long)__float_as_uint(1.f) << 32 | 0xfffffffeu;
    for (int i = lr.x + threadIdx.x; i < lr.y; i += blockDim.x) {
        const int s = conn[i];
        if (s >= 0 && s < D.max_keyframes && D.map[s] == row.w) D.cnt[s] = 0;
    }
    __syncthreads();
    const int nf = min(max(fn_all[row.x], 0), bow_cap);
    unsigned long long best = ~0ull;
    for (int c = lr.z + warp; c < lr.w; c += 8) {
        int cnt, first;
        const float sc = warp_l1_score(fw_all + (int64_t)row.x * bow_cap, fv_all + (int64_t)row.x * bow_cap, nf, cw + (int64_t)c * bow_cap,
                                       cv + (int64_t)c * bow_cap, min(max(cn[c], 0), bow_cap), lane, cnt, first);
        const unsigned bits = __float_as_uint(sc);
        best = min(best, (unsigned long long)(bits & 0x7fffffffu) << 32 | (unsigned)(c - lr.z) << 1 | bits >> 31);
    }
    if (lane == 0) atomicMin(&s_min, best);
    __syncthreads();
    if (threadIdx.x == 0) min_score[row.x] = __uint_as_float((unsigned)(s_min >> 32) | (unsigned)(s_min & 1) << 31);
}

__device__ void sort_with_slots(uint64_t* key, int32_t* slot, int n_pow2) {         // ascending, padding = all ones
    for (int k = 2; k <= n_pow2; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = threadIdx.x; i < n_pow2; i += blockDim.x) {
                const int p = i ^ j;
                if (p > i) {
                    const uint64_t a = key[i], b = key[p];
                    if ((a > b) == ((i & k) == 0)) { key[i] = b; key[p] = a; const int32_t s = slot[i]; slot[i] = slot[p]; slot[p] = s; }
                }
            }
            __syncthreads();
        }
}

// :224-308 for one row: the gate, mRelocScore, lKFsSharingWords order of the scored key frames, accumulation over the covisibility table, retention,
// dedupe.  stats: key frames sharing a word, maxCommonWords, nscores, candidates before the cap.
// kLoop: DetectLoopCandidates' :107-193 instead, on the counts kfdb_loop_prep_kernel left (connected key frames do not share): only the scored key
// frames with si >= minScore are listed, a neighbour adds its si of this query if it is above the gate, bestAccScore starts at minScore, and
// mRelocScore is not touched.
template <bool kLoop>
__global__ void __launch_bounds__(kRowThreads) kfdb_row_kernel(const KfdbDev D, const int4* __restrict__ rows, const int32_t* __restrict__ covis,
                                                               int p2, int32_t* __restrict__ cand, int cand_cap, int32_t* __restrict__ ncand,
                                                               int32_t* __restrict__ stats, const float* __restrict__ min_score) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int4 row = rows[blockIdx.x];
    uint64_t* key = reinterpret_cast<uint64_t*>(smem);             // [p2] sort keys (first common word's index << 40 | add counter), then (acc, pBestKF)
    int32_t* kslot = reinterpret_cast<int32_t*>(key + p2);          // [p2] the slot of each key
    __shared__ int s_share, s_max, s_nsc, s_best, s_scored;
    const int tid = threadIdx.x, f = row.x, map = row.w, len = row.z;
    const float min_si = kLoop ? min_score[f] : 0.f;                // lScoreAndMatch's least si and bestAccScore's start
    const int32_t* grp = D.group + row.y;
    if (tid == 0) { s_share = 0; s_max = 0; s_nsc = 0; s_best = __float_as_int(min_si); s_scored = 0; }
    __syncthreads();
    int share = 0, mx = 0;
    for (int p = tid; p < len; p += kRowThreads) {
        const int c = D.cnt[grp[p]];
        share += c > 0; mx = max(mx, c);
    }
    atomicAdd(&s_share, share); atomicMax(&s_max, mx);
    __syncthreads();
    const int nshare = s_share, maxc = s_max;
    const int minc = __float2int_rz(__fmul_rn((float)maxc, 0.8f));  // :235
    // :242-253 the scored key frames write mRelocScore; they are listed in any order here and sorted below
    for (int p = tid; p < len; p += kRowThreads) {
        const int s = grp[p];
        if (nshare > 0 && D.cnt[s] > minc) {
            if (kLoop) atomicAdd(&s_scored, 1);
            else D.score[s] = D.si[s];
            if (kLoop && !(D.si[s] >= min_si)) continue;            // :136
            const int q = atomicAdd(&s_nsc, 1);
            key[q] = ((uint64_t)D.first[s] << 40) | D.seq[s];
            kslot[q] = s;
        }
    }
    __syncthreads();
    const int nsc = s_nsc;
    int n2 = 1;
    while (n2 < nsc) n2 <<= 1;
    for (int q = nsc + tid; q < n2; q += kRowThreads) { key[q] = ~0ull; kslot[q] = -1; }
    __syncthreads();
    if (nsc > 1) sort_with_slots(key, kslot, n2);
    // :262-287 accumulation by covisibility: neighbours that share a word in this query (mnRelocQuery == F->mnId), fresh or stale mRelocScore (Q16).
    // The loop query's neighbours (:159) are listed in this query and above the gate, so every score it reads is this query's si.
    for (int q = tid; q < nsc; q += kRowThreads) {
        const int s = kslot[q];
        float best = D.si[s], acc = best;
        int pbest = s;
        for (int k = 0; k < 10; ++k) {
            const int nb = covis[(int64_t)s * 10 + k];
            if (nb < 0 || nb >= D.max_keyframes || D.map[nb] != map || D.cnt[nb] <= (kLoop ? minc : 0)) continue;
            const float sc = kLoop ? D.si[nb] : D.score[nb];
            acc = __fadd_rn(acc, sc);
            if (sc > best) { pbest = nb; best = sc; }
        }
        key[q] = ((uint64_t)(uint32_t)__float_as_int(acc) << 32) | (uint32_t)pbest;
        if (acc > min_si) atomicMax(&s_best, __float_as_int(acc)); // non-negative floats order as their bits (-0 as the least)
    }
    __syncthreads();
    const float keep_above = __fmul_rn(0.75f, __int_as_float(s_best));   // :290
    // :291-306 retention, then the first entry of each pBestKF in list order
    for (int q = tid; q < nsc; q += kRowThreads)
        if (__int_as_float((int)(key[q] >> 32)) > keep_above) D.mark[(uint32_t)key[q]] = INT_MAX;
    __syncthreads();
    for (int q = tid; q < nsc; q += kRowThreads)
        if (__int_as_float((int)(key[q] >> 32)) > keep_above) atomicMin(&D.mark[(uint32_t)key[q]], q);
    __syncthreads();
    int total = 0;
    int32_t* out = cand + (int64_t)f * cand_cap;
    for (int q0 = 0; q0 < nsc; q0 += kRowThreads) {
        const int q = q0 + tid;
        const bool keep = q < nsc && __int_as_float((int)(key[q] >> 32)) > keep_above && __ldcg(&D.mark[(uint32_t)key[q]]) == q;
        const int pos = block_ordered_slot<kRowThreads>(keep, total);
        if (pos >= 0 && pos < cand_cap) out[pos] = (int32_t)(uint32_t)key[q];
    }
    for (int q = total + tid; q < cand_cap; q += kRowThreads) out[q] = -1;
    if (tid == 0) {
        ncand[f] = min(total, cand_cap);
        stats[4 * f] = nshare; stats[4 * f + 1] = maxc; stats[4 * f + 2] = kLoop ? s_scored : nsc; stats[4 * f + 3] = total;
    }
}

// the host-side checks of a query: map[f] == -1 skips row f; the others name distinct known maps of at most kMaxQueryKeyframes key frames.  On success
// rows holds (row, group offset, group length, map) of every queried row and *max_len the largest group.
int kfdb_plan_query(const sgs_kfdb* db, const char* fn, int nframes, const int32_t* map, std::vector<int4>& rows, int* max_len) {
    rows.clear();
    *max_len = 0;
    std::vector<uint8_t> used(db->max_maps, 0);
    for (int f = 0; f < nframes; ++f) {
        const int m = map[f];
        if (m == -1) continue;
        if (m < 0 || m >= db->max_maps) { set_error("%s: row %d names map %d (max_maps %d)", fn, f, m, db->max_maps); return SGS_ERR_INVALID; }
        if (used[m]) { set_error("%s: map %d is named by two rows of one call", fn, m); return SGS_ERR_INVALID; }
        used[m] = 1;
        const int off = db->group_off[m], len = db->group_off[m + 1] - off;
        if (len > kMaxQueryKeyframes) { set_error("%s: map %d holds %d key frames, a query takes at most %d", fn, m, len, kMaxQueryKeyframes); return SGS_ERR_UNSUPPORTED; }
        rows.push_back(make_int4(f, off, len, m));
        *max_len = std::max(*max_len, len);
    }
    return SGS_OK;
}

// the loop query's inputs beyond the relocalisation query's: per queried row (connected ids begin, end, covisible rows begin, end) and the arrays
struct KfdbLoop {
    std::vector<int4> ranges;
    const int32_t* conn; const int32_t* cov_word; const double* cov_value; const int32_t* cov_n; float* min_score;
};

// pair kernel, [loop prep kernel,] row kernel: the relocalisation query, or the loop query when loop is not NULL
int launch_query(sgs_kfdb* db, const char* fn, const std::vector<int4>& rows, int max_len, const int32_t* d_bow_word, const double* d_bow_value,
                 const int32_t* d_bow_n, int bow_cap, const int32_t* d_covis, int32_t* d_cand, int cand_cap, int32_t* d_ncand, int32_t* d_stats,
                 const KfdbLoop* loop, cudaStream_t st) {
    if (rows.empty()) return SGS_OK;
    SGS_CUDA_TRY_AT(fn, cudaSetDevice(db->device));
    const int nq = (int)rows.size();
    SGS_CUDA_TRY_AT(fn, cudaMemcpyAsync(db->d_rows, rows.data(), sizeof(int4) * nq, cudaMemcpyHostToDevice, st));
    KfdbDev D{db->d_word, db->d_value, db->d_n, db->d_seq, db->d_map, db->d_group, db->max_words, db->max_keyframes,
              db->d_score, db->d_cnt, db->d_first, db->d_si, db->d_mark};
    if (max_len > 0) {
        kfdb_pair_kernel<<<dim3((max_len + 7) / 8, nq), 256, 0, st>>>(D, db->d_rows, d_bow_word, d_bow_value, d_bow_n, bow_cap);
        SGS_CUDA_TRY_AT(fn, cudaGetLastError());
    }
    if (loop) {
        SGS_CUDA_TRY_AT(fn, cudaMemcpyAsync(db->d_loop, loop->ranges.data(), sizeof(int4) * nq, cudaMemcpyHostToDevice, st));
        kfdb_loop_prep_kernel<<<nq, 256, 0, st>>>(D, db->d_rows, db->d_loop, d_bow_word, d_bow_value, d_bow_n, bow_cap, loop->conn, loop->cov_word,
                                                  loop->cov_value, loop->cov_n, loop->min_score);
        SGS_CUDA_TRY_AT(fn, cudaGetLastError());
    }
    int p2 = 1;
    while (p2 < max_len) p2 <<= 1;
    const size_t smem = 12 * (size_t)p2 + 16;
    auto row_kernel = loop ? kfdb_row_kernel<true> : kfdb_row_kernel<false>;
    if (smem > 40 * 1024) SGS_CUDA_TRY_AT(fn, cudaFuncSetAttribute(row_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    row_kernel<<<nq, kRowThreads, smem, st>>>(D, db->d_rows, d_covis, p2, d_cand, cand_cap, d_ncand, d_stats, loop ? loop->min_score : nullptr);
    SGS_CUDA_TRY_AT(fn, cudaGetLastError());
    return SGS_OK;
}

int kfdb_launch_query(sgs_kfdb* db, const char* fn, const std::vector<int4>& rows, int max_len, const int32_t* d_bow_word, const double* d_bow_value,
                      const int32_t* d_bow_n, int bow_cap, const int32_t* d_covis, int32_t* d_cand, int cand_cap, int32_t* d_ncand, int32_t* d_stats,
                      cudaStream_t st) {
    return launch_query(db, fn, rows, max_len, d_bow_word, d_bow_value, d_bow_n, bow_cap, d_covis, d_cand, cand_cap, d_ncand, d_stats, nullptr, st);
}

}  // namespace sgs

using namespace sgs;

namespace {
// the live slots grouped by map onto the device, after a change of the bookkeeping
int publish_groups(sgs_kfdb* db, const char* fn, cudaStream_t st) {
    const int M = db->max_maps, K = db->max_keyframes;
    std::vector<int32_t> count(M + 1, 0);
    for (int s = 0; s < K; ++s) if (db->slot_map[s] >= 0) ++count[db->slot_map[s] + 1];
    for (int m = 0; m < M; ++m) count[m + 1] += count[m];
    db->group_off = count;
    db->group.assign(std::max(count[M], 1), 0);
    for (int s = 0; s < K; ++s) if (db->slot_map[s] >= 0) db->group[count[db->slot_map[s]]++] = s;
    SGS_CUDA_TRY_AT(fn, cudaSetDevice(db->device));
    SGS_CUDA_TRY_AT(fn, cudaMemcpyAsync(db->d_map, db->slot_map.data(), 4 * (size_t)K, cudaMemcpyHostToDevice, st));
    SGS_CUDA_TRY_AT(fn, cudaMemcpyAsync(db->d_group, db->group.data(), 4 * db->group.size(), cudaMemcpyHostToDevice, st));
    return SGS_OK;
}
}  // namespace

extern "C" {

SGS_API void sgs_kfdb_destroy(sgs_kfdb* db) { delete db; }

SGS_API int sgs_kfdb_create(int device, int max_maps, int max_keyframes, int max_words, sgs_kfdb** out) {
    const char* const fn = "sgs_kfdb_create";
    if (!out || max_maps < 1 || max_keyframes < 1 || max_words < 1) { set_error("%s: bad argument", fn); return SGS_ERR_INVALID; }
    *out = nullptr;
    SGS_CUDA_TRY_AT(fn, cudaSetDevice(device));
    auto db = std::make_unique<sgs_kfdb>(device);
    db->max_maps = max_maps; db->max_keyframes = max_keyframes; db->max_words = max_words;
    db->slot_map.assign(max_keyframes, -1); db->slot_seq.assign(max_keyframes, 0); db->group_off.assign(max_maps + 1, 0); db->group.assign(1, 0);
    HandleResources& R = db->res;
    const size_t K = max_keyframes, W = max_words;
    SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_word, K * W * 4)); SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_value, K * W * 8)); SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_n, K * 4));
    SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_seq, K * 8)); SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_score, K * 4)); SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_map, K * 4));
    SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_group, K * 4)); SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_cnt, K * 4)); SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_first, K * 4));
    SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_si, K * 4)); SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_mark, K * 4)); SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_add_slot, K * 4));
    SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_add_seq, K * 8)); SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_rows, sizeof(int4) * (size_t)max_maps));
    SGS_CUDA_TRY_AT(fn, R.alloc(&db->d_loop, sizeof(int4) * (size_t)max_maps));
    SGS_CUDA_TRY_AT(fn, cudaMemset(db->d_score, 0, K * 4)); SGS_CUDA_TRY_AT(fn, cudaMemset(db->d_n, 0, K * 4));
    if (publish_groups(db.get(), fn, nullptr) != SGS_OK) return SGS_ERR_CUDA;
    SGS_CUDA_TRY_AT(fn, cudaDeviceSynchronize());
    *out = db.release();
    return SGS_OK;
}

SGS_API int sgs_kfdb_add(sgs_kfdb* db, int n, const int32_t* slot, const int32_t* map, const int32_t* d_bow_word, const double* d_bow_value,
                         const int32_t* d_bow_n, int bow_cap, void* stream) {
    const char* const fn = "sgs_kfdb_add";
    if (!db || n < 0 || (n > 0 && (!slot || !map || !d_bow_word || !d_bow_value || !d_bow_n || bow_cap < 1))) { set_error("%s: bad argument", fn); return SGS_ERR_INVALID; }
    if (n == 0) return SGS_OK;
    const int K = db->max_keyframes;
    if (n > K) { set_error("%s: %d key frames in one call, the handle has %d slots", fn, n, K); return SGS_ERR_INVALID; }
    std::vector<uint8_t> seen(K, 0);
    for (int i = 0; i < n; ++i) {
        if (slot[i] < 0 || slot[i] >= K) { set_error("%s: slot %d out of range [0, %d)", fn, slot[i], K); return SGS_ERR_INVALID; }
        if (db->slot_map[slot[i]] >= 0 || seen[slot[i]]) { set_error("%s: slot %d is already live", fn, slot[i]); return SGS_ERR_INVALID; }
        if (map[i] < 0 || map[i] >= db->max_maps) { set_error("%s: map %d out of range [0, %d)", fn, map[i], db->max_maps); return SGS_ERR_INVALID; }
        seen[slot[i]] = 1;
    }
    if (db->next_seq + (uint64_t)n > kSeqLimit) { set_error("%s: the add counter is exhausted", fn); return SGS_ERR_CAPACITY; }
    cudaStream_t st = (cudaStream_t)stream;
    SGS_CUDA_TRY_AT(fn, cudaSetDevice(db->device));
    std::vector<int32_t> bn(n);
    SGS_CUDA_TRY_AT(fn, cudaMemcpyAsync(bn.data(), d_bow_n, 4 * (size_t)n, cudaMemcpyDeviceToHost, st));
    SGS_CUDA_TRY_AT(fn, cudaStreamSynchronize(st));
    for (int i = 0; i < n; ++i)
        if (bn[i] < 0 || bn[i] > db->max_words || bn[i] > bow_cap) {
            set_error("%s: BowVector %d has %d words (max_words %d, bow_cap %d)", fn, i, bn[i], db->max_words, bow_cap); return SGS_ERR_INVALID; }
    std::vector<uint64_t> seq(n);
    for (int i = 0; i < n; ++i) seq[i] = db->next_seq + (uint64_t)i;
    SGS_CUDA_TRY_AT(fn, cudaMemcpyAsync(db->d_add_slot, slot, 4 * (size_t)n, cudaMemcpyHostToDevice, st));
    SGS_CUDA_TRY_AT(fn, cudaMemcpyAsync(db->d_add_seq, seq.data(), 8 * (size_t)n, cudaMemcpyHostToDevice, st));
    kfdb_add_kernel<<<n, 128, 0, st>>>(db->d_add_slot, db->d_add_seq, d_bow_word, d_bow_value, d_bow_n, bow_cap, db->max_words, db->d_word, db->d_value,
                                       db->d_n, db->d_seq, db->d_score);
    SGS_CUDA_TRY_AT(fn, cudaGetLastError());
    for (int i = 0; i < n; ++i) { db->slot_map[slot[i]] = map[i]; db->slot_seq[slot[i]] = seq[i]; }
    db->next_seq += (uint64_t)n;
    return publish_groups(db, fn, st);
}

SGS_API int sgs_kfdb_erase(sgs_kfdb* db, int n, const int32_t* slot, void* stream) {
    const char* const fn = "sgs_kfdb_erase";
    if (!db || n < 0 || (n > 0 && !slot)) { set_error("%s: bad argument", fn); return SGS_ERR_INVALID; }
    std::vector<uint8_t> seen(db->max_keyframes, 0);
    for (int i = 0; i < n; ++i) {
        if (slot[i] < 0 || slot[i] >= db->max_keyframes || db->slot_map[slot[i]] < 0 || seen[slot[i]]) {
            set_error("%s: slot %d is not live", fn, slot[i]); return SGS_ERR_INVALID; }
        seen[slot[i]] = 1;
    }
    if (n == 0) return SGS_OK;
    for (int i = 0; i < n; ++i) db->slot_map[slot[i]] = -1;
    return publish_groups(db, fn, (cudaStream_t)stream);
}

SGS_API int sgs_kfdb_clear(sgs_kfdb* db, int map, void* stream) {
    const char* const fn = "sgs_kfdb_clear";
    if (!db || map < 0 || map >= db->max_maps) { set_error("%s: bad argument", fn); return SGS_ERR_INVALID; }
    for (int32_t& m : db->slot_map) if (m == map) m = -1;
    return publish_groups(db, fn, (cudaStream_t)stream);
}

SGS_API int sgs_kfdb_reloc_scores(const sgs_kfdb* db, float* out) {
    if (!db || !out) { set_error("sgs_kfdb_reloc_scores: bad argument"); return SGS_ERR_INVALID; }
    SGS_CUDA_TRY_AT("sgs_kfdb_reloc_scores", cudaSetDevice(db->device));
    SGS_CUDA_TRY_AT("sgs_kfdb_reloc_scores", cudaMemcpy(out, db->d_score, 4 * (size_t)db->max_keyframes, cudaMemcpyDeviceToHost));
    return SGS_OK;
}

SGS_API int sgs_kfdb_reloc_candidates_device(sgs_kfdb* db, int nframes, const int32_t* map, const int32_t* d_bow_word, const double* d_bow_value,
                                             const int32_t* d_bow_n, int bow_cap, const int32_t* d_covis, int32_t* d_cand, int cand_cap, int32_t* d_ncand,
                                             int32_t* d_stats, void* stream) {
    const char* const fn = "sgs_kfdb_reloc_candidates_device";
    if (!db || !map || nframes < 1 || !d_bow_word || !d_bow_value || !d_bow_n || !d_covis || !d_cand || !d_ncand || !d_stats || cand_cap < 1 || bow_cap < 1) {
        set_error("%s: bad argument", fn); return SGS_ERR_INVALID; }
    if (bow_cap > kMaxBowCap) { set_error("%s: bow_cap %d above %d", fn, bow_cap, kMaxBowCap); return SGS_ERR_UNSUPPORTED; }
    std::vector<int4> rows;
    int max_len = 0;
    const int rc = kfdb_plan_query(db, fn, nframes, map, rows, &max_len);
    if (rc != SGS_OK) return rc;
    return kfdb_launch_query(db, fn, rows, max_len, d_bow_word, d_bow_value, d_bow_n, bow_cap, d_covis, d_cand, cand_cap, d_ncand, d_stats, (cudaStream_t)stream);
}

// CSR offsets off[0 .. nframes] (host): from 0 or more, not decreasing
static bool offsets_ok(const int32_t* off, int nframes) {
    if (off[0] < 0) return false;
    for (int f = 0; f < nframes; ++f) if (off[f + 1] < off[f]) return false;
    return true;
}

SGS_API int sgs_kfdb_loop_candidates_device(sgs_kfdb* db, int nframes, const int32_t* map, const int32_t* d_bow_word, const double* d_bow_value,
                                            const int32_t* d_bow_n, int bow_cap, const int32_t* conn_off, const int32_t* d_conn, const int32_t* cov_off,
                                            const int32_t* d_cov_word, const double* d_cov_value, const int32_t* d_cov_n, const int32_t* d_covis,
                                            int32_t* d_cand, int cand_cap, int32_t* d_ncand, int32_t* d_stats, float* d_min_score, void* stream) {
    const char* const fn = "sgs_kfdb_loop_candidates_device";
    if (!db || !map || nframes < 1 || !d_bow_word || !d_bow_value || !d_bow_n || !conn_off || !cov_off || !d_covis || !d_cand || !d_ncand || !d_stats ||
        !d_min_score || cand_cap < 1 || bow_cap < 1) {
        set_error("%s: bad argument", fn); return SGS_ERR_INVALID; }
    if (bow_cap > kMaxBowCap) { set_error("%s: bow_cap %d above %d", fn, bow_cap, kMaxBowCap); return SGS_ERR_UNSUPPORTED; }
    if (!offsets_ok(conn_off, nframes) || !offsets_ok(cov_off, nframes)) { set_error("%s: CSR offsets negative or decreasing", fn); return SGS_ERR_INVALID; }
    if ((conn_off[nframes] > conn_off[0] && !d_conn) || (cov_off[nframes] > cov_off[0] && (!d_cov_word || !d_cov_value || !d_cov_n))) {
        set_error("%s: connected ids or covisible BowVectors given without their arrays", fn); return SGS_ERR_INVALID; }
    std::vector<int4> rows;
    int max_len = 0;
    const int rc = kfdb_plan_query(db, fn, nframes, map, rows, &max_len);
    if (rc != SGS_OK) return rc;
    KfdbLoop loop{{}, d_conn, d_cov_word, d_cov_value, d_cov_n, d_min_score};
    for (const int4& r : rows) loop.ranges.push_back(make_int4(conn_off[r.x], conn_off[r.x + 1], cov_off[r.x], cov_off[r.x + 1]));
    return launch_query(db, fn, rows, max_len, d_bow_word, d_bow_value, d_bow_n, bow_cap, d_covis, d_cand, cand_cap, d_ncand, d_stats, &loop,
                        (cudaStream_t)stream);
}

}  // extern "C"
