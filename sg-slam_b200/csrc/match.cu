// match.cu -- projection matchers of ORBmatcher on the GPU, batched over independent frames (one block per frame).
//
//   match_lastframe_kernel : ORBmatcher::SearchByProjection(Frame&, const Frame&, th, bMono)   src/ORBmatcher.cc:1332-1472
//   match_localmap_kernel  : ORBmatcher::SearchByProjection(Frame&, vector<MapPoint*>&, th)    src/ORBmatcher.cc:45-129
//
// Both reference loops are order dependent (a keypoint already holding a map point with Observations()>0 is skipped,
// last writer wins).  Exact restatement in three phases per frame:
//   1. the Frame grid (Frame::AssignFeaturesToGrid, src/Frame.cc:257-272) as a counting sort of the keypoints by cell
//      (cell = ix*48+iy, ascending keypoint index inside a cell): ascending position in that array == the iteration order of
//      Frame::GetFeaturesInArea (src/Frame.cc:354-407);
//   2. every map point scores its window in parallel (one THREAD per point: windows hold a handful of candidates) IGNORING
//      claims -> optimistic best (and second best);
//   3. one warp resolves the points in index order, 32 at a time: a point whose optimistic keypoints are neither claimed nor
//      tentatively claimed by an earlier point of the chunk is final; the first blocked point of a chunk is rescanned with
//      the claims in force (rare), then the rest of the chunk is re-evaluated.  This reproduces the sequential semantics.
// The sequential "dist < best" / "dist < second" updates keep the two smallest candidates under the order
// (distance, iteration position): a thread walking its window in iteration order gets them with the same comparisons.
#include <cuda_runtime.h>

#include <vector>

#include "match_dev.cuh"
#include "sgs_common.h"

namespace sgs {

constexpr int kMatchThreads = 256;
constexpr int kGridCols = 64, kGridRows = 48;         // FRAME_GRID_COLS / ROWS, include/Frame.h:39-40
constexpr int kGridCells = kGridCols * kGridRows;
constexpr uint32_t kNoKey = 0xFFFFFFFFu;

struct FrameSmem {
    uint16_t* order;     // [cap]  keypoint indices sorted by (cell, index)
    float* kx; float* ky; float* ur;
    uint8_t* oct;
    uint8_t* claimed;    // 1 = holds a map point with Observations() > 0
    uint8_t* tent;       // tentative claims of the chunk being resolved (lane + 1, 0 = none)
    int32_t* cell_start; // [kGridCells + 1]
    int32_t* cursor;     // [kGridCells] scatter cursors
};

__host__ __device__ inline size_t frame_smem_bytes(int cap) {
    const size_t c = (size_t)((cap + 15) & ~15);
    return c * (2 + 4 + 4 + 4 + 1 + 1 + 1) + (size_t)(kGridCells + 1) * 4 + (size_t)kGridCells * 4 + 256;
}

__device__ __forceinline__ void carve(uint8_t* base, int cap, FrameSmem& s) {
    const size_t c = (size_t)((cap + 15) & ~15);
    s.kx = reinterpret_cast<float*>(base); base += c * 4;
    s.ky = reinterpret_cast<float*>(base); base += c * 4;
    s.ur = reinterpret_cast<float*>(base); base += c * 4;
    s.cell_start = reinterpret_cast<int32_t*>(base); base += (size_t)(kGridCells + 1) * 4;
    s.cursor = reinterpret_cast<int32_t*>(base); base += (size_t)kGridCells * 4;
    s.order = reinterpret_cast<uint16_t*>(base); base += c * 2;
    s.oct = base; base += c;
    s.claimed = base; base += c;
    s.tent = base;
}

struct GridScale { float w_inv, h_inv; };

// Frame::mfGridElementWidthInv / mfGridElementHeightInv (src/Frame.cc:183-184)
__device__ __forceinline__ GridScale grid_scale(const sgs_camera& cam) {
    return {__fdiv_rn((float)kGridCols, __fsub_rn(cam.max_x, cam.min_x)), __fdiv_rn((float)kGridRows, __fsub_rn(cam.max_y, cam.min_y))};
}

// Frame::PosInGrid (src/Frame.cc:409-419): round() is half away from zero; cell = ix * kGridRows + iy
__device__ __forceinline__ bool pos_in_grid(const sgs_camera& cam, GridScale g, float x, float y, int& cell) {
    const int px = (int)roundf(__fmul_rn(__fsub_rn(x, cam.min_x), g.w_inv));
    const int py = (int)roundf(__fmul_rn(__fsub_rn(y, cam.min_y), g.h_inv));
    cell = px * kGridRows + py;
    return px >= 0 && px < kGridCols && py >= 0 && py < kGridRows;
}

// The cells Frame::GetFeaturesInArea (src/Frame.cc:354-407) visits for the window of half-size r around (x, y): columns min_cx..max_cx,
// rows min_cy..max_cy.  False when the window misses the grid.
__device__ __forceinline__ bool feature_window(const sgs_camera& cam, GridScale g, float x, float y, float r, int& min_cx, int& max_cx, int& min_cy,
                                               int& max_cy) {
    min_cx = max(0, (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(x, cam.min_x), r), g.w_inv)));
    max_cx = min(kGridCols - 1, (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(x, cam.min_x), r), g.w_inv)));
    min_cy = max(0, (int)floorf(__fmul_rn(__fsub_rn(__fsub_rn(y, cam.min_y), r), g.h_inv)));
    max_cy = min(kGridRows - 1, (int)ceilf(__fmul_rn(__fadd_rn(__fsub_rn(y, cam.min_y), r), g.h_inv)));
    return min_cx < kGridCols && max_cx >= 0 && min_cy < kGridRows && max_cy >= 0;
}

// counting sort by cell; entries of a cell end up in ascending keypoint index (== push_back order of AssignFeaturesToGrid)
__device__ void build_frame_grid(const sgs_camera& cam, const sgs_keypoint* __restrict__ kps, const float* __restrict__ uright, int n, FrameSmem& s) {
    __shared__ int s_scan[kMatchThreads];
    const GridScale g = grid_scale(cam);
    const int tid = threadIdx.x;
    for (int c = tid; c <= kGridCells; c += kMatchThreads) s.cell_start[c] = 0;
    __syncthreads();
    // histogram (cell id kept in `order` temporarily is not needed: recomputed in the scatter pass)
    for (int i = tid; i < n; i += kMatchThreads) {
        const sgs_keypoint kp = kps[i];
        s.kx[i] = kp.x; s.ky[i] = kp.y; s.oct[i] = (uint8_t)kp.octave; s.ur[i] = uright ? uright[i] : -1.f;
        int cell;
        if (pos_in_grid(cam, g, kp.x, kp.y, cell)) atomicAdd(&s.cell_start[cell + 1], 1);
    }
    __syncthreads();
    // inclusive scan of cell_start[1..kGridCells] (12 cells per thread + block scan of the partial sums)
    constexpr int kPer = kGridCells / kMatchThreads;   // 3072 / 256 = 12
    int local = 0;
    for (int k = 0; k < kPer; ++k) local += s.cell_start[1 + tid * kPer + k];
    s_scan[tid] = local;
    __syncthreads();
    for (int o = 1; o < kMatchThreads; o <<= 1) {
        const int v = tid >= o ? s_scan[tid - o] : 0;
        __syncthreads();
        s_scan[tid] += v;
        __syncthreads();
    }
    int run = s_scan[tid] - local;
    for (int k = 0; k < kPer; ++k) {
        const int c = tid * kPer + k;
        const int cnt = s.cell_start[1 + c];
        s.cursor[c] = run;
        run += cnt;
        s.cell_start[1 + c] = run;
    }
    __syncthreads();
    // scatter (unordered inside a cell), then order each cell's few entries by keypoint index
    for (int i = tid; i < n; i += kMatchThreads) {
        int cell;
        if (pos_in_grid(cam, g, s.kx[i], s.ky[i], cell)) s.order[atomicAdd(&s.cursor[cell], 1)] = (uint16_t)i;
    }
    __syncthreads();
    for (int c = tid; c < kGridCells; c += kMatchThreads) {
        const int b = s.cell_start[c], e = s.cell_start[c + 1];
        for (int i = b + 1; i < e; ++i) {               // insertion sort: cells hold ~0.3 keypoints on average
            const uint16_t v = s.order[i];
            int j = i - 1;
            while (j >= b && s.order[j] > v) { s.order[j + 1] = s.order[j]; --j; }
            s.order[j + 1] = v;
        }
    }
    __syncthreads();
}

struct TopK { uint32_t k[kTopK]; int ngated; };  // keys ascending; key = dist << 16 | position in the sorted array; 0xFFFFFFFF = none

__device__ __forceinline__ void topk_init(TopK& t) {
#pragma unroll
    for (int i = 0; i < kTopK; ++i) t.k[i] = 0xFFFFFFFFu;
    t.ngated = 0;
}

__device__ __forceinline__ void topk_insert(TopK& t, uint32_t k) {   // insertion into the sorted kTopK-array (keys are unique)
#pragma unroll
    for (int i = 0; i < kTopK; ++i) {
        const uint32_t lo = min(t.k[i], k);
        k = max(t.k[i], k);
        t.k[i] = lo;
    }
}

// Frame::GetFeaturesInArea + the candidate loop shared by both matchers.  A group of `gsize` lanes (1 or kGroup) shares one
// window: lane `gl` of the group takes the entries j = beg+gl, beg+gl+gsize, ... of every cell column; the caller min-reduces
// the (dist, position) keys across the group, which gives exactly the sequential loop's best / second best.
//   use_claims : skip keypoints whose `claimed` flag is set (phase-3 rescans); phase 2 passes false
// Returns the kTopK smallest (dist, position) keys seen by this lane and how many candidates passed the gates;
// *ncand accumulates this lane's share of |vIndices|.
__device__ TopK scan_window(const sgs_camera& cam, const FrameSmem& s, const uint4* __restrict__ cur_desc, float x, float y, float r,
                            int min_level, int max_level, const uint4& d0, const uint4& d1, bool use_claims, float ur_pred, float ur_tol,
                            int* ncand, int gl = 0, int gsize = 1) {
    TopK t; topk_init(t);
    int min_cx, max_cx, min_cy, max_cy;
    if (!feature_window(cam, grid_scale(cam), x, y, r, min_cx, max_cx, min_cy, max_cy)) return t;
    const bool check_levels = (min_level > 0) || (max_level >= 0);
    int cnt = 0;
    for (int ix = min_cx; ix <= max_cx; ++ix) {
        // cells (ix, min_cy..max_cy) are contiguous in the sorted array
        const int beg = s.cell_start[ix * kGridRows + min_cy], end = s.cell_start[ix * kGridRows + max_cy + 1];
        for (int j = beg + gl; j < end; j += gsize) {
            const int idx = s.order[j];
            const int o = s.oct[idx];
            if (check_levels) {
                if (o < min_level) continue;
                if (max_level >= 0 && o > max_level) continue;
            }
            const float dx = __fsub_rn(s.kx[idx], x), dy = __fsub_rn(s.ky[idx], y);
            if (!(fabsf(dx) < r && fabsf(dy) < r)) continue;
            ++cnt;                                            // member of vIndices
            if (use_claims && s.claimed[idx]) continue;       // :87-89 / :1407-1409
            const float ur = s.ur[idx];
            if (ur > 0.f) {                                   // :91-96 / :1411-1417
                const float er = fabsf(__fsub_rn(ur_pred, ur));
                if (er > ur_tol) continue;
            }
            const uint32_t k = ((uint32_t)descriptor_distance(d0, d1, __ldg(&cur_desc[2 * idx]), __ldg(&cur_desc[2 * idx + 1])) << 16) | (uint32_t)j;
            topk_insert(t, k);
            ++t.ngated;
        }
    }
    if (ncand) *ncand += cnt;
    return t;
}

constexpr int kGroup = 4;   // lanes cooperating on one map point in phase 2

__device__ __forceinline__ TopK group_topk(TopK t) {   // merge over the kGroup lanes of a group (xor butterfly stays inside it)
#pragma unroll
    for (int o = kGroup >> 1; o > 0; o >>= 1) {
        uint32_t other[kTopK];
#pragma unroll
        for (int i = 0; i < kTopK; ++i) other[i] = __shfl_xor_sync(0xffffffffu, t.k[i], o);
        t.ngated += __shfl_xor_sync(0xffffffffu, t.ngated, o);
#pragma unroll
        for (int i = 0; i < kTopK; ++i) topk_insert(t, other[i]);
    }
    return t;
}

// First two candidates of a point's list whose keypoints are not claimed (claims only ever remove candidates, so this is what
// the sequential loop would find); need_rescan: the list ran out although the window held more than kTopK candidates.
__device__ __forceinline__ void select_unclaimed(const FrameSmem& s, const uint32_t (&cand)[kTopK], int ngated, int want, uint32_t& k1, uint32_t& k2,
                                                 bool& need_rescan) {
    k1 = kNoKey; k2 = kNoKey;
    int found = 0;
#pragma unroll
    for (int c = 0; c < kTopK; ++c) {
        const uint32_t key = cand[c];
        if (key != kNoKey && !s.claimed[s.order[key & 0xFFFFu]]) {
            if (found == 0) k1 = key; else if (found == 1) k2 = key;
            ++found;
        }
    }
    need_rescan = found < want && ngated > kTopK;
}

// Ordered resolution of one chunk of <= 32 points by one warp (lane == point).  `Policy` supplies:
//   decide(keys, keypoints) -> accept + target keypoint, rescan() -> complete candidate list under the current claims,
//   record(target) (histogram), commit(target) (writes the match and the claim).
// Returns the number of accepted points in the chunk (warp-uniform).
template <class Policy>
__device__ int resolve_chunk(FrameSmem& s, Policy& pol, bool have_point, const uint32_t (&cand)[kTopK], int ngated) {
    const int lane = threadIdx.x & 31;
    const unsigned lt = (1u << lane) - 1;
    const int want = pol.uses_second() ? 2 : 1;
    bool pending = have_point && cand[0] != kNoKey;
    int accepted = 0;
    for (;;) {
        if (!__ballot_sync(0xffffffffu, pending)) break;
        uint32_t k1 = kNoKey, k2 = kNoKey;
        bool need_rescan = false, acc = false;
        int i1 = -1, i2 = -1, target = -1;
        if (pending) {
            select_unclaimed(s, cand, ngated, want, k1, k2, need_rescan);
            if (k1 != kNoKey) {
                i1 = s.order[k1 & 0xFFFFu];
                i2 = k2 != kNoKey ? (int)s.order[k2 & 0xFFFFu] : -1;
                acc = pol.decide(k1, k2, i1, i2, target);
            }
        }
        const bool claims = pending && !need_rescan && acc && pol.blocks_others();
        {   // the lowest claiming lane per keypoint records a tentative claim
            const unsigned same = __match_any_sync(0xffffffffu, claims ? target : -1 - lane);
            if (claims && (same & lt) == 0) s.tent[target] = (uint8_t)(lane + 1);
        }
        __syncwarp();
        bool blocked = false;
        if (pending) {
            blocked = need_rescan;
            if (!blocked && k1 != kNoKey && (acc || !pol.reject_is_final())) {
                const int t1 = s.tent[i1], t2 = (want == 2 && i2 >= 0) ? s.tent[i2] : 0;
                blocked = (t1 != 0 && t1 - 1 < lane) || (t2 != 0 && t2 - 1 < lane);
            }
        }
        const unsigned bm = __ballot_sync(0xffffffffu, blocked);
        const int fb = bm ? __ffs(bm) - 1 : 32;
        __syncwarp();
        if (claims) s.tent[target] = 0;                                  // clear the scratch
        __syncwarp();
        // finalize every pending lane below the first blocked one
        const bool fin = pending && lane < fb;
        const bool fin_acc = fin && acc;
        {
            const unsigned fm = __ballot_sync(0xffffffffu, fin_acc);
            if (fin_acc) {
                const unsigned same = __match_any_sync(fm, target);
                pol.record(target);                                       // histogram / events (order irrelevant)
                if ((same >> lane) == 1u) pol.commit(target);             // last writer wins: highest lane of the group
            }
            accepted += __popc(fm);
        }
        if (fin) pending = false;
        __syncwarp();
        // the first blocked lane is next in sequence: decide it against the claims now in force
        if (fb < 32) {
            bool a2 = false;
            if (lane == fb) {
                uint32_t n1, n2; bool rs;
                select_unclaimed(s, cand, ngated, want, n1, n2, rs);
                if (rs) { const TopK t = pol.rescan(); n1 = t.k[0]; n2 = t.k[1]; }
                int tgt = -1;
                if (n1 != kNoKey) {
                    const int j1 = s.order[n1 & 0xFFFFu];
                    const int j2 = n2 != kNoKey ? (int)s.order[n2 & 0xFFFFu] : -1;
                    a2 = pol.decide(n1, n2, j1, j2, tgt);
                }
                if (a2) { pol.record(tgt); pol.commit(tgt); }
                pending = false;
            }
            accepted += __shfl_sync(0xffffffffu, a2 ? 1 : 0, fb);
            __syncwarp();
        }
    }
    return accepted;
}

// end of both projection matchers: the frame's |vIndices| total (summed over the block) and its match count
__device__ __forceinline__ void write_totals(int ncand, int nmatch, unsigned long long* ncand_out, int32_t* nmatches_out) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) ncand += __shfl_xor_sync(0xffffffffu, ncand, o);
    if ((threadIdx.x & 31) == 0 && ncand) atomicAdd(ncand_out, (unsigned long long)ncand);
    if (threadIdx.x == 0) *nmatches_out = nmatch;
}

// ---------------------------------------------------------------------------------------------------------------------
struct LastPolicy {
    const LastFrameArgs& A; FrameSmem& s; const uint4* cur_desc; const sgs_keypoint* kps; int32_t* cur_mp; int* hist; int* n_event;
    int64_t lo; int point; PointPre pp;
    __device__ bool uses_second() const { return false; }
    __device__ bool reject_is_final() const { return true; }     // best distance > TH_HIGH: no candidate can be accepted
    __device__ bool blocks_others() const { return A.kf_mode || ((A.last_flags[lo + point] >> 1) & 1) != 0; }
    __device__ bool decide(uint32_t k1, uint32_t, int i1, int, int& target) const { target = i1; return (int)(k1 >> 16) <= A.orb_dist; }   // :1430 / :1559
    __device__ TopK rescan() const {
        const uint4* dm = reinterpret_cast<const uint4*>(A.last_desc + 32 * (lo + point));
        return scan_window(A.cam, s, cur_desc, pp.u, pp.v, pp.radius, pp.min_level, pp.max_level, __ldg(dm), __ldg(dm + 1), true,
                           __fsub_rn(pp.u, __fmul_rn(A.cam.bf, pp.invz)), A.kf_mode ? __int_as_float(0x7f800000) : pp.radius, nullptr);
    }
    __device__ void record(int target) const {
        if (!A.check_ori) return;
        const int bin = rotation_bin(A.last_angle[lo + point], kps[target].angle);      // :1438-1443
        atomicAdd(&hist[bin], 1);
        A.events[lo + atomicAdd(n_event, 1)] = (bin << 16) | target;
    }
    __device__ void commit(int target) const {
        cur_mp[target] = point;                                                   // :1432 last writer wins
        s.claimed[target] = A.kf_mode ? 1 : ((A.last_flags[lo + point] >> 1) & 1);     // KeyFrame variant: any assigned keypoint is skipped (:1543)
    }
};

__global__ void __launch_bounds__(kMatchThreads) match_lastframe_kernel(const __grid_constant__ LastFrameArgs A) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ int hist[kHistoLen];
    __shared__ int s_nmatch, s_nevent;
    __shared__ float s_pose[20];     // Rcw (9), tcw (3), forward/backward flags, Ow (3)
    const int f = blockIdx.x;
    if (A.frame_enable && !A.frame_enable[f]) return;      // block-uniform
    const int n = min(A.cur_n[f], A.cur_cap);
    const int nlast = min(A.last_n[f], A.last_cap);
    FrameSmem s;
    carve(smem, A.cur_cap, s);
    const sgs_keypoint* kps = A.cur_kps + (int64_t)f * A.cur_cap;
    const uint4* cur_desc = reinterpret_cast<const uint4*>(A.cur_desc + (int64_t)f * A.cur_cap * 32);
    int32_t* cur_mp = A.cur_mp + (int64_t)f * A.cur_cap;
    const int64_t lo = (int64_t)f * A.last_cap;
    if (threadIdx.x < kHistoLen) hist[threadIdx.x] = 0;
    if (threadIdx.x == 0) {
        s_nmatch = 0; s_nevent = 0;
        // Rcw, tcw, twc = -Rcw^T tcw, tlc = Rlw twc + tlw (:1342-1351).  cv::gemm on CV_32F: the transposed product takes the general path
        // (double accumulator, one rounding); the plain product takes the small-matrix path (gemm3_row).
        const float* Tc = A.tcw_cur + 16 * f; const float* Tl = A.kf_mode ? Tc : A.tcw_last + 16 * f;
        float twc[3];
        for (int r = 0; r < 3; ++r) {
            double acc = 0.0;
            for (int k = 0; k < 3; ++k) acc = __dadd_rn(acc, __dmul_rn((double)(-Tc[4 * k + r]), (double)Tc[4 * k + 3]));
            twc[r] = (float)acc;
        }
        const float tlc2 = gemm3_row(Tl[8], Tl[9], Tl[10], twc, Tl[11]);
        const float mb = __fdiv_rn(A.cam.bf, A.cam.fx);       // Frame.cc:196
        for (int r = 0; r < 3; ++r) { for (int c = 0; c < 3; ++c) s_pose[3 * r + c] = Tc[4 * r + c]; s_pose[9 + r] = Tc[4 * r + 3]; }
        s_pose[12] = (!A.kf_mode && tlc2 > mb && !A.mono) ? 1.f : 0.f;
        s_pose[13] = (!A.kf_mode && -tlc2 > mb && !A.mono) ? 1.f : 0.f;
        s_pose[14] = twc[0]; s_pose[15] = twc[1]; s_pose[16] = twc[2];       // Ow = -Rcw^T tcw (KeyFrame variant, :1480)
    }
    build_frame_grid(A.cam, kps, A.cur_uright + (int64_t)f * A.cur_cap, n, s);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const bool has = cur_mp[i] >= 0;
        s.claimed[i] = has ? (A.cur_mp_obs_in ? A.cur_mp_obs_in[(int64_t)f * A.cur_cap + i] : 1) : 0;
        s.tent[i] = 0;
    }
    __syncthreads();
    const bool fwd = s_pose[12] != 0.f, bwd = s_pose[13] != 0.f;
    PointPre* pre = A.pre + lo;
    int ncand = 0;
    // phase 2: optimistic scoring, kGroup lanes per last-frame point (uniform trip count so that the group shuffles are safe)
    const int gl = threadIdx.x & (kGroup - 1);
    const int ngroups = blockDim.x / kGroup;
    for (int i0 = 0; i0 < nlast; i0 += ngroups) {
        const int i = i0 + threadIdx.x / kGroup;
        PointPre pp; pp.valid = 0; pp.ngated = 0; pp.u = pp.v = pp.invz = pp.radius = 0.f; pp.min_level = pp.max_level = 0;
        TopK t; topk_init(t);
        if (i < nlast && (A.last_flags[lo + i] & 1)) {
            const float* X = A.last_xyz + 3 * (lo + i);
            float xc[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) xc[r] = gemm3_row(s_pose[3 * r], s_pose[3 * r + 1], s_pose[3 * r + 2], X, s_pose[9 + r]);   // Rcw * x3Dw + tcw
            const float invz = (float)__ddiv_rn(1.0, (double)xc[2]);                       // :1369 / :1506
            if (A.kf_mode || !(invz < 0.f)) {
                const float u = __fadd_rn(__fmul_rn(__fmul_rn(A.cam.fx, xc[0]), invz), A.cam.cx);
                const float v = __fadd_rn(__fmul_rn(__fmul_rn(A.cam.fy, xc[1]), invz), A.cam.cy);
                if (!(u < A.cam.min_x || u > A.cam.max_x) && !(v < A.cam.min_y || v > A.cam.max_y)) {
                    bool ok = true;
                    int oct, mn, mx;
                    if (A.kf_mode) {          // :1517-1531: distance inside the scale-invariance range, level from MapPoint::PredictScale
                        const float px = __fsub_rn(X[0], s_pose[14]), py = __fsub_rn(X[1], s_pose[15]), pz = __fsub_rn(X[2], s_pose[16]);
                        const float dist = (float)sqrt(((double)px * px + (double)py * py) + (double)pz * pz);
                        const float maxd = A.kf_max_dist[lo + i];
                        ok = !(dist < __fmul_rn(0.8f, A.kf_min_dist[lo + i]) || dist > __fmul_rn(1.2f, maxd));
                        oct = predict_scale(maxd, dist, A.log_sf, A.cam.nlevels);
                        mn = oct - 1; mx = oct + 1;
                    } else {
                        oct = A.last_octave[lo + i];
                        if (fwd) { mn = oct; mx = -1; } else if (bwd) { mn = 0; mx = oct; } else { mn = oct - 1; mx = oct + 1; }
                    }
                    if (ok) {
                        const float radius = __fmul_rn(A.th, A.cam.scale_factors[oct]);
                        pp.valid = 1; pp.u = u; pp.v = v; pp.invz = invz; pp.radius = radius; pp.min_level = mn; pp.max_level = mx;
                        const uint4* dm = reinterpret_cast<const uint4*>(A.last_desc + 32 * (lo + i));
                        const float ur_pred = __fsub_rn(u, __fmul_rn(A.cam.bf, invz));
                        t = scan_window(A.cam, s, cur_desc, u, v, radius, mn, mx, __ldg(dm), __ldg(dm + 1), false, ur_pred,
                                        A.kf_mode ? __int_as_float(0x7f800000) : radius, &ncand, gl, kGroup);
                    }
                }
            }
        }
        t = group_topk(t);
#pragma unroll
        for (int c = 0; c < kTopK; ++c) pp.k[c] = t.k[c];
        pp.ngated = (int16_t)min(t.ngated, 32767);
        if (gl == 0 && i < nlast) pre[i] = pp;
    }
    __syncthreads();
    // phase 3: ordered resolution by warp 0, 32 points at a time
    if (threadIdx.x < 32) {
        int nmatch = 0;
        for (int c0 = 0; c0 < nlast; c0 += 32) {
            const int i = c0 + threadIdx.x;
            LastPolicy pol{A, s, cur_desc, kps, cur_mp, hist, &s_nevent, lo, i, PointPre()};
            bool have = false;
            if (i < nlast) { pol.pp = pre[i]; have = pol.pp.valid != 0; }
            else { for (int c = 0; c < kTopK; ++c) pol.pp.k[c] = kNoKey; }
            nmatch += resolve_chunk(s, pol, have, pol.pp.k, pol.pp.ngated);
        }
        if (threadIdx.x == 0) s_nmatch = nmatch;
    }
    __syncthreads();
    if (A.check_ori) {                                             // :1451-1470
        int removed = drop_outside_main_bins(hist, A.events + lo, s_nevent, cur_mp);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) removed += __shfl_xor_sync(0xffffffffu, removed, o);
        __syncthreads();
        if ((threadIdx.x & 31) == 0 && removed) atomicSub(&s_nmatch, removed);
    }
    __syncthreads();
    write_totals(ncand, s_nmatch, &A.ncand[f], &A.nmatches[f]);
}

// ---------------------------------------------------------------------------------------------------------------------
struct LocalPolicy {
    const sgs_localmap_batch& A; FrameSmem& s; const uint4* cur_desc; int32_t* f_mp; uint8_t* f_obs; int64_t lo; int point;
    __device__ bool uses_second() const { return true; }
    __device__ bool reject_is_final() const { return false; }    // a ratio-test rejection can flip once a top-2 keypoint is claimed
    __device__ bool blocks_others() const { return A.mp_obs[lo + point] != 0; }
    __device__ bool decide(uint32_t k1, uint32_t k2, int i1, int i2, int& target) const {
        target = i1;
        const int best_dist = (int)(k1 >> 16);
        if (best_dist > kThHigh) return false;                                                     // :116
        const int best_level = s.oct[i1];
        int best_level2 = -1, best_dist2 = 256;
        if (i2 >= 0) { best_dist2 = (int)(k2 >> 16); best_level2 = s.oct[i2]; }
        if (best_level == best_level2 && (float)best_dist > __fmul_rn(A.nnratio, (float)best_dist2)) return false;   // :118-119
        return true;
    }
    __device__ void window(float& rr, int& lvl) const {
        lvl = A.level[lo + point];
        float r = ((double)A.view_cos[lo + point] > 0.998) ? 2.5f : 4.0f;   // RadiusByViewingCos :131-137 (compared in double)
        if (A.th != 1.0f) r = __fmul_rn(r, A.th);                           // bFactor :50,:67-68
        rr = __fmul_rn(r, A.cam.scale_factors[lvl]);
    }
    __device__ TopK rescan() const {
        float rr; int lvl;
        window(rr, lvl);
        const uint4* dm = reinterpret_cast<const uint4*>(A.mp_desc + 32 * (lo + point));
        return scan_window(A.cam, s, cur_desc, A.proj_x[lo + point], A.proj_y[lo + point], rr, lvl - 1, lvl, __ldg(dm), __ldg(dm + 1), true,
                           A.proj_xr[lo + point], rr, nullptr);
    }
    __device__ void record(int) const {}
    __device__ void commit(int target) const {
        f_mp[target] = A.id_base + point;
        const uint8_t ob = A.mp_obs[lo + point];
        f_obs[target] = ob;
        s.claimed[target] = ob ? 1 : 0;
    }
};

// cur_cap / mp_cap: the matcher's capacities, lpre: its per-point scratch [nframes][mp_cap].  The values that come beside the ABI struct are
// __grid_constant__ like it: the kernel reads them from the parameter bank where it uses them instead of holding them in registers throughout.
__global__ void __launch_bounds__(kMatchThreads) match_localmap_kernel(const __grid_constant__ sgs_localmap_batch A, const __grid_constant__ int cur_cap,
                                                                       LocalPre* const __grid_constant__ lpre, const __grid_constant__ int mp_cap) {
    extern __shared__ __align__(16) uint8_t smem[];
    __shared__ int s_nmatch;
    const int f = blockIdx.x;
    const int n = min(A.cur_n[f], cur_cap);
    const int nmp = min(A.mp_n[f], mp_cap);
    FrameSmem s;
    carve(smem, cur_cap, s);
    const sgs_keypoint* kps = A.cur_kps + (int64_t)f * cur_cap;
    const uint4* cur_desc = reinterpret_cast<const uint4*>(A.cur_desc + (int64_t)f * cur_cap * 32);
    int32_t* f_mp = A.f_mp + (int64_t)f * cur_cap;
    uint8_t* f_obs = A.f_mp_obs + (int64_t)f * cur_cap;
    const int64_t lo = (int64_t)f * mp_cap;
    build_frame_grid(A.cam, kps, A.cur_uright + (int64_t)f * cur_cap, n, s);
    for (int i = threadIdx.x; i < n; i += blockDim.x) { s.claimed[i] = (f_mp[i] >= 0 && f_obs[i]) ? 1 : 0; s.tent[i] = 0; }
    __syncthreads();
    LocalPre* pre = lpre + lo;
    int ncand = 0;
    const int gl = threadIdx.x & (kGroup - 1);
    const int ngroups = blockDim.x / kGroup;
    for (int i0 = 0; i0 < nmp; i0 += ngroups) {
        const int i = i0 + threadIdx.x / kGroup;
        TopK t; topk_init(t);
        if (i < nmp && A.mp_inview[lo + i]) {
            LocalPolicy pol{A, s, cur_desc, f_mp, f_obs, lo, i};
            float rr; int lvl;
            pol.window(rr, lvl);
            const uint4* dm = reinterpret_cast<const uint4*>(A.mp_desc + 32 * (lo + i));
            t = scan_window(A.cam, s, cur_desc, A.proj_x[lo + i], A.proj_y[lo + i], rr, lvl - 1, lvl, __ldg(dm), __ldg(dm + 1), false,
                            A.proj_xr[lo + i], rr, &ncand, gl, kGroup);
        }
        t = group_topk(t);
        if (gl == 0 && i < nmp) {
            LocalPre pp;
#pragma unroll
            for (int c = 0; c < kTopK; ++c) pp.k[c] = t.k[c];
            pp.ngated = t.ngated;
            pre[i] = pp;
        }
    }
    __syncthreads();
    if (threadIdx.x < 32) {
        int nmatch = 0;
        for (int c0 = 0; c0 < nmp; c0 += 32) {
            const int i = c0 + threadIdx.x;
            LocalPolicy pol{A, s, cur_desc, f_mp, f_obs, lo, i};
            LocalPre pp;
            if (i < nmp) pp = pre[i];
            else { for (int c = 0; c < kTopK; ++c) pp.k[c] = kNoKey; pp.ngated = 0; }
            nmatch += resolve_chunk(s, pol, i < nmp, pp.k, pp.ngated);
        }
        if (threadIdx.x == 0) s_nmatch = nmatch;
    }
    __syncthreads();
    write_totals(ncand, s_nmatch, reinterpret_cast<unsigned long long*>(A.ncand) + f, &A.nmatches[f]);
}

// ---------------------------------------------------------------------------------------------------------------------
// Search half of ORBmatcher::Fuse(pKF, vpMapPoints, th) (src/ORBmatcher.cc:829-980, LocalMapping::SearchInNeighbors).  Every map point is
// independent (the reference's side effects -- Replace / AddObservation -- do not feed back into the search), so the block only shares
// the key frame's grid: kGroup lanes per map point scan its window, the best (distance, grid position) key is min-reduced over the
// group, which is the first minimum of the reference's loop over vIndices.
__global__ void __launch_bounds__(kMatchThreads) fuse_search_kernel(const __grid_constant__ sgs_fuse_batch A, const __grid_constant__ float log_sf) {
    extern __shared__ __align__(16) uint8_t smem[];
    FrameSmem s;
    carve(smem, A.kf_cap, s);
    const int f = blockIdx.x;
    const int n = min(A.kf_n[f], A.kf_cap), nmp = min(A.mp_n[f], A.mp_cap);
    const sgs_keypoint* kps = A.kf_kps + (int64_t)f * A.kf_cap;
    const uint4* kf_desc = reinterpret_cast<const uint4*>(A.kf_desc + (int64_t)f * A.kf_cap * 32);
    build_frame_grid(A.cam, kps, A.kf_uright + (int64_t)f * A.kf_cap, n, s);
    const float* T = A.tcw + 16 * (int64_t)f; const float* O = A.ow + 3 * (int64_t)f;
    const int64_t lo = (int64_t)f * A.mp_cap;
    const GridScale g = grid_scale(A.cam);
    const int gl = threadIdx.x & (kGroup - 1), ngroups = blockDim.x / kGroup;
    // variant 3 (SearchByProjection(KeyFrame*, Scw, vpPoints, vpMatched, th)): the reference visits the points in order and a feature claimed by an
    // earlier point is invisible to later ones.  A wave of ngroups points searches in parallel against the claims made so far; one thread then walks
    // the wave in order and accepts picks until it meets a pick that an earlier point of the same wave has just taken -- that point (and the ones
    // behind it) search again.  A pick that is still free after the earlier claims is the same pick the sequential loop would make.
    const bool claim = A.sim3_variant == 3;
    int32_t* matched = claim ? A.kf_matched + (int64_t)f * A.kf_cap : nullptr;
    __shared__ int s_pick[kMatchThreads / kGroup], s_pick_dist[kMatchThreads / kGroup], s_first, s_nm;
    if (threadIdx.x == 0) s_nm = 0;
    for (int i0 = 0; i0 < nmp; i0 += ngroups) {
      const int grp = threadIdx.x / kGroup, cnt = min(ngroups, nmp - i0);
      int first = 0;
      do {
        const int i = i0 + grp;
        uint32_t best = kNoKey;
        if (i < nmp && grp >= first && A.mp_valid[lo + i]) {
            const float* X = A.mp_xyz + 3 * (lo + i);
            float pc[3];
#pragma unroll
            for (int r = 0; r < 3; ++r) pc[r] = gemm3_row(T[4 * r], T[4 * r + 1], T[4 * r + 2], X, T[4 * r + 3]);   // Rcw * p3Dw + tcw
            if (A.sim3_variant == 2) {          // p3Dc2 = sR21 * p3Dc1 + t21
                const float* S = A.xform2 + 12 * (int64_t)f;
                float q[3];
#pragma unroll
                for (int r = 0; r < 3; ++r) q[r] = gemm3_row(S[3 * r], S[3 * r + 1], S[3 * r + 2], pc, S[9 + r]);
                pc[0] = q[0]; pc[1] = q[1]; pc[2] = q[2];
            }
            bool ok = !(pc[2] < 0.0f);
            const float invz = (A.sim3_variant == 1 || A.sim3_variant == 2) ? (float)__ddiv_rn(1.0, (double)pc[2]) : __fdiv_rn(1.f, pc[2]);
            const float u = __fadd_rn(__fmul_rn(A.cam.fx, __fmul_rn(pc[0], invz)), A.cam.cx), v = __fadd_rn(__fmul_rn(A.cam.fy, __fmul_rn(pc[1], invz)), A.cam.cy);
            ok = ok && (u >= A.cam.min_x && u < A.cam.max_x && v >= A.cam.min_y && v < A.cam.max_y);        // KeyFrame::IsInImage
            const float ur = __fsub_rn(u, __fmul_rn(A.cam.bf, invz));
            const float maxd = A.mp_max_dist[lo + i];
            const bool cam2 = A.sim3_variant == 2;
            const float px = cam2 ? pc[0] : __fsub_rn(X[0], O[0]), py = cam2 ? pc[1] : __fsub_rn(X[1], O[1]), pz = cam2 ? pc[2] : __fsub_rn(X[2], O[2]);
            const float dist = (float)sqrt(((double)px * px + (double)py * py) + (double)pz * pz);
            ok = ok && !(dist < __fmul_rn(0.8f, A.mp_min_dist[lo + i]) || dist > __fmul_rn(1.2f, maxd));
            const float* N = A.mp_normal + 3 * (lo + i);
            ok = ok && (cam2 || !((((double)px * N[0] + (double)py * N[1]) + (double)pz * N[2]) < 0.5 * (double)dist));
            if (ok) {
                const int lvl = predict_scale(maxd, dist, log_sf, A.cam.nlevels);
                const float r = __fmul_rn(A.th, A.cam.scale_factors[lvl]);
                int min_cx, max_cx, min_cy, max_cy;
                if (feature_window(A.cam, g, u, v, r, min_cx, max_cx, min_cy, max_cy)) {
                    const uint4* dm = reinterpret_cast<const uint4*>(A.mp_desc + 32 * (lo + i));
                    const uint4 d0 = __ldg(dm), d1 = __ldg(dm + 1);
                    for (int ix = min_cx; ix <= max_cx; ++ix) {
                        const int beg = s.cell_start[ix * kGridRows + min_cy], end = s.cell_start[ix * kGridRows + max_cy + 1];
                        for (int j = beg + gl; j < end; j += kGroup) {
                            const int idx = s.order[j];
                            const float ex = __fsub_rn(u, s.kx[idx]), ey = __fsub_rn(v, s.ky[idx]);
                            if (!(fabsf(ex) < r && fabsf(ey) < r)) continue;          // GetFeaturesInArea: |kp - (u, v)| < r (same value as distx = kp - x)
                            const int o = s.oct[idx];
                            if (o < lvl - 1 || o > lvl) continue;
                            if (claim && matched[idx] >= 0) continue;                  // if(vpMatched[idx]) continue;  (:374)
                            const float kr = s.ur[idx];
                            if (A.sim3_variant) {
                            } else if (kr >= 0.f) {
                                const float er = __fsub_rn(ur, kr);
                                const float e2 = __fadd_rn(__fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey)), __fmul_rn(er, er));
                                if ((double)__fmul_rn(e2, A.inv_level_sigma2[o]) > 7.8) continue;
                            } else {
                                const float e2 = __fadd_rn(__fmul_rn(ex, ex), __fmul_rn(ey, ey));
                                if ((double)__fmul_rn(e2, A.inv_level_sigma2[o]) > 5.99) continue;
                            }
                            const uint32_t k = ((uint32_t)descriptor_distance(d0, d1, __ldg(&kf_desc[2 * idx]), __ldg(&kf_desc[2 * idx + 1])) << 16) | (uint32_t)j;
                            best = min(best, k);
                        }
                    }
                }
            }
        }
#pragma unroll
        for (int o = kGroup >> 1; o > 0; o >>= 1) best = min(best, __shfl_xor_sync(0xffffffffu, best, o));
        if (!claim) {
            if (gl == 0 && i < nmp) {
                A.best_idx[lo + i] = best == kNoKey ? -1 : (int)s.order[best & 0xFFFFu];
                A.best_dist[lo + i] = best == kNoKey ? 256 : (int)(best >> 16);
            }
            break;
        }
        if (gl == 0 && grp >= first && grp < cnt) {
            s_pick[grp] = best == kNoKey ? -1 : (int)s.order[best & 0xFFFFu];
            s_pick_dist[grp] = best == kNoKey ? 256 : (int)(best >> 16);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int k = first;
            for (; k < cnt; ++k) {
                const int idx = s_pick[k], d = s_pick_dist[k];
                const bool take = idx >= 0 && d <= kThLow;                             // if(bestDist<=TH_LOW)  (:393)
                if (take && matched[idx] >= 0) break;                                  // taken by an earlier point of this wave: search again
                if (take) { matched[idx] = i0 + k; s_nm = s_nm + 1; }
                A.best_idx[lo + i0 + k] = take ? idx : -1;
                A.best_dist[lo + i0 + k] = d;
            }
            s_first = k;
        }
        __syncthreads();
        first = s_first;
      } while (first < cnt);
    }
    if (claim) {
        __syncthreads();
        if (threadIdx.x == 0 && A.nmatches) A.nmatches[f] = s_nm;
    }
}

// ORBmatcher::SearchForInitialization (src/ORBmatcher.cc:407-522), one block per (F1, F2) pair.  The reference loop is order dependent (a feature of
// F2 remembers the best distance that claimed it, a better later keypoint steals it), so the keypoints of F1 are visited one after the other; the
// block shares the candidate scan of each: every thread folds its candidates into (best key, second-best distance), the pairs are merged with the
// rule of the sequential update (strict <, first candidate in grid order wins ties), thread 0 applies :462-489.
struct BestTwo { uint32_t best; uint32_t second; };      // best = dist << 16 | position in the grid order (kNoKey = none); second = distance (0xFFFFFFFF = none)
__device__ __forceinline__ BestTwo merge_two(BestTwo a, BestTwo b) {
    BestTwo r;
    const uint32_t lo = min(a.best, b.best), hi = max(a.best, b.best);
    r.best = lo;
    r.second = min(min(a.second, b.second), hi == kNoKey ? 0xFFFFFFFFu : (hi >> 16));
    return r;
}

__global__ void __launch_bounds__(kMatchThreads) search_init_kernel(const __grid_constant__ sgs_init_batch A) {
    extern __shared__ __align__(16) uint8_t smem[];
    FrameSmem s;
    carve(smem, A.f2_cap, s);
    int32_t* mdist = reinterpret_cast<int32_t*>(smem + frame_smem_bytes(A.f2_cap));      // vMatchedDistance
    int32_t* m21 = mdist + A.f2_cap;                                                        // vnMatches21
    int8_t* bin_of = reinterpret_cast<int8_t*>(m21 + A.f2_cap);                             // rotation bin a keypoint of F1 was pushed to, or -1
    __shared__ int hist[kHistoLen];
    __shared__ BestTwo s_part[kMatchThreads / 32];
    __shared__ int s_nm;
    const int f = blockIdx.x, tid = threadIdx.x;
    const int n1 = min(A.f1_n[f], A.f1_cap), n2 = min(A.f2_n[f], A.f2_cap);
    const sgs_keypoint* k1 = A.f1_kps + (int64_t)f * A.f1_cap;
    const sgs_keypoint* k2 = A.f2_kps + (int64_t)f * A.f2_cap;
    const uint4* d1 = reinterpret_cast<const uint4*>(A.f1_desc + (int64_t)f * A.f1_cap * 32);
    const uint4* d2 = reinterpret_cast<const uint4*>(A.f2_desc + (int64_t)f * A.f2_cap * 32);
    float* prev = A.prev_xy + (int64_t)f * A.f1_cap * 2;
    int32_t* m12 = A.match12 + (int64_t)f * A.f1_cap;
    build_frame_grid(A.cam, k2, nullptr, n2, s);
    for (int i = tid; i < n2; i += kMatchThreads) { mdist[i] = 0x7fffffff; m21[i] = -1; }
    for (int i = tid; i < A.f1_cap; i += kMatchThreads) { bin_of[i] = -1; m12[i] = -1; }
    if (tid < kHistoLen) hist[tid] = 0;
    if (tid == 0) s_nm = 0;
    __syncthreads();
    const GridScale g = grid_scale(A.cam);
    const float r = (float)A.window_size;
    for (int i1 = 0; i1 < n1; ++i1) {
        if (k1[i1].octave > 0) continue;                                                    // level1 > 0 (:424-426), block-uniform
        const float x = prev[2 * i1], y = prev[2 * i1 + 1];
        int min_cx, max_cx, min_cy, max_cy;                                                 // GetFeaturesInArea(x, y, windowSize, 0, 0)
        if (!feature_window(A.cam, g, x, y, r, min_cx, max_cx, min_cy, max_cy)) continue;
        const uint4 a0 = __ldg(&d1[2 * i1]), a1 = __ldg(&d1[2 * i1 + 1]);
        BestTwo t;
        t.best = kNoKey; t.second = 0xFFFFFFFFu;
        for (int ix = min_cx; ix <= max_cx; ++ix) {
            const int beg = s.cell_start[ix * kGridRows + min_cy], end = s.cell_start[ix * kGridRows + max_cy + 1];
            for (int j = beg + tid; j < end; j += kMatchThreads) {
                const int idx = s.order[j];
                if (s.oct[idx] > 0) continue;                                               // maxLevel = 0
                if (!(fabsf(__fsub_rn(s.kx[idx], x)) < r && fabsf(__fsub_rn(s.ky[idx], y)) < r)) continue;
                const uint32_t d = (uint32_t)descriptor_distance(a0, a1, __ldg(&d2[2 * idx]), __ldg(&d2[2 * idx + 1]));
                if (mdist[idx] <= (int)d) continue;                                         // if(vMatchedDistance[i2]<=dist) continue;  (:447)
                const uint32_t key = (d << 16) | (uint32_t)j;
                if (key < t.best) { if (t.best != kNoKey) t.second = min(t.second, t.best >> 16); t.best = key; }
                else t.second = min(t.second, d);
            }
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            BestTwo u;
            u.best = __shfl_xor_sync(0xffffffffu, t.best, o); u.second = __shfl_xor_sync(0xffffffffu, t.second, o);
            t = merge_two(t, u);
        }
        if ((tid & 31) == 0) s_part[tid >> 5] = t;
        __syncthreads();
        if (tid == 0) {
            BestTwo b = s_part[0];
            for (int w = 1; w < kMatchThreads / 32; ++w) b = merge_two(b, s_part[w]);
            if (b.best != kNoKey) {
                const int best_d = (int)(b.best >> 16), idx2 = s.order[b.best & 0xFFFFu];
                const float second_f = b.second == 0xFFFFFFFFu ? 2147483648.f : (float)(int)b.second;     // (float)INT_MAX
                if (best_d <= kThLow && (float)best_d < __fmul_rn(second_f, A.nnratio)) {
                    if (m21[idx2] >= 0) { m12[m21[idx2]] = -1; s_nm = s_nm - 1; }
                    m12[i1] = idx2; m21[idx2] = i1; mdist[idx2] = best_d; s_nm = s_nm + 1;
                    if (A.check_orientation) {
                        const int bin = rotation_bin(k1[i1].angle, k2[idx2].angle);
                        hist[bin] = hist[bin] + 1; bin_of[i1] = (int8_t)bin;
                    }
                }
            }
        }
        __syncthreads();
    }
    if (A.check_orientation) {
        __shared__ int keep[3];
        if (tid == 0) three_maxima(hist, keep[0], keep[1], keep[2]);
        __syncthreads();
        int removed = 0;
        for (int i = tid; i < n1; i += kMatchThreads) {
            const int b = bin_of[i];
            if (b >= 0 && b != keep[0] && b != keep[1] && b != keep[2] && m12[i] >= 0) { m12[i] = -1; ++removed; }
        }
        if (removed) atomicSub(&s_nm, removed);
        __syncthreads();
    }
    for (int i = tid; i < n1; i += kMatchThreads)
        if (m12[i] >= 0) { prev[2 * i] = s.kx[m12[i]]; prev[2 * i + 1] = s.ky[m12[i]]; }     // :517-519
    if (tid == 0 && A.nmatches) A.nmatches[f] = s_nm;
}

// One block of kMatchThreads per frame.  The frame grid keeps keypoint indices in 16 bits, so no capacity may exceed 65535, and `smem` bytes
// of dynamic shared memory hold it (plus the kernel's own per-keypoint arrays).
template <class... Params, class... Args>
static int launch_per_frame(void (*kernel)(Params...), size_t smem, int cap, int nframes, cudaStream_t st, const Args&... args) {
    if (smem > 200 * 1024 || cap > 65535) { set_error("matcher: capacity %d too large for shared memory", cap); return SGS_ERR_UNSUPPORTED; }
    SGS_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<nframes, kMatchThreads, smem, st>>>(args...);
    SGS_CUDA_TRY(cudaGetLastError());
    return SGS_OK;
}

int launch_matcher(const LastFrameArgs& A, int nframes, cudaStream_t st) {
    return launch_per_frame(match_lastframe_kernel, frame_smem_bytes(A.cur_cap), A.cur_cap, nframes, st, A);
}
int launch_matcher(const sgs_localmap_batch& A, int cur_cap, LocalPre* pre, int mp_cap, int nframes, cudaStream_t st) {
    return launch_per_frame(match_localmap_kernel, frame_smem_bytes(cur_cap), cur_cap, nframes, st, A, cur_cap, pre, mp_cap);
}
int launch_matcher(const sgs_fuse_batch& A, float log_sf, int nframes, cudaStream_t st) {
    return launch_per_frame(fuse_search_kernel, frame_smem_bytes(A.kf_cap), A.kf_cap, nframes, st, A, log_sf);
}
int launch_matcher(const sgs_init_batch& A, int nframes, cudaStream_t st) {     // + vMatchedDistance, vnMatches21 and the rotation bins of F1
    const size_t smem = frame_smem_bytes(A.f2_cap) + (size_t)A.f2_cap * 8 + (size_t)((A.f1_cap + 15) & ~15);
    return launch_per_frame(search_init_kernel, smem, max(A.f1_cap, A.f2_cap), nframes, st, A);
}

}  // namespace sgs
