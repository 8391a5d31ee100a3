// quadtree_core.h -- deterministic, data-parallel restatement of ORBextractor::DistributeOctTree
// (src/ORBextractor.cc:540-764) + ExtractorNode::DivideNode (:482-538).
//
// GPU-first formulation (not a translation of the std::list/pointer code):
//   * every split position of the reference's quadtree is a pure function of the root rectangle
//     (halfX = ceil(w/2)), so each candidate's path (2 bits per depth) is computed independently;
//   * candidates are sorted once by (root, path): every node of every depth is then a contiguous
//     range [lo,hi) of the sorted array, and "DivideNode" is three binary searches;
//   * the std::list order (push_front of children, erase of parents) is reproduced by rebuilding
//     an index array per pass:  new = children of the processed nodes in reverse processing order
//     (n4..n1 inside a group) followed by the untouched nodes in their old order;
//   * the (size, pointer) stable_sort tie-break is defined as node creation sequence (quirk Q1).
//
// The same code runs inside one CUDA block (Ctx = CudaCtx) and, for CPU-side verification of the
// logic, single-threaded on the host (Ctx = HostCtx; tests/test_quadtree_host.py).  Code between two
// ctx.sync() calls is written as independent strided loops, so any thread count gives the same result.
#pragma once
#include <cstdint>

#include "sgs_common.h"

namespace sgs {

struct QtGeom {
    int32_t n_ini;      // number of root strips
    float h_x;          // strip width (float, as in the reference)
    int32_t root_h;     // maxBorderY - minBorderY
    int32_t n_cols, w_cell, h_cell;  // FAST cell grid: defines the reference's candidate order (tie-break of equal responses)
    int32_t n_target;   // N
};

// candidate word: x (12 bits) | y (12 bits) << 12 | score << 24, coordinates relative to (minBorderX, minBorderY)
SGS_HD uint32_t qt_pack(int x, int y, int score) { return (uint32_t)x | ((uint32_t)y << 12) | ((uint32_t)score << 24); }
SGS_HD int qt_x(uint32_t c) { return (int)(c & 0xFFFu); }
SGS_HD int qt_y(uint32_t c) { return (int)((c >> 12) & 0xFFFu); }
SGS_HD int qt_score(uint32_t c) { return (int)(c >> 24); }

// (root << 24) | 12 x 2-bit child codes, most significant = first division.  Child code: bit0 = right, bit1 = bottom
// (n1=0, n2=1, n3=2, n4=3 of DivideNode).
SGS_HD uint32_t qt_path_key(int x, int y, const QtGeom& g) {
    int r = (int)((float)x / g.h_x);                      // vpIniNodes[kp.pt.x/hX]  (:571)
    if (r > g.n_ini - 1) r = g.n_ini - 1;
    int ulx = (int)(g.h_x * (float)r), urx = (int)(g.h_x * (float)(r + 1));  // :555-556
    int uly = 0, bry = g.root_h;
    uint32_t path = 0;
#pragma unroll
    for (int d = 0; d < kQtDepth; ++d) {
        const int mx = ulx + ((urx - ulx + 1) >> 1);      // UL.x + ceil((UR.x-UL.x)/2)  (:484)
        const int my = uly + ((bry - uly + 1) >> 1);
        const uint32_t bx = (x < mx) ? 0u : 1u;           // kp.pt.x < n1.UR.x  (:516)
        const uint32_t by = (y < my) ? 0u : 1u;
        path = (path << 2) | (by << 1) | bx;
        if (bx) ulx = mx; else urx = mx;
        if (by) uly = my; else bry = my;
    }
    return ((uint32_t)r << 24) | path;
}

// position of a candidate in the reference's vToDistributeKeys order: cells row-major, pixels row-major inside a cell
// (:790-826).  Smaller = earlier.  Interior of cell (i,j) starts at relative coordinate 3 + j*w_cell.
SGS_HD uint64_t qt_order_key(uint32_t c, const QtGeom& g) {
    const int x = qt_x(c), y = qt_y(c);
    const int j = (x - 3) / g.w_cell, i = (y - 3) / g.h_cell;
    return ((uint64_t)i << 32) | ((uint64_t)j << 24) | ((uint64_t)y << 12) | (uint64_t)x;
}

struct QtWork {
    // sorted keys: (path_key << 32) | candidate word; n_sort = power of two >= n, padded with ~0
    uint64_t* keys;
    int n, n_sort;
    // node pool (structure of arrays), capacity pool_cap
    int32_t* lo; int32_t* hi; int32_t* seq; uint8_t* depth; uint8_t* flag;  // flag: 1 = processed in this pass
    int32_t* free_list; int pool_cap;
    // list order ping-pong, expansion set, child boundaries, child ids
    int32_t* list_a; int32_t* list_b;
    int32_t* exp_a; int32_t* exp_b;       // expansion candidates (node ids): current / next
    uint64_t* exp_key;                    // sort keys of the fine phase
    int32_t* bnd;                         // [cap][3] child boundaries of exp_a entries
    int32_t* child;                       // [cap][4] child node ids (-1 = empty child)
    // scalars shared between threads (live in shared memory on the device)
    int32_t* sc;                          // [16] scratch scalars
};

enum { QS_LEN = 0, QS_NEXP, QS_NFREE, QS_SEQ, QS_FINISH, QS_FINE, QS_NOUT, QS_NNEXT, QS_PREV, QS_NTOEXP };

// number of int32-equivalents needed for the node-side arrays given the node capacity
SGS_HD int qt_pool_cap(int n_target, int n_ini) { return 2 * (n_target > 4 * n_ini ? n_target : 4 * n_ini) + 4 * n_ini + 16; }

// Bitonic sort of n_sort (a power of two) unique keys.  Stages with a partner distance j > 32 run across the whole block (one barrier each);
// the remaining stages of every merge only touch aligned chunks of 64 keys, which one group of threads (a warp on the device, the single
// host thread in the check build) finishes chunk by chunk with its own cheap synchronisation.  The keys are unique, so the result does not
// depend on how the network is scheduled.
template <class Ctx>
SGS_HD void qt_bitonic_sort(Ctx& ctx, uint64_t* a, int n_sort) {
    const int W = ctx.group();
    const int ngroups = ctx.nthreads() / W, gid = ctx.tid() / W, gl = ctx.tid() % W;
    const int chunk = n_sort < 64 ? n_sort : 64;
    for (int k = 2; k <= n_sort; k <<= 1) {
        int j = k >> 1;
        for (; j > 32; j >>= 1) {
            for (int t = ctx.tid(); t < (n_sort >> 1); t += ctx.nthreads()) {
                // t-th compare-exchange of this stage
                const int i = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                const int p = i | j;
                const bool up = ((i & k) == 0);
                const uint64_t x = a[i], y = a[p];
                if ((x > y) == up) { a[i] = y; a[p] = x; }
            }
            ctx.sync();
        }
        for (int base = gid * chunk; base < n_sort; base += ngroups * chunk) {
            for (int jj = j; jj > 0; jj >>= 1) {
                for (int t = gl; t < (chunk >> 1); t += W) {
                    const int i = base + (((t & ~(jj - 1)) << 1) | (t & (jj - 1)));
                    const int p = i | jj;
                    const bool up = ((i & k) == 0);
                    const uint64_t x = a[i], y = a[p];
                    if ((x > y) == up) { a[i] = y; a[p] = x; }
                }
                ctx.group_sync();
            }
        }
        ctx.sync();
    }
}

// first index in [lo,hi) whose child code at `depth` is >= code
SGS_HD int qt_lower_bound(const uint64_t* keys, int lo, int hi, int depth, uint32_t code) {
    const int sh = 32 + 2 * (kQtDepth - 1 - depth);
    while (lo < hi) {
        const int mid = (lo + hi) >> 1;
        const uint32_t c = (uint32_t)(keys[mid] >> sh) & 3u;
        if (c < code) lo = mid + 1; else hi = mid;
    }
    return lo;
}

// Runs the whole distribution for one (frame, level).  `cands` holds n packed candidates (any order).  Writes the selected
// candidates (packed words) to out[] in the reference's output order and returns their number through *n_out.
// All QtWork arrays must be sized by the caller: keys[n_sort], node arrays[pool_cap], lists[pool_cap], bnd[3*pool_cap],
// child[4*pool_cap].
template <class Ctx>
SGS_HD void qt_distribute(Ctx& ctx, const uint32_t* cands, const QtGeom& g, QtWork& w, uint32_t* out, int out_cap, int32_t* n_out) {
    const int n = w.n;
    const int N = g.n_target;
    if (n == 0) {
        if (ctx.tid() == 0) *n_out = 0;
        ctx.sync();
        return;
    }
    // 1. path keys + sort
    for (int i = ctx.tid(); i < w.n_sort; i += ctx.nthreads()) {
        uint64_t k = ~0ull;
        if (i < n) {
            const uint32_t c = cands[i];
            k = ((uint64_t)qt_path_key(qt_x(c), qt_y(c), g) << 32) | c;
        }
        w.keys[i] = k;
    }
    ctx.sync();
    qt_bitonic_sort(ctx, w.keys, w.n_sort);
    // 2. roots (:549-586): non-empty strips in x order; depth 0
    if (ctx.tid() == 0) {
        int len = 0, pos = 0, seq = 0;
        for (int r = 0; r < g.n_ini; ++r) {
            int lo = pos;
            // end of this root's range: first key with root > r
            int a = pos, b = n;
            while (a < b) { const int mid = (a + b) >> 1; if ((int)(w.keys[mid] >> 56) <= r) a = mid + 1; else b = mid; }
            pos = a;
            const int id = r;
            w.lo[id] = lo; w.hi[id] = pos; w.depth[id] = 0; w.seq[id] = seq++; w.flag[id] = 0;
            if (pos > lo) w.list_a[len++] = id;
        }
        int nfree = 0;
        for (int id = w.pool_cap - 1; id >= g.n_ini; --id) w.free_list[nfree++] = id;
        // empty roots are simply never referenced again
        w.sc[QS_LEN] = len; w.sc[QS_NFREE] = nfree; w.sc[QS_SEQ] = seq;
        w.sc[QS_FINISH] = 0; w.sc[QS_FINE] = 0; w.sc[QS_NNEXT] = 0;
    }
    ctx.sync();
    int32_t* list_cur = w.list_a;
    int32_t* list_new = w.list_b;
    int32_t* exp_cur = w.exp_a;
    int32_t* exp_next = w.exp_b;
    // 3. passes
    for (;;) {
        if (w.sc[QS_FINISH]) break;
        const int len = w.sc[QS_LEN];
        const bool fine = w.sc[QS_FINE] != 0;
        // 3a. processing order
        if (!fine) {
            // coarse pass (:601-666): every node with more than one point, in list order
            if (ctx.tid() == 0) {
                int ne = 0;
                for (int i = 0; i < len; ++i) { const int id = list_cur[i]; if (w.hi[id] - w.lo[id] > 1) exp_cur[ne++] = id; }
                w.sc[QS_NEXP] = ne;
            }
            ctx.sync();
        } else {
            // fine pass (:676-739): nodes recorded by the previous pass sorted by (size, creation seq), processed largest first
            const int ne = w.sc[QS_NNEXT];
            for (int i = ctx.tid(); i < ne; i += ctx.nthreads()) {
                const int id = exp_next[i];
                w.exp_key[i] = ((uint64_t)(uint32_t)(w.hi[id] - w.lo[id]) << 32) | (uint32_t)w.seq[id];
            }
            ctx.sync();
            for (int i = ctx.tid(); i < ne; i += ctx.nthreads()) {
                const uint64_t k = w.exp_key[i];
                int rank = 0;
                for (int j = 0; j < ne; ++j) rank += (w.exp_key[j] > k) ? 1 : 0;  // keys are unique (seq)
                exp_cur[rank] = exp_next[i];
            }
            if (ctx.tid() == 0) w.sc[QS_NEXP] = ne;
            ctx.sync();
        }
        const int ne = w.sc[QS_NEXP];
        // 3b. child boundaries of every node that may be divided in this pass (independent => parallel)
        for (int e = ctx.tid(); e < ne; e += ctx.nthreads()) {
            const int id = exp_cur[e];
            const int lo = w.lo[id], hi = w.hi[id], d = w.depth[id];
            const int b1 = qt_lower_bound(w.keys, lo, hi, d, 1u);
            const int b2 = qt_lower_bound(w.keys, b1, hi, d, 2u);
            const int b3 = qt_lower_bound(w.keys, b2, hi, d, 3u);
            w.bnd[3 * e + 0] = b1; w.bnd[3 * e + 1] = b2; w.bnd[3 * e + 2] = b3;
        }
        ctx.sync();
        // 3c. apply in processing order (serial: it is the reference's sequential list surgery, <= N steps)
        if (ctx.tid() == 0) {
            int size = len, nfree = w.sc[QS_NFREE], seq = w.sc[QS_SEQ];
            int processed = 0, nnext = 0, n_to_expand = 0;
            for (int e = 0; e < ne; ++e) {
                const int id = exp_cur[e];
                const int lo = w.lo[id], hi = w.hi[id], d = w.depth[id];
                const int b[5] = {lo, w.bnd[3 * e], w.bnd[3 * e + 1], w.bnd[3 * e + 2], hi};
                int nchild = 0;
                for (int q = 0; q < 4; ++q) {
                    int cid = -1;
                    if (b[q + 1] > b[q]) {
                        cid = w.free_list[--nfree];
                        w.lo[cid] = b[q]; w.hi[cid] = b[q + 1]; w.depth[cid] = (uint8_t)(d + 1); w.seq[cid] = seq++; w.flag[cid] = 0;
                        ++nchild;
                        if (b[q + 1] - b[q] > 1) { exp_next[nnext++] = cid; ++n_to_expand; }
                    }
                    w.child[4 * e + q] = cid;
                }
                w.flag[id] = 1;
                size += nchild - 1;
                ++processed;
                if (fine && size >= N) break;  // :731-732
            }
            // new list = children groups in reverse processing order (n4..n1 inside a group) + untouched nodes in old order
            int pos = 0;
            for (int e = processed - 1; e >= 0; --e)
                for (int q = 3; q >= 0; --q) { const int cid = w.child[4 * e + q]; if (cid >= 0) list_new[pos++] = cid; }
            for (int i = 0; i < len; ++i) { const int id = list_cur[i]; if (!w.flag[id]) list_new[pos++] = id; }
            for (int e = 0; e < processed; ++e) { const int id = exp_cur[e]; w.flag[id] = 0; w.free_list[nfree++] = id; }
            // bookkeeping of the reference's loop conditions
            int finish = 0, go_fine = fine ? 1 : 0;
            if (size >= N || size == len) finish = 1;                 // :670-673 / :735-736
            else if (!fine && (size + n_to_expand * 3) > N) go_fine = 1;  // :674
            w.sc[QS_LEN] = pos; w.sc[QS_NFREE] = nfree; w.sc[QS_SEQ] = seq;
            w.sc[QS_NNEXT] = nnext; w.sc[QS_FINISH] = finish; w.sc[QS_FINE] = go_fine;
        }
        ctx.sync();
        { int32_t* t = list_cur; list_cur = list_new; list_new = t; }
    }
    // 4. best response per node, first candidate (reference order) wins ties (:742-763)
    const int len = w.sc[QS_LEN];
    for (int i = ctx.tid(); i < len; i += ctx.nthreads()) {
        const int id = list_cur[i];
        uint64_t best = 0; uint32_t best_c = 0;
        for (int k = w.lo[id]; k < w.hi[id]; ++k) {
            const uint32_t c = (uint32_t)w.keys[k];
            const uint64_t score = ((uint64_t)qt_score(c) << 44) | ((~qt_order_key(c, g)) & ((1ull << 44) - 1));
            if (score > best || k == w.lo[id]) { best = score; best_c = c; }
        }
        if (i < out_cap) out[i] = best_c;
    }
    if (ctx.tid() == 0) *n_out = len;
    ctx.sync();
}

}  // namespace sgs
