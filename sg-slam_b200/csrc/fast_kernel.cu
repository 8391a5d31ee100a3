// fast_kernel.cu -- FAST-9-16 + cell-local 3x3 NMS + per-cell threshold fallback (ComputeKeyPointsOctTree, FAST part,
// src/ORBextractor.cc:766-830; cv::FAST semantics pinned in tests/test_oracle_golden.py).
//
// Design: ONE WARP PER CELL (a cell == one cv::FAST call of the reference), 8 independent warps per block, no block
// barriers.  Each warp
//   0. pulls its cell view (+3 px ring halo) into its private shared-memory tile with ONE TMA tensor copy
//      (cp.async.bulk.tensor.3d, per-level tensor map {x, y, frame}) completing on a per-warp mbarrier -- or with plain loads
//      when a level is not TMA-addressable.  The innermost TMA coordinate must be 16-byte aligned (an unaligned x
//      raises "illegal instruction"), so the box starts at xa = (x0-4) & ~15 and the view sits `off` = x0 - xa
//      (4..19) columns into the tile; the packed phase works on smem-aligned words and masks the partial first/last word;
//   A. compass pre-test on 4 pixels per instruction: VABSDIFF4.U8 against the 4 compass ring pixels (0,4,8,12), a carry-free
//      packed "> t" test, and "at least two of four" in three LOP3s (any 9-arc contains >= 2 compass pixels);
//   B. survivors: scalar sign-aware compass re-check, full 16-pixel segment test at the lower threshold, exact score with the
//      packed-16-bit sliding minimum (VIMNMX.S16x2) -> score map;
//   C. NMS against the 8 neighbours in the (cell-local) score map, choice between iniTh and minTh, emission of packed
//      candidates through one global atomic per cell.
// Facts used:  score(p) >= t  <=>  p is a corner at threshold t;  the NMS predicate is threshold independent (neighbours below the
// threshold are below score(p) anyway);  the candidate order inside a level is irrelevant (the quadtree sorts).
#include <cuda.h>
#include <cuda_runtime.h>

#include "extract_dev.cuh"
#include "extract_kernels.h"

namespace sgs {

constexpr int kFastWarps = 8;

struct FastTileGeom {
    int32_t tp, th;          // tile pitch (bytes, multiple of 16) and rows
    int32_t list_cap;        // entries of the per-warp position list
    int32_t warp_stride;     // bytes of shared memory per warp (multiple of 128)
    int32_t use_tma;
    int32_t frame0;          // frame index of P's frame 0 inside the tensor maps (chunked calls shift P's pointers, the maps stay whole)
};

// ---- exact FAST score -------------------------------------------------------------------------------------------------------
// max over the 16 contiguous 9-arcs of max(min d, -max d) - 1 with d_k = v - r_k, evaluated for d and -d at once in packed 16-bit
// lanes biased by +256 (lo = v - r_k + 256, hi = r_k - v + 256, both in [1,511]): one IMAD builds a lane pair
// (r_k * 0xFFFF + C), then a sliding minimum over windows of 2, 4, 8, 9 ring positions with VIMNMX.U16x2.
// (A plain 32-bit `max(best, max(mn9, -mx9))` formulation is MISCOMPILED by CUDA 12.9 ptxas -O3 for sm_100a -- the negation is
//  folded into a 3-input VIMNMX3 incorrectly; tools/ptxas_minmax_repro.cu reproduces it.  This form never negates a max result.)
__device__ __forceinline__ int fast_score16(int v, const int (&r)[16]) {
    const unsigned C = (unsigned)(v + 256) + ((unsigned)(256 - v) << 16);
    unsigned p[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) p[k] = (unsigned)r[k] * 0xFFFFu + C;
    unsigned w2[16], w4[16], w8[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) w2[k] = __vminu2(p[k], p[(k + 1) & 15]);
#pragma unroll
    for (int k = 0; k < 16; ++k) w4[k] = __vminu2(w2[k], w2[(k + 2) & 15]);
#pragma unroll
    for (int k = 0; k < 16; ++k) w8[k] = __vminu2(w4[k], w4[(k + 4) & 15]);
    unsigned best = 0;
#pragma unroll
    for (int k = 0; k < 16; ++k) best = __vmaxu2(best, __vminu2(w8[k], p[(k + 8) & 15]));
    const int lo = (int)(best & 0xFFFFu), hi = (int)(best >> 16);
    return (lo > hi ? lo : hi) - 257;
}

// bytes of `ad` strictly greater than t (0 <= t <= 126) -> 0x80 in that byte, carry-free
__device__ __forceinline__ uint32_t gt_flags(uint32_t ad, uint32_t k127_minus_t) {
    return (((ad & 0x7f7f7f7fu) + k127_minus_t) | ad) & 0x80808080u;
}

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

template <bool kTma>
__global__ void __launch_bounds__(kFastWarps * 32) fast_warp_cells_kernel(const __grid_constant__ DevPlan P, const __grid_constant__ FastTmaMaps M,
                                                                          const FastCell* __restrict__ cells, int ncells, int nitems,
                                                                          const FastTileGeom G) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int item = blockIdx.x * kFastWarps + warp;
    if (item >= nitems) return;                       // whole warp exits together; no block barriers below
    const int f = item / ncells;
    const FastCell c = cells[item - f * ncells];
    const DevLevel& L = P.lv[c.level];
    const int TP = G.tp;
    uint8_t* tile = smem + (size_t)warp * G.warp_stride;
    uint8_t* score = tile + TP * G.th;                // (th + 2) rows: row r of the view lives at score row r + 1
    uint16_t* list = reinterpret_cast<uint16_t*>(score + TP * (G.th + 2));
    uint64_t* mbar = reinterpret_cast<uint64_t*>(tile + G.warp_stride - 16);
    const int w = c.x1 - c.x0, h = c.y1 - c.y0;       // view size
    const int xa = ((int)c.x0 - 4) & ~15;             // 16-byte aligned box origin (TMA requirement)
    const int off = (int)c.x0 - xa;                   // tile column of view column 0 (4..19)
    const int iw = w - 6, ih = h - 6;                 // interior: tile columns [off+3, off+3+iw), rows [3, 3+ih)

    // ---- 0. tile load ------------------------------------------------------------------------------------------------------
    if (kTma) {
        if (lane == 0) {
            const uint32_t mb = smem_u32(mbar);
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mb));
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mb), "r"((uint32_t)(TP * G.th)) : "memory");
            asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
                         ::"r"(smem_u32(tile)), "l"(reinterpret_cast<uint64_t>(&M.m[c.level])), "r"(xa), "r"((int)c.y0), "r"(f + G.frame0), "r"(mb)
                         : "memory");
        }
    } else {
        const uint8_t* img = L.img + (int64_t)f * L.fstride + (int64_t)c.y0 * L.pitch + c.x0;
        for (int y = 0; y < h; ++y)
            for (int x = lane; x < w; x += 32) tile[y * TP + off + x] = __ldg(img + (int64_t)y * L.pitch + x);
    }
    // zero the score map while the copy is in flight
    {
        uint4* s4 = reinterpret_cast<uint4*>(score);
        const int n4 = TP * (G.th + 2) / 16;
        for (int i = lane; i < n4; i += 32) s4[i] = make_uint4(0, 0, 0, 0);
    }
    if (kTma) {
        const uint32_t mb = smem_u32(mbar);
        uint32_t done = 0;
        while (!done) {
            asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(mb) : "memory");
        }
    }
    __syncwarp();

    // ---- detection at one threshold: returns the number of NMS survivors, their tile positions are list[0..n) ----------------
    // The reference runs cv::FAST at iniTh and, only when that leaves the cell empty, again at minTh (:810-817).  Scores do not
    // depend on the threshold, and a neighbour that is not a corner at the current threshold counts as 0 in the NMS, so each pass
    // only needs the corners of ITS threshold: the (rare) second pass simply redoes the cell at the lower threshold.
    const int ix0 = off + 3, ix1 = off + 3 + iw;       // interior tile columns [ix0, ix1)
    const int a0 = ix0 & ~3;                            // first smem-aligned word touching the interior
    const int nw = (ix1 - a0 + 3) >> 2;                 // aligned 4-pixel words per interior row (<= 16)
    const uint32_t inv_nw = (65536u + nw - 1) / nw;     // row = item / nw by multiply-shift (exact for item < 4096)
    auto detect = [&](const int t) -> int {
        // A. packed compass pre-test (sign-agnostic superset)
        const uint32_t kk = (uint32_t)(127 - (t < 126 ? t : 126)) * 0x01010101u;
        int nlist = 0;                                  // warp-uniform
        for (int i0 = 0; i0 < ih * nw; i0 += 32) {
            const int it = i0 + lane;
            const int row = (int)(((uint32_t)it * inv_nw) >> 16), col = it - row * nw;
            uint32_t flags = 0;
            int pos = 0;
            if (it < ih * nw) {
                pos = (row + 3) * TP + a0 + 4 * col;
                const uint32_t* rp = reinterpret_cast<const uint32_t*>(tile + pos);
                const uint32_t cc = rp[0], ll = rp[-1], rr = rp[1];
                const uint32_t up = *reinterpret_cast<const uint32_t*>(tile + pos - 3 * TP);
                const uint32_t dn = *reinterpret_cast<const uint32_t*>(tile + pos + 3 * TP);
                const uint32_t p4 = __byte_perm(cc, rr, 0x6543), p12 = __byte_perm(ll, cc, 0x4321);
                const uint32_t f0 = gt_flags(__vabsdiffu4(dn, cc), kk), f8 = gt_flags(__vabsdiffu4(up, cc), kk);
                const uint32_t f4 = gt_flags(__vabsdiffu4(p4, cc), kk), f12 = gt_flags(__vabsdiffu4(p12, cc), kk);
                flags = (f0 & f4) | (f8 & f12) | ((f0 | f4) & (f8 | f12));
                const int x = a0 + 4 * col;
                const int lead = ix0 - x;               // bytes of this word left of the interior
                const int over = x + 4 - ix1;           // bytes right of the interior
                if (lead > 0) flags &= 0x80808080u << (8 * lead);
                if (over > 0) flags &= 0x80808080u >> (8 * over);
            }
            const unsigned any = __ballot_sync(0xffffffffu, flags != 0);
            if (any) {
                const int cnt = __popc(flags);
                int incl = cnt;                         // inclusive warp scan of the per-lane survivor counts
#pragma unroll
                for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
                int dst = nlist + incl - cnt;
                uint32_t fl = flags;
                while (fl) {
                    const int b = (__ffs(fl) - 1) >> 3; // byte index 0..3
                    fl &= fl - 1;
                    list[dst++] = (uint16_t)(pos + b);
                }
                nlist += __shfl_sync(0xffffffffu, incl, 31);
            }
        }
        __syncwarp();
        // B1. scalar sign-aware compass re-check, survivors compacted in place
        int nb1 = 0;
        for (int i0 = 0; i0 < nlist; i0 += 32) {
            const int i = i0 + lane;
            bool pass = false;
            int pos = 0;
            if (i < nlist) {
                pos = list[i];
                const uint8_t* p = tile + pos;
                const int v = p[0];
                const int hi = v + t, lo = v - t;
                const int r0 = p[3 * TP], r4 = p[3], r8 = p[-3 * TP], r12 = p[-3];
                const int nb = (r0 > hi) + (r4 > hi) + (r8 > hi) + (r12 > hi);
                const int nd = (r0 < lo) + (r4 < lo) + (r8 < lo) + (r12 < lo);
                pass = (nb >= 2) | (nd >= 2);
            }
            const unsigned m = __ballot_sync(0xffffffffu, pass);
            __syncwarp();                               // reads of list[i0..i0+31] precede the in-place writes
            if (pass) list[nb1 + __popc(m & ((1u << lane) - 1))] = (uint16_t)pos;
            nb1 += __popc(m);
        }
        __syncwarp();
        // B2. exact score; p is a corner at t  <=>  score >= t; corners compacted in place
        int ncorner = 0;
        for (int i0 = 0; i0 < nb1; i0 += 32) {
            const int i = i0 + lane;
            bool corner = false;
            int pos = 0;
            if (i < nb1) {
                pos = list[i];
                const uint8_t* p = tile + pos;
                int r[16];
                r[0] = p[3 * TP]; r[1] = p[3 * TP + 1]; r[2] = p[2 * TP + 2]; r[3] = p[TP + 3]; r[4] = p[3]; r[5] = p[-TP + 3];
                r[6] = p[-2 * TP + 2]; r[7] = p[-3 * TP + 1]; r[8] = p[-3 * TP]; r[9] = p[-3 * TP - 1]; r[10] = p[-2 * TP - 2];
                r[11] = p[-TP - 3]; r[12] = p[-3]; r[13] = p[TP - 3]; r[14] = p[2 * TP - 2]; r[15] = p[3 * TP - 1];
                const int sc = fast_score16(p[0], r);
                corner = sc >= t;
                if (corner) score[pos + TP] = (uint8_t)sc;
            }
            const unsigned m = __ballot_sync(0xffffffffu, corner);
            __syncwarp();
            if (corner) list[ncorner + __popc(m & ((1u << lane) - 1))] = (uint16_t)pos;
            ncorner += __popc(m);
        }
        __syncwarp();
        // C. NMS against the 8 neighbours (cell-local: the score map is zero outside the interior)
        int nkept = 0;
        for (int i0 = 0; i0 < ncorner; i0 += 32) {
            const int i = i0 + lane;
            bool keep = false;
            int pos = 0;
            if (i < ncorner) {
                pos = list[i];
                const uint8_t* q = score + pos + TP;
                const int sc = q[0];
                keep = sc > q[-1] && sc > q[1] && sc > q[-TP - 1] && sc > q[-TP] && sc > q[-TP + 1] && sc > q[TP - 1] && sc > q[TP] && sc > q[TP + 1];
            }
            const unsigned m = __ballot_sync(0xffffffffu, keep);
            __syncwarp();
            if (keep) list[nkept + __popc(m & ((1u << lane) - 1))] = (uint16_t)pos;
            nkept += __popc(m);
        }
        __syncwarp();
        return nkept;
    };
    int nkept = detect(P.ini_th);
    if (nkept == 0) nkept = detect(P.min_th);
    const int total = nkept;
    if (total == 0) return;
    int base = 0;
    if (lane == 0) base = atomicAdd(&P.cand_count[f * P.nlevels + c.level], total);
    base = __shfl_sync(0xffffffffu, base, 0);
    if (base + total > L.cand_cap) { if (lane == 0) atomicExch(P.error_flag, 1); return; }
    uint32_t* out = L.cand + (int64_t)f * P.cand_fstride + base;
    int written = 0;
    for (int i0 = 0; i0 < nkept; i0 += 32) {
        const int i = i0 + lane;
        int pos = 0, s = 0;
        bool emit = false;
        if (i < nkept) { pos = list[i]; s = score[pos + TP]; emit = true; }
        const unsigned m = __ballot_sync(0xffffffffu, emit);
        if (emit) {
            const int y = pos / TP, x = pos - y * TP - off;         // tile column `off` == view column 0
            out[written + __popc(m & ((1u << lane) - 1))] = qt_pack(c.x0 + x - kMinBorder, c.y0 + y - kMinBorder, s);
        }
        written += __popc(m);
    }
}

FastLaunchPlan make_fast_launch_plan(const OrbPlan& PL) {
    FastLaunchPlan fp;
    int mw = 7, mh = 7, area = 1;
    for (const FastCell& c : PL.cells) {
        const int w = c.x1 - c.x0, h = c.y1 - c.y0;
        if (w > mw) mw = w;
        if (h > mh) mh = h;
        if ((w - 6) * (h - 6) > area) area = (w - 6) * (h - 6);
    }
    fp.tp = (19 + mw + 4 + 15) / 16 * 16;  // view starts at tile column off <= 19; >= 4 readable bytes right of the last interior word
    fp.th = mh;
    fp.list_cap = area;
    const int bytes = fp.tp * fp.th + fp.tp * (fp.th + 2) + 2 * ((area + 7) & ~7) + 16;
    fp.warp_stride = (bytes + 127) / 128 * 128;
    fp.smem_bytes = (size_t)fp.warp_stride * kFastWarps;
    return fp;
}

cudaError_t configure_fast_smem(size_t smem_bytes) {
    cudaError_t e = cudaFuncSetAttribute(fast_warp_cells_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
    if (e != cudaSuccess) return e;
    return cudaFuncSetAttribute(fast_warp_cells_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
}

void launch_fast_v2(const DevPlan& P, const FastTmaMaps& M, bool use_tma, const FastLaunchPlan& fp, const FastCell* d_cells, int ncells, int frame0, cudaStream_t st) {
    const int nitems = ncells * P.nframes;
    const int nblocks = (nitems + kFastWarps - 1) / kFastWarps;
    FastTileGeom G;
    G.tp = fp.tp; G.th = fp.th; G.list_cap = fp.list_cap; G.warp_stride = fp.warp_stride; G.use_tma = use_tma ? 1 : 0; G.frame0 = frame0;
    if (use_tma) fast_warp_cells_kernel<true><<<nblocks, kFastWarps * 32, fp.smem_bytes, st>>>(P, M, d_cells, ncells, nitems, G);
    else fast_warp_cells_kernel<false><<<nblocks, kFastWarps * 32, fp.smem_bytes, st>>>(P, M, d_cells, ncells, nitems, G);
}

// ---- TMA tensor maps (driver entry point resolved at run time: no link dependency on libcuda) --------------------------------
typedef CUresult (*PFN_encode_tiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                     const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

bool encode_level_map(CUtensorMap* out, const void* base, int w, int h, int pitch, int64_t fstride, int nframes, int box_w, int box_h) {
    static PFN_encode_tiled fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qres;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = (PFN_encode_tiled)p;
        cudaGetLastError();
    }
    if (!fn) return false;
    if (((uintptr_t)base & 15) || (pitch & 15) || (fstride & 15) || box_w > 256 || box_h > 256) return false;
    cuuint64_t gdim[3] = {(cuuint64_t)w, (cuuint64_t)h, (cuuint64_t)nframes};
    cuuint64_t gstr[2] = {(cuuint64_t)pitch, (cuuint64_t)fstride};
    cuuint32_t box[3] = {(cuuint32_t)box_w, (cuuint32_t)box_h, 1};
    cuuint32_t est[3] = {1, 1, 1};
    return fn(out, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, const_cast<void*>(base), gdim, gstr, box, est, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
              CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace sgs
