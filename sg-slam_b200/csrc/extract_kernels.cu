// extract_kernels.cu -- hand-written sm_90a kernels of the batched ORB extractor.
//
// Stage            reference (src/ORBextractor.cc)                kernel
//   pyramid        ComputePyramid :1108-1133 (cv::resize)          resize_level_kernel   (1 launch per level >= 1, all frames)
//   FAST + NMS     ComputeKeyPointsOctTree :766-830 (cv::FAST)     fast_warp_cells_kernel (fast_kernel.cu; 1 launch: all levels, all frames)
//   distribution   DistributeOctTree :540-764                      quadtree_kernel       (1 launch: block per (level, frame))
//   blur           GaussianBlur :1086-1087                         blur_tile_kernel      (blur_kernel.cu, 1 launch per level)
//   orient + BRIEF IC_Angle :78-105, computeOrbDescriptor :109-148 describe_kernel       (1 launch: warp per keypoint)
//
// All integer stages are bit-exact by construction; float work uses explicitly rounded intrinsics (no FMA).
#include <cuda_runtime.h>

#include "extract_dev.cuh"
#include "extract_kernels.h"

namespace sgs {

// 256 BRIEF point pairs (x0,y0,x1,y1) as int8; lane i of a warp reads its 32 bytes with two 128-bit loads
__device__ __align__(16) const int8_t g_pattern[1024] = {
#include "orb_pattern.inc"
};

// --------------------------------------------------------------------------------------------------------------------
// Pyramid: cv::resize(INTER_LINEAR) for CV_8UC1 in its 11-bit fixed-point form.  Each thread produces 4 consecutive
// pixels of one output row (one 32-bit store); tables hold (src index, w0, w1) per output column / row.
// --------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) resize_level_kernel(const uint8_t* __restrict__ src, int sw, int sh, int spitch, int64_t sfstride,
                                                           uint8_t* __restrict__ dst, int dw, int dh, int dpitch, int64_t dfstride,
                                                           const short4* __restrict__ xtab, const short4* __restrict__ ytab) {
    const int x4 = (blockIdx.x * 32 + threadIdx.x) * 4;
    const int y = blockIdx.y * 8 + threadIdx.y;
    if (x4 >= dw || y >= dh) return;
    const uint8_t* S = src + (int64_t)blockIdx.z * sfstride;
    uint8_t* D = dst + (int64_t)blockIdx.z * dfstride;
    const short4 ty = __ldg(&ytab[y]);
    const int sy0 = ty.x, sy1 = min(sy0 + 1, sh - 1);
    const int b0 = ty.y, b1 = ty.z;
    const uint8_t* r0 = S + (int64_t)sy0 * spitch;
    const uint8_t* r1 = S + (int64_t)sy1 * spitch;
    uint32_t packed = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int x = x4 + i;
        int v = 0;
        if (x < dw) {
            const short4 tx = __ldg(&xtab[x]);
            const int sx0 = tx.x, sx1 = min(sx0 + 1, sw - 1);
            const int a0 = tx.y, a1 = tx.z;
            const int h0 = (int)__ldg(r0 + sx0) * a0 + (int)__ldg(r0 + sx1) * a1;
            const int h1 = (int)__ldg(r1 + sx0) * a0 + (int)__ldg(r1 + sx1) * a1;
            v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
            v = min(max(v, 0), 255);
        }
        packed |= (uint32_t)v << (8 * i);
    }
    *reinterpret_cast<uint32_t*>(D + (int64_t)y * dpitch + x4) = packed;  // dpitch is a multiple of 16: in-bounds
}

void launch_resize(const DevPlan& P, int level, cudaStream_t st) {
    const DevLevel& s = P.lv[level - 1];
    const DevLevel& d = P.lv[level];
    dim3 block(32, 8), grid((d.w + 127) / 128, (d.h + 7) / 8, P.nframes);
    resize_level_kernel<<<grid, block, 0, st>>>(s.img, s.w, s.h, s.pitch, s.fstride, d.img_w, d.w, d.h, d.pitch, d.fstride, d.xtab, d.ytab);
}

// --------------------------------------------------------------------------------------------------------------------
// Quadtree distribution: one block per (level, frame) running qt_distribute (quadtree_core.h).
// Shared memory: node-side arrays (sized for the largest level) + sort keys when they fit; otherwise the keys live in a
// global scratch area (pathological candidate counts, e.g. pure-noise images).
// --------------------------------------------------------------------------------------------------------------------
constexpr int kQtThreads = 256;

struct CudaCtx {
    __device__ __forceinline__ int tid() const { return threadIdx.x; }
    __device__ __forceinline__ int nthreads() const { return blockDim.x; }
    __device__ __forceinline__ void sync() const { __syncthreads(); }
    __device__ __forceinline__ int group() const { return 32; }                     // a warp synchronises by itself
    __device__ __forceinline__ void group_sync() const { __syncwarp(); }
};

__host__ __device__ inline size_t qt_node_bytes(int cap) {
    // lo, hi, seq, free, list_a, list_b, exp_a, exp_b : 8 x int32 ; exp_key : u64 ; bnd : 3 x int32 ; child : 4 x int32 ; depth, flag : 2 x u8
    return (size_t)cap * (8 * 4 + 8 + 3 * 4 + 4 * 4 + 2) + 64 + 16 * 4;
}

__global__ void __launch_bounds__(kQtThreads) quadtree_kernel(const __grid_constant__ DevPlan P, int smem_key_cap, int node_cap, uint64_t* __restrict__ key_scratch,
                                                              int64_t key_scratch_fstride, const int64_t* __restrict__ key_scratch_off) {
    extern __shared__ __align__(16) uint8_t smem[];
    const int level = blockIdx.x, f = blockIdx.y;
    const DevLevel& L = P.lv[level];
    const int n = min(P.cand_count[f * P.nlevels + level], L.cand_cap);
    int n_sort = 1;
    while (n_sort < n) n_sort <<= 1;
    QtWork w;
    uint8_t* p = smem;
    w.exp_key = reinterpret_cast<uint64_t*>(p); p += (size_t)node_cap * 8;
    w.lo = reinterpret_cast<int32_t*>(p); p += (size_t)node_cap * 4;
    w.hi = reinterpret_cast<int32_t*>(p); p += (size_t)node_cap * 4;
    w.seq = reinterpret_cast<int32_t*>(p); p += (size_t)node_cap * 4;
    w.free_list = reinterpret_cast<int32_t*>(p); p += (size_t)node_cap * 4;
    w.list_a = reinterpret_cast<int32_t*>(p); p += (size_t)node_cap * 4;
    w.list_b = reinterpret_cast<int32_t*>(p); p += (size_t)node_cap * 4;
    w.exp_a = reinterpret_cast<int32_t*>(p); p += (size_t)node_cap * 4;
    w.exp_b = reinterpret_cast<int32_t*>(p); p += (size_t)node_cap * 4;
    w.bnd = reinterpret_cast<int32_t*>(p); p += (size_t)node_cap * 12;
    w.child = reinterpret_cast<int32_t*>(p); p += (size_t)node_cap * 16;
    w.sc = reinterpret_cast<int32_t*>(p); p += 16 * 4;
    w.depth = p; p += node_cap;
    w.flag = p; p += node_cap;
    p = smem + ((p - smem + 15) & ~(size_t)15);
    w.pool_cap = qt_pool_cap(L.qt.n_target, L.qt.n_ini);
    w.n = n; w.n_sort = n_sort;
    if (n_sort <= smem_key_cap) w.keys = reinterpret_cast<uint64_t*>(p);
    else w.keys = key_scratch + (int64_t)f * key_scratch_fstride + key_scratch_off[level];
    CudaCtx ctx;
    uint32_t* out = P.kp_stage + (int64_t)f * P.kp_stage_per_frame + L.kp_off;
    qt_distribute(ctx, L.cand + (int64_t)f * P.cand_fstride, L.qt, w, out, L.kp_cap, &P.kp_stage_n[f * P.nlevels + level]);
}

void launch_quadtree(const DevPlan& P, int smem_key_cap, int node_cap, size_t smem_bytes, uint64_t* key_scratch, int64_t key_scratch_fstride,
                     const int64_t* d_key_scratch_off, cudaStream_t st) {
    dim3 grid(P.nlevels, P.nframes);
    quadtree_kernel<<<grid, kQtThreads, smem_bytes, st>>>(P, smem_key_cap, node_cap, key_scratch, key_scratch_fstride, d_key_scratch_off);
}

cudaError_t configure_quadtree_smem(size_t smem_bytes) {
    return cudaFuncSetAttribute(quadtree_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem_bytes);
}

size_t quadtree_node_bytes(int cap) { return qt_node_bytes(cap); }

// --------------------------------------------------------------------------------------------------------------------
// Orientation (intensity centroid over the 749-pixel disc) + rotated BRIEF, one warp per keypoint.
//   lanes 0..30 own the patch rows dy = lane-15 for the moments; lane i owns descriptor byte i.
//   cos/sin follow the contract of SURVEY Appendix A9: (float)cos((double)angle_rad).
// Also writes the final cv::KeyPoint records (coordinates scaled to level 0, :1096-1102) and the per-frame count.
// --------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) describe_kernel(const __grid_constant__ DevPlan P) {
    const int f = blockIdx.y;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int k = blockIdx.x * 8 + warp;
    // locate keypoint k of this frame: levels are concatenated 0..L-1 (:1076-1105); lane l holds the count of level l
    int nl = 0;
    if (lane < P.nlevels) nl = min(P.kp_stage_n[f * P.nlevels + lane], P.lv[lane].kp_cap);
    int incl = nl;
#pragma unroll
    for (int o = 1; o < kMaxLevels; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
    const int total = __shfl_sync(0xffffffffu, incl, P.nlevels - 1);
    const unsigned below = __ballot_sync(0xffffffffu, lane < P.nlevels && incl <= k);   // levels entirely before keypoint k
    const int level = __popc(below);
    const int idx = k - (level ? __shfl_sync(0xffffffffu, incl, level ? level - 1 : 0) : 0);
    if (k == 0 && lane == 0) {
        P.out_count[f] = min(total, P.out_cap);
        if (total > P.out_cap) atomicExch(P.error_flag, 2);
    }
    if (k >= total || k >= P.out_cap) return;
    const DevLevel& L = P.lv[level];
    const uint32_t c = P.kp_stage[(int64_t)f * P.kp_stage_per_frame + L.kp_off + idx];
    const int kx = qt_x(c) + kMinBorder, ky = qt_y(c) + kMinBorder;
    // --- IC_Angle: lane == patch column u = lane-15; every row is one coalesced <= 31-byte segment ---
    int m10 = 0, m01 = 0;
    {
        const int u = lane - 15;
        const int au = u < 0 ? -u : u;
        const uint8_t* ctr = L.img + (int64_t)f * L.fstride + (int64_t)ky * L.pitch + kx + u;
        int colsum = 0;
#pragma unroll
        for (int v = -kHalfPatch; v <= kHalfPatch; ++v) {
            const int d = P.umax[v < 0 ? -v : v];
            if (lane < 31 && au <= d) {
                const int val = __ldg(ctr + (int64_t)v * L.pitch);
                colsum += val;
                m01 += v * val;
            }
        }
        m10 = u * colsum;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        m10 += __shfl_xor_sync(0xffffffffu, m10, o);
        m01 += __shfl_xor_sync(0xffffffffu, m01, o);
    }
    const float angle = dev_fast_atan2((float)m01, (float)m10);
    // --- rotated BRIEF ---
    const float factor_pi = (float)(3.14159265358979323846 / (double)180.f);
    const float ang = __fmul_rn(angle, factor_pi);
    float cs = 0.f;                                   // lane 0: cos, lane 1: sin (FP64 libm calls are long: do them once)
    if (lane == 0) cs = (float)cos((double)ang);
    if (lane == 1) cs = (float)sin((double)ang);
    const float a = __shfl_sync(0xffffffffu, cs, 0), b = __shfl_sync(0xffffffffu, cs, 1);
    const uint8_t* center = L.blur + (int64_t)f * L.bfstride + (int64_t)ky * L.bpitch + kx;
    __align__(16) int8_t pat[32];
    *reinterpret_cast<int4*>(pat) = __ldg(reinterpret_cast<const int4*>(g_pattern + lane * 32));
    *reinterpret_cast<int4*>(pat + 16) = __ldg(reinterpret_cast<const int4*>(g_pattern + lane * 32 + 16));
    int byte = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
        const float x0 = (float)pat[4 * j], y0 = (float)pat[4 * j + 1], x1 = (float)pat[4 * j + 2], y1 = (float)pat[4 * j + 3];
        const int r0 = dev_cv_round(__fadd_rn(__fmul_rn(x0, b), __fmul_rn(y0, a)));
        const int c0 = dev_cv_round(__fsub_rn(__fmul_rn(x0, a), __fmul_rn(y0, b)));
        const int r1 = dev_cv_round(__fadd_rn(__fmul_rn(x1, b), __fmul_rn(y1, a)));
        const int c1 = dev_cv_round(__fsub_rn(__fmul_rn(x1, a), __fmul_rn(y1, b)));
        const int t0 = __ldg(center + (int64_t)r0 * L.bpitch + c0);
        const int t1 = __ldg(center + (int64_t)r1 * L.bpitch + c1);
        byte |= (t0 < t1) << j;
    }
    P.out_desc[((int64_t)f * P.out_cap + k) * 32 + lane] = (uint8_t)byte;
    if (lane == 0) {
        sgs_keypoint kp;
        kp.x = (level == 0) ? (float)kx : __fmul_rn((float)kx, L.scale);
        kp.y = (level == 0) ? (float)ky : __fmul_rn((float)ky, L.scale);
        kp.size = L.patch_size;
        kp.angle = angle;
        kp.response = (float)qt_score(c);
        kp.octave = level;
        kp.class_id = -1;
        P.out_kps[(int64_t)f * P.out_cap + k] = kp;
    }
}

void launch_describe(const DevPlan& P, cudaStream_t st) {
    dim3 grid((P.out_cap + 7) / 8, P.nframes);
    describe_kernel<<<grid, 256, 0, st>>>(P);
}

}  // namespace sgs
