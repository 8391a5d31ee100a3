// conv1x1_tc.cuh -- the detector's 1x1 convolutions (66 of the 70 convolutions of mobilenetv3_ssdlite_voc.param, 90 % of its MACs;
// Detector2D.cc:39-45 runs them through ncnn) as a Hopper-native GEMM:
//     out[p][co] = tail(bias[co] + sum_ci X[p][ci] * W[co][ci])          X: NHWC activations [pixels of all frames][Cin], W: [Cout][Cin]
//   * operands reach shared memory by TMA (cp.async.bulk.tensor.2d, 128-byte swizzle, out-of-range rows / channels zero-filled) through a ring of
//     stages guarded by mbarriers; the weight tile of the CTA stays resident in shared memory when it fits,
//   * the contraction is wgmma.mma_async (tf32, m64nNk8 with N = the tile's output channels): each of the two consumer warpgroups owns 64 pixels of
//     the 128-pixel tile and the whole output-channel tile, the activations enter as register fragments read from the swizzled stage, the weights
//     as shared-memory descriptors,
//   * FP32-grade accuracy: every operand is x = hi + lo with hi, lo exactly representable in TF32 (round-to-nearest split); each k-step issues
//     lo*hi + hi*lo + hi*hi (the dropped lo*lo term is < 2^-22 relative).  Weights are split once at load time, activations in registers,
//   * epilogue straight from the accumulator registers: bias -> fused element-wise tail -> NHWC store (each warp store covers whole 32-byte sectors).
// One CTA = two consumer warpgroups + one TMA producer warpgroup, persistent over the pixel tiles of one output-channel tile: the producer refills the
// ring while the consumers run the epilogue of the previous tile.  Narrow tiles run two CTAs per SM, so one CTA's epilogue overlaps the other's MMAs.
#pragma once
#include <cuda.h>
#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>
#include <type_traits>
#include <vector>

#include "host_stage.cuh"

namespace sgs {
namespace tc {

constexpr int kBM = 128;        // pixels per tile = two wgmma M = 64 warpgroups
constexpr int kBK = 32;         // floats per k-block = one 128-byte swizzle row (16 = one 64-byte row for layers with at most 16 input channels)
constexpr int kMaxStages = 8;
constexpr int kWN = 32;         // output-channel granule of a tile (the narrowest wgmma, m64n32k8)
constexpr int kMaxNT = 256;     // output channels per tile (128 accumulator registers per consumer thread)
constexpr int kMaxChunks = kMaxNT / kWN;
constexpr int kThreads = 3 * 128;       // two consumer warpgroups + the producer warpgroup (one thread of it issues the loads)
// Narrow tiles (one 32-channel chunk) run two CTAs per SM (conv1x1_tc_kernel): the accumulators and the split fragments of a k-block then fit the
// 80 registers per thread that two 384-thread CTAs leave.  (Two CTAs of 64-channel tiles measured slower than one: see DESIGN.md section 4.)
constexpr int kNarrowChunks = 1;
constexpr int kNarrowSmem = 110 * 1024; // dynamic shared memory of such a CTA: two fit the 228 KB of an SM with their 1 KB reserves and static barriers

// ---------------------------------------------------------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_addr(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count)); }
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) { asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory"); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "WAIT_%=:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra DONE_%=;\n\t"
        "bra WAIT_%=;\n\t"
        "DONE_%=:\n\t}" ::"r"(bar), "r"(parity) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int x, int y, uint32_t bar) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(dst), "l"(map), "r"(x), "r"(y), "r"(bar)
                 : "memory");
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_wait_all() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }
// d[64 x N] += a[64 x 8] (register fragment) * b[N x 8]^T (K-major tile in shared memory), N = 32 ... 256 in steps of 32.  d holds N / 2 floats per
// thread in the wgmma register order: d[4j + 2h + q] is row g + 8h, column 8j + 2t + q of the warp's 16 rows (g = lane / 4, t = lane % 4), so the first
// 16 floats are the m64n32 accumulator of columns 0-31, the next 16 that of columns 32-63, and so on.
#define SGS_WGMMA_HEAD(n) "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n" #n "k8.f32.tf32.tf32 "
#define SGS_WGMMA_IN "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc)
#define SGS_ACC8(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7])
template <int N>
__device__ __forceinline__ void wgmma_tf32(float (&d)[N / 2], const uint32_t (&a)[4], uint64_t bdesc) {
    static_assert(N % 32 == 0 && N >= 32 && N <= 256, "m64nNk8 with N a multiple of 32 up to 256");
    if constexpr (N == 32)
        asm volatile(SGS_WGMMA_HEAD(32)
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, {%16, %17, %18, %19}, %20, p, 1, 1;\n\t}"
                     : SGS_ACC8(0), SGS_ACC8(8)
                     : SGS_WGMMA_IN : "memory");
    else if constexpr (N == 64)
        asm volatile(SGS_WGMMA_HEAD(64)
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
                     : SGS_ACC8(0), SGS_ACC8(8), SGS_ACC8(16), SGS_ACC8(24)
                     : SGS_WGMMA_IN : "memory");
    else if constexpr (N == 96)
        asm volatile(SGS_WGMMA_HEAD(96)
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, {%48, %49, %50, %51}, %52, p, 1, 1;\n\t}"
                     : SGS_ACC8(0), SGS_ACC8(8), SGS_ACC8(16), SGS_ACC8(24), SGS_ACC8(32), SGS_ACC8(40)
                     : SGS_WGMMA_IN : "memory");
    else if constexpr (N == 128)
        asm volatile(SGS_WGMMA_HEAD(128)
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
                     : SGS_ACC8(0), SGS_ACC8(8), SGS_ACC8(16), SGS_ACC8(24), SGS_ACC8(32), SGS_ACC8(40), SGS_ACC8(48), SGS_ACC8(56)
                     : SGS_WGMMA_IN : "memory");
    else if constexpr (N == 160)
        asm volatile(SGS_WGMMA_HEAD(160)
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
        " %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79}, {%80, %81, %82, %83}, %84, p, 1, 1;\n\t}"
                     : SGS_ACC8(0), SGS_ACC8(8), SGS_ACC8(16), SGS_ACC8(24), SGS_ACC8(32), SGS_ACC8(40), SGS_ACC8(48), SGS_ACC8(56), SGS_ACC8(64), SGS_ACC8(72)
                     : SGS_WGMMA_IN : "memory");
    else if constexpr (N == 192)
        asm volatile(SGS_WGMMA_HEAD(192)
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
        " %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, {%96, %97, %98, %99}, %100, p, 1, 1;\n\t}"
                     : SGS_ACC8(0), SGS_ACC8(8), SGS_ACC8(16), SGS_ACC8(24), SGS_ACC8(32), SGS_ACC8(40), SGS_ACC8(48), SGS_ACC8(56), SGS_ACC8(64), SGS_ACC8(72), SGS_ACC8(80), SGS_ACC8(88)
                     : SGS_WGMMA_IN : "memory");
    else if constexpr (N == 224)
        asm volatile(SGS_WGMMA_HEAD(224)
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
        " %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95,"
        " %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111}, {%112, %113, %114, %115}, %116, p, 1, 1;\n\t}"
                     : SGS_ACC8(0), SGS_ACC8(8), SGS_ACC8(16), SGS_ACC8(24), SGS_ACC8(32), SGS_ACC8(40), SGS_ACC8(48), SGS_ACC8(56), SGS_ACC8(64), SGS_ACC8(72), SGS_ACC8(80), SGS_ACC8(88), SGS_ACC8(96), SGS_ACC8(104)
                     : SGS_WGMMA_IN : "memory");
    else if constexpr (N == 256)
        asm volatile(SGS_WGMMA_HEAD(256)
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31,"
        " %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63,"
        " %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95,"
        " %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, {%128, %129, %130, %131}, %132, p, 1, 1;\n\t}"
                     : SGS_ACC8(0), SGS_ACC8(8), SGS_ACC8(16), SGS_ACC8(24), SGS_ACC8(32), SGS_ACC8(40), SGS_ACC8(48), SGS_ACC8(56), SGS_ACC8(64), SGS_ACC8(72), SGS_ACC8(80), SGS_ACC8(88), SGS_ACC8(96), SGS_ACC8(104), SGS_ACC8(112), SGS_ACC8(120)
                     : SGS_WGMMA_IN : "memory");
}
#undef SGS_ACC8
#undef SGS_WGMMA_IN
#undef SGS_WGMMA_HEAD

// wgmma shared-memory descriptor of a K-major tile whose rows are one swizzle row (ROWB = 128 or 64 bytes) and whose 8-row groups are 8 * ROWB
// bytes apart: start >> 4 | LBO (unused by swizzled K-major tiles) << 16 | SBO << 32 | layout << 62 (SWIZZLE_128B = 1, SWIZZLE_64B = 2).
// A k-step inside the swizzle row advances the start address by its byte offset (the tiles are aligned to the swizzle pattern).  The same
// descriptor serves any N: the wgmma's k extent (8 floats = 32 bytes) stays inside one swizzle row, so LBO is never used, and its N / 8 row groups
// are read SBO apart -- the NT rows of a weight tile are one such run.
template <int ROWB>
__device__ __forceinline__ uint64_t kmajor_desc(uint32_t saddr) {
    static_assert(ROWB == 128 || ROWB == 64, "one swizzle row per tile row");
    return (uint64_t)((saddr & 0x3ffffu) >> 4) | (1ull << 16) | ((uint64_t)((8 * ROWB) >> 4) << 32) | ((uint64_t)(ROWB == 128 ? 1 : 2) << 62);
}
// byte offset of element (row, k) of a tile written by TMA with the 128- / 64-byte swizzle (16-byte pieces XORed with the row's position in the pattern)
template <int ROWB>
__device__ __forceinline__ uint32_t swz_offset(int row, int k) {
    const int sw = ROWB == 128 ? (row & 7) : ((row >> 1) & 3);
    return (uint32_t)(row * ROWB + ((((k >> 2) ^ sw) << 4) | ((k & 3) << 2)));
}

// x = hi + lo, both TF32 (round to nearest, ties away, by integer arithmetic on the bit pattern)
__device__ __forceinline__ void split_tf32(uint32_t x, uint32_t& hi, uint32_t& lo) {
    hi = (x + 0x1000u) & 0xffffe000u;
    lo = (__float_as_uint(__fsub_rn(__uint_as_float(x), __uint_as_float(hi))) + 0x1000u) & 0xffffe000u;
}

struct TcGeom {
    int npix, Cin, Cout;          // rows of X, channels in / out
    int NT, KB, stages;           // output channels per tile (multiple of kWN), k-blocks, pipeline depth of the operand ring
    int m_tiles;                  // 128-pixel tiles
    int b_resident;               // the CTA's weight tile (all k-blocks, hi + lo) is loaded once and stays in shared memory
    int HW;                       // pixels per frame (output addressing)
    int64_t frame_stride;         // floats between consecutive frames of the output
    int64_t base_off;             // float offset of frame 0 of the output inside `out`
    int pitch;                    // floats between consecutive pixels of the output
    int vec_ok;                   // 8-byte aligned channel pairs: float2 stores
    int coalesce;                 // contiguous [pixel][channel] output (frame_stride == HW * pitch): a pixel's row address needs no division by HW
};

#ifdef SGS_GEMM_TRACE
// Probe build only (tools/gemm_tile_trace.py): clock64() stamps of the first kTraceTiles tiles of CTA (0, 0), by role (consumer warpgroup 0, 1,
// producer) and CTA-local tile: TR_START tile start, TR_RING clocks spent in ring waits (summed over the tile's k-blocks), TR_ISSUED last wgmma
// issued, TR_DRAINED its wait_group returned, TR_EPI_END epilogue done, TR_KWAIT clocks in the k-loop's wait_group (summed).
constexpr int kTraceTiles = 16;
enum { TR_START, TR_RING, TR_ISSUED, TR_DRAINED, TR_EPI_END, TR_KWAIT, TR_EVENTS };
__device__ long long g_gemm_trace[3][kTraceTiles][TR_EVENTS];
#define SGS_STAMP() clock64()
#define SGS_TRACE(on, role, tile, ev, v) do { if ((on) && blockIdx.x == 0 && blockIdx.y == 0 && (tile) < kTraceTiles) g_gemm_trace[role][tile][ev] = (v); } while (0)
#else
#define SGS_STAMP() 0ll
#define SGS_TRACE(on, role, tile, ev, v) do { } while (0)
#endif

// Persistent, warp-specialised.  CTA (x, y) owns output-channel tile y and walks the pixel tiles x, x + gridDim.x, ...
//   warps 0-3, 4-7 : consumer warpgroups (pixels 0-63 / 64-127 of the tile): split the activation fragments, issue the wgmma, run the epilogue
//   warps 8-11     : producer warpgroup, registers handed to the consumers (setmaxnreg); one thread issues the TMA loads of the activation k-blocks (and of the weight k-blocks unless resident) into a ring of `stages` slots
// mbarriers: full[s] (TMA -> consumers), empty[s] (every consumer warp's MMAs on slot s have completed -> producer), bfull (resident weights).
// EpiFn: struct with  template <int N> __device__ void run(float (&v)[N], int64_t idx0) const   applied to N consecutive channels of one pixel;
// idx0 = pixel * Cout + channel (the NHWC index of same-shape operand tensors).
// NC: the 32-channel chunks of the tile (NT == 32 * NC); each split term of a k-step is one m64n(NT)k8 wgmma over the whole tile.  Narrow tiles
// (NC = kNarrowChunks) run two CTAs per SM (ctas_per_sm): each CTA's epilogue -- the stores and the fused tail's operand loads -- overlaps the other
// CTA's MMAs; every thread keeps the at most 80 registers that two 384-thread CTAs leave (no setmaxnreg split).  Wide tiles run one CTA per SM with
// the 232 / 40 split.
template <int NC>
constexpr int ctas_per_sm() { return NC <= kNarrowChunks ? 2 : 1; }
template <class EpiFn, int BKT, int NC>
__global__ void __launch_bounds__(kThreads, ctas_per_sm<NC>()) conv1x1_tc_kernel(const __grid_constant__ CUtensorMap mapA, const __grid_constant__ CUtensorMap mapBh,
                                                              const __grid_constant__ CUtensorMap mapBl, const float* __restrict__ bias,
                                                              float* __restrict__ out, const TcGeom G, const EpiFn epi) {
    static_assert(NC >= 1 && NC <= kMaxChunks, "chunks per tile");
    constexpr int NT = NC * kWN;
    constexpr bool kSplitRegs = ctas_per_sm<NC>() == 1;
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    __shared__ __align__(8) uint64_t s_full[kMaxStages], s_empty[kMaxStages], s_bfull;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int n0 = blockIdx.y * G.NT;
    constexpr int ROWB = BKT * 4;                                             // bytes per operand row = one swizzle row
    constexpr int KS = BKT / 8;                                               // k-steps per k-block
    const uint32_t a_bytes = kBM * ROWB, b_bytes = (uint32_t)G.NT * ROWB;
    const uint32_t stage_bytes = a_bytes + (G.b_resident ? 0u : 2 * b_bytes);
    const uint32_t sbase = (smem_addr(smem_raw) + 1023u) & ~1023u;
    const uint8_t* gbase = smem_raw + (sbase - smem_addr(smem_raw));
    const uint32_t bres = sbase + (uint32_t)G.stages * stage_bytes;          // resident weights: [kb][hi | lo]
    const int my_tiles = (G.m_tiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;

    if (tid == 0) {
        for (int s = 0; s < G.stages; ++s) { mbar_init(smem_addr(&s_full[s]), 1); mbar_init(smem_addr(&s_empty[s]), 8); }
        mbar_init(smem_addr(&s_bfull), 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (tid == 256) {
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapA) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapBh) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"(&mapBl) : "memory");
    }
    __syncthreads();

    if (warp >= 8) {
        // ------------------------------------------------------------------------------------------------ TMA producer
        if constexpr (kSplitRegs) asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
        if (warp == 8 && lane == 0) {
            if (G.b_resident) {
                mbar_expect_tx(smem_addr(&s_bfull), (uint32_t)G.KB * 2 * b_bytes);
                for (int kb = 0; kb < G.KB; ++kb) {
                    tma_load_2d(bres + (uint32_t)kb * 2 * b_bytes, &mapBh, kb * BKT, n0, smem_addr(&s_bfull));
                    tma_load_2d(bres + (uint32_t)kb * 2 * b_bytes + b_bytes, &mapBl, kb * BKT, n0, smem_addr(&s_bfull));
                }
            }
            uint32_t g = 0;
            for (int it = 0; it < my_tiles; ++it) {
                SGS_TRACE(true, 2, it, TR_START, SGS_STAMP());
                long long ring_wait = 0;
                const int m0 = ((int)blockIdx.x + it * (int)gridDim.x) * kBM;
                for (int kb = 0; kb < G.KB; ++kb, ++g) {
                    const uint32_t s = g % (uint32_t)G.stages, ph = (g / (uint32_t)G.stages) & 1u;
                    const long long w0 = SGS_STAMP();
                    mbar_wait(smem_addr(&s_empty[s]), ph ^ 1u);
                    ring_wait += SGS_STAMP() - w0;
                    const uint32_t st = sbase + s * stage_bytes, bar = smem_addr(&s_full[s]);
                    mbar_expect_tx(bar, a_bytes + (G.b_resident ? 0u : 2 * b_bytes));
                    tma_load_2d(st, &mapA, kb * BKT, m0, bar);
                    if (!G.b_resident) {
                        tma_load_2d(st + a_bytes, &mapBh, kb * BKT, n0, bar);
                        tma_load_2d(st + a_bytes + b_bytes, &mapBl, kb * BKT, n0, bar);
                    }
                }
                SGS_TRACE(true, 2, it, TR_RING, ring_wait);
                SGS_TRACE(true, 2, it, TR_ISSUED, SGS_STAMP());
            }
        }
        return;
    }

    // ---------------------------------------------------------------------------------------------------- consumers
    // Fragment ownership (wgmma m64nNk8, tf32): warp w of the warpgroup owns rows 16w + g and 16w + g + 8 (g = lane / 4); the A fragment holds
    // columns t and t + 4 of the k-step (t = lane % 4), the accumulator the channel pairs 8j + 2t, j = 0..NT/8-1 (wgmma_tf32: acc[4j + 2h + q]).
    if constexpr (kSplitRegs) asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int wg = warp >> 2, g = lane >> 2, t = lane & 3;
    const int r0 = 64 * wg + 16 * (warp & 3) + g;                            // tile row of fragment rows 0 (and r0 + 8)
    const int ncol = min(NT, G.Cout - n0);                                   // real output channels of this tile (uniform)
    const bool tr = (tid & 127) == 0;                                         // the warpgroup's trace thread (probe build only)
    (void)tr;
    // bias of channel n0 + 2t + d at bias_t[d]: the epilogue's loads then differ by constant offsets (one base address, not one per channel pair)
    const float* bias_t = bias ? bias + n0 + 2 * t : nullptr;
    if (G.b_resident) mbar_wait(smem_addr(&s_bfull), 0);
    float acc[NT / 2];
    uint32_t g_ring = 0;
    for (int it = 0; it < my_tiles; ++it) {
        SGS_TRACE(tr, wg, it, TR_START, SGS_STAMP());
        long long ring_wait = 0, k_wait = 0, issued = 0;
#pragma unroll
        for (int i = 0; i < NT / 2; ++i) acc[i] = 0.f;
        for (int kb = 0; kb < G.KB; ++kb, ++g_ring) {
            const uint32_t s = g_ring % (uint32_t)G.stages, ph = (g_ring / (uint32_t)G.stages) & 1u;
            const long long w0 = SGS_STAMP();
            mbar_wait(smem_addr(&s_full[s]), ph);
            ring_wait += SGS_STAMP() - w0;
            const uint8_t* sa = gbase + (size_t)s * stage_bytes;
            const uint32_t bh0 = G.b_resident ? bres + (uint32_t)kb * 2 * b_bytes : sbase + s * stage_bytes + a_bytes;
            const int ksteps = min(BKT, G.Cin - kb * BKT + 7) >> 3;          // 8-wide k-steps that hold real channels (the rest is zero fill)
            uint32_t ah[KS][4], al[KS][4];
#pragma unroll
            for (int j = 0; j < KS; ++j) {
                if (j < ksteps) {
                    const uint32_t x0 = *reinterpret_cast<const uint32_t*>(sa + swz_offset<ROWB>(r0, 8 * j + t));
                    const uint32_t x1 = *reinterpret_cast<const uint32_t*>(sa + swz_offset<ROWB>(r0 + 8, 8 * j + t));
                    const uint32_t x2 = *reinterpret_cast<const uint32_t*>(sa + swz_offset<ROWB>(r0, 8 * j + t + 4));
                    const uint32_t x3 = *reinterpret_cast<const uint32_t*>(sa + swz_offset<ROWB>(r0 + 8, 8 * j + t + 4));
                    split_tf32(x0, ah[j][0], al[j][0]); split_tf32(x1, ah[j][1], al[j][1]);
                    split_tf32(x2, ah[j][2], al[j][2]); split_tf32(x3, ah[j][3], al[j][3]);
                }
            }
            wgmma_fence();
#pragma unroll
            for (int j = 0; j < KS; ++j) {
                if (j < ksteps) {                                            // every output element sees lo*hi, hi*lo, hi*hi of each k-step, in that order
                    const uint32_t b = bh0 + (uint32_t)(j * 32);
                    wgmma_tf32<NT>(acc, al[j], kmajor_desc<ROWB>(b));
                    wgmma_tf32<NT>(acc, ah[j], kmajor_desc<ROWB>(b + b_bytes));
                    wgmma_tf32<NT>(acc, ah[j], kmajor_desc<ROWB>(b));
                }
            }
            wgmma_commit();
            issued = SGS_STAMP();
            wgmma_wait_all();
            k_wait += SGS_STAMP() - issued;
            __syncwarp();
            if (lane == 0) mbar_arrive(smem_addr(&s_empty[s]));              // this warp's MMAs on slot s are complete
        }
        SGS_TRACE(tr, wg, it, TR_ISSUED, issued);
        SGS_TRACE(tr, wg, it, TR_DRAINED, SGS_STAMP());
        SGS_TRACE(tr, wg, it, TR_RING, ring_wait);
        SGS_TRACE(tr, wg, it, TR_KWAIT, k_wait);

        // ------------------------------------------------------------------------------------------------ epilogue
        // Wide tiles load the bias of a chunk's 8 channels of this thread before the chunk's first store, so the 8 loads are in flight together.
        // (Loaded at each use, behind the branches on the column, every load's latency stood between two stores: the epilogue of a 128 x 256
        // tile took 7 x its MMAs, DESIGN.md section 6.)  Narrow tiles load at each use: their 80 registers leave no room for the 8 values.
        const int pt = ((int)blockIdx.x + it * (int)gridDim.x) * kBM + r0;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int p = pt + 8 * h;
            if (p >= G.npix) continue;
            int64_t off = (int64_t)p * G.pitch;
            if (!G.coalesce) { const int f = p / G.HW; off = (int64_t)f * G.frame_stride + (int64_t)(p - f * G.HW) * G.pitch; }
            float* o = out + G.base_off + off + n0;
            const int64_t idx = (int64_t)p * G.Cout + n0;
#pragma unroll
            for (int c = 0; c < NC; ++c) {
                if (c * kWN >= ncol) break;
                float bc[8];                                                 // bias of channels 8j + 2t + q, j = 4c .. 4c + 3, at bc[2(j - 4c) + q]
                if constexpr (kSplitRegs) {
#pragma unroll
                    for (int i = 0; i < 8; ++i) {
                        const int j = 4 * c + i / 2, q = i & 1;
                        bc[i] = bias_t && 8 * j + 2 * t + q < ncol ? __ldg(bias_t + 8 * j + q) : 0.f;
                    }
                }
                auto bias_of = [&](int j, int q) {
                    if constexpr (kSplitRegs) return bc[2 * (j - 4 * c) + q];
                    else return bias_t ? __ldg(bias_t + 8 * j + q) : 0.f;
                };
#pragma unroll
                for (int j = 4 * c; j < 4 * c + 4; ++j) {                      // 8-channel groups of the 32-channel chunk c
                    const int col = 8 * j + 2 * t;
                    if (col + 1 < ncol && G.vec_ok) {
                        float v[2] = {__fadd_rn(acc[4 * j + 2 * h], bias_of(j, 0)), __fadd_rn(acc[4 * j + 2 * h + 1], bias_of(j, 1))};
                        epi.template run<2>(v, idx + col);
                        *reinterpret_cast<float2*>(o + col) = make_float2(v[0], v[1]);
                    } else {
#pragma unroll
                        for (int q = 0; q < 2; ++q) {
                            if (col + q < ncol) {
                                float one[1] = {__fadd_rn(acc[4 * j + 2 * h + q], bias_of(j, q))};
                                epi.template run<1>(one, idx + col + q);
                                o[col + q] = one[0];
                            }
                        }
                    }
                }
            }
        }
        SGS_TRACE(tr, wg, it, TR_EPI_END, SGS_STAMP());
    }
}
#undef SGS_TRACE
#undef SGS_STAMP

// ---------------------------------------------------------------------------------------------------------------- host side
typedef CUresult (*PFN_tmap_encode)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
inline PFN_tmap_encode tmap_encoder() {
    static PFN_tmap_encode fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess) fn = (PFN_tmap_encode)p;
        cudaGetLastError();
    }
    return fn;
}
// 2-D FP32 tensor [rows][cols] with `pitch` floats between rows; box = bk floats (one 128- or 64-byte swizzle row) x box_rows, zero fill outside
inline bool encode_kmajor_map(CUtensorMap* m, const float* base, int64_t rows, int cols, int64_t pitch, int box_rows, int bk) {
    PFN_tmap_encode fn = tmap_encoder();
    if (!fn || ((uintptr_t)base & 15) || (pitch & 3) || box_rows < 1 || box_rows > 256 || (bk != 32 && bk != 16)) return false;
    cuuint64_t gdim[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    cuuint64_t gstr[1] = {(cuuint64_t)pitch * 4};
    cuuint32_t box[2] = {(cuuint32_t)bk, (cuuint32_t)box_rows};
    cuuint32_t est[2] = {1, 1};
    return fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), gdim, gstr, box, est, CU_TENSOR_MAP_INTERLEAVE_NONE, bk == 32 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B,
              CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

struct GemmPlan {
    int Cin = 0, Cout = 0, NT = 0, n_tiles = 0, KB = 0, BK = kBK, stages = 0, smem_bytes = 0, Kp = 0, Np = 0, b_resident = 0;
    float* d_whi = nullptr; float* d_wlo = nullptr;
    CUtensorMap map_hi, map_lo;
};

inline void split_tf32_host(float x, float& hi, float& lo) {
    uint32_t b; memcpy(&b, &x, 4);
    uint32_t h = (b + 0x1000u) & 0xffffe000u;
    memcpy(&hi, &h, 4);
    const float r = x - hi;       // exact
    memcpy(&b, &r, 4);
    uint32_t l = (b + 0x1000u) & 0xffffe000u;
    memcpy(&lo, &l, 4);
}

// Tiling of one layer (no device access): output-channel tiles of at most kMaxNT channels (a multiple of the 32-channel wgmma width), weights
// resident when all their k-blocks fit in 128 KB, ring depth from what is left of the 227 KB of shared memory a CTA may use.  Narrow tiles (at most
// 32 channels, two CTAs per SM) fit everything in kNarrowSmem: weights resident when a ring of two stages still fits beside them.
// m_tiles (128-pixel tiles of the largest batch, 0 = unknown) picks the number of output-channel tiles: every tile of a pixel block re-reads the
// activations and pays the pipeline's fill, so fewer, wider tiles win as long as they still fill the machine.  The cost of a plan is modelled as
// waves of the persistent grid (one CTA per SM) x (NT + 100)  and the cheapest tile count between Cout / 256 and Cout / 128 is taken.
constexpr int kPlanSMs = 132;
inline void plan_tiling(int Cin, int Cout, GemmPlan* P, int force_nt = 0, int m_tiles = 0) {
    P->Cin = Cin; P->Cout = Cout;
    int nt = (Cout + 127) / 128;
    if (m_tiles > 0) {
        double best = 1e300;
        for (int n = (Cout + kMaxNT - 1) / kMaxNT; n <= (Cout + 127) / 128; ++n) {
            const int w = ((Cout + n - 1) / n + kWN - 1) & ~(kWN - 1);
            const long long waves = ((long long)m_tiles * n + kPlanSMs - 1) / kPlanSMs;
            const double cost = (double)waves * (w + 100);
            if (cost < best) { best = cost; nt = n; }
        }
    }
    P->NT = force_nt > 0 ? force_nt : ((Cout + nt - 1) / nt + kWN - 1) & ~(kWN - 1);
    P->n_tiles = (Cout + P->NT - 1) / P->NT;
    P->BK = Cin <= 16 ? 16 : kBK;                                        // at most 16 input channels: 64-byte operand rows, half the ring slot
    P->KB = (Cin + P->BK - 1) / P->BK;
    P->Kp = P->KB * P->BK; P->Np = P->n_tiles * P->NT;
    const int a_stage = kBM * P->BK * 4, b_block = 2 * P->NT * P->BK * 4;
    const int b_all = P->KB * b_block;
    const bool narrow = P->NT <= kNarrowChunks * kWN;            // two CTAs per SM: each gets at most kNarrowSmem
    const int cap = narrow ? kNarrowSmem : 226 * 1024;
    P->b_resident = (narrow ? b_all + 2 * a_stage + 1024 <= cap : b_all <= 128 * 1024) ? 1 : 0;
    const int budget = cap - 1024 - (P->b_resident ? b_all : 0);
    const int stage_bytes = a_stage + (P->b_resident ? 0 : b_block);
    int st = budget / stage_bytes;
    if (st > kMaxStages) st = kMaxStages;
    if (st < 2) st = 2;
    P->stages = st;
    P->smem_bytes = st * stage_bytes + (P->b_resident ? b_all : 0) + 1024;
}

// Splits and uploads W [Cout][Cin] into buffers owned by `res`, picks the tiling.  Returns false when TMA is unavailable or an allocation fails.
inline bool plan_weights(HandleResources& res, const float* W, int Cin, int Cout, GemmPlan* P, int force_nt = 0, int m_tiles = 0) {
    plan_tiling(Cin, Cout, P, force_nt, m_tiles);
    std::vector<float> hi((size_t)P->Np * P->Kp, 0.f), lo((size_t)P->Np * P->Kp, 0.f);
    for (int co = 0; co < Cout; ++co)
        for (int c = 0; c < Cin; ++c) split_tf32_host(W[(size_t)co * Cin + c], hi[(size_t)co * P->Kp + c], lo[(size_t)co * P->Kp + c]);
    if (res.alloc(&P->d_whi, hi.size() * 4) != cudaSuccess) return false;
    if (res.alloc(&P->d_wlo, lo.size() * 4) != cudaSuccess) return false;
    if (cudaMemcpy(P->d_whi, hi.data(), hi.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess) return false;
    if (cudaMemcpy(P->d_wlo, lo.data(), lo.size() * 4, cudaMemcpyHostToDevice) != cudaSuccess) return false;
    return encode_kmajor_map(&P->map_hi, P->d_whi, P->Np, P->Kp, P->Kp, P->NT, P->BK) && encode_kmajor_map(&P->map_lo, P->d_wlo, P->Np, P->Kp, P->Kp, P->NT, P->BK);
}

// x / c.  For c == 6 (the hard-swish / hard-sigmoid divisor of the model) the quotient comes from the reciprocal and one FMA correction:
// q = RN(x * r), q' = RN(q + RN(x - 6q) * r), which equals the correctly rounded RN(x / 6) for every float with |x| >= 2^-100 and for zeros up to the
// sign of zero (verified exhaustively on the host over all 2^32 bit patterns); below 2^-100 it may differ from the IEEE quotient in the last bit of a
// denormal.  Both the fused and the layer-by-layer execution use this function.  (The generic IEEE division takes its slow path whenever the dividend is
// zero -- half of all hard-swish outputs.)
__device__ __forceinline__ float div6(float x) {         // correctly rounded x / 6 without the division subroutine
    const float r = 0x1.555556p-3f;                     // RN(1/6)
    const float q = __fmul_rn(x, r);
    return __fmaf_rn(__fmaf_rn(-6.0f, q, x), r, q);
}
__device__ __forceinline__ float div_scalar(float x, float c) { return c == 6.0f ? div6(x) : __fdiv_rn(x, c); }

inline int sm_count() {
    static int n = 0;
    if (!n) { int dev = 0; cudaGetDevice(&dev); if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1) n = kPlanSMs; }
    return n;
}

// mapA: encode_kmajor_map over the input activations (any number of rows >= npix; box kBM rows, P.BK columns)
template <class EpiFn>
inline bool launch_conv1x1_tc_map(const GemmPlan& P, const CUtensorMap& mapA, int npix, const float* bias, float* out, int HW, int64_t frame_stride, int64_t base_off,
                                  int pitch, const EpiFn& epi, cudaStream_t st) {
    if (P.NT % kWN || P.NT > kMaxNT || P.stages > kMaxStages) return false;
    TcGeom G;
    G.npix = npix; G.Cin = P.Cin; G.Cout = P.Cout; G.NT = P.NT; G.KB = P.KB; G.stages = P.stages;
    G.m_tiles = (npix + kBM - 1) / kBM; G.b_resident = P.b_resident;
    G.HW = HW; G.frame_stride = frame_stride; G.base_off = base_off; G.pitch = pitch;
    G.vec_ok = ((pitch & 1) == 0 && (frame_stride & 1) == 0 && (base_off & 1) == 0 && (((uintptr_t)out) & 7) == 0) ? 1 : 0;
    G.coalesce = (frame_stride == 0 || frame_stride == (int64_t)HW * pitch) ? 1 : 0;
    const bool narrow = P.NT <= kNarrowChunks * kWN;
    if (narrow && P.smem_bytes > kNarrowSmem) return false;
    auto go = [&](auto kern) -> bool {
        if (cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, 226 * 1024) != cudaSuccess) return false;   // cheap; per device
        // one wave of persistent CTAs: as many per SM as the registers and shared memory hold (two for narrow tiles, one otherwise)
        int per_sm = 1;
        if (narrow && (cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, (int)cudaSharedmemCarveoutMaxShared) != cudaSuccess ||
                       cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, kThreads, P.smem_bytes) != cudaSuccess || per_sm < 1))
            return false;
        int gx = sm_count() * per_sm / P.n_tiles;
        if (gx < 1) gx = 1;
        if (gx > G.m_tiles) gx = G.m_tiles;
        kern<<<dim3(gx, P.n_tiles), kThreads, P.smem_bytes, st>>>(mapA, P.map_hi, P.map_lo, bias, out, G, epi);
        return true;
    };
    // one instance per k-block width and tile width: the wgmma's N is a compile-time constant
    auto by_width = [&](auto bk) -> bool {
        constexpr int BKT = decltype(bk)::value;
        switch (P.NT / kWN) {
        case 1: return go(conv1x1_tc_kernel<EpiFn, BKT, 1>);
        case 2: return go(conv1x1_tc_kernel<EpiFn, BKT, 2>);
        case 3: return go(conv1x1_tc_kernel<EpiFn, BKT, 3>);
        case 4: return go(conv1x1_tc_kernel<EpiFn, BKT, 4>);
        case 5: return go(conv1x1_tc_kernel<EpiFn, BKT, 5>);
        case 6: return go(conv1x1_tc_kernel<EpiFn, BKT, 6>);
        case 7: return go(conv1x1_tc_kernel<EpiFn, BKT, 7>);
        case 8: return go(conv1x1_tc_kernel<EpiFn, BKT, 8>);
        }
        return false;
    };
    static_assert(kMaxChunks == 8, "one case per tile width");
    const bool ok = P.BK == 16 ? by_width(std::integral_constant<int, 16>{}) : by_width(std::integral_constant<int, 32>{});
    if (!ok) return false;
    return cudaGetLastError() == cudaSuccess;
}

}  // namespace tc
}  // namespace sgs
