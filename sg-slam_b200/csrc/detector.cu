// detector.cu -- Detector2D (src/Detector2D.cc:16-89): batched FP32 forward of the ncnn graph the reference loads
// (Thirdparty/ncnn_model/mobilenetv3_ssdlite_voc.param/.bin, MobileNetV3 backbone + SSDLite heads, 408 layers) and the post-processing of
// its "detection_out" rows into Object2D / potential-dynamic boxes.
//
// The handle parses the ncnn text graph and weight blob itself, infers every blob shape for the fixed 3x300x300 input (Detector2D.h:70),
// folds the constant sub-graphs (MemoryData scalars, PriorBox, their Concat) on the host, and turns the rest into a flat list of kernels:
//   preprocess     : Mat::from_pixels_resize + substract_mean_normalize (Detector2D.cc:39-40), fixed-point bilinear (bit-exact with cv::resize)
//   conv1x1        : 90 % of the MACs; out[p][co] = bias[co] + sum_ci X[p][ci] * W[co][ci] over the pixels of all frames, as a TMA-fed wgmma
//                    GEMM with error-compensated TF32 operands (conv1x1_tc.cuh), bias + fused element-wise tail in its epilogue
//   dwconv / conv  : depth-wise 3x3 / 5x5 (channel-vectorised) and the few dense convolutions the GEMM does not take (first layer, Cin not a multiple of 4)
//   eltwise        : whatever element-wise chain could not be attached to a producer
//   softmax, detection-output (per class: threshold, sort, top-k, greedy NMS; per frame: merge, top-k, Detector2D.cc:52-88)
// Element-wise layers (BinaryOp with a constant / a tensor / the chain's own start value, Clip, ReLU) that follow a producer are applied in
// the producer's epilogue in graph order, one rounding per op, so fused and unfused execution give identical bits.
// Layout: every 3-D blob is [frames][h][w][c] FP32 (channels innermost): both GEMM operands are K-major for wgmma (tf32) and TMA-addressable, the
// depth-wise kernels read channel vectors, and ncnn's Permute(order 3: c,h,w -> h,w,c) in front of the SSD heads becomes an alias -- the head
// convolutions write straight into the concatenated mbox_loc / mbox_conf buffers.  sgs_detector_blob transposes back to ncnn's c,h,w on read-out.
// Activations live in a pool planned by liveness.
#include <cuda_runtime.h>

#include <algorithm>
#include <cmath>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <sstream>
#include <stdexcept>

#include "conv1x1_tc.cuh"
#include "sgs_common.h"

namespace sgs {
namespace det {

using tc::div_scalar;
using tc::div6;

// ---------------------------------------------------------------------------------------------------------------- element-wise tail
enum { E_ADD = 0, E_SUB = 1, E_MUL = 2, E_DIV = 3, E_CLIP = 4, E_RELU = 5 };   // 0..3 = ncnn BinaryOp op_type
enum { SRC_SCALAR = 0, SRC_TENSOR = 1, SRC_START = 2 };
struct EpiStep {
    int op, src, rev;       // rev: the running value is the SECOND operand (matters for sub / div)
    float a, b;             // scalar operand / clip bounds
    const float* t;         // same-shape tensor operand
};
constexpr int kMaxEpi = 8;
struct Epi {
    int n, kind;
    EpiStep s[kMaxEpi];
};

enum { EK_GENERIC = 0, EK_NONE, EK_RELU, EK_CLIP, EK_HSWISH, EK_ADD_T, EK_SE_TAIL, EK_SE_MUL };   // Epi::kind: recognised tails run as straight-line code;
// the divisor of the three hard-swish / hard-sigmoid kinds is exactly 6 (checked at classification: other divisors take the generic tail)

template <int KIND>
__device__ __forceinline__ float apply_epi(const Epi& e, float v, int64_t idx) {
    if constexpr (KIND == EK_NONE) return v;
    else if constexpr (KIND == EK_RELU) return fmaxf(v, 0.f);
    else if constexpr (KIND == EK_CLIP) return fminf(fmaxf(v, e.s[0].a), e.s[0].b);
    else if constexpr (KIND == EK_HSWISH)                // v * clip(v + a) / b   (add scalar, clip, mul(rev) start, div scalar)
        return div6(__fmul_rn(v, fminf(fmaxf(__fadd_rn(v, e.s[0].a), e.s[1].a), e.s[1].b)));
    else if constexpr (KIND == EK_ADD_T) return __fadd_rn(v, __ldg(e.s[0].t + idx));
    else if constexpr (KIND == EK_SE_TAIL)               // t1 * (clip(v + a) / b) + t2   (add scalar, clip, div scalar, mul(rev) tensor, add tensor)
        return __fadd_rn(__fmul_rn(__ldg(e.s[3].t + idx), div6(fminf(fmaxf(__fadd_rn(v, e.s[0].a), e.s[1].a), e.s[1].b))), __ldg(e.s[4].t + idx));
    else if constexpr (KIND == EK_SE_MUL)                // t1 * (clip(v + a) / b)   (add scalar, clip, div scalar, mul(rev) tensor): hard-sigmoid gate
        return __fmul_rn(__ldg(e.s[3].t + idx), div6(fminf(fmaxf(__fadd_rn(v, e.s[0].a), e.s[1].a), e.s[1].b)));
    else {
        const float v0 = v;
        for (int i = 0; i < e.n; ++i) {
            const EpiStep& s = e.s[i];
            if (s.op == E_CLIP) { v = fminf(fmaxf(v, s.a), s.b); continue; }
            if (s.op == E_RELU) { v = fmaxf(v, 0.f); continue; }
            const float o = s.src == SRC_SCALAR ? s.a : (s.src == SRC_START ? v0 : __ldg(s.t + idx));
            const float x = s.rev ? o : v, y = s.rev ? v : o;
            v = s.op == E_ADD ? __fadd_rn(x, y) : s.op == E_SUB ? __fsub_rn(x, y) : s.op == E_MUL ? __fmul_rn(x, y) : div_scalar(x, y);
        }
        return v;
    }
}

// Runs `body` with the tail kind as a compile-time constant.  In a kernel the (block-uniform) switch is taken once per thread, not once per output;
// on the host it picks the GEMM instantiation of the kind.
template <int KIND> struct EpiKind { static constexpr int value = KIND; };
template <class F>
__host__ __device__ __forceinline__ void epi_dispatch(int kind, F&& body) {
    switch (kind) {
    case EK_NONE: body(EpiKind<EK_NONE>{}); break;
    case EK_RELU: body(EpiKind<EK_RELU>{}); break;
    case EK_CLIP: body(EpiKind<EK_CLIP>{}); break;
    case EK_HSWISH: body(EpiKind<EK_HSWISH>{}); break;
    case EK_ADD_T: body(EpiKind<EK_ADD_T>{}); break;
    case EK_SE_TAIL: body(EpiKind<EK_SE_TAIL>{}); break;
    case EK_SE_MUL: body(EpiKind<EK_SE_MUL>{}); break;
    default: body(EpiKind<EK_GENERIC>{}); break;
    }
}

// Four consecutive channels of one pixel (idx % 4 == 0, 16-byte aligned operand tensors): the tensor operands of the recognised tails are fetched
// as one float4 each instead of four scalar loads (the element order and roundings are those of apply_epi).
template <int KIND>
__device__ __forceinline__ void apply_epi4(const Epi& e, float (&v)[4], int64_t idx) {
    if constexpr (KIND == EK_ADD_T) {
        const float4 t = __ldg(reinterpret_cast<const float4*>(e.s[0].t + idx));
        v[0] = __fadd_rn(v[0], t.x); v[1] = __fadd_rn(v[1], t.y); v[2] = __fadd_rn(v[2], t.z); v[3] = __fadd_rn(v[3], t.w);
    } else if constexpr (KIND == EK_SE_TAIL || KIND == EK_SE_MUL) {
        const float4 t1 = __ldg(reinterpret_cast<const float4*>(e.s[3].t + idx));
        float4 t2 = make_float4(0.f, 0.f, 0.f, 0.f);
        if constexpr (KIND == EK_SE_TAIL) t2 = __ldg(reinterpret_cast<const float4*>(e.s[4].t + idx));
        const float a[4] = {t1.x, t1.y, t1.z, t1.w}, b[4] = {t2.x, t2.y, t2.z, t2.w};
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            const float g = __fmul_rn(a[q], div6(fminf(fmaxf(__fadd_rn(v[q], e.s[0].a), e.s[1].a), e.s[1].b)));
            v[q] = KIND == EK_SE_TAIL ? __fadd_rn(g, b[q]) : g;
        }
    } else {
#pragma unroll
        for (int q = 0; q < 4; ++q) v[q] = apply_epi<KIND>(e, v[q], idx + q);
    }
}

// The tail on N consecutive channels v of one pixel, the first at flat index idx0: as float4 groups when N % 4 == 0 and idx0 % 4 == 0, else one
// channel at a time.  ALIGNED: the caller knows that idx0 % 4 == 0, and the test is not made at run time.
template <int KIND, bool ALIGNED = false, int N>
__device__ __forceinline__ void apply_epi_n(const Epi& e, float (&v)[N], int64_t idx0) {
    static_assert(!ALIGNED || N % 4 == 0, "ALIGNED takes whole float4 groups");
    if constexpr (N % 4 == 0) {
        if (ALIGNED || (idx0 & 3) == 0) {
#pragma unroll
            for (int q = 0; q < N; q += 4) {
                float w[4] = {v[q], v[q + 1], v[q + 2], v[q + 3]};
                apply_epi4<KIND>(e, w, idx0 + q);
                v[q] = w[0]; v[q + 1] = w[1]; v[q + 2] = w[2]; v[q + 3] = w[3];
            }
            return;
        }
    }
    if constexpr (!ALIGNED)
#pragma unroll
        for (int q = 0; q < N; ++q) v[q] = apply_epi<KIND>(e, v[q], idx0 + q);
}

// The tail as the functor conv1x1_tc_kernel takes, with the kind fixed at compile time: one instantiation of the GEMM per kind, so that the epilogue
// carries the code of one tail only (with a run-time switch every tail is inlined at every call site of the epilogue, and the kernel's code outgrows
// the instruction cache).
template <int KIND>
struct EpiFnK {
    Epi e;
    template <int N>
    __device__ __forceinline__ void run(float (&v)[N], int64_t idx0) const { apply_epi_n<KIND>(e, v, idx0); }
};

// ---------------------------------------------------------------------------------------------------------------- kernels
// Mat::from_pixels_resize(..., PIXEL_RGB, w, h, 300, 300) + substract_mean_normalize (norm = 1).  11-bit fixed-point bilinear, the arithmetic
// of cv::resize INTER_LINEAR on 8-bit data: horizontal pass keeps value*2048, vertical pass ((b0*(r0>>4))>>16) + ((b1*(r1>>4))>>16) + 2) >> 2.
__device__ __forceinline__ void resize_coeff(int d, double scale, int sn, int& s, int& a0, int& a1) {
    float f = (float)((d + 0.5) * scale - 0.5);
    s = (int)floorf(f);
    f = __fsub_rn(f, (float)s);
    if (s < 0) { s = 0; f = 0.f; }
    if (s >= sn - 1) { s = sn - 2; f = 1.f; }
    a0 = max(-32768, min(32767, __float2int_rn(__fmul_rn(__fsub_rn(1.f, f), 2048.f))));
    a1 = max(-32768, min(32767, __float2int_rn(__fmul_rn(f, 2048.f))));
}

// The coefficients depend on the destination coordinate only: one small table per source geometry (source index, the two 11-bit weights; columns, then
// rows), rebuilt when the camera size changes -- the float / double evaluation of resize_coeff per pixel made the resize instruction-bound (81 % issue-active).
__global__ void __launch_bounds__(256) preprocess_table_kernel(int sw, int sh, int T, int* __restrict__ tab) {
    const int d = blockIdx.x * 256 + threadIdx.x;
    if (d >= T) return;
    int s, a0, a1;
    resize_coeff(d, (double)sw / T, sw, s, a0, a1);
    tab[d] = s; tab[T + d] = a0; tab[2 * T + d] = a1;
    resize_coeff(d, (double)sh / T, sh, s, a0, a1);
    tab[3 * T + d] = s; tab[4 * T + d] = a0; tab[5 * T + d] = a1;
}

__global__ void __launch_bounds__(256) preprocess_kernel(const uint8_t* __restrict__ rgb, int64_t frame_stride, int pitch, int T, const int* __restrict__ tab,
                                                         float m0, float m1, float m2, float* __restrict__ out) {
    const int f = blockIdx.y, i = blockIdx.x * 256 + threadIdx.x;
    if (i >= T * T) return;
    const int dy = i / T, dx = i - dy * T;
    const int sx = __ldg(tab + dx), a0 = __ldg(tab + T + dx), a1 = __ldg(tab + 2 * T + dx);
    const int sy = __ldg(tab + 3 * T + dy), b0 = __ldg(tab + 4 * T + dy), b1 = __ldg(tab + 5 * T + dy);
    const uint8_t* r0 = rgb + f * frame_stride + (int64_t)sy * pitch + sx * 3;
    const uint8_t* r1 = r0 + pitch;
    const float mean[3] = {m0, m1, m2};
    float* o = out + ((int64_t)f * T * T + i) * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const int h0 = r0[c] * a0 + r0[c + 3] * a1, h1 = r1[c] * a0 + r1[c + 3] * a1;
        int v = (((b0 * (h0 >> 4)) >> 16) + ((b1 * (h1 >> 4)) >> 16) + 2) >> 2;
        v = max(0, min(255, v));
        o[c] = __fsub_rn((float)v, mean[c]);
    }
}

struct ConvGeom {
    int Cin, Cout, H, W, OH, OW, k, stride, pad, dil;
};

// depth-wise K x K, stride S on [frame][h][w][c]: V channels (float4 when C % 4 == 0) x XT consecutive outputs of one row per thread; the
// K + (XT-1)S input vectors of each kernel row are loaded once and shared by the XT windows.  Weights transposed to [ky][kx][c] at load time.
// Each output accumulates ky-major / kx-minor from zero, then the bias.
template <int K, int S, int V, int YT>
__global__ void __launch_bounds__(256) dwconv_kernel(const float* __restrict__ in, const float* __restrict__ Wt, const float* __restrict__ bias,
                                                     float* __restrict__ out, ConvGeom g, int64_t total, Epi epi) {
    constexpr int XT = 4, NX = (XT - 1) * S + K, NY = (YT - 1) * S + K;      // outputs per thread: YT rows x XT columns; input rows / columns they need
    const int64_t t0 = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (t0 >= total) return;
    const int cv = g.Cout / V, owq = (g.OW + XT - 1) / XT, ohq = (g.OH + YT - 1) / YT;
    const int c = (int)(t0 % cv) * V;
    int64_t t = t0 / cv;
    const int ox0 = (int)(t % owq) * XT; t /= owq;
    const int oy0 = (int)(t % ohq) * YT;
    const int64_t f = t / ohq;
    float acc[YT][XT][V];
#pragma unroll
    for (int y = 0; y < YT; ++y)
#pragma unroll
        for (int o = 0; o < XT; ++o)
#pragma unroll
            for (int q = 0; q < V; ++q) acc[y][o][q] = 0.f;
    const int ix0 = ox0 * S - g.pad;
    const bool xin = ix0 >= 0 && ix0 + NX <= g.W;
    const int cst = g.Cout >> 2;             // float4 stride between neighbouring pixels
    // input rows in ascending order: output row y takes kernel row ky = r - y * S of input row r, so every output still accumulates ky-major / kx-minor
#pragma unroll
    for (int r = 0; r < NY; ++r) {
        const int iy = oy0 * S - g.pad + r;
        if (iy < 0 || iy >= g.H) continue;
        const float* row = in + ((f * g.H + iy) * (int64_t)g.W) * g.Cout + c;
        float x[NX][V];
        if (V == 4 && xin) {                 // every tap column inside the row: one pointer, a 32-bit stride, no per-tap tests
            const float4* p4 = reinterpret_cast<const float4*>(row + (int64_t)ix0 * g.Cout);
#pragma unroll
            for (int j = 0; j < NX; ++j) { const float4 q = __ldg(p4 + j * cst); x[j][0] = q.x; x[j][1] = q.y; x[j][2] = q.z; x[j][3] = q.w; }
        } else
#pragma unroll
        for (int j = 0; j < NX; ++j) {
            const int ix = ix0 + j;
            if (ix >= 0 && ix < g.W) {
                if constexpr (V == 4) { const float4 q = __ldg(reinterpret_cast<const float4*>(row + (int64_t)ix * g.Cout)); x[j][0] = q.x; x[j][1] = q.y; x[j][2] = q.z; x[j][3] = q.w; }
                else x[j][0] = __ldg(row + (int64_t)ix * g.Cout);
            } else {
#pragma unroll
                for (int q = 0; q < V; ++q) x[j][q] = 0.f;
            }
        }
#pragma unroll
        for (int y = 0; y < YT; ++y) {
            const int ky = r - y * S;
            if (ky < 0 || ky >= K) continue;                 // compile-time after unrolling
#pragma unroll
            for (int kx = 0; kx < K; ++kx) {
                float w[V];
                if constexpr (V == 4) { const float4 q = __ldg(reinterpret_cast<const float4*>(Wt + c) + (ky * K + kx) * cst); w[0] = q.x; w[1] = q.y; w[2] = q.z; w[3] = q.w; }
                else w[0] = __ldg(Wt + (ky * K + kx) * g.Cout + c);
#pragma unroll
                for (int o = 0; o < XT; ++o)
#pragma unroll
                    for (int q = 0; q < V; ++q) acc[y][o][q] = fmaf(w[q], x[o * S + kx][q], acc[y][o][q]);      // padding taps contribute w * 0
            }
        }
    }
    float b[V];
#pragma unroll
    for (int q = 0; q < V; ++q) b[q] = bias ? __ldg(bias + c + q) : 0.f;
    epi_dispatch(epi.kind, [&](auto kind) {
        constexpr int EK = decltype(kind)::value;
#pragma unroll
        for (int y = 0; y < YT; ++y) {
            if (oy0 + y >= g.OH) break;
            const int64_t o0 = ((f * g.OH + oy0 + y) * (int64_t)g.OW + ox0) * g.Cout + c;
#pragma unroll
            for (int o = 0; o < XT; ++o) {
                if (ox0 + o >= g.OW) break;
                const int64_t oi = o0 + (int64_t)o * g.Cout;
                float r[V];
#pragma unroll
                for (int q = 0; q < V; ++q) r[q] = __fadd_rn(acc[y][o][q], b[q]);
                apply_epi_n<EK, V == 4>(epi, r, oi);                   // V == 4: Cout % 4 == 0 and c % 4 == 0
                if constexpr (V == 4) *reinterpret_cast<float4*>(out + oi) = make_float4(r[0], r[1], r[2], r[3]);
                else out[oi] = r[0];
            }
        }
    });
}

// dense k x k convolution on [frame][h][w][c] for the layers the GEMM does not take (the network's first layer 3 -> 16, 3x3 stride 2, and the 1x1
// convolutions whose Cin is not a multiple of 4): one output pixel x kCot output channels per thread, the weights of the channel block staged
// in shared memory as [ky][kx][ci][kCot] so that every input value is loaded once and used kCot times.  Output addressing as in the GEMM
// (frame stride / base offset / pitch), so that a head convolution of this kind could write into a concatenated buffer as well.
constexpr int kCot = 8;
__global__ void __launch_bounds__(256) conv_small_kernel(const float* __restrict__ in, const float* __restrict__ Wt, const float* __restrict__ bias,
                                                         float* __restrict__ out, ConvGeom g, int64_t out_frame_stride, int64_t out_base, Epi epi) {
    extern __shared__ __align__(16) float sw[];
    const int co0 = blockIdx.y * kCot, f = blockIdx.z;
    const int taps = g.Cin * g.k * g.k;
    for (int e = threadIdx.x; e < taps * kCot; e += 256) {
        const int tp = e / kCot, o = e % kCot;                 // tp = (ky * k + kx) * Cin + ci
        const int ci = tp % g.Cin, kk = tp / g.Cin;
        sw[e] = co0 + o < g.Cout ? __ldg(Wt + ((int64_t)(co0 + o) * g.Cin + ci) * g.k * g.k + kk) : 0.f;
    }
    __syncthreads();
    const int p = blockIdx.x * 256 + threadIdx.x;
    if (p >= g.OH * g.OW) return;
    const int oy = p / g.OW, ox = p - oy * g.OW;
    float acc[kCot];
#pragma unroll
    for (int o = 0; o < kCot; ++o) acc[o] = 0.f;
    for (int ky = 0; ky < g.k; ++ky) {
        const int iy = oy * g.stride - g.pad + ky * g.dil;
        if (iy < 0 || iy >= g.H) continue;
        for (int kx = 0; kx < g.k; ++kx) {
            const int ix = ox * g.stride - g.pad + kx * g.dil;
            if (ix < 0 || ix >= g.W) continue;
            const float* src = in + (((int64_t)f * g.H + iy) * g.W + ix) * g.Cin;
            const float* wp = sw + (ky * g.k + kx) * g.Cin * kCot;
            for (int ci = 0; ci < g.Cin; ++ci) {
                const float x = __ldg(src + ci);
#pragma unroll
                for (int o = 0; o < kCot; ++o) acc[o] = fmaf(wp[ci * kCot + o], x, acc[o]);
            }
        }
    }
    float* orow = out + out_base + (int64_t)f * out_frame_stride + (int64_t)p * g.Cout;
    const int64_t idx0 = ((int64_t)f * g.OH * g.OW + p) * g.Cout;
    const bool vec = co0 + kCot <= g.Cout && (g.Cout & 3) == 0 && ((out_base | out_frame_stride) & 3) == 0;
    epi_dispatch(epi.kind, [&](auto kind) {
        constexpr int EK = decltype(kind)::value;
        float r[kCot];
        if (vec) {
#pragma unroll
            for (int o = 0; o < kCot; o += 4) {
                float w[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) w[q] = __fadd_rn(acc[o + q], bias ? __ldg(bias + co0 + o + q) : 0.f);
                apply_epi_n<EK, true>(epi, w, idx0 + co0 + o);         // vec: Cout % 4 == 0 and co0 % 8 == 0
                *reinterpret_cast<float4*>(orow + co0 + o) = make_float4(w[0], w[1], w[2], w[3]);
            }
        } else {
#pragma unroll
            for (int o = 0; o < kCot; ++o) {
                const int co = co0 + o;
                float w[1] = {0.f};
                if (co < g.Cout) { w[0] = __fadd_rn(acc[o], bias ? __ldg(bias + co) : 0.f); apply_epi_n<EK>(epi, w, idx0 + co); }
                r[o] = w[0];
            }
#pragma unroll
            for (int o = 0; o < kCot; ++o) if (co0 + o < g.Cout) orow[co0 + o] = r[o];
        }
    });
}

// The network's first layer as its own kernel (3 -> 16 channels, 3x3, stride 2, pad 1: 0.82 ms per 512 frames through the generic kernel above, the largest
// single launch of the detector; 0.55 ms here): one output pixel x all 16 channels per thread, the 27 x 16 weights in shared memory as [tap][channel]
// (warp-wide broadcast reads), every loop unrolled.  Same accumulation order per output channel as conv_small_kernel (ky, kx, ci from zero, then the bias).
__global__ void __launch_bounds__(256) conv_first_kernel(const float* __restrict__ in, const float* __restrict__ Wt, const float* __restrict__ bias,
                                                         float* __restrict__ out, ConvGeom g, Epi epi) {
    __shared__ __align__(16) float sw[27 * 16];
    const int f = blockIdx.y;
    for (int e = threadIdx.x; e < 27 * 16; e += 256) {
        const int tp = e >> 4, o = e & 15;                     // tp = (ky * 3 + kx) * 3 + ci
        const int ci = tp % 3, kk = tp / 3;
        sw[e] = __ldg(Wt + ((int64_t)o * 3 + ci) * 9 + kk);
    }
    __syncthreads();
    const int p = blockIdx.x * 256 + threadIdx.x;
    if (p >= g.OH * g.OW) return;
    const int oy = p / g.OW, ox = p - oy * g.OW;
    float acc[16];
#pragma unroll
    for (int o = 0; o < 16; ++o) acc[o] = 0.f;
    const float* img = in + (int64_t)f * g.H * g.W * 3;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
        const int iy = oy * 2 - 1 + ky;
        if (iy < 0 || iy >= g.H) continue;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const int ix = ox * 2 - 1 + kx;
            if (ix < 0 || ix >= g.W) continue;
            const float* src = img + ((int64_t)iy * g.W + ix) * 3;
#pragma unroll
            for (int ci = 0; ci < 3; ++ci) {
                const float x = __ldg(src + ci);
                const float4* w4 = reinterpret_cast<const float4*>(sw + ((ky * 3 + kx) * 3 + ci) * 16);
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const float4 w = w4[q];
                    acc[4 * q] = fmaf(w.x, x, acc[4 * q]); acc[4 * q + 1] = fmaf(w.y, x, acc[4 * q + 1]);
                    acc[4 * q + 2] = fmaf(w.z, x, acc[4 * q + 2]); acc[4 * q + 3] = fmaf(w.w, x, acc[4 * q + 3]);
                }
            }
        }
    }
    const int64_t idx0 = ((int64_t)f * g.OH * g.OW + p) * 16;
    epi_dispatch(epi.kind, [&](auto kind) {
        constexpr int EK = decltype(kind)::value;
#pragma unroll
        for (int o = 0; o < 16; o += 4) {
            float w[4];
#pragma unroll
            for (int q = 0; q < 4; ++q) w[q] = __fadd_rn(acc[o + q], bias ? __ldg(bias + o + q) : 0.f);
            apply_epi_n<EK, true>(epi, w, idx0 + o);
            *reinterpret_cast<float4*>(out + idx0 + o) = make_float4(w[0], w[1], w[2], w[3]);
        }
    });
}

__global__ void __launch_bounds__(256) eltwise_kernel(const float* __restrict__ in, float* __restrict__ out, int64_t total, Epi epi) {
    const int64_t idx = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (idx >= total) return;
    epi_dispatch(epi.kind, [&](auto kind) {
        float v[1] = {__ldg(in + idx)};
        apply_epi_n<decltype(kind)::value>(epi, v, idx);
        out[idx] = v[0];
    });
}

// Concat piece: per frame n floats from src (frame stride n) to dst + off (frame stride dst_n)
__global__ void __launch_bounds__(256) concat_copy_kernel(const float* __restrict__ src, int64_t n, float* __restrict__ dst, int64_t dst_n, int64_t off,
                                                          int64_t total) {
    const int64_t idx = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (idx >= total) return;
    const int64_t f = idx / n, i = idx - f * n;
    dst[f * dst_n + off + i] = __ldg(src + idx);
}

// Softmax over the innermost axis (w = classes) of a 2-D blob: max-subtract, exp, sum, divide.  One row per thread; rows of at most 32 classes
// stay in registers (one read and one write of the row), longer rows take the three-pass form.  Same operations in the same order either way.
__global__ void __launch_bounds__(256) softmax_rows_kernel(const float* __restrict__ in, float* __restrict__ out, int ncls, int64_t rows) {
    const int64_t r = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (r >= rows) return;
    const float* x = in + r * ncls;
    float* y = out + r * ncls;
    if (ncls <= 32) {
        float v[32];
#pragma unroll
        for (int c = 0; c < 32; ++c) v[c] = c < ncls ? __ldg(x + c) : 0.f;
        float m = v[0];
#pragma unroll
        for (int c = 1; c < 32; ++c) if (c < ncls) m = fmaxf(m, v[c]);
        float s = 0.f;
#pragma unroll
        for (int c = 0; c < 32; ++c) if (c < ncls) { v[c] = expf(__fsub_rn(v[c], m)); s = __fadd_rn(s, v[c]); }
#pragma unroll
        for (int c = 0; c < 32; ++c) if (c < ncls) y[c] = __fdiv_rn(v[c], s);
        return;
    }
    float m = x[0];
    for (int c = 1; c < ncls; ++c) m = fmaxf(m, x[c]);
    float s = 0.f;
    for (int c = 0; c < ncls; ++c) { const float e = expf(__fsub_rn(x[c], m)); y[c] = e; s = __fadd_rn(s, e); }
    for (int c = 0; c < ncls; ++c) y[c] = __fdiv_rn(y[c], s);
}

// ---- DetectionOutput
struct DetOutParams {
    int ncls, nprior, nms_topk, keep_topk;
    float nms_thr, conf_thr;
};

__device__ __forceinline__ float4 decode_box(const float* __restrict__ loc, const float* __restrict__ prior, const float* __restrict__ var, int i) {
    const float4 l = *reinterpret_cast<const float4*>(loc + 4 * (int64_t)i);
    const float4 pb = __ldg(reinterpret_cast<const float4*>(prior) + i), v = __ldg(reinterpret_cast<const float4*>(var) + i);
    const float pw = __fsub_rn(pb.z, pb.x), ph = __fsub_rn(pb.w, pb.y);
    const float pcx = __fmul_rn(__fadd_rn(pb.x, pb.z), 0.5f), pcy = __fmul_rn(__fadd_rn(pb.y, pb.w), 0.5f);
    const float cx = __fadd_rn(__fmul_rn(__fmul_rn(v.x, l.x), pw), pcx), cy = __fadd_rn(__fmul_rn(__fmul_rn(v.y, l.y), ph), pcy);
    const float w = __fmul_rn(expf(__fmul_rn(v.z, l.z)), pw), h = __fmul_rn(expf(__fmul_rn(v.w, l.w)), ph);
    const float hw = __fmul_rn(w, 0.5f), hh = __fmul_rn(h, 0.5f);
    return make_float4(__fsub_rn(cx, hw), __fsub_rn(cy, hh), __fadd_rn(cx, hw), __fadd_rn(cy, hh));
}

__device__ __forceinline__ void bitonic_sort_u64(unsigned long long* keys, int n /* power of two */) {
    for (int k = 2; k <= n; k <<= 1)
        for (int j = k >> 1; j > 0; j >>= 1) {
            __syncthreads();
            for (int i = threadIdx.x; i < n; i += blockDim.x) {
                const int ixj = i ^ j;
                if (ixj > i) {
                    const unsigned long long a = keys[i], b = keys[ixj];
                    const bool up = (i & k) == 0;
                    if ((a > b) == up) { keys[i] = b; keys[ixj] = a; }
                }
            }
        }
    __syncthreads();
}

// One block per (class >= 1, frame): candidates with score > conf_thr, descending score (ties: lower prior index first), first nms_topk,
// greedy NMS (drop when inter/union > nms_thr against any kept box).  Kept entries go to picked[f][cls-1][0..count) as sort keys
// (~score bits, class, prior) for the per-frame merge.
constexpr int kDetSortCap = 4096;
__global__ void __launch_bounds__(256) detout_class_kernel(const float* __restrict__ loc, const float* __restrict__ conf, const float* __restrict__ prior,
                                                           const float* __restrict__ var, DetOutParams P, unsigned long long* __restrict__ picked,
                                                           int32_t* __restrict__ picked_n) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);                 // [kDetSortCap]
    float4* box = reinterpret_cast<float4*>(keys + kDetSortCap);                                // [nms_topk]
    int* kept = reinterpret_cast<int*>(box + P.nms_topk);                                       // [nms_topk]
    __shared__ int s_n, s_kept;
    const int cls = blockIdx.x + 1, f = blockIdx.y;
    const float* cf = conf + (int64_t)f * P.nprior * P.ncls;
    const float* lf = loc + (int64_t)f * P.nprior * 4;
    if (threadIdx.x == 0) { s_n = 0; s_kept = 0; }
    __syncthreads();
    for (int i = threadIdx.x; i < P.nprior; i += blockDim.x) {
        const float s = cf[(int64_t)i * P.ncls + cls];
        if (s > P.conf_thr) {
            const int slot = atomicAdd(&s_n, 1);
            if (slot < kDetSortCap) keys[slot] = ((unsigned long long)(~__float_as_uint(s)) << 32) | (unsigned)i;
        }
    }
    __syncthreads();
    const int n = min(s_n, kDetSortCap);
    unsigned long long* dst = picked + ((int64_t)f * (P.ncls - 1) + (cls - 1)) * P.nms_topk;
    if (n == 0) { if (threadIdx.x == 0) picked_n[f * (P.ncls - 1) + cls - 1] = 0; return; }
    int np2 = 1;
    while (np2 < n) np2 <<= 1;
    for (int i = n + threadIdx.x; i < np2; i += blockDim.x) keys[i] = ~0ull;
    bitonic_sort_u64(keys, np2);
    const int m = min(n, P.nms_topk);
    for (int i = threadIdx.x; i < m; i += blockDim.x) box[i] = decode_box(lf, prior, var, (int)(keys[i] & 0xffffffffu));
    __syncthreads();
    for (int i = 0; i < m; ++i) {
        const float4 b = box[i];
        const float area = __fmul_rn(__fsub_rn(b.z, b.x), __fsub_rn(b.w, b.y));
        const int nk = s_kept;
        int sup = 0;
        for (int q = threadIdx.x; q < nk; q += blockDim.x) {
            const float4 a = box[kept[q]];
            float inter = 0.f;
            if (!(b.x > a.z || b.z < a.x || b.y > a.w || b.w < a.y))
                inter = __fmul_rn(__fsub_rn(fminf(a.z, b.z), fmaxf(a.x, b.x)), __fsub_rn(fminf(a.w, b.w), fmaxf(a.y, b.y)));
            const float uni = __fsub_rn(__fadd_rn(__fmul_rn(__fsub_rn(a.z, a.x), __fsub_rn(a.w, a.y)), area), inter);
            if (__fdiv_rn(inter, uni) > P.nms_thr) sup = 1;
        }
        sup = __syncthreads_or(sup);
        if (!sup && threadIdx.x == 0) { kept[s_kept] = i; s_kept = s_kept + 1; }
        __syncthreads();
    }
    const int nk = s_kept;
    for (int q = threadIdx.x; q < nk; q += blockDim.x) {
        const unsigned long long k = keys[kept[q]];
        dst[q] = (k & 0xffffffff00000000ull) | ((unsigned long long)cls << 16) | (k & 0xffffu);
    }
    if (threadIdx.x == 0) picked_n[f * (P.ncls - 1) + cls - 1] = nk;
}

struct PostParams {      // Detector2D.cc:52-88
    float det_thr, dyn_thr, target;
    int img_w, img_h, person, rows_cap, max_boxes;
};

// One block per frame: all kept entries of all classes, descending score, first keep_topk -> detection_out rows; then the reference's
// sequential pass over the rows (thread 0; <= keep_topk rows).
constexpr int kMergeCap = 8192;
__global__ void __launch_bounds__(256) detout_merge_kernel(const float* __restrict__ loc, const float* __restrict__ prior, const float* __restrict__ var,
                                                           DetOutParams P, const unsigned long long* __restrict__ picked, const int32_t* __restrict__ picked_n,
                                                           PostParams Q, float* __restrict__ rows, int32_t* __restrict__ nrows, sgs_object2d* __restrict__ objects,
                                                           int32_t* __restrict__ nobjects, sgs_rect* __restrict__ dyn_map, int32_t* __restrict__ ndyn_map,
                                                           sgs_rect* __restrict__ dyn_rm, int32_t* __restrict__ ndyn_rm, uint8_t* __restrict__ have_dyn_rm,
                                                           int32_t* __restrict__ status) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem_raw);   // [kMergeCap]
    float* srow = reinterpret_cast<float*>(keys + kMergeCap);                       // [keep_topk][6]
    __shared__ int s_n;
    const int f = blockIdx.x;
    if (threadIdx.x == 0) s_n = 0;
    __syncthreads();
    for (int c = 0; c < P.ncls - 1; ++c) {
        const int n = picked_n[f * (P.ncls - 1) + c];
        const unsigned long long* src = picked + ((int64_t)f * (P.ncls - 1) + c) * P.nms_topk;
        __shared__ int s_base;
        if (threadIdx.x == 0) { s_base = s_n; s_n = min(kMergeCap, s_n + n); }
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += blockDim.x)
            if (s_base + i < kMergeCap) keys[s_base + i] = src[i];
        __syncthreads();
    }
    const int n = s_n;
    int np2 = 1;
    while (np2 < n) np2 <<= 1;
    for (int i = n + threadIdx.x; i < np2; i += blockDim.x) keys[i] = ~0ull;
    if (n > 1) bitonic_sort_u64(keys, np2);
    __syncthreads();
    const int m = min(n, P.keep_topk);
    const float* lf = loc + (int64_t)f * P.nprior * 4;
    for (int i = threadIdx.x; i < m; i += blockDim.x) {
        const unsigned long long k = keys[i];
        const float4 b = decode_box(lf, prior, var, (int)(k & 0xffffu));
        float* r = srow + i * 6;
        r[0] = (float)(int)((k >> 16) & 0xffffu);
        r[1] = __uint_as_float(~(unsigned)(k >> 32));
        r[2] = b.x; r[3] = b.y; r[4] = b.z; r[5] = b.w;
    }
    __syncthreads();
    if (rows)
        for (int i = threadIdx.x; i < m * 6; i += blockDim.x) rows[(int64_t)f * Q.rows_cap * 6 + i] = srow[i];
    if (threadIdx.x != 0) return;
    if (nrows) nrows[f] = m;
    int no = 0, nm = 0, nr = 0, nnp = 0, over = 0;                  // objects, person boxes (mapping / rejection), non-person objects
    for (int i = 0; i < m; ++i) {
        const float* v = srow + i * 6;
        const int lab = (int)v[0];
        if (!(v[1] > Q.det_thr || (v[1] > Q.dyn_thr && lab == Q.person))) continue;
        float c[4];
        for (int q = 0; q < 4; ++q) c[q] = __fdiv_rn(fminf(fmaxf(__fmul_rn(v[2 + q], Q.target), 0.f), __fsub_rn(Q.target, 1.f)), Q.target);
        const float x1 = __fmul_rn(c[0], (float)Q.img_w), y1 = __fmul_rn(c[1], (float)Q.img_h);
        const float x2 = __fmul_rn(c[2], (float)Q.img_w), y2 = __fmul_rn(c[3], (float)Q.img_h);
        sgs_rect r;
        r.x = x1; r.y = y1; r.w = __fsub_rn(x2, x1); r.h = __fsub_rn(y2, y1);
        if (objects) { sgs_object2d o; o.id = lab; o.prob = v[1]; o.rect = r; objects[(int64_t)f * Q.rows_cap + no] = o; }
        ++no;
        if (lab == Q.person) {
            if (nm < Q.max_boxes) { if (dyn_map) dyn_map[(int64_t)f * Q.max_boxes + nm] = r; ++nm; } else over = 1;
            if ((double)v[1] > 0.2) {                                  // `object2d.prob > 0.2`: float against a double literal (Detector2D.cc:78)
                if (nr < Q.max_boxes) { if (dyn_rm) dyn_rm[(int64_t)f * Q.max_boxes + nr] = r; ++nr; } else over = 1;
            }
        } else ++nnp;
    }
    if (nobjects) nobjects[f] = no;
    if (ndyn_map) ndyn_map[f] = nm;
    if (ndyn_rm) ndyn_rm[f] = nr;
    // Frame.cc:482-491 copies the detector's flag only when mvObjects2D (the NON-person objects, Detector2D.cc:84-85) is not empty; otherwise the Frame
    // member stays uninitialised (include/Frame.h:112) -- defined here as false (DESIGN.md, quirk Q12) -- and bPreFrameHavePotentialDynamicObj = false.
    if (have_dyn_rm) have_dyn_rm[f] = (nr > 0 && nnp > 0) ? 1 : 0;
    if (status) status[f] = over;
}

// ---------------------------------------------------------------------------------------------------------------- graph (host)
struct Layer {
    std::string type, name;
    std::vector<std::string> in, out;
    std::map<int, std::vector<double>> prm;
    std::vector<float> weight, bias, data;
    double p(int k, double d) const { auto it = prm.find(k); return it == prm.end() || it->second.empty() ? d : it->second[0]; }
    int pi(int k, int d) const { return (int)p(k, d); }
    const std::vector<double>* arr(int k) const { auto it = prm.find(k); return it == prm.end() ? nullptr : &it->second; }
};

struct Blob {
    std::string name;
    int dims = 0, c = 1, h = 1, w = 1;
    int64_t n = 0;
    int producer = -1;
    int root = -1;                 // blob whose storage this one aliases (Split / Flatten / Reshape outputs)
    bool is_const = false;
    bool hwc = false;              // 3-D blob stored [h][w][c] (every activation); Permute(3) outputs alias their input and are "native" again
    std::vector<float> cval;       // constant-folded value
    int buf = -1;                  // pool buffer of the root
    float* dev = nullptr;
};

enum OpKind { OP_CONV1X1, OP_CONV_DIRECT, OP_DWCONV, OP_ELTWISE, OP_CONCAT_COPY, OP_SOFTMAX };
struct EpiStepH { int op, src, rev; float a, b; int tblob; };
struct Op {
    OpKind kind;
    int layer = -1;
    int in = -1, out = -1;         // blob ids (roots resolved at launch)
    std::vector<EpiStepH> epi;
    ConvGeom g{};
    float* d_w = nullptr; float* d_b = nullptr;
    int64_t off = 0;               // concat offset (copy pieces, and convolutions that write straight into a concatenated buffer: `cat`)
    bool cat = false;
    tc::GemmPlan gp;               // OP_CONV1X1: split weights, tiling, weight tensor maps
    CUtensorMap map_in;            // OP_CONV1X1: the input activations [max_frames * H * W][Cin]
};

}  // namespace det
}  // namespace sgs

using namespace sgs;
using namespace sgs::det;

struct sgs_detector {
    explicit sgs_detector(int dev) : device(dev), res(dev) {}
    int device, max_frames = 0, flags = 0;
    HandleResources res;              // nothing in plan-only mode (flags bit 1)
    float det_thr = 0, dyn_thr = 0;
    int T = 300;
    std::vector<Layer> layers;
    std::vector<Blob> blobs;
    std::map<std::string, int> blob_id;
    std::vector<Op> ops;
    int input_blob = -1, loc_blob = -1, conf_blob = -1;
    DetOutParams dp{};
    std::vector<float*> pool;          // activation buffers (max_frames x size)
    std::vector<int64_t> pool_size;
    float* d_prior = nullptr; float* d_var = nullptr;
    unsigned long long* d_picked = nullptr; int32_t* d_picked_n = nullptr;
    // host-call scratch
    uint8_t* d_img = nullptr; size_t d_img_cap = 0;
    int* d_pre_tab = nullptr; int pre_w = 0, pre_h = 0;       // resize coefficient table of the last source geometry (preprocess_table_kernel)
    sgs_object2d* d_obj = nullptr; int32_t* d_cnt = nullptr;
    int last_frames = 0;
    // optional per-kernel timing (sgs_detector_set_profiling): events around every launch of a call, read back at the next call / by sgs_detector_kernel_times
    StageTimer timer;
};

namespace {

int root_of(const sgs_detector& D, int b) { while (D.blobs[b].root != b) b = D.blobs[b].root; return b; }

int parse_param(const char* path, std::vector<Layer>& layers) {
    std::ifstream fs(path);
    if (!fs) { set_error("sgs_detector_create: cannot open %s", path); return SGS_ERR_INVALID; }
    std::string line;
    long magic = 0; int nl = 0, nb = 0;
    if (!(fs >> magic) || magic != 7767517) { set_error("sgs_detector_create: %s is not an ncnn text param file", path); return SGS_ERR_INVALID; }
    fs >> nl >> nb;
    std::getline(fs, line);
    while (std::getline(fs, line)) {
        std::istringstream ss(line);
        Layer L; int nin = 0, nout = 0;
        if (!(ss >> L.type >> L.name >> nin >> nout)) continue;
        if (nin < 0 || nout < 0 || nin > 64 || nout > 64) { set_error("sgs_detector_create: layer %s declares %d inputs / %d outputs", L.name.c_str(), nin, nout); return SGS_ERR_INVALID; }
        L.in.resize(nin); L.out.resize(nout);
        for (auto& s : L.in) ss >> s;
        for (auto& s : L.out) ss >> s;
        std::string kv;
        while (ss >> kv) {
            const size_t eq = kv.find('=');
            if (eq == std::string::npos) { set_error("sgs_detector_create: bad token '%s' in layer %s", kv.c_str(), L.name.c_str()); return SGS_ERR_INVALID; }
            int key = atoi(kv.substr(0, eq).c_str());
            std::string val = kv.substr(eq + 1);
            std::vector<double> v;
            if (key <= -23300) {                                  // array: -23300-id=count,v0,v1,...
                key = -(key + 23300);
                std::istringstream vs(val); std::string tok; bool first = true; size_t cnt = 0;
                while (std::getline(vs, tok, ',')) { if (first) { const int c = atoi(tok.c_str()); if (c < 0 || c > 4096) { set_error("sgs_detector_create: array of %d values in layer %s", c, L.name.c_str()); return SGS_ERR_INVALID; } cnt = (size_t)c; first = false; } else v.push_back(atof(tok.c_str())); }
                v.resize(cnt);
            } else v.push_back(atof(val.c_str()));
            L.prm[key] = v;
        }
        layers.push_back(std::move(L));
    }
    if ((int)layers.size() != nl) { set_error("sgs_detector_create: %s declares %d layers, %zu read", path, nl, layers.size()); return SGS_ERR_INVALID; }
    return SGS_OK;
}

int load_bin(const char* path, std::vector<Layer>& layers) {
    std::ifstream fs(path, std::ios::binary);
    if (!fs) { set_error("sgs_detector_create: cannot open %s", path); return SGS_ERR_INVALID; }
    std::vector<char> buf((std::istreambuf_iterator<char>(fs)), std::istreambuf_iterator<char>());
    size_t off = 0;
    auto take = [&](std::vector<float>& dst, size_t n) -> bool {
        if (off + 4 * n > buf.size()) return false;
        dst.resize(n); if (n) memcpy(dst.data(), buf.data() + off, 4 * n); off += 4 * n; return true;      // n == 0 (a hostile count): no null pointers into memcpy
    };
    for (auto& L : layers) {
        if (L.type == "Convolution" || L.type == "ConvolutionDepthWise") {
            uint32_t tag = 1;
            if (off + 4 <= buf.size()) memcpy(&tag, buf.data() + off, 4);
            off += 4;
            if (tag != 0) { set_error("sgs_detector_create: layer %s: only raw float32 weights are supported (storage tag %#x)", L.name.c_str(), tag); return SGS_ERR_UNSUPPORTED; }
            if (L.pi(6, 0) < 0 || L.pi(0, 0) < 0 || !take(L.weight, (size_t)L.pi(6, 0))) { set_error("sgs_detector_create: %s truncated at layer %s", path, L.name.c_str()); return SGS_ERR_INVALID; }
            if (L.pi(5, 0) && !take(L.bias, (size_t)L.pi(0, 0))) { set_error("sgs_detector_create: %s truncated at layer %s", path, L.name.c_str()); return SGS_ERR_INVALID; }
        } else if (L.type == "MemoryData") {
            const size_t n = (size_t)std::max(1, L.pi(0, 0)) * std::max(1, L.pi(1, 0)) * std::max(1, L.pi(2, 0));
            if (!take(L.data, n)) { set_error("sgs_detector_create: %s truncated at layer %s", path, L.name.c_str()); return SGS_ERR_INVALID; }
        }
    }
    if (off != buf.size()) { set_error("sgs_detector_create: %s has %zu bytes, the graph consumes %zu", path, buf.size(), off); return SGS_ERR_INVALID; }
    return SGS_OK;
}

// ncnn PriorBox: row 0 = corner boxes (normalised), row 1 = variances.  Keys 14/15 (mmdetection-style stride / centre) are both set in the
// reference model: stride = ceil(image / feature) and first centre = offset * (stride - 1).
void prior_box(const Layer& L, int fw, int fh, int iw, int ih, std::vector<float>& out) {
    const std::vector<double> none;
    const auto& mins = L.arr(0) ? *L.arr(0) : none; const auto& maxs = L.arr(1) ? *L.arr(1) : none; const auto& ars = L.arr(2) ? *L.arr(2) : none;
    const float var[4] = {(float)L.p(3, 0.1), (float)L.p(4, 0.1), (float)L.p(5, 0.2), (float)L.p(6, 0.2)};
    const int flip = L.pi(7, 1), clip = L.pi(8, 0);
    int image_w = L.pi(9, 0), image_h = L.pi(10, 0);
    if (image_w == -233) image_w = iw;
    if (image_h == -233) image_h = ih;
    float step_w = (float)L.p(11, -233.0), step_h = (float)L.p(12, -233.0);
    if (step_w == -233.f) step_w = (float)image_w / (float)fw;
    if (step_h == -233.f) step_h = (float)image_h / (float)fh;
    const float offset = (float)L.p(13, 0.0);
    if (L.pi(14, 0)) { step_w = (float)std::ceil((double)image_w / fw); step_h = (float)std::ceil((double)image_h / fh); }
    const int centre_mm = L.pi(15, 0);
    std::vector<float> box;
    const float fiw = (float)image_w, fih = (float)image_h;
    for (int i = 0; i < fh; ++i)
        for (int j = 0; j < fw; ++j) {
            volatile float cx, cy;
            if (centre_mm) { cx = offset * (step_w - 1.f) + (float)j * step_w; cy = offset * (step_h - 1.f) + (float)i * step_h; }
            else { cx = offset * step_w + (float)j * step_w; cy = offset * step_h + (float)i * step_h; }
            auto put = [&](float bw, float bh) {
                volatile float hw = bw * 0.5f, hh = bh * 0.5f;
                box.push_back((cx - hw) / fiw); box.push_back((cy - hh) / fih); box.push_back((cx + hw) / fiw); box.push_back((cy + hh) / fih);
            };
            for (size_t k = 0; k < mins.size(); ++k) {
                const float mn = (float)mins[k];
                put(mn, mn);
                if (!maxs.empty()) { const float s = (float)std::sqrt((double)(mn * (float)maxs[k])); put(s, s); }
                for (double ard : ars) {
                    const float r = (float)std::sqrt((double)(float)ard);
                    const float bw = mn * r, bh = mn / r;
                    put(bw, bh);
                    if (flip) put(bh, bw);
                }
            }
        }
    if (clip) for (auto& v : box) v = std::min(std::max(v, 0.f), 1.f);
    out = box;
    for (size_t i = 0; i < box.size() / 4; ++i) for (int q = 0; q < 4; ++q) out.push_back(var[q]);
}

bool is_eltwise(const Layer& L) { return L.type == "ReLU" || L.type == "Clip" || L.type == "BinaryOp"; }

int upload(sgs_detector* D, const std::vector<float>& h, float** d) {
    *d = nullptr;
    if (h.empty() || (D->flags & 2)) return SGS_OK;
    SGS_CUDA_TRY(D->res.alloc(d, h.size() * sizeof(float)));
    SGS_CUDA_TRY(cudaMemcpy(*d, h.data(), h.size() * sizeof(float), cudaMemcpyHostToDevice));
    return SGS_OK;
}

// ---- graph builder.  sgs_detector_create runs wire_graph, infer_shapes, schedule and plan_pool in this order, then allocate unless the handle is
// plan-only.

// Which blobs each layer reads and writes, and which layers read each blob: set up once from the layer list, read by every later step.
struct Wiring {
    std::vector<std::vector<int>> in, out;     // blob ids, per layer
    std::vector<std::vector<int>> readers;     // layer indices, per blob
};

int wire_graph(sgs_detector* D, Wiring& w) {
    auto& Ls = D->layers;
    auto& B = D->blobs;
    auto blob = [&](const std::string& n) -> int {
        auto it = D->blob_id.find(n);
        if (it != D->blob_id.end()) return it->second;
        Blob b; b.name = n; b.root = (int)B.size();
        B.push_back(b); D->blob_id[n] = (int)B.size() - 1;
        return (int)B.size() - 1;
    };
    w.in.assign(Ls.size(), {});
    w.out.assign(Ls.size(), {});
    for (size_t i = 0; i < Ls.size(); ++i) {
        for (auto& n : Ls[i].in) {
            if (!D->blob_id.count(n)) { set_error("sgs_detector_create: layer %s reads undefined blob %s", Ls[i].name.c_str(), n.c_str()); return SGS_ERR_INVALID; }
            w.in[i].push_back(blob(n));
        }
        for (auto& n : Ls[i].out) { const int b = blob(n); B[b].producer = (int)i; w.out[i].push_back(b); }
    }
    w.readers.assign(B.size(), {});
    for (size_t i = 0; i < Ls.size(); ++i) for (int b : w.in[i]) w.readers[b].push_back((int)i);
    return SGS_OK;
}

// ---- shapes, aliases and constants
void set3(Blob& b, int c, int h, int w) { b.dims = 3; b.c = c; b.h = h; b.w = w; b.n = (int64_t)c * h * w; }

int infer_conv(sgs_detector* D, const Wiring& w, int i) {
    const Layer& L = D->layers[i];
    const Blob& s = D->blobs[w.in[i][0]];
    const int k = L.pi(1, 1), dil = L.pi(2, 1), st = L.pi(3, 1), pad = L.pi(4, 0), cout = L.pi(0, 0);
    if (s.dims != 3 || L.pi(11, k) != k || L.pi(12, dil) != dil || L.pi(13, st) != st || L.pi(14, pad) != pad || pad < 0) {
        set_error("sgs_detector_create: layer %s: only square kernels with symmetric explicit padding are supported", L.name.c_str()); return SGS_ERR_UNSUPPORTED; }
    const int oh = (s.h + 2 * pad - dil * (k - 1) - 1) / st + 1, ow = (s.w + 2 * pad - dil * (k - 1) - 1) / st + 1;
    Blob& o = D->blobs[w.out[i][0]];
    set3(o, cout, oh, ow);
    o.hwc = true;
    if (!s.hwc) { set_error("sgs_detector_create: layer %s convolves a blob that is not an activation map", L.name.c_str()); return SGS_ERR_UNSUPPORTED; }
    const bool dw = L.type == "ConvolutionDepthWise";
    const int group = dw ? L.pi(7, 1) : 1;
    if (dw && !(group == s.c && cout == s.c && cout <= 65535 && dil == 1 && (k == 3 || k == 5) && (st == 1 || st == 2))) { set_error("sgs_detector_create: layer %s: grouped convolution other than depth-wise 3x3/5x5 with stride 1/2 is not supported", L.name.c_str()); return SGS_ERR_UNSUPPORTED; }
    const int64_t expect = dw ? (int64_t)cout * k * k : (int64_t)cout * s.c * k * k;
    if ((int64_t)L.weight.size() != expect) { set_error("sgs_detector_create: layer %s: weight size %zu, expected %lld", L.name.c_str(), L.weight.size(), (long long)expect); return SGS_ERR_INVALID; }
    return SGS_OK;
}

int infer_detection_output(sgs_detector* D, const Wiring& w, int i) {
    const Layer& L = D->layers[i];
    auto& B = D->blobs;
    if (w.in[i].size() != 3 || !B[w.in[i][2]].is_const) { set_error("sgs_detector_create: DetectionOutput %s: expects location, confidence and constant prior boxes", L.name.c_str()); return SGS_ERR_UNSUPPORTED; }
    const Blob& pr = B[w.in[i][2]];
    DetOutParams& P = D->dp;
    P.ncls = L.pi(0, 0); P.nms_thr = (float)L.p(1, 0.05); P.nms_topk = L.pi(2, 300); P.keep_topk = L.pi(3, 100); P.conf_thr = (float)L.p(4, 0.5);
    P.nprior = pr.w / 4;
    D->loc_blob = w.in[i][0]; D->conf_blob = w.in[i][1];
    if (B[D->loc_blob].n != (int64_t)P.nprior * 4 || B[D->conf_blob].n != (int64_t)P.nprior * P.ncls || P.ncls < 2 || P.ncls > 256 || P.nprior > kDetSortCap ||
        P.nms_topk < 1 || P.nms_topk > 1024 || P.keep_topk < 1 || P.keep_topk > 1024 || (int64_t)(P.ncls - 1) * P.nms_topk > kMergeCap) {
        set_error("sgs_detector_create: DetectionOutput %s: sizes outside what the kernels take (priors %d of at most %d, classes %d)", L.name.c_str(), P.nprior, kDetSortCap, P.ncls); return SGS_ERR_UNSUPPORTED; }
    std::vector<float> pb(pr.cval.begin(), pr.cval.begin() + pr.w), vr(pr.cval.begin() + pr.w, pr.cval.end());
    int rc = upload(D, pb, &D->d_prior); if (rc) return rc;
    rc = upload(D, vr, &D->d_var); if (rc) return rc;
    Blob& o = B[w.out[i][0]]; o.dims = 2; o.h = P.keep_topk; o.w = 6; o.n = 0;
    return SGS_OK;
}

// Every blob's shape for the fixed input; Split / Permute(3) / Flatten / Reshape outputs become aliases (root), constant sub-graphs are folded.
int infer_shapes(sgs_detector* D, const Wiring& w) {
    auto& B = D->blobs;
    for (size_t i = 0; i < D->layers.size(); ++i) {
        const Layer& L = D->layers[i];
        auto in0 = [&]() -> Blob& { return B[w.in[i][0]]; };
        int rc = SGS_OK;
        if (L.type == "Input") { set3(B[w.out[i][0]], 3, D->T, D->T); B[w.out[i][0]].hwc = true; D->input_blob = w.out[i][0]; }
        else if (L.type == "MemoryData") {
            Blob& o = B[w.out[i][0]];
            o.dims = 1; o.w = (int)L.data.size(); o.n = o.w; o.is_const = true; o.cval = L.data;
            if (L.pi(1, 0) > 0 || L.pi(2, 0) > 0 || o.n != 1) { set_error("sgs_detector_create: MemoryData %s: only scalar constants are supported", L.name.c_str()); return SGS_ERR_UNSUPPORTED; }
        } else if (L.type == "Split") {
            for (int o : w.out[i]) { Blob& ob = B[o]; const Blob& s = in0(); ob.dims = s.dims; ob.c = s.c; ob.h = s.h; ob.w = s.w; ob.n = s.n; ob.root = w.in[i][0]; ob.is_const = s.is_const; ob.cval = s.cval; ob.hwc = s.hwc; }
        } else if (L.type == "Convolution" || L.type == "ConvolutionDepthWise") rc = infer_conv(D, w, (int)i);
        else if (is_eltwise(L)) {
            const Blob& s = in0(); Blob& o = B[w.out[i][0]];
            o.dims = s.dims; o.c = s.c; o.h = s.h; o.w = s.w; o.n = s.n; o.hwc = s.hwc;
            if (L.type == "BinaryOp") {
                // the kernels read a tensor operand at the value's flat [h][w][c] index: only an operand of the value's own shape and layout is that
                // element (ncnn would broadcast other shapes; a flattened or permuted view orders the elements differently)
                const Blob& t = B[w.in[i][1]];
                const bool same = t.dims == s.dims && t.c == s.c && t.h == s.h && t.w == s.w && t.hwc == s.hwc;
                if (s.is_const || !(t.is_const ? t.n == 1 : same)) { set_error("sgs_detector_create: BinaryOp %s: unsupported operand shapes", L.name.c_str()); return SGS_ERR_UNSUPPORTED; }
                if (!t.is_const && root_of(*D, w.in[i][0]) == root_of(*D, w.in[i][1])) {
                    set_error("sgs_detector_create: BinaryOp %s: both operands are the same blob (x op x is not supported)", L.name.c_str()); return SGS_ERR_UNSUPPORTED; }
                if (L.pi(0, 0) < 0 || L.pi(0, 0) > 3) { set_error("sgs_detector_create: BinaryOp %s: op_type %d not supported", L.name.c_str(), L.pi(0, 0)); return SGS_ERR_UNSUPPORTED; }
            }
        }
        else if (L.type == "Permute") {
            const Blob& s = in0();
            if (s.dims != 3 || L.pi(0, 0) != 3 || !s.hwc) { set_error("sgs_detector_create: Permute %s: only order_type 3 on 3-D activation maps is supported", L.name.c_str()); return SGS_ERR_UNSUPPORTED; }
            set3(B[w.out[i][0]], s.h, s.w, s.c);
            B[w.out[i][0]].root = w.in[i][0];                 // (c,h,w) -> (h,w,c) is how the activation is stored already: an alias, in ncnn's "native" order from here on
        } else if (L.type == "Flatten") {
            const Blob& s = in0(); Blob& o = B[w.out[i][0]];
            if (s.hwc && s.c > 1 && s.h * s.w > 1) { set_error("sgs_detector_create: Flatten %s of an un-permuted activation map is not supported", L.name.c_str()); return SGS_ERR_UNSUPPORTED; }
            o.dims = 1; o.w = (int)s.n; o.n = s.n; o.root = w.in[i][0]; o.is_const = s.is_const; o.cval = s.cval;
        } else if (L.type == "Reshape") {
            const Blob& s = in0(); Blob& o = B[w.out[i][0]];
            const int rw = L.pi(0, -233), rh = L.pi(1, -233);
            if (rw <= 0 || L.pi(2, -233) != -233 || (s.hwc && s.c > 1 && s.h * s.w > 1)) { set_error("sgs_detector_create: Reshape %s: unsupported target", L.name.c_str()); return SGS_ERR_UNSUPPORTED; }
            if (rh == -233) { o.dims = 1; o.w = rw; } else { o.dims = 2; o.w = rw; o.h = rh == -1 ? (int)(s.n / rw) : rh; }
            o.n = s.n; o.root = w.in[i][0];
            if ((int64_t)o.w * o.h != s.n) { set_error("sgs_detector_create: Reshape %s: element count mismatch", L.name.c_str()); return SGS_ERR_INVALID; }
        } else if (L.type == "Concat") {
            Blob& o = B[w.out[i][0]];
            const Blob& f = in0();
            const int axis = L.pi(0, 0);
            bool all_const = true; int64_t total = 0;
            for (int b : w.in[i]) { all_const = all_const && B[b].is_const; total += B[b].n; }
            if (f.dims == 1 && axis == 0) { o.dims = 1; o.w = (int)total; o.n = total; }
            else if (f.dims == 2 && axis == 1 && all_const) {       // rows concatenated along w (prior boxes)
                o.dims = 2; o.h = f.h; int ow = 0; for (int b : w.in[i]) ow += B[b].w; o.w = ow; o.n = (int64_t)o.h * ow;
            } else { set_error("sgs_detector_create: Concat %s: unsupported axis / rank", L.name.c_str()); return SGS_ERR_UNSUPPORTED; }
            if (all_const) {
                o.is_const = true; o.cval.resize(o.n);
                if (o.dims == 1) { int64_t off = 0; for (int b : w.in[i]) { std::copy(B[b].cval.begin(), B[b].cval.end(), o.cval.begin() + off); off += B[b].n; } }
                else for (int r = 0; r < o.h; ++r) { int64_t off = 0; for (int b : w.in[i]) { std::copy(B[b].cval.begin() + (int64_t)r * B[b].w, B[b].cval.begin() + (int64_t)(r + 1) * B[b].w, o.cval.begin() + (int64_t)r * o.w + off); off += B[b].w; } }
            }
        } else if (L.type == "Softmax") {
            const Blob& s = in0(); Blob& o = B[w.out[i][0]];
            if (s.dims != 2 || L.pi(0, 0) != 1) { set_error("sgs_detector_create: Softmax %s: only the inner axis of a 2-D blob is supported", L.name.c_str()); return SGS_ERR_UNSUPPORTED; }
            o.dims = 2; o.h = s.h; o.w = s.w; o.n = s.n;
        } else if (L.type == "PriorBox") {
            const Blob& fm = B[w.in[i][0]]; const Blob& im = B[w.in[i][1]];
            Blob& o = B[w.out[i][0]];
            prior_box(L, fm.w, fm.h, im.w, im.h, o.cval);
            o.is_const = true; o.dims = 2; o.h = 2; o.w = (int)(o.cval.size() / 2); o.n = (int64_t)o.cval.size();
        } else if (L.type == "DetectionOutput") rc = infer_detection_output(D, w, (int)i);
        else { set_error("sgs_detector_create: layer type %s (%s) is not supported", L.type.c_str(), L.name.c_str()); return SGS_ERR_UNSUPPORTED; }
        if (rc) return rc;
    }
    if (D->input_blob < 0 || D->loc_blob < 0) { set_error("sgs_detector_create: the graph has no Input / DetectionOutput layer"); return SGS_ERR_INVALID; }
    return SGS_OK;
}

// ---- scheduling: the kernel list, and which element-wise layers each kernel applies in its epilogue.  absorbed[l]: layer l is a step of an
// earlier kernel's tail and gets no kernel of its own.

// Layers reading blob b or any alias of it, in graph order (aliases never chain through compute layers).
std::vector<int> readers_of_root(const sgs_detector& D, const Wiring& w, int b) {
    std::vector<int> r; const int rb = root_of(D, b);
    for (size_t q = 0; q < D.blobs.size(); ++q)
        if (!D.blobs[q].is_const && root_of(D, (int)q) == rb)
            for (int l : w.readers[q]) { const std::string& t = D.layers[l].type; if (t != "Split" && t != "Flatten" && t != "Reshape" && t != "Permute") r.push_back(l); }
    std::sort(r.begin(), r.end());
    return r;
}

// Layer li as one step of a tail whose running value is vblob, in the kernel of layer owner_layer; false when it cannot be one.  ReLU (slope 0) and
// Clip of the value are steps.  A BinaryOp is a step when the value is one operand (rev: the second) and the other is a scalar constant
// (SRC_SCALAR), the tail's start value start_blob when that is not the value itself (SRC_START; -1: no start value), or a tensor whose producer
// runs before the owner (SRC_TENSOR).  The value combined with itself is not a step.
bool step_of(const sgs_detector& D, const Wiring& w, int li, int vblob, int start_blob, int owner_layer, EpiStepH& st) {
    const Layer& L = D.layers[li];
    const auto& B = D.blobs;
    st = EpiStepH{0, SRC_SCALAR, 0, 0.f, 0.f, -1};
    if (L.type == "ReLU") { if (L.p(0, 0.0) != 0.0) return false; st.op = E_RELU; return root_of(D, w.in[li][0]) == root_of(D, vblob); }
    if (L.type == "Clip") { st.op = E_CLIP; st.a = (float)L.p(0, -3.4e38); st.b = (float)L.p(1, 3.4e38); return root_of(D, w.in[li][0]) == root_of(D, vblob); }
    if (L.type != "BinaryOp") return false;
    const int a = w.in[li][0], b = w.in[li][1];
    const bool va = root_of(D, a) == root_of(D, vblob), vb = !B[b].is_const && root_of(D, b) == root_of(D, vblob);
    if (!va && !vb) return false;
    st.op = L.pi(0, 0);
    st.rev = va ? 0 : 1;
    const int o = va ? b : a;
    if (B[o].is_const) { st.src = SRC_SCALAR; st.a = B[o].cval[0]; return true; }
    if (start_blob >= 0 && root_of(D, o) == root_of(D, start_blob) && root_of(D, o) != root_of(D, vblob)) { st.src = SRC_START; return true; }
    if (va && vb) return false;                                                 // x op x: infer_shapes refuses it, no kernel computes it
    if (B[root_of(D, o)].producer < owner_layer) { st.src = SRC_TENSOR; st.tblob = o; return true; }
    return false;
}

// The tail of the convolution owner_layer, whose output is out_blob.  The chain grows greedily: the next step is the first not yet absorbed
// element-wise reader (in graph order) of the running value that step_of takes, with out_blob as the start value, up to kMaxEpi steps.  The tail
// is the longest prefix of the chain whose intermediate blobs are read only inside the prefix, so that nothing needs a value the fused kernel does
// not store.  Marks its layers absorbed; returns the blob the tail's last step writes (out_blob for an empty tail).
int build_tail(const sgs_detector& D, const Wiring& w, std::vector<char>& absorbed, int owner_layer, int out_blob, std::vector<EpiStepH>& tail) {
    std::vector<int> chain_layers; std::vector<int> chain_blobs{out_blob};
    std::vector<EpiStepH> steps;
    int cur = out_blob;
    while ((int)steps.size() < kMaxEpi) {
        int next = -1; EpiStepH st{};
        for (int l : readers_of_root(D, w, cur)) {
            if (std::find(chain_layers.begin(), chain_layers.end(), l) != chain_layers.end() || !is_eltwise(D.layers[l]) || absorbed[l]) continue;
            if (step_of(D, w, l, cur, out_blob, owner_layer, st)) { next = l; break; }
        }
        if (next < 0) break;
        chain_layers.push_back(next); steps.push_back(st); cur = w.out[next][0]; chain_blobs.push_back(cur);
    }
    int best = 0;
    for (int m = 1; m <= (int)steps.size(); ++m) {
        bool ok = true;
        for (int j = 0; j < m && ok; ++j)
            for (int l : readers_of_root(D, w, chain_blobs[j]))
                if (std::find(chain_layers.begin(), chain_layers.begin() + m, l) == chain_layers.begin() + m) { ok = false; break; }
        if (ok) best = m;
    }
    tail.assign(steps.begin(), steps.begin() + best);
    for (int j = 0; j < best; ++j) absorbed[chain_layers[j]] = 1;
    return chain_blobs[best];
}

// Extends a stand-alone element-wise kernel (layer owner_layer, its output out_blob) by the layers that follow it: while the running value has one
// reader, and that reader is a not yet absorbed element-wise layer that step_of takes, it becomes the next step, up to kMaxEpi steps in all.  With
// one reader per value no step ever needs to be cut off again, unlike build_tail.  No step is SRC_START: the start value of a stand-alone chain
// is its input, which SRC_START does not mean.  Returns the blob the last step writes.
int eltwise_chain(const sgs_detector& D, const Wiring& w, std::vector<char>& absorbed, int owner_layer, int out_blob, std::vector<EpiStepH>& steps) {
    int cur = out_blob;
    EpiStepH st{};
    while ((int)steps.size() < kMaxEpi) {
        auto cs = readers_of_root(D, w, cur);
        if (cs.size() != 1 || !is_eltwise(D.layers[cs[0]]) || absorbed[cs[0]] || !step_of(D, w, cs[0], cur, -1, owner_layer, st)) break;
        absorbed[cs[0]] = 1; steps.push_back(st); cur = w.out[cs[0]][0];
    }
    return cur;
}

// The tail kinds the kernels run as straight-line code (Epi::kind); each reproduces the generic loop operation for operation (same operand
// order, one rounding each).
int epi_kind(const std::vector<EpiStepH>& h) {
    const int n = (int)h.size();
    auto is = [&](int i, int op, int src) { return h[i].op == op && (op >= E_CLIP || h[i].src == src); };
    if (n == 0) return EK_NONE;
    if (n == 1 && h[0].op == E_RELU) return EK_RELU;
    if (n == 1 && h[0].op == E_CLIP) return EK_CLIP;
    if (n == 1 && is(0, E_ADD, SRC_TENSOR)) return EK_ADD_T;                  // addition commutes: rev is irrelevant
    if (n == 4 && is(0, E_ADD, SRC_SCALAR) && h[1].op == E_CLIP && is(2, E_MUL, SRC_START) && is(3, E_DIV, SRC_SCALAR) && !h[3].rev && h[3].a == 6.0f) return EK_HSWISH;
    if (n == 5 && is(0, E_ADD, SRC_SCALAR) && h[1].op == E_CLIP && is(2, E_DIV, SRC_SCALAR) && !h[2].rev && h[2].a == 6.0f && is(3, E_MUL, SRC_TENSOR) && is(4, E_ADD, SRC_TENSOR))
        return EK_SE_TAIL;
    if (n == 4 && is(0, E_ADD, SRC_SCALAR) && h[1].op == E_CLIP && is(2, E_DIV, SRC_SCALAR) && !h[2].rev && h[2].a == 6.0f && is(3, E_MUL, SRC_TENSOR)) return EK_SE_MUL;
    return EK_GENERIC;
}

// The SSD head outputs.  When every piece is the (permuted, flattened) [h][w][c] output of a convolution that nothing else reads, and none of those
// convolutions' tails reads a tensor, the convolutions write their rows straight into the concatenated buffer; otherwise, and in diagnostic mode,
// each piece is copied by a kernel of its own.
void schedule_concat(sgs_detector* D, const Wiring& w, int i) {
    std::vector<int> prod;
    bool direct = !(D->flags & 1);
    for (int b : w.in[i]) {
        const int r = root_of(*D, b);
        int q = -1;
        for (size_t o = 0; o < D->ops.size(); ++o) if (root_of(*D, D->ops[o].out) == r && !D->ops[o].cat) q = (int)o;
        const auto cs = readers_of_root(*D, w, r);
        bool ok = q >= 0 && (D->ops[q].kind == OP_CONV1X1 || D->ops[q].kind == OP_CONV_DIRECT) && cs.size() == 1 && cs[0] == i && D->blobs[r].hwc;
        if (ok) for (auto& st : D->ops[q].epi) if (st.src == SRC_TENSOR) ok = false;
        direct = direct && ok;
        prod.push_back(q);
    }
    int64_t off = 0;
    for (size_t j = 0; j < w.in[i].size(); ++j) {
        const int b = w.in[i][j];
        if (direct) { Op& po = D->ops[prod[j]]; po.out = w.out[i][0]; po.cat = true; po.off = off; }
        else { Op op; op.kind = OP_CONCAT_COPY; op.layer = i; op.in = b; op.out = w.out[i][0]; op.off = off; D->ops.push_back(op); }
        off += D->blobs[b].n;
    }
}

// The kernel list in graph order.  A convolution takes the tail build_tail finds; an element-wise layer no tail took gets a kernel of its own on
// whichever operand step_of takes as the running value (the first, else a tensor second), extended by eltwise_chain.  Diagnostic mode (flags
// bit 0) fuses nothing: one kernel per computing layer.
int schedule(sgs_detector* D, const Wiring& w) {
    const bool diag = D->flags & 1;
    std::vector<char> absorbed(D->layers.size(), 0);
    for (int i = 0; i < (int)D->layers.size(); ++i) {
        const Layer& L = D->layers[i];
        const bool conv = L.type == "Convolution" || L.type == "ConvolutionDepthWise";
        if (absorbed[i] || !(conv || is_eltwise(L) || L.type == "Concat" || L.type == "Softmax")) continue;
        Op op; op.layer = i; op.in = w.in[i][0]; op.out = w.out[i][0];
        if (conv) {
            const Blob& s = D->blobs[op.in]; const Blob& o = D->blobs[op.out];
            op.g = ConvGeom{s.c, o.c, s.h, s.w, o.h, o.w, L.pi(1, 1), L.pi(3, 1), L.pi(4, 0), L.pi(2, 1)};
            if (L.type == "ConvolutionDepthWise") op.kind = OP_DWCONV;
            else op.kind = (op.g.k == 1 && op.g.stride == 1 && op.g.pad == 0 && s.c % 4 == 0) ? OP_CONV1X1 : OP_CONV_DIRECT;
            if (!diag) op.out = build_tail(*D, w, absorbed, i, op.out, op.epi);
            int rc = SGS_OK;
            if (op.kind == OP_CONV1X1) {
                const int m_tiles = (int)std::min<int64_t>(((int64_t)D->max_frames * op.g.OH * op.g.OW + tc::kBM - 1) / tc::kBM, 1 << 30);      // pixel tiles of a full batch
                if (D->flags & 2) tc::plan_tiling(op.g.Cin, op.g.Cout, &op.gp, 0, m_tiles);
                else if (!tc::plan_weights(D->res, L.weight.data(), op.g.Cin, op.g.Cout, &op.gp, 0, m_tiles)) { set_error("sgs_detector_create: layer %s: the wgmma GEMM could not be set up (TMA tensor maps need a CUDA 12 driver; %s)", L.name.c_str(), cudaGetErrorString(cudaGetLastError())); return SGS_ERR_CUDA; }
            } else if (op.kind == OP_DWCONV) {                    // [c][ky][kx] -> [ky][kx][c]: channel vectors
                std::vector<float> wt(L.weight.size());
                const int kk = op.g.k * op.g.k;
                for (int c = 0; c < op.g.Cout; ++c) for (int t = 0; t < kk; ++t) wt[(size_t)t * op.g.Cout + c] = L.weight[(size_t)c * kk + t];
                rc = upload(D, wt, &op.d_w);
            } else rc = upload(D, L.weight, &op.d_w);
            if (rc) return rc;
            rc = upload(D, L.bias, &op.d_b); if (rc) return rc;
        } else if (is_eltwise(L)) {
            op.kind = OP_ELTWISE;
            EpiStepH st{};
            if (!step_of(*D, w, i, op.in, -1, i, st)) {
                if (L.type == "BinaryOp" && !D->blobs[w.in[i][1]].is_const) op.in = w.in[i][1];
                if (!step_of(*D, w, i, op.in, -1, i, st)) { set_error("sgs_detector_create: layer %s cannot be scheduled", L.name.c_str()); return SGS_ERR_UNSUPPORTED; }
            }
            op.epi.push_back(st);
            if (!diag) op.out = eltwise_chain(*D, w, absorbed, i, op.out, op.epi);
        } else if (L.type == "Concat") {
            if (!D->blobs[op.out].is_const) schedule_concat(D, w, i);
            continue;
        } else op.kind = OP_SOFTMAX;
        D->ops.push_back(op);
    }
    return SGS_OK;
}

// ---- activation pool.  A root's buffer is free again after the last kernel that reads it (or any alias); a free buffer is reused best-fit, or the
// largest one grows.  With every blob kept (flags bit 0 or 2) no buffer is ever reused.
void plan_pool(sgs_detector* D) {
    auto& B = D->blobs;
    const bool keep = D->flags & 5;
    std::vector<int> last(B.size(), -1);
    auto touch = [&](int b, int opi) { const int r = root_of(*D, b); last[r] = std::max(last[r], opi); };
    for (size_t q = 0; q < D->ops.size(); ++q) {
        touch(D->ops[q].in, (int)q);
        for (auto& s : D->ops[q].epi) if (s.src == SRC_TENSOR) touch(s.tblob, (int)q);
    }
    touch(D->loc_blob, 1 << 30); touch(D->conf_blob, 1 << 30); touch(D->input_blob, -1);
    std::vector<int> free_list;
    auto acquire = [&](int64_t n) -> int {
        int best = -1;
        for (size_t q = 0; q < free_list.size(); ++q)
            if (D->pool_size[free_list[q]] >= n && (best < 0 || D->pool_size[free_list[q]] < D->pool_size[free_list[best]])) best = (int)q;
        if (best >= 0) { const int b = free_list[best]; free_list.erase(free_list.begin() + best); return b; }
        if (!free_list.empty() && !keep) {        // grow the largest free buffer instead of adding one
            int big = 0;
            for (size_t q = 1; q < free_list.size(); ++q) if (D->pool_size[free_list[q]] > D->pool_size[free_list[big]]) big = (int)q;
            const int b = free_list[big]; free_list.erase(free_list.begin() + big); D->pool_size[b] = n; return b;
        }
        D->pool_size.push_back(n); return (int)D->pool_size.size() - 1;
    };
    B[root_of(*D, D->input_blob)].buf = acquire(B[D->input_blob].n);
    for (size_t q = 0; q < D->ops.size(); ++q) {
        const int r = root_of(*D, D->ops[q].out);
        if (B[r].buf < 0) B[r].buf = acquire(B[r].n);
        if (keep) continue;
        // buffers whose last reader is this kernel go back to the pool (after it: in/out never alias)
        for (size_t b = 0; b < B.size(); ++b)
            if (B[b].root == (int)b && B[b].buf >= 0 && last[b] == (int)q) free_list.push_back(B[b].buf);
        const int ri = root_of(*D, D->input_blob);
        if (q == 0 && last[ri] <= 0 && std::find(free_list.begin(), free_list.end(), B[ri].buf) == free_list.end()) free_list.push_back(B[ri].buf);
        if (last[r] < 0 && r != root_of(*D, D->loc_blob) && r != root_of(*D, D->conf_blob)) free_list.push_back(B[r].buf);   // never read: dead output
    }
}

// ---- device memory: the pool buffers (max_frames x size), every blob's address in them, the GEMMs' activation tensor maps, the DetectionOutput scratch.
int allocate(sgs_detector* D) {
    auto& B = D->blobs;
    D->pool.assign(D->pool_size.size(), nullptr);
    for (size_t q = 0; q < D->pool_size.size(); ++q) SGS_CUDA_TRY(D->res.alloc(&D->pool[q], (size_t)D->pool_size[q] * D->max_frames * sizeof(float)));
    for (auto& b : B) { const int r = root_of(*D, (int)(&b - &B[0])); if (B[r].buf >= 0) b.dev = D->pool[B[r].buf]; }
    for (auto& op : D->ops)                                   // the GEMMs' activation operand: [max_frames * H * W][Cin], rows past the batch are never stored
        if (op.kind == OP_CONV1X1 && !tc::encode_kmajor_map(&op.map_in, B[op.in].dev, (int64_t)D->max_frames * op.g.H * op.g.W, op.g.Cin, op.g.Cin, tc::kBM, op.gp.BK)) {
            set_error("sgs_detector_create: layer %s: cuTensorMapEncodeTiled failed", D->layers[op.layer].name.c_str()); return SGS_ERR_CUDA; }
    SGS_CUDA_TRY(D->res.alloc(&D->d_picked, (size_t)D->max_frames * (D->dp.ncls - 1) * D->dp.nms_topk * sizeof(unsigned long long)));
    SGS_CUDA_TRY(D->res.alloc(&D->d_picked_n, (size_t)D->max_frames * (D->dp.ncls - 1) * sizeof(int32_t)));
    SGS_CUDA_TRY(D->res.alloc(&D->d_obj, (size_t)D->dp.keep_topk * sizeof(sgs_object2d)));
    SGS_CUDA_TRY(D->res.alloc(&D->d_cnt, 4 * sizeof(int32_t)));
    return SGS_OK;
}

Epi make_epi(const sgs_detector* D, const std::vector<EpiStepH>& h) {
    Epi e; e.n = (int)h.size(); e.kind = epi_kind(h);
    for (int i = 0; i < e.n; ++i) {
        e.s[i].op = h[i].op; e.s[i].src = h[i].src; e.s[i].rev = h[i].rev; e.s[i].a = h[i].a; e.s[i].b = h[i].b;
        e.s[i].t = h[i].src == SRC_TENSOR ? D->blobs[h[i].tblob].dev : nullptr;
    }
    return e;
}

inline unsigned nblk(int64_t total) { return (unsigned)((total + 255) / 256); }

// Depth-wise convolutions: V = 4 channels per thread (float4) when Cout % 4 == 0, and then two output rows per thread on maps of 4 rows or more
// (the K + S input rows serve both: 1.5x / 1.67x fewer row loads for 3x3 / 5x5 at stride 1).
template <int K, int S>
void launch_dwconv(const float* in, const Op& op, float* out, int F, const Epi& epi, cudaStream_t st) {
    auto go = [&](auto kernel, int V, int YT) {
        const int64_t total = (int64_t)F * ((op.g.OH + YT - 1) / YT) * ((op.g.OW + 3) / 4) * (op.g.Cout / V);
        kernel<<<nblk(total), 256, 0, st>>>(in, op.d_w, op.d_b, out, op.g, total, epi);
    };
    if (op.g.Cout % 4) go(dwconv_kernel<K, S, 1, 1>, 1, 1);
    else if (op.g.OH >= 4) go(dwconv_kernel<K, S, 4, 2>, 4, 2);
    else go(dwconv_kernel<K, S, 4, 1>, 4, 1);
}

}  // namespace

extern "C" {

int sgs_detector_create(const char* param_path, const char* bin_path, int max_frames, float det_thr, float dyn_thr, int flags, int device,
                        sgs_detector** out) {
    if (!out || !param_path || !bin_path || max_frames < 1) { set_error("sgs_detector_create: bad argument"); return SGS_ERR_INVALID; }
    *out = nullptr;
    if (!(flags & 2)) SGS_CUDA_TRY(cudaSetDevice(device));
    auto D = std::make_unique<sgs_detector>(device);
    D->max_frames = max_frames; D->flags = flags; D->det_thr = det_thr; D->dyn_thr = dyn_thr;
    int rc = SGS_OK;
    try {                                              // malformed files must come back as a status, never as an exception through the C ABI
        rc = parse_param(param_path, D->layers);
        if (rc == SGS_OK) rc = load_bin(bin_path, D->layers);
        Wiring w;
        if (rc == SGS_OK) rc = wire_graph(D.get(), w);
        if (rc == SGS_OK) rc = infer_shapes(D.get(), w);
        if (rc == SGS_OK) rc = schedule(D.get(), w);
        if (rc == SGS_OK) plan_pool(D.get());
        if (rc == SGS_OK && !(flags & 2)) rc = allocate(D.get());
    } catch (const std::exception& ex) {
        set_error("sgs_detector_create: %s while reading %s / %s", ex.what(), param_path, bin_path);
        rc = SGS_ERR_INVALID;
    }
    if (rc == SGS_OK && !(flags & 2)) {
        cudaError_t e = cudaFuncSetAttribute(detout_merge_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kMergeCap * 8 + D->dp.keep_topk * 24);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(detout_class_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kDetSortCap * 8 + D->dp.nms_topk * 20);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(conv_small_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024);
        if (e != cudaSuccess) { set_error("sgs_detector_create: cudaFuncSetAttribute -> %s", cudaGetErrorString(e)); rc = SGS_ERR_CUDA; }
    }
    if (rc != SGS_OK) return rc;
    D->timer = StageTimer((int)D->ops.size() + 3);
    *out = D.release();
    return SGS_OK;
}

void sgs_detector_destroy(sgs_detector* D) { delete D; }

int sgs_detector_info(const sgs_detector* D, int* rows_cap, int* input_size, int* num_layers, int* num_kernels) {
    if (!D) { set_error("sgs_detector_info: NULL handle"); return SGS_ERR_INVALID; }
    if (rows_cap) *rows_cap = D->dp.keep_topk;
    if (input_size) *input_size = D->T;
    if (num_layers) *num_layers = (int)D->layers.size();
    if (num_kernels) *num_kernels = (int)D->ops.size() + 3;
    return SGS_OK;
}

int sgs_detector_set_profiling(sgs_detector* D, int enable) {
    if (!D || (D->flags & 2)) { set_error("sgs_detector_set_profiling: NULL or plan-only handle"); return SGS_ERR_INVALID; }
    SGS_CUDA_TRY(cudaSetDevice(D->device));
    SGS_CUDA_TRY(D->timer.enable(D->res, enable != 0));
    return SGS_OK;
}

int sgs_detector_kernel_times(sgs_detector* D, double* ms_total, int cap, int* nkernels, int* ncalls) {
    if (!D || !nkernels || !ncalls) { set_error("sgs_detector_kernel_times: NULL"); return SGS_ERR_INVALID; }
    const int nk = (int)D->ops.size() + 3;
    *nkernels = nk; *ncalls = 0;
    if (!D->timer.on()) return SGS_OK;
    SGS_CUDA_TRY(cudaSetDevice(D->device));
    D->timer.fold();        // a failed wait leaves the last call out of the totals
    *ncalls = D->timer.calls();
    if (ms_total) { if (cap < nk) { set_error("sgs_detector_kernel_times: %d entries needed", nk); return SGS_ERR_CAPACITY; } for (int i = 0; i < nk; ++i) ms_total[i] = D->timer.totals()[i]; }
    return SGS_OK;
}

int sgs_detector_detect_device(sgs_detector* D, const uint8_t* d_rgb, int64_t frame_stride, int pitch, int width, int height, int nframes,
                               float* d_rows, int32_t* d_nrows, sgs_object2d* d_objects, int32_t* d_nobjects, sgs_rect* d_dyn_map,
                               int32_t* d_ndyn_map, sgs_rect* d_dyn_rm, int32_t* d_ndyn_rm, uint8_t* d_have_dyn_rm, int max_boxes,
                               int32_t* d_status, void* stream) {
    if (D && (D->flags & 2)) { set_error("sgs_detector_detect_device: the handle is plan-only (flags bit 1)"); return SGS_ERR_UNSUPPORTED; }
    if (!D || !d_rgb || nframes < 1 || nframes > D->max_frames || nframes > 65535 || width < 2 || height < 2 || pitch < width * 3 || max_boxes < 0 ||
        ((d_dyn_map || d_dyn_rm) && max_boxes < 1)) {
        set_error("sgs_detector_detect_device: bad argument (nframes %d of max %d, %dx%d pitch %d)", nframes, D ? D->max_frames : 0, width, height, pitch);
        return SGS_ERR_INVALID;
    }
    SGS_CUDA_TRY(cudaSetDevice(D->device));
    cudaStream_t st = (cudaStream_t)stream;
    const int F = nframes, T = D->T;
    auto& B = D->blobs;
    StageTimer& timer = D->timer;
    timer.begin();
    int stage = 0;
    if (!D->d_pre_tab) SGS_CUDA_TRY(D->res.alloc(&D->d_pre_tab, (size_t)6 * T * sizeof(int)));
    if (D->pre_w != width || D->pre_h != height) {          // stream-ordered in front of the resize; calls on one handle are serial (they share the activation pool)
        preprocess_table_kernel<<<nblk(T), 256, 0, st>>>(width, height, T, D->d_pre_tab);
        D->pre_w = width; D->pre_h = height;
    }
    timer.mark(stage++, st);
    preprocess_kernel<<<dim3(nblk((int64_t)T * T), F), 256, 0, st>>>(d_rgb, frame_stride, pitch, T, D->d_pre_tab, 123.675f, 116.28f, 103.53f, B[D->input_blob].dev);
    for (const Op& op : D->ops) {
        timer.mark(stage++, st);
        const Blob& bi = B[op.in]; const Blob& bo = B[op.out];
        const Epi epi = make_epi(D, op.epi);
        switch (op.kind) {
        case OP_CONV1X1: {
            const int HW = op.g.OH * op.g.OW; const int64_t npix = (int64_t)F * HW;
            if (npix >= (1ll << 31) - 256) { set_error("sgs_detector_detect_device: batch too large for 32-bit pixel indices"); return SGS_ERR_UNSUPPORTED; }
            const int64_t fstride = op.cat ? bo.n : (int64_t)HW * op.g.Cout;
            bool launched = false;
            epi_dispatch(epi.kind, [&](auto kind) {
                launched = tc::launch_conv1x1_tc_map(op.gp, op.map_in, (int)npix, op.d_b, bo.dev, HW, fstride, op.cat ? op.off : 0, op.g.Cout, EpiFnK<decltype(kind)::value>{epi}, st);
            });
            if (!launched) {
                set_error("sgs_detector_detect_device: layer %s: GEMM launch failed (%s)", D->layers[op.layer].name.c_str(), cudaGetErrorString(cudaGetLastError())); return SGS_ERR_CUDA; }
            break;
        }
        case OP_CONV_DIRECT: {
            const size_t wbytes = (size_t)op.g.Cin * op.g.k * op.g.k * kCot * sizeof(float);
            if (wbytes > 96 * 1024) { set_error("sgs_detector_detect_device: layer %s: %zu bytes of weights per channel block do not fit shared memory", D->layers[op.layer].name.c_str(), wbytes); return SGS_ERR_UNSUPPORTED; }
            const int64_t fstride = op.cat ? bo.n : (int64_t)op.g.OH * op.g.OW * op.g.Cout;
            if (!op.cat && op.g.k == 3 && op.g.Cin == 3 && op.g.Cout == 16 && op.g.stride == 2 && op.g.pad == 1 && op.g.dil == 1) {
                conv_first_kernel<<<dim3(nblk((int64_t)op.g.OH * op.g.OW), F), 256, 0, st>>>(bi.dev, op.d_w, op.d_b, bo.dev, op.g, epi);
                break;
            }
            conv_small_kernel<<<dim3(nblk((int64_t)op.g.OH * op.g.OW), (op.g.Cout + kCot - 1) / kCot, F), 256, wbytes, st>>>(bi.dev, op.d_w, op.d_b, bo.dev, op.g, fstride,
                                                                                                                        op.cat ? op.off : 0, epi);
            break;
        }
        case OP_DWCONV: {
            if (op.g.k == 3) (op.g.stride == 1 ? launch_dwconv<3, 1> : launch_dwconv<3, 2>)(bi.dev, op, bo.dev, F, epi, st);
            else (op.g.stride == 1 ? launch_dwconv<5, 1> : launch_dwconv<5, 2>)(bi.dev, op, bo.dev, F, epi, st);
            break;
        }
        case OP_ELTWISE: {
            const int64_t total = (int64_t)F * bo.n;
            eltwise_kernel<<<nblk(total), 256, 0, st>>>(bi.dev, bo.dev, total, epi);
            break;
        }
        case OP_CONCAT_COPY: {
            const int64_t total = (int64_t)F * bi.n;
            concat_copy_kernel<<<nblk(total), 256, 0, st>>>(bi.dev, bi.n, bo.dev, bo.n, op.off, total);
            break;
        }
        case OP_SOFTMAX: {
            const int64_t rows = (int64_t)F * bo.h;
            softmax_rows_kernel<<<nblk(rows), 256, 0, st>>>(bi.dev, bo.dev, bo.w, rows);
            break;
        }
        }
    }
    const DetOutParams P = D->dp;
    timer.mark(stage++, st);
    detout_class_kernel<<<dim3(P.ncls - 1, F), 256, kDetSortCap * 8 + P.nms_topk * 20, st>>>(B[D->loc_blob].dev, B[D->conf_blob].dev, D->d_prior, D->d_var, P,
                                                                                                D->d_picked, D->d_picked_n);
    PostParams Q{D->det_thr, D->dyn_thr, (float)T, width, height, 15, P.keep_topk, max_boxes};
    timer.mark(stage++, st);
    detout_merge_kernel<<<F, 256, kMergeCap * 8 + P.keep_topk * 24, st>>>(B[D->loc_blob].dev, D->d_prior, D->d_var, P, D->d_picked, D->d_picked_n, Q, d_rows,
                                                                          d_nrows, d_objects, d_nobjects, d_dyn_map, d_ndyn_map, d_dyn_rm, d_ndyn_rm,
                                                                          d_have_dyn_rm, d_status);
    timer.end(st);
    SGS_CUDA_TRY(cudaGetLastError());
    D->last_frames = F;
    return SGS_OK;
}

int sgs_detect(sgs_detector* D, const uint8_t* rgb, int width, int height, int pitch, sgs_object2d* objects, int cap, int* n) {
    if (!D || !rgb || !n || (cap > 0 && !objects) || width < 2 || height < 2 || pitch < width * 3) { set_error("sgs_detect: bad argument"); return SGS_ERR_INVALID; }
    SGS_CUDA_TRY(cudaSetDevice(D->device));
    const int64_t bytes = (int64_t)pitch * height;
    SGS_CUDA_TRY(D->res.grow(&D->d_img, &D->d_img_cap, (size_t)bytes));
    SGS_CUDA_TRY(cudaMemcpy(D->d_img, rgb, (size_t)bytes, cudaMemcpyHostToDevice));
    int rc = sgs_detector_detect_device(D, D->d_img, bytes, pitch, width, height, 1, nullptr, nullptr, D->d_obj, D->d_cnt, nullptr, nullptr, nullptr, nullptr, nullptr, 0,
                                        nullptr, nullptr);
    if (rc != SGS_OK) return rc;
    int32_t cnt = 0;
    SGS_CUDA_TRY(cudaMemcpy(&cnt, D->d_cnt, sizeof(cnt), cudaMemcpyDeviceToHost));
    *n = cnt;
    if (cnt > cap) { set_error("sgs_detect: %d objects, capacity %d", cnt, cap); return SGS_ERR_CAPACITY; }
    if (cnt > 0) SGS_CUDA_TRY(cudaMemcpy(objects, D->d_obj, (size_t)cnt * sizeof(sgs_object2d), cudaMemcpyDeviceToHost));
    return SGS_OK;
}

int sgs_detector_describe(const sgs_detector* D, char* out, int64_t cap, int64_t* n) {
    if (!D || !n) { set_error("sgs_detector_describe: bad argument"); return SGS_ERR_INVALID; }
    static const char* kind[] = {"conv1x1", "conv", "dwconv", "eltwise", "concat", "softmax"};
    static const char* opn[] = {"add", "sub", "mul", "div", "clip", "relu"};
    std::ostringstream ss;
    int64_t pool_floats = 0;
    for (int64_t v : D->pool_size) pool_floats += v;
    ss << "layers " << D->layers.size() << " kernels " << D->ops.size() + 3 << " pool_buffers " << D->pool_size.size() << " pool_floats_per_frame " << pool_floats << "\n";
    for (const Op& op : D->ops) {
        const Blob& bi = D->blobs[op.in]; const Blob& bo = D->blobs[op.out];
        ss << kind[op.kind] << ' ' << D->layers[op.layer].name << " in " << bi.name << " buf " << D->blobs[root_of(*D, op.in)].buf << " out " << bo.name << " buf "
           << D->blobs[root_of(*D, op.out)].buf << " n " << bo.n;
        if (op.kind <= OP_DWCONV) ss << " geom " << op.g.Cin << 'x' << op.g.H << 'x' << op.g.W << "->" << op.g.Cout << 'x' << op.g.OH << 'x' << op.g.OW << " k" << op.g.k << " s" << op.g.stride << " p" << op.g.pad;
        if (op.kind <= OP_DWCONV && op.g.dil != 1) ss << " d" << op.g.dil;
        if (op.kind == OP_CONCAT_COPY || op.cat) ss << " off " << op.off;
        if (op.kind == OP_CONV1X1) ss << " tile " << op.gp.NT << "x" << op.gp.n_tiles << " kb " << op.gp.KB << "x" << op.gp.BK << " stages " << op.gp.stages << (op.gp.b_resident ? " wres" : "")
                                    << " smem " << op.gp.smem_bytes << " wgmma m64n" << op.gp.NT << "k8";
        for (const auto& s : op.epi) {
            ss << " | " << opn[s.op] << (s.rev ? "(rev)" : "");
            if (s.op <= E_DIV) { if (s.src == SRC_SCALAR) ss << ' ' << s.a; else if (s.src == SRC_START) ss << " start"; else ss << ' ' << D->blobs[s.tblob].name << " buf " << D->blobs[root_of(*D, s.tblob)].buf; }
            else if (s.op == E_CLIP) ss << ' ' << s.a << ' ' << s.b;
        }
        ss << "\n";
    }
    const std::string str = ss.str();
    *n = (int64_t)str.size() + 1;
    if (*n > cap) { set_error("sgs_detector_describe: %lld bytes, capacity %lld", (long long)*n, (long long)cap); return SGS_ERR_CAPACITY; }
    if (out) memcpy(out, str.c_str(), str.size() + 1);
    return SGS_OK;
}

int sgs_detector_blob(sgs_detector* D, const char* name, int frame, float* out, int64_t cap, int64_t* n) {
    if (!D || !name || !n) { set_error("sgs_detector_blob: bad argument"); return SGS_ERR_INVALID; }
    if (!(D->flags & 5)) { set_error("sgs_detector_blob: the handle keeps no blobs (flags bit 0 or 2)"); return SGS_ERR_UNSUPPORTED; }
    auto it = D->blob_id.find(name);
    if (it == D->blob_id.end()) { set_error("sgs_detector_blob: no blob named %s", name); return SGS_ERR_INVALID; }
    const Blob& b = D->blobs[it->second];
    if (b.is_const) {
        *n = (int64_t)b.cval.size();
        if (*n > cap) { set_error("sgs_detector_blob: %lld floats, capacity %lld", (long long)*n, (long long)cap); return SGS_ERR_CAPACITY; }
        if (out) memcpy(out, b.cval.data(), b.cval.size() * sizeof(float));
        return SGS_OK;
    }
    if (!b.dev || b.n == 0 || frame < 0 || frame >= D->last_frames) { set_error("sgs_detector_blob: blob %s is not materialised / bad frame", name); return SGS_ERR_INVALID; }
    *n = b.n;
    if (b.n > cap) { set_error("sgs_detector_blob: %lld floats, capacity %lld", (long long)b.n, (long long)cap); return SGS_ERR_CAPACITY; }
    SGS_CUDA_TRY(cudaSetDevice(D->device));
    SGS_CUDA_TRY(cudaDeviceSynchronize());
    if (b.hwc && b.dims == 3 && b.c > 1 && b.h * b.w > 1) {        // stored [h][w][c]; ncnn's order is [c][h][w]
        std::vector<float> tmp((size_t)b.n);
        SGS_CUDA_TRY(cudaMemcpy(tmp.data(), b.dev + (int64_t)frame * b.n, (size_t)b.n * sizeof(float), cudaMemcpyDeviceToHost));
        const int hw = b.h * b.w;
        for (int p = 0; p < hw; ++p) for (int c = 0; c < b.c; ++c) out[(size_t)c * hw + p] = tmp[(size_t)p * b.c + c];
        return SGS_OK;
    }
    SGS_CUDA_TRY(cudaMemcpy(out, b.dev + (int64_t)frame * b.n, (size_t)b.n * sizeof(float), cudaMemcpyDeviceToHost));
    return SGS_OK;
}

}  // extern "C"
