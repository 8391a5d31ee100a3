// lk_kernel.cu -- cv::calcOpticalFlowPyrLK as called by Frame::RmDynamicPointWithSemanticAndGeometry (src/Frame.cc:445):
// I = current gray, J = previous gray, window 21x21, 4 pyramid levels, <= 30 iterations or |delta|^2 <= 1e-4.
// Follows OpenCV video/lkpyramid.cpp: cv::pyrDown levels (bit-exact integers), Scharr derivatives of I (int16, zero outside the
// image), 14-bit fixed-point bilinear window extraction, float 2x2 solve.  Sums of integer products are accumulated EXACTLY
// (int32/int64) and rounded once, and every float step is an explicit round-to-nearest intrinsic, so the result equals the int64
// restatement tests/lk_exact.py bit for bit (tests/test_gpu_lk_exact.py); OpenCV accumulates the sums in float in SIMD order, so
// positions agree with it to ~1e-4 px, not bit-for-bit (tolerance stated in tests/test_gpu_lk.py).  status/err are not produced (the reference ignores them, quirk Q4); a level
// that fails leaves the running estimate untouched (SURVEY A10).
//
// Like buildOpticalFlowPyramid, every level is stored with a border of kLkPad pixels (REFLECT_101) and has a derivative image
// (dx | dy << 16, zero border), so the tracker reads windows straight through the image edge without any per-pixel border logic.
// One warp per point; the 21x21 window is tiled over the lanes (7x2 pixels each + one pixel of the last column) and lives in
// registers for the whole level; no shared memory.
#include <cuda_runtime.h>

#include <cstdint>
#include <memory>
#include <vector>

#include "host_stage.cuh"
#include "internal_launch.cuh"
#include "sgs_common.h"

namespace sgs {

constexpr int kWin = 21, kLkMaxLevel = 3, kLkMaxCount = 30;
static_assert(kLkMaxLevel + 1 == sizeof(LkPyramid::off) / sizeof(int64_t), "LkPyramid describes every level");
constexpr int kLkWarps = 4;

constexpr int kLkPad = 24;            // the window reaches 22 px past the image on every side

struct LkLevels {                     // pointers address pixel (0, 0) of frame 0 of each padded level
    const uint8_t* I[kLkMaxLevel + 1]; const uint8_t* J[kLkMaxLevel + 1]; const uint32_t* D[kLkMaxLevel + 1];
    int32_t w[kLkMaxLevel + 1], h[kLkMaxLevel + 1], pitch[kLkMaxLevel + 1];      // pitch in pixels, shared by image and derivative planes
    int64_t fstride[kLkMaxLevel + 1];                                            // pixels between frames
    int32_t max_level;
};

__device__ __forceinline__ int lk_refl(int i, int n) {
    while (i < 0 || i >= n) i = (i < 0) ? -i : 2 * (n - 1) - i;
    return i;
}

// cv::pyrDown, CV_8U: separable [1 4 6 4 1], exact integer sums, (v + 128) >> 8, BORDER_REFLECT_101.  The source is a padded level
// whose border is already filled, so the 5x5 taps need no border logic.  Four outputs per thread: source columns 8 tx - 4 .. 8 tx + 11
// arrive as four aligned words per row (pixel (0, 0) of a padded plane is 8-byte aligned, rows are 16-byte multiples).
__global__ void __launch_bounds__(256) lk_pyrdown_kernel(const uint8_t* __restrict__ src, int spitch, int64_t sfstride,
                                                         uint8_t* __restrict__ dst, int dw, int dh, int dpitch, int64_t dfstride) {
    const int tx = blockIdx.x * 32 + (threadIdx.x & 31), y = blockIdx.y * 8 + (threadIdx.x >> 5);
    const int x0 = 4 * tx;
    if (x0 >= dw || y >= dh) return;
    const uint8_t* S = src + (int64_t)blockIdx.z * sfstride + (int64_t)(2 * y - 2) * spitch + (2 * x0 - 4);
    int acc[4] = {0, 0, 0, 0};
#pragma unroll
    for (int r = 0; r < 5; ++r) {
        const uint32_t* row = reinterpret_cast<const uint32_t*>(S + (int64_t)r * spitch);       // 4-byte aligned (8 tx - 4 past an 8-aligned origin)
        const uint4 q = make_uint4(__ldg(row), __ldg(row + 1), __ldg(row + 2), __ldg(row + 3));
        int b[11];          // source columns 2 x0 - 2 .. 2 x0 + 8
        b[0] = (q.x >> 16) & 255; b[1] = q.x >> 24;
        b[2] = q.y & 255; b[3] = (q.y >> 8) & 255; b[4] = (q.y >> 16) & 255; b[5] = q.y >> 24;
        b[6] = q.z & 255; b[7] = (q.z >> 8) & 255; b[8] = (q.z >> 16) & 255; b[9] = q.z >> 24;
        b[10] = q.w & 255;
        const int wr = r == 2 ? 6 : (r == 1 || r == 3) ? 4 : 1;
#pragma unroll
        for (int i = 0; i < 4; ++i) acc[i] += (b[2 * i + 2] * 6 + (b[2 * i + 1] + b[2 * i + 3]) * 4 + b[2 * i] + b[2 * i + 4]) * wr;
    }
    uint8_t* D = dst + (int64_t)blockIdx.z * dfstride + (int64_t)y * dpitch + x0;
    if (x0 + 3 < dw) {
        *reinterpret_cast<uint32_t*>(D) = (uint32_t)((acc[0] + 128) >> 8) | ((uint32_t)((acc[1] + 128) >> 8) << 8) | ((uint32_t)((acc[2] + 128) >> 8) << 16) |
                                          ((uint32_t)((acc[3] + 128) >> 8) << 24);
    } else {
#pragma unroll
        for (int i = 0; i < 4; ++i) if (x0 + i < dw) D[i] = (uint8_t)((acc[i] + 128) >> 8);
    }
}

// Interior of a padded level: optional copy from an unpadded source (level 0; src == dst interior when cv::pyrDown already wrote it)
// and the Scharr derivatives (calcScharrDeriv: REFLECT_101 at the image edge) stored as dx | dy << 16.
//   t0(x) = 3 (s[y-1][x] + s[y+1][x]) + 10 s[y][x],  t1(x) = s[y+1][x] - s[y-1][x];  dx = t0(x+1) - t0(x-1),  dy = 3 (t1(x-1) + t1(x+1)) + 10 t1(x)
// kVec: four pixels per thread from aligned 32-bit loads (needs 4-byte aligned rows and w % 4 == 0); otherwise one pixel per thread.
template <bool kVec>
__global__ void __launch_bounds__(256) lk_interior_kernel(const uint8_t* __restrict__ src, int spitch, int64_t sfstride, uint8_t* dst, bool copy,
                                                          uint32_t* __restrict__ deriv, int w, int h, int pitch, int64_t fstride) {
    const int tx = blockIdx.x * 32 + (threadIdx.x & 31), Y = blockIdx.y * 8 + (threadIdx.x >> 5);
    const int X = kVec ? 4 * tx : tx;
    if (X >= w || Y >= h) return;
    const uint8_t* S = src + (int64_t)blockIdx.z * sfstride;
    const int ym = Y == 0 ? (h > 1 ? 1 : 0) : Y - 1, yp = Y == h - 1 ? (h > 1 ? h - 2 : 0) : Y + 1;
    const uint8_t* r0 = S + (int64_t)ym * spitch; const uint8_t* r1 = S + (int64_t)Y * spitch; const uint8_t* r2 = S + (int64_t)yp * spitch;
    const int64_t o = (int64_t)blockIdx.z * fstride + (int64_t)Y * pitch + X;
    if (kVec) {
        const int xm = X == 0 ? 1 : X - 1, xp = X + 4 >= w ? w - 2 : X + 4;
        const uint32_t w0 = __ldg(reinterpret_cast<const uint32_t*>(r0 + X)), w1 = __ldg(reinterpret_cast<const uint32_t*>(r1 + X)),
                       w2 = __ldg(reinterpret_cast<const uint32_t*>(r2 + X));
        int a[6], b[6], c[6];          // columns X-1 .. X+4 of the three rows
        a[0] = __ldg(r0 + xm); b[0] = __ldg(r1 + xm); c[0] = __ldg(r2 + xm);
        a[5] = __ldg(r0 + xp); b[5] = __ldg(r1 + xp); c[5] = __ldg(r2 + xp);
#pragma unroll
        for (int i = 0; i < 4; ++i) { a[i + 1] = (w0 >> (8 * i)) & 255; b[i + 1] = (w1 >> (8 * i)) & 255; c[i + 1] = (w2 >> (8 * i)) & 255; }
        int t0[6], t1[6];
#pragma unroll
        for (int i = 0; i < 6; ++i) { t0[i] = (a[i] + c[i]) * 3 + b[i] * 10; t1[i] = c[i] - a[i]; }
        uint4 d;
        uint32_t* dp = &d.x;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int dx = t0[i + 2] - t0[i], dy = (t1[i] + t1[i + 2]) * 3 + t1[i + 1] * 10;
            dp[i] = ((uint32_t)dx & 0xffffu) | ((uint32_t)dy << 16);
        }
        *reinterpret_cast<uint4*>(deriv + o) = d;
        if (copy) *reinterpret_cast<uint32_t*>(dst + o) = w1;
    } else {
        const int xm = X == 0 ? (w > 1 ? 1 : 0) : X - 1, xp = X == w - 1 ? (w > 1 ? w - 2 : 0) : X + 1;
        const int t0m = (r0[xm] + r2[xm]) * 3 + r1[xm] * 10, t0p = (r0[xp] + r2[xp]) * 3 + r1[xp] * 10;
        const int t1m = r2[xm] - r0[xm], t1c = r2[X] - r0[X], t1p = r2[xp] - r0[xp];
        const int dx = t0p - t0m, dy = (t1m + t1p) * 3 + t1c * 10;
        deriv[o] = ((uint32_t)dx & 0xffffu) | ((uint32_t)dy << 16);
        if (copy) dst[o] = r1[X];
    }
}

// REFLECT_101 border of a padded level from its interior.  One thread per border pixel: `band` rows above and below the image span
// the padded width, the side bands span the image rows.
__global__ void __launch_bounds__(256) lk_border_kernel(uint8_t* dst, int w, int h, int pitch, int64_t fstride) {
    const int pw = w + 2 * kLkPad;
    const int n_tb = 2 * kLkPad * pw, n_side = 2 * kLkPad * h;
    const int i = blockIdx.x * 256 + threadIdx.x;
    if (i >= n_tb + n_side) return;
    int X, Y;
    if (i < n_tb) { const int r = i / pw; X = i - r * pw - kLkPad; Y = r < kLkPad ? r - kLkPad : h + (r - kLkPad); }
    else { const int j = i - n_tb; const int r = j / (2 * kLkPad), c = j - r * (2 * kLkPad); Y = r; X = c < kLkPad ? c - kLkPad : w + (c - kLkPad); }
    uint8_t* F = dst + (int64_t)blockIdx.z * fstride;
    F[(int64_t)Y * pitch + X] = F[(int64_t)lk_refl(Y, h) * pitch + lk_refl(X, w)];
}

// Exact warp sum of per-lane int32 partials with the hardware reduction (redux.sync): |partial| < 2^29, so the low 16 bits and the
// (signed) high part are reduced separately in int32 without overflow and recombined in int64.  Every lane gets the total.
__device__ __forceinline__ long long warp_sum_exact(int v) {
    const int lo = __reduce_add_sync(0xffffffffu, v & 0xffff), hi = __reduce_add_sync(0xffffffffu, v >> 16);
    return (long long)hi * 65536 + lo;
}

__device__ __forceinline__ int lk_descale(int x, int n) { return (x + (1 << (n - 1))) >> n; }

// Three neighbouring pixels of one image row as the bytes (p0, p1, p1, p2): the low half feeds the bilinear taps of column 0, the high half those of
// column 1 (IDP.2A: two 16-bit weights x two bytes + accumulator in one instruction, same issue rate as one IMAD).
// d = c + a.lo16 * b.byte0 + a.hi16 * b.byte1 (lo) / ... byte2, byte3 (hi): SIGNED 16-bit halves (w11 = 16384 - w00 - w01 - w10 can be -1) x unsigned bytes
__device__ __forceinline__ int dp2a_lo_su(uint32_t a, uint32_t b, int c) { int d; asm("dp2a.lo.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ int dp2a_hi_su(uint32_t a, uint32_t b, int c) { int d; asm("dp2a.hi.s32.u32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c)); return d; }
__device__ __forceinline__ uint32_t lk_pack_weights(int lo, int hi) { return ((uint32_t)lo & 0xffffu) | ((uint32_t)hi << 16); }

// Read from an arbitrarily aligned address with two aligned 32-bit loads (the padded planes have 256 bytes of slack behind the last row).
__device__ __forceinline__ uint32_t lk_load_row3(const uint8_t* p) {
    const uintptr_t a = reinterpret_cast<uintptr_t>(p);
    const uint32_t* q = reinterpret_cast<const uint32_t*>(a & ~(uintptr_t)3);
    const uint32_t x = __funnelshift_r(__ldg(q), __ldg(q + 1), 8u * (uint32_t)(a & 3));      // bytes p[0..3]
    return __byte_perm(x, 0, 0x2110);
}

__device__ __forceinline__ void lk_weights(float a, float b, int& w00, int& w01, int& w10, int& w11) {
    w00 = __float2int_rn(__fmul_rn(__fmul_rn(__fsub_rn(1.f, a), __fsub_rn(1.f, b)), 16384.f));
    w01 = __float2int_rn(__fmul_rn(__fmul_rn(a, __fsub_rn(1.f, b)), 16384.f));
    w10 = __float2int_rn(__fmul_rn(__fmul_rn(__fsub_rn(1.f, a), b), 16384.f));
    w11 = 16384 - w00 - w01 - w10;
}


// Window set-up of one level, in the tiled ownership of lk_mismatch_tiles (see there): each lane reads the 8x3 pixels of I and the
// 8x3 derivative words under its 7x2 window pixels (+ 2x2 for its pixel of column 20) from the padded planes and interpolates I, Ix,
// Iy with the 14-bit weights.  Outputs stay in registers: C = 256 - 512 Iw, GX = Ix, GY = Iy; s11/s12/s22 are this lane's share of
// the gradient matrix (exact in int32: 15 terms of < 2^24.1).
__device__ __forceinline__ void lk_setup_tiles(const uint8_t* __restrict__ img, const uint32_t* __restrict__ der, int pitch, int ipx, int ipy,
                                               int k2, int g7, int erow, int lane, int w00, int w01, int w10, int w11,
                                               int (&C)[14], int (&GX)[14], int (&GY)[14], int& Ce, int& GXe, int& GYe,
                                               int& s11, int& s12, int& s22) {
    uint32_t Rw[8];                  // row r of the 8x3 tile of I as bytes (p0, p1, p1, p2): the two horizontal pixel pairs of the lane's two columns
    int Dx[8][3], Dy[8][3];
    {
        const int64_t o = (int64_t)(ipy + g7) * pitch + (ipx + k2);
        const uint8_t* p = img + o; const uint32_t* q = der + o;
#pragma unroll
        for (int r = 0; r < 8; ++r) {
            Rw[r] = lk_load_row3(p);
#pragma unroll
            for (int x = 0; x < 3; ++x) {
                const uint32_t d = __ldg(q + x);
                Dx[r][x] = (int)(short)(d & 0xffffu); Dy[r][x] = (int)d >> 16;
            }
            p += pitch; q += pitch;
        }
    }
    const uint32_t wt = lk_pack_weights(w00, w01), wb = lk_pack_weights(w10, w11);
    int a11 = 0, a12 = 0, a22 = 0;
#pragma unroll
    for (int r = 0; r < 7; ++r)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            const int ival = (c == 0 ? dp2a_lo_su(wt, Rw[r], dp2a_lo_su(wb, Rw[r + 1], 256)) : dp2a_hi_su(wt, Rw[r], dp2a_hi_su(wb, Rw[r + 1], 256))) >> 9;
            const int ixv = (Dx[r][c] * w00 + Dx[r][c + 1] * w01 + Dx[r + 1][c] * w10 + Dx[r + 1][c + 1] * w11 + 8192) >> 14;
            const int iyv = (Dy[r][c] * w00 + Dy[r][c + 1] * w01 + Dy[r + 1][c] * w10 + Dy[r + 1][c + 1] * w11 + 8192) >> 14;
            C[2 * r + c] = 256 - 512 * ival; GX[2 * r + c] = ixv; GY[2 * r + c] = iyv;
            a11 += ixv * ixv; a12 += ixv * iyv; a22 += iyv * iyv;
        }
    if (lane >= 30) a11 = a12 = a22 = 0;
    // the pixel of column 20
    const int64_t oe = (int64_t)(ipy + erow) * pitch + (ipx + 20);
    const uint8_t* pe = img + oe; const uint32_t* qe = der + oe;
    const int e00 = __ldg(pe), e01 = __ldg(pe + 1), e10 = __ldg(pe + pitch), e11 = __ldg(pe + pitch + 1);
    const uint32_t d00 = __ldg(qe), d01 = __ldg(qe + 1), d10 = __ldg(qe + pitch), d11 = __ldg(qe + pitch + 1);
    const int ival = (e00 * w00 + e01 * w01 + e10 * w10 + e11 * w11 + 256) >> 9;
    const int ixv = ((int)(short)(d00 & 0xffffu) * w00 + (int)(short)(d01 & 0xffffu) * w01 + (int)(short)(d10 & 0xffffu) * w10 + (int)(short)(d11 & 0xffffu) * w11 + 8192) >> 14;
    const int iyv = (((int)d00 >> 16) * w00 + ((int)d01 >> 16) * w01 + ((int)d10 >> 16) * w10 + ((int)d11 >> 16) * w11 + 8192) >> 14;
    Ce = 256 - 512 * ival; GXe = lane < kWin ? ixv : 0; GYe = lane < kWin ? iyv : 0;
    s11 = a11 + GXe * GXe; s12 = a12 + GXe * GYe; s22 = a22 + GYe * GYe;
}

// Mismatch vector of one iteration.  The 21x21 window is tiled over the warp: lane = 10 g + k (k < 10, g < 3) owns window columns
// 2k, 2k+1 of rows 7g .. 7g+6 (14 pixels, held in registers: C = 256 - 512 Iw folds the descale rounding and the subtraction of the
// template into the first multiply-add), and lanes 0..20 each own one pixel of the left-over column 20.  Lanes 30, 31 repeat the
// work of lane 29 and are masked out.  Every lane loads its own 8x3 (+2x2) bytes of J from the padded plane and keeps them while the
// iterations stay on the same integer position (the usual case: steps are sub-pixel); the sums per lane are < 15 * 2^25: exact in int32.
__device__ __forceinline__ void lk_load_j_tile(const uint8_t* __restrict__ img, int pitch, int inx, int iny, int k2, int g7, int erow, uint32_t (&v)[8], uint32_t& e) {
    const uint8_t* p = img + (int64_t)(iny + g7) * pitch + (inx + k2);
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        v[r] = lk_load_row3(p);
        p += pitch;
    }
    const uint8_t* q = img + (int64_t)(iny + erow) * pitch + (inx + 20);
    e = (uint32_t)__ldg(q) | ((uint32_t)__ldg(q + 1) << 8) | ((uint32_t)__ldg(q + pitch) << 16) | ((uint32_t)__ldg(q + pitch + 1) << 24);
}

// v[r] = packed row r of the lane's 8x3 tile of J (lk_load_row3), e = the 2x2 pixels under its pixel of column 20 (top pair | bottom pair << 16);
// wt = w00 | w01 << 16, wb = w10 | w11 << 16.  
__device__ __forceinline__ void lk_mismatch_tiles(const uint32_t (&v)[8], uint32_t e, bool lane30, uint32_t wt, uint32_t wb,
                                                  const int (&C)[14], const int (&GX)[14], const int (&GY)[14], int Ce, int GXe, int GYe, int& s1, int& s2) {
    int a1 = 0, a2 = 0, b1 = 0, b2 = 0;
#pragma unroll
    for (int r = 0; r < 7; ++r) {
        const int da = dp2a_lo_su(wt, v[r], dp2a_lo_su(wb, v[r + 1], C[2 * r])) >> 9;
        const int db = dp2a_hi_su(wt, v[r], dp2a_hi_su(wb, v[r + 1], C[2 * r + 1])) >> 9;
        a1 += da * GX[2 * r]; a2 += da * GY[2 * r];
        b1 += db * GX[2 * r + 1]; b2 += db * GY[2 * r + 1];
    }
    if (lane30) { a1 = 0; a2 = 0; b1 = 0; b2 = 0; }
    const int de = dp2a_lo_su(wt, e, dp2a_hi_su(wb, e, Ce)) >> 9;
    s1 = a1 + b1 + de * GXe; s2 = a2 + b2 + de * GYe;
}

// points come either from keypoints (kps != nullptr: kp.x, kp.y) or from a plain float2 array
// (111 registers: 4 blocks of 4 warps per SM; asking for 5 or 6 resident blocks measured equal / 10 % slower)
__global__ void __launch_bounds__(kLkWarps * 32) lk_track_kernel(const __grid_constant__ LkLevels L, const sgs_keypoint* __restrict__ kps,
                                                                 const float2* __restrict__ pts, const int32_t* __restrict__ counts, int cap,
                                                                 const int32_t* __restrict__ prev_index, float2* __restrict__ out) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int f = blockIdx.y;
    const int p = blockIdx.x * kLkWarps + warp;
    const int n = counts ? min(counts[f], cap) : cap;
    if (p >= n) return;
    // row of L.J that plays the role of the previous image; < 0 (stream steps, a stream's first frame): the frame's own image
    const int fj = prev_index ? prev_index[f] : f;
    const int64_t pi = (int64_t)f * cap + p;
    float ptx, pty;
    if (kps) { ptx = kps[pi].x; pty = kps[pi].y; } else { const float2 q = pts[pi]; ptx = q.x; pty = q.y; }
    const int tl = min(lane, 29);
    const int k2 = 2 * (tl % 10), g7 = 7 * (tl / 10), erow = min(lane, kWin - 1);      // this lane's tile of the window (see lk_mismatch_tiles)
    const float half_win = 10.f;                       // (winSize - 1) * 0.5
    const float flt_scale = 1.f / (1 << 20);
    float nx = 0.f, ny = 0.f;
    for (int level = L.max_level; level >= 0; --level) {
        const int lw = L.w[level], lh = L.h[level];
        const int pitch = L.pitch[level];
        const uint8_t* Iimg = L.I[level] + (int64_t)f * L.fstride[level];
        const uint32_t* Dimg = L.D[level] + (int64_t)f * L.fstride[level];
        const uint8_t* Jimg = fj < 0 ? Iimg : L.J[level] + (int64_t)fj * L.fstride[level];
        const float sc = 1.f / (float)(1 << level);
        float px = __fmul_rn(ptx, sc), py = __fmul_rn(pty, sc);
        float qx, qy;
        if (level == L.max_level) { qx = px; qy = py; } else { qx = __fmul_rn(nx, 2.f); qy = __fmul_rn(ny, 2.f); }
        nx = qx; ny = qy;
        px = __fsub_rn(px, half_win); py = __fsub_rn(py, half_win);
        const int ipx = (int)floorf(px), ipy = (int)floorf(py);
        if (ipx < -kWin || ipx >= lw || ipy < -kWin || ipy >= lh) continue;
        int w00, w01, w10, w11;
        lk_weights(__fsub_rn(px, (float)ipx), __fsub_rn(py, (float)ipy), w00, w01, w10, w11);
        int s11, s12, s22;
        int C[14], GX[14], GY[14], Ce, GXe, GYe;
        lk_setup_tiles(Iimg, Dimg, pitch, ipx, ipy, k2, g7, erow, lane, w00, w01, w10, w11, C, GX, GY, Ce, GXe, GYe, s11, s12, s22);
        const float A11 = __fmul_rn((float)warp_sum_exact(s11), flt_scale), A12 = __fmul_rn((float)warp_sum_exact(s12), flt_scale),
                    A22 = __fmul_rn((float)warp_sum_exact(s22), flt_scale);
        float D = __fsub_rn(__fmul_rn(A11, A22), __fmul_rn(A12, A12));
        const float dd = __fsub_rn(A11, A22);
        const float min_eig = __fdiv_rn(__fsub_rn(__fadd_rn(A22, A11), __fsqrt_rn(__fadd_rn(__fmul_rn(dd, dd), __fmul_rn(__fmul_rn(4.f, A12), A12)))),
                                        (float)(2 * kWin * kWin));
        if (min_eig < 1e-4f || D < 1.1920928955078125e-7f) continue;
        D = __fdiv_rn(1.f, D);
        qx = __fsub_rn(qx, half_win); qy = __fsub_rn(qy, half_win);
        float pdx = 0.f, pdy = 0.f;
        uint32_t jv[8], je = 0;
        int tile_x = 0x7fffffff, tile_y = 0x7fffffff;
        for (int j = 0; j < kLkMaxCount; ++j) {
            const int inx = (int)floorf(qx), iny = (int)floorf(qy);
            if (inx < -kWin || inx >= lw || iny < -kWin || iny >= lh) break;
            lk_weights(__fsub_rn(qx, (float)inx), __fsub_rn(qy, (float)iny), w00, w01, w10, w11);
            if (inx != tile_x || iny != tile_y) { lk_load_j_tile(Jimg, pitch, inx, iny, k2, g7, erow, jv, je); tile_x = inx; tile_y = iny; }
            int s1, s2;
            lk_mismatch_tiles(jv, je, lane >= 30, lk_pack_weights(w00, w01), lk_pack_weights(w10, w11), C, GX, GY, Ce, GXe, GYe, s1, s2);
            const float B1 = __fmul_rn((float)warp_sum_exact(s1), flt_scale), B2 = __fmul_rn((float)warp_sum_exact(s2), flt_scale);
            const float dx = __fmul_rn(__fsub_rn(__fmul_rn(A12, B2), __fmul_rn(A22, B1)), D);
            const float dy = __fmul_rn(__fsub_rn(__fmul_rn(A12, B1), __fmul_rn(A11, B2)), D);
            qx = __fadd_rn(qx, dx); qy = __fadd_rn(qy, dy);
            nx = __fadd_rn(qx, half_win); ny = __fadd_rn(qy, half_win);
            if (__dadd_rn(__dmul_rn((double)dx, (double)dx), __dmul_rn((double)dy, (double)dy)) <= 0.01 * 0.01) break;        // Point2f::ddot is double
            if (j > 0 && (double)fabsf(__fadd_rn(dx, pdx)) < 0.01 && (double)fabsf(__fadd_rn(dy, pdy)) < 0.01) {
                nx = __fsub_rn(nx, __fmul_rn(dx, 0.5f)); ny = __fsub_rn(ny, __fmul_rn(dy, 0.5f));
                break;
            }
            pdx = dx; pdy = dy;
        }
    }
    if (lane == 0) out[pi] = make_float2(nx, ny);
}

}  // namespace sgs

using namespace sgs;

struct sgs_lk {
    explicit sgs_lk(int dev) : device(dev), res(dev) {}
    int device, w = 0, h = 0, max_batch = 0, max_level = 0;
    int lw[kLkMaxLevel + 1], lh[kLkMaxLevel + 1], lp[kLkMaxLevel + 1];      // level sizes; lp = padded pitch in pixels
    int64_t lfs[kLkMaxLevel + 1], loff[kLkMaxLevel + 1];                    // pixels per padded frame; offset of the level inside a pyramid buffer
    int64_t lorg[kLkMaxLevel + 1];                                          // offset of pixel (0, 0) inside a padded frame
    int64_t pyr_elems = 0;
    HandleResources res;
    uint8_t* d_pyrI = nullptr; uint8_t* d_pyrJ = nullptr;     // padded levels 0..max_level, each [max_batch][h + 2 pad][pitch]
    uint32_t* d_der = nullptr;                                // derivative planes of I, same geometry (borders stay zero)
    // staging for the single-pair host API
    uint8_t* d_img = nullptr; float* d_pts = nullptr; float* d_out = nullptr; int pts_cap = 0;
    cudaStream_t st = nullptr;
    // optional stage timing (pyramid build, tracker), same contract as sgs_extractor_set_profiling
    StageTimer timer{2};
};

namespace {
int lk_bad(const char* m) { set_error("%s", m); return SGS_ERR_INVALID; }

// padded pyramid (+ derivative planes when d_der != nullptr) of `nframes` images
void build_pyramid(sgs_lk* k, const uint8_t* d_l0, int pitch0, int64_t fstride0, uint8_t* d_pyr, uint32_t* d_der, int nframes, cudaStream_t st) {
    for (int l = 0; l <= k->max_level; ++l) {
        uint8_t* dst = d_pyr + k->loff[l] + k->lorg[l];
        const int w = k->lw[l], h = k->lh[l];
        if (l > 0) {
            const uint8_t* src = d_pyr + k->loff[l - 1] + k->lorg[l - 1];
            dim3 grid(((w + 3) / 4 + 31) / 32, (h + 7) / 8, nframes);
            lk_pyrdown_kernel<<<grid, 256, 0, st>>>(src, k->lp[l - 1], k->lfs[l - 1], dst, w, h, k->lp[l], k->lfs[l]);
        }
        const uint8_t* src = l == 0 ? d_l0 : dst;
        const int sp = l == 0 ? pitch0 : k->lp[l];
        const int64_t sfs = l == 0 ? fstride0 : k->lfs[l];
        if (d_der) {
            uint32_t* der = d_der + k->loff[l] + k->lorg[l];
            const bool vec = (w & 3) == 0 && w >= 8 && (((uintptr_t)src | (uintptr_t)sp | (uintptr_t)sfs) & 3) == 0;
            if (vec) {
                dim3 grid((w / 4 + 31) / 32, (h + 7) / 8, nframes);
                lk_interior_kernel<true><<<grid, 256, 0, st>>>(src, sp, sfs, dst, l == 0, der, w, h, k->lp[l], k->lfs[l]);
            } else {
                dim3 grid((w + 31) / 32, (h + 7) / 8, nframes);
                lk_interior_kernel<false><<<grid, 256, 0, st>>>(src, sp, sfs, dst, l == 0, der, w, h, k->lp[l], k->lfs[l]);
            }
        } else if (l == 0) {
            cudaMemcpy3DParms c = {};
            c.srcPtr = make_cudaPitchedPtr(const_cast<uint8_t*>(d_l0), (size_t)pitch0, (size_t)w, (size_t)(fstride0 / pitch0));
            c.dstPtr = make_cudaPitchedPtr(dst - k->lorg[0], (size_t)k->lp[0], (size_t)k->lp[0], (size_t)(h + 2 * kLkPad));
            c.dstPos = make_cudaPos(kLkPad, kLkPad, 0);
            c.extent = make_cudaExtent((size_t)w, (size_t)h, (size_t)nframes);
            c.kind = cudaMemcpyDeviceToDevice;
            if (fstride0 % pitch0 == 0) cudaMemcpy3DAsync(&c, st);
            else for (int f = 0; f < nframes; ++f)
                cudaMemcpy2DAsync(dst + (int64_t)f * k->lfs[0], (size_t)k->lp[0], d_l0 + (int64_t)f * fstride0, (size_t)pitch0, (size_t)w, (size_t)h, cudaMemcpyDeviceToDevice, st);
        }
        const int nborder = 2 * kLkPad * (w + 2 * kLkPad) + 2 * kLkPad * h;
        dim3 gb((nborder + 255) / 256, 1, nframes);
        lk_border_kernel<<<gb, 256, 0, st>>>(dst, w, h, k->lp[l], k->lfs[l]);
    }
}

// j_store (may be NULL): padded levels in the geometry of d_pyrJ holding the previous images, row d_prev_index[f] for frame f (< 0: its own image)
int run_lk(sgs_lk* k, const uint8_t* d_cur, const uint8_t* d_prev, const int32_t* d_prev_index, int nframes, size_t frame_stride, int pitch,
           const sgs_keypoint* d_kps, const float* d_pts, const int32_t* d_counts, int cap, float* d_out, cudaStream_t st, const uint8_t* j_store = nullptr) {
    k->timer.begin();
    k->timer.mark(0, st);
    build_pyramid(k, d_cur, pitch, (int64_t)frame_stride, k->d_pyrI, k->d_der, nframes, st);
    const bool same_batch = d_prev_index != nullptr;     // previous images are other frames of the same batch (or the store): no J pyramid to build
    if (!same_batch) build_pyramid(k, d_prev, pitch, (int64_t)frame_stride, k->d_pyrJ, nullptr, nframes, st);
    LkLevels L;
    L.max_level = k->max_level;
    for (int l = 0; l <= kLkMaxLevel; ++l) {
        if (l <= k->max_level) {
            const int64_t o = k->loff[l] + k->lorg[l];
            L.w[l] = k->lw[l]; L.h[l] = k->lh[l]; L.pitch[l] = k->lp[l]; L.fstride[l] = k->lfs[l];
            L.I[l] = k->d_pyrI + o; L.J[l] = (j_store ? j_store : same_batch ? k->d_pyrI : k->d_pyrJ) + o; L.D[l] = k->d_der + o;
        } else { L.I[l] = L.J[l] = nullptr; L.D[l] = nullptr; L.w[l] = L.h[l] = L.pitch[l] = 0; L.fstride[l] = 0; }
    }
    k->timer.mark(1, st);
    dim3 grid((cap + kLkWarps - 1) / kLkWarps, nframes);
    lk_track_kernel<<<grid, kLkWarps * 32, 0, st>>>(L, d_kps, reinterpret_cast<const float2*>(d_pts), d_counts, cap, d_prev_index, reinterpret_cast<float2*>(d_out));
    k->timer.end(st);
    SGS_CUDA_TRY(cudaGetLastError());
    return SGS_OK;
}
}  // namespace

namespace sgs {
LkPyramid lk_pyramid(const sgs_lk* k) {
    LkPyramid p;
    p.I = k->d_pyrI; p.bytes = k->pyr_elems + 256; p.max_level = k->max_level;
    for (int l = 0; l <= kLkMaxLevel; ++l) { p.off[l] = l <= k->max_level ? k->loff[l] : 0; p.frame_bytes[l] = l <= k->max_level ? k->lfs[l] : 0; }
    return p;
}

int lk_track_from_store(sgs_lk* k, const uint8_t* d_cur, int nframes, size_t frame_stride, int pitch, const sgs_keypoint* d_kps, const int32_t* d_counts,
                        int cap, const uint8_t* d_store, const int32_t* d_row, float* d_prev_xy, cudaStream_t st) {
    return run_lk(k, d_cur, nullptr, d_row, nframes, frame_stride, pitch, d_kps, nullptr, d_counts, cap, d_prev_xy, st, d_store);
}
}  // namespace sgs

extern "C" {

SGS_API int sgs_lk_set_profiling(sgs_lk* k, int enable) {
    if (!k) return lk_bad("sgs_lk_set_profiling: NULL");
    SGS_CUDA_TRY(cudaSetDevice(k->device));
    SGS_CUDA_TRY(k->timer.enable(k->res, enable != 0));
    return SGS_OK;
}

SGS_API int sgs_lk_stage_times(sgs_lk* k, double* ms_total2, int* ncalls) {
    if (!k || !ms_total2 || !ncalls) return lk_bad("sgs_lk_stage_times: NULL");
    k->timer.fold();        // a failed wait leaves the last call out of the totals
    ms_total2[0] = k->timer.totals()[0]; ms_total2[1] = k->timer.totals()[1]; *ncalls = k->timer.calls();
    return SGS_OK;
}

SGS_API void sgs_lk_destroy(sgs_lk* k) { delete k; }

SGS_API int sgs_lk_create(int width, int height, int max_batch, int device, sgs_lk** out) {
    if (!out || width < 24 || height < 24 || max_batch < 1) return lk_bad("sgs_lk_create: bad argument");
    *out = nullptr;
    SGS_CUDA_TRY(cudaSetDevice(device));
    auto k = std::make_unique<sgs_lk>(device);
    k->w = width; k->h = height; k->max_batch = max_batch;
    int64_t off = 0;
    k->max_level = 0;
    for (int l = 0; l <= kLkMaxLevel; ++l) {     // buildOpticalFlowPyramid stops when a level would not be larger than the window
        if (l == 0) { k->lw[0] = width; k->lh[0] = height; }
        else {
            const int nw = (k->lw[l - 1] + 1) / 2, nh = (k->lh[l - 1] + 1) / 2;
            if (nw <= kWin || nh <= kWin) break;
            k->lw[l] = nw; k->lh[l] = nh; k->max_level = l;
        }
        k->lp[l] = (k->lw[l] + 2 * kLkPad + 15) & ~15;
        k->lfs[l] = (int64_t)k->lp[l] * (k->lh[l] + 2 * kLkPad);
        k->lorg[l] = (int64_t)kLkPad * k->lp[l] + kLkPad;
        k->loff[l] = off;
        off += k->lfs[l] * max_batch;
    }
    k->pyr_elems = off;
    SGS_CUDA_TRY_AT("sgs_lk_create", k->res.stream(&k->st));
    SGS_CUDA_TRY_AT("sgs_lk_create", k->res.alloc(&k->d_pyrI, (size_t)off + 256));
    SGS_CUDA_TRY_AT("sgs_lk_create", k->res.alloc(&k->d_pyrJ, (size_t)off + 256));
    SGS_CUDA_TRY_AT("sgs_lk_create", k->res.alloc(&k->d_der, 4 * (size_t)off + 256));
    SGS_CUDA_TRY_AT("sgs_lk_create", cudaMemset(k->d_der, 0, 4 * (size_t)off + 256));        // the borders of the derivative planes are never written again
    *out = k.release();
    return SGS_OK;
}

SGS_API int sgs_lk_track_batch_device(sgs_lk* k, const uint8_t* d_cur, const uint8_t* d_prev, const int32_t* d_prev_index, int nframes,
                                      size_t frame_stride, int pitch, const sgs_keypoint* d_kps, const int32_t* d_counts, int cap, float* d_prev_xy,
                                      void* stream) {
    if (!k || !d_cur || (!d_prev && !d_prev_index) || !d_kps || !d_counts || !d_prev_xy) return lk_bad("sgs_lk_track_batch_device: NULL argument");
    if (nframes < 1 || nframes > k->max_batch || cap < 1) return lk_bad("sgs_lk_track_batch_device: nframes/cap out of range");
    if (pitch < k->w || frame_stride < (size_t)pitch * k->h) return lk_bad("sgs_lk_track_batch_device: pitch/frame_stride too small");
    return run_lk(k, d_cur, d_prev, d_prev_index, nframes, frame_stride, pitch, d_kps, nullptr, d_counts, cap, d_prev_xy, stream ? (cudaStream_t)stream : k->st);
}

SGS_API int sgs_lk_track(sgs_lk* k, const uint8_t* cur, const uint8_t* prev, int pitch, const float* pts, int n, float* out) {
    if (!k || !cur || !prev || n < 0 || (n > 0 && (!pts || !out))) return lk_bad("sgs_lk_track: bad argument");
    if (n == 0) return SGS_OK;
    SGS_CUDA_TRY(cudaSetDevice(k->device));
    const int dp = (k->w + 15) & ~15;
    if (!k->d_img) SGS_CUDA_TRY(k->res.alloc(&k->d_img, (size_t)2 * dp * k->h));
    if (n > k->pts_cap) {
        k->pts_cap = 0;
        SGS_CUDA_TRY(k->res.regrow(&k->d_pts, 8 * (size_t)n));
        SGS_CUDA_TRY(k->res.regrow(&k->d_out, 8 * (size_t)n));
        k->pts_cap = n;
    }
    SGS_CUDA_TRY(cudaMemcpy2DAsync(k->d_img, dp, cur, pitch, k->w, k->h, cudaMemcpyHostToDevice, k->st));
    SGS_CUDA_TRY(cudaMemcpy2DAsync(k->d_img + (size_t)dp * k->h, dp, prev, pitch, k->w, k->h, cudaMemcpyHostToDevice, k->st));
    SGS_CUDA_TRY(cudaMemcpyAsync(k->d_pts, pts, 8 * (size_t)n, cudaMemcpyHostToDevice, k->st));
    int rc = run_lk(k, k->d_img, k->d_img + (size_t)dp * k->h, nullptr, 1, (size_t)dp * k->h, dp, nullptr, k->d_pts, nullptr, n, k->d_out, k->st);
    if (rc != SGS_OK) return rc;
    SGS_CUDA_TRY(cudaMemcpyAsync(out, k->d_out, 8 * (size_t)n, cudaMemcpyDeviceToHost, k->st));
    SGS_CUDA_TRY(cudaStreamSynchronize(k->st));
    return SGS_OK;
}

SGS_API int sgs_lk_read_level(sgs_lk* k, int which, int level, uint8_t* out, int out_pitch) {   // parity accessor: frame 0 of the last call
    if (!k || !out || level < 1 || level > k->max_level) return lk_bad("sgs_lk_read_level: bad argument");
    SGS_CUDA_TRY(cudaSetDevice(k->device));
    SGS_CUDA_TRY(cudaStreamSynchronize(k->st));
    SGS_CUDA_TRY(cudaMemcpy2D(out, out_pitch, (which ? k->d_pyrJ : k->d_pyrI) + k->loff[level] + k->lorg[level], k->lp[level], k->lw[level], k->lh[level],
                              cudaMemcpyDeviceToHost));
    return SGS_OK;
}

SGS_API int sgs_lk_read_padded(sgs_lk* k, int which, int level, int frame, uint8_t* img, uint32_t* deriv, int* pad) {   // parity accessor: a whole padded level
    if (!k || !img || (which != 0 && which != 1) || (which == 1 && deriv) || level < 0 || level > k->max_level || frame < 0 || frame >= k->max_batch)
        return lk_bad("sgs_lk_read_padded: bad argument");
    SGS_CUDA_TRY(cudaSetDevice(k->device));
    SGS_CUDA_TRY(cudaStreamSynchronize(k->st));
    const int64_t o = k->loff[level] + (int64_t)frame * k->lfs[level];
    const size_t pw = (size_t)k->lw[level] + 2 * kLkPad, ph = (size_t)k->lh[level] + 2 * kLkPad;
    SGS_CUDA_TRY(cudaMemcpy2D(img, pw, (which ? k->d_pyrJ : k->d_pyrI) + o, k->lp[level], pw, ph, cudaMemcpyDeviceToHost));
    if (deriv) SGS_CUDA_TRY(cudaMemcpy2D(deriv, 4 * pw, k->d_der + o, 4 * (size_t)k->lp[level], 4 * pw, ph, cudaMemcpyDeviceToHost));
    if (pad) *pad = kLkPad;
    return SGS_OK;
}

}  // extern "C"
