// match_rules.cuh -- the ORBmatcher rules that more than one device matcher restates (match.cu, bow.cu, hamming.cu, frame_geom.cu).
// Every helper keeps the reference's order of operations with individually rounded intrinsics (the build uses -fmad=false), so a
// matcher that calls it stays bit-exact; a fix to one of these rules is made here once.
#pragma once
#include <cuda_runtime.h>

#include <cstdint>

#include "sgs_logf.h"

namespace sgs {

constexpr int kThHigh = 100, kThLow = 50, kHistoLen = 30;   // TH_HIGH, TH_LOW, HISTO_LENGTH: src/ORBmatcher.cc:37-39

// ORBmatcher::DescriptorDistance (src/ORBmatcher.cc:1649-1665 == DBoW2 FORB::distance): Hamming distance of two 256-bit descriptors
__device__ __forceinline__ int descriptor_distance(const uint4& a0, const uint4& a1, const uint4& b0, const uint4& b1) {
    return __popc(a0.x ^ b0.x) + __popc(a0.y ^ b0.y) + __popc(a0.z ^ b0.z) + __popc(a0.w ^ b0.w) +
           __popc(a1.x ^ b1.x) + __popc(a1.y ^ b1.y) + __popc(a1.z ^ b1.z) + __popc(a1.w ^ b1.w);
}

// rotation-histogram bin of a match whose keypoint angles are angle_a and angle_b (e.g. src/ORBmatcher.cc:1438-1443)
__device__ __forceinline__ int rotation_bin(float angle_a, float angle_b) {
    float rot = __fsub_rn(angle_a, angle_b);
    if (rot < 0.f) rot = __fadd_rn(rot, 360.f);
    const int bin = (int)roundf(__fmul_rn(rot, (float)kHistoLen / 360.0f));
    return bin == kHistoLen ? 0 : bin;
}

// ORBmatcher::ComputeThreeMaxima (src/ORBmatcher.cc:1603-1645): the three fullest bins, -1 for a bin under a tenth of the fullest
__device__ __forceinline__ void three_maxima(const int* hist, int& i1, int& i2, int& i3) {
    int m1 = 0, m2 = 0, m3 = 0;
    i1 = i2 = i3 = -1;
    for (int i = 0; i < kHistoLen; ++i) {
        const int sz = hist[i];
        if (sz > m1) { m3 = m2; m2 = m1; m1 = sz; i3 = i2; i2 = i1; i1 = i; }
        else if (sz > m2) { m3 = m2; m2 = sz; i3 = i2; i2 = i; }
        else if (sz > m3) { m3 = sz; i3 = i; }
    }
    if ((float)m2 < __fmul_rn(0.1f, (float)m1)) { i2 = -1; i3 = -1; }
    else if ((float)m3 < __fmul_rn(0.1f, (float)m1)) { i3 = -1; }
}

// The rotation-consistency filter after the matching loop (e.g. src/ORBmatcher.cc:1451-1470), order independent: every thread of the
// block takes events e = threadIdx.x, threadIdx.x + blockDim.x, ... of the list (bin << 16 | slot) and clears out[slot] when the bin is
// not one of the three main bins of `hist`.  Returns how many matches this thread removed.
__device__ __forceinline__ int drop_outside_main_bins(const int* hist, const int32_t* events, int nevent, int32_t* out) {
    int i1, i2, i3;
    three_maxima(hist, i1, i2, i3);
    int removed = 0;
    for (int e = threadIdx.x; e < nevent; e += blockDim.x) {
        const int ev = events[e];
        const int bin = ev >> 16;
        if (bin != i1 && bin != i2 && bin != i3) { out[ev & 0xFFFF] = -1; ++removed; }
    }
    return removed;
}

// MapPoint::PredictScale (src/MapPoint.cc:400-418): ceil(log(maxDistance / dist) / log(scaleFactor)) with libm's logf, clamped to the pyramid
__device__ __forceinline__ int predict_scale(float max_dist, float dist, float log_sf, int nlevels) {
    const int s = (int)ceilf(__fdiv_rn(glibc_logf(__fdiv_rn(max_dist, dist)), log_sf));
    return s < 0 ? 0 : (s >= nlevels ? nlevels - 1 : s);
}

// One row of a plain 3x3 * 3x1 (+ C) cv::gemm on CV_32F, which takes OpenCV's small-matrix path: float products summed in float, left to
// right, then (float)((double)sum + (double)c).  Pinned against cv2.gemm (tests/golden/make_golden_frustum.py).
__device__ __forceinline__ float gemm3_row(float r0, float r1, float r2, const float* x, float c) {
    const float sum = __fadd_rn(__fadd_rn(__fmul_rn(r0, x[0]), __fmul_rn(r1, x[1])), __fmul_rn(r2, x[2]));
    return (float)__dadd_rn((double)sum, (double)c);
}

}  // namespace sgs
