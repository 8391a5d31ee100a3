// grab.cu -- the image half of Tracking::GrabImageRGBD (src/Tracking.cc:206-251) for a batch of frames:
//   colour -> gray : cvtColor(CV_RGB2GRAY / CV_BGR2GRAY) of 8-bit 3-channel frames (:214-227), OpenCV's fixed-point formula
//                    Y = (9798 R + 19235 G + 3735 B + 2^14) >> 15 (quirk Q14 in DESIGN.md); Camera.RGB picks the channel that gets the R weight;
//   raw depth      : convertTo(CV_32F, mDepthMapFactor) (:229-230) of uint16 or float32 frames, one float32 multiply (float)raw * factor.
// One launch converts both for every frame of the batch; each thread handles four consecutive pixels of one row.
#include <cuda_runtime.h>

#include <cmath>

#include "sgs_common.h"

namespace sgs {

template <class DepthT>
__global__ void __launch_bounds__(256) grab_rgbd_kernel(const uint8_t* __restrict__ rgb, int64_t rgb_stride, int rgb_pitch, int r_chan,
                                                        const uint8_t* __restrict__ depth, int64_t depth_stride, int depth_pitch, float factor,
                                                        int width, int height, uint8_t* __restrict__ gray, int64_t gray_stride, int gray_pitch,
                                                        uint8_t* __restrict__ dout, int64_t dout_stride, int dout_pitch) {
    const int qw = (width + 3) >> 2;
    const int q = blockIdx.x * 256 + threadIdx.x;
    if (q >= qw * height) return;
    const int64_t f = blockIdx.y;
    const int y = q / qw, x0 = (q - y * qw) * 4, n = min(4, width - x0);
    if (gray) {
        const uint8_t* s = rgb + f * rgb_stride + (int64_t)y * rgb_pitch + 3 * x0;
        uint8_t* d = gray + f * gray_stride + (int64_t)y * gray_pitch + x0;
        for (int i = 0; i < n; ++i) {
            const uint32_t r = s[3 * i + r_chan], g = s[3 * i + 1], b = s[3 * i + 2 - r_chan];
            d[i] = (uint8_t)((9798u * r + 19235u * g + 3735u * b + (1u << 14)) >> 15);
        }
    }
    if (dout) {
        const DepthT* s = reinterpret_cast<const DepthT*>(depth + f * depth_stride + (int64_t)y * depth_pitch) + x0;
        float* d = reinterpret_cast<float*>(dout + f * dout_stride + (int64_t)y * dout_pitch) + x0;
        for (int i = 0; i < n; ++i) d[i] = __fmul_rn((float)s[i], factor);
    }
}

}  // namespace sgs

using namespace sgs;

extern "C" {

SGS_API int sgs_grab_rgbd_batch_device(const uint8_t* d_rgb, size_t rgb_stride, int rgb_pitch, const void* d_depth, size_t depth_stride, int depth_pitch,
                                       const sgs_rgbd_format* fmt, int width, int height, int nframes, uint8_t* d_gray, size_t gray_stride, int gray_pitch,
                                       float* d_depth_out, size_t depth_out_stride, int depth_out_pitch, void* stream) {
    auto bad = [](const char* m) { set_error("sgs_grab_rgbd_batch_device: %s", m); return (int)SGS_ERR_INVALID; };
    if (!fmt) return bad("NULL format");
    if (fmt->depth_type != 0 && fmt->depth_type != 1) return bad("depth_type is neither 0 (uint16) nor 1 (float32)");
    if (!std::isfinite(fmt->depth_map_factor) || !(fmt->depth_map_factor > 0.f)) return bad("depth_map_factor is not a finite positive number");
    if (width < 1 || height < 1 || nframes < 1 || nframes > 65535) return bad("width, height or nframes out of range");
    if (!d_rgb != !d_gray || !d_depth != !d_depth_out || (!d_gray && !d_depth_out)) return bad("colour / gray and depth in / out come in pairs, at least one pair");
    const size_t W = width, Hh = height, esz = fmt->depth_type == 0 ? 2 : 4;
    if (d_gray && (rgb_pitch < 3 * width || rgb_stride < (size_t)rgb_pitch * Hh || gray_pitch < width || gray_stride < (size_t)gray_pitch * Hh))
        return bad("colour or gray pitch / frame stride too small");
    if (d_depth_out) {
        if ((size_t)depth_pitch < esz * W || depth_stride < (size_t)depth_pitch * Hh || (size_t)depth_out_pitch < 4 * W || depth_out_stride < (size_t)depth_out_pitch * Hh)
            return bad("depth pitch / frame stride too small");
        if (depth_pitch % esz || depth_stride % esz || (uintptr_t)d_depth % esz || depth_out_pitch % 4 || depth_out_stride % 4 || (uintptr_t)d_depth_out % 4)
            return bad("depth pitch, frame stride or pointer not a multiple of the element size");
    }
    const int qw = (width + 3) / 4;
    const dim3 grid((unsigned)(((int64_t)qw * height + 255) / 256), nframes);
    auto k = fmt->depth_type == 0 ? grab_rgbd_kernel<uint16_t> : grab_rgbd_kernel<float>;
    k<<<grid, 256, 0, (cudaStream_t)stream>>>(d_rgb, (int64_t)rgb_stride, rgb_pitch, fmt->rgb ? 0 : 2, (const uint8_t*)d_depth, (int64_t)depth_stride, depth_pitch,
                                              fmt->depth_map_factor, width, height, d_gray, (int64_t)gray_stride, gray_pitch, (uint8_t*)d_depth_out,
                                              (int64_t)depth_out_stride, depth_out_pitch);
    SGS_CUDA_TRY(cudaGetLastError());
    return SGS_OK;
}

}  // extern "C"
