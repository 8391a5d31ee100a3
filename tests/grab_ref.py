"""numpy restatement of the two image conversions of Tracking::GrabImageRGBD (src/Tracking.cc:206-251), the device kernels of
sg-slam_b200/csrc/grab.cu: cvtColor(RGB2GRAY / BGR2GRAY) of 8-bit 3-channel frames and convertTo(CV_32F, mDepthMapFactor).  Pinned against cv2 by
tests/test_grab_rgbd.py."""
import numpy as np

FACTORS = (np.float32(1 / 5000), np.float32(1 / 5208), np.float32(1.0))     # mDepthMapFactor of TUM1 / TUM2 (DepthMapFactor 5000 / 5208) and astra (1)


def to_gray(rgb, rgb_order):
    """OpenCV's 15-bit fixed-point luma: Y = (9798 R + 19235 G + 3735 B + 2^14) >> 15; rgb_order (Camera.RGB) != 0 gives byte 0 the R weight."""
    c = np.asarray(rgb).astype(np.uint32)
    r, b = (c[..., 0], c[..., 2]) if rgb_order else (c[..., 2], c[..., 0])
    return ((9798 * r + 19235 * c[..., 1] + 3735 * b + (1 << 14)) >> 15).astype(np.uint8)


def to_depth(raw, factor):
    """(float)raw * (float)factor, one float32 multiply."""
    return np.asarray(raw).astype(np.float32) * np.float32(factor)


def all_triples():
    """Every 8-bit RGB triple once: a 4096 x 4096 x 3 image, pixel i = (i >> 16, (i >> 8) & 255, i & 255)."""
    i = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([i >> 16, (i >> 8) & 255, i & 255], -1).astype(np.uint8).reshape(4096, 4096, 3)


def frames_from_buffer(buf, nframes, h, row_bytes, pitch, stride, dtype):
    """[F, h, row_bytes / itemsize] view of frames stored `stride` bytes apart with rows `pitch` bytes apart in the flat byte buffer `buf`."""
    out = np.stack([np.stack([buf[f * stride + y * pitch: f * stride + y * pitch + row_bytes] for y in range(h)]) for f in range(nframes)])
    return np.ascontiguousarray(out).view(dtype)
