"""Writes tests/golden/grab_rgbd.npz: small batches of colour and raw depth frames in padded layouts (odd sizes, row pitches and frame strides that
are not multiples of the row, depth values 0 and 65535) with what cv2 computes for them: cvtColor(RGB2GRAY) and cvtColor(BGR2GRAY) of every frame, and
cv2.multiply(depth, factor, dtype=CV_32F) at the TUM1, TUM2 and astra factors.  The GPU tests read it because the GPU machine may lack cv2.

    python tests/golden/make_golden_grab.py"""
import os
import sys

import cv2
import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import grab_ref as GR  # noqa: E402

# (width, height, frames, depth type 0 = uint16 / 1 = float32, colour pitch padding, colour stride padding, depth pitch padding, depth stride padding)
CASES = [(1, 1, 2, 0, 1, 3, 2, 2), (7, 5, 3, 0, 5, 11, 6, 4), (33, 17, 2, 0, 3, 7, 2, 10), (61, 47, 3, 0, 13, 1, 14, 6), (45, 31, 2, 1, 7, 9, 12, 8)]


def main():
    rng = np.random.RandomState(14)
    out = {'factors': np.array(GR.FACTORS, np.float32)}
    for k, (w, h, nf, dt, rp, rs, dp, ds) in enumerate(CASES):
        esz = 2 if dt == 0 else 4
        rgb_pitch = 3 * w + rp; rgb_stride = rgb_pitch * h + rs
        d_pitch = esz * w + dp; d_stride = d_pitch * h + ds
        rgb_buf = rng.randint(0, 256, nf * rgb_stride).astype(np.uint8)
        d_buf = rng.randint(0, 256, nf * d_stride).astype(np.uint8)
        rgb = GR.frames_from_buffer(rgb_buf, nf, h, 3 * w, rgb_pitch, rgb_stride, np.uint8).reshape(nf, h, w, 3)
        if dt == 0:
            raw = rng.randint(0, 65536, (nf, h, w)).astype(np.uint16)
            raw.flat[0] = 0; raw.flat[-1] = 65535; raw.flat[len(raw.flat) // 2] = 65535
        else:
            raw = rng.uniform(0, 10, (nf, h, w)).astype(np.float32)
            raw.flat[0] = 0
        for f in range(nf):
            for y in range(h):
                o = f * d_stride + y * d_pitch
                d_buf[o:o + esz * w] = raw[f, y].view(np.uint8)
        out['c%d_meta' % k] = np.array([w, h, nf, dt, rgb_pitch, rgb_stride, d_pitch, d_stride], np.int64)
        out['c%d_rgb' % k] = rgb_buf
        out['c%d_depth' % k] = d_buf
        out['c%d_gray_rgb' % k] = np.stack([cv2.cvtColor(np.ascontiguousarray(rgb[f]), cv2.COLOR_RGB2GRAY).reshape(h, w) for f in range(nf)])
        out['c%d_gray_bgr' % k] = np.stack([cv2.cvtColor(np.ascontiguousarray(rgb[f]), cv2.COLOR_BGR2GRAY).reshape(h, w) for f in range(nf)])
        for j, fac in enumerate(GR.FACTORS):
            out['c%d_depth_f%d' % (k, j)] = np.stack([cv2.multiply(np.ascontiguousarray(raw[f]), float(fac), dtype=cv2.CV_32F).reshape(h, w)
                                                      for f in range(nf)])
    out['ncases'] = np.array(len(CASES))
    np.savez_compressed(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'grab_rgbd.npz'), **out)


if __name__ == '__main__':
    main()
