"""Camera geometries, device-buffer layouts and rounding cases for the detector's input resize (preprocess_table_kernel + preprocess_kernel of
detector.cu: Mat::from_pixels_resize to 300 x 300 + mean subtraction), for tests/test_detector_resize_cases.py (CPU) and
tests/test_gpu_detector_resize.py (GPU, bit for bit against detector_oracle.preprocess).

  GEOMETRIES  (width, height): the benchmark's and the usual datasets' cameras, 1080p, the identity and an exact 2x, odd sizes on both sides of 300,
              and enlarged axes down to the 2-pixel minimum (the s < 0 and s >= sn - 1 clamps of the coefficients);
  LAYOUTS     how a batch lies in device memory: dense, an odd pitch 3W + 5, a frame stride past H * pitch (gaps filled with MARKER), stride 0 (every
              frame reads frame 0), a base pointer 1 to 3 bytes past an aligned address;
  exact halves: the destination columns / rows whose float32 weight * 2048 lands exactly on .5, where the rounding convention of the 11-bit
              coefficients decides the weight (cv2 rounds half to even, a +-0.5-and-truncate cast rounds half away from zero);
  plans       the detector's GEMM plans at 8 frames and at the benchmark's batch sizes (plan-only handles)."""
import numpy as np

import detector_oracle as DO

T = DO.TARGET
GEOMETRIES = [(640, 480), (1280, 720), (752, 480), (1241, 376), (1920, 1080), (300, 300), (600, 600), (301, 299), (150, 100), (2, 2), (2, 600),
              (600, 2)]
LAYOUTS = ('dense', 'pitch', 'gap', 'zero', 'offset')
MARKER = 0xA5
PROBE = 8                      # frames per call of the small-batch handles (DM.PROBE_FRAMES)
SM_TILES = 2 * 132             # persistent GEMM CTAs at most (two per SM on narrow tiles, 132 SMs): a CTA walks m_tiles / SM_TILES pixel tiles or more
# pixel tiles per persistent CTA on a graph's largest GEMM layer at 512 frames, at least (the wide-tail graph's largest GEMM map is 75 x 75)
SCALE_TILES = {'reference': 100, 'mini': 100, 'wide_tails': 80}


def exact_halves(dn, sn):
    """Destination positions (of dn, from sn source pixels) where one of the two weights, as float32 product with 2048, is exactly k + 0.5: recorded
    from the restatement's own coefficient code (detector_oracle.resize_coeffs calls its rounding on weight 0, then weight 1, per position)."""
    seen = []

    def rnd(v):
        seen.append(v % 1 == 0.5)
        return DO.round_half_even(v)

    DO.resize_coeffs(dn, sn, rnd)
    return np.nonzero(np.array(seen).reshape(dn, 2).any(1))[0]


def half_table():
    """{source size: exact-half destination positions} over every width and height of GEOMETRIES"""
    return {n: exact_halves(T, n) for n in sorted({n for g in GEOMETRIES for n in g})}


def frames(w, h, n, seed):
    """n distinct uint8 frames h x w x 3: uniform noise (every weight of the resize matters; the geometries go down to 2 pixels)"""
    return np.random.default_rng(seed * 7919 + w * 31 + h).integers(0, 256, (n, h, w, 3), dtype=np.uint8)


def half_image(w, h, seed=0):
    """An image of w x h on which the half-to-even and the half-away-from-zero coefficients give different input blobs (at every exact-half column
    and row: tests/test_detector_resize_cases.py proves it): black and white noise, so that a coefficient one unit off moves the horizontal sums by
    up to 255 / 2048 of a grey level and many of the 300 pixels of each such column or row cross a rounding boundary."""
    return (np.random.default_rng(seed + w * 7 + h).integers(0, 2, (h, w, 3)) * 255).astype(np.uint8)


def pack(fr, layout, marker=MARKER):
    """The batch fr [F, H, W, 3] laid out in one byte buffer as `layout` says: (buffer uint8 [n], byte offset of frame 0, frame_stride, pitch).
    Bytes outside the frames' pixels (pitch padding, stride gaps, the bytes before an offset base) hold marker."""
    F, H, W, _ = fr.shape
    pitch, off = W * 3, 0
    stride = H * pitch
    if layout == 'pitch':
        pitch = W * 3 + 5
        stride = H * pitch
    elif layout == 'gap':
        pitch = W * 3 + 5
        stride = H * pitch + 4099
    elif layout == 'zero':
        stride = 0
    elif layout == 'offset':
        off = 1 + (W + H) % 3
        pitch = W * 3 + 5
        stride = H * pitch + 2
    elif layout != 'dense':
        raise ValueError(layout)
    nstored = 1 if stride == 0 else F
    buf = np.full(off + max(stride, H * pitch) * nstored + 64, marker, np.uint8)
    for f in range(nstored):
        base = off + f * stride
        for y in range(H):
            buf[base + y * pitch: base + y * pitch + W * 3] = fr[f, y].reshape(-1)
    return buf, off, stride, pitch


def expected_blobs(fr, layout):
    """The restatement's input blob of every frame of the call (stride 0: frame 0's, for every frame)"""
    ref = [DO.preprocess(f) for f in (fr[:1] if layout == 'zero' else fr)]
    return [ref[0 if layout == 'zero' else f] for f in range(len(fr))]


def plans(pp, bp, max_frames, flags=0):
    """The conv1x1 lines of a plan-only handle's describe() (detector_model.parse_plan)"""
    import detector_model as DM
    from pysgs import binding as B
    d = B.Detector(pp, bp, max_frames=max_frames, flags=flags | B.DET_PLAN_ONLY)
    try:
        return DM.parse_plan(d.describe())
    finally:
        d.close()


def pool_bytes(pp, bp, max_frames, flags):
    """Activation pool of a handle of max_frames frames, from the pool size per frame describe() reports"""
    from pysgs import binding as B
    d = B.Detector(pp, bp, max_frames=max_frames, flags=flags | B.DET_PLAN_ONLY)
    try:
        return int(d.describe().split()[7]) * 4 * max_frames
    finally:
        d.close()


def tiles_per_cta(p, frames_):
    """The fewest pixel tiles a persistent CTA of plan line p walks at frames_ frames per call (at most SM_TILES CTAs per output-channel tile)"""
    return -(-frames_ * p['h'] * p['w'] // 128) // SM_TILES


def bench_batches():
    """{config: (width, height, batch)} of the benchmark"""
    import bench
    return {k: (c['W'], c['H'], c['batch']) for k, c in bench.CONFIGS.items()}
