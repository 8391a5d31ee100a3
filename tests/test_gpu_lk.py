"""GPU parity of the LK stage (src/Frame.cc:445) through the C ABI against the CPU oracle and the cv2 golden vectors.
Integer stages (cv::pyrDown levels) are bit-exact; tracked positions are tolerance-based: the GPU sums the integer products
exactly and rounds once, OpenCV/the oracle accumulate in float, so iterations can differ in the last bits."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle as O  # noqa: E402
from pysgs import binding as B  # noqa: E402
from pysgs import synth  # noqa: E402

# pixels: median / 99th percentile as for the oracle vs cv2 (tests/test_lk.py); a converging iteration can stop one step apart when
# the float sums differ in the last bit, so a handful of points (<= 0.3 %) may differ by up to 0.25 px (thresholds downstream: 0.2 / 1.0 px)
TOL_MAX, TOL_OUTLIER, TOL_P99, TOL_MEDIAN = 0.25, 0.02, 2e-3, 2e-4


def _check(mine, ref):
    d = np.abs(mine - ref).max(1)
    assert np.median(d) <= TOL_MEDIAN and np.quantile(d, 0.99) <= TOL_P99 and d.max() <= TOL_MAX, (np.median(d), np.quantile(d, 0.99), d.max())
    assert (d > TOL_OUTLIER).sum() <= max(1, int(0.003 * len(d))), int((d > TOL_OUTLIER).sum())


def test_lk_against_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, 'lk_320x240.npz'))
    lk = B.LK(320, 240)
    try:
        got = lk.track(g['cur'], g['prev'], g['pts'])
        _check(got, g['tracked'])
        assert np.array_equal(lk.read_level(0, 3), g['pyr3'])
        for l in (1, 2, 3):
            assert np.array_equal(lk.read_level(0, l), O.lk_pyr_level(g['cur'], l))
            assert np.array_equal(lk.read_level(1, l), O.lk_pyr_level(g['prev'], l))
    finally:
        lk.close()


def test_lk_point_buffers_regrow(golden_dir):
    """sgs_lk_track on one handle with a small, a larger and again a small point count (the point buffers grow once): every result is what a
    fresh handle returns."""
    g = np.load(os.path.join(golden_dir, 'lk_320x240.npz'))
    pts = g['pts']
    lk = B.LK(320, 240)
    try:
        for sel in (pts[:40], pts, pts[-90:]):
            fresh = B.LK(320, 240)
            try:
                want = fresh.track(g['cur'], g['prev'], sel)
            finally:
                fresh.close()
            assert np.array_equal(lk.track(g['cur'], g['prev'], sel), want), len(sel)
    finally:
        lk.close()


def test_lk_against_oracle_on_stream():
    frames, _ = synth.stream_s2(3, 640, 480, seed=2)
    lk = B.LK(640, 480)
    try:
        for a, b in ((1, 0), (2, 1)):
            k, _ = O.extract(frames[a])
            pts = np.stack([k['x'], k['y']], 1).astype(np.float32)
            _check(lk.track(frames[a], frames[b], pts), O.lk_track(frames[a], frames[b], pts))
        # points whose window leaves the image / flat regions / identical images (zero flow)
        pts = np.array([[0.5, 0.5], [639.0, 479.0], [320.3, 2.2], [5.0, 470.0], [100.5, 100.5]], np.float32)
        _check(lk.track(frames[1], frames[0], pts), O.lk_track(frames[1], frames[0], pts))
        same = lk.track(frames[1], frames[1], pts)
        assert np.abs(same - pts).max() < 1e-3
        flat = np.full((480, 640), 90, np.uint8)
        assert np.array_equal(lk.track(flat, flat, pts), pts)      # min-eigenvalue gate: the input point comes back unchanged (A10)
    finally:
        lk.close()


def test_lk_batch_device_matches_single():
    import torch
    frames, _ = synth.stream_s2(4, 640, 480, seed=5)
    ex = B.Extractor(640, 480, max_batch=3)
    lk = B.LK(640, 480, max_batch=3)
    try:
        cur = torch.from_numpy(frames[1:4].copy()).cuda(); prev = torch.from_numpy(frames[0:3].copy()).cuda()
        st = torch.cuda.Stream(); torch.cuda.synchronize()
        ex.extract_batch_device(cur.data_ptr(), 3, 640 * 480, 640, st.cuda_stream)
        kptr, dptr, cptr, cap = ex.results_device()
        out = torch.zeros(3, cap, 2, dtype=torch.float32, device='cuda')
        lk.track_batch_device(cur.data_ptr(), prev.data_ptr(), 3, 640 * 480, 640, kptr, cptr, cap, out.data_ptr(), st.cuda_stream)
        st.synchronize()
        kps, desc, n = ex.fetch(3, st.cuda_stream)
        o = out.cpu().numpy()
        for f in range(3):
            pts = np.stack([kps[f, :n[f]]['x'], kps[f, :n[f]]['y']], 1)
            _check(o[f, :n[f]], O.lk_track(frames[1 + f], frames[f], pts))
    finally:
        ex.close(); lk.close()
