"""lk_track_kernel and the padded pyramid it reads, bit for bit against the exact-sum restatement (tests/lk_exact.py), through all
three entry points.  No tolerance anywhere: every window sum is an exact integer sum and every float step an explicit
round-to-nearest intrinsic, so each tracked position must equal the restatement's to the last bit, and every padded image and
derivative plane (border included) byte for byte.  tests/test_lk_exact.py ties the restatement to cv2.

Sizes: every golden size (752x480, 1241x376, 641x481, 90x60, 43x43, 42x42) plus 640x480 and 24x24, so the scalar Scharr path,
the scalar pyrDown tail store, odd level widths and max_level 0 / 1 all run; and the large-flow, flat, 0/255 noise and checker pairs."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import lk_exact as X  # noqa: E402
from pysgs import binding as B  # noqa: E402

SIZES = X.GOLDEN_SIZES + X.EXTRA_SIZES


def _same(got, exp, pts, what):
    bad = np.nonzero((got.view(np.uint32) != exp.view(np.uint32)).any(1))[0]
    rows = [(int(i), pts[i].tolist(), got[i].tolist(), exp[i].tolist()) for i in bad[:10]]
    assert got.tobytes() == exp.tobytes(), (what, '%d of %d points differ' % (len(bad), len(pts)), rows)


def _check_planes(lk, frame, cur, prev, what):
    """Padded levels of batch frame `frame` (and its derivative planes) against the restatement; prev=None: J was not built."""
    for level, lv in enumerate(X.pyramid(cur)):
        img, der = lk.read_padded(0, level, frame)
        assert np.array_equal(img, X.padded(lv)), (what, 'I', level)
        assert np.array_equal(der, X.padded_deriv(lv)), (what, 'dI', level)
    if prev is not None:
        for level, lv in enumerate(X.pyramid(prev)):
            assert np.array_equal(lk.read_padded(1, level, frame)[0], X.padded(lv)), (what, 'J', level)


@pytest.mark.parametrize('name,cur,prev,pts', [pytest.param(*c, id=c[0]) for c in X.cases()])
def test_single_pair_bit_exact(name, cur, prev, pts):
    h, w = cur.shape
    lk = B.LK(w, h)
    try:
        got = lk.track(cur, prev, pts)
        exp, _ = X.track(cur, prev, pts)
        _same(got, exp, pts, name)
        _check_planes(lk, 0, cur, prev, name)
    finally:
        lk.close()


def _frames(w, h, seed):
    """Four distinct frames of one size: a stream pair and its mirror images."""
    cur, prev = X.image_pair(w, h, seed)
    return [cur, prev, np.ascontiguousarray(cur[::-1, ::-1]), np.ascontiguousarray(prev[:, ::-1])]


def _points(w, h, seed, nframes):
    base = X.point_set(w, h, seed + 100)
    return [base + np.float32(0.37 * f) for f in range(nframes)]


def _upload_frames(torch, frames, pitch, stride, rng):
    """The frames at `pitch` bytes per row and `stride` bytes per frame; the bytes between rows and frames are random."""
    h, w = frames[0].shape
    buf = rng.randint(0, 256, len(frames) * stride + pitch).astype(np.uint8)
    for f, img in enumerate(frames):
        for y in range(h):
            buf[f * stride + y * pitch:f * stride + y * pitch + w] = img[y]
    return torch.from_numpy(buf).cuda()


def _run_batch(torch, lk, d_cur, d_prev, prev_index, nframes, stride, pitch, pts, counts, cap):
    kps = np.zeros((nframes, cap), B.KP_DTYPE)
    for f in range(nframes):
        m = min(len(pts[f]), cap)
        kps[f, :m]['x'], kps[f, :m]['y'] = pts[f][:m, 0], pts[f][:m, 1]
    d_kps = torch.from_numpy(kps.view(np.uint8).reshape(-1)).cuda()
    d_counts = torch.from_numpy(np.asarray(counts, np.int32)).cuda()
    sentinel = np.full((nframes, cap, 2), -12345.5, np.float32)
    out = torch.from_numpy(sentinel).cuda()
    d_pidx = torch.from_numpy(np.asarray(prev_index, np.int32)).cuda() if prev_index is not None else None
    st = torch.cuda.Stream()
    torch.cuda.synchronize()
    lk.track_batch_device(d_cur.data_ptr(), d_prev.data_ptr() if d_prev is not None else 0, nframes, stride, pitch, d_kps.data_ptr(),
                          d_counts.data_ptr(), cap, out.data_ptr(), st.cuda_stream, d_prev_index=d_pidx.data_ptr() if d_pidx is not None else 0)
    st.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize('w,h,seed', SIZES)
@pytest.mark.parametrize('layout', ['odd_pitch', 'aligned'])
def test_batch_with_prev_bit_exact(w, h, seed, layout):
    """sgs_lk_track_batch_device with a second array of previous images.  'odd_pitch': pitch % 4 != 0 (the scalar Scharr path at
    level 0) and a frame stride that is no multiple of the pitch (the previous images are copied frame by frame);
    'aligned': 16-byte pitch and a stride of whole rows (one 3-D copy, the vector path wherever the width allows)."""
    import torch
    frames = _frames(w, h, seed)
    cur, prev = frames[:3], [frames[1], frames[0], frames[3]]
    if layout == 'odd_pitch':
        pitch = w + 1 if (w + 1) % 4 else w + 2
        stride = pitch * h + 37
    else:
        pitch = (w + 15) & ~15
        stride = pitch * (h + 1)
    pts = _points(w, h, seed, 3)
    cap = len(pts[0])
    counts = [cap, cap - 7, cap]
    rng = np.random.RandomState(seed)
    lk = B.LK(w, h, max_batch=3)
    try:
        d_cur = _upload_frames(torch, cur, pitch, stride, rng); d_prev = _upload_frames(torch, prev, pitch, stride, rng)
        got = _run_batch(torch, lk, d_cur, d_prev, None, 3, stride, pitch, pts, counts, cap)
        for f in range(3):
            n = counts[f]
            exp, _ = X.track(cur[f], prev[f], pts[f][:n])
            _same(got[f, :n], exp, pts[f], (w, h, layout, f))
            assert np.all(got[f, n:] == np.float32(-12345.5)), 'entries past counts[f] were written'
        for f in (0, 2):
            _check_planes(lk, f, cur[f], prev[f], (w, h, layout, f))
    finally:
        lk.close()


@pytest.mark.parametrize('w,h,seed', SIZES)
def test_batch_with_prev_index_bit_exact(w, h, seed):
    """sgs_lk_track_batch_device with d_prev_index: one pyramid serves as current and previous images (the tracker's and the
    benchmark's path).  A permutation with a frame that is its own previous frame, counts[f] == 0, and counts[f] > cap (clamped)."""
    import torch
    frames = _frames(w, h, seed)
    prev_index = [2, 0, 3, 3]
    pts = _points(w, h, seed, 4)
    cap = len(pts[0]) - 20
    counts = [cap, 0, cap + 50, cap - 3]
    pitch = w + 1 if (w + 1) % 4 else w + 2
    stride = pitch * h + 5
    lk = B.LK(w, h, max_batch=4)
    try:
        d_cur = _upload_frames(torch, frames, pitch, stride, np.random.RandomState(seed + 1))
        got = _run_batch(torch, lk, d_cur, None, prev_index, 4, stride, pitch, pts, counts, cap)
        for f in range(4):
            n = min(counts[f], cap)
            if n:
                exp, _ = X.track(frames[f], frames[prev_index[f]], pts[f][:n])
                _same(got[f, :n], exp, pts[f], (w, h, f))
            assert np.all(got[f, n:] == np.float32(-12345.5)), 'entries past counts[f] were written'
        for f in (0, 3):
            _check_planes(lk, f, frames[f], None, (w, h, f))
    finally:
        lk.close()
