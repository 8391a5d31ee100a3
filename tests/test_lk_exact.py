"""The exact-sum LK restatement (tests/lk_exact.py) against the real cv2, on the CPU.  tests/test_gpu_lk_exact.py pins the kernel to
the restatement bit for bit; this file pins the restatement to cv2, so together they carry the kernel's cv2 semantics.
- Pyramid levels, Scharr planes and the level count are integer results: equal to cv2 bit for bit at every golden size and level.
- Tracked positions: cv2 sums in float in SIMD order, the restatement exactly, so they meet the tolerance tests/test_gpu_lk.py
  states for the kernel.
- The test cases reach every branch of the tracker, and the largest per-lane window sum stays inside warp_sum_exact's range."""
import os

import numpy as np
import pytest

import lk_exact as X
import oracle as O

# tests/test_gpu_lk.py: median / 99th percentile / every point, and at most 0.3 % of the points beyond 0.02 px
TOL_MAX, TOL_OUTLIER, TOL_P99, TOL_MEDIAN = 0.25, 0.02, 2e-3, 2e-4


def _check(mine, ref, pts):
    d = np.abs(mine - ref).max(1)
    bad = np.nonzero(d > TOL_OUTLIER)[0]
    rows = [(int(i), pts[i].tolist(), mine[i].tolist(), ref[i].tolist()) for i in bad]
    assert np.median(d) <= TOL_MEDIAN and np.quantile(d, 0.99) <= TOL_P99 and d.max() <= TOL_MAX, (np.median(d), np.quantile(d, 0.99), d.max(), rows)
    assert len(bad) <= max(1, int(0.003 * len(d))), rows


@pytest.fixture(scope='module')
def sizes_golden(golden_dir):
    return np.load(os.path.join(golden_dir, 'lk_sizes.npz'))


@pytest.mark.parametrize('w,h,seed', X.GOLDEN_SIZES)
def test_pyramid_and_scharr_equal_cv2(sizes_golden, w, h, seed):
    g = sizes_golden
    key = '%dx%d' % (w, h)
    cur, prev = X.image_pair(w, h, seed)
    assert [X.digest(cur), X.digest(prev)] == list(g[key + '_images']), 'the seeded test images changed'
    sizes = X.level_sizes(w, h)
    assert len(sizes) - 1 == int(g[key + '_max_level'])
    assert [l.shape[::-1] for l in X.pyramid(cur)] == sizes
    lv = cur
    for level, (d_img, d_dx, d_dy) in enumerate(g[key + '_digests']):     # the cv2.pyrDown chain to level 3, kept or not
        if level:
            lv = X.pyr_down(lv)
        dx, dy = X.scharr(lv)
        assert (X.digest(lv), X.digest(dx), X.digest(dy)) == (d_img, d_dx, d_dy), (key, level)


def test_padded_border_equals_cv2():
    """The PAD-pixel REFLECT_101 border, also where it is wider than the level (22 px wide levels exist: 43x43 -> 22x22)."""
    cv2 = pytest.importorskip('cv2')
    rng = np.random.RandomState(3)
    for w, h in ((22, 22), (23, 40), (94, 60)):
        img = rng.randint(0, 256, (h, w)).astype(np.uint8)
        ref = cv2.copyMakeBorder(img, X.PAD, X.PAD, X.PAD, X.PAD, cv2.BORDER_REFLECT_101)
        assert np.array_equal(X.padded(img), ref), (w, h)


def test_tracks_match_cv2_golden_320x240(golden_dir):
    g = np.load(os.path.join(golden_dir, 'lk_320x240.npz'))
    out, _ = X.track(g['cur'], g['prev'], g['pts'])
    _check(out, g['tracked'], g['pts'])


@pytest.mark.parametrize('w,h,seed', X.GOLDEN_SIZES)
def test_tracks_match_cv2_golden_sizes(sizes_golden, w, h, seed):
    key = '%dx%d' % (w, h)
    cur, prev = X.image_pair(w, h, seed)
    pts = sizes_golden[key + '_pts']
    out, _ = X.track(cur, prev, pts)
    _check(out, sizes_golden[key + '_tracked'], pts)


def test_tracks_match_oracle_on_stream():
    from pysgs import synth
    frames, _ = synth.stream_s2(3, 640, 480, seed=2)
    for a, b in ((1, 0), (2, 1)):
        k, _ = O.extract(frames[a])
        pts = np.stack([k['x'], k['y']], 1).astype(np.float32)
        out, _ = X.track(frames[a], frames[b], pts)
        _check(out, O.lk_track(frames[a], frames[b], pts), pts)


@pytest.fixture(scope='module')
def tracked_cases():
    return [(name, cur, pts) + X.track(cur, prev, pts) for name, cur, prev, pts in X.cases()]


def test_cases_reach_every_branch(tracked_cases):
    total = {k: 0 for k in X.COUNTERS}
    for name, cur, pts, out, info in tracked_cases:
        for k in X.COUNTERS:
            total[k] += int(info[k].sum())
        sizes = X.level_sizes(cur.shape[1], cur.shape[0])
        for level in sorted({0, len(sizes) - 1}):
            lw, lh = sizes[level]
            for axis, lim in (('ipx', lw), ('ipy', lh)):
                seen = set(info[axis][:, level].tolist())
                assert {-X.WIN, lim - 1, -X.WIN - 1, lim} <= seen, (name, level, axis)
    print('branch counters over all cases:', total)
    assert all(total[k] > 0 for k in X.COUNTERS), total


def test_window_sums_fit_warp_sum_exact(tracked_cases):
    """warp_sum_exact adds per-lane int32 partials that must stay below 2^29.  The worst case, 15 pixels x 8160 x 4080, is 0.93 * 2^29;
    0/255 noise and the 2-pixel checker reach Scharr's +-4080 and the largest intensity differences."""
    worst = {name: info['max_lane'] for name, _, _, _, info in tracked_cases}
    print('largest per-lane partial (fraction of 2^29):', {k: round(v / 2.0 ** 29, 3) for k, v in worst.items()})
    assert max(worst.values()) < 1 << 29
    noise = [cur for name, cur, _, _, _ in tracked_cases if name == 'noise_200x120'][0]
    assert max(np.abs(d.astype(np.int32)).max() for d in X.scharr(noise)) == 4080
    # the contrast cases drive the sums well beyond the smooth images
    assert min(worst['noise_200x120'], worst['checker_200x120']) > 2 * max(v for k, v in worst.items() if k[0].isdigit())
