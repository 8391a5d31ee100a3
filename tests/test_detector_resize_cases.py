"""CPU checks of the detector's input-resize cases (tests/detector_resize_cases.py) and of the plans the detector runs at the benchmark's batch sizes.

  * the exact-half coefficient positions, per source size, pinned: these are the destination columns / rows where the rounding convention of the
    11-bit coefficients decides a weight (the project rounds half to even, as cv2 does; ncnn's from_pixels_resize at those points is unverified);
  * the half-rounding images separate the two conventions at every such column or row and nowhere else, and cv2 takes the half-to-even side;
  * the layouts put every pixel where (offset, frame_stride, pitch) says and the marker everywhere else;
  * plan-only handles of the reference model (when present), the mini graph and the wide-tail graph at 8 frames and at each benchmark batch: the
    persistent GEMM CTAs walk at least 100 pixel tiles each on the largest layers at the benchmark's batches, and the 8-vs-512 plan table."""
import os

import numpy as np
import pytest

import detector_model as DM
import detector_oracle as DO
import detector_resize_cases as RC

REAL = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle', '_ref', 'ncnn_model', 'mobilenetv3_ssdlite_voc')

# source size -> exact-half destination positions (of 300)
HALVES_640 = [240, 254, 255, 269, 270, 284, 285, 299]
HALF_COUNTS = {640: 8, 480: 0, 1280: 32, 720: 0, 752: 19, 1241: 35, 376: 9, 1920: 56, 1080: 6, 300: 0, 600: 0, 301: 8, 299: 8, 150: 0, 100: 0,
               2: 0}


def test_exact_half_positions_are_pinned():
    table = RC.half_table()
    print('\nexact-half coefficient positions (destination columns / rows of 300) per source size:')
    for n, pos in table.items():
        print('  %5d: %2d  %s' % (n, len(pos), ' '.join(map(str, pos))))
    assert list(table[640]) == HALVES_640
    assert {n: len(p) for n, p in table.items()} == HALF_COUNTS
    assert list(table[301]) == list(table[299])
    for n, pos in table.items():
        # at an exact half the two weights are k + 0.5 and 2047 - k + 0.5 (they sum to 2048): one of them has an even integer part, so the two
        # conventions give different coefficients at every exact-half position and agree everywhere else
        even, away = DO.resize_coeffs(RC.T, n)[1], DO.resize_coeffs(RC.T, n, DO.round_half_away)[1]
        assert list(np.nonzero((even != away).any(1))[0]) == list(pos), n
        assert (np.abs(even - away) <= 1).all() and (even.sum(1) == 2048).all() and (away.sum(1) == 2048 + (even != away).any(1)).all(), n


def test_rounding_helpers():
    for v, e, a in ((1160.5, 1160, 1161), (887.5, 888, 888), (0.5, 0, 1), (2.4999, 2, 2), (-0.5, 0, -1), (-1.5, -2, -2), (2047.5, 2048, 2048)):
        assert DO.round_half_even(v) == e and DO.round_half_away(v) == a, v


def _diff_mask(img):
    a = DO.preprocess(img)
    b = DO.preprocess(img, DO.round_half_away)
    return (a != b).any(0)                      # [dy][dx]


@pytest.mark.parametrize('w,h', [g for g in RC.GEOMETRIES if len(RC.exact_halves(RC.T, g[0])) or len(RC.exact_halves(RC.T, g[1]))])
def test_half_images_separate_the_conventions(w, h):
    """The two restatements differ on the half-rounding image, in every affected column and row and only there."""
    hx, hy = RC.exact_halves(RC.T, w), RC.exact_halves(RC.T, h)
    d = _diff_mask(RC.half_image(w, h))
    allowed = np.zeros_like(d)
    allowed[:, hx] = True
    allowed[hy, :] = True
    assert not (d & ~allowed).any(), 'differences outside the exact-half columns / rows'
    # every exact-half column differs in some row that is not itself an exact-half row, and likewise every exact-half row
    plain_rows = np.setdiff1d(np.arange(RC.T), hy); plain_cols = np.setdiff1d(np.arange(RC.T), hx)
    assert all(d[plain_rows, x].any() for x in hx), [x for x in hx if not d[plain_rows, x].any()]
    assert all(d[y, plain_cols].any() for y in hy), [y for y in hy if not d[y, plain_cols].any()]


@pytest.mark.parametrize('w,h', [(640, 480), (1280, 720), (752, 480), (1241, 376), (1920, 1080)])
def test_cv2_rounds_the_halves_to_even(w, h):
    """Shrinking on both axes (where cv2 4.13 and the restatement agree bit for bit, test_detector.py::test_resize_matches_cv2)."""
    cv2 = pytest.importorskip('cv2')
    img = RC.half_image(w, h)
    c = cv2.resize(img, (RC.T, RC.T), interpolation=cv2.INTER_LINEAR)
    assert np.array_equal(c, DO.resize_bilinear_u8c3(img, RC.T, RC.T))
    assert not np.array_equal(c, DO.resize_bilinear_u8c3(img, RC.T, RC.T, DO.round_half_away))


@pytest.mark.parametrize('layout', RC.LAYOUTS)
def test_layouts(layout):
    w, h, n = 7, 5, 3
    fr = RC.frames(w, h, n, 1)
    buf, off, stride, pitch = RC.pack(fr, layout)
    assert pitch >= 3 * w and 0 <= off <= 3
    assert {'dense': stride == h * pitch == h * w * 3, 'pitch': stride == h * pitch and pitch == 3 * w + 5, 'gap': stride > h * pitch, 'zero': stride == 0,
            'offset': 1 <= off <= 3}[layout]
    seen = np.zeros(len(buf), bool)
    for f in range(n):
        for y in range(h):
            at = off + f * stride + y * pitch
            assert buf[at: at + 3 * w].tobytes() == fr[0 if stride == 0 else f, y].tobytes()
            seen[at: at + 3 * w] = True
    assert (buf[~seen] == RC.MARKER).all() and (~seen).sum() >= (0 if layout in ('dense', 'zero') else n * h * 5)
    assert all(np.array_equal(e, DO.preprocess(fr[0 if layout == 'zero' else f])) for f, e in enumerate(RC.expected_blobs(fr, layout)))


def test_frames_are_distinct():
    for w, h in RC.GEOMETRIES:
        fr = RC.frames(w, h, 3, 0)
        assert len({f.tobytes() for f in fr}) == 3, (w, h)


# ---------------------------------------------------------------------------------------------------------------- plans at the benchmark's batches
def _graphs(tmp):
    g = [('mini', *DM.write_mini_model(os.path.join(tmp, 'mini'), 0)), ('wide_tails', *DM.write_wide_tail_model(os.path.join(tmp, 'wide'), 0)[:2])]
    if os.path.exists(REAL + '.param'):
        g.insert(0, ('reference', REAL + '.param', REAL + '.bin'))
    return g


def _key(p):
    return (p['nt'], p['n_tiles'], p['stages'], p['wres'])


def test_plans_at_the_benchmark_batches(tmp_path):
    batches = sorted({b for _, _, b in RC.bench_batches().values()})
    assert 512 in batches and 192 in batches
    changed = {}
    for name, pp, bp in _graphs(str(tmp_path)):
        small = RC.plans(pp, bp, RC.PROBE)
        print('\n%s: conv1x1 plans whose (NT, n_tiles, stages, wres) differ from those at %d frames:' % (name, RC.PROBE))
        for b in batches:
            big = RC.plans(pp, bp, b)
            assert [p['name'] for p in big] == [p['name'] for p in small]
            assert all((p['bk'], p['kb']) == (q['bk'], q['kb']) for p, q in zip(big, small)), 'the k-blocking depends on Cin only'
            diff = [(p, q) for p, q in zip(small, big) if _key(p) != _key(q)]
            changed[(name, b)] = len(diff)
            for p, q in diff:
                print('  %4d frames  %-28s %4d -> %4d @ %3dx%-3d  NT %3d x %d st %d%s  ->  NT %3d x %d st %d%s' % (
                    b, p['name'][:28], p['cin'], p['cout'], p['h'], p['w'], p['nt'], p['n_tiles'], p['stages'], ' wres' if p['wres'] else '',
                    q['nt'], q['n_tiles'], q['stages'], ' wres' if q['wres'] else ''))
            # the largest layers: every persistent CTA walks 80 to 100 pixel tiles or more at 512 frames (a few at 8 frames)
            top = max(RC.tiles_per_cta(q, b) for q in big)
            few = max(RC.tiles_per_cta(p, RC.PROBE) for p in small)
            print('  %4d frames: %d plans differ; largest layer %d pixel tiles per persistent CTA (%d at %d frames)' % (b, len(diff), top, few, RC.PROBE))
            if b == 512:
                assert top >= RC.SCALE_TILES[name] and few < 10, (name, top, few)
    if any(n == 'reference' for n, _ in changed):
        assert changed[('reference', 512)] >= 1, 'the planner picks the same tiling at 8 and 512 frames'
    assert changed[('mini', 512)] == 0            # at most 126 output channels: one tile whatever the batch
