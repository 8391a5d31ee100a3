"""Constructed cases for the dynamic-feature rejection (Frame::RmDynamicPointWithSemanticAndGeometry, src/Frame.cc:560-604) and a plain
restatement of it.  numpy only, no device.

The restatement follows CheckEpiLineDistToRmDynamicPoint (:613-627) and isInDynamicRegion (:629-652) one IEEE operation per step, in float64
with no FMA (numpy ufuncs round every multiply and add on its own), the box end r.x + r.w a float32 add, and the restore-all guard (:599)
`kept < nfeatures * 0.1` in double.  A case is one frame: the inputs, what the restatement says of them (keep, dist, nkeep, restored) and a
proof, a function that asserts the case really takes the path it is named for -- so that a case which drifted off its edge fails loudly
instead of passing for the wrong reason.

Batch-only inputs: `nboxes` is what the batch entry point is given for the frame (clamped there to [0, max_boxes]; the single-frame entry
point gets the clamped list), `count` the frame's keypoint count (clamped to [0, cap]).  nfeatures 0 keeps the restore guard from ever
firing, so that the verdicts show in the compacted output."""
import math
from fractions import Fraction

import numpy as np

MAX_BOXES = 4
IN_BOX, OUT_BOX = 0.2, 1.0
THRESHOLD_F = np.array([0, 0, 0, 0, 0, 1, 0, -1, 0], np.float64)   # a = 0, b = 1, c = -y: the distance is |py - y|
W, H = 640, 480
WHOLE_IMAGE = (-1.0, -1.0, W + 2.0, H + 2.0)
KEEP_D, BOX_D, DROP_D = 0.1, 0.5, 2.0      # |py - y| under THRESHOLD_F: kept anywhere, kept only outside a box, removed anywhere

f32 = np.float32


def up32(v):
    return np.nextafter(f32(v), f32(np.inf))


def down32(v):
    return np.nextafter(f32(v), f32(-np.inf))


# ---- the restatement ---------------------------------------------------------------------------------------------------------------

def box_count(nboxes, max_boxes=MAX_BOXES):
    return max(0, min(int(nboxes), max_boxes))


def in_any_box(xy, boxes, nboxes, max_boxes=MAX_BOXES):
    """isInDynamicRegion over the first nboxes boxes (clamped): x > r.x && x < fl32(r.x + r.w) && y > r.y && y < fl32(r.y + r.h)."""
    xy = np.asarray(xy, np.float32).reshape(-1, 2)
    x, y = xy[:, 0], xy[:, 1]
    inside = np.zeros(len(xy), bool)
    for r in np.asarray(boxes, np.float32).reshape(-1, 4)[:box_count(nboxes, max_boxes)]:
        rx, ry, rw, rh = (f32(v) for v in r)
        inside |= (x > rx) & (x < f32(rx + rw)) & (y > ry) & (y < f32(ry + rh))
    return inside


def epi_dist(cur, prev, F):
    """|a px + b py + c| / sqrt(a^2 + b^2) with (a, b, c) = F (x, y, 1), every product and sum rounded on its own."""
    c32 = np.asarray(cur, np.float32).reshape(-1, 2); p32 = np.asarray(prev, np.float32).reshape(-1, 2)
    x, y = c32[:, 0].astype(np.float64), c32[:, 1].astype(np.float64)
    px, py = p32[:, 0].astype(np.float64), p32[:, 1].astype(np.float64)
    F = np.asarray(F, np.float64)
    F = F.reshape(9) if F.size == 9 else F.reshape(-1, 9).T       # one F, or one per keypoint
    with np.errstate(all='ignore'):
        a = (x * F[0] + y * F[1]) + F[2]
        b = (x * F[3] + y * F[4]) + F[5]
        c = (x * F[6] + y * F[7]) + F[8]
        son = np.abs((a * px + b * py) + c)
        mom = np.sqrt(a * a + b * b)
        return son / mom


def restate(cur, prev, F, boxes, nboxes, have_dyn, nfeatures, max_boxes=MAX_BOXES):
    """(keep uint8 [n], dist float64 [n], nkeep, restored).  F None: the empty matrix (quirk Q11), everything kept, distances 0."""
    cur = np.asarray(cur, np.float32).reshape(-1, 2)
    n = len(cur)
    inb = in_any_box(cur, boxes, nboxes, max_boxes) if have_dyn else np.zeros(n, bool)
    if F is None:
        keep, dist = np.ones(n, bool), np.zeros(n)
    else:
        dist = epi_dist(cur, prev, F)
        keep = dist < np.where(inb, IN_BOX, OUT_BOX)          # NaN compares false: removed
    nkeep = int(keep.sum())
    return keep.astype(np.uint8), dist, nkeep, bool(have_dyn) and float(nkeep) < nfeatures * 0.1


def expected(c, n=None):
    """The restatement of case c over its first n keypoints (default: all)."""
    n = len(c['cur']) if n is None else n
    return restate(c['cur'][:n], c['prev'][:n], c['F'], c['boxes'], c['nboxes'], c['have_dyn'], c['nfeatures'])


def single_frame_boxes(c):
    """What the single-frame entry point is given: the boxes the batch kernel reads after clamping nboxes."""
    return np.asarray(c['boxes'], np.float32).reshape(-1, 4)[:box_count(c['nboxes'])]


# ---- the restatement with one operation changed: what a kernel that contracts or reorders the distance would compute -----------------

def fma(a, b, c):
    """a * b + c rounded once (exact rational arithmetic, then one rounding to double)."""
    return float(Fraction(a) * Fraction(b) + Fraction(c))


def _lin(u, v, F, i, variant, tag):
    if variant == 'fma_' + tag + '_x':
        return fma(u, F[i], v * F[i + 1]) + F[i + 2]
    if variant == 'fma_' + tag + '_y':
        return fma(v, F[i + 1], u * F[i]) + F[i + 2]
    return (u * F[i] + v * F[i + 1]) + F[i + 2]


def epi_dist_variant(x, y, px, py, F, variant):
    """One keypoint's distance with `variant` applied (None: the restatement itself, in Python floats)."""
    x, y, px, py = float(f32(x)), float(f32(y)), float(f32(px)), float(f32(py))
    F = [float(v) for v in np.asarray(F, np.float64).reshape(9)]
    a = _lin(x, y, F, 0, variant, 'a'); b = _lin(x, y, F, 3, variant, 'b'); c = _lin(x, y, F, 6, variant, 'c')
    if variant == 'fma_son_a':
        s = fma(a, px, b * py) + c
    elif variant == 'fma_son_b':
        s = fma(b, py, a * px) + c
    elif variant == 'son_reordered':
        s = a * px + (b * py + c)
    else:
        s = (a * px + b * py) + c
    if variant == 'fma_mom_a':
        m2 = fma(a, a, b * b)
    elif variant == 'fma_mom_b':
        m2 = fma(b, b, a * a)
    else:
        m2 = a * a + b * b
    son, mom = abs(s), math.sqrt(m2)
    return son * (1.0 / mom) if variant == 'reciprocal' else son / mom


VARIANTS = ('fma_a_x', 'fma_a_y', 'fma_b_x', 'fma_b_y', 'fma_c_x', 'fma_c_y', 'fma_son_a', 'fma_son_b', 'fma_mom_a', 'fma_mom_b',
            'son_reordered', 'reciprocal')


# ---- case construction -------------------------------------------------------------------------------------------------------------

CASES = []


def _case(name, cur, prev, F, boxes=(), have_dyn=False, nfeatures=0, nboxes=None, count=None, proof=None, follower=None,
          register=True):
    cur = np.asarray(cur, np.float32).reshape(-1, 2); prev = np.asarray(prev, np.float32).reshape(-1, 2)
    boxes = np.asarray(boxes, np.float32).reshape(-1, 4)
    assert len(cur) == len(prev) and len(boxes) <= MAX_BOXES, name
    c = dict(name=name, cur=cur, prev=prev, F=None if F is None else np.asarray(F, np.float64).reshape(9), boxes=boxes,
             nboxes=len(boxes) if nboxes is None else nboxes, have_dyn=bool(have_dyn), nfeatures=nfeatures,
             count=len(cur) if count is None else count, follower=follower)
    c['keep'], c['dist'], c['nkeep'], c['restored'] = expected(c)
    c['proof'] = (lambda: proof(c)) if proof else (lambda: None)
    if register:
        CASES.append(c)
    return c


def _box_around(x, y, r=1.0):
    return (x - r, y - r, 2 * r, 2 * r)


def _with(c, **over):
    """The restatement of c with some inputs changed (for proofs)."""
    d = dict(c, **over)
    return restate(d['cur'], d['prev'], d['F'], d['boxes'], d['nboxes'], d['have_dyn'], d['nfeatures'])


def _threshold_cases():
    # (A) THRESHOLD_F, distances at the float32 neighbours of 0.2 (on the row y = 0 the distance is the float32 py itself; on y = 240 it is
    # a multiple of 2^-16), each inside a box and outside
    lo0, hi0 = down32(0.2), f32(0.2)                               # f32(0.2) > 0.2 (double)
    hi240 = down32(240.2)
    while float(hi240) - 240.0 <= 0.2:
        hi240 = up32(hi240)
    lo240 = down32(hi240)
    ys = [0.0, 0.0, 240.0, 240.0]; pys = [lo0, hi0, lo240, hi240]
    xs = [50.0, 150.0, 250.0, 350.0]
    cur = np.stack([xs, ys], 1); prev = np.stack([xs, pys], 1)

    def near_02(c, inside):
        d = c['dist']
        assert d[0] < 0.2 < d[1] and d[2] < 0.2 < d[3], d
        assert d[0] == float(lo0) and d[1] == float(hi0) and d[3] - d[2] == 2.0 ** -16, 'adjacent representable distances'
        assert in_any_box(c['cur'], c['boxes'], len(c['boxes'])).tolist() == [inside] * 4
        assert c['keep'].tolist() == ([1, 0, 1, 0] if inside else [1, 1, 1, 1])
    _case('epi_f32_neighbours_of_0.2_in_box', cur, prev, THRESHOLD_F, [_box_around(x, y) for x, y in zip(xs, ys)], have_dyn=True,
          proof=lambda c: near_02(c, True))
    _case('epi_f32_neighbours_of_0.2_outside_box', cur, prev, THRESHOLD_F, [(500, 300, 50, 50)], have_dyn=True, proof=lambda c: near_02(c, False))

    # (B) THRESHOLD_F, distance exactly 1.0 (py - y = 1) and exactly nextafter(1.0, 0) (y = 2^-53, py = 1: 1 - 2^-53 is a double)
    tiny = f32(2.0 ** -53)
    cur = np.array([[60, 0.0], [160, tiny], [260, 100.0], [360, 0.0], [460, tiny]], np.float32)
    prev = np.array([[60, 1.0], [160, 1.0], [260, 101.0], [360, 1.0], [460, 1.0]], np.float32)
    boxes = [_box_around(360, 0.0), _box_around(460, 0.0)]

    def exactly_one(c):
        assert c['dist'].tolist() == [1.0, np.nextafter(1.0, 0), 1.0, 1.0, np.nextafter(1.0, 0)], c['dist']
        assert in_any_box(c['cur'], c['boxes'], 2).tolist() == [False, False, False, True, True]
        assert c['keep'].tolist() == [0, 1, 0, 0, 0]
    _case('epi_exactly_1.0_and_below', cur, prev, THRESHOLD_F, boxes, have_dyn=True, proof=exactly_one)

    # (C) THRESHOLD_F with F[8] = t: on the row y = 0 with py = 0, +-ulp the distance is t's double neighbours and t itself
    for t, thr_name, inside in ((0.2, '0.2', True), (1.0, '1.0', False)):
        F = THRESHOLD_F.copy(); F[8] = t
        below, above = np.nextafter(t, 0) - t, np.nextafter(t, 2) - t        # 2^-55, 2^-55 at 0.2; -2^-53, 2^-52 at 1.0
        xs = [100.0, 200.0, 300.0]
        cur = np.array([[x, 0.0] for x in xs], np.float32); prev = np.array([[7.0, below], [7.0, 0.0], [7.0, above]], np.float32)
        boxes = [_box_around(x, 0.0) for x in xs] if inside else [(0, 100, 640, 380)]

        def exact(c, t=t, inside=inside):
            assert c['dist'].tolist() == [np.nextafter(t, 0), t, np.nextafter(t, 2)], c['dist']
            assert in_any_box(c['cur'], c['boxes'], len(c['boxes'])).tolist() == [inside] * 3
            assert c['keep'].tolist() == [1, 0, 0]
        _case('epi_double_neighbours_of_%s_%s_box' % (thr_name, 'in' if inside else 'outside'), cur, prev, F, boxes, have_dyn=True, proof=exact)


def _assert(cond, msg=''):
    assert cond, msg
    return True


def _near_threshold(thr, seed, n=200000):
    """Keypoints, previous points and general Fs (a, b != 0, the magnitudes of a real fundamental matrix) whose restated distance lies
    within one ulp of thr: seeded draws with F[8] solved for the distance, kept where the rounded distance landed that close."""
    rng = np.random.RandomState(seed)
    x, y, px, py = (rng.uniform(20, hi, n).astype(np.float32).astype(np.float64) for hi in (620, 460, 620, 460))
    F = np.stack([rng.normal(0, s, n) for s in (1e-5, 1e-4, 1e-2, 1e-4, 1e-5, 1e-2, 1e-2, 1e-2, 0)], 1)
    a = (x * F[:, 0] + y * F[:, 1]) + F[:, 2]; b = (x * F[:, 3] + y * F[:, 4]) + F[:, 5]
    F[:, 8] = (thr * np.sqrt(a * a + b * b) - (a * px + b * py)) - (x * F[:, 6] + y * F[:, 7])
    d = epi_dist(np.stack([x, y], 1), np.stack([px, py], 1), F)
    near = np.nonzero(np.abs(d - thr) <= np.spacing(thr))[0]
    return [((x[k], y[k]), (px[k], py[k]), F[k]) for k in near]


def _general_f_cases():
    hits = {thr: _near_threshold(thr, 1000 + int(1000 * thr)) for thr in (IN_BOX, OUT_BOX)}
    for variant in VARIANTS:
        for thr, inside in ((IN_BOX, True), (OUT_BOX, False)):
            for k, (xy, pxy, F) in enumerate(hits[thr]):
                if (epi_dist_variant(*xy, *pxy, F, None) < thr) != (epi_dist_variant(*xy, *pxy, F, variant) < thr):
                    del hits[thr][k]
                    break
            else:
                raise AssertionError('no general-F point found for %s at %g' % (variant, thr))
            boxes = [_box_around(*xy)] if inside else [(0, 0, 5, 5)]

            def flips(c, variant=variant, thr=thr, inside=inside):
                (x, y), (px, py) = c['cur'][0], c['prev'][0]
                F = c['F']
                assert F[0] != 0 and abs(F[0]) < 1 and in_any_box(c['cur'], c['boxes'], 1)[0] == inside
                a = (float(x) * F[0] + float(y) * F[1]) + F[2]; b = (float(x) * F[3] + float(y) * F[4]) + F[5]
                assert a != 0 and b != 0, 'a general line'
                d = c['dist'][0]
                assert abs(d - thr) <= np.spacing(thr) and d == epi_dist_variant(x, y, px, py, F, None), d
                assert (d < thr) != (epi_dist_variant(x, y, px, py, F, variant) < thr), 'the variant flips the verdict'
            _case('epi_general_F_%s_near_%g' % (variant, thr), [xy], [pxy], F, boxes, have_dyn=True, proof=flips)


def _box_edge_cases():
    # x from 100.1 + 50.3 and y from 120.3 + 40.7: both float32 adds round DOWN, so a box end computed in double would contain the
    # keypoint placed on the float32 end.  Points at |py - y| = 0.5: removed inside a box, kept outside.
    for name, (rx, rw, ry, rh) in (('rounds_down', (100.1, 50.3, 120.3, 40.7)), ('rounds_up', (0.1, 0.2, 0.1, 0.2))):
        rx, rw, ry, rh = (f32(v) for v in (rx, rw, ry, rh))
        ex, ey = f32(rx + rw), f32(ry + rh)
        mx, my = f32(rx + rw / 2), f32(ry + rh / 2)
        xs = [rx, up32(rx), ex, down32(ex), mx, mx, mx, mx]
        ys = [my, my, my, my, ry, up32(ry), ey, down32(ey)]
        inside = [False, True, False, True, False, True, False, True]
        cur = np.stack([xs, ys], 1).astype(np.float32)
        prev = cur.copy(); prev[:, 1] = cur[:, 1] + f32(BOX_D)

        def edges(c, ex=ex, ey=ey, rx=rx, rw=rw, ry=ry, rh=rh, name=name, inside=inside):
            exact_x, exact_y = Fraction(float(rx)) + Fraction(float(rw)), Fraction(float(ry)) + Fraction(float(rh))
            if name == 'rounds_down':
                assert Fraction(float(ex)) < exact_x and Fraction(float(ey)) < exact_y, 'the float32 end lies below the real end'
            else:
                assert Fraction(float(ex)) > exact_x and Fraction(float(ey)) > exact_y, 'the float32 end lies above the real end'
            assert in_any_box(c['cur'], c['boxes'], 1).tolist() == inside
            assert ((0.2 < c['dist']) & (c['dist'] < 1.0)).all()
            assert c['keep'].tolist() == [0 if i else 1 for i in inside]
        _case('box_edges_float32_end_%s' % name, cur, prev, THRESHOLD_F, [(rx, ry, rw, rh)], have_dyn=True, proof=edges)

    # zero-width and zero-height boxes contain nothing, not even their own corner
    cur = np.array([[200, 210], [up32(200), 210], [300, 310], [300, up32(310)]], np.float32)
    prev = cur.copy(); prev[:, 1] += f32(BOX_D)
    boxes = [(200, 200, 0, 20), (290, 310, 20, 0)]

    def zero(c):
        assert not in_any_box(c['cur'], c['boxes'], 2).any() and c['keep'].all()
        widened = c['boxes'].copy(); widened[0, 2] = 1; widened[1, 3] = 1
        assert in_any_box(c['cur'], widened, 2).tolist() == [False, True, False, True], 'the points lie where a box of width 1 would hold them'
    _case('box_zero_width_and_height', cur, prev, THRESHOLD_F, boxes, have_dyn=True, proof=zero)

    # overlapping boxes; a point inside only the last of four boxes
    cur = np.array([[105, 105], [95, 95], [115, 115], [130, 130], [400, 400], [10, 470]], np.float32)
    prev = cur.copy(); prev[:, 1] += f32(BOX_D)
    boxes = [(90, 90, 20, 20), (100, 100, 20, 20), (500, 10, 30, 30), (380, 380, 40, 40)]

    def overlap(c):
        per_box = [in_any_box(c['cur'], c['boxes'][b:b + 1], 1).tolist() for b in range(4)]
        assert per_box[0] == [True, True, False, False, False, False] and per_box[1] == [True, False, True, False, False, False]
        assert per_box[3] == [False, False, False, False, True, False] and not any(per_box[2])
        assert c['keep'].tolist() == [0, 0, 0, 1, 0, 1]
    _case('box_overlapping_and_only_the_last', cur, prev, THRESHOLD_F, boxes, have_dyn=True, proof=overlap)


def _boxes_ignored_cases():
    rng = np.random.RandomState(7)
    cur = np.stack([rng.uniform(10, W - 10, 40), rng.uniform(10, H - 10, 40)], 1).astype(np.float32)
    prev = cur.copy(); prev[:, 1] += f32(BOX_D)
    whole = [WHOLE_IMAGE] * 4

    def all_kept_but(c, **over):
        assert c['keep'].all() and c['nkeep'] == len(c['cur'])
        assert not _with(c, **over)[0].any(), 'the ignored boxes would remove every point'
    # nboxes 7 > max_boxes 4: the batch kernel clamps; unclamped it would read the next frame's boxes, which cover the image
    small = [(0, 0, 3, 3), (5, 0, 3, 3), (10, 0, 3, 3), (15, 0, 3, 3)]

    def clamped(c):
        assert c['keep'].all()
        assert not restate(c['cur'], c['prev'], c['F'], np.concatenate([c['boxes'], np.array(whole, np.float32)]), 7, True, 0, 8)[0].any(), \
            'the boxes past max_boxes would remove every point'
    _case('boxes_nboxes_above_max_boxes', cur, prev, THRESHOLD_F, small, have_dyn=True, nboxes=7, proof=clamped,
          follower='boxes_have_dyn_0_with_boxes')
    _case('boxes_have_dyn_0_with_boxes', cur, prev, THRESHOLD_F, whole, have_dyn=False, proof=lambda c: all_kept_but(c, have_dyn=True))
    _case('boxes_nboxes_0_with_have_dyn', cur, prev, THRESHOLD_F, whole, have_dyn=True, nboxes=0, proof=lambda c: all_kept_but(c, nboxes=4))
    _case('boxes_whole_image_box_past_nboxes', cur, prev, THRESHOLD_F, [(0, 0, 3, 3), WHOLE_IMAGE], have_dyn=True, nboxes=1,
          proof=lambda c: all_kept_but(c, nboxes=2))
    _case('boxes_negative_nboxes', cur, prev, THRESHOLD_F, whole, have_dyn=True, nboxes=-3, proof=lambda c: all_kept_but(c, nboxes=4))


def prev_for(cur, pattern, box=None):
    """Previous points that give keypoints `cur` the verdicts `pattern` under THRESHOLD_F (1 kept: |py - y| 0.5 outside the box, 0.1
    inside; 0 removed: 2.0)."""
    cur = np.asarray(cur, np.float32).reshape(-1, 2)
    inb = in_any_box(cur, [box], 1) if box is not None else np.zeros(len(cur), bool)
    d = np.where(np.asarray(pattern, bool), np.where(inb, KEEP_D, BOX_D), DROP_D).astype(np.float32)
    prev = cur.copy(); prev[:, 1] = cur[:, 1] + d
    return prev


def _verdict_frame(pattern, seed, box=None):
    """Keypoints at seeded positions with the verdicts `pattern` (prev_for)."""
    rng = np.random.RandomState(seed)
    n = len(pattern)
    cur = np.stack([rng.uniform(0, W, n), rng.uniform(0, H, n)], 1).astype(np.float32)
    return cur, prev_for(cur, pattern, box)


def large_frame(n, kind='runs'):
    """A frame of n keypoints with the shape pattern `kind`, kept out of CASES (for the capacity limit of the batch entry point)."""
    pattern = shape_pattern(kind, n)
    cur, prev = _verdict_frame(pattern, 7000 + n)
    return _case('large_n%d_%s' % (n, kind), cur, prev, THRESHOLD_F, [], proof=lambda c: _assert(c['keep'].tolist() == pattern.tolist()),
                 register=False)


def _restore_cases():
    box = (200, 150, 200, 200)
    for nf, kept, restored in ((1000, 100, False), (1000, 99, True), (1005, 101, False), (1005, 100, True)):
        pattern = np.zeros(160, np.uint8); pattern[np.random.RandomState(kept).permutation(160)[:kept]] = 1
        cur, prev = _verdict_frame(pattern, nf + kept, box)

        def guard(c, nf=nf, kept=kept, restored=restored, pattern=pattern):
            assert c['keep'].tolist() == pattern.tolist() and c['nkeep'] == kept and c['restored'] == restored
            assert in_any_box(c['cur'], c['boxes'], 1).any(), 'some kept points lie in the box'
            assert abs(kept - nf * 0.1) <= 1, 'at the bound'
            if nf == 1000 and not restored:
                assert float(kept) == nf * 0.1, 'on the bound: <= would restore'
            if nf == 1005 and restored:
                assert kept == nf // 10, 'integer nfeatures / 10 would not restore'
        _case('restore_nf%d_keep%d' % (nf, kept), cur, prev, THRESHOLD_F, [box], have_dyn=True, nfeatures=nf, proof=guard)
    cur, prev = _verdict_frame(np.zeros(50, np.uint8), 77, box)
    _case('restore_have_dyn_0_keep0', cur, prev, THRESHOLD_F, [box], have_dyn=False, nfeatures=1000,
          proof=lambda c: _assert(c['nkeep'] == 0 and not c['restored'] and _with(c, have_dyn=True)[3]))
    # a negative keypoint count: an empty frame in the batch (counts_out 0) even though the guard fires for it
    _case('restore_negative_count', cur[:0], prev[:0], THRESHOLD_F, [box], have_dyn=True, nfeatures=1000, count=-5,
          proof=lambda c: _assert(c['nkeep'] == 0 and c['restored']))


def _degenerate_f_cases():
    rng = np.random.RandomState(11)
    n = 24
    cur = np.stack([rng.uniform(10, W - 10, n), rng.uniform(10, H - 10, n)], 1).astype(np.float32)
    prev = (cur + rng.uniform(-0.3, 0.3, (n, 2))).astype(np.float32)
    box = [(0, 0, W / 2, H)]

    def empty(c):
        assert c['keep'].all() and (c['dist'] == 0).all()
        as_matrix = np.array([np.nan, 0, 0, 0, 0, 1, 0, -1, 0])
        assert not _with(c, F=as_matrix)[0].any(), 'read as a matrix, the NaN marker would remove every point'
    _case('F_empty', cur, prev, None, box, have_dyn=True, proof=empty)
    F = THRESHOLD_F.copy(); F[4] = np.nan
    _case('F_nan_past_the_marker', cur, prev, F, box, have_dyn=True, proof=lambda c: _assert(np.isnan(c['dist']).all() and not c['keep'].any()))
    _case('F_all_zero', cur, prev, np.zeros(9), box, have_dyn=True, proof=lambda c: _assert(np.isnan(c['dist']).all() and not c['keep'].any()))
    F = np.zeros(9); F[8] = 1.0
    _case('F_no_line_anywhere', cur, prev, F, box, have_dyn=True, proof=lambda c: _assert(np.isinf(c['dist']).all() and not c['keep'].any()))
    # a = x - x0, b = y - y0, c = 1: at (x0, y0) the line is 0 = 1 (distance 1 / 0); elsewhere (prev 0, 0) the distance is 1 / |(x, y) - (x0, y0)|
    x0, y0 = cur[0]
    F = np.array([1, 0, -float(x0), 0, 1, -float(y0), 0, 0, 1], np.float64)
    p0 = np.zeros_like(cur)

    def one_point(c, x0=x0, y0=y0):
        assert (c['cur'][0] == (x0, y0)).all() and np.isinf(c['dist'][0]) and c['keep'][0] == 0
        assert np.all(np.hypot(c['cur'][1:, 0] - x0, c['cur'][1:, 1] - y0) >= 5) and c['keep'][1:].all()
    _case('F_no_line_through_one_point', cur, p0, F, [], proof=one_point)
    bad = prev.copy()
    bad[1] = (np.nan, bad[1, 1]); bad[3] = (bad[3, 0], np.nan); bad[5] = (np.inf, bad[5, 1]); bad[7] = (bad[7, 0], -np.inf)
    prev_ok = cur.copy(); prev_ok[:, 1] += f32(KEEP_D)
    bad_t = prev_ok.copy(); bad_t[[1, 3, 5, 7]] = bad[[1, 3, 5, 7]]

    def nonfinite(c):
        assert not c['keep'][[1, 3, 5, 7]].any() and c['keep'][[0, 2, 4, 6]].all()
        assert np.isnan(c['dist'][[1, 3, 5]]).all() and np.isinf(c['dist'][7]), 'under a = 0, 0 * inf is NaN'
    _case('prev_point_nan_and_inf', cur, bad_t, THRESHOLD_F, box, have_dyn=True, proof=nonfinite)


SHAPE_NS = (0, 1, 31, 32, 255, 256, 257, 511, 1100)


def shape_pattern(kind, n):
    """1 kept, 0 removed"""
    i = np.arange(n)
    if kind == 'none_removed':
        return np.ones(n, np.uint8)
    if kind == 'all_removed':
        return np.zeros(n, np.uint8)
    if kind == 'alternate':
        return (i % 2 == 0).astype(np.uint8)
    if kind == 'runs':            # removed runs that straddle lane 32 and thread 256 boundaries: [20, 45), [250, 270), [500, 530), [760, 800)
        rm = ((i >= 20) & (i < 45)) | ((i >= 250) & (i < 270)) | ((i >= 500) & (i < 530)) | ((i >= 760) & (i < 800))
        return (~rm).astype(np.uint8)
    if kind == 'first_removed':
        return (i != 0).astype(np.uint8)
    if kind == 'last_removed':
        return (i != n - 1).astype(np.uint8)
    raise ValueError(kind)


SHAPE_KINDS = ('none_removed', 'all_removed', 'alternate', 'runs', 'first_removed', 'last_removed')


def _shape_cases():
    for n in SHAPE_NS:
        for kind in SHAPE_KINDS if n else ('none_removed',):
            pattern = shape_pattern(kind, n)
            cur, prev = _verdict_frame(pattern, 5000 + n)
            _case('shape_n%d_%s' % (n, kind), cur, prev, THRESHOLD_F, [], proof=lambda c, p=pattern: _assert(c['keep'].tolist() == p.tolist()))
    # a count above the capacity (the batch runs give this case a capacity of exactly its 1100 keypoints)
    pattern = shape_pattern('runs', 1100)
    cur, prev = _verdict_frame(pattern, 6100)
    _case('shape_count_above_cap', cur, prev, THRESHOLD_F, [], count=1500,
          proof=lambda c: _assert(c['count'] > len(c['cur']) and c['keep'].tolist() == pattern.tolist()))


_threshold_cases()
_general_f_cases()
_box_edge_cases()
_boxes_ignored_cases()
_restore_cases()
_degenerate_f_cases()
_shape_cases()

BY_NAME = {c['name']: c for c in CASES}
assert len(BY_NAME) == len(CASES), 'case names are unique'
