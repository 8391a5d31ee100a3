"""Constructed images for the ORB extractor (numpy only, no device): each image is built so that one named path of the FAST cells
(sg-slam_b200/csrc/fast_kernel.cu), the quadtree distribution (quadtree_core.h), the orientation / descriptor kernel (describe_kernel) or the
planner (orb_plan.cpp) MUST be taken.  Every case carries a proof -- an assertion on the oracle's per-stage output (oracle.ExtractDump) that
only holds if that path was taken -- so that an edit to a builder cannot quietly turn a case into an easy one.

The building block is the dot: one pixel of value b + s + 1 (or b - s - 1) on a flat background b is an isolated FAST corner of score
exactly s, and none of its neighbours is a corner.  Dots whose offsets are neither 8-adjacent nor on each other's 3-px ring give exactly the
planted candidate set with the planted scores.

A case is a dict: name, img (uint8 [h, w]), p (nfeatures, scale, nlevels, ini, mn as the extractor takes them), proof(dump), and a geometry
key (w, h, p) under which cases are batched together.  refusals() lists the parameter sets sgs_extractor_create must refuse, with the
status and a word of the message."""
import math

import numpy as np

import oracle as O

f32 = np.float32
MIN_BORDER = 16                       # EDGE_THRESHOLD - 3: FAST cells and candidate coordinates start here (src/ORBextractor.cc:786)
RING = [(0, 3), (1, 3), (2, 2), (3, 1), (3, 0), (3, -1), (2, -2), (1, -3), (0, -3), (-1, -3), (-2, -2), (-3, -1), (-3, 0), (-3, 1), (-2, 2), (-1, 3)]
RING_SET = set(RING)
QT_DEPTH = 12                         # divisions the device's path keys encode (kQtDepth)
SMEM_LIMIT, KEY_SMEM = 200 * 1024, 96 * 1024   # extractor.cu: shared-memory budget of the quadtree block and of its sort keys


def P(nfeatures=1000, scale=1.2, nlevels=1, ini=20, mn=7):
    return dict(nfeatures=nfeatures, scale=scale, nlevels=nlevels, ini=ini, mn=mn)


def oparams(p):
    return O.params(p['nfeatures'], p['scale'], p['nlevels'], p['ini'], p['mn'])


# ---- geometry restated from ComputeKeyPointsOctTree / DistributeOctTree / the extractor's quadtree budget --------------------------------
_CELLS = {}


def cells(w, h):
    """FAST cells of a level: (i, j, x0, y0, x1, y1) views in the reference's order (src/ORBextractor.cc:790-826), level coordinates.
    The interior -- where corners are reported -- is [x0 + 3, x1 - 3) x [y0 + 3, y1 - 3)."""
    if (w, h) not in _CELLS:
        mbx, mby = w - MIN_BORDER, h - MIN_BORDER
        W, H = mbx - MIN_BORDER, mby - MIN_BORDER
        nc, nr = W // 30, H // 30
        wc, hc = -(-W // nc), -(-H // nr)
        out = {}
        for i in range(nr):
            y0 = MIN_BORDER + i * hc
            if y0 >= mby - 3:
                continue
            y1 = min(y0 + hc + 6, mby)
            for j in range(nc):
                x0 = MIN_BORDER + j * wc
                if x0 >= mbx - 6:
                    continue
                out[i, j] = (i, j, x0, y0, min(x0 + wc + 6, mbx), y1)
        _CELLS[w, h] = (list(out.values()), out, wc, hc)
    return _CELLS[w, h][0]


def cell_of(w, h, x, y):
    """The cell whose interior holds level pixel (x, y), or None.  Interiors of neighbouring cells are adjacent and disjoint."""
    cells(w, h)
    _, by_ij, wc, hc = _CELLS[w, h]
    c = by_ij.get(((y - MIN_BORDER - 3) // hc, (x - MIN_BORDER - 3) // wc)) if x >= MIN_BORDER + 3 and y >= MIN_BORDER + 3 else None
    if c is not None and c[2] + 3 <= x < c[4] - 3 and c[3] + 3 <= y < c[5] - 3:
        return c
    return None


def qt_roots(w, h):
    """(n_ini, hX, root height) of DistributeOctTree (:544-560) for a level of w x h."""
    W, H = w - 2 * MIN_BORDER, h - 2 * MIN_BORDER
    n = int(round(float(f32(W) / f32(H))))
    return n, f32(W) / f32(n), H


def qt_root(w, h, x):
    """Root strip of a candidate at relative x: (int)(kp.pt.x / hX) (:571)."""
    n, hx, _ = qt_roots(w, h)
    return min(int(f32(x) / hx), n - 1)


def qt_path(w, h, x, y):
    """Child codes (bit 0 right, bit 1 bottom) of the reference's DivideNode for a candidate at relative (x, y), QT_DEPTH divisions deep."""
    n, hx, rh = qt_roots(w, h)
    r = qt_root(w, h, x)
    ulx, urx, uly, bry = int(hx * f32(r)), int(hx * f32(r + 1)), 0, rh
    codes = []
    for _ in range(QT_DEPTH):
        mx, my = ulx + math.ceil((urx - ulx) / 2), uly + math.ceil((bry - uly) / 2)
        bx, by = int(x >= mx), int(y >= my)
        codes.append(bx | by << 1)
        ulx, urx = (mx, urx) if bx else (ulx, mx)
        uly, bry = (my, bry) if by else (uly, my)
    return r, codes


def split_division(w, h, a, b):
    """1-based division at which two candidates (relative coordinates) first land in different children; 0 = different roots, None = never."""
    ra, ca = qt_path(w, h, *a)
    rb, cb = qt_path(w, h, *b)
    if ra != rb:
        return 0
    for d in range(QT_DEPTH):
        if ca[d] != cb[d]:
            return d + 1
    return None


def plan_levels(w, h, p):
    """Level sizes of ComputePyramid (cvRound(w * invScale), float arithmetic, from the oracle) and the scale tables."""
    t = O.orb_tables(oparams(p))
    return [O.level_size(oparams(p), w, h, l) for l in range(p['nlevels'])], t


def max_nlevels(w, h, scale, cap=16):
    for L in range(cap, 0, -1):
        sizes, _ = plan_levels(w, h, P(scale=scale, nlevels=L))
        if all(lw - 2 * MIN_BORDER >= 30 and lh - 2 * MIN_BORDER >= 30 and round((lw - 32) / (lh - 32)) >= 1 for lw, lh in sizes):
            return L
    return 0


def qt_node_cap(w, h, p):
    """Node capacity of the device quadtree: the largest qt_pool_cap over the levels (quadtree_core.h)."""
    sizes, t = plan_levels(w, h, p)
    cap = 0
    for (lw, lh), n in zip(sizes, t['nPerLevel']):
        ni = qt_roots(lw, lh)[0]
        cap = max(cap, 2 * max(int(n), 4 * ni) + 4 * ni + 16)
    return cap


def qt_node_bytes(cap):
    return (cap * 70 + 128 + 15) & ~15          # extract_kernels.cu qt_node_bytes, rounded to 16 as extractor.cu does


def qt_accepts(w, h, p):
    return qt_node_bytes(qt_node_cap(w, h, p)) + 8 * 1024 <= SMEM_LIMIT


def smem_key_cap(w, h, p):
    """Largest candidate count per level whose sort keys stay in shared memory (4096, 2048 or 1024 by nfeatures)."""
    nb, cap = qt_node_bytes(qt_node_cap(w, h, p)), 4096
    while nb + cap * 8 > KEY_SMEM and cap > 1024:
        cap >>= 1
    return cap


def max_nfeatures(w, h, p):
    """Largest nfeatures the shared-memory quadtree accepts for this geometry (binary search on the plan formulas)."""
    lo, hi = 1, 1 << 16
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if qt_accepts(w, h, dict(p, nfeatures=mid)):
            lo = mid
        else:
            hi = mid - 1
    return lo


# ---- images ----------------------------------------------------------------------------------------------------------------------------
def dots(w, h, pts, b=40):
    """Flat image b with dots (x, y, s[, sign]) in level-0 coordinates: value b + s + 1 (sign +1) or b - s - 1 (sign -1)."""
    img = np.full((h, w), b, np.int32)
    for d in pts:
        x, y, s = d[:3]
        sg = d[3] if len(d) > 3 else 1
        img[y, x] = b + sg * (s + 1)
    assert img.min() >= 0 and img.max() <= 255
    return img.astype(np.uint8)


def check_spacing(pts):
    """No dot on another's 3-px ring (8-adjacent pairs are built on purpose by the NMS cases and checked by their proofs)."""
    for a in range(len(pts)):
        for c in range(a + 1, len(pts)):
            dx, dy = pts[c][0] - pts[a][0], pts[c][1] - pts[a][1]
            assert (dx, dy) not in RING_SET and (-dx, -dy) not in RING_SET, (pts[a], pts[c])


# ---- proofs on the oracle's dump -------------------------------------------------------------------------------------------------------
def cand_set(d, lvl=0):
    c = d.cands[lvl]
    return {(int(x) + MIN_BORDER, int(y) + MIN_BORDER, int(s)) for x, y, s in c}


def kp_set(d, octave=0):
    k = d.kps[d.kps['octave'] == octave]
    return {(int(x), int(y), int(r)) for x, y, r in zip(k['x'], k['y'], k['response'])}


def exact_cands(expected, lvl=0):
    expected = {(int(x), int(y), int(s)) for x, y, s in expected}

    def proof(d):
        got = cand_set(d, lvl)
        assert got == expected, 'candidates: missing %s, extra %s' % (sorted(expected - got)[:6], sorted(got - expected)[:6])
    return proof


def all_of(*fs):
    def proof(d):
        for f in fs:
            f(d)
    return proof


def case(name, img, p, proof, **extra):
    return dict(name=name, img=np.ascontiguousarray(img, np.uint8), p=p, proof=proof, key=(img.shape[1], img.shape[0], tuple(sorted(p.items()))), **extra)


# ---- FAST ------------------------------------------------------------------------------------------------------------------------------
def interior_centres(w, h, n, step=12, margin=8):
    """The first n points of a grid of `step` px that lie in a cell interior, `margin` px away from the FAST border (level-0 coordinates)."""
    out = []
    for y in range(MIN_BORDER + 3 + margin, h - MIN_BORDER - 3 - margin, step):
        for x in range(MIN_BORDER + 3 + margin, w - MIN_BORDER - 3 - margin, step):
            if cell_of(w, h, x, y) is not None:
                out.append((x, y))
            if len(out) == n:
                return out
    raise AssertionError('image too small for %d points' % n)


def fast_threshold_cases():
    """Per-cell fallback and scores at the thresholds: in separate cells dots of score ini, ini - 1, mn, mn - 1; one cell holding an ini dot and a
    dot between mn and ini (the fallback must not run there).  Proof: the exact candidate set and the oracle's fallback count (every cell
    without a corner at ini falls back)."""
    out = []
    w, h = 640, 480
    cl = cells(w, h)
    for ini, mn in ((20, 7), (1, 1), (127, 126), (200, 130), (254, 254)):
        for sign in (1, -1):
            b = (0 if sign > 0 else 255) if ini > 100 else (40 if sign > 0 else 200)
            scores = sorted({ini, ini - 1, mn, mn - 1} - {0})
            pts = []
            for k, s in enumerate(scores):
                i, j, x0, y0, x1, y1 = cl[3 * k + 25]
                pts.append((x0 + 10, y0 + 12, s, sign))
            pair_cell = None
            if mn < ini:
                i, j, x0, y0, x1, y1 = pair_cell = cl[60]
                pts += [(x0 + 8, y0 + 8, ini, sign), (x0 + 20, y0 + 22, max(mn, ini - 5), sign)]
            check_spacing(pts)
            exp = [(x, y, s) for x, y, s, _ in pts if s >= mn and not (pair_cell and s < ini and cell_of(w, h, x, y) == pair_cell)]
            with_ini = {cell_of(w, h, x, y) for x, y, s, _ in pts if s >= ini}
            nfb = len(cl) - len(with_ini)

            def fb(d, nfb=nfb):
                assert d.nfallback == nfb, (d.nfallback, nfb)
            out.append(case('fast_th_%d_%d_%s' % (ini, mn, 'bright' if sign > 0 else 'dark'), dots(w, h, pts, b), P(ini=ini, mn=mn),
                            all_of(exact_cands(exp), fb)))
    return out


def fast_interior_edge_case():
    """Dots on the first and last interior column and row of every cell: the cells' x0 take every value mod 16, so the first and last
    interior word of the packed pre-test is masked at every tile offset.  Neighbouring cells' dots touch across each boundary (both kept:
    the NMS is cell-local).  Proof: the exact candidate set, and the x0 residues cover 0..15."""
    w, h = 640, 480
    cl = cells(w, h)
    assert {c[2] % 16 for c in cl} == set(range(16))
    pts = []
    for k, (i, j, x0, y0, x1, y1) in enumerate(cl):
        s = 20 + (k * 7) % 200
        fx, lx, fy, ly = x0 + 3, x1 - 4, y0 + 3, y1 - 4
        pts += [(fx, fy, s), (lx, ly, s + 1), (fx, ly, s + 2), (lx, fy, s)]
    return case('fast_interior_edges', dots(w, h, pts, 20), P(ini=20, mn=7), exact_cands(pts))


def fast_nms_cases():
    """Equal and unequal 8-adjacent dots inside a cell (equal: both suppressed; unequal: the higher kept) and straddling a cell boundary
    horizontally, vertically and diagonally (both kept whatever the scores).  Proof: the exact candidate set."""
    w, h = 640, 480
    cl = cells(w, h)
    pts, exp = [], []
    for k, (s1, s2) in enumerate(((30, 30), (30, 31), (45, 44))):
        i, j, x0, y0, x1, y1 = cl[45 + 2 * k]
        for dx, dy in ((1, 0), (0, 1), (1, 1), (1, -1)):
            bx, by = x0 + 6 + 6 * (dx + 1) * (dy + 2), y0 + 8 + 8 * (dy + 1)
            pts += [(bx, by, s1), (bx + dx, by + dy, s2)]
            if s1 > s2:
                exp.append((bx, by, s1))
            elif s2 > s1:
                exp.append((bx + dx, by + dy, s2))
    for k, (s1, s2) in enumerate(((30, 30), (30, 33))):
        i, j, x0, y0, x1, y1 = cl[130 + k]            # right / bottom neighbours exist
        lx, ly = x1 - 4, y1 - 4
        pr = [((lx, y0 + 10), (lx + 1, y0 + 10)), ((x0 + 10, ly), (x0 + 10, ly + 1)), ((lx, ly), (lx + 1, ly + 1))]
        for a, c in pr:
            assert cell_of(w, h, *a) != cell_of(w, h, *c)
            pts += [(a[0], a[1], s1), (c[0], c[1], s2)]
            exp += [(a[0], a[1], s1), (c[0], c[1], s2)]
    return case('fast_nms_adjacent', dots(w, h, pts, 60), P(ini=20, mn=7), exact_cands(exp))


def fast_arc_cases():
    """Arcs of 8 and 9 contiguous ring pixels at all 16 start positions (wrapping from 15 to 0), bright and dark.  The arc pixels differ from
    the background by 15 (never a corner at 20), the centre by 10 the other way, so the arc pixels differ from the centre by 25 and the other
    ring pixels by 10: the centre is a corner of score 24 exactly when its arc has 9 pixels.  Proof: the exact candidate set."""
    out = []
    w, h = 640, 480
    for sign in (1, -1):
        b = 100
        img = np.full((h, w), b, np.int32)
        cs = interior_centres(w, h, 32)
        exp = []
        for k, (cx, cy) in enumerate(cs):
            start, L = k % 16, 8 + k // 16
            img[cy, cx] = b - 10 * sign
            for q in range(L):
                dx, dy = RING[(start + q) % 16]
                img[cy + dy, cx + dx] = b + 15 * sign
            if L == 9:
                exp.append((cx, cy, 24))
        out.append(case('fast_arcs_%s' % ('bright' if sign > 0 else 'dark'), img.astype(np.uint8), P(ini=20, mn=20), exact_cands(exp)))
    return out


def fast_compass_cases():
    """Mixed-sign compass pixels, on ramps (a linear ramp has no FAST corner: the ring pixels beyond the threshold form one arc of at most 7).
    I = 128 + 8 * dy: every pixel of the ramp band has compass pixel 0 brighter and 8 darker by 24 > t (4 and 12 equal), so the packed
    sign-agnostic pre-test passes and the signed re-check fails.  I = 128 + 8 * |dy|: compass 0 and 8 are both brighter, the re-check passes
    and the segment test fails (two 3-pixel arcs).  Plus one dot in the clipped flat area.  Proof: the pre-test / re-check outcomes of the
    centre, restated, and the exact candidate set (the dot only)."""
    w, h, t = 640, 480, 20
    cx, cy = 300, 200
    yy, xx = np.mgrid[0:h, 0:w]
    out = []
    for name, ramp, dot in (('fast_compass_mixed_sign', yy - cy, (500, 100, 30, 1)), ('fast_compass_no_segment', np.abs(yy - cy), (100, 400, 30, -1))):
        img = np.clip(128 + 8 * ramp, 0, 255).astype(np.int32)
        x, y, s, sg = dot
        img[y, x] += sg * (s + 1)
        v = int(img[cy, cx])
        comp = [int(img[cy + dy, cx + dx]) - v for dx, dy in (RING[0], RING[4], RING[8], RING[12])]
        packed = sum(abs(c) > t for c in comp) >= 2
        signed = sum(c > t for c in comp) >= 2 or sum(c < -t for c in comp) >= 2
        assert packed and (signed == (name == 'fast_compass_no_segment'))
        out.append(case(name, img.astype(np.uint8), P(ini=t, mn=t), exact_cands([(x, y, s)])))
    return out


# ---- quadtree --------------------------------------------------------------------------------------------------------------------------
W0, H0 = 640, 480                    # one root [0, 608) x [0, 448) (relative coordinates); first split at (304, 224), then (152, 112), (76, 56)


def rel(x, y):
    return x - MIN_BORDER, y - MIN_BORDER


def kept(expected_xy_resp):
    exp = {(int(x), int(y), int(s)) for x, y, s in expected_xy_resp}

    def proof(d):
        got = kp_set(d)
        assert got == exp, 'keypoints: missing %s, extra %s' % (sorted(exp - got)[:6], sorted(got - exp)[:6])
    return proof


def qt_case(name, pts, N, keep, w=W0, h=H0, extra_proof=None):
    check_spacing(pts)
    fs = [exact_cands(pts), kept(keep)]
    if extra_proof:
        fs.append(extra_proof)
    return case(name, dots(w, h, pts, 30), P(nfeatures=N), all_of(*fs))


def quadtree_cases():
    out = []
    # coarse exit at size >= N: one dot per quadrant + a second in the top-left one; N = 4 -> the first pass ends it
    pts = [(66, 66, 30), (416, 66, 31), (66, 316, 32), (416, 316, 33), (80, 90, 34)]
    out.append(qt_case('qt_coarse_exit_at_N', pts, 4, pts[1:]))
    # the coarse pass has no mid-pass exit: with 2 roots of 4 quadrant dots each and N = 4, both roots are divided although the first one
    # alone already brings the list to N -> 8 keypoints
    w2 = 901
    n, hx, _ = qt_roots(w2, H0)
    assert n == 2
    pts = [(int(hx * f32(r)) + dx + MIN_BORDER, dy + MIN_BORDER, 30 + 4 * r + q) for r in range(2) for q, (dx, dy) in enumerate(((40, 40), (260, 40), (40, 300), (260, 300)))]
    assert [qt_root(w2, H0, x - MIN_BORDER) for x, _, _ in pts] == [0] * 4 + [1] * 4
    out.append(qt_case('qt_coarse_exit_two_roots', pts, 4, pts, w=w2))
    # coarse stall: 2 candidates in one quadrant, N = 1000 -> the first pass leaves one node: 1 keypoint
    pts = [(66, 66, 30), (96, 96, 31)]
    assert split_division(W0, H0, rel(66, 66), rel(96, 96)) == 3
    out.append(qt_case('qt_coarse_stall_pair', pts, 1000, pts[1:]))
    # coarse stall one pass later: the pair separates only at division 3, the second pass keeps it together and ends the distribution
    pts = [(66, 66, 30), (96, 96, 31), (416, 316, 32)]
    out.append(qt_case('qt_coarse_stall_second_pass', pts, 1000, pts[1:]))
    # coarse -> fine (4 + 3 * 4 > 6), fine pass breaks after 2 of 4 equal-size nodes: the last created (n4, then n3) go first (Q1)
    quads = [(16, 16), (320, 16), (16, 240), (320, 240)]
    pts = []
    for q, (qx, qy) in enumerate(quads):
        pts += [(qx + 30, qy + 30, 40 + 2 * q), (qx + 200, qy + 150, 41 + 2 * q)]
    for a in range(0, 8, 2):
        assert split_division(W0, H0, rel(*pts[a][:2]), rel(*pts[a + 1][:2])) == 2
    out.append(qt_case('qt_fine_break_q1_equal_sizes', pts, 6, pts[4:] + [pts[1], pts[3]]))
    # fine pass over unequal sizes: the 3-dot quadrant first (largest), then n4; the break at N = 7
    pts3 = pts[:2] + [(16 + 200, 16 + 30, 39)] + pts[2:]
    assert split_division(W0, H0, rel(*pts3[0][:2]), rel(*pts3[2][:2])) == 2
    out.append(qt_case('qt_fine_break_q1_sizes', pts3, 7, pts3[:3] + pts3[6:] + [pts3[4]]))
    # a fine pass ending in a stall: two close pairs (separate at division 3), 2 + 3 * 2 > 5 -> fine; neither pair splits -> finish
    pts = [(66, 66, 30), (96, 96, 31), (366, 290, 33), (396, 320, 32)]
    assert split_division(W0, H0, rel(366, 290), rel(396, 320)) == 3
    out.append(qt_case('qt_fine_stall', pts, 5, [pts[1], pts[2]]))
    # equal responses in one final node: across cells the first cell in row-major cell order wins, inside a cell the first pixel row-major
    a, c = (16 + 40, 16 + 10), (16 + 10, 16 + 40)
    assert cell_of(W0, H0, *a)[:2] == (0, 1) and cell_of(W0, H0, *c)[:2] == (1, 0)
    out.append(qt_case('qt_tie_across_cells', [(a[0], a[1], 30), (c[0], c[1], 30)], 1000, [(a[0], a[1], 30)]))
    a, c = (16 + 20, 16 + 5), (16 + 5, 16 + 10)
    assert cell_of(W0, H0, *a) == cell_of(W0, H0, *c)
    out.append(qt_case('qt_tie_in_cell', [(a[0], a[1], 30), (c[0], c[1], 30)], 1000, [(a[0], a[1], 30)]))
    out += root_boundary_cases()
    out += candidate_count_cases()
    out.append(depth12_case())
    return out


def root_boundary_cases():
    """Wide levels with 2, 9 and 42 quadtree roots and a non-integer strip width hX: dots at every inner strip boundary B = (int)(r * hX) and at
    B - 1 and B + 1.  The dot at B is the column x == UR.x of the strip on its left (it lies outside that strip's rectangle).  Each strip's
    dots sit in different quadrants, so every dot is kept.  Proof: the root each dot lands in (restated), and every dot kept."""
    out = []
    for w, h in ((901, 480), (4096, 480), (4096, 128)):
        n, hx, rh = qt_roots(w, h)
        assert n >= 2 and float(hx) != int(hx)
        pts, outside = [], 0
        for r in range(1, n):
            B = int(hx * f32(r))
            for dx, yr in ((-1, rh // 8), (0, rh - rh // 8 - 1), (1, rh // 3)):
                x = B + dx
                if cell_of(w, h, x + MIN_BORDER, yr + MIN_BORDER) is None:
                    continue
                root = qt_root(w, h, x)
                if dx == 0 and root == r - 1:
                    outside += 1                       # x == UR.x of root r - 1
                assert root == (r if dx == 1 else r - 1) or dx == 0
                pts.append((x + MIN_BORDER, yr + MIN_BORDER, 30 + len(pts) % 200))
        assert outside >= 1
        out.append(qt_case('qt_roots_%dx%d_n%d' % (w, h, n), pts, 1000, pts, w=w, h=h))
    return out


def lattice(w, h, n, step=4):
    """n dots on a 4-px lattice inside the cell interiors (never adjacent, never on a ring), scores cycling through 20..219."""
    pts = []
    for y in range(MIN_BORDER + 3, h - MIN_BORDER - 3, step):
        for x in range(MIN_BORDER + 3, w - MIN_BORDER - 3, step):
            if len(pts) == n:
                return pts
            if cell_of(w, h, x, y) is not None:
                pts.append((x, y, 20 + (x * 7 + y * 13) % 200))
    assert len(pts) == n, (len(pts), n)
    return pts


def candidate_count_cases():
    """Candidate counts 1, 2, 63, 64, 65 (bitonic sorts of 1, 2, < 64 and exactly 64 keys, and the first one over a warp chunk), and the
    shared-memory key capacity - 1, +0, + 1 for an nfeatures in each of its three bands (4096, 2048, 1024): the first count over it sorts in
    global scratch.  Proof: the oracle's candidate count and the restated band."""
    out = []
    w, h = W0, H0
    for n in (1, 2, 63, 64, 65):
        pts = lattice(w, h, n)
        out.append(case('qt_count_%d' % n, dots(w, h, pts, 0), P(), exact_cands(pts)))
    for nf, cap in ((300, 4096), (500, 2048), (1000, 1024)):
        assert smem_key_cap(w, h, P(nfeatures=nf)) == cap
        for n in (cap - 1, cap, cap + 1):
            pts = lattice(w, h, n)

            def proof(d, n=n):
                assert len(d.cands[0]) == n
            out.append(case('qt_keys_nf%d_count%d' % (nf, n), dots(w, h, pts, 0), P(nfeatures=nf), all_of(proof, exact_cands(pts)), band=cap))
    return out


def depth12_case():
    """A 4096 x 4096 level and two horizontally adjacent dots on either side of a FAST cell boundary (both survive the cell-local NMS) that share
    their quadtree path for 11 divisions and separate at the 12th, the last one the device's path key encodes.  Dots Q_d peel off the pair's
    node at every earlier division, so each coarse pass splits one node and none stalls.  Proof: the restated split divisions (12 for the pair,
    1..11 for the Q_d) and every dot kept."""
    w = h = 4096
    cl = cells(w, h)
    bounds = sorted({c[2] + 3 for c in cl if c[1] > 0})
    rng = np.random.RandomState(12)
    for bx in bounds[40:]:
        for y in range(2000, 2004):
            a, b = rel(bx - 1, y), rel(bx, y)
            if split_division(w, h, a, b) != QT_DEPTH:
                continue
            pts = [(bx - 1, y), (bx, y)]
            ok = True
            for d in range(QT_DEPTH - 2, -1, -1):            # Q_d separates from the pair at division d + 1: seeded search in a box of the node's size
                found = None
                half = max(4, (w - 2 * MIN_BORDER) >> d)
                for _ in range(20000):
                    dx, dy = (int(v) for v in rng.randint(-half, half + 1, 2))
                    q = (bx - 1 + dx, y + dy)
                    if not (0 <= q[0] < w and 0 <= q[1] < h) or cell_of(w, h, *q) is None or split_division(w, h, a, rel(*q)) != d + 1:
                        continue
                    if all(max(abs(q[0] - p[0]), abs(q[1] - p[1])) >= 2 and (q[0] - p[0], q[1] - p[1]) not in RING_SET
                           and (p[0] - q[0], p[1] - q[1]) not in RING_SET for p in pts):
                        found = q
                        break
                if not found:
                    ok = False
                    break
                pts.append(found)
            if ok:
                dd = [(x, yy, 30 + k) for k, (x, yy) in enumerate(pts)]
                assert sorted(split_division(w, h, a, rel(x, yy)) for x, yy, _ in dd[1:]) == list(range(1, QT_DEPTH + 1))
                return qt_case('qt_depth12_pair_4096', dd[:1] + dd[2:] + dd[1:2], 1000, dd, w=w, h=h)
    raise AssertionError('no depth-12 pair found')


# ---- orientation and descriptor --------------------------------------------------------------------------------------------------------
def stamp_case(name, w, h, stamps, b=100, border_noise=False, p=None, proof=None):
    """Dots of score 40 with one low-contrast pixel (b + 2, never a corner) at disc offset (u, v) -- or none: m10 = 2u, m01 = 2v."""
    img = np.full((h, w), b, np.int32)
    if border_noise:
        rng = np.random.RandomState(7)
        m = np.zeros((h, w), bool); m[:4] = True; m[-4:] = True; m[:, :4] = True; m[:, -4:] = True
        img[m] = rng.randint(0, 256, int(m.sum()))
    exp = []
    for x, y, uv in stamps:
        img[y, x] = b + 41
        if uv is not None:
            img[y + uv[1], x + uv[0]] = b + 2
        exp.append((x, y, 40))
    img = img.astype(np.uint8)
    fs = [exact_cands(exp)]
    if proof:
        fs.append(proof)
    return case(name, img, p or P(), all_of(*fs))


def orientation_cases():
    """Stamps on a 4096 x 128 level, one per quadtree root (42 roots: a root with one candidate is never divided, so every stamp is kept).
    Offsets (+-5, 0), (0, +-5) and none give moments (m10, m01) = (+-10, 0), (0, +-10), (0, 0) and the angles 0, 180, 90, 270 and 0 exactly.
    Offsets at |u| == umax[v] and umax[v] + 1 put the one off-background pixel just inside or just outside the circular patch.  Proof: the
    oracle's moments of each kept keypoint (and the exact angles)."""
    out = []
    w, h = 4096, 128
    n, hx, _ = qt_roots(w, h)
    cs = [(int(hx * f32(r + 0.5)) + MIN_BORDER, h // 2) for r in range(n)]
    assert all(cell_of(w, h, *c) is not None and qt_root(w, h, c[0] - MIN_BORDER) == r for r, c in enumerate(cs))
    want = {(5, 0): 0.0, (0, 5): 90.0, (-5, 0): 180.0, (0, -5): 270.0, None: 0.0}
    st = [(cs[k][0], cs[k][1], uv) for k, uv in enumerate(want)]

    def angles(d, st=st):
        for x, y, uv in st:
            k = d.kps[(d.kps['x'] == x) & (d.kps['y'] == y)]
            assert len(k) == 1 and k['angle'][0] == want[uv], (x, y, uv, k['angle'])
            a, m01, m10 = O.ic_angle(d.pyramid[0], x, y)
            assert (m10, m01) == ((2 * uv[0], 2 * uv[1]) if uv else (0, 0))
    out.append(stamp_case('ori_axis_angles', w, h, st, proof=angles))
    # umax edge: a pixel at |u| == umax[v] is inside the disc, one at umax[v] + 1 outside
    umax = O.orb_tables(oparams(P()))['umax']
    st = []
    for v in (0, 3, 8, 10, 11, 13, 15):
        for du, su, sv in ((0, 1, 1), (1, 1, -1), (0, -1, -1), (1, -1, 1)):
            u = su * (int(umax[v]) + du)
            if abs(u) <= 15:
                st.append((u, sv * v))
    st = [(cs[k][0], cs[k][1], uv) for k, uv in enumerate(st)]
    assert len(st) <= n

    def edges(d, st=st):
        inside = 0
        for x, y, (u, v) in st:
            a, m01, m10 = O.ic_angle(d.pyramid[0], x, y)
            k = d.kps[(d.kps['x'] == x) & (d.kps['y'] == y)]
            assert len(k) == 1
            ins = abs(u) <= umax[abs(v)]
            inside += ins
            assert (m10, m01) == ((2 * u, 2 * v) if ins else (0, 0)), (u, v, m10, m01)
        assert 0 < inside < len(st)
    out.append(stamp_case('ori_umax_edges', w, h, st, proof=edges))
    return out


def border_descriptor_case():
    """Keypoints at the minimum legal border (first / last interior pixel of the corner cells) with angles near 45, 135, 225 and 315 degrees:
    their rotated BRIEF pattern reaches 17 px or more, into the pixels whose 7x7 blur reflects (BORDER_REFLECT_101) the random outer frame.
    Proof: O.pattern_extent of each kept keypoint's angle is >= 17."""
    w, h = W0, H0
    lo, hx, hy = MIN_BORDER + 3, w - MIN_BORDER - 4, h - MIN_BORDER - 4
    st = []
    for (x, y, sx, sy) in ((lo, lo, -1, -1), (hx, lo, 1, -1), (lo, hy, -1, 1), (hx, hy, 1, 1)):   # one per root quadrant: all kept
        best = max(((sx * u, sy * v) for u in range(3, 9) for v in range(3, 9) if abs(u - v) <= 2),
                   key=lambda uv: (O.pattern_extent(O.fast_atan2(2 * uv[1], 2 * uv[0])), -abs(abs(uv[0]) - abs(uv[1]))))
        st.append((x, y, best))

    def ext(d):
        for x, y, (u, v) in st:
            k = d.kps[(d.kps['x'] == x) & (d.kps['y'] == y)]
            assert len(k) == 1 and abs(float(k['angle'][0]) % 90 - 45) <= 15, k['angle']
            e = O.pattern_extent(float(k['angle'][0]))
            assert e >= 17 and min(x, y, w - 1 - x, h - 1 - y) - e <= 2, (x, y, e)   # a tap on a pixel whose blur reflected the frame
    return stamp_case('desc_border_45deg', w, h, st, border_noise=True, proof=ext)


# ---- budgets and geometry --------------------------------------------------------------------------------------------------------------
def budget_cases():
    from pysgs import synth
    out = []
    img = synth.frame_s1(640, 480, seed=21)
    for nf in (1, 7, 8, 9):
        p = P(nfeatures=nf, nlevels=8)

        def zero_levels(d, p=p):
            npl = O.orb_tables(oparams(p))['nPerLevel']
            z = [l for l in range(p['nlevels']) if npl[l] == 0 and len(d.cands[l]) > 1]
            assert z, npl
            assert any((d.kps['octave'] == l).sum() > 0 for l in z)       # an n_target = 0 level still keeps its first pass's nodes
        out.append(case('budget_nf%d_8lv' % nf, img, p, zero_levels))
    big = synth.frame_s1(1280, 960, seed=22)
    for sc, im in ((1.05, img), (1.5, big), (1.999, big)):
        L = max_nlevels(im.shape[1], im.shape[0], sc)
        p = P(nfeatures=1500, scale=sc, nlevels=L)

        def levels(d, L=L, sc=sc):
            assert L == 16 or sc > 1.1
            assert all(x is not None for x in d.pyramid) and sum(len(c) > 0 for c in d.cands) == L
        out.append(case('budget_scale%s_%dlv' % (str(sc).replace('.', 'p'), L), im, p, levels))
    def one_level(d):
        assert len(d.pyramid) == 1 and len(d.kps) >= 800 and (d.kps['octave'] == 0).all()
    out.append(case('budget_nlevels1', img, P(nfeatures=800, nlevels=1), one_level))
    # cvRound ties of the level size (round half to even): 644 * 0.625 = 402.5 -> 402, 484 * 0.625 = 302.5 -> 302; 636 -> 397.5 -> 398, 476 -> 297.5 -> 298
    for w, h, ew, eh in ((644, 484, 402, 302), (636, 476, 398, 298)):
        p = P(nfeatures=600, scale=1.6, nlevels=3)
        inv = O.orb_tables(oparams(p))['invScale'][1]
        for v, e in ((f32(w) * inv, ew), (f32(h) * inv, eh)):
            assert v % 1 == 0.5 and abs(v - e) == 0.5 and e % 2 == 0
        im = synth.frame_s1(w, h, seed=23)

        def tie(d, ew=ew, eh=eh):
            assert d.pyramid[1].shape == (eh, ew)
        out.append(case('budget_round_tie_%dx%d' % (w, h), im, p, tie))
    return out


def refusals():
    """(name, w, h, params, status, word of the message) for sgs_extractor_create.  The nfeatures limit is derived from the plan formulas."""
    SGS_ERR_INVALID, SGS_ERR_UNSUPPORTED = 1, 4
    nmax = max_nfeatures(640, 480, P(nlevels=1))
    return [('width_4097', 4097, 480, P(), SGS_ERR_INVALID, 'outside'),
            ('height_4097', 640, 4097, P(), SGS_ERR_INVALID, 'outside'),
            ('scale_2', 640, 480, P(scale=2.0, nlevels=3), SGS_ERR_UNSUPPORTED, 'INTER_AREA'),
            ('level_too_small', 640, 480, P(scale=1.5, nlevels=9), SGS_ERR_UNSUPPORTED, '30-px'),
            ('nfeatures_%d' % (nmax + 1), 640, 480, P(nfeatures=nmax + 1), SGS_ERR_UNSUPPORTED, 'nfeatures')], nmax


def accepted_limits():
    """Parameter sets at the edge of what sgs_extractor_create accepts: 4096 x 4096 and the largest nfeatures of the quadtree."""
    nmax = max_nfeatures(640, 480, P(nlevels=1))
    return [(4096, 4096, P()), (640, 480, P(nfeatures=nmax))]


def all_cases():
    out = fast_threshold_cases() + [fast_interior_edge_case(), fast_nms_cases()] + fast_arc_cases() + fast_compass_cases()
    out += quadtree_cases() + orientation_cases() + [border_descriptor_case()] + budget_cases()
    names = [c['name'] for c in out]
    assert len(set(names)) == len(names)
    return out
