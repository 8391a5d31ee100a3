"""Constructed inputs for the projection matchers (numpy only, no device): small frames plus maps built so that one hard path of the
ordered restatement in sg-slam_b200/csrc/match.cu MUST be taken.  Every case carries a proof -- an assertion on the oracle's result that
only holds if the path was taken (for example "point j matched the keypoint it ranks (j+1)-th") -- so that an edit to a builder cannot
quietly turn a case into an easy one.

A case is a dict: name, kind ('last', 'kf', 'local', 'sim3', 'init'), params (the per-launch scalars of the batched entry point), the
arrays of that matcher, bounds (min_x, min_y, max_x, max_y), paths (labels of the paths the proof demonstrates) and proof(result).
run_oracle(case) returns the oracle's result as a dict; the same dict layout is what the tests build from the reference and the device.

The last-frame, key-frame and Sim3 cases use the identity pose and points at depth 1, so that a projection is u = fx * X + cx with two
float32 roundings, which the builders invert exactly where a case needs a projection on a bound."""
import numpy as np

import oracle as O
import scenarios as S
from pysgs import synth

f32 = np.float32
CAM = dict(synth.TUM3)
SF = S.scale_factors()
W, H = 640, 480
FULL = (0.0, 0.0, float(W), float(H))
ID_BASE = 7
GRID_COLS, GRID_ROWS = 64, 48


def tum1_bounds():
    """Frame::ComputeImageBounds on TUM1's distortion: the undistorted corners (0,0) (w,0) (0,h) (w,h) of tests/golden/undistort.npz (cv2)."""
    import os
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'undistort.npz'))
    c = g['TUM1_und'][-4:]
    return (float(min(c[0, 0], c[2, 0])), float(min(c[0, 1], c[1, 1])), float(max(c[1, 0], c[3, 0])), float(max(c[2, 1], c[3, 1])))


def grid_inv(bounds):
    return f32(f32(GRID_COLS) / f32(f32(bounds[2]) - f32(bounds[0]))), f32(f32(GRID_ROWS) / f32(f32(bounds[3]) - f32(bounds[1])))


def _round_away(v):
    return int(np.sign(v) * np.floor(abs(float(v)) + 0.5))


def pos_in_grid(x, y, bounds):
    """Frame::PosInGrid (src/Frame.cc:409-419) in float32: (cell x, cell y) or None outside the grid."""
    wi, hi = grid_inv(bounds)
    px = _round_away(f32(f32(f32(x) - f32(bounds[0])) * wi)); py = _round_away(f32(f32(f32(y) - f32(bounds[1])) * hi))
    return (px, py) if 0 <= px < GRID_COLS and 0 <= py < GRID_ROWS else None


def grid_order(kps, bounds):
    """Keypoint indices in the iteration order of Frame::GetFeaturesInArea: cell ix * 48 + iy ascending, then index."""
    key = []
    for i, k in enumerate(kps):
        c = pos_in_grid(k['x'], k['y'], bounds)
        if c is not None:
            key.append((c[0] * GRID_ROWS + c[1], i))
    return [i for _, i in sorted(key)]


def _neighbours(v, n=400):
    """float32 values around v, n ulps either way."""
    v = f32(v)
    out = [v]
    lo = hi = v
    for _ in range(n):
        lo = np.nextafter(lo, f32(-np.inf)); hi = np.nextafter(hi, f32(np.inf))
        out += [lo, hi]
    return np.array(out, f32)


def proj(X, f, c):
    """u = fx * X * invz + cx at invz = 1 (identity pose, depth 1): the projection of all three pose-based matchers."""
    return f32(f32(f32(f) * f32(X)) + f32(c))


def solve_coord(target, f, c, mode='near'):
    """The camera coordinate X (depth 1) whose projection is `target` exactly ('eq'), the smallest projection >= target ('ge'), the
    largest < target ('lt') or the nearest one ('near')."""
    xs = _neighbours(f32((float(target) - float(c)) / float(f)))
    us = np.array([proj(x, f, c) for x in xs], f32)
    t = f32(target)
    if mode == 'eq':
        hit = xs[us == t]
        assert len(hit), ('no exact projection onto', target)
        return hit[0]
    if mode == 'ge':
        sel = us >= t; return xs[sel][np.argmin(us[sel])]
    if mode == 'lt':
        sel = us < t; return xs[sel][np.argmax(us[sel])]
    return xs[np.argmin(np.abs(us.astype(np.float64) - float(target)))]


def cell_coord(k, origin, inv, half=True):
    """A float32 coordinate x with (x - origin) * inv == k + 0.5 exactly (half=True) -- PosInGrid rounds it half away from zero."""
    t = f32(k + 0.5) if half else f32(k)
    for x in _neighbours(f32(float(origin) + float(t) / float(inv)), 2000):
        if f32(f32(x - f32(origin)) * inv) == t:
            return x
    return None


def _desc(rng):
    return rng.randint(0, 256, 32).astype(np.uint8)


def flip(d, bits):
    b = np.unpackbits(d)
    b[list(bits)] ^= 1
    return np.packbits(b)


def hamming(a, b):
    return int(np.unpackbits(a ^ b).sum())


class _Frame:
    """The current frame (or key frame) of a case: keypoints, descriptors, right coordinates."""

    def __init__(self, bounds=FULL):
        self.kps, self.desc, self.ur, self.bounds = [], [], [], bounds

    def kp(self, x, y, d, octave=0, angle=0.0, ur=-1.0):
        self.kps.append((f32(x), f32(y), octave, f32(angle))); self.desc.append(d); self.ur.append(f32(ur))
        return len(self.kps) - 1

    def arrays(self):
        k = np.zeros(len(self.kps), O.KP_DTYPE)
        for i, (x, y, o, a) in enumerate(self.kps):
            k[i]['x'], k[i]['y'], k[i]['octave'], k[i]['angle'] = x, y, o, a
        k['size'] = 31; k['response'] = 20; k['class_id'] = -1
        return dict(kps=k, desc=np.array(self.desc, np.uint8).reshape(-1, 32), uright=np.array(self.ur, f32), bounds=self.bounds)


class _Points:
    """Map points at depth 1 seen through the identity pose: (u, v) is where a point projects."""

    def __init__(self):
        self.rows = []

    def point(self, u, v, d, octave=0, angle=0.0, has=1, obs=1, mode=('near', 'near'), level=0):
        X = (solve_coord(u, CAM['fx'], CAM['cx'], mode[0]), solve_coord(v, CAM['fy'], CAM['cy'], mode[1]))
        self.rows.append(dict(X=X, d=d, octave=octave, angle=f32(angle), has=has, obs=obs, level=level))
        return len(self.rows) - 1

    def filler(self, n, rng):
        for _ in range(n):
            self.rows.append(dict(X=(f32(0), f32(0)), d=_desc(rng), octave=0, angle=f32(0), has=0, obs=1, level=0))

    def uv(self, i):
        X = self.rows[i]['X']
        return proj(X[0], CAM['fx'], CAM['cx']), proj(X[1], CAM['fy'], CAM['cy'])

    def xyz(self):
        return np.array([[r['X'][0], r['X'][1], 1.0] for r in self.rows], f32).reshape(-1, 3)

    def last(self):
        return dict(last_has=np.array([r['has'] for r in self.rows], np.uint8), last_xyz=self.xyz(),
                    last_desc=np.array([r['d'] for r in self.rows], np.uint8).reshape(-1, 32), last_obs=np.array([r['obs'] for r in self.rows], np.uint8),
                    last_oct=np.array([r['octave'] for r in self.rows], np.int32), last_angle=np.array([r['angle'] for r in self.rows], f32))

    def distances(self):
        """MapPoint::PredictScale inputs: mfMaxDistance chosen so that the predicted level is the point's `level` (Ow = 0), mfMinDistance far below."""
        xyz = self.xyz()
        dist = np.array([f32(np.sqrt(float(x) * float(x) + float(y) * float(y) + float(z) * float(z))) for x, y, z in xyz], f32)
        lvl = np.array([r['level'] for r in self.rows])
        maxd = np.where(lvl == 0, dist * 0.95, dist * 1.2 ** (lvl - 0.5)).astype(f32)
        lsf = O.logf(1.2)
        for i in range(len(dist)):
            got = int(np.ceil(f32(O.logf(f32(maxd[i] / dist[i])) / lsf)))
            assert max(got, 0) == lvl[i], (i, got, lvl[i])
        return dict(min_dist=(maxd / f32(1.2) ** 8).astype(f32), max_dist=maxd)

    def keyframe(self):
        d = self.distances()
        return dict(kf_valid=np.array([r['has'] for r in self.rows], np.uint8), last_xyz=self.xyz(),
                    last_desc=np.array([r['d'] for r in self.rows], np.uint8).reshape(-1, 32), last_angle=np.array([r['angle'] for r in self.rows], f32), **d)


EYE = np.eye(4, dtype=f32)
CASES = {}


def _case(name, kind, params, paths, proof, **arrays):
    CASES[name] = dict(name=name, kind=kind, params=params, paths=paths, proof=proof, cam=CAM, sf=SF, w=W, h=H, **arrays)


LAST = dict(th=15.0, mono=False, check_ori=True)
LAST_NO_ORI = dict(th=15.0, mono=False, check_ori=False)
KF = dict(th=10.0, orb_dist=7, check_ori=True)
LOCAL = dict(th=1.0, nnratio=0.8)
LOCAL_TH = dict(th=float(np.nextafter(f32(1.0), f32(2.0))), nnratio=0.8)
SIM3 = dict(th=10)
INIT = dict(window=20, nnratio=0.75, check_ori=True)


def _last_case(name, fr, P, params, paths, proof, Tcw_last=EYE, cur_mp=None, cur_obs=None):
    a = fr.arrays()
    n = len(a['kps'])
    _case(name, 'last', params, paths, proof, **a, **P.last(), Tcw_cur=EYE, Tcw_last=Tcw_last,
          cur_mp=np.full(n, -1, np.int32) if cur_mp is None else cur_mp, cur_obs=cur_obs)


# ---- pile-up: 10 keypoints in one window, 12 points with one descriptor; point j gets the keypoint it ranks j-th --------------------------
def _pile(kind, first, equal, seed):
    rng = np.random.RandomState(seed)
    fr, P = _Frame(), _Points()
    D = _desc(rng)
    for k in range(10):
        if equal:         # one distance for all, laid out against index order across cell boundaries (cells are 10 px wide)
            fr.kp(312 - 2 * k, 240 + 6 * (k % 2), flip(D, range(8 * k, 8 * k + 5)))
        else:
            fr.kp(300 + k, 238 + (k % 3), flip(D, range(k + 1)))
    P.filler(first, rng)
    for j in range(12):
        P.point(303.0 if equal else 305.0, 242.0 if equal else 240.0, D, level=0)
    a = fr.arrays()
    rank = grid_order(a['kps'], fr.bounds) if equal else list(range(10))
    if equal:
        assert rank != sorted(rank)
    return fr, P, rank


for _kind in ('last', 'kf'):
    for _first, _where in ((4, 'in_chunk'), (28, 'across_chunks')):
        for _equal in (False, True):
            _fr, _P, _rank = _pile(_kind, _first, _equal, 11 + _first + _equal)
            _nm = '%s_pile_%s_%s' % (_kind, _where, 'equal' if _equal else 'distinct')
            if _kind == 'last':
                def _proof(r, first=_first, rank=_rank):
                    # sequential: point first+j takes the keypoint ranked j; the last two find every candidate claimed
                    for j in range(10):
                        assert r['mp'][rank[j]] == first + j, (j, r['mp'])
                    assert r['nm'] == 10 and (r['mp'] >= 0).sum() == 10
                _last_case(_nm, _fr, _P, LAST, ['rescan', 'tentative_claim'], _proof)
            else:
                # key-frame variant: keypoint rank 2 is already assigned (skipped), ORBdist = 7
                a = _fr.arrays()
                cur_mp = np.full(len(a['kps']), -1, np.int32); cur_mp[_rank[2]] = 900
                if _equal:
                    def _proof(r, first=_first, rank=_rank):
                        # all distances 5 <= ORBdist: every free keypoint is taken in rank order, points 9.. find nothing
                        free = [k for k in rank if k != rank[2]]
                        for j, k in enumerate(free):
                            assert r['mp'][k] == first + j, (j, r['mp'])
                        assert r['mp'][rank[2]] == 900 and r['nm'] == 9
                else:
                    def _proof(r, first=_first):
                        # keypoint k sits at distance k + 1; point first+5 takes keypoint 6 at distance 7 == ORBdist, point first+6 would need
                        # keypoint 7 at distance 8 and is rejected -- and so is everyone after it, since a rejection claims nothing
                        want = {0: 0, 1: 1, 3: 2, 4: 3, 5: 4, 6: 5}
                        for k, j in want.items():
                            assert r['mp'][k] == first + j, (k, r['mp'])
                        assert r['mp'][2] == 900 and (r['mp'][7:] == -1).all() and r['nm'] == 6
                _case(_nm, 'kf', KF, ['rescan', 'tentative_claim', 'orb_dist_edge' if not _equal else 'grid_order_ties'], _proof,
                      **a, **_P.keyframe(), Tcw_cur=EYE, cur_mp=cur_mp)


# ---- pre-existing claims: the top four candidates of point 0 already hold an observed map point ----------------------------------------
def _preclaimed():
    rng = np.random.RandomState(3)
    fr, P = _Frame(), _Points()
    D = _desc(rng)
    for k in range(6):
        fr.kp(200 + 2 * k, 150, flip(D, range(k + 1)))
    P.point(205.0, 150.0, D); P.point(205.0, 150.0, D)
    cur_mp = np.array([700, 701, 702, 703, 800, -1], np.int32)
    cur_obs = np.array([1, 1, 1, 1, 0, 0], np.uint8)          # keypoint 4 holds a point without observations: not a claim

    def proof(r):
        assert list(r['mp']) == [700, 701, 702, 703, 0, 1] and r['nm'] == 2
    _last_case('last_preclaimed_top4', fr, P, LAST, ['rescan'], proof, cur_mp=cur_mp, cur_obs=cur_obs)


_preclaimed()


# ---- non-claiming writers: obs = 0 points overwrite one keypoint, an obs = 1 point writes last ----------------------------------------
def _lattice(fr, P, rng, rots, x0=40, y0=40, step=40, ncols=14, octave=0, kp_angle=0.0):
    """One keypoint and one point projecting onto it per rotation in `rots` (rot = point angle - keypoint angle); returns the keypoint indices."""
    ks = []
    for i, rot in enumerate(rots):
        x, y = x0 + step * (i % ncols), y0 + step * (i // ncols)
        d = _desc(rng)
        ks.append(fr.kp(x, y, d, octave, angle=kp_angle))
        P.point(x + 0.5, y - 0.5, flip(d, range(3)), octave, angle=kp_angle + rot)
    return ks


def _writers(check_ori):
    rng = np.random.RandomState(5)
    fr, P = _Frame(), _Points()
    bg = _lattice(fr, P, rng, [0.0] * 20)
    D = _desc(rng)
    A = fr.kp(500, 420, D, angle=10.0)
    for j, (obs, rot) in enumerate(((0, 0.0), (0, 0.0), (0, 180.0), (1, 0.0))):
        P.point(500.5, 420.5, flip(D, range(2 * j, 2 * j + 2)), obs=obs, angle=10.0 + rot)
    if check_ori:
        def proof(r):
            # four writes counted; the third writer's rotation bin (15) is discarded, which clears the keypoint although the last writer's bin is kept
            assert r['mp'][A] == -1 and r['nm'] == 20 + 4 - 1 and all(r['mp'][k] >= 0 for k in bg)
    else:
        def proof(r):
            assert r['mp'][A] == 23 and r['nm'] == 24
    _last_case('last_writers_%s' % ('ori' if check_ori else 'no_ori'), fr, P, LAST if check_ori else LAST_NO_ORI,
               ['last_writer'] + (['ori_clears_keypoint'] if check_ori else []), proof)


_writers(True)
_writers(False)


# ---- geometry on TUM1's image bounds --------------------------------------------------------------------------------------------------
def _geometry():
    B_ = tum1_bounds()
    mnx, mny, mxx, mxy = B_
    wi, hi = grid_inv(B_)
    rng = np.random.RandomState(8)
    fr, P = _Frame(B_), _Points()
    # (a) half-cell keypoint H with the same distance as G, one cell later in index order: round-half-away puts H in G's cell, behind G
    for k in range(20, 40, 2):
        xh = cell_coord(k, mnx, wi)
        if xh is not None:
            break
    assert f32(f32(xh - f32(mnx)) * wi) == f32(k + 0.5)
    xg = f32(mnx + (k + 1.2) / float(wi))
    D = _desc(rng)
    G = fr.kp(xg, 200, flip(D, range(0, 4)))
    Hh = fr.kp(xh, 200, flip(D, range(4, 8)))
    assert pos_in_grid(xh, 200, B_)[0] == k + 1 == pos_in_grid(xg, 200, B_)[0]
    p_half = P.point((float(xg) + float(xh)) / 2, 200.0, D)
    # (b) left border: keypoint O at cell coordinate -0.5 (outside the grid) with the best descriptor; u just inside min_x (u == min_x
    #     itself is not reachable: with this cx every projection near min_x is a multiple of 2^-15) and just outside it
    xo = cell_coord(-1, mnx, wi)
    assert f32(f32(xo - f32(mnx)) * wi) == f32(-0.5) and pos_in_grid(xo, 100, B_) is None
    D = _desc(rng)
    Oo = fr.kp(xo, 100, flip(D, range(1)))
    I1 = fr.kp(mnx + 2.0, 100, flip(D, range(1, 11)))
    p_left = P.point(mnx, 100.0, D, mode=('ge', 'near'))
    D = _desc(rng)
    I2 = fr.kp(mnx + 2.0, 330, flip(D, range(3)))
    p_left_out = P.point(mnx, 330.0, D, mode=('lt', 'near'))
    # (c) right border: u == max_x exactly (inclusive in the last-frame test); window clipped at cell 63
    D = _desc(rng)
    R = fr.kp(mxx - 6.0, 250, flip(D, range(3)))
    p_right = P.point(mxx, 250.0, D, mode=('eq', 'near'))
    # (d) top border with an outside keypoint just above row coordinate -0.5 (no float32 y lands on -0.5 exactly here), bottom border v == max_y exactly
    ys = _neighbours(f32(mny - 0.5 / float(hi)), 2000)
    yo = max(y for y in ys if f32(f32(y - f32(mny)) * hi) < f32(-0.5))
    assert pos_in_grid(300, yo, B_) is None
    D = _desc(rng)
    Ot = fr.kp(300, yo, flip(D, range(1)))
    T_ = fr.kp(300, mny + 2.0, flip(D, range(1, 9)))
    p_top = P.point(300.0, mny, D, mode=('near', 'ge'))
    D = _desc(rng)
    Bt = fr.kp(450, mxy - 5.0, flip(D, range(3)))
    p_bottom = P.point(450.0, mxy, D, mode=('near', 'eq'))
    assert P.uv(p_right)[0] == f32(mxx) and P.uv(p_bottom)[1] == f32(mxy)
    assert P.uv(p_left)[0] >= f32(mnx) and P.uv(p_left_out)[0] < f32(mnx) and P.uv(p_top)[1] >= f32(mny)

    def proof(r):
        mp = r['mp']
        assert mp[G] == p_half and mp[Hh] == -1                      # grid order: G before the half-cell keypoint of the same cell
        assert mp[I1] == p_left and mp[Oo] == -1 and mp[Ot] == -1 and mp[T_] == p_top
        assert mp[I2] == -1                                           # the point just left of min_x is never searched
        assert mp[R] == p_right and mp[Bt] == p_bottom and r['nm'] == 5
    _last_case('last_tum1_bounds', fr, P, LAST, ['grid_half_cell', 'outside_grid', 'bounds'], proof)


_geometry()


# ---- gate edges: stereo error == radius, TH_HIGH, level windows at octave 0 and nlevels - 1 -------------------------------------------
def _gates():
    rng = np.random.RandomState(9)
    fr, P = _Frame(), _Points()
    out = {}
    # stereo: er == radius (15) passes, one ulp more does not
    for name, y, above in (('s_eq', 60.0, False), ('s_above', 160.0, True)):
        D = _desc(rng)
        i = P.point(60.0, y, D)
        u, _ = P.uv(i)
        urp = f32(u - f32(f32(CAM['bf']) * f32(1.0)))
        ur = f32(urp - f32(15.0))
        while f32(abs(f32(urp - ur))) > f32(15.0):
            ur = np.nextafter(ur, f32(np.inf))
        while f32(abs(f32(urp - ur))) < f32(15.0):
            ur = np.nextafter(ur, f32(-np.inf))
        assert f32(abs(f32(urp - ur))) == f32(15.0)
        while above and f32(abs(f32(urp - ur))) == f32(15.0):       # the next error the subtraction can produce above the radius
            ur = np.nextafter(ur, f32(-np.inf))
        out[name] = (i, fr.kp(62, y, flip(D, range(1)), ur=ur), fr.kp(58, y, flip(D, range(1, 21))))
    # TH_HIGH: distance 100 is a match, 101 is not
    for name, y, nb in (('h100', 60.0, 100), ('h101', 160.0, 101)):
        D = _desc(rng)
        i = P.point(200.0, y, D)
        out[name] = (i, fr.kp(201, y, flip(D, range(nb))))
    # level windows: octave 0 searches levels -1..1, octave 7 levels 6..8 (the best keypoint sits one level outside)
    D = _desc(rng)
    i = P.point(330.0, 60.0, D, octave=0)
    out['l0'] = (i, fr.kp(331, 60, flip(D, range(1)), octave=2), fr.kp(329, 60, flip(D, range(1, 9)), octave=1))
    D = _desc(rng)
    i = P.point(480.0, 300.0, D, octave=7)
    out['l7'] = (i, fr.kp(500, 300, flip(D, range(1)), octave=5), fr.kp(460, 300, flip(D, range(1, 9)), octave=7))

    def proof(r):
        mp = r['mp']
        i, ks, kn = out['s_eq']; assert mp[ks] == i and mp[kn] == -1
        i, ks, kn = out['s_above']; assert mp[ks] == -1 and mp[kn] == i
        i, k = out['h100']; assert mp[k] == i
        i, k = out['h101']; assert mp[k] == -1
        for key in ('l0', 'l7'):
            i, kout, kin = out[key]; assert mp[kout] == -1 and mp[kin] == i
        assert r['nm'] == 5
    _last_case('last_gate_edges', fr, P, LAST, ['stereo_edge', 'th_high_edge', 'level_window_edges'], proof)


_gates()


def _motion(forward):
    """Forward (tlc_z > b) and backward (-tlc_z > b) motion: level windows [oct, inf) and [0, oct]; forward from octave 0 checks no level."""
    rng = np.random.RandomState(10 + forward)
    fr, P = _Frame(), _Points()
    T = np.eye(4, dtype=f32); T[2, 3] = 0.12 if forward else -0.12
    D0 = _desc(rng); D3 = _desc(rng)
    i0 = P.point(150.0, 150.0, D0, octave=0)
    a0 = fr.kp(151, 150, flip(D0, range(1)), octave=6)
    i3 = P.point(400.0, 300.0, D3, octave=3)
    best3 = fr.kp(401, 300, flip(D3, range(1)), octave=2 if forward else 4)
    ok3 = fr.kp(399, 300, flip(D3, range(1, 9)), octave=7 if forward else 0)

    def proof(r):
        mp = r['mp']
        assert mp[best3] == -1 and mp[ok3] == i3
        assert mp[a0] == (i0 if forward else -1) and r['nm'] == (2 if forward else 1)
    _last_case('last_%s_motion' % ('forward' if forward else 'backward'), fr, P, LAST, ['level_window_edges'], proof, Tcw_last=T)


_motion(True)
_motion(False)


# ---- rotation histogram: wrap of bin 30, ties between maxima, max2 / max3 at 0.1 * max1 ------------------------------------------------
def _hist(name, seed, rots, keep, paths):
    rng = np.random.RandomState(seed)
    fr, P = _Frame(), _Points()
    ks = _lattice(fr, P, rng, rots)

    def proof(r):
        got = [bool(r['mp'][k] >= 0) for k in ks]
        assert got == keep, (got, keep)
        assert r['nm'] == sum(keep)
    _last_case(name, fr, P, LAST, paths, proof)


_FACTOR = f32(f32(30) / f32(360))


def _bin(rot):
    return _round_away(f32(f32(rot) * _FACTOR))


assert _bin(359.0) == 30 and _bin(355.0) == 30
_hist('last_hist_wrap', 70, [0.0] * 10 + [359.0, 355.0, 175.0], [True] * 12 + [False], ['histogram_wrap'])
_ties = [37.0] * 5 + [85.0] * 5 + [133.0] * 5 + [157.0] * 5           # bins 3, 7, 11, 13, five each: the first three maxima win
assert [_bin(r) for r in (37.0, 85.0, 133.0, 157.0)] == [3, 7, 11, 13]
_hist('last_hist_ties', 71, _ties, [True] * 15 + [False] * 5, ['histogram_ties'])
assert f32(f32(0.1) * f32(20)) == f32(2.0)
_hist('last_hist_tenth_kept', 72, [0.0] * 20 + [60.0] * 2 + [108.0] * 2 + [200.0], [True] * 24 + [False], ['histogram_tenth'])
_hist('last_hist_tenth_dropped', 73, [0.0] * 20 + [60.0] + [108.0], [True] * 20 + [False] * 2, ['histogram_tenth'])


# ---- local map: ratio verdicts flipped by claims ---------------------------------------------------------------------------------------
def _local_case(name, fr, pts, params, paths, proof, f_mp=None, f_obs=None):
    a = fr.arrays()
    n = len(a['kps'])
    m = len(pts)
    g = lambda k, dt, dflt=0: np.array([p.get(k, dflt) for p in pts], dt)
    _case(name, 'local', params, paths, proof, **a, inview=g('inview', np.uint8, 1), projx=g('x', f32), projy=g('y', f32),
          projxr=g('xr', f32, -1.0), level=g('level', np.int32), viewcos=g('viewcos', f32, 0.99),
          mp_desc=np.array([p['d'] for p in pts], np.uint8).reshape(m, 32), mp_obs=g('obs', np.uint8, 1),
          f_mp=np.full(n, -1, np.int32) if f_mp is None else f_mp, f_obs=np.zeros(n, np.uint8) if f_obs is None else f_obs)


def _fillers(pts, n, rng):
    pts += [dict(inview=0, x=0.0, y=0.0, d=_desc(rng)) for _ in range(n)]


def _local_flip(promote, obs, i1, i2):
    """promote=False: an earlier point claims the later point's second-best keypoint, rejection -> acceptance.
    promote=True: an earlier point claims the best one and a same-level third candidate becomes second, acceptance -> rejection.
    obs = 0: the earlier point claims nothing, no flip."""
    rng = np.random.RandomState(20 + 2 * promote + obs + i2)
    fr = _Frame()
    Z = _desc(rng)
    if not promote:
        A = fr.kp(300, 200, flip(Z, range(0, 40)), octave=1)
        Bk = fr.kp(302, 200, flip(Z, range(40, 82)), octave=1)
        d1 = flip(flip(Z, range(40, 82)), range(82, 92))          # 10 from B, 92 from A
        C = None
    else:
        A = fr.kp(300, 200, flip(Z, range(0, 30)), octave=1)
        Bk = fr.kp(302, 200, flip(Z, range(30, 70)), octave=1)
        C = fr.kp(300, 202, flip(Z, range(70, 115)), octave=1)
        d1 = flip(flip(Z, range(0, 30)), range(115, 125))         # 10 from A
    pts = []
    _fillers(pts, i1, rng)
    pts.append(dict(x=301.0, y=201.0, d=d1, level=1, obs=obs))
    _fillers(pts, i2 - i1 - 1, rng)
    pts.append(dict(x=301.0, y=201.0, d=Z, level=1, obs=1))
    e1, e2 = ID_BASE + i1, ID_BASE + i2
    if not promote:
        def proof(r):
            mp = r['mp']
            assert mp[Bk] == e1
            assert mp[A] == (e2 if obs else -1) and r['nm'] == (2 if obs else 1)
    else:
        def proof(r):
            mp = r['mp']
            assert mp[A] == (e1 if obs else e2) and mp[Bk] == -1 and mp[C] == -1 and r['nm'] == (1 if obs else 2)
    where = 'in_chunk' if i1 // 32 == i2 // 32 else 'across_chunks'
    paths = (['ratio_flip'] + (['tentative_second'] if (where == 'in_chunk' and not promote) else ['tentative_claim'] if where == 'in_chunk' else [])) if obs else ['ratio_no_flip']
    _local_case('local_%s_%s_obs%d' % ('promote_third' if promote else 'free_second', where, obs), fr, pts, LOCAL, paths, proof)


for _promote in (False, True):
    for _obs in (1, 0):
        _local_flip(_promote, _obs, 3, 7)
        _local_flip(_promote, _obs, 20, 40)


def _local_pile(first):
    """Alternating octaves keep consecutive candidates on different levels, so every ratio test passes and only the claims decide."""
    rng = np.random.RandomState(30 + first)
    fr = _Frame()
    D = _desc(rng)
    for k in range(10):
        fr.kp(300 + k, 200 + (k % 3), flip(D, range(k + 1)), octave=k % 2)
    pts = []
    _fillers(pts, first, rng)
    pts += [dict(x=304.5, y=201.0, d=D, level=1, obs=1) for _ in range(12)]

    def proof(r):
        for k in range(10):
            assert r['mp'][k] == ID_BASE + first + k, (k, r['mp'])
        assert r['nm'] == 10
    _local_case('local_pile_%s' % ('in_chunk' if first < 20 else 'across_chunks'), fr, pts, LOCAL, ['rescan', 'tentative_claim'], proof)


_local_pile(4)
_local_pile(28)


def _local_gates():
    rng = np.random.RandomState(40)
    fr = _Frame()
    pts, out = [], {}
    c998 = f32(0.998)
    assert float(c998) > 0.998 and float(np.nextafter(c998, f32(0))) < 0.998
    # view_cos == 0.998f is > 0.998 in double: radius 2.5, the far keypoint (3 px) is outside; one ulp below: radius 4
    for name, y, vc in (('v_eq', 60.0, c998), ('v_below', 160.0, np.nextafter(c998, f32(0)))):
        D = _desc(rng)
        out[name] = (len(pts), fr.kp(103, y, flip(D, range(10))), fr.kp(101, y, flip(D, range(10, 40))))
        pts.append(dict(x=100.0, y=y, d=D, level=0, viewcos=vc))
    # TH_HIGH and the ratio exactly at nnratio: 40 > 0.8f * 50 is false (0.8f * 50 rounds to 40.0f), 41 > 40 is true
    for name, y, nb, ns in (('h100', 260.0, 100, None), ('h101', 360.0, 101, None), ('r40', 60.0, 40, 50), ('r41', 160.0, 41, 50)):
        D = _desc(rng)
        x = 250.0 if name[0] == 'h' else 400.0
        k = fr.kp(x + 1, y, flip(D, range(nb)))
        k2 = fr.kp(x - 1, y, flip(D, range(128, 128 + ns))) if ns else None
        out[name] = (len(pts), k, k2)
        pts.append(dict(x=x, y=y, d=D, level=0))
    assert f32(f32(0.8) * f32(50)) == f32(40)
    # level windows: level 0 searches -1..0, level 7 searches 6..7
    for name, y, lvl, bad, good in (('l0', 400.0, 0, 1, 0), ('l7', 300.0, 7, 5, 6)):
        D = _desc(rng)
        out[name] = (len(pts), fr.kp(551, y, flip(D, range(1)), octave=bad), fr.kp(549, y, flip(D, range(1, 9)), octave=good))
        pts.append(dict(x=550.0, y=y, d=D, level=lvl))

    def proof(r):
        mp = r['mp']
        i, kf_, kn = out['v_eq']; assert mp[kn] == ID_BASE + i and mp[kf_] == -1
        i, kf_, kn = out['v_below']; assert mp[kf_] == ID_BASE + i and mp[kn] == -1
        assert mp[out['h100'][1]] == ID_BASE + out['h100'][0] and mp[out['h101'][1]] == -1
        assert mp[out['r40'][1]] == ID_BASE + out['r40'][0] and mp[out['r41'][1]] == -1 and mp[out['r41'][2]] == -1
        for key in ('l0', 'l7'):
            i, kb, kg = out[key]; assert mp[kb] == -1 and mp[kg] == ID_BASE + i
        assert r['nm'] == 6
    _local_case('local_gate_edges', fr, pts, LOCAL, ['view_cos_edge', 'th_high_edge', 'ratio_edge', 'level_window_edges'], proof)


_local_gates()


def _local_th(params):
    """th == 1.0f leaves the radius alone (4 px: a keypoint exactly 4 px away is outside); any other th multiplies it."""
    rng = np.random.RandomState(41)
    fr = _Frame()
    D = _desc(rng)
    far = fr.kp(304.0, 200.0, flip(D, range(2)))
    near = fr.kp(301.0, 200.0, flip(D, range(2, 30)))
    pts = [dict(x=300.0, y=200.0, d=D, level=0)]
    one = params['th'] == 1.0

    def proof(r):
        assert r['mp'][far] == (-1 if one else ID_BASE) and r['mp'][near] == (ID_BASE if one else -1)
    _local_case('local_th_%s' % ('one' if one else 'above_one'), fr, pts, params, ['th_factor'], proof)


_local_th(LOCAL)
_local_th(LOCAL_TH)


# ---- Sim3 SearchByProjection (fuse kernel, variant 3): more than 64 points racing for one feature set -------------------------------
def _sim3_case(name, fr, P, paths, proof, matched=None):
    a = fr.arrays()
    kf = P.keyframe()
    xyz = kf['last_xyz'].astype(np.float64)
    nrm = (xyz / np.linalg.norm(xyz, axis=1, keepdims=True)).astype(f32)
    _case(name, 'sim3', SIM3, paths, proof, **a, **kf, Tcw_cur=EYE, Ow=np.zeros(3, f32), normal=nrm,
          matched=np.full(len(a['kps']), -1, np.int32) if matched is None else matched)


def _sim3_waves():
    rng = np.random.RandomState(50)
    fr, P = _Frame(), _Points()
    D = _desc(rng)
    dist = [30 + k // 4 for k in range(80)] + [50, 51]
    for k, d in enumerate(dist):
        fr.kp(300 - 8.1 + 1.8 * (k % 10), 200 - 8.1 + 1.8 * (k // 10), flip(D, range(d)))
    matched = np.full(len(dist), -1, np.int32); matched[5] = 999
    for _ in range(100):
        P.point(300.0, 200.0, D)

    def proof(r):
        m = r['matched']
        took = sorted(int(v) for v in m if 0 <= v < 999)
        assert took == list(range(80)) and r['nm'] == 80            # waves 1 and 2 both accept (points 64..79)
        assert m[80] == 79 and m[81] == -1 and m[5] == 999          # bestDist == 50 accepted, 51 not
    _sim3_case('sim3_waves', fr, P, ['wave_retry', 'th_low_edge'], proof, matched)


_sim3_waves()


def _sim3_bounds():
    B_ = tum1_bounds()
    rng = np.random.RandomState(51)
    fr, P = _Frame(B_), _Points()
    D = _desc(rng)
    R = fr.kp(B_[2] - 6.0, 250, flip(D, range(3)))
    p_r = P.point(B_[2], 250.0, D, mode=('eq', 'near'))          # u == max_x: KeyFrame::IsInImage is half-open
    D = _desc(rng)
    L_ = fr.kp(B_[0] + 2.0, 150, flip(D, range(3)))
    p_l = P.point(B_[0], 150.0, D, mode=('ge', 'near'))
    assert P.uv(p_r)[0] == f32(B_[2])

    def proof(r):
        assert r['matched'][R] == -1 and r['matched'][L_] == p_l and r['nm'] == 1
    _sim3_case('sim3_tum1_bounds', fr, P, ['bounds'], proof)


_sim3_bounds()


# ---- SearchForInitialization: steals, TH_LOW and the ratio at nnratio -----------------------------------------------------------------
def _init():
    rng = np.random.RandomState(60)
    f1, f2 = _Frame(), _Frame()
    prev = []
    ids = {}

    def one(name, xy, d, octave=0):
        ids[name] = f1.kp(xy[0], xy[1], d, octave); prev.append(xy)
    # steal: e matches X at 20, f (later, 10) steals it, g (10, equal) cannot and takes Y
    D = _desc(rng)
    X = f2.kp(100, 100, D); Y = f2.kp(104, 100, flip(D, range(200, 230)))
    one('e', (100.0, 100.0), flip(D, range(20))); one('f', (100.0, 100.0), flip(D, range(20, 30))); one('g', (100.0, 100.0), flip(D, range(30, 40)))
    # TH_LOW, nnratio 0.75: 50 vs 80 accepted, 51 rejected, 45 vs 60 rejected (45 < 45.0f is false), 44 vs 60 accepted
    for name, x, best, second in (('a', 300.0, 50, 80), ('b', 400.0, 51, None), ('c', 500.0, 45, 60), ('d', 600.0, 44, 60)):
        D = _desc(rng)
        ids['k' + name] = f2.kp(x + 1, 300, flip(D, range(best)))
        if second:
            f2.kp(x - 1, 300, flip(D, range(128, 128 + second)))
        one(name, (x, 300.0), D)
    # octave filters: an F1 keypoint above level 0 is skipped, an F2 keypoint above level 0 is not a candidate
    D = _desc(rng)
    ids['ko'] = f2.kp(200, 400, D, octave=1); ids['kz'] = f2.kp(202, 400, flip(D, range(5)))
    one('h', (200.0, 400.0), D, octave=1); one('i', (200.0, 400.0), flip(D, range(1)))
    a1, a2 = f1.arrays(), f2.arrays()

    def proof(r):
        m = r['m12']
        assert m[ids['e']] == -1 and m[ids['f']] == X and m[ids['g']] == Y
        assert m[ids['a']] == ids['ka'] and m[ids['b']] == -1 and m[ids['c']] == -1 and m[ids['d']] == ids['kd']
        assert m[ids['h']] == -1 and m[ids['i']] == ids['kz']
        assert r['nm'] == 5
    _case('init_steal_and_edges', 'init', INIT, ['steal', 'th_low_edge', 'ratio_edge'], proof, k1=a1['kps'], d1=a1['desc'], k2=a2['kps'], d2=a2['desc'],
          prev=np.array(prev, f32), bounds=FULL)


_init()


# ---------------------------------------------------------------------------------------------------------------------------------------
def frame_arrays(c, which=''):
    """O.FrameArrays of a case's current frame (which='') or of F1 / F2 of an initialisation case (which='1' / '2')."""
    if which:
        return O.FrameArrays(c['k' + which], np.full(len(c['k' + which]), -1, f32), c['d' + which], W, H, CAM['fx'], CAM['fy'], CAM['cx'], CAM['cy'],
                             CAM['bf'], SF, bounds=c['bounds'])
    return O.FrameArrays(c['kps'], c['uright'], c['desc'], W, H, CAM['fx'], CAM['fy'], CAM['cx'], CAM['cy'], CAM['bf'], SF, bounds=c['bounds'])


def run_oracle(c):
    p = c['params']
    k = c['kind']
    if k == 'last':
        nm, mp, nc = O.search_by_projection_last(frame_arrays(c), c['Tcw_cur'], c['Tcw_last'], c['last_has'], c['last_xyz'], c['last_desc'], c['last_obs'],
                                                 c['last_oct'], c['last_angle'], p['th'], mono=p['mono'], check_ori=p['check_ori'], cur_mp=c['cur_mp'],
                                                 cur_mp_obs=c['cur_obs'])
        return dict(nm=nm, mp=mp, ncand=nc)
    if k == 'kf':
        nm, mp, nc = O.search_by_projection_kf(frame_arrays(c), c['Tcw_cur'], c['kf_valid'], c['last_xyz'], c['last_desc'], c['last_angle'], c['min_dist'],
                                               c['max_dist'], p['th'], p['orb_dist'], p['check_ori'], cur_mp=c['cur_mp'])
        return dict(nm=nm, mp=mp, ncand=nc)
    if k == 'local':
        nm, mp, ob, nc = O.search_by_projection_local(frame_arrays(c), c['inview'], c['projx'], c['projy'], c['projxr'], c['level'], c['viewcos'], c['mp_desc'],
                                                      c['mp_obs'], p['th'], p['nnratio'], c['f_mp'], c['f_obs'], id_base=ID_BASE)
        return dict(nm=nm, mp=mp, obs=ob, ncand=nc)
    if k == 'sim3':
        nm, m = O.search_by_projection_sim3(frame_arrays(c), c['Tcw_cur'], c['Ow'], c['kf_valid'], c['last_xyz'], c['normal'], c['min_dist'], c['max_dist'],
                                            c['last_desc'], float(p['th']), c['matched'])
        return dict(nm=nm, matched=m)
    nm, m, pv = O.search_for_initialization(frame_arrays(c, '1'), frame_arrays(c, '2'), c['prev'], p['window'], p['nnratio'], p['check_ori'])
    return dict(nm=nm, m12=m, prev=pv)


def names(kind=None):
    return [n for n, c in CASES.items() if kind is None or c['kind'] == kind]


def path_counts():
    """{path label: number of cases whose proof demonstrates it}."""
    out = {}
    for c in CASES.values():
        for p in c['paths']:
            out[p] = out.get(p, 0) + 1
    return out
