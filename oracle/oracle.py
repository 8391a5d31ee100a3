"""ctypes binding of the CPU oracle (oracle/liboracle.so).  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module.  The product package (sg-slam_b200/) never does.
"""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None

KP_DTYPE = np.dtype([('x', '<f4'), ('y', '<f4'), ('size', '<f4'), ('angle', '<f4'), ('response', '<f4'),
                     ('octave', '<i4'), ('class_id', '<i4')])
assert KP_DTYPE.itemsize == 28


class OrbParams(C.Structure):
    _fields_ = [('nfeatures', C.c_int32), ('scaleFactor', C.c_float), ('nlevels', C.c_int32),
                ('iniThFAST', C.c_int32), ('minThFAST', C.c_int32)]


class SgoFrame(C.Structure):
    _fields_ = [('N', C.c_int32), ('keysUn', C.c_void_p), ('uRight', C.c_void_p), ('desc', C.c_void_p),
                ('minX', C.c_float), ('minY', C.c_float), ('maxX', C.c_float), ('maxY', C.c_float),
                ('fx', C.c_float), ('fy', C.c_float), ('cx', C.c_float), ('cy', C.c_float), ('bf', C.c_float),
                ('nlevels', C.c_int32), ('scaleFactors', C.c_void_p), ('logScaleFactor', C.c_float)]


def build(force=False):
    so = os.path.join(_HERE, 'liboracle.so')
    src = os.path.join(_HERE, 'sgs_oracle.cpp')
    if force or not os.path.exists(so) or (os.path.exists(src) and os.path.getmtime(src) > os.path.getmtime(so)):
        subprocess.check_call(['make', '-C', _HERE, '-s', 'liboracle.so'])
    return so


def lib():
    global _LIB
    if _LIB is None:
        _LIB = C.CDLL(build())
        _LIB.sgo_fast_atan2.restype = C.c_float
        _LIB.sgo_fast_atan2.argtypes = [C.c_float, C.c_float]
        _LIB.sgo_ic_angle.restype = C.c_float
        _LIB.sgo_extract_dump.restype = C.c_void_p
    return _LIB


_libm = None


def logf(x):
    """libm's float logarithm: what `log(float)` calls in the reference (mfLogScaleFactor = log(mfScaleFactor), src/Frame.cc:139; PredictScale,
    src/MapPoint.cc:402-418).  numpy's float32 log is a different implementation (1 ulp apart at 1.2f)."""
    global _libm
    if _libm is None:
        import ctypes.util
        _libm = C.CDLL(ctypes.util.find_library('m'))
        _libm.logf.restype = C.c_float; _libm.logf.argtypes = [C.c_float]
    return np.float32(_libm.logf(float(np.float32(x))))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def params(nfeatures=1000, scale=1.2, nlevels=8, ini=20, mn=7):
    return OrbParams(nfeatures, scale, nlevels, ini, mn)


def orb_tables(p):
    n = p.nlevels
    sc, isc, s2, is2 = (np.zeros(n, np.float32) for _ in range(4))
    npl = np.zeros(n, np.int32)
    umax = np.zeros(16, np.int32)
    lib().sgo_orb_tables(C.byref(p), _p(sc), _p(isc), _p(s2), _p(is2), _p(npl), _p(umax))
    return dict(scale=sc, invScale=isc, sigma2=s2, invSigma2=is2, nPerLevel=npl, umax=umax)


def level_size(p, w, h, level):
    lw, lh = C.c_int32(), C.c_int32()
    lib().sgo_level_size(C.byref(p), w, h, level, C.byref(lw), C.byref(lh))
    return lw.value, lh.value


def resize(src, dw, dh):
    src = np.ascontiguousarray(src, np.uint8)
    dst = np.zeros((dh, dw), np.uint8)
    lib().sgo_resize(_p(src), src.shape[1], src.shape[0], src.strides[0], _p(dst), dw, dh, dw)
    return dst


def fast_view(view, threshold, nms=True):
    """cv::FAST on a (possibly non-contiguous) 2-D uint8 view; returns int32 [n,3] (x, y, score)."""
    assert view.dtype == np.uint8 and view.strides[1] == 1
    h, w = view.shape
    out = np.zeros((max(1, w * h), 3), np.int32)
    n = lib().sgo_fast_view(C.c_void_p(view.ctypes.data), view.strides[0], w, h, threshold, int(nms), _p(out), out.shape[0])
    assert n >= 0
    return out[:n].copy()


def fast_level(img, ini=20, mn=7):
    img = np.ascontiguousarray(img, np.uint8)
    cap = img.size // 4 + 16
    out = np.zeros((cap, 3), np.float32)
    nf = C.c_int32()
    n = lib().sgo_fast_level(_p(img), img.shape[1], img.shape[0], img.strides[0], ini, mn, _p(out), cap, C.byref(nf))
    assert n >= 0
    return out[:n].copy(), nf.value


def octree(cands, minX, maxX, minY, maxY, N):
    cands = np.ascontiguousarray(cands, np.float32)
    sel = np.zeros(N + 64 + len(cands), np.int32)
    n = lib().sgo_octree(_p(cands), len(cands), minX, maxX, minY, maxY, N, _p(sel), len(sel))
    assert n >= 0
    return sel[:n].copy()


def fast_atan2(y, x):
    return lib().sgo_fast_atan2(float(y), float(x))


def ic_angle(img, x, y):
    img = np.ascontiguousarray(img, np.uint8)
    m01, m10 = C.c_int32(), C.c_int32()
    a = lib().sgo_ic_angle(_p(img), img.shape[1], img.shape[0], img.strides[0], C.c_float(x), C.c_float(y), C.byref(m01), C.byref(m10))
    return a, m01.value, m10.value


def blur(img):
    img = np.ascontiguousarray(img, np.uint8)
    out = np.zeros_like(img)
    lib().sgo_blur(_p(img), img.shape[1], img.shape[0], img.strides[0], _p(out), out.strides[0])
    return out


def brief(blurred, x, y, angle):
    blurred = np.ascontiguousarray(blurred, np.uint8)
    d = np.zeros(32, np.uint8)
    lib().sgo_brief(_p(blurred), blurred.shape[1], blurred.shape[0], blurred.strides[0], C.c_float(x), C.c_float(y), C.c_float(angle), _p(d))
    return d


def pattern_extent(angle):
    return lib().sgo_pattern_extent(C.c_float(angle))


def extract(img, p=None):
    p = p or params()
    img = np.ascontiguousarray(img, np.uint8)
    cap = p.nfeatures + 8 * p.nlevels + 64
    kps = np.zeros(cap, KP_DTYPE)
    desc = np.zeros((cap, 32), np.uint8)
    n = lib().sgo_extract(C.byref(p), _p(img), img.shape[1], img.shape[0], img.strides[0], _p(kps), _p(desc), cap)
    assert n >= 0, n
    return kps[:n].copy(), desc[:n].copy()


class ExtractDump:
    """Per-stage outputs of one oracle extraction (pyramid, candidates, blurred levels, final)."""

    def __init__(self, img, p=None):
        self.p = p or params()
        img = np.ascontiguousarray(img, np.uint8)
        L = lib()
        h = C.c_void_p(L.sgo_extract_dump(C.byref(self.p), _p(img), img.shape[1], img.shape[0], img.strides[0]))
        try:
            n = L.sgo_dump_nkps(h)
            self.kps = np.zeros(n, KP_DTYPE)
            self.desc = np.zeros((n, 32), np.uint8)
            if n:
                L.sgo_dump_kps(h, _p(self.kps), _p(self.desc))
            self.nfallback = L.sgo_dump_nfallback(h)
            self.pyramid, self.blurred, self.cands = [], [], []
            for lvl in range(self.p.nlevels):
                for which, dst in ((0, self.pyramid), (1, self.blurred)):
                    w, hh = C.c_int32(), C.c_int32()
                    sz = L.sgo_dump_level(h, lvl, which, C.byref(w), C.byref(hh), None)
                    if sz > 0:
                        a = np.zeros((hh.value, w.value), np.uint8)
                        L.sgo_dump_level(h, lvl, which, C.byref(w), C.byref(hh), _p(a))
                        dst.append(a)
                    else:
                        dst.append(None)
                nc = L.sgo_dump_cands(h, lvl, None, 0)
                c = np.zeros((max(nc, 1), 3), np.float32)
                L.sgo_dump_cands(h, lvl, _p(c), nc)
                self.cands.append(c[:nc].copy())
        finally:
            L.sgo_dump_free(h)


def hamming(a, b):
    a = np.ascontiguousarray(a, np.uint8); b = np.ascontiguousarray(b, np.uint8)
    return lib().sgo_hamming(_p(a), _p(b))


def bf_match(q, t):
    q = np.ascontiguousarray(q, np.uint8); t = np.ascontiguousarray(t, np.uint8)
    bi = np.zeros(len(q), np.int32); bd = np.zeros(len(q), np.int32); sd = np.zeros(len(q), np.int32)
    lib().sgo_bf_match(_p(q), len(q), _p(t), len(t), _p(bi), _p(bd), _p(sd))
    return bi, bd, sd


class FrameArrays:
    """Keeps the numpy arrays behind an SgoFrame alive.  bounds = (min_x, min_y, max_x, max_y) (Frame::ComputeImageBounds), default (0, 0, w, h)."""

    def __init__(self, keysUn, uRight, desc, w, h, fx, fy, cx, cy, bf, scaleFactors, bounds=None):
        self.keysUn = np.ascontiguousarray(keysUn, KP_DTYPE)
        self.uRight = np.ascontiguousarray(uRight, np.float32)
        self.desc = np.ascontiguousarray(desc, np.uint8)
        self.scaleFactors = np.ascontiguousarray(scaleFactors, np.float32)
        b = (0.0, 0.0, float(w), float(h)) if bounds is None else tuple(float(v) for v in bounds)
        self.c = SgoFrame(len(self.keysUn), self.keysUn.ctypes.data, self.uRight.ctypes.data, self.desc.ctypes.data,
                          *b, fx, fy, cx, cy, bf, len(self.scaleFactors),
                          self.scaleFactors.ctypes.data, float(logf(self.scaleFactors[1])) if len(self.scaleFactors) > 1 else 0.0)


def features_in_area(fr, x, y, r, minLevel=-1, maxLevel=-1):
    out = np.zeros(fr.c.N + 1, np.int32)
    n = lib().sgo_features_in_area(C.byref(fr.c), C.c_float(x), C.c_float(y), C.c_float(r), minLevel, maxLevel, _p(out), len(out))
    assert n >= 0
    return out[:n].copy()


def search_by_projection_last(cur, Tcw_cur, Tcw_last, last_has_mp, last_xyz, last_desc, last_obs, last_octave,
                              last_angle, th, mono=False, check_ori=True, cur_mp=None, cur_mp_obs=None):
    n = len(last_has_mp)
    Tc = np.ascontiguousarray(Tcw_cur, np.float32); Tl = np.ascontiguousarray(Tcw_last, np.float32)
    has = np.ascontiguousarray(last_has_mp, np.uint8); xyz = np.ascontiguousarray(last_xyz, np.float32)
    ld = np.ascontiguousarray(last_desc, np.uint8); lo = np.ascontiguousarray(last_obs, np.uint8)
    loct = np.ascontiguousarray(last_octave, np.int32); la = np.ascontiguousarray(last_angle, np.float32)
    mp = np.full(cur.c.N, -1, np.int32) if cur_mp is None else np.ascontiguousarray(cur_mp, np.int32).copy()
    mpo = None if cur_mp_obs is None else np.ascontiguousarray(cur_mp_obs, np.uint8)
    ncand = C.c_int64()
    nm = lib().sgo_search_by_projection_last(C.byref(cur.c), _p(Tc), _p(Tl), n, _p(has), _p(xyz), _p(ld), _p(lo), _p(loct),
                                             _p(la), C.c_float(th), int(mono), int(check_ori), _p(mp),
                                             _p(mpo) if mpo is not None else None, C.byref(ncand))
    return nm, mp, ncand.value


def search_by_projection_kf(cur, Tcw_cur, kf_valid, kf_xyz, kf_desc, kf_angle, min_dist, max_dist, th, orb_dist, check_ori=True, cur_mp=None,
                            log_scale_factor=None):
    """SearchByProjection(Frame&, KeyFrame*, sAlreadyFound, th, ORBdist) (src/ORBmatcher.cc:1474-1601): returns (nmatches, cur_mp, ncand)."""
    n = len(kf_valid)
    Tc = np.ascontiguousarray(Tcw_cur, np.float32)
    a = [np.ascontiguousarray(kf_valid, np.uint8), np.ascontiguousarray(kf_xyz, np.float32), np.ascontiguousarray(kf_desc, np.uint8),
         np.ascontiguousarray(kf_angle, np.float32), np.ascontiguousarray(min_dist, np.float32), np.ascontiguousarray(max_dist, np.float32)]
    mp = np.full(cur.c.N, -1, np.int32) if cur_mp is None else np.ascontiguousarray(cur_mp, np.int32).copy()
    if log_scale_factor is None:
        log_scale_factor = float(logf(1.2))
    ncand = C.c_int64()
    fn = lib().sgo_search_by_projection_kf
    fn.restype = C.c_int
    nm = fn(C.byref(cur.c), _p(Tc), n, *[_p(x) for x in a], C.c_float(th), int(orb_dist), int(check_ori), C.c_float(log_scale_factor), _p(mp),
            C.byref(ncand))
    return nm, mp, ncand.value


def search_by_projection_local(fr, inview, projx, projy, projxr, level, viewcos, mp_desc, mp_obs, th, nnratio,
                               f_mp, f_mp_obs, id_base=0):
    n = len(inview)
    a = [np.ascontiguousarray(inview, np.uint8), np.ascontiguousarray(projx, np.float32), np.ascontiguousarray(projy, np.float32),
         np.ascontiguousarray(projxr, np.float32), np.ascontiguousarray(level, np.int32), np.ascontiguousarray(viewcos, np.float32),
         np.ascontiguousarray(mp_desc, np.uint8), np.ascontiguousarray(mp_obs, np.uint8)]
    mp = np.ascontiguousarray(f_mp, np.int32).copy(); mpo = np.ascontiguousarray(f_mp_obs, np.uint8).copy()
    ncand = C.c_int64()
    nm = lib().sgo_search_by_projection_local(C.byref(fr.c), n, *[_p(x) for x in a], C.c_float(th), C.c_float(nnratio), id_base,
                                              _p(mp), _p(mpo), C.byref(ncand))
    return nm, mp, mpo, ncand.value


def dynreject(cur_xy, prev_xy, F, boxes, have_dyn, nfeatures):
    cur = np.ascontiguousarray(cur_xy, np.float32); prev = np.ascontiguousarray(prev_xy, np.float32)
    n = len(cur)
    Fm = None if F is None else np.ascontiguousarray(F, np.float64).reshape(9)
    bx = np.ascontiguousarray(boxes, np.float32).reshape(-1, 4) if boxes is not None and len(boxes) else np.zeros((0, 4), np.float32)
    keep = np.zeros(n, np.uint8); dist = np.zeros(n, np.float64); rest = C.c_int32()
    s = lib().sgo_dynreject(_p(cur), _p(prev), n, _p(Fm) if Fm is not None else None, _p(bx), len(bx), int(have_dyn), nfeatures,
                            _p(keep), _p(dist), C.byref(rest))
    return s, keep, dist, bool(rest.value)


def lk_track(I, J, pts):
    """calcOpticalFlowPyrLK(I, J, pts) with the reference's parameters (src/Frame.cc:445): returns the tracked points [n,2]."""
    I = np.ascontiguousarray(I, np.uint8); J = np.ascontiguousarray(J, np.uint8)
    p = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    out = np.zeros_like(p)
    lib().sgo_lk_track(_p(I), _p(J), I.shape[1], I.shape[0], I.strides[0], _p(p), len(p), _p(out))
    return out


def lk_pyr_level(img, level):
    img = np.ascontiguousarray(img, np.uint8)
    w, h = C.c_int32(), C.c_int32()
    lib().sgo_lk_pyr_level(_p(img), img.shape[1], img.shape[0], img.strides[0], level, None, C.byref(w), C.byref(h))
    out = np.zeros((h.value, w.value), np.uint8)
    lib().sgo_lk_pyr_level(_p(img), img.shape[1], img.shape[0], img.strides[0], level, _p(out), C.byref(w), C.byref(h))
    return out


def run7point(m1, m2):
    """fundam.cpp run7Point on 7 point pairs: list of 3x3 double matrices (1..3)."""
    a = np.ascontiguousarray(m1, np.float32).reshape(7, 2); b = np.ascontiguousarray(m2, np.float32).reshape(7, 2)
    F = np.zeros(27, np.float64)
    lib().sgo_run7point.restype = C.c_int
    n = lib().sgo_run7point(_p(a), _p(b), _p(F))
    return [F[9 * k:9 * k + 9].reshape(3, 3).copy() for k in range(max(n, 0))]


def find_fundamental_ransac(pts1, pts2, thresh=1.0, confidence=0.99, max_iters=1000, small_sample=True):
    """cv::findFundamentalMat(pts1, pts2, FM_RANSAC, thresh, confidence) (src/Frame.cc:469-472).
    Returns (F 3x3 float64 or None, mask uint8 [n], info int32 [3] = iterations run, inliers, final niters).
    Like OpenCV: 15 pairs and more -> RANSAC; 8..14 -> LMedS (pinned for 14 pairs, numerically arbitrary below -- see tests/test_fundamental.py);
    exactly 7 -> the first solution of the 7-point solver; fewer -> None.  (`small_sample` is kept for old call sites and ignored.)"""
    a = np.ascontiguousarray(pts1, np.float32).reshape(-1, 2); b = np.ascontiguousarray(pts2, np.float32).reshape(-1, 2)
    F = np.zeros(9, np.float64); mask = np.zeros(len(a), np.uint8); info = np.zeros(3, np.int32)
    if len(a) < 7:
        return None, mask, info
    fn = lib().sgo_find_fundamental_ransac
    fn.restype = C.c_int
    fn.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    ok = fn(_p(a), _p(b), len(a), float(thresh), float(confidence), int(max_iters), _p(F), _p(mask), _p(info))
    return (F.reshape(3, 3) if ok else None), mask, info


def select_static_pairs(cur, prev, boxes, prev_have_dyn):
    """src/Frame.cc:454-472: the point pairs handed to findFundamentalMat."""
    a = np.ascontiguousarray(cur, np.float32).reshape(-1, 2); b = np.ascontiguousarray(prev, np.float32).reshape(-1, 2)
    bx = np.ascontiguousarray(boxes, np.float32).reshape(-1, 4)
    s1 = np.zeros_like(a); s2 = np.zeros_like(b)
    lib().sgo_select_static_pairs.restype = C.c_int
    n = lib().sgo_select_static_pairs(_p(a), _p(b), len(a), _p(bx), len(bx), int(bool(prev_have_dyn)), _p(s1), _p(s2))
    return s1[:n], s2[:n]


def stereo_from_rgbd(kps, depth, bf, kps_un=None):
    """Frame::ComputeStereoFromRGBD (src/Frame.cc:893-914): (u_right, depth) per keypoint."""
    k = np.ascontiguousarray(kps); d = np.ascontiguousarray(depth, np.float32)
    ur = np.zeros(len(k), np.float32); dz = np.zeros(len(k), np.float32)
    ku = None if kps_un is None else np.ascontiguousarray(kps_un)
    lib().sgo_stereo_from_rgbd(_p(k), _p(ku) if ku is not None else None, len(k), _p(d), d.strides[0] // 4, C.c_float(bf), _p(ur), _p(dz))
    return ur, dz


def is_in_frustum(Tcw, cam, nlevels, log_scale_factor, xyz, normal, min_dist, max_dist, viewing_cos_limit=0.5):
    """Frame::isInFrustum for n map points.  cam = (fx, fy, cx, cy, bf, minX, minY, maxX, maxY).
    Returns dict(inview, proj_x, proj_y, proj_xr, level, view_cos)."""
    T = np.ascontiguousarray(Tcw, np.float32).reshape(16); cm = np.ascontiguousarray(cam, np.float32)
    X = np.ascontiguousarray(xyz, np.float32).reshape(-1, 3); N = np.ascontiguousarray(normal, np.float32).reshape(-1, 3)
    mn = np.ascontiguousarray(min_dist, np.float32); mx = np.ascontiguousarray(max_dist, np.float32)
    n = len(X)
    out = dict(inview=np.zeros(n, np.uint8), proj_x=np.zeros(n, np.float32), proj_y=np.zeros(n, np.float32), proj_xr=np.zeros(n, np.float32),
               level=np.zeros(n, np.int32), view_cos=np.zeros(n, np.float32))
    lib().sgo_is_in_frustum(_p(T), _p(cm), int(nlevels), C.c_float(log_scale_factor), C.c_float(viewing_cos_limit), n, _p(X), _p(N), _p(mn), _p(mx),
                            _p(out['inview']), _p(out['proj_x']), _p(out['proj_y']), _p(out['proj_xr']), _p(out['level']), _p(out['view_cos']))
    return out


def undistort_points(xy, fx, fy, cx, cy, dist5):
    """cv::undistortPoints(xy, K, dist, R=I, P=K) (Frame::UndistortKeyPoints, src/Frame.cc:654-684)."""
    a = np.ascontiguousarray(xy, np.float32).reshape(-1, 2); d = np.ascontiguousarray(dist5, np.float32)
    out = np.zeros_like(a)
    lib().sgo_undistort_points(_p(a), len(a), C.c_float(fx), C.c_float(fy), C.c_float(cx), C.c_float(cy), _p(d), _p(out))
    return out


class Vocabulary:
    """DBoW2 vocabulary tree as flat arrays: parent[i] of node i (node 0 = root, parent -1), node descriptors [n,32], leaf weights."""

    def __init__(self, k, L, parent, desc, weight):
        self.k, self.L = k, L
        self.parent = np.ascontiguousarray(parent, np.int32); self.desc = np.ascontiguousarray(desc, np.uint8); self.weight = np.ascontiguousarray(weight, np.float64)
        lib().sgo_voc_create.restype = C.c_void_p
        self.h = C.c_void_p(lib().sgo_voc_create(k, L, len(self.parent), _p(self.parent), _p(self.desc), _p(self.weight)))

    def __del__(self):
        try:
            lib().sgo_voc_free(self.h)
        except Exception:
            pass

    def transform(self, desc, levelsup=4):
        """Per feature: (word id, weight, node id at level L - levelsup) -- TemplatedVocabulary::transform, Frame::ComputeBoW (src/Frame.cc:421-428)."""
        d = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
        word = np.zeros(len(d), np.int32); w = np.zeros(len(d), np.float64); node = np.zeros(len(d), np.int32)
        lib().sgo_bow_transform(self.h, _p(d), len(d), int(levelsup), _p(word), _p(w), _p(node))
        return word, w, node


def bow_vector(word, weight):
    n = len(word)
    ow = np.zeros(n, np.int32); ov = np.zeros(n, np.float64)
    c = lib().sgo_bow_vector(_p(np.ascontiguousarray(word, np.int32)), _p(np.ascontiguousarray(weight, np.float64)), n, _p(ow), _p(ov))
    return ow[:c], ov[:c]


def search_by_bow(kf_node, kf_weight, kf_valid, kf_desc, kf_angle, f_node, f_weight, f_desc, f_angle, nnratio=0.7, check_ori=True):
    """ORBmatcher::SearchByBoW(KeyFrame*, Frame&, ...) (src/ORBmatcher.cc:159-290): (nmatches, match_f[j] = key-frame feature index or -1)."""
    a = [np.ascontiguousarray(kf_node, np.int32), np.ascontiguousarray(kf_weight, np.float64), np.ascontiguousarray(kf_valid, np.uint8),
         np.ascontiguousarray(kf_desc, np.uint8), np.ascontiguousarray(kf_angle, np.float32)]
    b = [np.ascontiguousarray(f_node, np.int32), np.ascontiguousarray(f_weight, np.float64), np.ascontiguousarray(f_desc, np.uint8), np.ascontiguousarray(f_angle, np.float32)]
    m = np.zeros(len(b[0]), np.int32)
    nm = lib().sgo_search_by_bow(len(a[0]), *[_p(x) for x in a], len(b[0]), *[_p(x) for x in b], C.c_float(nnratio), int(check_ori), _p(m))
    return nm, m


def search_by_bow_kfkf(node1, weight1, valid1, desc1, angle1, node2, weight2, valid2, desc2, angle2, nnratio=0.8, check_ori=True):
    """ORBmatcher::SearchByBoW(KeyFrame*, KeyFrame*, vpMatches12) (src/ORBmatcher.cc:524-657): (nmatches, match_1[i1] = feature of KF2 or -1)."""
    a = [np.ascontiguousarray(node1, np.int32), np.ascontiguousarray(weight1, np.float64), np.ascontiguousarray(valid1, np.uint8),
         np.ascontiguousarray(desc1, np.uint8), np.ascontiguousarray(angle1, np.float32)]
    b = [np.ascontiguousarray(node2, np.int32), np.ascontiguousarray(weight2, np.float64), np.ascontiguousarray(valid2, np.uint8),
         np.ascontiguousarray(desc2, np.uint8), np.ascontiguousarray(angle2, np.float32)]
    m = np.zeros(len(a[0]), np.int32)
    nm = lib().sgo_search_by_bow_kfkf(len(a[0]), *[_p(x) for x in a], len(b[0]), *[_p(x) for x in b], C.c_float(nnratio), int(check_ori), _p(m))
    return nm, m


def search_for_triangulation(k1, k2, F12, ex, ey, sigma2, scale, only_stereo=False, check_ori=True):
    """ORBmatcher::SearchForTriangulation (src/ORBmatcher.cc:659-827).  k1 / k2: dicts with node, weight, free, stereo, desc, xy, angle (+ octave for k2)."""
    f32, u8 = np.float32, np.uint8
    a = [np.ascontiguousarray(k1['node'], np.int32), np.ascontiguousarray(k1['weight'], np.float64), np.ascontiguousarray(k1['free'], u8), np.ascontiguousarray(k1['stereo'], u8),
         np.ascontiguousarray(k1['desc'], u8), np.ascontiguousarray(k1['xy'], f32), np.ascontiguousarray(k1['angle'], f32)]
    b = [np.ascontiguousarray(k2['node'], np.int32), np.ascontiguousarray(k2['weight'], np.float64), np.ascontiguousarray(k2['free'], u8), np.ascontiguousarray(k2['stereo'], u8),
         np.ascontiguousarray(k2['desc'], u8), np.ascontiguousarray(k2['xy'], f32), np.ascontiguousarray(k2['octave'], np.int32), np.ascontiguousarray(k2['angle'], f32)]
    Fm = np.ascontiguousarray(F12, f32).reshape(9); s2 = np.ascontiguousarray(sigma2, f32); sc = np.ascontiguousarray(scale, f32)
    m = np.zeros(len(a[0]), np.int32)
    nm = lib().sgo_search_for_triangulation(len(a[0]), *[_p(x) for x in a], len(b[0]), *[_p(x) for x in b], _p(Fm), C.c_float(ex), C.c_float(ey), _p(s2), _p(sc),
                                            int(only_stereo), int(check_ori), _p(m))
    return nm, m


def fuse_search(kf, Tcw, Ow, mp_valid, mp_xyz, mp_normal, min_dist, max_dist, mp_desc, th, inv_level_sigma2, log_scale_factor=None, sim3_variant=0, xform2=None):
    """Search half of ORBmatcher::Fuse(pKF, vpMapPoints, th) (src/ORBmatcher.cc:829-980): (best_idx, best_dist) per map point."""
    f32 = np.float32
    a = [np.ascontiguousarray(mp_valid, np.uint8), np.ascontiguousarray(mp_xyz, f32), np.ascontiguousarray(mp_normal, f32), np.ascontiguousarray(min_dist, f32),
         np.ascontiguousarray(max_dist, f32), np.ascontiguousarray(mp_desc, np.uint8)]
    n = len(a[0])
    bi = np.zeros(n, np.int32); bd = np.zeros(n, np.int32)
    if log_scale_factor is None:
        log_scale_factor = float(logf(1.2))
    T = np.ascontiguousarray(Tcw, f32); O_ = np.ascontiguousarray(Ow, f32); s2 = np.ascontiguousarray(inv_level_sigma2, f32)
    lib().sgo_fuse_search(C.byref(kf.c), _p(T), _p(O_), n, *[_p(x) for x in a], C.c_float(th), _p(s2), C.c_float(log_scale_factor), int(sim3_variant),
                          _p(np.ascontiguousarray(xform2, f32)) if xform2 is not None else None, _p(bi), _p(bd))
    return bi, bd


def search_by_projection_sim3(kf, Tcw, Ow, mp_valid, mp_xyz, mp_normal, min_dist, max_dist, mp_desc, th, kf_matched, log_scale_factor=None):
    """ORBmatcher::SearchByProjection(pKF, Scw, vpPoints, vpMatched, th) (src/ORBmatcher.cc:292-405) with Scw already decomposed into Tcw rows / Ow.
    kf_matched: int32 per key-frame feature, >= 0 = occupied; returns (nmatches, updated copy: claimed features hold the claiming point's index)."""
    f32 = np.float32
    a = [np.ascontiguousarray(mp_valid, np.uint8), np.ascontiguousarray(mp_xyz, f32), np.ascontiguousarray(mp_normal, f32), np.ascontiguousarray(min_dist, f32),
         np.ascontiguousarray(max_dist, f32), np.ascontiguousarray(mp_desc, np.uint8)]
    if log_scale_factor is None:
        log_scale_factor = float(logf(1.2))
    T = np.ascontiguousarray(Tcw, f32); O_ = np.ascontiguousarray(Ow, f32)
    m = np.ascontiguousarray(kf_matched, np.int32).copy()
    nm = lib().sgo_search_by_projection_sim3(C.byref(kf.c), _p(T), _p(O_), len(a[0]), *[_p(x) for x in a], C.c_float(th), C.c_float(log_scale_factor), _p(m))
    return nm, m


def search_for_initialization(f1, f2, prev_xy, window_size=100, nnratio=0.9, check_ori=True):
    """ORBmatcher::SearchForInitialization (src/ORBmatcher.cc:407-522): (nmatches, match12, updated vbPrevMatched)."""
    p = np.ascontiguousarray(prev_xy, np.float32).reshape(-1, 2).copy()
    m = np.zeros(f1.c.N, np.int32)
    nm = lib().sgo_search_for_initialization(C.byref(f1.c), C.byref(f2.c), _p(p), int(window_size), C.c_float(nnratio), int(check_ori), _p(m))
    return nm, m, p


def distinctive_descriptor(desc):
    """MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:242-307): index of the representative descriptor among desc [n,32]."""
    d = np.ascontiguousarray(desc, np.uint8).reshape(-1, 32)
    return int(lib().sgo_distinctive_descriptor(_p(d), len(d)))


def pose_optimization(Tcw, has_mp, xyz, kp_xy, octave, uright, inv_level_sigma2, fx, fy, cx, cy, bf):
    """Optimizer::PoseOptimization (src/Optimizer.cc:239-451): returns (n_inliers, Tcw_out 4x4 float32, outlier uint8 [n])."""
    f32 = np.float32
    T = np.ascontiguousarray(Tcw, f32).reshape(16)
    a = [np.ascontiguousarray(has_mp, np.uint8), np.ascontiguousarray(xyz, f32), np.ascontiguousarray(kp_xy, f32), np.ascontiguousarray(octave, np.int32),
         np.ascontiguousarray(uright, f32), np.ascontiguousarray(inv_level_sigma2, f32)]
    n = len(a[0])
    out = np.zeros(16, f32); outl = np.zeros(n, np.uint8)
    fn = lib().sgo_pose_optimization
    fn.restype = C.c_int
    r = fn(_p(T), n, *[_p(x) for x in a], C.c_float(fx), C.c_float(fy), C.c_float(cx), C.c_float(cy), C.c_float(bf), _p(out), _p(outl))
    return r, out.reshape(4, 4), outl


class SgoChainArgs(C.Structure):
    _fields_ = [('params', C.c_void_p), ('frames', C.c_void_p), ('nframes', C.c_int32), ('w', C.c_int32), ('h', C.c_int32), ('prev_index', C.c_void_p),
                ('boxes', C.c_void_p), ('nboxes', C.c_void_p), ('have_dyn', C.c_void_p), ('max_boxes', C.c_int32), ('depth', C.c_void_p), ('u_right_in', C.c_void_p),
                ('fx', C.c_float), ('fy', C.c_float), ('cx', C.c_float), ('cy', C.c_float), ('bf', C.c_float), ('scale_factors', C.c_void_p),
                ('log_scale_factor', C.c_float), ('point_cap', C.c_int32), ('last_xyz', C.c_void_p), ('last_desc', C.c_void_p), ('last_flags', C.c_void_p),
                ('last_octave', C.c_void_p), ('last_angle', C.c_void_p), ('last_n', C.c_void_p), ('tcw', C.c_void_p), ('th', C.c_float), ('cap', C.c_int32),
                ('kps', C.c_void_p), ('desc', C.c_void_p), ('counts', C.c_void_p), ('prev_xy', C.c_void_p), ('F', C.c_void_p), ('f_ok', C.c_void_p),
                ('keep', C.c_void_p), ('nkeep', C.c_void_p), ('restored', C.c_void_p), ('match', C.c_void_p), ('nmatch', C.c_void_p)]


def online_cpus():
    return int(lib().sgo_online_cpus())


class Chain:
    """The reference's per-frame tracking chain (extract -> LK -> findFundamentalMat -> dyn-reject -> SearchByProjection(cur, last)) for a batch of
    frames inside the C++ oracle (oracle/chain.cpp): one frame per task, `nthreads` pinned worker threads.  Inputs as bench.py builds them
    (make_track_inputs); `want_outputs` allocates the per-frame results for parity checks, otherwise only the counts come back."""

    def __init__(self, frames, pidx, ti, cam, cap, nfeatures=1000, th=15.0, want_outputs=True, p=None):
        self.p = p or params(nfeatures)
        self.a = {}
        keep = self.a
        keep['frames'] = np.ascontiguousarray(frames, np.uint8)
        B, h, w = keep['frames'].shape
        keep['pidx'] = np.ascontiguousarray(pidx, np.int32)
        keep['boxes'] = np.ascontiguousarray(ti['boxes'], np.float32); keep['nb'] = np.ascontiguousarray(ti['nb'], np.int32); keep['have'] = np.ascontiguousarray(ti['have'], np.uint8)
        keep['ur'] = np.ascontiguousarray(ti['ur'], np.float32)
        assert keep['ur'].shape[1] == cap
        keep['sf'] = np.ascontiguousarray(ti['sf'], np.float32)
        for k in ('lxyz', 'ldesc', 'lflags', 'loct', 'lang', 'ln', 'T'):
            keep[k] = np.ascontiguousarray(ti[k])
        pc = keep['lflags'].shape[1]
        o = self.out = {}
        o['counts'] = np.zeros(B, np.int32); o['nkeep'] = np.zeros(B, np.int32); o['restored'] = np.zeros(B, np.int32); o['nmatch'] = np.zeros(B, np.int32); o['f_ok'] = np.zeros(B, np.int32)
        if want_outputs:
            o['kps'] = np.zeros((B, cap), KP_DTYPE); o['desc'] = np.zeros((B, cap, 32), np.uint8); o['prev_xy'] = np.zeros((B, cap, 2), np.float32)
            o['F'] = np.zeros((B, 9), np.float64); o['keep'] = np.zeros((B, cap), np.uint8); o['match'] = np.full((B, cap), -1, np.int32)
        g = lambda k: o[k].ctypes.data if k in o else None
        self.args = SgoChainArgs(C.addressof(self.p), keep['frames'].ctypes.data, B, w, h, keep['pidx'].ctypes.data, keep['boxes'].ctypes.data, keep['nb'].ctypes.data,
                                 keep['have'].ctypes.data, keep['boxes'].shape[1], None, keep['ur'].ctypes.data, cam['fx'], cam['fy'], cam['cx'], cam['cy'], cam['bf'],
                                 keep['sf'].ctypes.data, float(logf(keep['sf'][1])), pc, keep['lxyz'].ctypes.data, keep['ldesc'].ctypes.data, keep['lflags'].ctypes.data,
                                 keep['loct'].ctypes.data, keep['lang'].ctypes.data, keep['ln'].ctypes.data, keep['T'].ctypes.data, th, cap,
                                 g('kps'), g('desc'), g('counts'), g('prev_xy'), g('F'), g('f_ok'), g('keep'), g('nkeep'), g('restored'), g('match'), g('nmatch'))
        self.nframes = B

    def run(self, first=0, count=None, nthreads=1, pin=True):
        count = self.nframes - first if count is None else count
        return int(lib().sgo_chain_batch(C.byref(self.args), int(first), int(count), int(nthreads), 1 if pin else 0))
