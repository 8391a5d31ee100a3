#!/usr/bin/env python3
"""Golden vectors for Frame::isInFrustum (src/Frame.cc:296-352) and Frame::ComputeStereoFromRGBD (:893-914), evaluated with the REAL OpenCV
matrix primitives the reference calls (cv2.gemm for Rcw*P+tcw and -Rcw.t()*tcw, cv2.norm, float32 scalar arithmetic), so that the double
accumulation / single rounding conventions of the oracle are pinned.  Run in the build container:  python tests/golden/make_golden_frustum.py"""
import ctypes
import ctypes.util
import math
import os

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
f32 = np.float32
_libm = ctypes.CDLL(ctypes.util.find_library('m'))
_libm.logf.restype = ctypes.c_float
_libm.logf.argtypes = [ctypes.c_float]


def logf(x):
    """libm's float logarithm -- what `log(float)` in Frame.cc:1017 / MapPoint.cc:411 calls (glibc 2.39 here)."""
    return f32(_libm.logf(float(x)))


def main():
    rs = np.random.RandomState(7)
    n = 4000
    ang = 0.3
    R = np.array([[math.cos(ang), 0, math.sin(ang)], [0.02, 1, -0.01], [-math.sin(ang), 0, math.cos(ang)]], f32)
    t = np.array([[0.3], [-0.1], [0.2]], f32)
    cam = np.array([535.4, 539.2, 320.1, 247.6, 40.0, 0, 0, 640, 480], f32)
    z = rs.uniform(-1, 8, n); pc = np.c_[rs.uniform(-0.75, 0.75, n) * z, rs.uniform(-0.55, 0.55, n) * z, z]       # camera coordinates, some outside the view
    xyz = ((pc - t[:, 0].astype(np.float64)) @ R.astype(np.float64)).astype(f32)                                     # world = R^T (pc - t)
    cen = (-R.T.astype(np.float64) @ t.astype(np.float64))[:, 0]
    to_cam = xyz.astype(np.float64) - cen; dist0 = np.linalg.norm(to_cam, axis=1)
    nrm = rs.normal(0, 1, (n, 3)); nrm = (nrm / np.linalg.norm(nrm, axis=1, keepdims=True))
    face = rs.uniform(size=n) < 0.7
    nrm[face] = (to_cam[face] / dist0[face, None]) + rs.normal(0, 0.3, (int(face.sum()), 3))            # MapPoint normals point from the camera to the point
    nrm = (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(f32)
    maxd = (dist0 * rs.uniform(0.6, 4.0, n)).astype(f32); mind = (maxd / f32(1.2) ** rs.randint(3, 9, n)).astype(f32)
    Ow = cv2.gemm(R, t, -1, None, 0, flags=cv2.GEMM_1_T)            # mOw = -mRcw.t()*mtcw: the MatExpr folds transpose and sign into one gemm call
    logsf = logf(f32(1.2))                                         # mfLogScaleFactor = log(mfScaleFactor), float overload
    out = dict(inview=np.zeros(n, np.uint8), proj_x=np.zeros(n, f32), proj_y=np.zeros(n, f32), proj_xr=np.zeros(n, f32), level=np.zeros(n, np.int32),
               view_cos=np.zeros(n, f32), level_arg=np.zeros(n, np.float64))
    fx, fy, cx, cy, bf = cam[:5]
    for i in range(n):
        P = xyz[i].reshape(3, 1)
        Pc = cv2.gemm(R, P, 1, t, 1)
        if Pc[2, 0] < f32(0):
            continue
        invz = f32(1.0) / Pc[2, 0]
        u = fx * Pc[0, 0] * invz + cx; v = fy * Pc[1, 0] * invz + cy
        if u < cam[5] or u > cam[7] or v < cam[6] or v > cam[8]:
            continue
        PO = P - Ow
        dist = f32(cv2.norm(PO))
        if dist < f32(0.8) * mind[i] or dist > f32(1.2) * maxd[i]:
            continue
        dot = float(PO[0, 0]) * float(nrm[i, 0]) + float(PO[1, 0]) * float(nrm[i, 1]) + float(PO[2, 0]) * float(nrm[i, 2])     # Mat::dot: double accumulator
        vc = f32(dot / float(dist))
        if vc < f32(0.5):
            continue
        ratio = maxd[i] / dist
        arg = float(logf(ratio)) / float(logsf)                          # logf(ratio) / mfLogScaleFactor in double, for diagnostics only
        lv = int(math.ceil(f32(logf(ratio) / logsf)))                    # MapPoint::PredictScale: float log, float division, ceil
        lv = 0 if lv < 0 else (7 if lv >= 8 else lv)
        out['inview'][i] = 1; out['proj_x'][i] = u; out['proj_y'][i] = v; out['proj_xr'][i] = u - bf * invz; out['level'][i] = lv; out['view_cos'][i] = vc
        out['level_arg'][i] = arg
    Tcw = np.eye(4, dtype=f32); Tcw[:3, :3] = R; Tcw[:3, 3] = t[:, 0]
    # ComputeStereoFromRGBD
    depth = (1.0 + rs.uniform(0, 3, (480, 640))).astype(f32); depth[rs.uniform(size=depth.shape) < 0.1] = 0
    kx = rs.uniform(0, 639.99, 500).astype(f32); ky = rs.uniform(0, 479.99, 500).astype(f32)
    d = depth[ky.astype(np.int32), kx.astype(np.int32)]
    ur = np.where(d > 0, kx - f32(40.0) / np.where(d > 0, d, 1).astype(f32), f32(-1)).astype(f32)
    dz = np.where(d > 0, d, f32(-1)).astype(f32)
    looked_up = np.zeros_like(depth); looked_up[ky.astype(np.int32), kx.astype(np.int32)] = d
    depth = looked_up                                                      # only the pixels under the keypoints are read: the rest is stored as 0 (keeps the file small)
    np.savez_compressed(os.path.join(HERE, 'frustum.npz'), Tcw=Tcw, cam=cam, xyz=xyz, normal=nrm, min_dist=mind, max_dist=maxd, logsf=logsf, depth=depth, kx=kx, ky=ky,
                        u_right=ur, depth_out=dz, cv2_version=np.array(cv2.__version__), **out)
    print('in view', int(out['inview'].sum()), 'of', n)


def make_undistort():
    """tests/golden/undistort.npz: cv2.undistortPoints(pts, K, D, None, K) with the TUM1 / TUM2 calibrations of the reference's Examples/*.yaml."""
    rs = np.random.RandomState(3)
    out = {}
    for name, (fx, fy, cx, cy, d) in {'TUM1': (517.306408, 516.469215, 318.643040, 255.313989, [0.262383, -0.953104, -0.005358, 0.002628, 1.163314]),
                                       'TUM2': (520.908620, 521.007327, 325.141442, 249.701764, [0.231222, -0.784899, -0.003257, -0.000105, 0.917205])}.items():
        K = np.array([[fx, 0, cx], [0, fy, cy], [0, 0, 1]], np.float32); D = np.array(d, np.float32)
        pts = np.c_[rs.uniform(0, 640, 1500), rs.uniform(0, 480, 1500)].astype(np.float32)
        pts = np.r_[pts, np.array([[0, 0], [640, 0], [0, 480], [640, 480]], np.float32)]
        out[name + '_K'] = np.array([K[0, 0], K[1, 1], K[0, 2], K[1, 2]], np.float32); out[name + '_D'] = D; out[name + '_pts'] = pts
        out[name + '_und'] = cv2.undistortPoints(pts.reshape(-1, 1, 2), K, D, None, K).reshape(-1, 2)
    np.savez_compressed(os.path.join(HERE, 'undistort.npz'), cv2_version=np.array(cv2.__version__), **out)


if __name__ == '__main__':
    main()
    make_undistort()
