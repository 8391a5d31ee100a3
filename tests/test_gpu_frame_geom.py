"""GPU parity of Frame::isInFrustum (+ MapPoint::PredictScale) and Frame::ComputeStereoFromRGBD through the C ABI against the golden
vectors made with the real cv2 primitives and against the CPU oracle.  Floats bit-identical; the predicted level is exact as well (libm's
logf restated for the device in sg-slam_b200/csrc/sgs_logf.h and pinned against the running libm by tests/test_host_logic.py)."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle as O  # noqa: E402
import scenarios as S  # noqa: E402
from pysgs import binding as B  # noqa: E402
from pysgs import synth  # noqa: E402


def _frustum_gpu(Tcw, cam9, xyz, normal, mind, maxd, counts, point_cap, limit=0.5):
    import torch
    F = len(counts)
    sf = S.scale_factors()
    cam = B.make_camera(640, 480, dict(fx=cam9[0], fy=cam9[1], cx=cam9[2], cy=cam9[3], bf=cam9[4]), sf)
    cam.min_x, cam.min_y, cam.max_x, cam.max_y = [float(x) for x in cam9[5:9]]
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d = dict(tcw=dev(Tcw.astype(np.float32)), xyz=dev(xyz), nrm=dev(normal), mn=dev(mind), mx=dev(maxd), n=dev(np.asarray(counts, np.int32)))
    o = dict(inview=torch.zeros((F, point_cap), dtype=torch.uint8, device='cuda'), proj_x=torch.zeros((F, point_cap), device='cuda'),
             proj_y=torch.zeros((F, point_cap), device='cuda'), proj_xr=torch.zeros((F, point_cap), device='cuda'),
             level=torch.zeros((F, point_cap), dtype=torch.int32, device='cuda'), view_cos=torch.zeros((F, point_cap), device='cuda'))
    a = B.FrustumBatch()
    a.cam = cam
    a.tcw, a.mp_xyz, a.mp_normal, a.mp_min_dist, a.mp_max_dist, a.mp_n = [t.data_ptr() for t in (d['tcw'], d['xyz'], d['nrm'], d['mn'], d['mx'], d['n'])]
    a.point_cap = point_cap; a.viewing_cos_limit = limit
    a.mp_inview, a.proj_x, a.proj_y, a.proj_xr, a.level, a.view_cos = [o[k].data_ptr() for k in ('inview', 'proj_x', 'proj_y', 'proj_xr', 'level', 'view_cos')]
    B.check(B.lib().sgs_frustum_batch_device(C.byref(a), F, C.c_void_p(0)))
    torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in o.items()}


def _same(out, ref, level_arg=None):
    """Everything bit-exact, the predicted pyramid level included (MapPoint::PredictScale through the restated libm logf, sgs_logf.h)."""
    assert np.array_equal(out['inview'], ref['inview'])
    for k in ('proj_x', 'proj_y', 'proj_xr', 'view_cos'):
        assert out[k].tobytes() == ref[k].tobytes(), k
    assert np.array_equal(out['level'], ref['level'])


def test_frustum_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, 'frustum.npz'))
    n = len(g['xyz'])
    out = _frustum_gpu(g['Tcw'].reshape(1, 16), g['cam'], g['xyz'].reshape(1, n, 3), g['normal'].reshape(1, n, 3), g['min_dist'].reshape(1, n),
                       g['max_dist'].reshape(1, n), [n], n)
    _same({k: v[0] for k, v in out.items()}, g, g['level_arg'])
    # the host entry point on the same inputs
    cam9 = g['cam']
    cam = B.make_camera(640, 480, dict(fx=cam9[0], fy=cam9[1], cx=cam9[2], cy=cam9[3], bf=cam9[4]), S.scale_factors())
    cam.min_x, cam.min_y, cam.max_x, cam.max_y = [float(x) for x in cam9[5:9]]
    h = dict(inview=np.full(n, 7, np.uint8), proj_x=np.zeros(n, np.float32), proj_y=np.zeros(n, np.float32), proj_xr=np.zeros(n, np.float32),
             level=np.zeros(n, np.int32), view_cos=np.zeros(n, np.float32))
    P = lambda a: np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)
    B.check(B.lib().sgs_frustum(C.byref(cam), P(g['Tcw'].astype(np.float32)), n, P(g['xyz']), P(g['normal']), P(g['min_dist']), P(g['max_dist']), 0.5,
                                *[P(h[k]) for k in ('inview', 'proj_x', 'proj_y', 'proj_xr', 'level', 'view_cos')], 0))
    _same(h, g, g['level_arg'])


def test_frustum_batch_against_oracle():
    rs = np.random.RandomState(5)
    F, cap = 5, 3000
    counts = [3000, 1, 2999, 0, 1234]
    cam9 = np.array([535.4, 539.2, 320.1, 247.6, 40.0, 0, 0, 640, 480], np.float32)
    Tcw = np.zeros((F, 16), np.float32); xyz = np.zeros((F, cap, 3), np.float32); nrm = np.zeros((F, cap, 3), np.float32)
    mn = np.zeros((F, cap), np.float32); mx = np.zeros((F, cap), np.float32)
    for f in range(F):
        a = rs.uniform(-0.4, 0.4); T = np.eye(4, dtype=np.float32)
        T[:3, :3] = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], np.float32); T[:3, 3] = rs.uniform(-0.5, 0.5, 3)
        Tcw[f] = T.reshape(16)
        z = rs.uniform(-1, 8, cap); pc = np.c_[rs.uniform(-0.8, 0.8, cap) * z, rs.uniform(-0.6, 0.6, cap) * z, z]
        xyz[f] = ((pc - T[:3, 3].astype(np.float64)) @ T[:3, :3].astype(np.float64)).astype(np.float32)
        cen = -T[:3, :3].T.astype(np.float64) @ T[:3, 3].astype(np.float64)
        tc = xyz[f].astype(np.float64) - cen; d0 = np.linalg.norm(tc, axis=1)
        nn = tc / d0[:, None] + rs.normal(0, 0.5, (cap, 3)); nrm[f] = (nn / np.linalg.norm(nn, axis=1, keepdims=True)).astype(np.float32)
        mx[f] = (d0 * rs.uniform(0.5, 5, cap)).astype(np.float32); mn[f] = (mx[f] / 1.2 ** rs.randint(2, 9, cap)).astype(np.float32)
    out = _frustum_gpu(Tcw, cam9, xyz, nrm, mn, mx, counts, cap)
    logsf = float(O.logf(1.2))
    for f in range(F):
        n = counts[f]
        ref = O.is_in_frustum(Tcw[f], cam9, 8, logsf, xyz[f, :n], nrm[f, :n], mn[f, :n], mx[f, :n], 0.5)
        _same({k: v[f, :n] for k, v in out.items()}, ref)
        assert not out['inview'][f, n:].any()          # rows past the count are cleared


def test_predict_scale_at_ceil_boundaries():
    """MapPoint::PredictScale (src/MapPoint.cc:402-418) where it is fragile: ratios mfMaxDistance / dist within a few ulps of 1.2^k, so that
    ceil(logf(ratio) / mfLogScaleFactor) flips on the last bit of logf.  Level must equal the oracle's (which calls the real libm) everywhere."""
    rs = np.random.RandomState(11)
    cap = 60000
    cam9 = np.array([535.4, 539.2, 320.1, 247.6, 40.0, 0, 0, 640, 480], np.float32)
    T = np.eye(4, dtype=np.float32).reshape(1, 16)
    z = rs.uniform(0.5, 6.0, cap).astype(np.float32)
    xyz = np.zeros((1, cap, 3), np.float32); xyz[0, :, 2] = z; xyz[0, :, 0] = (rs.uniform(-0.3, 0.3, cap) * z).astype(np.float32); xyz[0, :, 1] = (rs.uniform(-0.2, 0.2, cap) * z).astype(np.float32)
    dist = np.sqrt((xyz[0].astype(np.float64) ** 2).sum(1)).astype(np.float32)
    nrm = (xyz[0] / dist[:, None]).astype(np.float32).reshape(1, cap, 3)
    sf = np.float32(1.2); pw = np.ones(10, np.float32)
    for k in range(1, 10): pw[k] = pw[k - 1] * sf
    k = rs.randint(0, 10, cap)
    target = (pw[k] * dist).astype(np.float32)                      # ratio ~ 1.2^k
    off = rs.randint(-40, 41, cap).astype(np.int32)
    mx = (target.view(np.int32) + off).view(np.float32).reshape(1, cap)
    mn = (mx / np.float32(60.0)).astype(np.float32)
    out = _frustum_gpu(T, cam9, xyz, nrm, mn, mx, [cap], cap)
    logsf = float(O.logf(1.2))
    ref = O.is_in_frustum(T[0], cam9, 8, logsf, xyz[0], nrm[0], mn[0], mx[0], 0.5)
    assert ref['inview'].sum() > cap // 2
    _same({k_: v[0] for k_, v in out.items()}, ref)
    # the sweep really sits on the boundaries: neighbouring ulp offsets give different levels for a good share of the points
    lv = ref['level'][ref['inview'] > 0]
    assert len(np.unique(lv)) >= 8


def test_stereo_from_depth():
    import torch
    rs = np.random.RandomState(4)
    F, cap = 3, 1100
    depth = (0.5 + rs.uniform(0, 4, (F, 480, 640))).astype(np.float32); depth[rs.uniform(size=depth.shape) < 0.15] = 0
    kps = np.zeros((F, cap), B.KP_DTYPE); counts = np.array([1100, 700, 0], np.int32)
    kps['x'] = rs.uniform(0, 639.99, (F, cap)); kps['y'] = rs.uniform(0, 479.99, (F, cap))
    dk = torch.from_numpy(kps.view(np.uint8).reshape(-1)).cuda(); dd = torch.from_numpy(depth).cuda(); dc = torch.from_numpy(counts).cuda()
    ur = torch.zeros((F, cap), device='cuda'); dz = torch.zeros((F, cap), device='cuda')
    v = C.c_void_p
    B.check(B.lib().sgs_stereo_from_depth_batch_device(v(dk.data_ptr()), v(0), v(dc.data_ptr()), cap, F, v(dd.data_ptr()), 640 * 480, 640,
                                                       40.0, v(ur.data_ptr()), v(dz.data_ptr()), v(0)))
    torch.cuda.synchronize()
    ur = ur.cpu().numpy(); dz = dz.cpu().numpy()
    for f in range(F):
        n = counts[f]
        ru, rd = O.stereo_from_rgbd(kps[f, :n], depth[f], 40.0)
        assert ur[f, :n].tobytes() == ru.tobytes() and dz[f, :n].tobytes() == rd.tobytes()
        assert np.all(ur[f, n:] == -1)
    # one shared depth image (frame stride 0): every frame looks up frame 0's depth
    ur2 = torch.zeros((F, cap), device='cuda')
    B.check(B.lib().sgs_stereo_from_depth_batch_device(v(dk.data_ptr()), v(0), v(dc.data_ptr()), cap, F, v(dd.data_ptr()), 0, 640,
                                                       40.0, v(ur2.data_ptr()), v(0), v(0)))
    torch.cuda.synchronize()
    ru, _ = O.stereo_from_rgbd(kps[1, :counts[1]], depth[0], 40.0)
    assert ur2.cpu().numpy()[1, :counts[1]].tobytes() == ru.tobytes()


def test_undistort_and_image_bounds(golden_dir):
    import torch
    g = np.load(os.path.join(golden_dir, 'undistort.npz'))
    v = C.c_void_p
    for name in ('TUM1', 'TUM2'):
        K = g[name + '_K']; D = np.ascontiguousarray(g[name + '_D'], np.float32); pts = np.ascontiguousarray(g[name + '_pts'])
        out = np.zeros_like(pts)
        B.check(B.lib().sgs_undistort_points(pts.ctypes.data_as(v), len(pts), K[0], K[1], K[2], K[3],
                                             D.ctypes.data_as(v), out.ctypes.data_as(v), 0))
        assert out.tobytes() == g[name + '_und'].tobytes(), name
        b = np.zeros(4, np.float32)
        B.check(B.lib().sgs_image_bounds(640, 480, K[0], K[1], K[2], K[3], D.ctypes.data_as(v), b.ctypes.data_as(v), 0))
        c = g[name + '_und'][-4:]          # corners (0,0) (w,0) (0,h) (w,h)
        assert b[0] == min(c[0, 0], c[2, 0]) and b[2] == max(c[1, 0], c[3, 0]) and b[1] == min(c[0, 1], c[1, 1]) and b[3] == max(c[2, 1], c[3, 1])
        # batched keypoint form: two frames, the second shorter; everything but pt is copied
        cap = len(pts)
        kps = np.zeros((2, cap), B.KP_DTYPE); kps['x'] = pts[:, 0]; kps['y'] = pts[:, 1]; kps['octave'] = 3; kps['angle'] = 42.0
        counts = np.array([cap, 100], np.int32)
        dk = torch.from_numpy(kps.view(np.uint8).reshape(-1)).cuda(); dc = torch.from_numpy(counts).cuda(); du = torch.zeros_like(dk)
        B.check(B.lib().sgs_undistort_batch_device(v(dk.data_ptr()), v(dc.data_ptr()), cap, 2, K[0], K[1], K[2], K[3],
                                                   D.ctypes.data_as(v), v(du.data_ptr()), v(0)))
        torch.cuda.synchronize()
        un = du.cpu().numpy().view(B.KP_DTYPE).reshape(2, cap)
        assert np.stack([un['x'][0], un['y'][0]], 1).tobytes() == g[name + '_und'].tobytes()
        assert np.array_equal(un['octave'][1, :100], kps['octave'][1, :100]) and np.array_equal(un['x'][1, :100], un['x'][0, :100])
    zero = np.zeros(5, np.float32); b = np.zeros(4, np.float32)
    B.check(B.lib().sgs_image_bounds(640, 480, 500, 500, 320, 240, zero.ctypes.data_as(v), b.ctypes.data_as(v), 0))
    assert list(b) == [0, 0, 640, 480]
