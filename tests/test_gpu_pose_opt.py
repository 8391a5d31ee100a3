"""GPU Optimizer::PoseOptimization through the C ABI against the CPU restatement (tests/test_pose_opt.py explains why g2o itself is not the
reference here).  Tolerance: pose entries within one float32 ulp (both sides are FP64 with different summation orders, ~1e-12 apart on the double
pose; rounding that to float32 can add one ulp, no more); outlier flags and inlier counts identical.  tests/test_gpu_pose_opt_cases.py runs the
full case set."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle as O  # noqa: E402
import pose_cases as PC  # noqa: E402
import scenarios as S  # noqa: E402
from pysgs import binding as B  # noqa: E402


def _gpu(scs, cap, use_index):
    import torch
    F = len(scs)
    cam = B.make_camera(640, 480, scs[0]['cam'], S.scale_factors())
    kps = np.zeros((F, cap), B.KP_DTYPE); ur = np.full((F, cap), -1, np.float32); n = np.zeros(F, np.int32); T0 = np.zeros((F, 16), np.float32)
    has = np.zeros((F, cap), np.uint8); idx = np.full((F, cap), -1, np.int32)
    pcap = cap + 50
    pts = np.zeros((F, pcap if use_index else cap, 3), np.float32)
    rs = np.random.RandomState(0)
    for f, s in enumerate(scs):
        m = len(s['xy']); n[f] = m
        kps['x'][f, :m] = s['xy'][:, 0]; kps['y'][f, :m] = s['xy'][:, 1]; kps['octave'][f, :m] = s['octave']; ur[f, :m] = s['uright']; T0[f] = s['T0'].reshape(16)
        has[f, :m] = s['has']
        if use_index:
            perm = rs.permutation(pcap)[:m]
            pts[f, perm] = s['xyz']; idx[f, :m] = np.where(s['has'] == 1, perm, -1)
        else:
            pts[f, :m] = s['xyz']
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    t = dict(T0=dev(T0), kps=dev(kps.view(np.uint8).reshape(-1)), ur=dev(ur), n=dev(n), has=dev(has), idx=dev(idx), pts=dev(pts))
    Tout = torch.zeros((F, 16), device='cuda'); outl = torch.full((F, cap), 9, dtype=torch.uint8, device='cuda'); nin = torch.zeros(F, dtype=torch.int32, device='cuda')
    err = torch.zeros((F, cap, 3), dtype=torch.float64, device='cuda'); lvl = torch.zeros((F, cap), dtype=torch.uint8, device='cuda')
    a = B.PoseOptBatch()
    a.cam = cam
    a.tcw_in, a.kps, a.uright, a.n, a.cap = t['T0'].data_ptr(), t['kps'].data_ptr(), t['ur'].data_ptr(), t['n'].data_ptr(), cap
    a.has_mp = 0 if use_index else t['has'].data_ptr(); a.mp_index = t['idx'].data_ptr() if use_index else 0
    a.points_xyz, a.point_cap = t['pts'].data_ptr(), pcap
    for l in range(8):
        a.inv_level_sigma2[l] = float(scs[0]['inv_s2'][l])
    a.tcw_out, a.outlier, a.ninliers, a.scratch_err, a.scratch_level = Tout.data_ptr(), outl.data_ptr(), nin.data_ptr(), err.data_ptr(), lvl.data_ptr()
    B.check(B.lib().sgs_pose_optimization_batch_device(C.byref(a), F, C.c_void_p(0)))
    torch.cuda.synchronize()
    return Tout.cpu().numpy().reshape(F, 4, 4), outl.cpu().numpy(), nin.cpu().numpy()


def _host(s):
    """sgs_pose_optimization, the single-frame host entry point."""
    m = len(s['xy'])
    kps = np.zeros(m, B.KP_DTYPE); kps['x'] = s['xy'][:, 0]; kps['y'] = s['xy'][:, 1]; kps['octave'] = s['octave']
    s2 = np.zeros(16, np.float32); s2[:len(s['inv_s2'])] = s['inv_s2']
    T = np.zeros(16, np.float32); outl = np.full(m, 9, np.uint8); nin = C.c_int(-1)
    P = lambda a: np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)
    cam = B.make_camera(640, 480, s['cam'], S.scale_factors())
    B.check(B.lib().sgs_pose_optimization(C.byref(cam), P(s['T0'].astype(np.float32).reshape(16)), m, P(kps), P(s['uright'].astype(np.float32)), P(s['has']),
                                          P(s['xyz'].astype(np.float32)), P(s2), P(T), P(outl), C.byref(nin), 0))
    return T.reshape(4, 4), outl, nin.value


def _scenarios():
    scs = [S.pose_scenario(1), S.pose_scenario(2, n=300, outlier_frac=0.3), S.pose_scenario(3, n=1000, mono_frac=1.0), S.pose_scenario(4, n=1000, mono_frac=0.0, noise=1.0),
           S.pose_scenario(5, n=600, outlier_frac=0.0, noise=0.2), S.pose_scenario(6, n=900, pose_err=(0.08, 0.2))]
    few = dict(S.pose_scenario(7, n=40)); few['has'] = np.zeros(40, np.uint8); few['has'][:2] = 1; scs.append(few)           # < 3 correspondences
    few2 = dict(S.pose_scenario(8, n=40)); few2['has'] = np.zeros(40, np.uint8); few2['has'][:8] = 1; scs.append(few2)       # < 10 edges: one round
    return scs


def _check(f, s, T, outl, nin):
    c = s['cam']; m = len(s['xy'])
    rn, rT, ro = O.pose_optimization(s['T0'], s['has'], s['xyz'], s['xy'], s['octave'], s['uright'], s['inv_s2'], c['fx'], c['fy'], c['cx'], c['cy'], c['bf'])
    assert PC.ulp_distance(T, rT).max() <= 1, (f, int(PC.ulp_distance(T, rT).max()), np.abs(T - rT).max())
    used = s['has'] == 1
    assert np.array_equal(outl[:m][used], ro[used]), (f, int((outl[:m][used] != ro[used]).sum()))
    assert nin == rn, (f, nin, rn)


@pytest.mark.parametrize('use_index', [False, True])
def test_pose_optimization_batch(use_index):
    scs = _scenarios()
    T, outl, nin = _gpu(scs, 1000, use_index)
    for f, s in enumerate(scs):
        _check(f, s, T[f], outl[f], nin[f])


def test_pose_optimization_host_entry_point():
    for f, s in enumerate(_scenarios()):
        T, outl, nin = _host(s)
        _check(f, s, T, outl, nin)
        assert (outl[s['has'] == 0] == 0).all()             # the outlier flags are cleared before the optimisation
