"""Optimizer::PoseOptimization pinned against the REFERENCE'S OWN src/Optimizer.cc, src/Converter.cc and vendored g2o (oracle/_ref/liboptimizer_ref.so: every
file compiled unmodified from the reference tree; see oracle/Makefile, target ref_optimizer).  The image has no Eigen, so the library is built against the Eigen
stand-in of oracle/g2o_shim/Eigen (eager evaluation of Eigen's published formulas): what is pinned is the control flow and arithmetic of Optimizer.cc and g2o --
graph set-up, Levenberg with its lambda schedule and rejected trials, the Huber kernel, the four rounds with their chi-square re-classification, the early exits --
not Eigen's instruction order.  The oracle's sgo_pose_optimization (oracle/pose_opt.cpp, the checker of the GPU's pose_opt_kernel) must return the same inlier
count and the same outlier flags; the pose (float32 on both sides) must agree within 1e-6 -- on every case below it is in fact identical.  The frames are
pose_cases.reference_cases(), shared with the device kernel's tests.  No device needed."""
import ctypes as C
import os

import numpy as np
import pytest

import oracle as O
import pose_cases as PC

LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle', '_ref', 'liboptimizer_ref.so')
pytestmark = pytest.mark.skipif(not os.path.exists(LIB), reason='oracle/_ref/liboptimizer_ref.so not built (reference tree absent)')
v = C.c_void_p
POSE_TOL = 1e-6


def ref_pose_optimization(s):
    L = C.CDLL(LIB); L.ref_pose_optimization.restype = C.c_int
    c = s['cam']; f32 = np.float32
    T = np.ascontiguousarray(s['T0'], f32).reshape(16)
    a = [np.ascontiguousarray(s['has'], np.uint8), np.ascontiguousarray(s['xyz'], f32), np.ascontiguousarray(s['xy'], f32), np.ascontiguousarray(s['octave'], np.int32),
         np.ascontiguousarray(s['uright'], f32)]
    isig = np.ascontiguousarray(s['inv_s2'], f32)
    n = len(a[0]); out = np.zeros(16, f32); outl = np.zeros(n, np.uint8)
    r = L.ref_pose_optimization(T.ctypes.data_as(v), n, *[x.ctypes.data_as(v) for x in a], isig.ctypes.data_as(v), len(isig), C.c_float(c['fx']), C.c_float(c['fy']),
                                C.c_float(c['cx']), C.c_float(c['cy']), C.c_float(c['bf']), out.ctypes.data_as(v), outl.ctypes.data_as(v))
    return r, out.reshape(4, 4), outl


def oracle_pose_optimization(s):
    c = s['cam']
    return O.pose_optimization(s['T0'], s['has'], s['xyz'], s['xy'], s['octave'], s['uright'], s['inv_s2'], c['fx'], c['fy'], c['cx'], c['cy'], c['bf'])


def _same(s, tag):
    rn, rT, ro = ref_pose_optimization(s)
    on, oT, oo = oracle_pose_optimization(s)
    assert rn == on, (tag, rn, on)
    assert np.array_equal(ro, oo), (tag, int((ro != oo).sum()))
    assert np.abs(rT.astype(np.float64) - oT.astype(np.float64)).max() <= POSE_TOL, (tag, np.abs(rT - oT).max())
    return rn, bool(np.array_equal(rT, oT))


def _family(*fams):
    return [(name, s) for fam, name, s in PC.reference_cases() if fam in fams]


def test_tracking_like_frames():
    identical = 0
    for name, s in _family('plain'):
        n, same = _same(s, name)
        assert n > 300
        identical += same
    assert identical >= 20                                  # in practice all of them: both sides round the same double pose to float32


def test_hard_frames_rejected_trials_many_outliers_and_noise():
    for name, s in _family('hard', 'far'):                  # 45 % outliers and 1.5 px noise; starts 0.25 rad / 0.8 m away (rejected trials)
        _same(s, name)


def test_monocular_only_and_stereo_only():
    for name, s in _family('mono', 'stereo'):
        _same(s, name)


def test_early_exits():
    for name, s in _family('few'):                          # fewer than three correspondences: pose untouched, 0 returned (src/Optimizer.cc:338-339)
        n, same = _same(s, name)
        assert n == 0 and same
    for name, s in _family('edges', 'tiny'):                # fewer than ten edges: a single round (:427-428); ten and more: four; a tiny graph with outliers
        _same(s, name)


def test_points_behind_the_camera_and_exact_start():
    for name, s in _family('behind', 'exact'):              # negative depth (flagged in the first round); a start at the optimum (Levenberg's stop rules)
        _same(s, name)


def test_case_set_holds_the_61_reference_frames():
    assert len(PC.reference_cases()) == 61
