"""The PoseOptimization case set (tests/pose_cases.py) on the CPU, no device needed.

(a) Every case, designed ones included, gives the same result from the reference's own Optimizer.cc + g2o (oracle/_ref/liboptimizer_ref.so) as from
the restatement oracle/pose_opt.cpp: inlier count and outlier flags equal, pose within 1e-6 (the criterion of tests/test_optimizer_ref.py).

(b) Mutation power.  The device kernel is checked by equality with the restatement, so a kernel slip is caught exactly when the restatement with
the same slip differs from the unmodified one on some case.  Each mutant below is one plausible slip written as text substitutions on
oracle/pose_opt.cpp (which stands alone), compiled with the oracle's flags; a case catches it when the inlier count or a flag differs or a pose
entry moves by more than one float32 ulp -- the bar tests/test_gpu_pose_opt_cases.py holds the kernel to.  Every mutant not declared a survivor
must be caught by at least one case.

Some mutants are tied to the case family built for them (TARGETS): a case of that family must catch the mutant, so that the property the family
was built for stays true.  The stale-error quirk (after a rejected trial g2o restores the estimate but not the edges' error vectors, and the
classification reads them) matters only for the active edges of a round that ends on a rejected trial; pose_cases.stale_error_case() plants an edge
whose chi2 straddles the threshold between its stale and its fresh value.

The same edge's stale chi2 rounds to exactly 5.991f, so it also tells the chi-square test written `>=` from `>`, which differ for no other case:
no other final chi2 lands in that one-ulp window (4.8e-7 wide).  No mutant is declared a survivor today; the mechanism stays for one that must be."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import oracle as O
import pose_cases as PC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, 'oracle', '_ref', 'liboptimizer_ref.so')
SRC = os.path.join(ROOT, 'oracle', 'pose_opt.cpp')
CXXFLAGS = ['-O3', '-std=c++17', '-fPIC', '-shared', '-ffp-contract=off']          # oracle/Makefile's flags for liboracle.so
v = C.c_void_p

# (name, [(search, replace), ...], reason it survives or None)
MUTANTS = [
    ('huber_in_round_4', [('if (it == 2) e.robust = false;', 'if (it == 3) e.robust = false;')], None),
    ('stereo_invz_double', [('const float invz = 1.0f / p[2];', 'const double invz = 1.0 / p[2];')], None),
    ('lambda_tau_1e-4', [('lambda = 1e-5 * md;', 'lambda = 1e-4 * md;')], None),
    ('round_restarts_from_previous', [('P.est = se3_from_Rt(R0, t0);', 'if (it == 0) P.est = se3_from_Rt(R0, t0);')], None),
    ('nbad_factor_1e4', [('(iniChi - currentChi) * 1e3 < iniChi', '(iniChi - currentChi) * 1e4 < iniChi')], None),
    ('five_trials', [('while (rho < 0 && qmax < 10);', 'while (rho < 0 && qmax < 5);'), ('if (qmax == 10 ||', 'if (qmax == 5 ||')], None),
    ('single_round_below_9', [('if (P.edges.size() < 10) break;', 'if (P.edges.size() < 9) break;')], None),
    ('huber_delta_double', [('const float deltaMono = std::sqrt(5.991), deltaStereo', 'const double deltaMono = std::sqrt(5.991), deltaStereo')], None),
    ('classification_recomputes_errors', [('if (outlier[e.idx]) P.compute_error(e);', 'P.compute_error(e);')], None),
    ('chi2_test_ge', [('if (chi2 > (e.stereo ? chi2Stereo[it] : chi2Mono[it]))', 'if (chi2 >= (e.stereo ? chi2Stereo[it] : chi2Mono[it]))')], None),
]
TARGETS = {'five_trials': 'rejects', 'nbad_factor_1e4': 'nbad', 'single_round_below_9': 'nine', 'classification_recomputes_errors': 'stale',
           'chi2_test_ge': 'stale'}


def run_lib(L, s):
    """sgo_pose_optimization of library L on scenario s: (n_inliers, Tcw float32 [4][4], outlier flags)."""
    f32 = np.float32; c = s['cam']
    T = np.ascontiguousarray(s['T0'], f32).reshape(16)
    a = [np.ascontiguousarray(s['has'], np.uint8), np.ascontiguousarray(s['xyz'], f32), np.ascontiguousarray(s['xy'], f32), np.ascontiguousarray(s['octave'], np.int32),
         np.ascontiguousarray(s['uright'], f32), np.ascontiguousarray(s['inv_s2'], f32)]
    n = len(a[0]); out = np.zeros(16, f32); outl = np.zeros(n, np.uint8)
    r = L.sgo_pose_optimization(T.ctypes.data_as(v), n, *[x.ctypes.data_as(v) for x in a], C.c_float(c['fx']), C.c_float(c['fy']), C.c_float(c['cx']),
                                C.c_float(c['cy']), C.c_float(c['bf']), out.ctypes.data_as(v), outl.ctypes.data_as(v))
    return r, out.reshape(4, 4), outl


def differs(a, b):
    """Whether two results (n, T, flags) differ under the device test's bar: count or a flag, or a pose entry more than one float32 ulp apart."""
    return a[0] != b[0] or not np.array_equal(a[2], b[2]) or int(PC.ulp_distance(a[1], b[1]).max()) > 1


@pytest.mark.skipif(not os.path.exists(REF_LIB), reason='oracle/_ref/liboptimizer_ref.so not built (reference tree absent)')
def test_every_case_equals_the_reference():
    import test_optimizer_ref as R
    for fam, name, s in PC.all_cases():
        R._same(s, name)


def _build_mutant(src, pairs, path):
    for a, b in pairs:
        assert src.count(a) == 1, a                         # the substitution must keep hitting exactly one place in the restatement
        src = src.replace(a, b)
    cpp = path + '.cpp'
    with open(cpp, 'w') as f:
        f.write(src)
    subprocess.check_call(['g++', *CXXFLAGS, '-o', path, cpp])
    return C.CDLL(path)


@pytest.mark.skipif(shutil.which('g++') is None, reason='no g++ to build the mutants')
def test_every_mutant_is_caught(tmp_path):
    with open(SRC) as f:
        src = f.read()
    cases = PC.all_cases()
    base = [run_lib(O.lib(), s) for _, _, s in cases]
    unmodified = _build_mutant(src, [], str(tmp_path / 'unmodified.so'))
    for (_, name, s), b in zip(cases, base):               # the standalone build is the oracle
        assert not differs(run_lib(unmodified, s), b), name
    report = {}
    for mname, pairs, survivor in MUTANTS:
        L = _build_mutant(src, pairs, str(tmp_path / (mname + '.so')))
        caught = [(fam, name) for (fam, name, s), b in zip(cases, base) if differs(run_lib(L, s), b)]
        report[mname] = caught
        if survivor is None:
            assert caught, '%s: no case tells it from the restatement' % mname
            if mname in TARGETS:
                assert TARGETS[mname] in {f for f, _ in caught}, '%s: not caught by the %s cases built for it' % (mname, TARGETS[mname])
        else:
            assert not caught, '%s is caught by %s: it is no longer a survivor' % (mname, caught[:5])
    print({k: len(c) for k, c in report.items()})
