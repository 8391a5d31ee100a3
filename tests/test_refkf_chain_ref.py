"""The reference-key-frame chain -- what sgs_tracker_refkf_chain_device computes: Tracking::TrackReferenceKeyFrame (ComputeBoW, SearchByBoW with 0.7 and the
orientation check, the 15-match gate, PoseOptimization from the last frame's pose, the outlier discard) and TrackLocalMap after it -- pinned against the
REFERENCE'S OWN tracking code (ref_track_refkf_and_local_map of tests/cpp/refkf_ref_driver.cpp, compiled here as oracle/Makefile builds
oracle/_ref/libtracking_ref.so: src/Tracking.cc, ORBmatcher.cc, Optimizer.cc + vendored g2o unmodified).  The checker of the GPU chain, the composition of oracle functions in tests/refkf_cases.py (oracle_refkf), runs here on CPU-extracted
frames and must give the reference's BoW nmatches, the map point per keypoint after each half, the outlier flags, nmatchesMap's verdict, mnMatchesInliers,
both return values and both poses.  One frame runs TrackWithMotionModel first and fails it: the outliers its discard drops lie in the local map, and the
composition must leave them out of the local search exactly as the reference does (its seen_in).  No device needed."""
import ctypes as C
import glob
import os
import subprocess

import numpy as np
import pytest

import oracle as O
import refkf_cases as R
from pysgs import binding as B
from pysgs import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = '/root/reference/src/sg-slam'
G2O_OBJ = sorted(glob.glob(os.path.join(ROOT, 'oracle', '_ref', 'g2o_obj', '**', '*.o'), recursive=True))
pytestmark = pytest.mark.skipif(not (os.path.exists(os.path.join(REF, 'src', 'Tracking.cc')) and os.path.exists(os.path.join(ROOT, 'oracle', '_ref', 'libtracking_ref.so'))
                                     and G2O_OBJ), reason='reference tree / the tracking oracle absent')
W, H, TH = 640, 480, 15.0
v = C.c_void_p
RELOC, FEW, MOTION = 3, 2, 4          # frame 3 follows a relocalisation (th 5); frame 2's key frame has 12 features; frame 4 fails the motion model first


def _p(a):
    return a.ctypes.data_as(v)


@pytest.fixture(scope='module')
def reflib(tmp_path_factory):
    """tests/cpp/refkf_ref_driver.cpp built with the recipe of oracle/_ref/libtracking_ref.so (oracle/Makefile)"""
    out = str(tmp_path_factory.mktemp('refkf') / 'librefkf_ref.so')
    o = os.path.join(ROOT, 'oracle'); src = os.path.join(REF, 'src'); dbow = os.path.join(REF, 'Thirdparty', 'DBoW2', 'DBoW2')
    cmd = ['g++', '-O3', '-std=c++11', '-fPIC', '-shared', '-fvisibility=hidden', '-w', '-ffp-contract=off'] + \
          ['-I' + os.path.join(o, d) for d in ('', 'tracking_shim', 'g2o_shim', 'frame_shim', 'orbmatcher_shim')] + \
          ['-I' + REF, '-I' + os.path.join(REF, 'include'), '-I' + os.path.join(REF, 'Thirdparty', 'g2o'), '-include', os.path.join(o, 'tracking_shim', 'tracking_standins.h'),
           '-o', out, os.path.join(ROOT, 'tests', 'cpp', 'refkf_ref_driver.cpp')] + \
          [os.path.join(src, f) for f in ('Tracking.cc', 'Frame.cc', 'MapPoint.cc', 'ORBmatcher.cc', 'Optimizer.cc', 'Converter.cc', 'ORBextractor.cc')] + \
          [os.path.join(dbow, 'BowVector.cpp'), os.path.join(dbow, 'FeatureVector.cpp')] + G2O_OBJ + \
          ['-L' + o, '-l:liboracle.so', '-Wl,-rpath,' + o, '-l:libstdc++.so.6', '-pthread']
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    return out


def reference(lib, camv, sf, isig, cur, fnode, kf, knode, with_motion, ti, f, lm, pc, reloc):
    L = C.CDLL(lib)
    a = lambda x, dt: np.ascontiguousarray(x, dt)
    n, kn, m, nl = cur.c.N, int(kf['n']), int(ti['ln'][f]), lm['n']
    xy = a(np.stack([cur.keysUn['x'], cur.keysUn['y']], 1), np.float32)
    out = dict(okm=C.c_int32(), nm=C.c_int32(), okr=C.c_int32(), T1=np.zeros(16, np.float32), mp1=np.zeros(n, np.int32), okl=C.c_int32(),
               T2=np.zeros(16, np.float32), mp2=np.full(n, -1, np.int32), outl=np.zeros(n, np.uint8), inl=C.c_int32())
    keep = [a(cur.keysUn['octave'], np.int32), a(cur.keysUn['angle'], np.float32), a(fnode, np.int32),
            a(kf['xyz'][:kn], np.float32), a(kf['desc'][:kn], np.uint8), a(kf['flags'][:kn], np.uint8), a(kf['angle'][:kn], np.float32), a(knode, np.int32),
            a(kf['lid'][:max(kn, 1)], np.int32),
            a(ti['lxyz'][f, :m], np.float32), a(ti['ldesc'][f, :m], np.uint8), a(ti['lflags'][f, :m], np.uint8), a(ti['loct'][f, :m], np.int32),
            a(ti['lang'][f, :m], np.float32), a(lm['lid'][:max(m, 1)], np.int32), a(ti['Tc'][f], np.float32), a(ti['T'][f], np.float32)]
    lmk = [a(lm[k][:nl], dt) for k, dt in (('xyz', np.float32), ('nrm', np.float32), ('mn', np.float32), ('mx', np.float32), ('dsc', np.uint8), ('valid', np.uint8),
                                           ('obs', np.uint8))]
    L.ref_track_refkf_and_local_map(_p(camv), _p(a(sf, np.float32)), _p(isig), 8, n, _p(xy), _p(keep[0]), _p(keep[1]), _p(cur.uRight), _p(cur.desc), _p(keep[2]),
                                    kn, *[_p(x) for x in keep[3:9]], int(with_motion), m, *[_p(x) for x in keep[9:17]], int(reloc),
                                    nl, *[_p(x) for x in lmk], pc, C.byref(out['okm']), C.byref(out['nm']), C.byref(out['okr']), _p(out['T1']), _p(out['mp1']),
                                    C.byref(out['okl']), _p(out['T2']), _p(out['mp2']), _p(out['outl']), C.byref(out['inl']))
    return out


@pytest.mark.parametrize('k,L', [(3, 5), (10, 3)])
def test_refkf_composition_equals_the_reference_tracking_code(reflib, k, L):
    import bench
    nb = 6
    frames, boxes, unique = bench.make_frames(nb, 17, W, H, unique=nb)
    pidx = bench.prev_index(nb, unique)
    camd = dict(synth.TUM3)
    sf = synth.scale_factors(); cam = B.make_camera(W, H, camd, sf)
    NF = 1000; pc = NF + 64; cap = NF + 8 * 8 + 64; mcap = 1536
    kps = np.zeros((nb, cap), O.KP_DTYPE); desc = np.zeros((nb, cap, 32), np.uint8); cnt = np.zeros(nb, np.int32)
    for f in range(nb):
        kk, d = O.extract(frames[f])[:2]
        cnt[f] = len(kk); kps[f, :len(kk)] = kk; desc[f, :len(kk)] = d
    ti = bench.make_track_inputs(kps, desc, cnt, boxes, cap, pc, pidx, W, H, camd)
    ti['Tc'] = ti['T'].copy()
    ti['lflags'][:, 11::19] |= 4                                        # bad points (of the key frame, and of the last frame where it runs)
    ti['lflags'][MOTION] &= ~np.uint8(2)                                # no observations: the motion model fails on nmatchesMap, and so does the key frame
    # trap points of the motion-model frame: local-map points with octave <= 2 moved 6 px sideways, held by the last frame but not the key frame
    m4 = int(ti['ln'][MOTION])
    trap = np.nonzero((np.arange(m4) % 2 == 0) & (ti['loct'][MOTION, :m4] <= 2))[0][3::25]
    ti['lxyz'][MOTION, trap, 0] += 6.0 * ti['lxyz'][MOTION, trap, 2] / camd['fx']
    isig = np.zeros(16, np.float32); isig[:8] = 1.0 / (sf.astype(np.float32) ** 2)
    camv = np.array([camd['fx'], camd['fy'], camd['cx'], camd['cy'], camd['bf'], cam.min_x, cam.min_y, cam.max_x, cam.max_y], np.float32)
    voc = R.train_vocabulary(np.concatenate([desc[f, :cnt[f]] for f in range(nb)]), k, L, seed=k)
    V = O.Vocabulary(voc['k'], voc['L'], voc['parent'], voc['desc'], voc['weight'])
    rng = np.random.default_rng(k)
    seen = dict(gated=0, nomap=0, full=0, reloc=0, trap=0)
    for f in range(nb):
        n = int(cnt[f]); m = int(ti['ln'][f])
        cur = O.FrameArrays(kps[f, :n], ti['ur'][f, :n], desc[f, :n], W, H, camd['fx'], camd['fy'], camd['cx'], camd['cy'], camd['bf'], sf)
        lm = bench.make_local_map(f, kps[f], desc[f], n, ti, mcap, camd, sf, rng, W, H)
        for j in np.nonzero(lm['lid'][:m] >= 0)[0]:                   # one object per point: a linked local-map point carries the point's flags and position
            l = lm['lid'][j]
            lm['xyz'][l] = ti['lxyz'][f, j]; lm['obs'][l] = (ti['lflags'][f, j] >> 1) & 1; lm['valid'][l] = 0 if ti['lflags'][f, j] & 4 else 1
        kf = dict(desc=ti['ldesc'][f], angle=ti['lang'][f], xyz=ti['lxyz'][f], flags=ti['lflags'][f].copy(), lid=lm['lid'], n=12 if f == FEW else m)
        if f == MOTION:
            kf['flags'][trap] = 0
        kw_, fw_ = V.transform(kf['desc'][:kf['n']], 4), V.transform(cur.desc, 4)
        knode = np.where(kw_[1] > 0, kw_[2], -1); fnode = np.where(fw_[1] > 0, fw_[2], -1)        # the FeatureVector lists features of positive weight
        seen_in = None
        if f == MOTION:
            fl = ti['lflags'][f, :m]
            nm0, mp0, _ = O.search_by_projection_last(cur, ti['Tc'][f].reshape(4, 4), ti['T'][f].reshape(4, 4), fl & 1, ti['lxyz'][f, :m], ti['ldesc'][f, :m],
                                                      (fl >> 1) & 1, ti['loct'][f, :m], ti['lang'][f, :m], TH)
            seen_in = R.motion_discards(cur, mp0.copy(), int(nm0), ti, f, lm, camd, isig, TH)
            assert seen_in.sum() >= 1
        th_local = 5.0 if f == RELOC else 3.0
        r = R.oracle_refkf(cur, V, kf, ti['T'][f].reshape(4, 4), lm, seen_in, camd, camv, sf, isig, th_local, pc)
        g = reference(reflib, camv, sf, isig, cur, fnode, kf, knode, f == MOTION, ti, f, lm, pc, f == RELOC)
        st = r['stats']
        assert g['nm'].value == st[0], (f, g['nm'].value, st)
        if f == MOTION:
            assert g['okm'].value == 0
        if st[0] < 15:
            assert f == FEW and g['okr'].value == 0
            seen['gated'] += 1
            continue
        assert np.array_equal(g['mp1'], r['mp1']), (f, int((g['mp1'] != r['mp1']).sum()))
        assert g['okr'].value == int(st[4] >= 10), (f, st)
        assert np.abs(g['T1'].reshape(4, 4) - r['T1']).max() <= 1e-6, f
        assert np.array_equal(g['mp2'], r['mp']), (f, int((g['mp2'] != r['mp']).sum()))
        assert np.array_equal(g['outl'], r['outlier']), f
        assert g['inl'].value == st[7], (f, g['inl'].value, st)
        assert g['okl'].value == int(st[7] >= (50 if f == RELOC else 30)), (f, st)      # src/Tracking.cc:1003-1010
        assert np.abs(g['T2'].reshape(4, 4) - r['T2']).max() <= 1e-6, f
        seen['full'] += 1; seen['nomap'] += int(st[4] < 10); seen['reloc'] += int(f == RELOC)
        if f == MOTION:       # without the motion model's discards the local search would have matched some of them
            r0 = R.oracle_refkf(cur, V, kf, ti['T'][f].reshape(4, 4), lm, None, camd, camv, sf, isig, th_local, pc)
            seen['trap'] = int(np.sum((r0['mp'] >= pc) & (seen_in[np.maximum(r0['mp'] - pc, 0)] != 0)))
    assert seen['gated'] == 1 and seen['nomap'] >= 1 and seen['full'] == nb - 1 and seen['reloc'] == 1 and seen['trap'] >= 1, seen
