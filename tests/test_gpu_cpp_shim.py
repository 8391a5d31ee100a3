"""The reference-shaped C++ headers (include/sgslam/*.h: ORBextractor, ORBmatcher, RmDynamicPointsGeometry) compiled without
OpenCV and run on the GPU; the expected results are the CPU oracle's."""
import os
import subprocess

import numpy as np
import pytest

import oracle as O
import scenarios as S
from pysgs import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _build(out_dir):
    """Compiles tests/cpp/test_shim.cpp into out_dir (the source tree may be read-only)."""
    exe = os.path.join(out_dir, 'test_shim')
    src = os.path.join(ROOT, 'tests', 'cpp', 'test_shim.cpp')
    lib = os.path.join(ROOT, 'sg-slam_b200', 'lib')
    subprocess.check_call(['g++', '-O1', '-std=c++17', '-I', os.path.join(ROOT, 'include'), src, '-o', exe, '-L', lib, '-lsgs_cuda', '-Wl,-rpath,' + lib, '-ldl', '-lpthread', '-lrt'])
    return exe


def test_shim_compiles_without_gpu(tmp_path):
    _build(str(tmp_path))


@pytest.mark.gpu
def test_shim_on_gpu_built_in_tmp(tmp_path):
    exe = _build(str(tmp_path))
    img = synth.frame_s1(640, 480, 21)
    kps, desc = O.extract(img)
    s = S.random_lastframe_scenario(3, n_cur=900, n_last=1000)
    fo = O.FrameArrays(s['kps'], s['uright'], s['desc'], 640, 480, s['cam']['fx'], s['cam']['fy'], s['cam']['cx'], s['cam']['cy'], s['cam']['bf'], s['sf'])
    nm, mp, _ = O.search_by_projection_last(fo, s['Tcw_cur'], s['Tcw_last'], s['last_has'], s['last_xyz'], s['last_desc'], s['last_obs'], s['last_oct'], s['last_angle'], 15.0)
    d = S.dynreject_scenario(5, n=len(kps))
    dk = kps.copy(); dk['x'] = d['cur'][:, 0]; dk['y'] = d['cur'][:, 1]
    nkeep, keep, _, restored = O.dynreject(d['cur'], d['prev'], d['F'], d['boxes'], True, 1000)
    assert not restored
    path = tmp_path / 'scenario.bin'
    with open(path, 'wb') as f:
        np.array([640, 480, len(kps), len(s['kps']), len(s['last_has']), nm, nkeep, len(dk)], np.int32).tofile(f)
        img.tofile(f); kps.tofile(f); desc.tofile(f)
        s['kps'].tofile(f); s['uright'].astype(np.float32).tofile(f); s['desc'].tofile(f); s['sf'].astype(np.float32).tofile(f)
        s['Tcw_cur'].astype(np.float32).tofile(f); s['Tcw_last'].astype(np.float32).tofile(f)
        s['last_has'].astype(np.uint8).tofile(f); s['last_obs'].astype(np.uint8).tofile(f); s['last_xyz'].astype(np.float32).tofile(f)
        s['last_desc'].tofile(f); s['last_oct'].astype(np.int32).tofile(f); s['last_angle'].astype(np.float32).tofile(f); mp.astype(np.int32).tofile(f)
        dk.tofile(f); desc.tofile(f); d['prev'].astype(np.float32).tofile(f); d['F'].astype(np.float64).tofile(f)
        d['boxes'].astype(np.float32).tofile(f); keep.astype(np.uint8).tofile(f)
        # 4. LK + findFundamentalMat shims: a second frame of the stream, the oracle's tracks and its F on them
        frames, _ = synth.stream_s2(2, 640, 480, seed=9)
        k2, _ = O.extract(frames[1])
        pts = np.stack([k2['x'], k2['y']], 1).astype(np.float32)
        trk = O.lk_track(frames[1], frames[0], pts)
        Fo, _, _ = O.find_fundamental_ransac(pts, trk)
        assert Fo is not None
        np.array([len(pts)], np.int32).tofile(f); frames[1].tofile(f); frames[0].tofile(f); pts.tofile(f); trk.astype(np.float32).tofile(f)
        Fo.astype(np.float64).tofile(f)
        # 5. isInFrustum: points in front of a posed camera; distances chosen so that x/0.8*0.8 and x/1.2*1.2 round-trips cannot flip a gate
        rs = np.random.RandomState(8)
        nfr = 2000
        T = np.eye(4, dtype=np.float32); a = 0.2
        T[:3, :3] = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]], np.float32); T[:3, 3] = [0.2, -0.1, 0.3]
        z = rs.uniform(-1, 8, nfr); pc = np.c_[rs.uniform(-0.8, 0.8, nfr) * z, rs.uniform(-0.6, 0.6, nfr) * z, z]
        xyz = ((pc - T[:3, 3].astype(np.float64)) @ T[:3, :3].astype(np.float64)).astype(np.float32)
        cen = -T[:3, :3].T.astype(np.float64) @ T[:3, 3].astype(np.float64)
        tc = xyz.astype(np.float64) - cen; d0 = np.linalg.norm(tc, axis=1)
        nn = tc / d0[:, None] + rs.normal(0, 0.4, (nfr, 3)); nrm = (nn / np.linalg.norm(nn, axis=1, keepdims=True)).astype(np.float32)
        mx = (d0 * rs.choice([0.5, 1.7, 3.1], nfr)).astype(np.float32); mn = (mx / 5).astype(np.float32)
        mn = (np.float32(0.8) * mn / np.float32(0.8)).astype(np.float32); mx = (np.float32(1.2) * mx / np.float32(1.2)).astype(np.float32)   # fixed points of the round trip
        cam9 = np.array([535.4, 539.2, 320.1, 247.6, 40.0, 0, 0, 640, 480], np.float32)
        ref = O.is_in_frustum(T, cam9, 8, float(O.logf(1.2)), xyz, nrm, mn, mx, 0.5)
        np.array([nfr], np.int32).tofile(f); T.tofile(f); xyz.tofile(f); nrm.tofile(f); mn.tofile(f); mx.tofile(f)
        ref['inview'].tofile(f); ref['proj_x'].tofile(f); ref['proj_y'].tofile(f); ref['proj_xr'].tofile(f); ref['view_cos'].tofile(f); ref['level'].tofile(f)
        # 6. PoseOptimization
        ps = S.pose_scenario(12, n=700)
        pc = ps['cam']
        pn, pT, po = O.pose_optimization(ps['T0'], ps['has'], ps['xyz'], ps['xy'], ps['octave'], ps['uright'], ps['inv_s2'], pc['fx'], pc['fy'], pc['cx'], pc['cy'], pc['bf'])
        pk = np.zeros(700, O.KP_DTYPE); pk['x'] = ps['xy'][:, 0]; pk['y'] = ps['xy'][:, 1]; pk['octave'] = ps['octave']
        np.array([700], np.int32).tofile(f); ps['T0'].astype(np.float32).tofile(f); ps['xyz'].astype(np.float32).tofile(f); pk.tofile(f)
        ps['uright'].astype(np.float32).tofile(f); ps['inv_s2'][:8].astype(np.float32).tofile(f); ps['has'].astype(np.uint8).tofile(f); po.astype(np.uint8).tofile(f)
        pT.astype(np.float32).tofile(f); np.array([pn], np.int32).tofile(f)
        # 7. Detector2D::detect on the synthetic SSD graph of tests/detector_model.py
        import detector_model as DM
        import detector_oracle as DO
        import ncnn_model as NM
        dpp, dbp = DM.write_mini_model(str(tmp_path / 'model'), 0)
        layers = NM.parse_param(dpp); NM.load_weights(layers, dbp)
        rgb = DM.synthetic_rgb(480, 640, 1)
        _, (objs, _, _) = DO.detect(layers, rgb, 0.9, 0.01)
        np.array([640, 480, len(objs)], np.int32).tofile(f); rgb.tofile(f); objs[:, 0].astype(np.int32).tofile(f); objs[:, 1:].astype(np.float32).tofile(f)
        # 8./9. SearchByProjection(KeyFrame*, Scw, ...) and Fuse(KeyFrame*, vpMapPoints, th) through the class mirror: one key frame, one candidate list
        from test_match_sim3 import sim3_inputs
        ks, kOw, knrm, kmatched = sim3_inputs(31, 700, 1200)
        f32 = np.float32
        # the mirror recovers mfMin/MaxDistance from the *Invariance getters: use values that survive the 0.8 / 1.2 round trip
        kmin = ((f32(0.8) * ks['min_dist'].astype(f32)) / f32(0.8)).astype(f32); kmax = ((f32(1.2) * ks['max_dist'].astype(f32)) / f32(1.2)).astype(f32)
        kmin = ((f32(0.8) * kmin) / f32(0.8)).astype(f32); kmax = ((f32(1.2) * kmax) / f32(1.2)).astype(f32)
        kc = ks['cam']; sf8 = ks['sf'].astype(f32); inv8 = (1.0 / (sf8 * sf8)).astype(f32)
        kfo = O.FrameArrays(ks['kps'], ks['uright'], ks['desc'], 640, 480, kc['fx'], kc['fy'], kc['cx'], kc['cy'], kc['bf'], ks['sf'])
        nm3, m3 = O.search_by_projection_sim3(kfo, ks['Tcw_cur'], kOw, ks['kf_valid'], ks['last_xyz'], knrm, kmin, kmax, ks['last_desc'], 10.0, kmatched)
        assert nm3 > 30
        nk_, nmp_ = len(ks['kps']), len(ks['last_xyz'])
        rs9 = np.random.RandomState(99)
        kf_has = np.where(rs9.rand(nk_) < 0.3, rs9.randint(1, 6, nk_), -1).astype(np.int32)      # Observations() of the point the key frame already holds there
        pobs = rs9.randint(1, 6, nmp_).astype(np.int32); pinkf = (rs9.rand(nmp_) < 0.1).astype(np.uint8)
        fth = 3.0
        valid9 = (ks['kf_valid'].astype(bool) & ~pinkf.astype(bool)).astype(np.uint8)
        bi9, bd9 = O.fuse_search(kfo, ks['Tcw_cur'], kOw, valid9, ks['last_xyz'], knrm, kmin, kmax, ks['last_desc'], fth, inv8)
        # the reference's side-effect loop (src/ORBmatcher.cc:962-977) on the mock objects of test_shim.cpp
        kf_final = np.where(kf_has >= 0, -2, -1).astype(np.int32); ebad = np.zeros(nk_, np.uint8); pbad = (1 - ks['kf_valid']).astype(np.uint8); inkf = pinkf.copy(); nfused = 0
        pobs_run = pobs.copy()
        for i in range(nmp_):
            if pbad[i] or inkf[i] or bd9[i] > 50:
                continue
            j = bi9[i]
            if kf_final[j] != -1:                       # a point is already there (an original one, or a candidate added earlier in this call)
                holder_bad = ebad[j] if kf_final[j] == -2 else pbad[kf_final[j]]
                holder_obs = kf_has[j] if kf_final[j] == -2 else pobs_run[kf_final[j]]
                if not holder_bad:
                    if holder_obs > pobs_run[i]:
                        pbad[i] = 1
                    elif kf_final[j] == -2:
                        ebad[j] = 1
                    else:
                        pbad[kf_final[j]] = 1
            else:
                kf_final[j] = i; inkf[i] = 1; pobs_run[i] += 1
            nfused += 1
        assert nfused > 20 and ebad.sum() > 0
        np.array([nk_, nmp_, 10], np.int32).tofile(f); ks['kps'].tofile(f); ks['uright'].astype(f32).tofile(f); ks['desc'].tofile(f); sf8.tofile(f); inv8.tofile(f)
        np.array([kc['fx'], kc['fy'], kc['cx'], kc['cy'], kc['bf']], f32).tofile(f); ks['Tcw_cur'].astype(f32).tofile(f); kOw.astype(f32).tofile(f)
        ks['kf_valid'].astype(np.uint8).tofile(f); ks['last_xyz'].astype(f32).tofile(f); knrm.astype(f32).tofile(f); kmin.tofile(f); kmax.tofile(f); ks['last_desc'].tofile(f)
        kmatched.astype(np.int32).tofile(f); m3.astype(np.int32).tofile(f); np.array([nm3], np.int32).tofile(f)
        kf_has.tofile(f); pobs.tofile(f); pinkf.tofile(f); np.array([fth], f32).tofile(f); np.array([nfused], np.int32).tofile(f)
        kf_final.tofile(f); pbad.astype(np.uint8).tofile(f); ebad.tofile(f)
        # 10. SearchBySim3: both key frames share the features and the pose; each holds some of the candidate points at the features they resemble
        bi0, bd0 = O.fuse_search(kfo, ks['Tcw_cur'], kOw, np.ones(nmp_, np.uint8), ks['last_xyz'], knrm, kmin, kmax, ks['last_desc'], 3.0, inv8, sim3_variant=1)
        mp1 = np.full(nk_, -1, np.int32); mp2 = np.full(nk_, -1, np.int32)
        for i in np.argsort(bd0, kind='stable'):
            j = bi0[i]
            if j < 0 or bd0[i] > 70:
                continue
            if mp1[j] < 0 and rs9.rand() < 0.6:
                mp1[j] = i
            elif mp2[j] < 0:
                mp2[j] = i
        both = np.nonzero((mp1 >= 0) & (mp2 >= 0))[0]
        assert len(both) > 15
        pre = np.full(nk_, -1, np.int32); pre[both[:4]] = mp2[both[:4]]                       # vpMatches12 entries that are already set
        s12 = f32(1.02); a12 = 0.003
        R12 = np.array([[np.cos(a12), -np.sin(a12), 0], [np.sin(a12), np.cos(a12), 0], [0, 0, 1]], f32); t12 = np.array([0.01, -0.005, 0.008], f32)
        inv12 = f32(1.0 / np.float64(s12))
        sR12 = (R12 * s12).astype(f32); sR21 = (R12.T * inv12).astype(f32)
        t21 = np.array([-f32(f32(f32(sR21[r, 0] * t12[0]) + f32(sR21[r, 1] * t12[1])) + f32(sR21[r, 2] * t12[2])) for r in range(3)], f32)
        x21 = np.concatenate([sR21.reshape(9), t21]).astype(f32); x12 = np.concatenate([sR12.reshape(9), t12]).astype(f32)
        already1 = pre >= 0
        already2 = np.zeros(nk_, bool)
        for j in np.nonzero(already1)[0]:
            already2[np.nonzero(mp2 == pre[j])[0]] = True                                       # GetIndexInKeyFrame(pKF2)
        ok_pt = ks['kf_valid'].astype(bool)

        def direction(mp, already, xf):
            has = (mp >= 0) & ~already
            has &= np.where(mp >= 0, ok_pt[np.maximum(mp, 0)], False)
            g = np.maximum(mp, 0)
            bi_, bd_ = O.fuse_search(kfo, ks['Tcw_cur'], np.zeros(3, f32), has.astype(np.uint8), ks['last_xyz'][g], knrm[g], kmin[g], kmax[g], ks['last_desc'][g], 7.5, inv8,
                                     sim3_variant=2, xform2=xf)
            return np.where(bd_ <= 100, bi_, -1)
        vn1 = direction(mp1, already1, x21); vn2 = direction(mp2, already2, x12)
        exp12 = pre.copy(); nfound = 0
        for i1 in range(nk_):
            if vn1[i1] >= 0 and vn2[vn1[i1]] == i1:
                exp12[i1] = mp2[vn1[i1]]; nfound += 1
        assert nfound > 5
        np.array([nmp_, 0], np.int32).tofile(f); np.array([s12, 7.5], f32).tofile(f); R12.tofile(f); t12.tofile(f); mp1.tofile(f); mp2.tofile(f); pre.tofile(f); exp12.tofile(f)
        np.array([nfound], np.int32).tofile(f)
        # 11./12. SearchByBoW(KF, KF) and SearchForTriangulation through the class mirror (flattened FeatureVectors from the oracle's vocabulary transform)
        voc = S.random_vocabulary(17, k=10, L=3)
        V = O.Vocabulary(voc['k'], voc['L'], voc['parent'], voc['desc'], voc['weight'])
        n1_, n2_ = 900, 950
        bs = S.bow_pair_scenario(77, voc, n_kf=n1_, n_f=n2_, flips=30)
        rsb = np.random.RandomState(78)
        xy1 = np.c_[rsb.uniform(20, 620, n1_), rsb.uniform(20, 460, n1_)].astype(f32)
        d1b = np.unpackbits(bs['kf_desc'], axis=1).astype(np.int16); d2b = np.unpackbits(bs['f_desc'], axis=1).astype(np.int16)
        src_ = np.array([int(np.argmin(np.abs(d1b - d2b[j]).sum(1))) for j in range(n2_)])
        xy2 = np.c_[xy1[src_, 0] + rsb.uniform(-40, 40, n2_), xy1[src_, 1] + rsb.normal(0, 1.5, n2_)].astype(f32)
        oct2 = rsb.randint(0, 8, n2_).astype(np.int32)
        st = [rsb.choice([0, 1, 2], n1_, p=[0.5, 0.42, 0.08]).astype(np.uint8), rsb.choice([0, 1, 2], n2_, p=[0.5, 0.42, 0.08]).astype(np.uint8)]   # 0 no point, 1 point, 2 bad point
        ur = [np.where(rsb.rand(n1_) < 0.5, 100.0, -1.0).astype(f32), np.where(rsb.rand(n2_) < 0.5, 100.0, -1.0).astype(f32)]
        _, ow1, on1 = V.transform(bs['kf_desc'], 1); _, ow2, on2 = V.transform(bs['f_desc'], 1)
        F12 = np.array([[0, 0, 0], [0, 0, -1], [0, 1, 0]], f32)
        R2 = S.pose(0.01, -0.02, 0.015, (0, 0, 0))[:3, :3].astype(f32); t2 = np.array([0.3, -0.1, 0.2], f32); Cw = np.array([0.5, 0.2, -1.5], f32)
        camv = np.array([535.4, 539.2, 320.1, 247.6], f32)
        C2 = [f32(np.float64(f32(f32(f32(R2[r, 0] * Cw[0]) + f32(R2[r, 1] * Cw[1])) + f32(R2[r, 2] * Cw[2]))) + np.float64(t2[r])) for r in range(3)]
        invz2 = f32(1.0) / C2[2]
        ex = f32(f32(f32(camv[0] * C2[0]) * invz2) + camv[2]); ey = f32(f32(f32(camv[1] * C2[1]) * invz2) + camv[3])
        sig8 = (sf8 * sf8).astype(f32)
        nm11, m11 = O.search_by_bow_kfkf(on1, ow1, (st[0] == 1), bs['kf_desc'], bs['kf_angle'], on2, ow2, (st[1] == 1), bs['f_desc'], bs['f_angle'], nnratio=0.8, check_ori=True)
        k1 = dict(node=on1, weight=ow1, free=(st[0] == 0), stereo=(ur[0] >= 0), desc=bs['kf_desc'], xy=xy1, angle=bs['kf_angle'])
        k2 = dict(node=on2, weight=ow2, free=(st[1] == 0), stereo=(ur[1] >= 0), desc=bs['f_desc'], xy=xy2, octave=oct2, angle=bs['f_angle'])
        nm12, m12 = O.search_for_triangulation(k1, k2, F12, float(ex), float(ey), sig8, sf8, False, True)
        assert nm11 > 20 and nm12 > 20
        np.array([n1_, n2_, 0], np.int32).tofile(f)
        for q, (dsc, ang, xy, octv, onode, oweight) in enumerate([(bs['kf_desc'], bs['kf_angle'], xy1, np.zeros(n1_, np.int32), on1, ow1), (bs['f_desc'], bs['f_angle'], xy2, oct2, on2, ow2)]):
            kk = np.zeros(len(dsc), O.KP_DTYPE); kk['x'] = xy[:, 0]; kk['y'] = xy[:, 1]; kk['angle'] = ang; kk['octave'] = octv
            kk.tofile(f); ur[q].tofile(f); dsc.tofile(f); np.asarray(onode, np.int32).tofile(f); (np.asarray(oweight) > 0).astype(np.uint8).tofile(f); st[q].tofile(f)
        R2.tofile(f); t2.tofile(f); Cw.tofile(f); camv.tofile(f); F12.tofile(f); sig8.tofile(f); sf8.tofile(f)
        np.array([nm11], np.int32).tofile(f); m11.astype(np.int32).tofile(f); np.array([nm12], np.int32).tofile(f); m12.astype(np.int32).tofile(f)
        # 13. SearchForInitialization through the class mirror
        from test_match_init import init_scenario
        isc = init_scenario(5)
        inm, im12, iprev = O.search_for_initialization(isc['f1'], isc['f2'], isc['prev'], 100, 0.9, True)
        assert inm > 40
        np.array([len(isc['k1']), len(isc['k2']), 100], np.int32).tofile(f); isc['k1'].tofile(f); isc['d1'].tofile(f); isc['k2'].tofile(f); isc['d2'].tofile(f)
        isc['prev'].astype(f32).tofile(f); iprev.astype(f32).tofile(f); np.array([inm], np.int32).tofile(f); im12.astype(np.int32).tofile(f)
    out = subprocess.run([exe, str(path), dpp, dbp], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr
    assert 'OK shim' in out.stdout
