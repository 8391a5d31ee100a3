"""sgs_tracker_pose_chain_device: the rest of Tracking::TrackWithMotionModel (src/Tracking.cc:926-967: wide-window retry, PoseOptimization, discarding the
outliers) and Tracking::TrackLocalMap (:969-1000 with SearchLocalPoints :1262-1312: seen / bad points left out, isInFrustum + PredictScale,
SearchByProjection(F, local points, th), PoseOptimization, mnMatchesInliers) in one device call after sgs_tracker_track_lk, against the same chain composed
from the CPU oracle's functions.  Indices, flags and counters are compared exactly -- the oracle's second half runs from the GPU's first pose, so that a
1e-7 difference of the optimiser cannot move a projection across a grid cell -- and the poses within the optimiser's tolerance (1e-5, tests/test_gpu_pose_opt.py)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle as O  # noqa: E402
from pysgs import binding as B  # noqa: E402
from pysgs import synth  # noqa: E402

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

W, H, NF, TH = 640, 480, 1000, 15.0


def oracle_chain(f, cur, nm0, mp0, ti, lm, cam, camd, sf, isig, th, tcw_motion_gpu=None):
    """Returns a dict with the chain's outputs for frame f, composed from the oracle's functions."""
    pc = ti['lxyz'].shape[1]
    m = int(ti['ln'][f]); fl = ti['lflags'][f, :m]
    Tc = ti['Tc'][f].reshape(4, 4); Tl = ti['T'][f].reshape(4, 4)
    st = np.zeros(8, np.int64)
    st[0] = nm0; mp = mp0.copy(); nm = nm0
    if nm < 20:
        st[1] = 1
        nm, mp, _ = O.search_by_projection_last(cur, Tc, Tl, fl & 1, ti['lxyz'][f, :m], ti['ldesc'][f, :m], (fl >> 1) & 1, ti['loct'][f, :m], ti['lang'][f, :m], 2 * th)
    st[2] = nm
    N = cur.c.N
    has = (mp >= 0).astype(np.uint8)
    xyz = np.zeros((N, 3), np.float32); xyz[mp >= 0] = ti['lxyz'][f, mp[mp >= 0]]
    kxy = np.stack([cur.keysUn['x'], cur.keysUn['y']], 1)
    _, T1, out1 = O.pose_optimization(Tc, has, xyz, kxy, cur.keysUn['octave'], cur.uRight, isig, camd['fx'], camd['fy'], camd['cx'], camd['cy'], camd['bf'])
    seen = np.zeros(len(lm['valid']), np.uint8)
    obs = np.zeros(N, np.uint8)
    nmatches = nm; nmap = 0
    for i in range(N):
        if mp[i] >= 0:
            lid = lm['lid'][mp[i]]
            if lid >= 0: seen[lid] = 1
            if out1[i]:
                mp[i] = -1; nmatches -= 1
            else:
                if fl[mp[i]] & 2: nmap += 1
                if fl[mp[i]] & 4: mp[i] = -1
                else: obs[i] = (fl[mp[i]] >> 1) & 1
    st[3] = nmatches; st[4] = nmap
    T1u = T1 if tcw_motion_gpu is None else tcw_motion_gpu.reshape(4, 4)
    n = lm['n']
    fr = O.is_in_frustum(T1u, cam, 8, float(O.logf(sf[1])), lm['xyz'][:n], lm['nrm'][:n], lm['mn'][:n], lm['mx'][:n], 0.5)
    inview = fr['inview'] & lm['valid'][:n] & (1 - seen[:n])
    st[5] = int(inview.sum())
    nml, mp2, obs2, _ = O.search_by_projection_local(cur, inview, fr['proj_x'], fr['proj_y'], fr['proj_xr'], fr['level'], fr['view_cos'], lm['dsc'][:n], lm['obs'][:n], 3.0, 0.8,
                                                     mp, obs, id_base=pc)
    st[6] = nml
    has2 = (mp2 >= 0).astype(np.uint8)
    xyz2 = np.zeros((N, 3), np.float32)
    a = (mp2 >= 0) & (mp2 < pc); b = mp2 >= pc
    xyz2[a] = ti['lxyz'][f, mp2[a]]; xyz2[b] = lm['xyz'][mp2[b] - pc]
    _, T2, out2 = O.pose_optimization(T1u, has2, xyz2, kxy, cur.keysUn['octave'], cur.uRight, isig, camd['fx'], camd['fy'], camd['cx'], camd['cy'], camd['bf'])
    out2 = out2 & has2
    st[7] = int(((mp2 >= 0) & (out2 == 0) & (obs2 != 0)).sum())
    return dict(T1=T1, T2=T2, mp=mp2, outlier=out2, stats=st)


def test_pose_chain_against_the_oracle_functions():
    import bench
    import torch
    nb, unique = 12, 6
    frames, boxes, unique = bench.make_frames(nb, 11, W, H, unique=unique)
    pidx = bench.prev_index(nb, unique)
    camd = dict(synth.TUM3)
    sf = synth.scale_factors(); cam = B.make_camera(W, H, camd, sf)
    mcap = 1536
    trk = B.Tracker(W, H, cam, NF, 1.2, 8, 20, 7, max_batch=nb, point_cap=NF + 64, max_boxes=4, device=0)
    cap, pcap = trk.cap, trk.point_cap
    L, v = B.lib(), C.c_void_p
    P = lambda a: a.ctypes.data_as(v)
    kps = np.zeros((nb, cap), B.KP_DTYPE); desc = np.zeros((nb, cap, 32), np.uint8); n = np.zeros(nb, np.int32)
    B.check(L.sgs_tracker_extract(trk.h, P(frames), nb, W * H, W, P(kps), P(desc), cap, P(n)))
    ti = bench.make_track_inputs(kps, desc, n, boxes, cap, pcap, pidx, W, H, camd)
    ti['lflags'][:, 9::23] |= 4                                         # some last-frame points are bad
    # poses: identity for most frames; two frames start with a yaw / pitch error of ~60 px (beyond every window at th = 15: 15 * 1.2^7 = 53.7 px, inside the
    # windows of the coarse octaves at 2 th); one frame has no last-frame points at all
    Tc = ti['T'].copy()
    def rot(axis, ang):
        c, s_ = np.cos(ang), np.sin(ang)
        R = np.eye(4, dtype=np.float32)
        if axis == 'y': R[0, 0] = c; R[0, 2] = s_; R[2, 0] = -s_; R[2, 2] = c
        else: R[1, 1] = c; R[1, 2] = -s_; R[2, 1] = s_; R[2, 2] = c
        return R.reshape(16)
    Tc[3] = rot('y', 60.0 / camd['fx']); Tc[7] = rot('x', -58.0 / camd['fy'])
    ti['ln'][5] = 0
    ti['ln'][3] = 300; ti['ln'][7] = 300          # few enough last-frame points that the chance matches at th = 15 stay below 20
    ti['Tc'] = Tc
    o = dict(kps=np.zeros((nb, cap), B.KP_DTYPE), desc=np.zeros((nb, cap, 32), np.uint8), ur=np.zeros((nb, cap), np.float32), cnt=np.zeros(nb, np.int32),
             mp=np.zeros((nb, cap), np.int32), nm=np.zeros(nb, np.int32))
    track_lk = lambda: B.check(L.sgs_tracker_track_lk(trk.h, nb, P(ti['pidx']), P(ti['ur']), v(0), P(ti['boxes']), P(ti['nb']), P(ti['have']), P(ti['lxyz']), P(ti['ldesc']),
                                                      P(ti['lflags']), P(ti['loct']), P(ti['lang']), P(ti['ln']), P(Tc), P(ti['T']), TH, 0, 1, P(o['kps']),
                                                      P(o['desc']), P(o['ur']), P(o['cnt']), P(o['mp']), P(o['nm'])))
    track_lk()
    rng = np.random.default_rng(5)
    lms = [bench.make_local_map(f, o['kps'][f], o['desc'][f], int(o['cnt'][f]), ti, mcap, camd, sf, rng, W, H) for f in range(nb)]
    stack = lambda k, dt: np.ascontiguousarray(np.stack([m[k] for m in lms]).astype(dt))
    dev = {k: torch.from_numpy(a).cuda() for k, a in dict(lxyz=ti['lxyz'], ldesc=ti['ldesc'], lflags=ti['lflags'], loct=ti['loct'], lang=ti['lang'], ln=ti['ln'], Tc=Tc, Tl=ti['T'],
                                                          lid=stack('lid', np.int32), xyz=stack('xyz', np.float32), nrm=stack('nrm', np.float32), mn=stack('mn', np.float32),
                                                          mx=stack('mx', np.float32), dsc=stack('dsc', np.uint8), valid=stack('valid', np.uint8), obs=stack('obs', np.uint8),
                                                          n=np.array([m['n'] for m in lms], np.int32)).items()}
    outd = dict(T1=torch.zeros((nb, 16), device='cuda'), T2=torch.zeros((nb, 16), device='cuda'), mp=torch.zeros((nb, cap), dtype=torch.int32, device='cuda'),
                outl=torch.zeros((nb, cap), dtype=torch.uint8, device='cuda'), st=torch.zeros((nb, 8), dtype=torch.int32, device='cuda'))
    isig = np.zeros(16, np.float32); isig[:8] = 1.0 / (sf.astype(np.float32) ** 2)
    a = B.PoseChainBatch()
    D = lambda k: dev[k].data_ptr()
    a.last_xyz, a.last_desc, a.last_flags, a.last_octave, a.last_angle, a.last_n = D('lxyz'), D('ldesc'), D('lflags'), D('loct'), D('lang'), D('ln')
    a.tcw_cur, a.tcw_last, a.th, a.mono, a.check_orientation, a.last_local_id = D('Tc'), D('Tl'), TH, 0, 1, D('lid')
    a.mp_xyz, a.mp_normal, a.mp_min_dist, a.mp_max_dist, a.mp_desc, a.mp_valid, a.mp_obs, a.mp_n, a.mp_cap = D('xyz'), D('nrm'), D('mn'), D('mx'), D('dsc'), D('valid'), D('obs'), D('n'), mcap
    a.th_local, a.nnratio_local = 3.0, 0.8
    for l in range(16): a.inv_level_sigma2[l] = float(isig[l])
    a.tcw_motion, a.tcw_final, a.f_mp, a.outlier, a.stats = outd['T1'].data_ptr(), outd['T2'].data_ptr(), outd['mp'].data_ptr(), outd['outl'].data_ptr(), outd['st'].data_ptr()
    # a first chain with a smaller local-map capacity (it reads the first mp_cap rows of the local map): the checked call below runs on the scratch
    # regrown for mcap and a recreated local-map matcher, after track_lk has restored the matches the first chain changed
    a.mp_cap = 256
    B.check(L.sgs_tracker_pose_chain_device(trk.h, C.byref(a), nb, v(0)))
    first = {k: x.copy() for k, x in o.items()}
    track_lk()
    assert all(np.array_equal(o[k], first[k]) for k in o)
    a.mp_cap = mcap
    B.check(L.sgs_tracker_pose_chain_device(trk.h, C.byref(a), nb, v(0)))
    torch.cuda.synchronize()
    g = {k: t.cpu().numpy() for k, t in outd.items()}
    trk.close()
    camv = np.array([camd['fx'], camd['fy'], camd['cx'], camd['cy'], camd['bf'], cam.min_x, cam.min_y, cam.max_x, cam.max_y], np.float32)
    retried = 0; added = 0
    for f in range(nb):
        m = int(o['cnt'][f])
        cur = O.FrameArrays(o['kps'][f, :m], o['ur'][f, :m], o['desc'][f, :m], W, H, camd['fx'], camd['fy'], camd['cx'], camd['cy'], camd['bf'], sf)
        r = oracle_chain(f, cur, int(o['nm'][f]), o['mp'][f, :m].copy(), ti, lms[f], camv, camd, sf, isig, TH, tcw_motion_gpu=g['T1'][f])
        assert np.array_equal(g['st'][f], r['stats']), (f, g['st'][f], r['stats'])
        assert np.array_equal(g['mp'][f, :m], r['mp']), f
        assert np.array_equal(g['outl'][f, :m], r['outlier']), f
        assert np.abs(g['T1'][f].reshape(4, 4) - r['T1']).max() <= 1e-5 and np.abs(g['T2'][f].reshape(4, 4) - r['T2']).max() <= 1e-5, f
        retried += int(r['stats'][1]); added += int(r['stats'][6])
    print('frames retried with 2 th: %d; matches added by the local-map search: %d; stats per frame:\n%s' % (retried, added, g['st']))
    assert retried >= 2 and added > 20 * nb
