"""sgs_tracker_refkf_chain_device: Tracking::TrackReferenceKeyFrame (src/Tracking.cc:796-838: ComputeBoW, SearchByBoW(reference key frame, frame) with 0.7
and the orientation check, the 15-match gate, PoseOptimization from the last frame's pose, the outlier discard) and TrackLocalMap after it, in one device
call after sgs_tracker_track_lk, against the same chain composed from the CPU oracle's functions (tests/refkf_cases.py).  Indices, flags and counters are
compared exactly, the poses within the optimiser's tolerance (1e-5); the local half of the oracle runs from the GPU's first pose as in
tests/test_gpu_pose_chain.py.  The reference key frame of every frame is its previous frame (bench.make_track_inputs' last-frame arrays), the local map
bench.make_local_map's; the vocabularies are trained on the frames' descriptors."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle as O  # noqa: E402
import refkf_cases as R  # noqa: E402
from pysgs import binding as B  # noqa: E402
from pysgs import synth  # noqa: E402

W, H, NF, TH = 640, 480, 1000, 15.0
SENT = -7


class GpuVoc(B._Handle):
    def __init__(self, voc):
        v = C.c_void_p
        super().__init__(B.lib().sgs_vocabulary_create, B.lib().sgs_vocabulary_destroy, 0, voc['k'], voc['L'], len(voc['parent']), voc['parent'].ctypes.data_as(v),
                         np.ascontiguousarray(voc['desc']).ctypes.data_as(v), voc['weight'].ctypes.data_as(v))


def _setup(nb=12):
    import bench
    import torch
    frames, boxes, unique = bench.make_frames(nb, 11, W, H, unique=6)
    pidx = bench.prev_index(nb, unique)
    camd = dict(synth.TUM3)
    sf = synth.scale_factors(); cam = B.make_camera(W, H, camd, sf)
    trk = B.Tracker(W, H, cam, NF, 1.2, 8, 20, 7, max_batch=nb, point_cap=NF + 64, max_boxes=4, device=0)
    cap, pcap = trk.cap, trk.point_cap
    L, v = B.lib(), C.c_void_p
    P = lambda a: a.ctypes.data_as(v)
    kps = np.zeros((nb, cap), B.KP_DTYPE); desc = np.zeros((nb, cap, 32), np.uint8); n = np.zeros(nb, np.int32)
    B.check(L.sgs_tracker_extract(trk.h, P(frames), nb, W * H, W, P(kps), P(desc), cap, P(n)))
    ti = bench.make_track_inputs(kps, desc, n, boxes, cap, pcap, pidx, W, H, camd)
    ti['Tc'] = ti['T'].copy()
    # trap points: local-map points (every other last-frame point) with octave <= 2 moved 6 px sideways -- the motion model's search still matches them,
    # its PoseOptimization rejects them, and the local search after the reference key frame would take them again unless they count as seen
    trap = np.zeros(ti['lflags'].shape, bool)
    for f in range(nb):
        m = int(ti['ln'][f])
        cand = np.nonzero((np.arange(m) % 2 == 0) & (ti['loct'][f, :m] <= 2))[0][5::40]
        trap[f, cand] = True
        ti['lxyz'][f, cand, 0] += 6.0 * ti['lxyz'][f, cand, 2] / camd['fx']
    o = dict(kps=np.zeros((nb, cap), B.KP_DTYPE), desc=np.zeros((nb, cap, 32), np.uint8), ur=np.zeros((nb, cap), np.float32), cnt=np.zeros(nb, np.int32),
             mp=np.zeros((nb, cap), np.int32), nm=np.zeros(nb, np.int32))

    def track_lk():
        B.check(L.sgs_tracker_track_lk(trk.h, nb, P(ti['pidx']), P(ti['ur']), v(0), P(ti['boxes']), P(ti['nb']), P(ti['have']), P(ti['lxyz']), P(ti['ldesc']),
                                       P(ti['lflags']), P(ti['loct']), P(ti['lang']), P(ti['ln']), P(ti['Tc']), P(ti['T']), TH, 0, 1, P(o['kps']),
                                       P(o['desc']), P(o['ur']), P(o['cnt']), P(o['mp']), P(o['nm'])))
    track_lk()
    rng = np.random.default_rng(5)
    lms = [bench.make_local_map(f, o['kps'][f], o['desc'][f], int(o['cnt'][f]), ti, 1536, camd, sf, rng, W, H) for f in range(nb)]
    isig = np.zeros(16, np.float32); isig[:8] = 1.0 / (sf.astype(np.float32) ** 2)
    camv = np.array([camd['fx'], camd['fy'], camd['cx'], camd['cy'], camd['bf'], cam.min_x, cam.min_y, cam.max_x, cam.max_y], np.float32)
    return dict(nb=nb, trk=trk, cap=cap, pc=pcap, ti=ti, o=o, lms=lms, camd=camd, sf=sf, isig=isig, camv=camv, track_lk=track_lk, trap=trap, torch=torch)


def _local_map_fields(a, dev, mcap):
    D = lambda k: dev[k].data_ptr()
    a.mp_xyz, a.mp_normal, a.mp_min_dist, a.mp_max_dist, a.mp_desc, a.mp_valid, a.mp_obs, a.mp_n, a.mp_cap = D('xyz'), D('nrm'), D('mn'), D('mx'), D('dsc'), D('valid'), D('obs'), D('n'), mcap


def _pose_chain(s, dev, mcap):
    """one pose chain call; returns its outputs and the motion discards (host copies)"""
    torch = s['torch']
    nb, cap = s['nb'], s['cap']
    out = dict(T1=torch.zeros((nb, 16), device='cuda'), T2=torch.zeros((nb, 16), device='cuda'), mp=torch.zeros((nb, cap), dtype=torch.int32, device='cuda'),
               outl=torch.zeros((nb, cap), dtype=torch.uint8, device='cuda'), st=torch.zeros((nb, 8), dtype=torch.int32, device='cuda'))
    a = B.PoseChainBatch()
    D = lambda k: dev[k].data_ptr()
    a.last_xyz, a.last_desc, a.last_flags, a.last_octave, a.last_angle, a.last_n = D('lxyz'), D('ldesc'), D('lflags'), D('loct'), D('lang'), D('ln')
    a.tcw_cur, a.tcw_last, a.th, a.mono, a.check_orientation, a.last_local_id = D('Tc'), D('Tl'), TH, 0, 1, D('lid')
    _local_map_fields(a, dev, mcap)
    a.th_local, a.nnratio_local = 3.0, 0.8
    for l in range(16): a.inv_level_sigma2[l] = float(s['isig'][l])
    a.tcw_motion, a.tcw_final, a.f_mp, a.outlier, a.stats = out['T1'].data_ptr(), out['T2'].data_ptr(), out['mp'].data_ptr(), out['outl'].data_ptr(), out['st'].data_ptr()
    B.check(B.lib().sgs_tracker_pose_chain_device(s['trk'].h, C.byref(a), nb, C.c_void_p(0)))
    d = C.c_void_p()
    B.check(B.lib().sgs_tracker_motion_discards_device(s['trk'].h, C.byref(d)))
    disc = np.zeros((nb, mcap), np.uint8)
    s['torch'].cuda.synchronize()
    B.check(B.lib().sgs_memcpy_d2h(disc.ctypes.data_as(C.c_void_p), d, disc.nbytes))
    return {k: t.cpu().numpy() for k, t in out.items()}, disc


def _refkf_batch(s, dev, kd, mcap, outd, th_local, enable, seen):
    a = B.RefKfBatch()
    D = lambda k: dev[k].data_ptr()
    a.kf_node, a.kf_weight, a.kf_desc, a.kf_angle, a.kf_xyz, a.kf_flags, a.kf_n, a.kf_local_id = (kd[k].data_ptr() for k in ('node', 'weight', 'desc', 'angle', 'xyz', 'flags', 'n', 'lid'))
    a.tcw_last = D('Tl')
    a.frame_enable = enable.data_ptr() if enable is not None else None
    a.seen_in = seen.data_ptr() if seen is not None else None
    _local_map_fields(a, dev, mcap)
    a.th_local, a.nnratio_local = th_local, 0.8
    for l in range(16): a.inv_level_sigma2[l] = float(s['isig'][l])
    a.tcw_refkf, a.tcw_final, a.f_mp, a.outlier, a.stats = (outd[k].data_ptr() for k in ('T1', 'T2', 'mp', 'outl', 'st'))
    return a


@pytest.mark.parametrize('k,L', [(3, 5), (10, 3)])
def test_refkf_chain_against_the_oracle_functions(k, L):
    s = _setup()
    torch = s['torch']
    nb, cap, pc, ti, o, lms = s['nb'], s['cap'], s['pc'], s['ti'], s['o'], s['lms']
    mcap = 1536
    trk = s['trk']
    voc = R.train_vocabulary(np.concatenate([o['desc'][f, :o['cnt'][f]] for f in range(nb)]), k, L, seed=k)
    V = O.Vocabulary(voc['k'], voc['L'], voc['parent'], voc['desc'], voc['weight'])
    gv = GpuVoc(voc)
    # reference key frame of frame f: its previous frame without the trap points; some features bad; frame 5 has too few features for 15 matches;
    # frame 4's points have no observations (nmatchesMap < 10)
    kf = dict(desc=ti['ldesc'].copy(), angle=ti['lang'].copy(), xyz=ti['lxyz'].copy(), flags=ti['lflags'].copy(), n=ti['ln'].copy(),
              lid=np.stack([m['lid'] for m in lms]).astype(np.int32))
    kf['flags'][s['trap']] = 0
    kf['flags'][:, 11::19] |= 4
    kf['flags'][4] &= ~np.uint8(2)
    kf['n'][5] = 12
    kf['node'] = np.zeros(kf['flags'].shape, np.int32); kf['weight'] = np.zeros(kf['flags'].shape, np.float64)
    for f in range(nb):
        m = int(kf['n'][f])
        _, kf['weight'][f, :m], kf['node'][f, :m] = V.transform(kf['desc'][f, :m], 4)
    stack = lambda key, dt: np.ascontiguousarray(np.stack([m[key] for m in lms]).astype(dt))
    dev = {key: torch.from_numpy(np.ascontiguousarray(a)).cuda() for key, a in dict(
        lxyz=ti['lxyz'], ldesc=ti['ldesc'], lflags=ti['lflags'], loct=ti['loct'], lang=ti['lang'], ln=ti['ln'], Tc=ti['Tc'], Tl=ti['T'], lid=stack('lid', np.int32),
        xyz=stack('xyz', np.float32), nrm=stack('nrm', np.float32), mn=stack('mn', np.float32), mx=stack('mx', np.float32), dsc=stack('dsc', np.uint8),
        valid=stack('valid', np.uint8), obs=stack('obs', np.uint8), n=np.array([m['n'] for m in lms], np.int32)).items()}
    kd = {key: torch.from_numpy(np.ascontiguousarray(kf[key])).cuda() for key in ('node', 'weight', 'desc', 'angle', 'xyz', 'flags', 'n', 'lid')}
    try:
        # the pose chain, then (same frames) the pose chain again with a reference-key-frame chain in between: bit-identical outputs
        first, disc = _pose_chain(s, dev, mcap)
        s['track_lk']()
        seen = torch.from_numpy(disc).cuda()
        outd = dict(T1=torch.full((nb, 16), SENT, dtype=torch.float32, device='cuda'), T2=torch.full((nb, 16), SENT, dtype=torch.float32, device='cuda'),
                    mp=torch.full((nb, cap), SENT, dtype=torch.int32, device='cuda'), outl=torch.full((nb, cap), 7, dtype=torch.uint8, device='cuda'),
                    st=torch.full((nb, 8), SENT, dtype=torch.int32, device='cuda'))
        enabled = np.ones(nb, np.uint8); enabled[2] = 0
        th_of = np.where(np.arange(nb) % 3 == 0, 5.0, 3.0)                       # rows right after a relocalisation search with 5: two calls
        for th in (3.0, 5.0):
            en = torch.from_numpy((enabled & (th_of == th)).astype(np.uint8)).cuda()
            a = _refkf_batch(s, dev, kd, mcap, outd, th, en, seen)
            B.check(B.lib().sgs_tracker_refkf_chain_device(trk.h, gv.h, C.byref(a), nb, C.c_void_p(0)))
        second, disc2 = _pose_chain(s, dev, mcap)
        for key in first:
            assert np.array_equal(first[key], second[key]), key
        assert np.array_equal(disc, disc2)
        torch.cuda.synchronize()
        g = {key: t.cpu().numpy() for key, t in outd.items()}
    finally:
        gv.close()
        trk.close()
    camd, sf, isig, camv = s['camd'], s['sf'], s['isig'], s['camv']
    passed = gated = nomap = excluded = 0
    for f in range(nb):
        m = int(o['cnt'][f])
        cur = O.FrameArrays(o['kps'][f, :m], o['ur'][f, :m], o['desc'][f, :m], W, H, camd['fx'], camd['fy'], camd['cx'], camd['cy'], camd['bf'], sf)
        # the discard record of the pose chain
        assert np.array_equal(disc[f], R.motion_discards(cur, o['mp'][f, :m].copy(), int(o['nm'][f]), ti, f, lms[f], camd, isig, TH)), f
        if not enabled[f]:
            assert np.all(g['st'][f] == SENT) and np.all(g['mp'][f] == SENT) and np.all(g['outl'][f] == 7) and np.all(g['T1'][f] == SENT) and np.all(g['T2'][f] == SENT), f
            continue
        kff = {key: kf[key][f] for key in ('desc', 'angle', 'xyz', 'flags', 'lid')}; kff['n'] = kf['n'][f]
        r = R.oracle_refkf(cur, V, kff, ti['T'][f].reshape(4, 4), lms[f], disc[f], camd, camv, sf, isig, th_of[f], pc, tcw_first=g['T1'][f])
        assert np.array_equal(g['st'][f], r['stats']), (f, g['st'][f], r['stats'])
        if not r['stats'][1]:
            assert np.all(g['mp'][f] == SENT) and np.all(g['outl'][f] == 7) and np.all(g['T1'][f] == SENT) and np.all(g['T2'][f] == SENT), f
            gated += 1
            continue
        assert np.array_equal(g['mp'][f, :m], r['mp']), (f, int((g['mp'][f, :m] != r['mp']).sum()))
        assert np.array_equal(g['outl'][f, :m], r['outlier']), f
        assert np.abs(g['T1'][f].reshape(4, 4) - r['T1']).max() <= 1e-5 and np.abs(g['T2'][f].reshape(4, 4) - r['T2']).max() <= 1e-5, f
        passed += 1; nomap += int(r['stats'][4] < 10)
        # without the motion model's discards the local search takes some of them back
        r0 = R.oracle_refkf(cur, V, kff, ti['T'][f].reshape(4, 4), lms[f], None, camd, camv, sf, isig, th_of[f], pc, tcw_first=g['T1'][f])
        excluded += int(np.sum((r0['mp'] >= pc) & (disc[f][np.maximum(r0['mp'] - pc, 0)] != 0)))
    print('rows past the gate %d, stopped at it %d, nmatchesMap < 10: %d; discarded points the local search would have matched: %d; stats:\n%s'
          % (passed, gated, nomap, excluded, g['st']))
    assert gated >= 1 and nomap >= 1 and passed >= 7 and excluded >= 1
    assert int(disc.sum()) >= 1


def test_refkf_chain_refuses_bad_arguments():
    s = _setup(nb=2)
    torch = s['torch']
    nb, cap, ti, o, lms, trk = s['nb'], s['cap'], s['ti'], s['o'], s['lms'], s['trk']
    mcap = 1536
    voc = R.train_vocabulary(o['desc'][0, :o['cnt'][0]], 3, 5)
    gv = GpuVoc(voc)
    try:
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device='cuda')
        kd = dict(node=z((nb, s['pc']), torch.int32), weight=z((nb, s['pc']), torch.float64), desc=z((nb, s['pc'], 32), torch.uint8), angle=z((nb, s['pc']), torch.float32),
                  xyz=z((nb, s['pc'], 3), torch.float32), flags=z((nb, s['pc']), torch.uint8), n=torch.full((nb,), 20, dtype=torch.int32, device='cuda'),
                  lid=torch.full((nb, s['pc']), -1, dtype=torch.int32, device='cuda'))
        stack = lambda key, dt: np.ascontiguousarray(np.stack([m[key] for m in lms]).astype(dt))
        dev = {key: torch.from_numpy(a).cuda() for key, a in dict(Tl=ti['T'], xyz=stack('xyz', np.float32), nrm=stack('nrm', np.float32), mn=stack('mn', np.float32),
                                                                  mx=stack('mx', np.float32), dsc=stack('dsc', np.uint8), valid=stack('valid', np.uint8),
                                                                  obs=stack('obs', np.uint8), n=np.array([m['n'] for m in lms], np.int32)).items()}
        outd = dict(T1=torch.full((nb, 16), SENT, dtype=torch.float32, device='cuda'), T2=torch.full((nb, 16), SENT, dtype=torch.float32, device='cuda'),
                    mp=torch.full((nb, cap), SENT, dtype=torch.int32, device='cuda'), outl=torch.full((nb, cap), 7, dtype=torch.uint8, device='cuda'),
                    st=torch.full((nb, 8), SENT, dtype=torch.int32, device='cuda'))
        L, v = B.lib(), C.c_void_p
        call = lambda a, n=nb, voc_h=gv.h: L.sgs_tracker_refkf_chain_device(trk.h, voc_h, C.byref(a), n, v(0))
        a = _refkf_batch(s, dev, kd, mcap, outd, 3.0, None, None)
        for field in ('kf_node', 'kf_xyz', 'kf_n', 'tcw_last', 'mp_obs', 'stats'):
            bad = _refkf_batch(s, dev, kd, mcap, outd, 3.0, None, None)
            setattr(bad, field, None)
            assert call(bad) == B.SGS_ERR_INVALID, field
        assert call(a, n=0) == B.SGS_ERR_INVALID and call(a, n=nb + 1) == B.SGS_ERR_INVALID
        assert call(a, voc_h=None) == B.SGS_ERR_INVALID
        a.mp_cap = 0
        assert call(a) == B.SGS_ERR_INVALID
        torch.cuda.synchronize()
        assert all(bool((t == (7 if key == 'outl' else SENT)).all()) for key, t in outd.items())
        # a key frame with more features than the tracker's point_cap: that row's stats[0] = -1, nothing else written
        a.mp_cap = mcap
        kd['n'][1] = s['pc'] + 1
        B.check(call(a))
        torch.cuda.synchronize()
        st = outd['st'].cpu().numpy()
        assert list(st[1]) == [-1, 0, 0, 0, 0, 0, 0, 0] and bool((outd['mp'][1] == SENT).all()) and bool((outd['T1'][1] == SENT).all())
        assert st[0, 0] >= 0
    finally:
        gv.close()
        trk.close()
