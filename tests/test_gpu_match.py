"""GPU parity: Hamming / projection matchers / dyn-reject (through the C ABI) against the CPU oracle.
Integer results bit-exact; epipolar distances within 1e-5 (they are in fact identical FP64 values)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle as O  # noqa: E402
import scenarios as S  # noqa: E402
from pysgs import binding as B  # noqa: E402
from pysgs import synth  # noqa: E402


def test_hamming_pairs_and_known_answers():
    a = synth.descriptors_s5(5000, 1); b = synth.descriptors_s5(5000, 2)
    got = B.hamming_pairs(a, b)
    ref = np.unpackbits(a ^ b, axis=1).sum(1)
    assert np.array_equal(got, ref)
    z = np.zeros((3, 32), np.uint8); f = np.full((3, 32), 255, np.uint8)
    assert B.hamming_pairs(z, f).tolist() == [256, 256, 256] and B.hamming_pairs(z, z).tolist() == [0, 0, 0]
    assert all(O.hamming(a[i], b[i]) == got[i] for i in range(50))


@pytest.mark.parametrize('nq,nt', [(1, 1), (7, 300), (1000, 1000), (1000, 257), (130, 5000), (4096, 4096), (3, 0)])
def test_bf_matches_oracle(nq, nt):
    t = synth.descriptors_s5(max(nt, 1), 5)[:nt]
    q = synth.descriptors_near(synth.descriptors_s5(max(nq, 1), 5)[:nq] if nt == 0 else t[np.random.RandomState(nq).randint(0, nt, nq)], 6)
    gi, gd, gs = B.hamming_bf(q, t)
    if nt == 0:
        assert (gi == -1).all() and (gd == 256).all() and (gs == 256).all()
        return
    oi, od, os_ = O.bf_match(q, t)
    assert np.array_equal(gi, oi) and np.array_equal(gd, od) and np.array_equal(gs, os_)


def test_bf_tie_break_first_index_wins():
    t = np.zeros((600, 32), np.uint8)         # all identical: every distance ties
    q = np.zeros((40, 32), np.uint8); q[:, 0] = 1
    gi, gd, gs = B.hamming_bf(q, t)
    assert (gi == 0).all() and (gd == 1).all() and (gs == 1).all()


def test_bf_large_property():
    """BASELINE config 5 sizes: not oracle-checked pair by pair (too slow); size-independent properties instead."""
    n = 16384
    t = synth.descriptors_s5(n, 5)
    q = synth.descriptors_near(t, 6, maxflips=20)
    gi, gd, gs = B.hamming_bf(q, t)
    # the planted neighbour (<= 20 flips) must be found: random 256-bit strings are ~128 apart
    assert np.array_equal(gi, np.arange(n))
    assert np.array_equal(gd, np.unpackbits(q ^ t, axis=1).sum(1))
    assert (gs >= gd).all() and (gs > 60).all()
    # idempotence / self-match
    si, sd, _ = B.hamming_bf(t[:2048], t)
    assert np.array_equal(si, np.arange(2048)) and (sd == 0).all()


def _frames(s):
    fo = O.FrameArrays(s['kps'], s['uright'], s['desc'], s['w'], s['h'], s['cam']['fx'], s['cam']['fy'], s['cam']['cx'], s['cam']['cy'], s['cam']['bf'], s['sf'])
    fg = B.HostFrame(s['kps'], s['uright'], s['desc'], s['w'], s['h'], s['cam']['fx'], s['cam']['fy'], s['cam']['cx'], s['cam']['cy'], s['cam']['bf'], s['sf'])
    return fo, fg


@pytest.mark.parametrize('seed', range(6))
@pytest.mark.parametrize('th', [15.0, 30.0])
def test_search_by_projection_lastframe(seed, th):
    s = S.random_lastframe_scenario(seed, n_cur=1000 + 37 * seed, n_last=900 + 53 * seed, conflict=[0.0, 0.3, 0.6][seed % 3], mono=(seed == 5))
    fo, fg = _frames(s)
    args = (s['Tcw_cur'], s['Tcw_last'], s['last_has'], s['last_xyz'], s['last_desc'], s['last_obs'], s['last_oct'], s['last_angle'], th)
    for check_ori in (True, False):
        nm_o, mp_o, _ = O.search_by_projection_last(fo, *args, mono=s['mono'], check_ori=check_ori)
        nm_g, mp_g = B.match_project_lastframe(fg, *args, mono=s['mono'], check_ori=check_ori)
        assert nm_g == nm_o, (seed, th, check_ori)
        assert np.array_equal(mp_g, mp_o)
        assert nm_o > 50   # the scenario really matches something


def test_search_by_projection_lastframe_preexisting_matches():
    s = S.random_lastframe_scenario(7)
    fo, fg = _frames(s)
    rng = np.random.RandomState(1)
    pre = np.full(len(s['kps']), -1, np.int32); m = rng.rand(len(pre)) < 0.3; pre[m] = 5
    pre_obs = (rng.rand(len(pre)) < 0.5).astype(np.uint8)
    args = (s['Tcw_cur'], s['Tcw_last'], s['last_has'], s['last_xyz'], s['last_desc'], s['last_obs'], s['last_oct'], s['last_angle'], 15.0)
    nm_o, mp_o, _ = O.search_by_projection_last(fo, *args, cur_mp=pre, cur_mp_obs=pre_obs)
    nm_g, mp_g = B.match_project_lastframe(fg, *args, cur_mp=pre, cur_mp_obs=pre_obs)
    assert nm_g == nm_o and np.array_equal(mp_g, mp_o)


@pytest.mark.parametrize('seed', range(5))
def test_search_by_projection_localmap(seed):
    s = S.random_localmap_scenario(seed, n_cur=1000, n_mp=2500 + 100 * seed, conflict=[0.2, 0.5][seed % 2])
    fo, fg = _frames(s)
    for th, ratio in ((3.0, 0.8), (1.0, 0.8), (5.0, 0.6)):
        a = (s['inview'], s['projx'], s['projy'], s['projxr'], s['level'], s['viewcos'], s['mp_desc'], s['mp_obs'], th, ratio, s['f_mp'], s['f_obs'])
        nm_o, mp_o, ob_o, _ = O.search_by_projection_local(fo, *a)
        nm_g, mp_g, ob_g = B.match_project_localmap(fg, *a)
        assert nm_g == nm_o, (seed, th)
        assert np.array_equal(mp_g, mp_o) and np.array_equal(ob_g, ob_o)
        assert nm_o > 100


def test_matchers_on_extracted_frames():
    """End-to-end shaped case: frame k-1 keypoints with depth become map points, matched into frame k."""
    frames, _ = synth.stream_s2(2, 640, 480, seed=4, person=False)
    k0, d0 = O.extract(frames[0]); k1, d1 = O.extract(frames[1])
    depth = synth.depth_s1()
    cam = synth.TUM3; sf = S.scale_factors()
    z = depth[k0['y'].astype(np.int64), k0['x'].astype(np.int64)]
    Xw = np.stack([(k0['x'] - cam['cx']) * z / cam['fx'], (k0['y'] - cam['cy']) * z / cam['fy'], z], 1).astype(np.float32)
    z1 = depth[k1['y'].astype(np.int64), k1['x'].astype(np.int64)]
    ur = (k1['x'] - np.float32(cam['bf']) / z1).astype(np.float32)
    fo = O.FrameArrays(k1, ur, d1, 640, 480, cam['fx'], cam['fy'], cam['cx'], cam['cy'], cam['bf'], sf)
    fg = B.HostFrame(k1, ur, d1, 640, 480, cam['fx'], cam['fy'], cam['cx'], cam['cy'], cam['bf'], sf)
    T = np.eye(4, dtype=np.float32)
    ones = np.ones(len(k0), np.uint8)
    args = (T, T, ones, Xw, d0, ones, k0['octave'], k0['angle'], 15.0)
    nm_o, mp_o, _ = O.search_by_projection_last(fo, *args)
    nm_g, mp_g = B.match_project_lastframe(fg, *args)
    assert nm_g == nm_o and np.array_equal(mp_g, mp_o)


@pytest.mark.parametrize('seed', range(4))
def test_dynreject(seed):
    s = S.dynreject_scenario(seed, n=1000 + 13 * seed)
    for have_dyn in (True, False):
        so, ko, do, ro = O.dynreject(s['cur'], s['prev'], s['F'], s['boxes'], have_dyn, 1000)
        sg, kg, dg, rg = B.dynreject(s['cur'], s['prev'], s['F'], s['boxes'], have_dyn, 1000)
        assert sg == so and rg == ro and np.array_equal(kg, ko)
        assert np.all(np.abs(dg - do) <= 1e-5 * np.maximum(1.0, np.abs(do)))      # tolerance from BASELINE.json north_star
        assert np.array_equal(dg.view(np.uint64), do.view(np.uint64))              # and in fact bit-identical
        assert 0 < so < len(ko)
    # restore-all branch: almost everything rejected while a person box is present
    prev_bad = s['prev'] + 50
    so, ko, _, ro = O.dynreject(s['cur'], prev_bad, s['F'], s['boxes'], True, 1000)
    sg, kg, _, rg = B.dynreject(s['cur'], prev_bad, s['F'], s['boxes'], True, 1000)
    assert ro and rg and sg == so and np.array_equal(kg, ko)
    # empty F (quirk Q11): keep everything
    sg, kg, _, rg = B.dynreject(s['cur'], s['prev'], None, s['boxes'], True, 1000)
    assert sg == len(kg) and kg.all() and not rg
    # degenerate F (all zeros): distance is NaN -> everything removed, as in the reference
    so, ko, _, _ = O.dynreject(s['cur'], s['prev'], np.zeros(9), None, False, 1000)
    sg, kg, _, _ = B.dynreject(s['cur'], s['prev'], np.zeros(9), None, False, 1000)
    assert sg == so == 0 and not kg.any()


def test_dynreject_batch_device_compaction():
    import torch
    F_, cap = 5, 1100
    rng = np.random.RandomState(0)
    kps = np.zeros((F_, cap), B.KP_DTYPE); desc = rng.randint(0, 256, (F_, cap, 32)).astype(np.uint8)
    counts = np.array([1000, 1013, 0, 37, 1100], np.int32)
    prev = np.zeros((F_, cap, 2), np.float32); Fm = np.zeros((F_, 9)); boxes = np.zeros((F_, 4, 4), np.float32)
    nb = np.array([2, 0, 1, 2, 2], np.int32); have = np.array([1, 0, 1, 1, 1], np.uint8)
    refs = []
    for f in range(F_):
        s = S.dynreject_scenario(20 + f, n=cap)
        kps[f]['x'] = s['cur'][:, 0]; kps[f]['y'] = s['cur'][:, 1]; kps[f]['octave'] = rng.randint(0, 8, cap); kps[f]['angle'] = rng.rand(cap)
        prev[f] = s['prev'] if f != 3 else s['prev'] + 40     # frame 3: restore-all branch
        Fm[f] = s['F'].reshape(9); boxes[f, :2] = s['boxes']
        if f == 4:
            Fm[f, 0] = np.nan                                  # empty F
        n = counts[f]
        so, ko, _, ro = O.dynreject(s['cur'][:n], prev[f, :n], None if f == 4 else Fm[f], boxes[f, :nb[f]], bool(have[f]), 1000)
        refs.append((so, ko, ro))
    t = {k: torch.from_numpy(v).cuda() for k, v in dict(kps=kps.view(np.uint8).reshape(F_, cap, 28), desc=desc, counts=counts, prev=prev, Fm=Fm, boxes=boxes, nb=nb, have=have).items()}
    ko_t = torch.zeros_like(t['kps']); do_t = torch.zeros_like(t['desc']); co_t = torch.zeros_like(t['counts']); keep_t = torch.zeros(F_, cap, dtype=torch.uint8, device='cuda')
    torch.cuda.synchronize()
    B.dynreject_batch_device(t['kps'].data_ptr(), t['desc'].data_ptr(), t['counts'].data_ptr(), cap, F_, t['prev'].data_ptr(), t['Fm'].data_ptr(),
                             t['boxes'].data_ptr(), t['nb'].data_ptr(), 4, t['have'].data_ptr(), 1000, ko_t.data_ptr(), do_t.data_ptr(), co_t.data_ptr(), keep_t.data_ptr(), 0)
    torch.cuda.synchronize()
    co = co_t.cpu().numpy(); ko = ko_t.cpu().numpy().reshape(F_, cap * 28).view(B.KP_DTYPE).reshape(F_, cap); do_ = do_t.cpu().numpy(); keep = keep_t.cpu().numpy()
    for f in range(F_):
        so, kref, ro = refs[f]
        n = counts[f]
        assert np.array_equal(keep[f, :n], kref)
        sel = np.arange(n) if ro else np.nonzero(kref)[0]
        assert co[f] == len(sel)
        assert ko[f, :len(sel)].tobytes() == kps[f][sel].tobytes()
        assert np.array_equal(do_[f, :len(sel)], desc[f][sel])


@pytest.mark.parametrize('seed,ncur,nkf,orb_dist,th', [(1, 1000, 1000, 100, 10.0), (2, 1500, 800, 64, 3.0), (3, 300, 2000, 100, 10.0), (4, 1000, 1000, 50, 15.0)])
def test_keyframe_projection_matcher(seed, ncur, nkf, orb_dist, th):
    """SearchByProjection(Frame&, KeyFrame*, sAlreadyFound, th, ORBdist) (relocalisation, src/ORBmatcher.cc:1474-1601)."""
    s = S.keyframe_scenario(seed, n_cur=ncur, n_kf=nkf, conflict=0.4)
    cam = s['cam']
    fo = O.FrameArrays(s['kps'], s['uright'], s['desc'], 640, 480, cam['fx'], cam['fy'], cam['cx'], cam['cy'], cam['bf'], s['sf'])
    fg = B.HostFrame(s['kps'], s['uright'], s['desc'], 640, 480, cam['fx'], cam['fy'], cam['cx'], cam['cy'], cam['bf'], s['sf'])
    for ori in (True, False):
        nm_o, mp_o, _ = O.search_by_projection_kf(fo, s['Tcw_cur'], s['kf_valid'], s['last_xyz'], s['last_desc'], s['last_angle'], s['min_dist'], s['max_dist'], th,
                                                  orb_dist, ori, s['cur_mp'])
        nm_g, mp_g = B.match_project_keyframe(fg, s['Tcw_cur'], s['kf_valid'], s['last_xyz'], s['last_desc'], s['last_angle'], s['min_dist'], s['max_dist'], th,
                                              orb_dist, ori, s['cur_mp'])
        assert nm_g == nm_o and np.array_equal(mp_g, mp_o)
        assert nm_o > 20
        assert np.array_equal(mp_g[s['cur_mp'] >= 0], s['cur_mp'][s['cur_mp'] >= 0])        # keypoints that already held a map point are never touched


@pytest.mark.parametrize('seed,ncur,nmp,th,sim3', [(1, 1000, 1000, 3.0, 0), (2, 1500, 3000, 3.0, 0), (3, 400, 2000, 5.0, 0), (4, 1000, 2000, 4.0, 1), (5, 1000, 2000, 7.5, 2)])
def test_fuse_search(seed, ncur, nmp, th, sim3):
    """Search half of ORBmatcher::Fuse(KeyFrame*, vpMapPoints, th) (src/ORBmatcher.cc:829-980)."""
    import ctypes as C
    import torch
    s = S.keyframe_scenario(seed, n_cur=ncur, n_kf=nmp, conflict=0.3)
    cam = s['cam']; sf = s['sf'].astype(np.float32)
    rs = np.random.RandomState(seed + 7)
    R = s['Tcw_cur'][:3, :3].astype(np.float64); t = s['Tcw_cur'][:3, 3].astype(np.float64)
    Ow = (-(R.T @ t)).astype(np.float32)
    to = s['last_xyz'].astype(np.float64) - Ow.astype(np.float64); d = np.linalg.norm(to, axis=1)
    nrm = to / np.maximum(d[:, None], 1e-9) + rs.normal(0, 0.6, (nmp, 3)); nrm = (nrm / np.linalg.norm(nrm, axis=1, keepdims=True)).astype(np.float32)
    inv_s2 = (1.0 / (sf * sf)).astype(np.float32)
    xf = None
    if sim3 == 2:          # [sR21 | t21]: a small similarity on top of the key-frame pose
        a_ = 0.004; sc = 1.01
        xf = np.concatenate([(sc * np.array([[np.cos(a_), -np.sin(a_), 0], [np.sin(a_), np.cos(a_), 0], [0, 0, 1]])).reshape(9), [0.01, -0.005, 0.02]]).astype(np.float32)
    fo = O.FrameArrays(s['kps'], s['uright'], s['desc'], 640, 480, cam['fx'], cam['fy'], cam['cx'], cam['cy'], cam['bf'], s['sf'])
    bi_o, bd_o = O.fuse_search(fo, s['Tcw_cur'], Ow, s['kf_valid'], s['last_xyz'], nrm, s['min_dist'], s['max_dist'], s['last_desc'], th, inv_s2, sim3_variant=sim3, xform2=xf)
    assert (bi_o >= 0).sum() > 30 and (bd_o[bi_o >= 0] <= 50).sum() > 10
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    kcap, mcap = ncur + 5, nmp + 3
    pad = lambda a, cap: np.concatenate([a, np.zeros((cap - len(a),) + a.shape[1:], a.dtype)])[None]
    t_ = dict(kps=dev(pad(s['kps'], kcap).view(np.uint8).reshape(-1)), kd=dev(pad(s['desc'], kcap)), ur=dev(pad(s['uright'].astype(np.float32), kcap)), kn=dev(np.array([ncur], np.int32)),
              T=dev(s['Tcw_cur'].astype(np.float32).reshape(1, 16)), ow=dev(Ow.reshape(1, 3)), xyz=dev(pad(s['last_xyz'], mcap)), nrm=dev(pad(nrm, mcap)),
              mn=dev(pad(s['min_dist'], mcap)), mx=dev(pad(s['max_dist'], mcap)), md=dev(pad(s['last_desc'], mcap)), mv=dev(pad(s['kf_valid'], mcap)), mn_=dev(np.array([nmp], np.int32)))
    bi = torch.zeros((1, mcap), dtype=torch.int32, device='cuda'); bd = torch.zeros((1, mcap), dtype=torch.int32, device='cuda')
    a = B.FuseBatch()
    a.cam = B.make_camera(640, 480, cam, s['sf'])
    a.kf_kps, a.kf_desc, a.kf_uright, a.kf_n, a.kf_cap = t_['kps'].data_ptr(), t_['kd'].data_ptr(), t_['ur'].data_ptr(), t_['kn'].data_ptr(), kcap
    a.tcw, a.ow, a.mp_xyz, a.mp_normal, a.mp_min_dist, a.mp_max_dist = t_['T'].data_ptr(), t_['ow'].data_ptr(), t_['xyz'].data_ptr(), t_['nrm'].data_ptr(), t_['mn'].data_ptr(), t_['mx'].data_ptr()
    a.mp_desc, a.mp_valid, a.mp_n, a.mp_cap, a.th = t_['md'].data_ptr(), t_['mv'].data_ptr(), t_['mn_'].data_ptr(), mcap, th
    for l in range(8):
        a.inv_level_sigma2[l] = float(inv_s2[l])
    a.sim3_variant = sim3
    if xf is not None:
        t_['xf'] = dev(xf.reshape(1, 12)); a.xform2 = t_['xf'].data_ptr()
    a.best_idx, a.best_dist = bi.data_ptr(), bd.data_ptr()
    B.check(B.lib().sgs_fuse_search_batch_device(C.byref(a), 1, C.c_void_p(0)))
    torch.cuda.synchronize()
    assert np.array_equal(bi.cpu().numpy()[0, :nmp], bi_o) and np.array_equal(bd.cpu().numpy()[0, :nmp], bd_o)
    # the host entry point on the same inputs
    fg = B.HostFrame(s['kps'], s['uright'], s['desc'], 640, 480, cam['fx'], cam['fy'], cam['cx'], cam['cy'], cam['bf'], s['sf'])
    nm_h, bi_h, bd_h = _fuse_search_host(fg, s['Tcw_cur'], Ow, s, nrm, th, inv_s2, sim3, xf, None)
    assert np.array_equal(bi_h, bi_o) and np.array_equal(bd_h, bd_o) and nm_h == 0


def _fuse_search_host(fg, Tcw, Ow, s, nrm, th, inv_s2, sim3, xf, kf_matched):
    """sgs_fuse_search, the single-frame host entry point: (nmatches, best_idx, best_dist); kf_matched is updated in place."""
    import ctypes as C
    nmp = len(s['kf_valid'])
    P = lambda a: None if a is None else np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)
    bi = np.full(nmp, 7, np.int32); bd = np.full(nmp, 7, np.int32); nm = C.c_int(-1)
    B.check(B.lib().sgs_fuse_search(C.byref(fg.c), P(Tcw.astype(np.float32).reshape(16)), P(Ow.astype(np.float32)), nmp, P(s['kf_valid']), P(s['last_xyz']), P(nrm),
                                    P(s['min_dist']), P(s['max_dist']), P(s['last_desc']), th, P(inv_s2), sim3, P(xf), P(bi), P(bd),
                                    P(kf_matched), C.byref(nm), 0))
    return nm.value, bi, bd


@pytest.mark.parametrize('seed,ncur,nmp,th', [(11, 600, 900, 10), (12, 300, 1500, 10), (13, 800, 800, 4), (14, 1000, 3000, 10)])
def test_search_by_projection_sim3(seed, ncur, nmp, th):
    """ORBmatcher::SearchByProjection(KeyFrame*, Scw, vpPoints, vpMatched, th) (src/ORBmatcher.cc:292-405): ordered claims, two key frames per call."""
    import ctypes as C
    import torch
    from test_match_sim3 import sim3_inputs
    inv_s2 = None
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    kcap, mcap = ncur + 5, nmp + 3
    pad = lambda a, cap: np.concatenate([a, np.zeros((cap - len(a),) + a.shape[1:], a.dtype)])
    per = []
    for k in range(2):
        s, Ow, nrm, matched = sim3_inputs(seed + 100 * k, ncur, nmp)
        cam = s['cam']
        fo = O.FrameArrays(s['kps'], s['uright'], s['desc'], 640, 480, cam['fx'], cam['fy'], cam['cx'], cam['cy'], cam['bf'], s['sf'])
        nm_o, m_o = O.search_by_projection_sim3(fo, s['Tcw_cur'], Ow, s['kf_valid'], s['last_xyz'], nrm, s['min_dist'], s['max_dist'], s['last_desc'], float(th), matched)
        assert nm_o > 30
        per.append((s, Ow, nrm, matched, nm_o, m_o))
    st = lambda f: np.stack([f(p) for p in per])
    t_ = dict(kps=dev(st(lambda p: pad(p[0]['kps'], kcap)).view(np.uint8).reshape(-1)), kd=dev(st(lambda p: pad(p[0]['desc'], kcap))),
              ur=dev(st(lambda p: pad(p[0]['uright'].astype(np.float32), kcap))), kn=dev(np.array([ncur, ncur], np.int32)),
              T=dev(st(lambda p: p[0]['Tcw_cur'].astype(np.float32).reshape(16))), ow=dev(st(lambda p: p[1])), xyz=dev(st(lambda p: pad(p[0]['last_xyz'], mcap))),
              nrm=dev(st(lambda p: pad(p[2], mcap))), mn=dev(st(lambda p: pad(p[0]['min_dist'], mcap))), mx=dev(st(lambda p: pad(p[0]['max_dist'], mcap))),
              md=dev(st(lambda p: pad(p[0]['last_desc'], mcap))), mv=dev(st(lambda p: pad(p[0]['kf_valid'], mcap))), mn_=dev(np.array([nmp, nmp], np.int32)),
              matched=dev(st(lambda p: np.concatenate([p[3], np.full(kcap - ncur, -1, np.int32)]))))
    bi = torch.zeros((2, mcap), dtype=torch.int32, device='cuda'); bd = torch.zeros((2, mcap), dtype=torch.int32, device='cuda'); nm = torch.zeros(2, dtype=torch.int32, device='cuda')
    a = B.FuseBatch()
    a.cam = B.make_camera(640, 480, per[0][0]['cam'], per[0][0]['sf'])
    a.kf_kps, a.kf_desc, a.kf_uright, a.kf_n, a.kf_cap = t_['kps'].data_ptr(), t_['kd'].data_ptr(), t_['ur'].data_ptr(), t_['kn'].data_ptr(), kcap
    a.tcw, a.ow, a.mp_xyz, a.mp_normal, a.mp_min_dist, a.mp_max_dist = t_['T'].data_ptr(), t_['ow'].data_ptr(), t_['xyz'].data_ptr(), t_['nrm'].data_ptr(), t_['mn'].data_ptr(), t_['mx'].data_ptr()
    a.mp_desc, a.mp_valid, a.mp_n, a.mp_cap, a.th = t_['md'].data_ptr(), t_['mv'].data_ptr(), t_['mn_'].data_ptr(), mcap, float(th)
    a.sim3_variant = 3
    a.best_idx, a.best_dist, a.kf_matched, a.nmatches = bi.data_ptr(), bd.data_ptr(), t_['matched'].data_ptr(), nm.data_ptr()
    B.check(B.lib().sgs_fuse_search_batch_device(C.byref(a), 2, C.c_void_p(0)))
    torch.cuda.synchronize()
    got = t_['matched'].cpu().numpy(); bi_h = bi.cpu().numpy()
    for k, (s, Ow, nrm, matched, nm_o, m_o) in enumerate(per):
        assert int(nm[k].item()) == nm_o
        assert np.array_equal(got[k, :ncur], m_o) and (got[k, ncur:] == -1).all()
        claimed = np.nonzero((matched < 0) & (m_o >= 0))[0]
        assert np.array_equal(np.sort(bi_h[k, m_o[claimed]]), np.sort(claimed))             # best_idx[i] = the feature point i claimed
        assert (bi_h[k, :nmp] >= 0).sum() == nm_o
        # the host entry point on the same key frame
        fg = B.HostFrame(s['kps'], s['uright'], s['desc'], 640, 480, s['cam']['fx'], s['cam']['fy'], s['cam']['cx'], s['cam']['cy'], s['cam']['bf'], s['sf'])
        km = matched.astype(np.int32).copy()
        nm_h, bi_1, _ = _fuse_search_host(fg, s['Tcw_cur'], Ow, s, nrm, float(th), None, 3, None, km)
        assert nm_h == nm_o and np.array_equal(km, m_o) and np.array_equal(bi_1, bi_h[k, :nmp])
    a.kf_matched = None
    with pytest.raises(B.SgsError):
        B.check(B.lib().sgs_fuse_search_batch_device(C.byref(a), 2, C.c_void_p(0)))


@pytest.mark.parametrize('window,ori', [(100, True), (100, False), (40, True)])
def test_search_for_initialization(window, ori):
    """ORBmatcher::SearchForInitialization (src/ORBmatcher.cc:407-522): order-dependent distance book-keeping, two pairs per call + the host entry point."""
    import ctypes as C
    import torch
    from test_match_init import init_scenario
    sc = [init_scenario(seed) for seed in (1, 2)]
    ref = [O.search_for_initialization(s['f1'], s['f2'], s['prev'], window, 0.9, ori) for s in sc]
    assert all(r[0] > 40 for r in ref)
    n1, n2 = len(sc[0]['k1']), len(sc[0]['k2'])
    c1, c2 = n1 + 7, n2 + 5
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    pad = lambda a, cap: np.concatenate([a, np.zeros((cap - len(a),) + a.shape[1:], a.dtype)])
    t_ = dict(k1=dev(np.stack([pad(s['k1'], c1) for s in sc]).view(np.uint8).reshape(-1)), d1=dev(np.stack([pad(s['d1'], c1) for s in sc])),
              k2=dev(np.stack([pad(s['k2'], c2) for s in sc]).view(np.uint8).reshape(-1)), d2=dev(np.stack([pad(s['d2'], c2) for s in sc])),
              n1=dev(np.array([n1, n1], np.int32)), n2=dev(np.array([n2, n2], np.int32)), prev=dev(np.stack([pad(s['prev'], c1) for s in sc])))
    m = torch.zeros((2, c1), dtype=torch.int32, device='cuda'); nm = torch.zeros(2, dtype=torch.int32, device='cuda')
    a = B.InitBatch()
    a.cam = B.make_camera(640, 480, sc[0]['cam'], sc[0]['sf'])
    a.f1_kps, a.f1_desc, a.f1_n, a.f1_cap = t_['k1'].data_ptr(), t_['d1'].data_ptr(), t_['n1'].data_ptr(), c1
    a.f2_kps, a.f2_desc, a.f2_n, a.f2_cap = t_['k2'].data_ptr(), t_['d2'].data_ptr(), t_['n2'].data_ptr(), c2
    a.prev_xy, a.window_size, a.nnratio, a.check_orientation, a.match12, a.nmatches = t_['prev'].data_ptr(), window, 0.9, int(ori), m.data_ptr(), nm.data_ptr()
    B.check(B.lib().sgs_search_for_initialization_batch_device(C.byref(a), 2, C.c_void_p(0)))
    torch.cuda.synchronize()
    mh = m.cpu().numpy(); ph = t_['prev'].cpu().numpy()
    for k, (nm_o, m_o, p_o) in enumerate(ref):
        assert int(nm[k].item()) == nm_o and np.array_equal(mh[k, :n1], m_o) and (mh[k, n1:] == -1).all()
        assert np.array_equal(ph[k, :n1], p_o)
    # host entry point on the first pair
    s = sc[0]
    sf = np.ascontiguousarray(s['sf'], np.float32)
    def view(k, d):
        v = B.FrameView(); v.n = len(k); v.keys_un = k.ctypes.data; v.u_right = None; v.desc = d.ctypes.data
        v.min_x, v.min_y, v.max_x, v.max_y = 0.0, 0.0, 640.0, 480.0
        v.nlevels = 8; v.scale_factors = sf.ctypes.data
        return v
    k1 = np.ascontiguousarray(s['k1']); k2 = np.ascontiguousarray(s['k2']); d1 = np.ascontiguousarray(s['d1']); d2 = np.ascontiguousarray(s['d2'])
    v1, v2 = view(k1, d1), view(k2, d2)
    prev = s['prev'].copy(); mo = np.zeros(n1, np.int32); nmo = C.c_int()
    B.check(B.lib().sgs_search_for_initialization(C.byref(v1), C.byref(v2), prev.ctypes.data_as(C.c_void_p), window, 0.9, int(ori), mo.ctypes.data_as(C.c_void_p), C.byref(nmo), 0))
    assert nmo.value == ref[0][0] and np.array_equal(mo, ref[0][1]) and np.array_equal(prev, ref[0][2])


def test_distinctive_descriptor_batch():
    """MapPoint::ComputeDistinctiveDescriptors (src/MapPoint.cc:242-307): median-of-distances representative, first minimum wins."""
    import ctypes as C
    import torch
    rs = np.random.RandomState(8)
    P, cap = 3000, 64
    counts = rs.randint(0, 65, P).astype(np.int32); counts[:6] = [0, 1, 2, 3, 64, 33]
    desc = np.zeros((P, cap, 32), np.uint8)
    for p in range(P):
        base = rs.randint(0, 2, 256).astype(np.uint8)
        for i in range(counts[p]):
            b = base.copy(); b[rs.choice(256, rs.randint(0, 60), replace=False)] ^= 1
            desc[p, i] = np.packbits(b)
        if counts[p] >= 4 and p % 5 == 0:
            desc[p, 2] = desc[p, 1]                                   # exact duplicates: ties between rows
    dd = torch.from_numpy(desc).cuda(); dc = torch.from_numpy(counts).cuda(); out = torch.full((P,), -3, dtype=torch.int32, device='cuda')
    v = C.c_void_p
    B.check(B.lib().sgs_distinctive_descriptor_batch_device(v(dd.data_ptr()), v(dc.data_ptr()), cap, P, v(out.data_ptr()), v(0)))
    torch.cuda.synchronize()
    got = out.cpu().numpy()
    for p in range(P):
        assert got[p] == O.distinctive_descriptor(desc[p, :counts[p]]), (p, counts[p])
