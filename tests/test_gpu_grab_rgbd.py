"""RGB-D frames as the camera delivers them (Tracking::GrabImageRGBD + the RGB-D Frame constructor + TrackWithMotionModel's matcher call):
  - sgs_grab_rgbd_batch_device bit for bit against the numpy restatement (tests/grab_ref.py, itself pinned against cv2) and the committed cv2 fixture;
  - sgs_tracker_step_rgbd_device with k1 = 0 against the existing entry points called one by one on host-converted inputs, and
    sgs_tracker_step_rgbd (host buffers) against the device step;
  - with TUM1.yaml's distortion: mvKeysUn, mvuRight, mvDepth, the matches and the following pose chain against their pinned pieces;
  - the argument checks."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import detector_model as DM  # noqa: E402
import grab_ref as GR  # noqa: E402
import oracle as O  # noqa: E402
from pysgs import binding as B  # noqa: E402
from pysgs import synth  # noqa: E402

W, H, NF, TH = 640, 480, 1000, 15.0
v = C.c_void_p
P = lambda a: a.ctypes.data_as(v)
TUM1 = dict(fx=517.306408, fy=516.469215, cx=318.643040, cy=255.313989, bf=40.0)
TUM1_DIST = (0.262383, -0.953104, -0.005358, 0.002628, 1.163314)


def fmt_of(rgb, depth_type, factor, dist=(0, 0, 0, 0, 0)):
    f = B.RgbdFormat(rgb, depth_type, factor)
    for i, d in enumerate(dist):
        f.dist_coef[i] = d
    return f


def dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8) if a.dtype.fields else a).cuda()


def grab(d_rgb, rgb_stride, rgb_pitch, d_depth, d_stride, d_pitch, fmt, w, h, nf, gray_pitch, depth_pitch_f):
    """Runs the conversion into padded output frames filled with a sentinel; returns (gray [F,h,w], depth [F,h,w]) and checks the padding."""
    import torch
    gs, ds = gray_pitch * h + 5, depth_pitch_f * h + 3
    g = torch.full((nf * gs,), 0xA5, dtype=torch.uint8, device='cuda')
    d = torch.full((nf * ds,), -7.0, dtype=torch.float32, device='cuda')
    B.check(B.lib().sgs_grab_rgbd_batch_device(d_rgb, rgb_stride, rgb_pitch, d_depth, d_stride, d_pitch, C.byref(fmt), w, h, nf, g.data_ptr(), gs, gray_pitch,
                                               d.data_ptr(), ds * 4, depth_pitch_f * 4, v(0)))
    torch.cuda.synchronize()
    g, d = g.cpu().numpy(), d.cpu().numpy()
    gf = np.stack([g[f * gs: f * gs + h * gray_pitch].reshape(h, gray_pitch) for f in range(nf)])
    df = np.stack([d[f * ds: f * ds + h * depth_pitch_f].reshape(h, depth_pitch_f) for f in range(nf)])
    assert (gf[:, :, w:] == 0xA5).all() and (df[:, :, w:] == -7.0).all(), 'writes past the row'
    assert all((g[f * gs + h * gray_pitch:(f + 1) * gs] == 0xA5).all() and (d[f * ds + h * depth_pitch_f:(f + 1) * ds] == -7.0).all() for f in range(nf))
    return gf[:, :, :w], df[:, :, :w]


@pytest.mark.parametrize('rgb_order', [1, 0])
def test_grab_every_triple(rgb_order):
    img = GR.all_triples()
    raw = np.arange(1 << 24, dtype=np.uint32).astype(np.uint16).reshape(4096, 4096)
    d_img, d_raw, d_f = dev(img), dev(raw), dev(raw.astype(np.float32) * np.float32(0.001))
    for depth_type, d_in, pitch, host in ((0, d_raw, 4096 * 2, raw), (1, d_f, 4096 * 4, raw.astype(np.float32) * np.float32(0.001))):
        for factor in (GR.FACTORS[0], np.float32(1.0)):
            g, d = grab(d_img.data_ptr(), 4096 * 4096 * 3, 4096 * 3, d_in.data_ptr(), pitch * 4096, pitch, fmt_of(rgb_order, depth_type, factor), 4096, 4096, 1,
                        4096 + 16, 4096 + 4)
            assert np.array_equal(g[0], GR.to_gray(img, rgb_order))
            assert d[0].tobytes() == GR.to_depth(host, factor).tobytes(), (depth_type, factor)


def test_grab_fixture_batches(golden_dir):
    z = np.load(os.path.join(golden_dir, 'grab_rgbd.npz'))
    for k in range(int(z['ncases'])):
        w, h, nf, dt, rp, rs, dp, ds = (int(x) for x in z['c%d_meta' % k])
        d_rgb, d_depth = dev(z['c%d_rgb' % k]), dev(z['c%d_depth' % k])
        for rgb_order, key in ((1, 'gray_rgb'), (0, 'gray_bgr')):
            for j, fac in enumerate(z['factors']):
                g, d = grab(d_rgb.data_ptr(), rs, rp, d_depth.data_ptr(), ds, dp, fmt_of(rgb_order, dt, fac), w, h, nf, w + 3, w + 1)
                assert np.array_equal(g, z['c%d_%s' % (k, key)]), (k, key)
                assert d.tobytes() == z['c%d_depth_f%d' % (k, j)].tobytes(), (k, j)


# ---- the step ------------------------------------------------------------------------------------------------------------------------------
NB = 6
PIDX = np.array([0, 0, 1, 2, 3, 4], np.int32)


@pytest.fixture(scope='module')
def scene(tmp_path_factory):
    """Colour S2 frames (blended with the synthetic detector's scenes, so that the mini SSD graph fires on the person class), TUM-style raw depth,
    and the last-frame inputs built from a first extraction of the restated gray frames."""
    import bench
    rgb, depth, gt = synth.stream_s2_rgbd(NB, W, H, seed=5)
    rgb = np.ascontiguousarray(np.stack([(DM.synthetic_rgb(H, W, 10 + i).astype(np.float32) * 0.25 + rgb[i] * 0.75).astype(np.uint8) for i in range(NB)]))
    pp, bp = DM.write_mini_model(str(tmp_path_factory.mktemp('det')), 0)
    gray = GR.to_gray(rgb, 1)
    sf = synth.scale_factors()
    trk = B.Tracker(W, H, B.make_camera(W, H, synth.TUM3, sf), NF, 1.2, 8, 20, 7, max_batch=NB, point_cap=NF + 64, max_boxes=4, device=0)
    cap = trk.cap
    kps = np.zeros((NB, cap), B.KP_DTYPE); desc = np.zeros((NB, cap, 32), np.uint8); n = np.zeros(NB, np.int32)
    B.check(B.lib().sgs_tracker_extract(trk.h, P(gray), NB, W * H, W, P(kps), P(desc), cap, P(n)))
    trk.close()
    ti = bench.make_track_inputs(kps, desc, n, gt, cap, NF + 64, PIDX, W, H, dict(synth.TUM3))
    return dict(rgb=rgb, depth=depth, gray=gray, ti=ti, pp=pp, bp=bp, sf=sf)


def last_args(d):
    return [d[k].data_ptr() for k in ('lxyz', 'ldesc', 'lflags', 'loct', 'lang', 'ln', 'T', 'T')]


def dev_inputs(sc):
    return {k: dev(sc['ti'][k]) for k in ('lxyz', 'ldesc', 'lflags', 'loct', 'lang', 'ln', 'T', 'pidx')}


def results(trk, nb):
    """The tracker's device results after a step / track call, on the host."""
    L, cap = B.lib(), trk.cap
    k, d, u, c, m, nm, nc = (v() for _ in range(7))
    B.check(L.sgs_tracker_results_device(trk.h, C.byref(k), C.byref(d), C.byref(u), C.byref(c), C.byref(m), C.byref(nm), C.byref(nc)))
    bx, nbx, hv = v(), v(), v()
    B.check(L.sgs_tracker_boxes_device(trk.h, C.byref(bx), C.byref(nbx), C.byref(hv)))
    r = dict(kps=np.zeros((nb, cap), B.KP_DTYPE), desc=np.zeros((nb, cap, 32), np.uint8), ur=np.zeros((nb, cap), np.float32), cnt=np.zeros(nb, np.int32),
             mp=np.zeros((nb, cap), np.int32), nm=np.zeros(nb, np.int32), boxes=np.zeros((nb, trk.max_boxes, 4), np.float32), nb=np.zeros(nb, np.int32),
             have=np.zeros(nb, np.uint8))
    for key, p in (('kps', k), ('desc', d), ('ur', u), ('cnt', c), ('mp', m), ('nm', nm), ('boxes', bx), ('nb', nbx), ('have', hv)):
        B.memcpy_d2h(r[key], p.value)
    return r


def frame_results(trk, nb):
    ku, dz = v(), v()
    B.check(B.lib().sgs_tracker_frame_device(trk.h, C.byref(ku), C.byref(dz)))
    return B.memcpy_d2h(np.zeros((nb, trk.cap), B.KP_DTYPE), ku.value), B.memcpy_d2h(np.zeros((nb, trk.cap), np.float32), dz.value)


def assert_same(a, b, keys=('cnt', 'nm', 'nb', 'have')):
    for k in keys:
        assert np.array_equal(a[k], b[k]), k
    for f in range(len(a['cnt'])):
        c, nbx = a['cnt'][f], a['nb'][f]
        assert a['kps'][f, :c].tobytes() == b['kps'][f, :c].tobytes() and np.array_equal(a['desc'][f, :c], b['desc'][f, :c]), f
        assert np.array_equal(a['mp'][f, :c], b['mp'][f, :c]) and a['ur'][f, :c].tobytes() == b['ur'][f, :c].tobytes(), f
        assert a['boxes'][f, :nbx].tobytes() == b['boxes'][f, :nbx].tobytes(), f


def test_step_rgbd_equals_the_stages_one_by_one_and_the_host_step(scene):
    import torch
    L = B.lib()
    sc = scene
    cam = B.make_camera(W, H, synth.TUM3, sc['sf'])
    trk = B.Tracker(W, H, cam, NF, 1.2, 8, 20, 7, max_batch=NB, point_cap=NF + 64, max_boxes=4, device=0)
    det = B.Detector(sc['pp'], sc['bp'], max_frames=NB, det_thr=0.9, dyn_thr=0.01)
    d = dev_inputs(sc)
    d_rgb, d_depth = dev(sc['rgb']), dev(sc['depth'])
    factor = np.float32(1 / 5000)
    # 1. one by one: extract on the restated gray, the detector into the tracker's arrays, LK, F, depth lookup on the float depth, track
    d_gray = dev(sc['gray']); d_depthf = dev(GR.to_depth(sc['depth'], factor))
    B.check(L.sgs_tracker_extract_device(trk.h, d_gray.data_ptr(), NB, W * H, W, v(0)))
    B.check(L.sgs_tracker_detect_device(trk.h, det.h, d_rgb.data_ptr(), H * W * 3, W * 3, W, H, NB, v(0)))
    torch.cuda.synchronize()
    B.check(L.sgs_tracker_lk_device(trk.h, d_gray.data_ptr(), NB, W * H, W, d['pidx'].data_ptr(), v(0)))
    B.check(L.sgs_tracker_fundamental_device(trk.h, NB, None, None, None, d['pidx'].data_ptr(), v(0)))
    B.check(L.sgs_tracker_stereo_device(trk.h, NB, d_depthf.data_ptr(), W * H, W, v(0)))
    B.check(L.sgs_tracker_track_device(trk.h, NB, None, None, None, None, None, None, *last_args(d), TH, 0, 1, v(0)))
    torch.cuda.synchronize()
    r1 = results(trk, NB)
    assert r1['nb'].sum() > 0, 'the synthetic detector must produce person boxes for this test to mean something'
    # 2. the device step on colour + raw uint16 depth
    fmt = fmt_of(1, B.DEPTH_U16, factor)
    B.check(L.sgs_tracker_step_rgbd_device(trk.h, det.h, d_rgb.data_ptr(), H * W * 3, W * 3, d_depth.data_ptr(), H * W * 2, W * 2, C.byref(fmt), NB,
                                           d['pidx'].data_ptr(), *last_args(d), TH, 0, 1, v(0)))
    torch.cuda.synchronize()
    r2 = results(trk, NB)
    assert_same(r1, r2)
    kun, dz = frame_results(trk, NB)
    for f in range(NB):
        c = r2['cnt'][f]
        assert kun[f, :c].tobytes() == r2['kps'][f, :c].tobytes(), 'k1 = 0: mvKeysUn = mvKeys'
        k = r2['kps'][f, :c]
        z = GR.to_depth(sc['depth'][f], factor)[k['y'].astype(np.int64), k['x'].astype(np.int64)]
        assert np.array_equal(dz[f, :c], np.where(z > 0, z, np.float32(-1))), f
    # 3. the host step (float32 depth in a padded layout this time: same metres, read in place with factor 1) equals the device step
    ti = sc['ti']
    dpitch = W * 4 + 64
    hd = np.zeros((NB, H, dpitch // 4), np.float32); hd[:, :, :W] = GR.to_depth(sc['depth'], factor)
    o = dict(kps=np.zeros((NB, trk.cap), B.KP_DTYPE), desc=np.zeros((NB, trk.cap, 32), np.uint8), ur=np.zeros((NB, trk.cap), np.float32), cnt=np.zeros(NB, np.int32),
             mp=np.zeros((NB, trk.cap), np.int32), nm=np.zeros(NB, np.int32), boxes=np.zeros((NB, 4, 4), np.float32), nb=np.zeros(NB, np.int32), have=np.zeros(NB, np.uint8))
    kun3 = np.zeros((NB, trk.cap), B.KP_DTYPE); dz3 = np.zeros((NB, trk.cap), np.float32)
    fmt_f = fmt_of(1, B.DEPTH_F32, 1.0)
    B.check(L.sgs_tracker_step_rgbd(trk.h, det.h, P(sc['rgb']), H * W * 3, W * 3, P(hd), H * dpitch, dpitch, C.byref(fmt_f), NB, P(ti['pidx']), P(ti['lxyz']),
                                    P(ti['ldesc']), P(ti['lflags']), P(ti['loct']), P(ti['lang']), P(ti['ln']), P(ti['T']), P(ti['T']), TH, 0, 1,
                                    *[P(o[k]) for k in ('kps', 'desc', 'ur', 'cnt', 'mp', 'nm', 'boxes', 'nb', 'have')], P(kun3), P(dz3)))
    assert_same(r2, o)
    for f in range(NB):
        c = o['cnt'][f]
        assert kun3[f, :c].tobytes() == kun[f, :c].tobytes() and dz3[f, :c].tobytes() == dz[f, :c].tobytes(), f
    trk.close(); det.close()


def test_step_rgbd_with_distortion(scene):
    """TUM1.yaml: the step's mvKeysUn / mvuRight / mvDepth / matches equal their pinned pieces on the compacted keypoints, and the pose chain after it
    equals the oracle composition of tests/test_gpu_pose_chain.py on the undistorted frame."""
    import bench
    import torch
    from test_gpu_pose_chain import oracle_chain
    L = B.lib()
    sc, ti, sf = scene, scene['ti'], scene['sf']
    dist = np.array(TUM1_DIST, np.float32)
    bounds = np.zeros(4, np.float32)
    B.check(L.sgs_image_bounds(W, H, TUM1['fx'], TUM1['fy'], TUM1['cx'], TUM1['cy'], P(dist), P(bounds), 0))
    cam = B.make_camera(W, H, TUM1, sf)
    cam.min_x, cam.min_y, cam.max_x, cam.max_y = (float(b) for b in bounds)
    trk = B.Tracker(W, H, cam, NF, 1.2, 8, 20, 7, max_batch=NB, point_cap=NF + 64, max_boxes=4, device=0)
    det = B.Detector(sc['pp'], sc['bp'], max_frames=NB, det_thr=0.9, dyn_thr=0.01)
    cap = trk.cap
    d = dev_inputs(sc)
    factor = np.float32(1 / 5000)
    d_rgb, d_depth, d_depthf = dev(sc['rgb']), dev(sc['depth']), dev(GR.to_depth(sc['depth'], factor))
    fmt = fmt_of(1, B.DEPTH_U16, factor, TUM1_DIST)
    B.check(L.sgs_tracker_step_rgbd_device(trk.h, det.h, d_rgb.data_ptr(), H * W * 3, W * 3, d_depth.data_ptr(), H * W * 2, W * 2, C.byref(fmt), NB,
                                           d['pidx'].data_ptr(), *last_args(d), TH, 0, 1, v(0)))
    torch.cuda.synchronize()
    r = results(trk, NB)
    kun, dz = frame_results(trk, NB)
    # mvKeysUn, mvuRight, mvDepth from the pinned per-point entry points applied to the compacted keypoints
    kp_d, cnt_d = dev(r['kps']), dev(r['cnt'])
    kun_ref = torch.zeros((NB, cap * 28), dtype=torch.uint8, device='cuda')
    ur_ref = torch.zeros((NB, cap), dtype=torch.float32, device='cuda'); dz_ref = torch.zeros((NB, cap), dtype=torch.float32, device='cuda')
    B.check(L.sgs_undistort_batch_device(kp_d.data_ptr(), cnt_d.data_ptr(), cap, NB, TUM1['fx'], TUM1['fy'], TUM1['cx'], TUM1['cy'], P(dist), kun_ref.data_ptr(), v(0)))
    B.check(L.sgs_stereo_from_depth_batch_device(kp_d.data_ptr(), kun_ref.data_ptr(), cnt_d.data_ptr(), cap, NB, d_depthf.data_ptr(), W * H, W, TUM1['bf'],
                                                 ur_ref.data_ptr(), dz_ref.data_ptr(), v(0)))
    torch.cuda.synchronize()
    kun_ref = kun_ref.cpu().numpy().view(B.KP_DTYPE).reshape(NB, cap); ur_ref = ur_ref.cpu().numpy(); dz_ref = dz_ref.cpu().numpy()
    moved = 0
    for f in range(NB):
        c = r['cnt'][f]
        assert kun[f, :c].tobytes() == kun_ref[f, :c].tobytes(), f
        assert r['ur'][f, :c].tobytes() == ur_ref[f, :c].tobytes() and dz[f, :c].tobytes() == dz_ref[f, :c].tobytes(), f
        moved += int((kun[f, :c]['x'] != r['kps'][f, :c]['x']).sum())
        # SearchByProjection(cur, last) on the frame view built from mvKeysUn
        fr = B.HostFrame(kun[f, :c], r['ur'][f, :c], r['desc'][f, :c], W, H, TUM1['fx'], TUM1['fy'], TUM1['cx'], TUM1['cy'], TUM1['bf'], sf)
        fr.c.min_x, fr.c.min_y, fr.c.max_x, fr.c.max_y = cam.min_x, cam.min_y, cam.max_x, cam.max_y
        m = int(ti['ln'][f]); fl = ti['lflags'][f, :m]
        nm, mp = B.match_project_lastframe(fr, ti['T'][f].reshape(4, 4), ti['T'][f].reshape(4, 4), fl & 1, ti['lxyz'][f, :m], ti['ldesc'][f, :m], (fl >> 1) & 1,
                                           ti['loct'][f, :m], ti['lang'][f, :m], TH)
        assert nm == r['nm'][f] and np.array_equal(mp, r['mp'][f, :c]), f
    assert moved > 0.9 * r['cnt'].sum(), 'the distortion must move the keypoints'
    # the pose chain after the RGB-D step reads mvKeysUn
    mcap = 1536
    rng = np.random.default_rng(5)
    lms = [bench.make_local_map(f, kun[f], r['desc'][f], int(r['cnt'][f]), ti, mcap, TUM1, sf, rng, W, H) for f in range(NB)]
    stack = lambda k, dt: np.ascontiguousarray(np.stack([m[k] for m in lms]).astype(dt))
    lm = {k: dev(a) for k, a in dict(lid=stack('lid', np.int32), xyz=stack('xyz', np.float32), nrm=stack('nrm', np.float32), mn=stack('mn', np.float32),
                                      mx=stack('mx', np.float32), dsc=stack('dsc', np.uint8), valid=stack('valid', np.uint8), obs=stack('obs', np.uint8),
                                      n=np.array([m['n'] for m in lms], np.int32)).items()}
    outd = dict(T1=torch.zeros((NB, 16), device='cuda'), T2=torch.zeros((NB, 16), device='cuda'), mp=torch.zeros((NB, cap), dtype=torch.int32, device='cuda'),
                outl=torch.zeros((NB, cap), dtype=torch.uint8, device='cuda'), st=torch.zeros((NB, 8), dtype=torch.int32, device='cuda'))
    isig = np.zeros(16, np.float32); isig[:8] = 1.0 / (sf.astype(np.float32) ** 2)
    a = B.PoseChainBatch()
    a.last_xyz, a.last_desc, a.last_flags, a.last_octave, a.last_angle, a.last_n, a.tcw_cur, a.tcw_last = last_args(d)
    a.th, a.mono, a.check_orientation, a.last_local_id = TH, 0, 1, lm['lid'].data_ptr()
    a.mp_xyz, a.mp_normal, a.mp_min_dist, a.mp_max_dist = lm['xyz'].data_ptr(), lm['nrm'].data_ptr(), lm['mn'].data_ptr(), lm['mx'].data_ptr()
    a.mp_desc, a.mp_valid, a.mp_obs, a.mp_n, a.mp_cap = lm['dsc'].data_ptr(), lm['valid'].data_ptr(), lm['obs'].data_ptr(), lm['n'].data_ptr(), mcap
    a.th_local, a.nnratio_local = 3.0, 0.8
    for l in range(16):
        a.inv_level_sigma2[l] = float(isig[l])
    a.tcw_motion, a.tcw_final, a.f_mp, a.outlier, a.stats = outd['T1'].data_ptr(), outd['T2'].data_ptr(), outd['mp'].data_ptr(), outd['outl'].data_ptr(), outd['st'].data_ptr()
    B.check(L.sgs_tracker_pose_chain_device(trk.h, C.byref(a), NB, v(0)))
    torch.cuda.synchronize()
    g = {k: t.cpu().numpy() for k, t in outd.items()}
    camv = np.array([TUM1['fx'], TUM1['fy'], TUM1['cx'], TUM1['cy'], TUM1['bf'], cam.min_x, cam.min_y, cam.max_x, cam.max_y], np.float32)
    tid = dict(ti, Tc=ti['T'])
    for f in range(NB):
        c = int(r['cnt'][f])
        cur = O.FrameArrays(kun[f, :c], r['ur'][f, :c], r['desc'][f, :c], W, H, TUM1['fx'], TUM1['fy'], TUM1['cx'], TUM1['cy'], TUM1['bf'], sf)
        cur.c.minX, cur.c.minY, cur.c.maxX, cur.c.maxY = cam.min_x, cam.min_y, cam.max_x, cam.max_y
        o = oracle_chain(f, cur, int(r['nm'][f]), r['mp'][f, :c].copy(), tid, lms[f], camv, TUM1, sf, isig, TH, tcw_motion_gpu=g['T1'][f])
        assert np.array_equal(g['st'][f], o['stats']), (f, g['st'][f], o['stats'])
        assert np.array_equal(g['mp'][f, :c], o['mp']) and np.array_equal(g['outl'][f, :c], o['outlier']), f
        assert np.abs(g['T1'][f].reshape(4, 4) - o['T1']).max() <= 1e-5 and np.abs(g['T2'][f].reshape(4, 4) - o['T2']).max() <= 1e-5, f
    trk.close(); det.close()


def test_invalid_arguments_are_refused_before_anything_runs(scene):
    import torch
    L = B.lib()
    sc, ti = scene, scene['ti']
    trk = B.Tracker(W, H, B.make_camera(W, H, synth.TUM3, sc['sf']), NF, 1.2, 8, 20, 7, max_batch=NB, point_cap=NF + 64, max_boxes=4, device=0)
    det = B.Detector(sc['pp'], sc['bp'], max_frames=NB, det_thr=0.9, dyn_thr=0.01)
    d = dev_inputs(sc)
    d_rgb, d_depth = dev(sc['rgb']), dev(sc['depth'])
    g_out, z_out = torch.zeros(W * H, dtype=torch.uint8, device='cuda'), torch.zeros(W * H, dtype=torch.float32, device='cuda')
    cap = trk.cap
    outs = [np.zeros((NB, cap), B.KP_DTYPE), np.zeros((NB, cap, 32), np.uint8), np.zeros((NB, cap), np.float32), np.zeros(NB, np.int32),
            np.zeros((NB, cap), np.int32), np.zeros(NB, np.int32)]
    ok = dict(rgb_stride=H * W * 3, rgb_pitch=W * 3, depth_stride=H * W * 2, depth_pitch=W * 2, fmt=fmt_of(1, 0, 1 / 5000), nframes=NB, pidx=PIDX)
    cases = [dict(nframes=0), dict(nframes=NB + 1), dict(pidx=np.array([0, 0, 1, 2, 3, 6], np.int32)), dict(pidx=np.array([-1, 0, 1, 2, 3, 4], np.int32)),
             dict(rgb_pitch=W * 3 - 1), dict(rgb_stride=H * W * 3 - 1), dict(depth_pitch=W * 2 - 2), dict(depth_stride=H * W * 2 - 2), dict(depth_pitch=W * 2 + 1, depth_stride=H * (W * 2 + 1)),
             dict(fmt=fmt_of(1, 2, 1 / 5000)), dict(fmt=fmt_of(1, -1, 1 / 5000)), dict(fmt=fmt_of(1, 0, 0.0)), dict(fmt=fmt_of(1, 0, -1.0)),
             dict(fmt=fmt_of(1, 0, float('nan'))), dict(fmt=fmt_of(1, 0, float('inf')))]
    for case in cases:
        a = dict(ok, **case)
        rc = L.sgs_tracker_step_rgbd(trk.h, det.h, P(sc['rgb']), a['rgb_stride'], a['rgb_pitch'], P(sc['depth']), a['depth_stride'], a['depth_pitch'], C.byref(a['fmt']),
                                     a['nframes'], P(np.ascontiguousarray(a['pidx'])), P(ti['lxyz']), P(ti['ldesc']), P(ti['lflags']), P(ti['loct']), P(ti['lang']),
                                     P(ti['ln']), P(ti['T']), P(ti['T']), TH, 0, 1, *[P(x) for x in outs], None, None, None, None, None)
        assert rc == B.SGS_ERR_INVALID, case
        if 'pidx' not in case:
            rc = L.sgs_tracker_step_rgbd_device(trk.h, det.h, d_rgb.data_ptr(), a['rgb_stride'], a['rgb_pitch'], d_depth.data_ptr(), a['depth_stride'], a['depth_pitch'],
                                                C.byref(a['fmt']), a['nframes'], d['pidx'].data_ptr(), *last_args(d), TH, 0, 1, v(0))
            assert rc == B.SGS_ERR_INVALID, case
        if set(case) <= {'rgb_pitch', 'rgb_stride', 'depth_pitch', 'depth_stride', 'fmt'}:
            rc = L.sgs_grab_rgbd_batch_device(d_rgb.data_ptr(), a['rgb_stride'], a['rgb_pitch'], d_depth.data_ptr(), a['depth_stride'], a['depth_pitch'], C.byref(a['fmt']),
                                              W, H, 1, g_out.data_ptr(), W * H, W, z_out.data_ptr(), W * H * 4, W * 4, v(0))
            assert rc == B.SGS_ERR_INVALID, case
    rc = L.sgs_tracker_frame_device(trk.h, None, None)
    assert rc == B.SGS_ERR_INVALID, 'no RGB-D step has run on this handle'
    trk.close(); det.close()
