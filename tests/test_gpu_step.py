"""The whole front end in one call (sgs_tracker_step): Detector2D::detect on its own stream -> person boxes in the tracker's device arrays ->
consumed in stream order by findFundamentalMat (previous-frame boxes) and the dynamic-feature rejection (src/Frame.cc:474-500 joins the detector
thread at the same place).  Checked against the same stages called one by one through the C ABI with the boxes carried over by hand, bit for bit.
The host-buffer track entry points (sgs_tracker_track with a host prev_xy and F, sgs_tracker_track_lk with a host F) are checked against
sgs_tracker_track_lk with F on the device, and the argument refusals of the gray-frame host entry points against what they leave behind.
The synthetic SSD graph of tests/detector_model.py is used because it does fire on the person class (the trained model sees no people in S2 textures)."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import detector_model as DM  # noqa: E402
import scenarios as S  # noqa: E402
from pysgs import binding as B  # noqa: E402
from pysgs import synth  # noqa: E402

W, H, NF, TH = 640, 480, 1000, 15.0
NB = 6
v = C.c_void_p
P = lambda a: a.ctypes.data_as(v)
LAST = ('lxyz', 'ldesc', 'lflags', 'loct', 'lang', 'ln', 'T', 'T')      # the eight last-frame arrays, in argument order (tcw_cur, tcw_last)
OUTS = ('kps', 'desc', 'ur', 'cnt', 'mp', 'nm')


@pytest.fixture(scope='module')
def scene(tmp_path_factory):
    """An S2 stream blended with colour frames the synthetic detector fires on, the tracker and detector, the extraction results, the track
    inputs made from them and the detector's boxes read back to the host."""
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    import bench
    import torch
    pp, bp = DM.write_mini_model(str(tmp_path_factory.mktemp('det')), 0)
    frames, gt = synth.stream_s2(NB, W, H, seed=5)
    rgb = np.stack([DM.synthetic_rgb(H, W, 10 + i) for i in range(NB)])          # colour frames the synthetic detector fires on
    frames = np.ascontiguousarray((rgb.astype(np.float32).mean(3) * 0.25 + frames * 0.75).astype(np.uint8))
    pidx = np.array([0, 0, 1, 2, 3, 4], np.int32)
    sf = S.scale_factors(); cam = B.make_camera(W, H, synth.TUM3, sf)
    trk = B.Tracker(W, H, cam, NF, 1.2, 8, 20, 7, max_batch=NB, point_cap=NF + 64, max_boxes=4, device=0)
    det = B.Detector(pp, bp, max_frames=NB, det_thr=0.9, dyn_thr=0.01)
    cap = trk.cap
    kps = np.zeros((NB, cap), B.KP_DTYPE); desc = np.zeros((NB, cap, 32), np.uint8); n = np.zeros(NB, np.int32)
    B.check(B.lib().sgs_tracker_extract(trk.h, P(frames), NB, W * H, W, P(kps), P(desc), cap, P(n)))
    ti = bench.make_track_inputs(kps, desc, n, gt, cap, trk.point_cap, pidx, W, H, dict(synth.TUM3))
    # the detector on the colour frames, boxes carried over to the host by hand
    d_rgb = torch.from_numpy(rgb).cuda()
    d_bx = torch.zeros((NB, 4, 4), device='cuda'); d_nb = torch.zeros(NB, dtype=torch.int32, device='cuda'); d_hv = torch.zeros(NB, dtype=torch.uint8, device='cuda')
    det.detect_device(d_rgb.data_ptr(), H * W * 3, W * 3, W, H, NB, d_dyn_rm=d_bx.data_ptr(), d_ndyn_rm=d_nb.data_ptr(), d_have_dyn_rm=d_hv.data_ptr(), max_boxes=4)
    torch.cuda.synchronize()
    bx, nbx, hv = d_bx.cpu().numpy(), d_nb.cpu().numpy(), d_hv.cpu().numpy()
    assert nbx.sum() > 0, 'the synthetic detector must produce person boxes for the tests to mean something'
    yield dict(trk=trk, det=det, frames=frames, rgb=rgb, pidx=pidx, cap=cap, ti=ti, bx=bx, nbx=nbx, hv=hv)
    trk.close(); det.close()


def _outs(cap):
    return dict(kps=np.zeros((NB, cap), B.KP_DTYPE), desc=np.zeros((NB, cap, 32), np.uint8), ur=np.zeros((NB, cap), np.float32), cnt=np.zeros(NB, np.int32),
                mp=np.zeros((NB, cap), np.int32), nm=np.zeros(NB, np.int32))


def _extract(sc, frames=None):
    cap = sc['cap']
    kps = np.zeros((NB, cap), B.KP_DTYPE); desc = np.zeros((NB, cap, 32), np.uint8); n = np.zeros(NB, np.int32)
    B.check(B.lib().sgs_tracker_extract(sc['trk'].h, P(sc['frames'] if frames is None else frames), NB, W * H, W, P(kps), P(desc), cap, P(n)))


def _track_lk(sc, o, F=None, nboxes=None, have=None, ti=None):
    ti = ti or sc['ti']
    return B.lib().sgs_tracker_track_lk(sc['trk'].h, NB, P(sc['pidx']), P(ti['ur']), None if F is None else P(F), P(ti.get('bx', sc['bx'])),
                                        P(sc['nbx'] if nboxes is None else nboxes), P(sc['hv'] if have is None else have), *[P(ti[k]) for k in LAST],
                                        TH, 0, 1, *[P(o[k]) for k in OUTS])


def _overwrite_then_extract(sc):
    """Leaves other values in every device array a host track call uploads or falls back on, then extracts the scene's frames again: LK and
    the device F of other frames, a host F of ones, zero u_right and boxes, other last-frame points.  A call that skips an upload, reads the
    wrong F or does not wait for its uploads then computes something else."""
    ti = sc['ti']
    other = dict(ti, ur=np.zeros_like(ti['ur']), bx=np.zeros_like(sc['bx']), lxyz=ti['lxyz'] * 2, ldesc=ti['ldesc'] ^ 0xFF)
    _extract(sc, np.ascontiguousarray(sc['frames'][::-1]))
    zn, zh = np.zeros_like(sc['nbx']), np.zeros_like(sc['hv'])
    B.check(_track_lk(sc, _outs(sc['cap']), nboxes=zn, have=zh, ti=other))
    B.check(_track_lk(sc, _outs(sc['cap']), F=np.ones((NB, 9)), nboxes=zn, have=zh, ti=other))
    _extract(sc)


def _assert_same_results(o1, o2, u_right=True):
    assert np.array_equal(o1['cnt'], o2['cnt']) and np.array_equal(o1['nm'], o2['nm'])
    for f in range(NB):
        c = o1['cnt'][f]
        assert o1['kps'][f, :c].tobytes() == o2['kps'][f, :c].tobytes() and np.array_equal(o1['desc'][f, :c], o2['desc'][f, :c])
        assert np.array_equal(o1['mp'][f, :c], o2['mp'][f, :c])
        if u_right:
            assert o1['ur'][f, :c].tobytes() == o2['ur'][f, :c].tobytes()


def test_step_equals_the_stages_called_one_by_one(scene):
    sc = scene
    trk, det, ti, cap, pidx, bx, nbx, hv = sc['trk'], sc['det'], sc['ti'], sc['cap'], sc['pidx'], sc['bx'], sc['nbx'], sc['hv']
    L = B.lib()
    # 1. stage by stage: extract (host), detector (host frames one by one -> boxes by hand), track_lk with those boxes
    _extract(sc)
    o1 = _outs(cap)
    B.check(_track_lk(sc, o1))
    # 2. one call
    o2 = _outs(cap)
    bo = np.zeros((NB, 4, 4), np.float32); nbo = np.zeros(NB, np.int32); hvo = np.zeros(NB, np.uint8)
    T = ti['T']
    B.check(L.sgs_tracker_step(trk.h, det.h, P(sc['frames']), W * H, W, P(sc['rgb']), W * H * 3, W * 3, NB, P(pidx), P(ti['ur']), P(ti['lxyz']), P(ti['ldesc']),
                               P(ti['lflags']), P(ti['loct']), P(ti['lang']), P(ti['ln']), P(T), P(T), TH, 0, 1, P(o2['kps']), P(o2['desc']), P(o2['ur']), P(o2['cnt']),
                               P(o2['mp']), P(o2['nm']), P(bo), P(nbo), P(hvo)))
    assert np.array_equal(nbo, nbx) and np.array_equal(hvo, hv)
    for f in range(NB):
        assert bo[f, :nbx[f]].tobytes() == bx[f, :nbx[f]].tobytes()
    _assert_same_results(o1, o2)
    # the boxes matter: with the person boxes removed the rejection keeps a different set on at least one frame
    o3 = _outs(cap)
    B.check(_track_lk(sc, o3, nboxes=np.zeros_like(nbx), have=np.zeros_like(hv)))
    if hv.any():
        assert not np.array_equal(o3['cnt'], o1['cnt'])


def test_host_track_and_host_F_equal_track_lk_with_F_on_the_device(scene):
    sc = scene
    trk, ti, cap = sc['trk'], sc['ti'], sc['cap']
    L = B.lib()
    _extract(sc)
    o1 = _outs(cap)
    B.check(_track_lk(sc, o1))                 # F == NULL: LK and findFundamentalMat on the device
    pp, pF = v(), v()
    B.check(L.sgs_tracker_prev_xy_device(trk.h, C.byref(pp))); B.check(L.sgs_tracker_fundamental_device_ptr(trk.h, C.byref(pF), None))
    prev = B.memcpy_d2h(np.zeros((NB, cap, 2), np.float32), pp.value); F = B.memcpy_d2h(np.zeros((NB, 9), np.float64), pF.value)
    assert np.isnan(F[0, 0]) and np.isfinite(F[1:, 0]).any(), 'frame 0 has no previous frame; the others must give the host F something to carry'
    # sgs_tracker_track_lk with that F from the host
    _overwrite_then_extract(sc)
    o2 = _outs(cap)
    B.check(_track_lk(sc, o2, F=F))
    _assert_same_results(o1, o2)
    # the host F is what the rejection reads: an empty F (NaN) keeps every keypoint, and the counts move
    _overwrite_then_extract(sc)
    o_nan = _outs(cap)
    B.check(_track_lk(sc, o_nan, F=np.full((NB, 9), np.nan)))
    assert not np.array_equal(o_nan['cnt'], o1['cnt'])
    # sgs_tracker_track with that prev_xy, the host u_right, that F and the boxes
    ptrs = [P(prev), P(ti['ur']), P(F), P(sc['bx']), P(sc['nbx']), P(sc['hv'])] + [P(ti[k]) for k in LAST]
    _overwrite_then_extract(sc)
    o3 = _outs(cap)
    trk.track(NB, ptrs, TH, 0, 1, [P(o3[k]) for k in OUTS])
    _assert_same_results(o1, o3)
    # u_right_out == NULL: the other outputs are written all the same
    _overwrite_then_extract(sc)
    o4 = _outs(cap)
    trk.track(NB, ptrs, TH, 0, 1, [None if k == 'ur' else P(o4[k]) for k in OUTS])
    _assert_same_results(o1, o4, u_right=False)


def _device_results(trk, cap):
    """(device pointers, host copies) of what sgs_tracker_results_device exposes"""
    p = [v() for _ in range(7)]
    B.check(B.lib().sgs_tracker_results_device(trk.h, *[C.byref(x) for x in p]))
    shapes = [((NB, cap), B.KP_DTYPE), ((NB, cap, 32), np.uint8), ((NB, cap), np.float32), (NB, np.int32), ((NB, cap), np.int32), (NB, np.int32), (NB, np.uint64)]
    return [x.value for x in p], [B.memcpy_d2h(np.zeros(s, d), x.value).tobytes() for (s, d), x in zip(shapes, p)]


def test_gray_host_entry_points_refuse_bad_arguments_before_anything_runs(scene):
    sc = scene
    trk, det, ti, cap, pidx = sc['trk'], sc['det'], sc['ti'], sc['cap'], sc['pidx']
    L = B.lib()
    _extract(sc)
    B.check(_track_lk(sc, _outs(cap)))
    before = _device_results(trk, cap)
    o = {'out_' + k: a for k, a in _outs(cap).items()}
    outs = tuple(o)
    ok = dict(nframes=NB, pidx=pidx, prev=np.zeros((NB, cap, 2), np.float32), F=np.zeros((NB, 9), np.float64), rgb_pitch=W * 3, rgb_stride=H * W * 3,
              **{k: ti[k] for k in ('ur', 'lxyz', 'ldesc', 'lflags', 'loct', 'lang', 'ln')}, tc=ti['T'], tl=ti['T'], **o)
    last = ('lxyz', 'ldesc', 'lflags', 'loct', 'lang', 'ln', 'tc', 'tl')
    ptr = lambda a, k: None if a[k] is None else P(a[k])

    def step(a):
        return L.sgs_tracker_step(trk.h, det.h, P(sc['frames']), W * H, W, P(sc['rgb']), a['rgb_stride'], a['rgb_pitch'], a['nframes'], ptr(a, 'pidx'), ptr(a, 'ur'),
                                  *[ptr(a, k) for k in last], TH, 0, 1, *[ptr(a, k) for k in outs], None, None, None)

    def track_lk(a):
        return L.sgs_tracker_track_lk(trk.h, a['nframes'], ptr(a, 'pidx'), ptr(a, 'ur'), None, P(sc['bx']), P(sc['nbx']), P(sc['hv']), *[ptr(a, k) for k in last],
                                      TH, 0, 1, *[ptr(a, k) for k in outs])

    def track(a):
        return L.sgs_tracker_track(trk.h, a['nframes'], ptr(a, 'prev'), ptr(a, 'ur'), ptr(a, 'F'), P(sc['bx']), P(sc['nbx']), P(sc['hv']), *[ptr(a, k) for k in last],
                                   TH, 0, 1, *[ptr(a, k) for k in outs])

    common = [dict(nframes=0), dict(nframes=NB + 1), dict(ur=None)] + [{k: None} for k in last] + [{k: None} for k in outs if k != 'out_ur']
    with_pidx = [dict(pidx=np.array([-1, 0, 1, 2, 3, 4], np.int32)), dict(pidx=np.array([0, 0, 1, 2, 3, NB], np.int32))]
    entries = (('sgs_tracker_step', step, common + with_pidx + [dict(rgb_pitch=W * 3 - 1), dict(rgb_stride=H * W * 3 - 1)]),
               ('sgs_tracker_track_lk', track_lk, common + with_pidx),
               ('sgs_tracker_track', track, common))
    for name, call, cases in entries:
        for case in cases:
            rc = call(dict(ok, **case))
            assert rc == B.SGS_ERR_INVALID, (name, case)
            assert L.sgs_last_error().decode().startswith(name + ':'), (name, case, L.sgs_last_error())
    assert not any(np.frombuffer(a.tobytes(), np.uint8).any() for a in o.values()), 'a refused call writes no output'
    assert _device_results(trk, cap) == before, 'a refused call leaves the results of the last good call'
