"""The whole front end in one call (sgs_tracker_step): Detector2D::detect on its own stream -> person boxes in the tracker's device arrays ->
consumed in stream order by findFundamentalMat (previous-frame boxes) and the dynamic-feature rejection (src/Frame.cc:474-500 joins the detector
thread at the same place).  Checked against the same stages called one by one through the C ABI with the boxes carried over by hand, bit for bit.
The synthetic SSD graph of tests/detector_model.py is used because it does fire on the person class (the trained model sees no people in S2 textures)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import detector_model as DM  # noqa: E402
import scenarios as S  # noqa: E402
from pysgs import binding as B  # noqa: E402
from pysgs import synth  # noqa: E402

W, H, NF, TH = 640, 480, 1000, 15.0


def _inputs(frames, boxes_gt, kps, desc, counts, cap, pcap, pidx):
    import bench
    return bench.make_track_inputs(kps, desc, counts, boxes_gt, cap, pcap, pidx, W, H, dict(synth.TUM3))


def test_step_equals_the_stages_called_one_by_one(tmp_path):
    import sys, os
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    pp, bp = DM.write_mini_model(str(tmp_path), 0)
    nb = 6
    frames, gt = synth.stream_s2(nb, W, H, seed=5)
    rgb = np.stack([DM.synthetic_rgb(H, W, 10 + i) for i in range(nb)])          # colour frames the synthetic detector fires on
    frames = np.ascontiguousarray((rgb.astype(np.float32).mean(3) * 0.25 + frames * 0.75).astype(np.uint8))
    pidx = np.array([0, 0, 1, 2, 3, 4], np.int32)
    sf = S.scale_factors(); cam = B.make_camera(W, H, synth.TUM3, sf)
    trk = B.Tracker(W, H, cam, NF, 1.2, 8, 20, 7, max_batch=nb, point_cap=NF + 64, max_boxes=4, device=0)
    det = B.Detector(pp, bp, max_frames=nb, det_thr=0.9, dyn_thr=0.01)
    cap = trk.cap
    L, v = B.lib(), C.c_void_p
    P = lambda a: a.ctypes.data_as(v)
    # 1. stage by stage: extract (host), detector (host frames one by one -> boxes by hand), track_lk with those boxes
    kps = np.zeros((nb, cap), B.KP_DTYPE); desc = np.zeros((nb, cap, 32), np.uint8); n = np.zeros(nb, np.int32)
    B.check(L.sgs_tracker_extract(trk.h, P(frames), nb, W * H, W, P(kps), P(desc), cap, P(n)))
    ti = _inputs(frames, gt, kps, desc, n, cap, trk.point_cap, pidx)
    import torch
    d_rgb = torch.from_numpy(rgb).cuda()
    d_bx = torch.zeros((nb, 4, 4), device='cuda'); d_nb = torch.zeros(nb, dtype=torch.int32, device='cuda'); d_hv = torch.zeros(nb, dtype=torch.uint8, device='cuda')
    det.detect_device(d_rgb.data_ptr(), H * W * 3, W * 3, W, H, nb, d_dyn_rm=d_bx.data_ptr(), d_ndyn_rm=d_nb.data_ptr(), d_have_dyn_rm=d_hv.data_ptr(), max_boxes=4)
    torch.cuda.synchronize()
    bx, nbx, hv = d_bx.cpu().numpy(), d_nb.cpu().numpy(), d_hv.cpu().numpy()
    assert nbx.sum() > 0, 'the synthetic detector must produce person boxes for this test to mean something'
    o1 = dict(kps=np.zeros((nb, cap), B.KP_DTYPE), desc=np.zeros((nb, cap, 32), np.uint8), ur=np.zeros((nb, cap), np.float32), cnt=np.zeros(nb, np.int32),
              mp=np.zeros((nb, cap), np.int32), nm=np.zeros(nb, np.int32))
    T = ti['T']
    B.check(L.sgs_tracker_track_lk(trk.h, nb, P(pidx), P(ti['ur']), v(0), P(bx), P(nbx), P(hv), P(ti['lxyz']), P(ti['ldesc']), P(ti['lflags']), P(ti['loct']), P(ti['lang']),
                                   P(ti['ln']), P(T), P(T), TH, 0, 1, P(o1['kps']), P(o1['desc']), P(o1['ur']), P(o1['cnt']), P(o1['mp']), P(o1['nm'])))
    # 2. one call
    o2 = {k: np.zeros_like(a) for k, a in o1.items()}
    bo = np.zeros((nb, 4, 4), np.float32); nbo = np.zeros(nb, np.int32); hvo = np.zeros(nb, np.uint8)
    B.check(L.sgs_tracker_step(trk.h, det.h, P(frames), W * H, W, P(rgb), W * H * 3, W * 3, nb, P(pidx), P(ti['ur']), P(ti['lxyz']), P(ti['ldesc']),
                               P(ti['lflags']), P(ti['loct']), P(ti['lang']), P(ti['ln']), P(T), P(T), TH, 0, 1, P(o2['kps']), P(o2['desc']), P(o2['ur']), P(o2['cnt']),
                               P(o2['mp']), P(o2['nm']), P(bo), P(nbo), P(hvo)))
    assert np.array_equal(nbo, nbx) and np.array_equal(hvo, hv)
    for f in range(nb):
        assert bo[f, :nbx[f]].tobytes() == bx[f, :nbx[f]].tobytes()
    assert np.array_equal(o1['cnt'], o2['cnt']) and np.array_equal(o1['nm'], o2['nm'])
    for f in range(nb):
        c = o1['cnt'][f]
        assert o1['kps'][f, :c].tobytes() == o2['kps'][f, :c].tobytes() and np.array_equal(o1['desc'][f, :c], o2['desc'][f, :c])
        assert np.array_equal(o1['mp'][f, :c], o2['mp'][f, :c]) and o1['ur'][f, :c].tobytes() == o2['ur'][f, :c].tobytes()
    # the boxes matter: with the person boxes removed the rejection keeps a different set on at least one frame
    z = np.zeros_like(nbx); zh = np.zeros_like(hv)
    o3 = {k: np.zeros_like(a) for k, a in o1.items()}
    B.check(L.sgs_tracker_track_lk(trk.h, nb, P(pidx), P(ti['ur']), v(0), P(bx), P(z), P(zh), P(ti['lxyz']), P(ti['ldesc']), P(ti['lflags']), P(ti['loct']), P(ti['lang']),
                                   P(ti['ln']), P(T), P(T), TH, 0, 1, P(o3['kps']), P(o3['desc']), P(o3['ur']), P(o3['cnt']), P(o3['mp']), P(o3['nm'])))
    if hv.any():
        assert not np.array_equal(o3['cnt'], o1['cnt'])
    trk.close(); det.close()
