#!/usr/bin/env python3
"""Experiment: does splitting the device-resident batch over two tracker handles on two streams (so that the latency-bound kernels of one half
overlap the throughput-bound kernels of the other) raise frames/s?  Prints ms per 512 frames for 1, 2 and 4 handles."""
import ctypes as C
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, 'sg-slam_b200'), os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'tests'), ROOT]
import bench as BN  # noqa: E402
from pysgs import binding as B, synth  # noqa: E402
import scenarios as S  # noqa: E402

W, H, NF, TH = 640, 480, 1000, 15.0
NB = 512
L, v = B.lib(), C.c_void_p
frames, boxes, unique = BN.make_frames(NB, seed=2)
pidx = BN.prev_index(NB, unique)
sf = S.scale_factors(); cam = B.make_camera(W, H, synth.TUM3, sf)
d_depth = torch.from_numpy(synth.depth_s1(W, H).astype(np.float32)).cuda()


def build(nh):
    hb = NB // nh
    hs = []
    for i in range(nh):
        sl = slice(i * hb, (i + 1) * hb)
        trk = B.Tracker(W, H, cam, NF, 1.2, 8, 20, 7, max_batch=hb, point_cap=NF + 64, max_boxes=4, device=0)
        cap = trk.cap
        st = torch.cuda.Stream()
        d_frames = torch.from_numpy(frames[sl]).cuda(); d_pidx = torch.from_numpy(np.ascontiguousarray(pidx[sl] - i * hb)).cuda()
        # inputs of the track stage: dummy last-frame points (zeros are fine for timing shape? no: use real ones from a set-up pass)
        hk = np.zeros((hb, cap), B.KP_DTYPE); hd = np.zeros((hb, cap, 32), np.uint8); hn = np.zeros(hb, np.int32)
        exh = L.sgs_tracker_extractor(trk.h)
        B.check(L.sgs_tracker_extract_device(trk.h, d_frames.data_ptr(), hb, W * H, W, st.cuda_stream))
        B.check(L.sgs_extractor_fetch(exh, hb, hk.ctypes.data_as(v), hd.ctypes.data_as(v), cap, hn.ctypes.data_as(v), st.cuda_stream))
        ti = BN.make_track_inputs(hk, hd, hn, boxes[sl], None, cap, NF + 64, pidx[sl] - i * hb)
        dv = {k: torch.from_numpy(np.ascontiguousarray(ti[k])).cuda() for k in ('ur', 'boxes', 'nb', 'have', 'lxyz', 'ldesc', 'lflags', 'loct', 'lang', 'ln', 'T')}
        hs.append(dict(trk=trk, st=st, d_frames=d_frames, d_pidx=d_pidx, dv=dv, hb=hb))
    return hs


def step(h):
    trk, st, hb, dv = h['trk'], h['st'], h['hb'], h['dv']
    B.check(L.sgs_tracker_extract_device(trk.h, h['d_frames'].data_ptr(), hb, W * H, W, st.cuda_stream))
    B.check(L.sgs_tracker_lk_device(trk.h, h['d_frames'].data_ptr(), hb, W * H, W, h['d_pidx'].data_ptr(), st.cuda_stream))
    B.check(L.sgs_tracker_fundamental_device(trk.h, hb, dv['boxes'].data_ptr(), dv['nb'].data_ptr(), dv['have'].data_ptr(), h['d_pidx'].data_ptr(), st.cuda_stream))
    B.check(L.sgs_tracker_stereo_device(trk.h, hb, d_depth.data_ptr(), 0, W, st.cuda_stream))
    ptrs = [0, 0] + [dv[k].data_ptr() for k in ('boxes', 'nb', 'have', 'lxyz', 'ldesc', 'lflags', 'loct', 'lang', 'ln', 'T', 'T')]
    B.check(L.sgs_tracker_track_device(trk.h, hb, 0, *ptrs, TH, 0, 1, st.cuda_stream))


for nh in (1, 2, 4):
    hs = build(nh)
    for _ in range(3):
        for h in hs:
            step(h)
    torch.cuda.synchronize()
    K = 20
    t0 = time.perf_counter()
    for _ in range(K):
        for h in hs:
            step(h)
    torch.cuda.synchronize()
    dt = (time.perf_counter() - t0) / K
    print('%d handle(s): %.3f ms per %d frames -> %.0f frames/s' % (nh, dt * 1e3, NB, NB / dt), flush=True)
    for h in hs:
        h['trk'].close()
