"""The reference-key-frame chain against the pose chain, one JSON line on stdout.

After one RGB-D step of 512 frames (640x480, 1000 features; sgs_tracker_step_rgbd from pinned host buffers), times on the device (CUDA events around
one call): sgs_tracker_pose_chain_device, then sgs_tracker_refkf_chain_device with (a) every row enabled and (b) 8 of the rows enabled, seen_in = the
pose chain's motion discards, alternated over --rounds rounds on the same inputs (the step is repeated before each round, untimed, because the pose
chain rewrites the step's matches in place).  The reference key frame of every frame is its previous frame (bench.make_track_inputs' last-frame
arrays) with its FeatureVector from a vocabulary trained on the frames' descriptors (k = 10, L = 5); the local maps are bench.make_local_map's.
Medians are reported with the card name and power limit read in the same run.  Without a device it stops at the first device call.

    python tools/bench_refkf_chain.py [--frames 512] [--rounds 5]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'sg-slam_b200'), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

W, H, NFEAT, TH, MCAP = 640, 480, 1000, 15.0, 1536


def card():
    try:
        name, limit = subprocess.check_output(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit', '--format=csv,noheader,nounits'],
                                              text=True).strip().splitlines()[0].split(', ')
        return name, float(limit)
    except Exception:
        import torch
        return torch.cuda.get_device_name(0), None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=512)
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--enabled', type=int, default=8, help='rows enabled in the sparse case')
    args = ap.parse_args()
    import bench
    from pysgs import synth
    NB = args.frames
    frames, boxes, unique = bench.make_frames(NB, 2, W, H)
    pidx = bench.prev_index(NB, unique)
    camd = dict(synth.TUM3)
    sf = synth.scale_factors()
    raw = np.rint(synth.depth_s1(W, H).astype(np.float64) * 5000).astype(np.uint16)
    sparse = np.zeros(NB, np.uint8); sparse[np.linspace(0, NB - 1, min(args.enabled, NB)).astype(int)] = 1
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_refkf_chain.py needs a CUDA device (host inputs for %d frames built)' % NB)
    import detector_model as DM
    import oracle as O
    import refkf_cases as R
    from pysgs import binding as B
    L, v = B.lib(), C.c_void_p
    name, power_limit = card()
    cam = B.make_camera(W, H, camd, sf)
    trk = B.Tracker(W, H, cam, NFEAT, 1.2, 8, 20, 7, max_batch=NB, point_cap=NFEAT + 64, max_boxes=4, device=0)
    cap, pcap = trk.cap, trk.point_cap
    if os.path.exists(bench.MODEL + '.param'):
        pp, bp = bench.MODEL + '.param', bench.MODEL + '.bin'
    else:
        pp, bp = DM.write_mini_model(tempfile.mkdtemp(), 0)
    det = B.Detector(pp, bp, max_frames=NB, det_thr=0.9, dyn_thr=0.01)
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    h_gray, h_rgb, h_depth = pin(frames), pin(synth.gray_to_rgb(frames)), pin(np.broadcast_to(raw, (NB, H, W)))
    kps = np.zeros((NB, cap), B.KP_DTYPE); desc = np.zeros((NB, cap, 32), np.uint8); n = np.zeros(NB, np.int32)
    B.check(L.sgs_tracker_extract(trk.h, v(h_gray.data_ptr()), NB, W * H, W, kps.ctypes.data, desc.ctypes.data, cap, n.ctypes.data))
    ti = bench.make_track_inputs(kps, desc, n, boxes, cap, pcap, pidx, W, H, camd)
    hp = {k: pin(ti[k]) for k in ('pidx', 'lxyz', 'ldesc', 'lflags', 'loct', 'lang', 'ln', 'T')}
    last = [v(hp[k].data_ptr()) for k in ('lxyz', 'ldesc', 'lflags', 'loct', 'lang', 'ln', 'T', 'T')]
    outs = {k: np.zeros(s, dt) for k, s, dt in (('kps', (NB, cap), B.KP_DTYPE), ('desc', (NB, cap, 32), np.uint8), ('ur', (NB, cap), np.float32),
                                                 ('cnt', NB, np.int32), ('mp', (NB, cap), np.int32), ('nm', NB, np.int32), ('boxes', (NB, 16), np.float32),
                                                 ('nb', NB, np.int32), ('have', NB, np.uint8), ('kun', (NB, cap), B.KP_DTYPE), ('dz', (NB, cap), np.float32))}
    o = [outs[k].ctypes.data_as(v) for k in ('kps', 'desc', 'ur', 'cnt', 'mp', 'nm', 'boxes', 'nb', 'have', 'kun', 'dz')]
    fmt = B.RgbdFormat(1, B.DEPTH_U16, np.float32(1 / 5000))

    def step():
        B.check(L.sgs_tracker_step_rgbd(trk.h, det.h, v(h_rgb.data_ptr()), W * H * 3, W * 3, v(h_depth.data_ptr()), W * H * 2, W * 2, C.byref(fmt), NB,
                                        v(hp['pidx'].data_ptr()), *last, TH, 0, 1, *o))
    step()
    rng = np.random.default_rng(3)
    lms = [bench.make_local_map(f, outs['kun'][f], outs['desc'][f], int(outs['cnt'][f]), ti, MCAP, camd, sf, rng, W, H) for f in range(NB)]
    voc = R.train_vocabulary(np.concatenate([outs['desc'][f, :outs['cnt'][f]] for f in range(0, NB, max(1, NB // 16))]), 10, 5, seed=1)
    V = O.Vocabulary(voc['k'], voc['L'], voc['parent'], voc['desc'], voc['weight'])
    gvoc = v()
    B.check(L.sgs_vocabulary_create(0, voc['k'], voc['L'], len(voc['parent']), voc['parent'].ctypes.data_as(v), np.ascontiguousarray(voc['desc']).ctypes.data_as(v),
                                    voc['weight'].ctypes.data_as(v), C.byref(gvoc)))
    knode = np.zeros((NB, pcap), np.int32); kweight = np.zeros((NB, pcap), np.float64)
    for f in range(NB):
        m = int(ti['ln'][f])
        _, kweight[f, :m], knode[f, :m] = V.transform(ti['ldesc'][f, :m], 4)
    stack = lambda key, dt: np.ascontiguousarray(np.stack([m[key] for m in lms]).astype(dt))
    dev = {k: torch.from_numpy(np.ascontiguousarray(a)).cuda() for k, a in dict(
        lxyz=ti['lxyz'], ldesc=ti['ldesc'], lflags=ti['lflags'], loct=ti['loct'], lang=ti['lang'], ln=ti['ln'], T=ti['T'], lid=stack('lid', np.int32),
        xyz=stack('xyz', np.float32), nrm=stack('nrm', np.float32), mn=stack('mn', np.float32), mx=stack('mx', np.float32), dsc=stack('dsc', np.uint8),
        valid=stack('valid', np.uint8), obs=stack('obs', np.uint8), n=np.array([m['n'] for m in lms], np.int32), knode=knode, kweight=kweight,
        sparse=sparse).items()}
    D = lambda k: dev[k].data_ptr()
    isig = np.zeros(16, np.float32); isig[:8] = 1.0 / (sf.astype(np.float32) ** 2)
    out = dict(T1=torch.zeros((NB, 16), device='cuda'), T2=torch.zeros((NB, 16), device='cuda'), mp=torch.zeros((NB, cap), dtype=torch.int32, device='cuda'),
               outl=torch.zeros((NB, cap), dtype=torch.uint8, device='cuda'), st=torch.zeros((NB, 8), dtype=torch.int32, device='cuda'))
    pc = B.PoseChainBatch()
    pc.last_xyz, pc.last_desc, pc.last_flags, pc.last_octave, pc.last_angle, pc.last_n = D('lxyz'), D('ldesc'), D('lflags'), D('loct'), D('lang'), D('ln')
    pc.tcw_cur, pc.tcw_last, pc.th, pc.mono, pc.check_orientation, pc.last_local_id = D('T'), D('T'), TH, 0, 1, D('lid')
    rk = B.RefKfBatch()
    rk.kf_node, rk.kf_weight, rk.kf_desc, rk.kf_angle, rk.kf_xyz, rk.kf_flags, rk.kf_n, rk.kf_local_id = D('knode'), D('kweight'), D('ldesc'), D('lang'), D('lxyz'), D('lflags'), D('ln'), D('lid')
    rk.tcw_last = D('T')
    for a in (pc, rk):
        a.mp_xyz, a.mp_normal, a.mp_min_dist, a.mp_max_dist, a.mp_desc, a.mp_valid, a.mp_obs, a.mp_n, a.mp_cap = D('xyz'), D('nrm'), D('mn'), D('mx'), D('dsc'), D('valid'), D('obs'), D('n'), MCAP
        a.th_local, a.nnratio_local = 3.0, 0.8
        for l in range(16): a.inv_level_sigma2[l] = float(isig[l])
        a.tcw_final, a.f_mp, a.outlier, a.stats = out['T2'].data_ptr(), out['mp'].data_ptr(), out['outl'].data_ptr(), out['st'].data_ptr()
    pc.tcw_motion = out['T1'].data_ptr(); rk.tcw_refkf = out['T1'].data_ptr()
    stream = torch.cuda.Stream()
    st = stream.cuda_stream

    def timed(fn):
        e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
        e0.record(stream); fn(); e1.record(stream); torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    def refkf(enable):
        rk.frame_enable = enable
        B.check(L.sgs_tracker_refkf_chain_device(trk.h, gvoc, C.byref(rk), NB, v(st)))
    t = {'pose_chain_ms': [], 'refkf_all_rows_ms': [], 'refkf_sparse_rows_ms': []}
    passed = 0
    for r in range(args.rounds + 1):                 # round 0 warms every shape up
        step()
        ms = timed(lambda: B.check(L.sgs_tracker_pose_chain_device(trk.h, C.byref(pc), NB, v(st))))
        disc = v()
        B.check(L.sgs_tracker_motion_discards_device(trk.h, C.byref(disc)))
        rk.seen_in = disc.value
        ms_all = timed(lambda: refkf(None))
        if r == 0:
            passed = int(out['st'][:, 1].sum().item())
        ms_sparse = timed(lambda: refkf(D('sparse')))
        if r:
            t['pose_chain_ms'].append(ms); t['refkf_all_rows_ms'].append(ms_all); t['refkf_sparse_rows_ms'].append(ms_sparse)
    L.sgs_vocabulary_destroy(gvoc)
    det.close(); trk.close()
    res = {'gpu': name, 'power_limit_w': power_limit, 'frames': NB, 'width': W, 'height': H, 'features': NFEAT, 'mp_cap': MCAP, 'rounds': args.rounds,
           'sparse_rows_enabled': int(sparse.sum()), 'rows_past_15_matches_all_enabled': passed}
    res.update({k: float(np.median(x)) for k, x in t.items()})
    print(json.dumps(res))


if __name__ == '__main__':
    main()
