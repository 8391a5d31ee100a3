"""The RGB-D step against the gray step, one JSON line on stdout.

Times sgs_tracker_step_rgbd (colour + raw uint16 depth from host memory; gray, mvKeysUn, mvuRight and mvDepth computed on the device) and
sgs_tracker_step (gray + colour frames and a host-computed u_right) in the same process, alternated, at 640x480, 1000 features, 512 frames per step,
from pinned host buffers.  The colour frames carry the gray frame in all three channels, so that the two steps extract the same keypoints and
differ only in what they upload and convert.  Also reports the H2D bytes per frame of each step (from the shapes), the device time of the
conversion kernel (sgs_grab_rgbd_batch_device, CUDA events) against its algorithmic bytes, and the card name and power limit read in the same run.

    python tools/bench_rgbd_step.py [--frames 512] [--steps 10] [--warmup 2]"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'sg-slam_b200'), ROOT):
    if p not in sys.path:
        sys.path.insert(0, p)

W, H, NFEAT, TH = 640, 480, 1000, 15.0


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
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--rounds', type=int, default=3, help='alternations of the two steps; the median step time of each is reported')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_rgbd_step.py needs a CUDA device')
    import bench
    import detector_model as DM
    from pysgs import binding as B
    from pysgs import synth
    L, v = B.lib(), C.c_void_p
    NB = args.frames
    name, power_limit = card()
    frames, boxes, unique = bench.make_frames(NB, 2, W, H)
    pidx = bench.prev_index(NB, unique)
    camd = dict(synth.TUM3)
    sf = synth.scale_factors()
    trk = B.Tracker(W, H, B.make_camera(W, H, camd, sf), NFEAT, 1.2, 8, 20, 7, max_batch=NB, point_cap=NFEAT + 64, max_boxes=4, device=0)
    cap, pcap = trk.cap, trk.point_cap
    if os.path.exists(bench.MODEL + '.param'):
        det_kind, (pp, bp) = 'trained model', (bench.MODEL + '.param', bench.MODEL + '.bin')
    else:
        det_kind, (pp, bp) = 'synthetic graph of tests/detector_model.py', DM.write_mini_model(tempfile.mkdtemp(), 0)
    det = B.Detector(pp, bp, max_frames=NB, det_thr=0.9, dyn_thr=0.01)
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    h_gray, h_rgb = pin(frames), pin(synth.gray_to_rgb(frames))
    raw = np.rint(synth.depth_s1(W, H).astype(np.float64) * 5000).astype(np.uint16)
    h_depth = pin(np.broadcast_to(raw, (NB, H, W)))
    kps = np.zeros((NB, cap), B.KP_DTYPE); desc = np.zeros((NB, cap, 32), np.uint8); n = np.zeros(NB, np.int32)
    B.check(L.sgs_tracker_extract(trk.h, v(h_gray.data_ptr()), NB, W * H, W, kps.ctypes.data, desc.ctypes.data, cap, n.ctypes.data))
    ti = bench.make_track_inputs(kps, desc, n, boxes, cap, pcap, pidx, W, H, camd)
    hp = {k: pin(ti[k]) for k in ('pidx', 'ur', 'lxyz', 'ldesc', 'lflags', 'loct', 'lang', 'ln', 'T')}
    last = [v(hp[k].data_ptr()) for k in ('lxyz', 'ldesc', 'lflags', 'loct', 'lang', 'ln', 'T', 'T')]
    outs = {k: pin(np.zeros(s, dt)) for k, s, dt in (('kps', (NB, cap * 28), np.uint8), ('desc', (NB, cap, 32), np.uint8), ('ur', (NB, cap), np.float32),
                                                      ('cnt', NB, np.int32), ('mp', (NB, cap), np.int32), ('nm', NB, np.int32), ('boxes', (NB, 16), np.float32),
                                                      ('nb', NB, np.int32), ('have', NB, np.uint8), ('kun', (NB, cap * 28), np.uint8), ('dz', (NB, cap), np.float32))}
    o = lambda *ks: [v(outs[k].data_ptr()) for k in ks]
    fmt = B.RgbdFormat(1, B.DEPTH_U16, np.float32(1 / 5000))

    def step_gray():
        B.check(L.sgs_tracker_step(trk.h, det.h, v(h_gray.data_ptr()), W * H, W, v(h_rgb.data_ptr()), W * H * 3, W * 3, NB, v(hp['pidx'].data_ptr()),
                                   v(hp['ur'].data_ptr()), *last, TH, 0, 1, *o('kps', 'desc', 'ur', 'cnt', 'mp', 'nm', 'boxes', 'nb', 'have')))

    def step_rgbd():
        B.check(L.sgs_tracker_step_rgbd(trk.h, det.h, v(h_rgb.data_ptr()), W * H * 3, W * 3, v(h_depth.data_ptr()), W * H * 2, W * 2, C.byref(fmt), NB,
                                        v(hp['pidx'].data_ptr()), *last, TH, 0, 1, *o('kps', 'desc', 'ur', 'cnt', 'mp', 'nm', 'boxes', 'nb', 'have', 'kun', 'dz')))

    def timed(fn):
        t0 = time.perf_counter()
        for _ in range(args.steps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / args.steps

    step_gray(); g_out = {k: outs[k].numpy().copy() for k in ('kps', 'cnt')}
    step_rgbd(); r_out = {k: outs[k].numpy().copy() for k in ('kps', 'cnt')}
    same_keypoints = bool(np.array_equal(g_out['cnt'], r_out['cnt']) and np.array_equal(g_out['kps'], r_out['kps']))
    for _ in range(args.warmup):
        step_gray(); step_rgbd()
    tg, tr = [], []
    for _ in range(args.rounds):
        tg.append(timed(step_gray)); tr.append(timed(step_rgbd))
    tg, tr = float(np.median(tg)), float(np.median(tr))
    # the conversion kernel alone on device frames, CUDA events over many launches
    d_rgb, d_raw = h_rgb.cuda(), h_depth.cuda()
    d_gray = torch.empty((NB, H, W), dtype=torch.uint8, device='cuda'); d_dep = torch.empty((NB, H, W), dtype=torch.float32, device='cuda')
    grab = lambda: B.check(L.sgs_grab_rgbd_batch_device(v(d_rgb.data_ptr()), W * H * 3, W * 3, v(d_raw.data_ptr()), W * H * 2, W * 2, C.byref(fmt), W, H, NB,
                                                        v(d_gray.data_ptr()), W * H, W, v(d_dep.data_ptr()), W * H * 4, W * 4, v(torch.cuda.current_stream().cuda_stream)))
    for _ in range(3):
        grab()
    nl = 50
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(nl):
        grab()
    e1.record(); torch.cuda.synchronize()
    grab_ms = e0.elapsed_time(e1) / nl
    grab_ok = bool(np.array_equal(d_gray.cpu().numpy(), frames)) and bool(np.array_equal(d_dep[0].cpu().numpy(), raw.astype(np.float32) * np.float32(1 / 5000)))
    grab_bytes = NB * (W * H * 3 + W * H * 2 + W * H + W * H * 4)
    last_bytes = pcap * (12 + 32 + 1 + 4 + 4) + 4 + 2 * 64
    h2d = {'step': W * H + W * H * 3 + cap * 4 + 4 + last_bytes, 'step_rgbd': W * H * 3 + W * H * 2 + 4 + last_bytes}
    print(json.dumps({
        'gpu': name, 'power_limit_w': power_limit, 'frames_per_step': NB, 'width': W, 'height': H, 'features': NFEAT, 'detector': det_kind,
        'step_frames_per_s': NB / tg, 'step_rgbd_frames_per_s': NB / tr, 'step_ms': tg * 1e3, 'step_rgbd_ms': tr * 1e3,
        'h2d_bytes_per_frame': h2d, 'h2d_image_bytes_per_frame': {'step': W * H * 4, 'step_rgbd': W * H * 5},
        'grab_kernel_ms': grab_ms, 'grab_bytes': grab_bytes, 'grab_gb_per_s': grab_bytes / grab_ms / 1e6,
        'same_keypoints_both_steps': same_keypoints, 'grab_parity': grab_ok,
        'note': 'pinned host buffers, calls synchronise; colour = gray in three channels; step times are medians of %d alternated rounds of %d steps'
                % (args.rounds, args.steps)}))
    trk.close(); det.close()


if __name__ == '__main__':
    main()
