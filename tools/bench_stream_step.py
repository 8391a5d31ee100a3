"""Live RGB-D streams, one new frame per stream per call: the stream step against the batch step that re-sends each previous frame.  One JSON line.

  (A) sgs_tracker_step_rgbd_stream(_device): S streams (default 512), one new frame each per call; the previous frames stay in the tracker's slots.
  (B) sgs_tracker_step_rgbd(_device) with prev_index: the only batch route to the same results -- S/2 streams per call, each as its previous frame
      (again: upload, gray, extraction, detector, pyramid) plus its new frame.
Both run on one tracker (the batch calls leave the slots alone), 640x480, 1000 features, the reference's trained detector when build() staged it.
Each stream alternates between two consecutive frames of a synthetic camera path, so LK and F see real motion.  Reported for device-resident and
pinned host buffers: new frames per second of A and B (medians of alternated rounds), whether the new frames' outputs of A and B are identical, the
device time of the slot commit and of the per-call resolve (kernel times from torch.profiler), and the card name and power limit read in the same run.

    python tools/bench_stream_step.py [--streams 512] [--steps 10] [--warmup 2] [--rounds 5]"""
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
    ap.add_argument('--streams', type=int, default=512)
    ap.add_argument('--steps', type=int, default=10)
    ap.add_argument('--warmup', type=int, default=2)
    ap.add_argument('--rounds', type=int, default=5, help='alternations of A and B; the median call time of each is reported')
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit('bench_stream_step.py needs a CUDA device')
    import bench
    import detector_model as DM
    from pysgs import binding as B
    from pysgs import synth
    L, v = B.lib(), C.c_void_p
    S = args.streams
    S2 = S // 2
    name, power_limit = card()
    # frames 0..S: consecutive frames of the bench's camera paths; call k gives stream s frame s + (k & 1)
    frames, boxes, unique = bench.make_frames(S + 1, 2, W, H)
    camd = dict(synth.TUM3)
    sf = synth.scale_factors()
    trk = B.Tracker(W, H, B.make_camera(W, H, camd, sf), NFEAT, 1.2, 8, 20, 7, max_batch=S, point_cap=NFEAT + 64, max_boxes=4, device=0)
    cap, pcap = trk.cap, trk.point_cap
    if os.path.exists(bench.MODEL + '.param'):
        det_kind, (pp, bp) = 'trained model', (bench.MODEL + '.param', bench.MODEL + '.bin')
    else:
        det_kind, (pp, bp) = 'synthetic graph of tests/detector_model.py', DM.write_mini_model(tempfile.mkdtemp(), 0)
    det = B.Detector(pp, bp, max_frames=S, det_thr=0.9, dyn_thr=0.01)
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    rgb = synth.gray_to_rgb(frames)
    raw = np.ascontiguousarray(np.broadcast_to(np.rint(synth.depth_s1(W, H).astype(np.float64) * 5000).astype(np.uint16), (S + 1, H, W)))
    kps = np.zeros((S, cap), B.KP_DTYPE); desc = np.zeros((S, cap, 32), np.uint8); n = np.zeros(S, np.int32)
    B.check(L.sgs_tracker_extract(trk.h, frames[:S].ctypes.data, S, W * H, W, kps.ctypes.data, desc.ctypes.data, cap, n.ctypes.data))
    ti = bench.make_track_inputs(kps, desc, n, boxes[:S], cap, pcap, bench.prev_index(S, unique), W, H, camd)
    LAST = ('lxyz', 'ldesc', 'lflags', 'loct', 'lang', 'ln', 'T', 'T')
    # (A): the S + 1 frames once; call k starts at frame k & 1.  (B): per parity, the S/2 new frames followed by their previous frames
    a_rgb, a_dep = pin(rgb), pin(raw)
    b_rows = [np.concatenate([np.arange(S2) + o, np.arange(S2) + 1 - o]) for o in (0, 1)]
    b_rgb, b_dep = [pin(rgb[r]) for r in b_rows], [pin(raw[r]) for r in b_rows]
    b_pidx = np.concatenate([np.arange(S2) + S2, np.arange(S2)]).astype(np.int32)      # previous frames are not first frames: no row is its own predecessor
    h = dict(a_last=[pin(ti[k]) for k in LAST], b_last=[pin(np.concatenate([ti[k][:S2], ti[k][:S2]])) for k in LAST], slot=pin(np.arange(S, dtype=np.int32)),
             pidx=pin(b_pidx))
    d = {k: ([x.cuda() for x in t] if isinstance(t, list) else t.cuda()) for k, t in h.items()}
    d_a_rgb, d_a_dep, d_b_rgb, d_b_dep = a_rgb.cuda(), a_dep.cuda(), [x.cuda() for x in b_rgb], [x.cuda() for x in b_dep]
    outs = {k: pin(np.zeros(s, dt)) for k, s, dt in (('kps', (S, cap * 28), np.uint8), ('desc', (S, cap, 32), np.uint8), ('ur', (S, cap), np.float32),
                                                     ('cnt', S, np.int32), ('mp', (S, cap), np.int32), ('nm', S, np.int32), ('boxes', (S, 16), np.float32),
                                                     ('nb', S, np.int32), ('have', S, np.uint8), ('kun', (S, cap * 28), np.uint8), ('dz', (S, cap), np.float32))}
    o = [v(outs[k].data_ptr()) for k in ('kps', 'desc', 'ur', 'cnt', 'mp', 'nm', 'boxes', 'nb', 'have', 'kun', 'dz')]
    fmt = B.RgbdFormat(1, B.DEPTH_U16, np.float32(1 / 5000))
    fb_rgb, fb_dep = W * H * 3, W * H * 2
    ptrs = lambda ts: [v(t.data_ptr()) for t in ts]
    k = dict(a=0, b=0)

    def a_dev():
        off = k['a'] & 1; k['a'] += 1
        B.check(L.sgs_tracker_step_rgbd_stream_device(trk.h, det.h, v(d_a_rgb.data_ptr() + off * fb_rgb), fb_rgb, W * 3, v(d_a_dep.data_ptr() + off * fb_dep),
                                                      fb_dep, W * 2, C.byref(fmt), S, v(d['slot'].data_ptr()), None, *ptrs(d['a_last']), TH, 0, 1, None))

    def b_dev():
        off = k['b'] & 1; k['b'] += 1
        B.check(L.sgs_tracker_step_rgbd_device(trk.h, det.h, v(d_b_rgb[off].data_ptr()), fb_rgb, W * 3, v(d_b_dep[off].data_ptr()), fb_dep, W * 2, C.byref(fmt),
                                               2 * S2, v(d['pidx'].data_ptr()), *ptrs(d['b_last']), TH, 0, 1, None))

    def a_host():
        off = k['a'] & 1; k['a'] += 1
        B.check(L.sgs_tracker_step_rgbd_stream(trk.h, det.h, v(a_rgb.data_ptr() + off * fb_rgb), fb_rgb, W * 3, v(a_dep.data_ptr() + off * fb_dep), fb_dep, W * 2,
                                               C.byref(fmt), S, v(h['slot'].data_ptr()), None, *ptrs(h['a_last']), TH, 0, 1, *o))

    def b_host():
        off = k['b'] & 1; k['b'] += 1
        B.check(L.sgs_tracker_step_rgbd(trk.h, det.h, v(b_rgb[off].data_ptr()), fb_rgb, W * 3, v(b_dep[off].data_ptr()), fb_dep, W * 2, C.byref(fmt), 2 * S2,
                                        v(h['pidx'].data_ptr()), *ptrs(h['b_last']), TH, 0, 1, *o))

    def snapshot(nf):
        """The device results of the last call, frames [0, nf): compacted keypoints, descriptors, matches, F and its info, LK positions."""
        p = [v() for _ in range(10)]
        B.check(L.sgs_tracker_results_device(trk.h, *[C.byref(x) for x in p[:7]]))
        B.check(L.sgs_tracker_fundamental_device_ptr(trk.h, C.byref(p[7]), C.byref(p[8])))
        B.check(L.sgs_tracker_prev_xy_device(trk.h, C.byref(p[9])))
        torch.cuda.synchronize()
        get = lambda i, nbytes: B.memcpy_d2h(np.zeros(nbytes, np.uint8), p[i].value)
        return [get(0, nf * cap * 28), get(1, nf * cap * 32), get(2, nf * cap * 4), get(3, nf * 4), get(4, nf * cap * 4), get(5, nf * 4), get(7, nf * 72),
                get(8, nf * 16), get(9, nf * cap * 8)]

    # parity: stream s of A and row s of B see the same new frame (s + 1 - 1) after the same previous frame, itself not a first frame
    same = {}
    for kind, (fa, fbb) in (('device', (a_dev, b_dev)), ('host', (a_host, b_host))):
        k['a'] = k['b'] = 0
        fa(); fa(); fa()                          # A: frames s, s+1, s: the previous frame (s+1) is not a first frame
        ra = snapshot(S2)
        k['b'] = 0
        fbb()                                     # B, parity 0: new frames s after previous frames s+1
        rb = snapshot(S2)
        cnt = np.frombuffer(ra[3].tobytes(), np.int32)
        same[kind] = bool(all(np.array_equal(x, y) for x, y in zip(ra, rb))) and int(cnt.sum()) > 0

    def timed(fn):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(args.steps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / args.steps

    res = {}
    for kind, (fa, fbb) in (('device', (a_dev, b_dev)), ('host', (a_host, b_host))):
        for _ in range(args.warmup):
            fa(); fbb()
        ta, tb = [], []
        for _ in range(args.rounds):
            ta.append(timed(fa)); tb.append(timed(fbb))
        ta, tb = float(np.median(ta)), float(np.median(tb))
        res[kind] = {'A_new_frames_per_s': S / ta, 'B_new_frames_per_s': S2 / tb, 'A_ms_per_call': ta * 1e3, 'B_ms_per_call': tb * 1e3,
                     'A_over_B': (S / ta) / (S2 / tb), 'outputs_identical': same[kind]}
    # device time of the per-call stream kernels, from the profiler's kernel records over a few device calls
    from torch.profiler import ProfilerActivity, profile
    ncalls = 4
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(ncalls):
            a_dev()
        torch.cuda.synchronize()
    kt = {}
    for e in prof.events():
        for key in ('stream_commit_kernel', 'stream_resolve_kernel', 'lk_track_kernel'):
            if key in e.name and e.device_type.name == 'CUDA':
                kt[key] = kt.get(key, 0.0) + e.device_time / 1e3 / ncalls
    print(json.dumps({
        'gpu': name, 'power_limit_w': power_limit, 'streams': S, 'width': W, 'height': H, 'features': NFEAT, 'detector': det_kind,
        'device': res['device'], 'host_pinned': res['host'], 'kernel_ms_per_call': kt,
        'note': 'A: %d new frames per call (stream step); B: %d previous + %d new frames per call (batch step with prev_index); medians of %d alternated '
                'rounds of %d calls; kernel times from torch.profiler over %d device calls' % (S, S2, S2, args.rounds, args.steps, ncalls)}))
    trk.close(); det.close()


if __name__ == '__main__':
    main()
