#!/usr/bin/env python3
"""Secondary measurements (not the driver's bench line): BASELINE config 5 (Hamming BF sweep 1k..64k) and config 3's extraction
geometry (1280x720, 2000 features).  Prints one JSON line per measurement."""
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(ROOT, 'sg-slam_b200'), os.path.join(ROOT, 'oracle')]
from pysgs import binding as B, synth  # noqa: E402


def ev_time(fn, reps, st):
    for _ in range(3):
        fn()
    st.synchronize()
    e0, e1 = torch.cuda.Event(True), torch.cuda.Event(True)
    with torch.cuda.stream(st):
        e0.record(st)
        for _ in range(reps):
            fn()
        e1.record(st)
    st.synchronize()
    return e0.elapsed_time(e1) / reps


def hamming_sweep():
    peaks = json.load(open(os.path.join(ROOT, 'MEASURED_PEAKS.json'))) if os.path.exists(os.path.join(ROOT, 'MEASURED_PEAKS.json')) else {'hbm_gbs': 6650.0}
    st = torch.cuda.Stream()
    for n in (1024, 2048, 4096, 8192, 16384, 32768, 65536):
        t = synth.descriptors_s5(n, 5); q = synth.descriptors_near(t, 6, 40) if n <= 16384 else synth.descriptors_s5(n, 7)
        dq, dt = torch.from_numpy(q).cuda(), torch.from_numpy(t).cuda()
        di, db, ds = (torch.empty(n, dtype=torch.int32, device='cuda') for _ in range(3))
        scr = torch.empty(max(1, B.hamming_bf_scratch_elems(n, n)), dtype=torch.int32, device='cuda')
        f = lambda: B.hamming_bf_device(dq.data_ptr(), n, dt.data_ptr(), n, di.data_ptr(), db.data_ptr(), ds.data_ptr(), scr.data_ptr(), st.cuda_stream)
        ms = ev_time(f, 20 if n <= 16384 else 5, st)
        pairs = n * n / (ms * 1e-3)
        alg_bytes = 32 * 2 * n + 12 * n
        print(json.dumps({'bench': 'hamming_bf', 'n': n, 'm': n, 'ms': ms, 'pairs_per_s': pairs, 'popc32_per_s': 8 * pairs,
                          'alg_GBps': alg_bytes / (ms * 1e-3) / 1e9, 'frac_hbm': alg_bytes / (ms * 1e-3) / 1e9 / peaks['hbm_gbs'],
                          'bound': 'POPC/ALU (operands reused from shared memory), not HBM'}), flush=True)


def extract_config_b():
    w, h, nf, nb = 1280, 720, 2000, 128
    frames = np.stack([synth.frame_s1(w, h, 40 + i) for i in range(8)])
    frames = np.tile(frames, (nb // 8, 1, 1))
    ex = B.Extractor(w, h, nf, 1.2, 8, 20, 7, max_batch=nb)
    d = torch.from_numpy(frames).cuda()
    st = torch.cuda.Stream()
    ex.set_profiling(True)
    ms = ev_time(lambda: ex.extract_batch_device(d.data_ptr(), nb, w * h, w, st.cuda_stream), 10, st)
    stage, ncalls = ex.stage_times()
    kps, desc, n = ex.fetch(nb, st.cuda_stream)
    print(json.dumps({'bench': 'extract_1280x720_2000', 'frames_per_step': nb, 'ms_per_step': ms, 'frames_per_s': nb / (ms * 1e-3), 'mean_keypoints': float(n.mean()),
                      'stage_ms': [s / max(1, ncalls) for s in stage], 'alg_bytes_per_frame': 16234083,
                      'alg_GBps': 16234083 * nb / (ms * 1e-3) / 1e9}), flush=True)
    ex.close()


if __name__ == '__main__':
    which = sys.argv[1] if len(sys.argv) > 1 else 'all'
    if which in ('all', 'hamming'):
        hamming_sweep()
    if which in ('all', 'b'):
        extract_config_b()
