"""Per-layer roofline of the detector's 1x1-convolution GEMMs (conv1x1_tc_kernel) on the real model at the flagship batch.

For every conv1x1 line of sgs_detector_describe: kind, layer, K -> N, map, fused tail kind, measured ms per call (CUDA events around every launch,
sgs_detector_set_profiling), algorithmic bytes (FP32 NHWC activations in + out, the tail's same-shape tensor operands, the weights once), the floor
and achieved / floor.  The floor of a layer is the larger of
  - its bytes at the HBM3 data-sheet bandwidth (3.35 TB/s), and
  - its MACs times three (the lo*hi, hi*lo, hi*hi TF32 passes) at 132 SMs x 1024 TF32 MAC/clk x 1.98 GHz.
The card name, power limit and SM clock are read in the same run.

Usage: python tools/detector_layer_roofline.py [--frames 512] [--calls 10] [--json PATH]"""
import argparse
import json
import os
import re
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, 'sg-slam_b200'), os.path.join(ROOT, 'tests')):
    sys.path.insert(0, p)

REAL = os.path.join(ROOT, 'oracle', '_ref', 'ncnn_model', 'mobilenetv3_ssdlite_voc')
HBM_BPS = 3.35e12
MAC_PER_S = 132 * 1024 * 1.98e9


def tail_kind(tail):
    """the planner's classification (epi_kind in detector.cu), from the describe text of the tail"""
    steps = [s.strip() for s in tail.split('|') if s.strip()]
    ops = [s.split()[0] for s in steps]
    tensor = [bool(re.match(r'(?:add|mul|sub|div)(?:\(rev\))? [0-9A-Za-z_]+ buf', s)) for s in steps]
    if not steps:
        return 'none', 0
    n = sum(tensor)
    if ops == ['relu']:
        return 'relu', 0
    if ops == ['clip']:
        return 'clip', 0
    if ops == ['add'] and n == 1:
        return 'add_t', 1
    if len(ops) == 4 and ops[2].startswith('mul') and 'start' in steps[2]:
        return 'hswish', 0
    if len(ops) == 5 and n == 2:
        return 'se_tail', 2
    if len(ops) == 4 and n == 1:
        return 'se_mul', 1
    return 'generic', n


def gpu_info():
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.sm,clocks.max.sm', '--format=csv,noheader'], capture_output=True, text=True,
                             timeout=20).stdout.strip().splitlines()[0]
        return dict(zip(('name', 'power_limit', 'sm_clock', 'max_sm_clock'), [x.strip() for x in out.split(',')]))
    except Exception as e:  # noqa: BLE001
        return {'error': str(e)}


def table(describe_text, kernel_ms, ncalls, nframes):
    ops = [l for l in describe_text.split('\n')[1:] if l]
    rows = []
    for j, op in enumerate(ops):
        if not op.startswith('conv1x1 '):
            continue
        t = kernel_ms[j + 1] / max(1, ncalls)
        cin, hh, ww, cout = [int(x) for x in re.search(r'geom (\d+)x(\d+)x(\d+)->(\d+)x', op).groups()]
        tile = re.search(r'tile (\d+)x(\d+) kb (\d+)x(\d+) stages (\d+)', op).groups()
        tail = op.split('|', 1)[1] if '|' in op else ''
        kind, nt = tail_kind(tail)
        npx = hh * ww * nframes
        nbytes = (cin + cout + nt * cout) * 4.0 * npx + 4.0 * cin * cout
        floor = max(nbytes / HBM_BPS, 3.0 * cin * cout * npx / MAC_PER_S) * 1e3
        rows.append(dict(layer=op.split()[1], K=cin, N=cout, map='%dx%d' % (hh, ww), tail=kind, nt=int(tile[0]), n_tiles=int(tile[1]), bk=int(tile[3]),
                         stages=int(tile[4]), ms=t, bytes=nbytes, floor_ms=floor, ratio=t / floor if floor > 0 else float('inf')))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--frames', type=int, default=512)
    ap.add_argument('--calls', type=int, default=10)
    ap.add_argument('--json', default=None)
    args = ap.parse_args()
    import torch
    from pysgs import binding as B
    import detector_model as DM
    if not torch.cuda.is_available():
        raise SystemExit('detector_layer_roofline.py needs a CUDA device')
    if not os.path.exists(REAL + '.param'):
        raise SystemExit('%s.param is not staged (build() copies it)' % REAL)
    info = gpu_info()
    F, W, H = args.frames, 640, 480
    det = B.Detector(REAL + '.param', REAL + '.bin', max_frames=F)
    base = np.stack([DM.synthetic_rgb(H, W, s) for s in range(8)])
    d = torch.from_numpy(base[np.arange(F) % 8]).cuda()
    nd = torch.zeros(F, dtype=torch.int32, device='cuda'); boxes = torch.zeros((F, 4, 4), device='cuda'); have = torch.zeros(F, dtype=torch.uint8, device='cuda')

    def run():
        det.detect_device(d.data_ptr(), H * W * 3, W * 3, W, H, F, d_dyn_rm=boxes.data_ptr(), d_ndyn_rm=nd.data_ptr(), d_have_dyn_rm=have.data_ptr(), max_boxes=4)

    for _ in range(3):
        run()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.calls):
        run()
    e1.record(); torch.cuda.synchronize()
    call_ms = e0.elapsed_time(e1) / args.calls
    det.set_profiling(1)
    run()                                   # the times of a call are collected at the next one
    for _ in range(args.calls):
        run()
    torch.cuda.synchronize()
    kms, nc = det.kernel_times()
    det.set_profiling(0)
    rows = table(det.describe(), kms, nc, F)
    info_after = gpu_info()
    det.close()

    print('card %s, power limit %s, SM clock %s (max %s); after: SM clock %s' % (info.get('name'), info.get('power_limit'), info.get('sm_clock'),
                                                                                    info.get('max_sm_clock'), info_after.get('sm_clock')))
    print('%d frames of %dx%d per call, %d profiled calls; whole call without events %.2f ms' % (F, W, H, nc, call_ms))
    print('%-6s %-28s %5s %5s %-8s %-8s %4s %3s %2s %8s %9s %8s %6s' % ('kind', 'layer', 'K', 'N', 'map', 'tail', 'NT', 'BK', 'st', 'ms', 'MB', 'floor', 'x'))
    for r in rows:
        print('%-6s %-28s %5d %5d %-8s %-8s %4d %3d %2d %8.3f %9.1f %8.3f %6.2f' % ('gemm', r['layer'], r['K'], r['N'], r['map'], r['tail'], r['nt'], r['bk'],
                                                                               r['stages'], r['ms'], r['bytes'] / 1e6, r['floor_ms'], r['ratio']))
    tot, fl = sum(r['ms'] for r in rows), sum(r['floor_ms'] for r in rows)
    print('conv1x1 family: %d launches, %.3f ms per call, floor %.3f ms (x %.2f), %.1f GB, %.2f TB/s algorithmic' % (
        len(rows), tot, fl, tot / fl, sum(r['bytes'] for r in rows) / 1e9, sum(r['bytes'] for r in rows) / tot / 1e9))
    print('all kernels: %.3f ms per call (sum of per-kernel events)' % (sum(kms) / max(1, nc)))
    if args.json:
        os.makedirs(os.path.dirname(os.path.abspath(args.json)), exist_ok=True)
        with open(args.json, 'w') as f:
            json.dump(dict(gpu=info, gpu_after=info_after, frames=F, call_ms=call_ms, rows=rows, gemm_ms=tot, floor_ms=fl), f, indent=1)


if __name__ == '__main__':
    main()
