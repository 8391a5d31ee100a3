"""Joins an ncu launch list of one detector call (ncu --metrics gpu__time_duration.sum ... python tools/bench_detector.py --once B) with the kernel plan
(sgs_detector_describe): per kernel time, achieved GB/s and FP32-equivalent TFLOP/s of the 1x1-convolution GEMMs.  Usage: det_launch_table.py launches.csv [batch]"""
import collections
import csv
import os
import re
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'sg-slam_b200'))
from pysgs import binding as B  # noqa: E402

path = sys.argv[1]; F = int(sys.argv[2]) if len(sys.argv) > 2 else 128
m = os.path.join(ROOT, 'oracle', '_ref', 'ncnn_model', 'mobilenetv3_ssdlite_voc')
plan = B.Detector(m + '.param', m + '.bin', max_frames=F, det_thr=0.5, dyn_thr=0.1, flags=B.DET_PLAN_ONLY)
ops = [o for o in plan.describe().split('\n')[1:] if o]
rows = [r for r in csv.reader(open(path)) if len(r) > 5]
for i, r in enumerate(rows):
    if 'Kernel Name' in r:
        hdr = r; data = rows[i + 1:]; break
mv = hdr.index('Metric Value'); gi = hdr.index('Grid Size'); kn = hdr.index('Kernel Name')
first = next(i for i, r in enumerate(data) if 'preprocess_kernel' in r[kn])          # one call = preprocess ... detout_merge; the window may start mid-call
data = data[first:] + data[:first]
ts = [float(r[mv].replace(',', '')) / 1000 for r in data]
agg = collections.OrderedDict()
for r, t in zip(data, ts):
    name = re.sub(r'\(.*', '', r[kn]).replace('void ', '').replace('sgs::det::', '').replace('sgs::tc::', '')
    agg.setdefault(name, [0, 0.0]); agg[name][0] += 1; agg[name][1] += t
tot = sum(ts)
print('total %.1f us, %d launches, batch %d' % (tot, len(ts), F))
for k, (c, t) in sorted(agg.items(), key=lambda kv: -kv[1][1]):
    print('  %-60s %3d %9.1f us %5.1f%%' % (k[:60], c, t, 100 * t / tot))
out = []; gemm_t = 0.0; gemm_fl = 0.0
for j, op in enumerate(ops):
    t = ts[j + 1]
    g = re.search(r'geom (\S+)', op); kind = op.split()[0]
    tail = op.split('|', 1)[1][:44] if '|' in op else ''
    if kind == 'conv1x1':
        cin, hh, ww = [int(x) for x in g.group(1).split('->')[0].split('x')]; cout = int(g.group(1).split('->')[1].split('x')[0])
        npx = hh * ww * F; by = (cin + cout) * 4 * npx; fl = 2 * cin * cout * npx
        gemm_t += t; gemm_fl += fl
        tile = re.search(r'tile (\S+) kb (\S+) stages (\d+)( wres)?', op).group(0)
        out.append((t, '%3d %-8s %-26s %-34s %7.1f us %6.0f GB/s %6.1f TF |%s' % (j, kind, g.group(1), tile, t, by / t * 1e-3, fl / t * 1e-6, tail)))
    else:
        out.append((t, '%3d %-8s %-26s %-34s %7.1f us |%s' % (j, kind, g.group(1) if g else '', '', t, tail)))
print('1x1-convolution GEMMs: %.1f us for %.1f GFLOP = %.1f TFLOP/s FP32-equivalent (x3 on the TF32 tensor pipe)' % (gemm_t, gemm_fl * 1e-9, gemm_fl / gemm_t * 1e-6))
for t, s in sorted(out, key=lambda x: -x[0])[:int(sys.argv[3]) if len(sys.argv) > 3 else 40]:
    print(s)
