"""Per-tile clock trace of the detector's 1x1-convolution GEMM (conv1x1_tc_kernel) at the shapes of a few layers of the reference model.

Builds sg-slam_b200/probes/gemm_tile_trace.cu with -DSGS_GEMM_TRACE into a temporary directory (the product build has no stamps), runs one GEMM per
layer shape on seeded data at the flagship batch and prints, per layer, the mean clocks of each phase of the traced tiles of CTA (0, 0) next to the
per-tile budget:
  ring     waiting for a full ring slot (summed over the tile's k-blocks)
  kwait    inside the k-loop's wgmma.wait_group (summed)
  issue    tile start -> last wgmma issued (includes ring and the kwait of all but the last k-block)
  drain    last wgmma issued -> its wait_group returned
  epi      the epilogue (bias, tail, stores)
  period   clocks from one tile start to the next
  budget   MMA: the tile's three TF32 passes at 1024 MAC/clk; memory: its activation bytes in + out at 3.35 TB/s / 132 SMs / max SM clock.
The card name, power limit and SM clock are read in the same run.

Usage: python tools/gemm_tile_trace.py [--frames 512] [--csrc DIR] [--json PATH]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
from detector_layer_roofline import gpu_info  # noqa: E402

# (layer, Cin, Cout, map side, tail): the shapes of the reference model's layers (sgs_detector_describe of mobilenetv3_ssdlite_voc)
LAYERS = [('673', 40, 240, 38, 1), ('780', 112, 672, 19, 1), ('597', 16, 64, 150, 0), ('605', 24, 72, 75, 0)]
TR_START, TR_RING, TR_ISSUED, TR_DRAINED, TR_EPI_END, TR_KWAIT = range(6)


def build(csrc, outdir):
    exe = os.path.join(outdir, 'gemm_tile_trace')
    src = os.path.join(ROOT, 'sg-slam_b200', 'probes', 'gemm_tile_trace.cu')
    subprocess.check_call(['nvcc', '-O3', '-std=c++17', '-gencode', 'arch=compute_90a,code=sm_90a', '--expt-relaxed-constexpr', '-fmad=false',
                           '-DSGS_GEMM_TRACE', '-I', csrc, '-o', exe, src, '-lcuda'])
    return exe


def phases(r, clk_hz):
    """mean clocks per phase over the traced tiles of warpgroup 0 of CTA (0, 0) (both warpgroups work on every tile) from the probe's JSON line"""
    tiles = [s for s in r['trace'][0] if s[TR_EPI_END]]
    n = len(tiles)
    out = dict(ring=sum(s[TR_RING] for s in tiles) / n, kwait=sum(s[TR_KWAIT] for s in tiles) / n,
               issue=sum(s[TR_ISSUED] - s[TR_START] for s in tiles) / n, drain=sum(s[TR_DRAINED] - s[TR_ISSUED] for s in tiles) / n,
               epi=sum(s[TR_EPI_END] - s[TR_DRAINED] for s in tiles) / n, period=(tiles[-1][TR_EPI_END] - tiles[0][TR_START]) / n, tiles=n)
    k8 = -(-r['cin'] // 8) * 8
    out['budget_mma'] = 3.0 * 128 * r['nt'] * k8 / 1024
    out['budget_mem'] = 128 * (r['cin'] + r['cout'] / r['n_tiles']) * 4 / (3.35e12 / 132 / clk_hz)
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--frames', type=int, default=512)
    ap.add_argument('--csrc', default=os.path.join(ROOT, 'sg-slam_b200', 'csrc'), help='the csrc directory whose conv1x1_tc.cuh is traced (laid out like sg-slam_b200/csrc, e.g. a checkout of another revision)')
    ap.add_argument('--json', default=None)
    a = ap.parse_args()
    info = gpu_info()
    try:
        clk_hz = float(info['max_sm_clock'].split()[0]) * 1e6
    except (KeyError, ValueError):
        clk_hz = 1.98e9
    print('# %s' % json.dumps(info))
    rows = []
    with tempfile.TemporaryDirectory() as d:
        exe = build(a.csrc, d)
        for name, cin, cout, side, tail in LAYERS:
            r = json.loads(subprocess.check_output([exe, str(cin), str(cout), str(side), str(side), str(a.frames), str(tail)], text=True).strip())
            r['layer'] = name
            r['phases'] = phases(r, clk_hz)
            rows.append(r)
    print('%-5s %-14s %-20s %7s | %6s %6s %6s %6s %6s %7s | %8s %8s' % (
        'layer', 'K->N @map', 'plan', 'ms', 'ring', 'kwait', 'issue', 'drain', 'epi', 'period', 'mma bud', 'mem bud'))
    for r in rows:
        p = r['phases']
        plan = 'NT%d x%d st%d%s' % (r['nt'], r['n_tiles'], r['stages'], ' wres' if r['wres'] else '')
        print('%-5s %-14s %-20s %7.3f | %6.0f %6.0f %6.0f %6.0f %6.0f %7.0f | %8.0f %8.0f' % (
            r['layer'], '%d->%d @%d' % (r['cin'], r['cout'], r['h']), plan, r['ms'], p['ring'], p['kwait'], p['issue'], p['drain'], p['epi'],
            p['period'], p['budget_mma'], p['budget_mem']))
    print('# clocks per 128-pixel tile (means over the first %d tiles of CTA 0)' % rows[0]['phases']['tiles'])
    if a.json:
        with open(a.json, 'w') as f:
            json.dump(dict(gpu=info, layers=rows), f, indent=1)


if __name__ == '__main__':
    main()
