"""SHA-256 digests of what the detector's 1x1-convolution GEMM (conv1x1_tc.cuh) writes, on seeded synthetic graphs (tests/detector_model.py), for
tests/golden/make_golden_detector_gemm.py (which stores them) and tests/test_gpu_detector_gemm_schedule.py (which requires them bit for bit).

  diagnostic mode (every blob of every frame kept, tails run as kernels of their own): per frame, the output blob of every conv1x1 line of the plan
    - probe   : write_probe_model(GEMM_PROBES, seed 0) at PROBE_FRAMES frames
    - tails   : write_tail_model(seed 0), 3 frames of a 4-frame handle
    - short   : write_probe_model(GEMM_PROBES, seed 2): a full batch, then 3 frames on the same handle (the last pixel tile runs over stale rows)
    - narrow32: write_probe_model(NARROW32_PROBES, seed 5): at most 32 output channels from more than 16 input channels (32-float k-blocks), with
                resident and streamed weights
  fused mode (tails inside the GEMM epilogue): per frame, the detection rows, their count and the accepted objects at a low threshold (0.05), so that
  many boxes reach the rows
    - fused_probe, fused_tails, fused_narrow32 : the graphs above"""
import hashlib

import numpy as np

import detector_model as DM

DET_THR = 0.05
NARROW32_PROBES = [('gemm', 20, 24, 150), ('gemm', 72, 24, 75), ('gemm', 40, 10, 38), ('gemm', 112, 28, 19), ('gemm', 672, 16, 19)]


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def frames(seeds):
    return np.stack([DM.synthetic_rgb(480, 640, s) for s in seeds])


def _gemm_lines(det):
    return [p['name'] for p in DM.parse_plan(det.describe())]


def _diag(B, run, pp, bp, batches, max_frames):
    det = B.Detector(pp, bp, max_frames=max_frames, flags=B.DET_DIAGNOSTIC)
    for fr in batches:
        run(det, fr)
    nf = len(batches[-1])
    out = {n: np.array([sha(det.blob(n, f)) for f in range(nf)]) for n in _gemm_lines(det)}
    det.close()
    return out


def _fused(B, run, pp, bp, fr, max_frames):
    det = B.Detector(pp, bp, max_frames=max_frames, det_thr=DET_THR)
    o = run(det, fr)
    det.close()
    n = o['nrows']
    return {'rows': np.array([sha(o['rows'][f, :n[f]]) for f in range(len(fr))]), 'nrows': n.astype(np.int64),
            'objects': np.array([sha(o['objects'][f, :o['nobjects'][f]]) for f in range(len(fr))])}


def compute(B, run, workdir):
    """{case: {key: per-frame array}}.  B: pysgs.binding, run: test_gpu_detector._run, workdir: a directory for the generated graphs."""
    import os
    res = {}
    pp, bp, _ = DM.write_probe_model(os.path.join(workdir, 'probe'), DM.GEMM_PROBES, 0)
    full = frames(range(31, 31 + DM.PROBE_FRAMES))
    res['probe'] = _diag(B, run, pp, bp, [full], DM.PROBE_FRAMES)
    res['fused_probe'] = _fused(B, run, pp, bp, full, DM.PROBE_FRAMES)
    tp, tb = DM.write_tail_model(os.path.join(workdir, 'tails'), 0)
    tf = frames((61, 62, 63))
    res['tails'] = _diag(B, run, tp, tb, [tf], 4)
    res['fused_tails'] = _fused(B, run, tp, tb, tf, 4)
    sp, sb, _ = DM.write_probe_model(os.path.join(workdir, 'short'), DM.GEMM_PROBES, 2)
    res['short'] = _diag(B, run, sp, sb, [frames(range(41, 41 + DM.PROBE_FRAMES)), frames((51, 52, 53))], DM.PROBE_FRAMES)
    np_, nb, _ = DM.write_probe_model(os.path.join(workdir, 'narrow32'), NARROW32_PROBES, 5)
    nf = frames(range(91, 91 + DM.PROBE_FRAMES))
    res['narrow32'] = _diag(B, run, np_, nb, [nf], DM.PROBE_FRAMES)
    res['fused_narrow32'] = _fused(B, run, np_, nb, nf, DM.PROBE_FRAMES)
    return res


def flatten(res):
    return {'%s/%s' % (c, k): v for c, d in res.items() for k, v in d.items()}
