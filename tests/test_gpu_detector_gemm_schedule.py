"""The detector's 1x1-convolution GEMM (conv1x1_tc.cuh) computes the same bits under every schedule: the SHA-256 digests of
tests/golden/detector_gemm_digests.npz (make_golden_detector_gemm.py) were taken on an H100 with the one-CTA-per-SM schedule that stored each
channel group right after its tail.  Today narrow tiles (32 output channels) run two CTAs per SM with their own register budget and a ring that
fits half an SM's shared memory; every conv1x1 output blob of every frame (diagnostic mode) and the detection rows and objects of the fused tails
must still match.

The probe graph reaches both schedules (narrow: 16 -> 32 at 150x150 with about ten pixel tiles per CTA, the 1- to 32-channel expansions and probes;
wide: the 36- to 1000-channel ones), odd pitches and scalar stores, partial last pixel tiles, and a 3-frame call on a handle that
ran 8 frames before.  The tail graph puts every fused tail kind on a narrow GEMM; the
narrow32 graph has narrow tiles with 32-float k-blocks, resident and streamed (672 -> 16) weights."""
import os

import numpy as np
import pytest

import detector_gemm_digests as DG
import detector_model as DM
from pysgs import binding as B

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'detector_gemm_digests.npz')


def _narrow(p):
    return p['nt'] <= 32


def test_narrow_plans_fit_two_ctas_per_sm(tmp_path):
    """CPU: narrow plans (N-tiles of 32 channels) take at most 110 KB of shared memory, so that two CTAs
    share an SM; the probe graphs have narrow plans of both k-block widths (with resident and streamed weights) and wide ones, and wide plans keep the
    128 KB rule for resident weights."""
    plans = []
    for sub, probes in (('probe', DM.GEMM_PROBES), ('narrow32', DG.NARROW32_PROBES)):
        pp, bp, _ = DM.write_probe_model(str(tmp_path / sub), probes, 0)
        det = B.Detector(pp, bp, max_frames=DM.PROBE_FRAMES, flags=B.DET_PLAN_ONLY)
        plans += DM.parse_plan(det.describe())
        det.close()
    kinds = {(_narrow(p), p['bk']) for p in plans}
    assert kinds >= {(True, 16), (True, 32), (False, 32)}, kinds
    assert any(_narrow(p) and p['bk'] == 32 and not p['wres'] and p['kb'] > p['stages'] for p in plans)
    for p in plans:
        if _narrow(p):
            assert p['smem'] <= 110 * 1024 and p['stages'] >= 2, p['line']
        wb = p['kb'] * 2 * p['nt'] * p['bk'] * 4
        if not _narrow(p):
            assert p['wres'] == (wb <= 128 * 1024), p['line']


@pytest.mark.gpu
def test_gemm_outputs_match_the_golden_digests(tmp_path):
    from test_gpu_detector import _run
    gold = np.load(GOLDEN)
    got = DG.flatten(DG.compute(B, _run, str(tmp_path)))
    assert sorted(got) == sorted(gold.files)
    bad = [k for k in sorted(got) if not np.array_equal(got[k], gold[k])]
    assert not bad, 'outputs differ from the golden digests in %s' % ', '.join(bad)

