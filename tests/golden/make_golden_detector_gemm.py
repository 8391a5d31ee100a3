#!/usr/bin/env python3
"""Golden digests of the detector's 1x1-convolution GEMM outputs (tests/detector_gemm_digests.py) on seeded synthetic graphs: every conv1x1 output
blob per frame in diagnostic mode, and the detection rows / objects per frame in fused mode.  Taken on an H100 with the kernel schedule these
digests were first recorded from; any later schedule must reproduce them bit for bit (tests/test_gpu_detector_gemm_schedule.py).
Run on the GPU after build():  python tests/golden/make_golden_detector_gemm.py"""
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, 'sg-slam_b200'), os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import detector_gemm_digests as DG  # noqa: E402
from pysgs import binding as B  # noqa: E402
from test_gpu_detector import _run  # noqa: E402


def main():
    out = sys.argv[1] if len(sys.argv) > 1 else os.path.join(HERE, 'detector_gemm_digests.npz')
    with tempfile.TemporaryDirectory() as d:
        flat = DG.flatten(DG.compute(B, _run, d))
    np.savez_compressed(out, **flat)
    print('%d entries written to %s' % (len(flat), out))


if __name__ == '__main__':
    main()
