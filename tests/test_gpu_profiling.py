"""The stage timers of the extractor (5 stages), the LK tracker (2 stages) and the detector (one entry per kernel): with profiling off no call
is counted; enabled, two calls are counted once read back, every total is non-negative and they sum to a positive time; enabling again
starts from zero.  bench.py and the tools read these accessors."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import detector_model as DM  # noqa: E402
from pysgs import binding as B  # noqa: E402
from pysgs import synth  # noqa: E402


def _lk_set_profiling(lk, on):
    B.check(B.lib().sgs_lk_set_profiling(lk.h, int(on)))


def _lk_stage_times(lk):
    ms, n = (C.c_double * 2)(), C.c_int()
    B.check(B.lib().sgs_lk_stage_times(lk.h, ms, C.byref(n)))
    return list(ms), n.value


def _run_twice(call, set_profiling, times, nstages):
    ms, n = times()
    assert n == 0 and len(ms) == nstages and not any(ms)             # off: nothing counted
    call()
    assert times()[1] == 0
    set_profiling(True)
    call(); call()
    ms, n = times()
    assert n == 2 and len(ms) == nstages, (n, len(ms))
    assert min(ms) >= 0 and sum(ms) > 0, ms
    set_profiling(True)                                               # enabling again resets the totals and the count
    ms, n = times()
    assert n == 0 and not any(ms), (n, ms)
    call()
    assert times()[1] == 1


def test_extractor_stage_times():
    img = synth.frame_s1(640, 480, 1)
    ex = B.Extractor(640, 480, 1000, max_batch=1)
    try:
        _run_twice(lambda: ex.extract(img), ex.set_profiling, ex.stage_times, 5)
    finally:
        ex.close()


def test_lk_stage_times(golden_dir):
    g = np.load(os.path.join(golden_dir, 'lk_320x240.npz'))
    lk = B.LK(320, 240)
    try:
        _run_twice(lambda: lk.track(g['cur'], g['prev'], g['pts']), lambda on: _lk_set_profiling(lk, on), lambda: _lk_stage_times(lk), 2)
    finally:
        lk.close()


def test_detector_kernel_times(tmp_path):
    pp, bp = DM.write_mini_model(str(tmp_path), 0)
    det = B.Detector(pp, bp, max_frames=1)
    rgb = DM.synthetic_rgb(480, 640, 1)
    try:
        assert det.num_kernels > 3
        _run_twice(lambda: det.detect(rgb), det.set_profiling, det.kernel_times, det.num_kernels)
    finally:
        det.close()
