"""The dynamic-feature rejection's constructed cases (tests/dynreject_cases.py) on the CPU: every case's proof holds, the oracle's sgo_dynreject
equals the restatement on every case (verdicts, distance bits, kept count, restore flag), and -- when oracle/_ref/libframe_ref.so was built
from the reference tree -- the restatement's per-keypoint tests equal the reference's own Frame::CheckEpiLineDistToRmDynamicPoint and
Frame::isInDynamicRegion on every keypoint of every case.  No device needed; tests/test_gpu_dynreject_cases.py runs the same cases through
the device entry points."""
import ctypes as C
import os

import numpy as np
import pytest

import dynreject_cases as D
import oracle as O

NAMES = [c['name'] for c in D.CASES]
REF_LIB = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle', '_ref', 'libframe_ref.so')


def same_dist(got, want):
    """Distances equal bit for bit, NaN where NaN (a NaN's payload is not part of the result)."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.uint64), want[~nan].view(np.uint64))


@pytest.mark.parametrize('name', NAMES)
def test_case_takes_its_path(name):
    D.BY_NAME[name]['proof']()


def test_cases_cover_every_family():
    prefixes = {n.split('_')[0] for n in NAMES}
    assert prefixes == {'epi', 'box', 'boxes', 'restore', 'F', 'prev', 'shape'}
    assert sum(n.startswith('epi_general_F_') for n in NAMES) == 2 * len(D.VARIANTS)
    assert {c['count'] for c in D.CASES if c['count'] != len(c['cur'])} == {-5, 1500}


@pytest.mark.parametrize('name', NAMES)
def test_oracle_equals_restatement(name):
    c = D.BY_NAME[name]
    s, keep, dist, restored = O.dynreject(c['cur'], c['prev'], c['F'], D.single_frame_boxes(c), c['have_dyn'], c['nfeatures'])
    assert np.array_equal(keep, c['keep']) and same_dist(dist, c['dist'])
    assert s == c['nkeep'] and restored == c['restored']


@pytest.fixture(scope='module')
def ref():
    if not os.path.exists(REF_LIB):
        pytest.skip('oracle/_ref/libframe_ref.so not built (reference tree absent)')
    L = C.CDLL(REF_LIB)
    if not (hasattr(L, 'ref_frame_check_epi_line_dist') and hasattr(L, 'ref_frame_is_in_dynamic_region')):
        # a library built from an older oracle/frame_ref_driver.cpp, where the reference tree is out of reach of this build to redo it
        pytest.skip('oracle/_ref/libframe_ref.so predates the per-keypoint wrappers of oracle/frame_ref_driver.cpp (rebuild it from the reference tree)')
    L.ref_frame_check_epi_line_dist.restype = C.c_int
    L.ref_frame_check_epi_line_dist.argtypes = [C.c_float, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_double]
    L.ref_frame_is_in_dynamic_region.restype = C.c_int
    L.ref_frame_is_in_dynamic_region.argtypes = [C.c_float, C.c_float, C.c_void_p, C.c_int]
    return L


@pytest.mark.parametrize('name', [n for n in NAMES if not n.startswith('shape_')] + ['shape_n257_runs'])
def test_restatement_equals_reference_frame(ref, name):
    """Both of the reference's per-keypoint tests, called on every keypoint, against the restatement's."""
    c = D.BY_NAME[name]
    boxes = np.ascontiguousarray(D.single_frame_boxes(c), np.float32)
    inside = D.in_any_box(c['cur'], boxes, len(boxes))
    for i, ((x, y), (px, py)) in enumerate(zip(c['cur'], c['prev'])):
        assert ref.ref_frame_is_in_dynamic_region(x, y, boxes.ctypes.data, len(boxes)) == inside[i], (name, i)
    if c['F'] is None:
        return
    F = np.ascontiguousarray(c['F'], np.float64)
    d = D.epi_dist(c['cur'], c['prev'], F)
    for thr in (D.IN_BOX, D.OUT_BOX):
        got = [ref.ref_frame_check_epi_line_dist(x, y, px, py, F.ctypes.data, thr) for (x, y), (px, py) in zip(c['cur'], c['prev'])]
        assert got == (d < thr).astype(int).tolist(), (name, thr)
