"""The oracle of cv::findFundamentalMat(FM_RANSAC) (oracle/fundamental.cpp) on the constructed cases of tests/fm_cases.py: every case's
proof holds on the Python replay of OpenCV's loop, the replay returns what the oracle returns, and the oracle returns what cv2 returned
(tests/golden/fm_cases.npz: F to 1e-9, identical masks, identical emptiness; live cv2 as well when it can be imported).  Cases on which
cv2 4.13 throws (quirk Q15) are not pinned to cv2; there the oracle must still equal the replay."""
import os

import numpy as np
import pytest

import fm_cases as C
import oracle as O

CASES = C.cases()
IDS = [c['name'] for c in CASES]
G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'fm_cases.npz'))
F_TOL = 1e-9


def _oracle(c):
    return O.find_fundamental_ransac(c['m1'], c['m2'], **c['params'])


def test_golden_has_every_case():
    assert list(G['names']) == IDS
    assert str(G['cv2_version']) == '4.13.0'


@pytest.mark.parametrize('case', CASES, ids=IDS)
def test_proof_and_replay_equal_oracle(case):
    tr = C.check_proofs(case)
    F, mask, info = _oracle(case)
    assert (F is None) == (tr['F'] is None)
    if F is not None:
        assert np.array_equal(F, tr['F']) and np.array_equal(mask, tr['mask'])
        assert info[1] == tr['inliers']
    assert info[0] == tr['iterations']


def _against(case, status, Fg, maskg):
    F, mask, _ = _oracle(case)
    if status == 'empty':
        assert F is None
        return
    assert status == 'ok' and F is not None
    Fg = np.asarray(Fg, np.float64)
    assert Fg.shape in ((3, 3), (9, 3))         # exactly 7 pairs: the stacked solutions, the first is returned
    assert np.abs(F - Fg[:3]).max() <= F_TOL * max(1.0, np.abs(Fg[:3]).max())
    assert np.array_equal(mask, maskg)


@pytest.mark.parametrize('case', [c for c in CASES if c['group'] == 'pinned'], ids=[c['name'] for c in CASES if c['group'] == 'pinned'])
def test_oracle_equals_cv2_golden(case):
    k = case['name']
    assert np.array_equal(G[k + '_m1'], case['m1']) and np.array_equal(G[k + '_m2'], case['m2'])
    _against(case, str(G[k + '_status']), G[k + '_F'], G[k + '_mask'])


@pytest.mark.parametrize('case', CASES, ids=IDS)
def test_oracle_equals_live_cv2(case):
    cv2 = pytest.importorskip('cv2')
    p = case['params']
    try:
        F, mask = cv2.findFundamentalMat(case['m1'], case['m2'], cv2.FM_RANSAC, p['thresh'], p['confidence'], p['max_iters'])
    except cv2.error:
        assert case['group'] == 'raises'
        return
    assert case['group'] == 'pinned'
    empty = F is None or F.size == 0
    _against(case, 'empty' if empty else 'ok', F, None if empty else mask.ravel().astype(np.uint8))


def test_paths_covered():
    """Every path the cases are built for has at least one case."""
    paths = {p for c in CASES for p in c['paths']}
    assert {'draw_over_1000', 'draw_over_10000', 'later_draw_fails', 'adaptive_stop', 'tie', 'three_roots', 'max_iters',
            'thresh_normalised', 'confidence_normalised', 'seven', 'collinear', 'empty', 'redraw'} <= paths
    stops = {c['name'] for c in CASES if 'adaptive_stop' in c['paths']}
    assert len(stops) >= 5
