"""The device findFundamentalMat (sg-slam_b200/csrc/fundamental.cu) on the constructed cases of tests/fm_cases.py, through both entry points.
Every case must give what the Python replay of OpenCV's loop gives (itself equal to the oracle and, outside the cases where cv2 4.13 throws,
to cv2; tests/test_fundamental_cases.py): F to 1e-9, the same mask, and info = {pairs, inliers, iterations, status}.  On the cases where
cv2 throws (quirk Q15) a drawn sample has six collinear points, its 7x9 system has rank below 7 and any member of the larger null space
solves it: there the device's F is not pinned (its Gram-Schmidt completion picks another member than the oracle's Jacobi completion),
but it must be defined -- finite, or NaN with status 2 -- and the mask and info must still be the oracle's.

The batched launch carries every case as one frame of the sgs_keypoint layout, next to frames that exercise the launch itself: a frame
without a previous frame (status 3), fewer than 7 pairs, 12800 pairs (the 200 KB shared-memory limit) and the same frame with counts
above cap, and pair selections behind the previous frame's boxes that leave exactly 20 and 21 pairs or put points on a box's edges."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import fm_cases as C  # noqa: E402
import oracle as O  # noqa: E402
from pysgs import binding as B  # noqa: E402

CASES = C.cases()
IDS = [c['name'] for c in CASES]
F_TOL = 1e-9
CAP_MAX = 200 * 1024 // 16          # pairs per frame that fit the kernel's shared memory


def expected(m1, m2, thresh=1.0, confidence=0.99, max_iters=1000):
    """(F or None, mask, info[4]) of the replay, in the device's info layout."""
    tr = C.replay(m1, m2, thresh, confidence, max_iters)
    n = len(m1)
    status = 1 if n < 7 else (2 if tr['F'] is None else 0)
    return tr['F'], tr['mask'], np.array([n, tr['inliers'], tr['iterations'], status], np.int32)


def _same_F(F, Fref):
    return np.abs(F - Fref).max() <= F_TOL * max(1.0, np.abs(Fref).max())


def _check(F, info, want, name, pin_F=True):
    """F: the device's 3x3 output, NaN for "no matrix"."""
    Fw, _, iw = want
    assert np.array_equal(info, iw), (name, info, iw)
    if Fw is None:
        assert np.isnan(F).all() and info[3] != 0, name
    else:
        assert np.isfinite(F).all() and info[3] == 0, name
        assert _same_F(F, Fw) or not pin_F, name


@pytest.fixture(scope='module')
def want():
    return {c['name']: expected(c['m1'], c['m2'], **c['params']) for c in CASES}


@pytest.mark.parametrize('case', CASES, ids=IDS)
def test_single_frame_entry(case, want):
    F, mask, info = B.fundamental_ransac(case['m1'], case['m2'], **case['params'])
    w = want[case['name']]
    _check(np.full((3, 3), np.nan) if F is None else F, info, w, case['name'], case['group'] == 'pinned')
    assert np.array_equal(mask, w[1]), case['name']


def test_refuses_more_pairs_than_shared_memory_holds():
    import torch
    z = lambda nbytes: torch.zeros(nbytes, dtype=torch.uint8, device='cuda')
    kps, prev, cnt, F, info = z(28 * (CAP_MAX + 1)), z(8 * (CAP_MAX + 1)), z(4), z(72), z(16)
    with pytest.raises(B.SgsError) as e:
        B.fundamental_batch_device(kps.data_ptr(), prev.data_ptr(), cnt.data_ptr(), CAP_MAX + 1, 1, 0, 0, 0, 0, 0, F.data_ptr(), info.data_ptr())
    assert e.value.code == B.SGS_ERR_UNSUPPORTED


BOX = np.array([100.0, 100.0, 200.0, 200.0], np.float32)          # x, y, w, h: 100 < x < 300, 100 < y < 300 is inside


def _box_frame(seed, inside, outside, on_edge):
    """Previous points: `inside` strictly inside BOX, `outside` well outside, `on_edge` exactly on its four edges (kept: the test is
    strict); current points are the previous ones moved by a few pixels."""
    rs = np.random.RandomState(seed)
    prev = [rs.uniform(120, 280, (inside, 2)), np.c_[rs.uniform(320, 620, outside), rs.uniform(20, 460, outside)]]
    e = np.rint(rs.uniform(120, 280, on_edge))
    edge = np.array([[(100.0, v), (300.0, v), (v, 100.0), (v, 300.0)][i % 4] for i, v in enumerate(e)]).reshape(-1, 2)
    prev = np.concatenate(prev + [edge]).astype(np.float32)[rs.permutation(inside + outside + on_edge)]
    cur = (prev + rs.normal(0, 2.0, prev.shape) + np.array([3.0, -1.0])).astype(np.float32)
    return cur, prev


def _launch(frames, cap, params):
    """frames: list of dict(cur, prev, count, prev_index, have_dyn, boxes).  Returns (F [nf, 3, 3], info [nf, 4])."""
    import torch
    nf = len(frames)
    kps = np.zeros((nf, cap), O.KP_DTYPE); prev = np.zeros((nf, cap, 2), np.float32)
    counts = np.zeros(nf, np.int32); pidx = np.zeros(nf, np.int32); have = np.zeros(nf, np.uint8)
    boxes = np.zeros((nf, 1, 4), np.float32); nboxes = np.zeros(nf, np.int32)
    for f, fr in enumerate(frames):
        n = len(fr['cur'])
        kps['x'][f, :n] = fr['cur'][:, 0]; kps['y'][f, :n] = fr['cur'][:, 1]; prev[f, :n] = fr['prev']
        counts[f] = fr.get('count', n); pidx[f] = fr.get('prev_index', 0); have[f] = fr.get('have_dyn', 0)
        if fr.get('have_dyn'):
            boxes[f, 0] = BOX; nboxes[f] = 1
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()
    d = [dev(a) for a in (kps, prev, counts, boxes, nboxes, have, pidx)]
    d_F = torch.full((nf * 9,), -7.0, dtype=torch.float64, device='cuda'); d_info = torch.full((nf * 4,), -7, dtype=torch.int32, device='cuda')
    B.fundamental_batch_device(d[0].data_ptr(), d[1].data_ptr(), d[2].data_ptr(), cap, nf, d[3].data_ptr(), d[4].data_ptr(), d[5].data_ptr(), 1,
                               d[6].data_ptr(), d_F.data_ptr(), d_info.data_ptr(), **params)
    torch.cuda.synchronize()
    return d_F.cpu().numpy().reshape(nf, 3, 3), d_info.cpu().numpy().reshape(nf, 4)


def _param_key(p):
    return (p['thresh'], p['confidence'], p['max_iters'])


def test_batched_launch(want):
    """Frame 0 has no previous frame; frame 1 holds the boxes (its own previous frame is frame 0, so they filter); every other frame's
    previous frame is 0 (no boxes) unless it is a box frame (previous frame 1)."""
    cap = CAP_MAX
    big_cur, big_prev = C.two_view(7, cap, 0.5, 0.3)
    few_cur, few_prev = C.two_view(8, 5, 0.3, 0.0)
    b20, b21, bedge = _box_frame(1, 20, 20, 0), _box_frame(2, 20, 21, 0), _box_frame(3, 10, 18, 12)
    base = [dict(cur=few_cur, prev=few_prev, prev_index=0),                                   # 0: no previous frame -> status 3
            dict(cur=few_cur, prev=few_prev, prev_index=0, have_dyn=1),                       # 1: fewer than 7 pairs; holds the boxes
            dict(cur=big_cur, prev=big_prev, prev_index=0),                                   # 2: 12800 pairs
            dict(cur=big_cur, prev=big_prev, prev_index=0, count=cap + 1000),                 # 3: counts > cap: clipped to cap
            dict(cur=b20[0], prev=b20[1], prev_index=1),                                      # 4: 20 pairs outside the box -> all 40
            dict(cur=b21[0], prev=b21[1], prev_index=1),                                      # 5: 21 outside -> those 21
            dict(cur=bedge[0], prev=bedge[1], prev_index=1)]                                  # 6: 12 on the edges are outside -> 30
    sel = []
    for fr in base[4:]:
        s1, s2 = O.select_static_pairs(fr['cur'], fr['prev'], BOX[None], True)
        sel.append((s1, s2))
    assert [len(s[0]) for s in sel] == [40, 21, 30]
    groups = {}
    for c in CASES:
        groups.setdefault(_param_key(c['params']), []).append(c)
    for key, cs in groups.items():
        params = dict(thresh=key[0], confidence=key[1], max_iters=key[2])
        default = key == _param_key(C.DEFAULT)
        frames = (base if default else base[:1]) + [dict(cur=c['m1'], prev=c['m2'], prev_index=0) for c in cs]
        F, info = _launch(frames, cap if default else max(len(fr['cur']) for fr in frames), params)
        assert info[0, 3] == 3 and np.isnan(F[0]).all()
        off = len(frames) - len(cs)
        for j, c in enumerate(cs):
            _check(F[off + j], info[off + j], want[c['name']], c['name'], c['group'] == 'pinned')
        if not default:
            continue
        assert info[1, 0] == 5 and info[1, 3] == 1 and np.isnan(F[1]).all()
        w = expected(big_cur, big_prev)
        for f in (2, 3):
            _check(F[f], info[f], w, f'frame {f}')
        for f, (s1, s2) in zip((4, 5, 6), sel):
            _check(F[f], info[f], expected(s1, s2), f'frame {f}')
        F2, info2 = _launch(frames, cap, params)                     # a repeat launch gives the same bytes
        assert F2.tobytes() == F.tobytes() and info2.tobytes() == info.tobytes()
