"""pose_opt_kernel (Optimizer::PoseOptimization on the device) against the CPU restatement oracle/pose_opt.cpp on every case of tests/pose_cases.py:
the same inlier count, the same outlier flag on every keypoint holding a map point, and every pose entry within one float32 ulp.  Both sides
compute in FP64 and differ only in summation order (the kernel reduces over the block in a fixed tree), ~1e-12 on the double pose; one ulp is
what rounding that pose to float32 can add.  tests/test_pose_opt_cases.py shows the cases tell plausible one-line slips of the kernel from the
restatement under this bar.

Besides the cases one per frame, the runs cover the layouts the batch entry point accepts: every case in one launch, the cases permuted and repeated
past one wave of 132 blocks (each frame bit-identical to its run alone: the block reduction is deterministic and frames do not interact), scratch
buffers holding garbage, frames with n > cap and n = 0, has_mp values other than 1, the mp_index form with a second point array, and the
single-frame host entry point."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle as O  # noqa: E402
import pose_cases as PC  # noqa: E402
import scenarios as S  # noqa: E402
from pysgs import binding as B  # noqa: E402

CAM = PC.reference_cases()[0][2]['cam']


def _oracle(s):
    c = s['cam']
    return O.pose_optimization(s['T0'], s['has'], s['xyz'], s['xy'], s['octave'], s['uright'], s['inv_s2'], c['fx'], c['fy'], c['cx'], c['cy'], c['bf'])


def _launch(frames, cap=None, n_override=None, scratch_fill=False, index=None):
    """sgs_pose_optimization_batch_device on a list of scenarios, one frame each.  index=None: has_mp form; index=id_base2: mp_index form, keypoint i
    of frame f reading point id f_ids[f][i] (< id_base2: points_xyz, >= id_base2: points2_xyz), taken from each scenario's 'ids' / 'pts' / 'pts2'."""
    import torch
    F = len(frames)
    cap = cap or max(1, max(len(s['xy']) for s in frames))
    cam = B.make_camera(640, 480, CAM, S.scale_factors())
    kps = np.zeros((F, cap), B.KP_DTYPE); ur = np.full((F, cap), -1, np.float32); n = np.zeros(F, np.int32); T0 = np.zeros((F, 16), np.float32)
    has = np.zeros((F, cap), np.uint8)
    for f, s in enumerate(frames):
        m = min(len(s['xy']), cap); n[f] = len(s['xy'])
        kps['x'][f, :m] = s['xy'][:m, 0]; kps['y'][f, :m] = s['xy'][:m, 1]; kps['octave'][f, :m] = s['octave'][:m]; ur[f, :m] = s['uright'][:m]
        T0[f] = s['T0'].reshape(16); has[f, :m] = s['has'][:m]
    if n_override is not None:
        n[:] = n_override
    if index is None:
        pcap, pts = cap, np.zeros((F, cap, 3), np.float32)
        for f, s in enumerate(frames):
            m = min(len(s['xy']), cap); pts[f, :m] = s['xyz'][:m]
    else:
        pcap = max(len(s['pts']) for s in frames); pcap2 = max(len(s['pts2']) for s in frames)
        pts = np.zeros((F, pcap, 3), np.float32); pts2 = np.zeros((F, pcap2, 3), np.float32); idx = np.full((F, cap), -1, np.int32)
        for f, s in enumerate(frames):
            pts[f, :len(s['pts'])] = s['pts']; pts2[f, :len(s['pts2'])] = s['pts2']; idx[f, :len(s['ids'])] = s['ids']
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    keep = [dev(T0), dev(kps.view(np.uint8).reshape(-1)), dev(ur), dev(n), dev(has), dev(pts)]
    Tout = torch.zeros((F, 16), device='cuda'); outl = torch.full((F, cap), 9, dtype=torch.uint8, device='cuda'); nin = torch.full((F,), -7, dtype=torch.int32, device='cuda')
    err = torch.full((F, cap, 3), float('nan') if scratch_fill else 0.0, dtype=torch.float64, device='cuda')
    lvl = torch.full((F, cap), 1 if scratch_fill else 0, dtype=torch.uint8, device='cuda')
    a = B.PoseOptBatch()
    a.cam = cam
    a.tcw_in, a.kps, a.uright, a.n, a.cap = keep[0].data_ptr(), keep[1].data_ptr(), keep[2].data_ptr(), keep[3].data_ptr(), cap
    a.points_xyz, a.point_cap = keep[5].data_ptr(), pcap
    if index is None:
        a.has_mp, a.mp_index = keep[4].data_ptr(), 0
    else:
        keep += [dev(idx), dev(pts2)]
        a.has_mp, a.mp_index = 0, keep[6].data_ptr()
        a.points2_xyz, a.id_base2, a.point2_cap = keep[7].data_ptr(), index, pcap2
    for l in range(PC.NLEVELS):
        a.inv_level_sigma2[l] = float(PC.INV_S2[l])
    a.tcw_out, a.outlier, a.ninliers, a.scratch_err, a.scratch_level = Tout.data_ptr(), outl.data_ptr(), nin.data_ptr(), err.data_ptr(), lvl.data_ptr()
    B.check(B.lib().sgs_pose_optimization_batch_device(C.byref(a), F, C.c_void_p(0)))
    torch.cuda.synchronize()
    return Tout.cpu().numpy().reshape(F, 4, 4), outl.cpu().numpy(), nin.cpu().numpy()


def _check(name, s, T, outl, nin, ref=None):
    """Device result against the restatement; returns the largest ulp distance of the pose."""
    rn, rT, ro = ref if ref is not None else _oracle(s)
    m = len(s['xy']); used = s['has'] != 0
    assert nin == rn, (name, int(nin), rn)
    assert np.array_equal(outl[:m][used], ro[used]), (name, int((outl[:m][used] != ro[used]).sum()))
    ulp = int(PC.ulp_distance(T, rT).max())
    assert ulp <= 1, (name, ulp, float(np.abs(T.astype(np.float64) - rT).max()))
    return ulp


def test_every_case_in_one_launch_within_one_ulp():
    cases = PC.all_cases()
    T, outl, nin = _launch([s for _, _, s in cases])
    worst = {}
    for f, (fam, name, s) in enumerate(cases):
        worst[fam] = max(worst.get(fam, 0), _check(name, s, T[f], outl[f], nin[f]))
    print('largest pose distance in float32 ulps, per family:', worst)


def test_permuted_and_repeated_past_one_wave_bit_identical_to_single_runs():
    cases = [s for _, _, s in PC.all_cases()]
    alone = [_launch([s]) for s in cases]
    order = np.random.RandomState(5).permutation(np.tile(np.arange(len(cases)), 3))[:2 * 132 + 7]
    T, outl, nin = _launch([cases[i] for i in order], cap=1000)
    for f, i in enumerate(order):
        m = len(cases[i]['xy'])
        aT, ao, an = alone[i]
        assert T[f].tobytes() == aT[0].tobytes() and nin[f] == an[0], (f, int(i))
        assert np.array_equal(outl[f, :m], ao[0, :m]), (f, int(i))


def test_scratch_buffers_holding_garbage():
    cases = [c for c in PC.all_cases() if c[0] in ('plain', 'far', 'edges', 'nine', 'farstart', 'levels16')]
    T, outl, nin = _launch([s for _, _, s in cases], scratch_fill=True)
    for f, (_, name, s) in enumerate(cases):
        _check(name, s, T[f], outl[f], nin[f])


def test_n_above_cap_zero_n_and_has_values_other_than_one():
    rs = np.random.RandomState(7)
    base = [S.pose_scenario(600 + k, n=300, outlier_frac=0.25) for k in range(4)]
    cap = 240
    frames, ns, refs = [], [], []
    for k, s in enumerate(base):                          # n = 300 > cap = 240: only the first 240 keypoints take part
        frames.append(s); ns.append(300)
        refs.append(dict(s, xy=s['xy'][:cap], has=s['has'][:cap], xyz=s['xyz'][:cap], octave=s['octave'][:cap], uright=s['uright'][:cap]))
    for k in range(2):                                    # n = 0: nothing to optimise, the input pose comes back with no inlier
        frames.append(base[k]); ns.append(0); refs.append(None)
    for k, s in enumerate(base[:2]):                      # has_mp is a truth value: any non-zero byte holds a map point
        h = np.where(s['has'] != 0, rs.choice(np.array([1, 2, 128, 255], np.uint8), len(s['has'])), 0).astype(np.uint8)
        frames.append(dict(s, has=h, xy=s['xy'][:cap], xyz=s['xyz'][:cap], octave=s['octave'][:cap], uright=s['uright'][:cap]))
        frames[-1]['has'] = h[:cap]; ns.append(cap); refs.append(dict(frames[-1], has=(h[:cap] != 0).astype(np.uint8)))
    T, outl, nin = _launch(frames, cap=cap, n_override=np.array(ns, np.int32))
    for f, r in enumerate(refs):
        if r is None:
            assert nin[f] == 0 and T[f].tobytes() == frames[f]['T0'].astype(np.float32).tobytes(), f
            assert (outl[f] == 9).all(), f               # nothing is written for keypoints beyond n
            continue
        _check(f, r, T[f], outl[f], nin[f])
        assert (outl[f][r['has'] == 0] == 9).all(), f     # keypoints without a map point keep their flag


def _indexed(s, id_base2, rs):
    """s in the mp_index form: each keypoint with a map point reads it by id from one of two point arrays (ids on both sides of id_base2, in a
    shuffled order, with empty slots); keypoints 0 and 1 share one map point (the scenario's xyz is made equal so that the restatement sees the
    same input)."""
    s = dict(s); s['xyz'] = s['xyz'].copy(); s['has'] = s['has'].copy()
    m = len(s['xy'])
    s['has'][:2] = 1; s['xyz'][1] = s['xyz'][0]
    ids = np.full(m, -1, np.int32)
    n1 = m // 2 + 20; n2 = m - m // 2 + 20
    slots = np.r_[rs.permutation(n1)[:m // 2], id_base2 + rs.permutation(n2)[:m - m // 2]]
    slots = slots[rs.permutation(m)]
    pts = np.zeros((n1, 3), np.float32); pts2 = np.zeros((n2, 3), np.float32)
    for i in range(m):
        if s['has'][i]:
            ids[i] = slots[i]
    ids[1] = ids[0]
    for i in range(m):
        if ids[i] >= id_base2:
            pts2[ids[i] - id_base2] = s['xyz'][i]
        elif ids[i] >= 0:
            pts[ids[i]] = s['xyz'][i]
    assert (ids[s['has'] == 1] < id_base2).any() and (ids >= id_base2).any()
    s.update(ids=ids, pts=pts, pts2=pts2)
    return s


def test_mp_index_form_with_a_second_point_array():
    rs = np.random.RandomState(11)
    id_base2 = 100000
    cases = [c for c in PC.all_cases() if c[0] in ('plain', 'hard', 'mono', 'stereo', 'ten', 'farstart', 'levels16')]
    frames = [_indexed(s, id_base2, rs) for _, _, s in cases]
    T, outl, nin = _launch(frames, index=id_base2)
    for f, (_, name, _) in enumerate(cases):
        _check(name, frames[f], T[f], outl[f], nin[f])


def _host(s):
    """sgs_pose_optimization, the single-frame host entry point."""
    m = len(s['xy'])
    kps = np.zeros(m, B.KP_DTYPE); kps['x'] = s['xy'][:, 0]; kps['y'] = s['xy'][:, 1]; kps['octave'] = s['octave']
    T = np.zeros(16, np.float32); outl = np.full(m, 9, np.uint8); nin = C.c_int(-1)
    P = lambda a: np.ascontiguousarray(a).ctypes.data_as(C.c_void_p)
    cam = B.make_camera(640, 480, s['cam'], S.scale_factors())
    B.check(B.lib().sgs_pose_optimization(C.byref(cam), P(s['T0'].astype(np.float32).reshape(16)), m, P(kps), P(s['uright'].astype(np.float32)), P(s['has']),
                                          P(s['xyz'].astype(np.float32)), P(PC.INV_S2), P(T), P(outl), C.byref(nin), 0))
    return T.reshape(4, 4), outl, nin.value


def test_host_entry_point_on_a_subset():
    for fam, name, s in PC.all_cases():
        if fam in ('plain', 'exact', 'behind', 'few', 'nine', 'rejects', 'nbad', 'levels16') or name in ('farstart900_208', 'hard30', 'stereo50'):
            T, outl, nin = _host(s)
            _check(name, s, T, outl, nin)
            assert (outl[s['has'] == 0] == 0).all(), name   # the host entry point clears every flag
