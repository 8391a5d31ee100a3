"""The constructed bag-of-words cases of tests/bow_cases.py through the BATCHED device entry points sgs_bow_transform_batch_device and
sgs_match_bow_batch_device (all three modes), every case one frame of a launch.

Each matcher launch groups the cases that share the per-launch scalars (mode, nnratio, orientation check, only_stereo) and adds a frame
whose first side has count 0, one whose second side has count 0, and one whose counts exceed both caps (the kernel clamps them).  The caps
are the largest counts plus padding, once with kf_cap < f_cap and once the other way; the rows past each frame's counts hold copies of its
rows (what a kernel reading past a count would find and match), every output starts as a sentinel.  Required: every frame equals the
oracle exactly (matches and counts; the reference's own ORBmatcher.cc too where it was built), the case's proof holds, and every match_f
row past the count is -1.  Further: caps of 1, 4097 (just past a power of two) and 8192 on both sides with one full bucket (about 200 KB of
dynamic shared memory), 8193 refused without a launch, a node with 4096 children accepted and one with 4097 refused.  The transform runs on
every constructed tree (ORBvoc's shape included) and on one trained by DBoW2's own `create`: word, weight (bit pattern) and node equal the
oracle for every levelsup, padding rows keep their sentinels.  The host wrappers give the same results, and a repeated launch the same bytes."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import bow_cases as BC  # noqa: E402
import oracle as O  # noqa: E402
import test_bow_cases as TB  # noqa: E402
import test_gpu_bow as TG  # noqa: E402
from pysgs import binding as B  # noqa: E402

SENT = np.int32(0x5A5A5A5A)
SENT_W = -7.25
V = C.c_void_p
SIDE_A = ('node', 'weight', 'valid', 'desc', 'angle', 'stereo', 'xy')
SIDE_B = SIDE_A + ('octave',)


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


def _pad(rows, cap):
    """[cap, ...]: `rows` (at most cap of them), then the rows repeated."""
    rows = np.asarray(rows)
    out = np.zeros((cap,) + rows.shape[1:], rows.dtype)
    n = min(len(rows), cap)
    out[:n] = rows[:n]
    if n:
        out[n:] = rows[np.arange(cap - n) % n]
    return out


def _reference():
    return TB._matcher() if os.path.exists(TB.MATCHER_SO) else None


def frame(c, na=None, nb=None, proof=True):
    return dict(c=c, na=len(c['a']['node']) if na is None else na, nb=len(c['b']['node']) if nb is None else nb, proof=proof)


def launch(frames, kf_cap, f_cap):
    """One sgs_match_bow_batch_device call: returns (match_f [F][out cap], nmatches [F], padded sides) on the host."""
    import torch
    c0 = frames[0]['c']
    mode, p = c0['mode'], c0['params']
    pa = {k: np.stack([_pad(f['c']['a'][k], kf_cap) for f in frames]) for k in SIDE_A}
    pb = {k: np.stack([_pad(f['c']['b'][k], f_cap) for f in frames]) for k in SIDE_B}
    t = {('a', k): _dev(v) for k, v in pa.items()}
    t.update({('b', k): _dev(v) for k, v in pb.items()})
    na = _dev(np.array([f['na'] for f in frames], np.int32)); nb = _dev(np.array([f['nb'] for f in frames], np.int32))
    F12 = _dev(np.stack([f['c']['F12'].reshape(9) for f in frames])); ep = _dev(np.array([[f['c']['ex'], f['c']['ey']] for f in frames], np.float32))
    out_cap = f_cap if mode == 0 else kf_cap
    m = torch.full((len(frames), out_cap), int(SENT), dtype=torch.int32, device='cuda'); nm = torch.full((len(frames),), int(SENT), dtype=torch.int32, device='cuda')
    a = B.BowBatch()
    a.kf_node, a.kf_weight, a.kf_valid, a.kf_desc, a.kf_angle, a.kf_n, a.kf_cap = (t['a', 'node'].data_ptr(), t['a', 'weight'].data_ptr(), t['a', 'valid'].data_ptr(),
                                                                                   t['a', 'desc'].data_ptr(), t['a', 'angle'].data_ptr(), na.data_ptr(), kf_cap)
    a.f_node, a.f_weight, a.f_desc, a.f_angle, a.f_n, a.f_cap = (t['b', 'node'].data_ptr(), t['b', 'weight'].data_ptr(), t['b', 'desc'].data_ptr(),
                                                                 t['b', 'angle'].data_ptr(), nb.data_ptr(), f_cap)
    a.f_valid = t['b', 'valid'].data_ptr() if mode else None
    a.keyframe_pair, a.nnratio, a.check_orientation, a.only_stereo = mode, p['nnratio'], p['check_ori'], p['only_stereo']
    if mode == 2:
        a.kf_stereo, a.f_stereo, a.kf_xy, a.f_xy, a.f_octave = (t['a', 'stereo'].data_ptr(), t['b', 'stereo'].data_ptr(), t['a', 'xy'].data_ptr(),
                                                                t['b', 'xy'].data_ptr(), t['b', 'octave'].data_ptr())
        a.F12, a.epipole = F12.data_ptr(), ep.data_ptr()
        for l in range(len(BC.SF)):
            a.level_sigma2[l] = float(BC.SIGMA2[l]); a.scale_factors[l] = float(BC.SF[l])
    a.match_f, a.nmatches = m.data_ptr(), nm.data_ptr()
    B.check(B.lib().sgs_match_bow_batch_device(C.byref(a), len(frames), V(0)))
    return _host(m), _host(nm), pa, pb


def check(frames, kf_cap, f_cap, ref=None):
    m, nm, pa, pb = launch(frames, kf_cap, f_cap)
    for i, f in enumerate(frames):
        c = f['c']
        na, nb = min(f['na'], kf_cap), min(f['nb'], f_cap)
        sa = {k: v[i, :na] for k, v in pa.items()}; sb = {k: v[i, :nb] for k, v in pb.items()}
        o = BC.run_arrays(c['mode'], c['params'], sa, sb, c)
        n_out = nb if c['mode'] == 0 else na
        assert nm[i] == o['nm'] and np.array_equal(m[i, :n_out], o['m']), (c['name'], i, nm[i], o['nm'], np.nonzero(m[i, :n_out] != o['m'])[0][:8])
        assert (m[i, n_out:] == -1).all(), (c['name'], i, 'rows past the count must be -1')
        if ref is not None and na and nb:
            r = TB.ref_arrays(ref, c['mode'], c['params'], sa, sb, c)
            assert r['nm'] == nm[i] and np.array_equal(r['m'], m[i, :n_out]), (c['name'], 'reference')
        if f['proof'] and na == len(c['a']['node']) and nb == len(c['b']['node']):
            c['proof'](o)
    return m, nm


def _groups():
    out = {}
    for n in BC.names():
        c = BC.CASES[n]
        out.setdefault((c['mode'], tuple(sorted(c['params'].items()))), []).append(n)
    return list(out.values())


GROUPS = _groups()


def _frames(names):
    cs = [BC.CASES[n] for n in names]
    fr = [frame(c) for c in cs]
    fr += [frame(cs[0], na=0), frame(cs[0], nb=0)]
    return fr


@pytest.mark.parametrize('layout', ['kf_lt_f', 'kf_gt_f'])
@pytest.mark.parametrize('names', GROUPS, ids=['%s+%d' % (g[0], len(g) - 1) for g in GROUPS])
def test_matcher_cases_batched(names, layout):
    """Every constructed case as one frame of a launch, with count-0 frames and a frame whose counts exceed the caps."""
    fr = _frames(names)
    ma = max(len(f['c']['a']['node']) for f in fr); mb = max(len(f['c']['b']['node']) for f in fr)
    if layout == 'kf_lt_f':
        kf_cap = ma + 37; f_cap = max(mb, kf_cap) + 11
    else:
        f_cap = mb + 37; kf_cap = max(ma, f_cap) + 11
    assert (kf_cap < f_cap) == (layout == 'kf_lt_f')
    fr.append(frame(fr[0]['c'], na=kf_cap + 9, nb=f_cap + 9, proof=False))
    check(fr, kf_cap, f_cap, _reference())


@pytest.mark.parametrize('mode', [0, 1, 2])
def test_caps_of_one(mode):
    fr = [frame(BC.tiny(mode, 20)), frame(BC.tiny(mode, 51)), frame(BC.tiny(mode, 20), na=0), frame(BC.tiny(mode, 20), na=5, nb=5)]
    m, nm = check(fr, 1, 1, _reference())
    assert list(nm) == [1, 0, 0, 1]


@pytest.mark.parametrize('mode', [0, 1, 2])
def test_cap_4097(mode):
    """One side past 4096 (the bitonic arrays pad to 8192): the full root bucket with 4097 features a side, and a clamped copy."""
    c = BC.full_bucket(mode, 2048, extra=1)
    assert len(c['a']['node']) == len(c['b']['node']) == 4097
    check([frame(c), frame(c, na=5000, nb=4097 + 3, proof=False), frame(c, nb=0)], 4097, 4097)


@pytest.mark.parametrize('mode', [0, 1, 2])
def test_full_bucket_at_8192(mode):
    """8192 features on both sides, all in the root bucket: the largest shared-memory configuration (about 200 KB)."""
    c = BC.full_bucket(mode, 4096)
    m, nm = check([frame(c), frame(c, na=0)], 8192, 8192, _reference())
    assert nm[0] == 8192


@pytest.mark.parametrize('side', ['kf', 'f'])
def test_8193_features_are_refused(side):
    import torch
    kf_cap, f_cap = (8193, 8192) if side == 'kf' else (8192, 8193)
    z = lambda n, shape=(), dt=torch.int32: torch.zeros((n,) + shape, dtype=dt, device='cuda')
    t = dict(kn=z(kf_cap), kw=z(kf_cap, (), torch.float64), kv=z(kf_cap, (), torch.uint8), kd=z(kf_cap, (32,), torch.uint8), ka=z(kf_cap, (), torch.float32),
             fn=z(f_cap), fw=z(f_cap, (), torch.float64), fd=z(f_cap, (32,), torch.uint8), fa=z(f_cap, (), torch.float32), c=torch.ones(2, dtype=torch.int32, device='cuda'))
    m = torch.full((max(kf_cap, f_cap),), int(SENT), dtype=torch.int32, device='cuda'); nm = torch.full((1,), int(SENT), dtype=torch.int32, device='cuda')
    a = B.BowBatch()
    a.kf_node, a.kf_weight, a.kf_valid, a.kf_desc, a.kf_angle, a.kf_n, a.kf_cap = t['kn'].data_ptr(), t['kw'].data_ptr(), t['kv'].data_ptr(), t['kd'].data_ptr(), t['ka'].data_ptr(), t['c'].data_ptr(), kf_cap
    a.f_node, a.f_weight, a.f_desc, a.f_angle, a.f_n, a.f_cap = t['fn'].data_ptr(), t['fw'].data_ptr(), t['fd'].data_ptr(), t['fa'].data_ptr(), t['c'].data_ptr() + 4, f_cap
    a.nnratio, a.check_orientation, a.match_f, a.nmatches = 0.7, 1, m.data_ptr(), nm.data_ptr()
    assert B.lib().sgs_match_bow_batch_device(C.byref(a), 1, V(0)) == B.SGS_ERR_UNSUPPORTED
    assert (_host(m) == SENT).all() and _host(nm)[0] == SENT, 'nothing launched'


@pytest.mark.parametrize('k,rc', [(4096, B.SGS_OK), (4097, B.SGS_ERR_UNSUPPORTED)])
def test_vocabulary_child_limit(k, rc):
    parent = np.array([-1] + [0] * k, np.int32); desc = np.random.RandomState(k).randint(0, 256, (k + 1, 32)).astype(np.uint8); w = np.ones(k + 1)
    h = V()
    assert B.lib().sgs_vocabulary_create(0, 10, 1, k + 1, parent.ctypes.data_as(V), desc.ctypes.data_as(V), w.ctypes.data_as(V), C.byref(h)) == rc
    if rc == B.SGS_OK:
        B.lib().sgs_vocabulary_destroy(h)
    else:
        assert not h.value


class GpuVoc(B._Handle):
    def __init__(self, v):
        p = lambda a: np.ascontiguousarray(a).ctypes.data_as(V)
        super().__init__(B.lib().sgs_vocabulary_create, B.lib().sgs_vocabulary_destroy, 0, max(int(v['k']), 2), v['L'], len(v['parent']),
                         p(np.asarray(v['parent'], np.int32)), p(np.asarray(v['desc'], np.uint8)), p(np.asarray(v['weight'], np.float64)))


def transform_batched(gv, q, levelsup):
    """Three frames: the queries, count 0, and count above the cap (clamped); rows past each count are copies and must keep the sentinels."""
    import torch
    n = len(q); cap = n + 13
    desc = np.stack([_pad(q, cap)] * 3)
    counts = np.array([n, 0, cap + 5], np.int32)
    dd, dc = _dev(desc), _dev(counts)
    word = torch.full((3, cap), int(SENT), dtype=torch.int32, device='cuda'); w = torch.full((3, cap), SENT_W, dtype=torch.float64, device='cuda')
    node = torch.full((3, cap), int(SENT), dtype=torch.int32, device='cuda')
    B.check(B.lib().sgs_bow_transform_batch_device(gv.h, V(dd.data_ptr()), V(dc.data_ptr()), cap, 3, levelsup, V(word.data_ptr()), V(w.data_ptr()), V(node.data_ptr()), V(0)))
    return _host(word), _host(w), _host(node), desc[0]


def _check_transform(v, levelsups):
    gv = GpuVoc(v)
    try:
        Vo = O.Vocabulary(v['k'], v['L'], v['parent'], v['desc'], v['weight'])
        res = {}
        for ls in levelsups:
            word, w, node, padded = transform_batched(gv, v['queries'], ls)
            n, cap = len(v['queries']), word.shape[1]
            for f, cnt in ((0, n), (2, cap)):
                ow, owt, on = Vo.transform(padded[:cnt], ls)
                assert np.array_equal(word[f, :cnt], ow) and w[f, :cnt].tobytes() == owt.tobytes() and np.array_equal(node[f, :cnt], on), (v['name'], ls, f)
            assert (word[0, n:] == SENT).all() and (w[0, n:] == SENT_W).all() and (node[0, n:] == SENT).all(), (v['name'], 'padding rows written')
            assert (word[1] == SENT).all() and (w[1] == SENT_W).all() and (node[1] == SENT).all(), (v['name'], 'count-0 frame written')
            res[ls] = (word[0, :n], w[0, :n], node[0, :n])
        return res
    finally:
        gv.close()


@pytest.mark.parametrize('name', [v['name'] for v in BC.vocabularies(big=False)])
def test_transform_on_constructed_trees(name):
    v = {x['name']: x for x in BC.vocabularies(big=False)}[name]
    v['proof'](_check_transform(v, range(v['L'] + 2)))


def test_transform_orbvoc_shape():
    """k = 10, L = 6, 1.1 M nodes in depth-first order, 2000 descriptors at Frame::ComputeBoW's levelsup = 4 (and the rest)."""
    v = BC.orbvoc_shaped()
    v['proof'](_check_transform(v, range(v['L'] + 2)))


def test_transform_on_a_dbow2_trained_tree():
    """A tree trained by DBoW2's own create (nodes with fewer than k children), through the device transform."""
    L = TB.dbow2()
    h, v = TB.trained_vocabulary(L)
    L.dbow2_ref_free(V(h))
    _check_transform(v, range(v['L'] + 2))


SAMPLE = ['kf_claims_ori1', 'kf_hist_wrap', 'kf_ratio80_ori0', 'kfkf_claims_ori0', 'kfkf_hist_tie4', 'tri_claims_ori1', 'tri_epipole_ori0', 'tri_dsqr_ori1', 'tri_stereo1_ori0']


@pytest.mark.parametrize('name', SAMPLE)
def test_host_wrappers(name):
    """sgs_match_bow (mode 0) and sgs_match_bow_keyframes (modes 1, 2) on single cases equal the oracle."""
    c = BC.CASES[name]
    o = BC.run_oracle(c)
    a, b, p = c['a'], c['b'], c['params']
    if c['mode'] == 0:
        P = lambda x: np.ascontiguousarray(x).ctypes.data_as(V)
        m = np.full(len(b['node']), 7, np.int32); nm = C.c_int()
        B.check(B.lib().sgs_match_bow(len(a['node']), P(a['node']), P(a['weight']), P(a['valid']), P(a['desc']), P(a['angle']), len(b['node']), P(b['node']),
                                      P(b['weight']), P(b['desc']), P(b['angle']), p['nnratio'], p['check_ori'], m.ctypes.data_as(V), C.byref(nm), 0))
        nm = nm.value
    else:
        kw = dict(F12=c['F12'], epipole=np.array([c['ex'], c['ey']], np.float32), sigma2=BC.SIGMA2, sf=BC.SF, only_stereo=p['only_stereo']) if c['mode'] == 2 else {}
        nm, m = TG._match_bow_keyframes_host(c['mode'], a, b, p['nnratio'], p['check_ori'], **kw)
    assert nm == o['nm'] and np.array_equal(m, o['m']), name
    c['proof'](o)


def test_host_transform_wrapper():
    v = [x for x in BC.vocabularies(big=False) if x['name'] == 'voc_fan4096'][0]
    gv = GpuVoc(v)
    try:
        q = np.ascontiguousarray(v['queries']); n = len(q)
        word = np.zeros(n, np.int32); w = np.zeros(n, np.float64); node = np.zeros(n, np.int32)
        B.check(B.lib().sgs_bow_transform(gv.h, q.ctypes.data_as(V), n, 1, word.ctypes.data_as(V), w.ctypes.data_as(V), node.ctypes.data_as(V)))
        ow, owt, on = BC.run_voc_oracle(v, [1])[1]
        assert np.array_equal(word, ow) and w.tobytes() == owt.tobytes() and np.array_equal(node, on)
    finally:
        gv.close()


def test_repeat_launch_gives_identical_bytes():
    fr = _frames([g for g in GROUPS if 'tri_claims_ori1' in g][0])
    ma = max(len(f['c']['a']['node']) for f in fr); mb = max(len(f['c']['b']['node']) for f in fr)
    m1, n1, _, _ = launch(fr, ma + 3, mb + 5)
    m2, n2, _, _ = launch(fr, ma + 3, mb + 5)
    assert m1.tobytes() == m2.tobytes() and n1.tobytes() == n2.tobytes()
