"""GPU parity of DBoW2 transform and ORBmatcher::SearchByBoW(KeyFrame*, Frame&) through the C ABI against the CPU oracle: integer work,
bit-exact (word / node ids, weights as stored, assignments, counts)."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle as O  # noqa: E402
import scenarios as S  # noqa: E402
from pysgs import binding as B  # noqa: E402


class GpuVoc(B._Handle):
    def __init__(self, voc):
        v = C.c_void_p
        super().__init__(B.lib().sgs_vocabulary_create, B.lib().sgs_vocabulary_destroy, 0, voc['k'], voc['L'], len(voc['parent']), voc['parent'].ctypes.data_as(v),
                         np.ascontiguousarray(voc['desc']).ctypes.data_as(v), voc['weight'].ctypes.data_as(v))


def _transform_gpu(gv, desc, counts, levelsup):
    import torch
    F, cap = desc.shape[:2]
    dd = torch.from_numpy(np.ascontiguousarray(desc)).cuda(); dc = torch.from_numpy(np.asarray(counts, np.int32)).cuda()
    word = torch.full((F, cap), -7, dtype=torch.int32, device='cuda'); w = torch.zeros((F, cap), dtype=torch.float64, device='cuda'); node = torch.full((F, cap), -7, dtype=torch.int32, device='cuda')
    v = C.c_void_p
    B.check(B.lib().sgs_bow_transform_batch_device(gv.h, v(dd.data_ptr()), v(dc.data_ptr()), cap, F, levelsup, v(word.data_ptr()), v(w.data_ptr()), v(node.data_ptr()), v(0)))
    torch.cuda.synchronize()
    return word, w, node


@pytest.mark.parametrize('k,L', [(10, 3), (4, 5), (33, 2)])
def test_transform(k, L):
    voc = S.random_vocabulary(5 + k, k=k, L=L)
    V = O.Vocabulary(voc['k'], voc['L'], voc['parent'], voc['desc'], voc['weight'])
    gv = GpuVoc(voc)
    try:
        sc = [S.bow_pair_scenario(s, voc, n_kf=700, n_f=1) for s in (1, 2)]
        desc = np.stack([c['kf_desc'] for c in sc]); counts = [700, 333]
        for levelsup in (0, 1, 2, 4):
            word, w, node = _transform_gpu(gv, desc, counts, levelsup)
            word, w, node = word.cpu().numpy(), w.cpu().numpy(), node.cpu().numpy()
            for f in range(2):
                n = counts[f]
                ow, owt, on = V.transform(desc[f, :n], levelsup)
                assert np.array_equal(word[f, :n], ow) and np.array_equal(node[f, :n], on) and w[f, :n].tobytes() == owt.tobytes()
                assert np.all(word[f, n:] == -7)
    finally:
        gv.close()


@pytest.mark.parametrize('seed,nk,nf,flips,nnratio', [(1, 1000, 1000, 40, 0.7), (2, 1100, 400, 80, 0.6), (3, 50, 1100, 10, 0.9), (4, 1000, 1000, 0, 0.7)])
def test_search_by_bow(seed, nk, nf, flips, nnratio):
    import torch
    voc = S.random_vocabulary(9, k=10, L=3)
    V = O.Vocabulary(voc['k'], voc['L'], voc['parent'], voc['desc'], voc['weight'])
    gv = GpuVoc(voc)
    try:
        F, cap = 3, 1100
        scs = [S.bow_pair_scenario(seed * 10 + i, voc, n_kf=nk, n_f=nf, flips=flips) for i in range(F)]
        kd = np.zeros((F, cap, 32), np.uint8); fd = np.zeros((F, cap, 32), np.uint8); ka = np.zeros((F, cap), np.float32); fa = np.zeros((F, cap), np.float32)
        kv = np.zeros((F, cap), np.uint8)
        for i, s in enumerate(scs):
            kd[i, :nk] = s['kf_desc']; fd[i, :nf] = s['f_desc']; ka[i, :nk] = s['kf_angle']; fa[i, :nf] = s['f_angle']; kv[i, :nk] = s['kf_valid']
        kn = np.array([nk, nk, max(1, nk // 2)], np.int32); fn = np.array([nf, max(1, nf // 3), nf], np.int32)
        for levelsup in (1, 2):
            _, kw, knode = _transform_gpu(gv, kd, kn, levelsup); _, fw, fnode = _transform_gpu(gv, fd, fn, levelsup)
            dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
            t = dict(kv=dev(kv), kd=dev(kd), ka=dev(ka), kn=dev(kn), fd=dev(fd), fa=dev(fa), fn=dev(fn))
            for ori in (0, 1):
                m = torch.zeros((F, cap), dtype=torch.int32, device='cuda'); nm = torch.zeros(F, dtype=torch.int32, device='cuda')
                a = B.BowBatch()
                a.kf_node, a.kf_weight, a.kf_valid, a.kf_desc, a.kf_angle, a.kf_n, a.kf_cap = knode.data_ptr(), kw.data_ptr(), t['kv'].data_ptr(), t['kd'].data_ptr(), t['ka'].data_ptr(), t['kn'].data_ptr(), cap
                a.f_node, a.f_weight, a.f_desc, a.f_angle, a.f_n, a.f_cap = fnode.data_ptr(), fw.data_ptr(), t['fd'].data_ptr(), t['fa'].data_ptr(), t['fn'].data_ptr(), cap
                a.nnratio, a.check_orientation, a.match_f, a.nmatches = nnratio, ori, m.data_ptr(), nm.data_ptr()
                B.check(B.lib().sgs_match_bow_batch_device(C.byref(a), F, C.c_void_p(0)))
                torch.cuda.synchronize()
                mg, nmg = m.cpu().numpy(), nm.cpu().numpy()
                for f in range(F):
                    a_, b_ = int(kn[f]), int(fn[f])
                    _, okw, okn = V.transform(kd[f, :a_], levelsup); _, ofw, ofn = V.transform(fd[f, :b_], levelsup)
                    onm, om = O.search_by_bow(okn, okw, kv[f, :a_], kd[f, :a_], ka[f, :a_], ofn, ofw, fd[f, :b_], fa[f, :b_], nnratio, bool(ori))
                    assert nmg[f] == onm and np.array_equal(mg[f, :b_], om), (f, levelsup, ori)
                    assert np.all(mg[f, b_:] == -1)
                if flips <= 40 and nk >= 1000:
                    assert nmg[0] > 50
    finally:
        gv.close()


def test_host_variants():
    voc = S.random_vocabulary(21, k=10, L=3)
    V = O.Vocabulary(voc['k'], voc['L'], voc['parent'], voc['desc'], voc['weight'])
    gv = GpuVoc(voc)
    try:
        s = S.bow_pair_scenario(5, voc, n_kf=900, n_f=1000)
        v = C.c_void_p
        outs = []
        for d in (s['kf_desc'], s['f_desc']):
            n = len(d); word = np.zeros(n, np.int32); w = np.zeros(n, np.float64); node = np.zeros(n, np.int32)
            B.check(B.lib().sgs_bow_transform(gv.h, np.ascontiguousarray(d).ctypes.data_as(v), n, 1, word.ctypes.data_as(v), w.ctypes.data_as(v), node.ctypes.data_as(v)))
            ow, owt, on = V.transform(d, 1)
            assert np.array_equal(word, ow) and np.array_equal(node, on) and w.tobytes() == owt.tobytes()
            outs.append((w, node))
        (kw, kn), (fw, fn) = outs
        m = np.zeros(1000, np.int32); nm = C.c_int()
        P = lambda a: np.ascontiguousarray(a).ctypes.data_as(v)
        B.check(B.lib().sgs_match_bow(900, P(kn), P(kw), P(s['kf_valid']), P(s['kf_desc']), P(s['kf_angle']), 1000, P(fn), P(fw), P(s['f_desc']), P(s['f_angle']),
                                      0.7, 1, m.ctypes.data_as(v), C.byref(nm), 0))
        onm, om = O.search_by_bow(kn, kw, s['kf_valid'], s['kf_desc'], s['kf_angle'], fn, fw, s['f_desc'], s['f_angle'], 0.7, True)
        assert nm.value == onm and np.array_equal(m, om)
        B.check(B.lib().sgs_bow_transform(gv.h, None, 0, 1, None, None, None))              # nothing to transform: no device work
    finally:
        gv.close()


def _match_bow_keyframes_host(mode, k1, k2, nnratio, ori, F12=None, epipole=None, sigma2=None, sf=None, only_stereo=0):
    """sgs_match_bow_keyframes, the single-pair host entry point: (nmatches, match12)."""
    P = lambda a, dt=None: None if a is None else np.ascontiguousarray(a, dt).ctypes.data_as(C.c_void_p)
    side = lambda k: [P(k['node'], np.int32), P(k['weight'], np.float64), P(k['valid'], np.uint8), P(k['desc'], np.uint8), P(k['angle'], np.float32)]
    n1, n2 = len(k1['desc']), len(k2['desc'])
    m = np.full(n1, 7, np.int32); nm = C.c_int(-1)
    B.check(B.lib().sgs_match_bow_keyframes(mode, n1, *side(k1), n2, *side(k2), nnratio, int(ori), P(k1.get('stereo'), np.uint8), P(k2.get('stereo'), np.uint8),
                                            P(k1.get('xy'), np.float32), P(k2.get('xy'), np.float32), P(k2.get('octave'), np.int32), P(F12, np.float32),
                                            P(epipole, np.float32), P(sigma2, np.float32), P(sf, np.float32), 0 if sf is None else len(sf), int(only_stereo),
                                            P(m), C.byref(nm), 0))
    return nm.value, m


@pytest.mark.parametrize('seed,n1,n2,nnratio', [(1, 1000, 1000, 0.8), (2, 600, 1100, 0.75)])
def test_search_by_bow_keyframe_pair(seed, n1, n2, nnratio):
    """SearchByBoW(KeyFrame*, KeyFrame*, vpMatches12) (loop closing, src/ORBmatcher.cc:524-657)."""
    import torch
    voc = S.random_vocabulary(13, k=10, L=3)
    V = O.Vocabulary(voc['k'], voc['L'], voc['parent'], voc['desc'], voc['weight'])
    gv = GpuVoc(voc)
    try:
        cap = 1100
        s = S.bow_pair_scenario(seed + 40, voc, n_kf=n1, n_f=n2, flips=40)
        rs = np.random.RandomState(seed)
        valid2 = (rs.rand(n2) < 0.8).astype(np.uint8)
        pad = lambda a, n, shape, dt: np.concatenate([a, np.zeros((cap - n,) + shape, dt)])[None]
        d1 = pad(s['kf_desc'], n1, (32,), np.uint8); d2 = pad(s['f_desc'], n2, (32,), np.uint8)
        a1 = pad(s['kf_angle'], n1, (), np.float32); a2 = pad(s['f_angle'], n2, (), np.float32)
        v1 = pad(s['kf_valid'], n1, (), np.uint8); v2 = pad(valid2, n2, (), np.uint8)
        c1 = np.array([n1], np.int32); c2 = np.array([n2], np.int32)
        _, w1, nd1 = _transform_gpu(gv, d1, c1, 1); _, w2, nd2 = _transform_gpu(gv, d2, c2, 1)
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        t = [dev(x) for x in (v1, d1, a1, c1, d2, a2, c2, v2)]
        _, ow1, on1 = V.transform(s['kf_desc'], 1); _, ow2, on2 = V.transform(s['f_desc'], 1)
        for ori in (0, 1):
            m = torch.zeros((1, cap), dtype=torch.int32, device='cuda'); nm = torch.zeros(1, dtype=torch.int32, device='cuda')
            a = B.BowBatch()
            a.kf_node, a.kf_weight, a.kf_valid, a.kf_desc, a.kf_angle, a.kf_n, a.kf_cap = nd1.data_ptr(), w1.data_ptr(), t[0].data_ptr(), t[1].data_ptr(), t[2].data_ptr(), t[3].data_ptr(), cap
            a.f_node, a.f_weight, a.f_desc, a.f_angle, a.f_n, a.f_cap = nd2.data_ptr(), w2.data_ptr(), t[4].data_ptr(), t[5].data_ptr(), t[6].data_ptr(), cap
            a.f_valid, a.keyframe_pair = t[7].data_ptr(), 1
            a.nnratio, a.check_orientation, a.match_f, a.nmatches = nnratio, ori, m.data_ptr(), nm.data_ptr()
            B.check(B.lib().sgs_match_bow_batch_device(C.byref(a), 1, C.c_void_p(0)))
            torch.cuda.synchronize()
            onm, om = O.search_by_bow_kfkf(on1, ow1, s['kf_valid'], s['kf_desc'], s['kf_angle'], on2, ow2, valid2, s['f_desc'], s['f_angle'], nnratio, bool(ori))
            assert int(nm.cpu()[0]) == onm and np.array_equal(m.cpu().numpy()[0, :n1], om) and onm > 30
            sel = om >= 0
            assert np.all(valid2[om[sel]] == 1) and len(set(om[sel].tolist())) == int(sel.sum())       # only good map points, each used once
            hnm, hm = _match_bow_keyframes_host(1, dict(node=on1, weight=ow1, valid=s['kf_valid'], desc=s['kf_desc'], angle=s['kf_angle']),
                                                dict(node=on2, weight=ow2, valid=valid2, desc=s['f_desc'], angle=s['f_angle']), nnratio, ori)
            assert hnm == onm and np.array_equal(hm, om)
    finally:
        gv.close()


@pytest.mark.parametrize('seed,only_stereo', [(1, 0), (2, 1), (3, 0)])
def test_search_for_triangulation(seed, only_stereo):
    """ORBmatcher::SearchForTriangulation + CheckDistEpipolarLine (src/ORBmatcher.cc:140-157, 659-827)."""
    import torch
    voc = S.random_vocabulary(17, k=10, L=3)
    V = O.Vocabulary(voc['k'], voc['L'], voc['parent'], voc['desc'], voc['weight'])
    gv = GpuVoc(voc)
    try:
        cap, n1, n2 = 1100, 1000, 1050
        s = S.bow_pair_scenario(seed + 70, voc, n_kf=n1, n_f=n2, flips=30)
        rs = np.random.RandomState(seed + 5)
        tgt_desc = s['f_desc']
        xy1 = np.c_[rs.uniform(20, 620, n1), rs.uniform(20, 460, n1)].astype(np.float32)
        # frame-2 features: re-derive which key-frame feature each one copies by nearest descriptor, place it on / near the epipolar line y2 = y1
        d1b = np.unpackbits(s['kf_desc'], axis=1).astype(np.int16); d2b = np.unpackbits(tgt_desc, axis=1).astype(np.int16)
        src = np.array([int(np.argmin(np.abs(d1b - d2b[j]).sum(1))) for j in range(n2)])
        xy2 = np.c_[xy1[src, 0] + rs.uniform(-40, 40, n2), xy1[src, 1] + rs.normal(0, 1.5, n2)].astype(np.float32)
        oct2 = rs.randint(0, 8, n2).astype(np.int32)
        free1 = (rs.rand(n1) < 0.8).astype(np.uint8); free2 = (rs.rand(n2) < 0.8).astype(np.uint8)
        st1 = (rs.rand(n1) < 0.5).astype(np.uint8); st2 = (rs.rand(n2) < 0.5).astype(np.uint8)
        F12 = np.array([[0, 0, 0], [0, 0, -1], [0, 1, 0]], np.float32)
        ex, ey = np.float32(320.5), np.float32(240.25)
        sf = S.scale_factors().astype(np.float32); sigma2 = (sf * sf).astype(np.float32)
        _, ow1, on1 = V.transform(s['kf_desc'], 1); _, ow2, on2 = V.transform(tgt_desc, 1)
        k1 = dict(node=on1, weight=ow1, free=free1, stereo=st1, desc=s['kf_desc'], xy=xy1, angle=s['kf_angle'])
        k2 = dict(node=on2, weight=ow2, free=free2, stereo=st2, desc=tgt_desc, xy=xy2, octave=oct2, angle=s['f_angle'])
        pad = lambda a, n, shape, dt: np.concatenate([np.asarray(a, dt), np.zeros((cap - n,) + shape, dt)])[None]
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
        D1 = pad(s['kf_desc'], n1, (32,), np.uint8); D2 = pad(tgt_desc, n2, (32,), np.uint8)
        c1 = np.array([n1], np.int32); c2 = np.array([n2], np.int32)
        _, w1, nd1 = _transform_gpu(gv, D1, c1, 1); _, w2, nd2 = _transform_gpu(gv, D2, c2, 1)
        t = dict(free1=dev(pad(free1, n1, (), np.uint8)), d1=dev(D1), a1=dev(pad(s['kf_angle'], n1, (), np.float32)), c1=dev(c1), st1=dev(pad(st1, n1, (), np.uint8)),
                 xy1=dev(pad(xy1, n1, (2,), np.float32)), free2=dev(pad(free2, n2, (), np.uint8)), d2=dev(D2), a2=dev(pad(s['f_angle'], n2, (), np.float32)), c2=dev(c2),
                 st2=dev(pad(st2, n2, (), np.uint8)), xy2=dev(pad(xy2, n2, (2,), np.float32)), o2=dev(pad(oct2, n2, (), np.int32)), F=dev(F12.reshape(1, 9)),
                 ep=dev(np.array([[ex, ey]], np.float32)))
        for ori in (0, 1):
            m = torch.zeros((1, cap), dtype=torch.int32, device='cuda'); nm = torch.zeros(1, dtype=torch.int32, device='cuda')
            a = B.BowBatch()
            a.kf_node, a.kf_weight, a.kf_valid, a.kf_desc, a.kf_angle, a.kf_n, a.kf_cap = nd1.data_ptr(), w1.data_ptr(), t['free1'].data_ptr(), t['d1'].data_ptr(), t['a1'].data_ptr(), t['c1'].data_ptr(), cap
            a.f_node, a.f_weight, a.f_desc, a.f_angle, a.f_n, a.f_cap = nd2.data_ptr(), w2.data_ptr(), t['d2'].data_ptr(), t['a2'].data_ptr(), t['c2'].data_ptr(), cap
            a.f_valid, a.keyframe_pair, a.nnratio, a.check_orientation = t['free2'].data_ptr(), 2, 0.6, ori
            a.kf_stereo, a.f_stereo, a.kf_xy, a.f_xy, a.f_octave, a.F12, a.epipole = t['st1'].data_ptr(), t['st2'].data_ptr(), t['xy1'].data_ptr(), t['xy2'].data_ptr(), t['o2'].data_ptr(), t['F'].data_ptr(), t['ep'].data_ptr()
            for l in range(8):
                a.level_sigma2[l] = float(sigma2[l]); a.scale_factors[l] = float(sf[l])
            a.only_stereo, a.match_f, a.nmatches = only_stereo, m.data_ptr(), nm.data_ptr()
            B.check(B.lib().sgs_match_bow_batch_device(C.byref(a), 1, C.c_void_p(0)))
            torch.cuda.synchronize()
            onm, om = O.search_for_triangulation(k1, k2, F12, ex, ey, sigma2, sf, bool(only_stereo), bool(ori))
            assert int(nm.cpu()[0]) == onm and np.array_equal(m.cpu().numpy()[0, :n1], om), (ori, int(nm.cpu()[0]), onm)
            assert onm > 20
            sel = om >= 0
            assert np.all(free1[sel] == 1) and np.all(free2[om[sel]] == 1)
            if only_stereo:
                assert np.all(st1[sel] == 1) and np.all(st2[om[sel]] == 1)
            hnm, hm = _match_bow_keyframes_host(2, dict(k1, valid=free1), dict(k2, valid=free2), 0.6, ori, F12=F12, epipole=np.array([ex, ey], np.float32),
                                                sigma2=sigma2, sf=sf, only_stereo=only_stereo)
            assert hnm == onm and np.array_equal(hm, om)
    finally:
        gv.close()


def test_vocabulary_loaded_from_files(tmp_path):
    """sgs_vocabulary_load (text and binary files of the reference's formats) gives the same transform as the tree built from arrays and as the oracle."""
    from test_vocabulary_files import write_binary, write_text
    voc = S.random_vocabulary(23, k=7, L=3)
    voc['weight'] = voc['weight'].astype(np.float32).astype(np.float64)          # representable in the binary format, so that both files hold the same tree
    V = O.Vocabulary(voc['k'], voc['L'], voc['parent'], voc['desc'], voc['weight'])
    write_text(tmp_path / 'v.txt', voc); write_binary(tmp_path / 'v.bin', voc)
    rs = np.random.RandomState(4)
    leaves = np.nonzero(voc['weight'] > 0)[0]
    d = voc['desc'][leaves[rs.randint(0, len(leaves), 500)]].copy()
    d[rs.rand(500) < 0.5, rs.randint(0, 32)] ^= 0x15
    ow, oweight, onode = V.transform(d, 1)
    v = C.c_void_p
    for name in ('v.txt', 'v.bin'):
        h = C.c_void_p()
        B.check(B.lib().sgs_vocabulary_load(str(tmp_path / name).encode(), 0, C.byref(h)))
        word = np.zeros(500, np.int32); w = np.zeros(500, np.float64); node = np.zeros(500, np.int32)
        B.check(B.lib().sgs_bow_transform(h, np.ascontiguousarray(d).ctypes.data_as(v), 500, 1, word.ctypes.data_as(v), w.ctypes.data_as(v), node.ctypes.data_as(v)))
        B.lib().sgs_vocabulary_destroy(h)
        assert np.array_equal(word, ow) and np.array_equal(w, oweight) and np.array_equal(node, onode), name
    with pytest.raises(B.SgsError):
        h = C.c_void_p()
        B.check(B.lib().sgs_vocabulary_load(str(tmp_path / 'missing.txt').encode(), 0, C.byref(h)))
