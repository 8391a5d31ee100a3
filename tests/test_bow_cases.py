"""The constructed bag-of-words cases of tests/bow_cases.py against the REFERENCE'S OWN code (no device):
- every matcher case: the oracle's SearchByBoW(KF, F), SearchByBoW(KF1, KF2) and SearchForTriangulation (oracle/bow.cpp) equal the
  reference's src/ORBmatcher.cc (oracle/_ref/liborbmatcher_ref.so) match for match, and the case's proof holds on that result;
- every constructed vocabulary: the oracle's transform equals DBoW2's own `transform` (oracle/_ref/libdbow2_ref.so) for levelsup 0 .. L + 1
  -- word, weight bit for bit, node -- on the tree written as a binary vocabulary file and read back by DBoW2's loadFromBinaryFile.
  The binary format is used because its phantom node (the eof() loop re-reads the last record) duplicates a sibling and is never selected,
  while the text loader's phantom has a zero descriptor.  The header's k only sizes DBoW2's reservations, so it is written as at most 20
  (the product's reader refuses more) and at least 2; the tree itself comes from the parent records.
Skipped only when the reference libraries were never built."""
import ctypes as C
import os

import numpy as np
import pytest

import bow_cases as BC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MATCHER_SO = os.path.join(ROOT, 'oracle', '_ref', 'liborbmatcher_ref.so')
DBOW2_SO = os.path.join(ROOT, 'oracle', '_ref', 'libdbow2_ref.so')


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def _matcher():
    if not os.path.exists(MATCHER_SO):
        pytest.skip('oracle/_ref/liborbmatcher_ref.so not built (reference tree absent)')
    L = C.CDLL(MATCHER_SO)
    for f in ('ref_search_by_bow', 'ref_search_by_bow_kfkf', 'ref_search_for_triangulation'):
        getattr(L, f).restype = C.c_int
    return L


def dbow2():
    if not os.path.exists(DBOW2_SO):
        pytest.skip('oracle/_ref/libdbow2_ref.so not built (reference tree absent)')
    L = C.CDLL(DBOW2_SO)
    for f in ('dbow2_ref_create', 'dbow2_ref_load_binary'):
        getattr(L, f).restype = C.c_void_p
    return L


def ref_arrays(L, mode, params, a, b, c):
    """The reference's ORBmatcher.cc on explicit side arrays: dict(nm, m) in the layout of bow_cases.run_arrays."""
    f32, u8, i32, f64 = np.float32, np.uint8, np.int32, np.float64
    g = lambda s, k, dt: np.ascontiguousarray(s[k], dt)
    r, ori = C.c_float(params['nnratio']), int(params['check_ori'])
    na, nb = len(a['node']), len(b['node'])
    if mode == 0:
        m = np.zeros(nb, i32)
        nm = L.ref_search_by_bow(na, _p(g(a, 'node', i32)), _p(g(a, 'weight', f64)), _p(g(a, 'valid', u8)), _p(g(a, 'desc', u8)), _p(g(a, 'angle', f32)),
                                 nb, _p(g(b, 'node', i32)), _p(g(b, 'weight', f64)), _p(g(b, 'desc', u8)), _p(g(b, 'angle', f32)), r, ori, _p(m))
    elif mode == 1:
        m = np.zeros(na, i32)
        nm = L.ref_search_by_bow_kfkf(na, _p(g(a, 'node', i32)), _p(g(a, 'weight', f64)), _p(g(a, 'valid', u8)), _p(g(a, 'desc', u8)), _p(g(a, 'angle', f32)),
                                      nb, _p(g(b, 'node', i32)), _p(g(b, 'weight', f64)), _p(g(b, 'valid', u8)), _p(g(b, 'desc', u8)), _p(g(b, 'angle', f32)), r, ori, _p(m))
    else:
        m = np.zeros(na, i32)
        A = [g(a, 'node', i32), g(a, 'weight', f64), g(a, 'valid', u8), g(a, 'stereo', u8), g(a, 'desc', u8), g(a, 'xy', f32), g(a, 'angle', f32)]
        B = [g(b, 'node', i32), g(b, 'weight', f64), g(b, 'valid', u8), g(b, 'stereo', u8), g(b, 'desc', u8), g(b, 'xy', f32), g(b, 'octave', i32), g(b, 'angle', f32)]
        nm = L.ref_search_for_triangulation(na, *[_p(x) for x in A], nb, *[_p(x) for x in B], _p(np.ascontiguousarray(c['F12'], f32).reshape(9).copy()),
                                            _p(np.ascontiguousarray(c['cw'], f32)), _p(BC.CAM), len(BC.SF), _p(BC.SIGMA2), _p(BC.SF), int(params['only_stereo']), ori, _p(m))
    return dict(nm=int(nm), m=m)


def ref_case(L, c):
    return ref_arrays(L, c['mode'], c['params'], c['a'], c['b'], c)


@pytest.mark.parametrize('name', BC.names())
def test_matcher_case_equals_the_reference(name):
    """SearchByBoW (both forms) and SearchForTriangulation on a constructed case: the oracle equals the reference's ORBmatcher.cc, and the
    case's proof -- the gate, ratio, claim, tie, bucket, histogram or epipolar path it was built for -- holds on that result."""
    c = BC.CASES[name]
    o = BC.run_oracle(c)
    r = ref_case(_matcher(), c)
    assert r['nm'] == o['nm'] and np.array_equal(r['m'], o['m']), (name, r['nm'], o['nm'], np.nonzero(r['m'] != o['m'])[0][:10])
    c['proof'](o)


@pytest.mark.parametrize('mode', [0, 1, 2])
@pytest.mark.parametrize('npairs,extra', [(4096, 0), (2048, 1)])
def test_full_root_bucket_equals_the_reference(mode, npairs, extra):
    """Every feature in the root bucket (levelsup >= L): 8192 (or 4097) features per side in one node, each duplicated key-frame
    descriptor claiming its first candidate and its copy the second."""
    c = BC.full_bucket(mode, npairs, extra)
    o = BC.run_oracle(c)
    r = ref_case(_matcher(), c)
    assert r['nm'] == o['nm'] and np.array_equal(r['m'], o['m'])
    c['proof'](o)


def write_binary(path, v):
    """saveToBinaryFile's layout (TemplatedVocabulary.h:1514-1535), written with one structured array (the ORBvoc-shaped tree has 1.1 M nodes)."""
    n = len(v['parent'])
    nch = np.bincount(v['parent'][1:], minlength=n)
    rec = np.zeros(n - 1, np.dtype([('parent', '<i4'), ('desc', 'u1', 32), ('weight', '<f4'), ('leaf', 'u1')]))
    assert rec.dtype.itemsize == 41
    rec['parent'] = v['parent'][1:]; rec['desc'] = v['desc'][1:]; rec['weight'] = v['weight'][1:]; rec['leaf'] = nch[1:] == 0
    assert np.array_equal(rec['weight'].astype(np.float64), v['weight'][1:]), 'weights must be float32-representable'
    k = int(min(max(int(nch.max()), 2), 20))
    with open(path, 'wb') as f:
        f.write(np.array([n, 41], '<u4').tobytes() + np.array([k, v['L'], 0, 0], '<i4').tobytes())
        f.write(rec.tobytes())


def ref_transform_from_file(L, path, queries, levelsups):
    h = L.dbow2_ref_load_binary(str(path).encode())
    assert h
    try:
        out = {}
        q = np.ascontiguousarray(queries, np.uint8)
        for ls in levelsups:
            word = np.zeros(len(q), np.int32); w = np.zeros(len(q), np.float64); node = np.zeros(len(q), np.int32)
            L.dbow2_ref_transform_each(C.c_void_p(h), _p(q), len(q), ls, _p(word), _p(w), _p(node))
            out[ls] = (word, w, node)
        return out
    finally:
        L.dbow2_ref_free(C.c_void_p(h))


@pytest.fixture(scope='module')
def vocabularies():
    return {v['name']: v for v in BC.vocabularies()}


@pytest.mark.parametrize('name', [v['name'] for v in BC.vocabularies(big=False)] + ['voc_orbvoc'])
def test_vocabulary_transform_equals_dbow2(name, vocabularies, tmp_path):
    """Planted sibling ties across 32-lane groups, fan-outs 1 .. 4096, an equidistant descriptor, single-child chains, stopped words and
    the ORBvoc shape: the oracle's transform equals DBoW2's for levelsup 0 .. L + 1, and the vocabulary's proof holds."""
    L = dbow2()
    v = vocabularies[name]
    write_binary(tmp_path / 'v.bin', v)
    ls = list(range(v['L'] + 2))
    r = ref_transform_from_file(L, tmp_path / 'v.bin', v['queries'], ls)
    o = BC.run_voc_oracle(v, ls)
    for l in ls:
        assert np.array_equal(o[l][0], r[l][0]) and o[l][1].tobytes() == r[l][1].tobytes() and np.array_equal(o[l][2], r[l][2]), (name, l)
    v['proof'](o)


def trained_vocabulary(L, seed=1, k=10, depth=4):
    """A tree trained by DBoW2's own `create` (k = 10): the lower levels hold so few descriptors that many nodes get fewer than k children.
    Returns (handle, tree as flat arrays with queries); the caller frees the handle."""
    import test_dbow2_ref as TD
    desc, image_of, nimg = TD._training(seed, nimages=10, per_image=100)
    h = L.dbow2_ref_create(_p(desc), _p(image_of), len(desc), nimg, k, depth)
    assert h
    v = TD._dump(L, h)
    nch = np.bincount(v['parent'][1:], minlength=len(v['parent']))
    inner = nch[nch > 0]
    assert (inner < k).sum() > 100 and inner.min() <= 2, 'variable fan-out down to two children'
    rs = np.random.RandomState(seed)
    leaves = np.nonzero(v['word_id'] >= 0)[0]
    q = v['desc'][leaves[rs.randint(0, len(leaves), 1500)]] ^ (rs.randint(0, 256, (1500, 32)) & rs.randint(0, 256, (1500, 32)) & rs.randint(0, 256, (1500, 32))).astype(np.uint8)
    q = np.concatenate([q, rs.randint(0, 256, (500, 32)).astype(np.uint8)])
    return h, dict(name='voc_trained', k=k, L=depth, parent=v['parent'], desc=v['desc'], weight=v['weight'], queries=q)


def test_trained_vocabulary_transform_equals_dbow2():
    """The same pin on a tree DBoW2's create trained (k = 10, L = 4), in memory."""
    import oracle as O
    L = dbow2()
    h, v = trained_vocabulary(L)
    try:
        V = O.Vocabulary(v['k'], v['L'], v['parent'], v['desc'], v['weight'])
        q = np.ascontiguousarray(v['queries'])
        for ls in range(v['L'] + 2):
            word = np.zeros(len(q), np.int32); w = np.zeros(len(q), np.float64); node = np.zeros(len(q), np.int32)
            L.dbow2_ref_transform_each(C.c_void_p(h), _p(q), len(q), ls, _p(word), _p(w), _p(node))
            ow, owt, on = V.transform(q, ls)
            assert np.array_equal(ow, word) and owt.tobytes() == w.tobytes() and np.array_equal(on, node), ls
    finally:
        L.dbow2_ref_free(C.c_void_p(h))
