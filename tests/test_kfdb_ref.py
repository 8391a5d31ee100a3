"""The key-frame database restatement (tests/kfdb_cases.py) -- what sgs_kfdb and sgs_kfdb_reloc_candidates_device compute -- pinned against the
REFERENCE'S OWN src/KeyFrameDatabase.cc, compiled unmodified with the real DBoW2 BowVector / ScoringObject / TemplatedVocabulary against the KeyFrame
and Frame stand-ins of tests/cpp/kfdb_ref_pre.h (driver: tests/cpp/kfdb_ref_driver.cpp).  Sequences of add / erase / clear / query, random and
constructed: candidate lists and every key frame's mRelocScore after each query must be equal, bit for bit.  No device needed."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import kfdb_cases as K
import oracle as O

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = '/root/reference/src/sg-slam'
DBOW = os.path.join(REF, 'Thirdparty', 'DBoW2')
pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(REF, 'src', 'KeyFrameDatabase.cc')), reason='reference tree absent')
v = C.c_void_p


def _p(a):
    return a.ctypes.data_as(v)


@pytest.fixture(scope='module')
def reflib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('kfdb') / 'libkfdb_ref.so')
    cmd = ['g++', '-O3', '-std=c++11', '-fPIC', '-shared', '-fvisibility=hidden', '-w', '-ffp-contract=off',
           '-I' + os.path.join(ROOT, 'oracle', 'dbow2_shim'), '-I' + REF, '-I' + os.path.join(REF, 'include'), '-I' + DBOW,
           '-include', os.path.join(ROOT, 'tests', 'cpp', 'kfdb_ref_pre.h'), '-o', out, os.path.join(ROOT, 'tests', 'cpp', 'kfdb_ref_driver.cpp'),
           os.path.join(REF, 'src', 'KeyFrameDatabase.cc')] + \
          [os.path.join(DBOW, 'DBoW2', f) for f in ('BowVector.cpp', 'FeatureVector.cpp', 'ScoringObject.cpp', 'FORB.cpp')] + \
          [os.path.join(DBOW, 'DUtils', f) for f in ('Random.cpp', 'Timestamp.cpp')] + ['-l:libstdc++.so.6', '-pthread']
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(out)
    L.kdb_create.restype = v
    return L


def run_reference(L, ops, nslots, covis, nmaps=4, nwords=1024):
    h = v(L.kdb_create(nwords, nmaps, nslots))
    for s in range(nslots):
        L.kdb_set_covis(h, s, _p(np.ascontiguousarray(covis[s], np.int32)))
    where, out = {}, []
    for op in ops:
        if op[0] == 'add':
            for s, m, (ids, vals) in zip(op[1], op[2], op[3]):
                ids = np.ascontiguousarray(ids, np.int32); vals = np.ascontiguousarray(vals, np.float64)
                L.kdb_add(h, s, m, len(ids), _p(ids), _p(vals)); where[s] = m
        elif op[0] == 'erase':
            for s in op[1]:
                L.kdb_erase(h, s, where.pop(s))
        elif op[0] == 'clear':
            L.kdb_clear(h, op[1]); where = {s: m for s, m in where.items() if m != op[1]}
        else:
            rows = []
            scores = np.zeros(nslots, np.float32)
            for m, (ids, vals) in zip(op[1], op[2]):
                ids = np.ascontiguousarray(ids, np.int32); vals = np.ascontiguousarray(vals, np.float64)
                cand = np.zeros(nslots, np.int32)
                n = L.kdb_query(h, m, len(ids), _p(ids), _p(vals), _p(cand), _p(scores))
                rows.append(cand[:n].tolist())
            out.append((rows, scores.copy()))
    L.kdb_free(h)
    return out


def _compare(ref, mine):
    assert len(ref) == len(mine)
    for q, ((rr, rs), (mr, ms)) in enumerate(zip(ref, mine)):
        assert [r for r in rr] == [m[0] for m in mr], q
        assert rs.tobytes() == ms.tobytes(), (q, np.nonzero(rs != ms)[0])


@pytest.mark.parametrize('seed', [1, 2, 3, 4])
def test_random_sequences_equal_the_reference(reflib, seed):
    ops, covis = K.random_sequence(seed)
    mine, seen = K.run_oracle(ops, len(covis), covis)
    _compare(run_reference(reflib, ops, len(covis), covis), mine)
    assert sum(len(r[0]) for rows, _ in mine for r in rows) > 20 and seen['stale'] > 0 and seen['noshare_nb'] > 0, seen


def test_constructed_sequence_equals_the_reference_and_forces_every_path(reflib):
    ops, covis = K.constructed_sequence()
    mine, seen = K.run_oracle(ops, len(covis), covis)
    _compare(run_reference(reflib, ops, len(covis), covis), mine)
    for k in ('tie', 'edge', 'stale', 'noshare_nb', 'dup_best', 'retain_tie', 'empty_frame', 'empty_map'):
        assert seen[k] > 0, (k, seen)


def test_bow_vector_restatement_on_edge_inputs():
    """Frame::ComputeBoW's BowVector from per-feature (word, weight): stopped words (weight 0) left out, repeated words summed in feature order,
    no features at all, every feature stopped -- oracle.bow_vector (pinned to the real transform by tests/test_dbow2_ref.py) against
    BowVector::addWeight + normalize(L1) written out."""
    rng = np.random.default_rng(5)
    word = rng.integers(0, 40, 300).astype(np.int32)
    weight = rng.uniform(0, 2, 300); weight[::7] = 0.0
    for w, wt in ((word, weight), (word[:0], weight[:0]), (word[:20], np.zeros(20))):
        ids, vals = O.bow_vector(w, wt)
        raw = {}
        for i in range(len(w)):
            if wt[i] > 0:
                raw[int(w[i])] = raw[int(w[i])] + wt[i] if int(w[i]) in raw else wt[i]
        rid, rv = K.normalized(list(raw.keys()), list(raw.values())) if raw else (np.zeros(0, np.int32), np.zeros(0))
        assert np.array_equal(ids, rid) and vals.tobytes() == np.asarray(rv, np.float64).tobytes()
