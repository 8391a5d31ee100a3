"""The loop-query restatement (tests/kfdb_loop_cases.py) -- what sgs_kfdb_loop_candidates_device computes -- pinned against the REFERENCE'S OWN
src/KeyFrameDatabase.cc, compiled unmodified with the real DBoW2 BowVector / ScoringObject / TemplatedVocabulary against the stand-ins of
tests/cpp/kfdb_loop_ref_pre.h (driver: tests/cpp/kfdb_loop_ref_driver.cpp, which computes DetectLoop's minScore with the vocabulary's own score).
Sequences of add / erase / clear / relocalisation and loop queries, random and constructed: candidate lists, stats and minScore of every loop
query, and the candidates and every key frame's mRelocScore after every relocalisation query, must be equal bit for bit.  No device needed."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import kfdb_loop_cases as KL

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = '/root/reference/src/sg-slam'
DBOW = os.path.join(REF, 'Thirdparty', 'DBoW2')
pytestmark = pytest.mark.skipif(not os.path.exists(os.path.join(REF, 'src', 'KeyFrameDatabase.cc')), reason='reference tree absent')
v = C.c_void_p


def _p(a):
    return a.ctypes.data_as(v)


@pytest.fixture(scope='module')
def reflib(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('kfdb_loop') / 'libkfdb_loop_ref.so')
    cmd = ['g++', '-O3', '-std=c++11', '-fPIC', '-shared', '-fvisibility=hidden', '-w', '-ffp-contract=off',
           '-I' + os.path.join(ROOT, 'oracle', 'dbow2_shim'), '-I' + REF, '-I' + os.path.join(REF, 'include'), '-I' + DBOW,
           '-include', os.path.join(ROOT, 'tests', 'cpp', 'kfdb_loop_ref_pre.h'), '-o', out, os.path.join(ROOT, 'tests', 'cpp', 'kfdb_loop_ref_driver.cpp'),
           os.path.join(REF, 'src', 'KeyFrameDatabase.cc')] + \
          [os.path.join(DBOW, 'DBoW2', f) for f in ('BowVector.cpp', 'FeatureVector.cpp', 'ScoringObject.cpp', 'FORB.cpp')] + \
          [os.path.join(DBOW, 'DUtils', f) for f in ('Random.cpp', 'Timestamp.cpp')] + ['-l:libstdc++.so.6', '-pthread']
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-3000:]
    L = C.CDLL(out)
    L.kdb_create.restype = v
    return L


def _bow_rows(bows):
    cap = max([len(b[0]) for b in bows] + [1])
    w = np.zeros((len(bows), cap), np.int32); x = np.zeros((len(bows), cap)); n = np.array([len(b[0]) for b in bows], np.int32)
    for i, (ids, vals) in enumerate(bows):
        w[i, :len(ids)] = ids; x[i, :len(ids)] = vals
    return w, x, n, cap


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
        elif op[0] == 'query':
            rows = []
            scores = np.zeros(nslots, np.float32)
            for m, (ids, vals) in zip(op[1], op[2]):
                ids = np.ascontiguousarray(ids, np.int32); vals = np.ascontiguousarray(vals, np.float64)
                cand = np.zeros(nslots, np.int32)
                n = L.kdb_query(h, m, len(ids), _p(ids), _p(vals), _p(cand), _p(scores))
                rows.append(cand[:n].tolist())
            out.append(('query', rows, scores.copy()))
        else:
            rows = []
            for m, (ids, vals), conn, covs, sf in zip(*op[1:]):
                if m < 0:
                    rows.append(None)
                    continue
                ids = np.ascontiguousarray(ids, np.int32); vals = np.ascontiguousarray(vals, np.float64)
                conn = np.ascontiguousarray(conn, np.int32)
                cw, cv, cn, cap = _bow_rows(covs)
                cand = np.zeros(nslots, np.int32); stats = np.zeros(4, np.int32); ms = np.zeros(1, np.float32)
                n = L.kdb_loop(h, m, sf, len(ids), _p(ids), _p(vals), len(conn), _p(conn), len(covs), cap, _p(cn), _p(cw), _p(cv), _p(cand),
                               _p(stats), _p(ms))
                rows.append((cand[:n].tolist(), stats.tolist(), ms[0]))
            out.append(('loop', rows))
    L.kdb_free(h)
    return out


def _compare(ref, mine):
    assert len(ref) == len(mine)
    for q, (r, m) in enumerate(zip(ref, mine)):
        assert r[0] == m[0], q
        if r[0] == 'query':
            assert r[1] == [x[0] for x in m[1]], q
            assert r[2].tobytes() == m[2].tobytes(), (q, np.nonzero(r[2] != m[2])[0])
        else:
            for f, (rr, mr) in enumerate(zip(r[1], m[1])):
                if rr is None:
                    assert mr is None
                    continue
                assert rr[0] == mr[0] and rr[1] == mr[1], (q, f, rr, mr)
                assert np.float32(rr[2]).tobytes() == np.float32(mr[2]).tobytes(), (q, f, rr[2], mr[2])


@pytest.mark.parametrize('seed', [1, 2, 3, 4])
def test_random_sequences_equal_the_reference(reflib, seed):
    ops, covis = KL.loop_sequence(seed)
    mine, db = KL.run_oracle(ops, len(covis), covis)
    _compare(run_reference(reflib, ops, len(covis), covis), mine)
    loops = [r for kind, *rest in mine if kind == 'loop' for r in rest[0] if r is not None]
    assert sum(len(r[0]) for r in loops) > 10 and sum(r[1][0] > r[1][2] for r in loops) > 0, db.lseen
    assert db.lseen['conn_most'] + db.lseen['conn_nb'] > 0 and db.lseen['self_cand'] > 0, db.lseen


def test_constructed_sequence_equals_the_reference_and_forces_every_path(reflib):
    ops, covis = KL.constructed_sequence()
    mine, db = KL.run_oracle(ops, len(covis), covis)
    _compare(run_reference(reflib, ops, len(covis), covis), mine)
    for k in ('conn_most', 'conn_nb', 'si_eq_min', 'nb_below_min', 'nb_edge', 'no_cov', 'cov_not_in_db', 'zero_min', 'retain_tie', 'dup_best',
              'empty_frame', 'empty_map', 'self_cand'):
        assert db.lseen[k] > 0, (k, db.lseen)
    # the zero minimum keeps the sign of the first zero score met: -0 (no common word)
    assert any(r is not None and r[2] == 0 and np.signbit(r[2]) for kind, *rest in mine if kind == 'loop' for r in rest[0])
