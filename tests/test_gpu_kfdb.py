"""The device BowVector (sgs_bow_vector_batch_device), the key-frame database (sgs_kfdb_*) and its relocalisation query
(sgs_kfdb_reloc_candidates_device, sgs_tracker_reloc_candidates_device) against the restatement of tests/kfdb_cases.py, which tests/test_kfdb_ref.py
pins to the reference's own KeyFrameDatabase.cc: BowVectors, candidate lists, stats and every slot's mRelocScore bit for bit over add / erase / clear /
query sequences."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import kfdb_cases as K  # noqa: E402
import oracle as O  # noqa: E402
import refkf_cases as R  # noqa: E402
from pysgs import binding as B  # noqa: E402
from test_gpu_refkf_chain import GpuVoc, _setup  # noqa: E402

SENT = 7777


def _torch():
    import torch
    return torch


class Db(B._Handle):
    def __init__(self, max_maps, max_keyframes, max_words):
        super().__init__(B.lib().sgs_kfdb_create, B.lib().sgs_kfdb_destroy, 0, max_maps, max_keyframes, max_words)
        self.K, self.W = max_keyframes, max_words

    def add(self, slots, maps, bows, expect=B.SGS_OK):
        t = _torch()
        cap = max([len(b[0]) for b in bows] + [1])
        w = np.zeros((len(bows), cap), np.int32); v = np.zeros((len(bows), cap)); n = np.array([len(b[0]) for b in bows], np.int32)
        for i, (ids, vals) in enumerate(bows):
            w[i, :len(ids)] = ids; v[i, :len(ids)] = vals
        dw, dv, dn = t.from_numpy(w).cuda(), t.from_numpy(v).cuda(), t.from_numpy(n).cuda()
        s = np.array(slots, np.int32); m = np.array(maps, np.int32)
        rc = B.lib().sgs_kfdb_add(self.h, len(slots), B._p(s), B._p(m), dw.data_ptr(), dv.data_ptr(), dn.data_ptr(), cap, None)
        assert rc == expect, B.lib().sgs_last_error()

    def erase(self, slots, expect=B.SGS_OK):
        s = np.array(slots, np.int32)
        assert B.lib().sgs_kfdb_erase(self.h, len(s), B._p(s), None) == expect

    def clear(self, m, expect=B.SGS_OK):
        assert B.lib().sgs_kfdb_clear(self.h, m, None) == expect

    def scores(self):
        _torch().cuda.synchronize()
        out = np.zeros(self.K, np.float32)
        B.check(B.lib().sgs_kfdb_reloc_scores(self.h, B._p(out)))
        return out

    def query(self, maps, bows, dcovis, cand_cap=64, expect=B.SGS_OK, prefill=None):
        t = _torch()
        F = len(maps); cap = max([len(b[0]) for b in bows] + [1])
        w = np.zeros((F, cap), np.int32); v = np.zeros((F, cap)); n = np.array([len(b[0]) for b in bows], np.int32)
        for i, (ids, vals) in enumerate(bows):
            w[i, :len(ids)] = ids; v[i, :len(ids)] = vals
        dw, dv, dn = t.from_numpy(w).cuda(), t.from_numpy(v).cuda(), t.from_numpy(n).cuda()
        cand = t.full((F, cand_cap), SENT, dtype=t.int32, device='cuda'); ncand = t.full((F,), SENT, dtype=t.int32, device='cuda')
        stats = t.full((F, 4), SENT, dtype=t.int32, device='cuda')
        m = np.array(maps, np.int32)
        rc = B.lib().sgs_kfdb_reloc_candidates_device(self.h, F, B._p(m), dw.data_ptr(), dv.data_ptr(), dn.data_ptr(), cap, dcovis.data_ptr(),
                                                      cand.data_ptr(), cand_cap, ncand.data_ptr(), stats.data_ptr(), None)
        assert rc == expect, B.lib().sgs_last_error()
        t.cuda.synchronize()
        return cand.cpu().numpy(), ncand.cpu().numpy(), stats.cpu().numpy()


def _check_row(got, want, cand_cap, q, f):
    cand, ncand, stats = got
    wc, ws = want
    assert list(stats[f]) == ws, (q, f, stats[f], ws)
    k = min(len(wc), cand_cap)
    assert ncand[f] == k and list(cand[f, :k]) == wc[:k] and (cand[f, k:] == -1).all(), (q, f, cand[f], wc)


def run_device(ops, covis, nmaps=4, cand_cap=64, split=False):
    """every query op's per-row device outputs and the scores after it; split: one call per row"""
    t = _torch()
    db = Db(nmaps, len(covis), 128)
    dcovis = t.from_numpy(np.ascontiguousarray(covis)).cuda()
    out = []
    for op in ops:
        if op[0] == 'add':
            db.add(op[1], op[2], op[3])
        elif op[0] == 'erase':
            db.erase(op[1])
        elif op[0] == 'clear':
            db.clear(op[1])
        else:
            if split:
                res = [db.query([m], [b], dcovis, cand_cap) for m, b in zip(op[1], op[2])]
                res = tuple(np.concatenate([r[i] for r in res]) for i in range(3))
            else:
                res = db.query(op[1], op[2], dcovis, cand_cap)
            out.append((res, db.scores()))
    db.close()
    return out


def _compare(dev, mine, cand_cap):
    assert len(dev) == len(mine)
    for q, ((got, sc), (rows, want_sc)) in enumerate(zip(dev, mine)):
        for f, want in enumerate(rows):
            _check_row(got, want, cand_cap, q, f)
        assert sc.tobytes() == want_sc.tobytes(), (q, np.nonzero(sc != want_sc)[0])


@pytest.mark.parametrize('seed', [1, 2, 3, 4, 5, 6])
def test_query_sequences_equal_the_restatement(seed):
    ops, covis = K.random_sequence(seed)
    mine, _ = K.run_oracle(ops, len(covis), covis)
    _compare(run_device(ops, covis), mine, 64)


def test_constructed_cases_and_truncation():
    ops, covis = K.constructed_sequence()
    mine, seen = K.run_oracle(ops, len(covis), covis)
    assert all(seen[k] > 0 for k in ('tie', 'edge', 'stale', 'noshare_nb', 'dup_best', 'retain_tie', 'empty_frame', 'empty_map')), seen
    _compare(run_device(ops, covis), mine, 64)
    # cand_cap 1: the count before the cap shows the truncation
    dev = run_device(ops, covis, cand_cap=1)
    _compare(dev, mine, 1)
    assert any(got[2][f, 3] > got[1][f] for got, _ in dev for f in range(len(got[1])))


def test_batched_rows_equal_one_call_per_row():
    ops, covis = K.random_sequence(7, nmaps=4, nops=60)
    a, b = run_device(ops, covis), run_device(ops, covis, split=True)
    assert any(len(op[1]) > 1 for op in ops if op[0] == 'query')
    for (ga, sa), (gb, sb) in zip(a, b):
        assert all(np.array_equal(x, y) for x, y in zip(ga, gb)) and sa.tobytes() == sb.tobytes()


def test_skipped_rows_and_refused_calls_change_nothing():
    t = _torch()
    ops, covis = K.random_sequence(3)
    nadd = next(i for i, op in enumerate(ops) if op[0] == 'query')
    mine, _ = K.run_oracle(ops[:nadd + 1], len(covis), covis)
    db = Db(4, len(covis), 64)
    dcovis = t.from_numpy(np.ascontiguousarray(covis)).cuda()
    live = {}
    for op in ops[:nadd]:
        if op[0] == 'add':
            db.add(op[1], op[2], op[3]); live.update(zip(op[1], op[2]))
        elif op[0] == 'erase':
            db.erase(op[1]); [live.pop(s) for s in op[1]]
        elif op[0] == 'clear':
            db.clear(op[1]); live = {s: m for s, m in live.items() if m != op[1]}
    free = next(s for s in range(len(covis)) if s not in live)
    some = next(iter(live))
    bow = K.random_bow(np.random.default_rng(0), 160, 10, 20)
    big = (np.arange(70, dtype=np.int32), np.full(70, 1 / 70))
    before = db.scores()
    db.add([some], [0], [bow], expect=B.SGS_ERR_INVALID)                  # already live
    db.add([len(covis)], [0], [bow], expect=B.SGS_ERR_INVALID)            # out of range
    db.add([free, free], [0, 0], [bow, bow], expect=B.SGS_ERR_INVALID)    # twice in one call
    db.add([free], [4], [bow], expect=B.SGS_ERR_INVALID)                  # unknown map
    db.add([free], [0], [big], expect=B.SGS_ERR_INVALID)                  # bow_n > max_words
    db.erase([free], expect=B.SGS_ERR_INVALID)                            # not live
    db.erase([some, some], expect=B.SGS_ERR_INVALID)
    db.clear(4, expect=B.SGS_ERR_INVALID)
    op = ops[nadd]
    db.query([op[1][0], op[1][0]], [op[2][0], op[2][0]], dcovis, expect=B.SGS_ERR_INVALID)     # one map twice
    db.query([7], [op[2][0]], dcovis, expect=B.SGS_ERR_INVALID)
    assert db.scores().tobytes() == before.tobytes()
    # the query with a skipped row (-1) in front: that row keeps its sentinels, the others equal the restatement
    got = db.query([-1] + op[1], [bow] + op[2], dcovis)
    assert (got[0][0] == SENT).all() and got[1][0] == SENT and (got[2][0] == SENT).all()
    rows, sc = mine[-1]
    for f, want in enumerate(rows):
        _check_row(tuple(x[1:] for x in got), want, 64, 0, f)
    assert db.scores().tobytes() == sc.tobytes()
    db.close()


@pytest.mark.parametrize('n', [1000, 8192])
def test_bow_vector_equals_the_restatement(n):
    t = _torch()
    rng = np.random.default_rng(n)
    F = 4
    word = rng.integers(0, 600 if n == 1000 else 5000, (F, n)).astype(np.int32)
    weight = rng.uniform(0, 3, (F, n)); weight[:, ::9] = 0.0
    counts = np.array([n, n - 17, 0, 1], np.int32)
    dw, dwt, dc = t.from_numpy(word).cuda(), t.from_numpy(weight).cuda(), t.from_numpy(counts).cuda()
    ow = t.full((F, n), -5, dtype=t.int32, device='cuda'); ov = t.zeros((F, n), dtype=t.float64, device='cuda'); on = t.zeros(F, dtype=t.int32, device='cuda')
    B.check(B.lib().sgs_bow_vector_batch_device(dw.data_ptr(), dwt.data_ptr(), dc.data_ptr(), n, F, ow.data_ptr(), ov.data_ptr(), on.data_ptr(), None))
    t.cuda.synchronize()
    ow, ov, on = ow.cpu().numpy(), ov.cpu().numpy(), on.cpu().numpy()
    for f in range(F):
        ids, vals = O.bow_vector(word[f, :counts[f]], weight[f, :counts[f]])
        assert on[f] == len(ids) and np.array_equal(ow[f, :on[f]], ids) and ov[f, :on[f]].tobytes() == vals.tobytes(), f


def test_tracker_entry_equals_the_calls_one_by_one():
    """ComputeBoW + the query on the tracker's frames equals sgs_bow_transform_batch_device + sgs_bow_vector_batch_device +
    sgs_kfdb_reloc_candidates_device on the same frames; disabled rows are not written."""
    t = _torch()
    s = _setup(nb=6)
    trk, nb, cap = s['trk'], s['nb'], s['cap']
    L = B.lib()
    o = s['o']
    voc = R.train_vocabulary(np.concatenate([o['desc'][f, :o['cnt'][f]] for f in range(nb)]), 8, 3, seed=1)
    gv = GpuVoc(voc)
    kps, desc, cnt = C.c_void_p(), C.c_void_p(), C.c_void_p()
    B.check(L.sgs_tracker_results_device(trk.h, C.byref(kps), C.byref(desc), None, C.byref(cnt), None, None, None))
    # the database: every frame's BowVector (as computed one by one) as key frames of maps 0..2, two per map
    word = t.zeros((nb, cap), dtype=t.int32, device='cuda'); wt = t.zeros((nb, cap), dtype=t.float64, device='cuda'); node = t.zeros_like(word)
    bw = t.zeros_like(word); bv = t.zeros_like(wt); bn = t.zeros(nb, dtype=t.int32, device='cuda')
    B.check(L.sgs_bow_transform_batch_device(gv.h, desc, cnt, cap, nb, 4, word.data_ptr(), wt.data_ptr(), node.data_ptr(), None))
    B.check(L.sgs_bow_vector_batch_device(word.data_ptr(), wt.data_ptr(), cnt, cap, nb, bw.data_ptr(), bv.data_ptr(), bn.data_ptr(), None))
    db = Db(3, 16, cap)
    slots = np.arange(nb, dtype=np.int32); maps = (np.arange(nb) % 3).astype(np.int32)
    B.check(L.sgs_kfdb_add(db.h, nb, B._p(slots), B._p(maps), bw.data_ptr(), bv.data_ptr(), bn.data_ptr(), cap, None))
    covis = np.full((16, 10), -1, np.int32)
    for f in range(nb):
        covis[f, 0] = (f + 3) % nb
    dcovis = t.from_numpy(covis).cuda()
    qmap = np.array([0, 1, 2, -1, 0, 0], np.int32)
    en = np.array([1, 1, 1, 0, 0, 0], np.uint8)
    cc = 8
    res = []
    for entry in (True, False):
        cand = t.full((nb, cc), SENT, dtype=t.int32, device='cuda'); ncand = t.full((nb,), SENT, dtype=t.int32, device='cuda')
        stats = t.full((nb, 4), SENT, dtype=t.int32, device='cuda')
        if entry:
            a = B.RelocBatch(B._p(qmap), B._p(en), dcovis.data_ptr(), cand.data_ptr(), cc, ncand.data_ptr(), stats.data_ptr())
            B.check(L.sgs_tracker_reloc_candidates_device(trk.h, gv.h, db.h, C.byref(a), nb, None))
        else:
            m = np.where(en != 0, qmap, -1).astype(np.int32)
            B.check(L.sgs_kfdb_reloc_candidates_device(db.h, nb, B._p(m), bw.data_ptr(), bv.data_ptr(), bn.data_ptr(), cap, dcovis.data_ptr(),
                                                       cand.data_ptr(), cc, ncand.data_ptr(), stats.data_ptr(), None))
        t.cuda.synchronize()
        res.append((cand.cpu().numpy(), ncand.cpu().numpy(), stats.cpu().numpy(), db.scores()))
    for x, y in zip(res[0], res[1]):
        assert np.array_equal(x, y)
    cand, ncand, stats, _ = res[0]
    assert (ncand[:3] >= 1).all() and (cand[3:] == SENT).all() and (ncand[3:] == SENT).all() and (stats[3:] == SENT).all()
    assert all(f in cand[f, :ncand[f]] for f in range(3))          # a frame finds its own key frame
    # the whole tracker path against the restatement: the frames' BowVectors from the oracle's transform
    V = O.Vocabulary(voc['k'], voc['L'], voc['parent'], voc['desc'], voc['weight'])
    ref = K.Database(16)
    fb = []
    for f in range(nb):
        w_, wt_, _ = V.transform(o['desc'][f, :o['cnt'][f]], 4)
        fb.append(O.bow_vector(w_, wt_))
        ref.add(f, int(maps[f]), *fb[f])
    for f in range(3):
        wc, ws = ref.query(int(qmap[f]), *fb[f], covis)
        _check_row((cand, ncand, stats), (wc, ws), cc, 0, f)
    db.close(); gv.close(); trk.close()
