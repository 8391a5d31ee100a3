"""The device loop query (sgs_kfdb_loop_candidates_device) against the restatement of tests/kfdb_loop_cases.py, which tests/test_kfdb_loop_ref.py
pins to the reference's own KeyFrameDatabase.cc: candidates, counts, stats and minScore bit for bit over add / erase / clear / relocalisation / loop
sequences, with the relocalisation query's results and mRelocScore unchanged by the loop queries between them."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import kfdb_cases as K  # noqa: E402
import kfdb_loop_cases as KL  # noqa: E402
import oracle as O  # noqa: E402
from pysgs import binding as B  # noqa: E402
from test_gpu_kfdb import SENT, Db, _check_row  # noqa: E402

FSENT = np.float32(7777.5)


def _torch():
    import torch
    return torch


def _rows(bows, cap):
    w = np.zeros((len(bows), cap), np.int32); v = np.zeros((len(bows), cap)); n = np.array([len(b[0]) for b in bows], np.int32)
    for i, (ids, vals) in enumerate(bows):
        w[i, :len(ids)] = ids; v[i, :len(ids)] = vals
    return w, v, n


def _offsets(lists):
    return np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int32)


class LoopArgs:
    """the device arrays of one loop call: rows' BowVectors, connected ids and covisible BowVectors in CSR form, outputs at their sentinels"""

    def __init__(self, bows, conns, covs, cand_cap=64):
        t = _torch()
        F = len(bows)
        self.cap = max([len(b[0]) for b in bows] + [len(c[0]) for cs in covs for c in cs] + [1])
        self.q = [t.from_numpy(a).cuda() for a in _rows(bows, self.cap)]
        self.conn_off = _offsets(conns)
        self.conn = t.from_numpy(np.array([s for c in conns for s in c] + [0], np.int32)).cuda()
        self.cov_off = _offsets(covs)
        self.cov = [t.from_numpy(a).cuda() for a in _rows([c for cs in covs for c in cs] + [(np.zeros(0, np.int32), np.zeros(0))], self.cap)]
        self.cand_cap = cand_cap
        self.cand = t.full((F, cand_cap), SENT, dtype=t.int32, device='cuda'); self.ncand = t.full((F,), SENT, dtype=t.int32, device='cuda')
        self.stats = t.full((F, 4), SENT, dtype=t.int32, device='cuda'); self.ms = t.full((F,), float(FSENT), dtype=t.float32, device='cuda')

    def call(self, db, maps, dcovis, **over):
        a = dict(db=db.h, F=len(maps), map=np.array(maps, np.int32), qw=self.q[0].data_ptr(), qv=self.q[1].data_ptr(), qn=self.q[2].data_ptr(),
                 cap=self.cap, conn_off=self.conn_off, conn=self.conn.data_ptr(), cov_off=self.cov_off, cw=self.cov[0].data_ptr(),
                 cv=self.cov[1].data_ptr(), cn=self.cov[2].data_ptr(), covis=dcovis.data_ptr(), cand=self.cand.data_ptr(), cc=self.cand_cap,
                 ncand=self.ncand.data_ptr(), stats=self.stats.data_ptr(), ms=self.ms.data_ptr())
        a.update(over)
        return B.lib().sgs_kfdb_loop_candidates_device(a['db'], a['F'], B._p(a['map']), a['qw'], a['qv'], a['qn'], a['cap'], B._p(a['conn_off']), a['conn'],
                                                       B._p(a['cov_off']), a['cw'], a['cv'], a['cn'], a['covis'], a['cand'], a['cc'], a['ncand'],
                                                       a['stats'], a['ms'], None)

    def result(self):
        _torch().cuda.synchronize()
        return self.cand.cpu().numpy(), self.ncand.cpu().numpy(), self.stats.cpu().numpy(), self.ms.cpu().numpy()


def loop_query(db, maps, bows, conns, covs, dcovis, cand_cap=64):
    a = LoopArgs(bows, conns, covs, cand_cap)
    rc = a.call(db, maps, dcovis)
    assert rc == B.SGS_OK, B.lib().sgs_last_error()
    return a.result()


def run_device(ops, covis, nmaps=4, cand_cap=64, split=False):
    """per query op: ('query', (cand, ncand, stats), mRelocScore table) or ('loop', (cand, ncand, stats, min_score)); split: one call per row"""
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
        elif op[0] == 'query':
            out.append(('query', db.query(op[1], op[2], dcovis, cand_cap), db.scores()))
        elif split:
            res = [loop_query(db, [m], [b], [c], [cv], dcovis, cand_cap) for m, b, c, cv in zip(*op[1:5])]
            out.append(('loop', tuple(np.concatenate([r[i] for r in res]) for i in range(4))))
        else:
            out.append(('loop', loop_query(db, op[1], op[2], op[3], op[4], dcovis, cand_cap)))
    db.close()
    return out


def _check_loop_row(got, want, cand_cap, q, f):
    _check_row(got[:3], want[:2], cand_cap, q, f)
    assert got[3][f].tobytes() == np.float32(want[2]).tobytes(), (q, f, got[3][f], want[2])


def _compare(dev, mine, cand_cap):
    assert len(dev) == len(mine)
    for q, (d, m) in enumerate(zip(dev, mine)):
        assert d[0] == m[0]
        if d[0] == 'query':
            for f, want in enumerate(m[1]):
                _check_row(d[1], want, cand_cap, q, f)
            assert d[2].tobytes() == m[2].tobytes(), (q, np.nonzero(d[2] != m[2])[0])
        else:
            for f, want in enumerate(m[1]):
                _check_loop_row(d[1], want, cand_cap, q, f)


@pytest.mark.parametrize('seed', [1, 2, 3, 4, 5, 6])
def test_loop_sequences_equal_the_restatement(seed):
    ops, covis = KL.loop_sequence(seed)
    mine, _ = KL.run_oracle(ops, len(covis), covis)
    _compare(run_device(ops, covis), mine, 64)


def test_constructed_cases_and_truncation():
    ops, covis = KL.constructed_sequence()
    mine, db = KL.run_oracle(ops, len(covis), covis)
    assert all(v > 0 for k, v in db.lseen.items() if k != 'truncated'), db.lseen
    _compare(run_device(ops, covis), mine, 64)
    dev = run_device(ops, covis, cand_cap=1)
    _compare(dev, mine, 1)
    assert any(r[1][2][f, 3] > r[1][1][f] for r in dev if r[0] == 'loop' for f in range(len(r[1][1])))


def test_batched_rows_equal_one_call_per_row():
    ops, covis = KL.loop_sequence(7, nmaps=4, nops=60)
    a, b = run_device(ops, covis), run_device(ops, covis, split=True)
    assert any(len(op[1]) > 1 for op in ops if op[0] == 'loop')
    for x, y in zip(a, b):
        assert all(np.array_equal(p, q) for p, q in zip(x[1], y[1]))


def test_relocalisation_is_unchanged_by_loop_queries():
    """the relocalisation query's candidates, stats and mRelocScore, with and without the loop queries between them"""
    ops, covis = KL.loop_sequence(8, nops=60)
    with_loops = [r for r in run_device(ops, covis) if r[0] == 'query']
    without = run_device([op for op in ops if op[0] != 'loop'], covis)
    assert len(with_loops) == len(without) > 5
    for x, y in zip(with_loops, without):
        assert all(np.array_equal(p, q) for p, q in zip(x[1], y[1])) and x[2].tobytes() == y[2].tobytes()


def test_skipped_rows_and_refused_calls_change_nothing():
    t = _torch()
    ops, covis = KL.loop_sequence(3)
    k = next(i for i, op in enumerate(ops) if op[0] == 'loop' and len(op[1]) > 1)
    mine, _ = KL.run_oracle(ops[:k + 1], len(covis), covis)
    db = Db(4, len(covis), 128)
    dcovis = t.from_numpy(np.ascontiguousarray(covis)).cuda()
    for op in ops[:k]:
        if op[0] == 'add':
            db.add(op[1], op[2], op[3])
        elif op[0] == 'erase':
            db.erase(op[1])
        elif op[0] == 'clear':
            db.clear(op[1])
        elif op[0] == 'query':
            db.query(op[1], op[2], dcovis)
        else:
            loop_query(db, op[1], op[2], op[3], op[4], dcovis)
    op = ops[k]
    before = db.scores()
    a = LoopArgs(op[2], op[3], op[4])
    E, U = B.SGS_ERR_INVALID, B.SGS_ERR_UNSUPPORTED
    m0 = op[1][0]
    bad_off = a.conn_off.copy(); bad_off[1] = bad_off[2] + 1
    neg_off = a.cov_off.copy(); neg_off[0] = -1
    many = np.full(len(op[1]) + 1, 1, np.int32); many[0] = 0
    for rc, over in ((E, dict(map=np.array([m0, m0], np.int32), F=2)), (E, dict(map=np.array([7], np.int32), F=1)), (E, dict(F=0)),
                     (E, dict(conn_off=bad_off)), (E, dict(cov_off=neg_off)), (E, dict(conn=None, conn_off=np.maximum(a.conn_off, many))),
                     (E, dict(cw=None, cov_off=np.maximum(a.cov_off, many))), (E, dict(ms=None)), (E, dict(cc=0)), (U, dict(cap=(1 << 23) + 1))):
        assert a.call(db, op[1], dcovis, **over) == rc, (over, B.lib().sgs_last_error())
    cand, ncand, stats, ms = a.result()
    assert (cand == SENT).all() and (ncand == SENT).all() and (stats == SENT).all() and (ms == FSENT).all()
    assert db.scores().tobytes() == before.tobytes()
    # the same query with a skipped row (-1) in front: that row keeps its sentinels, the others equal the restatement
    sk = (np.arange(3, dtype=np.int32), np.full(3, 1 / 3))
    got = loop_query(db, [-1] + op[1], [sk] + op[2], [[0, 1]] + op[3], [[sk]] + op[4], dcovis)
    assert (got[0][0] == SENT).all() and got[1][0] == SENT and (got[2][0] == SENT).all() and got[3][0] == FSENT
    for f, want in enumerate(mine[-1][1]):
        _check_loop_row(tuple(x[1:] for x in got), want, 64, 0, f)
    assert db.scores().tobytes() == before.tobytes()
    db.close()


@pytest.mark.parametrize('n', [1000, 8192])
def test_device_bow_vectors_equal_the_restatement(n):
    """key frames, new key frames and covisible key frames whose BowVectors come from sgs_bow_vector_batch_device (n features each), used in
    place: the query rows and the covisible rows are rows of the same device array"""
    t = _torch()
    L = B.lib()
    rng = np.random.default_rng(n + 1)
    nb = 16
    word = rng.integers(0, 600 if n == 1000 else 5000, (nb, n)).astype(np.int32)
    weight = rng.uniform(0, 3, (nb, n)); weight[:, ::9] = 0.0
    counts = np.full(nb, n, np.int32); counts[5] = n // 3
    dw, dwt, dc = t.from_numpy(word).cuda(), t.from_numpy(weight).cuda(), t.from_numpy(counts).cuda()
    bw = t.zeros((nb, n), dtype=t.int32, device='cuda'); bv = t.zeros((nb, n), dtype=t.float64, device='cuda'); bn = t.zeros(nb, dtype=t.int32, device='cuda')
    B.check(L.sgs_bow_vector_batch_device(dw.data_ptr(), dwt.data_ptr(), dc.data_ptr(), n, nb, bw.data_ptr(), bv.data_ptr(), bn.data_ptr(), None))
    t.cuda.synchronize()
    hw, hv, hn = bw.cpu().numpy(), bv.cpu().numpy(), bn.cpu().numpy()
    bows = [(hw[f, :hn[f]].copy(), hv[f, :hn[f]].copy()) for f in range(nb)]
    for f in (0, 5):
        ids, vals = O.bow_vector(word[f, :counts[f]], weight[f, :counts[f]])
        assert np.array_equal(bows[f][0], ids) and bows[f][1].tobytes() == vals.tobytes()
    # frames 0..11 are key frames of maps 0 and 1; frames 12 and 13 are new key frames of maps 0 and 1, frame 4 is queried after its own add
    covis = np.full((nb, 10), -1, np.int32)
    for s in range(12):
        covis[s, :4] = [(s + 2 * j) % 12 for j in (1, 2, 3, 4)]
    dcovis = t.from_numpy(covis).cuda()
    db = Db(2, nb, n)
    slots = np.arange(12, dtype=np.int32); maps = (slots % 2).astype(np.int32)
    B.check(L.sgs_kfdb_add(db.h, 12, B._p(slots), B._p(maps), bw.data_ptr(), bv.data_ptr(), bn.data_ptr(), n, None))
    ref = KL.LoopDatabase(nb)
    for s in range(12):
        ref.add(s, int(maps[s]), *bows[s])
    calls = [([0, 1], [12, 13], [[2, 6], [3]], [(0, 3), (3, 5)]),          # covisible rows: frames 0..2 and 3..4
             ([-1, 0], [15, 4], [[], [2]], [(6, 6), (6, 9)])]               # frame 4 (slot 4, map 0) after its own add; covisible frames 6..8
    for maps_q, rows, conns, cov in calls:
        F = len(rows)
        qw = t.stack([bw[r] for r in rows]); qv = t.stack([bv[r] for r in rows]); qn = t.stack([bn[r] for r in rows])
        conn_off = _offsets(conns); conn = t.from_numpy(np.array([s for c in conns for s in c] + [0], np.int32)).cuda()
        cov_off = np.array([cov[0][0]] + [c[1] for c in cov], np.int32)
        cand = t.full((F, 64), SENT, dtype=t.int32, device='cuda'); ncand = t.full((F,), SENT, dtype=t.int32, device='cuda')
        stats = t.full((F, 4), SENT, dtype=t.int32, device='cuda'); ms = t.full((F,), float(FSENT), dtype=t.float32, device='cuda')
        B.check(L.sgs_kfdb_loop_candidates_device(db.h, F, B._p(np.array(maps_q, np.int32)), qw.data_ptr(), qv.data_ptr(), qn.data_ptr(), n,
                                                  B._p(conn_off), conn.data_ptr(), B._p(cov_off), bw.data_ptr(), bv.data_ptr(), bn.data_ptr(),
                                                  dcovis.data_ptr(), cand.data_ptr(), 64, ncand.data_ptr(), stats.data_ptr(), ms.data_ptr(), None))
        t.cuda.synchronize()
        got = (cand.cpu().numpy(), ncand.cpu().numpy(), stats.cpu().numpy(), ms.cpu().numpy())
        for f, m in enumerate(maps_q):
            if m < 0:
                assert got[1][f] == SENT and got[3][f] == FSENT
                continue
            want = ref.loop(m, *bows[rows[f]], conns[f], [bows[c] for c in range(*cov[f])], covis, rows[f] if rows[f] < 12 else -1)
            _check_loop_row(got, want, 64, 0, f)
            assert got[2][f, 0] > 0 and got[1][f] > 0, (f, got[2][f])
    assert ref.lseen['self_cand'] == 1
    db.close()


def test_a_map_above_the_query_limit_is_refused():
    """a queried map of 16385 key frames: SGS_ERR_UNSUPPORTED before anything is enqueued; at 16384 (the row kernel's largest shared-memory sort)
    the same call runs"""
    t = _torch()
    n = 16385
    db = Db(2, n, 4)
    w = t.zeros((n, 4), dtype=t.int32, device='cuda'); w[:, 0] = t.arange(n, device='cuda', dtype=t.int32) % 50
    v = t.zeros((n, 4), dtype=t.float64, device='cuda'); v[:, 0] = 1.0
    cnt = t.ones(n, dtype=t.int32, device='cuda')
    slots = np.arange(n, dtype=np.int32)
    B.check(B.lib().sgs_kfdb_add(db.h, n, B._p(slots), B._p(np.zeros(n, np.int32)), w.data_ptr(), v.data_ptr(), cnt.data_ptr(), 4, None))
    dcovis = t.full((n, 10), -1, dtype=t.int32, device='cuda')
    bow = (np.array([7], np.int32), np.ones(1))
    a = LoopArgs([bow], [[7]], [[bow]])                              # slot 7 shares word 7 but is connected
    assert a.call(db, [0], dcovis) == B.SGS_ERR_UNSUPPORTED, B.lib().sgs_last_error()
    cand, ncand, stats, ms = a.result()
    assert (cand == SENT).all() and (ncand == SENT).all() and (stats == SENT).all() and (ms == FSENT).all()
    db.erase([n - 1])
    assert a.call(db, [0], dcovis) == B.SGS_OK, B.lib().sgs_last_error()
    cand, ncand, stats, ms = a.result()
    share = sum(1 for k in range(n - 1) if k % 50 == 7) - 1
    assert list(stats[0]) == [share, 1, share, share] and ncand[0] == 64 and ms[0] == 1.0     # minScore = score(bow, bow) = 1
    assert 7 not in cand[0] and all(k % 50 == 7 for k in cand[0])
    db.close()
