"""KeyFrameDatabase::DetectLoopCandidates (src/KeyFrameDatabase.cc:76-197) and LoopClosing::DetectLoop's minScore (src/LoopClosing.cc:124-138)
restated for the tests, on the database of tests/kfdb_cases.py, and the sequences the tests run: those of tests/kfdb_cases.py with loop queries
interleaved.

A loop op is ('loop', [map or -1], [(ids, vals)], [connected slots], [[covisible (ids, vals)]], [self slot or -1]): per row the new key frame's
BowVector, its connected set, the BowVectors of its covisible key frames, and the slot it occupies when it is already in the database (the
reference's driver then queries with that key frame; the device needs no such input).  The restatement is literal: per key frame mnLoopQuery /
mnLoopWords / mLoopScore, every query a new key frame id, the inverted file walked word by word with the connected set tested as the reference
tests it.  `lseen` counts the paths the loop queries took."""
import numpy as np

import kfdb_cases as K

F32 = np.float32


def min_score(fids, fvals, covs):
    """DetectLoop's minScore: from 1, the least float(L1Scoring::score) against the covisible BowVectors, in order, by strict <"""
    ms = F32(1)
    for ids, vals in covs:
        s = K.score_l1(np.asarray(fids, np.int32), np.asarray(fvals, np.float64), np.asarray(ids, np.int32), np.asarray(vals, np.float64))
        if s < ms:
            ms = s
    return ms


class LoopDatabase(K.Database):
    def __init__(self, max_keyframes):
        super().__init__(max_keyframes)
        self.loop_query = np.zeros(max_keyframes, np.int64)          # mnLoopQuery, mnLoopWords, mLoopScore of every slot
        self.loop_words = np.zeros(max_keyframes, np.int64)
        self.loop_score = np.zeros(max_keyframes, np.float32)
        self.next_id = 1                                             # LoopClosing never queries key frame 0
        self.lseen = dict(conn_most=0, conn_nb=0, si_eq_min=0, nb_below_min=0, nb_edge=0, no_cov=0, cov_not_in_db=0, zero_min=0, retain_tie=0,
                          dup_best=0, empty_frame=0, empty_map=0, self_cand=0, truncated=0)

    def loop(self, m, fids, fvals, conn, covs, covis, self_slot=-1, cand_cap=1 << 30):
        """(candidate slots, stats [4], minScore) of one new key frame of map m"""
        fids = np.asarray(fids, np.int32); fvals = np.asarray(fvals, np.float64)
        ms = min_score(fids, fvals, covs)
        slots = sorted((s for s, mm in self.map.items() if mm == m), key=lambda s: self.seq[s])
        live_bows = [self.bow[s] for s in slots]
        if not covs:
            self.lseen['no_cov'] += 1
        if any(not any(np.array_equal(ids, b[0]) and np.array_equal(vals, b[1]) for b in live_bows) for ids, vals in covs):
            self.lseen['cov_not_in_db'] += 1
        if ms == 0:
            self.lseen['zero_min'] += 1
        if not slots:
            self.lseen['empty_map'] += 1
        if len(fids) == 0:
            self.lseen['empty_frame'] += 1
        qid = self.next_id; self.next_id += 1
        connected = set(conn)
        inverted = {}
        for s in slots:
            for w in self.bow[s][0].tolist():
                inverted.setdefault(w, []).append(s)
        sharing = []
        for w in fids.tolist():                                      # :86-104
            for s in inverted.get(w, ()):
                if self.loop_query[s] != qid:
                    self.loop_words[s] = 0
                    if s not in connected:
                        self.loop_query[s] = qid
                        sharing.append(s)
                self.loop_words[s] += 1
        if not sharing:
            return [], [0, 0, 0, 0], ms
        maxc = max(int(self.loop_words[s]) for s in sharing)         # :113-118
        minc = int(F32(maxc) * F32(0.8))                             # :120
        common = {s: len(np.intersect1d(fids, self.bow[s][0])) for s in slots if s in connected}
        if any(c > maxc for c in common.values()):
            self.lseen['conn_most'] += 1
        nscores, matches = 0, []
        for s in sharing:                                            # :125-139
            if self.loop_words[s] > minc:
                nscores += 1
                si = K.score_l1(fids, fvals, *self.bow[s])
                self.loop_score[s] = si
                if si >= ms:
                    matches.append((si, s))
                    if si == ms:
                        self.lseen['si_eq_min'] += 1
        if not matches:
            return [], [len(sharing), maxc, nscores, 0], ms
        acc_list, best_acc = [], ms
        for si, s in matches:                                        # :148-173
            best, acc, pbest = si, si, s
            for nb in covis[s][:K.NEIGH].tolist():
                if nb < 0:
                    continue
                if common.get(nb, 0) > minc:
                    self.lseen['conn_nb'] += 1
                if self.loop_query[nb] == qid and self.loop_words[nb] > minc:
                    if self.loop_score[nb] < ms:
                        self.lseen['nb_below_min'] += 1
                    acc = F32(acc + self.loop_score[nb])
                    if self.loop_score[nb] > best:
                        pbest, best = nb, self.loop_score[nb]
                elif self.loop_query[nb] == qid and minc > 0 and self.loop_words[nb] == minc:
                    self.lseen['nb_edge'] += 1
            acc_list.append((acc, pbest))
            if acc > best_acc:
                best_acc = acc
        keep_above = F32(F32(0.75) * best_acc)                       # :176
        out, added = [], set()
        for acc, pbest in acc_list:                                  # :182-193
            if acc == keep_above:
                self.lseen['retain_tie'] += 1
            if acc > keep_above:
                if pbest in added:
                    self.lseen['dup_best'] += 1
                else:
                    out.append(pbest); added.add(pbest)
        if self_slot >= 0 and self_slot in out:
            self.lseen['self_cand'] += 1
        if len(out) > cand_cap:
            self.lseen['truncated'] += 1
        return out, [len(sharing), maxc, nscores, len(out)], ms


def run_oracle(ops, max_keyframes, covis, cand_cap=1 << 30):
    """per query op, in order: ('query', rows, mRelocScore table) or ('loop', rows of (candidates, stats, minScore)); the database (its seen and
    lseen path counts)"""
    db = LoopDatabase(max_keyframes)
    out = []
    for op in ops:
        if op[0] == 'add':
            for s, m, (ids, vals) in zip(op[1], op[2], op[3]):
                db.add(s, m, ids, vals)
        elif op[0] == 'erase':
            for s in op[1]:
                db.erase(s)
        elif op[0] == 'clear':
            db.clear(op[1])
        elif op[0] == 'query':
            out.append(('query', [db.query(m, ids, vals, covis, cand_cap) if m >= 0 else None for m, (ids, vals) in zip(op[1], op[2])],
                        db.score.copy()))
        else:
            out.append(('loop', [db.loop(m, ids, vals, conn, covs, covis, sf, cand_cap) if m >= 0 else None
                                 for m, (ids, vals), conn, covs, sf in zip(*op[1:])]))
    return out, db


def random_loop(rng, live, bows, nmaps, slots, nvoc):
    """one loop op on the live key frames {slot: map} with BowVectors {slot: (ids, vals)}: per map of a random subset, a new key frame (a random
    BowVector, or one of the map's key frames queried after its own add), connected slots (of the map, of other maps, not live, out of range) and
    0-4 covisible BowVectors (the map's key frames' or random ones)"""
    maps = rng.permutation(nmaps).tolist()[:int(rng.integers(1, nmaps + 1))]
    rows = ([], [], [], [], [])
    for m in maps:
        mine = sorted(s for s, mm in live.items() if mm == m)
        self_slot = int(rng.choice(mine)) if mine and rng.uniform() < 0.25 else -1
        bow = bows[self_slot] if self_slot >= 0 else K.random_bow(rng, nvoc, 0 if rng.uniform() < 0.05 else 10, 60)
        conn = [int(s) for s in rng.choice(mine, min(len(mine), int(rng.integers(0, 6))), replace=False)] if mine else []
        conn += [int(s) for s in rng.integers(-2, slots + 2, int(rng.integers(0, 3)))]
        conn = [s for s in conn if s != self_slot]
        covs = []
        for _ in range(int(rng.integers(0, 5))):
            covs.append(bows[int(rng.choice(mine))] if mine and rng.uniform() < 0.5 else K.random_bow(rng, nvoc, 5, 40))
        for r, x in zip(rows, (m, bow, conn, covs, self_slot)):
            r.append(x)
    return ('loop',) + rows


def loop_sequence(seed, nmaps=3, slots=48, nvoc=160, nops=40):
    """K.random_sequence(seed, ...) unchanged, with a loop op after about half of its ops"""
    ops, covis = K.random_sequence(seed, nmaps, slots, nvoc, nops)
    rng = np.random.default_rng(seed + 1000)
    live, bows, out = {}, {}, []
    for op in ops:
        out.append(op)
        if op[0] == 'add':
            live.update(zip(op[1], op[2])); bows.update(zip(op[1], op[3]))
        elif op[0] == 'erase':
            for s in op[1]:
                del live[s]
        elif op[0] == 'clear':
            live = {s: m for s, m in live.items() if m != op[1]}
        if rng.uniform() < 0.5:
            out.append(random_loop(rng, live, bows, nmaps, slots, nvoc))
    return out, covis


def constructed_sequence():
    """A sequence that forces each path of the loop query; map 0 carries the cases, map 1 stays empty.  Word values are dyadic, so every score is
    exact (the score of two L1-normalised BowVectors is the sum of the smaller value over their common words)."""
    covis = np.full((16, K.NEIGH), -1, np.int32)
    Q = (np.arange(1, 9, dtype=np.int32), np.full(8, 0.125))                               # eight words 1..8
    b2 = (np.arange(1, 7, dtype=np.int32), np.array([0.25, 0.25, 0.125, 0.125, 0.125, 0.125]))   # against Q: 6 words, 0.75
    b3 = (np.arange(1, 6, dtype=np.int32), np.array([0.25, 0.25, 0.25, 0.125, 0.125]))           # 5 words, 0.625
    b4 = (np.arange(1, 5, dtype=np.int32), np.full(4, 0.25))                                     # 4 words, 0.5
    off_db = (np.arange(1, 8, dtype=np.int32), np.array([0.25] + [0.125] * 6))                   # 0.875, no key frame of the database
    far = (np.array([100, 101], np.int32), np.array([0.5, 0.5]))                                 # no common word: score -0
    ops = []
    # slot 1 is connected and shares all eight words (more than any listed key frame: maxCommonWords stays 6, the gate int(6 * 0.8f) = 4);
    # slot 2 is listed with 6 words, slot 3 with 5, slot 4 with 4 (at the gate: not scored); slot 2's best neighbours are 3, 4 and 1
    ops.append(('add', [1, 2, 3, 4], [0] * 4, [Q, b2, b3, b4]))
    covis[2, :3] = [3, 4, 1]
    # minScore 0.75 from slot 2's own BowVector (slot 2: si == minScore, kept; slot 3: 0.625 below it, still added as slot 2's neighbour);
    # connected ids that are not live, negative or out of range are ignored; map 1 is empty and has no covisible key frame (minScore 1)
    ops.append(('loop', [0, 1], [Q, Q], [[1, 9, -1, 99], []], [[b2, off_db], []], [-1, -1]))
    ops.append(('query', [0], [Q]))
    # slot 2 queried after its own add, no covisible key frame: minScore 1 == its own score, it is its own candidate
    ops.append(('loop', [0], [b2], [[1]], [[]], [2]))
    # an empty BowVector; a covisible key frame without a common word: minScore -0
    ops.append(('loop', [0], [(np.zeros(0, np.int32), np.zeros(0))], [[]], [[far, b3]], [-1]))
    # the 0.75 tie: slot 6 scores exactly 0.75, slot 7 a little more, slot 8 scores 1 alone (minScore 0.5)
    ops.append(('clear', 0))
    q = (np.arange(1, 9, dtype=np.int32), np.concatenate([np.full(4, 0.125), np.full(4, 0.0625)]))
    q2 = (np.arange(1, 9, dtype=np.int32), np.concatenate([np.full(4, 0.125), np.full(3, 0.0625), [0.0625 + 2.0 ** -12]]))
    ops.append(('add', [6, 7, 8], [0, 0, 0], [q, q2, Q]))
    ops.append(('loop', [0], [Q], [[]], [[b4]], [-1]))
    # a duplicated pBestKF: slots 10 and 11 both have slot 12 (score 1) as their best neighbour
    ops.append(('add', [10, 11, 12], [0, 0, 0], [q, q2, Q]))
    covis[10, :1] = [12]; covis[11, :1] = [12]
    ops.append(('loop', [0], [Q], [[]], [[b4, far]], [-1]))
    return ops, covis
