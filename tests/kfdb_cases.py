"""KeyFrameDatabase (src/KeyFrameDatabase.cc:33-74) and DetectRelocalizationCandidates (:199-311) restated for the tests, one database per map as
sgs_kfdb keeps them, and the add / erase / clear / query sequences the tests run on it.

The restatement walks the inverted file the way the reference does (the frame's words ascending, each word's key frames in add order), scores with
DBoW2's L1Scoring (the float64 sum of |v - w| - |v| - |w| over the common words in ascending order, then -score / 2, rounded to float) and accumulates
in float.  mRelocScore is 0 after an add (the reference leaves it uninitialised: DESIGN.md Q16).  `seen` counts the paths each query took, so that a
test can assert the sequence forced them."""
import numpy as np

F32 = np.float32
NEIGH = 10


class Database:
    def __init__(self, max_keyframes):
        self.map, self.seq, self.bow = {}, {}, {}
        self.score = np.zeros(max_keyframes, np.float32)
        self.next_seq = 0
        self.seen = dict(tie=0, edge=0, stale=0, noshare_nb=0, dup_best=0, retain_tie=0, empty_frame=0, empty_map=0, truncated=0)

    def add(self, slot, m, ids, vals):
        self.map[slot] = m; self.seq[slot] = self.next_seq; self.next_seq += 1
        self.bow[slot] = (np.asarray(ids, np.int32), np.asarray(vals, np.float64))
        self.score[slot] = 0

    def erase(self, slot):
        del self.map[slot]

    def clear(self, m):
        for s in [s for s, mm in self.map.items() if mm == m]:
            del self.map[s]

    def query(self, m, fids, fvals, covis, cand_cap=1 << 30):
        """(candidate slots, stats [4]) of one frame against map m; updates mRelocScore like the reference."""
        fids = np.asarray(fids, np.int32); fvals = np.asarray(fvals, np.float64)
        slots = sorted((s for s, mm in self.map.items() if mm == m), key=lambda s: self.seq[s])
        if not slots:
            self.seen['empty_map'] += 1
        if len(fids) == 0:
            self.seen['empty_frame'] += 1
        inverted = {}                                               # mvInvertedFile of this map: each word's key frames in add order
        for s in slots:
            for w in self.bow[s][0].tolist():
                inverted.setdefault(w, []).append(s)
        cnt, order = {}, []
        for w in fids.tolist():                                     # :207-222
            for s in inverted.get(w, ()):
                if s not in cnt:
                    cnt[s] = 0; order.append(s)
                cnt[s] += 1
        if not order:
            return [], [0, 0, 0, 0]
        maxc = max(cnt.values())
        minc = int(F32(maxc) * F32(0.8))                            # :235
        if sum(c == maxc for c in cnt.values()) > 1:
            self.seen['tie'] += 1
        if minc > 0 and any(c == minc for c in cnt.values()):
            self.seen['edge'] += 1
        scored = []
        for s in order:                                             # :242-253
            if cnt[s] > minc:
                si = score_l1(fids, fvals, *self.bow[s])
                self.score[s] = si
                scored.append((si, s))
        acc_list, best_acc = [], F32(0)
        scored_set = {s for _, s in scored}
        for si, s in scored:                                        # :262-287
            best, acc, pbest = si, si, s
            for nb in covis[s][:NEIGH].tolist():
                if nb < 0:
                    continue
                if nb not in cnt:
                    self.seen['noshare_nb'] += 1
                    continue
                if nb not in scored_set:
                    self.seen['stale'] += 1
                acc = F32(acc + self.score[nb])
                if self.score[nb] > best:
                    pbest, best = nb, self.score[nb]
            acc_list.append((acc, pbest))
            if acc > best_acc:
                best_acc = acc
        keep_above = F32(F32(0.75) * best_acc)                      # :290
        out, added = [], set()
        for acc, pbest in acc_list:
            if acc == keep_above:
                self.seen['retain_tie'] += 1
            if acc > keep_above:
                if pbest in added:
                    self.seen['dup_best'] += 1
                else:
                    out.append(pbest); added.add(pbest)
        if len(out) > cand_cap:
            self.seen['truncated'] += 1
        return out, [len(order), maxc, len(scored), len(out)]


def score_l1(a_ids, a_vals, b_ids, b_vals):
    """float(L1Scoring::score(a, b)), ScoringObject.cpp:23-68"""
    _, ia, ib = np.intersect1d(a_ids, b_ids, assume_unique=True, return_indices=True)
    s = 0.0
    for i, j in zip(ia.tolist(), ib.tolist()):
        vi, wi = float(a_vals[i]), float(b_vals[j])
        s += abs(vi - wi) - abs(vi) - abs(wi)
    return F32(-s / 2.0)


def normalized(ids, raw):
    """a BowVector from raw per-word sums: ids ascending, values divided by their serial L1 norm (BowVector::normalize)"""
    o = np.argsort(ids)
    ids = np.asarray(ids, np.int32)[o]; raw = np.asarray(raw, np.float64)[o]
    norm = 0.0
    for v in raw.tolist():
        norm += abs(v)
    return ids, (raw / norm if norm > 0 else raw)


def random_bow(rng, nvoc, nmin, nmax):
    n = int(rng.integers(nmin, nmax + 1))
    ids = rng.choice(nvoc, n, replace=False)
    return normalized(ids, rng.uniform(0.05, 1.0, n))


def random_sequence(seed, nmaps=3, slots=48, nvoc=160, nops=40):
    """ops: ('add', [slot], [map], [(ids, vals)]), ('erase', [slot]), ('clear', map), ('query', [map or -1], [(ids, vals)]); covis [slots][10]"""
    rng = np.random.default_rng(seed)
    covis = np.full((slots, NEIGH), -1, np.int32)
    for s in range(slots):                                          # any other slots: of the same map, of other maps, not live
        nb = [t for t in rng.permutation(slots).tolist() if t != s][:int(rng.integers(0, NEIGH + 1))]
        covis[s, :len(nb)] = nb
    live, ops = {}, []
    for k in range(nops):
        r = rng.uniform()
        free = [s for s in range(slots) if s not in live]
        if (r < 0.45 or len(live) < 6) and free:
            ss = rng.choice(free, min(len(free), int(rng.integers(1, 5))), replace=False).tolist()
            ms = rng.integers(0, nmaps, len(ss)).tolist()
            ops.append(('add', ss, ms, [random_bow(rng, nvoc, 8, 40) for _ in ss]))
            live.update(zip(ss, ms))
        elif r < 0.55 and live:
            ss = rng.choice(sorted(live), min(len(live), int(rng.integers(1, 3))), replace=False).tolist()
            ops.append(('erase', ss))
            for s in ss:
                del live[s]
        elif r < 0.58:
            m = int(rng.integers(0, nmaps)); ops.append(('clear', m))
            live = {s: mm for s, mm in live.items() if mm != m}
        else:
            maps = rng.permutation(nmaps).tolist()[:int(rng.integers(1, nmaps + 1))]
            ops.append(('query', maps, [random_bow(rng, nvoc, 0 if k % 11 == 0 else 10, 60) for _ in maps]))
    return ops, covis


def constructed_sequence():
    """A sequence that forces each path of the query; map 0 carries the cases, map 1 stays empty.  Word values are dyadic, so every score is exact."""
    covis = np.full((16, NEIGH), -1, np.int32)
    eighth = np.full(8, 0.125)
    F = (np.arange(1, 9, dtype=np.int32), eighth)                   # eight words 1..8, 0.125 each
    ops = []
    # slots 0 and 1: all eight words (tie at maxCommonWords 8, score 1); slot 2: 6 of them (int(8 * 0.8f) = 6: at the edge, not scored);
    # slot 3: seven (scored); slot 4: one word (shares, far below the gate)
    # slot 9: seven words like slot 3
    seven = (np.arange(1, 8, dtype=np.int32), np.full(7, 1 / 7))
    ops.append(('add', [0, 1, 2, 3, 4, 9], [0] * 6, [F, F, (np.arange(1, 7, dtype=np.int32), np.full(6, 1 / 6)), seven,
                                                     (np.array([8], np.int32), np.ones(1)), seven]))
    covis[3, :3] = [4, 5, 2]                                        # 4 and 2 share words but are not scored; 5 never shares a word
    covis[9, :1] = [4]                                              # once slot 4's stale score is 1, it is pBestKF of both 3 and 9
    covis[0, :1] = [1]; covis[1, :1] = [0]
    ops.append(('add', [5], [0], [(np.array([100, 101], np.int32), np.array([0.5, 0.5]))]))
    ops.append(('query', [0, 1], [F, (np.arange(1, 4, dtype=np.int32), np.full(3, 1 / 3))]))     # map 1: no key frames
    # slot 4 scored alone (a frame of word 8 only), so that its score is stale in the next query
    ops.append(('query', [0], [(np.array([8], np.int32), np.ones(1))]))
    ops.append(('query', [0], [F]))
    ops.append(('query', [0], [(np.zeros(0, np.int32), np.zeros(0))]))    # empty BowVector
    # erase slot 0 and add it again: it moves behind slot 1 in every inverted list
    ops.append(('erase', [0]))
    ops.append(('add', [0], [0], [F]))
    ops.append(('query', [0], [F]))
    # the 0.75 tie: slot 6 scores exactly 0.75 (four words at 0.125, four at 0.0625), slot 7 a little more; slot 8 scores 1 alone
    ops.append(('clear', 0))
    q = (np.arange(1, 9, dtype=np.int32), np.concatenate([np.full(4, 0.125), np.full(4, 0.0625)]))
    q2 = (np.arange(1, 9, dtype=np.int32), np.concatenate([np.full(4, 0.125), np.full(3, 0.0625), [0.0625 + 2.0 ** -12]]))
    ops.append(('add', [6, 7, 8], [0, 0, 0], [q, q2, F]))
    ops.append(('query', [0], [F]))
    return ops, covis


def run_oracle(ops, max_keyframes, covis, cand_cap=1 << 30):
    """every query's (candidates, stats) per row and the mRelocScore table after it, and the path counts"""
    db = Database(max_keyframes)
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
        else:
            rows = [db.query(m, ids, vals, covis, cand_cap) if m >= 0 else None for m, (ids, vals) in zip(op[1], op[2])]
            out.append((rows, db.score.copy()))
    return out, db.seen
