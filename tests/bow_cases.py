"""Constructed inputs for the bag-of-words pieces (numpy only, no device): vocabulary trees and matcher inputs built so that one path of
sg-slam_b200/csrc/bow.cu (and of its CPU restatement oracle/bow.cpp) MUST be taken.  Every case carries a proof -- an assertion on the
oracle's result that holds only if the path was taken (for example "the third key-frame feature of the bucket matched its third choice,
because the first two claimed its first and second") -- so that an edit to a builder cannot quietly turn a hard case into an easy one.

Vocabulary case: name, k, L, parent / desc / weight (like scenarios.random_vocabulary; weights are float32-representable so that a binary
vocabulary file holds the same tree), queries [n][32] and proof(result), result = {levelsup: (word, weight, node)} from run_voc_oracle.

Matcher case: name, mode (0: SearchByBoW(KF, F), 1: SearchByBoW(KF1, KF2), 2: SearchForTriangulation), params (nnratio, check_ori,
only_stereo), side arrays `a` (key frame / first key frame) and `b` (frame / second key frame), the triangulation geometry (F12, the first
key frame's centre cw and the epipole (ex, ey) computed from it by the reference's expression) and proof(result).  run_oracle(case)
returns dict(nm, m): m is indexed by the frame's features in mode 0 and by the first key frame's features in modes 1 and 2 -- the layout
of the batched device entry point's match_f.  The tests build the same dict from the reference and from the device.

Descriptors are placed at exact Hamming distances: a candidate is its key-frame descriptor with a chosen number of distinct bits flipped,
fillers are uniform random descriptors (about 128 bits away; the builders re-draw any filler closer than FAR)."""
import numpy as np

import oracle as O
import scenarios as S

f32 = np.float32
TH_LOW = 50
FACTOR = f32(f32(30) / f32(360))                       # HISTO_LENGTH / 360.0f
SF = S.scale_factors().astype(f32)
SIGMA2 = (SF * SF).astype(f32)
CAM = np.array([535.4, 539.2, 320.1, 247.6, 40.0, 0, 0, 640, 480], f32)     # fx fy cx cy bf, image bounds
CW = np.array([0.31, -0.07, 2.5], f32)                 # the first key frame's centre in the second key frame's (identity) camera
F_LINE = np.array([[0, 0, 0], [0, 0, -1], [0, 1, 0]], f32)                 # l = x1' F12: the epipolar line of (x1, y1) is y2 = y1
FAR = 96


def hamming(a, b):
    return int(np.unpackbits(np.bitwise_xor(a, b)).sum())


_POPC = np.unpackbits(np.arange(256, dtype=np.uint8)[:, None], axis=1).sum(1).astype(np.int32)


def dist_matrix(A, B):
    """Hamming distances [len(A)][len(B)]."""
    return _POPC[A[:, None, :] ^ B[None, :, :]].sum(2)


def flip(d, n, rng):
    b = np.unpackbits(d)
    b[rng.choice(256, n, replace=False)] ^= 1
    return np.packbits(b)


def epipole(cw=CW):
    """(ex, ey) of src/ORBmatcher.cc:667-672 with the second key frame at the identity: C2 = Cw, invz = 1.0f / C2z, ex = fx*C2x*invz + cx."""
    invz = f32(1.0) / cw[2]
    return f32(f32(f32(CAM[0] * cw[0]) * invz) + CAM[2]), f32(f32(f32(CAM[1] * cw[1]) * invz) + CAM[3])


def _neighbours(v, n):
    v = f32(v)
    out = [v]
    lo = hi = v
    for _ in range(n):
        lo = np.nextafter(lo, f32(-np.inf)); hi = np.nextafter(hi, f32(np.inf))
        out += [lo, hi]
    return np.sort(np.array(out, f32))


# ---- vocabularies ------------------------------------------------------------------------------------------------------------------
def _weights(n, rng):
    return (rng.randint(1, 64, n) / 8.0).astype(np.float64)          # multiples of 1/8: exact in float32


def _fanout_vocab(k, seed):
    """L = 2: a root with k children, two leaves under each.  Ties planted between root children (0, 32), (31, 32), (0, 64) and
    (last, first) where k allows (some pairs straddle a 32-lane group); each planted query is equidistant from its two children and
    farther from all others; the leaves under the first child of every pair are stopped words (weight 0)."""
    rng = np.random.RandomState(seed)
    pairs = [p for p in ((0, 32), (31, 32), (0, 64), (k - 1, 0)) if max(p) < k and p[0] != p[1]]
    base = rng.randint(0, 256, 32).astype(np.uint8)
    child = rng.randint(0, 256, (k, 32)).astype(np.uint8)
    sets = {}
    for c in sorted({c for p in pairs for c in p}):
        sets[c] = rng.choice(256, 12, replace=False)
        bits = np.unpackbits(base); bits[sets[c]] ^= 1
        child[c] = np.packbits(bits)
    queries, winners = [], []
    for a, b in pairs:
        diff = np.nonzero(np.unpackbits(child[a] ^ child[b]))[0]
        sa = [i for i in diff if i in set(sets[a])]; sb = [i for i in diff if i in set(sets[b])]
        h = sa[:len(sa) // 2] + sb[:len(sb) - len(sb) // 2]            # half of the differing bits, from both sides
        bits = np.unpackbits(child[a]); bits[h] ^= 1
        q = np.packbits(bits)
        d = np.unpackbits(q[None] ^ child, axis=1).sum(1)
        assert d[a] == d[b] and (np.delete(d, [a, b]) > d[a]).all(), ('planted tie', k, a, b)
        queries.append(q); winners.append(min(a, b))
    parent = [-1] + [0] * k
    desc = [np.zeros(32, np.uint8)] + list(child)
    for c in range(k):
        for _ in range(2):
            parent.append(1 + c); desc.append(flip(child[c], 20, rng))
    parent = np.array(parent, np.int32); desc = np.stack(desc)
    weight = np.zeros(len(parent)); leaf = np.arange(1 + k, len(parent))
    weight[leaf] = _weights(len(leaf), rng)
    for w in winners:
        weight[parent == 1 + w] = 0.0
    nplant = len(queries)
    leaves = desc[leaf[rng.randint(0, len(leaf), 150)]]
    queries = np.concatenate([np.array(queries, np.uint8).reshape(-1, 32), np.stack([flip(d, rng.randint(0, 25), rng) for d in leaves]),
                              rng.randint(0, 256, (60, 32)).astype(np.uint8)])

    def proof(r):
        word, w, node = r[1]                                            # levelsup = L - 1: the node at level 1 = the root child taken
        for i, c in enumerate(winners):
            assert node[i] == 1 + c, ('the first of two equidistant children wins', k, pairs[i], node[i])
            assert w[i] == 0 and r[0][1][i] == 0, 'the planted query reaches a stopped word'
    return dict(name='voc_fan%d' % k, k=k, L=2, parent=parent, desc=desc, weight=weight, queries=queries, proof=proof, nplant=nplant)


def _equidistant_vocab(k, seed):
    """L = 1: every child of the root is 3 bits away from one descriptor (child 0 must win), and random descriptors tie on many children."""
    rng = np.random.RandomState(seed)
    q = rng.randint(0, 256, 32).astype(np.uint8)
    seen, child = set(), []
    while len(child) < k:
        s = tuple(sorted(rng.choice(256, 3, replace=False)))
        if s in seen:
            continue
        seen.add(s)
        bits = np.unpackbits(q); bits[list(s)] ^= 1
        child.append(np.packbits(bits))
    parent = np.array([-1] + [0] * k, np.int32); desc = np.stack([np.zeros(32, np.uint8)] + child)
    weight = np.zeros(k + 1); weight[1:] = _weights(k, rng)
    queries = np.concatenate([q[None], np.stack([flip(q, 4, rng) for _ in range(100)]), rng.randint(0, 256, (100, 32)).astype(np.uint8)])

    def proof(r):
        d = dist_matrix(q[None], desc[1:])[0]
        assert (d == 3).all() and r[0][0][0] == 0, 'equidistant from every child: child 0'
        dq = dist_matrix(queries[1:], desc[1:])
        ties = (dq == dq.min(1, keepdims=True)).sum(1) > 1
        assert ties.sum() > 50 and np.array_equal(r[0][0][1:], dq.argmin(1)), 'many ties, first child of the minimum'
    return dict(name='voc_equi%d' % k, k=k, L=1, parent=parent, desc=desc, weight=weight, queries=queries, proof=proof)


def _unbalanced_vocab(seed, L=6):
    """Eight children under the root, then variable fan-out (1, 2, 3 or 5) with single-child chains, leaves at every depth from 2 to L, identical siblings now and then."""
    rng = np.random.RandomState(seed)
    parent, desc, depth = [-1], [rng.randint(0, 256, 32).astype(np.uint8)], [0]
    stack = [0]
    while stack:
        p = stack.pop()
        if depth[p] == L or (depth[p] >= 2 and rng.rand() < 0.2):
            continue
        prev = None
        for _ in range(8 if p == 0 else int(rng.choice([1, 1, 1, 2, 3, 5]))):
            d = flip(desc[p], rng.randint(20, 70), rng)
            if prev is not None and rng.rand() < 0.1:
                d = prev.copy()
            prev = d
            parent.append(p); desc.append(d); depth.append(depth[p] + 1)
            stack.append(len(parent) - 1)
    parent = np.array(parent, np.int32); desc = np.stack(desc); desc[0] = 0; depth = np.array(depth)
    nch = np.bincount(parent[1:], minlength=len(parent))
    leaf = np.nonzero((nch == 0) & (np.arange(len(parent)) > 0))[0]
    weight = np.zeros(len(parent)); weight[leaf] = _weights(len(leaf), rng)
    weight[leaf[rng.rand(len(leaf)) < 0.1]] = 0.0
    queries = np.concatenate([np.stack([flip(d, rng.randint(0, 30), rng) for d in desc[leaf[rng.randint(0, len(leaf), 300)]]]),
                              rng.randint(0, 256, (100, 32)).astype(np.uint8)])

    def proof(r):
        assert (nch[1:] == 1).sum() > 10 and len(set(depth[leaf])) >= 3, 'chains and leaves at several depths'
        word, w, node = r[L - 1]                                        # node at level 1
        d = depth[np.nonzero(parent == 0)[0]]
        assert (d == 1).all() and set(node.tolist()) <= set(np.nonzero(parent == 0)[0].tolist())
        shallow = depth[_leaf_of(r, leaf)] < L
        assert shallow.any() and (r[0][2][shallow] == 0).all(), 'a leaf above level L leaves the node at the root (nid_level not reached)'
    return dict(name='voc_unbalanced%d' % seed, k=5, L=L, parent=parent, desc=desc, weight=weight, queries=queries, proof=proof)


def _leaf_of(r, leaf):
    return leaf[r[0][0]]                                                # word ids number the leaves in node-id order


def orbvoc_shaped(seed=0, k=10, L=6):
    """ORBvoc.txt's shape: a full k-ary tree of depth L in depth-first node order (about 1.1 M nodes for k = 10, L = 6; ids above 2^20),
    built level by level.  A node at level l on the path (c1 .. cl) has id sum_j (1 + c_j * size_j), size_j = nodes in a level-j subtree."""
    rng = np.random.RandomState(seed)
    size = [(k ** (L - l + 1) - 1) // (k - 1) for l in range(L + 1)]
    n = size[0]
    parent = np.full(n, -1, np.int32); desc = np.zeros((n, 32), np.uint8)
    ids = np.zeros(1, np.int64); dprev = rng.randint(0, 256, (1, 32)).astype(np.uint8)
    for l in range(1, L + 1):
        c = np.tile(np.arange(k), len(ids))
        pid = np.repeat(ids, k)
        nid = pid + 1 + c * size[l]
        mask = rng.randint(0, 256, (len(nid), 32)).astype(np.uint8) & rng.randint(0, 256, (len(nid), 32)).astype(np.uint8) & \
            rng.randint(0, 256, (len(nid), 32)).astype(np.uint8)       # about 32 flipped bits
        d = np.repeat(dprev, k, axis=0) ^ mask
        parent[nid] = pid; desc[nid] = d
        ids, dprev = nid, d
    weight = np.zeros(n); weight[ids] = _weights(len(ids), rng)
    weight[ids[rng.rand(len(ids)) < 0.02]] = 0.0
    pick = ids[rng.randint(0, len(ids), 2000)]
    q = desc[pick] ^ (rng.randint(0, 256, (2000, 32)).astype(np.uint8) & rng.randint(0, 256, (2000, 32)).astype(np.uint8) &
                      rng.randint(0, 256, (2000, 32)).astype(np.uint8) & rng.randint(0, 256, (2000, 32)).astype(np.uint8))

    def proof(r):
        assert n > 2 ** 20 and r[4][2].max() > 2 ** 20 and r[0][0].max() > 0.9 * k ** L, 'node and word ids of the full size'
        assert (np.diff(np.nonzero(parent == 0)[0]) == size[1]).all(), 'depth-first ids'
    return dict(name='voc_orbvoc', k=k, L=L, parent=parent, desc=desc, weight=weight, queries=q, proof=proof)


def vocabularies(big=True):
    v = [_fanout_vocab(k, 100 + k) for k in (1, 2, 10, 31, 32, 33, 64, 65, 4096)]
    v += [_equidistant_vocab(k, 7 + k) for k in (33, 65, 4096)]
    v += [_unbalanced_vocab(s) for s in (1, 2)]
    if big:
        v.append(orbvoc_shaped())
    return v


def run_voc_oracle(v, levelsups=None):
    V = O.Vocabulary(v['k'], v['L'], v['parent'], v['desc'], v['weight'])
    return {ls: V.transform(v['queries'], ls) for ls in (range(v['L'] + 2) if levelsups is None else levelsups)}


# ---- matcher inputs ----------------------------------------------------------------------------------------------------------------
class _Pair:
    """Rows of the two sides plus the expected outcome: (a, b) = a matched b, (a, None) / (None, b) = left unmatched."""

    def __init__(self, mode, nnratio, seed, root=False):
        self.mode, self.nnratio, self.root = mode, nnratio, root
        self.rng = np.random.RandomState(seed)
        self.a, self.b, self.expect = [], [], []
        self._node = seed + 1

    def node(self):
        """Node ids in no particular order, small and above 2^20."""
        if self.root:
            return 0
        self._node = (self._node * 48271) % 2147483647
        return self._node

    def add_a(self, desc, node, weight=1.0, valid=1, angle=0.0, stereo=1, xy=(0.0, 0.0)):
        self.a.append(dict(desc=desc, node=node, weight=weight, valid=valid, angle=angle, stereo=stereo, xy=xy))
        return len(self.a) - 1

    def add_b(self, desc, node, weight=1.0, valid=1, angle=0.0, stereo=1, xy=(0.0, 0.0), octave=0):
        self.b.append(dict(desc=desc, node=node, weight=weight, valid=valid, angle=angle, stereo=stereo, xy=xy, octave=octave))
        return len(self.b) - 1

    def rand(self):
        return self.rng.randint(0, 256, 32).astype(np.uint8)

    def filler(self, K):
        while True:
            d = self.rand()
            if hamming(d, K) >= FAR:
                return d

    def accepts(self, best1, best2):
        """The verdict the reference's SearchByBoW gives (no ratio test in triangulation); the ratio product is float32."""
        if self.mode == 2:
            return best1 <= TH_LOW
        gate = best1 <= TH_LOW if self.mode == 0 else best1 < TH_LOW
        return gate and f32(best1) < f32(self.nnratio) * f32(best2)


def _bucket(P, size, place, nkf=1, angle=0.0, kf_kw=None, node=None):
    """One node: `nkf` key-frame features with the same descriptor K and a bucket of `size` frame features, the one at position p at
    distance place[p] from K, the others fillers.  Returns (kf rows, frame rows by position, K)."""
    K = P.rand()
    n = P.node() if node is None else node
    ks = [P.add_a(K, n, angle=angle, **(kf_kw or {})) for _ in range(nkf)]
    bs = [P.add_b(flip(K, place[p], P.rng) if p in place else P.filler(K), n, angle=angle) for p in range(size)]
    for p, d in place.items():
        assert hamming(P.b[bs[p]]['desc'], K) == d
    return ks, bs, K


def _resolve(P, ks, bs, place):
    """Expected outcome of a bucket whose key-frame features share one descriptor: each takes the best free candidate in turn (the first
    of equal distances in SearchByBoW, the last in SearchForTriangulation) if the gates accept it."""
    free = dict(place)
    for k in ks:
        if not free:
            P.expect.append((k, None)); continue
        d = sorted(free.values())
        best = d[0]
        cand = [p for p in sorted(free) if free[p] == best]
        p = cand[-1] if P.mode == 2 else cand[0]
        best2 = d[1] if len(d) > 1 else FAR
        if P.accepts(best, best2):
            P.expect.append((k, bs[p])); del free[p]
        else:
            P.expect.append((k, None))
    for p in free:
        P.expect.append((None, bs[p]))


def probe(P, size, place, nkf=1):
    ks, bs, _ = _bucket(P, size, place, nkf)
    _resolve(P, ks, bs, place)


def _finish(name, P, ori=0, only_stereo=0, F12=F_LINE, cw=CW, exhaustive=True, why=''):
    def side(rows, octave):
        d = dict(node=np.array([r['node'] for r in rows], np.int32), weight=np.array([r['weight'] for r in rows], np.float64),
                 valid=np.array([r['valid'] for r in rows], np.uint8), desc=np.stack([r['desc'] for r in rows]).astype(np.uint8),
                 angle=np.array([r['angle'] for r in rows], f32), stereo=np.array([r['stereo'] for r in rows], np.uint8),
                 xy=np.array([r['xy'] for r in rows], f32).reshape(-1, 2))
        if octave:
            d['octave'] = np.array([r['octave'] for r in rows], np.int32)
        return d
    ex, ey = epipole(cw)
    c = dict(name=name, mode=P.mode, params=dict(nnratio=float(P.nnratio), check_ori=int(ori), only_stereo=int(only_stereo)),
             a=side(P.a, False), b=side(P.b, True), F12=np.ascontiguousarray(F12, f32), cw=np.ascontiguousarray(cw, f32), ex=ex, ey=ey)
    expect = list(P.expect)
    mode = P.mode

    def proof(o):
        m = o['m']
        for a, b in expect:
            if a is not None and b is not None:
                got = m[b] if mode == 0 else m[a]
                assert got == (a if mode == 0 else b), (name, why, 'expected match', a, b, got)
            elif b is None:
                assert (a not in m) if mode == 0 else m[a] == -1, (name, why, 'key-frame feature must stay unmatched', a)
            else:
                assert m[b] == -1 if mode == 0 else (b not in m), (name, why, 'frame feature must stay unmatched', b)
        if exhaustive:
            nexp = sum(1 for a, b in expect if a is not None and b is not None)
            assert o['nm'] == nexp == int((m >= 0).sum()), (name, why, o['nm'], nexp)
    c['proof'] = proof
    c['expect'] = expect
    return c


MODES = {0: 'kf', 1: 'kfkf', 2: 'tri'}


def _gates(mode, ori, seed):
    P = _Pair(mode, 0.7, seed)
    for d in (49, 50, 51):
        probe(P, 2, {0: d})
        probe(P, 33, {32: d})
    return _finish('%s_gate_ori%d' % (MODES[mode], ori), P, ori, why='best distance 49 / 50 / 51 against TH_LOW')


def _ratio(mode, ori, r, seed):
    P = _Pair(mode, r, seed)
    for b2 in (40, 60, 65):
        fl = int(np.floor(f32(r) * f32(b2)))
        for b1 in (fl - 1, fl, fl + 1):
            probe(P, 3, {2: b1, 0: b2})
    return _finish('%s_ratio%02d_ori%d' % (MODES[mode], int(round(r * 100)), ori), P, ori, why='best1 == fl(nnratio * best2) and its neighbours')


def _claims(mode, ori, seed, root=False):
    """Claim cascades three deep (cross-lane positions), equal best distances with and without the twin claimed first, equal distances
    in four lanes claimed one after the other, invalid map points / weight-0 features that would otherwise win, nodes on one side only."""
    P = _Pair(mode, 0.75, seed, root=root)
    probe(P, 3, {2: 30, 0: 10, 1: 20}, nkf=3)                              # three deep inside one bucket
    probe(P, 65, {33: 10, 1: 20, 63: 30, 64: 44}, nkf=3)                   # the same across 32-lane groups
    probe(P, 65, {0: 15, 31: 15, 32: 15, 63: 15}, nkf=4)                   # equal distances: ratio rejects all in SearchByBoW; last wins in triangulation
    # twins un-rejected: the earlier key-frame feature is a copy of twin 1 and claims it, the later one then takes twin 2
    K = P.rand(); n = P.node()
    t1, t2 = flip(K, 20, P.rng), flip(K, 20, P.rng)
    a0 = P.add_a(t1, n); a1 = P.add_a(K, n)
    x1 = P.add_b(t1 ^ 0, n); x2 = P.add_b(t2, n); P.add_b(P.filler(K), n)
    assert hamming(K, t1) == hamming(K, t2) == 20 and hamming(t1, t2) >= 20
    P.expect += [(a0, x1), (a1, x2)]
    # invalid map point / weight-0 key-frame feature first in the bucket, a weight-0 (and in modes 1, 2 an invalid) frame feature closest
    K = P.rand(); n = P.node()
    inv = P.add_a(K, n, valid=0); w0 = P.add_a(K, n, weight=0.0); ok = P.add_a(K, n)
    bw0 = P.add_b(flip(K, 2, P.rng), n, weight=0.0)
    bad = [P.add_b(flip(K, 3, P.rng), n, valid=0)] if mode else []
    x = P.add_b(flip(K, 12, P.rng), n); P.add_b(P.filler(K), n)
    P.expect += [(inv, None), (w0, None), (ok, x), (None, bw0)] + [(None, b) for b in bad]
    if not root:
        # nodes on one side only: an exact copy in another node never matches
        K = P.rand()
        lone = P.add_a(K, P.node()); other = P.add_b(K.copy(), P.node())
        P.expect += [(lone, None), (None, other)]
    return _finish('%s_%s_ori%d' % (MODES[mode], 'root' if root else 'claims', ori), P, ori, why='claims, twins, invalid rows, one-sided nodes')


def _buckets(mode, ori, seed):
    P = _Pair(mode, 0.7, seed)
    for size, pos in ((1, 0), (31, 30), (31, 0), (32, 31), (33, 32), (33, 31), (64, 63), (64, 32), (65, 64), (65, 63), (65, 0), (1000, 999), (1000, 517)):
        pl = {pos: 30}
        if size > 1:
            pl[(pos + 32) % size if (pos + 32) % size != pos else (pos + 1) % size] = 45
        probe(P, size, pl)
    return _finish('%s_buckets_ori%d' % (MODES[mode], ori), P, ori, why='bucket sizes 1 .. 1000, best at lane 0 / 31 / 32 / 63 / last')


def _angles_for(target):
    """(kf angle, frame angle) whose rot (with the + 360 of a negative difference) gives rot * factor == target exactly, or None."""
    for a0, b0 in ((None, 0.0), (0.0, None)):
        guess = float(target) / float(FACTOR)
        if a0 is None:
            cand = [(a, f32(0)) for a in _neighbours(guess, 200)]
        else:
            cand = [(f32(0), b) for b in _neighbours(360.0 - guess, 200)]
        for a, b in cand:
            rot = f32(a - b)
            if rot < 0:
                rot = f32(rot + f32(360))
            if f32(rot * FACTOR) == f32(target) and 0 <= a < 360 and 0 <= b < 360:
                return a, b
    return None


def _bin(a, b):
    rot = f32(f32(a) - f32(b))
    if rot < 0:
        rot = f32(rot + f32(360))
    v = float(f32(rot * FACTOR))
    bn = int(np.floor(v + 0.5))
    return 0 if bn == 30 else bn


def _hist(mode, name, units, seed, why):
    """units: list of (kf angle, frame angle, kept?) -- one sure match per unit in its own node; the rotation histogram keeps or drops it."""
    P = _Pair(mode, 0.75, seed)
    for a, b, keep in units:
        K = P.rand(); n = P.node()
        ka = P.add_a(K, n, angle=a, stereo=1); fb = P.add_b(flip(K, 8, P.rng), n, angle=b); P.add_b(P.filler(K), n, angle=b)
        P.expect.append((ka, fb) if keep else (ka, None))
    return _finish('%s_hist_%s' % (MODES[mode], name), P, ori=1, why=why)


def _counts_units(counts, keep_bins):
    u = []
    for bn, c in counts.items():
        for i in range(c):
            u.append((f32(bn * 12 + 0.25 * i) % f32(360), f32(0.25 * i), bn in keep_bins))
    return u


def _hist_cases(mode):
    out = []
    # rot * factor exactly at k + 0.5 rounds half away from zero (2.5 -> 3, not 2); one float below goes to the lower bin
    units = _counts_units({3: 4, 5: 4, 9: 4}, {3, 5, 9})
    for t, keep in ((2.5, True), (4.5, True), (8.5, True)):
        a, b = _angles_for(t)
        below = np.nextafter(a, f32(-np.inf)) if b == 0 else a
        b2 = b if b == 0 else np.nextafter(b, f32(np.inf))
        assert _bin(a, b) == int(t + 0.5) and _bin(below, b2) == int(t - 0.5)
        units += [(a, b, keep), (below, b2, False)]
    out.append(_hist(mode, 'half', units, 1, 'rot * factor at k + 0.5'))
    # rot = -tiny: + 360 gives 360.0f, bin 30, wrapped to bin 0; rot just under 360 and at 29.5 * 12 also wrap
    units = _counts_units({0: 4, 7: 4, 13: 4}, {0, 7, 13})
    a, b = _angles_for(29.5)
    units += [(f32(0), f32(1e-5), True), (f32(359.99), f32(0), True), (a, b, True)]
    below = (np.nextafter(a, f32(-np.inf)), b) if b == 0 else (a, np.nextafter(b, f32(np.inf)))
    assert _bin(f32(0), f32(1e-5)) == 0 and f32(f32(f32(0) - f32(1e-5)) + f32(360)) == f32(360) and _bin(*below) == 29
    units.append((below[0], below[1], False))
    out.append(_hist(mode, 'wrap', units, 2, 'negative rot wraps through bin 30 to bin 0'))
    out.append(_hist(mode, 'tie4', _counts_units({4: 3, 11: 3, 20: 3, 25: 3}, {4, 11, 20}), 3, 'four bins tied: the first three win'))
    out.append(_hist(mode, 'tie_top', _counts_units({2: 5, 6: 5, 8: 2, 9: 2}, {2, 6, 8}), 4, 'tied maxima'))
    for m1, m2, m3 in ((10, 1, 1), (11, 1, 1), (10, 5, 1), (11, 5, 1), (20, 2, 2), (21, 2, 2), (19, 2, 1)):
        lim = f32(0.1) * f32(m1)
        keep = {1} | ({17} if f32(m2) >= lim else set()) | ({23} if f32(m2) >= lim and f32(m3) >= lim else set())
        out.append(_hist(mode, 'tenth_%d_%d_%d' % (m1, m2, m3), _counts_units({1: m1, 17: m2, 23: m3}, keep), 5 + m1 + m2, 'max2 / max3 against 0.1f * max1'))
    return out


# ---- triangulation geometry -------------------------------------------------------------------------------------------------------
def _epipole_point(target, cw=CW):
    """A point (x2, y2) whose squared distance to the epipole, as the reference computes it in float, is exactly `target`."""
    ex, ey = epipole(cw)
    for x2 in _neighbours(f32(ex - np.sqrt(float(target))), 300):
        dx = f32(ex - x2); dx2 = f32(dx * dx)
        if dx2 > target:
            continue
        gap = float(target) - float(dx2)
        ys = _neighbours(f32(ey - np.sqrt(gap)), 300)
        dy = (ey - ys).astype(f32)
        s = (dx2 + (dy * dy).astype(f32)).astype(f32)
        hit = np.nonzero(s == f32(target))[0]
        if len(hit):
            return f32(x2), ys[hit[0]]
    raise AssertionError(('no point at', target))


def _tri_epipole(ori, seed):
    """The epipole gate (both sides without stereo) at equality and one float32 ulp inside, octaves 0, 1 and 7; the gate skipped because
    either side is stereo."""
    P = _Pair(2, 0.6, seed)
    for oc in (0, 1, 7):
        lim = f32(f32(100) * SF[oc])
        for target, keep in ((lim, True), (np.nextafter(lim, f32(0)), False)):
            x2, y2 = _epipole_point(target)
            for st1, st2 in ((0, 0), (1, 0), (0, 1)):
                K = P.rand(); n = P.node()
                a = P.add_a(K, n, stereo=st1, xy=(f32(50), y2))
                b = P.add_b(flip(K, 9, P.rng), n, stereo=st2, xy=(x2, y2), octave=oc)
                P.expect.append((a, b) if (keep or st1 or st2) else (a, None))
    return _finish('tri_epipole_ori%d' % ori, P, ori, why='epipole distance at 100 * scale[octave]')


def _tri_dsqr(ori, seed):
    """dsqr = num^2 / den next to 3.84 * sigma2[octave] (compared in double) for all 8 octaves: y1 = 0 and the line y2 = y1 make dsqr = y2^2."""
    P = _Pair(2, 0.6, seed)
    ex, _ = epipole()
    for oc in range(8):
        T = 3.84 * float(SIGMA2[oc])
        ys = _neighbours(f32(np.sqrt(T)), 40)
        ds = (ys * ys).astype(f32)
        below = ys[np.nonzero(ds.astype(np.float64) < T)[0][-1]]
        above = ys[np.nonzero(ds.astype(np.float64) >= T)[0][0]]
        for y2, keep in ((below, True), (above, False)):
            for st in (0, 1):
                K = P.rand(); n = P.node()
                a = P.add_a(K, n, stereo=0, xy=(f32(100), f32(0)))
                b = P.add_b(flip(K, 7, P.rng), n, stereo=st, xy=(f32(ex - 200), y2), octave=oc)
                P.expect.append((a, b) if keep else (a, None))
    return _finish('tri_dsqr_ori%d' % ori, P, ori, why='dsqr one float either side of 3.84 * sigma2')


def _tri_den0(ori, seed):
    """F12 = [[1,0,0],[0,1,0],[-x1,-y1,0]]: the epipolar line of the key-frame point (x1, y1) is degenerate (den == 0); a point
    elsewhere gets the line 3 x - 2 y = 0 through the origin."""
    P = _Pair(2, 0.6, seed)
    x1, y1 = f32(211.75), f32(97.5)
    K = P.rand(); n = P.node()
    a0 = P.add_a(K, n, xy=(x1, y1)); b0 = P.add_b(K.copy(), n, xy=(f32(0), f32(0)))
    K = P.rand(); n = P.node()
    a1 = P.add_a(K, n, xy=(x1 + 3, y1 - 2)); b1 = P.add_b(flip(K, 5, P.rng), n, xy=(f32(0), f32(0)))
    P.expect += [(a0, None), (None, b0), (a1, b1)]
    F = np.array([[1, 0, 0], [0, 1, 0], [-x1, -y1, 0]], f32)
    return _finish('tri_den0_ori%d' % ori, P, ori, F12=F, why='den == 0')


def _tri_only_stereo(ori, only, seed):
    P = _Pair(2, 0.6, seed)
    ex, ey = epipole()
    far = (f32(ex - 150), f32(ey))
    K = P.rand(); n = P.node()
    as_ = P.add_a(K, n, stereo=1, xy=far)
    xm = P.add_b(flip(K, 5, P.rng), n, stereo=0, xy=far); xs = P.add_b(flip(K, 20, P.rng), n, stereo=1, xy=far)
    K = P.rand(); n = P.node()
    am = P.add_a(K, n, stereo=0, xy=far); xs2 = P.add_b(K.copy(), n, stereo=1, xy=far); xm2 = P.add_b(flip(K, 30, P.rng), n, stereo=0, xy=far)
    if only:
        P.expect += [(as_, xs), (None, xm), (am, None), (None, xs2), (None, xm2)]
    else:
        P.expect += [(as_, xm), (None, xs), (am, xs2), (None, xm2)]
    return _finish('tri_stereo%d_ori%d' % (only, ori), P, ori, only_stereo=only, why='only_stereo with mixed flags')


def full_bucket(mode, npairs, extra=0, seed=0, nnratio=0.75):
    """Everything in the root bucket: npairs distinct descriptors, each held by two key-frame features, each with candidates at 10 and
    20 bits in shuffled positions (the first copy claims the 10, the second takes the 20), plus `extra` unmatched rows on both sides."""
    rng = np.random.RandomState(seed)
    K = rng.randint(0, 256, (npairs, 32)).astype(np.uint8)
    a_desc = np.repeat(K, 2, axis=0)
    c1 = np.stack([flip(k, 10, rng) for k in K]); c2 = np.stack([flip(k, 20, rng) for k in K])
    order = rng.permutation(2 * npairs)
    b_desc = np.concatenate([c1, c2])[order]
    pos = np.argsort(order)                                             # pos[i] = row of candidate i (c1: i < npairs, c2: i >= npairs)
    P = _Pair(mode, nnratio, seed + 1000)
    for d in a_desc:
        P.add_a(d, 0)
    for d in b_desc:
        P.add_b(d, 0)
    for i in range(extra):
        P.add_a(P.filler(K[0]), 0); P.add_b(P.filler(K[0]), 0)
    P.expect += [(2 * i, int(pos[i])) for i in range(npairs)] + [(2 * i + 1, int(pos[npairs + i])) for i in range(npairs)]
    return _finish('%s_full%d' % (MODES[mode], len(P.a)), P, 0, why='full root bucket')


def tiny(mode, d):
    P = _Pair(mode, 0.75, 50 + d)
    probe(P, 1, {0: d})
    return _finish('%s_tiny%d' % (MODES[mode], d), P, 0, why='one feature per side')


def _build():
    cases = []
    for mode in (0, 1, 2):
        for ori in (0, 1):
            cases.append(_gates(mode, ori, 10 + mode))
            if mode != 2:
                cases += [_ratio(mode, ori, r, 20 + mode) for r in (0.7, 0.75, 0.8)]
            cases.append(_claims(mode, ori, 30 + mode))
            cases.append(_claims(mode, ori, 40 + mode, root=True))
            cases.append(_buckets(mode, ori, 50 + mode))
        cases += _hist_cases(mode)
    for ori in (0, 1):
        cases += [_tri_epipole(ori, 60), _tri_dsqr(ori, 61), _tri_den0(ori, 62), _tri_only_stereo(ori, 0, 63), _tri_only_stereo(ori, 1, 64)]
    return {c['name']: c for c in cases}


CASES = _build()


def names(mode=None):
    return [n for n, c in CASES.items() if mode is None or c['mode'] == mode]


def run_arrays(mode, params, a, b, c):
    """The oracle on explicit side arrays (the case's, or a padded frame's rows up to its count)."""
    r, ori = params['nnratio'], bool(params['check_ori'])
    if mode == 0:
        nm, m = O.search_by_bow(a['node'], a['weight'], a['valid'], a['desc'], a['angle'], b['node'], b['weight'], b['desc'], b['angle'], r, ori)
    elif mode == 1:
        nm, m = O.search_by_bow_kfkf(a['node'], a['weight'], a['valid'], a['desc'], a['angle'], b['node'], b['weight'], b['valid'], b['desc'], b['angle'], r, ori)
    else:
        k1 = dict(a, free=a['valid']); k2 = dict(b, free=b['valid'])
        nm, m = O.search_for_triangulation(k1, k2, c['F12'], float(c['ex']), float(c['ey']), SIGMA2, SF, bool(params['only_stereo']), ori)
    return dict(nm=int(nm), m=m)


def run_oracle(c):
    return run_arrays(c['mode'], c['params'], c['a'], c['b'], c)
