"""Constructed inputs for findFundamentalMat(FM_RANSAC) (numpy only, no device): point sets built so that one hard path of the restatement in
sg-slam_b200/csrc/fundamental.cu MUST be taken.  Every case carries a proof -- an assertion on a pure-Python replay of OpenCV's estimator
loop (the MWC generator, getSubset's redraws, the accept / update-niters rules, LMedS's median) that only holds if the path was taken (for
example "the first draw needs 1000 < a <= 10000 attempts" or "the loop stops after iteration 9") -- so that an edit to a builder cannot
quietly turn a case into an easy one.  The replay takes the 7-point models from the oracle's run7point and does everything else itself;
tests/test_fundamental_cases.py checks that it returns what the oracle returns.

A case is a dict: name, group ('pinned': cv2 returns a matrix or nothing; 'raises': cv2 4.13 throws, see DESIGN.md quirk Q15), m1, m2
(float32 [n, 2]), params (thresh, confidence, max_iters as passed to the entry points), paths (labels) and proof(trace).

The collinearity-driven cases use integer coordinates, so that getSubset's FLT_EPSILON test is exact in every implementation.  Their
structure: in image 1 all points but one (p*) lie on the line y = 100; in image 2 p* sits at a centre c, `nh` points lie on the horizontal
line through c and the others on distinct rays from c.  A sample passes only when p* is drawn last and at most one of the six others is
on c's horizontal line, so a draw needs thousands of attempts; which attempt passes depends on the order of the points (a seeded
permutation), because the generator's index stream depends on n alone."""
import math

import numpy as np

import oracle as O

f32 = np.float32
M64 = (1 << 64) - 1
FLT_EPSILON = float(np.finfo(np.float32).eps)
DBL_MIN = float(np.finfo(np.float64).tiny)
RANSAC_ATTEMPTS, LMEDS_ATTEMPTS = 10000, 1000
DEFAULT = dict(thresh=1.0, confidence=0.99, max_iters=1000)


class Rng:
    """cv::RNG: multiply-with-carry, state (uint64)-1; uniform(0, n) = next() % n."""
    def __init__(self, state=M64):
        self.state = state

    def next(self):
        self.state = ((self.state & 0xffffffff) * 4164903690 + (self.state >> 32)) & M64
        return self.state & 0xffffffff


def collinear(p):
    """fundam.cpp haveCollinearPoints on the last of 7 points, for a stack p [T, 7, 2] of float32 samples: bool [T].  The differences are
    float32 subtractions (Point2f), the test is in double."""
    d = (p[:, :6, :] - p[:, 6:7, :]).astype(np.float64)
    out = np.zeros(len(p), bool)
    for j in range(6):
        for k in range(j):
            dx1, dy1, dx2, dy2 = d[:, j, 0], d[:, j, 1], d[:, k, 0], d[:, k, 1]
            out |= np.abs(dx2 * dy1 - dy2 * dx1) <= FLT_EPSILON * (np.abs(dx1) + np.abs(dy1) + np.abs(dx2) + np.abs(dy2))
    return out


class Sampler:
    """getSubset: one continuous stream of 7-index attempts (it depends on n alone); draw(cap) returns (indices, attempts) or (None, cap)."""
    CHUNK = 4096

    def __init__(self, m1, m2):
        self.m1, self.m2, self.n = np.asarray(m1, f32), np.asarray(m2, f32), len(m1)
        self.rng, self.idx, self.ok, self.pos = Rng(), np.zeros((0, 7), np.int64), np.zeros(0, bool), 0

    def _grow(self):
        r, n = self.rng, self.n
        out = np.zeros((self.CHUNK, 7), np.int64)
        for t in range(self.CHUNK):
            row = []
            for _ in range(7):
                v = r.next() % n
                while v in row:
                    v = r.next() % n
                row.append(v)
            out[t] = row
        ok = ~collinear(self.m1[out]) & ~collinear(self.m2[out])
        self.idx, self.ok = np.concatenate([self.idx, out]), np.concatenate([self.ok, ok])

    def draw(self, cap):
        while True:
            hit = np.flatnonzero(self.ok[self.pos:self.pos + cap])
            if len(hit) or len(self.ok) >= self.pos + cap:
                break
            self._grow()
        if not len(hit):
            self.pos += cap
            return None, cap
        a = int(hit[0]) + 1
        idx = self.idx[self.pos + a - 1]
        self.pos += a
        return idx, a


def errors(m1, m2, F):
    """FMEstimatorCallback::computeError in double, rounded to float, in OpenCV's operation order."""
    x1, y1 = m1[:, 0].astype(np.float64), m1[:, 1].astype(np.float64)
    x2, y2 = m2[:, 0].astype(np.float64), m2[:, 1].astype(np.float64)
    F = np.asarray(F, np.float64).ravel()
    with np.errstate(all='ignore'):          # a degenerate model gives 1 / 0
        a = F[0] * x1 + F[1] * y1 + F[2]; b = F[3] * x1 + F[4] * y1 + F[5]; c = F[6] * x1 + F[7] * y1 + F[8]
        s2 = 1. / (a * a + b * b); d2 = x2 * a + y2 * b + c
        a = F[0] * x2 + F[3] * y2 + F[6]; b = F[1] * x2 + F[4] * y2 + F[7]; c = F[2] * x2 + F[5] * y2 + F[8]
        s1 = 1. / (a * a + b * b); d1 = x1 * a + y1 * b + c
        return np.maximum(d1 * d1 * s1, d2 * d2 * s2).astype(f32)


def update_num_iters(p, ep, max_iters):
    """ptsetreg.cpp RANSACUpdateNumIters, modelPoints = 7.  Returns (niters, num / denom or None)."""
    p = min(max(p, 0.), 1.); ep = min(max(ep, 0.), 1.)
    num, denom = max(1. - p, DBL_MIN), 1. - math.pow(1. - ep, 7)
    if denom < DBL_MIN:
        return 0, None
    num, denom = math.log(num), math.log(denom)
    if denom >= 0 or -num >= max_iters * (-denom):
        return max_iters, None
    return int(np.rint(num / denom)), num / denom


def normalise(thresh, confidence):
    """fundam.cpp: thresh <= 0 -> 3, confidence outside (DBL_EPSILON, 1 - DBL_EPSILON) -> 0.99 (both branches)."""
    eps = float(np.finfo(np.float64).eps)
    return (3.0 if thresh <= 0 else thresh), (0.99 if confidence < eps or confidence > 1 - eps else confidence)


def replay(m1, m2, thresh=1.0, confidence=0.99, max_iters=1000):
    """cv::findFundamentalMat(m1, m2, FM_RANSAC, thresh, confidence, max_iters) step by step.  Returns a trace dict:
    branch ('empty', 'seven', 'lmeds', 'ransac'), F (3x3 or None), mask, inliers, iterations (samples evaluated), niters (final),
    draws (attempts of every draw, the failed one last as None), failed (index of the failed draw or None), nmodels (per iteration),
    scores (per iteration: inlier counts or medians of its models), accepts ((iteration, root, score) of every replacement of the best
    model), ratios (num / denom of every niters update that was not capped)."""
    m1, m2 = np.asarray(m1, f32).reshape(-1, 2), np.asarray(m2, f32).reshape(-1, 2)
    n = len(m1)
    thresh, confidence = normalise(thresh, confidence)
    tr = dict(branch='empty', F=None, mask=np.zeros(n, np.uint8), inliers=0, iterations=0, niters=0, draws=[], failed=None, nmodels=[],
              scores=[], accepts=[], ratios=[])
    if n < 7:
        return tr
    if n == 7:
        models = O.run7point(m1, m2)
        tr.update(branch='seven', nmodels=[len(models)], iterations=1, niters=1)
        if models:
            tr.update(F=models[0], mask=np.ones(n, np.uint8), inliers=7)
        return tr
    lmeds = n < 15
    S = Sampler(m1, m2)
    if lmeds:
        niters = max(update_num_iters(confidence, 0.45, max_iters)[0], 3)
        tr.update(branch='lmeds', niters=niters)
        best, best_med = None, math.inf
        it = 0
        while it < niters:
            idx, a = S.draw(LMEDS_ATTEMPTS)
            if idx is None:
                tr['draws'].append(None); tr['failed'] = it
                break
            tr['draws'].append(a)
            models = O.run7point(m1[idx], m2[idx])
            tr['nmodels'].append(len(models)); sc = []
            for k, F in enumerate(models):
                med = float(np.sort(errors(m1, m2, F), kind='stable')[n // 2])
                sc.append(med)
                if med < best_med:
                    best_med, best = med, F
                    tr['accepts'].append((it, k, med))
            tr['scores'].append(sc)
            it += 1
        tr['iterations'] = it
        if best is None or (tr['failed'] == 0):
            return tr
        sigma = max(2.5 * 1.4826 * (1 + 5. / (n - 7)) * math.sqrt(best_med), 0.001)
        mask = (errors(m1, m2, best) <= f32(sigma * sigma)).astype(np.uint8)
        tr['inliers'] = int(mask.sum())
        if tr['inliers'] >= 7:
            tr.update(F=best, mask=mask)
        return tr
    tr['branch'] = 'ransac'
    t = f32(thresh * thresh)
    niters, maxgood, best, best_mask = max(max_iters, 1), 0, None, None
    it = 0
    while it < niters:
        idx, a = S.draw(RANSAC_ATTEMPTS)
        if idx is None:
            tr['draws'].append(None); tr['failed'] = it
            break
        tr['draws'].append(a)
        models = O.run7point(m1[idx], m2[idx])
        tr['nmodels'].append(len(models)); sc = []
        for k, F in enumerate(models):
            mask = (errors(m1, m2, F) <= t).astype(np.uint8)
            good = int(mask.sum())
            sc.append(good)
            if good > max(maxgood, 6):
                best, best_mask, maxgood = F, mask, good
                niters, ratio = update_num_iters(confidence, (n - good) / n, niters)
                tr['accepts'].append((it, k, good))
                if ratio is not None:
                    tr['ratios'].append(ratio)
        tr['scores'].append(sc)
        it += 1
    tr.update(iterations=it, niters=niters, inliers=maxgood)
    if tr['failed'] == 0 or maxgood <= 0:
        tr['inliers'] = 0
        return tr
    tr.update(F=best, mask=best_mask)
    return tr


# ---- scene builders

def two_view(seed, n, noise, outlier_frac, integer=False):
    """Seeded two-view correspondences (the generator of tests/golden/make_golden_fm.py): n points at depth 2..6 seen by two cameras 0.05
    apart, Gaussian noise in pixels, a leading fraction of outliers displaced by up to 30 px, then shuffled.  integer=True rounds the
    coordinates, so that collinearity tests are exact."""
    rs = np.random.RandomState(seed)
    X = np.c_[rs.uniform(-2, 2, n), rs.uniform(-1.5, 1.5, n), rs.uniform(2, 6, n)]
    K = np.array([[535.4, 0, 320.1], [0, 539.2, 247.6], [0, 0, 1]])
    ang = 0.02
    R = np.array([[math.cos(ang), 0, math.sin(ang)], [0, 1, 0], [-math.sin(ang), 0, math.cos(ang)]])
    p1 = (K @ X.T).T; p1 = p1[:, :2] / p1[:, 2:]
    X2 = (R @ X.T).T + np.array([0.05, 0.01, 0.02]); p2 = (K @ X2.T).T; p2 = p2[:, :2] / p2[:, 2:]
    p1 = p1 + rs.normal(0, noise, p1.shape); p2 = p2 + rs.normal(0, noise, p2.shape)
    nout = int(n * outlier_frac)
    p2[:nout] += rs.uniform(-30, 30, (nout, 2))
    perm = rs.permutation(n)
    p1, p2 = p1[perm], p2[perm]
    if integer:
        p1, p2 = np.rint(p1), np.rint(p2)
    return p1.astype(f32), p2.astype(f32)


def line_and_rays(n, nh, seed):
    """The collinearity structure of the module docstring, in the order of a seeded permutation."""
    m1 = np.zeros((n, 2), f32); m2 = np.zeros((n, 2), f32)
    m1[:n - 1, 0] = np.arange(n - 1) * 7 + 50; m1[:n - 1, 1] = 100; m1[n - 1] = (300, 260)
    m2[n - 1] = (320, 240)
    rays = [(1, 1), (1, 2), (2, 1), (1, -1), (0, 1), (2, -1), (1, -2), (3, 1), (1, 3), (3, -1)]
    for j in range(nh):
        m2[j] = (320 + (j // 2 + 1) * 9 * (1 if j % 2 else -1), 240)
    for j in range(n - 1 - nh):
        m2[nh + j] = (320 + rays[j][0] * (5 + j), 240 + rays[j][1] * (5 + j))
    p = np.random.RandomState(seed).permutation(n)
    return m1[p], m2[p]


def first_draw(m1, m2, cap=RANSAC_ATTEMPTS):
    """Attempts the first getSubset call needs (None: more than cap)."""
    idx, a = Sampler(m1, m2).draw(cap)
    return None if idx is None else a


def _collinear_first_attempt(m1, m2):
    """Moves, in image 1, the last point of the generator's first 7-index attempt onto the line through the attempt's first two points
    (integer coordinates: exactly collinear), so that the first draw rejects one sample."""
    t = Sampler(m1, m2); t._grow()
    i0, i1, i6 = t.idx[0][0], t.idx[0][1], t.idx[0][6]
    m1 = m1.copy(); m1[i6] = 2 * m1[i1] - m1[i0]
    return m1, m2


def _case(name, group, m1, m2, paths, proof, **params):
    p = dict(DEFAULT); p.update(params)
    return dict(name=name, group=group, m1=np.asarray(m1, f32), m2=np.asarray(m2, f32), params=p, paths=paths, proof=proof)


def _stop_at(k, rounds_up=False):
    """The loop ends because niters fell to k (no failed draw), at iteration k."""
    def proof(c, tr):
        assert tr['failed'] is None and tr['iterations'] == tr['niters'] == k and tr['F'] is not None
        if rounds_up:      # the last update rounded num / denom up: truncation would stop one iteration earlier
            assert tr['ratios'] and tr['ratios'][-1] % 1 >= 0.5 and int(tr['ratios'][-1]) == k - 1
    return proof


def _lmeds_cap(c, tr):
    assert 1000 < first_draw(c['m1'], c['m2']) <= 10000 and tr['failed'] == 0 and tr['F'] is None


def _lmeds_iters(k):
    def proof(c, tr):
        assert tr['branch'] == 'lmeds' and tr['failed'] is None and tr['iterations'] == tr['niters'] == k
        assert replay(c['m1'], c['m2'])['iterations'] == 300 != k          # the default parameters run 300 samples
    return proof


def _tie(c, tr):
    wi, _, wg = tr['accepts'][-1]
    assert any(g == wg for j, sc in enumerate(tr['scores']) if j > wi for g in sc)        # a later model as good as the winner is not taken


def _later_root(c, tr):
    wi, wk, _ = tr['accepts'][-1]
    assert tr['nmodels'][wi] == 3 and wk >= 1


def _same_as(**ref):
    """Normalised parameters: the replay equals the one at the normalised values."""
    def proof(c, tr):
        p = dict(c['params']); p.update(ref)
        r = replay(c['m1'], c['m2'], **p)
        assert tr['F'] is not None and np.array_equal(tr['F'], r['F']) and np.array_equal(tr['mask'], r['mask']) and tr['iterations'] == r['iterations']
    return proof


def _holds(pred):
    def proof(c, tr):
        assert pred(c, tr)
    return proof


def _and(*proofs):
    def proof(c, tr):
        for p in proofs:
            p(c, tr)
    return proof


def _scene(seed, n, noise, of):
    return two_view(seed, n, noise, of)


def cases():
    out = []
    add = out.append
    # ---- LMedS (8..14 pairs): getSubset's default of 1000 attempts; niters from max_iters
    for n, nh, seed in [(10, 4, 84), (11, 5, 0), (12, 6, 2), (14, 8, 0)]:
        add(_case(f'lmeds_cap_n{n}', 'pinned', *line_and_rays(n, nh, seed), ['lmeds', 'draw_over_1000', 'empty'], _lmeds_cap))
    m1, m2 = _collinear_first_attempt(*two_view(3, 14, 0.5, 0.0, integer=True))
    add(_case('lmeds_redraw_control', 'pinned', m1, m2, ['lmeds', 'redraw'],
              _holds(lambda c, tr: 1 < tr['draws'][0] <= 1000 and tr['failed'] is None and tr['F'] is not None)))
    for mi, k in [(1, 3), (20, 20), (299, 299)]:
        add(_case(f'lmeds_max_iters_{mi}', 'pinned', *two_view(0, 14, 0.5, 0.2), ['lmeds', 'max_iters'], _lmeds_iters(k), max_iters=mi))
    add(_case('lmeds_max_iters_5000', 'pinned', *two_view(0, 14, 0.5, 0.2), ['lmeds', 'max_iters'],
              _holds(lambda c, tr: tr['iterations'] == tr['niters'] == 300), max_iters=5000))
    add(_case('lmeds_confidence_0p9', 'pinned', *two_view(1, 14, 0.5, 0.2), ['lmeds', 'confidence'], _lmeds_iters(150), confidence=0.9))
    # ---- RANSAC (15 pairs and more): 10000 attempts
    for n, nh, seed in [(15, 9, 1), (16, 10, 0)]:
        add(_case(f'ransac_first_draw_fails_n{n}', 'pinned', *line_and_rays(n, nh, seed), ['ransac', 'draw_over_10000', 'empty'],
                  _holds(lambda c, tr: first_draw(c['m1'], c['m2']) is None and tr['failed'] == 0 and tr['F'] is None)))
    for name, key, k, up in [('ransac_niters_zero', (66, 30, 0.1, 0.0), 1, False), ('ransac_stop_8', (30, 18, 0.1, 0.2), 8, True),
                             ('ransac_stop_9', (110, 40, 0.1, 0.1), 9, False), ('ransac_stop_9_rounded_up', (329, 25, 0.3, 0.0), 9, True),
                             ('ransac_stop_20', (28, 15, 0.6, 0.1), 20, True), ('ransac_stop_41', (33, 40, 0.1, 0.3), 41, False)]:
        proof = _stop_at(k, up) if k > 1 else _holds(lambda c, tr: tr['iterations'] == 1 and tr['niters'] == 0 and tr['inliers'] == len(c['m1']))
        add(_case(name, 'pinned', *_scene(*key), ['ransac', 'adaptive_stop'], proof))
    add(_case('ransac_tie', 'pinned', *_scene(5, 18, 0.1, 0.1), ['ransac', 'tie'], _tie))
    add(_case('ransac_later_root_wins', 'pinned', *_scene(0, 30, 0.3, 0.0), ['ransac', 'three_roots'], _later_root))
    # ---- parameters: limits and OpenCV's normalisation (thresh <= 0 -> 3, confidence outside (0, 1) -> 0.99)
    for mi in (1, 2):
        add(_case(f'ransac_max_iters_{mi}', 'pinned', *_scene(33, 40, 0.1, 0.3), ['ransac', 'max_iters'],
                  _holds(lambda c, tr: tr['iterations'] == c['params']['max_iters'] and tr['F'] is not None), max_iters=mi))
    heavy = two_view(0, 40, 0.3, 0.7)
    add(_case('ransac_max_iters_1000', 'pinned', *heavy, ['ransac', 'max_iters'], _and(
        _holds(lambda c, tr: tr['iterations'] == 1000 and tr['failed'] is None),
        _holds(lambda c, tr: replay(c['m1'], c['m2'], max_iters=5000)['iterations'] > 1000))))
    add(_case('ransac_max_iters_5000', 'pinned', *heavy, ['ransac', 'max_iters'],
              _holds(lambda c, tr: 1000 < tr['iterations'] == tr['niters'] < 5000), max_iters=5000))
    add(_case('ransac_max_iters_50', 'pinned', *heavy, ['ransac', 'max_iters'], _holds(lambda c, tr: tr['iterations'] == 50), max_iters=50))
    noisy = two_view(0, 40, 1.2, 0.1)
    for name, th in [('ransac_thresh_0', 0.0), ('ransac_thresh_negative', -1.0)]:
        add(_case(name, 'pinned', *noisy, ['ransac', 'thresh_normalised'], _and(
            _same_as(thresh=3.0), _holds(lambda c, tr: tr['inliers'] != replay(c['m1'], c['m2'], thresh=1.0)['inliers'])), thresh=th))
    mid = two_view(0, 40, 0.3, 0.3)
    add(_case('ransac_confidence_0', 'pinned', *mid, ['ransac', 'confidence_normalised'],        # unnormalised: niters 0 after the first model
              _and(_same_as(confidence=0.99), _holds(lambda c, tr: tr['iterations'] > 1 and len(tr['accepts']) >= 1)), confidence=0.0))
    add(_case('ransac_confidence_1', 'pinned', *mid, ['ransac', 'confidence_normalised'],        # unnormalised: niters stays at max_iters
              _and(_same_as(confidence=0.99), _holds(lambda c, tr: tr['iterations'] < 1000 and tr['failed'] is None)), confidence=1.0))
    add(_case('ransac_thresh_0p5_confidence_0p9', 'pinned', *two_view(1, 40, 0.3, 0.3), ['ransac', 'parameters'],
              _holds(lambda c, tr: tr['F'] is not None), thresh=0.5, confidence=0.9))
    add(_case('ransac_thresh_3_confidence_0p999', 'pinned', *two_view(2, 100, 0.8, 0.3), ['ransac', 'parameters'],
              _holds(lambda c, tr: tr['F'] is not None), thresh=3.0, confidence=0.999))
    # ---- exactly 7 pairs: the 7-point solver itself, without getSubset's collinearity test
    add(_case('seven_three_roots', 'pinned', *two_view(0, 7, 0.3, 0.0), ['seven'], _holds(lambda c, tr: tr['nmodels'] == [3])))
    m1, m2 = two_view(1, 7, 0.3, 0.0, integer=True)
    m1[6] = 2 * m1[1] - m1[0]
    add(_case('seven_collinear', 'pinned', m1, m2, ['seven', 'collinear'],
              _holds(lambda c, tr: collinear(c['m1'][None])[0] and tr['F'] is not None)))
    # ---- cv2 4.13 raises on these (quirk Q15): a drawn sample has six points on one line in image 1
    add(_case('lmeds_later_draw_fails_n14', 'raises', *line_and_rays(14, 8, 24), ['lmeds', 'later_draw_fails'],
              _holds(lambda c, tr: tr['draws'][0] <= 1000 and tr['failed'] is not None and tr['failed'] > 0)))
    add(_case('ransac_draw_over_1000_n15', 'raises', *line_and_rays(15, 9, 0), ['ransac', 'draw_over_1000'],
              _holds(lambda c, tr: 1000 < tr['draws'][0] <= 10000 and tr['iterations'] >= 1)))
    for n, nh, seed in [(15, 9, 3), (16, 10, 2)]:
        add(_case(f'ransac_later_draw_fails_n{n}', 'raises', *line_and_rays(n, nh, seed), ['ransac', 'later_draw_fails'],
                  _holds(lambda c, tr: tr['failed'] is not None and 0 < tr['failed'] == tr['iterations'] < tr['niters'])))
    return out


def check_proofs(case):
    """Replays the case and asserts its proof; returns the trace."""
    tr = replay(case['m1'], case['m2'], **case['params'])
    case['proof'](case, tr)
    return tr
