"""The detector's tail -- softmax_rows_kernel, detout_class_kernel and detout_merge_kernel (detector.cu) -- each on the exact input the GPU read.
Diagnostic mode keeps the pre-softmax confidences (mbox_conf), the Softmax output (mbox_conf_softmax), the location offsets (mbox_loc) and the prior
table (mbox_priorbox), so the references below are computed from the device's own blobs and nothing is carried in from earlier layers.  The graphs
are head-only (tests/detector_model.py: write_head_model, head_scene), most with zero head weights and planted biases, so that scores tie exactly and
every box is its prior box decoded with zero offsets.

Softmax, u = 2^-24, per row x (float32), d_c = x_c - max(x), R = float64 softmax of x:
  x_c - m rounds once (relative u), so expf sees d_c (1 + e) and exp(d_c e) is within |d_c| u of 1; expf itself is within 2 ulp <= 4 u (CUDA math
  documentation); the sum of the ncls exponentials is ncls - 1 sequential float additions of positive terms ((ncls - 1) u) plus the error of its
  terms (sum_j R_j (|d_j| + 4) u relative); the division rounds once (u).  First order, and 1 % for the second-order terms:
    |y_c - R_c| <= 1.01 u R_c ((|d_c| + 4) + (ncls - 1) + sum_j R_j (|d_j| + 4) + 1) + 2^-146
  (the absolute term covers exponentials in the subnormal range: the sum is at least 1, so y_c is at most e_c).
DetectionOutput: oracle/detector_oracle.py:detection_output on the device's loc / softmax / prior blobs.  With zero loc both sides decode the prior boxes
with the same float32 operations (expf(0) == 1) and the scores are the blob's values, so the rows must be identical bit for bit.  With random loc, expf and numpy's exp
may differ by a few ulp: labels, order and count must be identical, boxes within 8 u (|x_max - x_min| + |x|) per coordinate, and every NMS decision
of the scene is checked to lie further than 1e-5 (relative) from nms_thr in float64, so that no scene can flip on a last-bit difference.
Post-processing (Detector2D.cc:52-88): DO.postprocess on the device's own rows uses the kernel's single-rounded float32 operations in the kernel's
order: objects, person boxes, their counts, have_dyn_rm and status must be identical bit for bit."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import detector_model as DM  # noqa: E402
import detector_oracle as DO  # noqa: E402
import ncnn_model as NM  # noqa: E402
from pysgs import binding as B  # noqa: E402
from test_gpu_detector import _run  # noqa: E402

U = 2.0 ** -24
W, H = 640, 480
K_DET_SORT_CAP, K_MERGE_CAP = 4096, 8192                     # detector.cu


def softmax_bound(x):
    """(R, bound) of the docstring for rows x [rows][ncls] float32"""
    xd = np.asarray(x, np.float64)
    d = xd - xd.max(1, keepdims=True)
    e = np.exp(d)
    R = e / e.sum(1, keepdims=True)
    ncls = x.shape[1]
    tail = (R * (np.abs(d) + 4)).sum(1, keepdims=True)
    return R, 1.01 * U * R * ((np.abs(d) + 4) + (ncls - 1) + tail + 1) + 2.0 ** -146


def check_softmax(x, y, what):
    R, bound = softmax_bound(x)
    err = np.abs(y.astype(np.float64) - R)
    bad = np.argwhere(err > bound)
    assert len(bad) == 0, '%s: %d softmax outputs outside the bound, first (row, class) %s: %r vs %r' % (what, len(bad), tuple(bad[0]), y[tuple(bad[0])], R[tuple(bad[0])])
    return float((err / bound).max())


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _detout_layer(layers, **over):
    """the DetectionOutput layer, with parameters overridden by key number (p1 = nms_thr ... p4 = conf_thr)"""
    L = [l for l in layers if l.type == 'DetectionOutput'][0]
    M = NM.Layer(L.type, L.name, L.inputs, L.outputs, dict(L.params))
    for k, v in over.items():
        M.params[int(k[1:])] = v
    return M


class Head:
    """One diagnostic handle on a head graph, run on a batch; keeps the outputs and every frame's tail blobs."""

    def __init__(self, tmp, scene, frames, det_thr=0.9, dyn_thr=0.01, max_boxes=32, tag='', **over):
        kw = DM.head_scene(scene); kw.update(over)
        self.pp, self.bp, self.nprs = DM.write_head_model(str(tmp), name=scene + tag, **kw)
        self.layers = NM.parse_param(self.pp); NM.load_weights(self.layers, self.bp)
        self.L = _detout_layer(self.layers)
        self.ncls = kw['ncls']
        det = B.Detector(self.pp, self.bp, max_frames=max(8, len(frames)), det_thr=det_thr, dyn_thr=dyn_thr, flags=B.DET_DIAGNOSTIC)
        self.out = _run(det, frames, max_boxes)
        self.nf = len(frames)
        self.prior = det.blob('mbox_priorbox').reshape(2, -1)
        self.loc = [det.blob('mbox_loc', f) for f in range(self.nf)]
        self.x = [det.blob('mbox_conf', f).reshape(-1, self.ncls) for f in range(self.nf)]
        self.y = [det.blob('mbox_conf_softmax', f).reshape(-1, self.ncls) for f in range(self.nf)]
        self.rows_cap = det.rows_cap
        det.close()
        self.nprior = self.prior.shape[1] // 4

    def rows(self, f):
        return self.out['rows'][f, :self.out['nrows'][f]]

    def ref(self, f, **over):
        return DO.detection_output(_detout_layer(self.layers, **over) if over else self.L, self.loc[f], self.y[f], self.prior)

    def candidates(self, f):
        """per class >= 1: the number of priors scoring above conf_thr"""
        return (self.y[f][:, 1:] > np.float32(self.L.p(4))).sum(0)


def check_rows_exact(h, f):
    ref = h.ref(f)
    got = h.rows(f)
    assert len(got) == len(ref), 'frame %d: %d rows, restatement %d' % (f, len(got), len(ref))
    assert np.array_equal(_bits(got), _bits(ref)), 'frame %d: first differing row %d' % (f, np.argwhere((_bits(got) != _bits(ref)).any(1))[0, 0])
    return ref


def check_post(h, f, W_, H_, det_thr, dyn_thr, max_boxes=32):
    """objects / person boxes / counts / have_dyn_rm / status of frame f against DO.postprocess of the device's own rows, bit for bit"""
    o = h.out
    objs, dyn_map, dyn_rm = DO.postprocess(h.rows(f), W_, H_, det_thr, dyn_thr)
    no = o['nobjects'][f]
    assert no == len(objs)
    ob = o['objects'][f, :no]
    assert np.array_equal(ob['id'], objs[:, 0].astype(np.int32))
    assert np.array_equal(_bits(np.stack([ob['prob'], ob['x'], ob['y'], ob['w'], ob['h']], 1).reshape(-1, 5)), _bits(objs[:, 1:]))
    for key, ref in (('dyn_map', dyn_map), ('dyn_rm', dyn_rm)):
        k = o['n' + key][f]
        assert k == min(len(ref), max_boxes), key
        assert np.array_equal(_bits(o[key][f, :k]), _bits(ref[:k])), key
    have = 1 if len(dyn_rm) and (objs[:, 0] != DO.PERSON).any() else 0
    assert o['have'][f] == have
    assert o['status'][f] == (1 if max(len(dyn_map), len(dyn_rm)) > max_boxes else 0)
    return objs, dyn_map, dyn_rm, have


def _frames(seeds):
    return np.stack([DM.synthetic_rgb(H, W, s) for s in seeds])


@pytest.fixture(scope='module')
def planted(tmp_path_factory):
    return Head(tmp_path_factory.mktemp('planted'), 'planted', _frames([1]), det_thr=0.05, dyn_thr=0.01)


def test_softmax_on_its_own_input(planted, tmp_path):
    """ncls 21 and 32 (the register path) and 33 and 40 (the loop path), planted and random logits"""
    worst = [('planted 21', check_softmax(planted.x[0], planted.y[0], 'planted'))]
    for scene, ncls in (('random32', 32), ('random40', 40), ('cap', 33)):
        h = Head(tmp_path, scene, _frames([2, 3]) if scene != 'cap' else _frames([2]))
        assert h.ncls == ncls and h.x[0].shape[1] == ncls
        for f in range(h.nf):
            worst.append(('%s %d frame %d' % (scene, ncls, f), check_softmax(h.x[f], h.y[f], scene)))
            assert np.ptp(h.x[f]) > 0
    print('softmax: max error / bound ' + ', '.join('%s %.3f' % w for w in worst))


def test_planted_rows_bit_exact_ties_and_truncation(planted):
    """(c) exact ties inside a class and across classes, (d) nms_top_k truncation, (e) keep_top_k truncation; boxes are decoded prior boxes."""
    h = planted
    assert not h.loc[0].any(), 'planted loc must be exactly zero'
    ref = check_rows_exact(h, 0)
    nms_topk, keep_topk = h.L.p(2), h.L.p(3)
    cand = h.candidates(0)
    over = int((cand > nms_topk).sum())
    assert over >= 5, cand
    kept_all = DO.detection_output(_detout_layer(h.layers, p3=10 ** 6), h.loc[0], h.y[0], h.prior)
    assert len(kept_all) > keep_topk and len(ref) == keep_topk
    rows = h.rows(0)
    same = rows[1:, 1] == rows[:-1, 1]
    in_class = int((same & (rows[1:, 0] == rows[:-1, 0])).sum())
    across = int((same & (rows[1:, 0] != rows[:-1, 0])).sum())
    assert in_class > 0 and across > 0
    # the tie order on the device: score descending, then class, then prior index (each row's box is its prior decoded with zero offsets)
    pb = DO.decode_boxes(h.loc[0], h.prior)
    idx = np.array([np.flatnonzero((_bits(pb) == _bits(r[2:])).all(1))[0] for r in rows])
    key = list(zip(-rows[:, 1].astype(np.float64), rows[:, 0], idx))
    assert key == sorted(key)
    print('planted: %d classes with more than nms_top_k = %d candidates (max %d), %d kept before keep_top_k = %d, %d adjacent ties in a class, '
          '%d across classes' % (over, nms_topk, cand.max(), len(kept_all), keep_topk, in_class, across))


def test_postprocess_bit_exact(planted, tmp_path):
    """Borders, max_boxes overflow, person-only frames (quirk Q12: have_dyn_rm 0), on the planted rows."""
    h = planted
    objs, dyn_map, dyn_rm, have = check_post(h, 0, W, H, 0.05, 0.01)
    r = h.rows(0)
    assert (r[:, 2:] < 0).any() and (r[:, 2:] * np.float32(300) > np.float32(299)).any(), 'no box crosses an image border'
    assert have == 1 and len(dyn_rm) > 0 and (objs[:, 0] != DO.PERSON).any()
    # the same rows, fewer boxes than persons: clamped counts, status 1
    small = Head(tmp_path, 'planted', _frames([1]), det_thr=0.05, dyn_thr=0.01, max_boxes=4, tag='_small')
    assert small.rows(0).tobytes() == r.tobytes()
    _, dm, _, _ = check_post(small, 0, W, H, 0.05, 0.01, max_boxes=4)
    assert len(dm) > 4 and small.out['status'][0] == 1
    # only person rows pass the thresholds: person boxes for rejection, but no other object, so have_dyn_rm stays 0; another image size
    persons = Head(tmp_path, 'planted', _frames([1]), det_thr=0.99, dyn_thr=0.01, tag='_persons')
    objs, _, dr, have = check_post(persons, 0, W, H, 0.99, 0.01)
    assert len(dr) > 0 and (objs[:, 0] == DO.PERSON).all() and have == 0
    print('post-processing: %d objects, %d / %d person boxes; max_boxes 4: %d person boxes, status 1; person-only: %d objects, have_dyn_rm 0' %
          (len(h.rows(0)), len(dyn_map), len(dyn_rm), len(dm), len(objs)))


def test_nms_threshold_equal_to_iou(tmp_path):
    """(a) the max box of a 1x1 map, scored below the concentric min box, at IoU == nms_thr: kept (strict >); one ulp lower: suppressed."""
    probe = Head(tmp_path, 'iou', _frames([1]), tag='_probe')
    pb = DO.decode_boxes(probe.loc[0], probe.prior)                 # zero offsets: the boxes NMS compares
    assert probe.nprior == 2 and probe.y[0][0, 1] > probe.y[0][1, 1]
    t = DM.nms_iou(pb[0], pb[1])
    assert 0 < t < 1
    at = Head(tmp_path, 'iou', _frames([1]), tag='_at', nms_thr=t)
    assert np.float32(at.L.p(1)) == t and len(check_rows_exact(at, 0)) == 2, 'the box at IoU == nms_thr must be kept'
    below = Head(tmp_path, 'iou', _frames([1]), tag='_below', nms_thr=np.nextafter(t, np.float32(0)))
    assert len(check_rows_exact(below, 0)) == 1, 'the box at IoU one ulp above nms_thr must be suppressed'
    print('nms: IoU %r (%s): kept at nms_thr == IoU, suppressed one ulp lower' % (t, _bits(t)))


def test_score_equal_to_conf_thr(planted, tmp_path):
    """(b) conf_thr set to a score the device produced: entries scoring exactly that value are excluded; one ulp lower they are included."""
    h = planted
    sc = h.y[0][:, 1:]
    vals, counts = np.unique(sc[sc > np.float32(h.L.p(4))], return_counts=True)
    v = vals[np.argmax(np.where(np.isin(vals, h.rows(0)[:, 1]), counts, 0))]         # the most frequent score that makes it into the rows
    n_eq = int((sc == v).sum())
    assert n_eq > 1 and v in h.rows(0)[:, 1]
    at = Head(tmp_path, 'planted', _frames([1]), det_thr=0.05, tag='_thr_at', conf_thr=v)
    assert np.float32(at.L.p(4)) == v and at.y[0].tobytes() == h.y[0].tobytes()
    r = check_rows_exact(at, 0)
    assert (r[:, 1] > v).all()
    below = Head(tmp_path, 'planted', _frames([1]), det_thr=0.05, tag='_thr_below', conf_thr=np.nextafter(v, np.float32(0)))
    r2 = check_rows_exact(below, 0)
    assert (r2[:, 1] == v).any()
    print('conf_thr: %d entries score exactly %r: excluded at conf_thr == score, %d of them in the rows one ulp lower' % (n_eq, v, int((r2[:, 1] == v).sum())))


def test_at_the_caps(tmp_path):
    """(f) 4096 priors, all above conf_thr in every class (kDetSortCap entries per class), (33 - 1) * 256 = 8192 kept entries in the merge (kMergeCap)."""
    h = Head(tmp_path, 'cap', _frames([1]))
    assert h.nprior == K_DET_SORT_CAP
    cand = h.candidates(0)
    assert (cand == K_DET_SORT_CAP).all(), cand
    kept_all = DO.detection_output(_detout_layer(h.layers, p3=10 ** 6), h.loc[0], h.y[0], h.prior)
    assert len(kept_all) == (h.ncls - 1) * h.L.p(2) == K_MERGE_CAP
    ref = check_rows_exact(h, 0)
    assert len(ref) == h.L.p(3) == 1024
    print('caps: %d priors above conf_thr in each of %d classes, %d entries merged, %d rows' % (cand.min(), h.ncls - 1, len(kept_all), len(ref)))


def test_4097_priors_refused(tmp_path):
    kw = DM.head_scene('cap')
    kw['maps'] = kw['maps'] + [(1, 60.0, None, (), False)]
    kw['conf_bias'] = kw['conf_bias'] + [0.0]
    pp, bp, nprs = DM.write_head_model(str(tmp_path), name='cap4097', **kw)
    assert sum(n * m[0] ** 2 for n, m in zip(nprs, kw['maps'])) == K_DET_SORT_CAP + 1
    with pytest.raises(B.SgsError) as e:
        B.Detector(pp, bp, max_frames=1)
    assert e.value.code == B.SGS_ERR_UNSUPPORTED


def _nms_margin(h, f, boxes=None):
    """smallest |max IoU against the kept boxes - nms_thr| / nms_thr over every NMS decision of frame f, in float64 on the restatement's boxes"""
    boxes = DO.decode_boxes(h.loc[f], h.prior).astype(np.float64) if boxes is None else boxes
    thr, topk, cthr = float(np.float32(h.L.p(1))), h.L.p(2), np.float32(h.L.p(4))
    conf = h.y[f]
    margin, decisions = np.inf, 0
    for c in range(1, h.ncls):
        idx = np.nonzero(conf[:, c] > cthr)[0]
        idx = idx[np.lexsort((idx, -conf[idx, c]))][:topk]
        kept = []
        for i in idx:
            if kept:
                a, b = boxes[kept], boxes[i]
                iw = np.clip(np.minimum(a[:, 2], b[2]) - np.maximum(a[:, 0], b[0]), 0, None)
                ih = np.clip(np.minimum(a[:, 3], b[3]) - np.maximum(a[:, 1], b[1]), 0, None)
                inter = iw * ih
                iou = inter / ((a[:, 2] - a[:, 0]) * (a[:, 3] - a[:, 1]) + (b[2] - b[0]) * (b[3] - b[1]) - inter)
                m = iou.max()
                margin = min(margin, abs(m - thr) / thr); decisions += 1
                if m > thr:
                    continue
            kept.append(i)
    return margin, decisions


def check_rows_random(h, f):
    """labels, order, count identical; boxes within 8 u (|w| + |x|); every NMS decision more than 1e-5 from nms_thr"""
    margin, decisions = _nms_margin(h, f)
    assert margin > 1e-5, 'frame %d: an NMS decision lies within %.3g of nms_thr; the scene can flip on rounding' % (f, margin)
    ref, got = h.ref(f), h.rows(f)
    assert len(got) == len(ref)
    assert np.array_equal(_bits(got[:, :2]), _bits(ref[:, :2])), 'labels / scores / order'
    ext = np.abs(np.concatenate([ref[:, 4:6] - ref[:, 2:4]] * 2, 1))
    assert (np.abs(got[:, 2:].astype(np.float64) - ref[:, 2:]) <= 8 * U * (ext + np.abs(ref[:, 2:]))).all(), 'boxes'
    return ref, margin, decisions


def test_batch_of_eight_frames(tmp_path):
    """(g) random head weights, 8 different frames (frame 5 flat grey: no candidate at all): each frame's rows equal the restatement's on its own
    input and the rows of the same frame run alone; post-processing bit for bit."""
    frames = _frames([11, 12, 13, 14, 15, 16, 17, 18])
    frames[5] = (124, 116, 104)
    h = Head(tmp_path, 'random', frames, det_thr=0.5, dyn_thr=0.01)
    assert h.loc[0].any() and h.nf == 8
    cands = [int(h.candidates(f).sum()) for f in range(8)]
    assert cands[5] == 0 and h.out['nrows'][5] == 0 and min(c for i, c in enumerate(cands) if i != 5) > 0
    nrows = h.out['nrows']
    assert len(set(nrows.tolist())) >= 4, nrows
    margins = []
    for f in range(8):
        _, m, d = check_rows_random(h, f)
        margins.append((m, d))
        check_post(h, f, W, H, 0.5, 0.01)
    for f in (0, 5, 7):
        one = Head(tmp_path, 'random', frames[f:f + 1], det_thr=0.5, dyn_thr=0.01, tag='_one%d' % f)
        n = one.out['nrows'][0]
        assert n == nrows[f] and one.rows(0).tobytes() == h.rows(f).tobytes(), 'frame %d: rows depend on the batch' % f
        for k in ('nobjects', 'ndyn_map', 'ndyn_rm', 'have', 'status'):
            assert one.out[k][0] == h.out[k][f], k
    print('batch: candidates per frame %s, rows %s, smallest NMS margin %.3g over %d decisions' %
          (cands, nrows.tolist(), min(m for m, _ in margins), sum(d for _, d in margins)))


def test_random_heads_with_forty_classes(tmp_path):
    h = Head(tmp_path, 'random40', _frames([21, 22]))
    for f in range(2):
        assert h.out['nrows'][f] > 0
        check_rows_random(h, f)
        check_post(h, f, W, H, 0.9, 0.01)
