"""CPU checks of the helpers of tests/test_gpu_detector_head.py: the head-only graph writer (detector_model.write_head_model / head_scene), the
float32 IoU it plants as nms_thr, and the Softmax error bound, here on the restatement's own Softmax (oracle/detector_oracle.py).  The product's
graph builder runs in plan-only mode (no device needed) for the prior / merge caps."""
import numpy as np
import pytest

import detector_model as DM
import detector_oracle as DO
import ncnn_model as NM
from pysgs import binding as B
from test_gpu_detector_head import softmax_bound

SCENES = ('planted', 'iou', 'cap', 'random', 'random32', 'random40')


def _write(tmp_path, scene, **over):
    kw = DM.head_scene(scene); kw.update(over)
    pp, bp, nprs = DM.write_head_model(str(tmp_path), name=scene, **kw)
    layers = NM.parse_param(pp)
    used, total = NM.load_weights(layers, bp)
    assert used == total
    return kw, pp, bp, nprs, layers


@pytest.mark.parametrize('scene', SCENES)
def test_head_writer_round_trips(tmp_path, scene):
    kw, pp, bp, nprs, layers = _write(tmp_path, scene)
    L = [l for l in layers if l.type == 'DetectionOutput'][0]
    for key, name, default in ((1, 'nms_thr', 0.45), (4, 'conf_thr', 0.01)):
        assert np.float32(L.p(key)) == np.float32(kw.get(name, default)), name          # written with %.9g: the same float32 back
    assert (L.p(0), L.p(2), L.p(3)) == (kw['ncls'], kw.get('nms_topk', 300), kw.get('keep_topk', 100))
    heads = [l for l in layers if l.type == 'Convolution' and l.weight.shape[1] == 8 and l.weight.shape[2] == 1]
    assert len(heads) == 2 * len(kw['maps'])
    for i, npr in enumerate(nprs):
        cf, lc = heads[2 * i], heads[2 * i + 1]
        assert cf.weight.shape[0] == npr * kw['ncls'] and lc.weight.shape[0] == npr * 4
        assert np.array_equal(cf.bias.reshape(npr, kw['ncls']), np.broadcast_to(np.float32(kw['conf_bias'][i]), (npr, kw['ncls'])))
        if kw.get('weights', 'zero') == 'zero':
            assert not cf.weight.any() and not lc.weight.any() and not lc.bias.any()
    blobs = DO.forward(layers, DO.preprocess(DM.synthetic_rgb(480, 640, 1)), want='mbox_priorbox')
    nprior = sum(n * m[0] ** 2 for n, m in zip(nprs, kw['maps']))
    assert blobs['mbox_priorbox'].shape == (2, 4 * nprior)
    d = B.Detector(pp, bp, max_frames=8, flags=B.DET_DIAGNOSTIC | B.DET_PLAN_ONLY)
    d.close()


def test_sort_and_merge_caps_at_create(tmp_path):
    """4096 priors and (ncls - 1) * nms_top_k = 8192 are accepted; 4097 priors, or 8194 merge entries, are refused."""
    kw, pp, bp, nprs, _ = _write(tmp_path, 'cap')
    assert nprs[0] * kw['maps'][0][0] ** 2 == 4096 and (kw['ncls'] - 1) * kw['nms_topk'] == 8192
    B.Detector(pp, bp, max_frames=1, flags=B.DET_PLAN_ONLY).close()
    for over in (dict(maps=kw['maps'] + [(1, 60.0, None, (), False)], conf_bias=kw['conf_bias'] + [0.0]),
                 dict(ncls=18, nms_topk=482, conf_bias=[0.0])):
        _, pp, bp, nprs, _ = _write(tmp_path, 'cap', **over)
        with pytest.raises(B.SgsError) as e:
            B.Detector(pp, bp, max_frames=1, flags=B.DET_PLAN_ONLY)
        assert e.value.code == B.SGS_ERR_UNSUPPORTED


def _two_box_rows(boxes, scores, nms_thr):
    """DO.detection_output on two priors with zero loc, class 1 scored `scores`"""
    L = NM.Layer('DetectionOutput', 'd', [], [], {0: 2, 1: float(nms_thr), 2: 300, 3: 100, 4: 0.01})
    conf = np.stack([1 - np.float32(scores), np.float32(scores)], 1).astype(np.float32)
    prior = np.stack([np.asarray(boxes, np.float32).reshape(-1), np.tile(np.float32([0.1, 0.1, 0.2, 0.2]), len(boxes))])
    return DO.detection_output(L, np.zeros(4 * len(boxes), np.float32), conf, prior)


def test_planted_iou_matches_the_restatement(tmp_path):
    """nms_iou (the kernel's order) decides like DO.detection_output: kept at nms_thr == IoU, suppressed one ulp lower -- on the concentric pair
    of the 'iou' scene and on random overlapping pairs."""
    _, _, _, _, layers = _write(tmp_path, 'iou')
    pb = DO.forward(layers, DO.preprocess(DM.synthetic_rgb(480, 640, 1)), want='mbox_priorbox')['mbox_priorbox']
    pairs = [pb[0].reshape(-1, 4)]                                      # the concentric min / max prior boxes
    rng = np.random.default_rng(3)
    for _ in range(200):
        a = np.sort(rng.uniform(-0.2, 1.2, (2, 2)), 0).T.reshape(-1)[[0, 2, 1, 3]]
        b = a + rng.uniform(-0.1, 0.1, 4)
        b = np.array([min(b[0], b[2]), min(b[1], b[3]), max(b[0], b[2]), max(b[1], b[3])])
        pairs.append(np.float32([a, b]))
    reached = 0
    for boxes in pairs:
        prior = np.stack([np.asarray(boxes, np.float32).reshape(-1), np.tile(np.float32([0.1, 0.1, 0.2, 0.2]), 2)])
        dec = DO.decode_boxes(np.zeros(8, np.float32), prior)
        t = DM.nms_iou(dec[0], dec[1])
        if not 0 < t < 1:
            continue
        reached += 1
        assert len(_two_box_rows(boxes, [0.8, 0.6], t)) == 2
        assert len(_two_box_rows(boxes, [0.8, 0.6], np.nextafter(t, np.float32(0)))) == 1
    assert reached > 100


@pytest.mark.parametrize('scene', SCENES)
def test_softmax_bound_on_the_restatement(tmp_path, scene):
    """the bound of test_gpu_detector_head.py holds for the restatement's float32 Softmax (numpy exp, pairwise sum) on every scene's input"""
    kw, pp, bp, nprs, layers = _write(tmp_path, scene)
    blobs = DO.forward(layers, DO.preprocess(DM.synthetic_rgb(480, 640, 2)), want='mbox_conf_softmax')
    x = blobs['mbox_conf'].reshape(-1, kw['ncls'])
    y = blobs['mbox_conf_softmax']
    R, bound = softmax_bound(x)
    assert (np.abs(y - R) <= bound).all()
    assert np.ptp(x) > 0
