"""GPU parity of the detector (Detector2D::detect, src/Detector2D.cc:34-89) through the C ABI against the CPU restatement
(oracle/detector_oracle.py, PyTorch FP32).  PARITY UNPINNED with respect to ncnn itself (not available here): these tests prove GPU == restatement.
  * input blob (resize + mean): bit-exact;
  * every intermediate blob (diagnostic mode, one kernel per layer): max|diff| <= 2e-4 * max(1, max|ref|) per blob -- FP32 sums in a different
    order (the PyTorch restatement itself sits 1e-5 of the blob scale away from a float64 run of the same graph; 5e-5 observed near the end of the
    trained model);
  * fused / pooled execution == diagnostic execution, bit for bit (the fused tails apply the same roundings in the same order);
  * detection rows: same labels in the same order, scores and boxes within 2e-5; Object2D / dynamic boxes likewise."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import detector_model as DM  # noqa: E402
import detector_oracle as DO  # noqa: E402
import ncnn_model as NM  # noqa: E402
from pysgs import binding as B  # noqa: E402

REAL = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle', '_ref', 'ncnn_model', 'mobilenetv3_ssdlite_voc')
TOL = 2e-5


def _run(det, frames, max_boxes=32):
    """frames: [F, H, W, 3] uint8 -> dict of host arrays."""
    import torch
    F, H, W, _ = frames.shape
    d = torch.from_numpy(np.ascontiguousarray(frames)).cuda()
    return _run_ptr(det, d.data_ptr(), H * W * 3, W * 3, W, H, F, max_boxes)


def _run_ptr(det, d_rgb, frame_stride, pitch, W, H, F, max_boxes=32):
    """F frames of W x H at device address d_rgb, frame_stride / pitch bytes apart -> dict of host arrays."""
    import torch
    R = det.rows_cap
    o = dict(rows=torch.zeros((F, R, 6), device='cuda'), nrows=torch.zeros(F, dtype=torch.int32, device='cuda'),
             objects=torch.zeros((F, R, 6), device='cuda'), nobjects=torch.zeros(F, dtype=torch.int32, device='cuda'),
             dyn_map=torch.zeros((F, max_boxes, 4), device='cuda'), ndyn_map=torch.zeros(F, dtype=torch.int32, device='cuda'),
             dyn_rm=torch.zeros((F, max_boxes, 4), device='cuda'), ndyn_rm=torch.zeros(F, dtype=torch.int32, device='cuda'),
             have=torch.zeros(F, dtype=torch.uint8, device='cuda'), status=torch.zeros(F, dtype=torch.int32, device='cuda'))
    det.detect_device(d_rgb, frame_stride, pitch, W, H, F, *[o[k].data_ptr() for k in
                      ('rows', 'nrows', 'objects', 'nobjects', 'dyn_map', 'ndyn_map', 'dyn_rm', 'ndyn_rm', 'have')], max_boxes, o['status'].data_ptr())
    torch.cuda.synchronize()
    out = {k: v.cpu().numpy() for k, v in o.items()}
    out['objects'] = out['objects'].view(np.uint8).reshape(F, R, 24).copy().view(B.OBJ_DTYPE).reshape(F, R)
    return out


def _check_rows(out, f, rows_ref, post_ref, max_boxes=32):
    n = out['nrows'][f]
    assert n == len(rows_ref)
    rows = out['rows'][f, :n]
    assert np.array_equal(rows[:, 0], rows_ref[:, 0]), 'labels / order'
    assert np.abs(rows[:, 1:] - rows_ref[:, 1:]).max() <= TOL
    objs, dyn_map, dyn_rm = post_ref
    no = out['nobjects'][f]
    assert no == len(objs)
    o = out['objects'][f, :no]
    assert np.array_equal(o['id'], objs[:, 0].astype(np.int32))
    got = np.stack([o['prob'], o['x'], o['y'], o['w'], o['h']], 1)
    assert np.abs(got - objs[:, 1:]).max() <= TOL * 1280
    for key, ref in (('dyn_map', dyn_map), ('dyn_rm', dyn_rm)):
        k = out['n' + key][f]
        assert k == min(len(ref), max_boxes)
        assert np.abs(out[key][f, :k] - ref[:k]).max(initial=0) <= TOL * 1280
    # the flag the Frame ends up with (src/Frame.cc:482-491): person boxes for rejection AND at least one non-person object (quirk Q12)
    assert out['have'][f] == (1 if len(dyn_rm) and (objs[:, 0] != 15).any() else 0)
    assert out['status'][f] == (1 if max(len(dyn_map), len(dyn_rm)) > max_boxes else 0)


@pytest.fixture(scope='module')
def mini(tmp_path_factory):
    pp, bp = DM.write_mini_model(str(tmp_path_factory.mktemp('mini')), 0)
    layers = NM.parse_param(pp); NM.load_weights(layers, bp)
    return pp, bp, layers


def _blob_parity(pp, bp, layers, img, only=None):
    det = B.Detector(pp, bp, max_frames=1, flags=B.DET_DIAGNOSTIC)
    _run(det, img[None])
    ref = DO.forward(layers, DO.preprocess(img))
    first_bad = None
    for L in layers:
        if L.type in ('MemoryData', 'DetectionOutput'):
            continue
        for name in L.outputs:
            r = np.asarray(ref[name], np.float32).reshape(-1)
            g = det.blob(name)
            assert g.shape == r.shape, (L.type, name, g.shape, r.shape)
            if L.type in ('Input', 'Split') and name.startswith(('input', 'data')):
                assert np.array_equal(g, r), 'input blob must be bit-exact'
            err = np.abs(g - r) / max(1.0, float(np.abs(r).max()))
            if err.max() > 2e-4 and first_bad is None:
                first_bad = (L.type, L.name, name, float(err.max()), int(err.argmax()))
    det.close()
    assert first_bad is None, 'first mismatching layer: %s' % (first_bad,)


def test_every_blob_of_the_synthetic_graph(mini):
    pp, bp, layers = mini
    _blob_parity(pp, bp, layers, DM.synthetic_rgb(480, 640, 1))


def test_detections_of_the_synthetic_graph(mini):
    pp, bp, layers = mini
    frames = np.stack([DM.synthetic_rgb(480, 640, s) for s in (1, 2, 3)])
    fused = B.Detector(pp, bp, max_frames=4)
    diag = B.Detector(pp, bp, max_frames=4, flags=B.DET_DIAGNOSTIC)
    a, b = _run(fused, frames), _run(diag, frames)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), 'fused and per-layer execution differ in ' + k
    one = _run(fused, frames[1:2])
    assert one['rows'][0].tobytes() == a['rows'][1].tobytes() and one['nobjects'][0] == a['nobjects'][1], 'batch position changes the result'
    for f in range(3):
        rows_ref, post = DO.detect(layers, frames[f], 0.9, 0.01)
        assert (rows_ref[:, 0] == 15).any() or f > 0
        _check_rows(a, f, rows_ref, post)
    # small box capacity: clamped and flagged
    small = _run(fused, frames[:1], max_boxes=2)
    rows_ref, post = DO.detect(layers, frames[0], 0.9, 0.01)
    assert len(post[1]) > 2
    _check_rows(small, 0, rows_ref, post, max_boxes=2)
    # host entry point == device entry point
    objs = fused.detect(frames[0])
    assert objs.tobytes() == a['objects'][0, :a['nobjects'][0]].tobytes()
    fused.close(); diag.close()


def test_other_image_geometry_and_thresholds(mini):
    pp, bp, layers = mini
    img = DM.synthetic_rgb(720, 1280, 7)
    det = B.Detector(pp, bp, max_frames=2, det_thr=0.95, dyn_thr=0.5)
    out = _run(det, img[None])
    rows_ref, post = DO.detect(layers, img, 0.95, 0.5)
    _check_rows(out, 0, rows_ref, post)
    det.close()


def test_argument_errors(mini):
    import torch
    pp, bp, _ = mini
    det = B.Detector(pp, bp, max_frames=1)
    d = torch.zeros((2, 64, 64, 3), dtype=torch.uint8, device='cuda')
    with pytest.raises(B.SgsError) as e:
        det.detect_device(d.data_ptr(), 64 * 64 * 3, 64 * 3, 64, 64, 2)
    assert e.value.code == B.SGS_ERR_INVALID
    with pytest.raises(B.SgsError) as e:
        det.blob('input')
    assert e.value.code == B.SGS_ERR_UNSUPPORTED
    with pytest.raises(B.SgsError) as e:
        det.detect(np.zeros((1, 64, 3), np.uint8))
    assert e.value.code == B.SGS_ERR_INVALID
    det.close()


needs_real = pytest.mark.skipif(not os.path.exists(REAL + '.param'), reason='reference model copy (oracle/_ref/ncnn_model, made by build()) not present')


@pytest.fixture(scope='module')
def real():
    layers = NM.parse_param(REAL + '.param'); NM.load_weights(layers, REAL + '.bin')
    return layers


@needs_real
def test_every_blob_of_the_reference_model(real):
    _blob_parity(REAL + '.param', REAL + '.bin', real, DM.synthetic_rgb(480, 640, 11))


@needs_real
def test_detections_of_the_reference_model(real):
    frames = np.stack([DM.synthetic_rgb(480, 640, s) for s in (21, 22)])
    det = B.Detector(REAL + '.param', REAL + '.bin', max_frames=2, det_thr=0.9, dyn_thr=0.01)
    out = _run(det, frames)
    for f in range(2):
        rows_ref, post = DO.detect(real, frames[f], 0.9, 0.01)
        _check_rows(out, f, rows_ref, post)
    det.close()
