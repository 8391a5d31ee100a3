"""The detector's input resize + mean subtraction (preprocess_table_kernel + preprocess_kernel of detector.cu) bit for bit against the restatement
(detector_oracle.preprocess), at every camera geometry and device layout of tests/detector_resize_cases.py, read back from the input blob of
DET_DIAGNOSTIC handles of the synthetic mini graph.

  * every frame of 3-frame batches of distinct frames, at every geometry x layout (dense, pitch 3W + 5, frame stride past H * pitch with marker bytes
    in the gaps, stride 0, base pointer 1 to 3 bytes off); the marker's value changes nothing;
  * the half-rounding images: the device takes the half-to-even side of the exact-half coefficients, which the half-away-from-zero restatement does
    not (so the check can see the convention);
  * camera-size changes on one handle (the coefficient table is rebuilt per geometry): after every call of a sequence that mixes the host and the
    device entry points and goes small -> large -> small -> large, the input blob and the results equal those of a fresh handle;
  * the host entry point with a wide pitch returns the device entry point's objects."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import detector_model as DM  # noqa: E402
import detector_oracle as DO  # noqa: E402
import detector_resize_cases as RC  # noqa: E402
from pysgs import binding as B  # noqa: E402
from test_gpu_detector import _run_ptr  # noqa: E402

NF = 3


@pytest.fixture(scope='module')
def mini(tmp_path_factory):
    return DM.write_mini_model(str(tmp_path_factory.mktemp('mini_resize')), 0)


@pytest.fixture(scope='module')
def diag(mini):
    det = B.Detector(*mini, max_frames=NF, flags=B.DET_DIAGNOSTIC)
    yield det
    det.close()


def _device_call(det, fr, layout, marker=RC.MARKER):
    """fr laid out as `layout` in device memory, one detect_device call: the outputs of _run_ptr"""
    import torch
    buf, off, stride, pitch = RC.pack(fr, layout, marker)
    d = torch.from_numpy(buf).cuda()
    assert d.data_ptr() % 16 == 0
    F, H, W, _ = fr.shape
    return _run_ptr(det, d.data_ptr() + off, stride, pitch, W, H, F)


def _blobs(det, nf):
    return [det.blob('input', f) for f in range(nf)]


def _detect_host(det, img, pitch):
    """sgs_detect on img (H x W x 3) stored in rows of `pitch` bytes (the bytes past 3W hold the marker)"""
    H, W, _ = img.shape
    rows = np.full((H, pitch), RC.MARKER, np.uint8)
    rows[:, :3 * W] = img.reshape(H, -1)
    out = np.zeros(det.rows_cap, B.OBJ_DTYPE); n = C.c_int()
    B.check(B.lib().sgs_detect(det.h, rows.ctypes.data_as(C.c_void_p), W, H, pitch, out.ctypes.data_as(C.c_void_p), len(out), C.byref(n)))
    return out[:n.value]


@pytest.mark.parametrize('w,h', RC.GEOMETRIES)
def test_input_blob_at_every_layout(diag, w, h):
    fr = RC.frames(w, h, NF, 3)
    for layout in RC.LAYOUTS:
        _device_call(diag, fr, layout)
        got = _blobs(diag, NF)
        for f, ref in enumerate(RC.expected_blobs(fr, layout)):
            assert got[f].tobytes() == ref.reshape(-1).tobytes(), '%dx%d %s: frame %d differs from the restatement' % (w, h, layout, f)
        if layout == 'zero':
            assert got[0].tobytes() == got[1].tobytes() == got[2].tobytes()
        if layout in ('gap', 'offset'):          # the bytes between rows and frames are never read
            _device_call(diag, fr, layout, marker=0xFF - RC.MARKER)
            assert all(a.tobytes() == b.tobytes() for a, b in zip(_blobs(diag, NF), got)), '%dx%d %s: the marker bytes change the blob' % (w, h, layout)


HALF_GEOMETRIES = [g for g in RC.GEOMETRIES if len(RC.exact_halves(RC.T, g[0])) or len(RC.exact_halves(RC.T, g[1]))]


@pytest.mark.parametrize('w,h', HALF_GEOMETRIES)
def test_exact_halves_round_to_even(diag, w, h):
    img = RC.half_image(w, h)
    _device_call(diag, img[None], 'dense')
    got = diag.blob('input', 0).reshape(3, RC.T, RC.T)
    even, away = DO.preprocess(img), DO.preprocess(img, DO.round_half_away)
    assert got.tobytes() == even.tobytes(), 'the device resize differs from the half-to-even restatement'
    d = (got != away).any(0)
    allowed = np.zeros_like(d)
    allowed[:, RC.exact_halves(RC.T, w)] = True
    allowed[RC.exact_halves(RC.T, h), :] = True
    assert d.any() and not (d & ~allowed).any(), 'the device differs from the half-away restatement outside the exact-half columns / rows'


def test_geometry_changes_on_one_handle(mini):
    """A -> B -> A -> C, host and device calls mixed.  Every later geometry is at least as large as the first on both axes."""
    seq = [('host', 640, 480, 1), ('device', 1280, 720, 2), ('device', 640, 480, 3), ('host', 752, 480, 1), ('device', 752, 480, 2)]
    det = B.Detector(*mini, max_frames=NF, flags=B.DET_DIAGNOSTIC)
    for i, (entry, w, h, n) in enumerate(seq):
        fr = np.stack([DM.synthetic_rgb(h, w, 300 + 10 * i + k) for k in range(n)])
        fresh = B.Detector(*mini, max_frames=NF, flags=B.DET_DIAGNOSTIC)
        what = 'call %d (%s %dx%d)' % (i, entry, w, h)
        if entry == 'host':
            pitch = 3 * w + 67
            a, b = _detect_host(det, fr[0], pitch), _detect_host(fresh, fr[0], pitch)
            assert a.tobytes() == b.tobytes(), what + ': objects'
        else:
            a, b = _device_call(det, fr, 'pitch'), _device_call(fresh, fr, 'pitch')
            for k in a:
                assert a[k].tobytes() == b[k].tobytes(), what + ': ' + k
        for f in range(n):
            x = det.blob('input', f)
            assert x.tobytes() == fresh.blob('input', f).tobytes() == DO.preprocess(fr[f]).reshape(-1).tobytes(), what + ': input blob'
        fresh.close()
    det.close()


def test_host_entry_point_with_a_wide_pitch(mini):
    det = B.Detector(*mini, max_frames=1, det_thr=0.05)
    for w, h, seed in ((640, 480, 5), (1280, 720, 6)):
        img = DM.synthetic_rgb(h, w, seed)
        dev = _device_call(det, img[None], 'dense')
        objs = _detect_host(det, img, 3 * w + 129)
        assert len(objs) > 0 and objs.tobytes() == dev['objects'][0, :dev['nobjects'][0]].tobytes(), (w, h)
    det.close()
