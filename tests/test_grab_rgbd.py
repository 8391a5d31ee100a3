"""The image half of Tracking::GrabImageRGBD without a device: the numpy restatement of the colour -> gray and raw depth -> float conversions
(tests/grab_ref.py, which the device kernels are checked against) equals cv2 4.13 on every input the conversions can see, the committed fixture
agrees with it, the sgs_rgbd_format mirror has the compiler's layout and the RGB-D entry points are exported and typed from sgs_abi.h."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import grab_ref as GR
from pysgs import binding as B
from pysgs import synth
from test_abi_binding import INCLUDE, LAYOUT_C, _kind


@pytest.fixture(params=[True, False], ids=['ipp', 'no-ipp'])
def cv2_ipp(request):
    cv2 = pytest.importorskip('cv2')
    was = cv2.ipp.useIPP()
    cv2.ipp.setUseIPP(request.param)
    yield cv2
    cv2.ipp.setUseIPP(was)


@pytest.mark.parametrize('rgb_order', [1, 0])
def test_gray_equals_cv2_on_every_triple(cv2_ipp, rgb_order):
    img = GR.all_triples()
    code = cv2_ipp.COLOR_RGB2GRAY if rgb_order else cv2_ipp.COLOR_BGR2GRAY
    assert np.array_equal(cv2_ipp.cvtColor(img, code), GR.to_gray(img, rgb_order))


@pytest.mark.parametrize('rgb_order', [1, 0])
def test_gray_equals_cv2_at_scalar_tails_and_odd_sizes(cv2_ipp, rgb_order):
    rng = np.random.RandomState(3)
    code = cv2_ipp.COLOR_RGB2GRAY if rgb_order else cv2_ipp.COLOR_BGR2GRAY
    for w, h in [(w, 3) for w in range(1, 34)] + [(641, 479), (640, 480)]:
        img = rng.randint(0, 256, (h, w, 3)).astype(np.uint8)
        assert np.array_equal(cv2_ipp.cvtColor(img, code).reshape(h, w), GR.to_gray(img, rgb_order)), (w, h)


def test_the_two_channel_orders_differ():
    img = GR.all_triples()
    assert (GR.to_gray(img, 1) != GR.to_gray(img, 0)).sum() > 1 << 23


@pytest.mark.parametrize('factor', GR.FACTORS, ids=['tum1', 'tum2', 'astra'])
def test_depth_equals_cv2_for_every_uint16_and_random_float32(factor):
    cv2 = pytest.importorskip('cv2')
    raw = np.arange(1 << 16, dtype=np.uint16).reshape(256, 256)
    assert cv2.multiply(raw, float(factor), dtype=cv2.CV_32F).tobytes() == GR.to_depth(raw, factor).tobytes()
    f = np.random.RandomState(4).uniform(0, 20, (480, 640)).astype(np.float32)
    assert cv2.multiply(f, float(factor), dtype=cv2.CV_32F).tobytes() == GR.to_depth(f, factor).tobytes()


def test_fixture_equals_the_restatement(golden_dir):
    z = np.load(os.path.join(golden_dir, 'grab_rgbd.npz'))
    seen = set()
    for k in range(int(z['ncases'])):
        w, h, nf, dt, rp, rs, dp, ds = (int(v) for v in z['c%d_meta' % k])
        assert rs != rp * h and ds != dp * h and rp > 3 * w             # padded rows and frames
        rgb = GR.frames_from_buffer(z['c%d_rgb' % k], nf, h, 3 * w, rp, rs, np.uint8).reshape(nf, h, w, 3)
        raw = GR.frames_from_buffer(z['c%d_depth' % k], nf, h, (2 if dt == 0 else 4) * w, dp, ds, np.uint16 if dt == 0 else np.float32)
        seen |= {int(v) for v in raw.flat if dt == 0 and v in (0, 65535)}
        assert np.array_equal(GR.to_gray(rgb, 1), z['c%d_gray_rgb' % k]) and np.array_equal(GR.to_gray(rgb, 0), z['c%d_gray_bgr' % k])
        for j, fac in enumerate(z['factors']):
            assert GR.to_depth(raw, fac).tobytes() == z['c%d_depth_f%d' % (k, j)].tobytes(), (k, j)
    assert seen == {0, 65535}


def test_rgbd_format_mirror_matches_the_compiler_layout(tmp_path):
    cls, cname = B.RgbdFormat, 'sgs_rgbd_format'
    src = [LAYOUT_C, 'SIZE("%s", %s)' % (cls.__name__, cname)]
    want = {(cls.__name__, 'sizeof'): (0, C.sizeof(cls), 'struct')}
    for name, t in cls._fields_:
        src.append('FIELD("%s", %s, "%s", %s, %s)' % (cls.__name__, cname, name, name, name + '[0]' if issubclass(t, C.Array) else name))
        want[cls.__name__, name] = (getattr(cls, name).offset, getattr(cls, name).size, _kind(t))
    (tmp_path / 'layout.c').write_text('\n'.join(src) + '\nreturn 0; }\n')
    cc = subprocess.run(['cc', '-std=c11', '-I', INCLUDE, '-o', str(tmp_path / 'layout'), str(tmp_path / 'layout.c')], capture_output=True, text=True)
    assert cc.returncode == 0, cc.stderr
    got = {}
    for line in subprocess.check_output([str(tmp_path / 'layout')], text=True).splitlines():
        py, name, off, size, kind = line.split()
        got[py, name] = (int(off), int(size), kind)
    assert got == want


P, I32, Z, F32 = C.c_void_p, C.c_int32, C.c_size_t, C.c_float
NEW = {
    'sgs_grab_rgbd_batch_device': [P, Z, I32, P, Z, I32, P, I32, I32, I32, P, Z, I32, P, Z, I32, P],
    'sgs_tracker_step_rgbd_device': [P, P, P, Z, I32, P, Z, I32, P, I32, P] + [P] * 8 + [F32, I32, I32, P],
    'sgs_tracker_step_rgbd': [P, P, P, Z, I32, P, Z, I32, P, I32, P] + [P] * 8 + [F32, I32, I32] + [P] * 11,
    'sgs_tracker_frame_device': [P, P, P],
}


def test_rgbd_entry_points_are_exported_and_typed():
    L = B.lib()
    out = subprocess.check_output(['nm', '-D', '--defined-only', B.build()], text=True)
    exported = {l.split()[-1] for l in out.splitlines() if ' T ' in l}
    for name, args in NEW.items():
        assert name in exported and name in B.ABI_SYMBOLS, name
        assert B._SIGNATURES[name] == (C.c_int, args) and getattr(L, name).argtypes == args, name


def test_rgbd_format_from_settings():
    s = B.Settings(k1=0.262383, k2=-0.953104, p1=-0.005358, p2=0.002628, k3=1.163314, rgb=1, depth_map_factor=np.float32(1 / 5000))
    f = B.rgbd_format(s)
    assert (f.rgb, f.depth_type) == (1, B.DEPTH_U16) and f.depth_map_factor == s.depth_map_factor
    assert list(f.dist_coef) == [s.k1, s.k2, s.p1, s.p2, s.k3]


def test_colour_s2_stream():
    rgb, depth, boxes = synth.stream_s2_rgbd(3, 96, 64, seed=4, tex_w=160, tex_h=120, person=False)
    rgb2, depth2, _ = synth.stream_s2_rgbd(3, 96, 64, seed=4, tex_w=160, tex_h=120, person=False)
    assert np.array_equal(rgb, rgb2) and np.array_equal(depth, depth2)
    assert rgb.shape == (3, 64, 96, 3) and depth.dtype == np.uint16 and depth.shape == (3, 64, 96)
    assert not np.array_equal(rgb[..., 0], rgb[..., 1]) and not np.array_equal(GR.to_gray(rgb, 1), GR.to_gray(rgb, 0))
    assert np.array_equal(depth[1], np.rint(synth.depth_s1(96, 64).astype(np.float64) * 5000).astype(np.uint16))
