"""Writes tests/golden/orbextractor_ref.npz from the reference's own ORBextractor.cc (oracle/_ref/liborbextractor_ref.so, built by build() when the reference
tree is present): for every call tests/test_orbextractor_ref.py compares, the reference's keypoint count and digests of its keypoint and descriptor bytes, and
the (x, y, octave) of the address-order run.  Run from the repository root: python tests/golden/make_golden_orbextractor_ref.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'sg-slam_b200')]
import test_orbextractor_ref as T  # noqa: E402

assert T.HAVE_REF, T.LIB + ' not built'
out = {}


def record(img, **kw):
    k, d = T.ref_extract(img, **kw)
    out['same_' + T.call_key(img, **kw)] = T.digest(k, d)
    return len(k)


T.same = record                                   # every comparison of the test module now records the reference's side
T.test_s2_stream_frames()
for w, h, nf in [(640, 480, 1000), (1280, 720, 2000), (321, 243, 500), (752, 480, 1200)]:
    T.test_other_geometries(w, h, nf)
T.test_other_parameters()
T.test_degenerate_images()
from pysgs import synth  # noqa: E402
frames, _ = synth.stream_s2(3, 640, 480, seed=3)
for i, p in enumerate(T.address_order_points(frames)):
    out['address_order_%d' % i] = p.astype(np.float32)
np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'orbextractor_ref.npz'), **out)
print('%d entries' % len(out))
