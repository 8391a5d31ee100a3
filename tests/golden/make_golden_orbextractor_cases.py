"""Writes tests/golden/orbextractor_cases.npz from the reference's own ORBextractor.cc (oracle/_ref/liborbextractor_ref.so, built by build() when
the reference tree is present): for every case of tests/orb_cases.py the reference's keypoint count and digests of its keypoint and descriptor
bytes, and a digest of the case's image and parameters.  Run from the repository root: python tests/golden/make_golden_orbextractor_cases.py"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle'), os.path.join(ROOT, 'sg-slam_b200')]
import orb_cases as OC  # noqa: E402
import test_orbextractor_ref as T  # noqa: E402

assert T.HAVE_REF, T.LIB + ' not built'
out = {}
for c in OC.all_cases():
    p = c['p']
    k, d = T.ref_extract(c['img'], nfeatures=p['nfeatures'], scale=p['scale'], nlevels=p['nlevels'], ini=p['ini'], mn=p['mn'])
    out[c['name']] = T.digest(k, d)
    out['img_' + c['name']] = np.array([int(T.call_key(c['img'], **p)[:15], 16)], np.int64)
np.savez_compressed(os.path.join(ROOT, 'tests', 'golden', 'orbextractor_cases.npz'), **out)
print('%d entries' % len(out))
