"""The constructed extractor cases of tests/orb_cases.py against the REFERENCE'S OWN src/ORBextractor.cc (no device): for every case the
oracle's keypoints equal the reference's field for field and its descriptors byte for byte (the reference run on the monotone allocator,
quirk Q1), and the case's proof holds on the oracle's per-stage output.

Without the reference tree the comparison runs against tests/golden/orbextractor_cases.npz (written from the reference by
tests/golden/make_golden_orbextractor_cases.py): per case the keypoint count and SHA-256 digests of the keypoint and descriptor bytes."""
import os

import numpy as np
import pytest

import oracle as O
import orb_cases as OC
import test_orbextractor_ref as R

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'orbextractor_cases.npz')
CASES = OC.all_cases()
_golden = None


def golden():
    global _golden
    if _golden is None:
        _golden = dict(np.load(GOLDEN))
    return _golden


def reference(c):
    p = c['p']
    return R.ref_extract(c['img'], nfeatures=p['nfeatures'], scale=p['scale'], nlevels=p['nlevels'], ini=p['ini'], mn=p['mn'])


@pytest.mark.parametrize('c', CASES, ids=[c['name'] for c in CASES])
def test_case_against_reference(c):
    d = O.ExtractDump(c['img'], OC.oparams(c['p']))
    c['proof'](d)
    if R.HAVE_REF:
        kr, dr = reference(c)
        assert len(kr) == len(d.kps), (len(kr), len(d.kps))
        for f in O.KP_DTYPE.names:
            assert np.array_equal(kr[f].view(np.uint32), d.kps[f].view(np.uint32)), f
        assert kr.tobytes() == d.kps.tobytes()
        assert np.array_equal(dr, d.desc)
    else:
        ref = golden()[c['name']]
        assert ref[0] == len(d.kps), (ref[0], len(d.kps))
        assert np.array_equal(R.digest(d.kps, d.desc), ref), 'keypoints / descriptors differ from the reference\'s'


def test_golden_covers_every_case():
    """The digests were written from the same images: a builder change that alters a case must come with new digests."""
    g = golden()
    assert sorted(g) == sorted(['img_' + c['name'] for c in CASES] + [c['name'] for c in CASES])
    for c in CASES:
        assert int(g['img_' + c['name']][0]) == int(R.call_key(c['img'], **c['p'])[:15], 16), c['name']


def test_plan_limits_restated():
    """The nfeatures limit of the shared-memory quadtree at 640 x 480 with one level, from the plan formulas: 1393 accepted, 1394 refused;
    and the key capacity bands the count cases use."""
    assert OC.max_nfeatures(640, 480, OC.P(nlevels=1)) == 1393
    assert [OC.smem_key_cap(640, 480, OC.P(nfeatures=n)) for n in (300, 500, 1000)] == [4096, 2048, 1024]
