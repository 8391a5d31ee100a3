"""The host-pointer entry points (the single-frame calls the mirror headers make) up to the point where they reach the device:
argument checks, the outputs written before an early return, and the status codes.  No GPU needed; the calls that would reach a
device are checked to fail with SGS_ERR_CUDA only where there is none."""
import ctypes as C

import numpy as np
import pytest

from pysgs import binding as B

v = C.c_void_p


def _p(a):
    return a.ctypes.data_as(v)


def _skip_on_a_device():
    n = C.c_int(-1)
    if B.lib().sgs_device_count(C.byref(n)) == 0 and n.value > 0:
        pytest.skip('a CUDA device is present')


def _view(n):
    """A frame of n keypoints (arrays kept alive on the view)."""
    fv = B.FrameView()
    fv._a = (_z(n, B.KP_DTYPE), _z(n, np.float32), _z(n, np.uint8, (32,)), (1.2 ** np.arange(8)).astype(np.float32))
    fv.n = n
    fv.keys_un, fv.u_right, fv.desc = (a.ctypes.data for a in fv._a[:3])
    fv.max_x, fv.max_y, fv.fx, fv.fy, fv.cx, fv.cy, fv.bf = 640.0, 480.0, 500.0, 500.0, 320.0, 240.0, 40.0
    fv.nlevels, fv.scale_factors = 8, fv._a[3].ctypes.data
    return fv


def _z(n, dt, shape=()):
    return np.zeros((max(n, 0),) + shape, dt)


def _f(n, value, dt=np.int32):
    return np.full(max(n, 0), value, dt)


T = np.eye(4, dtype=np.float32).reshape(16)


def lastframe(ncur=3, nlast=4, drop=None):
    a = dict(has=_z(nlast, np.uint8), xyz=_z(nlast, np.float32, (3,)), desc=_z(nlast, np.uint8, (32,)), obs=_z(nlast, np.uint8), oct=_z(nlast, np.int32),
             ang=_z(nlast, np.float32), mp=_f(ncur, -1, np.int32))
    nm = C.c_int(-5)
    P = {k: (None if k == drop else _p(x)) for k, x in a.items()}
    rc = B.lib().sgs_match_project_lastframe(C.byref(_view(ncur)), _p(T), _p(T), nlast, P['has'], P['xyz'], P['desc'], P['obs'], P['oct'], P['ang'],
                                             15.0, 0, 1, P['mp'], None, C.byref(nm), 0)
    return rc, dict(nmatches=nm.value)


def keyframe(ncur=3, nkf=4, drop=None):
    a = dict(valid=_z(nkf, np.uint8), xyz=_z(nkf, np.float32, (3,)), desc=_z(nkf, np.uint8, (32,)), ang=_z(nkf, np.float32), mn=_z(nkf, np.float32),
             mx=_z(nkf, np.float32), mp=_f(ncur, -1, np.int32))
    nm = C.c_int(-5)
    P = {k: (None if k == drop else _p(x)) for k, x in a.items()}
    rc = B.lib().sgs_match_project_keyframe(C.byref(_view(ncur)), _p(T), nkf, P['valid'], P['xyz'], P['desc'], P['ang'], P['mn'], P['mx'], 10.0, 100, 1,
                                            P['mp'], C.byref(nm), 0)
    return rc, dict(nmatches=nm.value)


def localmap(ncur=3, nmp=4, drop=None):
    a = dict(inview=_z(nmp, np.uint8), px=_z(nmp, np.float32), py=_z(nmp, np.float32), pxr=_z(nmp, np.float32), lvl=_z(nmp, np.int32), vc=_z(nmp, np.float32),
             desc=_z(nmp, np.uint8, (32,)), obs=_z(nmp, np.uint8), mp=_f(ncur, -1, np.int32), mpo=_z(ncur, np.uint8))
    nm = C.c_int(-5)
    P = {k: (None if k == drop else _p(x)) for k, x in a.items()}
    rc = B.lib().sgs_match_project_localmap(C.byref(_view(ncur)), nmp, P['inview'], P['px'], P['py'], P['pxr'], P['lvl'], P['vc'], P['desc'], P['obs'],
                                            1.0, 0.8, 0, P['mp'], P['mpo'], C.byref(nm), 0)
    return rc, dict(nmatches=nm.value)


def fuse(nkf=3, nmp=4, drop=None):
    a = dict(valid=_z(nmp, np.uint8), xyz=_z(nmp, np.float32, (3,)), nrm=_z(nmp, np.float32, (3,)), mn=_z(nmp, np.float32), mx=_z(nmp, np.float32),
             desc=_z(nmp, np.uint8, (32,)), s2=np.ones(8, np.float32))
    bi = _f(nmp, 7, np.int32); bd = _f(nmp, 7, np.int32); nm = C.c_int(-5)
    P = {k: (None if k == drop else _p(x)) for k, x in a.items()}
    rc = B.lib().sgs_fuse_search(C.byref(_view(nkf)), _p(T), _p(np.zeros(3, np.float32)), nmp, P['valid'], P['xyz'], P['nrm'], P['mn'], P['mx'], P['desc'],
                                 3.0, P['s2'], 0, None, _p(bi), _p(bd), None, C.byref(nm), 0)
    return rc, dict(nmatches=nm.value, best_idx=bi, best_dist=bd)


def init(n1=3, n2=4, drop=None):
    a = dict(prev=_z(n1, np.float32, (2,)), m12=_f(n1, 7, np.int32))
    nm = C.c_int(-5)
    P = {k: (None if k == drop else _p(x)) for k, x in a.items()}
    rc = B.lib().sgs_search_for_initialization(C.byref(_view(n1)), C.byref(_view(n2)), P['prev'], 100, 0.9, 1, P['m12'], C.byref(nm), 0)
    return rc, dict(nmatches=nm.value, match12=a['m12'])


def bow_keyframes(n1=3, n2=4, drop=None, mode=1):
    a = dict(node1=_z(n1, np.int32), w1=_z(n1, np.float64), v1=_z(n1, np.uint8), d1=_z(n1, np.uint8, (32,)), a1=_z(n1, np.float32),
             node2=_z(n2, np.int32), w2=_z(n2, np.float64), v2=_z(n2, np.uint8), d2=_z(n2, np.uint8, (32,)), a2=_z(n2, np.float32), m12=_f(n1, 7, np.int32))
    nm = C.c_int(-5)
    P = {k: (None if k == drop else _p(x)) for k, x in a.items()}
    rc = B.lib().sgs_match_bow_keyframes(mode, n1, P['node1'], P['w1'], P['v1'], P['d1'], P['a1'], n2, P['node2'], P['w2'], P['v2'], P['d2'], P['a2'],
                                         0.75, 1, None, None, None, None, None, None, None, None, None, 8, 0, P['m12'], C.byref(nm), 0)
    return rc, dict(nmatches=nm.value, match12=a['m12'])


def match_bow(nkf=3, nf=4, drop=None):
    a = dict(kn=_z(nkf, np.int32), kw=_z(nkf, np.float64), kv=_z(nkf, np.uint8), kd=_z(nkf, np.uint8, (32,)), ka=_z(nkf, np.float32),
             fn=_z(nf, np.int32), fw=_z(nf, np.float64), fd=_z(nf, np.uint8, (32,)), fa=_z(nf, np.float32), mf=_f(nf, 7, np.int32))
    nm = C.c_int(-5)
    P = {k: (None if k == drop else _p(x)) for k, x in a.items()}
    rc = B.lib().sgs_match_bow(nkf, P['kn'], P['kw'], P['kv'], P['kd'], P['ka'], nf, P['fn'], P['fw'], P['fd'], P['fa'], 0.7, 1, P['mf'], C.byref(nm), 0)
    return rc, dict(nmatches=nm.value, match_f=a['mf'])


def hamming_pairs(n=4, drop=None):
    a = dict(a=_z(n, np.uint8, (32,)), b=_z(n, np.uint8, (32,)), dist=_z(n, np.int32))
    P = {k: (None if k == drop else _p(x)) for k, x in a.items()}
    return B.lib().sgs_hamming_pairs(P['a'], P['b'], n, P['dist'], 0), {}


def hamming_bf(nq=4, nt=4, drop=None):
    a = dict(q=_z(nq, np.uint8, (32,)), t=_z(nt, np.uint8, (32,)), bi=_z(nq, np.int32), bd=_z(nq, np.int32), sd=_z(nq, np.int32))
    P = {k: (None if k == drop else _p(x)) for k, x in a.items()}
    return B.lib().sgs_hamming_bf(P['q'], nq, P['t'], nt, P['bi'], P['bd'], P['sd'], 0), {}


def undistort(n=4, drop=None):
    a = dict(xy=_z(n, np.float32, (2,)), k=np.array([0.1, 0, 0, 0, 0], np.float32), out=_z(n, np.float32, (2,)))
    P = {k: (None if k == drop else _p(x)) for k, x in a.items()}
    return B.lib().sgs_undistort_points(P['xy'], n, 500, 500, 320, 240, P['k'], P['out'], 0), {}


def frustum(n=4, drop=None):
    cam = B.make_camera(640, 480, dict(fx=500.0, fy=500.0, cx=320.0, cy=240.0, bf=40.0), 1.2 ** np.arange(8))
    a = dict(cam=None, xyz=_z(n, np.float32, (3,)), nrm=_z(n, np.float32, (3,)), mn=_z(n, np.float32), mx=_z(n, np.float32), iv=_z(n, np.uint8),
             px=_z(n, np.float32), py=_z(n, np.float32), pxr=_z(n, np.float32), lvl=_z(n, np.int32), vc=_z(n, np.float32))
    P = {k: (None if k == drop else (C.byref(cam) if k == 'cam' else _p(x))) for k, x in a.items()}
    rc = B.lib().sgs_frustum(P['cam'], _p(T), n, P['xyz'], P['nrm'], P['mn'], P['mx'], 0.5, P['iv'], P['px'], P['py'], P['pxr'], P['lvl'], P['vc'], 0)
    return rc, {}


def pose(n=4, drop=None):
    cam = B.make_camera(640, 480, dict(fx=500.0, fy=500.0, cx=320.0, cy=240.0, bf=40.0), 1.2 ** np.arange(8))
    tin = (np.arange(16) + 0.5).astype(np.float32)
    a = dict(cam=None, kps=_z(n, B.KP_DTYPE), ur=_z(n, np.float32), has=_z(n, np.uint8), xyz=_z(n, np.float32, (3,)), s2=np.ones(16, np.float32),
             out=_f(n, 7, np.uint8))
    tout = _f(16, -3, np.float32); nin = C.c_int(-5)
    P = {k: (None if k == drop else (C.byref(cam) if k == 'cam' else _p(x))) for k, x in a.items()}
    rc = B.lib().sgs_pose_optimization(P['cam'], _p(tin), n, P['kps'], P['ur'], P['has'], P['xyz'], P['s2'], _p(tout), P['out'], C.byref(nin), 0)
    return rc, dict(tcw_out=tout, tcw_in=tin, ninliers=nin.value)


def dynreject(n=4, drop=None):
    a = dict(cur=_z(n, np.float32, (2,)), prev=_z(n, np.float32, (2,)), keep=_z(n, np.uint8))
    nk, rest = C.c_int(-5), C.c_int(-5)
    P = {k: (None if k == drop else _p(x)) for k, x in a.items()}
    rc = B.lib().sgs_dynreject(P['cur'], P['prev'], n, None, None, 0, 0, 1000, P['keep'], None, C.byref(nk), C.byref(rest), 0)
    return rc, dict(nkeep=nk.value, restored=rest.value)


def fundamental(n=8, drop=None):
    a = dict(p1=_z(n, np.float32, (2,)), p2=_z(n, np.float32, (2,)), F=_z(9, np.float64))
    P = {k: (None if k == drop else _p(x)) for k, x in a.items()}
    return B.lib().sgs_fundamental_ransac(P['p1'], P['p2'], n, 1.0, 0.99, 200, P['F'], None, None, 0), {}


def _invalid(name, rc):
    assert rc == B.SGS_ERR_INVALID, (name, rc)
    assert B.lib().sgs_last_error().decode().startswith(name), B.lib().sgs_last_error()


# (entry point, call, sizes of a call that would reach the device, a NULL array it must reject, a negative size it must reject)
CASES = [
    ('sgs_match_project_lastframe', lastframe, dict(ncur=3, nlast=4), 'xyz', dict(nlast=-1)),
    ('sgs_match_project_keyframe', keyframe, dict(ncur=3, nkf=4), 'mx', dict(nkf=-1)),
    ('sgs_match_project_localmap', localmap, dict(ncur=3, nmp=4), 'mpo', dict(nmp=-1)),
    ('sgs_fuse_search', fuse, dict(nkf=3, nmp=4), 'desc', dict(nmp=-1)),
    ('sgs_search_for_initialization', init, dict(n1=3, n2=4), 'prev', dict(n2=-1)),
    ('sgs_match_bow_keyframes', bow_keyframes, dict(n1=3, n2=4), 'a2', dict(n1=-1)),
    ('sgs_match_bow', match_bow, dict(nkf=3, nf=4), 'kv', dict(nf=-1)),
    ('sgs_hamming_pairs', hamming_pairs, dict(n=4), 'b', dict(n=-1)),
    ('sgs_hamming_bf', hamming_bf, dict(nq=4, nt=4), 'q', dict(nt=-1)),
    ('sgs_undistort_points', undistort, dict(n=4), 'k', dict(n=-1)),
    ('sgs_frustum', frustum, dict(n=4), 'cam', dict(n=-1)),
    ('sgs_pose_optimization', pose, dict(n=4), 'xyz', dict(n=-1)),
    ('sgs_dynreject', dynreject, dict(n=4), 'keep', dict(n=-1)),
    ('sgs_fundamental_ransac', fundamental, dict(n=8), 'p2', dict(n=0)),
]


@pytest.mark.parametrize('name,call,sizes,null,negative', CASES, ids=[c[0] for c in CASES])
def test_bad_arguments_are_rejected_by_name(name, call, sizes, null, negative):
    _invalid(name, call(**sizes, drop=null)[0])
    _invalid(name, call(**negative)[0])


def test_bow_entry_points_reject_bad_arguments():
    _invalid('sgs_match_bow_keyframes', bow_keyframes(mode=3)[0])
    _invalid('sgs_bow_transform', B.lib().sgs_bow_transform(None, None, 0, 1, None, None, None))


# (entry point, call, sizes with an empty side)
EMPTY = [
    ('sgs_match_project_lastframe', lastframe, [dict(ncur=0), dict(nlast=0)]),
    ('sgs_match_project_keyframe', keyframe, [dict(ncur=0), dict(nkf=0)]),
    ('sgs_match_project_localmap', localmap, [dict(ncur=0), dict(nmp=0)]),
    ('sgs_fuse_search', fuse, [dict(nkf=0), dict(nmp=0)]),
    ('sgs_search_for_initialization', init, [dict(n1=0), dict(n2=0)]),
    ('sgs_match_bow_keyframes', bow_keyframes, [dict(n1=0), dict(n2=0), dict(n2=0, mode=2)]),
    ('sgs_match_bow', match_bow, [dict(nkf=0), dict(nf=0)]),
    ('sgs_hamming_pairs', hamming_pairs, [dict(n=0)]),
    ('sgs_hamming_bf', hamming_bf, [dict(nq=0), dict(nq=0, nt=0)]),
    ('sgs_undistort_points', undistort, [dict(n=0)]),
    ('sgs_frustum', frustum, [dict(n=0)]),
    ('sgs_pose_optimization', pose, [dict(n=0)]),
]


@pytest.mark.parametrize('name,call,sizes', EMPTY, ids=[c[0] for c in EMPTY])
def test_empty_inputs_return_initial_outputs_without_a_device(name, call, sizes):
    for sz in sizes:
        rc, out = call(**sz)
        assert rc == B.SGS_OK, (name, sz, rc, B.lib().sgs_last_error())
        if 'nmatches' in out:
            assert out['nmatches'] == 0, (name, sz)
        for k in ('match12', 'match_f'):
            if k in out:
                assert (out[k] == -1).all(), (name, sz, out[k])
        if name == 'sgs_fuse_search':
            assert (out['best_idx'] == -1).all() and (out['best_dist'] == 256).all(), sz
        if name == 'sgs_pose_optimization':
            assert out['tcw_out'].tobytes() == out['tcw_in'].tobytes() and out['ninliers'] == 0


def test_projection_matchers_reject_more_than_8192_keypoints():
    for call, sz in ((lastframe, dict(nlast=4)), (keyframe, dict(nkf=4)), (localmap, dict(nmp=4))):
        rc, out = call(ncur=8193, **sz)
        assert rc == B.SGS_ERR_UNSUPPORTED, (call.__name__, rc)
        assert out['nmatches'] == 0


@pytest.mark.parametrize('name,call,sizes,null,negative', CASES, ids=[c[0] for c in CASES])
def test_first_device_call_fails_without_a_device(name, call, sizes, null, negative):
    _skip_on_a_device()
    rc, out = call(**sizes)
    assert rc == B.SGS_ERR_CUDA, (name, rc)
    if 'nmatches' in out:
        assert out['nmatches'] == 0


def test_dynreject_selects_the_device_even_when_empty():
    _skip_on_a_device()
    rc, out = dynreject(n=0)
    assert rc == B.SGS_ERR_CUDA
    assert out['nkeep'] == 0 and out['restored'] == 0
    rc, out = dynreject(n=4)
    assert rc == B.SGS_ERR_CUDA and out['nkeep'] == 4 and out['restored'] == 0           # written before the device is selected
