"""The constructed matcher cases of tests/match_cases.py through the BATCHED device entry points, every case one frame of a launch.

Each launch groups the cases that share the per-launch scalars and the camera (th, ratio, orientation check, image bounds) and adds a frame
with n = 0 and a frame without points; the last-frame launch also carries a disabled frame (frame_enable = 0).  Capacities are the largest
keypoint count + 37 and the largest point count + 11; the rows past each frame's counts hold copies of its data (what a kernel reading past
a count would pick up), every output row starts as a sentinel and ncand starts at zero.  Required: every enabled frame equals the oracle
and the reference's own ORBmatcher.cc exactly, the device ncand equals the oracle's |vIndices| count, the case's path proof holds, and the
disabled frame and every padding row still hold their sentinels.  The host-pointer wrappers (cur_cap == n) give the same results, a second
identical launch gives identical bytes, and the 8192-keypoint limit of the shared-memory grid is checked on both sides."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import match_cases as MC  # noqa: E402
import oracle as O  # noqa: E402
import scenarios as S  # noqa: E402
import test_orbmatcher_ref as TR  # noqa: E402
from pysgs import binding as B  # noqa: E402

SENT = np.int32(0x5A5A5A5A)
SENT_U8 = np.uint8(0xA5)
SENT_F = np.float32(-12345.5)
EXTRA_KP, EXTRA_PT = 37, 11
V = C.c_void_p


def _groups(kind):
    """The cases of `kind` split by launch: same params and same image bounds."""
    out = {}
    for n in MC.names(kind):
        c = MC.CASES[n]
        out.setdefault((tuple(sorted(c['params'].items())), c['bounds']), []).append(n)
    return list(out.values())


def _ids(groups):
    return ['%s+%d' % (g[0], len(g) - 1) for g in groups]


def _pad(rows, cap, fill=None):
    """[cap, ...]: `rows`, then `fill`, or without a fill the rows repeated."""
    rows = np.asarray(rows)
    out = np.zeros((cap,) + rows.shape[1:], rows.dtype)
    out[:len(rows)] = rows
    if fill is not None:
        out[len(rows):] = fill
    elif len(rows):
        out[len(rows):] = rows[np.arange(cap - len(rows)) % len(rows)]
    return out


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _host(t):
    import torch
    torch.cuda.synchronize()
    return t.cpu().numpy()


def _frames(names, disabled=False):
    """Frame specs of one launch: the cases, then one with n = 0, one without points, and optionally a disabled copy of the first case."""
    cs = [MC.CASES[n] for n in names]
    fr = [dict(case=c, n=None, m=None, enable=1) for c in cs]
    fr += [dict(case=cs[0], n=0, m=None, enable=1), dict(case=cs[0], n=None, m=0, enable=1)]
    if disabled:
        fr.append(dict(case=cs[0], n=None, m=None, enable=0))
    return fr


def _counts(f, n_all, m_all):
    return (n_all if f['n'] is None else f['n']), (m_all if f['m'] is None else f['m'])


def _reference(c):
    return TR.ref_case(TR._lib(), c) if os.path.exists(TR.LIB) else None


def _check_frame(f, n, m, got, oracle_key, out_key, inp, sent, nm, ncand=None):
    """One frame's output rows against the oracle / reference (or, for a frame that cannot match, against its input) and its padding."""
    c = f['case']
    if f['enable'] and n and m:
        o = MC.run_oracle(c)
        assert np.array_equal(got[:n], o[oracle_key]), (c['name'], out_key, got[:n], o[oracle_key])
        assert nm == o['nm'], (c['name'], nm, o['nm'])
        if ncand is not None:
            assert ncand == o['ncand'], (c['name'], ncand, o['ncand'])
        r = _reference(c)
        if r is not None:
            assert np.array_equal(got[:n], r[oracle_key]) and nm == r['nm'], c['name']
        c['proof'](o)
    else:
        assert np.array_equal(got[:n], inp[:n]), (c['name'], out_key)
        assert nm == (0 if f['enable'] else SENT) and (ncand is None or ncand == 0), (c['name'], nm, ncand)
    assert (got[n:] == sent).all(), (c['name'], out_key, 'padding row written')


# ---- SearchByProjection(Frame&, const Frame&) ----------------------------------------------------------------------------------------
def _run_last(names):
    fr = _frames(names, disabled=True)
    cs = [f['case'] for f in fr]
    F = len(fr)
    cap = max(len(c['kps']) for c in cs) + EXTRA_KP
    pcap = max(len(c['last_has']) for c in cs) + EXTRA_PT
    p = cs[0]['params']
    ns = [_counts(f, len(f['case']['kps']), len(f['case']['last_has'])) for f in fr]
    mp_in = np.stack([_pad(f['case']['cur_mp'][:n], cap, SENT) if f['enable'] else np.full(cap, SENT) for f, (n, _) in zip(fr, ns)])
    obs_in = np.stack([_pad(c['cur_obs'] if c['cur_obs'] is not None else np.ones(len(c['kps']), np.uint8), cap) for c in cs])
    flags = [c['last_has'] | (c['last_obs'] << 1) for c in cs]
    t = dict(kps=_dev(np.stack([_pad(c['kps'], cap) for c in cs]).view(np.uint8).reshape(-1)), desc=_dev(np.stack([_pad(c['desc'], cap) for c in cs])),
             ur=_dev(np.stack([_pad(c['uright'], cap) for c in cs])), n=_dev(np.array([n for n, _ in ns], np.int32)),
             xyz=_dev(np.stack([_pad(c['last_xyz'], pcap) for c in cs])), ld=_dev(np.stack([_pad(c['last_desc'], pcap) for c in cs])),
             fl=_dev(np.stack([_pad(x, pcap) for x in flags])), oct=_dev(np.stack([_pad(c['last_oct'], pcap) for c in cs])),
             ang=_dev(np.stack([_pad(c['last_angle'], pcap) for c in cs])), m=_dev(np.array([m for _, m in ns], np.int32)),
             tc=_dev(np.stack([c['Tcw_cur'].reshape(16) for c in cs])), tl=_dev(np.stack([c['Tcw_last'].reshape(16) for c in cs])),
             mp=_dev(mp_in), obs=_dev(obs_in), nm=_dev(np.full(F, SENT)), nc=_dev(np.zeros(F, np.uint64)),
             en=_dev(np.array([f['enable'] for f in fr], np.uint8)))
    a = B.LastFrameBatch()
    a.cam = B.make_camera(MC.W, MC.H, MC.CAM, MC.SF, bounds=cs[0]['bounds'])
    a.cur_kps, a.cur_desc, a.cur_uright, a.cur_n = t['kps'].data_ptr(), t['desc'].data_ptr(), t['ur'].data_ptr(), t['n'].data_ptr()
    a.last_xyz, a.last_desc, a.last_flags, a.last_octave = t['xyz'].data_ptr(), t['ld'].data_ptr(), t['fl'].data_ptr(), t['oct'].data_ptr()
    a.last_angle, a.last_n, a.tcw_cur, a.tcw_last = t['ang'].data_ptr(), t['m'].data_ptr(), t['tc'].data_ptr(), t['tl'].data_ptr()
    a.th, a.mono, a.check_orientation = p['th'], int(p['mono']), int(p['check_ori'])
    a.cur_mp, a.cur_mp_obs_in, a.nmatches, a.ncand, a.frame_enable = t['mp'].data_ptr(), t['obs'].data_ptr(), t['nm'].data_ptr(), t['nc'].data_ptr(), t['en'].data_ptr()
    mt = B.Matcher(F, cap, pcap)
    mt.lastframe_batch(a, F)
    out = dict(mp=_host(t['mp']), nm=_host(t['nm']), nc=_host(t['nc']))
    mt.close()
    return fr, ns, mp_in, out


@pytest.mark.parametrize('names', _groups('last'), ids=_ids(_groups('last')))
def test_lastframe_batch(names):
    fr, ns, mp_in, out = _run_last(names)
    for k, (f, (n, m)) in enumerate(zip(fr, ns)):
        _check_frame(f, n, m, out['mp'][k], 'mp', 'cur_mp', mp_in[k], SENT, out['nm'][k], int(out['nc'][k]))
    _, _, _, again = _run_last(names)
    assert all(again[k].tobytes() == out[k].tobytes() for k in out)
    for n in names:                                   # the host-pointer wrapper: one frame, cur_cap == n
        c = MC.CASES[n]; p = c['params']; o = MC.run_oracle(c)
        fg = B.HostFrame(c['kps'], c['uright'], c['desc'], MC.W, MC.H, MC.CAM['fx'], MC.CAM['fy'], MC.CAM['cx'], MC.CAM['cy'], MC.CAM['bf'], MC.SF, bounds=c['bounds'])
        nm, mp = B.match_project_lastframe(fg, c['Tcw_cur'], c['Tcw_last'], c['last_has'], c['last_xyz'], c['last_desc'], c['last_obs'], c['last_oct'],
                                           c['last_angle'], p['th'], mono=p['mono'], check_ori=p['check_ori'], cur_mp=c['cur_mp'], cur_mp_obs=c['cur_obs'])
        assert nm == o['nm'] and np.array_equal(mp, o['mp']), n


# ---- SearchByProjection(Frame&, KeyFrame*, sAlreadyFound, th, ORBdist) ---------------------------------------------------------------
def _run_kf(names):
    fr = _frames(names)
    cs = [f['case'] for f in fr]
    F = len(fr)
    cap = max(len(c['kps']) for c in cs) + EXTRA_KP
    pcap = max(len(c['kf_valid']) for c in cs) + EXTRA_PT
    p = cs[0]['params']
    ns = [_counts(f, len(f['case']['kps']), len(f['case']['kf_valid'])) for f in fr]
    mp_in = np.stack([_pad(f['case']['cur_mp'][:n], cap, SENT) for f, (n, _) in zip(fr, ns)])
    t = dict(kps=_dev(np.stack([_pad(c['kps'], cap) for c in cs]).view(np.uint8).reshape(-1)), desc=_dev(np.stack([_pad(c['desc'], cap) for c in cs])),
             ur=_dev(np.stack([_pad(c['uright'], cap) for c in cs])), n=_dev(np.array([n for n, _ in ns], np.int32)),
             xyz=_dev(np.stack([_pad(c['last_xyz'], pcap) for c in cs])), kd=_dev(np.stack([_pad(c['last_desc'], pcap) for c in cs])),
             kv=_dev(np.stack([_pad(c['kf_valid'], pcap) for c in cs])), ang=_dev(np.stack([_pad(c['last_angle'], pcap) for c in cs])),
             mn=_dev(np.stack([_pad(c['min_dist'], pcap) for c in cs])), mx=_dev(np.stack([_pad(c['max_dist'], pcap) for c in cs])),
             m=_dev(np.array([m for _, m in ns], np.int32)), tc=_dev(np.stack([c['Tcw_cur'].reshape(16) for c in cs])),
             mp=_dev(mp_in), nm=_dev(np.full(F, SENT)), nc=_dev(np.zeros(F, np.uint64)))
    a = B.KeyFrameBatch()
    a.cam = B.make_camera(MC.W, MC.H, MC.CAM, MC.SF, bounds=cs[0]['bounds'])
    a.cur_kps, a.cur_desc, a.cur_uright, a.cur_n = t['kps'].data_ptr(), t['desc'].data_ptr(), t['ur'].data_ptr(), t['n'].data_ptr()
    a.kf_xyz, a.kf_desc, a.kf_valid, a.kf_angle = t['xyz'].data_ptr(), t['kd'].data_ptr(), t['kv'].data_ptr(), t['ang'].data_ptr()
    a.kf_min_dist, a.kf_max_dist, a.kf_n, a.tcw_cur = t['mn'].data_ptr(), t['mx'].data_ptr(), t['m'].data_ptr(), t['tc'].data_ptr()
    a.th, a.orb_dist, a.check_orientation = p['th'], p['orb_dist'], int(p['check_ori'])
    a.cur_mp, a.nmatches, a.ncand = t['mp'].data_ptr(), t['nm'].data_ptr(), t['nc'].data_ptr()
    mt = B.Matcher(F, cap, pcap)
    B.check(B.lib().sgs_match_project_keyframe_batch_device(mt.h, C.byref(a), F, V(0)))
    out = dict(mp=_host(t['mp']), nm=_host(t['nm']), nc=_host(t['nc']))
    mt.close()
    return fr, ns, mp_in, out


@pytest.mark.parametrize('names', _groups('kf'), ids=_ids(_groups('kf')))
def test_keyframe_batch(names):
    fr, ns, mp_in, out = _run_kf(names)
    for k, (f, (n, m)) in enumerate(zip(fr, ns)):
        _check_frame(f, n, m, out['mp'][k], 'mp', 'cur_mp', mp_in[k], SENT, out['nm'][k], int(out['nc'][k]))
    _, _, _, again = _run_kf(names)
    assert all(again[k].tobytes() == out[k].tobytes() for k in out)
    for n in names:
        c = MC.CASES[n]; p = c['params']; o = MC.run_oracle(c)
        fg = B.HostFrame(c['kps'], c['uright'], c['desc'], MC.W, MC.H, MC.CAM['fx'], MC.CAM['fy'], MC.CAM['cx'], MC.CAM['cy'], MC.CAM['bf'], MC.SF, bounds=c['bounds'])
        nm, mp = B.match_project_keyframe(fg, c['Tcw_cur'], c['kf_valid'], c['last_xyz'], c['last_desc'], c['last_angle'], c['min_dist'], c['max_dist'],
                                          p['th'], p['orb_dist'], p['check_ori'], c['cur_mp'])
        assert nm == o['nm'] and np.array_equal(mp, o['mp']), n


# ---- SearchByProjection(Frame&, vector<MapPoint*>&, th) -------------------------------------------------------------------------------
def _run_local(names):
    fr = _frames(names)
    cs = [f['case'] for f in fr]
    F = len(fr)
    cap = max(len(c['kps']) for c in cs) + EXTRA_KP
    pcap = max(len(c['inview']) for c in cs) + EXTRA_PT
    p = cs[0]['params']
    ns = [_counts(f, len(f['case']['kps']), len(f['case']['inview'])) for f in fr]
    mp_in = np.stack([_pad(f['case']['f_mp'][:n], cap, SENT) for f, (n, _) in zip(fr, ns)])
    ob_in = np.stack([_pad(f['case']['f_obs'][:n], cap, SENT_U8) for f, (n, _) in zip(fr, ns)])
    pts = lambda key: _dev(np.stack([_pad(c[key], pcap) for c in cs]))
    t = dict(kps=_dev(np.stack([_pad(c['kps'], cap) for c in cs]).view(np.uint8).reshape(-1)), desc=_dev(np.stack([_pad(c['desc'], cap) for c in cs])),
             ur=_dev(np.stack([_pad(c['uright'], cap) for c in cs])), n=_dev(np.array([n for n, _ in ns], np.int32)),
             iv=pts('inview'), px=pts('projx'), py=pts('projy'), pr=pts('projxr'), lv=pts('level'), vc=pts('viewcos'), md=pts('mp_desc'), mo=pts('mp_obs'),
             m=_dev(np.array([m for _, m in ns], np.int32)), mp=_dev(mp_in), ob=_dev(ob_in), nm=_dev(np.full(F, SENT)), nc=_dev(np.zeros(F, np.uint64)))
    a = B.LocalMapBatch()
    a.cam = B.make_camera(MC.W, MC.H, MC.CAM, MC.SF, bounds=cs[0]['bounds'])
    a.cur_kps, a.cur_desc, a.cur_uright, a.cur_n = t['kps'].data_ptr(), t['desc'].data_ptr(), t['ur'].data_ptr(), t['n'].data_ptr()
    a.mp_inview, a.proj_x, a.proj_y, a.proj_xr, a.level = t['iv'].data_ptr(), t['px'].data_ptr(), t['py'].data_ptr(), t['pr'].data_ptr(), t['lv'].data_ptr()
    a.view_cos, a.mp_desc, a.mp_obs, a.mp_n = t['vc'].data_ptr(), t['md'].data_ptr(), t['mo'].data_ptr(), t['m'].data_ptr()
    a.th, a.nnratio, a.id_base = p['th'], p['nnratio'], MC.ID_BASE
    a.f_mp, a.f_mp_obs, a.nmatches, a.ncand = t['mp'].data_ptr(), t['ob'].data_ptr(), t['nm'].data_ptr(), t['nc'].data_ptr()
    mt = B.Matcher(F, cap, pcap)
    mt.localmap_batch(a, F)
    out = dict(mp=_host(t['mp']), ob=_host(t['ob']), nm=_host(t['nm']), nc=_host(t['nc']))
    mt.close()
    return fr, ns, (mp_in, ob_in), out


@pytest.mark.parametrize('names', _groups('local'), ids=_ids(_groups('local')))
def test_localmap_batch(names):
    fr, ns, (mp_in, ob_in), out = _run_local(names)
    for k, (f, (n, m)) in enumerate(zip(fr, ns)):
        _check_frame(f, n, m, out['mp'][k], 'mp', 'f_mp', mp_in[k], SENT, out['nm'][k], int(out['nc'][k]))
        _check_frame(f, n, m, out['ob'][k], 'obs', 'f_mp_obs', ob_in[k], SENT_U8, out['nm'][k], int(out['nc'][k]))
    _, _, _, again = _run_local(names)
    assert all(again[k].tobytes() == out[k].tobytes() for k in out)
    for n in names:
        c = MC.CASES[n]; p = c['params']; o = MC.run_oracle(c)
        fg = B.HostFrame(c['kps'], c['uright'], c['desc'], MC.W, MC.H, MC.CAM['fx'], MC.CAM['fy'], MC.CAM['cx'], MC.CAM['cy'], MC.CAM['bf'], MC.SF, bounds=c['bounds'])
        nm, mp, ob = B.match_project_localmap(fg, c['inview'], c['projx'], c['projy'], c['projxr'], c['level'], c['viewcos'], c['mp_desc'], c['mp_obs'],
                                              p['th'], p['nnratio'], c['f_mp'], c['f_obs'], id_base=MC.ID_BASE)
        assert nm == o['nm'] and np.array_equal(mp, o['mp']) and np.array_equal(ob, o['obs']), n


# ---- SearchByProjection(KeyFrame*, Scw, vpPoints, vpMatched, th): the fuse kernel's variant 3 -----------------------------------------
def _run_sim3(names):
    fr = _frames(names)
    cs = [f['case'] for f in fr]
    F = len(fr)
    cap = max(len(c['kps']) for c in cs) + EXTRA_KP
    pcap = max(len(c['kf_valid']) for c in cs) + EXTRA_PT
    p = cs[0]['params']
    ns = [_counts(f, len(f['case']['kps']), len(f['case']['kf_valid'])) for f in fr]
    km_in = np.stack([_pad(f['case']['matched'][:n], cap, SENT) for f, (n, _) in zip(fr, ns)])
    pts = lambda key: _dev(np.stack([_pad(c[key], pcap) for c in cs]))
    t = dict(kps=_dev(np.stack([_pad(c['kps'], cap) for c in cs]).view(np.uint8).reshape(-1)), desc=_dev(np.stack([_pad(c['desc'], cap) for c in cs])),
             ur=_dev(np.stack([_pad(c['uright'], cap) for c in cs])), n=_dev(np.array([n for n, _ in ns], np.int32)),
             T=_dev(np.stack([c['Tcw_cur'].reshape(16) for c in cs])), ow=_dev(np.stack([c['Ow'] for c in cs])), xyz=pts('last_xyz'), nrm=pts('normal'),
             mn=pts('min_dist'), mx=pts('max_dist'), md=pts('last_desc'), mv=pts('kf_valid'), m=_dev(np.array([m for _, m in ns], np.int32)),
             km=_dev(km_in), bi=_dev(np.full((F, pcap), SENT)), bd=_dev(np.full((F, pcap), SENT)), nm=_dev(np.full(F, SENT)))
    a = B.FuseBatch()
    a.cam = B.make_camera(MC.W, MC.H, MC.CAM, MC.SF, bounds=cs[0]['bounds'])
    a.kf_kps, a.kf_desc, a.kf_uright, a.kf_n, a.kf_cap = t['kps'].data_ptr(), t['desc'].data_ptr(), t['ur'].data_ptr(), t['n'].data_ptr(), cap
    a.tcw, a.ow, a.mp_xyz, a.mp_normal, a.mp_min_dist, a.mp_max_dist = t['T'].data_ptr(), t['ow'].data_ptr(), t['xyz'].data_ptr(), t['nrm'].data_ptr(), t['mn'].data_ptr(), t['mx'].data_ptr()
    a.mp_desc, a.mp_valid, a.mp_n, a.mp_cap, a.th = t['md'].data_ptr(), t['mv'].data_ptr(), t['m'].data_ptr(), pcap, float(p['th'])
    a.sim3_variant = 3
    a.best_idx, a.best_dist, a.kf_matched, a.nmatches = t['bi'].data_ptr(), t['bd'].data_ptr(), t['km'].data_ptr(), t['nm'].data_ptr()
    B.check(B.lib().sgs_fuse_search_batch_device(C.byref(a), F, V(0)))
    return fr, ns, km_in, dict(km=_host(t['km']), bi=_host(t['bi']), bd=_host(t['bd']), nm=_host(t['nm']))


def _claims(c, matched):
    """best_idx the variant-3 search must report: the feature each point claimed, -1 for the rest."""
    bi = np.full(len(c['kf_valid']), -1, np.int32)
    for k, (was, now) in enumerate(zip(c['matched'], matched)):
        if was < 0 and now >= 0:
            bi[now] = k
    return bi


@pytest.mark.parametrize('names', _groups('sim3'), ids=_ids(_groups('sim3')))
def test_sim3_batch(names):
    fr, ns, km_in, out = _run_sim3(names)
    for k, (f, (n, m)) in enumerate(zip(fr, ns)):
        c = f['case']
        _check_frame(f, n, m, out['km'][k], 'matched', 'kf_matched', km_in[k], SENT, out['nm'][k])
        want = _claims(c, MC.run_oracle(c)['matched']) if n and m else np.full(m, -1, np.int32)
        assert np.array_equal(out['bi'][k, :m], want), c['name']
        for i in np.nonzero(want >= 0)[0]:
            assert out['bd'][k, i] == MC.hamming(c['last_desc'][i], c['desc'][want[i]]) <= 50
        assert (out['bi'][k, m:] == SENT).all() and (out['bd'][k, m:] == SENT).all()
    _, _, _, again = _run_sim3(names)
    assert all(again[k].tobytes() == out[k].tobytes() for k in out)
    for n in names:                                   # sgs_fuse_search: the single-frame host entry point
        c = MC.CASES[n]; o = MC.run_oracle(c)
        fg = B.HostFrame(c['kps'], c['uright'], c['desc'], MC.W, MC.H, MC.CAM['fx'], MC.CAM['fy'], MC.CAM['cx'], MC.CAM['cy'], MC.CAM['bf'], MC.SF, bounds=c['bounds'])
        m = len(c['kf_valid'])
        P = lambda x: np.ascontiguousarray(x).ctypes.data_as(V)
        km = c['matched'].astype(np.int32).copy(); bi = np.full(m, 7, np.int32); bd = np.full(m, 7, np.int32); nm = C.c_int(-1)
        arrs = [np.ascontiguousarray(x) for x in (c['Tcw_cur'].reshape(16), c['Ow'], c['kf_valid'], c['last_xyz'], c['normal'], c['min_dist'], c['max_dist'], c['last_desc'])]
        B.check(B.lib().sgs_fuse_search(C.byref(fg.c), *[P(x) for x in arrs[:2]], m, *[P(x) for x in arrs[2:]], float(c['params']['th']), None, 3, None,
                                        P(bi), P(bd), P(km), C.byref(nm), 0))
        assert nm.value == o['nm'] and np.array_equal(km, o['matched']) and np.array_equal(bi, _claims(c, o['matched'])), n


# ---- SearchForInitialization ----------------------------------------------------------------------------------------------------------
def _run_init(names):
    fr = _frames(names)
    cs = [f['case'] for f in fr]
    F = len(fr)
    c2 = max(len(c['k2']) for c in cs) + EXTRA_KP
    c1 = max(len(c['k1']) for c in cs) + EXTRA_PT
    p = cs[0]['params']
    ns = [_counts(f, len(f['case']['k2']), len(f['case']['k1'])) for f in fr]        # (F2 keypoints, F1 keypoints)
    prev_in = np.stack([_pad(f['case']['prev'][:m], c1, SENT_F) for f, (_, m) in zip(fr, ns)])
    t = dict(k1=_dev(np.stack([_pad(c['k1'], c1) for c in cs]).view(np.uint8).reshape(-1)), d1=_dev(np.stack([_pad(c['d1'], c1) for c in cs])),
             k2=_dev(np.stack([_pad(c['k2'], c2) for c in cs]).view(np.uint8).reshape(-1)), d2=_dev(np.stack([_pad(c['d2'], c2) for c in cs])),
             n1=_dev(np.array([m for _, m in ns], np.int32)), n2=_dev(np.array([n for n, _ in ns], np.int32)), prev=_dev(prev_in),
             m12=_dev(np.full((F, c1), SENT)), nm=_dev(np.full(F, SENT)))
    a = B.InitBatch()
    a.cam = B.make_camera(MC.W, MC.H, MC.CAM, MC.SF, bounds=cs[0]['bounds'])
    a.f1_kps, a.f1_desc, a.f1_n, a.f1_cap = t['k1'].data_ptr(), t['d1'].data_ptr(), t['n1'].data_ptr(), c1
    a.f2_kps, a.f2_desc, a.f2_n, a.f2_cap = t['k2'].data_ptr(), t['d2'].data_ptr(), t['n2'].data_ptr(), c2
    a.prev_xy, a.window_size, a.nnratio, a.check_orientation = t['prev'].data_ptr(), p['window'], p['nnratio'], int(p['check_ori'])
    a.match12, a.nmatches = t['m12'].data_ptr(), t['nm'].data_ptr()
    B.check(B.lib().sgs_search_for_initialization_batch_device(C.byref(a), F, V(0)))
    return fr, ns, prev_in, dict(m12=_host(t['m12']), prev=_host(t['prev']), nm=_host(t['nm']))


def _view(k, d, c):
    v = B.FrameView(); v.n = len(k); v.keys_un = k.ctypes.data; v.u_right = None; v.desc = d.ctypes.data
    v.min_x, v.min_y, v.max_x, v.max_y = c['bounds']
    v.nlevels = len(MC.SF); v.scale_factors = MC.SF.ctypes.data
    return v


@pytest.mark.parametrize('names', _groups('init'), ids=_ids(_groups('init')))
def test_search_for_initialization_batch(names):
    fr, ns, prev_in, out = _run_init(names)
    for k, (f, (n2, n1)) in enumerate(zip(fr, ns)):
        c = f['case']
        if n1 and n2:
            o = MC.run_oracle(c)
            assert out['nm'][k] == o['nm'] and np.array_equal(out['m12'][k, :n1], o['m12']) and np.array_equal(out['prev'][k, :n1], o['prev']), c['name']
            r = _reference(c)
            if r is not None:
                assert out['nm'][k] == r['nm'] and np.array_equal(out['m12'][k, :n1], r['m12']) and np.array_equal(out['prev'][k, :n1], r['prev'])
            c['proof'](o)
        else:
            assert out['nm'][k] == 0 and np.array_equal(out['prev'][k, :n1], prev_in[k, :n1]) and (out['m12'][k, :n1] == -1).all()
        assert (out['m12'][k, n1:] == -1).all(), c['name']            # the kernel clears vnMatches12 over the whole capacity
        assert (out['prev'][k, n1:] == SENT_F).all(), c['name']
    _, _, _, again = _run_init(names)
    assert all(again[k].tobytes() == out[k].tobytes() for k in out)
    for n in names:
        c = MC.CASES[n]; p = c['params']; o = MC.run_oracle(c)
        k1, k2 = np.ascontiguousarray(c['k1']), np.ascontiguousarray(c['k2']); d1, d2 = np.ascontiguousarray(c['d1']), np.ascontiguousarray(c['d2'])
        v1, v2 = _view(k1, d1, c), _view(k2, d2, c)
        prev = c['prev'].copy(); mo = np.zeros(len(k1), np.int32); nmo = C.c_int()
        B.check(B.lib().sgs_search_for_initialization(C.byref(v1), C.byref(v2), prev.ctypes.data_as(V), p['window'], p['nnratio'], int(p['check_ori']),
                                                      mo.ctypes.data_as(V), C.byref(nmo), 0))
        assert nmo.value == o['nm'] and np.array_equal(mo, o['m12']) and np.array_equal(prev, o['prev']), n


# ---- image bounds and capacity --------------------------------------------------------------------------------------------------------
def test_tum1_bounds_are_the_device_image_bounds(golden_dir):
    """The bounds the geometry cases use are what sgs_image_bounds computes for TUM1."""
    g = np.load(os.path.join(golden_dir, 'undistort.npz'))
    K = g['TUM1_K']; D = np.ascontiguousarray(g['TUM1_D'], np.float32); b = np.zeros(4, np.float32)
    B.check(B.lib().sgs_image_bounds(640, 480, K[0], K[1], K[2], K[3], D.ctypes.data_as(V), b.ctypes.data_as(V), 0))
    assert tuple(float(x) for x in b) == MC.tum1_bounds()
    assert b[0] != 0 and b[1] != 0


def _crowded(n_cur, n_last, seed=3):
    """A last-frame scenario whose first 120 keypoints share one grid cell, with 60 points aimed into that cell."""
    s = S.random_lastframe_scenario(seed, n_cur=n_cur, n_last=n_last, conflict=0.3)
    k = s['kps']
    k['x'][:120] = (300.0 + 0.35 * (np.arange(120) % 12)).astype(np.float32)
    k['y'][:120] = (200.0 + 0.35 * (np.arange(120) // 12)).astype(np.float32)
    rng = np.random.RandomState(seed)
    cam = s['cam']
    u = 302.0 + rng.normal(0, 1.0, 60); v = 201.5 + rng.normal(0, 1.0, 60); z = rng.uniform(1.0, 3.0, 60)
    Xc = np.stack([(u - cam['cx']) * z / cam['fx'], (v - cam['cy']) * z / cam['fy'], z], 1)
    R = s['Tcw_cur'][:3, :3].astype(np.float64); t = s['Tcw_cur'][:3, 3].astype(np.float64)
    s['last_xyz'][:60] = ((Xc - t) @ R).astype(np.float32)
    tgt = rng.randint(0, 120, 60)
    s['last_desc'][:60] = s['desc'][tgt]
    s['last_desc'][:60, 0] ^= rng.randint(0, 256, 60).astype(np.uint8)
    s['last_oct'][:60] = k['octave'][tgt]; s['last_angle'][:60] = k['angle'][tgt]
    s['last_has'][:60] = 1
    s['uright'][:120] = -1.0
    return s


def test_capacity_8192_keypoints():
    """cur_cap = 8192 (the largest the 16-bit grid positions allow) with one frame of 8192 keypoints, one cell holding 120 of them."""
    s = _crowded(8192, 2000)
    cells = np.bincount([c[0] * 48 + c[1] for c in (MC.pos_in_grid(x, y, MC.FULL) for x, y in zip(s['kps']['x'], s['kps']['y'])) if c is not None])
    assert cells.max() > 16 and (cells > 16).sum() >= 1
    fo = TR._frame(s)
    args = (s['Tcw_cur'], s['Tcw_last'], s['last_has'], s['last_xyz'], s['last_desc'], s['last_obs'], s['last_oct'], s['last_angle'], 15.0)
    nm_o, mp_o, nc_o = O.search_by_projection_last(fo, *args)
    assert nm_o > 500 and (mp_o[:120] >= 0).sum() > 20
    if os.path.exists(TR.LIB):
        nm_r, mp_r = TR.ref_last(TR._lib(), s, 15.0, False, True)
        assert nm_r == nm_o and np.array_equal(mp_r, mp_o)
    n, m = 8192, 2000
    t = dict(kps=_dev(s['kps'].view(np.uint8).reshape(-1)), desc=_dev(s['desc']), ur=_dev(s['uright']), n=_dev(np.array([n], np.int32)),
             xyz=_dev(s['last_xyz']), ld=_dev(s['last_desc']), fl=_dev(s['last_has'] | (s['last_obs'] << 1)), oct=_dev(s['last_oct']), ang=_dev(s['last_angle']),
             m=_dev(np.array([m], np.int32)), tc=_dev(s['Tcw_cur'].reshape(16)), tl=_dev(s['Tcw_last'].reshape(16)), mp=_dev(np.full(n, -1, np.int32)),
             nm=_dev(np.full(1, SENT)), nc=_dev(np.zeros(1, np.uint64)))
    a = B.LastFrameBatch()
    a.cam = B.make_camera(640, 480, s['cam'], s['sf'])
    a.cur_kps, a.cur_desc, a.cur_uright, a.cur_n = t['kps'].data_ptr(), t['desc'].data_ptr(), t['ur'].data_ptr(), t['n'].data_ptr()
    a.last_xyz, a.last_desc, a.last_flags, a.last_octave = t['xyz'].data_ptr(), t['ld'].data_ptr(), t['fl'].data_ptr(), t['oct'].data_ptr()
    a.last_angle, a.last_n, a.tcw_cur, a.tcw_last = t['ang'].data_ptr(), t['m'].data_ptr(), t['tc'].data_ptr(), t['tl'].data_ptr()
    a.th, a.mono, a.check_orientation = 15.0, 0, 1
    a.cur_mp, a.nmatches, a.ncand = t['mp'].data_ptr(), t['nm'].data_ptr(), t['nc'].data_ptr()
    mt = B.Matcher(1, 8192, m)
    mt.lastframe_batch(a, 1)
    assert int(_host(t['nm'])[0]) == nm_o and np.array_equal(_host(t['mp']), mp_o) and int(_host(t['nc'])[0]) == nc_o
    mt.close()
    fg = B.HostFrame(s['kps'], s['uright'], s['desc'], 640, 480, s['cam']['fx'], s['cam']['fy'], s['cam']['cx'], s['cam']['cy'], s['cam']['bf'], s['sf'])
    nm_h, mp_h = B.match_project_lastframe(fg, *args)
    assert nm_h == nm_o and np.array_equal(mp_h, mp_o)


def test_capacity_8193_is_refused():
    h = V()
    assert B.lib().sgs_matcher_create(0, 1, 8193, 10, C.byref(h)) == B.SGS_ERR_UNSUPPORTED and not h.value
    s = S.random_lastframe_scenario(4, n_cur=8193, n_last=10)
    fg = B.HostFrame(s['kps'], s['uright'], s['desc'], 640, 480, s['cam']['fx'], s['cam']['fy'], s['cam']['cx'], s['cam']['cy'], s['cam']['bf'], s['sf'])
    mp = np.full(8193, -1, np.int32)
    with pytest.raises(B.SgsError) as e:
        B.match_project_lastframe(fg, s['Tcw_cur'], s['Tcw_last'], s['last_has'], s['last_xyz'], s['last_desc'], s['last_obs'], s['last_oct'], s['last_angle'],
                                  15.0, cur_mp=mp)
    assert e.value.code == B.SGS_ERR_UNSUPPORTED
