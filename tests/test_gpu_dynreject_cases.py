"""Every constructed case of tests/dynreject_cases.py through every device path of the dynamic-feature rejection, bit for bit against the
restatement there (tests/test_dynreject_cases.py pins the restatement to the oracle and to the reference's own Frame on the CPU):

  * sgs_dynreject (single frame): verdicts, distance bits, kept count, restore flag;
  * sgs_dynreject_batch_device: the cases packed into batches of mixed sizes, the ordered compaction of the 28-byte keypoint and 32-byte
    descriptor rows, the untouched rows and verdicts past each frame's count, keep_out NULL, capacity 1, counts above the capacity and below
    zero, and the largest capacity the kernel's shared memory takes (the next one is refused before anything is enqueued);
  * sgs_tracker_track: extracted frames with constructed previous points, F, boxes and u_right, so that the verdicts are chosen per
    keypoint -- the keypoints, descriptors and u_right that come back (compact_uright_kernel moves u_right with the rejection's own
    verdicts) and the map-point slots past the count."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import dynreject_cases as D  # noqa: E402
import scenarios as S  # noqa: E402
from pysgs import binding as B  # noqa: E402
from pysgs import synth  # noqa: E402

NAMES = [c['name'] for c in D.CASES]
CAP = 1100
SENTINEL = 0xA5
KEEP_SENTINEL = 0xEE
EMPTY_F = np.array([np.nan, 0, 0, 0, 0, 1, 0, -1, 0])     # F[0] NaN: the empty matrix; the rest would remove every point if it were read


def same_dist(got, want):
    """Distances equal bit for bit, NaN where NaN (a NaN's payload is not part of the result)."""
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got[~nan].view(np.uint64), want[~nan].view(np.uint64))


@pytest.mark.parametrize('name', NAMES)
def test_single_frame(name):
    c = D.BY_NAME[name]
    nk, keep, dist, restored = B.dynreject(c['cur'], c['prev'], c['F'], D.single_frame_boxes(c), c['have_dyn'], c['nfeatures'])
    assert np.array_equal(keep, c['keep']) and same_dist(dist, c['dist'])
    assert nk == c['nkeep'] and restored == c['restored']


def _pack(frames, cap, seed):
    """Host arrays of one batch.  frames: (case, count) pairs; rows past a frame's keypoints hold random bytes."""
    rng = np.random.RandomState(seed)
    nf = len(frames)
    kps = rng.randint(0, 256, (nf, cap * 28)).astype(np.uint8).view(B.KP_DTYPE)
    desc = rng.randint(0, 256, (nf, cap, 32)).astype(np.uint8)
    prev = rng.uniform(0, 640, (nf, cap, 2)).astype(np.float32)
    Fm = np.zeros((nf, 9)); boxes = np.zeros((nf, D.MAX_BOXES, 4), np.float32)
    counts = np.zeros(nf, np.int32); nboxes = np.zeros(nf, np.int32); have = np.zeros(nf, np.uint8)
    for f, (c, count) in enumerate(frames):
        m = min(len(c['cur']), cap)
        assert min(max(count, 0), cap) <= m, (c['name'], 'a frame reads only its own keypoints')
        kps['x'][f, :m], kps['y'][f, :m] = c['cur'][:m, 0], c['cur'][:m, 1]
        prev[f, :m] = c['prev'][:m]
        Fm[f] = EMPTY_F if c['F'] is None else c['F']
        boxes[f, :len(c['boxes'])] = c['boxes']
        counts[f], nboxes[f], have[f] = count, c['nboxes'], c['have_dyn']
        if c['follower']:
            assert f + 1 < nf and frames[f + 1][0]['name'] == c['follower'], 'the boxes past max_boxes are the next frame\'s'
            assert (frames[f + 1][0]['boxes'] == np.array(D.WHOLE_IMAGE, np.float32)).all()
    return dict(kps=kps, desc=desc, prev=prev, Fm=Fm, boxes=boxes, counts=counts, nboxes=nboxes, have=have)


def _launch(p, cap, nfeatures, with_keep=True):
    """One sgs_dynreject_batch_device call on outputs pre-filled with sentinels; returns (status, outputs as host arrays)."""
    import torch
    nf = len(p['counts'])
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    t = {k: dev(v.view(np.uint8) if k == 'kps' else v) for k, v in p.items()}
    kout = torch.full((nf, cap * 28), SENTINEL, dtype=torch.uint8, device='cuda')
    dout = torch.full((nf, cap, 32), SENTINEL, dtype=torch.uint8, device='cuda')
    cout = torch.full((nf,), -7, dtype=torch.int32, device='cuda')
    keep = torch.full((nf, cap), KEEP_SENTINEL, dtype=torch.uint8, device='cuda')
    torch.cuda.synchronize()
    try:
        B.dynreject_batch_device(t['kps'].data_ptr(), t['desc'].data_ptr(), t['counts'].data_ptr(), cap, nf, t['prev'].data_ptr(), t['Fm'].data_ptr(),
                                 t['boxes'].data_ptr(), t['nboxes'].data_ptr(), D.MAX_BOXES, t['have'].data_ptr(), nfeatures, kout.data_ptr(),
                                 dout.data_ptr(), cout.data_ptr(), keep.data_ptr() if with_keep else 0, 0)
        status = B.SGS_OK
    except B.SgsError as e:
        status = e.code
    torch.cuda.synchronize()
    return status, dict(kps=kout.cpu().numpy().view(B.KP_DTYPE), desc=dout.cpu().numpy(), counts=cout.cpu().numpy(), keep=keep.cpu().numpy())


def _check(frames, p, out, cap, nfeatures, with_keep=True):
    for f, (c, count) in enumerate(frames):
        n = min(max(count, 0), cap)
        keep, _, _, restored = D.restate(c['cur'][:n], c['prev'][:n], c['F'], c['boxes'], c['nboxes'], c['have_dyn'], nfeatures)
        sel = np.arange(n) if restored else np.nonzero(keep)[0]
        m = len(sel)
        assert out['counts'][f] == m, (c['name'], count)
        if with_keep:
            assert np.array_equal(out['keep'][f, :n], keep), c['name']
        assert (out['keep'][f, (n if with_keep else 0):] == KEEP_SENTINEL).all(), (c['name'], 'verdicts past the count are not written')
        assert out['kps'][f, :m].tobytes() == p['kps'][f, sel].tobytes(), c['name']
        assert out['desc'][f, :m].tobytes() == p['desc'][f, sel].tobytes(), c['name']
        assert (out['kps'][f, m:].view(np.uint8) == SENTINEL).all() and (out['desc'][f, m:] == SENTINEL).all(), (c['name'], 'rows past the count')


def _batches():
    """{id: (frames, cap, nfeatures)} of the batch runs: the cases of each nfeatures in one launch of mixed sizes; frames of every kind under
    nfeatures 1000 (empty, negative count, restored, empty F, normal); capacity 1."""
    by_nf = {}
    for c in D.CASES:
        by_nf.setdefault(c['nfeatures'], []).append((c, c['count']))
    out = {'nf%d' % nf: (frames, CAP, nf) for nf, frames in sorted(by_nf.items())}
    g = D.BY_NAME
    mixed = [(g['shape_n0_none_removed'], 0), (g['restore_negative_count'], -5), (g['restore_nf1000_keep99'], 160), (g['F_empty'], 24),
             (g['shape_n257_runs'], 257), (g['restore_nf1000_keep100'], 160), (g['shape_count_above_cap'], 1500), (g['F_all_zero'], 24)]
    out['mixed'] = (mixed, CAP, 1000)
    cap1 = [(g['shape_n1_none_removed'], 1), (g['shape_n1_all_removed'], 1), (g['shape_n31_alternate'], 5), (g['shape_n31_first_removed'], 31),
            (g['shape_n0_none_removed'], 0), (g['restore_negative_count'], -2), (g['restore_nf1000_keep99'], 1), (g['F_empty'], 3)]
    out['cap1'] = (cap1, 1, 1000)
    return out


BATCHES = _batches()


@pytest.mark.parametrize('batch', sorted(BATCHES))
def test_batch_device(batch):
    frames, cap, nf = BATCHES[batch]
    p = _pack(frames, cap, sorted(BATCHES).index(batch))
    st, out = _launch(p, cap, nf)
    assert st == B.SGS_OK
    _check(frames, p, out, cap, nf)
    st, out2 = _launch(p, cap, nf, with_keep=False)
    assert st == B.SGS_OK
    _check(frames, p, out2, cap, nf, with_keep=False)
    assert all(out[key].tobytes() == out2[key].tobytes() for key in ('kps', 'desc', 'counts')), 'keep_out NULL changes nothing else'


def test_batch_device_shared_memory_limit():
    """The kernel keeps one int per keypoint slot in shared memory, up to 160 KB: cap 40960 runs, 40961 is refused with nothing enqueued."""
    big = D.large_frame(40960)
    big['proof']()
    frames = [(big, 40960)]
    p = _pack(frames, 40960, 7)
    st, out = _launch(p, 40960, 0)
    assert st == B.SGS_OK
    _check(frames, p, out, 40960, 0)
    p2 = _pack(frames, 40961, 8)
    st, out = _launch(p2, 40961, 0)
    assert st == B.SGS_ERR_UNSUPPORTED and 'cap too large' in B.lib().sgs_last_error().decode()
    assert out['counts'][0] == -7 and (out['keep'] == KEEP_SENTINEL).all()
    assert (out['kps'].view(np.uint8) == SENTINEL).all() and (out['desc'] == SENTINEL).all()


# ---- sgs_tracker_track: the rejection and the u_right compaction on extracted frames -----------------------------------------------------

W, H, NF = 640, 480, 1000


def _tracker_inputs(kps, n, cap, frames_spec, ur):
    """Per-frame (pattern kind, box, have_dyn, empty F) -> prev_xy, F, boxes, nboxes, have_dyn, and the restatement's (keep, restored)."""
    nb = len(frames_spec)
    prev = np.zeros((nb, cap, 2), np.float32); F = np.zeros((nb, 9)); boxes = np.zeros((nb, 4, 4), np.float32)
    nboxes = np.zeros(nb, np.int32); have = np.zeros(nb, np.uint8); want = []
    for f, (pattern, box, hv, empty_f) in enumerate(frames_spec):
        cur = np.stack([kps['x'][f, :n[f]], kps['y'][f, :n[f]]], 1)
        prev[f, :n[f]] = D.prev_for(cur, pattern, box)
        F[f] = EMPTY_F if empty_f else D.THRESHOLD_F
        boxes[f, 0] = box; nboxes[f] = 1; have[f] = hv
        keep, _, nkeep, restored = D.restate(cur, prev[f, :n[f]], None if empty_f else D.THRESHOLD_F, [box], 1, hv, NF)
        assert np.array_equal(keep, pattern) or empty_f, 'the chosen verdicts'
        want.append(np.arange(n[f]) if restored else np.nonzero(keep)[0])
    return (prev, ur, F, boxes, nboxes, have), want


def test_tracker_track_compacts_u_right_with_the_rejection_verdicts():
    frames, _ = synth.stream_s2(2, W, H, seed=3)
    cam = synth.TUM3
    trk = B.Tracker(W, H, B.make_camera(W, H, cam, S.scale_factors()), NF, 1.2, 8, 20, 7, max_batch=2, point_cap=NF + 64, max_boxes=4, device=0)
    try:
        L = B.lib(); P = lambda a: a.ctypes.data_as(C.c_void_p)
        cap = trk.cap
        kps = np.zeros((2, cap), B.KP_DTYPE); desc = np.zeros((2, cap, 32), np.uint8); n = np.zeros(2, np.int32)
        B.check(L.sgs_tracker_extract(trk.h, P(frames), 2, W * H, W, P(kps), P(desc), cap, P(n)))
        assert (n > 300).all()
        ur = np.full((2, cap), -1, np.float32)
        for f in range(2):
            ur[f, :n[f]] = np.where(np.arange(n[f]) % 5 == 4, -1, 10 + f * 2000 + 0.25 * np.arange(n[f]))
        # the last frame: every extracted keypoint as a map point 2 m in front of the camera, so that the search fills cur_mp
        pc = NF + 64
        lxyz = np.zeros((2, pc, 3), np.float32); ldesc = np.zeros((2, pc, 32), np.uint8); lfl = np.zeros((2, pc), np.uint8)
        loct = np.zeros((2, pc), np.int32); lang = np.zeros((2, pc), np.float32); ln = np.minimum(n, pc).astype(np.int32)
        for f in range(2):
            m = ln[f]; k = kps[f, :m]
            lxyz[f, :m] = np.stack([(k['x'] - cam['cx']) * 2 / cam['fx'], (k['y'] - cam['cy']) * 2 / cam['fy'], np.full(m, 2.0)], 1)
            ldesc[f, :m] = desc[f, :m]; lfl[f, :m] = 3; loct[f, :m] = k['octave']; lang[f, :m] = k['angle']
        T = np.tile(np.eye(4, dtype=np.float32).reshape(1, 16), (2, 1))
        last = (lxyz, ldesc, lfl, loct, lang, ln, T, T)

        def track(spec):
            ins, want = _tracker_inputs(kps, n, cap, spec, ur)
            o = dict(kps=np.zeros((2, cap), B.KP_DTYPE), desc=np.zeros((2, cap, 32), np.uint8), ur=np.zeros((2, cap), np.float32),
                     cnt=np.zeros(2, np.int32), mp=np.zeros((2, cap), np.int32), nm=np.zeros(2, np.int32))
            trk.track(2, [P(a) for a in ins + last], 15.0, True, True, [P(o[k]) for k in ('kps', 'desc', 'ur', 'cnt', 'mp', 'nm')])
            for f in range(2):
                sel = want[f]; m = len(sel)
                assert o['cnt'][f] == m
                assert o['kps'][f, :m].tobytes() == kps[f, sel].tobytes() and np.array_equal(o['desc'][f, :m], desc[f, sel])
                assert o['ur'][f, :m].tobytes() == ur[f, sel].tobytes(), 'u_right moves with the keypoints'
                assert (o['mp'][f, m:] == -1).all()
            return o, want

        box = (150, 100, 300, 250)
        rng = np.random.RandomState(5)
        keep99 = np.zeros(n[0], np.uint8); keep99[rng.permutation(n[0])[:99]] = 1
        # a restored frame and an empty-F frame come back unchanged
        o1, w1 = track([(keep99, box, 1, False), (np.zeros(n[1], np.uint8), box, 1, True)])
        assert [len(w) for w in w1] == list(n) and (o1['mp'] >= 0).sum() > 100
        # 100 kept of 1000 features (not restored) and a frame with runs of removed keypoints across the 32 and 256 boundaries
        keep100 = np.zeros(n[0], np.uint8); keep100[rng.permutation(n[0])[:100]] = 1
        runs = D.shape_pattern('runs', n[1])
        o2, w2 = track([(keep100, box, 1, False), (runs, box, 1, False)])
        assert len(w2[0]) == 100 and len(w2[1]) == runs.sum() < n[1]
        assert all((o1['mp'][f, len(w2[f]):n[f]] >= 0).any() for f in range(2)), 'the slots past the new count held matches before'
    finally:
        trk.close()
