"""The RGB-D stream step (sgs_tracker_step_rgbd_stream / _device): one new frame per stream slot per call, each stream's previous frame kept in the
tracker.  Every case runs stream calls and the matching batch formulation -- sgs_tracker_step_rgbd_device on a batch that holds each stream's previous
frame, chained with prev_index -- and requires every output of every new frame to be equal bit for bit: keypoints, descriptors, counts, mvuRight,
matches, boxes and flag, mvKeysUn, mvDepth, F and its info, and the LK positions.  Each case proves from info and the boxes that the paths it is named
for were taken.  Inputs as in tests/test_gpu_grab_rgbd.py: S2 colour frames blended with the mini SSD graph's scenes, so that person boxes occur."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import detector_model as DM  # noqa: E402
import grab_ref as GR  # noqa: E402
from pysgs import binding as B  # noqa: E402
from pysgs import synth  # noqa: E402

W, H, NF, TH, MB = 640, 480, 1000, 15.0, 4
POOL = 16                       # distinct frames; frame content c of a stream is pool frame c, the last-frame inputs those built for c
FACTOR = np.float32(1 / 5000)
LAST = ('lxyz', 'ldesc', 'lflags', 'loct', 'lang', 'ln', 'T', 'T')
v = C.c_void_p
P = lambda a: a.ctypes.data_as(v)


def dev(a):
    import torch
    a = np.ascontiguousarray(a)
    return torch.from_numpy(a.view(np.uint8) if a.dtype.fields else a).cuda()


def fmt_of(depth_type, factor):
    return B.RgbdFormat(1, depth_type, factor)


@pytest.fixture(scope='module')
def pool(tmp_path_factory):
    import bench
    rgb, depth, gt = synth.stream_s2_rgbd(POOL, W, H, seed=5)
    rgb = np.ascontiguousarray(np.stack([(DM.synthetic_rgb(H, W, 10 + i).astype(np.float32) * 0.25 + rgb[i] * 0.75).astype(np.uint8) for i in range(POOL)]))
    pp, bp = DM.write_mini_model(str(tmp_path_factory.mktemp('det')), 0)
    sf = synth.scale_factors()
    cam = B.make_camera(W, H, synth.TUM3, sf)
    trk = B.Tracker(W, H, cam, NF, 1.2, 8, 20, 7, max_batch=POOL, point_cap=NF + 64, max_boxes=MB, device=0)
    cap = trk.cap
    kps = np.zeros((POOL, cap), B.KP_DTYPE); desc = np.zeros((POOL, cap, 32), np.uint8); n = np.zeros(POOL, np.int32)
    B.check(B.lib().sgs_tracker_extract(trk.h, P(GR.to_gray(rgb, 1)), POOL, W * H, W, P(kps), P(desc), cap, P(n)))
    trk.close()
    ti = bench.make_track_inputs(kps, desc, n, gt, cap, NF + 64, np.concatenate([[0], np.arange(POOL - 1)]), W, H, dict(synth.TUM3))
    return dict(rgb=rgb, depth=depth, ti=ti, pp=pp, bp=bp, cam=cam, sf=sf, d_rgb=dev(rgb), d_depth=dev(depth.view(np.int16)),      # int16: indexable on the device
                d_ti={k: dev(ti[k]) for k in set(LAST)})


class Run:
    """A tracker and its detector."""

    def __init__(self, pool, max_batch):
        self.trk = B.Tracker(W, H, pool['cam'], NF, 1.2, 8, 20, 7, max_batch=max_batch, point_cap=NF + 64, max_boxes=MB, device=0)
        self.det = B.Detector(pool['pp'], pool['bp'], max_frames=max_batch, det_thr=0.9, dyn_thr=0.01)

    def close(self):
        self.trk.close(); self.det.close()


def collect(trk, n):
    """Every output of the last step, per frame: the results, boxes, mvKeysUn / mvDepth, F / info, the LK positions and the extracted count."""
    L, cap = B.lib(), trk.cap
    p = [v() for _ in range(16)]
    B.check(L.sgs_tracker_results_device(trk.h, *[C.byref(x) for x in p[:7]]))
    B.check(L.sgs_tracker_boxes_device(trk.h, *[C.byref(x) for x in p[7:10]]))
    B.check(L.sgs_tracker_frame_device(trk.h, C.byref(p[10]), C.byref(p[11])))
    B.check(L.sgs_tracker_fundamental_device_ptr(trk.h, C.byref(p[12]), C.byref(p[13])))
    B.check(L.sgs_tracker_prev_xy_device(trk.h, C.byref(p[14])))
    ecap = C.c_int()
    B.check(L.sgs_extractor_results_device(L.sgs_tracker_extractor(trk.h), None, None, C.byref(p[15]), C.byref(ecap)))
    shapes = dict(kps=((n, cap), B.KP_DTYPE, 0), desc=((n, cap, 32), np.uint8, 1), ur=((n, cap), np.float32, 2), cnt=(n, np.int32, 3),
                  mp=((n, cap), np.int32, 4), nm=(n, np.int32, 5), boxes=((n, MB, 4), np.float32, 7), nb=(n, np.int32, 8), have=(n, np.uint8, 9),
                  kun=((n, cap), B.KP_DTYPE, 10), dz=((n, cap), np.float32, 11), F=((n, 9), np.float64, 12), info=((n, 4), np.int32, 13),
                  prev=((n, cap, 2), np.float32, 14), n_all=(n, np.int32, 15))
    r = {k: B.memcpy_d2h(np.zeros(s, dt), p[i].value) for k, (s, dt, i) in shapes.items()}
    return [{k: a[f] for k, a in r.items()} for f in range(n)]


def same_row(a, b, what):
    n_all, c, nbx = int(a['n_all']), int(a['cnt']), int(a['nb'])
    for k in ('n_all', 'cnt', 'nm', 'nb', 'have', 'info'):
        assert np.array_equal(a[k], b[k]), (what, k, a[k], b[k])
    for k in ('kps', 'desc', 'ur', 'mp', 'kun', 'dz'):
        assert a[k][:c].tobytes() == b[k][:c].tobytes(), (what, k)
    assert a['boxes'][:nbx].tobytes() == b['boxes'][:nbx].tobytes(), (what, 'boxes')
    assert a['F'].tobytes() == b['F'].tobytes(), (what, 'F')
    assert a['prev'][:n_all].tobytes() == b['prev'][:n_all].tobytes(), (what, 'prev_xy')


def device_inputs(pool, content):
    import torch
    idx = torch.as_tensor(np.asarray(content, np.int64), device='cuda')
    return pool['d_rgb'][idx].contiguous(), pool['d_depth'][idx].contiguous(), [pool['d_ti'][k][idx].contiguous() for k in LAST]


def stream_call(r, pool, content, slots, new=None):
    """sgs_tracker_step_rgbd_stream_device: frame i (pool frame content[i]) is the next frame of slot slots[i]."""
    import torch
    rgb, depth, last = device_inputs(pool, content)
    d_slot = dev(np.asarray(slots, np.int32))
    d_new = dev(np.asarray(new, np.uint8)) if new is not None else None
    r.trk.step_rgbd_stream_device(r.det, rgb.data_ptr(), H * W * 3, W * 3, depth.data_ptr(), H * W * 2, W * 2, fmt_of(B.DEPTH_U16, FACTOR), len(slots),
                                  d_slot.data_ptr(), d_new.data_ptr() if d_new is not None else 0, [t.data_ptr() for t in last], TH, 0, 1)
    torch.cuda.synchronize()
    return collect(r.trk, len(slots))


def batch_call(r, pool, content, pidx):
    """sgs_tracker_step_rgbd_device on pool frames `content` chained by prev_index `pidx`."""
    import torch
    rgb, depth, last = device_inputs(pool, content)
    d_pidx = dev(np.asarray(pidx, np.int32))
    B.check(B.lib().sgs_tracker_step_rgbd_device(r.trk.h, r.det.h, rgb.data_ptr(), H * W * 3, W * 3, depth.data_ptr(), H * W * 2, W * 2,
                                                 C.byref(fmt_of(B.DEPTH_U16, FACTOR)), len(content), d_pidx.data_ptr(), *[t.data_ptr() for t in last],
                                                 TH, 0, 1, v(0)))
    torch.cuda.synchronize()
    return collect(r.trk, len(content))


def host_call(r, pool, content, slots, new=None, depth_f32=False, pinned=False, rgb_pad=0, depth_pad=0, nframes=None, slot_arg=True):
    """sgs_tracker_step_rgbd_stream from host buffers; returns (rc, the host outputs per frame)."""
    import torch
    n = len(content)
    esz = 4 if depth_f32 else 2
    rp, dp = W * 3 + rgb_pad, W * esz + depth_pad
    alloc = (lambda s, dt: torch.zeros(s, dtype=dt, pin_memory=True).numpy()) if pinned else (lambda s, dt: np.zeros(s, torch.empty(0, dtype=dt).numpy().dtype))
    hr = alloc((n, H, rp), torch.uint8); hr[:, :, :W * 3] = pool['rgb'][content].reshape(n, H, W * 3)
    hd = alloc((n, H, dp // esz), torch.float32 if depth_f32 else torch.int16)
    if depth_f32:
        hd[:, :, :W] = GR.to_depth(pool['depth'][content], FACTOR)
    else:
        hd.view(np.uint16)[:, :, :W] = pool['depth'][content]
    fmt = fmt_of(B.DEPTH_F32, 1.0) if depth_f32 else fmt_of(B.DEPTH_U16, FACTOR)
    ti = pool['ti']
    last = [np.ascontiguousarray(ti[k][content]) for k in LAST]
    slot = np.asarray(slots, np.int32)
    newa = np.asarray(new, np.uint8) if new is not None else None
    cap = r.trk.cap
    o = dict(kps=np.zeros((n, cap), B.KP_DTYPE), desc=np.zeros((n, cap, 32), np.uint8), ur=np.zeros((n, cap), np.float32), cnt=np.zeros(n, np.int32),
             mp=np.zeros((n, cap), np.int32), nm=np.zeros(n, np.int32), boxes=np.zeros((n, MB, 4), np.float32), nb=np.zeros(n, np.int32),
             have=np.zeros(n, np.uint8), kun=np.zeros((n, cap), B.KP_DTYPE), dz=np.zeros((n, cap), np.float32))
    rc = B.lib().sgs_tracker_step_rgbd_stream(r.trk.h, r.det.h, P(hr), H * rp, rp, P(hd), H * dp, dp, C.byref(fmt), n if nframes is None else nframes,
                                             P(slot) if slot_arg else None, P(newa) if newa is not None else None, *[P(a) for a in last], TH, 0, 1,
                                             *[P(o[k]) for k in ('kps', 'desc', 'ur', 'cnt', 'mp', 'nm', 'boxes', 'nb', 'have', 'kun', 'dz')])
    return rc, [{k: a[f] for k, a in o.items()} for f in range(n)]


def host_rows(r, pool, content, slots, **kw):
    """A host stream call that must succeed: its rows as collect() sees them, after checking the host outputs against them."""
    rc, out = host_call(r, pool, content, slots, **kw)
    B.check(rc)
    rows = collect(r.trk, len(content))
    for f, (h, d) in enumerate(zip(out, rows)):
        c, nbx = int(d['cnt']), int(d['nb'])
        assert all(np.array_equal(h[k], d[k]) for k in ('cnt', 'nm', 'nb', 'have')), f
        assert all(h[k][:c].tobytes() == d[k][:c].tobytes() for k in ('kps', 'desc', 'ur', 'mp', 'kun', 'dz')), f
        assert h['boxes'][:nbx].tobytes() == d['boxes'][:nbx].tobytes(), f
    return rows


def filtered(row, prev_row):
    """The previous frame's flag and boxes took pairs out: more than 20 pairs outside the boxes, fewer than exist."""
    return bool(prev_row['have']) and 20 < row['info'][0] < row['n_all'] and row['info'][3] != 3


# ---- 1. a sequence: S streams x T frames as T calls, slot order shuffled every call --------------------------------------------------------------
def test_sequence_equals_the_batch_step(pool):
    S, T = 6, 5
    content = lambda s, t: (3 * s + t) % POOL
    rng = np.random.default_rng(1)
    rs = Run(pool, S)
    got = {}
    for t in range(T):
        order = [int(s) for s in rng.permutation(S)]
        for s, row in zip(order, stream_call(rs, pool, [content(s, t) for s in order], order)):
            got[s, t] = row
    rs.close()
    frames = [(s, t) for s in range(S) for t in range(T)]
    rb = Run(pool, S * T)
    rows = batch_call(rb, pool, [content(*f) for f in frames], [i if f[1] == 0 else i - 1 for i, f in enumerate(frames)])
    rb.close()
    for i, f in enumerate(frames):
        same_row(got[f], rows[i], f)
    assert all(got[s, 0]['info'][3] == 3 and np.isnan(got[s, 0]['F']).all() and got[s, 0]['cnt'] == got[s, 0]['n_all'] for s in range(S)), 'first frames'
    assert any(filtered(got[s, t], got[s, t - 1]) for s in range(S) for t in range(2, T)), 'no frame had its pairs filtered by the previous boxes'
    q13 = [s for s in range(S) if got[s, 0]['have'] and got[s, 0]['nb'] > 0 and got[s, 1]['info'][0] == got[s, 1]['n_all'] and got[s, 1]['info'][3] != 3]
    assert q13, 'no first frame with person boxes whose second frame uses every pair (quirk Q13)'


# ---- 2. gaps and restarts ------------------------------------------------------------------------------------------------------------------------
# stream A on slot 0 (restarted with new_stream at its third frame), B on slot 1, C on slot 2 (skips the second call), D on the never-used slot 3
GAP_CALLS = [([('A', 0), ('B', 0), ('C', 0)], [0, 1, 2], None),
             ([('B', 1), ('A', 1)], [1, 0], None),
             ([('C', 1), ('A', 2), ('B', 2), ('D', 0)], [2, 0, 1, 3], [0, 1, 0, 0]),
             ([('A', 3), ('C', 2)], [0, 2], [0, 0])]
GAP_CONTENT = dict(A=0, B=4, C=8, D=12)
GAP_FIRST = {('A', 0), ('B', 0), ('C', 0), ('A', 2), ('D', 0)}


def gap_batch(rb, pool):
    frames = [f for call in GAP_CALLS for f in call[0]]
    pidx = [i if f in GAP_FIRST else frames.index((f[0], f[1] - 1)) for i, f in enumerate(frames)]
    return dict(zip(frames, batch_call(rb, pool, [GAP_CONTENT[s] + t for s, t in frames], pidx)))


def test_gaps_and_restarts_equal_the_batch_step(pool):
    rs = Run(pool, 6)
    got = {}
    for frames, slots, new in GAP_CALLS:
        got.update(zip(frames, stream_call(rs, pool, [GAP_CONTENT[s] + t for s, t in frames], slots, new)))
    rs.close()
    rb = Run(pool, 16)
    ref = gap_batch(rb, pool)
    rb.close()
    for f in ref:
        same_row(got[f], ref[f], f)
    # C1 (after C skipped a call) and A3 (after A's restart) have a previous frame; A2, D0 and the first frames of the first call do not
    for f in got:
        assert (got[f]['info'][3] == 3) == (f in GAP_FIRST), f


# ---- 3. host buffers against device buffers ------------------------------------------------------------------------------------------------------
def test_host_variant_equals_device_variant(pool):
    rd, rh = Run(pool, 6), Run(pool, 6)
    kws = [dict(), dict(pinned=True, depth_f32=True, rgb_pad=48, depth_pad=64), dict(rgb_pad=3, depth_pad=2), dict(pinned=True, depth_f32=True)]
    for (frames, slots, new), kw in zip(GAP_CALLS, kws):
        content = [GAP_CONTENT[s] + t for s, t in frames]
        d = stream_call(rd, pool, content, slots, new)
        h = host_rows(rh, pool, content, slots, new=new, **kw)
        for f, a, b in zip(frames, d, h):
            same_row(a, b, (f, kw))
    rd.close(); rh.close()


# ---- 4. batch calls on the same handle leave the slots alone -------------------------------------------------------------------------------------
def pose_chain(r, pool, content, n):
    """sgs_tracker_pose_chain_device after the last step of r, on a synthetic local map (as tests/test_gpu_grab_rgbd.py builds it)."""
    import bench
    import torch
    ti = {k: a[content] for k, a in pool['ti'].items() if k != 'sf'}
    rows = collect(r.trk, n)
    mcap, cap, sf = 1536, r.trk.cap, pool['sf']
    rng = np.random.default_rng(5)
    lms = [bench.make_local_map(f, rows[f]['kun'], rows[f]['desc'], int(rows[f]['cnt']), ti, mcap, synth.TUM3, sf, rng, W, H) for f in range(n)]
    stack = lambda k, dt: dev(np.stack([m[k] for m in lms]).astype(dt))
    lm = dict(lid=stack('lid', np.int32), xyz=stack('xyz', np.float32), nrm=stack('nrm', np.float32), mn=stack('mn', np.float32), mx=stack('mx', np.float32),
              dsc=stack('dsc', np.uint8), valid=stack('valid', np.uint8), obs=stack('obs', np.uint8), n=dev(np.array([m['n'] for m in lms], np.int32)))
    last = [dev(ti[k]) for k in LAST]
    o = dict(T1=torch.zeros((n, 16), device='cuda'), T2=torch.zeros((n, 16), device='cuda'), mp=torch.zeros((n, cap), dtype=torch.int32, device='cuda'),
             outl=torch.zeros((n, cap), dtype=torch.uint8, device='cuda'), st=torch.zeros((n, 8), dtype=torch.int32, device='cuda'))
    a = B.PoseChainBatch()
    a.last_xyz, a.last_desc, a.last_flags, a.last_octave, a.last_angle, a.last_n, a.tcw_cur, a.tcw_last = [t.data_ptr() for t in last]
    a.th, a.mono, a.check_orientation, a.last_local_id = TH, 0, 1, lm['lid'].data_ptr()
    a.mp_xyz, a.mp_normal, a.mp_min_dist, a.mp_max_dist = lm['xyz'].data_ptr(), lm['nrm'].data_ptr(), lm['mn'].data_ptr(), lm['mx'].data_ptr()
    a.mp_desc, a.mp_valid, a.mp_obs, a.mp_n, a.mp_cap = lm['dsc'].data_ptr(), lm['valid'].data_ptr(), lm['obs'].data_ptr(), lm['n'].data_ptr(), mcap
    a.th_local, a.nnratio_local = 3.0, 0.8
    for l in range(8):
        a.inv_level_sigma2[l] = float(1.0 / np.float32(sf[l]) ** 2)
    a.tcw_motion, a.tcw_final, a.f_mp, a.outlier, a.stats = o['T1'].data_ptr(), o['T2'].data_ptr(), o['mp'].data_ptr(), o['outl'].data_ptr(), o['st'].data_ptr()
    B.check(B.lib().sgs_tracker_pose_chain_device(r.trk.h, C.byref(a), n, v(0)))
    torch.cuda.synchronize()
    return o['st'].cpu().numpy()


def test_batch_calls_between_stream_calls_change_nothing(pool):
    import torch
    calls = [([0, 4, 8], [0, 1, 2]), ([9, 1], [2, 0]), ([5, 2, 10], [1, 0, 2])]
    ra, rb = Run(pool, 4), Run(pool, 4)
    for content, slots in calls[:2]:
        for r in (ra, rb):
            stream_call(r, pool, content, slots)
    # on ra only: a batch RGB-D step over other frames, the pose chain after it, and the tracker's LK handle used directly
    bc = [12, 13, 14, 15]
    before = batch_call(ra, pool, bc, [0, 0, 1, 2])
    assert sum(int(r['nb']) for r in before) > 0
    assert pose_chain(ra, pool, bc, 4)[:, 0].sum() > 0
    gray = dev(GR.to_gray(pool['rgb'][bc], 1))
    k, c, prev = v(), v(), torch.zeros((4, ra.trk.cap, 2), dtype=torch.float32, device='cuda')
    B.check(B.lib().sgs_tracker_results_device(ra.trk.h, C.byref(k), None, None, C.byref(c), None, None, None))
    B.check(B.lib().sgs_lk_track_batch_device(B.lib().sgs_tracker_lk(ra.trk.h), gray.data_ptr(), gray.data_ptr() + W * H, None, 3, W * H, W, k.value, c.value,
                                              ra.trk.cap, prev.data_ptr(), v(0)))
    torch.cuda.synchronize()
    a = stream_call(ra, pool, *calls[2])
    b = stream_call(rb, pool, *calls[2])
    for i in range(len(a)):
        same_row(a[i], b[i], i)
    assert all(r['info'][3] != 3 for r in a)
    # and the pose chain after a stream call runs as after an RGB-D step
    assert pose_chain(ra, pool, calls[2][0], 3)[:, 0].sum() > 0
    ra.close(); rb.close()


# ---- 5. refusals change nothing ------------------------------------------------------------------------------------------------------------------
def test_refused_calls_change_no_slot(pool):
    import torch
    ra, rb = Run(pool, 4), Run(pool, 4)
    first = ([0, 4], [0, 1])
    for r in (ra, rb):
        host_rows(r, pool, *first)
    content = [5, 1]
    refused = [dict(nframes=0), dict(nframes=5), dict(slots=[-1, 1]), dict(slots=[0, 4]), dict(slots=[1, 1]), dict(slot_arg=False)]
    for case in refused:
        kw = dict(case)
        slots = kw.pop('slots', [1, 0])
        rc, _ = host_call(ra, pool, content, slots, **kw)
        assert rc == B.SGS_ERR_INVALID, case
        assert B.lib().sgs_last_error().decode().startswith('sgs_tracker_step_rgbd_stream:'), case
    rgb, depth, last = device_inputs(pool, content)
    d_slot = dev(np.array([1, 0], np.int32))
    for n, sp in ((0, d_slot.data_ptr()), (5, d_slot.data_ptr()), (2, None)):
        rc = B.lib().sgs_tracker_step_rgbd_stream_device(ra.trk.h, ra.det.h, rgb.data_ptr(), H * W * 3, W * 3, depth.data_ptr(), H * W * 2, W * 2,
                                                         C.byref(fmt_of(B.DEPTH_U16, FACTOR)), n, sp, None, *[t.data_ptr() for t in last], TH, 0, 1, v(0))
        assert rc == B.SGS_ERR_INVALID, n
    torch.cuda.synchronize()
    a = host_rows(ra, pool, content, [1, 0])
    b = host_rows(rb, pool, content, [1, 0])
    for i in range(2):
        same_row(a[i], b[i], i)
        assert a[i]['info'][3] != 3
    ra.close(); rb.close()


# ---- 6. at size ----------------------------------------------------------------------------------------------------------------------------------
def test_at_size_against_the_batch_formulation(pool):
    """64 streams x 20 calls with skips and restarts; every call against a batch of its new frames plus their previous frames."""
    S, T = 64, 20
    rng = np.random.default_rng(7)
    rs, rb = Run(pool, S), Run(pool, 2 * S)
    last = {}                               # stream -> (content of its last frame, whether that frame was a first frame)
    paths = dict(first=0, filtered=0, restart=0, skip=0)
    for t in range(T):
        order = [int(s) for s in rng.permutation([s for s in range(S) if t == 0 or (7 * s + t) % 9 != 0])]
        new = [1 if t > 0 and (5 * s + t) % 13 == 0 else 0 for s in order]
        content = [(3 * s + t) % POOL for s in order]
        got = stream_call(rs, pool, content, order, new)
        n = len(order)
        bc, pidx = list(content), list(range(n))
        for i, s in enumerate(order):
            if s in last and not new[i]:
                c, was_first = last[s]
                j = len(bc)
                bc.append(c); pidx[i] = j
                pidx.append(j if was_first else i)        # a previous frame that was not a first frame must not be its own predecessor (quirk Q13)
        ref = batch_call(rb, pool, bc, pidx)
        for i, s in enumerate(order):
            same_row(got[i], ref[i], (t, s))
            first = s not in last or bool(new[i])
            paths['first'] += first; paths['restart'] += s in last and bool(new[i])
            paths['skip'] += t > 1 and (7 * s + t - 1) % 9 == 0 and not first
            paths['filtered'] += (not first and pidx[pidx[i]] != pidx[i] and bool(ref[pidx[i]]['have']) and 20 < got[i]['info'][0] < got[i]['n_all'])
            assert (got[i]['info'][3] == 3) == first, (t, s)
            last[s] = (content[i], first)
    rs.close(); rb.close()
    assert all(paths.values()), paths
