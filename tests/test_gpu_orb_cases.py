"""Every constructed extractor case of tests/orb_cases.py through the device, bit for bit against the oracle's per-stage output
(oracle.ExtractDump): pyramid, sorted FAST candidates per level, blurred levels, keypoints (angles bitwise) and descriptors.  The same cases go
through every way a frame reaches the kernels: sgs_extract; sgs_extract_batch with the cases of one geometry in shuffled order;
sgs_extract_batch_device once on a 16-byte-aligned buffer (TMA tiles) and once on a base offset by 1..15 bytes with an odd pitch (plain-load
tiles); and a chunked pinned batch, whose second chunk addresses the TMA map with frame0 > 0.  The parameter sets sgs_extractor_create refuses
come back with their status and message and leave the library usable."""
import ctypes as C

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle as O  # noqa: E402
import orb_cases as OC  # noqa: E402
from pysgs import binding as B  # noqa: E402

CASES = OC.all_cases()
_dumps = {}


def dump(c):
    if c['name'] not in _dumps:
        _dumps[c['name']] = O.ExtractDump(c['img'], OC.oparams(c['p']))
    return _dumps[c['name']]


def extractor(c, max_batch=1):
    p = c['p']
    h, w = c['img'].shape
    return B.Extractor(w, h, p['nfeatures'], p['scale'], p['nlevels'], p['ini'], p['mn'], max_batch=max_batch)


def _sorted_cands(a):
    a = np.asarray(a, np.int64).reshape(-1, 3)
    return a[np.lexsort((a[:, 0], a[:, 1]))]


def same_as_oracle(kps, desc, d, name):
    assert len(kps) == len(d.kps), (name, len(kps), len(d.kps))
    for f in ('x', 'y', 'size', 'response', 'octave', 'class_id'):
        assert np.array_equal(kps[f], d.kps[f]), (name, f)
    assert np.array_equal(kps['angle'].view(np.uint32), d.kps['angle'].view(np.uint32)), (name, 'angles (bitwise)')
    assert kps.tobytes() == d.kps.tobytes(), name
    assert np.array_equal(desc, d.desc), (name, 'descriptors: %d rows differ' % int((desc != d.desc).any(1).sum()))


@pytest.mark.parametrize('c', CASES, ids=[c['name'] for c in CASES])
def test_case_every_stage(c):
    d = dump(c)
    ex = extractor(c)
    try:
        kps, desc = ex.extract(c['img'])
        for lvl in range(c['p']['nlevels']):
            assert np.array_equal(ex.read_level(0, lvl, False), d.pyramid[lvl]), 'pyramid level %d' % lvl
            got, ref = _sorted_cands(ex.read_candidates(0, lvl)), _sorted_cands(d.cands[lvl])
            assert np.array_equal(got, ref), 'FAST candidates level %d (%d vs %d)' % (lvl, len(got), len(ref))
            if d.blurred[lvl] is not None:
                assert np.array_equal(ex.read_level(0, lvl, True), d.blurred[lvl]), 'blur level %d' % lvl
        same_as_oracle(kps, desc, d, c['name'])
    finally:
        ex.close()


def groups(min_size=2):
    g = {}
    for c in CASES:
        g.setdefault(c['key'], []).append(c)
    return [v for v in g.values() if len(v) >= min_size]


def test_batches_of_one_geometry_in_shuffled_order():
    rng = np.random.RandomState(5)
    ran = 0
    for grp in groups():
        order = list(rng.permutation(len(grp))) + [0]              # a repeat of the first case as well
        frames = np.stack([grp[i]['img'] for i in order])
        ex = extractor(grp[0], max_batch=len(order))
        try:
            kps, desc, n = ex.extract_batch(frames)
        finally:
            ex.close()
        for f, i in enumerate(order):
            same_as_oracle(kps[f, :n[f]], desc[f, :n[f]], dump(grp[i]), grp[i]['name'])
        ran += len(order)
    assert ran >= 30


def _device_run(ex, frames, base_off, pitch):
    """Frames copied into one device buffer at byte offset base_off with row pitch `pitch`; sgs_extract_batch_device, then fetch."""
    import torch
    F, h, w = frames.shape
    fstride = pitch * h
    buf = torch.zeros(base_off + F * fstride + 64, dtype=torch.uint8, device='cuda')
    host = np.zeros(F * fstride, np.uint8)
    host.reshape(F, h, pitch)[:, :, :w] = frames
    buf[base_off:base_off + F * fstride].copy_(torch.from_numpy(host))
    torch.cuda.synchronize()
    ex.extract_batch_device(buf.data_ptr() + base_off, F, fstride, pitch)
    out = ex.fetch(F)
    del buf
    return out


def test_device_input_aligned_and_unaligned():
    """The TMA instance (aligned base, pitch and frame stride) and the plain-load instance (base offset by 1..15 bytes, odd pitch) must give the
    same bytes, equal to the oracle, on every geometry of the cases."""
    seen = {}
    for c in CASES:
        seen.setdefault(c['key'], []).append(c)
    for k, (key, grp) in enumerate(sorted(seen.items(), key=lambda kv: kv[1][0]['name'])):
        grp = grp[:4]
        frames = np.stack([c['img'] for c in grp])
        h, w = frames.shape[1:]
        ex = extractor(grp[0], max_batch=len(grp))
        try:
            ka, da, na = _device_run(ex, frames, 0, (w + 15) // 16 * 16)
            off = 1 + k % 15
            kb, db, nb = _device_run(ex, frames, off, w + 1 + 2 * (k % 7) if (w + 1) % 2 else w + 2 + 2 * (k % 7))
        finally:
            ex.close()
        assert np.array_equal(na, nb)
        for f, c in enumerate(grp):
            assert ka[f, :na[f]].tobytes() == kb[f, :nb[f]].tobytes() and np.array_equal(da[f, :na[f]], db[f, :nb[f]]), c['name']
            same_as_oracle(ka[f, :na[f]], da[f, :na[f]], dump(c), c['name'])


def test_chunked_pinned_batch_covers_cases():
    """64 pinned frames go up in two chunks; the cases sit in both, so the second chunk's tiles address the TMA map with frame0 = 32."""
    import torch
    grp = max(groups(), key=len)
    h, w = grp[0]['img'].shape
    nf = 64
    pick = [i % len(grp) for i in range(nf)]
    frames = np.stack([grp[i]['img'] for i in pick])
    ex = extractor(grp[0], max_batch=nf)
    try:
        pin = torch.from_numpy(frames).pin_memory()
        hk = torch.zeros((nf, ex.cap, 28), dtype=torch.uint8).pin_memory(); hd = torch.zeros((nf, ex.cap, 32), dtype=torch.uint8).pin_memory()
        n = np.zeros(nf, np.int32)
        B.check(B.lib().sgs_extract_batch(ex.h, C.c_void_p(pin.data_ptr()), nf, w * h, w, C.c_void_p(hk.data_ptr()), C.c_void_p(hd.data_ptr()), ex.cap,
                                          n.ctypes.data_as(C.c_void_p)))
    finally:
        ex.close()
    k = hk.numpy().reshape(nf, ex.cap * 28).view(B.KP_DTYPE).reshape(nf, ex.cap)
    for f in range(nf):
        c = grp[pick[f]]
        same_as_oracle(k[f, :n[f]], hd.numpy()[f, :n[f]], dump(c), '%s (frame %d)' % (c['name'], f))


def test_refusals_and_accepted_limits():
    refused, nmax = OC.refusals()
    assert nmax == 1393
    for name, w, h, p, status, word in refused:
        prm = B.OrbParams(p['nfeatures'], p['scale'], p['nlevels'], p['ini'], p['mn'])
        hdl = C.c_void_p()
        rc = B.lib().sgs_extractor_create(C.byref(prm), w, h, 1, 0, C.byref(hdl))
        msg = B.lib().sgs_last_error().decode()
        assert rc == status and not hdl.value and word in msg, (name, rc, msg)
    for w, h, p in OC.accepted_limits():
        ex = B.Extractor(w, h, p['nfeatures'], p['scale'], p['nlevels'], p['ini'], p['mn'])
        ex.close()
    # a refused call leaves its handle usable
    c = CASES[0]
    ex = extractor(c)
    try:
        kps = np.zeros(ex.cap, B.KP_DTYPE); desc = np.zeros((ex.cap, 32), np.uint8); n = C.c_int()
        img = np.zeros((c['img'].shape[0] + 1, c['img'].shape[1]), np.uint8)
        rc = B.lib().sgs_extract(ex.h, img.ctypes.data_as(C.c_void_p), img.shape[1], img.shape[0], img.shape[1], kps.ctypes.data_as(C.c_void_p),
                                 desc.ctypes.data_as(C.c_void_p), ex.cap, C.byref(n))
        assert rc == B.SGS_ERR_INVALID and 'geometry' in B.lib().sgs_last_error().decode()
        rc = B.lib().sgs_extract_batch(ex.h, c['img'].ctypes.data_as(C.c_void_p), 2, c['img'].size, c['img'].shape[1], kps.ctypes.data_as(C.c_void_p),
                                       desc.ctypes.data_as(C.c_void_p), ex.cap, C.byref(n))
        assert rc == B.SGS_ERR_INVALID and 'max_batch' in B.lib().sgs_last_error().decode()
        k, dsc = ex.extract(c['img'])
        same_as_oracle(k, dsc, dump(c), c['name'])
    finally:
        ex.close()
