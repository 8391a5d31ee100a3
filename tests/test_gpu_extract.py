"""GPU parity: the CUDA extractor (through the C ABI) against the CPU oracle and the golden fixtures.  Bit-exact."""
import ctypes as C
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import oracle as O  # noqa: E402
from pysgs import binding as B  # noqa: E402
from pysgs import synth  # noqa: E402


def _sorted_cands(c):
    c = np.asarray(c, np.int64).reshape(-1, 3)
    return c[np.lexsort((c[:, 0], c[:, 1]))]


def _check_against_oracle(img, nfeat=1000, nlev=8, stages=True):
    p = O.params(nfeat, 1.2, nlev, 20, 7)
    d = O.ExtractDump(img, p)
    ex = B.Extractor(img.shape[1], img.shape[0], nfeat, 1.2, nlev, 20, 7, max_batch=2)
    try:
        t = ex.tables(); to = O.orb_tables(p)
        assert t['nPerLevel'].tolist() == to['nPerLevel'].tolist()
        assert t['scale'].view(np.uint32).tolist() == to['scale'].view(np.uint32).tolist()
        kps, desc = ex.extract(img)
        if stages:
            for lvl in range(nlev):
                assert np.array_equal(ex.read_level(0, lvl, False), d.pyramid[lvl]), 'pyramid level %d' % lvl
                got = _sorted_cands(ex.read_candidates(0, lvl)); ref = _sorted_cands(d.cands[lvl])
                assert np.array_equal(got, ref), 'FAST candidates level %d (%d vs %d)' % (lvl, len(got), len(ref))
                if d.blurred[lvl] is not None:
                    assert np.array_equal(ex.read_level(0, lvl, True), d.blurred[lvl]), 'blur level %d' % lvl
        assert len(kps) == len(d.kps)
        for fld in ('x', 'y', 'size', 'response', 'octave', 'class_id'):
            assert np.array_equal(kps[fld], d.kps[fld]), fld
        assert np.array_equal(kps['angle'].view(np.uint32), d.kps['angle'].view(np.uint32)), 'angles (bitwise)'
        assert kps.tobytes() == d.kps.tobytes()
        assert np.array_equal(desc, d.desc), 'descriptors: %d rows differ' % int((desc != d.desc).any(1).sum())
    finally:
        ex.close()
    return len(kps)


def test_s1_640x480_all_stages():
    assert _check_against_oracle(synth.frame_s1(640, 480, 1)) > 900


@pytest.mark.parametrize('name', ['s1_640x480', 's1_320x240', 'noise_200x160'])
def test_against_golden_fixture(golden_dir, name):
    g = np.load(os.path.join(golden_dir, 'extract_%s.npz' % name))
    nfeat, nlev, ini, mn = [int(v) for v in g['params']]
    img = g['image']
    ex = B.Extractor(img.shape[1], img.shape[0], nfeat, 1.2, nlev, ini, mn)
    try:
        kps, desc = ex.extract(img)
        assert kps.tobytes() == g['kps'].tobytes()
        assert np.array_equal(desc, g['desc'])
        assert np.array_equal(ex.read_level(0, nlev - 1, False), g['pyr_last'])
        assert np.array_equal(ex.read_level(0, nlev - 1, True), g['blur_last'])
    finally:
        ex.close()


def test_other_geometries_and_params():
    _check_against_oracle(synth.frame_s1(1280, 720, 4), nfeat=2000)          # config B (2 quadtree roots)
    _check_against_oracle(synth.frame_s1(752, 480, 5), nfeat=1200, stages=False)
    _check_against_oracle(synth.frame_s1(333, 257, 6), nfeat=300, nlev=5)    # odd sizes, unaligned pitches


def test_edge_images():
    # constant image: no corners anywhere -> zero keypoints, like the reference (descriptors released, :1067)
    assert _check_against_oracle(np.full((480, 640), 77, np.uint8)) == 0
    # pure noise: tens of thousands of candidates per level -> exercises the global-memory sort path of the quadtree
    rng = np.random.RandomState(3)
    _check_against_oracle(rng.randint(0, 256, (480, 640)).astype(np.uint8))
    # checkerboard-ish texture with many equal FAST scores (tie-breaks)
    yy, xx = np.mgrid[0:240, 0:320]
    img = (((xx // 6 + yy // 6) % 2) * 120 + 60).astype(np.uint8)
    _check_against_oracle(img, nfeat=500)


def test_empty_image_returns_zero():
    ex = B.Extractor(640, 480)
    try:
        import ctypes as C
        n = C.c_int(5)
        B.check(B.lib().sgs_extract(ex.h, None, 640, 480, 640, None, None, 0, C.byref(n)))
        assert n.value == 0
    finally:
        ex.close()


def test_batch_matches_single_and_is_order_independent():
    frames, _ = synth.stream_s2(6, 640, 480, seed=2)
    ex = B.Extractor(640, 480, max_batch=6)
    ex1 = B.Extractor(640, 480, max_batch=1)
    try:
        kps, desc, n = ex.extract_batch(frames)
        for f in range(len(frames)):
            k1, d1 = ex1.extract(frames[f])
            assert n[f] == len(k1)
            assert kps[f, :n[f]].tobytes() == k1.tobytes() and np.array_equal(desc[f, :n[f]], d1)
            ko, do = O.extract(frames[f])
            assert k1.tobytes() == ko.tobytes() and np.array_equal(d1, do)
        # run-to-run determinism (atomics only order the unordered candidate lists)
        kps2, desc2, n2 = ex.extract_batch(frames)
        assert np.array_equal(n, n2) and kps.tobytes() == kps2.tobytes() and np.array_equal(desc, desc2)
    finally:
        ex.close(); ex1.close()


def test_strided_input_pitch():
    img = synth.frame_s1(640, 480, 9)
    padded = np.zeros((480, 700), np.uint8); padded[:, :640] = img
    ex = B.Extractor(640, 480)
    try:
        import ctypes as C
        kps = np.zeros(ex.cap, B.KP_DTYPE); desc = np.zeros((ex.cap, 32), np.uint8); n = C.c_int()
        B.check(B.lib().sgs_extract(ex.h, padded.ctypes.data_as(C.c_void_p), 640, 480, 700, kps.ctypes.data_as(C.c_void_p),
                                    desc.ctypes.data_as(C.c_void_p), ex.cap, C.byref(n)))
        ko, do = O.extract(img)
        assert kps[:n.value].tobytes() == ko.tobytes() and np.array_equal(desc[:n.value], do)
    finally:
        ex.close()


def test_device_resident_batch_with_torch():
    import torch
    frames, _ = synth.stream_s2(4, 640, 480, seed=11)
    ex = B.Extractor(640, 480, max_batch=4)
    try:
        d = torch.from_numpy(frames).cuda()
        st = torch.cuda.Stream()
        torch.cuda.synchronize()
        with torch.cuda.stream(st):
            ex.extract_batch_device(d.data_ptr(), 4, 640 * 480, 640, st.cuda_stream)
        kps, desc, counts = ex.fetch(4, st.cuda_stream)
        kptr, dptr, cptr, cap = ex.results_device()
        assert kptr and dptr and cptr and cap == ex.cap
        for f in range(4):
            ko, do = O.extract(frames[f])
            assert counts[f] == len(ko)
            assert kps[f, :counts[f]].tobytes() == ko.tobytes() and np.array_equal(desc[f, :counts[f]], do)
    finally:
        ex.close()


def test_large_pinned_batch_goes_up_in_chunks():
    """>= 64 pinned frames take the chunked upload path (copy stream ahead of the kernels): results must equal the unchunked ones."""
    import torch
    base, _ = synth.stream_s2(6, 640, 480, seed=12)
    nf = 70          # two chunks of 35
    frames = np.stack([np.roll(base[i % 6], 3 * (i // 6), 1) for i in range(nf)])
    ex = B.Extractor(640, 480, max_batch=nf)
    try:
        ref_k, ref_d, ref_n = ex.extract_batch(frames)                       # pageable input: staging path, one enqueue
        pin = torch.from_numpy(frames).pin_memory()
        hk = torch.zeros((nf, ex.cap, 28), dtype=torch.uint8).pin_memory(); hd = torch.zeros((nf, ex.cap, 32), dtype=torch.uint8).pin_memory()
        n = np.zeros(nf, np.int32)
        B.check(B.lib().sgs_extract_batch(ex.h, C.c_void_p(pin.data_ptr()), nf, 640 * 480, 640, C.c_void_p(hk.data_ptr()), C.c_void_p(hd.data_ptr()), ex.cap,
                                          n.ctypes.data_as(C.c_void_p)))
        assert np.array_equal(n, ref_n)
        k = hk.numpy().reshape(nf, ex.cap * 28).view(B.KP_DTYPE).reshape(nf, ex.cap)
        for f in range(nf):
            assert k[f, :n[f]].tobytes() == ref_k[f, :n[f]].tobytes() and np.array_equal(hd.numpy()[f, :n[f]], ref_d[f, :n[f]]), f
        for f in (0, 34, 35, 69):
            ok, od = O.extract(frames[f])
            assert k[f, :n[f]].tobytes() == ok.tobytes() and np.array_equal(hd.numpy()[f, :n[f]], od)
    finally:
        ex.close()
