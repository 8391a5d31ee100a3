"""The detector at the benchmark's batch sizes (bench.CONFIGS: 512 frames of 640 x 480, 192 frames of 1280 x 720), against the same frames run through
an 8-frame handle in 8-frame calls, bit for bit.

At the benchmark's batches the planner picks other GEMM tilings than at 8 frames (output-channel tiles, ring depth: the cost model counts waves of
the persistent grid), and each persistent GEMM CTA walks 100 or more pixel tiles on the largest layers instead of a few.  Every kernel computes an
element from the same operands in the same order at any batch size (the k-blocking depends on Cin only, and the tile width changes no bits:
tests/test_gpu_detector_wgmma_width.py), so the outputs must be identical, not close.

  frames   64 synthetic scenes, each repeated with a shift of a few pixels per repeat: every frame differs, and (proof) at least 95 % of the frames
           have detection rows of their own at a low threshold;
  graphs   the reference model (when build() staged it), the synthetic mini graph and the wide-tail graph;
  checks   one fused call at the full batch: per frame, rows, objects, dynamic boxes, their counts, the flag and the status equal the 8-frame calls';
           the same handle then called on 3 frames fewer and on 1 frame gives the same per-frame outputs; for the synthetic graphs, every blob of a
           DET_KEEP_BLOBS handle at the full batch equals the 8-frame handle's, per frame (SHA-256 digests)."""
import hashlib
import os
from functools import lru_cache

import numpy as np
import pytest

import detector_model as DM
import detector_resize_cases as RC
from pysgs import binding as B

REAL = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle', '_ref', 'ncnn_model', 'mobilenetv3_ssdlite_voc')
HAVE_REAL = os.path.exists(REAL + '.param')
CONFIGS = RC.bench_batches()
SCENES = 64
DET_THR = 0.05
POOL_LIMIT = 16 << 30
KEYS = ('rows', 'nrows', 'objects', 'nobjects', 'dyn_map', 'ndyn_map', 'dyn_rm', 'ndyn_rm', 'have', 'status')


@lru_cache(maxsize=None)
def scale_frames(w, h, n):
    """n frames h x w x 3: frame i is scene i % 64 shifted by (2k, 3k) pixels, k = i // 64 (np.roll: nothing leaves the frame)"""
    scenes = [DM.synthetic_rgb(h, w, 1000 + s) for s in range(SCENES)]
    out = np.empty((n, h, w, 3), np.uint8)
    for i in range(n):
        k = i // SCENES
        out[i] = np.roll(scenes[i % SCENES], (2 * k, 3 * k), axis=(0, 1))
    return out


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def test_batches_follow_the_benchmark():
    assert sorted((w, h, b) for w, h, b in CONFIGS.values()) == [(640, 480, 512), (1280, 720, 192)]
    for w, h, b in CONFIGS.values():
        fr = scale_frames(w, h, b)
        assert fr.shape == (b, h, w, 3) and len({_sha(f) for f in fr}) == b, (w, h, b)


@pytest.fixture(scope='module')
def graphs(tmp_path_factory):
    d = str(tmp_path_factory.mktemp('at_scale'))
    g = {'mini': DM.write_mini_model(os.path.join(d, 'mini'), 0), 'wide_tails': DM.write_wide_tail_model(os.path.join(d, 'wide'), 0)[:2]}
    if HAVE_REAL:
        g['reference'] = (REAL + '.param', REAL + '.bin')
    return g


needs_real = pytest.mark.skipif(not HAVE_REAL, reason='reference model copy (oracle/_ref/ncnn_model, made by build()) not present')
GRAPHS = [pytest.param('reference', marks=needs_real), 'mini', 'wide_tails']


def _frame(o, f):
    """frame f's outputs: every array cut at its count"""
    n = {k: int(o['n' + k][f]) for k in ('rows', 'objects', 'dyn_map', 'dyn_rm')}
    return {k: (o[k][f, :n[k]] if k in n else o[k][f]).tobytes() for k in KEYS}


def _small_batches(det, fr):
    from test_gpu_detector import _run
    parts = [_run(det, fr[i:i + RC.PROBE]) for i in range(0, len(fr), RC.PROBE)]
    return {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}


def _compare(what, got, ref, frames_):
    """frames_[i] of ref against frame i of got"""
    bad = []
    for i, f in enumerate(frames_):
        a, b = _frame(got, i), _frame(ref, f)
        bad += ['frame %d: %s' % (f, k) for k in KEYS if a[k] != b[k]]
    assert not bad, '%s: %d differences, first %s' % (what, len(bad), bad[:8])


def _check_scale(p, nb, name):
    """the full-batch handle's plan walks many pixel tiles per persistent CTA"""
    top = max(RC.tiles_per_cta(q, nb) for q in p)
    assert top >= RC.SCALE_TILES[name] or nb < 512, (name, nb, top)
    return top


@pytest.mark.gpu
@pytest.mark.parametrize('config', sorted(CONFIGS))
@pytest.mark.parametrize('name', GRAPHS)
def test_full_batch_equals_8_frame_calls(graphs, name, config):
    from test_gpu_detector import _run
    w, h, nb = CONFIGS[config]
    pp, bp = graphs[name]
    fr = scale_frames(w, h, nb)
    big = B.Detector(pp, bp, max_frames=nb, det_thr=DET_THR)
    small = B.Detector(pp, bp, max_frames=RC.PROBE, det_thr=DET_THR)
    top = _check_scale(DM.parse_plan(big.describe()), nb, name)
    ref = _small_batches(small, fr)
    small.close()
    digests = {_sha(ref['rows'][f, :ref['nrows'][f]]) for f in range(nb)}
    assert len(digests) >= 0.95 * nb, '%d distinct detection-row sets in %d frames' % (len(digests), nb)
    _compare('%s %s, %d frames in one call' % (name, config, nb), _run(big, fr), ref, range(nb))
    _compare('%s %s, %d frames after a full batch' % (name, config, nb - 3), _run(big, fr[:nb - 3]), ref, range(nb - 3))
    _compare('%s %s, frame %d alone after a full batch' % (name, config, nb - 1), _run(big, fr[nb - 1:]), ref, [nb - 1])
    big.close()
    print('\n%s %s: %d frames equal bit for bit (%d distinct row sets, %d+ pixel tiles per persistent CTA)' % (name, config, nb, len(digests), top))


def _blob_digests(det, names, nf):
    return {n: [_sha(det.blob(n, f)) for f in range(nf)] for n in names}


@pytest.mark.gpu
@pytest.mark.parametrize('config', sorted(CONFIGS))
@pytest.mark.parametrize('name', ['mini', 'wide_tails'])
def test_every_blob_at_the_full_batch(graphs, name, config):
    from test_gpu_detector import _run
    w, h, nb = CONFIGS[config]
    pp, bp = graphs[name]
    need = RC.pool_bytes(pp, bp, nb, B.DET_KEEP_BLOBS)
    if need > POOL_LIMIT:
        pytest.skip('DET_KEEP_BLOBS pool of %.1f GB at %d frames' % (need / 2 ** 30, nb))
    fr = scale_frames(w, h, nb)
    big = B.Detector(pp, bp, max_frames=nb, flags=B.DET_KEEP_BLOBS)
    lines = big.describe().splitlines()[1:]
    names = ['input'] + list(dict.fromkeys(l.split()[l.split().index('out') + 1] for l in lines))
    _check_scale(DM.parse_plan(big.describe()), nb, name)
    _run(big, fr)
    got = _blob_digests(big, names, nb)
    big.close()
    small = B.Detector(pp, bp, max_frames=RC.PROBE, flags=B.DET_KEEP_BLOBS)
    ref = {n: [] for n in names}
    for i in range(0, nb, RC.PROBE):
        _run(small, fr[i:i + RC.PROBE])
        for n, d in _blob_digests(small, names, RC.PROBE).items():
            ref[n] += d
    small.close()
    bad = [(n, f) for n in names for f in range(nb) if got[n][f] != ref[n][f]]
    assert not bad, '%d (blob, frame) pairs differ; in graph order, first: %s' % (len(bad), bad[:8])
    print('\n%s %s: %d blobs x %d frames equal bit for bit (pool %.2f GB)' % (name, config, len(names), nb, need / 2 ** 30))
