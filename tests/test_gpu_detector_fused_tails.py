"""The detector GEMM's fused element-wise tails on wide tiles (conv1x1_tc.cuh, 64 to 256 output channels per tile), read back from fused execution.

The production schedule applies each GEMM's tail (ReLU, clip, hard-swish, +tensor, SE gate, SE tail or the generic chain: EpiFnK / apply_epi of
detector.cu) in the epilogue, and reuses activation buffers.  DET_KEEP_BLOBS (flags bit 2) plans that same schedule but gives every materialised
blob a buffer of its own, so that a fused tail's output can be read and compared, element by element, with diagnostic mode (bit 0: every layer its
own kernel).  The graph is write_wide_tail_model (tests/detector_model.py): every tail kind at every tile width NT = 32 ... 256, both k-block
widths, streamed weights, several N-tiles with a partial last one, odd channel counts (scalar stores) and partial last pixel tiles.

  CPU (plan-only handles): the plan reaches every (kind, NT) cell and edge; bit 2 plans the kernels of flags 0; every (kind, NT, BK) of the reference
       model's fused tails at 8 and 512 frames is among the graph's;
  GPU: each GEMM's pre-tail output against float64 (_gemm_check of test_gpu_detector_kernels.py); fused == per-layer bit for bit; the per-layer tail
       == a float32 numpy restatement of the ncnn layers bit for bit; pooling changes no detection; stale rows of an earlier batch and a frame's
       batch position change no tail output; and on the reference model every blob both handles hold is equal bit for bit."""
import os
import re

import numpy as np
import pytest

import detector_model as DM
from pysgs import binding as B

REAL = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle', '_ref', 'ncnn_model', 'mobilenetv3_ssdlite_voc')
needs_real = pytest.mark.skipif(not os.path.exists(REAL + '.param'), reason='reference model copy (oracle/_ref/ncnn_model, made by build()) not present')
F = DM.PROBE_FRAMES
DET_THR = 0.05


def _describe(pp, bp, flags, max_frames=F):
    d = B.Detector(pp, bp, max_frames=max_frames, flags=flags | B.DET_PLAN_ONLY)
    txt = d.describe()
    d.close()
    return txt


@pytest.fixture(scope='module')
def graph(tmp_path_factory):
    return DM.write_wide_tail_model(str(tmp_path_factory.mktemp('wide_tails')), 0)


@pytest.fixture(scope='module')
def plan(graph):
    return DM.plan_tails(_describe(graph[0], graph[1], 0))


def _cells(plans):
    return {(p['kind'], p['nt'], p['bk']) for p in plans if p['kind'] != 'none'}


def _table(cells):
    kinds = sorted({k for k, _, _ in cells}, key=lambda k: DM.TAIL_KINDS.index(k))
    return '\n'.join('  %-8s %s' % (k, '  '.join('%3d:%s' % (nt, '/'.join(str(bk) for bk in (16, 32) if (k, nt, bk) in cells) or '-')
                                                 for nt in range(32, 257, 32))) for k in kinds)


# ---------------------------------------------------------------------------------------------------------------- CPU: plans
def test_plan_covers_every_tail_kind_at_every_width(graph, plan):
    info = graph[2]
    by_out = {p['out']: p for p in plan}
    for c in info:
        p = by_out[c['out']]
        assert p['kind'] == c['kind'] and (p['cin'], p['cout'], p['h']) == (c['cin'], c['cout'], c['hw']), p['line']
    tailed = [p for p in plan if p['kind'] != 'none']
    assert len(tailed) == len(info), [p['line'] for p in tailed if p['out'] not in {c['out'] for c in info}]
    cells = {(p['kind'], p['nt']) for p in tailed}
    missing = [(k, nt) for k in DM.TAIL_KINDS for nt in range(32, 257, 32) if (k, nt) not in cells]
    assert not missing, missing
    for k in DM.TAIL_KINDS:
        assert {p['bk'] for p in tailed if p['kind'] == k} == {16, 32}, k
    for k in ('hswish', 'se_tail'):
        assert any(not p['wres'] and p['kb'] > 1 for p in tailed if p['kind'] == k), 'streamed weights under ' + k
    for k in DM.TENSOR_TAILS:
        ps = [p for p in tailed if p['kind'] == k]
        # several N-tiles (operand index n0 + col), the last one short by at least a 32-channel chunk (the chunk cut-off)
        assert any(p['n_tiles'] >= 2 and p['cout'] - p['nt'] * (p['n_tiles'] - 1) <= p['nt'] - 32 for p in ps), k
        assert any(p['cout'] % 2 and p['nt'] > 32 for p in ps), 'odd Cout on a wide tile (scalar stores) under ' + k
    assert any(p['n_tiles'] >= 4 for p in tailed if p['kind'] == 'hswish')
    assert any(-(-F * p['h'] * p['w'] // 128) > 2 * 132 for p in tailed), 'several pixel tiles per persistent CTA'
    for p in tailed:
        assert (F * p['h'] * p['w']) % 128, 'partial last pixel tile: ' + p['line']
    print('\nwide-tail graph at %d frames, (kind: NT:BK):\n%s' % (F, _table(_cells(plan))))


def _plan_lines(text):
    """describe() lines without buffer numbers; the first line without the pool size"""
    lines = text.splitlines()
    return [' '.join(lines[0].split()[:4])] + [re.sub(r' buf -?\d+', '', l) for l in lines[1:]]


def test_keep_blobs_plans_the_fused_schedule(graph, tmp_path):
    """flags bit 2 changes the activation pool only: the kernel list, the fused tails and the concatenation-direct heads are those of flags 0."""
    models = [graph[:2], DM.write_mini_model(str(tmp_path / 'mini'), 0), DM.write_tail_model(str(tmp_path / 'tails'), 0)]
    if os.path.exists(REAL + '.param'):
        models.append((REAL + '.param', REAL + '.bin'))
    for pp, bp in models:
        fused, keep = _describe(pp, bp, 0), _describe(pp, bp, B.DET_KEEP_BLOBS)
        assert _plan_lines(fused) == _plan_lines(keep), pp
        assert ' | ' in fused and ' off ' in fused                     # tails and concatenation-direct heads are there to compare
        pool = lambda t: int(t.split()[5])                              # noqa: E731
        assert pool(keep) > pool(fused), pp
        assert _plan_lines(_describe(pp, bp, B.DET_KEEP_BLOBS | B.DET_DIAGNOSTIC)) == _plan_lines(_describe(pp, bp, B.DET_DIAGNOSTIC))


@needs_real
def test_the_reference_models_wide_tails_are_covered(plan):
    """Every (tail kind, NT, BK) the reference model's plan fuses, at 8 and at 512 frames per batch, is a cell of the wide-tail graph."""
    ours = _cells(plan)
    print('\nwide-tail graph at %d frames:\n%s' % (F, _table(ours)))
    for mf in (8, 512):
        ref = _cells(DM.plan_tails(_describe(REAL + '.param', REAL + '.bin', 0, mf)))
        print('reference model at %d frames:\n%s' % (mf, _table(ref)))
        assert ref and not ref - ours, sorted(ref - ours)


# ---------------------------------------------------------------------------------------------------------------- GPU
def _frames(seeds):
    return np.stack([DM.synthetic_rgb(480, 640, s) for s in seeds])


def _grab(det, name, nf):
    """[frame][n] float32 in ncnn's c,h,w order"""
    return np.stack([det.blob(name, f) for f in range(nf)])


def _pc(a, c):
    """[frame][c * pixels] -> [frame * pixel][c]"""
    return a.reshape(a.shape[0], c, -1).transpose(0, 2, 1).reshape(-1, c)


def _first_diff(what, a, b, c, nt):
    """None if a and b ([frame][c * pixels]) are equal bit for bit, else where they first differ: frame, pixel, channel, N-tile, 32-channel chunk"""
    d = np.argwhere(a.view(np.uint32) != b.view(np.uint32))
    if not len(d):
        return None
    f, i = d[0]
    ch, pix = divmod(int(i), a.shape[1] // c)
    return ('%s: %d of %d values differ; first at frame %d, pixel %d, channel %d (N-tile %d of width %d, chunk %d, column %d of the chunk): %r vs %r' %
            (what, len(d), a.size, f, pix, ch, ch // nt, nt, ch % nt // 32, ch % 32, a[f, i], b[f, i]))


@pytest.fixture(scope='module')
def runs(graph):
    """The same 8 frames through a diagnostic, a DET_KEEP_BLOBS and a flags-0 handle of the wide-tail graph; every blob the checks need, read back."""
    from test_gpu_detector import _run
    pp, bp, info, _ = graph
    frames = _frames(range(101, 101 + F))
    diag = B.Detector(pp, bp, max_frames=F, det_thr=DET_THR, flags=B.DET_DIAGNOSTIC)
    keep = B.Detector(pp, bp, max_frames=F, det_thr=DET_THR, flags=B.DET_KEEP_BLOBS)
    fused = B.Detector(pp, bp, max_frames=F, det_thr=DET_THR)
    out = {'diag': _run(diag, frames), 'keep': _run(keep, frames), 'fused': _run(fused, frames)}
    fused.close()
    names = {n for c in info for n in [c['x'], c['y'], c['out']] + c['ops']}
    D = {n: _grab(diag, n, F) for n in sorted(names)}
    K = {c['out']: _grab(keep, c['out'], F) for c in info}
    nt = {p['out']: p['nt'] for p in DM.parse_plan(keep.describe())}
    yield dict(frames=frames, det=out, D=D, K=K, nt=nt, keep=keep)
    keep.close(); diag.close()


@pytest.mark.gpu
def test_pre_tail_gemms_against_float64(graph, runs):
    from test_gpu_detector_kernels import _gemm_check
    info = graph[2]
    for c in info:
        name = '%s %d -> %d @ %dx%d' % (c['kind'], c['cin'], c['cout'], c['hw'], c['hw'])
        r, t = _gemm_check(name, _pc(runs['D'][c['x']], c['cin']), _pc(runs['D'][c['y']], c['cout']), c['w'], c['b'])
        assert r * 16 <= t, '%s: compensated error %.3g is not 16x below plain TF32 (%.3g)' % (name, r, t)


@pytest.mark.gpu
def test_fused_tails_equal_per_layer_execution(graph, runs):
    info = graph[2]
    bad = [e for e in (_first_diff('%s %d -> %d @ %dx%d (%s)' % (c['kind'], c['cin'], c['cout'], c['hw'], c['hw'], c['out']), runs['K'][c['out']],
                                   runs['D'][c['out']], c['cout'], runs['nt'][c['out']]) for c in info) if e]
    assert not bad, '\n'.join(bad)


def _div6(v):
    """ncnn BinaryOp div by the MemoryData scalar 6 as the kernels compute it (div6 of conv1x1_tc.cuh): the correctly rounded quotient -- numpy's --
    for |v| >= 2^-100, and +0 for a zero of either sign (the FMA correction adds zeros of opposite sign)"""
    tiny = (v != 0) & (np.abs(v) < 2.0 ** -100)
    assert not tiny.any(), 'a division input in (0, 2^-100), where div6 may differ from the IEEE quotient'
    q = v / np.float32(6)
    q[q == 0] = np.float32(0)
    return q


def _clip(v):
    return np.minimum(np.maximum(v, np.float32(0)), np.float32(6))


def _restate(kind, y, t):
    """the tail's ncnn layers in float32 and in graph order, on the pre-tail output y and the operands t"""
    f32 = np.float32
    if kind == 'relu':
        return np.maximum(y, f32(0))
    if kind == 'clip':
        return _clip(y)
    if kind == 'hswish':
        return _div6(y * _clip(y + f32(3)))
    if kind == 'add':
        return y + t[0]
    if kind == 'generic':
        return np.maximum(y * f32(0.5), f32(0))
    g = t[0] * _div6(_clip(y + f32(3)))
    return g if kind == 'se_gate' else g + t[1]


@pytest.mark.gpu
def test_per_layer_tails_equal_a_float32_restatement(graph, runs):
    """Ties the element-wise kernels -- and through the fused == per-layer check the fused epilogue -- to IEEE float32."""
    info = graph[2]
    D = runs['D']
    bad = []
    for c in info:
        ref = _restate(c['kind'], D[c['y']], [D[n] for n in c['ops']])
        assert ref.dtype == np.float32
        e = _first_diff('%s %d -> %d @ %dx%d (%s)' % (c['kind'], c['cin'], c['cout'], c['hw'], c['hw'], c['out']), D[c['out']], ref, c['cout'],
                        runs['nt'][c['out']])
        if e:
            bad.append(e)
    assert not bad, '\n'.join(bad)
    # the tails saw both sides of their breakpoints
    y = np.concatenate([D[c['y']].ravel() for c in info if c['kind'] in ('hswish', 'se_gate', 'se_tail')])
    assert (y < -3).any() and ((y > -3) & (y < 3)).any() and (y > 3).any()


@pytest.mark.gpu
def test_pooling_changes_no_detection(runs):
    det = runs['det']
    assert det['fused']['nrows'].min() > 0
    for k in ('rows', 'nrows', 'objects', 'nobjects'):
        assert det['fused'][k].tobytes() == det['keep'][k].tobytes() == det['diag'][k].tobytes(), k


@pytest.mark.gpu
def test_unmaterialised_blobs_stay_unreadable(graph, runs):
    """A blob absorbed into a tail and a head output written straight into the concatenation have no buffer under DET_KEEP_BLOBS either."""
    info = graph[2]
    for name in (info[0]['y'], graph[3][0]):
        with pytest.raises(B.SgsError) as e:
            runs['keep'].blob(name, 0)
        assert e.value.code == B.SGS_ERR_INVALID and 'not materialised' in str(e.value), name


@pytest.mark.gpu
def test_stale_rows_and_batch_position(graph, runs):
    """A 3-frame call after a full batch runs its last pixel tile over rows the full batch left behind: the tails' outputs equal a fresh handle's bit
    for bit.  And a frame's tail outputs do not depend on its position in the batch."""
    from test_gpu_detector import _run
    pp, bp, info, _ = graph
    keep, frames = runs['keep'], runs['frames']
    short = frames[[2, 6, 3]]
    _run(keep, short)
    stale = {c['out']: _grab(keep, c['out'], 3) for c in info}
    fresh_det = B.Detector(pp, bp, max_frames=F, flags=B.DET_KEEP_BLOBS)
    _run(fresh_det, short)
    for c in info:
        assert stale[c['out']].tobytes() == _grab(fresh_det, c['out'], 3).tobytes(), '%s: a 3-frame call depends on what an earlier call left' % c['out']
    fresh_det.close()
    perm = np.array([5, 1, 2, 3, 4, 0, 7, 6])
    _run(keep, frames[perm])
    for c in info:
        assert _grab(keep, c['out'], F).tobytes() == runs['K'][c['out']][perm].tobytes(), '%s: a frame\'s output depends on its batch position' % c['out']


@needs_real
@pytest.mark.gpu
def test_reference_model_fused_equals_per_layer():
    """Every blob that both a DET_KEEP_BLOBS and a diagnostic handle of the reference model hold, on 3 frames, bit for bit.  max_frames = 8: the
    diagnostic plan holds 30.5 M floats per frame (about 122 MB), so the two handles take about 2 GB of device memory; at this batch the plan fuses
    hard-swish at NT 96 / 128 / 160 / 256, the SE gate and tail at 96 / 128, +tensor at 96 / 128 and clip at 64 / 128 into wide tiles."""
    from test_gpu_detector import _run
    frames = _frames((21, 22, 23))
    keep = B.Detector(REAL + '.param', REAL + '.bin', max_frames=8, flags=B.DET_KEEP_BLOBS)
    diag = B.Detector(REAL + '.param', REAL + '.bin', max_frames=8, flags=B.DET_DIAGNOSTIC)
    a, b = _run(keep, frames), _run(diag, frames)
    plans = DM.plan_tails(keep.describe())
    geo = {p['out']: p for p in plans}
    outs = [l.split()[l.split().index('out') + 1] for l in keep.describe().splitlines()[1:]]
    compared, tails, bad = 0, set(), []
    for name in dict.fromkeys(outs):
        x = _grab(keep, name, 3)
        y = _grab(diag, name, 3)
        assert x.shape == y.shape, name
        p = geo.get(name)
        p = p if p and p['cout'] * p['h'] * p['w'] == x.shape[1] else None           # a GEMM's own output (not a concatenation it writes into)
        e = _first_diff(name, x, y, p['cout'] if p else 1, p['nt'] if p else 1 << 30)
        if e:
            bad.append(e)
        compared += 1
        if p and p['kind'] != 'none':
            tails.add((p['kind'], p['nt']))
    keep.close(); diag.close()
    assert not bad, '\n'.join(bad)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), k
    print('\nreference model: %d blobs equal bit for bit; fused (tail, NT) among them: %s' % (compared, sorted(tails)))
    assert tails >= {('hswish', 128), ('hswish', 160), ('hswish', 256), ('se_gate', 96), ('se_gate', 128), ('se_tail', 96), ('se_tail', 128),
                     ('add', 96), ('add', 128), ('clip', 64), ('clip', 128)}, sorted(tails)
