"""The detector's direct kernels -- depth-wise (dwconv_kernel), dense (conv_small_kernel), first layer (conv_first_kernel) -- and its stand-alone
element-wise kernel (eltwise_kernel) with every fused tail, read back from fused execution.

The graph is write_direct_tail_model (tests/detector_model.py): every tail kind (ReLU, clip, hard-swish, +tensor, SE gate, SE tail, the generic
chain) on every depth-wise variant (V = 1; V = 4 with two and with one output row per thread), on conv_small_kernel's float4, partial-block and
scalar paths, and on the first-layer kernel; bias-free and dilated convolutions, and bias-free 1x1 GEMMs on a narrow and a wide tile; SSD head
pieces written straight into the concatenated buffers at offsets and frame strides that are and are not multiples of 4; and element-wise chains that build_tail cuts, that outgrow kMaxEpi, that use sub,
div, rev, clip bounds other than 0..6 and tensor operands on either side, and that read the tail's start value.

  CPU (plan-only handles): every intended (kernel, variant, kind) cell is planned; the concatenation-direct pieces and the step lists of the chains;
       DET_KEEP_BLOBS plans the kernels of flags 0; the reference model's direct-kernel tail cells are among the graph's; the memory both GPU
       handles take; the planner refuses BinaryOp operands of another shape or layout and x op x, and still plans the graphs it took before.
  GPU: every tailed convolution's pre-tail output against float64 on the diagnostic handle's own input; DET_KEEP_BLOBS (fused) == diagnostic
       (per-layer) bit for bit for every blob the fused schedule materialises; every element-wise layer's diagnostic output == a float32 numpy
       restatement; both sides of the hard-swish / hard-sigmoid breakpoints reached; stale rows and batch position; equal detections."""
import os
import re

import numpy as np
import pytest

import detector_model as DM
import ncnn_model as NM
from pysgs import binding as B
from test_gpu_detector_fused_tails import REAL, _describe, _div6, _plan_lines, needs_real

F = DM.PROBE_FRAMES
DET_THR = 0.05
MEM_BUDGET = 1 << 30          # bytes of activation pool the GPU tests hold at once, at F frames (test_memory_budget)


@pytest.fixture(scope='module')
def graph(tmp_path_factory):
    return DM.write_direct_tail_model(str(tmp_path_factory.mktemp('direct_tails')), 0)


# ---------------------------------------------------------------------------------------------------------------- plan parsing
def _launch(line):
    """(kernel, variant) that detector_detect_device launches for a describe() line: dwconv variants by launch_dwconv (V1: Cout % 4 != 0; V4Y2:
    OH >= 4; V4Y1), conv_first_kernel for a 3 -> 16 3x3/s2/p1 undilated convolution not written into a concatenation, else conv_small_kernel:
    float4 stores when Cout % 4 == 0 and the output base and frame stride are multiples of 4 (the last 8-channel block scalar when Cout % 8 != 0),
    else scalar ('scalar/unaligned': Cout % 4 == 0, but the offset or the frame stride is not)."""
    t = line.split()
    if t[0] in ('eltwise', 'conv1x1', 'concat', 'softmax'):
        return t[0], '-'
    m = re.search(r' n (\d+) geom (\d+)x\d+x\d+->(\d+)x(\d+)x(\d+) k(\d+) s(\d+) p(\d+)(?: d(\d+))?', line)
    n, cin, cout, oh, ow, k, s, p, d = (int(v) if v else 1 for v in m.groups())
    off = re.search(r' off (\d+)', line)
    if t[0] == 'dwconv':
        return 'dwconv', 'V1' if cout % 4 else ('V4Y2' if oh >= 4 else 'V4Y1')
    if not off and (k, cin, cout, s, p, d) == (3, 3, 16, 2, 1, 1):
        return 'conv_first', '-'
    base, stride = (int(off.group(1)), n) if off else (0, oh * ow * cout)
    if cout % 4:
        return 'conv_small', 'scalar'
    if (base | stride) & 3:
        return 'conv_small', 'scalar/unaligned'
    return 'conv_small', 'float4' if cout % 8 == 0 else 'float4+scalar block'


def _plan(text):
    """describe() lines after the first as dicts: op, name, inp, out, kernel, variant, ks, steps, kind, off, line"""
    out = []
    for l in text.splitlines()[1:]:
        t = l.split()
        steps = DM.tail_steps(l)
        kern, var = _launch(l)
        ks = re.search(r' k(\d+) s(\d+)', l)
        off = re.search(r' off (\d+)', l)
        out.append(dict(op=t[0], name=t[1], inp=t[t.index('in') + 1], out=t[t.index('out') + 1], kernel=kern, variant=var, ks=tuple(map(int, ks.groups())) if ks else None,
                        steps=steps, kind=DM.epi_kind(steps), off=int(off.group(1)) if off else None, line=l))
    return out


def _cells(plan, kernels=('dwconv', 'conv_small', 'conv_first', 'eltwise')):
    return {(p['kernel'], p['variant'], p['kind']) for p in plan if p['kernel'] in kernels and p['kind'] != 'none'}


CONV_VARIANT = {16: 'float4', 12: 'float4+scalar block', 5: 'scalar'}


def _channels(plan):
    """channels of every blob a plan writes (1 for blobs that are not activation maps): a convolution's Cout, an element-wise kernel's input's"""
    ch = {'input': 3}
    for p in plan:
        g = re.search(r'->(\d+)x', p['line'])
        if g and p['off'] is None:
            ch[p['out']] = int(g.group(1))
        elif p['op'] == 'eltwise':
            ch[p['out']] = ch.get(re.sub(r'_splitncnn_\d+$', '', p['inp']), 1)
    return ch


def _intended(c):
    """(kernel, variant) a case of the graph is built to reach"""
    if c['family'] == 'dw':
        return 'dwconv', c['variant']
    if c['family'] == 'stem':
        return 'conv_first', '-'
    if c['family'] == 'conv':
        return 'conv_small', CONV_VARIANT[c['conv']['cout']]
    if c['family'] == 'gemm':
        return 'conv1x1', '-'
    return None


def _table(cells):
    rows = sorted({(k, v) for k, v, _ in cells})
    return '\n'.join('  %-11s %-20s %s' % (k, v, ' '.join('%-7s' % (kd if (k, v, kd) in cells else '-') for kd in DM.TAIL_KINDS)) for k, v in rows)


@pytest.fixture(scope='module')
def plan(graph):
    return _plan(_describe(graph[0], graph[1], 0))


# ---------------------------------------------------------------------------------------------------------------- CPU: plans
def test_plan_covers_every_cell(graph, plan):
    info = graph[2]
    by_out = {p['out']: p for p in plan}
    for c in info:
        if c['family'] in ('dw', 'conv', 'stem', 'gemm'):
            p = by_out[c['out']]
            assert (p['kernel'], p['variant']) == _intended(c) and p['kind'] == c['kind'], (c['case'], p['line'])
            assert p['ks'] == (c['conv']['k'], c['conv']['s']), p['line']
            assert bool(re.search(r' p\d+ d2 ', p['line'])) == (c['conv']['dil'] == 2), p['line']
    want = {_intended(c) + (k,) for c in info if c['family'] in ('dw', 'conv') for k in DM.TAIL_KINDS}
    want |= {('conv_first', '-', k) for k in DM.TAIL_KINDS}
    got = _cells(plan)
    assert not want - got, sorted(want - got)
    # each (K, S) meets every depth-wise variant, and at least one tensor-reading kind
    dw = [p for p in plan if p['kernel'] == 'dwconv' and p['kind'] != 'none']
    for ks in DM.DW_KS:
        assert {p['variant'] for p in dw if p['ks'] == ks} == set(DM.DW_VARIANTS), ks
        assert any(p['kind'] in DM.TENSOR_TAILS for p in dw if p['ks'] == ks), ks
    # bias-free convolutions on every direct kernel and dilation in conv_small_kernel
    free = [c for c in info if c['conv']['b'] is None]
    assert {_intended(c) for c in free} >= {('dwconv', v) for v in DM.DW_VARIANTS} | {('conv_small', 'float4'), ('conv_small', 'scalar'),
                                                                                     ('conv_first', '-'), ('conv1x1', '-')}
    # the bias-free GEMMs: one narrow tile (NT 32, bias loaded at each use) and one wide (NT >= 64, bias loaded per chunk)
    gemm = {p['out']: p for p in DM.parse_plan('\n'.join(p['line'] for p in plan))}
    assert sorted(gemm[c['out']]['nt'] > 32 for c in free if c['family'] == 'gemm') == [False, True]
    assert any(c['conv']['dil'] == 2 and by_out[c['out']]['kernel'] == 'conv_small' for c in info if c['family'] == 'conv')
    print('\ndirect-tail graph at %d frames, (kernel, variant): kinds\n%s' % (F, _table(got)))


def test_concatenation_direct_pieces(graph, plan):
    """The head pieces are conv_small_kernel launches writing straight into mbox_conf (3003 floats per frame: not a multiple of 4) and mbox_loc."""
    heads = [p for p in plan if p['name'] in graph[3]]
    assert len(heads) == 6 and all(p['op'] == 'conv' for p in heads), [p['line'] for p in heads]
    conf = [(p['off'], p['variant'], p['kind']) for p in heads if p['out'] == 'mbox_conf']
    loc = [(p['off'], p['variant'], p['kind']) for p in heads if p['out'] == 'mbox_loc']
    assert conf == [(0, 'scalar/unaligned', 'hswish'), (2100, 'scalar', 'relu'), (2667, 'scalar/unaligned', 'generic')], conf
    assert loc == [(0, 'float4', 'clip'), (400, 'float4+scalar block', 'generic'), (508, 'float4', 'hswish')], loc
    assert all(' n 3003 ' in p['line'] for p in heads if p['out'] == 'mbox_conf') and all(' n 572 ' in p['line'] for p in heads if p['out'] == 'mbox_loc')
    assert not [p for p in plan if p['op'] == 'concat']


def _norm(steps):
    """steps with tensor operands named by the blob they split from"""
    return [(op, rev, src, re.sub(r'_splitncnn_\d+$', '', v) if src == 'tensor' else v) for op, rev, src, v in steps]


def test_chain_step_lists(graph, plan):
    """build_tail's longest valid prefix, kMaxEpi, eltwise_chain's one-reader rule, and the steps of the sub / div / rev / clip and start chains."""
    by_out = {p['out']: p for p in plan}
    ch = {c['kind']: c for c in graph[2] if c['family'] == 'chain'}

    def line(blob):
        return by_out[blob]['op'], _norm(by_out[blob]['steps'])

    a, r, m, c, s, q = ch['cut']['outs']
    assert line(r) == ('dwconv', [('add', False, 'scalar', 1.0), ('relu', False, None, ())])
    assert line(m) == ('eltwise', [('mul', False, 'scalar', 2.0)])
    assert line(c) == ('eltwise', [('clip', False, None, (-1.0, 2.5))])
    assert line(s) == ('eltwise', [('sub', False, 'scalar', 0.25)])
    assert line(q) == ('eltwise', [('relu', False, None, ())])
    assert a not in by_out
    outs = ch['long']['outs']
    assert line(outs[7]) == ('conv', [('add', False, 'scalar', 0.5), ('mul', False, 'scalar', 1.5), ('relu', False, None, ()), ('sub', False, 'scalar', 0.25),
                                      ('clip', False, None, (-2.0, 3.0)), ('mul', False, 'scalar', 0.75), ('add', False, 'scalar', -0.125),
                                      ('div', False, 'scalar', 1.25)])
    assert line(outs[9]) == ('eltwise', [('mul', False, 'scalar', 2.0), ('relu', False, None, ())])
    t1, tpos = ch['ops']['ops']
    assert line(ch['ops']['out']) == ('dwconv', [('sub', False, 'scalar', 0.5), ('sub', True, 'tensor', t1), ('div', False, 'scalar', 0.75),
                                                 ('clip', False, None, (-1.0, 2.5)), ('add', False, 'scalar', 2.0), ('div', True, 'tensor', t1),
                                                 ('div', False, 'tensor', tpos)])
    assert line(ch['start']['out']) == ('conv', [('relu', False, None, ()), ('add', True, 'start', None)])
    assert by_out[ch['start']['out']]['kind'] == by_out[ch['ops']['out']]['kind'] == 'generic'
    assert sum(p['op'] == 'eltwise' for p in plan) == 5


def test_keep_blobs_plans_the_fused_schedule(graph):
    pp, bp = graph[:2]
    fused, keep = _describe(pp, bp, 0), _describe(pp, bp, B.DET_KEEP_BLOBS)
    assert _plan_lines(fused) == _plan_lines(keep)
    assert _plan_lines(_describe(pp, bp, B.DET_KEEP_BLOBS | B.DET_DIAGNOSTIC)) == _plan_lines(_describe(pp, bp, B.DET_DIAGNOSTIC))


def test_memory_budget(graph):
    """The most the GPU tests hold at once, F frames each: the runs fixture's diagnostic, DET_KEEP_BLOBS and flags-0 handles, and the second
    DET_KEEP_BLOBS handle of the stale-rows test (the fixture has closed its flags-0 and diagnostic handles by then, but they are counted).  Their
    activation pools fit MEM_BUDGET."""
    pool = lambda t: int(t.split()[7])           # noqa: E731  pool_floats_per_frame
    pp, bp = graph[:2]
    keep, diag, fused = (pool(_describe(pp, bp, f)) for f in (B.DET_KEEP_BLOBS, B.DET_DIAGNOSTIC, 0))
    total = (2 * keep + diag + fused) * F * 4
    print('\npool floats per frame: keep %d, diagnostic %d, flags 0 %d; %.0f MB at %d frames' % (keep, diag, fused, total / 1e6, F))
    assert total <= MEM_BUDGET


@needs_real
def test_the_reference_models_direct_tails_are_covered(plan):
    ours = _cells(plan, ('dwconv', 'conv_small', 'conv_first'))
    for mf in (8, 512):
        ref = _cells(_plan(_describe(REAL + '.param', REAL + '.bin', 0, mf)), ('dwconv', 'conv_small', 'conv_first'))
        print('\nreference model at %d frames:\n%s' % (mf, _table(ref)))
        assert ref and not ref - ours, sorted(ref - ours)


# ---------------------------------------------------------------------------------------------------------------- CPU: planner fixes
def _binop_graph(dirpath, form):
    """Stem and depth-wise chain to 19x19 (16 channels), a BinaryOp 'probe_op' of the given operand form, and a minimal SSD head."""
    g = DM.Graph(1)
    data = g.add('Input', [], name='input')
    x = {150: g.conv(data, 3, 16, 3, 2, 1, gain=1 / 64)}
    for a, b in zip(DM.CHAIN[:3], DM.CHAIN[1:4]):
        x[b] = g.conv(x[a], 16, 16, 3, 2, 1, dw=True)
    a = g.conv(x[19], 16, 8)                                                   # 8 x 19 x 19 = 2888 floats
    if form == 'same':
        t = g.conv(x[19], 16, 8)
    elif form == 'shape':
        t = g.conv(x[38], 16, 2)                                                # 2 x 38 x 38 = 2888 floats
    elif form == 'flat':
        t = g.add('Flatten', [g.add('Permute', [g.conv(x[19], 16, 8)], '0=3')])
    elif form == 'permuted':                                                     # 19 x 19 x 19 both ways: the shapes agree, the element order does not
        a = g.conv(x[19], 16, 19)
        t = g.add('Permute', [g.conv(x[19], 16, 19)], '0=3')
    elif form == 'self':
        t = a
    g.add('BinaryOp', [a, t], '0=0', name='probe_op')
    DM._head(g, data, [(x[19], 16)], 4, '-23300=1,60.000000 -23301=1,105.0 -23302=1,2.000000 7=1')
    os.makedirs(dirpath, exist_ok=True)
    pp, bp = os.path.join(dirpath, form + '.param'), os.path.join(dirpath, form + '.bin')
    g.write(pp, bp)
    return pp, bp


@pytest.mark.parametrize('form', ['shape', 'flat', 'permuted', 'self'])
def test_binop_operands_the_kernels_cannot_index_are_refused(tmp_path, form):
    pp, bp = _binop_graph(str(tmp_path), form)
    with pytest.raises(B.SgsError) as e:
        _describe(pp, bp, 0)
    assert e.value.code == B.SGS_ERR_UNSUPPORTED and 'probe_op' in str(e.value), str(e.value)
    assert ('same blob' in str(e.value)) == (form == 'self'), str(e.value)


def test_same_shape_operands_still_plan(tmp_path):
    pp, bp = _binop_graph(str(tmp_path), 'same')
    assert re.search(r' \| add(\(rev\))? \S+ buf ', _describe(pp, bp, 0))                 # fused into the second operand's GEMM


def test_the_test_graphs_still_create(tmp_path, graph):
    models = [DM.write_mini_model(str(tmp_path / 'mini'), 0), DM.write_tail_model(str(tmp_path / 'tails'), 0),
              DM.write_wide_tail_model(str(tmp_path / 'wide'), 0)[:2], graph[:2]]
    if os.path.exists(REAL + '.param'):
        models.append((REAL + '.param', REAL + '.bin'))
    for pp, bp in models:
        for flags in (0, B.DET_DIAGNOSTIC):
            assert _describe(pp, bp, flags).startswith('layers '), pp


# ---------------------------------------------------------------------------------------------------------------- GPU
def _frames(seeds):
    return np.stack([DM.synthetic_rgb(480, 640, s) for s in seeds])


def _grab(det, name, nf):
    """[frame][n] float32 in ncnn's c,h,w order"""
    return np.stack([det.blob(name, f) for f in range(nf)])


def _outs(text):
    return list(dict.fromkeys(p['out'] for p in _plan(text)))


@pytest.fixture(scope='module')
def runs(graph):
    """The same 8 frames through a diagnostic, a DET_KEEP_BLOBS and a flags-0 handle; every blob each schedule materialises, read back."""
    from test_gpu_detector import _run
    pp, bp, info, _ = graph
    frames = _frames(range(201, 201 + F))
    diag = B.Detector(pp, bp, max_frames=F, det_thr=DET_THR, flags=B.DET_DIAGNOSTIC)
    keep = B.Detector(pp, bp, max_frames=F, det_thr=DET_THR, flags=B.DET_KEEP_BLOBS)
    fused = B.Detector(pp, bp, max_frames=F, det_thr=DET_THR)
    out = {'diag': _run(diag, frames), 'keep': _run(keep, frames), 'fused': _run(fused, frames)}
    fused.close()
    dplan = _plan(diag.describe())
    D = {n: _grab(diag, n, F) for n in ['input'] + _outs(diag.describe())}
    kplan = _plan(keep.describe())
    K = {n: _grab(keep, n, F) for n in _outs(keep.describe())}
    diag.close()
    yield dict(frames=frames, det=out, D=D, K=K, kplan=kplan, dplan=dplan, keep=keep)
    keep.close()


def _shape(c, which):
    """[channels, h, w] of a convolution's input or output"""
    if which == 'in':
        return c['cin'], c['hw'], c['hw']
    oh = (c['hw'] + 2 * c['p'] - c['dil'] * (c['k'] - 1) - 1) // c['s'] + 1
    return c['cout'], oh, oh


@pytest.mark.gpu
def test_pre_tail_outputs_against_float64(graph, runs):
    from test_gpu_detector_kernels import _direct_check, _gemm_check, _pc
    D = runs['D']
    for c in graph[2]:
        cv = c['conv']
        X, Y = D[cv['in']].reshape((F,) + _shape(cv, 'in')), D[cv['out']].reshape((F,) + _shape(cv, 'out'))
        name = '%s %s %s (%s)' % (c['family'], c['kind'], c['variant'], cv['out'])
        if c['family'] == 'gemm':                     # bias-free 1x1 GEMM: the compensated-TF32 bound of test_gpu_detector_kernels.py
            r, t = _gemm_check(name, _pc(X), _pc(Y), cv['w'].reshape(cv['cout'], cv['cin']), np.zeros(cv['cout']))
            assert r * 16 <= t, '%s: compensated error %.3g is not 16x below plain TF32 (%.3g)' % (name, r, t)
        else:
            _direct_check(name, cv, X, Y)


def _first_diff(what, a, b, chans, variant, pieces=None):
    """None if a and b ([frame][n], ncnn order) are equal bit for bit, else where they first differ: frame, pixel and channel of a 3-D blob
    (chans channels), or the head piece ([(name, offset, n, channels, variant)]) and its pixel and channel for a concatenation"""
    d = np.argwhere(a.view(np.uint32) != b.view(np.uint32))
    if not len(d):
        return None
    f, i = (int(v) for v in d[0])
    if pieces:
        nm, off, _, ch, variant = [p for p in pieces if p[1] <= i < p[1] + p[2]][0]
        pix, c = divmod(i - off, ch)
        where = 'piece %s, pixel %d, channel %d' % (nm, pix, c)
    else:
        c, pix = divmod(i, a.shape[1] // chans)
        where = 'pixel %d, channel %d' % (pix, c)
    return '%s [%s]: %d of %d values differ; first at frame %d, %s: %r vs %r' % (what, variant, len(d), a.size, f, where, a[f, i], b[f, i])


@pytest.mark.gpu
def test_fused_equals_per_layer_execution(graph, runs):
    """Every blob the fused schedule materialises -- each tail's output, each stand-alone chain's, the concatenated head -- equals the
    diagnostic handle's bit for bit."""
    info = graph[2]
    K, D, kplan = runs['K'], runs['D'], runs['kplan']
    assert {c['out'] for c in info if c['family'] != 'cat'} <= set(K) and {'mbox_conf', 'mbox_loc'} <= set(K)
    chans = _channels(kplan)
    heads = {c['conv']['out']: c for c in info if c['family'] == 'cat'}
    bad = []
    for n in K:
        ps = [p for p in kplan if p['out'] == n]
        pieces = [(p['name'], p['off'], heads[p['name']]['conv']['cout'] * _shape(heads[p['name']]['conv'], 'out')[1] ** 2,
                   heads[p['name']]['conv']['cout'], p['variant']) for p in ps if p['off'] is not None]
        e = _first_diff('%s (%s)' % (n, ps[0]['kernel']), K[n], D[n], chans.get(n, 1), ps[0]['variant'], pieces)
        if e:
            bad.append(e)
    assert not bad, '\n'.join(bad)


def _restate(op, a, b):
    """one ncnn element-wise layer in float32: a op b for BinaryOp (b a scalar or a same-shape tensor), Clip (b = bounds), ReLU"""
    f32 = np.float32
    if op == 'relu':
        return np.maximum(a, f32(0))
    if op == 'clip':
        return np.minimum(np.maximum(a, f32(b[0])), f32(b[1]))
    if op == 'add':
        return a + b
    if op == 'sub':
        return a - b
    if op == 'mul':
        return a * b
    if np.ndim(b) == 0 and b == 6:
        return _div6(a)
    q = a / b                                          # IEEE; the kernels' div_scalar takes div6 for an operand of exactly 6: +0 for a zero quotient
    q[(b == f32(6)) & (q == 0)] = f32(0)
    return q


@pytest.mark.gpu
def test_per_layer_results_equal_a_float32_restatement(graph, runs):
    """Every ReLU, Clip and BinaryOp layer of the graph, run on its own kernel by the diagnostic handle, against numpy float32 on the same inputs."""
    D, chans = runs['D'], _channels(runs['dplan'])
    layers = NM.parse_param(graph[0]); NM.load_weights(layers, graph[1])
    src, const = {}, {}
    for L in layers:
        if L.type == 'Split':
            for o in L.outputs:
                src[o] = src.get(L.inputs[0], L.inputs[0])
        elif L.type == 'MemoryData':
            const[L.outputs[0]] = np.float32(L.data.reshape(-1)[0])
    val = lambda n: const[src.get(n, n)] if src.get(n, n) in const else D[src.get(n, n)]        # noqa: E731
    checked, bad = 0, []
    with np.errstate(divide='raise', over='raise', invalid='raise'):
        for L in layers:
            if L.type not in ('ReLU', 'Clip', 'BinaryOp'):
                continue
            if L.type == 'BinaryOp':
                op = ('add', 'sub', 'mul', 'div')[int(L.p(0, 0))]
                ref = _restate(op, val(L.inputs[0]), val(L.inputs[1]))
            else:
                ref = _restate(L.type.lower(), val(L.inputs[0]), (L.p(0), L.p(1)))
            assert ref.dtype == np.float32, L.name
            e = _first_diff('%s %s' % (L.type, L.name), D[L.outputs[0]], ref, chans[L.outputs[0]], 'eltwise_kernel')
            if e:
                bad.append(e)
            checked += 1
    assert not bad, '\n'.join(bad)
    print('\n%d element-wise layers equal their float32 restatement' % checked)


@pytest.mark.gpu
def test_breakpoints_are_reached(graph, runs):
    """The hard-swish / hard-sigmoid inputs of each (kernel, variant) -- and of each head piece and GEMM on its own -- lie on both sides of -3
    and of 3."""
    groups = {}
    for c in graph[2]:
        if c['kind'] in ('hswish', 'se_gate', 'se_tail'):
            key = _intended(c) if c['family'] in ('dw', 'conv', 'stem') else (c['family'], c['conv']['out'])
            groups.setdefault(key, []).append(runs['D'][c['conv']['out']].ravel())
    assert len(groups) == 3 + 3 + 1 + 2 + 2                  # dwconv variants, conv_small paths, conv_first, GEMMs, head pieces
    for key, ys in groups.items():
        y = np.concatenate(ys)
        assert (y < -3).any() and ((y > -3) & (y < 3)).any() and (y > 3).any(), (key, y.min(), y.max())


@pytest.mark.gpu
def test_stale_rows_and_batch_position(graph, runs):
    """A 3-frame call after a full batch equals a fresh handle's, and a frame's outputs do not depend on its position in the batch."""
    from test_gpu_detector import _run
    pp, bp = graph[:2]
    keep, frames, K = runs['keep'], runs['frames'], runs['K']
    short = frames[[2, 6, 3]]
    _run(keep, short)
    fresh = B.Detector(pp, bp, max_frames=F, flags=B.DET_KEEP_BLOBS)
    try:
        _run(fresh, short)
        for n in K:
            assert _grab(keep, n, 3).tobytes() == _grab(fresh, n, 3).tobytes(), '%s: a 3-frame call depends on what an earlier call left' % n
    finally:
        fresh.close()
    perm = np.array([5, 1, 2, 3, 4, 0, 7, 6])
    _run(keep, frames[perm])
    for n in K:
        assert _grab(keep, n, F).tobytes() == K[n][perm].tobytes(), '%s: a frame\'s output depends on its batch position' % n


@pytest.mark.gpu
def test_detections_do_not_depend_on_the_schedule(runs):
    det = runs['det']
    assert det['fused']['nrows'].min() > 0
    for k in det['fused']:
        assert det['fused'][k].tobytes() == det['keep'][k].tobytes() == det['diag'][k].tobytes(), k
