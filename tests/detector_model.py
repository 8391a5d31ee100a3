"""Synthetic SSD graphs in ncnn's text/bin format for the detector tests: same layer vocabulary and export idioms as the reference model
(Thirdparty/ncnn_model/mobilenetv3_ssdlite_voc.param: hard-swish as add/clip/mul/div with MemoryData scalars, spatial SE tail, residual adds,
SSDLite heads, mmdetection-style PriorBox, DetectionOutput), random weights, a few thousand priors."""
import os
import struct

import numpy as np


class Graph:
    def __init__(self, seed):
        self.rng = np.random.default_rng(seed)
        self.layers = []      # [type, name, ins, outs, param string, [arrays]]
        self.consts = {}
        self.uid = 0

    def name(self, p='b'):
        self.uid += 1
        return '%s%d' % (p, self.uid)

    def add(self, typ, ins, params='', weights=(), nout=1, name=None):
        name = name or self.name('l')
        outs = [name] if nout == 1 else ['%s_%d' % (name, i) for i in range(nout)]
        self.layers.append([typ, name, list(ins), outs, params, list(weights)])
        return outs[0] if nout == 1 else outs

    def const(self, v):
        n = self.name('c')
        self.layers.insert(1, ['MemoryData', n, [], [n], '0=1', [np.array([v], np.float32)]])
        return n

    def conv(self, x, cin, cout, k=1, s=1, p=0, gain=1.0, dw=False, w=None, b=None, name=None):
        fan = k * k * (1 if dw else cin)
        if w is None:
            w = (self.rng.standard_normal((cout, 1 if dw else cin, k, k)) * gain * np.sqrt(2.0 / fan)).astype(np.float32)
        if b is None:
            b = (self.rng.standard_normal(cout) * 0.1).astype(np.float32)
        prm = '0=%d 1=%d 11=%d 2=1 12=1 3=%d 13=%d 4=%d 14=%d 5=1 6=%d' % (cout, k, k, s, s, p, p, w.size)
        if dw:
            prm += ' 7=%d' % cout
        return self.add('ConvolutionDepthWise' if dw else 'Convolution', [x], prm, [np.zeros(1, np.uint32), w, b], name=name)

    def relu(self, x): return self.add('ReLU', [x])
    def clip(self, x): return self.add('Clip', [x], '0=0.000000 1=6.000000')
    def binop(self, a, b, op): return self.add('BinaryOp', [a, b], '0=%d' % op)

    def hswish(self, x):
        return self.binop(self.binop(x, self.clip(self.binop(x, self.const(3.0), 0)), 2), self.const(6.0), 3)

    def hsigmoid(self, x):
        return self.binop(self.clip(self.binop(x, self.const(3.0), 0)), self.const(6.0), 3)

    def finalize(self):
        """ncnn graphs are single-consumer: insert Split layers."""
        out = []
        use = {}
        for L in self.layers:
            for i in L[2]:
                use[i] = use.get(i, 0) + 1
        renamed = {}
        for L in self.layers:
            ins = []
            for i in L[2]:
                if i in renamed:
                    ins.append(renamed[i].pop())
                else:
                    ins.append(i)
            L = [L[0], L[1], ins, L[3], L[4], L[5]]
            out.append(L)
            for o in L[3]:
                if use.get(o, 0) > 1:
                    names = ['%s_splitncnn_%d' % (o, q) for q in range(use[o])]
                    out.append(['Split', 'splitncnn_' + o, [o], names, '', []])
                    renamed[o] = names[:]
        self.layers = out

    def write(self, param_path, bin_path):
        self.finalize()
        nblobs = sum(len(L[3]) for L in self.layers)
        with open(param_path, 'w') as f:
            f.write('7767517\n%d %d\n' % (len(self.layers), nblobs))
            for typ, name, ins, outs, prm, _ in self.layers:
                f.write('%-24s %-24s %d %d %s %s\n' % (typ, name, len(ins), len(outs), ' '.join(ins + outs), prm))
        with open(bin_path, 'wb') as f:
            for L in self.layers:
                for a in L[5]:
                    f.write(np.ascontiguousarray(a).tobytes())


def write_mini_model(dirpath, seed=0, conf_gain=1.0, person_bias=2.0, many_priors=False):
    g = Graph(seed)
    data = g.add('Input', [], name='input')
    x = g.hswish(g.conv(data, 3, 8, 3, 2, 1))                                     # 8 x 150 x 150
    x = g.relu(g.conv(x, 8, 16)); x = g.relu(g.conv(x, 16, 16, 3, 2, 1, dw=True))  # 75
    x0 = g.conv(x, 16, 8)
    # SE + residual block
    y = g.hswish(g.conv(x0, 8, 24)); y = g.hswish(g.conv(y, 24, 24, 5, 1, 2, dw=True)); y = g.conv(y, 24, 8)
    se = g.conv(g.relu(g.conv(y, 8, 6)), 6, 8)
    x = g.binop(g.binop(y, g.hsigmoid(se), 2), x0, 0)
    # plain residual
    r = g.conv(g.relu(g.conv(g.relu(g.conv(x, 8, 16)), 16, 16, 3, 1, 1, dw=True)), 16, 8)
    x = g.binop(r, x, 0)
    x = g.clip(g.conv(g.clip(g.conv(x, 8, 8, 5, 2, 2, dw=True)), 8, 32))          # 38
    f1 = g.clip(g.conv(g.clip(g.conv(x, 32, 32, 3, 2, 1, dw=True)), 32, 32))     # 19
    f2 = g.clip(g.conv(g.clip(g.conv(g.clip(g.conv(f1, 32, 16)), 16, 16, 3, 2, 1, dw=True)), 16, 32))   # 10
    ncls = 21
    locs, confs, priors = [], [], []
    specs = [(x if many_priors else f1, 32, '-23300=1,60.000000 -23301=1,105.0 -23302=1,2.000000', 4), (f2, 32, '-23300=1,105.000000 -23301=1,150.0 -23302=2,2.000000,3.0', 6)]
    for k, (f, c, pb, npr) in enumerate(specs):
        cf = g.conv(g.clip(g.conv(f, c, c, 3, 1, 1, dw=True)), c, npr * ncls, gain=conf_gain)
        g.layers[-1][5][2][15::ncls] += np.float32(person_bias)            # make the person class (id 15) show up among the detections
        confs.append(g.add('Flatten', [g.add('Permute', [cf], '0=3')]))
        lc = g.conv(g.clip(g.conv(f, c, c, 3, 1, 1, dw=True)), c, npr * 4)
        locs.append(g.add('Flatten', [g.add('Permute', [lc], '0=3')]))
        priors.append(g.add('PriorBox', [f, data], pb + ' 3=0.100000 4=0.100000 5=0.200000 6=0.200000 7=1 8=0 9=-233 10=-233 11=-233.000000 12=-233.000000 13=0.500000 14=1 15=1'))
    loc = g.add('Concat', locs, '0=0', name='mbox_loc')
    conf = g.add('Concat', confs, '0=0', name='mbox_conf')
    pri = g.add('Concat', priors, '0=1', name='mbox_priorbox')
    sm = g.add('Softmax', [g.add('Reshape', [conf], '0=%d 1=-1' % ncls)], '0=1 1=1')
    g.add('DetectionOutput', [loc, g.add('Flatten', [sm]), pri], '0=%d 1=0.450000 2=300 3=100 4=0.010000' % ncls, name='detection_out')
    os.makedirs(dirpath, exist_ok=True)
    pp, bp = os.path.join(dirpath, 'mini.param'), os.path.join(dirpath, 'mini.bin')
    g.write(pp, bp)
    return pp, bp


CHAIN = (150, 75, 38, 19, 10, 5, 3, 2, 1)        # map sizes of the probe graphs' depth-wise 3x3/s2 chain below the 150x150 stem output


def _head(g, data, feats, npr, prior_params, ncls=21, person_bias=2.0):
    """SSD head over [(blob, channels)]: conf / loc 1x1 convolutions -> Permute -> Flatten -> Concat, PriorBox, Softmax, DetectionOutput."""
    locs, confs, priors = [], [], []
    for f, c in feats:
        cf = g.conv(f, c, npr * ncls)
        g.layers[-1][5][2][15::ncls] += np.float32(person_bias)
        confs.append(g.add('Flatten', [g.add('Permute', [cf], '0=3')]))
        locs.append(g.add('Flatten', [g.add('Permute', [g.conv(f, c, npr * 4)], '0=3')]))
        priors.append(g.add('PriorBox', [f, data], prior_params + ' 3=0.100000 4=0.100000 5=0.200000 6=0.200000 8=0 9=-233 10=-233 11=-233.000000 '
                                                                   '12=-233.000000 13=0.500000 14=1 15=1'))
    loc = g.add('Concat', locs, '0=0', name='mbox_loc')
    conf = g.add('Concat', confs, '0=0', name='mbox_conf')
    pri = g.add('Concat', priors, '0=1', name='mbox_priorbox')
    sm = g.add('Softmax', [g.add('Reshape', [conf], '0=%d 1=-1' % ncls)], '0=1 1=1')
    g.add('DetectionOutput', [loc, g.add('Flatten', [sm]), pri], '0=%d 1=0.450000 2=300 3=100 4=0.010000' % ncls, name='detection_out')


def _probe_weights(rng, cin, cout, mode):
    """Weights [cout][cin][1][1] and bias of a probe GEMM.  'dense': normal; 'onehot': one full-mantissa float32 per output channel at input channel
    perm[co % cin] (a permutation, repeated when cout > cin); 'pow2': the same pattern with powers of two and a zero bias; 'zero': zeros."""
    b = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    if mode == 'dense':
        return (rng.standard_normal((cout, cin, 1, 1)) * np.sqrt(2.0 / cin)).astype(np.float32), b
    if mode == 'zero':
        return np.zeros((cout, cin, 1, 1), np.float32), np.zeros(cout, np.float32)
    w = np.zeros((cout, cin, 1, 1), np.float32)
    src = rng.permutation(cin)[np.arange(cout) % cin]
    sign = np.where(rng.random(cout) < 0.5, -1.0, 1.0)
    if mode == 'onehot':
        v = (sign * rng.uniform(0.5, 2.0, cout)).astype(np.float32)
        v = (v.view(np.uint32) | np.uint32(0x00000fff)).view(np.float32)         # low mantissa bits set: the hi / lo residual of the split is never zero
    elif mode == 'pow2':
        v = (sign * np.exp2(rng.integers(-3, 4, cout))).astype(np.float32)
        b = np.zeros(cout, np.float32)
    else:
        raise ValueError(mode)
    w[np.arange(cout), src, 0, 0] = v
    return w, b


def write_probe_model(dirpath, probes, seed=0, c0=16, weights='dense', name='probe'):
    """A graph that puts chosen convolution shapes on real activations, for kernel-level parity checks in diagnostic mode.

    Input 3x300x300 -> dense 3x3/s2 stem 3 -> c0 (no activation; per-channel gains 2^[-3, 3] give signed values of varied magnitude) -> a chain of
    depth-wise 3x3/s2 layers down to the smallest map a probe needs (CHAIN).  Each probe hangs off the chain at its map size and is a dead end:
      ('gemm', cin, cout, hw)           1x1 convolution (the wgmma GEMM when cin % 4 == 0), fed by a 1x1 expansion c0 -> cin unless cin == c0;
                                        its weights follow `weights` (see _probe_weights), every other layer is dense;
      ('dw', c, k, s, hw)               depth-wise k x k / stride s, padding k // 2, fed by an expansion c0 -> c unless c == c0;
      ('conv', cin, cout, k, s, hw)     dense k x k / stride s, padding k // 2, fed the same way.
    A minimal SSD head (4 priors per location, 21 classes) on the 19x19 map closes the graph.
    Returns (param path, bin path, convs): convs maps every convolution layer name to a dict with 'role' (stem / chain / expand / probe / head), 'dw',
    'in' / 'out' (blob names), 'cin', 'cout', 'k', 's', 'p', 'hw' (input map size), 'w' ([cout][cin or 1][k][k] float32) and 'b'."""
    g = Graph(seed)
    convs = {}

    def conv(role, x, cin, cout, hw, k=1, s=1, dw=False, w=None, b=None, gain=1.0):
        y = g.conv(x, cin, cout, k, s, k // 2, gain=gain, dw=dw, w=w, b=b, name=g.name('%s_%s' % (name, role)))
        L = g.layers[-1]
        convs[y] = dict(role=role, dw=dw, cin=cin, cout=cout, k=k, s=s, p=k // 2, hw=hw, w=L[5][1], b=L[5][2], out=y, **{'in': x})
        return y

    data = g.add('Input', [], name='input')
    ws = (g.rng.standard_normal((c0, 3, 3, 3)) * np.sqrt(2.0 / 27) * np.exp2(g.rng.uniform(-3, 3, (c0, 1, 1, 1))) / 64).astype(np.float32)
    chain = {150: conv('stem', data, 3, c0, 300, 3, 2, w=ws)}
    smallest = min([19] + [p[-1] for p in probes])
    for a, bsz in zip(CHAIN, CHAIN[1:]):
        if bsz < smallest:
            break
        chain[bsz] = conv('chain', chain[a], c0, c0, a, 3, 2, dw=True, gain=1.5)

    def feed(c, hw):
        return chain[hw] if c == c0 else conv('expand', chain[hw], c0, c, hw)

    for pr in probes:
        if pr[0] == 'gemm':
            _, cin, cout, hw = pr
            w, b = _probe_weights(g.rng, cin, cout, weights)
            conv('probe', feed(cin, hw), cin, cout, hw, w=w, b=b)
        elif pr[0] == 'dw':
            _, c, k, s, hw = pr
            conv('probe', feed(c, hw), c, c, hw, k, s, dw=True)
        elif pr[0] == 'conv':
            _, cin, cout, k, s, hw = pr
            conv('probe', feed(cin, hw), cin, cout, hw, k, s)
        else:
            raise ValueError(pr)
    n0 = len(g.layers)
    _head(g, data, [(chain[19], c0)], 4, '-23300=1,60.000000 -23301=1,105.0 -23302=1,2.000000 7=1')
    for L in g.layers[n0:]:
        if L[0] == 'Convolution':
            convs[L[3][0]] = dict(role='head', dw=False, cin=c0, cout=len(L[5][2]), k=1, s=1, p=0, hw=19, w=L[5][1], b=L[5][2], out=L[3][0],
                                  **{'in': chain[19]})
    os.makedirs(dirpath, exist_ok=True)
    pp, bp = os.path.join(dirpath, name + '.param'), os.path.join(dirpath, name + '.bin')
    g.write(pp, bp)
    return pp, bp, convs


def write_tail_model(dirpath, seed=0, name='tails'):
    """Odd channel counts through the fused epilogues.  A 16-channel 19x19 map feeds seven 1x1 GEMMs 16 -> 7, one per tail kind the planner
    recognises (ReLU, clip, hard-swish, +tensor, SE gate, SE tail) plus a generic chain (mul by a scalar, ReLU); each result goes back through a
    dense 1x1 convolution 7 -> 16 added onto the map.  The SSD head has 3 priors per location (min, max, one aspect ratio, no flip) on 19x19 and
    10x10: 63-channel confidence pieces, the second at the odd concat offset 19 * 19 * 63 = 22743, written straight into mbox_conf."""
    g = Graph(seed)
    data = g.add('Input', [], name='input')
    x = g.conv(data, 3, 16, 3, 2, 1, gain=1 / 64)                                # activations of order one
    for _ in range(3):
        x = g.relu(g.conv(x, 16, 16, 3, 2, 1, dw=True))                           # 75, 38, 19
    f = x

    def gm():
        return g.conv(f, 16, 7, gain=2.0)

    a = g.relu(gm())                                                              # relu
    cl = g.clip(gm())                                                             # clip
    hs = g.hswish(gm())                                                           # hard-swish
    ad = g.binop(gm(), a, 0)                                                      # + tensor
    se = g.binop(cl, g.hsigmoid(gm()), 2)                                         # SE gate
    st = g.binop(g.binop(hs, g.hsigmoid(gm()), 2), ad, 0)                         # SE tail
    gen = g.relu(g.binop(gm(), g.const(0.5), 2))                                  # generic
    h = f
    for t in (a, cl, hs, ad, se, st, gen):
        h = g.binop(g.conv(t, 7, 16, gain=0.5), h, 0)
    h2 = g.relu(g.conv(h, 16, 16, 3, 2, 1, dw=True))                              # 10
    _head(g, data, [(h, 16), (h2, 16)], 3, '-23300=1,60.000000 -23301=1,105.0 -23302=1,2.000000 7=0')
    os.makedirs(dirpath, exist_ok=True)
    pp, bp = os.path.join(dirpath, name + '.param'), os.path.join(dirpath, name + '.bin')
    g.write(pp, bp)
    return pp, bp


# GEMM shapes (cin, cout, map) for the parity tests, at PROBE_FRAMES frames per batch: BK = 16 (cin <= 16) and 32 with a partial last k-step /
# k-block (20, 36, 100, 964), streamed weights with more k-blocks than ring stages (960, 964), cout < 32 and odd (1, 21, 63: scalar stores),
# an exact tile (32, 256), one channel past a tile (257), several output-channel tiles (600, 1000), 1 / 4 / 25 / 9 pixels per frame, and
# 150 x 150 x 8 pixels (about ten 128-pixel tiles per persistent CTA).  The expansions c0 -> cin are GEMMs as well.
PROBE_FRAMES = 8
GEMM_PROBES = [('gemm', 16, 32, 150), ('gemm', 4, 21, 38), ('gemm', 12, 1, 1), ('gemm', 20, 63, 19), ('gemm', 36, 257, 10), ('gemm', 100, 600, 5),
               ('gemm', 32, 256, 2), ('gemm', 960, 1000, 19), ('gemm', 964, 256, 3)]
# depth-wise: V = 1 (c = 6, 10) and V = 4, k 3 / 5, stride 1 / 2, output maps under 4 rows (YT = 1) and larger, widths that are not a multiple of 4
# (the chain itself adds 3x3/s2 on 16 channels at every size); dense: 3x3 with cin % 4 != 0, 1x1 / stride 2, 1x1 with cin % 4 != 0 and odd cout
KERNEL_PROBES = [('dw', 6, 5, 1, 19), ('dw', 10, 3, 1, 5), ('dw', 6, 3, 2, 10), ('dw', 10, 5, 2, 3), ('dw', 16, 5, 1, 38), ('dw', 16, 5, 2, 19),
                 ('dw', 16, 3, 1, 3), ('dw', 20, 3, 1, 10), ('conv', 6, 8, 3, 1, 19), ('conv', 16, 12, 1, 2, 19), ('conv', 6, 5, 1, 1, 10),
                 ('conv', 10, 20, 3, 2, 10)]


def check_probe_plans(plans):
    """The plan features the GEMM parity tests rely on, on the conv1x1 lines (parse_plan) of a probe graph built from GEMM_PROBES at PROBE_FRAMES."""
    by = {(p['cin'], p['cout'], p['h']): p for p in plans}
    for _, cin, cout, hw in GEMM_PROBES:
        assert (cin, cout, hw) in by, (cin, cout, hw)
    assert by[(16, 32, 150)]['bk'] == 16 and by[(4, 21, 38)]['bk'] == 16 and by[(12, 1, 1)]['bk'] == 16                  # 64-byte swizzle
    for cin in (20, 36, 100):
        assert by[[k for k in by if k[0] == cin][0]]['bk'] == 32
    assert any(p['bk'] == 32 and p['cin'] % 8 for p in plans) and any(p['bk'] == 32 and p['cin'] % 32 and p['kb'] > 1 for p in plans)
    for key in ((960, 1000, 19), (964, 256, 3)):
        p = by[key]
        assert not p['wres'] and p['kb'] > p['stages'], p['line']                                                     # the ring wraps inside a tile
    assert by[(960, 1000, 19)]['n_tiles'] >= 3 and by[(100, 600, 5)]['n_tiles'] >= 3                                 # several output-channel tiles
    assert by[(36, 257, 10)]['n_tiles'] >= 2 and by[(32, 256, 2)]['nt'] * by[(32, 256, 2)]['n_tiles'] == 256
    assert by[(16, 32, 150)]['nt'] == 32 and by[(16, 32, 150)]['n_tiles'] == 1
    assert -(-PROBE_FRAMES * 150 * 150 // 128) >= 10 * 132                                                           # ~10 pixel tiles per CTA
    for key in ((12, 1, 1), (4, 21, 38), (20, 63, 19)):
        assert by[key]['cout'] % 2 and by[key]['off'] is None                                                         # odd pitch: scalar stores
    assert by[(12, 1, 1)]['nt'] == 32 and by[(4, 21, 38)]['nt'] == 32                                                 # fewer than 32 real channels


def parse_plan(describe_text):
    """The conv1x1 lines of sgs_detector_describe as dicts: name, cin, cout, h, w, nt, n_tiles, kb, bk, stages, wres, smem, off (or None), line."""
    import re
    out = []
    for l in describe_text.splitlines():
        if not l.startswith('conv1x1 '):
            continue
        m = re.search(r'geom (\d+)x(\d+)x(\d+)->(\d+)x(\d+)x(\d+) .* tile (\d+)x(\d+) kb (\d+)x(\d+) stages (\d+)( wres)? smem (\d+)', l)
        cin, h, w, cout, _, _, nt, ntl, kb, bk, st, wres, smem = m.groups()
        off = re.search(r' off (\d+)', l)
        out.append(dict(name=l.split()[1], out=l.split()[l.split().index('out') + 1], cin=int(cin), cout=int(cout), h=int(h), w=int(w), nt=int(nt),
                        n_tiles=int(ntl), kb=int(kb), bk=int(bk), stages=int(st), wres=bool(wres), smem=int(smem), off=int(off.group(1)) if off else None,
                        line=l))
    return out


def head_prior_count(maps):
    """Priors per location of each head map (hw, min_size, max_size or None, aspect ratios, flip): min box, max box, each ratio (and its flip)."""
    return [1 + (mx is not None) + len(ars) * (2 if flip else 1) for _, _, mx, ars, flip in maps]


def _f9(v):
    """a float32 parameter as ncnn text that reads back as the same float32"""
    return '%.9g' % float(np.float32(v))


def write_head_model(dirpath, maps, ncls, weights='zero', conf_bias=None, loc_bias=None, nms_thr=0.45, nms_topk=300, keep_topk=100, conf_thr=0.01,
                     seed=0, c=8, conf_gain=1.0, loc_gain=1.0, name='head'):
    """A graph that is mostly SSD head, for the Softmax / DetectionOutput parity tests.

    Input 3x300x300 -> dense 3x3/s2 stem 3 -> c + ReLU -> depth-wise 3x3/s2 + ReLU chain (CHAIN).  A map size off the chain is reached from the
    nearest larger chain map of the same parity by unpadded depth-wise 5x5 / 3x3 layers (-4 / -2 per layer).  Each entry of `maps`,
    (hw, min_size, max_size or None, aspect ratios, flip), gets a conf and a loc 1x1 convolution and a PriorBox (head_prior_count priors per
    location, mmdetection centres, no clip), concatenated in order into mbox_conf / mbox_loc / mbox_priorbox, then
    Reshape -> Softmax (blob mbox_conf_softmax) -> Flatten -> DetectionOutput with the given parameters, written so that they read back as the
    same float32.
      weights='zero'    head weights are zero: conf_bias[i] ([npr][ncls], broadcast) and loc_bias[i] ([npr][4], default 0) are the outputs at every
                        location of map i, so every location of a prior type scores the same and, with loc 0, every box is its prior box decoded with zero offsets
                        (the same float32 operations on the device and in the restatement);
      weights='random'  normal head weights (gain conf_gain / loc_gain); biases as given, else random.
    Returns (param path, bin path, priors per location of each map)."""
    g = Graph(seed)
    data = g.add('Input', [], name='input')
    chain = {150: g.relu(g.conv(data, 3, c, 3, 2, 1, gain=1 / 64))}
    for a, b in zip(CHAIN, CHAIN[1:]):
        chain[b] = g.relu(g.conv(chain[a], c, c, 3, 2, 1, dw=True, gain=1.5))
    nprs = head_prior_count(maps)
    locs, confs, priors = [], [], []
    for i, ((hw, mn, mx, ars, flip), npr) in enumerate(zip(maps, nprs)):
        size = min(s for s in CHAIN if s >= hw and (s - hw) % 2 == 0)
        f = chain[size]
        while size > hw:
            k = 5 if size - hw >= 4 else 3
            f = g.relu(g.conv(f, c, c, k, 1, 0, dw=True, gain=1.5))
            size -= k - 1
        zero = weights == 'zero'
        if not zero and weights != 'random':
            raise ValueError(weights)
        cb = conf_bias[i] if conf_bias is not None else (None if not zero else 0.0)
        lb = loc_bias[i] if loc_bias is not None else (None if not zero else 0.0)
        cb = None if cb is None else np.broadcast_to(np.asarray(cb, np.float32), (npr, ncls)).reshape(-1).copy()
        lb = None if lb is None else np.broadcast_to(np.asarray(lb, np.float32), (npr, 4)).reshape(-1).copy()
        cf = g.conv(f, c, npr * ncls, gain=conf_gain, w=np.zeros((npr * ncls, c, 1, 1), np.float32) if zero else None, b=cb)
        confs.append(g.add('Flatten', [g.add('Permute', [cf], '0=3')]))
        lc = g.conv(f, c, npr * 4, gain=loc_gain, w=np.zeros((npr * 4, c, 1, 1), np.float32) if zero else None, b=lb)
        locs.append(g.add('Flatten', [g.add('Permute', [lc], '0=3')]))
        pb = '-23300=1,%s' % _f9(mn)
        if mx is not None:
            pb += ' -23301=1,%s' % _f9(mx)
        if ars:
            pb += ' -23302=%d,%s' % (len(ars), ','.join(_f9(a) for a in ars))
        priors.append(g.add('PriorBox', [f, data], pb + ' 3=0.100000 4=0.100000 5=0.200000 6=0.200000 7=%d 8=0 9=-233 10=-233 11=-233.000000 '
                                                        '12=-233.000000 13=0.500000 14=1 15=1' % (1 if flip else 0)))
    loc = g.add('Concat', locs, '0=0', name='mbox_loc')
    conf = g.add('Concat', confs, '0=0', name='mbox_conf')
    pri = g.add('Concat', priors, '0=1', name='mbox_priorbox')
    sm = g.add('Softmax', [g.add('Reshape', [conf], '0=%d 1=-1' % ncls)], '0=1 1=1', name='mbox_conf_softmax')
    g.add('DetectionOutput', [loc, g.add('Flatten', [sm]), pri], '0=%d 1=%s 2=%d 3=%d 4=%s' % (ncls, _f9(nms_thr), nms_topk, keep_topk, _f9(conf_thr)),
          name='detection_out')
    os.makedirs(dirpath, exist_ok=True)
    pp, bp = os.path.join(dirpath, name + '.param'), os.path.join(dirpath, name + '.bin')
    g.write(pp, bp)
    return pp, bp, nprs


HEAD_MAPS = [(19, 60.0, 105.0, (2.0,), True), (10, 105.0, 150.0, (2.0, 3.0), True)]        # 19 * 19 * 4 + 10 * 10 * 6 = 2044 priors
CAP_MAP = (32, 30.0, 45.0, (2.0,), True)                                                 # 32 * 32 * 4 = 4096 priors (kDetSortCap)


def head_scene(name):
    """write_head_model keyword arguments of the graphs of tests/test_gpu_detector_head.py.
      planted  zero head weights, 21 classes; conf logits per (prior type, class) from {-3, 0, 1, 2.5} (background 2): exact score ties inside a
               class (every location of a prior type) and across classes (equal logits of one prior type); the person class (15) high on one prior
               type of the 10x10 map; several classes with more candidates than nms_top_k,
               keep_top_k 200 (a score tie across two classes falls inside it);
      iou      one 1x1 map with a min and a max box (concentric): class 1 scores the min box above the max box;
      cap      4096 priors, 33 classes, every prior above conf_thr in every class (logits {-0.5, 0, 0.5}), nms_thr 1 (nothing suppressed),
               nms_top_k 256: (33 - 1) * 256 = 8192 kept entries reach the merge (kMergeCap), keep_top_k 1024;
      random   random head weights and biases, 21 classes (random32 / random40: 32 / 40, the last Softmax register width and the loop path),
               conf_thr 0.3; candidates depend on the frame."""
    rng = np.random.default_rng(5)
    if name == 'planted':
        nprs = head_prior_count(HEAD_MAPS)
        cb = [rng.choice(np.array([-3.0, 0.0, 1.0, 2.5], np.float32), (n, 21)) for n in nprs]
        for b in cb:
            b[:, 0] = 2.0
        cb[1][2, 15] = 4.0
        return dict(maps=HEAD_MAPS, ncls=21, conf_bias=cb, keep_topk=200)
    if name == 'iou':
        return dict(maps=[(1, 60.0, 105.0, (), False)], ncls=2, conf_bias=[[[0.0, 1.0], [0.0, 0.0]]])
    if name == 'cap':
        return dict(maps=[CAP_MAP], ncls=33, conf_bias=[rng.choice(np.array([-0.5, 0.0, 0.5], np.float32), (4, 33))], nms_thr=1.0, nms_topk=256,
                    keep_topk=1024, conf_thr=0.001)
    if name in ('random', 'random32', 'random40'):
        ncls = int(name[6:] or 21)
        cb = [np.concatenate([np.full((n, 1), 4.0), rng.normal(0, 0.5, (n, ncls - 1))], 1) for n in head_prior_count(HEAD_MAPS)]
        return dict(maps=HEAD_MAPS, ncls=ncls, weights='random', conf_bias=cb, conf_gain=2.0, loc_gain=1.0, conf_thr=0.3, seed=7,
                    nms_topk=300 if ncls == 21 else 200)
    raise ValueError(name)


def nms_iou(a, b):
    """float32 IoU of box b against kept box a ([xmin, ymin, xmax, ymax]) in detout_class_kernel's operation order"""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    inter = np.float32(0)
    if not (b[0] > a[2] or b[2] < a[0] or b[1] > a[3] or b[3] < a[1]):
        inter = (min(a[2], b[2]) - max(a[0], b[0])) * (min(a[3], b[3]) - max(a[1], b[1]))
    area = (b[2] - b[0]) * (b[3] - b[1])
    return np.float32(inter / ((a[2] - a[0]) * (a[3] - a[1]) + area - inter))


def synthetic_rgb(h, w, seed):
    rng = np.random.default_rng(seed)
    img = np.full((h, w, 3), 110, np.float32) + rng.normal(0, 6, (h, w, 3))
    for _ in range(60):
        x0, y0 = rng.integers(0, w - 8), rng.integers(0, h - 8)
        x1, y1 = min(w, x0 + rng.integers(8, w // 3)), min(h, y0 + rng.integers(8, h // 3))
        img[y0:y1, x0:x1] = rng.integers(0, 256, 3)
    return np.clip(img, 0, 255).astype(np.uint8)
