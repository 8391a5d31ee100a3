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

    def conv(self, x, cin, cout, k=1, s=1, p=0, gain=1.0, dw=False, w=None, b=None, name=None, bias=True, dil=1):
        """bias=False: bias_term 0 (5=0) and no bias floats in the weight file; dil: dilation (2= / 12=)"""
        fan = k * k * (1 if dw else cin)
        if w is None:
            w = (self.rng.standard_normal((cout, 1 if dw else cin, k, k)) * gain * np.sqrt(2.0 / fan)).astype(np.float32)
        if b is None and bias:
            b = (self.rng.standard_normal(cout) * 0.1).astype(np.float32)
        prm = '0=%d 1=%d 11=%d 2=%d 12=%d 3=%d 13=%d 4=%d 14=%d 5=%d 6=%d' % (cout, k, k, dil, dil, s, s, p, p, int(bias), w.size)
        if dw:
            prm += ' 7=%d' % cout
        return self.add('ConvolutionDepthWise' if dw else 'Convolution', [x], prm, [np.zeros(1, np.uint32), w] + ([b] if bias else []), name=name)

    def relu(self, x): return self.add('ReLU', [x])
    def clip(self, x, lo=0.0, hi=6.0): return self.add('Clip', [x], '0=%f 1=%f' % (lo, hi))
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


TAIL_KINDS = ('relu', 'clip', 'hswish', 'add', 'se_gate', 'se_tail', 'generic')      # the tails epi_kind (detector.cu) recognises, and its generic chain
TENSOR_TAILS = ('add', 'se_gate', 'se_tail')                                        # the kinds that read same-shape operand tensors
TAIL_OPERANDS = {'add': 1, 'se_gate': 1, 'se_tail': 2}                              # operand tensors t1, t2 each kind reads


def _tail(g, kind, y, ops):
    """The tail `kind` after y, as ncnn exports it (ops: the operand blobs t1, t2); returns its last blob:
      relu     ReLU(y)                      clip     Clip(y, 0, 6)                  hswish   y * Clip(y + 3, 0, 6) / 6
      add      y + t1                       se_gate  t1 * (Clip(y + 3, 0, 6) / 6)   se_tail  t1 * (Clip(y + 3, 0, 6) / 6) + t2
      generic  ReLU(y * 0.5)"""
    if kind == 'relu':
        return g.relu(y)
    if kind == 'clip':
        return g.clip(y)
    if kind == 'hswish':
        return g.hswish(y)
    if kind == 'add':
        return g.binop(y, ops[0], 0)
    if kind == 'se_gate':
        return g.binop(ops[0], g.hsigmoid(y), 2)
    if kind == 'se_tail':
        return g.binop(g.binop(ops[0], g.hsigmoid(y), 2), ops[1], 0)
    if kind == 'generic':
        return g.relu(g.binop(y, g.const(0.5), 2))
    raise ValueError(kind)


def _wide_tail_cases():
    """Cases (kind, cin, cout, hw) of write_wide_tail_model, planned at PROBE_FRAMES frames per batch (plan_tiling's cost model, one H100 of 132 SMs):
      grid    every kind at every tile width NT = 32 ... 256 with Cin 40 (two 32-float k-blocks, the second partial): Cout <= 128 on the 19x19 map (one
              N-tile of roundup32(Cout), 23 pixel tiles), Cout 129-256 on 38x38 (91 pixel tiles: one N-tile of roundup32(Cout) is cheaper than two);
              Cout = NT or NT - 4 (a partial last 8-channel group) in a checkerboard over (kind, NT);
      Cin 16  (16-float k-blocks) ReLU at NT 32 and 64 and +tensor at NT 32 (the reference model has these), clip at 128, hard-swish at 256, the
              generic chain at 192, and three of the cases below;
      extras  streamed weights (Cin 96: 3 k-blocks of 2 x NT x 32 floats > 128 KB) under hard-swish (NT 256) and the SE tail (NT 224); each tensor kind
              on Cout 400 at 38x38 (two N-tiles of 224, 176 real channels in the second: its chunk 6 is cut off) and on the odd Cout 161 (NT 192,
              scalar stores); hard-swish on Cout 1000 at 10x10 (eight N-tiles of 128, the last with 104 channels); the SE tail on 75x75 (352 pixel
              tiles: several per persistent CTA).  Every map leaves a partial last pixel tile (8 * hw^2 is not a multiple of 128)."""
    cases = []
    for i, kind in enumerate(TAIL_KINDS):
        for j in range(8):
            nt = 32 * (j + 1)
            cases.append((kind, 40, nt - 4 if (i + j) % 2 else nt, 19 if nt <= 128 else 38))
    cases += [('relu', 16, 30, 19), ('relu', 16, 64, 19), ('add', 16, 32, 19), ('clip', 16, 124, 19), ('hswish', 16, 252, 38), ('generic', 16, 190, 38),
              ('hswish', 96, 256, 38), ('se_tail', 96, 224, 38), ('add', 40, 400, 38), ('se_gate', 16, 400, 38), ('se_tail', 40, 400, 38),
              ('add', 16, 161, 38), ('se_gate', 40, 161, 38), ('se_tail', 16, 161, 38), ('hswish', 40, 1000, 10), ('se_tail', 40, 96, 75)]
    return cases


WIDE_TAIL_CASES = _wide_tail_cases()


def write_wide_tail_model(dirpath, seed=0, cases=WIDE_TAIL_CASES, name='wide_tails'):
    """Fused element-wise tails on 1x1 GEMMs of chosen shapes, for the fused == per-layer and float32 restatement checks of
    tests/test_gpu_detector_fused_tails.py.  The trunk is write_probe_model's (3x3/s2 stem 3 -> 16 with per-channel gains, depth-wise 3x3/s2 chain);
    a feed of `cin` channels at map `hw` is the chain map itself (cin 16) or one dense 1x1 expansion 16 -> cin, shared by every case on it.  Each
    case (kind, cin, cout, hw) hangs a dense 1x1 GEMM y = W x + b (cin -> cout) off its feed and puts the tail after it, as ncnn exports it:
      relu     ReLU(y)                      clip     Clip(y, 0, 6)                  hswish   y * Clip(y + 3, 0, 6) / 6
      add      y + t1                       se_gate  t1 * (Clip(y + 3, 0, 6) / 6)   se_tail  t1 * (Clip(y + 3, 0, 6) / 6) + t2
      generic  ReLU(y * 0.5)
    t1, t2: further dense 1x1 convolutions cin -> cout of the same feed, written before y so that they exist when y's GEMM runs.  Each tail output
    is a dead end; write_probe_model's minimal SSD head on the 19x19 map closes the graph.
    Returns (param path, bin path, info, head): info[i] = dict(kind, cin, cout, hw, x (feed blob), y (the GEMM's output blob), ops (operand blobs
    t1, t2), out (the tail's final blob), w ([cout][cin] float32), b) of cases[i]; head = the output blobs of the head convolutions."""
    g = Graph(seed)
    data = g.add('Input', [], name='input')
    ws = (g.rng.standard_normal((16, 3, 3, 3)) * np.sqrt(2.0 / 27) * np.exp2(g.rng.uniform(-3, 3, (16, 1, 1, 1))) / 64).astype(np.float32)
    chain = {150: g.conv(data, 3, 16, 3, 2, 1, w=ws)}
    smallest = min([19] + [c[3] for c in cases])
    for a, bsz in zip(CHAIN, CHAIN[1:]):
        if bsz < smallest:
            break
        chain[bsz] = g.conv(chain[a], 16, 16, 3, 2, 1, dw=True, gain=1.5)
    feeds = {}

    def feed(cin, hw):
        if (cin, hw) not in feeds:
            feeds[(cin, hw)] = chain[hw] if cin == 16 else g.conv(chain[hw], 16, cin)
        return feeds[(cin, hw)]

    info = []
    for kind, cin, cout, hw in cases:
        x = feed(cin, hw)
        ops = [g.conv(x, cin, cout) for _ in range(TAIL_OPERANDS.get(kind, 0))]
        y = g.conv(x, cin, cout, name=g.name('wide_%s_' % kind))
        w, b = g.layers[-1][5][1].reshape(cout, cin), g.layers[-1][5][2]
        info.append(dict(kind=kind, cin=cin, cout=cout, hw=hw, x=x, y=y, ops=ops, out=_tail(g, kind, y, ops), w=w, b=b))
    n0 = len(g.layers)
    _head(g, data, [(chain[19], 16)], 4, '-23300=1,60.000000 -23301=1,105.0 -23302=1,2.000000 7=1')
    head = [L[3][0] for L in g.layers[n0:] if L[0] == 'Convolution']
    os.makedirs(dirpath, exist_ok=True)
    pp, bp = os.path.join(dirpath, name + '.param'), os.path.join(dirpath, name + '.bin')
    g.write(pp, bp)
    return pp, bp, info, head


DW_KS = ((3, 1), (3, 2), (5, 1), (5, 2))
# depth-wise variant -> (channels, {stride: input map}): V1 (odd C: one channel per thread), V4Y2 (float4, two output rows per thread: output map
# 19x19, odd and not a multiple of 4 wide), V4Y1 (float4, one row: output maps of 2 and 3 rows)
DW_VARIANTS = {'V1': (7, {1: 5, 2: 10}), 'V4Y2': (16, {1: 19, 2: 38}), 'V4Y1': (24, {1: 2, 2: 5})}
# dense direct shapes (cin, k, s, dil, input map), rotated over the conv_small_kernel cases
CONV_SHAPES = ((6, 3, 1, 1, 19), (10, 3, 2, 1, 19), (16, 1, 2, 1, 19), (6, 1, 1, 1, 10), (6, 3, 1, 2, 10))


def _direct_tail_cases():
    """Cases of write_direct_tail_model, each ('dw', kind, variant, k, s, bias) / ('conv', kind, cout, shape index, bias) / ('stem', kind, bias) /
    ('gemm', kind, cout, bias) / ('cat',) / ('chain', name):
      dw     every TAIL_KINDS entry in each depth-wise variant of DW_VARIANTS (dwconv_kernel<K, S, V, YT>), (K, S) rotating over DW_KS with the kind
             and the variant, so that each of 3/1, 3/2, 5/1, 5/2 meets every variant and at least one tensor-reading kind; one bias-free case
             (relu) per variant;
      conv   every kind on Cout 16 (float4 path), Cout 12 (second 8-channel block partial: scalar path) and Cout 5 (scalar), CONV_SHAPES rotating
             (3x3 s1 Cin 6, 3x3 s2 Cin 10, 1x1 s2, 1x1 Cin 6, 3x3 dilation 2), all through conv_small_kernel; bias-free cases on the float4 path
             (hswish, Cout 16) and the scalar path (relu, Cout 5);
      stem   one 3 -> 16 3x3/s2 stem per kind off the input (conv_first_kernel), its tensor operands further stems; one bias-free stem (clip);
      gemm   bias-free 1x1 GEMMs 16 -> Cout on the 19x19 chain map (the null bias of conv1x1_tc_kernel): Cout 24 on a narrow tile (NT 32, two CTAs
             per SM, bias loaded at each use) under hard-swish, Cout 100 on a wide tile (NT 128, bias loaded per chunk) under the SE tail;
      cat    the SSD head: 3x3 conv_small_kernel pieces with non-tensor tails written straight into mbox_conf / mbox_loc, on the 5x5 (4 priors),
             3x3 (3 priors) and 2x2 (4 priors) maps: mbox_conf is 2100 + 567 + 336 = 3003 floats per frame, so its 84-channel first piece sits at
             offset 0 (a multiple of 4) with a frame stride that is not, and its third piece at the odd offset 2667;
      chain  'cut': a depth-wise output whose tail's second value has a second element-wise reader: build_tail keeps the longest valid prefix
             (add, relu), the rest runs through eltwise_kernel, one of whose values has two readers again (eltwise_chain stops there);
             'long': ten steps after a 3x3 conv: eight fused, two in one stand-alone eltwise_kernel;
             'ops': sub, sub(rev) by a tensor first operand, div 0.75, clip(-1, 2.5), add 2, div(rev) of that tensor, div by a tensor >= 1;
             'start': y + relu(y) (SRC_START inside a generic tail)."""
    cases = []
    for v, var in enumerate(DW_VARIANTS):
        for i, kind in enumerate(TAIL_KINDS):
            k, s = DW_KS[(i + v) % 4]
            cases.append(('dw', kind, var, k, s, True))
        cases.append(('dw', 'relu', var, *DW_KS[(v + 2) % 4], False))
    j = 0
    for cout in (16, 12, 5):
        for kind in TAIL_KINDS:
            cases.append(('conv', kind, cout, j % len(CONV_SHAPES), True))
            j += 1
    cases += [('conv', 'hswish', 16, 0, False), ('conv', 'relu', 5, 1, False)]
    cases += [('stem', kind, True) for kind in TAIL_KINDS] + [('stem', 'clip', False)]
    cases += [('gemm', 'hswish', 24, False), ('gemm', 'se_tail', 100, False)]
    cases += [('cat',)] + [('chain', n) for n in ('cut', 'long', 'ops', 'start')]
    return cases


DIRECT_TAIL_CASES = _direct_tail_cases()
CAT_PIECES = ((5, 4, 'hswish', 'clip'), (3, 3, 'relu', 'generic'), (2, 4, 'generic', 'hswish'))      # (map, priors, conf tail, loc tail)


def write_direct_tail_model(dirpath, seed=0, cases=DIRECT_TAIL_CASES, name='direct_tails'):
    """Fused element-wise tails on the direct kernels (depth-wise, conv_small_kernel, conv_first_kernel) and stand-alone element-wise chains, for
    tests/test_gpu_detector_direct_tails.py; 8-frame batches (PROBE_FRAMES).  The trunk is write_probe_model's (3x3/s2 stem 3 -> 16 with
    per-channel gains, depth-wise 3x3/s2 chain down to 2x2, here with a third of the gain); a feed of c channels at map hw is the chain map
    itself (c 16) or one dense 1x1 expansion 16 -> c.  Tails as _tail writes them; tensor operands are convolutions of the tailed layer's own geometry on the same feed, written
    before it.  The SSD head is the 'cat' case (every case list needs it: it closes the graph).
    Returns (param path, bin path, info, head): info[i] = dict(case, family ('dw' / 'conv' / 'stem' / 'gemm' / 'cat' / 'chain'), kind, variant (dw),
    conv (the tailed convolution: in, out, dw, cin, cout, k, s, p, dil, hw, w, b or None), ops (operand blobs), out (the tail's last blob)) for each
    tailed convolution of cases[i] (the 'cat' case: one entry per head piece; 'chain' entries carry outs, every blob of the chain);
    head = the head convolutions' outputs."""
    g = Graph(seed)
    data = g.add('Input', [], name='input')
    ws = (g.rng.standard_normal((16, 3, 3, 3)) * np.sqrt(2.0 / 27) * np.exp2(g.rng.uniform(-3, 3, (16, 1, 1, 1))) / 64).astype(np.float32)
    chain = {150: g.conv(data, 3, 16, 3, 2, 1, w=ws)}
    for a, bsz in zip(CHAIN, CHAIN[1:]):
        if bsz < 2:
            break
        chain[bsz] = g.conv(chain[a], 16, 16, 3, 2, 1, dw=True, gain=0.5)          # activations stay of order one down the chain
    feeds = {}

    def feed(c, hw):
        if (c, hw) not in feeds:
            feeds[(c, hw)] = chain[hw] if c == 16 else g.conv(chain[hw], 16, c)
        return feeds[(c, hw)]

    def conv(x, cin, cout, k, s, hw, dw=False, dil=1, bias=True, gain=1.0, tag='d'):
        p = dil * (k // 2)
        y = g.conv(x, cin, cout, k, s, p, gain=gain, dw=dw, bias=bias, dil=dil, name=g.name(tag))
        L = g.layers[-1]
        return y, dict(dw=dw, cin=cin, cout=cout, k=k, s=s, p=p, dil=dil, hw=hw, w=L[5][1], b=L[5][2] if bias else None, out=y, **{'in': x})

    info, head = [], []
    for case in cases:
        fam = case[0]
        if fam in ('dw', 'conv', 'stem', 'gemm'):
            kind, bias = case[1], case[-1]
            if fam == 'dw':
                _, _, var, k, s, _ = case
                c, maps = DW_VARIANTS[var]
                x, geo = feed(c, maps[s]), dict(cin=c, cout=c, k=k, s=s, hw=maps[s], dw=True)
            elif fam == 'conv':
                cin, k, s, dil, hw = CONV_SHAPES[case[3]]
                x, geo = feed(cin, hw), dict(cin=cin, cout=case[2], k=k, s=s, hw=hw, dil=dil)
            elif fam == 'gemm':
                x, geo = chain[19], dict(cin=16, cout=case[2], k=1, s=1, hw=19)
            else:
                x, geo = data, dict(cin=3, cout=16, k=3, s=2, hw=300, gain=1 / 16)
            ops = [conv(x, **geo)[0] for _ in range(TAIL_OPERANDS.get(kind, 0))]
            y, cv = conv(x, bias=bias, tag='%s_%s_' % (fam, kind), **geo)
            info.append(dict(case=case, family=fam, kind=kind, variant=case[2] if fam == 'dw' else None, conv=cv, ops=ops, out=_tail(g, kind, y, ops)))
        elif fam == 'chain':
            info.append(_chain_case(g, case, feed, conv))
        elif fam != 'cat':
            raise ValueError(case)
    ncls = 21
    locs, confs, priors = [], [], []
    for hw, npr, ck, lk in CAT_PIECES:
        f = chain[hw]
        for what, cout, kind, dst in (('conf', npr * ncls, ck, confs), ('loc', npr * 4, lk, locs)):
            y, cv = conv(f, 16, cout, 3, 1, hw, gain=2.5 if kind == 'hswish' else 1.0, tag='cat_%s_' % what)     # hard-swish inputs past +-3
            if what == 'conf':
                cv['b'][15::ncls] += np.float32(2.0)                              # the person class (15) shows up among the detections
            head.append(y)
            out = _tail(g, kind, y, [])
            info.append(dict(case=('cat',), family='cat', kind=kind, variant=what, conv=cv, ops=[], out=out))
            dst.append(g.add('Flatten', [g.add('Permute', [out], '0=3')]))
        priors.append(g.add('PriorBox', [f, data], '-23300=1,60.000000 -23301=1,105.0 -23302=1,2.000000 7=%d 3=0.100000 4=0.100000 5=0.200000 '
                                                   '6=0.200000 8=0 9=-233 10=-233 11=-233.000000 12=-233.000000 13=0.500000 14=1 15=1' % (npr == 4)))
    loc = g.add('Concat', locs, '0=0', name='mbox_loc')
    conf = g.add('Concat', confs, '0=0', name='mbox_conf')
    pri = g.add('Concat', priors, '0=1', name='mbox_priorbox')
    sm = g.add('Softmax', [g.add('Reshape', [conf], '0=%d 1=-1' % ncls)], '0=1 1=1')
    g.add('DetectionOutput', [loc, g.add('Flatten', [sm]), pri], '0=%d 1=0.450000 2=300 3=100 4=0.010000' % ncls, name='detection_out')
    os.makedirs(dirpath, exist_ok=True)
    pp, bp = os.path.join(dirpath, name + '.param'), os.path.join(dirpath, name + '.bin')
    g.write(pp, bp)
    return pp, bp, info, head


def _chain_case(g, case, feed, conv):
    """The element-wise chains of _direct_tail_cases ('chain', name): info entry with outs = every blob the chain writes, in graph order"""
    nm = case[1]
    sc = g.const
    if nm == 'cut':                                   # depth-wise 3x3/s1 on 16 channels at 19x19 (V4Y2)
        y, cv = conv(feed(16, 19), 16, 16, 3, 1, 19, dw=True, tag='chain_cut_')
        a = g.binop(y, sc(1.0), 0); r = g.relu(a); m = g.binop(r, sc(2.0), 2); c = g.clip(m, -1.0, 2.5); s = g.binop(r, sc(0.25), 1); q = g.relu(m)
        outs, ops = [a, r, m, c, s, q], []
    elif nm == 'long':                                # 3x3/s1 conv_small_kernel 6 -> 12 at 19x19
        y, cv = conv(feed(6, 19), 6, 12, 3, 1, 19, tag='chain_long_')
        v, outs = y, []
        for op, val in ((0, 0.5), (2, 1.5), ('relu', None), (1, 0.25), ('clip', (-2.0, 3.0)), (2, 0.75), (0, -0.125), (3, 1.25), (2, 2.0), ('relu', None)):
            v = g.relu(v) if op == 'relu' else g.clip(v, *val) if op == 'clip' else g.binop(v, sc(val), op)
            outs.append(v)
        ops = []
    elif nm == 'ops':                                 # depth-wise 5x5/s1 on 16 channels at 19x19 (V4Y2)
        x = feed(16, 19)
        t1 = conv(x, 16, 16, 5, 1, 19, dw=True)[0]
        tpos = g.binop(g.relu(conv(x, 16, 16, 5, 1, 19, dw=True)[0]), sc(1.0), 0)          # >= 1: a divisor bounded away from zero
        y, cv = conv(x, 16, 16, 5, 1, 19, dw=True, tag='chain_ops_')
        a1 = g.binop(y, sc(0.5), 1); a2 = g.binop(t1, a1, 1); a3 = g.binop(a2, sc(0.75), 3); a4 = g.clip(a3, -1.0, 2.5)
        a5 = g.binop(a4, sc(2.0), 0); a6 = g.binop(t1, a5, 3); a7 = g.binop(a6, tpos, 3)
        outs, ops = [a1, a2, a3, a4, a5, a6, a7], [t1, tpos]
    elif nm == 'start':                               # 1x1 conv_small_kernel 6 -> 5 at 10x10
        y, cv = conv(feed(6, 10), 6, 5, 1, 1, 10, tag='chain_start_')
        r = g.relu(y)
        outs, ops = [r, g.binop(y, r, 0)], []
    else:
        raise ValueError(nm)
    return dict(case=case, family='chain', kind=nm, variant=None, conv=cv, ops=ops, out=outs[-1], outs=outs)


def plan_tails(describe_text):
    """parse_plan of describe_text, each line with 'steps' (the fused element-wise steps after ' | ': (op, rev, src, value) with src 'scalar' /
    'start' / 'tensor', value the scalar, the clip bounds or the operand blob) and 'kind': epi_kind's classification of the steps (detector.cu) --
    'none', one of TAIL_KINDS.  Like epi_kind it ignores (rev) on add and mul, and takes the hard-swish / hard-sigmoid forms only with the divisor 6
    and an un-reversed division."""
    out = []
    for p in parse_plan(describe_text):
        p['steps'] = tail_steps(p['line'])
        p['kind'] = epi_kind(p['steps'])
        out.append(p)
    return out


def tail_steps(line):
    """the element-wise steps of a describe() line (after ' | ') as plan_tails gives them"""
    steps = []
    for s in line.split(' | ')[1:]:
        t = s.split()
        op, rev = t[0].replace('(rev)', ''), t[0].endswith('(rev)')
        if op in ('relu', 'clip'):
            steps.append((op, rev, None, tuple(float(v) for v in t[1:])))
        elif t[1] == 'start':
            steps.append((op, rev, 'start', None))
        elif len(t) == 4 and t[2] == 'buf':                  # '<blob> buf <n>' (blob names may be numbers)
            steps.append((op, rev, 'tensor', t[1]))
        else:
            steps.append((op, rev, 'scalar', float(t[1])))
    return steps


def epi_kind(steps):
    """epi_kind's tail kind of the (op, rev, src, value) steps of plan_tails"""
    def is_(i, op, src=None):
        return steps[i][0] == op and (src is None or steps[i][2] == src)

    def div6(i):
        return is_(i, 'div', 'scalar') and not steps[i][1] and steps[i][3] == 6.0

    n = len(steps)
    if n == 0:
        return 'none'
    if n == 1 and is_(0, 'relu'):
        return 'relu'
    if n == 1 and is_(0, 'clip'):
        return 'clip'
    if n == 1 and is_(0, 'add', 'tensor'):
        return 'add'
    if n == 4 and is_(0, 'add', 'scalar') and is_(1, 'clip') and is_(2, 'mul', 'start') and div6(3):
        return 'hswish'
    if n == 5 and is_(0, 'add', 'scalar') and is_(1, 'clip') and div6(2) and is_(3, 'mul', 'tensor') and is_(4, 'add', 'tensor'):
        return 'se_tail'
    if n == 4 and is_(0, 'add', 'scalar') and is_(1, 'clip') and div6(2) and is_(3, 'mul', 'tensor'):
        return 'se_gate'
    return 'generic'


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
