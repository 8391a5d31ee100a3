"""The detector's convolution kernels against float64, each on the exact input the GPU read: diagnostic mode (flags bit 0) keeps every blob of every
frame, so a kernel's input X and output Y are both read back and the reference R is recomputed from X alone -- no error carried in from earlier
layers, and the bounds can be tight.  The graphs come from tests/detector_model.py (write_probe_model / write_tail_model): shapes the synthetic SSD
graph never reaches (several k-blocks and N-tiles, streamed weights, odd channel counts and concat offsets, 1-pixel maps, 8-frame batches).

1x1 GEMM (conv1x1_tc.cuh), u = 2^-24, S = |X| @ |W|^T, K = Cin:
  (a) dense random weights: |Y - R| <= (ALPHA + BETA * ceil(K / 8)) * u * S + u * |R| for every element, and max(|Y - R| / S) at most 1/16 of the same
      statistic for plain TF32 (tf32(X) @ tf32(W)^T, exact accumulation) on the same data;
  (b) one full-mantissa weight per output channel: |Y - x w - b| <= 2^-20 |x w| + u |Y|  (plain TF32 or a lost cross term: ~2^-12);
  (c) one power-of-two weight per output channel, zero bias: Y == w * (hi(x) + lo(x)) exactly (every product and partial sum is exact), so any
      wrong swizzle offset, fragment row, k-step, tile offset, frame offset or store shows up at a known (frame, pixel, channel).
Depth-wise and dense direct convolutions: |Y - R| <= 2 n u S + u |R|, n = products per output (k^2 or k^2 Cin), FP32 FMA chains from zero + bias."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import detector_model as DM  # noqa: E402
import detector_oracle as DO  # noqa: E402
import ncnn_model as NM  # noqa: E402
from pysgs import binding as B  # noqa: E402
from test_gpu_detector import _check_rows, _run  # noqa: E402

U = 2.0 ** -24
F = DM.PROBE_FRAMES
# Error model of one GEMM output, derivation:
#   split: x = hi + lo + e with |x - hi| <= 2^-11 |x| (round to 11 significant bits) and |e| <= 2^-11 |x - hi| <= 2^-22 |x|; the same for w.  The kernel
#     forms lo_x hi_w + hi_x lo_w + hi_x hi_w = x w - (lo_x lo_w + e_x w + (hi_x + lo_x) e_w), so each product is off by at most
#     (2^-22 (1 + 2^-11)^2 + 2^-22 + 2^-22 (1 + 2^-22)) |x w| < 3.001 * 2^-22 |x w| = 12.004 u |x w|; summed over k that is 12.004 u S;
#   products: 11 x 11 significant bits, exact in FP32;
#   accumulation: each wgmma k8 step adds 8 exact products to the FP32 accumulator.  Allowing for terms aligned to the largest exponent and truncated
#     (not rounded) to 24 bits, each of the 9 operands loses less than 2u of the largest magnitude and the normalised result another 2u: at most
#     20 u (|acc| + sum |p|) <= 20 u S per step (to first order), three steps (lo*hi, hi*lo, hi*hi) per 8-wide k-step: 60 u S per ceil(K / 8);
#   bias: one rounded addition, u |R| (plus u times the error above, covered by the slack in ALPHA).
ALPHA, BETA = 13, 60


def _frames(seeds):
    return np.stack([DM.synthetic_rgb(480, 640, s) for s in seeds])


def _grab(det, name, c, hw, nf):
    """a blob of the first nf frames as [frame][c][h][w] (sgs_detector_blob returns ncnn's c,h,w order)"""
    return np.stack([det.blob(name, f).reshape(c, hw, hw) for f in range(nf)])


def _pc(a):
    """[frame][c][h][w] -> [frame * pixel][c]"""
    return a.transpose(0, 2, 3, 1).reshape(-1, a.shape[1])


def _out_hw(c):
    return (c['hw'] + 2 * c['p'] - c.get('dil', 1) * (c['k'] - 1) - 1) // c['s'] + 1


def _probe_run(pp, bp, convs, runs, names=None, max_frames=F):
    """One diagnostic handle; runs the batches in `runs` in turn, then reads X and Y of the convolutions `names` for every frame of the last one."""
    det = B.Detector(pp, bp, max_frames=max_frames, flags=B.DET_DIAGNOSTIC)
    for frames in runs:
        _run(det, frames)
    nf = len(runs[-1])
    out = {}
    for n in (names if names is not None else convs):
        c = convs[n]
        out[n] = (_grab(det, c['in'], c['cin'], c['hw'], nf), _grab(det, n, c['cout'], _out_hw(c), nf))
    plan = det.describe()
    det.close()
    return out, plan


def _tf32(a):
    """round to nearest, ties away, to TF32 (10 explicit mantissa bits) on the bit pattern -- split_tf32 of conv1x1_tc.cuh"""
    b = np.ascontiguousarray(a, np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xffffe000)).view(np.float32)


def _split(a):
    hi = _tf32(a)
    return hi, _tf32(np.asarray(a, np.float32) - hi)          # the float32 difference is exact


def _gemm_check(name, X, Y, W, b):
    """(a) on X [pixels][K], Y [pixels][N], W [N][K]: returns (max |Y - R| / S, the same for plain TF32)."""
    Xd, Wd = X.astype(np.float64), W.astype(np.float64)
    R = Xd @ Wd.T + b
    S = np.abs(Xd) @ np.abs(Wd).T
    err = np.abs(Y - R)
    bound = (ALPHA + BETA * math.ceil(X.shape[1] / 8)) * U * S + U * np.abs(R)
    bad = np.argwhere(err > bound)
    assert len(bad) == 0, '%s: %d elements outside the bound, first (pixel, channel) %s: %r vs %r' % (name, len(bad), tuple(bad[0]), Y[tuple(bad[0])], R[tuple(bad[0])])
    T = _tf32(X).astype(np.float64) @ _tf32(W).astype(np.float64).T + b
    m = S > 0
    return float((err[m] / S[m]).max()), float((np.abs(T - R)[m] / S[m]).max())


def _gemm_names(plan):
    return [p['name'] for p in DM.parse_plan(plan)]


@pytest.fixture(scope='module')
def dense(tmp_path_factory):
    pp, bp, convs = DM.write_probe_model(str(tmp_path_factory.mktemp('probe')), DM.GEMM_PROBES + DM.KERNEL_PROBES, 0)
    data, plan = _probe_run(pp, bp, convs, [_frames(range(31, 31 + F))])
    return convs, data, plan


def test_probe_plans_on_the_device(dense):
    DM.check_probe_plans(DM.parse_plan(dense[2]))


def test_gemm_dense_weights_against_float64(dense):
    convs, data, plan = dense
    names = _gemm_names(plan)
    assert len(names) >= 2 * len(DM.GEMM_PROBES)
    for n in names:
        c = convs[n]
        X, Y = data[n]
        r, t = _gemm_check(n, _pc(X), _pc(Y), c['w'].reshape(c['cout'], c['cin']), c['b'])
        print('gemm %-16s %4d -> %4d @ %3dx%-3d x %d frames: max|Y-R|/S %.3g, plain TF32 %.3g, ratio %.0f' %
              (n, c['cin'], c['cout'], c['hw'], c['hw'], F, r, t, t / r if r > 0 else float('inf')))
        assert r * 16 <= t, '%s: compensated error %.3g is not 16x below plain TF32 (%.3g)' % (n, r, t)


@pytest.fixture(scope='module')
def one_hot(tmp_path_factory):
    res = {}
    for mode, seed in (('onehot', 3), ('pow2', 4)):
        pp, bp, convs = DM.write_probe_model(str(tmp_path_factory.mktemp(mode)), DM.GEMM_PROBES, seed, weights=mode)
        probes = [n for n, c in convs.items() if c['role'] == 'probe']
        data, _ = _probe_run(pp, bp, convs, [_frames(range(71, 71 + F))], probes)
        res[mode] = [(n, convs[n]) + data[n] for n in probes]
    return res


def _one_hot_parts(c, X):
    W = c['w'].reshape(c['cout'], c['cin'])
    src = np.argmax(W != 0, axis=1)
    assert np.count_nonzero(W) == c['cout']
    return src, W[np.arange(c['cout']), src]


def test_gemm_compensation_per_element(one_hot):
    for n, c, X, Y in one_hot['onehot']:
        X, Y = _pc(X), _pc(Y)
        src, w = _one_hot_parts(c, X)
        xw = X[:, src].astype(np.float64) * w.astype(np.float64)
        e = np.abs(Y - xw - c['b'])
        ok = e <= 2.0 ** -20 * np.abs(xw) + U * np.abs(Y)
        bad = np.argwhere(~ok)
        assert len(bad) == 0, '%s: %d elements, first (pixel, channel) %s: error %.3g of |x w| %.3g' % (n, len(bad), tuple(bad[0]), e[tuple(bad[0])], abs(xw[tuple(bad[0])]))
        m = xw != 0
        print('gemm one-hot %-16s %4d -> %4d: max |Y - x w - b| / |x w| = %.3g' % (n, c['cin'], c['cout'], (e[m] / np.abs(xw[m])).max()))


def test_gemm_routing_bit_exact(one_hot):
    for n, c, X, Y in one_hot['pow2']:
        hw = c['hw']
        X, Y = _pc(X), _pc(Y)
        assert np.all((X == 0) | (np.abs(X) >= 2.0 ** -100)), 'inputs must be zeros or normal numbers well above the denormal range'
        src, w = _one_hot_parts(c, X)
        assert np.all(c['b'] == 0) and np.all(np.abs(np.frexp(w)[0]) == 0.5)
        hi, lo = _split(X[:, src])
        expect = (hi.astype(np.float64) + lo.astype(np.float64)) * w.astype(np.float64)
        bad = np.argwhere(Y.astype(np.float64) != expect)
        if len(bad):
            p, co = bad[0]
            raise AssertionError('%s: %d of %d outputs differ; first at frame %d, pixel %d, channel %d (input channel %d): %r, expected %r' %
                                 (n, len(bad), Y.size, p // (hw * hw), p % (hw * hw), co, src[co], Y[p, co], expect[p, co]))


def test_short_batch_and_batch_position(tmp_path):
    """A call with fewer frames than max_frames runs its last pixel tile over rows an earlier call left behind: every frame must still pass (a) and
    equal a fresh handle's output bit for bit.  And a frame's outputs do not depend on its position in the batch."""
    pp, bp, convs = DM.write_probe_model(str(tmp_path), DM.GEMM_PROBES, 2)
    det = B.Detector(pp, bp, max_frames=F, flags=B.DET_PLAN_ONLY)
    names = _gemm_names(det.describe())
    det.close()
    full, short = _frames(range(41, 41 + F)), _frames((51, 52, 53))
    stale, _ = _probe_run(pp, bp, convs, [full, short], names)
    fresh, _ = _probe_run(pp, bp, convs, [short], names)
    for n in names:
        c = convs[n]
        X, Y = stale[n]
        assert Y.shape[0] == 3 and Y.tobytes() == fresh[n][1].tobytes(), '%s: output of a 3-frame call depends on what an earlier call left' % n
        r, t = _gemm_check(n, _pc(X), _pc(Y), c['w'].reshape(c['cout'], c['cin']), c['b'])
        assert r * 16 <= t, n
    perm = np.array([5, 1, 2, 3, 4, 0, 7, 6])
    a, _ = _probe_run(pp, bp, convs, [full], names)
    b, _ = _probe_run(pp, bp, convs, [full[perm]], names)
    for n in names:
        assert a[n][1][perm].tobytes() == b[n][1].tobytes(), '%s: a frame\'s output depends on its batch position' % n


def _direct_ref(c, X):
    """float64 convolution of X [frame][cin][h][w] with ncnn weights [cout][cin or 1][k][k], symmetric zero padding, dilation c['dil'] (default 1),
    bias c['b'] (None: none): (R, S) as [frame][cout][oh][ow]"""
    k, s, p, d, oh = c['k'], c['s'], c['p'], c.get('dil', 1), _out_hw(c)
    Xp = np.pad(X.astype(np.float64), ((0, 0), (0, 0), (p, p), (p, p)))
    W = c['w'].astype(np.float64)
    R = np.zeros((X.shape[0], c['cout'], oh, oh)); S = np.zeros_like(R)
    for ky in range(k):
        for kx in range(k):
            patch = Xp[:, :, ky * d:ky * d + s * (oh - 1) + 1:s, kx * d:kx * d + s * (oh - 1) + 1:s]
            if c['dw']:
                wk = W[:, 0, ky, kx][None, :, None, None]
                R += patch * wk; S += np.abs(patch) * np.abs(wk)
            else:
                R += np.einsum('fchw,oc->fohw', patch, W[:, :, ky, kx]); S += np.einsum('fchw,oc->fohw', np.abs(patch), np.abs(W[:, :, ky, kx]))
    return (R if c['b'] is None else R + c['b'][None, :, None, None]), S


def _direct_check(n, c, X, Y):
    R, S = _direct_ref(c, X)
    nprod = c['k'] ** 2 * (1 if c['dw'] else c['cin'])
    err = np.abs(Y - R)
    bad = np.argwhere(err > 2 * nprod * U * S + U * np.abs(R))
    assert len(bad) == 0, '%s: %d elements outside the bound, first (frame, channel, y, x) %s: %r vs %r' % (n, len(bad), tuple(bad[0]), Y[tuple(bad[0])], R[tuple(bad[0])])


def test_depthwise_and_direct_convolutions_against_float64(dense, tmp_path):
    convs, data, plan = dense
    kinds = {l.split()[1]: l.split()[0] for l in plan.splitlines()[1:]}
    direct = [n for n in convs if kinds.get(n) in ('dwconv', 'conv')]
    assert sum(kinds[n] == 'conv' for n in direct) == 1 + sum(p[0] == 'conv' for p in DM.KERNEL_PROBES)    # stem (16 channels: conv_first_kernel)
    assert sum(kinds[n] == 'dwconv' for n in direct) == len(DM.CHAIN) - 1 + sum(p[0] == 'dw' for p in DM.KERNEL_PROBES)
    for n in direct:
        _direct_check(n, convs[n], *data[n])
    # a 12-channel stem takes conv_small_kernel
    pp, bp, convs = DM.write_probe_model(str(tmp_path), [('conv', 7, 9, 3, 2, 19), ('dw', 12, 5, 1, 5)], 6, c0=12)
    stem = [n for n, c in convs.items() if c['role'] == 'stem']
    data, plan = _probe_run(pp, bp, convs, [_frames((81, 82, 83))], max_frames=4)
    for n in convs:
        if convs[n]['role'] != 'head' and (convs[n]['dw'] or convs[n]['k'] > 1 or convs[n]['cin'] % 4):
            _direct_check(n, convs[n], *data[n])
    assert len(stem) == 1 and (' %s ' % stem[0]) in plan and convs[stem[0]]['cout'] == 12


def test_odd_heads_and_every_fused_tail(tmp_path):
    """63-channel confidence pieces (the second at the odd offset 22743) and 7-channel GEMMs with each tail kind: fused == per-layer bit for bit, and
    the detections equal the restatement's (the odd pitches and offsets take the epilogue's scalar stores)."""
    pp, bp = DM.write_tail_model(str(tmp_path), 0)
    layers = NM.parse_param(pp); NM.load_weights(layers, bp)
    frames = _frames((61, 62, 63))
    fused = B.Detector(pp, bp, max_frames=4)
    diag = B.Detector(pp, bp, max_frames=4, flags=B.DET_DIAGNOSTIC)
    a, b = _run(fused, frames), _run(diag, frames)
    for k in a:
        assert a[k].tobytes() == b[k].tobytes(), 'fused and per-layer execution differ in ' + k
    assert a['nrows'].min() > 0
    for f in range(3):
        rows_ref, post = DO.detect(layers, frames[f], 0.9, 0.01)
        _check_rows(a, f, rows_ref, post)
    fused.close(); diag.close()
