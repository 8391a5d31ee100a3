"""CPU checks of the detector's test infrastructure and host logic: the oracle's fixed-point resize against cv2 (the one pinned piece), the ncnn
param/bin reader, the oracle's PriorBox / DetectionOutput invariants, and the product's graph builder in plan-only mode (no device needed):
every hard-swish / SE tail / residual add of the synthetic graph must end up fused into its producer, and the kernel list must be shorter than the
layer list.  PARITY UNPINNED for the network itself: ncnn is not available here (see oracle/detector_oracle.py)."""
import os

import numpy as np
import pytest

import detector_model as DM
import detector_oracle as DO
import ncnn_model as NM
from pysgs import binding as B

REAL = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'oracle', '_ref', 'ncnn_model', 'mobilenetv3_ssdlite_voc')


def test_resize_matches_cv2():
    cv2 = pytest.importorskip('cv2')
    # camera-sized inputs (shrinking on both axes) are bit-identical; when an axis is enlarged cv2 4.13 differs by one grey level on ~0.1 % of
    # the pixels (its own vector path), the reference never does that (640x480 / 1280x720 frames)
    for seed, (h, w, exact) in enumerate([(480, 640, True), (720, 1280, True), (300, 300, True), (601, 450, True), (211, 517, False), (37, 1000, False)]):
        img = np.random.default_rng(seed).integers(0, 256, (h, w, 3), dtype=np.uint8)
        a = DO.resize_bilinear_u8c3(img, 300, 300).astype(int); b = cv2.resize(img, (300, 300), interpolation=cv2.INTER_LINEAR).astype(int)
        assert np.abs(a - b).max() <= (0 if exact else 1) and (a != b).mean() < 0.01


def test_reader_consumes_the_whole_blob(tmp_path):
    pp, bp = DM.write_mini_model(str(tmp_path), 0)
    layers = NM.parse_param(pp)
    used, total = NM.load_weights(layers, bp)
    assert used == total
    assert sum(L.type == 'Split' for L in layers) > 5 and layers[0].type == 'Input'


def test_oracle_detection_invariants(tmp_path):
    pp, bp = DM.write_mini_model(str(tmp_path), 0)
    layers = NM.parse_param(pp); NM.load_weights(layers, bp)
    img = DM.synthetic_rgb(480, 640, 1)
    blobs = DO.forward(layers, DO.preprocess(img))
    rows = blobs['detection_out']
    sm = [L for L in layers if L.type == 'Softmax'][0].outputs[0]
    assert np.allclose(blobs[sm].sum(1), 1, atol=1e-5)
    pri = blobs['mbox_priorbox']
    assert pri.shape == (2, 4 * (19 * 19 * 4 + 10 * 10 * 6))
    # first prior of the 19x19 map: stride ceil(300/19) = 16, centre 0.5*(16-1) = 7.5, min size 60
    assert np.allclose(pri[0, :4], [(7.5 - 30) / 300, (7.5 - 30) / 300, (7.5 + 30) / 300, (7.5 + 30) / 300])
    assert np.allclose(pri[1, :4], [0.1, 0.1, 0.2, 0.2])
    assert len(rows) == 100 and np.all(np.diff(rows[:, 1]) <= 0) and np.all(rows[:, 0] >= 1)
    # greedy NMS: no two rows of one class overlap by more than the threshold
    for c in np.unique(rows[:, 0]):
        b = rows[rows[:, 0] == c][:, 2:]
        for i in range(len(b)):
            for j in range(i):
                iw = min(b[i, 2], b[j, 2]) - max(b[i, 0], b[j, 0]); ih = min(b[i, 3], b[j, 3]) - max(b[i, 1], b[j, 1])
                inter = max(iw, 0) * max(ih, 0)
                union = (b[i, 2] - b[i, 0]) * (b[i, 3] - b[i, 1]) + (b[j, 2] - b[j, 0]) * (b[j, 3] - b[j, 1]) - inter
                assert inter / union <= 0.45 + 1e-6
    objs, dyn_map, dyn_rm = DO.postprocess(rows, 640, 480, 0.9, 0.01)
    assert len(dyn_map) == (rows[:, 0] == 15).sum() and len(dyn_map) > 0
    assert np.all(objs[:, 2] >= 0) and np.all(objs[:, 2] + objs[:, 4] <= 640)


def test_oracle_convolutions_against_a_direct_sum(tmp_path):
    """The oracle evaluates Convolution / ConvolutionDepthWise with torch.conv2d; here the same outputs are recomputed at random positions as explicit
    float64 sums over the ncnn weight layout [out][in/group][kh][kw] with ncnn's stride / symmetric zero padding, for every convolution of the graph."""
    pp, bp = DM.write_mini_model(str(tmp_path), 0)
    layers = NM.parse_param(pp); NM.load_weights(layers, bp)
    blobs = DO.forward(layers, DO.preprocess(DM.synthetic_rgb(480, 640, 3)))
    rs = np.random.RandomState(0)
    checked = 0
    for L in layers:
        if L.type not in ('Convolution', 'ConvolutionDepthWise'):
            continue
        x = blobs[L.inputs[0]].astype(np.float64); y = blobs[L.outputs[0]]
        k, s, p = L.p(1), L.p(3, 1), L.p(4, 0)
        cout, oh, ow = y.shape
        assert oh == (x.shape[1] + 2 * p - k) // s + 1 and ow == (x.shape[2] + 2 * p - k) // s + 1
        xp = np.pad(x, ((0, 0), (p, p), (p, p)))
        for _ in range(12):
            co, oy, ox = rs.randint(cout), rs.randint(oh), rs.randint(ow)
            win = xp[:, oy * s:oy * s + k, ox * s:ox * s + k]
            if L.type == 'ConvolutionDepthWise':
                v = (win[co] * L.weight[co, 0].astype(np.float64)).sum()
            else:
                v = (win * L.weight[co].astype(np.float64)).sum()
            v += float(L.bias[co]) if L.bias is not None else 0.0
            assert abs(v - float(y[co, oy, ox])) <= 1e-4 * max(1.0, abs(v)), (L.name, co, oy, ox)
            checked += 1
    assert checked >= 200


def _describe(pp, bp, flags):
    d = B.Detector(pp, bp, max_frames=4, flags=flags | B.DET_PLAN_ONLY)
    txt = d.describe(); info = (d.num_layers, d.num_kernels)
    d.close()
    return txt, info


def test_plan_fuses_elementwise_tails(tmp_path):
    pp, bp = DM.write_mini_model(str(tmp_path), 0)
    txt, (nl, nk) = _describe(pp, bp, 0)
    lines = txt.splitlines()[1:]
    assert nl == 96 and nk == len(lines) + 3 and nk < nl // 2
    assert not any(l.startswith('eltwise') for l in lines)                       # every element-wise layer found a producer
    assert sum('| add 3 | clip 0 6 | mul(rev) start | div 6' in l for l in lines) == 3         # hard-swish x3
    se = [l for l in lines if '| add 3 | clip 0 6 | div 6 | mul(rev)' in l]
    assert len(se) == 1 and se[0].startswith('conv ') and se[0].count('| add') == 2            # SE tail + residual, Cin = 6 -> direct kernel
    # no kernel writes a buffer it also reads (input or tensor operand)
    for l in lines:
        t = l.split()
        out_buf = t[t.index('out') + 2 + 0] if False else t[t.index('out') + 3]
        in_bufs = [t[i + 1] for i, x in enumerate(t) if x == 'buf'][0:1] + [t[i + 1] for i, x in enumerate(t) if x == 'buf'][2:]
        assert out_buf not in in_bufs, l
    # diagnostic mode: one kernel per layer that computes something, nothing fused
    txt2, (_, nk2) = _describe(pp, bp, B.DET_DIAGNOSTIC)
    assert nk2 > nk and '|' not in ''.join(l for l in txt2.splitlines()[1:] if not l.startswith(('eltwise', 'conv', 'dwconv')))
    assert sum(l.startswith('eltwise') for l in txt2.splitlines()) >= 20


def test_probe_graphs_reach_the_planned_gemm_features(tmp_path):
    """The probe graph of tests/test_gpu_detector_kernels.py, planned at the batch the GPU test runs: every GEMM plan feature its parity checks
    rely on is reached (BK 16 / 32, partial k-steps, streamed weights with a wrapping ring, several N-tiles, odd output pitches), so that a planner
    change cannot retire a case unnoticed; the odd-head graph fuses one tail of each kind into a 7-channel GEMM and writes a 63-channel
    confidence piece at the odd offset 22743."""
    pp, bp, convs = DM.write_probe_model(str(tmp_path), DM.GEMM_PROBES + DM.KERNEL_PROBES, 0)
    d = B.Detector(pp, bp, max_frames=DM.PROBE_FRAMES, flags=B.DET_PLAN_ONLY)
    txt = d.describe()
    d.close()
    plans = DM.parse_plan(txt)
    DM.check_probe_plans(plans)
    assert {p['name'] for p in plans} == {n for n, c in convs.items() if not c['dw'] and c['k'] == 1 and c['s'] == 1 and c['cin'] % 4 == 0}
    ops = [l.split()[0] for l in txt.splitlines()[1:]]
    assert ops.count('conv') == 1 + sum(p[0] == 'conv' for p in DM.KERNEL_PROBES) and txt.splitlines()[1].startswith('conv ')
    pp, bp = DM.write_tail_model(str(tmp_path / 'tails'), 0)
    d = B.Detector(pp, bp, max_frames=4, flags=B.DET_PLAN_ONLY)
    txt = d.describe()
    d.close()
    tails = [p['line'].split(' | ', 1)[1] if ' | ' in p['line'] else '' for p in DM.parse_plan(txt) if p['cout'] == 7]
    assert len(tails) == 7
    pats = ['^relu$', '^clip 0 6$', r'^add 3 \| clip 0 6 \| mul\(rev\) start \| div 6$', r'^add \S+ buf \d+$',
            r'^add 3 \| clip 0 6 \| div 6 \| mul\(rev\) \S+ buf \d+$', r'^add 3 \| clip 0 6 \| div 6 \| mul\(rev\) \S+ buf \d+ \| add \S+ buf \d+$',
            r'^mul 0.5 \| relu$']
    import re
    for pat in pats:
        assert sum(bool(re.match(pat, t)) for t in tails) == 1, (pat, tails)
    heads = {(p['cout'], p['off']) for p in DM.parse_plan(txt) if p['off'] is not None}
    assert heads == {(63, 0), (63, 22743), (12, 0), (12, 4332)}


def test_gemm_plans_stay_inside_what_the_kernel_launches(tmp_path):
    """Plans of 1x1 convolutions with 4 <= Cin <= 4096 (multiples of 4) and 1 <= Cout <= 4096 on maps of 1 to 150 pixels a side, at batches of 1,
    8 and 64 frames: the shared memory fits a CTA (226 KB), the ring has 2..8 stages, the N-tile is a multiple of the 32-channel wgmma width of at
    most 256 channels and the tiles cover Cout without an empty one -- launch_conv1x1_tc_map rejects anything else at run time."""
    rng = np.random.default_rng(5)
    cins = [4, 8, 12, 16, 20, 28, 32, 36, 60, 64, 100, 128, 132, 252, 256, 260, 512, 964, 1024, 2044, 4096]
    couts = [1, 2, 31, 32, 33, 63, 96, 127, 129, 255, 256, 257, 300, 511, 513, 600, 1000, 1025, 2049, 4095, 4096]
    pairs = list(zip(cins, rng.permutation(couts)))
    pairs += [(4096, 4096), (4096, 1), (4, 4096), (256, 512), (1024, 1000)]
    maps = [1, 2, 5, 19, 38, 150]
    probes = [('gemm', cin, int(cout), maps[i % len(maps)]) for i, (cin, cout) in enumerate(pairs)]
    pp, bp, _ = DM.write_probe_model(str(tmp_path), probes, 1, weights='zero')
    seen = 0
    for mf in (1, 8, 64):
        d = B.Detector(pp, bp, max_frames=mf, flags=B.DET_PLAN_ONLY)
        plans = DM.parse_plan(d.describe())
        d.close()
        for p in plans:
            assert p['smem'] <= 226 * 1024, p['line']
            assert 2 <= p['stages'] <= 8, p['line']
            assert p['nt'] % 32 == 0 and 32 <= p['nt'] <= 256, p['line']
            assert p['nt'] * (p['n_tiles'] - 1) < p['cout'] <= p['nt'] * p['n_tiles'], p['line']
            assert p['bk'] == (16 if p['cin'] <= 16 else 32) and p['kb'] == -(-p['cin'] // p['bk']), p['line']
            seen += 1
    assert seen >= 3 * len(pairs)


def test_folded_prior_boxes_match_the_oracle_bitwise(tmp_path):
    """The product folds PriorBox + Concat on the host at create time; in plan-only diagnostic mode the constant is readable without a device."""
    pp, bp = DM.write_mini_model(str(tmp_path), 0)
    layers = NM.parse_param(pp); NM.load_weights(layers, bp)
    ref = DO.forward(layers, DO.preprocess(DM.synthetic_rgb(480, 640, 1)), want='mbox_priorbox')['mbox_priorbox']
    d = B.Detector(pp, bp, max_frames=1, flags=B.DET_DIAGNOSTIC | B.DET_PLAN_ONLY)
    got = d.blob('mbox_priorbox')
    d.close()
    assert got.tobytes() == np.ascontiguousarray(ref, np.float32).tobytes()
    if os.path.exists(REAL + '.param'):
        layers = NM.parse_param(REAL + '.param'); NM.load_weights(layers, REAL + '.bin')
        pri = [DO.prior_boxes(L, fw, fw, 300, 300) for L, fw in zip([l for l in layers if l.type == 'PriorBox'], (19, 10, 5, 3, 2, 1))]
        ref = np.concatenate(pri, axis=1)
        d = B.Detector(REAL + '.param', REAL + '.bin', max_frames=1, flags=B.DET_DIAGNOSTIC | B.DET_PLAN_ONLY)
        got = d.blob('mbox_priorbox')
        d.close()
        assert got.size == 2 * 9072 and got.tobytes() == np.ascontiguousarray(ref, np.float32).tobytes()


def test_create_reports_bad_files(tmp_path):
    pp, bp = DM.write_mini_model(str(tmp_path), 0)
    with pytest.raises(B.SgsError) as e:
        B.Detector(str(tmp_path / 'missing.param'), bp, flags=B.DET_PLAN_ONLY)
    assert e.value.code == B.SGS_ERR_INVALID
    short = tmp_path / 'short.bin'
    short.write_bytes(open(bp, 'rb').read()[:-8])
    with pytest.raises(B.SgsError) as e:
        B.Detector(pp, str(short), flags=B.DET_PLAN_ONLY)
    assert e.value.code == B.SGS_ERR_INVALID
    big_pp, big_bp = DM.write_mini_model(str(tmp_path / 'big'), 0, many_priors=True)          # 38x38x4 + 10x10x6 priors: more than one sort pass holds
    with pytest.raises(B.SgsError) as e:
        B.Detector(big_pp, big_bp, flags=B.DET_PLAN_ONLY)
    assert e.value.code == B.SGS_ERR_UNSUPPORTED and 'priors 6376' in str(e.value)
    bad = tmp_path / 'bad.param'
    bad.write_text(open(pp).read().replace('Softmax', 'LSTM'))
    with pytest.raises(B.SgsError) as e:
        B.Detector(str(bad), bp, flags=B.DET_PLAN_ONLY)
    assert e.value.code == B.SGS_ERR_UNSUPPORTED


@pytest.mark.skipif(not os.path.exists(REAL + '.param'), reason='reference model copy (oracle/_ref/ncnn_model, made by build()) not present')
def test_plan_of_the_reference_model():
    txt, (nl, nk) = _describe(REAL + '.param', REAL + '.bin', 0)
    lines = txt.splitlines()
    assert nl == 408 and nk == 105 and not any(l.startswith(('eltwise', 'permute', 'concat')) for l in lines)
    # [h][w][c] activations: the 12 Permute layers are aliases and the 12 SSD head convolutions write straight into mbox_loc / mbox_conf
    heads = [l for l in lines if ' out mbox_loc ' in l or ' out mbox_conf ' in l]
    assert len(heads) == 12 and all(l.startswith('conv1x1 ') and ' off ' in l for l in heads)
    offs = sorted(int(l.split(' off ')[1].split()[0]) for l in heads if ' out mbox_conf ' in l)
    assert offs == [0, 30324, 42924, 46074, 47208, 47544]
    # every 1x1 convolution of the model with Cin % 4 == 0 is planned for the wgmma GEMM: 66 of the 70 convolutions
    assert sum(l.startswith('conv1x1 ') for l in lines) == 66 and sum(l.startswith('conv ') for l in lines) == 4
    layers = NM.parse_param(REAL + '.param')
    used, total = NM.load_weights(layers, REAL + '.bin')
    assert used == total == 9693828


def test_batched_cpu_baseline_detector_matches_the_oracle(tmp_path):
    """bench.py's CPU baseline runs the restatement on chunks of frames with PyTorch tensors end to end (oracle/detector_batched.py).  It must be the same
    detector as the parity checker: identical DetectionOutput rows for identical head outputs (vectorised NMS), and the same detections from pixels (scores to
    2e-5: batched / channels-last convolutions may round differently from the single-frame ones)."""
    import detector_batched as DB
    import torch
    models = [DM.write_mini_model(str(tmp_path), 0)] + ([(REAL + '.param', REAL + '.bin')] if os.path.exists(REAL + '.param') else [])
    for pp, bp in models:
        layers = NM.parse_param(pp); NM.load_weights(layers, bp)
        bd = DB.BatchedDetector(layers)
        imgs = [DM.synthetic_rgb(480, 640, s) for s in (1, 2, 3)]
        xb = torch.from_numpy(np.stack([DO.preprocess(f) for f in imgs])).contiguous(memory_format=torch.channels_last)
        L, loc, conf, prior = bd.forward(xb)
        for i in range(len(imgs)):
            a = DO.detection_output(L, loc[i].numpy(), conf[i].numpy(), prior)
            b = DB.detection_output_fast(L, loc[i].numpy(), conf[i].numpy(), prior)
            assert a.shape == b.shape and np.array_equal(a, b)
        got = bd.detect(imgs, chunk=2)
        for f, (rows, post) in zip(imgs, got):
            ref_rows, ref_post = DO.detect(layers, f)
            assert rows.shape == ref_rows.shape
            if len(rows):
                assert np.array_equal(rows[:, 0], ref_rows[:, 0]) and np.abs(rows[:, 1:] - ref_rows[:, 1:]).max() < 2e-5
            assert all(x.shape == y.shape for x, y in zip(post, ref_post))
