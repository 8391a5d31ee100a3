"""TEST INFRASTRUCTURE: CPU FP32 restatement of Detector2D::detect (src/Detector2D.cc:34-89) — ncnn forward of the
MobileNetV3-SSDLite graph (Thirdparty/ncnn_model/mobilenetv3_ssdlite_voc.param) interpreted layer by layer with PyTorch CPU ops, plus the
reference's post-processing of the "detection_out" rows.

PARITY UNPINNED: ncnn is an un-vendored, unpinned dependency (ThirdpartyBuild.sh:21) and is not installed here, so nothing below was run
against ncnn itself.  Layer semantics are restated from ncnn's published layer definitions; the two places where that restatement carries a
real assumption are marked ASSUMPTION.  Pinned pieces: the input resize against cv2.resize (ncnn documents from_pixels_resize as
OpenCV-compatible fixed-point bilinear); the post-processing of the rows against the reference's own Detector2D.cc compiled unmodified
(tests/test_detector2d_ref.py); PriorBox and DetectionOutput against OpenCV's dnn implementation of the same Caffe-SSD layers that ncnn ported
(tests/test_detector_cv2.py: same rows to 1e-6); the convolutions are PyTorch's.  Still carried as assumptions: ncnn's two mmdetection switches of
PriorBox and the order of equal scores.
"""
import math
import numpy as np
import torch
import torch.nn.functional as F

TARGET = 300                                   # Detector2D.h:70
MEAN = (123.675, 116.28, 103.53)               # Detector2D.h:71 (norm_vals are all 1, :72)
PERSON = 15                                    # Detector2D.cc:74


def resize_bilinear_u8c3(img, dw, dh):
    """Mat::from_pixels_resize (Detector2D.cc:39): fixed-point bilinear, 11-bit coefficients, the same arithmetic as cv::resize INTER_LINEAR
    on 8-bit data: horizontal pass keeps value*2048, vertical pass is ((b0*(r0>>4))>>16) + ((b1*(r1>>4))>>16) + 2) >> 2."""
    sh, sw, ch = img.shape
    def coeffs(dn, sn):
        scale = sn / dn
        idx = np.zeros(dn, np.int64); a = np.zeros((dn, 2), np.int64)
        for d in range(dn):
            f = np.float32((d + 0.5) * scale - 0.5)
            s = int(math.floor(f)); f = np.float32(f - s)
            if s < 0: s, f = 0, np.float32(0)
            if s >= sn - 1: s, f = sn - 2, np.float32(1)
            idx[d] = s
            def sat(v):
                v = float(v); r = int(np.rint(v))        # saturate_cast<short>(float): round half to even
                return max(-32768, min(32767, r))
            a[d, 0] = sat((np.float32(1) - f) * np.float32(2048)); a[d, 1] = sat(f * np.float32(2048))
        return idx, a
    xi, xa = coeffs(dw, sw); yi, ya = coeffs(dh, sh)
    src = img.astype(np.int64)
    rows = src[:, xi, :] * xa[None, :, 0, None] + src[:, xi + 1, :] * xa[None, :, 1, None]      # sh x dw x ch, scaled by 2048
    r0 = rows[yi] >> 4; r1 = rows[yi + 1] >> 4
    out = (((ya[:, 0, None, None] * r0) >> 16) + ((ya[:, 1, None, None] * r1) >> 16) + 2) >> 2
    return np.clip(out, 0, 255).astype(np.uint8)


def preprocess(rgb):
    """u8 HxWx3 -> float32 3x300x300, mean-subtracted (Detector2D.cc:39-40).  Channel order is kept as given (PIXEL_RGB = no swap)."""
    small = resize_bilinear_u8c3(rgb, TARGET, TARGET)
    x = small.astype(np.float32).transpose(2, 0, 1).copy()
    for c in range(3):
        x[c] = (x[c] - np.float32(MEAN[c])) * np.float32(1.0)
    return x


def prior_boxes(L, fw, fh, iw, ih):
    """ncnn PriorBox -> (2, 4*fw*fh*num_prior): row 0 corner boxes (normalised), row 1 variances."""
    mins, maxs, ars = L.p(0, []), L.p(1, []), L.p(2, [])
    var = [np.float32(L.p(3, 0.1)), np.float32(L.p(4, 0.1)), np.float32(L.p(5, 0.2)), np.float32(L.p(6, 0.2))]
    flip, clip = L.p(7, 1), L.p(8, 0)
    image_w = L.p(9, 0); image_h = L.p(10, 0)
    if image_w == -233: image_w = iw
    if image_h == -233: image_h = ih
    step_w = np.float32(L.p(11, -233.0)); step_h = np.float32(L.p(12, -233.0))
    if step_w == -233: step_w = np.float32(image_w) / np.float32(fw)
    if step_h == -233: step_h = np.float32(image_h) / np.float32(fh)
    offset = np.float32(L.p(13, 0.0))
    # ASSUMPTION (keys 14/15, both 1 in this model: the graph was exported from an mmdetection SSD): the anchor stride is the integer
    # ceil(image / feature) and the first centre sits at offset*(stride-1), mmdetection's ((stride-1)/2) convention.
    if L.p(14, 0):
        step_w = np.float32(math.ceil(image_w / fw)); step_h = np.float32(math.ceil(image_h / fh))
    centre_mm = L.p(15, 0)
    out = []
    half = np.float32(0.5)
    for i in range(fh):
        for j in range(fw):
            if centre_mm:
                cx = offset * (step_w - np.float32(1)) + np.float32(j) * step_w
                cy = offset * (step_h - np.float32(1)) + np.float32(i) * step_h
            else:
                cx = offset * step_w + np.float32(j) * step_w
                cy = offset * step_h + np.float32(i) * step_h
            def put(bw, bh):
                out.extend([(cx - bw * half) / np.float32(image_w), (cy - bh * half) / np.float32(image_h),
                            (cx + bw * half) / np.float32(image_w), (cy + bh * half) / np.float32(image_h)])
            for k, mn in enumerate(mins):
                mn = np.float32(mn)
                put(mn, mn)
                if maxs:
                    s = np.float32(math.sqrt(float(mn * np.float32(maxs[k]))))
                    put(s, s)
                for ar in ars:
                    r = np.float32(math.sqrt(float(np.float32(ar))))
                    bw, bh = mn * r, mn / r
                    put(bw, bh)
                    if flip:
                        put(bh, bw)
    box = np.array(out, np.float32)
    if clip:
        box = np.clip(box, 0, 1)
    return np.stack([box, np.tile(np.array(var, np.float32), len(box) // 4)])


def decode_boxes(loc, prior):
    """DetectionOutput's box decoding: prior boxes moved by the location offsets scaled by the prior variances -> [prior][xmin, ymin, xmax, ymax]"""
    loc = loc.reshape(-1, 4).astype(np.float32); pb = prior[0].reshape(-1, 4); var = prior[1].reshape(-1, 4)
    half = np.float32(0.5)
    pw = pb[:, 2] - pb[:, 0]; ph = pb[:, 3] - pb[:, 1]
    pcx = (pb[:, 0] + pb[:, 2]) * half; pcy = (pb[:, 1] + pb[:, 3]) * half
    cx = var[:, 0] * loc[:, 0] * pw + pcx; cy = var[:, 1] * loc[:, 1] * ph + pcy
    w = np.exp(var[:, 2] * loc[:, 2]).astype(np.float32) * pw; h = np.exp(var[:, 3] * loc[:, 3]).astype(np.float32) * ph
    return np.stack([cx - w * half, cy - h * half, cx + w * half, cy + h * half], 1).astype(np.float32)


def detection_output(L, loc, conf, prior):
    """ncnn DetectionOutput: decode with the prior variances, per-class threshold + top-k + greedy NMS, global top-k.
    Returns rows [label, score, xmin, ymin, xmax, ymax] (normalised coordinates)."""
    ncls, nms_thr, nms_topk, keep_topk, conf_thr = L.p(0), np.float32(L.p(1, 0.05)), L.p(2, 300), L.p(3, 100), np.float32(L.p(4, 0.5))
    conf = conf.reshape(-1, ncls).astype(np.float32)
    boxes = decode_boxes(loc, prior)
    rows = []
    for c in range(1, ncls):
        idx = np.nonzero(conf[:, c] > conf_thr)[0]
        # descending score; ties (not ordered by ncnn's quicksort in any documented way) broken by prior index
        idx = idx[np.lexsort((idx, -conf[idx, c]))][:nms_topk]
        picked = []
        for i in idx:
            b = boxes[i]; area = (b[2] - b[0]) * (b[3] - b[1])
            a = boxes[picked].T                                  # every kept box at once: the same float32 operations, element by element
            apart = (b[0] > a[2]) | (b[2] < a[0]) | (b[1] > a[3]) | (b[3] < a[1])
            inter = np.where(apart, np.float32(0), (np.minimum(a[2], b[2]) - np.maximum(a[0], b[0])) * (np.minimum(a[3], b[3]) - np.maximum(a[1], b[1])))
            union = (a[2] - a[0]) * (a[3] - a[1]) + area - inter
            if not (inter / union > nms_thr).any():
                picked.append(i)
        rows += [(c, conf[i, c], i) for i in picked]
    rows.sort(key=lambda r: (-r[1], r[0], r[2]))
    rows = rows[:keep_topk]
    return np.array([[c, s, *boxes[i]] for c, s, i in rows], np.float32).reshape(-1, 6)


def forward(layers, x, want=None, keep_all=False):
    """Interprets the graph on one 3xHxW float32 input.  Returns the blob dictionary (numpy arrays in ncnn's dims order c,h,w / h,w / w)."""
    blobs = {}
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    for L in layers:
        ins = [blobs[n] for n in L.inputs]
        ty = L.type
        if ty == 'Input':
            out = [x.astype(np.float32)]
        elif ty == 'MemoryData':
            out = [L.data.copy()]
        elif ty == 'Split':
            out = [ins[0]] * len(L.outputs)
        elif ty in ('Convolution', 'ConvolutionDepthWise'):
            y = F.conv2d(t(ins[0])[None], t(L.weight), t(L.bias) if L.bias is not None else None, stride=(L.p(13, L.p(3, 1)), L.p(3, 1)),
                         padding=(L.p(14, L.p(4, 0)), L.p(4, 0)), dilation=(L.p(12, L.p(2, 1)), L.p(2, 1)), groups=L.group)
            out = [y[0].numpy()]
        elif ty == 'ReLU':
            out = [np.maximum(ins[0], np.float32(0))]
        elif ty == 'Clip':
            out = [np.minimum(np.maximum(ins[0], np.float32(L.p(0))), np.float32(L.p(1)))]
        elif ty == 'BinaryOp':
            a, b = ins
            if b.ndim == 1 and b.size == 1: b = b.reshape(())            # scalar constant
            elif b.ndim == 3 and a.ndim == 3 and b.shape[1:] == (1, 1): pass  # per-channel broadcast (c,1,1)
            op = L.p(0, 0)
            out = [{0: np.add, 1: np.subtract, 2: np.multiply, 3: np.divide}[op](a, b).astype(np.float32)]
        elif ty == 'Permute':
            assert L.p(0) == 3 and ins[0].ndim == 3                        # order c w h in ncnn's (w,h,c) notation = CHW -> HWC
            out = [np.ascontiguousarray(ins[0].transpose(1, 2, 0))]
        elif ty == 'Flatten':
            out = [ins[0].reshape(-1)]
        elif ty == 'Concat':
            out = [np.concatenate(ins, axis=L.p(0, 0))]
        elif ty == 'Reshape':
            w, h = L.p(0), L.p(1, -233)
            out = [ins[0].reshape(h, w) if h != -233 else ins[0].reshape(w)]
        elif ty == 'Softmax':
            assert ins[0].ndim == 2 and L.p(0) == 1
            z = ins[0]; m = z.max(axis=1, keepdims=True); e = np.exp(z - m).astype(np.float32)
            out = [(e / e.sum(axis=1, keepdims=True, dtype=np.float32)).astype(np.float32)]
        elif ty == 'PriorBox':
            fm, im = ins
            out = [prior_boxes(L, fm.shape[2], fm.shape[1], im.shape[2], im.shape[1])]
        elif ty == 'DetectionOutput':
            out = [detection_output(L, ins[0], ins[1], ins[2])]
        else:
            raise NotImplementedError(ty)
        for n, o in zip(L.outputs, out):
            blobs[n] = o
        if want is not None and want in L.outputs:
            break
    return blobs


def postprocess(rows, img_w, img_h, det_thr, dyn_thr):
    """Detector2D.cc:52-88: threshold, scale to the image, split person boxes.  Returns (objects, dynamic_for_mapping, dynamic_for_rm)
    as float32 arrays; objects rows are [id, prob, x, y, w, h] in detection order (all accepted rows, persons included)."""
    ts = np.float32(TARGET)
    objs, dyn_map, dyn_rm = [], [], []
    for v in rows:
        lab = int(v[0])
        if v[1] > np.float32(det_thr) or (v[1] > np.float32(dyn_thr) and lab == PERSON):
            c = [np.float32(min(max(v[k] * ts, np.float32(0)), ts - np.float32(1))) / ts for k in (2, 3, 4, 5)]
            x1, y1, x2, y2 = c[0] * np.float32(img_w), c[1] * np.float32(img_h), c[2] * np.float32(img_w), c[3] * np.float32(img_h)
            r = [x1, y1, x2 - x1, y2 - y1]
            objs.append([lab, v[1], *r])
            if lab == PERSON:
                dyn_map.append(r)
                if float(v[1]) > 0.2: dyn_rm.append(r)          # `object2d.prob > 0.2`: the float against the DOUBLE literal (Detector2D.cc:78; pinned by tests/test_detector2d_ref.py)
    f = lambda a, k: np.array(a, np.float32).reshape(-1, k)
    return f(objs, 6), f(dyn_map, 4), f(dyn_rm, 4)


def detect(layers, rgb, det_thr=0.9, dyn_thr=0.01):
    blobs = forward(layers, preprocess(rgb))
    rows = blobs['detection_out']
    return rows, postprocess(rows, rgb.shape[1], rgb.shape[0], det_thr, dyn_thr)
