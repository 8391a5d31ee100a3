"""Exact-sum restatement of the GPU LK tracker (lk_track_kernel in sg-slam_b200/csrc/lk_kernel.cu) and of the padded pyramid it
reads, in numpy.  No GPU, no cv2.

The kernel's arithmetic is fully specified: every window sum is a sum of integer products accumulated exactly (warp_sum_exact),
and every float step after that is an explicit __f*_rn / __d*_rn intrinsic (the library is built with -fmad=false).  So this
file sums in int64 (order-free: none of the kernel's lane tiling or dp2a packing matters) and then takes the same float32 /
float64 steps in the same order; the kernel must match it bit for bit.  Every float intermediate is a float32 or float64 array or
scalar exactly where the kernel has one (a float64 numpy scalar would silently promote a float32 expression).

track() also returns which branches each point took at each level, and the largest per-lane partial sum in the kernel's tiling,
so the tests can show that their data reaches every path.

The second half builds the test cases shared by tests/test_lk_exact.py (CPU) and tests/test_gpu_lk_exact.py (GPU)."""
import hashlib

import numpy as np

WIN, MAX_LEVEL, MAX_COUNT, PAD = 21, 3, 30, 24      # PAD = kLkPad: border of every padded plane
W_BITS = 14
f32, f64 = np.float32, np.float64
HALF_WIN = f32(10.0)                  # (winSize - 1) * 0.5
FLT_SCALE = f32(1.0 / (1 << 20))
MIN_EIG = f32(1e-4)
FLT_EPSILON = f32(2.0 ** -23)
EPS2 = 0.01 * 0.01                    # the convergence threshold, squared in double

# per point and level: how often each branch of lk_track_kernel was taken
COUNTERS = (
    'setup_outside',    # the window origin failed the ipx/ipy gate
    'setup_gated',      # min_eig < 1e-4 or D < FLT_EPSILON
    'left_image',       # an iteration's window origin left the image (break, estimate untouched)
    'converged',        # |delta|^2 <= 0.01^2
    'half_step',        # oscillation: the estimate moves back by half a step
    'max_iter',         # all 30 iterations ran
    'w11_setup',        # w11 == 16384 - w00 - w01 - w10 == -1 in the set-up weights
    'w11_iter',         # ... in an iteration's weights (count)
    'tile_reload',      # the integer window origin changed between iterations (the kernel reloads its J tile; count)
)


def level_sizes(w, h):
    """(w, h) of every level buildOpticalFlowPyramid keeps for a 21x21 window and maxLevel 3: it stops when the next level
    would not be larger than the window, (w + 1) / 2 <= 21 or (h + 1) / 2 <= 21."""
    sizes = [(w, h)]
    while len(sizes) <= MAX_LEVEL:
        nw, nh = (sizes[-1][0] + 1) // 2, (sizes[-1][1] + 1) // 2
        if nw <= WIN or nh <= WIN:
            break
        sizes.append((nw, nh))
    return sizes


def reflect101(i, n):
    """BORDER_REFLECT_101 index, periodic for any offset (lk_refl)."""
    i = np.asarray(i, np.int64)
    if n == 1:
        return np.zeros_like(i)
    p = 2 * (n - 1)
    i = np.abs(i) % p
    return np.where(i >= n, p - i, i)


def pyr_down(img):
    """cv::pyrDown for CV_8U: separable [1 4 6 4 1], exact integer sums, (v + 128) >> 8, REFLECT_101, size ((w + 1) / 2, (h + 1) / 2)."""
    s = np.asarray(img).astype(np.int64)
    h, w = s.shape
    taps = ((-2, 1), (-1, 4), (0, 6), (1, 4), (2, 1))
    xs, ys = 2 * np.arange((w + 1) // 2), 2 * np.arange((h + 1) // 2)
    r = sum(k * s[:, reflect101(xs + o, w)] for o, k in taps)
    v = sum(k * r[reflect101(ys + o, h)] for o, k in taps)
    return ((v + 128) >> 8).astype(np.uint8)


def pyramid(img):
    img = np.ascontiguousarray(img, np.uint8)
    levels = [img]
    for _ in level_sizes(img.shape[1], img.shape[0])[1:]:
        levels.append(pyr_down(levels[-1]))
    return levels


def scharr(img):
    """calcScharrDeriv: dx, dy as int16 with REFLECT_101 at the image edge (cv2.Scharr(img, CV_16S, ..., BORDER_REFLECT_101))."""
    s = np.asarray(img).astype(np.int32)
    h, w = s.shape
    ym, yp = reflect101(np.arange(h) - 1, h), reflect101(np.arange(h) + 1, h)
    xm, xp = reflect101(np.arange(w) - 1, w), reflect101(np.arange(w) + 1, w)
    t0 = 3 * (s[ym] + s[yp]) + 10 * s
    t1 = s[yp] - s[ym]
    dx = t0[:, xp] - t0[:, xm]
    dy = 3 * (t1[:, xm] + t1[:, xp]) + 10 * t1
    return dx.astype(np.int16), dy.astype(np.int16)


def padded(img):
    """A level with its PAD-pixel REFLECT_101 border, [h + 2 PAD, w + 2 PAD] uint8."""
    h, w = img.shape
    return img[reflect101(np.arange(-PAD, h + PAD), h)[:, None], reflect101(np.arange(-PAD, w + PAD), w)[None, :]]


def padded_deriv(img):
    """The derivative plane of a level as the kernel stores it: dx | dy << 16 (uint32), zero in the PAD-pixel border."""
    h, w = img.shape
    dx, dy = scharr(img)
    d = np.zeros((h + 2 * PAD, w + 2 * PAD), np.uint32)
    d[PAD:PAD + h, PAD:PAD + w] = dx.view(np.uint16).astype(np.uint32) | (dy.view(np.uint16).astype(np.uint32) << 16)
    return d


def _weights(a, b):
    """lk_weights: 14-bit bilinear weights from float32 products, rounded half to even; w11 takes the remainder (can be -1)."""
    one, s = f32(1), f32(1 << W_BITS)
    w00 = np.rint((one - a) * (one - b) * s).astype(np.int64)
    w01 = np.rint(a * (one - b) * s).astype(np.int64)
    w10 = np.rint((one - a) * b * s).astype(np.int64)
    return w00, w01, w10, (1 << W_BITS) - w00 - w01 - w10


def _window(plane, ox, oy):
    """The 22x22 pixels under the window whose origin (image coordinates) is (ox, oy), from a padded plane: [m, 22, 22] int64."""
    r = (oy + PAD)[:, None] + np.arange(WIN + 1)
    c = (ox + PAD)[:, None] + np.arange(WIN + 1)
    return plane[r[:, :, None], c[:, None, :]].astype(np.int64)


def _interp(P, w, shift):
    """descale(p00 w00 + p01 w01 + p10 w10 + p11 w11, shift) over the 21x21 window (arithmetic shift, as the kernel's >>)."""
    w00, w01, w10, w11 = (x[:, None, None] for x in w)
    s = P[:, :-1, :-1] * w00 + P[:, :-1, 1:] * w01 + P[:, 1:, :-1] * w10 + P[:, 1:, 1:] * w11
    return (s + (1 << (shift - 1))) >> shift


def _to_f32(s):
    """(float)(long long): the sums stay below 2^53, so the float64 step is exact and the float32 step is the one rounding."""
    return s.astype(f64).astype(f32)


def lane_partials(P):
    """Per-lane partial sums of the [m, 21, 21] products P in lk_track_kernel's tiling: lane 10 g + k (g < 3, k < 10) owns window
    columns 2k, 2k + 1 of rows 7g .. 7g + 6, and lanes 0..20 each own row `lane` of column 20.  Returns [m, 30]; lanes 30 and 31
    contribute nothing."""
    m = P.shape[0]
    lanes = P[:, :, :20].reshape(m, 3, 7, 10, 2).sum(axis=(2, 4)).reshape(m, 30)
    lanes[:, :WIN] += P[:, :, 20]
    return lanes


def _max_lane(*prods):
    return max([int(np.abs(lane_partials(p)).max()) for p in prods if p.shape[0]] + [0])


def track(cur, prev, pts):
    """lk_track_kernel for one image pair: I = cur (the points' image), J = prev.  Returns (out [n, 2] float32, info) where info
    holds the COUNTERS ([n, levels] int32 each), 'ipx' / 'ipy' ([n, levels] window origins at set-up) and 'max_lane' (the largest
    |per-lane partial sum| of the kernel's tiling over every window sum taken)."""
    cur = np.ascontiguousarray(cur, np.uint8); prev = np.ascontiguousarray(prev, np.uint8)
    assert cur.shape == prev.shape
    pts = np.ascontiguousarray(pts, f32).reshape(-1, 2)
    sizes = level_sizes(cur.shape[1], cur.shape[0])
    nl, n = len(sizes), len(pts)
    LI, LJ = pyramid(cur), pyramid(prev)
    info = {k: np.zeros((n, nl), np.int32) for k in COUNTERS}
    info['ipx'] = np.zeros((n, nl), np.int64); info['ipy'] = np.zeros((n, nl), np.int64)
    max_lane = 0
    nx, ny = np.zeros(n, f32), np.zeros(n, f32)
    for level in range(nl - 1, -1, -1):
        lw, lh = sizes[level]
        I = padded(LI[level])
        dxp, dyp = (np.pad(d, PAD) for d in scharr(LI[level]))
        J = padded(LJ[level])
        sc = f32(1.0 / (1 << level))
        px, py = pts[:, 0] * sc, pts[:, 1] * sc
        if level == nl - 1:
            qx, qy = px.copy(), py.copy()
        else:
            qx, qy = nx * f32(2), ny * f32(2)
        nx, ny = qx.copy(), qy.copy()
        px, py = px - HALF_WIN, py - HALF_WIN
        ipx, ipy = np.floor(px).astype(np.int64), np.floor(py).astype(np.int64)
        info['ipx'][:, level], info['ipy'][:, level] = ipx, ipy
        inside = (ipx >= -WIN) & (ipx < lw) & (ipy >= -WIN) & (ipy < lh)
        info['setup_outside'][~inside, level] = 1
        idx = np.nonzero(inside)[0]
        w = _weights(px[idx] - ipx[idx].astype(f32), py[idx] - ipy[idx].astype(f32))
        info['w11_setup'][idx[w[3] == -1], level] = 1
        Iw = _interp(_window(I, ipx[idx], ipy[idx]), w, W_BITS - 5)
        Ix = _interp(_window(dxp, ipx[idx], ipy[idx]), w, W_BITS)
        Iy = _interp(_window(dyp, ipx[idx], ipy[idx]), w, W_BITS)
        max_lane = max(max_lane, _max_lane(Ix * Ix, Ix * Iy, Iy * Iy))
        A11 = _to_f32((Ix * Ix).sum((1, 2))) * FLT_SCALE
        A12 = _to_f32((Ix * Iy).sum((1, 2))) * FLT_SCALE
        A22 = _to_f32((Iy * Iy).sum((1, 2))) * FLT_SCALE
        D = A11 * A22 - A12 * A12
        dd = A11 - A22
        min_eig = (A22 + A11 - np.sqrt(dd * dd + f32(4) * A12 * A12)) / f32(2 * WIN * WIN)
        gated = (min_eig < MIN_EIG) | (D < FLT_EPSILON)
        info['setup_gated'][idx[gated], level] = 1
        keep = ~gated
        idx, Iw, Ix, Iy, A11, A12, A22 = idx[keep], Iw[keep], Ix[keep], Iy[keep], A11[keep], A12[keep], A22[keep]
        Dinv = f32(1) / D[keep]
        sx, sy = qx[idx] - HALF_WIN, qy[idx] - HALF_WIN
        pdx, pdy = np.zeros(len(idx), f32), np.zeros(len(idx), f32)
        last_x, last_y = np.zeros(len(idx), np.int64), np.zeros(len(idx), np.int64)
        act = np.arange(len(idx))          # positions into idx of the points still iterating
        for j in range(MAX_COUNT):
            inx, iny = np.floor(sx[act]).astype(np.int64), np.floor(sy[act]).astype(np.int64)
            out = (inx < -WIN) | (inx >= lw) | (iny < -WIN) | (iny >= lh)
            info['left_image'][idx[act[out]], level] = 1
            act, inx, iny = act[~out], inx[~out], iny[~out]
            if not len(act):
                break
            g = idx[act]
            w = _weights(sx[act] - inx.astype(f32), sy[act] - iny.astype(f32))
            info['w11_iter'][g[w[3] == -1], level] += 1
            if j > 0:
                info['tile_reload'][g[(inx != last_x[act]) | (iny != last_y[act])], level] += 1
            last_x[act], last_y[act] = inx, iny
            diff = _interp(_window(J, inx, iny), w, W_BITS - 5) - Iw[act]
            p1, p2 = diff * Ix[act], diff * Iy[act]
            max_lane = max(max_lane, _max_lane(p1, p2))
            B1 = _to_f32(p1.sum((1, 2))) * FLT_SCALE
            B2 = _to_f32(p2.sum((1, 2))) * FLT_SCALE
            a11, a12, a22, d = A11[act], A12[act], A22[act], Dinv[act]
            dx = (a12 * B2 - a22 * B1) * d
            dy = (a12 * B1 - a11 * B2) * d
            sx[act] = sx[act] + dx; sy[act] = sy[act] + dy
            nx[g], ny[g] = sx[act] + HALF_WIN, sy[act] + HALF_WIN
            dx64, dy64 = dx.astype(f64), dy.astype(f64)
            conv = dx64 * dx64 + dy64 * dy64 <= EPS2
            osc = ~conv & (j > 0) & (np.abs(dx + pdx[act]).astype(f64) < 0.01) & (np.abs(dy + pdy[act]).astype(f64) < 0.01)
            nx[g[osc]] = nx[g[osc]] - dx[osc] * f32(0.5)
            ny[g[osc]] = ny[g[osc]] - dy[osc] * f32(0.5)
            info['converged'][g[conv], level] = 1
            info['half_step'][g[osc], level] = 1
            pdx[act], pdy[act] = dx, dy
            act = act[~(conv | osc)]
        else:
            info['max_iter'][idx[act], level] = 1
    info['max_lane'] = max_lane
    return np.stack([nx, ny], 1), info


# ------------------------------------------------------------------------------------------------------------------------------
# Test cases shared by the CPU and GPU tests
# ------------------------------------------------------------------------------------------------------------------------------

# (w, h, seed): EuRoC (level 3 width 94, not a multiple of 4), KITTI (odd widths at levels 0-2), odd 641x481, and small images
# with max_level 1 (90x60, 43x43) and 0 (42x42)
GOLDEN_SIZES = ((752, 480, 41), (1241, 376, 42), (641, 481, 43), (90, 60, 44), (43, 43, 45), (42, 42, 46))
EXTRA_SIZES = ((640, 480, 47), (24, 24, 48))


def digest(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def image_pair(w, h, seed):
    """(cur, prev): two consecutive frames of a seeded synthetic stream (pan of about 1 px per frame)."""
    from pysgs import synth
    frames, _ = synth.stream_s2(2, w, h, seed=seed, tex_w=w + 160, tex_h=h + 120, person=False)
    return frames[1], frames[0]


def point_set(w, h, seed, n_random=200):
    """Points that reach the tracker's edges:
    - on every image border and corner;
    - window origins at ipx / ipy == -21 and == lw - 1 (the last ones the gate admits) and one step past them, at level 0 and at
      the top level;
    - a dense sub-pixel grid (small fractional parts make w11 == -1);
    - uniform points over the image and a little beyond it."""
    rng = np.random.RandomState(seed)
    sizes = level_sizes(w, h)
    cx, cy = w / 2.0, h / 2.0
    p = []
    for x in (0.0, 0.5, 1.0, w - 1.0, w - 0.5, w - 1e-3):
        for y in (0.0, 0.25, cy, h - 1.0, h - 0.5):
            p += [(x, y), (y * w / h, x * h / w)]
    for L in sorted({0, len(sizes) - 1}):
        lw, lh = sizes[L]
        s = float(1 << L)
        xs = (-10.75 * s, (lw + 9.25) * s, -11.25 * s, (lw + 10.25) * s)
        ys = (-10.75 * s, (lh + 9.25) * s, -11.25 * s, (lh + 10.25) * s)
        p += [(x, cy) for x in xs] + [(cx, y) for y in ys] + [(x, y) for x in xs[:2] for y in ys[:2]]
    g = np.arange(12) / 12.0
    fr = np.array([0.0, 1e-4, 3e-4, 1e-3, 0.03, 0.5 - 1e-4, 0.5, 0.97, 0.9997])
    bx, by = rng.uniform(12, w - 12), rng.uniform(12, h - 12)
    p += [(bx + a + 3 * i, by + b + 3 * k) for i, a in enumerate(fr) for k, b in enumerate(fr)]
    p += [(bx + 0.3 + a, by + 2.1 + b) for a in g for b in g]
    r = np.stack([rng.uniform(-15, w + 15, n_random), rng.uniform(-15, h + 15, n_random)], 1)
    r[: n_random // 2] = np.floor(r[: n_random // 2]) + rng.uniform(0, 2e-3, (n_random // 2, 2))
    return np.concatenate([np.array(p, np.float64), r]).astype(np.float32)


def _shifted_pair(w, h, seed, sx, sy):
    """A texture and the same texture moved by (sx, sy) px: true flow (-sx, -sy) from cur into prev, larger than one level's reach."""
    from pysgs import synth
    tex = synth.texture(w + 2 * abs(sx) + 8, h + 2 * abs(sy) + 8, seed)
    x0, y0 = abs(sx) + 4, abs(sy) + 4
    return tex[y0:y0 + h, x0:x0 + w].copy(), tex[y0 - sy:y0 - sy + h, x0 - sx:x0 - sx + w].copy()


def special_cases():
    """Pairs beyond the smooth stream: large flow, flat patches, and 0/255 noise (Scharr reaches +-4080, the largest window sums)."""
    rng = np.random.RandomState(7)
    w, h = 641, 481
    out = []
    cur, prev = _shifted_pair(w, h, 51, 19, -13)
    out.append(('shift_641x481', cur, prev, point_set(w, h, 52)))
    cur, prev = image_pair(w, h, 53)
    cur[100:260, 50:300] = 90; prev[100:260, 50:300] = 90
    cur[300:, 400:] = 200
    flat = np.stack([rng.uniform(60, 290, 60), rng.uniform(110, 250, 60)], 1)
    out.append(('flat_641x481', cur, prev, np.concatenate([flat.astype(np.float32), point_set(w, h, 54, 40)])))
    w, h = 200, 120
    noise = (rng.randint(0, 2, (h + 8, w + 8)) * 255).astype(np.uint8)
    cur, prev = noise[4:4 + h, 4:4 + w].copy(), noise[5:5 + h, 3:3 + w].copy()
    flip = rng.randint(0, 20, (h, w)) == 0
    prev[flip] = 255 - prev[flip]
    out.append(('noise_200x120', cur, prev, point_set(w, h, 55)))
    yy, xx = np.mgrid[0:h, 0:w]
    checker = ((((xx + 3 * yy // 4) // 2) % 2) * 255).astype(np.uint8)
    out.append(('checker_200x120', checker, np.roll(checker, (1, 1), (0, 1)).copy(), point_set(w, h, 56, 40)))
    return out


def cases():
    """Every (name, cur, prev, pts) the exactness tests run: the golden sizes, 640x480, 24x24 and the special pairs."""
    out = []
    for w, h, seed in GOLDEN_SIZES + EXTRA_SIZES:
        cur, prev = image_pair(w, h, seed)
        out.append(('%dx%d' % (w, h), cur, prev, point_set(w, h, seed + 100)))
    return out + special_cases()
