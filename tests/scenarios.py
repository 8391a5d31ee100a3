"""Seeded matcher / dyn-reject scenarios shared by the GPU parity tests and the bench (numpy only)."""
import numpy as np

from pysgs import synth

KP_DTYPE = np.dtype([('x', '<f4'), ('y', '<f4'), ('size', '<f4'), ('angle', '<f4'), ('response', '<f4'),
                     ('octave', '<i4'), ('class_id', '<i4')])


def scale_factors(nlevels=8, sf=1.2):
    s = [np.float32(1.0)]
    for _ in range(1, nlevels):
        s.append(np.float32(np.float64(s[-1]) * np.float64(np.float32(sf))))
    return np.array(s, np.float32)


def pose(rx=0.0, ry=0.0, rz=0.0, t=(0, 0, 0)):
    cx, sx, cy, sy, cz, sz = np.cos(rx), np.sin(rx), np.cos(ry), np.sin(ry), np.cos(rz), np.sin(rz)
    Rx = np.array([[1, 0, 0], [0, cx, -sx], [0, sx, cx]]); Ry = np.array([[cy, 0, sy], [0, 1, 0], [-sy, 0, cy]])
    Rz = np.array([[cz, -sz, 0], [sz, cz, 0], [0, 0, 1]])
    T = np.eye(4)
    T[:3, :3] = Rz @ Ry @ Rx
    T[:3, 3] = t
    return T.astype(np.float32)


def random_lastframe_scenario(seed, n_cur=1000, n_last=1000, w=640, h=480, conflict=0.3, flips=60, mono=False):
    """Current frame = random keypoints/descriptors; last-frame map points are built to project near chosen current
    keypoints (several points may choose the same keypoint -> claim conflicts), with noisy descriptors."""
    rng = np.random.RandomState(seed)
    cam = dict(synth.TUM3)
    sf = scale_factors()
    kps = np.zeros(n_cur, KP_DTYPE)
    kps['x'] = rng.uniform(0, w, n_cur).astype(np.float32)
    kps['y'] = rng.uniform(0, h, n_cur).astype(np.float32)
    kps['octave'] = rng.randint(0, 8, n_cur)
    kps['angle'] = rng.uniform(0, 360, n_cur).astype(np.float32)
    kps['size'] = 31; kps['response'] = 20; kps['class_id'] = -1
    desc = rng.randint(0, 256, (n_cur, 32)).astype(np.uint8)
    depth = rng.uniform(0.5, 6.0, n_cur).astype(np.float32)
    has_depth = rng.rand(n_cur) < 0.8
    uright = np.where(has_depth, kps['x'] - np.float32(cam['bf']) / depth, np.float32(-1)).astype(np.float32)
    Tcw_cur = pose(0.01, -0.02, 0.015, (0.03, -0.01, 0.05 if seed % 3 else -0.2))
    Tcw_last = pose(0.0, 0.0, 0.0, (0.0, 0.0, 0.12 if seed % 2 else 0.0))
    # pick targets: with probability `conflict` reuse a previously used keypoint
    target = np.zeros(n_last, np.int64)
    for i in range(n_last):
        target[i] = target[rng.randint(0, i)] if (i > 0 and rng.rand() < conflict) else rng.randint(0, n_cur)
    jit = rng.normal(0, 3.0, (n_last, 2))
    u = kps['x'][target] + jit[:, 0]; v = kps['y'][target] + jit[:, 1]
    z = np.where(has_depth[target], depth[target], rng.uniform(0.5, 6.0, n_last)) * rng.uniform(0.98, 1.02, n_last)
    # camera-frame point then world = Rcw^T (Xc - tcw)
    Xc = np.stack([(u - cam['cx']) * z / cam['fx'], (v - cam['cy']) * z / cam['fy'], z], 1)
    R = Tcw_cur[:3, :3].astype(np.float64); t = Tcw_cur[:3, 3].astype(np.float64)
    Xw = (Xc - t) @ R  # R^T (Xc - t)
    bits = np.unpackbits(desc[target], axis=1)
    for i in range(n_last):
        nf = rng.randint(0, flips + 1)
        bits[i, rng.choice(256, nf, replace=False)] ^= 1
    last_desc = np.packbits(bits, axis=1)
    last_oct = np.clip(kps['octave'][target] + rng.randint(-1, 2, n_last), 0, 7).astype(np.int32)
    last_angle = ((kps['angle'][target] + rng.normal(0, 8, n_last) + (rng.rand(n_last) < 0.15) * rng.uniform(0, 360, n_last)) % 360).astype(np.float32)
    last_has = (rng.rand(n_last) < 0.9).astype(np.uint8)
    last_obs = (rng.rand(n_last) < 0.6).astype(np.uint8)
    # a few points behind the camera / outside the image
    bad = rng.rand(n_last) < 0.03
    Xw[bad] *= -1
    return dict(w=w, h=h, cam=cam, sf=sf, kps=kps, desc=desc, uright=uright, Tcw_cur=Tcw_cur, Tcw_last=Tcw_last,
                last_has=last_has, last_xyz=Xw.astype(np.float32), last_desc=last_desc, last_obs=last_obs, last_oct=last_oct,
                last_angle=last_angle, mono=mono)


def random_localmap_scenario(seed, n_cur=1000, n_mp=3000, w=640, h=480, conflict=0.3, flips=70):
    rng = np.random.RandomState(seed + 500)
    s = random_lastframe_scenario(seed, n_cur, 10, w, h)
    kps, desc = s['kps'], s['desc']
    target = np.zeros(n_mp, np.int64)
    for i in range(n_mp):
        target[i] = target[rng.randint(0, i)] if (i > 0 and rng.rand() < conflict) else rng.randint(0, n_cur)
    projx = (kps['x'][target] + rng.normal(0, 2.0, n_mp)).astype(np.float32)
    projy = (kps['y'][target] + rng.normal(0, 2.0, n_mp)).astype(np.float32)
    projxr = (np.where(s['uright'][target] > 0, s['uright'][target], projx - 10) + rng.normal(0, 2.0, n_mp)).astype(np.float32)
    level = np.clip(kps['octave'][target] + rng.randint(0, 2, n_mp), 0, 7).astype(np.int32)
    viewcos = rng.uniform(0.99, 1.0, n_mp).astype(np.float32)
    bits = np.unpackbits(desc[target], axis=1)
    for i in range(n_mp):
        nf = rng.randint(0, flips + 1)
        bits[i, rng.choice(256, nf, replace=False)] ^= 1
    mp_desc = np.packbits(bits, axis=1)
    inview = (rng.rand(n_mp) < 0.85).astype(np.uint8)
    mp_obs = (rng.rand(n_mp) < 0.9).astype(np.uint8)
    f_mp = np.full(n_cur, -1, np.int32)
    pre = rng.rand(n_cur) < 0.2   # matches left by the motion-model step
    f_mp[pre] = 100000 + np.arange(pre.sum())
    f_obs = (pre & (rng.rand(n_cur) < 0.7)).astype(np.uint8)
    s.update(dict(inview=inview, projx=projx, projy=projy, projxr=projxr, level=level, viewcos=viewcos, mp_desc=mp_desc, mp_obs=mp_obs,
                  f_mp=f_mp, f_obs=f_obs))
    return s


def dynreject_scenario(seed, n=1000, w=640, h=480, nboxes=2):
    rng = np.random.RandomState(seed + 900)
    cur = np.stack([rng.uniform(19, w - 19, n), rng.uniform(19, h - 19, n)], 1).astype(np.float32)
    # a plausible fundamental matrix: pure translation + small rotation, from K
    cam = synth.TUM3
    K = np.array([[cam['fx'], 0, cam['cx']], [0, cam['fy'], cam['cy']], [0, 0, 1.0]])
    tx = np.array([0.05, -0.01, 0.02]) + rng.normal(0, 0.01, 3)
    Tx = np.array([[0, -tx[2], tx[1]], [tx[2], 0, -tx[0]], [-tx[1], tx[0], 0]])
    R = pose(0.004, -0.006, 0.003)[:3, :3].astype(np.float64)
    E = Tx @ R
    Kinv = np.linalg.inv(K)
    F = Kinv.T @ E @ Kinv
    F /= np.abs(F).max()
    # previous points: on the epipolar line of the current point (inlier) +- noise, some gross outliers
    prev = np.zeros_like(cur)
    for i in range(n):
        l = F @ np.array([cur[i, 0], cur[i, 1], 1.0])
        # closest point on the line to cur[i] shifted a little along the line
        a, b, c = l
        d = (a * cur[i, 0] + b * cur[i, 1] + c) / (a * a + b * b)
        p = np.array([cur[i, 0] - a * d, cur[i, 1] - b * d]) + rng.uniform(-3, 3) * np.array([-b, a]) / np.hypot(a, b)
        noise = rng.normal(0, 0.4) if rng.rand() < 0.8 else rng.normal(0, 5.0)
        prev[i] = p + noise * np.array([a, b]) / np.hypot(a, b)
    boxes = np.zeros((nboxes, 4), np.float32)
    for b in range(nboxes):
        boxes[b] = (rng.uniform(0, w - 200), rng.uniform(0, h - 300), rng.uniform(80, 200), rng.uniform(150, 300))
    return dict(cur=cur, prev=prev.astype(np.float32), F=F, boxes=boxes)


def keyframe_scenario(seed, n_cur=1000, n_kf=1000, **kw):
    """Relocalisation search (src/ORBmatcher.cc:1474): the last-frame scenario re-read as a key frame -- map points with a scale-invariance
    range around their distance (so that the predicted level spreads over the pyramid, some points fall outside the range), a few current
    keypoints already holding a map point."""
    s = random_lastframe_scenario(seed, n_cur=n_cur, n_last=n_kf, **kw)
    rng = np.random.RandomState(seed + 1000)
    R = s['Tcw_cur'][:3, :3].astype(np.float64); t = s['Tcw_cur'][:3, 3].astype(np.float64)
    cen = -R.T @ t
    d = np.linalg.norm(s['last_xyz'].astype(np.float64) - cen, axis=1)
    lvl = rng.randint(0, 8, n_kf)
    maxd = (d * 1.2 ** (lvl - rng.uniform(0.05, 0.95, n_kf))).astype(np.float32)          # ceil(log(maxd/d)/log 1.2) == lvl, away from the boundaries
    out = rng.rand(n_kf) < 0.05
    maxd[out] = (d[out] * 0.5).astype(np.float32)                                            # beyond 1.2 maxd: skipped
    mind = (maxd / np.float32(1.2) ** 8).astype(np.float32)
    cur_mp = np.where(rng.rand(n_cur) < 0.1, 5000 + np.arange(n_cur), -1).astype(np.int32)
    s.update(kf_valid=(rng.rand(n_kf) < 0.9).astype(np.uint8), min_dist=mind, max_dist=maxd, cur_mp=cur_mp)
    return s


def random_vocabulary(seed, k=10, L=3, stop_frac=0.02):
    """A DBoW2-shaped vocabulary tree (k children per node, L levels, every leaf at level L) in DEPTH-FIRST node order like ORBvoc.txt:
    parent[], node descriptors, leaf weights (a few leaves have weight 0 = stopped words).  Children descriptors are noisy copies of the
    parent's so that the greedy descent is meaningful, with some exact ties between siblings."""
    rng = np.random.RandomState(seed)
    parent = [-1]; desc = [np.zeros(32, np.uint8)]; level = [0]

    def grow(pid, lvl):
        base = np.unpackbits(desc[pid]) if lvl > 0 else rng.randint(0, 2, 256).astype(np.uint8)
        prev = None
        for c in range(k):
            bits = base.copy()
            nfl = rng.randint(20, 70)
            bits[rng.choice(256, nfl, replace=False)] ^= 1
            d = np.packbits(bits)
            if prev is not None and rng.rand() < 0.05:
                d = prev.copy()                                  # identical siblings: the first one must win
            prev = d
            nid = len(parent)
            parent.append(pid); desc.append(d); level.append(lvl + 1)
            if lvl + 1 < L:
                grow(nid, lvl + 1)
    grow(0, 0)
    parent = np.array(parent, np.int32); desc = np.stack(desc); level = np.array(level)
    weight = np.zeros(len(parent), np.float64)
    leaves = level == L
    weight[leaves] = rng.uniform(0.5, 9.0, int(leaves.sum()))
    weight[leaves & (rng.rand(len(parent)) < stop_frac)] = 0.0
    return dict(k=k, L=L, parent=parent, desc=desc, weight=weight)


def bow_pair_scenario(seed, voc, n_kf=1000, n_f=1000, flips=40):
    """Key frame and frame descriptors that share structure: each frame feature is a noisy copy of some key-frame feature (several frame
    features may copy the same one, so claims and ratio tests matter); descriptors sit near vocabulary leaves."""
    rng = np.random.RandomState(seed)
    leaves = np.nonzero(voc['weight'] > 0)[0]
    src = voc['desc'][leaves[rng.randint(0, len(leaves), n_kf)]]
    bits = np.unpackbits(src, axis=1)
    for i in range(n_kf):
        bits[i, rng.choice(256, rng.randint(0, 30), replace=False)] ^= 1
    kf_desc = np.packbits(bits, axis=1)
    tgt = rng.randint(0, n_kf, n_f)
    fb = np.unpackbits(kf_desc[tgt], axis=1)
    for j in range(n_f):
        fb[j, rng.choice(256, rng.randint(0, flips + 1), replace=False)] ^= 1
    f_desc = np.packbits(fb, axis=1)
    kf_angle = rng.uniform(0, 360, n_kf).astype(np.float32)
    f_angle = ((kf_angle[tgt] - 25 + rng.normal(0, 6, n_f) + (rng.rand(n_f) < 0.15) * rng.uniform(0, 360, n_f)) % 360).astype(np.float32)
    kf_valid = (rng.rand(n_kf) < 0.85).astype(np.uint8)
    return dict(kf_desc=kf_desc, f_desc=f_desc, kf_angle=kf_angle, f_angle=f_angle, kf_valid=kf_valid)


def pose_scenario(seed, n=800, outlier_frac=0.15, noise=0.5, mono_frac=0.2, pose_err=(0.02, 0.05), nlevels=8):
    """Motion-only BA input: map points seen from a true pose, keypoints = projections + noise (a fraction is gross outliers), some without
    depth (monocular observations); the initial pose is the true pose perturbed by pose_err = (rotation rad, translation m).  Octaves are
    drawn from the `nlevels` levels of a 1.2 pyramid."""
    rng = np.random.RandomState(seed)
    cam = dict(synth.TUM3)
    sf = scale_factors(nlevels).astype(np.float32)
    T_true = pose(0.03, -0.02, 0.01, (0.1, -0.05, 0.2))
    Xc = np.c_[rng.uniform(-1.5, 1.5, n), rng.uniform(-1.0, 1.0, n), rng.uniform(1.0, 6.0, n)]
    R = T_true[:3, :3].astype(np.float64); t = T_true[:3, 3].astype(np.float64)
    Xw = ((Xc - t) @ R).astype(np.float32)
    octave = rng.randint(0, nlevels, n).astype(np.int32)
    u = cam['fx'] * Xc[:, 0] / Xc[:, 2] + cam['cx']; v = cam['fy'] * Xc[:, 1] / Xc[:, 2] + cam['cy']
    sig = noise * sf[octave]
    xy = np.stack([u + rng.normal(0, 1, n) * sig, v + rng.normal(0, 1, n) * sig], 1)
    ur = xy[:, 0] - cam['bf'] / Xc[:, 2] + rng.normal(0, 1, n) * sig
    out = rng.rand(n) < outlier_frac
    xy[out] += rng.uniform(-40, 40, (int(out.sum()), 2))
    ur = np.where(rng.rand(n) < mono_frac, -1.0, ur)
    has = (rng.rand(n) < 0.8).astype(np.uint8)
    T0 = (pose(pose_err[0], -pose_err[0] / 2, pose_err[0] / 3, (pose_err[1], -pose_err[1] / 2, pose_err[1])) @ T_true.astype(np.float64)).astype(np.float32)
    inv_s2 = (1.0 / (sf * sf)).astype(np.float32)
    return dict(cam=cam, T_true=T_true, T0=T0, has=has, xyz=Xw, xy=xy.astype(np.float32), octave=octave, uright=ur.astype(np.float32), inv_s2=inv_s2, gross=out)
