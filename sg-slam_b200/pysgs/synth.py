"""Seeded synthetic inputs (numpy only) for tests and bench -- SURVEY.md section 8(d), S1..S5.

The generators are deterministic functions of their seed so the CPU oracle and the GPU path
see byte-identical inputs.  No cv2 / no GPU required.
"""
import numpy as np

# intrinsics of /root/reference/src/sg-slam/Examples/TUM3.yaml:8-11,25
TUM3 = dict(fx=535.4, fy=539.2, cx=320.1, cy=247.6, bf=40.0)


def _blur3(img, sigma=0.7):
    k = np.exp(-0.5 * (np.arange(-1, 2) / sigma) ** 2)
    k /= k.sum()
    p = np.pad(img, 1, mode='reflect')
    t = k[0] * p[:, :-2] + k[1] * p[:, 1:-1] + k[2] * p[:, 2:]
    return k[0] * t[:-2] + k[1] * t[1:-1] + k[2] * t[2:]


def texture(w, h, seed, nrect=None):
    """S1-style texture: random axis-aligned rectangles (5..80 px, +-90 around 128) + N(0,4) + 3x3 blur."""
    rng = np.random.RandomState(seed)
    if nrect is None:
        nrect = max(8, int(400 * (w * h) / (640 * 480)))
    img = np.full((h, w), 128.0, np.float64)
    for _ in range(nrect):
        rw, rh = rng.randint(5, 81, 2)
        x0 = rng.randint(-rw // 2, w - rw // 2)
        y0 = rng.randint(-rh // 2, h - rh // 2)
        v = rng.uniform(-90, 90)
        img[max(y0, 0):max(y0 + rh, 0), max(x0, 0):max(x0 + rw, 0)] = 128 + v
    img += rng.normal(0, 4, img.shape)
    img = _blur3(img)
    return np.clip(np.rint(img), 0, 255).astype(np.uint8)


def frame_s1(w=640, h=480, seed=1):
    """S1: one gray frame."""
    return texture(w, h, seed)


def depth_s1(w=640, h=480, seed=1):
    """S1 depth (float32 metres): tilted plane 1..4 m + noise."""
    rng = np.random.RandomState(seed + 1000)
    yy, xx = np.mgrid[0:h, 0:w]
    d = 1.0 + 3.0 * (0.6 * xx / w + 0.4 * yy / h) + rng.normal(0, 0.01, (h, w))
    return d.astype(np.float32)


def _sample_bilinear(tex, xs, ys):
    x0 = np.floor(xs).astype(np.int64); y0 = np.floor(ys).astype(np.int64)
    fx = xs - x0; fy = ys - y0
    x0 = np.clip(x0, 0, tex.shape[1] - 2); y0 = np.clip(y0, 0, tex.shape[0] - 2)
    t = tex.astype(np.float64)
    v = (t[y0, x0] * (1 - fx) * (1 - fy) + t[y0, x0 + 1] * fx * (1 - fy) + t[y0 + 1, x0] * (1 - fx) * fy + t[y0 + 1, x0 + 1] * fx * fy)
    return v


def stream_s2(nframes=16, w=640, h=480, seed=2, tex_w=1024, tex_h=768, person=True):
    """S2: 'walking_xyz-shaped' stream: smooth pan (<=3 px/frame, <=0.5 deg/frame roll) over a big S1-style texture with one
    160x320 'person' rectangle moving >=4 px/frame against the pan.  Returns (frames u8 [n,h,w], boxes [n,4] x,y,w,h float32)."""
    rng = np.random.RandomState(seed)
    tex = texture(tex_w, tex_h, seed + 17)
    ptex = texture(160, 320, seed + 23, nrect=60)
    frames = np.zeros((nframes, h, w), np.uint8)
    boxes = np.zeros((nframes, 4), np.float32)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    cx0, cy0 = (tex_w - w) / 2.0, (tex_h - h) / 2.0
    for k in range(nframes):
        t = k / max(1, nframes - 1) if nframes > 1 else 0.0
        ph = 2 * np.pi * k / 420.0
        ox = cx0 + 0.8 * cx0 * np.sin(ph)            # <= ~2.3 px/frame
        oy = cy0 + 0.8 * cy0 * np.sin(1.7 * ph + 0.3)
        roll = np.deg2rad(4.0) * np.sin(0.9 * ph)    # <= ~0.06 deg/frame
        c, s = np.cos(roll), np.sin(roll)
        xc, yc = xx - w / 2.0, yy - h / 2.0
        xs = ox + w / 2.0 + c * xc - s * yc
        ys = oy + h / 2.0 + s * xc + c * yc
        img = _sample_bilinear(tex, xs, ys)
        if person:
            px = (40 + 5.0 * k) % (w - 160)
            py = 100 + 20 * np.sin(0.21 * k)
            x0, y0 = int(round(px)), int(round(py))
            hh = min(320, h - y0)
            img[y0:y0 + hh, x0:x0 + 160] = ptex[:hh, :]
            boxes[k] = (x0, y0, 160, hh)
        img += rng.normal(0, 1.5, img.shape)
        frames[k] = np.clip(np.rint(img), 0, 255).astype(np.uint8)
        del t
    return frames, boxes


def stream_s2_rgbd(nframes=16, w=640, h=480, seed=2, **kw):
    """Colour RGB-D variant of S2: the S2 frames of `seed` in three channels that differ -- c0 = frame + N(0,3), c1 = frame + N(0,3),
    c2 = 255 - frame + N(0,3), so that the two channel orders give different gray images -- and the S1 depth plane stored TUM-style as
    uint16 = round(d * 5000) for every frame.  Returns (colour u8 [n,h,w,3], depth u16 [n,h,w], boxes [n,4])."""
    frames, boxes = stream_s2(nframes, w, h, seed=seed, **kw)
    rng = np.random.RandomState(seed + 31)
    g = frames.astype(np.float64)
    ch = [g, g, 255.0 - g]
    rgb = np.stack([np.clip(np.rint(c + rng.normal(0, 3, g.shape)), 0, 255) for c in ch], -1).astype(np.uint8)
    depth = np.rint(depth_s1(w, h).astype(np.float64) * 5000).astype(np.uint16)
    return rgb, np.ascontiguousarray(np.broadcast_to(depth, (nframes, h, w))), boxes


def descriptors_s5(n, seed=5):
    """S5: uniform random 256-bit descriptors [n,32] u8."""
    rng = np.random.RandomState(seed)
    return rng.randint(0, 256, (n, 32)).astype(np.uint8)


def descriptors_near(train, seed=6, maxflips=40):
    """S5 near-duplicate variant: query = train with 0..maxflips random bit flips per row."""
    rng = np.random.RandomState(seed)
    q = train.copy()
    bits = np.unpackbits(q, axis=1)
    for i in range(len(q)):
        nf = rng.randint(0, maxflips + 1)
        idx = rng.choice(256, nf, replace=False)
        bits[i, idx] ^= 1
    return np.packbits(bits, axis=1)


def scale_factors(nlevels=8, sf=1.2):
    """mvScaleFactor of ORBextractor (src/ORBextractor.cc:416-421): float32 chain 1, 1.2, 1.44, ..."""
    s = [np.float32(1.0)]
    for _ in range(1, nlevels):
        s.append(np.float32(np.float64(s[-1]) * np.float64(np.float32(sf))))
    return np.array(s, np.float32)


def gray_to_rgb(frames):
    """Colour frames for the detector: the gray frame in all three channels ([n,h,w] -> [n,h,w,3] uint8)."""
    return np.ascontiguousarray(np.repeat(frames[..., None], 3, axis=-1))
