#!/usr/bin/env python3
"""Golden vectors for the LK stage at image sizes beyond 640x480 / 320x240: EuRoC 752x480, KITTI 1241x376, 641x481, and the small
images 90x60 / 43x43 (one pyramid level above level 0) and 42x42 (level 0 only).  Everything stored comes from the REAL cv2:
- SHA-256 digests of the cv2.pyrDown levels and of the cv2.Scharr(..., CV_16S, BORDER_REFLECT_101) dx / dy planes of every level;
- the level count of cv2.buildOpticalFlowPyramid(img, (21, 21), 3);
- cv2.calcOpticalFlowPyrLK tracks with the reference's parameters (winSize 21x21, maxLevel 3, COUNT|EPS 30 / 0.01).
The images are not stored: the tests regenerate them from their pysgs.synth seeds (tests/lk_exact.py) and check them against the
stored digests.
Run in the build container (needs cv2):  python tests/golden/make_golden_lk_sizes.py"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, 'sg-slam_b200'), os.path.join(ROOT, 'tests')]
import lk_exact as X  # noqa: E402  (image and point generators only; the vectors themselves come from cv2)


def main():
    out = {'cv2_version': np.array(cv2.__version__)}
    for w, h, seed in X.GOLDEN_SIZES:
        key = '%dx%d' % (w, h)
        cur, prev = X.image_pair(w, h, seed)
        pts = X.point_set(w, h, seed + 100)
        nlev, _ = cv2.buildOpticalFlowPyramid(cur, (21, 21), 3)
        digests = []
        lv = cur
        for level in range(X.MAX_LEVEL + 1):
            if level:
                lv = cv2.pyrDown(lv)
            dx = cv2.Scharr(lv, cv2.CV_16S, 1, 0, borderType=cv2.BORDER_REFLECT_101)
            dy = cv2.Scharr(lv, cv2.CV_16S, 0, 1, borderType=cv2.BORDER_REFLECT_101)
            digests.append([X.digest(lv), X.digest(dx), X.digest(dy)])
        nxt, st, _ = cv2.calcOpticalFlowPyrLK(cur, prev, pts, None, winSize=(21, 21), maxLevel=3,
                                             criteria=(cv2.TERM_CRITERIA_COUNT | cv2.TERM_CRITERIA_EPS, 30, 0.01))
        out[key + '_images'] = np.array([X.digest(cur), X.digest(prev)])
        out[key + '_max_level'] = np.array(nlev, np.int32)
        out[key + '_digests'] = np.array(digests)          # [level][image, dx, dy], cv2.pyrDown chain to level 3
        out[key + '_pts'] = pts
        out[key + '_tracked'] = nxt.reshape(-1, 2).astype(np.float32)
        out[key + '_status'] = st.reshape(-1).astype(np.uint8)
        print(key, 'max_level', nlev, 'points', len(pts), 'status ok', int(st.sum()))
    np.savez_compressed(os.path.join(HERE, 'lk_sizes.npz'), **out)


if __name__ == '__main__':
    main()
