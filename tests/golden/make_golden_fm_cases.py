#!/usr/bin/env python3
"""Golden results of the REAL cv2.findFundamentalMat(m1, m2, FM_RANSAC, thresh, confidence, max_iters) on the constructed cases of
tests/fm_cases.py.  Per case: the input pairs, status ('ok', 'empty': cv2 returned no matrix, 'raises': cv2 threw), F (stacked 3k x 3 as
cv2 returns it; (0, 3) unless ok) and the mask ((0,) unless ok).  Run in the build container:  python tests/golden/make_golden_fm_cases.py"""
import os
import sys

import cv2
import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path[:0] = [os.path.join(ROOT, 'tests'), os.path.join(ROOT, 'oracle')]
import fm_cases  # noqa: E402


def run_cv2(case):
    p = case['params']
    try:
        F, mask = cv2.findFundamentalMat(case['m1'], case['m2'], cv2.FM_RANSAC, p['thresh'], p['confidence'], p['max_iters'])
    except cv2.error:
        return 'raises', np.zeros((0, 3)), np.zeros(0, np.uint8)
    if F is None or F.size == 0:
        return 'empty', np.zeros((0, 3)), np.zeros(0, np.uint8)
    return 'ok', F, mask.ravel().astype(np.uint8)


def main():
    out = {}
    names = []
    for c in fm_cases.cases():
        status, F, mask = run_cv2(c)
        assert (status == 'raises') == (c['group'] == 'raises'), (c['name'], status)
        names.append(c['name'])
        out[c['name'] + '_m1'] = c['m1']; out[c['name'] + '_m2'] = c['m2']
        out[c['name'] + '_status'] = np.array(status); out[c['name'] + '_F'] = F; out[c['name'] + '_mask'] = mask
        print(c['name'], status, F.shape, int(mask.sum()))
    out['names'] = np.array(names); out['cv2_version'] = np.array(cv2.__version__)
    np.savez_compressed(os.path.join(HERE, 'fm_cases.npz'), **out)


if __name__ == '__main__':
    main()
