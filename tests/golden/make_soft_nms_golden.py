"""Pin tools/soft_nms_oracle.py's Soft-NMS results -> tests/golden/soft_nms.npz.

Cases (threshold 0.05 unless named): 700 seeded random candidates under each method and parameter (linear at
N_t 0.3 and 0.5, gaussian at sigma 0.5 and 0.1); tied scores on overlapping boxes; identical boxes (IoU 1: the linear
weight 0 drops them, the Gaussian weight is exp(-1/sigma)); a pair at IoU exactly 0.5 (not decayed by linear at
N_t = 0.5); zero-area boxes; a score that decays to exactly the threshold (dropped); an all-disjoint set (picked in
score order, scores bit-unchanged); an empty and a one-candidate image.

Per case the file keeps the method and parameters, the inputs (the seed and the SHA-256 of the inputs for the random
cases, the inputs themselves for the crafted ones) and the picked anchors with their float32 scores.  For every
Gaussian weight the oracle evaluates it records the distance of its float64 value to the nearest float32 rounding
boundary, in float64 ulps, and stores the smallest (`gaussian_margin_ulps`): while it is well above 1, a one-ulp
difference between two float64 exp implementations cannot change a weight.

usage: python tests/golden/make_soft_nms_golden.py"""
import hashlib
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(REPO, 'tools'))
import soft_nms_oracle as S  # noqa: E402

THRESHOLD = 0.05
RANDOM_N = 700


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return np.frombuffer(h.digest(), dtype=np.uint8)


def crafted():
    """name -> (boxes, scores, anchors, threshold) of the hand-made cases"""
    f = np.float32
    c = {}
    # tied scores on overlapping boxes: ties go to the lower anchor index, then the decays separate them
    c['ties'] = ([[0, 0, 10, 10], [1, 1, 11, 11], [2, 0, 12, 10], [0, 2, 10, 12], [30, 30, 40, 40], [31, 30, 41, 40]],
                 [0.8, 0.8, 0.8, 0.6, 0.6, 0.6], [7, 3, 5, 2, 9, 8], THRESHOLD)
    c['identical'] = ([[5, 5, 25, 25]] * 4 + [[100, 100, 120, 130]] * 3, [0.9, 0.7, 0.7, 0.3, 0.6, 0.6, 0.2],
                      [4, 1, 2, 3, 0, 6, 5], THRESHOLD)
    # [0,0,3,1] and [1,0,4,1]: intersection 2, union 4 -> IoU exactly 0.5
    c['iou_half'] = ([[0, 0, 3, 1], [1, 0, 4, 1], [0, 0, 3, 2]], [0.9, 0.8, 0.4], [0, 1, 2], THRESHOLD)
    c['zero_area'] = ([[5, 5, 5, 15], [5, 5, 15, 5], [5, 5, 5, 5], [0, 0, 10, 10], [5, 5, 15, 15], [5, 5, 5, 15]],
                      [0.9, 0.85, 0.8, 0.7, 0.65, 0.6], [10, 11, 12, 13, 14, 15], THRESHOLD)
    # [0,0,4,1] then [0,0,3,1]: IoU 0.75, linear weight 0.25: 0.5 * 0.25 = 0.125 == threshold -> dropped;
    # [0,0,4,2] (IoU 0.5 with the first) stays
    c['to_threshold'] = ([[0, 0, 4, 1], [0, 0, 3, 1], [0, 0, 4, 2]], [0.9, 0.5, 0.6], [0, 1, 2], 0.125)
    rng = np.random.default_rng(11)
    g = np.stack(np.meshgrid(np.arange(8), np.arange(8)), -1).reshape(-1, 2) * 20.0
    dis = np.concatenate([g, g + 10], 1)
    c['disjoint'] = (dis, rng.uniform(0.1, 1, 64), rng.permutation(64), THRESHOLD)
    c['empty'] = (np.zeros((0, 4)), np.zeros(0), np.zeros(0, np.int64), THRESHOLD)
    c['one'] = ([[1, 2, 30, 40]], [0.3], [17], THRESHOLD)
    return {k: (np.asarray(b, f).reshape(-1, 4), np.asarray(s, f), np.asarray(a, np.int64), t)
            for k, (b, s, a, t) in c.items()}


PARAMS = [('linear', 0.3, 0.5), ('linear', 0.5, 0.5), ('gaussian', 0.5, 0.5), ('gaussian', 0.5, 0.1)]


def cases():
    """list of (name, method, iou_threshold, sigma, threshold, boxes, scores, anchors, seed or -1)"""
    out = []
    for i, (method, nt, sigma) in enumerate(PARAMS):
        b, s, a = S.random_candidates(100 + i, RANDOM_N, threshold=THRESHOLD)
        out.append(('random_%s_%g_%g' % (method, nt, sigma), method, nt, sigma, THRESHOLD, b, s, a, 100 + i))
    for name, (b, s, a, thr) in crafted().items():
        for method, nt, sigma in (PARAMS[1], PARAMS[2]) if name != 'to_threshold' else (PARAMS[1],):
            out.append(('%s_%s' % (name, method), method, nt, sigma, thr, b, s, a, -1))
    return out


def main():
    data, names, margins = {}, [], []
    for name, method, nt, sigma, thr, b, s, a, seed in cases():
        m = []
        pa, ps = S.soft_nms(b, s, a, method, nt, sigma, thr, margin=m)
        margins += m
        p = name + '/'
        names.append(name)
        data.update({p + 'method': np.array(method), p + 'params': np.array([nt, sigma, thr], np.float64),
                     p + 'picks': pa, p + 'scores': ps, p + 'seed': np.array([seed])})
        if seed >= 0:
            data[p + 'input_sha256'] = digest(b, s, a)
        else:
            data.update({p + 'boxes': b, p + 'in_scores': s, p + 'anchors': a})
        print('%-28s %4d candidates %4d picks' % (name, len(s), len(pa)))
    data['cases'] = np.array(names)
    data['gaussian_margin_ulps'] = np.array([min(margins)])
    print('smallest Gaussian rounding margin: %.1f float64 ulps' % min(margins))
    np.savez_compressed(os.path.join(HERE, 'soft_nms.npz'), **data)


if __name__ == '__main__':
    main()
