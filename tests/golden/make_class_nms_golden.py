"""Pin torchvision's per-class NMS -> tests/golden/class_nms.npz.

For every case the file keeps the inputs (the seed and the SHA-256 of the inputs for the random cases, the inputs
themselves for the crafted ones) and three keep lists, from torchvision 0.26 on the CPU at IoU threshold 0.5:
  vanilla : torchvision.ops.boxes._batched_nms_vanilla -- torchvision.ops.nms per class, then a sort by score
  batched : torchvision.ops.batched_nms, which takes the coordinate trick for up to 1000 boxes on the CPU
  trick   : torchvision.ops.boxes._batched_nms_coordinate_trick -- one nms over boxes offset by class * (max + 1) in fp32
`trick_differs` marks the cases whose trick keep set differs from the vanilla one: the offset rounds coordinates, so
IoUs near the threshold can change.

Cases: ties within and across classes; identical boxes under different classes; a pair at IoU exactly 0.5 and one just
above it; a single class; about 700 candidates of 20 and of 80 classes; about 3000 and 6000 candidates of 80 classes;
a pair whose IoU the coordinate trick rounds to the threshold; an empty image.

usage: python tests/golden/make_class_nms_golden.py"""
import hashlib
import os
import sys

import numpy as np
import torch
import torchvision
from torchvision.ops import boxes as tvb

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(REPO, 'tools'))
import class_nms_oracle as C  # noqa: E402

IOU = 0.5


def digest(*arrays):
    h = hashlib.sha256()
    for a in arrays:
        h.update(np.ascontiguousarray(a).tobytes())
    return np.frombuffer(h.digest(), dtype=np.uint8)


def crafted():
    """name -> (boxes, scores, classes)"""
    c = {}
    # equal scores: overlapping boxes of one class, and of two classes
    c['ties'] = ([[0, 0, 10, 10], [1, 1, 11, 11], [2, 0, 12, 10], [0, 2, 10, 12], [30, 30, 40, 40], [31, 30, 41, 40],
                  [0, 0, 10, 10], [1, 1, 11, 11]],
                 [0.8, 0.8, 0.8, 0.6, 0.6, 0.6, 0.8, 0.6], [1, 1, 2, 1, 0, 0, 0, 2])
    c['identical'] = ([[5, 5, 25, 25]] * 6, [0.9, 0.8, 0.7, 0.6, 0.5, 0.4], [0, 1, 2, 0, 1, 2])
    # [0,0,3,1] / [1,0,4,1]: IoU exactly 0.5 (both kept); [20,0,23,1] / [20.99,0,24,1]: intersection 2.01, union 4,
    # IoU 0.5025 (the second suppressed)
    c['iou_half'] = ([[0, 0, 3, 1], [1, 0, 4, 1], [20, 0, 23, 1], [20.99, 0, 24, 1]], [0.9, 0.8, 0.9, 0.8],
                     [3, 3, 3, 3])
    b, s, _ = C.random_class_candidates(5, 300, 1)
    c['one_class'] = (b, s, np.zeros(300, np.int32))
    # IoU just above 0.5 in fp32; offset by 79 * (max + 1) the coordinates round and the IoU falls to 0.5 or below, so
    # the coordinate trick keeps both boxes of class 79
    c['trick_rounding'] = ([[251.6432647705078, 370.86181640625, 280.864013671875, 428.3642883300781],
                            [261.3834533691406, 370.86181640625, 290.6042175292969, 428.3642883300781],
                            [10, 10, 50, 50]], [0.9, 0.8, 0.7], [79, 79, 0])
    c['empty'] = (np.zeros((0, 4)), np.zeros(0), np.zeros(0))
    return {k: (np.asarray(b, np.float32).reshape(-1, 4), np.asarray(s, np.float32), np.asarray(cl, np.int32))
            for k, (b, s, cl) in c.items()}


RANDOM = [('random_k20', 21, 700, 20), ('random_k80', 22, 700, 80), ('random_3000', 23, 3000, 20),
          ('random_6000', 24, 6000, 80)]


def main():
    data, names, differs = {}, [], []
    cases = [(n, b, s, cl, -1) for n, (b, s, cl) in crafted().items()]
    for name, seed, n, K in RANDOM:
        b, s, cl = C.random_class_candidates(seed, n, K)
        cases.append((name, b, s, cl, seed))
    for name, b, s, cl, seed in cases:
        tb, ts, tc = torch.from_numpy(b), torch.from_numpy(s), torch.from_numpy(cl.astype(np.int64))
        vanilla = tvb._batched_nms_vanilla(tb, ts, tc, IOU).numpy()
        batched = torchvision.ops.batched_nms(tb, ts, tc, IOU).numpy()
        trick = tvb._batched_nms_coordinate_trick(tb, ts, tc, IOU).numpy()
        p = name + '/'
        names.append(name)
        data.update({p + 'vanilla': vanilla, p + 'batched': batched, p + 'trick': trick, p + 'seed': np.array([seed]),
                     p + 'K': np.array([int(cl.max()) + 1 if len(cl) else 0])})
        if seed >= 0:
            data[p + 'input_sha256'] = digest(b, s, cl)
            data[p + 'n'] = np.array([len(s)])
        else:
            data.update({p + 'boxes': b, p + 'scores': s, p + 'classes': cl})
        d = set(trick.tolist()) != set(vanilla.tolist())
        if d:
            differs.append(name)
        print('%-12s %5d candidates %5d kept%s' % (name, len(s), len(vanilla), '  (coordinate trick differs)' if d else ''))
    data['cases'] = np.array(names)
    data['trick_differs'] = np.array(differs)
    data['torchvision'] = np.array(torchvision.__version__)
    np.savez_compressed(os.path.join(HERE, 'class_nms.npz'), **data)


if __name__ == '__main__':
    main()
