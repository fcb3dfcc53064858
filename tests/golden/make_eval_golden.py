"""Pin tools/voc_eval_oracle.py against the reference's OWN evaluation code.  compute_overlap, _compute_ap and evaluate
are cut out of the reference's eval.py with `ast` and executed unmodified; _get_detections / _get_annotations are bound
to the synthetic per-image lists below (detections selected from padded model outputs as eval.py:107-133 does).
Output -> tests/golden/voc_eval.npz: the padded per-image inputs, the ground truth and the reference's results.

The synthetic set: 300 images, 7 classes, tie-free scores, and each of these cases at least once: a class with
detections but no ground truth (5), a class with ground truth but no detections (6), images without ground truth, two
detections on one ground truth, a best-overlap ground truth already taken while another one overlaps >= 0.5, an IoU of
exactly 0.5, a zero-area ground truth, and one class with more than 2,000 records.

usage: python tests/golden/make_eval_golden.py     (needs a checkout of the reference repository in EFFDET_REFERENCE)"""
import ast
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get('EFFDET_REFERENCE')          # path of a checkout of the reference repository
assert REF, 'set EFFDET_REFERENCE to a checkout of the reference repository'
sys.path.insert(0, os.path.join(REPO, 'tools'))
import voc_eval_oracle as V  # noqa: E402

K, NIMG, C, THR, MAX_DET = 7, 300, 120, 0.05, 100


def make_set(seed=3):
    rng = np.random.RandomState(seed)
    gts, counts = [], rng.randint(0, 5, size=NIMG)
    counts[::9] = 0                                                    # images without ground truth
    for i in range(NIMG):
        xy = rng.uniform(0, 400, size=(counts[i], 2))
        wh = rng.uniform(8, 120, size=(counts[i], 2))
        lab = rng.choice([0, 0, 0, 1, 2, 3, 4, 6], size=counts[i])
        gts.append(np.concatenate([xy, xy + wh, lab[:, None]], axis=1).astype(np.float64))
    scores = np.zeros((NIMG, C), np.float32)
    labels = np.zeros((NIMG, C), np.int64)
    boxes = np.zeros((NIMG, C, 4), np.float32)
    n_det = rng.randint(0, C + 1, size=NIMG)
    n_det[::13] = 0
    scale = rng.uniform(0.5, 1.6, size=NIMG).astype(np.float32)
    scale[:8] = 1.0                                                    # the hand-made cases are in image coordinates
    # tie-free scores: distinct float32 values over the whole set, some of them below the threshold
    pool = np.unique(rng.uniform(0.0, 1.0, size=NIMG * C * 2).astype(np.float32))
    pool = pool[rng.permutation(pool.shape[0])][:NIMG * C]
    assert pool.shape[0] == NIMG * C
    for i in range(NIMG):
        n = n_det[i]
        scores[i, :n] = np.sort(pool[i * C:i * C + n])[::-1]          # NMS output order: score descending
        for k in range(n):
            g = gts[i]
            if g.shape[0] and rng.rand() < 0.6:                         # near a ground-truth box (scaled to the input)
                j = rng.randint(g.shape[0])
                bx = g[j, :4] + rng.normal(0, 6, size=4)
                lab = int(g[j, 4]) if rng.rand() < 0.85 else rng.randint(0, 6)
                lab = 0 if lab == 6 else lab                            # class 6 keeps no detection
            else:
                xy = rng.uniform(0, 400, size=2)
                bx = np.concatenate([xy, xy + rng.uniform(8, 120, size=2)])
                lab = rng.choice([0, 0, 1, 2, 3, 4, 5])
            boxes[i, k] = bx * scale[i]
            labels[i, k] = lab
    # hand-made cases on images 0..4 (scale 1, exactly representable coordinates)
    def put(i, rows, dets):
        gts[i] = np.array(rows, dtype=np.float64).reshape(-1, 5)
        n_det[i] = len(dets)
        top = np.sort(pool[i * C:i * C + C])[::-1]
        top = top[top > 0.5]
        for k, (bx, lab) in enumerate(dets):
            scores[i, k], labels[i, k], boxes[i, k] = top[k], lab, bx
        scores[i, len(dets):], labels[i, len(dets):], boxes[i, len(dets):] = 0, 0, 0
    put(0, [[10, 10, 20, 20, 1]], [([10, 10, 20, 20], 1), ([11, 10, 20, 20], 1)])              # two dets, one GT
    put(1, [[0, 0, 10, 10, 2], [0, 1, 10, 11, 2]], [([0, 0, 10, 10], 2), ([0, 0, 10, 10], 2)])  # best GT taken
    put(2, [[0, 0, 1, 1, 3]], [([0, 0, 2, 1], 3)])                                              # IoU exactly 0.5
    put(3, [[5, 5, 5, 9, 4], [30, 30, 40, 40, 4]], [([5, 5, 5, 9], 4), ([4, 5, 6, 9], 4), ([30, 30, 40, 40], 4)])
    put(4, [[50, 50, 60, 60, 2]], [([50, 50, 60, 60], 5)])                                      # class 5: no GT
    return scores, labels, boxes, n_det.astype(np.int32), scale, gts


def selected(scores, labels, boxes, count, scale):
    return [V.select_detections(scores[i, :count[i]], labels[i, :count[i]], boxes[i, :count[i]], float(scale[i]), THR,
                                MAX_DET, K) for i in range(NIMG)]


if __name__ == '__main__':
    scores, labels, boxes, count, scale, gts = make_set()
    all_det = selected(scores, labels, boxes, count, scale)
    all_ann = [[g[g[:, 4] == c, :4].copy() for c in range(K)] for g in gts]
    assert V.overlaps(all_det[2][3], all_ann[2][3])[0, 0] == 0.5
    recs = [sum(d[c].shape[0] for d in all_det) for c in range(K)]
    assert recs[0] > 2000 and recs[5] > 0 and recs[6] == 0, recs
    assert sum(a[6].shape[0] for a in all_ann) > 0 and sum(a[5].shape[0] for a in all_ann) == 0

    src = open(os.path.join(REF, 'eval.py')).read()
    ns = {'np': np}
    for node in ast.parse(src).body:
        if getattr(node, 'name', None) in ('compute_overlap', '_compute_ap', 'evaluate'):
            exec(compile(ast.Module([node], []), 'eval.py', 'exec'), ns)
    ns['_get_detections'] = lambda generator, retinanet, **kw: all_det
    ns['_get_annotations'] = lambda generator: all_ann

    class _Gen:
        def num_classes(self):
            return K

        def __len__(self):
            return NIMG

        def label_to_name(self, label):
            return str(label)

    ref_mean, ref_aps = ns['evaluate'](_Gen(), None, iou_threshold=0.5, score_threshold=THR, max_detections=MAX_DET)
    o_mean, o_aps = V.evaluate(all_det, all_ann, K, 0.5)
    assert o_mean == ref_mean and all(o_aps[c] == ref_aps[c] for c in range(K)), (o_aps, ref_aps)
    assert all(type(o_aps[c][0]) is type(ref_aps[c][0]) for c in range(K))
    rows = np.concatenate(gts, axis=0)
    np.savez_compressed(os.path.join(HERE, 'voc_eval.npz'), scores=scores, labels=labels.astype(np.int8), boxes=boxes,
                        count=count, scale=scale, gt_rows=rows, gt_counts=np.array([g.shape[0] for g in gts], np.int32),
                        ap=np.array([ref_aps[c][0] for c in range(K)], np.float64),
                        num_annotations=np.array([ref_aps[c][1] for c in range(K)], np.float64),
                        mean_ap=np.array([ref_mean]), config=np.array([K, MAX_DET]), thresholds=np.array([THR, 0.5]))
    print('voc_eval.npz written; oracle == reference code; records per class', recs)
