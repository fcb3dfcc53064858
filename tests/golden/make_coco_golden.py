"""Pin tools/coco_eval_oracle.py against the reference's OWN COCO evaluation code.  evaluate_coco is cut out of the
reference's eval.py with `ast` and executed unmodified on a fake dataset (an instances dict, image_ids not sorted) and a
fake model that returns fixed (scores, labels, boxes) per image; COCOeval and coco.loadRes are bound to the oracle.
Output -> tests/golden/coco_eval.npz: the reference's result list (collection) and the oracle's precision, recall and
stats on it.  The set itself is regenerated from its seed by make_set(), which the tests import.

The set: 300 images, 12 categories with non-contiguous ids, and each of these cases at least once: crowd ground truth,
zero-area ground truth, annotation areas of exactly 32^2 and 96^2, a category with detections but no ground truth
(id 70), a category with ground truth but no detections (id 90), a model label that maps to no ground-truth category,
images with neither, an (image, category) with more than 100 detections, scores tied across images and inside an
image, an IoU of exactly 0.5, and an image whose rows go below the threshold and back above it.

usage: python tests/golden/make_coco_golden.py     (needs a checkout of the reference repository in EFFDET_REFERENCE)"""
import ast
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(REPO, 'tools'))
import coco_eval_oracle as O  # noqa: E402

CAT_IDS = [1, 3, 4, 7, 10, 15, 22, 23, 40, 41, 70, 90]
LABEL_TO_COCO = {i: c for i, c in enumerate(CAT_IDS)}
LABEL_TO_COCO[12] = 99                                               # a model label without a ground-truth category
NIMG, C, THR = 300, 160, 0.05


def make_set(seed=11):
    """-> (instances dict, image_ids in dataset order, scores [N,C] f32, labels [N,C] i64, boxes [N,C,4] f32 (x1,y1,x2,y2
    in network input coordinates), count [N] i32, scale [N] f32); rows of an image are in NMS order"""
    rng = np.random.RandomState(seed)
    ids = rng.choice(np.arange(1, 100000), size=NIMG, replace=False).tolist()
    images = [{'id': i, 'width': 640, 'height': 480} for i in ids]
    anns, aid = [], 1
    scores = np.zeros((NIMG, C), np.float32)
    labels = np.zeros((NIMG, C), np.int64)
    boxes = np.zeros((NIMG, C, 4), np.float32)
    count = np.zeros(NIMG, np.int32)
    scale = rng.uniform(0.5, 1.6, size=NIMG).astype(np.float32)
    scale[:8] = 1.0
    tied = (np.arange(1, 64) / 64.0).astype(np.float32)             # tied scores across and inside images
    for n in range(NIMG):
        gts = []
        ng = 0 if n % 11 == 0 else rng.randint(0, 9)
        for _ in range(ng):
            lab = rng.choice([0, 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 11])
            x, y = rng.uniform(0, 500, size=2)
            w, h = rng.uniform(2, 160, size=2)
            area = w * h if rng.rand() < 0.8 else w * h * rng.uniform(0.4, 1.0)
            crowd = int(rng.rand() < 0.06)
            gts.append((lab, [float(x), float(y), float(w), float(h)], float(area), crowd))
        if n % 17 == 3:
            gts.append((1, [10.0, 10.0, 0.0, 5.0], 0.0, 0))                         # zero-area ground truth
        if n % 23 == 4:
            gts.append((2, [50.0, 60.0, 32.0, 32.0], 1024.0, 0))                    # area exactly 32^2
            gts.append((2, [150.0, 60.0, 96.0, 96.0], 9216.0, 0))                   # area exactly 96^2
        nd = 0 if (n % 11 == 0 and n % 2 == 0) else rng.randint(0, C - 20)
        rows = []
        for _ in range(nd):
            if gts and rng.rand() < 0.6:
                lab, (x, y, w, h), _, _ = gts[rng.randint(len(gts))]
                bx = np.array([x, y, x + w, y + h]) + rng.normal(0, 4, size=4)
                lab = lab if rng.rand() < 0.85 else rng.randint(0, 13)
            else:
                x, y = rng.uniform(0, 500, size=2)
                bx = np.array([x, y, x + rng.uniform(4, 150), y + rng.uniform(4, 150)])
                lab = rng.choice([0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 12])
            lab = 10 if lab == 11 else lab                                          # id 90 keeps no detection
            s = tied[rng.randint(tied.size)] if rng.rand() < 0.3 else np.float32(rng.uniform(0.0, 1.0))
            rows.append((float(s), lab, bx * scale[n]))
        rows.sort(key=lambda r: -r[0])                                              # NMS order: score descending
        for k, (s, lab, bx) in enumerate(rows):
            scores[n, k], labels[n, k], boxes[n, k] = s, lab, bx
        count[n] = len(rows)
        for lab, bb, area, crowd in gts:
            anns.append({'id': aid, 'image_id': ids[n], 'category_id': CAT_IDS[lab], 'bbox': bb, 'area': area,
                         'iscrowd': crowd})
            aid += 1
    # hand-made images (scale 1)
    def put(n, rows):
        scores[n], labels[n], boxes[n] = 0, 0, 0
        for k, (s, lab, bx) in enumerate(rows):
            scores[n, k], labels[n, k], boxes[n, k] = s, lab, bx
        count[n] = len(rows)
    put(1, [(0.9, 3, [0, 0, 2, 1])])                                                 # IoU exactly 0.5 with ...
    anns.append({'id': aid, 'image_id': ids[1], 'category_id': CAT_IDS[3], 'bbox': [0.0, 0.0, 1.0, 1.0],
                 'area': 1.0, 'iscrowd': 0})                                        # ... this ground truth
    aid += 1
    put(5, [(float(np.float32(1.0 - k / 256.0)), 0, [3 * k, 0, 3 * k + 20, 20]) for k in range(130)])  # > 100 rows
    put(6, [(0.8, 4, [0, 0, 10, 10]), (0.04, 4, [0, 0, 11, 11]), (0.7, 4, [0, 0, 12, 12])])       # below, then above
    put(7, [(0.6, 2, [5, 5, 30, 30]), (0.6, 2, [5, 5, 31, 31]), (0.6, 2, [6, 5, 30, 30])])        # ties in an image
    put(0, [])                                                                       # neither (n % 11 == 0)
    inst = {'images': images, 'categories': [{'id': c, 'name': 'c%d' % c} for c in CAT_IDS], 'annotations': anns}
    return inst, ids, scores, labels, boxes, count, scale


def oracle_results(inst, ids, scores, labels, boxes, count, scale):
    out = []
    for n in range(len(ids)):
        k = count[n]
        out += O.collect(ids[n], scores[n, :k], labels[n, :k], boxes[n, :k], float(scale[n]),
                         LABEL_TO_COCO.__getitem__, THR)
    return out


def results_array(results):
    return np.array([[r['image_id'], r['category_id'], r['score']] + list(r['bbox']) for r in results], np.float64)


if __name__ == '__main__':
    import torch
    REF = os.environ.get('EFFDET_REFERENCE')          # path of a checkout of the reference repository
    assert REF, 'set EFFDET_REFERENCE to a checkout of the reference repository'
    inst, ids, scores, labels, boxes, count, scale = make_set()
    assert ids != sorted(ids)

    class _Img:
        def __init__(self, n):
            self.n = n

        def permute(self, *a):
            return self

        def cuda(self):
            return self

        def float(self):
            return self

        def unsqueeze(self, dim):
            return self

    class _Model:
        def eval(self):
            pass

        def train(self):
            pass

        def __call__(self, x):
            k = count[x.n]
            return (torch.from_numpy(scores[x.n, :k].copy()), torch.from_numpy(labels[x.n, :k].copy()),
                    torch.from_numpy(boxes[x.n, :k].copy()))

    class _Dataset:
        set_name = 'golden'
        image_ids = ids
        coco = O.COCO(inst)

        def __len__(self):
            return NIMG

        def __getitem__(self, n):
            return {'img': _Img(n), 'scale': float(scale[n])}

        def label_to_coco_label(self, label):
            return LABEL_TO_COCO[label]

    runs = []

    class _Eval(O.COCOeval):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            runs.append(self)

    src = open(os.path.join(REF, 'eval.py')).read()
    ns = {'np': np, 'torch': torch, 'json': json, 'COCOeval': _Eval}
    for node in ast.parse(src).body:
        if getattr(node, 'name', None) == 'evaluate_coco':
            exec(compile(ast.Module([node], []), 'eval.py', 'exec'), ns)
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            ns['evaluate_coco'](_Dataset(), _Model())
            ref_results = json.load(open('golden_bbox_results.json'))
        finally:
            os.chdir(cwd)
    E = runs[0]
    mine = oracle_results(inst, ids, scores, labels, boxes, count, scale)
    assert json.dumps(mine, indent=4) == json.dumps(ref_results, indent=4)
    assert O.iou([[0.0, 0.0, 2.0, 1.0]], [[0.0, 0.0, 1.0, 1.0]], [0])[0, 0] == 0.5
    K = len(CAT_IDS)
    P, Rc = E.eval['precision'], E.eval['recall']
    assert (P[:, :, CAT_IDS.index(90)] == 0).all() and (P[:, :, CAT_IDS.index(70)] == -1).all()
    print('\n'.join(E.lines))
    np.savez_compressed(os.path.join(HERE, 'coco_eval.npz'), results=results_array(ref_results), precision=P, recall=Rc,
                        stats=np.asarray(E.stats, np.float64))
    print('coco_eval.npz written: %d results, oracle collection == reference collection' % len(ref_results))
