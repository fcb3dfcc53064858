"""COCO box mAP on the device (csrc/coco_eval.cu, models/evaluation.py) against tools/coco_eval_oracle.py, which
tests/golden/make_coco_golden.py pins to the reference's own evaluate_coco (tests/golden/coco_eval.npz).

CPU: the oracle equals the fixture, hand-worked COCOeval cases, the ground-truth grouping, argument refusals, and a
cross-check against pycocotools where it is installed.
GPU: the accumulator equals the fixture bit for bit in any batching, the collection and results() equal the
reference's, ties follow the stable order, add() is sync-free and capturable, a random 80-category set equals the
oracle, and evaluate_coco on a real D0 equals COCOeval on its own results file and agrees with the reference loop."""
import json
import os
import sys

import numpy as np
import pytest
import torch

import effdet_oracle as EO

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'tools'))
sys.path.insert(0, os.path.join(HERE, 'golden'))
import coco_eval_oracle as O  # noqa: E402
import make_coco_golden as MG  # noqa: E402

gpu = pytest.mark.gpu


def _fixture():
    return np.load(os.path.join(HERE, 'golden', 'coco_eval.npz'))


def _same(got, want):
    for g, w in zip(got, want):
        g, w = np.asarray(g), np.asarray(w)
        assert g.shape == w.shape and g.dtype == w.dtype
        assert np.array_equal(g, w), np.argwhere(g != w)[:5]


def _run_oracle(inst, results, ids):
    return O.evaluate(inst, results, ids)


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------

def test_oracle_equals_reference_fixture():
    st = _fixture()
    inst, ids, *rest = MG.make_set()
    results = MG.oracle_results(inst, ids, *rest)
    assert np.array_equal(MG.results_array(results), st['results'])
    _same(_run_oracle(inst, results, ids), (st['stats'], st['precision'], st['recall']))


def _case(gts, dets, cats=(1, 2), images=(1, 2, 3)):
    """gts: (image, cat, [x,y,w,h], area, crowd); dets: (image, cat, [x,y,w,h], score) -> (stats, precision, recall)"""
    inst = {'images': [{'id': i} for i in images], 'categories': [{'id': c} for c in cats],
            'annotations': [{'id': n + 1, 'image_id': i, 'category_id': c, 'bbox': list(map(float, b)), 'area': float(a),
                             'iscrowd': cr} for n, (i, c, b, a, cr) in enumerate(gts)]}
    res = [{'image_id': i, 'category_id': c, 'bbox': list(map(float, b)), 'score': s} for i, c, b, s in dets]
    return O.evaluate(inst, res, list(images))


T50, T55, T95 = 0, 1, 9          # IoU threshold indices
ONE = 1.0 / (1.0 + np.spacing(1))  # precision after one TP and no FP: tp / ((fp + tp) + eps)
ALL, SMALL, MEDIUM, LARGE = 0, 1, 2, 3


def test_known_answers():
    # equal IoU: the later ground truth in the list wins
    _, p, r = _case([(1, 1, [0, 0, 2, 1], 2, 0), (1, 1, [1, 0, 2, 1], 2, 0)],
                    [(1, 1, [0, 0, 3, 1], 0.9), (1, 1, [0, 0, 2, 1], 0.8)])
    # d0 IoU 2/3 with both: takes the LATER (g2); d1 IoU 1 with g1 (free) and 1/3 with g2: TP.  Two TPs, recall 1
    assert r[T50, 0, ALL, 2] == 1.0 and p[T50, 100, 0, ALL, 2] == 1.0
    # at .55 the same; if the first one had won, d1 (IoU 1 with g1) would be the FP -> recall 0.5
    assert r[T55, 0, ALL, 2] == 1.0
    # one crowd ground truth absorbs two detections, both ignored; a regular gt elsewhere keeps npig = 1
    _, p, r = _case([(1, 1, [0, 0, 10, 10], 100, 1), (2, 1, [0, 0, 10, 10], 100, 0)],
                    [(1, 1, [0, 0, 10, 10], 0.9), (1, 1, [0, 0, 9, 10], 0.8), (2, 1, [0, 0, 10, 10], 0.7)])
    assert r[T50, 0, ALL, 2] == 1.0 and p[T50, 100, 0, ALL, 2] == ONE       # the crowd matches are not FPs
    # break on an ignored ground truth after a regular match: g0 regular (IoU .6), g1 crowd (IoU 1 in crowd terms)
    _, p, r = _case([(1, 1, [0, 0, 10, 10], 100, 0), (1, 1, [0, 0, 6, 10], 60, 1)],
                    [(1, 1, [0, 0, 6, 10], 0.9)])
    assert r[T50, 0, ALL, 2] == 1.0 and r[T95, 0, ALL, 2] == 0.0          # TP at .5 on g0, not absorbed by the crowd
    # IoU exactly at the threshold matches (0.5 exactly representable)
    _, p, r = _case([(1, 1, [0, 0, 1, 1], 1, 0)], [(1, 1, [0, 0, 2, 1], 0.9)])
    assert r[T50, 0, ALL, 2] == 1.0 and r[T55, 0, ALL, 2] == 0.0
    # area exactly 32^2 counts in small and medium; 96^2 in medium and large
    _, p, r = _case([(1, 1, [0, 0, 32, 32], 1024, 0), (2, 1, [0, 0, 96, 96], 9216, 0)],
                    [(1, 1, [0, 0, 32, 32], 0.9), (2, 1, [0, 0, 96, 96], 0.8)])
    assert r[T50, 0, SMALL, 2] == 1.0 and r[T50, 0, MEDIUM, 2] == 1.0 and r[T50, 0, LARGE, 2] == 1.0
    assert p[T50, 100, 0, MEDIUM, 2] == 1.0
    # an unmatched detection outside the area range is ignored: small range, a large FP does not cost precision
    _, p, r = _case([(1, 1, [0, 0, 10, 10], 100, 0)], [(1, 1, [50, 50, 50, 50], 0.95), (1, 1, [0, 0, 10, 10], 0.9)])
    assert p[T50, 100, 0, SMALL, 2] == ONE and p[T50, 100, 0, ALL, 2] == 0.5
    # maxDets 1 and 10: a TP at rank 2 / rank 11 of its image does not count below that cap
    dets = [(1, 1, [100 + 20 * k, 0, 10, 10], 0.9 - 0.01 * k) for k in range(11)] + [(1, 1, [0, 0, 10, 10], 0.5)]
    _, p, r = _case([(1, 1, [0, 0, 10, 10], 100, 0)], dets)
    assert r[T50, 0, ALL, 0] == 0.0 and r[T50, 0, ALL, 1] == 0.0 and r[T50, 0, ALL, 2] == 1.0
    assert p[T50, 0, 0, ALL, 2] == 1.0 / 12
    # a category without ground truth is -1 and excluded from the means; recall thresholds past the maximum recall: 0
    stats, p, r = _case([(1, 1, [0, 0, 10, 10], 100, 0), (2, 1, [0, 0, 10, 10], 100, 0)],
                        [(1, 1, [0, 0, 10, 10], 0.9), (3, 2, [0, 0, 10, 10], 0.9)])
    assert (p[:, :, 1] == -1).all() and (r[:, 1] == -1).all()
    assert r[T50, 0, ALL, 2] == 0.5 and p[T50, 50, 0, ALL, 2] == ONE and p[T50, 51, 0, ALL, 2] == 0.0
    assert stats[8] == 0.5 and stats[1] == np.mean([ONE] * 51 + [0.0] * 50)
    # ties across images follow the sorted image ids, not the dataset order: image 1 (FP) before image 2 (TP)
    g, d = [(2, 1, [0, 0, 10, 10], 100, 0)], [(2, 1, [0, 0, 10, 10], 0.5), (1, 1, [0, 0, 10, 10], 0.5)]
    for images in ((2, 1), (1, 2)):
        _, p, r = _case(g, d, images=images)
        assert p[T50, 100, 0, ALL, 2] == 0.5, images                        # FP first: precision 1/2 at recall 1


def test_ground_truth_grouping_order():
    """COCOAccumulator groups the ground truth by (image rank, category index) and keeps annotation order inside a
    group; annotations of unknown images or categories are left out; crowd and zero-area ones stay"""
    from models.evaluation import COCOAccumulator
    inst = {'images': [{'id': 9}, {'id': 4}], 'categories': [{'id': 7}, {'id': 3}],
            'annotations': [{'id': 1, 'image_id': 9, 'category_id': 7, 'bbox': [0, 0, 1, 1], 'area': 1, 'iscrowd': 0},
                            {'id': 2, 'image_id': 4, 'category_id': 7, 'bbox': [1, 0, 0, 1], 'area': 0, 'iscrowd': 0},
                            {'id': 3, 'image_id': 9, 'category_id': 7, 'bbox': [2, 0, 1, 1], 'area': 1, 'iscrowd': 1},
                            {'id': 4, 'image_id': 9, 'category_id': 3, 'bbox': [3, 0, 1, 1], 'area': 1, 'iscrowd': 0},
                            {'id': 5, 'image_id': 5, 'category_id': 3, 'bbox': [4, 0, 1, 1], 'area': 1, 'iscrowd': 0},
                            {'id': 6, 'image_id': 9, 'category_id': 8, 'bbox': [5, 0, 1, 1], 'area': 1, 'iscrowd': 0}]}

    acc = COCOAccumulator(inst, [9, 4], {0: 3, 1: 7}, device='cpu')        # host grouping, CPU tensors
    assert acc.ids_by_rank == [4, 9] and acc.cat_ids == [3, 7] and acc.max_gt == 2
    rows = acc.gt.numpy()
    # groups: (rank 0 = id 4, cat 3): -, (0, 7): ann 2, (1 = id 9, 3): ann 4, (1, 7): anns 1, 3 in that order
    assert rows[:, 0].tolist() == [1, 3, 0, 2] and rows[:, 5].tolist() == [0, 0, 0, 1]
    assert acc.gt_offsets.tolist() == [0, 0, 1, 2, 4]


def test_coco_entry_points_refuse_bad_arguments():
    """each refusal returns -1, names the entry point and comes before any device work (never-dereferenced pointers),
    so these calls run without a GPU"""
    from models import _native
    _native.build()
    lib = _native.load()
    f = 1 << 20

    def refused(rc, what):
        msg = lib.effdet_last_error().decode()
        assert rc == -1 and what in msg, (rc, msg)

    def sel(*, sc=f, B=2, C=50, thr=0.05, K=80, n=10, cap=1000, box=f, meta=f, rank=f):
        return lib.effdet_coco_select_batch(sc, f, box, f, f, rank, B, C, thr, f, 80, K, n, cap, f, f, meta, f, f, f, f,
                                            f, f, 0, None)

    refused(sel(K=256), 'num_categories=256')
    refused(sel(n=(1 << 18) + 1), 'num_images')
    refused(sel(cap=(1 << 25) + 1), 'capacity')
    refused(sel(thr=-0.1), 'score_threshold')
    refused(sel(sc=None), 'null')
    refused(sel(rank=None), 'null')
    refused(sel(B=0), 'B=0')
    refused(sel(box=f + 4), 'aligned')
    refused(sel(meta=f + 8), 'aligned')

    def match(*, iou_type=1, nthr=10, K=80, gt=f, max_gt=3, flags=f, B=2):
        return lib.effdet_coco_match(f, f, f, f, f, B, gt, f, 10, K, max_gt, f, nthr, iou_type, flags, f, 0, None)

    refused(match(iou_type=2), 'bbox')
    refused(match(nthr=11), 'num_iou_thrs')
    refused(match(K=256), 'num_categories=256')
    refused(match(max_gt=257), 'max_gt')
    refused(match(gt=None), 'null')
    refused(match(flags=None), 'null')
    refused(match(B=11), 'B=11')

    assert lib.effdet_coco_accumulate_workspace(1 << 25, 1 << 18, 255) > 0
    assert lib.effdet_coco_accumulate_workspace((1 << 25) + 1, 10, 20) == -1
    ws = lib.effdet_coco_accumulate_workspace(1000, 10, 20)

    def acc(*, nr=101, md=(1, 10, 100), ws_bytes=ws, w=f, prec=f):
        return lib.effdet_coco_accumulate(f, f, f, f, f, f, f, f, nr, *md, 1000, 10, 20, prec, f, w, ws_bytes, 0, None)

    refused(acc(nr=100), 'num_rec_thrs')
    refused(acc(md=(1, 10, 50)), 'max_dets')
    refused(acc(prec=None), 'null')
    refused(acc(ws_bytes=ws - 8), 'workspace')
    refused(acc(w=f + 8), 'aligned')


def test_oracle_equals_pycocotools_where_installed():
    pc = pytest.importorskip('pycocotools.cocoeval', reason='pycocotools is not installed: the cross-check against '
                             'the real COCOeval does not run here')
    from pycocotools.coco import COCO
    inst, ids, *rest = MG.make_set()
    results = MG.oracle_results(inst, ids, *rest)
    gt = COCO()
    gt.dataset = json.loads(json.dumps(inst))
    gt.createIndex()
    E = pc.COCOeval(gt, gt.loadRes(json.loads(json.dumps(results))), 'bbox')
    E.params.imgIds = list(ids)
    E.evaluate()
    E.accumulate()
    E.summarize()
    st = _fixture()
    _same((np.asarray(E.stats), E.eval['precision'], E.eval['recall']), (st['stats'], st['precision'], st['recall']))


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------

def _dev():
    return torch.device('cuda:0')


def _detections(arrs, i0, i1):
    from models._ops import Detections
    scores, labels, boxes, count = arrs
    d = _dev()
    return Detections(*(torch.from_numpy(np.ascontiguousarray(a[i0:i1])).to(d) for a in (scores, labels, boxes, count)))


def _accumulate(inst, ids, scores, labels, boxes, count, scale, batch, label_map=None, **kw):
    from models.evaluation import COCOAccumulator
    lm = MG.LABEL_TO_COCO if label_map is None else label_map
    acc = COCOAccumulator(inst, ids, lm.__getitem__, num_labels=len(lm), device=_dev(), **kw)
    n = len(ids)
    for i0 in range(0, n, batch):
        i1 = min(n, i0 + batch)
        acc.add(_detections((scores, labels, boxes, count), i0, i1), [float(s) for s in scale[i0:i1]])
    return acc


@gpu
@pytest.mark.parametrize('batch', [1, 7, 64])
def test_accumulator_equals_fixture(batch):
    st = _fixture()
    inst, ids, *arrs = MG.make_set()
    acc = _accumulate(inst, ids, *arrs, batch)
    stats, p, r = acc.compute()
    _same((stats, p, r), (st['stats'], st['precision'], st['recall']))
    if batch == 7:
        want = MG.oracle_results(inst, ids, *arrs)
        got = acc.results()
        assert json.dumps(got, indent=4) == json.dumps(want, indent=4)         # collection and JSON bytes
        assert np.array_equal(MG.results_array(got), st['results'])


@gpu
def test_tied_scores_follow_the_stable_order():
    """equal scores across two images and inside one: the device follows COCOeval's stable order (sorted image id,
    then NMS order), and the reversed tie order gives another result, so the test can see it"""
    inst = {'images': [{'id': 5}, {'id': 2}], 'categories': [{'id': 1}],
            'annotations': [{'id': 1, 'image_id': 2, 'category_id': 1, 'bbox': [0, 0, 10, 10], 'area': 100,
                             'iscrowd': 0},
                            {'id': 2, 'image_id': 5, 'category_id': 1, 'bbox': [40, 0, 10, 10], 'area': 100,
                             'iscrowd': 0}]}
    ids = [5, 2]                                            # dataset order: image 5 first; COCOeval: image 2 first
    scores = np.array([[0.5, 0.5], [0.5, 0.5]], np.float32)
    labels = np.zeros((2, 2), np.int64)
    boxes = np.array([[[40, 0, 50, 10], [80, 0, 90, 10]], [[60, 0, 70, 10], [0, 0, 10, 10]]], np.float32)
    count = np.array([2, 2], np.int32)
    scale = np.ones(2, np.float32)
    results = []
    for n in range(2):
        results += O.collect(ids[n], scores[n], labels[n], boxes[n], 1.0, {0: 1}.__getitem__)
    want = O.evaluate(inst, results, ids)
    # the same records with the tie order reversed inside each image: another precision curve
    rev = [dict(r) for r in results]
    rev = rev[1::-1] + rev[:1:-1]
    assert not np.array_equal(O.evaluate(inst, rev, ids)[1], want[1])
    acc = _accumulate(inst, ids, scores, labels, boxes, count, scale, 2, label_map={0: 1})
    _same(acc.compute(), want)


@gpu
def test_add_is_sync_free_and_capturable():
    """add() under torch.cuda.set_sync_debug_mode('error') raises nothing; an add() captured in a CUDA graph and
    replayed leaves the accumulator exactly where the eager add() does"""
    from models.evaluation import COCOAccumulator
    inst, ids, *arrs = MG.make_set()
    scale = arrs[-1]
    B = 16
    dets = _detections(arrs[:4], 0, B)
    scales = [float(s) for s in scale[:B]]
    mk = lambda: COCOAccumulator(inst, ids, MG.LABEL_TO_COCO.__getitem__, num_labels=13, device=_dev())  # noqa: E731
    torch.cuda.synchronize()
    eager = mk()
    torch.cuda.set_sync_debug_mode('error')
    try:
        eager.add(dets, scales)
    finally:
        torch.cuda.set_sync_debug_mode(0)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        mk().add(dets, scales)                                                 # warm-up off the capture
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graphed = mk()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        graphed.add(dets, scales)
    g.replay()
    torch.cuda.synchronize()
    for name in ('rec_box', 'rec_score', 'rec_meta', 'flags', 'cursor', 'image_offset', 'image_count', 'status',
                 'npig'):
        assert torch.equal(getattr(graphed, name), getattr(eager, name)), name
    assert int(eager.cursor) > 0 and int(eager.npig.sum()) > 0


def _random_set(n_img=500, K=80, seed=3, C=300):
    rng = np.random.RandomState(seed)
    cat_ids = sorted(rng.choice(np.arange(1, 200), size=K, replace=False).tolist())
    ids = rng.choice(np.arange(1, 10 ** 6), size=n_img, replace=False).tolist()
    anns, aid = [], 1
    scores = np.zeros((n_img, C), np.float32)
    labels = np.zeros((n_img, C), np.int64)
    boxes = np.zeros((n_img, C, 4), np.float32)
    count = rng.randint(0, C + 1, size=n_img).astype(np.int32)
    scale = rng.uniform(0.6, 1.4, size=n_img).astype(np.float32)
    for n in range(n_img):
        g = []
        for _ in range(rng.poisson(7)):
            x, y, w, h = rng.uniform(0, 400), rng.uniform(0, 400), rng.uniform(1, 200), rng.uniform(1, 200)
            k = rng.randint(K)
            g.append((k, [x, y, x + w, y + h]))
            anns.append({'id': aid, 'image_id': ids[n], 'category_id': cat_ids[k], 'bbox': [x, y, w, h],
                         'area': w * h, 'iscrowd': int(rng.rand() < 0.05)})
            aid += 1
        s = np.sort(np.round(rng.uniform(0, 1, size=count[n]) * 512) / 512).astype(np.float32)[::-1]
        scores[n, :count[n]] = s
        for k in range(count[n]):
            if g and rng.rand() < 0.5:
                lab, bx = g[rng.randint(len(g))]
                bx = np.array(bx) + rng.normal(0, 5, size=4)
            else:
                lab = rng.randint(K)
                x, y = rng.uniform(0, 400, size=2)
                bx = np.array([x, y, x + rng.uniform(2, 200), y + rng.uniform(2, 200)])
            labels[n, k], boxes[n, k] = lab, bx * scale[n]
    inst = {'images': [{'id': i} for i in ids], 'categories': [{'id': c} for c in cat_ids], 'annotations': anns}
    return inst, ids, {k: c for k, c in enumerate(cat_ids)}, scores, labels, boxes, count, scale


@gpu
def test_random_80_category_set_equals_oracle():
    inst, ids, lm, scores, labels, boxes, count, scale = _random_set()
    results = []
    for n in range(len(ids)):
        results += O.collect(ids[n], scores[n, :count[n]], labels[n, :count[n]], boxes[n, :count[n]],
                             float(scale[n]), lm.__getitem__)
    want = O.evaluate(inst, results, ids)
    acc = _accumulate(inst, ids, scores, labels, boxes, count, scale, 32, label_map=lm)
    _same(acc.compute(), want)


class _CocoDataset:
    """the CocoDataset interface evaluate_coco uses"""
    set_name = 'd0case'

    def __init__(self, images, scales, inst, ids, K):
        self.images, self.scales, self.image_ids, self.K = images, scales, ids, K
        self.coco = O.COCO(inst)

    def __len__(self):
        return len(self.images)

    def __getitem__(self, i):
        return {'img': self.images[i], 'scale': self.scales[i]}

    def label_to_coco_label(self, label):
        return 2 * label + 1


def _reference_evaluate_coco():
    """the reference's evaluate_coco loop (eval.py:260-338; its collection is pinned by the fixture): one model(image)
    per image, host collection, and the oracle's COCOeval"""
    def run(dataset, model, threshold=0.05):
        results, image_ids = [], []
        with torch.no_grad():
            for index in range(len(dataset)):
                data = dataset[index]
                s, l, b = model(data['img'].permute(2, 0, 1).cuda().float().unsqueeze(dim=0))
                results += O.collect(dataset.image_ids[index], s.cpu().numpy(), l.cpu().numpy(), b.cpu().numpy(),
                                     data['scale'], dataset.label_to_coco_label, threshold)
                image_ids.append(dataset.image_ids[index])
        return results, O.evaluate(dataset.coco.dataset, results, image_ids)
    return run


def _d0_case():
    """D0 with well-conditioned weights, 20 random 256x256 images, ground truth on the model's own detections above a
    wide score gap s* (one copy each), plus unmatched boxes outside the image and one image without ground truth"""
    from models import EfficientDet
    K = 80
    cfg = EO.make_config('efficientdet-d0', num_classes=K, W_bifpn=64, D_bifpn=2)
    m = EfficientDet(num_classes=K, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    m.load_state_dict(EO.init_state_dict(cfg, seed=1, mode='wellcond'))
    m = m.to(_dev()).eval()
    m.threshold = 0.65
    x = EO.synthetic_batch(20, size=256, seed=31)[0]
    images = [x[i].permute(1, 2, 0).contiguous() for i in range(20)]
    scales = [1.0 if i % 2 else 0.8 for i in range(20)]
    ids = [int(v) for v in np.random.RandomState(4).permutation(np.arange(100, 120))]
    inst = {'images': [{'id': i} for i in ids], 'categories': [{'id': 2 * k + 1} for k in range(K)], 'annotations': []}
    ds = _CocoDataset(images, scales, inst, ids, K)
    res, _ = _reference_evaluate_coco()(ds, m)
    sc = np.unique([r['score'] for r in res])
    lo, hi = int(0.3 * sc.size), int(0.7 * sc.size)
    j = lo + int(np.argmax(np.diff(sc[lo:hi])))
    s_star, gap = 0.5 * (sc[j] + sc[j + 1]), sc[j + 1] - sc[j]
    assert gap > 1e-5, gap
    anns = []
    for r in res:
        if r['score'] > s_star and r['image_id'] != ids[3]:
            x, y, w, h = r['bbox']
            anns.append({'id': len(anns) + 1, 'image_id': r['image_id'], 'category_id': r['category_id'],
                         'bbox': [x, y, w, h], 'area': w * h, 'iscrowd': 0})
    for i in ids:
        anns.append({'id': len(anns) + 1, 'image_id': i, 'category_id': 15, 'bbox': [1000, 1000, 10, 10], 'area': 100,
                     'iscrowd': 0})
    inst['annotations'] = anns
    ds.s_star = s_star
    return m, ds


@gpu
def test_evaluate_coco_end_to_end_equals_reference_loop(monkeypatch, tmp_path, capsys):
    """evaluate_coco with batch_size 8 (two graphed batches, an eager remainder) returns exactly the stats COCOeval
    gives on the results file it writes, and that file and those stats agree with the reference loop's; then again
    with max_candidates small enough that images overflow NMS and are redone eagerly.  The reference loop runs the
    network again, and two passes differ in the last bits (the order of the SE-mean fp32 atomics): where an NMS
    decision sits at an IoU within that noise of the threshold, one pass keeps a row the other drops, so the
    comparison with the second pass allows that noise."""
    from models import evaluation
    m, ds = _d0_case()
    want_res, want = _reference_evaluate_coco()(ds, m)
    assert 0 < want[0][1] < 1
    monkeypatch.chdir(tmp_path)
    for cap in (None, 'small'):
        m.eval()
        if cap == 'small':
            with torch.no_grad():
                x = torch.stack([ds[i]['img'].permute(2, 0, 1) for i in range(20)]).to(_dev())
                cls, _, _ = m._raw_predictions(x)
            counts = sorted((cls.max(dim=2)[0] > m.threshold).sum(dim=1).tolist())
            assert counts[0] > 0 and counts[-1] > counts[10]
            monkeypatch.setattr(evaluation, 'MAX_CANDIDATES', counts[10])
        got = evaluation.evaluate_coco(ds, m, batch_size=8)
        assert m.training                                                       # model.train() at the end
        res = json.load(open('d0case_bbox_results.json'))
        _same((got,), (O.evaluate(ds.coco.dataset, res, ds.image_ids)[0],))   # bit for bit on its own collection
        assert abs(len(res) - len(want_res)) <= len(want_res) // 100
        assert np.abs(got - want[0]).max() < 1e-3, (got, want[0])
        top = lambda rs: sorted(r['score'] for r in rs if r['score'] > ds.s_star)         # noqa: E731
        assert abs(len(top(res)) - len(top(want_res))) <= 2
    assert 'Average Precision  (AP) @[ IoU=0.50:0.95 | area=   all | maxDets=100 ]' in capsys.readouterr().out
    m.eval()
    m.is_training = True
    with pytest.raises(RuntimeError, match='inference mode'):
        evaluation.evaluate_coco(ds, m)
