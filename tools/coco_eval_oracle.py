"""CPU float64 restatement of the reference's COCO evaluation (eval.py:260-338) and of pycocotools' COCOeval for
iouType 'bbox' with default Params, written fresh in NumPy without importing pycocotools.  Tests and
tools/bench_coco_eval.py compare the device path (csrc/coco_eval.cu, models/evaluation.py) against it; it is pinned
to the reference's own evaluate_coco by tests/golden/make_coco_golden.py -> tests/golden/coco_eval.npz.

  collect         eval.py:280-311 for one image: boxes /= scale, x,y,w,h, rows up to the first score < threshold
  COCO.loadRes    pycocotools COCO.loadRes for bbox results: area = w*h, id = index + 1, iscrowd = 0
  COCOeval        COCOeval.evaluate (_prepare, computeIoU, evaluateImg), accumulate and summarize
  iou             maskApi.c bbIou
"""
import copy
import json

import numpy as np

AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ['all', 'small', 'medium', 'large']
MAX_DETS = [1, 10, 100]


def iou_thresholds():
    """Params.setDetParams' iouThrs"""
    return np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)


def recall_thresholds():
    """Params.setDetParams' recThrs"""
    return np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)


def collect(image_id, scores, labels, boxes, scale, label_to_coco_label, threshold=0.05):
    """eval.py:280-311 for one image's model output (rows in NMS order) -> list of result dicts"""
    boxes = np.array(boxes, dtype=np.float32).reshape(-1, 4) / np.float32(scale)
    boxes[:, 2] -= boxes[:, 0]
    boxes[:, 3] -= boxes[:, 1]
    out = []
    for i in range(boxes.shape[0]):
        score = float(scores[i])
        if score < threshold:
            break
        out.append({'image_id': image_id, 'category_id': label_to_coco_label(int(labels[i])), 'score': float(score),
                    'bbox': [float(v) for v in boxes[i]]})
    return out


def iou(d, g, iscrowd):
    """maskApi.c bbIou: d [m,4], g [n,4] (x,y,w,h) fp64 -> [m,n]; each operation rounded on its own"""
    o = np.zeros((len(d), len(g)))
    for j, (G, crowd) in enumerate(zip(g, iscrowd)):
        ga = G[2] * G[3]
        for i, D in enumerate(d):
            da = D[2] * D[3]
            w = min(D[2] + D[0], G[2] + G[0]) - max(D[0], G[0])
            if w <= 0:
                continue
            h = min(D[3] + D[1], G[3] + G[1]) - max(D[1], G[1])
            if h <= 0:
                continue
            i_ = w * h
            u = da if crowd else (da + ga) - i_
            o[i, j] = i_ / u
    return o


class COCO:
    """the parts of pycocotools' COCO that evaluate_coco and COCOeval use, over an instances dict"""

    def __init__(self, dataset):
        self.dataset = dataset

    def loadRes(self, res):
        if isinstance(res, str):
            with open(res) as f:
                res = json.load(f)
        anns = copy.deepcopy(res)
        ids = {img['id'] for img in self.dataset['images']}
        assert {a['image_id'] for a in anns} <= ids, 'Results do not correspond to current coco set'
        for i, a in enumerate(anns):
            bb = a['bbox']
            a['area'] = bb[2] * bb[3]
            a['id'] = i + 1
            a['iscrowd'] = 0
        return COCO({'images': self.dataset['images'], 'categories': copy.deepcopy(self.dataset['categories']),
                     'annotations': anns})


class Params:
    def __init__(self, gt):
        self.imgIds = sorted(img['id'] for img in gt.dataset['images'])
        self.catIds = sorted(c['id'] for c in gt.dataset['categories'])
        self.iouThrs = iou_thresholds()
        self.recThrs = recall_thresholds()
        self.maxDets = list(MAX_DETS)
        self.areaRng = [list(a) for a in AREA_RNG]
        self.areaRngLbl = list(AREA_LBL)


def group(anns, img_ids, cat_ids):
    """COCOeval._prepare: per (image, category) the annotations in annotation order"""
    imgs, cats = set(img_ids), set(cat_ids)
    out = {}
    for a in anns:
        if a['image_id'] in imgs and a['category_id'] in cats:
            out.setdefault((a['image_id'], a['category_id']), []).append(a)
    return out


class COCOeval:
    """COCOeval(cocoGt, cocoDt, 'bbox'): evaluate(), accumulate() and summarize() with default Params"""

    def __init__(self, cocoGt, cocoDt, iouType='bbox'):
        assert iouType == 'bbox', iouType
        self.cocoGt, self.cocoDt = cocoGt, cocoDt
        self.params = Params(cocoGt)
        self.eval, self.stats = {}, []

    def evaluate(self):
        p = self.params
        p.imgIds = list(np.unique(p.imgIds))
        p.catIds = list(np.unique(p.catIds))
        self._gts = group(self.cocoGt.dataset['annotations'], p.imgIds, p.catIds)
        self._dts = group(self.cocoDt.dataset['annotations'], p.imgIds, p.catIds)
        self.evalImgs = [self.evaluate_img(i, c, a) for c in p.catIds for a in p.areaRng for i in p.imgIds]

    def evaluate_img(self, img, cat, rng):
        """computeIoU + evaluateImg for maxDet = maxDets[-1]"""
        p = self.params
        gt, dt = self._gts.get((img, cat), []), self._dts.get((img, cat), [])
        if not gt and not dt:
            return None
        dt = [dt[i] for i in np.argsort([-d['score'] for d in dt], kind='mergesort')][:p.maxDets[-1]]
        ious = iou([d['bbox'] for d in dt], [g['bbox'] for g in gt], [int(g['iscrowd']) for g in gt])
        g_ig = [1 if (g.get('iscrowd', 0) or g['area'] < rng[0] or g['area'] > rng[1]) else 0 for g in gt]
        order = np.argsort(g_ig, kind='mergesort')
        gt = [gt[i] for i in order]
        gt_ig = np.array([g_ig[i] for i in order])
        ious = ious[:, order] if len(gt) and len(dt) else ious
        crowd = [int(g['iscrowd']) for g in gt]
        T, G, D = len(p.iouThrs), len(gt), len(dt)
        gtm, dtm, dt_ig = np.zeros((T, G)), np.zeros((T, D)), np.zeros((T, D))
        if G and D:
            for ti, t in enumerate(p.iouThrs):
                for di, d in enumerate(dt):
                    best, m = min([t, 1 - 1e-10]), -1
                    for gi in range(G):
                        if gtm[ti, gi] > 0 and not crowd[gi]:
                            continue
                        if m > -1 and gt_ig[m] == 0 and gt_ig[gi] == 1:
                            break
                        if ious[di, gi] < best:
                            continue
                        best, m = ious[di, gi], gi
                    if m == -1:
                        continue
                    dt_ig[ti, di] = gt_ig[m]
                    dtm[ti, di] = gt[m]['id']
                    gtm[ti, m] = d['id']
        out = np.array([d['area'] < rng[0] or d['area'] > rng[1] for d in dt]).reshape((1, D))
        dt_ig = np.logical_or(dt_ig, np.logical_and(dtm == 0, np.repeat(out, T, 0)))
        return {'dtMatches': dtm, 'dtScores': [d['score'] for d in dt], 'gtIgnore': gt_ig, 'dtIgnore': dt_ig}

    def accumulate(self):
        p = self.params
        T, R, K, A, M = len(p.iouThrs), len(p.recThrs), len(p.catIds), len(p.areaRng), len(p.maxDets)
        precision, recall = -np.ones((T, R, K, A, M)), -np.ones((T, K, A, M))
        I0, A0 = len(p.imgIds), len(p.areaRng)
        for k in range(K):
            for a in range(A):
                for m, max_det in enumerate(p.maxDets):
                    E = [e for e in self.evalImgs[k * A0 * I0 + a * I0:k * A0 * I0 + (a + 1) * I0] if e is not None]
                    if not E:
                        continue
                    scores = np.concatenate([e['dtScores'][0:max_det] for e in E])
                    inds = np.argsort(-scores, kind='mergesort')
                    dtm = np.concatenate([e['dtMatches'][:, 0:max_det] for e in E], axis=1)[:, inds]
                    dt_ig = np.concatenate([e['dtIgnore'][:, 0:max_det] for e in E], axis=1)[:, inds]
                    gt_ig = np.concatenate([e['gtIgnore'] for e in E])
                    npig = np.count_nonzero(gt_ig == 0)
                    if npig == 0:
                        continue
                    tps = np.logical_and(dtm, np.logical_not(dt_ig))
                    fps = np.logical_and(np.logical_not(dtm), np.logical_not(dt_ig))
                    tp_sum = np.cumsum(tps, axis=1).astype(dtype=np.float64)
                    fp_sum = np.cumsum(fps, axis=1).astype(dtype=np.float64)
                    for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                        nd = len(tp)
                        rc = tp / npig
                        pr = (tp / (fp + tp + np.spacing(1))).tolist()
                        recall[t, k, a, m] = rc[-1] if nd else 0
                        for i in range(nd - 1, 0, -1):
                            if pr[i] > pr[i - 1]:
                                pr[i - 1] = pr[i]
                        q = np.zeros((R,))
                        for ri, pi in enumerate(np.searchsorted(rc, p.recThrs, side='left')):
                            if pi >= nd:
                                break
                            q[ri] = pr[pi]
                        precision[t, :, k, a, m] = q
        self.eval = {'precision': precision, 'recall': recall}

    def summarize(self):
        self.stats, self.lines = summarize(self.eval['precision'], self.eval['recall'], self.params.iouThrs)
        for line in self.lines:
            print(line)


def summarize(precision, recall, iou_thrs=None):
    """COCOeval.summarize for bbox -> (stats [12], the 12 printed lines)"""
    iou_thrs = iou_thresholds() if iou_thrs is None else iou_thrs
    fmt = ' {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}'
    lines = []

    def one(ap, thr=None, area='all', max_dets=100):
        a, m = [AREA_LBL.index(area)], [MAX_DETS.index(max_dets)]
        s = precision if ap else recall
        if thr is not None:
            s = s[np.where(thr == iou_thrs)[0]]
        s = s[:, :, :, a, m] if ap else s[:, :, a, m]
        mean = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        thr_s = '{:0.2f}:{:0.2f}'.format(iou_thrs[0], iou_thrs[-1]) if thr is None else '{:0.2f}'.format(thr)
        lines.append(fmt.format('Average Precision' if ap else 'Average Recall', '(AP)' if ap else '(AR)', thr_s, area,
                                max_dets, mean))
        return mean

    stats = np.zeros((12,))
    stats[0] = one(1)
    stats[1] = one(1, .5)
    stats[2] = one(1, .75)
    stats[3] = one(1, area='small')
    stats[4] = one(1, area='medium')
    stats[5] = one(1, area='large')
    stats[6] = one(0, max_dets=1)
    stats[7] = one(0, max_dets=10)
    stats[8] = one(0)
    stats[9] = one(0, area='small')
    stats[10] = one(0, area='medium')
    stats[11] = one(0, area='large')
    return stats, lines


def evaluate(gt_dataset, results, image_ids):
    """eval.py:318-333 on a result list -> (stats, precision, recall)"""
    gt = COCO(gt_dataset)
    E = COCOeval(gt, gt.loadRes(results), 'bbox')
    E.params.imgIds = list(image_ids)
    E.evaluate()
    E.accumulate()
    stats, _ = summarize(E.eval['precision'], E.eval['recall'], E.params.iouThrs)
    return stats, E.eval['precision'], E.eval['recall']
