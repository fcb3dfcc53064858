"""CPU float64 restatement of the reference's VOC evaluation (eval.py:165-257), written fresh in NumPy.  Tests and
tools/bench_eval.py compare the device path (csrc/voc_eval.cu, models/evaluation.py) against it; it is pinned to the
reference's own code by tests/golden/make_eval_golden.py -> tests/golden/voc_eval.npz.

One deliberate difference: records of a class are sorted with a STABLE argsort (ties keep the append order: image, then
rank inside the image).  The reference calls np.argsort(-scores) with the default introsort, whose order among equal
scores is a NumPy implementation detail; on tie-free scores the two agree exactly.

  get_detections   eval.py:76-136, driving model(image) one image at a time (selection as in select_detections)
  get_annotations  eval.py:139-162
  evaluate         eval.py:185-257 on those lists -> (mean AP, {label: (AP, num_annotations)})
  pairwise_sum     the summation order of np.sum on a contiguous float64 array (the AP kernel follows it)
"""
import numpy as np

EPS = np.finfo(np.float64).eps


def select_detections(scores, labels, boxes, scale, score_threshold, max_detections, num_classes):
    """eval.py:107-133 for one image -> list over labels of [k,5] float64 (x1,y1,x2,y2,score); stable on ties"""
    boxes = np.asarray(boxes, dtype=np.float32).copy()
    boxes /= scale
    keep = np.where(scores > score_threshold)[0]
    if keep.shape[0] == 0:
        return [np.zeros((0, 5)) for _ in range(num_classes)]
    order = keep[np.argsort(-scores[keep], kind='stable')[:max_detections]]
    det = np.concatenate([boxes[order], scores[order][:, None], labels[order][:, None]], axis=1)
    return [det[det[:, -1] == c, :-1] for c in range(num_classes)]


def get_detections(generator, model, score_threshold=0.05, max_detections=100):
    """the reference's batch-1 loop: one forward per image, three host reads, host selection"""
    import torch
    out = []
    with torch.no_grad():
        for i in range(len(generator)):
            data = generator[i]
            scores, labels, boxes = model(data['img'].permute(2, 0, 1).cuda().float().unsqueeze(dim=0))
            out.append(select_detections(scores.cpu().numpy(), labels.cpu().numpy(), boxes.cpu().numpy(), data['scale'],
                                         score_threshold, max_detections, generator.num_classes()))
    return out


def get_annotations(generator):
    K = generator.num_classes()
    out = []
    for i in range(len(generator)):
        a = generator.load_annotations(i)
        out.append([a[a[:, 4] == c, :4].copy() for c in range(K)])
    return out


def overlaps(d, g):
    """IoU of detections d [k,>=4] against ground truth g [n,4], compute_overlap's operation order"""
    area_g = (g[:, 2] - g[:, 0]) * (g[:, 3] - g[:, 1])
    iw = np.maximum(np.minimum(d[:, 2:3], g[:, 2]) - np.maximum(d[:, 0:1], g[:, 0]), 0)
    ih = np.maximum(np.minimum(d[:, 3:4], g[:, 3]) - np.maximum(d[:, 1:2], g[:, 1]), 0)
    ua = np.maximum(((d[:, 2] - d[:, 0]) * (d[:, 3] - d[:, 1]))[:, None] + area_g - iw * ih, EPS)
    return (iw * ih) / ua


def match(dets, gts, iou_threshold):
    """greedy TP flags of one (image, class): dets in their order, the first best ground truth, each taken once"""
    tp = np.zeros(dets.shape[0])
    if gts.shape[0] == 0 or dets.shape[0] == 0:
        return tp
    ov = overlaps(dets, gts)
    taken = set()
    for k in range(dets.shape[0]):
        j = int(np.argmax(ov[k]))
        if ov[k, j] >= iou_threshold and j not in taken:
            tp[k] = 1
            taken.add(j)
    return tp


def average_precision(scores, tp, num_annotations):
    flags = tp[np.argsort(-scores, kind='stable')]
    tp = np.cumsum(flags)
    fp = np.cumsum(1 - flags)
    recall = tp / num_annotations
    precision = tp / np.maximum(tp + fp, EPS)
    mrec = np.concatenate(([0.], recall, [1.]))
    mpre = np.concatenate(([0.], precision, [0.]))
    mpre = np.maximum.accumulate(mpre[::-1])[::-1]
    i = np.where(mrec[1:] != mrec[:-1])[0]
    return np.sum((mrec[i + 1] - mrec[i]) * mpre[i + 1])


def evaluate(all_detections, all_annotations, num_classes, iou_threshold=0.5):
    """eval.py:191-257 without the prints -> (np.mean of the APs, {label: (AP, num_annotations)})"""
    aps = {}
    for c in range(num_classes):
        scores, tps, n_ann = [], [], 0.0
        for dets, anns in zip(all_detections, all_annotations):
            n_ann += anns[c].shape[0]
            scores.append(dets[c][:, 4])
            tps.append(match(dets[c], anns[c], iou_threshold))
        if n_ann == 0:
            aps[c] = 0, 0
            continue
        aps[c] = average_precision(np.concatenate(scores), np.concatenate(tps), n_ann), n_ann
    return np.mean([aps[c][0] for c in range(num_classes)]), aps


def pairwise_sum(a):
    """np.sum of a contiguous float64 array, as numpy's pairwise_sum adds it: below 8 elements left to right; up to
    128 elements eight running sums over whole blocks of 8, combined ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the tail
    left to right; above 128 the halves split at n/2 rounded down to a multiple of 8, each summed the same way."""
    a = np.asarray(a, dtype=np.float64)
    n = a.shape[0]
    if n < 8:
        r = np.float64(-0.0)
        for v in a:
            r = r + v
        return r
    if n <= 128:
        r = a[:8].copy()
        i = 8
        while i < n - n % 8:
            r = r + a[i:i + 8]
            i += 8
        res = ((r[0] + r[1]) + (r[2] + r[3])) + ((r[4] + r[5]) + (r[6] + r[7]))
        for v in a[i:]:
            res = res + v
        return res
    h = n // 2
    h -= h % 8
    return pairwise_sum(a[:h]) + pairwise_sum(a[h:])
