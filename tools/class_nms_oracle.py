"""Class-aware NMS in NumPy: the restatement csrc/detect.cu's per-class and multi-label paths are held to bit for bit.

    per-class hard NMS   for every class c, oracle/effdet_oracle.py::nms_greedy (torchvision's CPU nms: stable
                         descending sort, fp32 IoU, suppress iff IoU > thr) on that class's candidates in index order;
                         the keep sets merged in (score desc, index asc) order.  The keep sets are torchvision 0.26's
                         _batched_nms_vanilla; its final sort is not stable, so on ties this order is the stable one.
    per-class Soft-NMS   tools/soft_nms_oracle.py::soft_nms run class by class; a pick decays only its own class, so
                         the global pick order is the merge of the per-class pick lists by (score at the pick desc,
                         index asc).
    multi-label top-k    every (anchor a, class k) pair with cls[a, k] > threshold, p = a*K + k, ordered by the key
                         (~order(score) << 32) | p -- score descending, p ascending -- and cut to the first top_k;
                         slot i is the i-th pair, and slots stand for anchors in the per-class NMS that follows.

tests/test_class_nms.py holds this against tests/golden/class_nms.npz (written with torchvision by
tests/golden/make_class_nms_golden.py) on the CPU and the device against this on the GPU.
"""
import os
import sys

import numpy as np
import torch

_HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(_HERE), 'oracle'))
sys.path.insert(0, _HERE)
import effdet_oracle as O  # noqa: E402
import soft_nms_oracle as S  # noqa: E402

MODES = ('agnostic', 'per_class', 'multi_label')


def _merge(idx, scores):
    """idx (distinct ints) in (score desc, idx asc) order"""
    idx = np.asarray(idx, np.int64)
    if idx.size == 0:
        return idx
    return idx[np.lexsort((idx, -np.asarray(scores, np.float32)[idx]))]


def per_class_nms(boxes, scores, classes, iou_threshold):
    """boxes [n,4], scores [n] float32, classes [n] -> kept indices int64 in (score desc, index asc) order"""
    boxes = np.asarray(boxes, np.float32).reshape(-1, 4)
    scores = np.asarray(scores, np.float32).reshape(-1)
    classes = np.asarray(classes).reshape(-1)
    keep = []
    for c in np.unique(classes):
        idx = np.flatnonzero(classes == c)
        k = O.nms_greedy(torch.from_numpy(boxes[idx]), torch.from_numpy(scores[idx]), iou_threshold).numpy()
        keep.append(idx[k])
    return _merge(np.concatenate(keep) if keep else np.zeros(0, np.int64), scores)


def per_class_soft_nms(boxes, scores, classes, anchors, method, iou_threshold=0.5, sigma=0.5, threshold=0.0):
    """Soft-NMS within each class -> (picked anchors int64, their scores at the pick float32), in global pick order"""
    boxes = np.asarray(boxes, np.float32).reshape(-1, 4)
    scores = np.asarray(scores, np.float32).reshape(-1)
    classes, anchors = np.asarray(classes).reshape(-1), np.asarray(anchors, np.int64).reshape(-1)
    pa, ps = [], []
    for c in np.unique(classes):
        i = np.flatnonzero(classes == c)
        a, s = S.soft_nms(boxes[i], scores[i], anchors[i], method, iou_threshold, sigma, threshold)
        pa.append(a)
        ps.append(s)
    if not pa:
        return np.zeros(0, np.int64), np.zeros(0, np.float32)
    pa, ps = np.concatenate(pa), np.concatenate(ps)
    order = np.lexsort((pa, -ps))
    return pa[order], ps[order]


def pair_keys(cls_b):
    """cls_b [A,K] float32 -> uint64 keys (~order(score) << 32) | p of every pair, p = a*K + k"""
    v = np.asarray(cls_b, np.float32).reshape(-1).view(np.uint32)
    order = np.where(v & np.uint32(0x80000000), ~v, v | np.uint32(0x80000000))
    return ((~order).astype(np.uint64) << np.uint64(32)) | np.arange(v.size, dtype=np.uint64)


def topk_pairs(cls_b, threshold, top_k):
    """the multi-label selection of one image: pair indices p of the best min(top_k, pairs above threshold) pairs,
    in (score desc, p asc) order"""
    flat = np.asarray(cls_b, np.float32).reshape(-1)
    keys = pair_keys(cls_b)[flat > np.float32(threshold)]
    return (np.sort(keys)[:top_k] & np.uint64(0xffffffff)).astype(np.int64)


def candidates(cand, b, mode, threshold, top_k, cls=None):
    """image b's candidates in slot order -> (boxes [n,4], scores [n], classes [n], index [n]).
    cand: NumPy (boxes [B,A,4], scores [B,A], classes [B,A], count [B], keys [B,npad]) as
    effdet_detect_candidates_batch writes them; the decoded box of every anchor is used for its pairs as well.
    agnostic / per_class: the anchors above the threshold, index = anchor.  multi_label (cls [B,A,K] needed): the
    top-k pairs, index = slot (their rank)."""
    boxes, scores, classes, count, keys = cand
    if mode != 'multi_label':
        a = np.asarray(keys[b][:int(count[b])]).astype(np.int64) & 0xffffffff
        return boxes[b][a], scores[b][a], classes[b][a], a
    K = cls.shape[2]
    p = topk_pairs(cls[b], threshold, top_k)
    a = p // K
    return boxes[b][a], np.asarray(cls[b], np.float32).reshape(-1)[p], (p % K).astype(np.int32), np.arange(len(p))


def detect(cand, b, mode, nms, threshold, iou_threshold, sigma=0.5, top_k=5000, cls=None):
    """the detections of image b -> (scores float32, classes int64, boxes [n,4] float32) in output order"""
    bx, sc, cl, idx = candidates(cand, b, mode, threshold, top_k, cls)
    if nms == 'hard':
        if mode == 'agnostic':
            k = O.nms_greedy(torch.from_numpy(np.ascontiguousarray(bx)), torch.from_numpy(np.ascontiguousarray(sc)),
                             iou_threshold).numpy()
        else:
            k = per_class_nms(bx, sc, cl, iou_threshold)
        return sc[k].astype(np.float32), cl[k].astype(np.int64), bx[k].astype(np.float32)
    if mode == 'agnostic':
        pa, ps = S.soft_nms(bx, sc, idx, nms, iou_threshold, sigma, threshold)
    else:
        pa, ps = per_class_soft_nms(bx, sc, cl, idx, nms, iou_threshold, sigma, threshold)
    pos = {int(v): i for i, v in enumerate(idx)}
    k = np.asarray([pos[int(v)] for v in pa], np.int64)
    return ps, cl[k].astype(np.int64) if len(k) else np.zeros(0, np.int64), bx[k].reshape(-1, 4).astype(np.float32)


def random_class_candidates(seed, n, K, size=512.0, clusters=24, threshold=0.05, ties=0.2):
    """n seeded candidates of K classes: soft_nms_oracle.random_candidates' boxes and scores (many overlaps, a fraction
    `ties` of repeated scores) with seeded classes -> (boxes [n,4] float32, scores [n] float32, classes [n] int32)"""
    boxes, scores, _ = S.random_candidates(seed, n, size=size, clusters=clusters, threshold=threshold, ties=ties)
    classes = np.random.default_rng(seed + 7919).integers(0, K, n).astype(np.int32)
    return boxes, scores, classes
