"""Soft-NMS (Bodla et al., Soft-NMS -- Improving Object Detection With One Line of Code, ICCV 2017, Algorithm 1) in
NumPy, vectorised over the live candidates of each pick, with the arithmetic pinned so that the device
(csrc/soft_nms.cu, effdet_soft_nms_batch) and this restatement agree bit for bit:

    live = all candidates, s = their scores (float32)
    while live is not empty:
        m = argmax over live of s                      ties: lower anchor index
        emit (m, s[m]); remove m from live
        for j in live:
            ov = IoU(box[m], box[j])                   float32, each operation rounded on its own (no FMA);
                                                       an intersection of 0 gives ov = 0 with no division
            linear:   w = 1 - ov if float64(ov) > iou_threshold else 1
            gaussian: w = float32(exp(-(float64(ov) * ov) / sigma))            float64, rounded once
            s[j] = float32(s[j] * w)
            if not s[j] > threshold: remove j from live

tests/test_soft_nms.py holds this against a literal one-candidate-at-a-time transcription of the loop above and the
device against this, and tests/golden/make_soft_nms_golden.py pins the fixture's results.
"""
import numpy as np

METHODS = ('linear', 'gaussian')


def iou(box, boxes):
    """float32 IoU of one box [4] with boxes [n, 4]: csrc/detect.cu iou_gt's operations, 0 where the intersection is 0"""
    box = np.asarray(box, np.float32)
    boxes = np.asarray(boxes, np.float32).reshape(-1, 4)
    zero = np.float32(0)
    width = np.maximum(np.minimum(box[2], boxes[:, 2]) - np.maximum(box[0], boxes[:, 0]), zero)
    height = np.maximum(np.minimum(box[3], boxes[:, 3]) - np.maximum(box[1], boxes[:, 1]), zero)
    inter = width * height
    sa = (box[2] - box[0]) * (box[3] - box[1])
    sb = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1])
    hit = inter != 0
    ov = np.zeros(len(boxes), np.float32)
    ov[hit] = inter[hit] / ((sa + sb[hit]) - inter[hit])
    return ov


def gaussian_double(ov, sigma):
    """the float64 value the Gaussian weight is rounded from"""
    o = np.asarray(ov, np.float32).astype(np.float64)
    return np.exp(-(o * o) / np.float64(sigma))


def weights(ov, method, iou_threshold, sigma):
    """float32 decay weights of IoUs ov [n]"""
    ov = np.asarray(ov, np.float32)
    if method == 'linear':
        return np.where(ov.astype(np.float64) > iou_threshold, np.float32(1) - ov, np.float32(1)).astype(np.float32)
    if method == 'gaussian':
        return gaussian_double(ov, sigma).astype(np.float32)
    raise ValueError('method must be one of %s' % (METHODS,))


def rounding_margin(ov, sigma):
    """smallest distance, in float64 ulps, from a Gaussian weight's float64 value to the nearest point where its float32
    rounding changes (the midpoint to a neighbouring float32), over the IoUs ov > 0.  A float64 exp that is off by one
    ulp changes the float32 weight only where this is below 1.  inf when there is no ov > 0."""
    ov = np.asarray(ov, np.float32)
    ov = ov[ov > 0]
    if ov.size == 0:
        return np.inf
    e = gaussian_double(ov, sigma)
    f = e.astype(np.float32)
    up = np.nextafter(f, np.float32(np.inf)).astype(np.float64)
    down = np.nextafter(f, np.float32(-np.inf)).astype(np.float64)
    fd = f.astype(np.float64)
    dist = np.minimum(np.abs(e - (fd + up) / 2), np.abs(e - (fd + down) / 2))
    return float(np.min(dist / np.spacing(e)))


def soft_nms(boxes, scores, anchors, method, iou_threshold=0.5, sigma=0.5, threshold=0.0, margin=None):
    """boxes [n,4], scores [n] float32 (the candidates, every score > threshold), anchors [n] distinct int
    -> (picked anchors int64 [k], their scores at the pick float32 [k]), in pick order.
    margin: a list that receives rounding_margin of every pick's Gaussian weights (for the fixture script)."""
    boxes = np.asarray(boxes, np.float32).reshape(-1, 4)
    s = np.array(scores, np.float32).reshape(-1)
    anchors = np.asarray(anchors, np.int64).reshape(-1)
    thr = np.float32(threshold)
    live = np.flatnonzero(s > thr)
    out_a, out_s = [], []
    while live.size:
        top = s[live].max()
        tied = live[s[live] == top]
        m = tied[np.argmin(anchors[tied])]
        out_a.append(anchors[m])
        out_s.append(s[m])
        live = live[live != m]
        if not live.size:
            break
        ov = iou(boxes[m], boxes[live])
        if margin is not None and method == 'gaussian':
            margin.append(rounding_margin(ov, sigma))
        s[live] = s[live] * weights(ov, method, iou_threshold, sigma)
        live = live[s[live] > thr]
    return np.asarray(out_a, np.int64), np.asarray(out_s, np.float32)


def soft_nms_candidates(boxes, scores, classes, count, keys, b, method, iou_threshold, sigma, threshold):
    """Soft-NMS of image b of effdet_detect_candidates_batch's outputs (NumPy arrays boxes [B,A,4], scores [B,A],
    classes [B,A], count [B], keys [B,npad]) -> (scores [k], classes [k] int64, boxes [k,4], anchors [k])"""
    n = int(count[b])
    idx = np.asarray(keys[b][:n]).astype(np.int64) & 0xffffffff
    a, s = soft_nms(boxes[b][idx], scores[b][idx], idx, method, iou_threshold, sigma, threshold)
    return s, np.asarray(classes[b][a], np.int64), np.asarray(boxes[b][a], np.float32), a


def random_candidates(seed, n, size=512.0, clusters=24, threshold=0.05, ties=0.2):
    """n seeded candidates: boxes around a few cluster centres (so that many pairs overlap), scores in
    (threshold, 1) with a fraction `ties` repeating earlier scores, distinct anchors in [0, 4n) -> (boxes [n,4]
    float32, scores [n] float32, anchors [n] int64)"""
    rng = np.random.default_rng(seed)
    centres = rng.uniform(0, size, (max(1, clusters), 2))
    c = centres[rng.integers(0, len(centres), n)] + rng.normal(0, size / 40, (n, 2))
    wh = rng.uniform(size / 64, size / 8, (n, 2))
    boxes = np.concatenate([c - wh / 2, c + wh / 2], axis=1).clip(0, size).astype(np.float32)
    scores = rng.uniform(threshold, 1.0, n).astype(np.float32)
    scores[scores <= np.float32(threshold)] = np.float32(0.5)
    rep = rng.random(n) < ties
    if n > 1:
        scores[rep] = scores[rng.integers(0, n, int(rep.sum()))]
    anchors = rng.permutation(4 * max(n, 1))[:n].astype(np.int64)
    return boxes, scores, anchors
