"""VOC mean average precision on the device: eval.py::evaluate (eval.py:165-257) over csrc/voc_eval.cu.

    acc = VOCAccumulator(num_classes, num_images)
    for each batch:  acc.add(detections, scales, annotations)     # launches only: no host read, capturable
    mean_ap, aps = acc.compute()                                   # the one read -> what eval.py::evaluate returns

`evaluate(generator, model)` is a drop-in for eval.py::evaluate that runs the network in batches through a
GraphedDetect and accumulates on the device; it prints and returns what the reference does.

Records of one class with equal scores are ordered by image, then by rank inside the image: the order a stable sort of
the reference's append order gives (the reference's np.argsort leaves ties to NumPy's introsort).  On tie-free scores
the results equal the reference's float64 values exactly.

`evaluate_coco(dataset, model)` is the same for eval.py::evaluate_coco over csrc/coco_eval.cu: COCOAccumulator runs
pycocotools' COCOeval (bbox, default Params) on the device and needs neither pycocotools nor a host read per batch.
"""
import json

import numpy as np
import torch

from . import _native as N
from . import _ops
from . import pipeline
from .graph_step import GraphedDetect, GraphedRawDetect

# candidate rows per image that the graphed detection keeps before NMS: None = every anchor, so no image overflows; with
# an integer, an image with more candidates is redone eagerly
MAX_CANDIDATES = None


class VOCAccumulator:
    """Device-side state of one VOC evaluation over `num_images` images, filled batch by batch in image order.

    Every image owns `max_detections` record slots, so the buffers are sized at construction and add() needs no count
    from the device.  add() uploads the batch's ground truth from pinned memory and launches the selection and the
    matching; compute() launches the AP and reads the result back once."""

    def __init__(self, num_classes, num_images, iou_threshold=0.5, score_threshold=0.05, max_detections=100,
                 device='cuda:0'):
        self.K, self.num_images, self.max_det = int(num_classes), int(num_images), int(max_detections)
        self.iou_threshold, self.score_threshold = float(iou_threshold), float(score_threshold)
        self.device = torch.device(device)
        R = self.num_images * self.max_det
        ws = int(N.load().effdet_voc_ap_workspace(R, self.K))
        if ws < 0:
            raise N.EffdetNativeError('VOCAccumulator: %s' % N.last_error())
        dev = self.device
        self.dets = torch.zeros((R, 5), device=dev, dtype=torch.float32)
        self.labels = torch.full((R,), -1, device=dev, dtype=torch.int32)
        self.tp = torch.zeros((R,), device=dev, dtype=torch.uint8)
        self.overflow = torch.zeros((self.num_images,), device=dev, dtype=torch.int32)
        self.gt_count = torch.zeros((self.K,), device=dev, dtype=torch.int64)
        self.workspace = torch.empty((ws,), device=dev, dtype=torch.uint8)
        self.result = torch.empty((2 * self.K,), device=dev, dtype=torch.float64)
        self.images = 0                       # images added so far: the next batch's first image
        self._staged = None                   # pinned host copies of the last batch (captured copies read them)

    def add(self, detections, scales, annotations):
        """detections: _ops.Detections of B images (scores [B,C], classes [B,C] int64, boxes [B,C,4], count [B] int32,
        -1 = NMS overflow), as GraphedDetect / _ops.detect_batch(..., cap=C) return them; scales: B per-image box
        scales (eval.py's data['scale']); annotations: B float64 arrays [n,5] (x1,y1,x2,y2,label) in original image
        coordinates, as generator.load_annotations returns them."""
        scores, classes, boxes, count = detections
        B, C = scores.shape
        if self.images + B > self.num_images:
            raise N.EffdetNativeError('VOCAccumulator: %d images added to %d, but it was built for %d'
                                      % (B, self.images, self.num_images))
        if len(annotations) != B or len(scales) != B:
            raise N.EffdetNativeError('VOCAccumulator.add: %d images, %d annotation arrays and %d scales'
                                      % (B, len(annotations), len(scales)))
        anns = [np.asarray(a, dtype=np.float64).reshape(-1, 5) for a in annotations]
        counts = np.array([a.shape[0] for a in anns], dtype=np.int64)
        offs = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
        num_gt = int(offs[-1])
        rows = np.concatenate(anns, axis=0) if num_gt else np.zeros((1, 5))
        host = [torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
                for a in (rows, offs, np.asarray(scales, dtype=np.float32).reshape(B))]
        self._staged = host
        rows_d, offs_d, scale_d = (t.to(self.device, non_blocking=True) for t in host)
        class_off = torch.empty((B, self.K + 1), device=self.device, dtype=torch.int32)
        r0 = self.images * self.max_det
        dets, labels = self.dets[r0:], self.labels[r0:]
        N.call('effdet_eval_select_batch', scores, N.f32(scores.contiguous(), 'scores'), N.ptr(classes.contiguous()),
               N.f32(boxes.contiguous(), 'boxes'), N.ptr(count.contiguous()), N.ptr(scale_d), B, C,
               self.score_threshold, self.max_det, self.K, N.ptr(dets), N.ptr(labels), N.ptr(class_off),
               N.ptr(self.overflow[self.images:]))
        N.call('effdet_voc_match', scores, N.ptr(dets), N.ptr(class_off), N.ptr(rows_d), N.ptr(offs_d), num_gt, B,
               self.max_det, self.K, self.iou_threshold, N.ptr(self.tp[r0:]), N.ptr(self.gt_count))
        self.images += B

    def compute(self):
        """-> (mean AP, {label: (AP, num_annotations)}) exactly as eval.py::evaluate returns them: (0, 0) for a label
        without ground truth.  The mean is np.mean over the labels' APs, on the host, as the reference takes it."""
        K = self.K
        N.call('effdet_voc_ap', self.dets, N.ptr(self.dets), N.ptr(self.labels), N.ptr(self.tp), N.ptr(self.gt_count),
               self.num_images * self.max_det, K, N.ptr(self.result), N.ptr(self.result[K:]), N.ptr(self.workspace),
               self.workspace.numel())
        host = torch.cat([self.result, self.overflow.double()]).cpu().numpy()        # the one device->host read
        bad = np.nonzero(host[2 * K:])[0]
        if bad.size:
            raise N.EffdetNativeError('VOCAccumulator: images %s overflowed NMS (more candidates than the detection '
                                      'was built for); redo them eagerly before add()' % bad.tolist())
        aps = {}
        for c in range(K):
            aps[c] = (0, 0) if host[K + c] == 0 else (np.float64(host[c]), float(host[K + c]))
        return np.mean([aps[c][0] for c in range(K)]), aps


def _padded(trip):
    """one eager detection triple -> Detections of one image"""
    s, c, b = trip
    n = s.numel()
    if n == 0:
        s, c, b = s.new_zeros(1), torch.zeros(1, dtype=torch.int64, device=s.device), s.new_zeros(1, 4)
    count = torch.full((1,), n, dtype=torch.int32, device=s.device)
    return _ops.Detections(s.reshape(1, -1).contiguous(), c.reshape(1, -1).contiguous(), b.reshape(1, -1, 4).contiguous(),
                           count)


def _add_batch(acc, out, cls, reg, anchors, hw, model, scales, *per_image):
    """adds the padded detections of one batch to acc (a VOCAccumulator or a COCOAccumulator: acc.add(detections,
    scales, *per_image)); images that overflowed NMS are redone eagerly from the network outputs (one [B] int32 read)
    and added one by one, in image order"""
    counts = out.count.tolist()
    b0 = 0
    for b, m in enumerate(counts + [None]):
        if m is not None and m >= 0:
            continue
        if b > b0:
            acc.add(_ops.Detections(*(t[b0:b] for t in out)), scales[b0:b], *(p[b0:b] for p in per_image))
        if m is None:
            break
        trip = _ops.detect_batch(cls[b:b + 1], reg[b:b + 1], anchors, hw[0], hw[1], **model.postprocess())[0]
        acc.add(_padded(trip), scales[b:b + 1], *(p[b:b + 1] for p in per_image))
        b0 = b + 1


def _detect_raw(dataset, model, acc, batch_size, per_image, progress_base, collater, num_workers):
    """_detect_all for a dataset of decoded samples: a DataLoader with collate_fn=collater (a RawCollater) yields raw
    batches, full batches replay one GraphedRawDetect (the Resizer chain runs at the head of its graph), and the
    remainder runs eagerly.  A batch whose bytes do not fit the graph rebuilds it with at least twice the capacity."""
    loader = torch.utils.data.DataLoader(dataset, batch_size=batch_size, shuffle=False, num_workers=num_workers,
                                         collate_fn=collater, pin_memory=True)
    n = len(dataset)
    dev = next(model.parameters()).device
    graphed = None
    i0 = 0
    with torch.no_grad():
        for raw in loader:
            idx = range(i0, i0 + raw.B)
            i0 += raw.B
            hw = raw.S, raw.S
            if raw.B == batch_size:
                if graphed is not None and raw.data_bytes > graphed.max_bytes:
                    need = max(2 * graphed.max_bytes, raw.data_bytes)
                    # inference graphs hold no state: rebuild, after dropping every reference into the old graph's
                    # pool (its outputs from the previous batch included), so the two pools are not held together
                    out = cls = reg = anchors = graphed = None
                    graphed = GraphedRawDetect(model, raw, max_bytes=need, max_candidates=MAX_CANDIDATES)
                if graphed is None:
                    graphed = GraphedRawDetect(model, raw, max_candidates=MAX_CANDIDATES)
                out, scales = graphed(raw)
                cls, reg, anchors = graphed.cls, graphed.reg, graphed.anchors
            else:
                images = pipeline.raw_images(raw, dev)
                cls, reg, anchors = model._raw_predictions(images)
                out = _ops.detect_batch(cls, reg, anchors, hw[0], hw[1], cap=_ops.candidate_cap(MAX_CANDIDATES, cls),
                                        **model.postprocess())
                scales = raw.scales
            _add_batch(acc, out, cls, reg, anchors, hw, model, scales, *per_image(idx))
            for i in idx:
                print('{}/{}'.format(i + progress_base, n), end='\r')


def _detect_all(dataset, model, acc, batch_size, per_image, progress_base, collater=None, num_workers=0):
    """runs the network over the whole dataset, batch_size images per pass (full batches replay one GraphedDetect, the
    remainder runs eagerly), and adds every batch to acc in image order.  per_image(indices) -> the lists acc.add()
    takes after the scales; progress_base: the number the progress line shows for image 0.  With a collater, the
    dataset yields decoded samples and _detect_raw runs instead."""
    if collater is not None:
        return _detect_raw(dataset, model, acc, batch_size, per_image, progress_base, collater, num_workers)
    n = len(dataset)
    dev = next(model.parameters()).device
    graphed = None
    with torch.no_grad():
        for i0 in range(0, n, batch_size):
            idx = range(i0, min(n, i0 + batch_size))
            data = [dataset[i] for i in idx]
            images = torch.stack([d['img'].permute(2, 0, 1).to(dev).float() for d in data])
            hw = images.shape[2], images.shape[3]
            if len(idx) == batch_size:
                if graphed is None:
                    graphed = GraphedDetect(model, images, max_candidates=MAX_CANDIDATES)
                out = graphed(images)
                cls, reg, anchors = graphed.cls, graphed.reg, graphed.anchors
            else:
                cls, reg, anchors = model._raw_predictions(images)
                out = _ops.detect_batch(cls, reg, anchors, hw[0], hw[1], cap=_ops.candidate_cap(MAX_CANDIDATES, cls),
                                        **model.postprocess())
            _add_batch(acc, out, cls, reg, anchors, hw, model, [d['scale'] for d in data], *per_image(idx))
            for i in idx:
                print('{}/{}'.format(i + progress_base, n), end='\r')


def _refuse_jitter(collater, what):
    if getattr(collater, 'scale_jitter', None) is not None:
        raise N.EffdetNativeError('%s: the collater has scale_jitter=%r, but evaluation never jitters; pass a '
                                  'RawCollater without scale_jitter' % (what, collater.scale_jitter))


def _refuse_training(model, what):
    if model.training or model.is_training:
        raise N.EffdetNativeError('%s needs a model in inference mode (model.eval() and model.is_training = False)'
                                  % what)


def evaluate(generator, retinanet, iou_threshold=0.5, score_threshold=0.05, max_detections=100, save_path=None,
             batch_size=16, collater=None, num_workers=0):
    """Drop-in for eval.py::evaluate (eval.py:165-257): the same generator interface (`generator[i]` -> {'img' [H,W,3],
    'scale'}, load_annotations, num_classes, label_to_name, len), the same prints and return value.  The network runs
    `batch_size` images per pass (full batches replay one GraphedDetect, the remainder runs eagerly), and selection,
    matching and AP run on the device.  save_path is accepted and unused, as in the reference.

    collater=pipeline.RawCollater(pixel_scale=255): `generator[i]` yields decoded samples ({'img': uint8 [h,w,3],
    'annot'}, as DeviceCollater takes them) instead; a DataLoader(generator, batch_size, num_workers=num_workers,
    collate_fn=collater, pin_memory=True) batches them and the Resizer chain runs on the device, bit-identical to the
    host chain, inside a GraphedRawDetect.  Ground truth still comes from generator.load_annotations.  A collater with
    scale_jitter is refused."""
    _refuse_jitter(collater, 'evaluate')
    _refuse_training(retinanet, 'evaluate')
    n, K = len(generator), generator.num_classes()
    dev = next(retinanet.parameters()).device
    acc = VOCAccumulator(K, n, iou_threshold, score_threshold, max_detections, device=dev)
    _detect_all(generator, retinanet, acc, batch_size, lambda idx: [[generator.load_annotations(i) for i in idx]], 1,
                collater, num_workers)
    mean_ap, aps = acc.compute()
    print('\nmAP:')
    for label in range(K):
        print('{}: {}'.format(generator.label_to_name(label), aps[label][0]))
    print('avg mAP: {}'.format(mean_ap))
    return mean_ap, aps


# ---- COCO ------------------------------------------------------------------------------------------------------------
COCO_AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
COCO_AREA_LBL = ['all', 'small', 'medium', 'large']
COCO_MAX_DETS = [1, 10, 100]
COCO_MAX_GT = 256                      # ground truths of one (image, category) the matching kernel holds
COCO_MAX_RECORDS = 1 << 25
COCO_BBOX = 1                          # EFFDET_COCO_BBOX


def coco_iou_thresholds():
    """pycocotools Params.iouThrs, computed as setDetParams computes it"""
    return np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)


def coco_recall_thresholds():
    """pycocotools Params.recThrs, computed as setDetParams computes it"""
    return np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)


def coco_summarize(precision, recall):
    """COCOeval.summarize for bbox on precision [10,101,K,4,3] and recall [10,K,4,3] -> (stats [12], the 12 lines it
    prints): the mean over the entries > -1 of each slice, -1 for an empty slice"""
    thrs = coco_iou_thresholds()
    fmt = ' {:<18} {} @[ IoU={:<9} | area={:>6s} | maxDets={:>3d} ] = {:0.3f}'
    spec = [(1, None, 'all', 100), (1, .5, 'all', 100), (1, .75, 'all', 100), (1, None, 'small', 100),
            (1, None, 'medium', 100), (1, None, 'large', 100), (0, None, 'all', 1), (0, None, 'all', 10),
            (0, None, 'all', 100), (0, None, 'small', 100), (0, None, 'medium', 100), (0, None, 'large', 100)]
    stats, lines = np.zeros((12,)), []
    for n, (ap, thr, area, max_dets) in enumerate(spec):
        a, m = [COCO_AREA_LBL.index(area)], [COCO_MAX_DETS.index(max_dets)]
        s = precision if ap else recall
        if thr is not None:
            s = s[np.where(thr == thrs)[0]]
        s = s[:, :, :, a, m] if ap else s[:, :, a, m]
        stats[n] = -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
        iou = '{:0.2f}:{:0.2f}'.format(thrs[0], thrs[-1]) if thr is None else '{:0.2f}'.format(thr)
        lines.append(fmt.format('Average Precision' if ap else 'Average Recall', '(AP)' if ap else '(AR)', iou, area,
                                max_dets, stats[n]))
    return stats, lines


class COCOAccumulator:
    """Device-side state of one COCO box evaluation (pycocotools COCOeval, iouType 'bbox', default Params) over the
    images `image_ids`, filled batch by batch in that (dataset) order.

        acc = COCOAccumulator(dataset.coco, dataset.image_ids, dataset.label_to_coco_label)
        for each batch:  acc.add(detections, scales)     # launches only: no host read, capturable
        stats, precision, recall = acc.compute()          # the one read
        results = acc.results()                           # the detection list eval.py writes (one more read)

    ground_truth: an instances dict, or an object with .dataset (pycocotools' COCO).  Its ground truth is grouped by
    (image, category) in annotation order and uploaded once; crowd annotations and annotations of any size are kept, as
    COCOeval keeps them.  label_to_category: model label -> category id (a callable, a dict or a sequence), for labels
    0 .. num_labels-1 (default: one label per ground-truth category).  A record is one detection with score >=
    score_threshold; the record buffer holds max_records (default 1000 per image), and compute() says what would have
    been enough when it runs out."""

    def __init__(self, ground_truth, image_ids, label_to_category, num_labels=None, score_threshold=0.05,
                 max_records=None, device='cuda:0'):
        gt = ground_truth.dataset if hasattr(ground_truth, 'dataset') else ground_truth
        self.image_ids = list(image_ids)
        if len(set(self.image_ids)) != len(self.image_ids):
            raise N.EffdetNativeError('COCOAccumulator: image_ids has duplicates')
        self.ids_by_rank = sorted(self.image_ids)                     # COCOeval's imgIds: np.unique
        self.cat_ids = sorted(c['id'] for c in gt['categories'])      # COCOeval's catIds
        self.K, self.num_images = len(self.cat_ids), len(self.image_ids)
        self.label_to_category = label_to_category if callable(label_to_category) else label_to_category.__getitem__
        self.num_labels = int(num_labels) if num_labels is not None else (
            self.K if callable(label_to_category) else len(label_to_category))
        self.score_threshold = float(score_threshold)
        cap = 1000 * self.num_images if max_records is None else int(max_records)
        self.capacity = min(cap, COCO_MAX_RECORDS)
        self.device = dev = torch.device(device)
        rank = {i: q for q, i in enumerate(self.ids_by_rank)}
        cat = {c: k for k, c in enumerate(self.cat_ids)}
        K, n = self.K, self.num_images
        label_cat = []
        for lab in range(self.num_labels):
            try:
                label_cat.append(cat.get(self.label_to_category(lab), -1))
            except (KeyError, IndexError):
                label_cat.append(-1)
        keys, rows = [], []
        for a in gt['annotations']:
            q, k = rank.get(a['image_id']), cat.get(a['category_id'])
            if q is None or k is None:
                continue
            if a['id'] == 0:
                raise N.EffdetNativeError('COCOAccumulator: annotation id 0 (COCOeval takes a match to it for no match)')
            keys.append(q * K + k)
            rows.append(list(a['bbox']) + [a['area'], 1.0 if a.get('iscrowd', 0) else 0.0])
        keys = np.array(keys, dtype=np.int64)
        order = np.argsort(keys, kind='stable')                        # grouped by (image, category), annotation order
        rows = np.array(rows, dtype=np.float64).reshape(-1, 6)[order]
        per_group = np.bincount(keys, minlength=n * K)
        self.max_gt = int(per_group.max()) if keys.size else 0
        if self.max_gt > COCO_MAX_GT:
            raise N.EffdetNativeError('COCOAccumulator: %d ground truths in one (image, category); at most %d'
                                      % (self.max_gt, COCO_MAX_GT))
        self.num_gt = rows.shape[0]
        ws = int(N.load().effdet_coco_accumulate_workspace(self.capacity, n, K))
        if ws < 0:
            raise N.EffdetNativeError('COCOAccumulator: %s' % N.last_error())
        up = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)                       # noqa: E731
        self.gt = up(rows if rows.shape[0] else np.zeros((1, 6)))
        self.gt_offsets = up(np.concatenate([[0], np.cumsum(per_group)]).astype(np.int32))
        self.image_rank = up(np.array([rank[i] for i in self.image_ids], dtype=np.int32))
        self.label_category = up(np.array(label_cat, dtype=np.int32))
        self.iou_thrs, self.rec_thrs = up(coco_iou_thresholds()), up(coco_recall_thresholds())
        R = self.capacity
        self.rec_box = torch.zeros((R, 4), device=dev, dtype=torch.float32)
        self.rec_score = torch.zeros((R,), device=dev, dtype=torch.float32)
        self.rec_meta = torch.full((R, 4), -1, device=dev, dtype=torch.int32)
        self.flags = torch.zeros((R, 4), device=dev, dtype=torch.int32)
        self.cursor = torch.zeros((1,), device=dev, dtype=torch.int64)
        self.image_offset = torch.zeros((n,), device=dev, dtype=torch.int32)
        self.image_count = torch.zeros((n,), device=dev, dtype=torch.int32)
        self.status = torch.zeros((n,), device=dev, dtype=torch.int32)
        self.npig = torch.zeros((K * 4,), device=dev, dtype=torch.int64)
        self.workspace = torch.empty((ws,), device=dev, dtype=torch.uint8)
        self.precision = torch.empty((10 * 101 * K * 4 * 3,), device=dev, dtype=torch.float64)
        self.recall = torch.empty((10 * K * 4 * 3,), device=dev, dtype=torch.float64)
        self.images = 0                       # images added so far: the next batch's first image
        self.num_records = None               # records asked for, known after compute()
        self.summary = None                   # the 12 lines COCOeval.summarize prints, after compute()
        self._staged = None                   # pinned host copy of the last batch's scales (captured copies read it)

    def add(self, detections, scales):
        """detections: _ops.Detections of B images (scores [B,C], classes [B,C] int64, boxes [B,C,4], count [B] int32,
        -1 = NMS overflow) in NMS order, as GraphedDetect / _ops.detect_batch(..., cap=C) return them; scales: B
        per-image box scales (eval.py's data['scale'])"""
        scores, classes, boxes, count = detections
        B, C = scores.shape
        if self.images + B > self.num_images:
            raise N.EffdetNativeError('COCOAccumulator: %d images added to %d, but it was built for %d'
                                      % (B, self.images, self.num_images))
        if len(scales) != B:
            raise N.EffdetNativeError('COCOAccumulator.add: %d images and %d scales' % (B, len(scales)))
        host = torch.from_numpy(np.asarray(scales, dtype=np.float32).reshape(B).copy()).pin_memory()
        self._staged = host
        scale_d = host.to(self.device, non_blocking=True)
        batch_off = torch.empty((B,), device=self.device, dtype=torch.int32)
        batch_cnt = torch.empty((B,), device=self.device, dtype=torch.int32)
        ranks = self.image_rank[self.images:self.images + B]
        N.call('effdet_coco_select_batch', scores, N.f32(scores.contiguous(), 'scores'), N.ptr(classes.contiguous()),
               N.f32(boxes.contiguous(), 'boxes'), N.ptr(count.contiguous()), N.ptr(scale_d), N.ptr(ranks), B, C,
               self.score_threshold, N.ptr(self.label_category), self.num_labels, self.K, self.num_images,
               self.capacity, N.ptr(self.rec_box), N.ptr(self.rec_score), N.ptr(self.rec_meta), N.ptr(self.cursor),
               N.ptr(self.image_offset), N.ptr(self.image_count), N.ptr(self.status[self.images:]), N.ptr(batch_off),
               N.ptr(batch_cnt))
        N.call('effdet_coco_match', scores, N.ptr(self.rec_box), N.ptr(self.rec_meta), N.ptr(batch_off),
               N.ptr(batch_cnt), N.ptr(ranks), B, N.ptr(self.gt), N.ptr(self.gt_offsets), self.num_images, self.K,
               self.max_gt, N.ptr(self.iou_thrs), 10, COCO_BBOX, N.ptr(self.flags), N.ptr(self.npig))
        self.images += B

    def compute(self):
        """-> (stats [12], precision [10,101,K,4,3], recall [10,K,4,3]) as COCOeval's stats and eval['precision'] /
        eval['recall'] hold them (float64)"""
        if self.images != self.num_images:
            raise N.EffdetNativeError('COCOAccumulator: %d of %d images were added' % (self.images, self.num_images))
        K, n = self.K, self.num_images
        N.call('effdet_coco_accumulate', self.rec_score, N.ptr(self.rec_score), N.ptr(self.rec_meta),
               N.ptr(self.flags), N.ptr(self.cursor), N.ptr(self.image_offset), N.ptr(self.image_count),
               N.ptr(self.npig), N.ptr(self.rec_thrs), 101, *COCO_MAX_DETS, self.capacity, n, K,
               N.ptr(self.precision), N.ptr(self.recall), N.ptr(self.workspace), self.workspace.numel())
        host = torch.cat([self.precision, self.recall, self.status.double(), self.cursor.double()]).cpu().numpy()
        P, Rc = 10 * 101 * K * 12, 10 * K * 12
        status, asked = host[P + Rc:P + Rc + n], int(host[-1])
        bad = np.nonzero(status == 1)[0]
        if bad.size:
            raise N.EffdetNativeError('COCOAccumulator: images %s overflowed NMS (more candidates than the detection '
                                      'was built for); redo them eagerly before add()' % bad.tolist())
        if asked > self.capacity:
            raise N.EffdetNativeError('COCOAccumulator: %d records did not fit max_records=%d; max_records=%d would '
                                      'have been enough' % (asked, self.capacity, asked))
        self.num_records = asked
        precision, recall = host[:P].reshape(10, 101, K, 4, 3), host[P:P + Rc].reshape(10, K, 4, 3)
        stats, self.summary = coco_summarize(precision, recall)
        return stats, precision, recall

    def results(self):
        """the detection list eval.py::evaluate_coco builds (eval.py:300-308), in dataset order: image_id,
        category_id, score and bbox (x, y, w, h) as Python numbers"""
        if self.num_records is None:
            self.num_records = min(int(self.cursor.item()), self.capacity)
        m = self.num_records
        rows = torch.cat([self.rec_box[:m], self.rec_score[:m, None], self.rec_meta[:m, :3].view(torch.float32)],
                         dim=1).cpu()                                 # one device->host read
        box, score = rows[:, :4].tolist(), rows[:, 4].tolist()
        meta = rows[:, 5:].contiguous().view(torch.int32).tolist()
        cats = {}
        out = []
        for b, s, (label, _, q) in zip(box, score, meta):
            if label not in cats:
                cats[label] = self.label_to_category(label)
            out.append({'image_id': self.ids_by_rank[q], 'category_id': cats[label], 'score': s, 'bbox': b})
        return out


def evaluate_coco(dataset, model, threshold=0.05, batch_size=16, max_records=None, collater=None, num_workers=0):
    """Drop-in for eval.py::evaluate_coco (eval.py:260-338): the same dataset interface (`dataset[i]` -> {'img'
    [H,W,3], 'scale'}, image_ids, label_to_coco_label, coco, set_name, len), the same progress line, results file
    ({set_name}_bbox_results.json) and summary, with COCOeval's evaluation run on the device (no pycocotools needed).
    Returns COCOeval's 12 stats (None when there are no detections, as the reference returns early); the model is set
    back to training mode at the end, as the reference does.  collater=pipeline.RawCollater(): the dataset yields
    decoded samples and the Resizer chain runs on the device, as in evaluate().  max_records (default 1000 per image)
    bounds the records above threshold; with model.class_nms = 'multi_label' an image can have more than 1000, and then
    the refusal names the max_records that would fit.  A collater with scale_jitter is refused."""
    _refuse_jitter(collater, 'evaluate_coco')
    _refuse_training(model, 'evaluate_coco')
    dev = next(model.parameters()).device
    acc = COCOAccumulator(dataset.coco, dataset.image_ids, dataset.label_to_coco_label, score_threshold=threshold,
                          max_records=max_records, device=dev)
    _detect_all(dataset, model, acc, batch_size, lambda idx: [], 0, collater, num_workers)
    stats, _, _ = acc.compute()
    results = acc.results()
    if not len(results):
        return None
    with open('{}_bbox_results.json'.format(dataset.set_name), 'w') as f:
        json.dump(results, f, indent=4)
    for line in acc.summary:
        print(line)
    model.train()
    return stats
