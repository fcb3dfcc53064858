"""VOC mean average precision on the device: eval.py::evaluate (eval.py:165-257) over csrc/voc_eval.cu.

    acc = VOCAccumulator(num_classes, num_images)
    for each batch:  acc.add(detections, scales, annotations)     # launches only: no host read, capturable
    mean_ap, aps = acc.compute()                                   # the one read -> what eval.py::evaluate returns

`evaluate(generator, model)` is a drop-in for eval.py::evaluate that runs the network in batches through a
GraphedDetect and accumulates on the device; it prints and returns what the reference does.

Records of one class with equal scores are ordered by image, then by rank inside the image: the order a stable sort of
the reference's append order gives (the reference's np.argsort leaves ties to NumPy's introsort).  On tie-free scores
the results equal the reference's float64 values exactly.
"""
import numpy as np
import torch

from . import _native as N
from . import _ops
from .graph_step import GraphedDetect

# candidate rows per image that the graphed detection keeps before NMS; an image with more is redone eagerly
MAX_CANDIDATES = 8192


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


def _add_batch(acc, out, cls, reg, anchors, hw, model, scales, annotations):
    """adds the padded detections of one batch; images that overflowed NMS are redone eagerly from the network outputs
    (one [B] int32 read) and added one by one, in image order"""
    counts = out.count.tolist()
    b0 = 0
    for b, m in enumerate(counts + [None]):
        if m is not None and m >= 0:
            continue
        if b > b0:
            acc.add(_ops.Detections(*(t[b0:b] for t in out)), scales[b0:b], annotations[b0:b])
        if m is None:
            break
        trip = _ops.detect_batch(cls[b:b + 1], reg[b:b + 1], anchors, hw[0], hw[1], model.threshold,
                                 model.iou_threshold)[0]
        acc.add(_padded(trip), scales[b:b + 1], annotations[b:b + 1])
        b0 = b + 1


def evaluate(generator, retinanet, iou_threshold=0.5, score_threshold=0.05, max_detections=100, save_path=None,
             batch_size=16):
    """Drop-in for eval.py::evaluate (eval.py:165-257): the same generator interface (`generator[i]` -> {'img' [H,W,3],
    'scale'}, load_annotations, num_classes, label_to_name, len), the same prints and return value.  The network runs
    `batch_size` images per pass (full batches replay one GraphedDetect, the remainder runs eagerly), and selection,
    matching and AP run on the device.  save_path is accepted and unused, as in the reference."""
    if retinanet.training or retinanet.is_training:
        raise N.EffdetNativeError('evaluate needs a model in inference mode (model.eval() and '
                                  'model.is_training = False)')
    n, K = len(generator), generator.num_classes()
    dev = next(retinanet.parameters()).device
    acc = VOCAccumulator(K, n, iou_threshold, score_threshold, max_detections, device=dev)
    graphed = None
    with torch.no_grad():
        for i0 in range(0, n, batch_size):
            idx = range(i0, min(n, i0 + batch_size))
            data = [generator[i] for i in idx]
            images = torch.stack([d['img'].permute(2, 0, 1).to(dev).float() for d in data])
            hw = images.shape[2], images.shape[3]
            if len(idx) == batch_size:
                if graphed is None:
                    graphed = GraphedDetect(retinanet, images, max_candidates=MAX_CANDIDATES)
                out = graphed(images)
                cls, reg, anchors = graphed.cls, graphed.reg, graphed.anchors
            else:
                cls, reg, anchors = retinanet._raw_predictions(images)
                out = _ops.detect_batch(cls, reg, anchors, hw[0], hw[1], retinanet.threshold, retinanet.iou_threshold,
                                        cap=min(MAX_CANDIDATES, cls.shape[1]))
            _add_batch(acc, out, cls, reg, anchors, hw, retinanet, [d['scale'] for d in data],
                       [generator.load_annotations(i) for i in idx])
            for i in idx:
                print('{}/{}'.format(i + 1, n), end='\r')
    mean_ap, aps = acc.compute()
    print('\nmAP:')
    for label in range(K):
        print('{}: {}'.format(generator.label_to_name(label), aps[label][0]))
    print('avg mAP: {}'.format(mean_ap))
    return mean_ap, aps
