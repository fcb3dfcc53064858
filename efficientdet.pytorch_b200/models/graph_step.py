"""CUDA-graph execution of the training step (forward + FocalLoss + backward, optionally the fused optimizer), and of
inference (GraphedDetect, at the end of this file).

Every kernel of the hot path is launched on the caller's stream with device-resident arguments and no host
synchronisation (the C ABI never syncs, FocalLoss reads its upstream gradients from device memory), so the ~480
launches of a step can be captured once and replayed: the host cost of a step drops from ~12-16 ms of ctypes calls to
one cudaGraphLaunch, which matters as soon as the GPU finishes a step faster than Python can issue it.

    step = GraphedTrainStep(model, images_example, annotations_example)          # model.train(); freeze_bn() first
    loss = step(images, annotations)      # copies into the static inputs, replays, returns the static loss tensor
    ... model parameters' .grad now hold this step's gradients (same tensors every step)

Without an optimizer the graph reads the packed weights / folded BatchNorm its warm-up derived into the caches of
models/_ops.py; anything that invalidates them (load_state_dict, train(), eval(), freeze_bn(), building a step with an
optimizer) means building this step again.

Build it BEFORE any eager step, or after every reference to earlier eager losses / outputs has been dropped: a live autograd
graph keeps the parameters' gradient accumulators bound to the stream it ran on (the legacy stream), and the engine
may not touch that stream while another one is capturing.

Shapes are static by default: every call takes images and annotations of the example's shapes.  Drop-connect keeps
working: torch.rand inside a captured region advances the Philox offset on every replay.

Capacity mode, for the batches a DataLoader with collate_fn=collater yields.  The collater pads each batch to the
largest annotation count in THAT batch, and the last batch of an epoch is short unless drop_last is set.  With
`max_annotations=Gcap` the example images fix a capacity of Bcap images of H x W, and the graph is captured on a static
[Bcap, Gcap, 5] annotation table plus its device-side counts (models/losses.py).  Every call then takes images
[B, 3, H, W] with 1 <= B <= Bcap and annotations [B, G, 5] with G <= Gcap, from the host or the device: the images go
to the first B rows of the static input and the rest is zero-filled; one launch packs the annotations (each image's
labelled rows first, the rest -1) and writes the counts; then the graph replays.  The loss is the mean over the B real
images; the padding images are excluded from it and their gradients are exactly zero, and the frozen BatchNorm and the
per-image squeeze-excite keep them from touching the real images.  A short batch costs a full-capacity step.  Images
with more than Gcap annotations, more than Bcap images or another H x W are refused before anything is launched.

    step = GraphedTrainStep(model, images_example, annotations_example, optimizer=opt, max_annotations=256)
    for idx, (images, annotations) in enumerate(train_loader):       # any batch size up to Bcap, ragged annotations
        loss = step(images, annotations, update=(idx + 1) % k == 0)

Training with the optimizer in the graph.  With `optimizer=FusedClipAdamW(...)` every call is one micro-step of the
reference loop (train.py:95-133): forward, loss, backward, gradients added to the persistent accumulators that
`p.grad` then refers to (skipped when the loss is exactly 0), and, when `update` is true and the loss is non-zero, the
clip + AdamW update, which also empties the accumulators.  The loop as a user writes it, with k =
--grad_accumulation_steps:

    opt = FusedClipAdamW(model.parameters(), lr=lr, max_norm=0.1)    # opt.load_state_dict(...) here, if resuming
    scheduler = torch.optim.lr_scheduler.ReduceLROnPlateau(opt, patience=3)
    step = GraphedTrainStep(model, images_example, annotations_example, optimizer=opt)
    for epoch in range(num_epoch):
        opt.zero_grad()
        losses = []
        for idx, (images, annotations) in enumerate(train_loader):
            loss = step(images, annotations, update=(idx + 1) % k == 0)
            losses.append(loss.clone())                    # stays on the device: no synchronisation per step
        losses = torch.stack(losses)
        scheduler.step(float(losses[losses != 0].mean()))  # the reference averages the non-skipped losses
        torch.save({'optimizer': opt.state_dict(), ...})  # true step counts: one device read

The step counters and learning rates live in device memory: each call writes the `update` flag, and the lr of any
param group whose `group['lr']` changed, into their device scalars before the replay (launches, no synchronisation),
so schedulers work without recapture.  betas, eps, weight_decay and max_norm are fixed at capture; changing them
raises.  Building the step leaves parameters, moments and step counts untouched: the warm-up runs forward and backward
only.  Under DDP every call must update (`update=True`); gradient accumulation across DDP micro-steps is not
supported.  Any other optimizer has its `step()` captured as is (the warm-up then runs it too) and allows
`update=True` only.

With an optimizer in the graph the packed-weight / folded-BN derivations are captured as well: they re-run on every
replay because the weights change without Python seeing it.  For the same reason, eager use of the model between
replays needs `model.eval()` / `model.train()` (or `_ops.invalidate_caches()`) first.
"""
import torch

from . import _ops
from .fused_optim import FusedClipAdamW


class GraphedTrainStep:
    """model: the EfficientDet module, or its DistributedDataParallel wrapper.  For DDP the NCCL gradient all-reduces are
    captured with the step (torch's documented recipe: NCCL >= 2.9.6, TORCH_NCCL_ASYNC_ERROR_HANDLING=0 before
    init_process_group, the DDP wrapper CONSTRUCTED inside a side-stream context, >= 11 eager warm-up iterations);
    gradients then have to flow through DDP's AccumulateGrad hooks, so the captured step calls loss.backward()."""

    def __init__(self, model, images, annotations, optimizer=None, warmup=3, max_annotations=None):
        if not images.is_cuda:
            raise _ops.N.EffdetNativeError('GraphedTrainStep needs CUDA example inputs')
        self.ddp = isinstance(model, torch.nn.parallel.DistributedDataParallel)
        if self.ddp:
            warmup = max(warmup, 11)
        self.model = model
        self.optimizer = optimizer
        self.fused = isinstance(optimizer, FusedClipAdamW)
        self.static_images = images.clone()
        self.static_counts = None
        if max_annotations is None:
            self.static_annots = annotations.clone()
        else:
            if isinstance(max_annotations, bool) or not isinstance(max_annotations, int) or max_annotations < 1:
                raise _ops.N.EffdetNativeError('GraphedTrainStep: max_annotations must be an integer >= 1, got %r'
                                               % (max_annotations,))
            if images.dim() != 4:
                raise _ops.N.EffdetNativeError('GraphedTrainStep: example images must be [Bcap, 3, H, W], got %s'
                                               % (tuple(images.shape),))
            self.static_annots = torch.full((images.shape[0], max_annotations, 5), -1.0, dtype=torch.float32,
                                            device=images.device)
            self.static_counts = torch.zeros((1 + images.shape[0],), dtype=torch.int32, device=images.device)
            self._check_batch(images, annotations)
            self._load_batch(images, annotations)
        params = [p for p in model.parameters() if p.requires_grad]
        side = torch.cuda.Stream(device=images.device)
        side.wait_stream(torch.cuda.current_stream(images.device))
        with torch.cuda.stream(side):
            for _ in range(warmup):                                   # fills allocator pools, caches, cuFuncSetAttribute
                self._eager_step(params)
        torch.cuda.current_stream(images.device).wait_stream(side)
        torch.cuda.synchronize(images.device)
        if optimizer is not None:
            _ops.invalidate_caches()                                  # capture the weight re-packing with the step
        if self.fused:
            optimizer._bind_graph([p for p in params if p.grad is not None])
        self.graph = torch.cuda.CUDAGraph()
        for p in params:
            p.grad = None
        n0 = _ops.N.launch_count()
        try:
            with torch.cuda.graph(self.graph):
                self.static_loss = self._eager_step(params, zero=False, capture=True)
        except RuntimeError as e:
            if 'legacy stream' in str(e) or 'previous error during capture' in str(e):
                raise _ops.N.EffdetNativeError(
                    'GraphedTrainStep: the autograd engine tried to synchronise with the legacy default stream during '
                    'capture.  The gradient accumulators of the parameters remember the stream of an earlier eager step '
                    'for as long as that step\'s graph is alive: drop every reference to earlier losses / outputs '
                    '(`del loss`) before building the graphed step, or run eager steps under a side stream.') from e
            raise
        self.library_launches = _ops.N.launch_count() - n0            # kernels of this library recorded into the graph
        self.params = params
        if self.fused:
            optimizer._graph_captured()
            # capture recorded the weight packing without running it: eager calls derive their own until a replay
            _ops.invalidate_caches()

    def _eager_step(self, params, zero=True, capture=False):
        if zero:
            for p in params:
                p.grad = None
        inputs = [self.static_images, self.static_annots]
        if self.static_counts is not None:
            inputs.append(self.static_counts)
        cl, rl = self.model(inputs)
        loss = cl.mean() + rl.mean()
        # torch.autograd.grad, not .backward(): AccumulateGrad nodes remember the stream of an earlier eager step (the
        # legacy stream if the caller still holds that step's loss) and would make it wait on the capturing stream --
        # cudaErrorStreamCaptureImplicit.  The returned tensors live in the graph's pool: every replay rewrites them.
        if self.ddp:
            loss.backward()
        else:
            grads = torch.autograd.grad(loss, params, allow_unused=True)
            for p, g in zip(params, grads):
                p.grad = g
        if self.fused:
            if capture:                                              # the warm-up leaves the optimizer untouched
                self.optimizer._graph_launch({p: p.grad for p in params}, loss)
        elif self.optimizer is not None:
            self.optimizer.step()
        return loss.detach()

    def _check_batch(self, images, annotations):
        """capacity mode: refuse a batch that does not fit, before anything is launched"""
        cap = tuple(self.static_images.shape)
        Bcap, Gcap = cap[0], self.static_annots.shape[1]
        if images.dim() != 4 or tuple(images.shape[1:]) != cap[1:]:
            raise _ops.N.EffdetNativeError('GraphedTrainStep was captured for images [B <= %d, %d, %d, %d], got %s'
                                           % (cap + (tuple(images.shape),)))
        B = images.shape[0]
        if not 1 <= B <= Bcap:
            raise _ops.N.EffdetNativeError('GraphedTrainStep: a batch of %d images does not fit the capacity of %d '
                                           'images of the example' % (B, Bcap))
        if annotations.dim() != 3 or annotations.shape[0] != B or annotations.shape[2] != 5:
            raise _ops.N.EffdetNativeError('GraphedTrainStep: annotations must be [B=%d, G, 5], got %s'
                                           % (B, tuple(annotations.shape)))
        G = annotations.shape[1]
        if G > Gcap:
            raise _ops.N.EffdetNativeError('GraphedTrainStep: a batch with %d annotation rows per image does not fit '
                                           'max_annotations=%d; build the step with max_annotations=%d or more'
                                           % (G, Gcap, G))

    def _load_batch(self, images, annotations):
        """capacity mode: images into the static input (zeros after them), annotations packed with their counts"""
        B = images.shape[0]
        self.static_images[:B].copy_(images, non_blocking=True)
        if B < self.static_images.shape[0]:
            self.static_images[B:].zero_()
        if annotations.shape[1] == 0:                                # no rows at all: one -1 row, as collater writes
            annotations = torch.full((B, 1, 5), -1.0)
        annotations = annotations.to(device=self.static_annots.device, dtype=torch.float32, non_blocking=True)
        _ops.pack_annotations(annotations.contiguous(), self.static_annots, self.static_counts)

    def __call__(self, images, annotations, update=True):
        """One micro-step.  update: run the optimizer after it (train.py:115 `(idx + 1) % k == 0`); with
        FusedClipAdamW the update is skipped on the device when the step's loss is exactly zero."""
        if self.static_counts is not None:
            self._check_batch(images, annotations)
        if self.fused:
            if self.ddp and not update:
                raise _ops.N.EffdetNativeError('GraphedTrainStep: update=False (gradient accumulation) is not supported '
                                               'under DistributedDataParallel; call it with update=True')
            self.optimizer._graph_prepare(update)
        elif not update:
            raise _ops.N.EffdetNativeError('GraphedTrainStep: update=False (gradient accumulation) needs '
                                           'optimizer=FusedClipAdamW(...)')
        if self.static_counts is not None:
            self._load_batch(images, annotations)
        else:
            self.static_images.copy_(images, non_blocking=True)
            self.static_annots.copy_(annotations, non_blocking=True)
        self.graph.replay()
        return self.static_loss


class GraphedDetect:
    """CUDA-graph execution of inference: network forward + decode + threshold + NMS of a whole batch as one replay,
    with no host synchronisation.

        det = GraphedDetect(model, example_images, max_candidates=8192)   # model.eval(), model.is_training False
        out = det(images)        # copies into the static input, one replay -> _ops.Detections (padded, on the device)
        dets = det.to_list(out)  # one device->host read -> B triples exactly as model.detect_batch(images) returns them

    out.scores [B,C], out.classes [B,C] int64, out.boxes [B,C,4] and out.count [B] int32 (kept rows; -1 when the image
    has more than C candidates above the threshold) are static tensors: every call rewrites them.  C is max_candidates,
    or the anchor count A when that is smaller (an image never has more than A candidates); max_candidates=None sets
    C = A, so every anchor may be a candidate and no image overflows.  to_list redoes overflowed images eagerly from the
    network outputs of the last replay.  Calls take images of the example's shape only.

    Memory that max_candidates costs per image is linear in C: 32 bytes per row of keep indices and padded outputs,
    plus the NMS workspace, which is the mask C * ceil(C/64) * 8 bytes up to C = _ops.NMS_CHUNK and the mask of one
    chunk (2 MiB at NMS_CHUNK = 4096) above it.  At D7 1536x1536 (A = 441 936) C = A costs about 16 MB per image.  The
    decoded anchors and their sort keys (24 bytes per anchor plus 8 per power-of-two padded anchor) do not depend on C.

    The packed weights and folded BatchNorm are derived inside the graph, so replays follow in-place weight updates
    (load_state_dict, EMA copies).  The score and IoU thresholds are fixed at capture."""

    def __init__(self, model, images, max_candidates=8192, warmup=2):
        if model.training or model.is_training:
            raise _ops.N.EffdetNativeError('GraphedDetect needs a model in inference mode (model.eval() and '
                                           'model.is_training = False)')
        if not images.is_cuda:
            raise _ops.N.EffdetNativeError('GraphedDetect needs CUDA example images')
        self.model = model
        self.max_candidates = None if max_candidates is None else int(max_candidates)
        self.threshold, self.iou_threshold = model.threshold, model.iou_threshold
        self.static_images = images.clone()
        dev = images.device
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side):
            for _ in range(warmup):                                   # anchor table, allocator pools, smem opt-ins
                self._run()
        torch.cuda.current_stream(dev).wait_stream(side)
        torch.cuda.synchronize(dev)
        _ops.invalidate_caches()                                      # capture the weight packing and BN folding
        self.graph = torch.cuda.CUDAGraph()
        n0 = _ops.N.launch_count()
        with torch.cuda.graph(self.graph):
            self.cls, self.reg, self.anchors, self.out = self._run()
        self.library_launches = _ops.N.launch_count() - n0            # kernels of this library recorded into the graph
        # capture recorded the weight packing without running it: the cache entries it made hold nothing until a
        # replay.  Dropping them makes eager calls derive their own; the graph keeps its copies in its private pool.
        _ops.invalidate_caches()

    @torch.no_grad()
    def _run(self):
        cls, reg, anchors = self.model._raw_predictions(self.static_images)
        out = _ops.detect_batch(cls, reg, anchors, self.static_images.shape[2], self.static_images.shape[3],
                                self.threshold, self.iou_threshold, cap=_ops.candidate_cap(self.max_candidates, cls))
        return cls, reg, anchors, out

    def __call__(self, images):
        if (self.model.threshold, self.model.iou_threshold) != (self.threshold, self.iou_threshold):
            raise _ops.N.EffdetNativeError(
                'GraphedDetect: threshold / iou_threshold changed from (%r, %r) at capture to (%r, %r); build a new '
                'GraphedDetect' % (self.threshold, self.iou_threshold, self.model.threshold, self.model.iou_threshold))
        if images.shape != self.static_images.shape:
            raise _ops.N.EffdetNativeError('GraphedDetect was captured for images of shape %s, got %s'
                                           % (tuple(self.static_images.shape), tuple(images.shape)))
        self.static_images.copy_(images, non_blocking=True)
        self.graph.replay()
        return self.out

    def to_list(self, out):
        """out (the result of the latest call) -> list of B triples [scores[K_b], classes[K_b] int64, boxes[K_b,4]]"""
        res = []
        for b, m in enumerate(out.count.tolist()):                   # the one device->host read
            if m < 0:
                res.append(_ops.detect_batch(self.cls[b:b + 1], self.reg[b:b + 1], self.anchors,
                                             self.static_images.shape[2], self.static_images.shape[3], self.threshold,
                                             self.iou_threshold)[0])
            else:
                res.append([out.scores[b, :m], out.classes[b, :m], out.boxes[b, :m]])
        return res
