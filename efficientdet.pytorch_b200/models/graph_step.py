"""CUDA-graph execution of the training step (forward + FocalLoss + backward, optionally the fused optimizer), and of
inference (GraphedDetect, and GraphedFrameDetect for demo.py's frames, at the end of this file).

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

Raw-batch mode, for a DataLoader whose workers decode: collate_fn=pipeline.RawCollater(...) yields RawBatch blobs
(uint8 images, Resizer geometry, flips, annotation rows) without touching CUDA.  Built on one of them, the step is
capacity mode with Bcap = its B, max_annotations (required) rows per image and max_bytes (default: Bcap times its
largest image) bytes of PIXELS -- the rows have their own bound, Bcap * max_annotations.  (GraphedRawDetect has no
max_annotations and counts rows and pixels together in its max_bytes.)  The captured region starts with the Resizer
chain into the static images and the annotation packing (effdet_collate_pack_annots), so a call is one host-to-device
copy of the blob and one replay.  Batches with more images, pixel bytes or rows per image are refused before anything
is copied.

    loader = DataLoader(dataset, batch_size, num_workers=4, collate_fn=RawCollater(pixel_scale=255), pin_memory=True)
    step = None
    for idx, raw in enumerate(loader):
        step = step or GraphedTrainStep(model, raw, optimizer=opt, max_annotations=256)
        loss = step(raw, update=(idx + 1) % k == 0)

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
import numpy as np
import torch

from . import _ops
from . import pipeline
from .fused_optim import FusedClipAdamW


class GraphedTrainStep:
    """model: the EfficientDet module, or its DistributedDataParallel wrapper.  For DDP the NCCL gradient all-reduces are
    captured with the step (torch's documented recipe: NCCL >= 2.9.6, TORCH_NCCL_ASYNC_ERROR_HANDLING=0 before
    init_process_group, the DDP wrapper CONSTRUCTED inside a side-stream context, >= 11 eager warm-up iterations);
    gradients then have to flow through DDP's AccumulateGrad hooks, so the captured step calls loss.backward()."""

    def __init__(self, model, images, annotations=None, optimizer=None, warmup=3, max_annotations=None, max_bytes=None):
        self.raw = None
        if isinstance(images, pipeline.RawBatch):
            images = self._init_raw(model, images, annotations, max_annotations, max_bytes)
        elif annotations is None:
            raise _ops.N.EffdetNativeError('GraphedTrainStep: example annotations are needed with example images')
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
        if self.raw is not None:
            self.static_annots = torch.full((self.raw['Bcap'], max_annotations, 5), -1.0, dtype=torch.float32,
                                            device=images.device)
            self.static_counts = torch.zeros((1 + self.raw['Bcap'],), dtype=torch.int32, device=images.device)
        elif max_annotations is None:
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
            # a raw-batch step is built while a DataLoader's pin thread allocates pinned memory: capture in
            # thread-local mode, so that thread's CUDA calls do not invalidate this thread's capture
            with torch.cuda.graph(self.graph, capture_error_mode='global' if self.raw is None else 'thread_local'):
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

    def _init_raw(self, model, example, annotations, max_annotations, max_bytes):
        """raw-batch mode: the static device copy of a raw batch laid out for Bcap = example.B images, with room for
        Bcap * max_annotations rows and max_bytes pixel bytes (pixels only, unlike GraphedRawDetect's max_bytes) ->
        example images for the capture (zeros)"""
        err = _ops.N.EffdetNativeError
        if annotations is not None:
            raise err('GraphedTrainStep(model, raw_batch, ...): a RawBatch carries its annotations; pass optimizer, '
                      'max_annotations and max_bytes by keyword')
        if isinstance(max_annotations, bool) or not isinstance(max_annotations, int) or max_annotations < 1:
            raise err('GraphedTrainStep: a RawBatch example needs max_annotations, an integer >= 1, got %r'
                      % (max_annotations,))
        dev = next(model.parameters()).device
        if dev.type != 'cuda':
            raise err('GraphedTrainStep needs a model on a CUDA device')
        Bcap = example.B
        cap_bytes = Bcap * int(example.image_bytes.max()) if max_bytes is None else int(max_bytes)
        _, total = pipeline.raw_layout(Bcap, Bcap * max_annotations, cap_bytes)
        self.raw = dict(Bcap=Bcap, Gcap=max_annotations, max_bytes=cap_bytes, S=example.S,
                        pixel_scale=example.pixel_scale, blob=torch.empty((total,), dtype=torch.uint8, device=dev))
        self._check_raw(example)
        self._load_raw(example)
        return torch.zeros((Bcap, 3, example.S, example.S), device=dev)

    def _check_raw(self, raw):
        """raw-batch mode: refuse a batch that does not fit, before anything is copied or launched"""
        err, c = _ops.N.EffdetNativeError, self.raw
        if not isinstance(raw, pipeline.RawBatch):
            raise err('GraphedTrainStep was built on a RawBatch: call it as step(raw_batch, update=...)')
        if (raw.S, raw.pixel_scale) != (c['S'], c['pixel_scale']):
            raise err('GraphedTrainStep was captured for common size %d and pixel_scale %r, got %d and %r'
                      % (c['S'], c['pixel_scale'], raw.S, raw.pixel_scale))
        if not 1 <= raw.B <= c['Bcap']:
            raise err('GraphedTrainStep: a batch of %d images does not fit the capacity of %d images of the example'
                      % (raw.B, c['Bcap']))
        if raw.nbytes > c['max_bytes']:
            raise err('GraphedTrainStep: a batch of %d pixel bytes does not fit max_bytes=%d; build the step with '
                      'max_bytes=%d or more' % (raw.nbytes, c['max_bytes'], raw.nbytes))
        if raw.max_rows > c['Gcap']:
            raise err('GraphedTrainStep: a batch with %d annotation rows per image does not fit max_annotations=%d; '
                      'build the step with max_annotations=%d or more' % (raw.max_rows, c['Gcap'], raw.max_rows))

    def _load_raw(self, raw):
        """raw-batch mode: the batch laid out for Bcap images (a short batch gets zero entries for the unused images,
        in a new host blob) -> one host-to-device copy into the static blob"""
        blob = raw.at_capacity(self.raw['Bcap'], pin=raw.blob.is_pinned()).blob
        self.raw['blob'][:blob.numel()].copy_(blob, non_blocking=True)

    def _unpack_raw(self):
        """the head of the captured region in raw-batch mode: Normalizer -> flip -> Resizer -> pad into the static
        images (padding images are zeros), then the annotations collated and packed with their counts"""
        c = self.raw
        pipeline.launch_raw_resize(self.static_images, c['blob'], c['Bcap'], c['pixel_scale'])
        pipeline.launch_raw_pack(c['blob'], c['Bcap'], self.static_annots, self.static_counts)

    def _eager_step(self, params, zero=True, capture=False):
        if zero:
            for p in params:
                p.grad = None
        if self.raw is not None:
            self._unpack_raw()
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

    def __call__(self, images, annotations=None, update=True):
        """One micro-step.  update: run the optimizer after it (train.py:115 `(idx + 1) % k == 0`); with
        FusedClipAdamW the update is skipped on the device when the step's loss is exactly zero.  A step built on a
        RawBatch is called as step(raw_batch, update=...)."""
        if self.raw is not None:
            if annotations is not None:
                raise _ops.N.EffdetNativeError('GraphedTrainStep was built on a RawBatch: call it as '
                                               'step(raw_batch, update=...)')
            self._check_raw(images)
        elif annotations is None:
            raise _ops.N.EffdetNativeError('GraphedTrainStep: call it as step(images, annotations, update=...)')
        elif self.static_counts is not None:
            self._check_batch(images, annotations)
        if self.fused:
            if self.ddp and not update:
                raise _ops.N.EffdetNativeError('GraphedTrainStep: update=False (gradient accumulation) is not supported '
                                               'under DistributedDataParallel; call it with update=True')
            self.optimizer._graph_prepare(update)
        elif not update:
            raise _ops.N.EffdetNativeError('GraphedTrainStep: update=False (gradient accumulation) needs '
                                           'optimizer=FusedClipAdamW(...)')
        if self.raw is not None:
            self._load_raw(images)
        elif self.static_counts is not None:
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
    (load_state_dict, EMA copies).  The post-processing settings (threshold, iou_threshold, nms, soft_nms_sigma,
    class_nms, pre_nms_top_k) are fixed at capture: changing one on the model makes the next call raise.  With
    class_nms='multi_label', C is also clamped to the min(pre_nms_top_k, A*K) candidate slots of an image."""

    _capture_error_mode = 'global'

    def __init__(self, model, images, max_candidates=8192, warmup=2):
        if model.training or model.is_training:
            raise _ops.N.EffdetNativeError('GraphedDetect needs a model in inference mode (model.eval() and '
                                           'model.is_training = False)')
        if not images.is_cuda:
            raise _ops.N.EffdetNativeError('GraphedDetect needs CUDA example images')
        self.model = model
        self.max_candidates = None if max_candidates is None else int(max_candidates)
        self.post = model.postprocess()
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
        with torch.cuda.graph(self.graph, capture_error_mode=self._capture_error_mode):
            self.cls, self.reg, self.anchors, self.out = self._run()
        self.library_launches = _ops.N.launch_count() - n0            # kernels of this library recorded into the graph
        # capture recorded the weight packing without running it: the cache entries it made hold nothing until a
        # replay.  Dropping them makes eager calls derive their own; the graph keeps its copies in its private pool.
        _ops.invalidate_caches()

    @torch.no_grad()
    def _run(self):
        cls, reg, anchors = self.model._raw_predictions(self.static_images)
        out = _ops.detect_batch(cls, reg, anchors, self.static_images.shape[2], self.static_images.shape[3],
                                cap=_ops.candidate_cap(self.max_candidates, cls), **self.post)
        return cls, reg, anchors, out

    def _check_thresholds(self):
        now = self.model.postprocess()
        if now != self.post:
            raise _ops.N.EffdetNativeError('%s: the post-processing settings changed from %r at capture to %r; build a '
                                           'new %s' % (type(self).__name__, self.post, now, type(self).__name__))

    def __call__(self, images):
        self._check_thresholds()
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
                                             self.static_images.shape[2], self.static_images.shape[3], **self.post)[0])
            else:
                res.append([out.scores[b, :m], out.classes[b, :m], out.boxes[b, :m]])
        return res


class GraphedFrameDetect(GraphedDetect):
    """demo.py's Detect.process (demo.py:71-104) for a batch of frames as one CUDA-graph replay: the test transform
    (pipeline.frame_transform's kernel) at the head of GraphedDetect's captured region, decode + NMS after the network,
    and demo.py's per-box arithmetic (pipeline.frame_boxes) at its tail.

        det = GraphedFrameDetect(model, example_frames)           # model.eval(), model.is_training False
        for boxes, labels, scores in det(frames):                 # frames: list of uint8 [h, w, 3] BGR arrays
            ...  # boxes int32 [n, 4], labels int64 [n], scores int32 [n]: demo.py's bboxes, label indices, bbox_scores

    The example frames fix the capacity: Bcap = len(example_frames) frames and their total byte count.  A call takes
    1 .. Bcap frames of any sizes whose bytes fit; it copies them and their geometry into pinned staging, issues the
    host-to-device copies, replays once and reads back the counts and the kept rows (two device->host reads, no
    per-box Python).  Frames of new sizes replay without recapture; unused capacity runs as zero padding frames.  A
    frame that overflows max_candidates (None: every anchor may be a candidate, no frame overflows) is redone eagerly
    from the replay's network outputs.  The network input is height x width, demo.py's size_image."""

    def __init__(self, model, example_frames, height=512, width=512, max_candidates=None, warmup=2):
        frames = pipeline.check_frames(example_frames, 'GraphedFrameDetect')
        self.H, self.W = int(height), int(width)
        if not (1 <= self.H <= 65535 and 1 <= self.W <= 65535):
            raise _ops.N.EffdetNativeError('GraphedFrameDetect: height=%r, width=%r must be in [1, 65535]'
                                           % (height, width))
        dev = next(model.parameters()).device
        if dev.type != 'cuda':
            raise _ops.N.EffdetNativeError('GraphedFrameDetect needs a model on a CUDA device')
        self.capacity = len(frames)
        self.byte_capacity = sum(f.size for f in frames)
        self._pix_h = torch.empty((self.byte_capacity,), dtype=torch.uint8).pin_memory()
        self._offs_h = torch.zeros((self.capacity,), dtype=torch.int64).pin_memory()
        self._hw_h = torch.zeros((self.capacity, 2), dtype=torch.int32).pin_memory()
        self._pix = torch.empty((self.byte_capacity,), dtype=torch.uint8, device=dev)
        self._offs = torch.empty((self.capacity,), dtype=torch.int64, device=dev)
        self._hw = torch.empty((self.capacity, 2), dtype=torch.int32, device=dev)
        self._load(frames)
        super().__init__(model, torch.zeros((self.capacity, 3, self.H, self.W), device=dev), max_candidates, warmup)

    def _load(self, frames):
        """staging <- frames (padding frames h = w = 0 after them), then the host->device copies"""
        B = len(frames)
        flat, offs = pipeline.concat_pinned(frames, self._pix_h)
        self._offs_h.zero_()
        self._hw_h.zero_()
        self._offs_h.numpy()[:B] = offs
        self._hw_h.numpy()[:B] = [f.shape[:2] for f in frames]
        self._pix[:flat.numel()].copy_(flat, non_blocking=True)
        self._offs.copy_(self._offs_h, non_blocking=True)
        self._hw.copy_(self._hw_h, non_blocking=True)

    @torch.no_grad()
    def _run(self):
        pipeline.launch_frame_transform(self.static_images, self._pix, self._offs, self._hw)
        cls, reg, anchors, out = super()._run()
        self.rows, self.counts = pipeline.frame_boxes(out, self._hw, self.H, self.W)
        return cls, reg, anchors, out

    def __call__(self, frames):
        """frames: list of 1 .. capacity uint8 [h, w, 3] arrays -> per frame (boxes int32 [n, 4], labels int64 [n],
        scores int32 [n]) as NumPy arrays"""
        frames = pipeline.check_frames(frames, 'GraphedFrameDetect')
        B, nbytes = len(frames), sum(f.size for f in frames)
        if B > self.capacity or nbytes > self.byte_capacity:
            raise _ops.N.EffdetNativeError(
                'GraphedFrameDetect: %d frames of %d bytes do not fit the capacity of %d frames and %d bytes of the '
                'example frames' % (B, nbytes, self.capacity, self.byte_capacity))
        self._check_thresholds()
        self._load(frames)
        self.graph.replay()
        counts = self.counts[:B].tolist()                             # device->host read 1 of 2
        top = max(counts + [0])
        rows = self.rows[:B, :top].cpu().numpy() if top else None      # device->host read 2 of 2
        res = []
        for b, n in enumerate(counts):
            if n < 0:
                r = self._redo(b)
            else:
                r = rows[b, :n] if n else np.zeros((0, 6), np.int32)
            res.append((np.ascontiguousarray(r[:, :4]), r[:, 4].astype(np.int64), np.ascontiguousarray(r[:, 5])))
        return res

    def _redo(self, b):
        """rows of a frame that overflowed the candidate cap: eager NMS on the replay's network outputs"""
        from .evaluation import _padded
        trip = _ops.detect_batch(self.cls[b:b + 1], self.reg[b:b + 1], self.anchors, self.H, self.W, **self.post)[0]
        rows, counts = pipeline.frame_boxes(_padded(trip), self._hw[b:b + 1], self.H, self.W)
        return rows[0, :int(counts[0])].cpu().numpy()


class GraphedRawDetect(GraphedDetect):
    """GraphedDetect fed by raw batches (pipeline.RawCollater's output): the Resizer chain (Normalizer -> Resizer ->
    zero pad, effdet_resize_normalize_pad) at the head of the captured region, then the network, decode and NMS (hard
    or Soft-NMS, from model.postprocess()).

        det = GraphedRawDetect(model, example_raw_batch)          # model.eval(), model.is_training False
        out, scales = det(raw_batch)    # one host-to-device copy, one replay -> padded Detections, float64 [B] scales

    The example fixes the capacity: Bcap = example.B images, and max_bytes bytes of annotation rows AND pixels together
    (RawBatch.data_bytes, the blob after its fixed sections; default: Bcap times the example's largest image plus the
    example's rows).  This differs from GraphedTrainStep's max_bytes, which counts pixels only because its rows are
    bounded by max_annotations; detection reads no rows, so it bounds the blob's size alone.  A call takes 1 ..
    Bcap images whose bytes fit; the unused capacity runs as zero padding images, whose rows of `out` are to be
    ignored.  out is the static output of GraphedDetect: every call rewrites it."""

    # built while a DataLoader's pin thread allocates pinned memory (evaluate(..., collater=)): another thread's CUDA
    # calls must not invalidate the capture
    _capture_error_mode = 'thread_local'

    def __init__(self, model, example, max_bytes=None, max_candidates=None, warmup=2):
        err = _ops.N.EffdetNativeError
        if not isinstance(example, pipeline.RawBatch):
            raise err('GraphedRawDetect needs a RawBatch example (pipeline.RawCollater output)')
        dev = next(model.parameters()).device
        if dev.type != 'cuda':
            raise err('GraphedRawDetect needs a model on a CUDA device')
        self.capacity, self.S, self.pixel_scale = example.B, example.S, example.pixel_scale
        if max_bytes is None:
            max_bytes = (self.capacity * int(example.image_bytes.max()) + 15) // 16 * 16 + \
                (40 * example.rows + 15) // 16 * 16
        self.max_bytes = int(max_bytes)
        fixed = pipeline.raw_layout(self.capacity, 0, 0)[0]['rows']
        self._blob = torch.empty((fixed + self.max_bytes,), dtype=torch.uint8, device=dev)
        self._check_raw(example)
        self._load_raw(example)
        super().__init__(model, torch.zeros((self.capacity, 3, self.S, self.S), device=dev), max_candidates, warmup)

    def _check_raw(self, raw):
        err = _ops.N.EffdetNativeError
        if not isinstance(raw, pipeline.RawBatch):
            raise err('GraphedRawDetect takes RawBatch inputs (pipeline.RawCollater output)')
        if (raw.S, raw.pixel_scale) != (self.S, self.pixel_scale):
            raise err('GraphedRawDetect was captured for common size %d and pixel_scale %r, got %d and %r'
                      % (self.S, self.pixel_scale, raw.S, raw.pixel_scale))
        if not 1 <= raw.B <= self.capacity:
            raise err('GraphedRawDetect: a batch of %d images does not fit the capacity of %d images of the example'
                      % (raw.B, self.capacity))
        if raw.data_bytes > self.max_bytes:
            raise err('GraphedRawDetect: a batch of %d bytes of rows and pixels does not fit max_bytes=%d; build it '
                      'with max_bytes=%d or more' % (raw.data_bytes, self.max_bytes, raw.data_bytes))

    def _load_raw(self, raw):
        blob = raw.at_capacity(self.capacity, pin=raw.blob.is_pinned()).blob
        self._blob[:blob.numel()].copy_(blob, non_blocking=True)

    @torch.no_grad()
    def _run(self):
        pipeline.launch_raw_resize(self.static_images, self._blob, self.capacity, self.pixel_scale)
        return super()._run()

    def __call__(self, raw):
        """raw: a RawBatch of 1 .. capacity images -> (padded Detections of `capacity` rows, raw.scales)"""
        self._check_thresholds()
        self._check_raw(raw)
        self._load_raw(raw)
        self.graph.replay()
        return self.out, raw.scales
