"""Device-side versions of the two steps that sit either side of the hot path in the reference's loops
(SURVEY.md 8(f) ranks 2 and 3), as thin host wrappers over csrc/pipeline.cu:

  DeviceCollater      Normalizer -> Augmenter flip -> [Resizer's cv2.resize] -> zero pad -> collater -> .cuda().float()
                      (datasets/augmentation.py:69-150; train.py:105-106): the DataLoader workers only decode to uint8;
                      everything else happens in two launches on the GPU, bit-identical to NumPy (and, with
                      resize=True, to OpenCV's generic INTER_LINEAR resize).
  select_detections   eval.py:105-128 after NMS: boxes /= scale, score threshold, top-100, per-label split, without
                      the three .cpu().numpy() round trips per image.
  frame_transform     demo.py's test transform (get_augumentation('test'): cv2.resize of the uint8 frame, Normalize,
                      ToTensor) + unsqueeze / stack + .to(device), in one launch; frame_boxes is demo.py's per-box
                      arithmetic on the padded detections.  GraphedFrameDetect (models/graph_step.py) runs both around
                      the network in one CUDA graph.
"""
import ctypes

import numpy as np
import torch

from . import _native as N

MEAN = (0.485, 0.456, 0.406)        # datasets/augmentation.py:144-145
STD = (0.229, 0.224, 0.225)


def resizer_geometry(h, w, common_size):
    """Resizer's host arithmetic (datasets/augmentation.py:99-107), in Python floats -> (scale, resized_h, resized_w)"""
    if h > w:
        scale = common_size / h
        return scale, common_size, int(w * scale)
    scale = common_size / w
    return scale, int(h * scale), common_size


def concat_pinned(imgs, staging=None):
    """uint8 arrays back to back in pinned host memory -> (flat pinned uint8 tensor, int64 [B] byte offsets).
    staging: a pinned uint8 tensor of at least the total size to write into, instead of a new allocation."""
    nbytes = [im.size for im in imgs]
    offs = np.concatenate([[0], np.cumsum(nbytes)[:-1]]).astype(np.int64)
    if staging is None:
        return torch.from_numpy(np.concatenate([im.reshape(-1) for im in imgs])).pin_memory(), offs
    flat = staging[:sum(nbytes)]
    np.concatenate([im.reshape(-1) for im in imgs], out=flat.numpy())
    return flat, offs


def check_samples(samples, S, resize, who, resize_who):
    """the sample checks of DeviceCollater and RawCollater -> (C-contiguous uint8 images, sizes int32 [B, 2], box scales
    float64 [B], resized sizes int32 [B, 2]).  Raises before anything is copied; who / resize_who name the caller in the
    messages (resize_who in the refusal of 'scale', which only the Resizer path makes)."""
    imgs = [np.ascontiguousarray(s['img']) for s in samples]
    for im in imgs:
        if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3 or im.shape[0] < 1 or im.shape[1] < 1 or \
                (not resize and (im.shape[0] > S or im.shape[1] > S)):
            raise N.EffdetNativeError('%s: images must be uint8 [h,w,3] with h,w >= 1%s, got %s %s'
                                      % (who, '' if resize else ' and <= %d' % S, im.dtype, im.shape))
    sizes = np.array([[im.shape[0], im.shape[1]] for im in imgs], dtype=np.int32)
    if resize:
        if any('scale' in s for s in samples):
            raise N.EffdetNativeError("%s: a sample carries 'scale', but the Resizer computes each image's scale "
                                      "itself" % resize_who)
        geo = [resizer_geometry(int(h), int(w), S) for h, w in sizes]
        for (h, w), (_, rh, rw) in zip(sizes, geo):
            if rh < 1 or rw < 1:
                raise N.EffdetNativeError('%s: a %dx%d image resizes to %dx%d at common size %d' % (who, h, w, rh, rw, S))
        scales = np.array([g[0] for g in geo], dtype=np.float64)
        resized = np.array([[g[1], g[2]] for g in geo], dtype=np.int32)
    else:
        scales = np.array([float(s.get('scale', 1.0)) for s in samples], dtype=np.float64)
        resized = sizes
    return imgs, sizes, scales, resized


class DeviceCollater:
    """collate_fn replacement: call with a list of samples {'img': uint8 [h,w,3] ndarray, 'annot': [n,5] float64 ndarray,
    optional 'flip': bool, optional 'scale': float}; returns (images float32 [B,3,S,S], annotations float32 [B,G,5])
    on `device` -- what train.py:105-106 hands to the model.

    resize=False (default): images enter at their final resolution (h, w <= S) and are only normalized, flipped and
      padded; a sample's 'scale' (default 1) scales its boxes.
    resize=True: the whole Normalizer -> Augmenter -> Resizer chain of train.py:176-196.  Images of any size are
      resized so the long side is S (cv2.resize INTER_LINEAR, OpenCV's generic algorithm, on the float64 normalized
      image), and the boxes are scaled by Resizer's scale.  A sample must not carry 'scale': the Resizer computes it.
    pixel_scale=None: the Normalizer's input is float32(u8), as CocoDataset delivers it.  pixel_scale=255: it is
      float32(u8) / 255, as VOCDetection delivers it (datasets/voc0712.py:109); pass the decoded uint8 image.
    return_scales=True: return (images, annotations, scales), scales a float64 [B] ndarray of the per-image box scales
      (eval.py's data['scale']), in the form VOCAccumulator.add() takes."""

    def __init__(self, common_size=512, device='cuda:0', resize=False, pixel_scale=None, return_scales=False):
        self.S = int(common_size)
        self.device = torch.device(device)
        self.resize = bool(resize)
        if pixel_scale not in (None, 255):
            raise N.EffdetNativeError('DeviceCollater: pixel_scale must be None (COCO) or 255 (VOC), got %r'
                                      % (pixel_scale,))
        self.pixel_scale = pixel_scale
        self.return_scales = bool(return_scales)
        self._mean = (ctypes.c_double * 3)(*MEAN)
        self._std = (ctypes.c_double * 3)(*STD)

    def __call__(self, samples):
        B, S, dev = len(samples), self.S, self.device
        imgs, sizes, scales, resized = check_samples(samples, S, self.resize, 'DeviceCollater',
                                                     'DeviceCollater(resize=True)')
        flat, offs = concat_pinned(imgs)
        flips = np.array([1 if s.get('flip') else 0 for s in samples], dtype=np.uint8)
        anns = [np.asarray(s['annot'], dtype=np.float64).reshape(-1, 5) for s in samples]
        counts = np.array([a.shape[0] for a in anns], dtype=np.int32)
        row_off = np.concatenate([[0], np.cumsum(counts)]).astype(np.int32)
        G = max(int(counts.max()), 1)                                  # collater: one all -1 row when nobody has boxes
        rows = np.concatenate(anns, axis=0) if counts.sum() else np.zeros((1, 5))
        d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=True)   # noqa: E731
        pix_d, offs_d, hw_d, flip_d = flat.to(dev, non_blocking=True), d(offs), d(sizes), d(flips)
        rows_d, roff_d, sc_d, w_d = d(rows), d(row_off), d(scales), d(sizes[:, 1].copy())
        out = torch.empty((B, 3, S, S), device=dev, dtype=torch.float32)
        ann = torch.empty((B, G, 5), device=dev, dtype=torch.float32)
        if self.resize or self.pixel_scale is not None:
            # without resize, resized == sizes: the kernel copies each image (cv2.resize to its own size is a copy)
            N.call('effdet_resize_normalize_pad', out, N.ptr(pix_d), N.ptr(offs_d), N.ptr(hw_d), N.ptr(d(resized)),
                   N.ptr(flip_d), N.f32(out), B, S, self.pixel_scale or 1, self._mean, self._std,
                   nbytes=float(flat.numel() + 4 * out.numel()))
        else:
            N.call('effdet_normalize_pad', out, N.ptr(pix_d), N.ptr(offs_d), N.ptr(hw_d), N.ptr(flip_d), N.f32(out), B, S,
                   self._mean, self._std, nbytes=float(flat.numel() + 4 * out.numel()))
        N.call('effdet_collate_annots', out, N.ptr(rows_d), N.ptr(roff_d), N.ptr(sc_d), N.ptr(flip_d), N.ptr(w_d), N.f32(ann),
               B, G)
        if self.return_scales:
            return out, ann, scales
        return out, ann


# ---- raw batches: what DataLoader workers hand to the graphed steps ---------------------------------------------------
RAW_HEADER = 8          # int64 header entries: B, pixel bytes, rows, layout capacity, common size, pixel scale, 0, 0
_MEAN64 = (ctypes.c_double * 3)(*MEAN)
_STD64 = (ctypes.c_double * 3)(*STD)


def raw_layout(capacity, rows, nbytes):
    """byte offset of every section of a raw batch whose per-image sections hold `capacity` images, with `rows`
    annotation rows and `nbytes` pixel bytes -> (dict name -> offset, total bytes).  Every section starts on a 16-byte
    boundary; the sections up to 'rows' depend on the capacity alone."""
    sizes = [('header', 8 * RAW_HEADER), ('offsets', 8 * capacity), ('hw', 8 * capacity), ('resized_hw', 8 * capacity),
             ('flips', capacity), ('scales', 8 * capacity), ('row_offsets', 4 * (capacity + 1)), ('rows', 40 * rows),
             ('pixels', nbytes)]
    off, at = {}, 0
    for name, n in sizes:
        off[name] = at
        at += (n + 15) // 16 * 16
    return off, at


_SECTIONS = {'header': (torch.int64, RAW_HEADER), 'offsets': (torch.int64, 1), 'hw': (torch.int32, 2),
             'resized_hw': (torch.int32, 2), 'flips': (torch.uint8, 1), 'scales': (torch.float64, 1),
             'row_offsets': (torch.int32, 1)}


def raw_section(blob, capacity, name):
    """a typed view of one fixed section of a raw batch (host or device) laid out for `capacity` images: header int64
    [8], offsets int64 [cap], hw / resized_hw int32 [cap, 2], flips uint8 [cap], scales float64 [cap], row_offsets
    int32 [cap + 1]"""
    off, _ = raw_layout(capacity, 0, 0)
    dtype, width = _SECTIONS[name]
    n = RAW_HEADER if name == 'header' else (capacity + 1 if name == 'row_offsets' else capacity * width)
    v = blob[off[name]:off[name] + n * dtype.itemsize].view(dtype)
    return v.reshape(capacity, width) if width == 2 else v


def _assemble(capacity, S, pixel_scale, sizes, resized, flips, scales, counts, rows, pixels, pin=False):
    """one raw batch blob laid out for `capacity` >= B images: entries b >= B of the per-image sections are zero (an
    image with h = 0 is padding to the resize kernel).  pixels: a list of uint8 arrays, back to back."""
    B = len(sizes)
    image_bytes = sizes[:, 0].astype(np.int64) * sizes[:, 1] * 3
    nbytes, R = int(image_bytes.sum()), int(counts.sum())
    off, total = raw_layout(capacity, R, nbytes)
    blob = torch.empty((total,), dtype=torch.uint8, pin_memory=pin)
    a = blob.numpy()
    p0 = off['pixels']
    a[:p0] = 0                                                   # header tail, row slots and padding: deterministic
    a[p0 + nbytes:] = 0

    def put(name, arr):
        arr = np.ascontiguousarray(arr).reshape(-1).view(np.uint8)
        a[off[name]:off[name] + arr.size] = arr

    put('header', np.array([B, nbytes, R, capacity, S, pixel_scale or 1, 0, 0], np.int64))
    put('offsets', p0 + np.concatenate([[0], np.cumsum(image_bytes)[:-1]]).astype(np.int64))   # from the blob's start
    put('hw', sizes.astype(np.int32))
    put('resized_hw', resized.astype(np.int32))
    put('flips', flips.astype(np.uint8))
    put('scales', scales.astype(np.float64))
    put('row_offsets', np.concatenate([[0], np.cumsum(counts)]).astype(np.int32))
    put('rows', rows.astype(np.float64))
    np.concatenate([np.asarray(p).reshape(-1) for p in pixels] or [np.zeros(0, np.uint8)], out=a[p0:p0 + nbytes])
    return RawBatch(blob, capacity, S, pixel_scale, counts, image_bytes, scales)


class RawBatch:
    """A batch as DataLoader workers can build it without CUDA: decoded uint8 images, the Resizer's geometry, the flips
    and the ragged annotation rows in ONE contiguous uint8 host tensor (`blob`), so that a graphed step needs one
    host-to-device copy.  Sections, each 16-byte aligned (raw_layout): header int64 [8] (B, pixel bytes, rows, layout
    capacity, common size, pixel scale), byte offsets int64 [cap] (from the blob's start), hw and resized_hw int32
    [cap, 2], flips uint8 [cap], Resizer scales float64 [cap], row offsets int32 [cap + 1], rows float64 [R, 5], pixels.
    A collated batch is laid out for its own B images (capacity == B).

    Host-side facts, for the capacity checks without a device read: B, counts (rows per image), image_bytes, nbytes,
    and scales (float64 [B], eval.py's data['scale'], as VOCAccumulator.add() takes them)."""

    def __init__(self, blob, capacity, S, pixel_scale, counts, image_bytes, scales):
        self.blob = blob
        self.capacity, self.S, self.pixel_scale = int(capacity), int(S), pixel_scale
        self.counts = np.asarray(counts, dtype=np.int32)
        self.image_bytes = np.asarray(image_bytes, dtype=np.int64)
        self.scales = np.asarray(scales, dtype=np.float64)
        self.B, self.nbytes, self.rows = len(self.counts), int(self.image_bytes.sum()), int(self.counts.sum())

    def __len__(self):
        return self.B

    @property
    def max_rows(self):
        """the most annotation rows of one image (what max_annotations must hold)"""
        return int(self.counts.max()) if self.B else 0

    @property
    def data_bytes(self):
        """bytes of the rows and pixel sections: the blob's size after its fixed, capacity-sized sections"""
        return (40 * self.rows + 15) // 16 * 16 + (self.nbytes + 15) // 16 * 16

    def section(self, name):
        return raw_section(self.blob, self.capacity, name)

    def pin_memory(self):
        """a copy in pinned memory (DataLoader(pin_memory=True) calls this in its pin thread)"""
        return RawBatch(self.blob.pin_memory(), self.capacity, self.S, self.pixel_scale, self.counts, self.image_bytes,
                        self.scales)

    def at_capacity(self, capacity, pin=False):
        """the same batch laid out for `capacity` >= B images (zero entries for the unused ones): what a graph captured
        for `capacity` images reads"""
        if capacity == self.capacity:
            return self
        B = self.B
        off, _ = raw_layout(self.capacity, self.rows, self.nbytes)
        a = self.blob.numpy()
        rows = a[off['rows']:off['rows'] + 40 * self.rows].view(np.float64).reshape(-1, 5)
        return _assemble(capacity, self.S, self.pixel_scale, self.section('hw')[:B].numpy(),
                         self.section('resized_hw')[:B].numpy(), self.section('flips')[:B].numpy(), self.scales,
                         self.counts, rows, [a[off['pixels']:off['pixels'] + self.nbytes]], pin=pin)


class RawCollater:
    """collate_fn for DataLoader workers: takes DeviceCollater(resize=True)'s samples ({'img': uint8 [h,w,3], 'annot':
    float64 [n,5], optional 'flip'}, no 'scale'), refuses what it refuses, and returns a RawBatch.  It never touches
    CUDA, so it runs in forked workers after the parent has initialised CUDA; GraphedTrainStep / GraphedRawDetect run
    the Normalizer -> Augmenter flip -> Resizer -> collater chain on the device, bit-identical to DeviceCollater.
    pixel_scale: None (COCO, float32(u8)) or 255 (VOC, float32(u8) / 255), as DeviceCollater."""

    def __init__(self, common_size=512, pixel_scale=None):
        if pixel_scale not in (None, 255):
            raise N.EffdetNativeError('RawCollater: pixel_scale must be None (COCO) or 255 (VOC), got %r' % (pixel_scale,))
        self.S, self.pixel_scale = int(common_size), pixel_scale

    def __call__(self, samples):
        imgs, sizes, scales, resized = check_samples(samples, self.S, True, 'RawCollater', 'RawCollater')
        flips = np.array([1 if s.get('flip') else 0 for s in samples], dtype=np.uint8)
        anns = [np.asarray(s['annot'], dtype=np.float64).reshape(-1, 5) for s in samples]
        counts = np.array([a.shape[0] for a in anns], dtype=np.int32)
        rows = np.concatenate(anns, axis=0) if counts.sum() else np.zeros((0, 5))
        return _assemble(len(samples), self.S, self.pixel_scale, sizes, resized, flips, scales, counts, rows, imgs)


def launch_raw_resize(out, blob, capacity, pixel_scale):
    """effdet_resize_normalize_pad of a raw batch in device memory laid out for `capacity` images into out float32
    [capacity, 3, S, S]; the geometry arguments point into the blob, and padding entries (h = 0) write zeros"""
    S = out.shape[2]
    sec = lambda name: raw_section(blob, capacity, name)               # noqa: E731
    N.call('effdet_resize_normalize_pad', out, N.ptr(blob), N.ptr(sec('offsets')), N.ptr(sec('hw')),
           N.ptr(sec('resized_hw')), N.ptr(sec('flips')), N.f32(out), capacity, S, pixel_scale or 1, _MEAN64, _STD64,
           nbytes=float(blob.numel() + 4 * out.numel()))


def launch_raw_pack(blob, capacity, annots, counts):
    """effdet_collate_pack_annots of a raw batch in device memory laid out for `capacity` images into the static table
    annots float32 [capacity, Gcap, 5] and counts int32 [1 + capacity]"""
    sec = lambda name: raw_section(blob, capacity, name)               # noqa: E731
    rows = blob[raw_layout(capacity, 0, 0)[0]['rows']:]
    N.call('effdet_collate_pack_annots', annots, N.ptr(sec('header')), N.ptr(rows), N.ptr(sec('row_offsets')),
           N.ptr(sec('scales')), N.ptr(sec('flips')), N.ptr(sec('hw')), N.f32(annots), N.ptr(counts), capacity,
           annots.shape[1])


def raw_images(raw, device='cuda:0'):
    """the images of a raw batch on the device, eagerly: float32 [B, 3, S, S], bit-identical to DeviceCollater(S,
    resize=True, pixel_scale=raw.pixel_scale)"""
    blob = raw.blob.to(device, non_blocking=raw.blob.is_pinned())
    out = torch.empty((raw.capacity, 3, raw.S, raw.S), device=blob.device, dtype=torch.float32)
    launch_raw_resize(out, blob, raw.capacity, raw.pixel_scale)
    return out[:raw.B]


def select_detections(scores, labels, boxes, scale, score_threshold=0.05, max_detections=100, num_classes=80):
    """eval.py:105-128 on the device.  scores [n] f32, labels [n] i64, boxes [n,4] f32 (the model's eval-mode output).
    -> (dets [m,5] f32 grouped by label, labels [m] i32, class_offsets [num_classes+1] i32): detections of label c are
    dets[class_offsets[c]:class_offsets[c+1]], each (x1,y1,x2,y2,score) with boxes already divided by scale."""
    dev = scores.device
    n = int(scores.numel())
    dets = torch.empty((max_detections, 5), device=dev, dtype=torch.float32)
    labs = torch.empty((max_detections,), device=dev, dtype=torch.int32)
    offs = torch.empty((num_classes + 1,), device=dev, dtype=torch.int32)
    cnt = torch.empty((1,), device=dev, dtype=torch.int32)
    sc = scores.contiguous() if n else None
    N.call('effdet_eval_select', dets, N.f32(sc, 'scores'), N.ptr(labels.contiguous() if n else None),
           N.f32(boxes.contiguous() if n else None, 'boxes'), n, float(scale), float(score_threshold), int(max_detections),
           int(num_classes), N.f32(dets), N.ptr(labs), N.ptr(offs), N.ptr(cnt))
    m = int(cnt.item())
    return dets[:m], labs[:m], offs


def check_frames(frames, who):
    """demo.py's frames as the device path takes them: a non-empty list of uint8 [h, w, 3] arrays with h, w >= 1
    (cv2.imread's BGR layout) -> the same frames as C-contiguous arrays.  Raises before anything is copied."""
    if isinstance(frames, np.ndarray) or not len(frames):
        raise N.EffdetNativeError('%s: frames must be a non-empty list of uint8 [h, w, 3] arrays' % who)
    out = []
    for f in frames:
        f = np.asarray(f)
        if f.dtype != np.uint8 or f.ndim != 3 or f.shape[2] != 3 or f.shape[0] < 1 or f.shape[1] < 1:
            raise N.EffdetNativeError('%s: frames must be uint8 [h, w, 3] with h, w >= 1, got %s %s'
                                      % (who, f.dtype, f.shape))
        out.append(np.ascontiguousarray(f))
    if len(out) > 65535:
        raise N.EffdetNativeError('%s: %d frames exceed 65535' % (who, len(out)))
    return out


_FRAME_MEAN = (ctypes.c_float * 3)(*MEAN)      # albumentations.Normalize's arguments, datasets/augmentation.py:44-45
_FRAME_STD = (ctypes.c_float * 3)(*STD)


def launch_frame_transform(out, pixels, offsets, hw):
    """effdet_frame_transform of the frames in device memory (pixels uint8, offsets int64 [B], hw int32 [B, 2], h == 0
    for padding) into out float32 [B, 3, H, W]"""
    B, _, H, W = out.shape
    N.call('effdet_frame_transform', out, N.ptr(pixels), N.ptr(offsets), N.ptr(hw), N.f32(out), B, H, W, _FRAME_MEAN,
           _FRAME_STD, nbytes=float(pixels.numel() + 4 * out.numel()))


def frame_transform(frames, height=512, width=512, device='cuda:0'):
    """demo.py's `self.transform(image=img)['image'].to(device).unsqueeze(0)` (demo.py:75-78) for a list of uint8
    [h, w, 3] BGR frames of any sizes -> float32 [B, 3, height, width] on `device`, bit-identical to albumentations
    0.5.2's Resize (OpenCV's uint8 INTER_LINEAR) + Normalize + ToTensor, stacked.  Eager: one launch."""
    frames = check_frames(frames, 'frame_transform')
    if not (1 <= int(height) <= 65535 and 1 <= int(width) <= 65535):
        raise N.EffdetNativeError('frame_transform: height=%r, width=%r must be in [1, 65535]' % (height, width))
    dev = torch.device(device)
    flat, offs = concat_pinned(frames)
    sizes = np.array([f.shape[:2] for f in frames], dtype=np.int32)
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev, non_blocking=True)   # noqa: E731
    out = torch.empty((len(frames), 3, int(height), int(width)), device=dev, dtype=torch.float32)
    launch_frame_transform(out, flat.to(dev, non_blocking=True), d(offs), d(sizes))
    return out


def frame_boxes(detections, hw, height, width):
    """demo.py:86-104 on padded detections (scores [B,C], classes [B,C] int64, boxes [B,C,4], count [B] int32, as
    GraphedDetect returns them) of frames hw int32 [B, 2] on the device, for a network input of height x width
    -> (rows int32 [B, C, 6] (x1, y1, x2, y2, label, score) valid below counts[b], counts int32 [B]: -1 for a frame that
    overflowed the candidate cap, 0 for a padding frame).  No host read: capturable."""
    scores, classes, boxes, count = detections
    B, C = scores.shape
    rows = torch.empty((B, C, 6), device=scores.device, dtype=torch.int32)
    counts = torch.empty((B,), device=scores.device, dtype=torch.int32)
    if classes.dtype != torch.int64 or count.dtype != torch.int32 or hw.dtype != torch.int32 or hw.numel() != 2 * B:
        raise N.EffdetNativeError('frame_boxes: classes must be int64, count and hw int32 [B] / [B, 2]')
    N.call('effdet_frame_boxes', scores, N.f32(scores, 'scores'), N.ptr(classes.contiguous()), N.f32(boxes, 'boxes'),
           N.ptr(count.contiguous()), N.ptr(hw.contiguous()), B, C, int(height), int(width), N.ptr(rows), N.ptr(counts))
    return rows, counts
