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
        imgs = [np.ascontiguousarray(s['img']) for s in samples]
        for im in imgs:
            if im.dtype != np.uint8 or im.ndim != 3 or im.shape[2] != 3 or im.shape[0] < 1 or im.shape[1] < 1 or \
                    (not self.resize and (im.shape[0] > S or im.shape[1] > S)):
                raise N.EffdetNativeError('DeviceCollater: images must be uint8 [h,w,3] with h,w >= 1%s, got %s %s'
                                          % ('' if self.resize else ' and <= %d' % S, im.dtype, im.shape))
        sizes = np.array([[im.shape[0], im.shape[1]] for im in imgs], dtype=np.int32)
        if self.resize:
            if any('scale' in s for s in samples):
                raise N.EffdetNativeError("DeviceCollater(resize=True): a sample carries 'scale', but the Resizer "
                                          "computes each image's scale itself")
            geo = [resizer_geometry(int(h), int(w), S) for h, w in sizes]
            for (h, w), (_, rh, rw) in zip(sizes, geo):
                if rh < 1 or rw < 1:
                    raise N.EffdetNativeError('DeviceCollater: a %dx%d image resizes to %dx%d at common size %d'
                                              % (h, w, rh, rw, S))
            scales = np.array([g[0] for g in geo], dtype=np.float64)
            resized = np.array([[g[1], g[2]] for g in geo], dtype=np.int32)
        else:
            scales = np.array([float(s.get('scale', 1.0)) for s in samples], dtype=np.float64)
            resized = sizes
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
