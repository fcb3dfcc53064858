"""CPU restatement of the reference's training-time input chain with its resize, written fresh in NumPy from the rules
below.  tests/test_pipeline_resize.py compares the device path (csrc/pipeline.cu effdet_resize_normalize_pad,
models/pipeline.py DeviceCollater(resize=True)) against it; it is pinned to the reference's own code (with OpenCV's
generic, non-optimized resize) by tests/golden/make_resize_golden.py -> tests/golden/pipeline_resize.npz.

  resizer_geometry             Resizer's host arithmetic (datasets/augmentation.py:99-107): scale and resized size
  resize_linear                cv2.resize(img, (rw, rh)) of a float64 [h,w,3] image, INTER_LINEAR, generic path
  normalize_resize_pad_collate Normalizer -> Augmenter flip -> Resizer -> collater -> .float()  (train.py:105)

The resize rules (OpenCV's INTER_LINEAR for CV_64FC3 without SIMD or IPP):
  * the same size: a copy;
  * both scale factors src/dst exactly 2 (within DBL_EPSILON): the 2x2 box mean ((S00 + S01) + S10) + S11) * 0.25;
  * otherwise, per output column, scale = 1.0 / (dst / src), f = float32((d + 0.5) * scale - 0.5), s = floor(f),
    f -= s in float32, coefficients (1 - f, f) in float32 used as float64.  Columns: s < 0 gives (s, f) = (0, 0);
    s + 1 >= w makes the column single-tap (D = S[s]), with (s, f) = (w - 1, 0) when s >= w - 1.  Rows: f is NOT
    clamped; both row indices s and s + 1 are clamped into [0, h - 1], so the first and last rows of an upscale are
    H(0) * (1 - f) + H(0) * f, which can differ from H(0) in the last bit.
  * the horizontal pass runs on the two source rows, the vertical pass combines them: H(r0) * b0 + H(r1) * b1, every
    product and sum rounded separately in float64.
"""
import numpy as np

MEAN = np.array([[[0.485, 0.456, 0.406]]])          # datasets/augmentation.py:144-145 (float64)
STD = np.array([[[0.229, 0.224, 0.225]]])
DBL_EPSILON = np.finfo(np.float64).eps


def resizer_geometry(h, w, common_size):
    """datasets/augmentation.py:99-107 with Python floats -> (scale, resized_height, resized_width)"""
    if h > w:
        scale = common_size / h
        return scale, common_size, int(w * scale)
    scale = common_size / w
    return scale, int(h * scale), common_size


def _taps(dst, src):
    """per output index: (s, f float32, single-tap mask) before any clamping"""
    scale = 1.0 / (dst / src)
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = f - s.astype(np.float32)
    return s, f


def resize_linear(img, rh, rw):
    """img float64 [h,w,3] -> float64 [rh,rw,3]"""
    h, w = img.shape[:2]
    if (h, w) == (rh, rw):
        return img.copy()
    if abs(1.0 / (rw / w) - 2) < DBL_EPSILON and abs(1.0 / (rh / h) - 2) < DBL_EPSILON:
        s = img[:2 * rh, :2 * rw]
        return (((s[0::2, 0::2] + s[0::2, 1::2]) + s[1::2, 0::2]) + s[1::2, 1::2]) * 0.25
    sx, fx = _taps(rw, w)
    fx[sx < 0] = 0
    sx[sx < 0] = 0
    single = sx + 1 >= w
    fx[sx >= w - 1] = 0
    sx[sx >= w - 1] = w - 1
    ax0 = (np.float32(1) - fx).astype(np.float64)[None, :, None]
    ax1 = fx.astype(np.float64)[None, :, None]
    sx1 = np.minimum(sx + 1, w - 1)
    hz = np.where(single[None, :, None], img[:, sx], img[:, sx] * ax0 + img[:, sx1] * ax1)      # [h, rw, 3]
    sy, fy = _taps(rh, h)
    r0, r1 = np.clip(sy, 0, h - 1), np.clip(sy + 1, 0, h - 1)
    by0 = (np.float32(1) - fy).astype(np.float64)[:, None, None]
    by1 = fy.astype(np.float64)[:, None, None]
    return hz[r0] * by0 + hz[r1] * by1


def normalize(img_u8, pixel_scale=None):
    """Normalizer on the dataset's pixels: float32(u8) (COCO) or float32(u8) / 255 in float32 (VOC) -> float64"""
    x = img_u8.astype(np.float32)
    if pixel_scale is not None:
        x = x / np.float32(pixel_scale)
    return (x - MEAN) / STD


def synthetic_batch(seed, sizes, n_boxes):
    """the fixture's inputs, regenerated from a seed (RandomState's stream is fixed across NumPy versions): uint8
    [h,w,3] images and float64 [n,5] boxes (x1,y1,x2,y2,label) inside each image"""
    rng = np.random.RandomState(seed)
    images, annots = [], []
    for (h, w), n in zip(sizes, n_boxes):
        images.append(rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8))
        xs, ys = np.sort(rng.rand(n, 2) * w, axis=1), np.sort(rng.rand(n, 2) * h, axis=1)
        annots.append(np.concatenate([xs[:, :1], ys[:, :1], xs[:, 1:], ys[:, 1:],
                                      rng.randint(0, 20, size=(n, 1)).astype(np.float64)], axis=1))
    return images, annots


def normalize_resize_pad_collate(images_u8, annots, flips, common_size, pixel_scale=None):
    """images_u8: list of [h,w,3] uint8; annots: list of [n,5] float64; flips: list of bool; pixel_scale: None (COCO)
    or 255 (VOC).  -> (float32 [B,3,S,S], float32 [B,G,5], float64 [B] scales)"""
    S = common_size
    B = len(images_u8)
    imgs, anns, scales = [], [], []
    for b in range(B):
        img = normalize(images_u8[b], pixel_scale)
        ann = np.asarray(annots[b], dtype=np.float64).reshape(-1, 5).copy()
        if flips[b]:                                                          # Augmenter
            img = img[:, ::-1, :]
            cols = img.shape[1]
            x1, x2 = ann[:, 0].copy(), ann[:, 2].copy()
            ann[:, 0] = cols - x2
            ann[:, 2] = cols - x1
        scale, rh, rw = resizer_geometry(img.shape[0], img.shape[1], S)       # Resizer
        new = np.zeros((S, S, 3))
        new[:rh, :rw] = resize_linear(img, rh, rw)
        ann[:, :4] *= scale
        imgs.append(new)
        anns.append(ann)
        scales.append(scale)
    G = max(a.shape[0] for a in anns)                                         # collater
    pad = np.ones((B, max(G, 1), 5), dtype=np.float32) * -1
    for b, a in enumerate(anns):
        if a.shape[0] > 0:
            pad[b, :a.shape[0], :] = a
    stacked = np.stack(imgs, axis=0)
    return stacked.transpose(0, 3, 1, 2).astype(np.float32), pad, np.array(scales, dtype=np.float64)
