"""CPU restatement of demo.py's per-frame path (Detect.process, demo.py:71-104), written fresh in NumPy from the rules
below.  tests/test_frame_detect.py compares the device path (csrc/pipeline.cu effdet_frame_transform and
effdet_frame_boxes, models/pipeline.py frame_transform, models/graph_step.py GraphedFrameDetect) against it; it is pinned
to OpenCV 4.13.0 and to demo.py's own expressions by tests/golden/make_frame_golden.py -> tests/golden/frame_transform.npz.

  resize_u8        cv2.resize(img, (W, H), interpolation=INTER_LINEAR) of a uint8 [h,w,3] frame (CV_8UC3)
  normalize        albumentations 0.5.2 Normalize(mean, std, max_pixel_value=255) + ToTensor on the resized frame
  transform        get_augumentation(phase='test') + unsqueeze / stack: frames -> float32 [B,3,H,W]
  frame_boxes      demo.py:86-104 on one frame's kept detections -> int32 (x1, y1, x2, y2), labels, int32 scores

The resize rules (OpenCV's INTER_LINEAR for CV_8U, with and without its optimized code paths):
  * the same size: a copy (albumentations does not even call cv2.resize then);
  * both scale factors src/dst exactly 2 (within DBL_EPSILON): INTER_AREA's 2x2 box, (S00 + S01 + S10 + S11 + 2) >> 2;
  * otherwise, per axis, scale = 1.0 / (dst / src), f = float32((d + 0.5) * scale - 0.5), s = floor(f), f -= s in
    float32.  Columns: s < 0 gives (s, f) = (0, 0); s >= w - 1 gives (s, f) = (w - 1, 0) and the second tap index is
    clamped to w - 1.  Rows: f is kept; both row indices s and s + 1 are clamped into [0, h - 1].
    Fixed-point taps a0 = rint(float32((1 - f) * 2048)), a1 = rint(float32(f * 2048)) (round half to even), b0, b1
    likewise for rows.  H(r) = S[r][s] * a0 + S[r][s + 1] * a1 (int32, scale 2^11);
    out = clamp_u8((((H(r0) >> 4) * b0 >> 16) + ((H(r1) >> 4) * b1 >> 16) + 2) >> 2), arithmetic shifts: OpenCV's
    vector rounding, which is not the scalar (H(r0) * b0 + H(r1) * b1 + 2^21) >> 22.

Normalize (albumentations/augmentations/functional.py, 0.5.2): mean = float32(mean) * 255 and std = float32(std) * 255
as float32 arrays, den = reciprocal(std) in float32, then img = float32(u8); img -= mean; img *= den, each a float32
operation of its own.  ToTensor is moveaxis(img / 1, -1, 0).astype(float32), exact.  The channels stay in the frame's
BGR order: the demo applies the RGB mean and std to cv2.imread's BGR channels.
"""
import numpy as np

MEAN = (0.485, 0.456, 0.406)                         # datasets/augmentation.py:44-45
STD = (0.229, 0.224, 0.225)
DBL_EPSILON = np.finfo(np.float64).eps
COEF = 2048                                           # OpenCV's INTER_RESIZE_COEF_SCALE


def _taps(dst, src):
    """per output index: (s, f float32) before any clamping"""
    scale = 1.0 / (dst / src)
    f = ((np.arange(dst, dtype=np.float64) + 0.5) * scale - 0.5).astype(np.float32)
    s = np.floor(f).astype(np.int64)
    f = f - s.astype(np.float32)
    return s, f


def _fixed(f):
    """float32 tap weight -> (rint((1 - f) * 2048), rint(f * 2048)) as int64"""
    one = np.float32(1)
    a0 = np.rint((one - f) * np.float32(COEF)).astype(np.int64)
    a1 = np.rint(f * np.float32(COEF)).astype(np.int64)
    return a0, a1


def resize_u8(img, H, W):
    """img uint8 [h,w,3] -> uint8 [H,W,3], cv2.resize INTER_LINEAR for CV_8UC3"""
    h, w = img.shape[:2]
    if (h, w) == (H, W):
        return img.copy()
    src = img.astype(np.int64)
    if abs(1.0 / (W / w) - 2) < DBL_EPSILON and abs(1.0 / (H / h) - 2) < DBL_EPSILON:
        s = src[:2 * H, :2 * W]
        return ((s[0::2, 0::2] + s[0::2, 1::2] + s[1::2, 0::2] + s[1::2, 1::2] + 2) >> 2).astype(np.uint8)
    sx, fx = _taps(W, w)
    fx[sx < 0] = 0
    sx[sx < 0] = 0
    fx[sx >= w - 1] = 0
    sx[sx >= w - 1] = w - 1
    sx1 = np.minimum(sx + 1, w - 1)
    a0, a1 = _fixed(fx)
    hz = src[:, sx] * a0[None, :, None] + src[:, sx1] * a1[None, :, None]             # [h, W, 3], scale 2^11
    sy, fy = _taps(H, h)
    r0, r1 = np.clip(sy, 0, h - 1), np.clip(sy + 1, 0, h - 1)
    b0, b1 = _fixed(fy)
    v = (((hz[r0] >> 4) * b0[:, None, None]) >> 16) + (((hz[r1] >> 4) * b1[:, None, None]) >> 16)
    return np.clip((v + 2) >> 2, 0, 255).astype(np.uint8)


def normalize(img_u8, mean=MEAN, std=STD):
    """albumentations 0.5.2 Normalize + ToTensor: uint8 [H,W,3] -> float32 [3,H,W]"""
    m = np.array(mean, dtype=np.float32)
    m *= 255.0
    s = np.array(std, dtype=np.float32)
    s *= 255.0
    den = np.reciprocal(s, dtype=np.float32)
    img = img_u8.astype(np.float32)
    img -= m
    img *= den
    return np.moveaxis(img / 1, -1, 0).astype(np.float32)


def transform(frames, height=512, width=512):
    """get_augumentation(phase='test') on each uint8 [h,w,3] frame, stacked -> float32 [B,3,height,width]"""
    return np.stack([normalize(resize_u8(f, height, width)) for f in frames])


def frame_boxes(boxes, labels, scores, frame_hw, size_hw=(512, 512), float64=False):
    """demo.py:86-104 on one frame's kept detections: boxes float32 [n,4] in network-input pixels, labels [n], scores
    float32 [n]; frame_hw the frame's (h, w), size_hw demo's size_image (the network input's (H, W)).
    -> (int32 [n,4] (x1, y1, x2, y2), int64 [n] labels, int32 [n] scores).

    Box: int(bbox[k] * frame side / size side).  With NumPy >= 2 (NEP 50) bbox[k] is a float32 scalar and the Python
    ints stay weak, so the product and the quotient are float32 operations (the default).  float64=True is the NumPy
    1.x reading, where the scalar expression is evaluated in float64.
    Score: int(np.around(s, 2) * 100) = trunc(rint(s *f 100) /f 100 *f 100), float32 operations, rint half to even."""
    boxes = np.asarray(boxes, dtype=np.float32).reshape(-1, 4)
    scores = np.asarray(scores, dtype=np.float32).reshape(-1)
    h, w = frame_hw
    dt = np.float64 if float64 else np.float32
    side = np.array([w, h, w, h], dtype=dt)
    size = np.array([size_hw[1], size_hw[0], size_hw[1], size_hw[0]], dtype=dt)
    xy = np.trunc(boxes.astype(dt) * side / size).astype(np.int32)
    hundred = np.float32(100)
    sc = np.trunc(np.rint(scores * hundred) / hundred * hundred).astype(np.int32)
    return xy, np.asarray(labels, dtype=np.int64).reshape(-1), sc


def synthetic_frames(seed, sizes):
    """uint8 [h,w,3] frames regenerated from a seed (RandomState's stream is fixed across NumPy versions): a smooth
    gradient plus noise, so that neighbouring pixels are correlated as in a photograph and the interpolation is not
    dominated by full-range jumps"""
    rng = np.random.RandomState(seed)
    out = []
    for h, w in sizes:
        yy, xx = np.meshgrid(np.linspace(0, 1, h), np.linspace(0, 1, w), indexing='ij')
        base = np.stack([xx * 200, yy * 200, (xx + yy) * 100], axis=-1)
        noise = rng.randint(-60, 61, size=(h, w, 3))
        out.append(np.clip(base + noise, 0, 255).astype(np.uint8))
    return out
