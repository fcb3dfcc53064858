"""Pin tools/frame_oracle.py against what demo.py's Detect.process (demo.py:71-104) computes per frame.

  * the resize is OpenCV's own: cv2.resize(frame, (W, H), interpolation=INTER_LINEAR), which albumentations 0.5.2's
    Resize calls (a frame already of the target size is returned as is).  It runs with the default (optimized) code
    path, as albumentations calls it, and every case is rerun with cv2.setUseOptimized(False), which must agree.
  * Normalize and ToTensor are albumentations 0.5.2's lines (albumentations/augmentations/functional.py normalize,
    albumentations/pytorch/functional.py img_to_tensor), restated below: albumentations is not installed here.
  * the box and score expressions are cut out of demo.py with `ast` (its Assign statements at lines 88-91 and
    100-101) and executed unmodified on crafted float32 boxes and scores; demo.py itself cannot be imported (it needs
    albumentations, skimage and matplotlib and parses arguments at import).

The frames are regenerated from seeds (frame_oracle.synthetic_frames); the file keeps, per case, the geometry, the
input digest and the SHA-256 of each frame's float32 [3, H, W] output, and its first row.  A sweep of further
geometries checks the oracle against cv2 on both code paths without storing outputs.

usage: python tests/golden/make_frame_golden.py     (needs a checkout of the reference repository in EFFDET_REFERENCE)"""
import ast
import hashlib
import os
import sys

import cv2
import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = os.environ.get('EFFDET_REFERENCE')          # path of a checkout of the reference repository
assert REF, 'set EFFDET_REFERENCE to a checkout of the reference repository'
sys.path.insert(0, os.path.join(REPO, 'tools'))
import frame_oracle as F  # noqa: E402


def albu_normalize(img, mean, std, max_pixel_value=255.0):     # albumentations 0.5.2 functional.normalize
    mean = np.array(mean, dtype=np.float32)
    mean *= max_pixel_value
    std = np.array(std, dtype=np.float32)
    std *= max_pixel_value
    denominator = np.reciprocal(std, dtype=np.float32)
    img = img.astype(np.float32)
    img -= mean
    img *= denominator
    return img


def albu_to_tensor(im):                                          # albumentations 0.5.2 pytorch img_to_tensor
    return torch.from_numpy(np.moveaxis(im / (255.0 if im.dtype == np.uint8 else 1), -1, 0).astype(np.float32))


def reference_transform(frame, H, W):
    if frame.shape[:2] != (H, W):
        frame = cv2.resize(frame, (W, H), interpolation=cv2.INTER_LINEAR)
    return albu_to_tensor(albu_normalize(frame, F.MEAN, F.STD)).numpy()


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


# name: (seed, [(h, w)], (H, W))
CASES = {
    'vga_512': (31, [(480, 640)], (512, 512)),
    'hd_512': (32, [(720, 1280)], (512, 512)),
    'fullhd_512': (33, [(1080, 1920)], (512, 512)),
    'voc_512': (34, [(375, 500)], (512, 512)),
    'exact2x_512': (35, [(1024, 1024)], (512, 512)),
    'identity_512': (36, [(512, 512)], (512, 512)),
    'tiny_512': (37, [(7, 5), (1, 1), (1, 300), (300, 1)], (512, 512)),
    'mixed_512': (38, [(480, 640), (1, 1), (1024, 1024), (720, 1280), (7, 5), (512, 512), (375, 500), (300, 1)],
                  (512, 512)),
    'vga_384x640': (39, [(480, 640)], (384, 640)),
    'hd_384x640': (40, [(720, 1280)], (384, 640)),
    'fullhd_384x640': (41, [(1080, 1920)], (384, 640)),
    'mixed_384x640': (42, [(375, 500), (768, 1280), (384, 640), (1, 300), (7, 5)], (384, 640)),
}

out = {'cv2_version': np.array(cv2.__version__), 'numpy_version': np.array(np.__version__), 'cases': np.array(list(CASES))}
for name, (seed, sizes, (H, W)) in CASES.items():
    frames = F.synthetic_frames(seed, sizes)
    cv2.setUseOptimized(True)
    ref = np.stack([reference_transform(f, H, W) for f in frames])
    cv2.setUseOptimized(False)
    gen = np.stack([reference_transform(f, H, W) for f in frames])
    cv2.setUseOptimized(True)
    assert np.array_equal(ref, gen), 'optimized and generic cv2.resize differ (%s)' % name
    assert np.array_equal(ref, F.transform(frames, H, W)), 'oracle != reference (%s)' % name
    p = name + '/'
    out.update({p + 'seed': np.array([seed]), p + 'sizes': np.array(sizes, dtype=np.int32),
                p + 'target': np.array([H, W], dtype=np.int32),
                p + 'input_sha256': digest(np.concatenate([f.reshape(-1) for f in frames])),
                p + 'output_sha256': np.stack([digest(o) for o in ref]), p + 'first_row': ref[:, :, 0, :]})
    print('%-16s %-60s -> %dx%d: cv2 (both paths) == oracle' % (name, sizes, H, W))

# further geometries, checked and not stored: the oracle against cv2 on uniform noise, both code paths
rng = np.random.RandomState(43)
swept = 0
for h, w in [(1, 2), (2, 1), (2, 2), (3, 17), (33, 65), (100, 1000), (257, 129), (599, 801), (768, 768), (1536, 1536),
             (2000, 2000), (1200, 1600), (1, 1920), (1080, 1)]:
    img = rng.randint(0, 256, size=(h, w, 3)).astype(np.uint8)
    for H, W in [(512, 512), (384, 640), (128, 768), (768, 128), (h * 2, w * 2), (max(h // 2, 1), max(w // 2, 1))]:
        want = F.resize_u8(img, H, W)
        for opt in (True, False):
            cv2.setUseOptimized(opt)
            assert np.array_equal(cv2.resize(img, (W, H), interpolation=cv2.INTER_LINEAR), want), (h, w, H, W, opt)
            swept += 1
cv2.setUseOptimized(True)
print('sweep: %d further resizes equal the oracle' % swept)
out['sweep_count'] = np.array([swept])

# demo.py's box and score expressions, cut out of the file and executed as written
src = open(os.path.join(REF, 'demo.py')).read()
assigns = {}
for node in ast.walk(ast.parse(src)):
    if isinstance(node, ast.Assign) and node.lineno in (88, 89, 90, 91, 100):
        assigns[node.targets[0].id] = compile(ast.Expression(node.value), 'demo.py:%d' % node.lineno, 'eval')
assert sorted(assigns) == ['score', 'x1', 'x2', 'y1', 'y2'], sorted(assigns)


class _Detect:
    def __init__(self, size_image):
        self.size_image = size_image


class _Frame:
    def __init__(self, h, w):
        self.shape = (h, w, 3)


def demo_box(bbox, frame_hw, size_hw):
    env = {'bbox': np.asarray(bbox, dtype=np.float32), 'origin_img': _Frame(*map(int, frame_hw)),   # Python ints,
           'self': _Detect(tuple(map(int, size_hw))), 'np': np}                                     # as ndarray.shape
    return [int(eval(assigns[k], env)) for k in ('x1', 'y1', 'x2', 'y2')]


def demo_score(s):
    env = {'scores': torch.tensor([s], dtype=torch.float32), 'j': 0, 'np': np}
    return int(eval(assigns['score'], env))                    # bbox_scores.append(int(score)), demo.py:112


# boxes: at 0, at the network input's edge, random, and values where float32 and float64 arithmetic truncate apart
box_rng = np.random.RandomState(44)
geoms = [((480, 640), (512, 512)), ((720, 1280), (512, 512)), ((1080, 1920), (512, 512)), ((375, 500), (512, 512)),
         ((7, 5), (512, 512)), ((1, 300), (512, 512)), ((480, 640), (384, 640)), ((1080, 1920), (384, 640))]
b_in, b_hw, b_size = [], [], []
for hw, size in geoms:
    H, W = size
    b_in += [[0, 0, 0, 0], [W, H, W, H], [0, 0, W, H]]
    b_hw += [hw] * 3
    b_size += [size] * 3
    for _ in range(8):
        b_in.append(np.sort(box_rng.rand(2) * W).tolist()[:1] + np.sort(box_rng.rand(2) * H).tolist()[:1]
                    + [box_rng.rand() * W, box_rng.rand() * H])
        b_hw.append(hw)
        b_size.append(size)
    # truncation splits of this geometry: float32 neighbours of the box values whose outputs are integers
    near = (np.arange(hw[1] + 1, dtype=np.float64) * W / hw[1]).astype(np.float32)
    cand = np.concatenate([near, np.nextafter(near, np.float32(-1)), np.nextafter(near, np.float32(W + 1))])
    cand = cand[(cand >= 0) & (cand <= W)]
    x32 = np.trunc(cand * np.float32(hw[1]) / np.float32(W))
    x64 = np.trunc(cand.astype(np.float64) * hw[1] / W)
    for v in cand[x32 != x64][:3]:
        b_in.append([v, 0, v, H])
        b_hw.append(hw)
        b_size.append(size)
b_in = np.array(b_in, dtype=np.float32)
b_hw = np.array(b_hw, dtype=np.int32)
b_size = np.array(b_size, dtype=np.int32)
b_out = np.array([demo_box(b, hw, sz) for b, hw, sz in zip(b_in, b_hw, b_size)], dtype=np.int32)
b_f64 = np.concatenate([F.frame_boxes(b[None], [0], [0], hw, sz, float64=True)[0] for b, hw, sz in zip(b_in, b_hw, b_size)])
b_f32 = np.concatenate([F.frame_boxes(b[None], [0], [0], hw, sz)[0] for b, hw, sz in zip(b_in, b_hw, b_size)])
assert np.array_equal(b_out, b_f32), 'oracle != demo.py (boxes)'
split = (b_f64 != b_f32).any(axis=1)
assert split.sum() >= 8, 'too few float32 / float64 truncation splits: %d' % split.sum()
print('boxes: %d rows equal demo.py; %d where the NumPy 1.x (float64) reading truncates differently'
      % (len(b_in), split.sum()))

# scores: every k / 100 and its float32 neighbours, half-way points k / 100 + 0.005, and random scores
ks = np.arange(0, 101, dtype=np.float64)
base = np.concatenate([ks / 100, (ks[:-1] + 0.5) / 100]).astype(np.float32)
s_in = np.unique(np.concatenate([base, np.nextafter(base, np.float32(2)), np.nextafter(base, np.float32(-1)),
                                 box_rng.rand(200).astype(np.float32)]))
s_in = s_in[(s_in >= 0) & (s_in <= 1)]
s_out = np.array([demo_score(float(s)) for s in s_in], dtype=np.int32)
assert np.array_equal(s_out, F.frame_boxes(np.zeros((len(s_in), 4)), np.zeros(len(s_in)), s_in, (1, 1))[2])
naive = np.round(s_in.astype(np.float64) * 100).astype(np.int32)
print('scores: %d equal demo.py; %d differ from round(100 * s)' % (len(s_in), (naive != s_out).sum()))
assert (naive != s_out).sum() > 0
out.update({'boxes/in': b_in, 'boxes/frame_hw': b_hw, 'boxes/size_hw': b_size, 'boxes/out': b_out,
            'boxes/out_numpy1': b_f64, 'scores/in': s_in, 'scores/out': s_out})
np.savez_compressed(os.path.join(HERE, 'frame_transform.npz'), **out)
print('frame_transform.npz written with OpenCV', cv2.__version__, 'and NumPy', np.__version__)
