"""Pin tools/jitter_oracle.py against the reference's OWN input chain at a drawn common size.  As in
make_resize_golden.py, Normalizer, Augmenter and Resizer are cut out of datasets/augmentation.py with `ast` and executed
unmodified (albumentations is not installed, so the module cannot be imported), VOC's pixel encoding is the line of
datasets/voc0712.py that produces it, and cv2 runs with setUseOptimized(False) (OpenCV's generic resize).  Each image
goes through Resizer.__call__(sample, common_size=L); the S x S window at (y0, x0) is sliced from its L x L output
afterwards, zero-padded where it runs past it, and cast with .float().  Its boxes are the Resizer's (flipped, scaled),
shifted by (x0, y0), clamped to [0, S] in float64, cast to float32, and dropped when their label is -1 or their float32
area is zero.  Outputs -> tests/golden/pipeline_jitter.npz.

The images are regenerated from seeds (resize_oracle.synthetic_batch; every third row gets label -1), so the file holds,
per case, the geometry (drawn and raised L, resized sizes, scales, windows), the input digest, the SHA-256 of the float32
window batch, each window's first two rows and its last row inside the resized image, and the packed boxes with their
counts.

usage: python tests/golden/make_jitter_golden.py     (needs a checkout of the reference repository in EFFDET_REFERENCE)"""
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
import jitter_oracle as J  # noqa: E402
import resize_oracle as R  # noqa: E402

tree = ast.parse(open(os.path.join(REF, 'datasets', 'augmentation.py')).read())
ns = {'np': np, 'torch': torch, 'cv2': cv2}
for node in tree.body:
    if getattr(node, 'name', None) in {'Augmenter', 'Normalizer', 'Resizer'}:
        exec(compile(ast.Module([node], []), 'augmentation.py', 'exec'), ns)
voc_line = next(l.strip() for l in open(os.path.join(REF, 'datasets', 'voc0712.py')) if '/255.' in l)
assert voc_line == 'img = img.astype(np.float32)/255.', voc_line

# name: (seed, S, VOC encoding, [(h, w)], flips, boxes per image, drawn L per image, window per image)
# window: 'origin' (0, 0), 'far' (rh - S, rw - S), 'mid' (half of those), or (y0, x0)
CASES = {
    'voc_L_below_S': (21, 512, True, [(375, 500), (500, 375), (7, 5)], [1, 0, 1], [4, 3, 2], [300, 400, 200],
                      ['origin'] * 3),
    'coco_L_equal_S': (22, 512, False, [(480, 640), (427, 640)], [0, 1], [4, 3], [512, 512], ['origin'] * 2),
    'coco_L_above_S_windows': (23, 256, False, [(375, 500)] * 3, [0, 1, 0], [9, 9, 9], [512] * 3,
                               ['origin', 'far', 'mid']),
    'voc_L_above_S_windows': (28, 384, True, [(480, 640), (640, 480)], [1, 0], [7, 7], [700, 600], ['far', 'mid']),
    'voc_upscale_1024': (24, 512, True, [(375, 500)], [1], [12], [1024], ['mid']),
    'coco_box2x_crop': (25, 512, False, [(2048, 1536), (2048, 1536)], [0, 1], [6, 6], [1024, 1024],
                        [(300, 200), 'far']),
    'voc_copy_crop': (26, 512, True, [(700, 600)], [1], [6], [700], [(100, 50)]),
    'coco_raise_L': (27, 512, False, [(1, 700), (900, 2), (40, 30)], [0, 1, 1], [2, 2, 2], [300, 100, 9],
                     ['far', 'mid', 'origin']),
}


def geometry(h, w, L, S, where):
    """the raise of L (smallest valid common size >= L, found by stepping), the Resizer's geometry, the window"""
    while min(R.resizer_geometry(h, w, L)[1:]) < 1:
        L += 1
    scale, rh, rw = R.resizer_geometry(h, w, L)
    far = (max(rh - S, 0), max(rw - S, 0))
    y0, x0 = {'origin': (0, 0), 'far': far, 'mid': (far[0] // 2, far[1] // 2)}.get(where, where) \
        if isinstance(where, str) else where
    assert 0 <= y0 <= far[0] and 0 <= x0 <= far[1], (h, w, L, where)
    return L, scale, rh, rw, y0, x0


def reference(img, ann, fl, voc, L, S, y0, x0):
    if voc:
        env = {'np': np, 'img': img}
        exec(voc_line, env)                                        # datasets/voc0712.py:109
        img = env['img']
    s = ns['Normalizer']()({'img': img, 'annot': ann.copy()})
    if fl:
        s = ns['Augmenter']()(s, flip_x=2.0)                       # np.random.rand() < 2.0 -> always flips
    r = ns['Resizer']()(s, common_size=L)
    full = r['img'].numpy()
    win = np.zeros((S, S, 3))
    part = full[y0:y0 + S, x0:x0 + S]
    win[:part.shape[0], :part.shape[1]] = part
    a = r['annot'].numpy().copy()
    a[:, [0, 2]] = np.clip(a[:, [0, 2]] - x0, 0, S)
    a[:, [1, 3]] = np.clip(a[:, [1, 3]] - y0, 0, S)
    f = a.astype(np.float32)
    keep = (f[:, 4] != -1) & (f[:, 2] > f[:, 0]) & (f[:, 3] > f[:, 1])
    return torch.from_numpy(win).permute(2, 0, 1).float().numpy(), f[keep], r['scale']


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


def case_inputs(seed, sizes, nbox):
    images, annots = R.synthetic_batch(seed, sizes, nbox)
    for a in annots:
        a[2::3, 4] = -1
    return images, annots


out = {'cv2_version': np.array(cv2.__version__), 'cases': np.array(list(CASES))}
cv2.setUseOptimized(False)
for name, (seed, S, voc, sizes, flips, nbox, drawn, where) in CASES.items():
    images, annots = case_inputs(seed, sizes, nbox)
    geo = [geometry(h, w, L, S, wh) for (h, w), L, wh in zip(sizes, drawn, where)]
    wins, kept, last = [], [], []
    for b, (img, ann, fl) in enumerate(zip(images, annots, flips)):
        L, scale, rh, rw, y0, x0 = geo[b]
        win, k, ref_scale = reference(img, ann, fl, voc, L, S, y0, x0)
        assert ref_scale == scale, name
        o_win = J.crop_image(img, fl, rh, rw, y0, x0, S, 255 if voc else None)
        o_k = J.crop_boxes(ann, fl, img.shape[1], scale, y0, x0, S)
        assert np.array_equal(win, o_win), 'oracle != reference (images, %s, %d)' % (name, b)
        assert np.array_equal(k, o_k), 'oracle != reference (boxes, %s, %d)' % (name, b)
        wins.append(win)
        kept.append(k)
        last.append(win[:, max(min(rh - y0, S), 1) - 1, :])
    wins = np.stack(wins)
    table, counts = J.pack(kept, len(sizes), max(1, max(len(k) for k in kept)))
    p = name + '/'
    out.update({p + 'seed': np.array([seed]), p + 'common': np.array([S]), p + 'voc': np.array([voc]),
                p + 'sizes': np.array(sizes, dtype=np.int32), p + 'flips': np.array(flips, dtype=np.uint8),
                p + 'n_boxes': np.array(nbox, dtype=np.int32), p + 'drawn_L': np.array(drawn, dtype=np.int32),
                p + 'L': np.array([g[0] for g in geo], dtype=np.int32),
                p + 'scales': np.array([g[1] for g in geo], dtype=np.float64),
                p + 'resized': np.array([g[2:4] for g in geo], dtype=np.int32),
                p + 'crops': np.array([g[4:6] for g in geo], dtype=np.int32),
                p + 'input_sha256': digest(np.concatenate([im.reshape(-1) for im in images])),
                p + 'images_sha256': digest(wins), p + 'top_rows': wins[:, :, :2, :], p + 'last_rows': np.stack(last),
                p + 'annots': table, p + 'counts': counts})
    print('%-24s S=%4d %s L=%s windows=%s kept=%s: reference == oracle'
          % (name, S, 'VOC ' if voc else 'COCO', [g[0] for g in geo], [g[4:6] for g in geo], counts[1:].tolist()))
cv2.setUseOptimized(True)
np.savez_compressed(os.path.join(HERE, 'pipeline_jitter.npz'), **out)
print('pipeline_jitter.npz written with OpenCV', cv2.__version__)
