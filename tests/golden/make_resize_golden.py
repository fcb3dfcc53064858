"""Pin tools/resize_oracle.py against the reference's OWN input chain.  datasets/augmentation.py cannot be imported here
(albumentations is not installed), so Normalizer, Augmenter, Resizer and collater are cut out of the reference file with
`ast` and executed unmodified; VOC's pixel encoding is the line of datasets/voc0712.py that produces it, executed from the
reference source.  Outputs -> tests/golden/pipeline_resize.npz.

Resizer calls cv2.resize on the float64 image.  The expected output is OpenCV's generic algorithm, so the reference runs
with cv2.setUseOptimized(False); the default (SIMD/IPP) path of the same OpenCV build is run too, and its digest and its
largest distance to the generic path are recorded per case, as well as the largest distance over a sweep of N(0,1)
images at common sizes 512, 768 and 1536.

The images are regenerated from seeds (resize_oracle.synthetic_batch), so the file holds, per case, the geometry, the
input digest, the SHA-256 of the float32 image batch, its first two rows and each image's last resized row, the
annotations and the scales.

usage: python tests/golden/make_resize_golden.py     (needs a checkout of the reference repository in EFFDET_REFERENCE)"""
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
import resize_oracle as R  # noqa: E402

tree = ast.parse(open(os.path.join(REF, 'datasets', 'augmentation.py')).read())
ns = {'np': np, 'torch': torch, 'cv2': cv2}
for node in tree.body:
    if getattr(node, 'name', None) in {'collater', 'Augmenter', 'Normalizer', 'Resizer'}:
        exec(compile(ast.Module([node], []), 'augmentation.py', 'exec'), ns)
voc_line = next(l.strip() for l in open(os.path.join(REF, 'datasets', 'voc0712.py')) if '/255.' in l)
assert voc_line == 'img = img.astype(np.float32)/255.', voc_line

# name: (seed, common size, VOC encoding, [(h, w)], flips, boxes per image)
CASES = {
    'voc_512': (11, 512, True, [(375, 500), (500, 375), (7, 5), (1, 1), (300, 1), (1, 300)],
                [True, False, True, False, True, True], [3, 1, 1, 0, 2, 1]),
    'coco_512': (12, 512, False, [(480, 640), (427, 640), (1024, 768), (384, 512)], [True, False, True, True], [4, 2, 0, 3]),
    'coco_512_elongated': (13, 512, False, [(300, 1200), (1200, 300), (2, 3), (375, 500)], [False, True, True, False],
                           [2, 1, 1, 2]),
    'voc_768': (14, 768, True, [(427, 640), (375, 500), (5, 7)], [True, False, False], [2, 3, 1]),
    'coco_768': (15, 768, False, [(480, 640), (1024, 768), (11, 13)], [False, True, True], [1, 0, 2]),
    'voc_512_no_boxes': (16, 512, True, [(333, 500), (12, 9)], [False, True], [0, 0]),
}


def reference(images, annots, flips, S, voc):
    samples = []
    for img, ann, fl in zip(images, annots, flips):
        if voc:
            env = {'np': np, 'img': img}
            exec(voc_line, env)                                    # datasets/voc0712.py:109
            img = env['img']
        s = ns['Normalizer']()({'img': img, 'annot': ann.copy()})
        if fl:
            s = ns['Augmenter']()(s, flip_x=2.0)                   # np.random.rand() < 2.0 -> always flips
        samples.append(ns['Resizer']()(s, common_size=S))
    imgs, ann = ns['collater'](samples)
    return imgs.float().numpy(), ann.numpy(), np.array([s['scale'] for s in samples], dtype=np.float64)


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


out = {'cv2_version': np.array(cv2.__version__), 'cases': np.array(list(CASES))}
for name, (seed, S, voc, sizes, flips, nbox) in CASES.items():
    images, annots = R.synthetic_batch(seed, sizes, nbox)
    cv2.setUseOptimized(False)
    imgs, ann, scales = reference(images, annots, flips, S, voc)
    o_imgs, o_ann, o_scales = R.normalize_resize_pad_collate(images, annots, flips, S, pixel_scale=255 if voc else None)
    assert np.array_equal(imgs, o_imgs), 'oracle != reference (images, %s)' % name
    assert np.array_equal(ann, o_ann) and np.array_equal(scales, o_scales), 'oracle != reference (annotations, %s)' % name
    cv2.setUseOptimized(True)
    opt, _, _ = reference(images, annots, flips, S, voc)
    rh = np.array([R.resizer_geometry(h, w, S)[1] for h, w in sizes])
    p = name + '/'
    out.update({p + 'seed': np.array([seed]), p + 'common': np.array([S]), p + 'voc': np.array([voc]),
                p + 'sizes': np.array(sizes, dtype=np.int32), p + 'flips': np.array(flips, dtype=np.uint8),
                p + 'n_boxes': np.array(nbox, dtype=np.int32),
                p + 'input_sha256': digest(np.concatenate([im.reshape(-1) for im in images])),
                p + 'images_sha256': digest(imgs), p + 'top_rows': imgs[:, :, :2, :],
                p + 'last_rows': np.stack([imgs[b, :, rh[b] - 1, :] for b in range(len(sizes))]),
                p + 'annots': ann, p + 'scales': scales,
                p + 'optimized_sha256': digest(opt), p + 'optimized_gap': np.array([np.abs(opt - imgs).max()])})
    print('%-20s S=%4d %s: reference == oracle; optimized cv2 differs by up to %.3g'
          % (name, S, 'VOC ' if voc else 'COCO', np.abs(opt - imgs).max()))

# the optimized path's distance on float64 N(0,1) images, per common size (Resizer geometry of each source size)
rng = np.random.RandomState(17)
sweep = []
for S in (512, 768, 1536):
    worst = 0.0
    for h, w in [(375, 500), (480, 640), (427, 640), (333, 500), (500, 353), (612, 612)]:
        img = rng.standard_normal((h, w, 3))
        _, rh, rw = R.resizer_geometry(h, w, S)
        cv2.setUseOptimized(False)
        gen = cv2.resize(img, (rw, rh))
        assert np.array_equal(gen, R.resize_linear(img, rh, rw)), (S, h, w)
        cv2.setUseOptimized(True)
        worst = max(worst, float(np.abs(cv2.resize(img, (rw, rh)) - gen).max()))
    sweep.append(worst)
    print('N(0,1) sweep S=%4d: generic == oracle; optimized cv2 differs by up to %.3g' % (S, worst))
cv2.setUseOptimized(True)
out['normal_sweep_common'] = np.array([512, 768, 1536])
out['normal_sweep_optimized_gap'] = np.array(sweep)
np.savez_compressed(os.path.join(HERE, 'pipeline_resize.npz'), **out)
print('pipeline_resize.npz written with OpenCV', cv2.__version__)
