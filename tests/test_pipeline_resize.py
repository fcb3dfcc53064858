"""The input chain with Resizer (datasets/augmentation.py:94-150, train.py:105): tools/resize_oracle.py against the
fixture generated from the reference's own code with OpenCV's generic resize (tests/golden/make_resize_golden.py), and --
on the GPU -- DeviceCollater(resize=True) (csrc/pipeline.cu effdet_resize_normalize_pad) against the same fixture, bit
for bit, for both pixel encodings and every geometry in it."""
import ctypes
import hashlib
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'tools'))
import resize_oracle as R  # noqa: E402

G = os.path.join(HERE, 'golden')


def _fixture():
    return np.load(os.path.join(G, 'pipeline_resize.npz'))


def _sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


def _case(st, name):
    p = name + '/'
    sizes = [tuple(int(v) for v in s) for s in st[p + 'sizes']]
    images, annots = R.synthetic_batch(int(st[p + 'seed'][0]), sizes, [int(n) for n in st[p + 'n_boxes']])
    assert np.array_equal(_sha(np.concatenate([im.reshape(-1) for im in images])), st[p + 'input_sha256'])
    return (images, annots, [bool(f) for f in st[p + 'flips']], int(st[p + 'common'][0]),
            255 if bool(st[p + 'voc'][0]) else None)


def _check(st, name, imgs, ann, scales):
    p = name + '/'
    sizes = st[p + 'sizes']
    S = int(st[p + 'common'][0])
    rh = [R.resizer_geometry(int(h), int(w), S)[1] for h, w in sizes]
    assert imgs.dtype == np.float32 and imgs.shape == (len(sizes), 3, S, S)
    assert np.array_equal(imgs[:, :, :2, :], st[p + 'top_rows']), name
    assert np.array_equal(np.stack([imgs[b, :, rh[b] - 1, :] for b in range(len(sizes))]), st[p + 'last_rows']), name
    assert np.array_equal(_sha(imgs), st[p + 'images_sha256']), name
    assert ann.dtype == np.float32 and np.array_equal(ann, st[p + 'annots']), name
    assert np.array_equal(np.asarray(scales, dtype=np.float64), st[p + 'scales']), name


def test_oracle_equals_reference_fixture():
    st = _fixture()
    names = [str(n) for n in st['cases']]
    assert len(names) == 6 and str(st['cv2_version'])
    geometries = set()
    for name in names:
        images, annots, flips, S, enc = _case(st, name)
        imgs, ann, scales = R.normalize_resize_pad_collate(images, annots, flips, S, pixel_scale=enc)
        _check(st, name, imgs, ann, scales)
        geometries |= {(im.shape[0], im.shape[1], S) for im in images}
    # the geometries the fixture is there to cover: upscale, downscale, exact 2x, identity, elongated, 1-pixel sides
    for g in [(375, 500, 512), (7, 5, 512), (480, 640, 512), (427, 640, 512), (1024, 768, 512), (384, 512, 512),
              (300, 1200, 512), (300, 1, 512), (1, 300, 512), (1, 1, 512), (427, 640, 768)]:
        assert g in geometries, g


def test_oracle_resize_rules():
    """the branches of resize_linear on hand-checkable inputs"""
    img = np.arange(4 * 6 * 3, dtype=np.float64).reshape(4, 6, 3) * 0.5
    assert np.array_equal(R.resize_linear(img, 4, 6), img)                               # same size: a copy
    half = R.resize_linear(img, 2, 3)                                                    # exact 2x: 2x2 box mean
    assert np.array_equal(half[1, 2], (((img[2, 4] + img[2, 5]) + img[3, 4]) + img[3, 5]) * 0.25)
    one = R.resize_linear(img[:, :1], 8, 1)                                              # a 1-pixel-wide column
    assert one.shape == (8, 1, 3) and np.allclose(one[:, 0, 0], np.interp((np.arange(8) + 0.5) / 2 - 0.5,
                                                                          np.arange(4), img[:, 0, 0]))


def test_resizer_geometry_matches_reference_arithmetic():
    from models.pipeline import resizer_geometry
    for h, w, S in [(375, 500, 512), (500, 375, 512), (333, 333, 512), (1, 700, 512), (300, 1200, 768), (7, 5, 1536)]:
        assert resizer_geometry(h, w, S) == R.resizer_geometry(h, w, S)
    assert resizer_geometry(333, 333, 512)[1:] == (int(333 * (512 / 333)), 512)       # h == w takes the width branch


def test_argument_refusals_before_launch():
    """the C entry point and DeviceCollater refuse bad arguments before anything touches the device, so these calls
    run without a GPU"""
    from models import _native
    from models._native import EffdetNativeError
    from models.pipeline import DeviceCollater
    _native.build()
    lib = _native.load()
    fake = 1 << 20
    m3 = (ctypes.c_double * 3)(1.0, 1.0, 1.0)
    assert lib.effdet_resize_normalize_pad(fake, fake, fake, None, fake, fake, 1, 512, 1, m3, m3, 0, None) == -1
    assert 'resize_normalize_pad' in lib.effdet_last_error().decode()
    assert lib.effdet_resize_normalize_pad(fake, fake, fake, fake, fake, fake, 1, 512, 7, m3, m3, 0, None) == -1
    assert 'pixel_scale 7' in lib.effdet_last_error().decode()
    assert lib.effdet_resize_normalize_pad(fake, fake, fake, fake, fake, fake, 0, 512, 1, m3, m3, 0, None) == -1

    ok = np.zeros((4, 5, 3), np.uint8)
    box = np.zeros((0, 5))
    col = DeviceCollater(512, resize=True, pixel_scale=255)
    bad = [np.zeros((4, 5, 3), np.float32), np.zeros((4, 5, 2), np.uint8), np.zeros((4, 5), np.uint8),
           np.zeros((0, 5, 3), np.uint8), np.zeros((4, 0, 3), np.uint8),
           np.zeros((1, 700, 3), np.uint8)]                                 # Resizer: int(1 * 512 / 700) == 0 rows
    for im in bad:
        with pytest.raises(EffdetNativeError):
            col([dict(img=ok, annot=box), dict(img=im, annot=box)])
    with pytest.raises(EffdetNativeError, match='scale'):
        col([dict(img=ok, annot=box, scale=1.0)])
    with pytest.raises(EffdetNativeError, match='pixel_scale'):
        DeviceCollater(512, resize=True, pixel_scale=256)
    with pytest.raises(EffdetNativeError, match='<= 512'):                  # without resize: larger images refused
        DeviceCollater(512, pixel_scale=255)([dict(img=np.zeros((513, 5, 3), np.uint8), annot=box)])


@pytest.mark.gpu
def test_device_collater_resize_bit_exact():
    from models.pipeline import DeviceCollater
    st = _fixture()
    for name in [str(n) for n in st['cases']]:
        images, annots, flips, S, enc = _case(st, name)
        samples = [dict(img=im, annot=a, flip=f) for im, a, f in zip(images, annots, flips)]
        imgs, ann, scales = DeviceCollater(S, 'cuda:0', resize=True, pixel_scale=enc, return_scales=True)(samples)
        _check(st, name, imgs.cpu().numpy(), ann.cpu().numpy(), scales)
        want, _, _ = R.normalize_resize_pad_collate(images, annots, flips, S, pixel_scale=enc)
        assert np.array_equal(imgs.cpu().numpy(), want), name
        # the default return value is the pair, as without resize
        pair = DeviceCollater(S, 'cuda:0', resize=True, pixel_scale=enc)(samples)
        assert len(pair) == 2 and torch.equal(pair[0], imgs) and torch.equal(pair[1], ann)


@pytest.mark.gpu
def test_device_collater_without_resize_unchanged():
    """resize=False keeps the pad-only path and its output (tests/golden/pipeline_input.npz); with pixel_scale=255 it
    pads VOC-encoded images, each copied at its own size"""
    from models.pipeline import DeviceCollater
    st = np.load(os.path.join(G, 'pipeline_input.npz'))
    images, off = [], 0
    for h, w in st['sizes']:
        images.append(st['pixels'][off:off + h * w * 3].reshape(h, w, 3))
        off += h * w * 3
    annots, r = [], 0
    for n in st['ann_counts']:
        annots.append(st['ann_rows'][r:r + n])
        r += n
    flips = [bool(f) for f in st['flips']]
    S = int(st['common'][0])
    samples = [dict(img=im, annot=a, flip=f) for im, a, f in zip(images, annots, flips)]
    imgs, ann = DeviceCollater(common_size=S, device='cuda:0')(samples)
    assert np.array_equal(imgs.cpu().numpy(), st['out_images']) and np.array_equal(ann.cpu().numpy(), st['out_annots'])
    imgs, ann, sc = DeviceCollater(common_size=S, device='cuda:0', pixel_scale=255, return_scales=True)(samples)
    want = np.zeros((len(images), S, S, 3))
    for b, im in enumerate(images):
        v = R.normalize(im, 255)
        want[b, :im.shape[0], :im.shape[1]] = v[:, ::-1] if flips[b] else v
    assert np.array_equal(imgs.cpu().numpy(), want.transpose(0, 3, 1, 2).astype(np.float32))
    assert np.array_equal(ann.cpu().numpy(), st['out_annots']) and np.array_equal(sc, np.ones(len(images)))


@pytest.mark.gpu
def test_d0_train_step_from_device_collater():
    """one D0 512x512 training step fed by DeviceCollater(resize=True) and by the oracle's batch: the batches are equal
    bit for bit, so the step computes the same losses and gradients.  Two passes of the network over the same batch may
    differ in the last bits (the SE means are fp32 atomics), hence bounds of 1e-5 on the losses and 1e-3 of each
    gradient's largest entry."""
    import effdet_oracle as O
    from models import EfficientDet
    from models.pipeline import DeviceCollater
    dev = torch.device('cuda:0')
    sizes = [(375, 500), (480, 640)]
    images, annots = R.synthetic_batch(21, sizes, [3, 2])
    flips = [True, False]
    imgs, ann = DeviceCollater(512, 'cuda:0', resize=True, pixel_scale=255)(
        [dict(img=im, annot=a, flip=f) for im, a, f in zip(images, annots, flips)])
    w_imgs, w_ann, _ = R.normalize_resize_pad_collate(images, annots, flips, 512, pixel_scale=255)
    assert np.array_equal(imgs.cpu().numpy(), w_imgs) and np.array_equal(ann.cpu().numpy(), w_ann)

    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
    m.load_state_dict(O.init_state_dict(cfg, seed=5))
    m = m.to(dev).eval()                                      # drop-connect off: both steps see the same function
    m.is_training = True

    def step(x, a):
        m.zero_grad(set_to_none=True)
        cl, rl = m([x, a])
        (cl.mean() + rl.mean()).backward()
        return cl.detach().item(), rl.detach().item(), [p.grad.detach().clone() for p in m.parameters() if p.grad is not None]

    c1, r1, g1 = step(imgs, ann)
    c2, r2, g2 = step(torch.from_numpy(w_imgs).to(dev), torch.from_numpy(w_ann).to(dev))
    assert r1 > 0 and c1 > 0 and len(g1) == len(g2) > 0
    assert abs(c1 - c2) <= 1e-5 * abs(c2) and abs(r1 - r2) <= 1e-5 * abs(r2), (c1, c2, r1, r2)
