"""Input-path timing on one GPU: the reference's per-image host chain (Normalizer -> Augmenter -> Resizer with
cv2.resize -> collater -> .cuda().float()) against DeviceCollater(resize=True), for a batch of VOC-sized (375x500) and
of COCO-sized (480x640) images.

  host    : wall clock of the chain per batch on this process's cores (OpenCV's default, optimized path, with its own
            thread pool), including the float64 host-to-device copy and the .float() on the device
  device  : CUDA events per batch around the copy of the uint8 bytes from pinned memory, effdet_resize_normalize_pad and
            effdet_collate_annots; the kernel's algorithmic bytes (uint8 read + fp32 [B,3,S,S] written) over its time
            against the H100 SXM data-sheet HBM3 bandwidth (3.35 TB/s)

The device output is checked bit for bit against tools/resize_oracle.py on the timed batch first.
usage: python tools/bench_input.py [--batch 32] [--common 512] [--reps 50] [--out FILE]
Prints one JSON line with the card name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import cv2
import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(REPO, 'efficientdet.pytorch_b200'), os.path.join(REPO, 'tools')):
    sys.path.insert(0, p)
import resize_oracle as R  # noqa: E402
from models import _native as N  # noqa: E402
from models.pipeline import MEAN, STD, DeviceCollater  # noqa: E402

HBM_TBS = 3.35


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
    return torch.cuda.get_device_name(0), q


def host_chain(images, annots, flips, S, voc, dev):
    """the reference's training transform and collate, per image, as train.py:176-196 and :105 run them"""
    mean, std = np.array([[MEAN]]), np.array([[STD]])
    imgs, anns = [], []
    for img, ann, fl in zip(images, annots, flips):
        x = img.astype(np.float32) / 255. if voc else img
        x = (x.astype(np.float32) - mean) / std
        ann = ann.copy()
        if fl:
            x = x[:, ::-1, :]
            x1 = ann[:, 0].copy()
            ann[:, 0] = x.shape[1] - ann[:, 2]
            ann[:, 2] = x.shape[1] - x1
        scale, rh, rw = R.resizer_geometry(x.shape[0], x.shape[1], S)
        new = np.zeros((S, S, 3))
        new[:rh, :rw] = cv2.resize(x, (rw, rh))
        ann[:, :4] *= scale
        imgs.append(new)
        anns.append(ann)
    batch = torch.from_numpy(np.stack(imgs, axis=0)).permute(0, 3, 1, 2)
    G = max(a.shape[0] for a in anns)
    pad = torch.ones((len(anns), max(G, 1), 5)) * -1
    for b, a in enumerate(anns):
        pad[b, :a.shape[0]] = torch.from_numpy(a)
    out = batch.to(dev).float(), pad.to(dev)
    torch.cuda.synchronize(dev)
    return out


def measure(label, h, w, B, S, voc, reps, dev):
    images, annots = R.synthetic_batch(5, [(h, w)] * B, [4] * B)
    flips = [b % 2 == 0 for b in range(B)]
    samples = [dict(img=im, annot=a, flip=f) for im, a, f in zip(images, annots, flips)]
    col = DeviceCollater(S, dev, resize=True, pixel_scale=255 if voc else None)
    got, ann = col(samples)
    want, want_ann, _ = R.normalize_resize_pad_collate(images, annots, flips, S, pixel_scale=255 if voc else None)
    exact = bool(np.array_equal(got.cpu().numpy(), want) and np.array_equal(ann.cpu().numpy(), want_ann))

    host_chain(images[:2], annots[:2], flips[:2], S, voc, dev)                    # warm-up
    host = []
    for _ in range(max(3, reps // 10)):
        t0 = time.perf_counter()
        host_chain(images, annots, flips, S, voc, dev)
        host.append(time.perf_counter() - t0)

    flat = torch.from_numpy(np.concatenate([im.reshape(-1) for im in images])).pin_memory()
    dst = torch.empty_like(flat, device=dev)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    for _ in range(5):
        dst.copy_(flat, non_blocking=True)
        col(samples)
    torch.cuda.synchronize(dev)
    h2d, kern, coll, wall = [], [], [], []
    for _ in range(reps):
        ev[0].record()
        dst.copy_(flat, non_blocking=True)
        ev[1].record()
        N.PROFILER = N.Profiler()
        t0 = time.perf_counter()
        col(samples)
        torch.cuda.synchronize(dev)
        wall.append(time.perf_counter() - t0)
        recs = {name: e0.elapsed_time(e1) for name, _, e0, e1 in N.PROFILER.recs}
        N.PROFILER = None
        h2d.append(ev[0].elapsed_time(ev[1]))
        kern.append(recs['effdet_resize_normalize_pad'])
        coll.append(recs['effdet_collate_annots'])
    med = lambda a: float(np.median(a))                                           # noqa: E731
    nbytes = flat.numel() + 4 * B * 3 * S * S
    k_ms = med(kern)
    return dict(case=label, h=h, w=w, batch=B, common=S, bit_exact_vs_oracle=exact,
                host_ms_per_batch=round(med(host) * 1e3, 2), host_ms_per_image=round(med(host) * 1e3 / B, 3),
                h2d_uint8_ms=round(med(h2d), 4), h2d_uint8_bytes=int(flat.numel()),
                resize_kernel_ms=round(k_ms, 4), collate_annots_ms=round(med(coll), 4),
                device_collater_wall_ms=round(med(wall) * 1e3, 3),
                kernel_bytes=int(nbytes), kernel_gb_per_s=round(nbytes / k_ms / 1e6, 1),
                kernel_hbm_fraction=round(nbytes / k_ms / 1e6 / (HBM_TBS * 1e3), 3),
                host_to_device_ratio=round(med(host) * 1e3 / (med(h2d) + k_ms + med(coll)), 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batch', type=int, default=32)
    ap.add_argument('--common', type=int, default=512)
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--out', default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_input.py measures on a GPU'
    dev = torch.device('cuda:0')
    name, power = card()
    res = dict(gpu=name, nvidia_smi=power, host_cores=len(os.sched_getaffinity(0)), cv2=cv2.__version__,
               cv2_threads=cv2.getNumThreads(), torch=torch.__version__,
               cases=[measure('voc', 375, 500, a.batch, a.common, True, a.reps, dev),
                      measure('coco', 480, 640, a.batch, a.common, False, a.reps, dev)])
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
