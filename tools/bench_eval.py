"""VOC evaluation timing on one GPU: the device accumulator (models/evaluation.py) against the host accumulation, and
evaluate() end to end against the reference-style loop (one image per forward, host selection and accumulation).

usage: python tools/bench_eval.py [--images 4952] [--e2e-images 256] [--batch 16]
Prints one JSON line with the card name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(REPO, 'efficientdet.pytorch_b200'), os.path.join(REPO, 'oracle'), os.path.join(REPO, 'tools')):
    sys.path.insert(0, p)
import effdet_oracle as O  # noqa: E402
import voc_eval_oracle as V  # noqa: E402
from models import EfficientDet, evaluation  # noqa: E402
from models._ops import Detections  # noqa: E402


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True).stdout.strip()
    return torch.cuda.get_device_name(0), q


def synthetic(n, K, per_image, seed=0):
    """padded detections (per_image rows, all above the threshold) and 1..4 ground-truth boxes per image"""
    rng = np.random.RandomState(seed)
    scores = rng.uniform(0.06, 1.0, size=(n, per_image)).astype(np.float32)
    scores = -np.sort(-scores, axis=1)
    labels = rng.randint(0, K, size=(n, per_image)).astype(np.int64)
    xy = rng.uniform(0, 400, size=(n, per_image, 2))
    boxes = np.concatenate([xy, xy + rng.uniform(10, 100, size=(n, per_image, 2))], axis=2).astype(np.float32)
    gts = []
    for i in range(n):
        g = rng.randint(1, 5)
        pick = rng.randint(0, per_image, size=g)
        gts.append(np.concatenate([boxes[i, pick] + rng.normal(0, 4, size=(g, 4)), labels[i, pick, None]], axis=1))
    return scores, labels, boxes, np.full(n, per_image, np.int32), np.ones(n, np.float32), gts


def accumulation(n, K, batch, reps=3):
    scores, labels, boxes, count, scale, gts = synthetic(n, K, 100)
    dets = [V.select_detections(scores[i], labels[i], boxes[i], 1.0, 0.05, 100, K) for i in range(n)]
    anns = [[g[g[:, 4] == c, :4] for c in range(K)] for g in gts]
    t0 = time.perf_counter()
    host = V.evaluate(dets, anns, K)
    host_s = time.perf_counter() - t0
    d = torch.device('cuda:0')
    batches = [Detections(*(torch.from_numpy(a[i:i + batch]).to(d) for a in (scores, labels, boxes, count)))
               for i in range(0, n, batch)]

    def run():
        acc = evaluation.VOCAccumulator(K, n, device=d)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t = time.perf_counter()
        e0.record()
        for j, b in enumerate(batches):
            acc.add(b, [1.0] * b.scores.shape[0], gts[j * batch:(j + 1) * batch])
        res = acc.compute()                                           # ends in the one read, i.e. a synchronise
        e1.record()
        torch.cuda.synchronize()
        return res, time.perf_counter() - t, e0.elapsed_time(e1) / 1e3

    run()                                                             # warm-up
    times = [run() for _ in range(reps)]
    res = times[0][0]
    assert res[0] == host[0] and all(res[1][c] == host[1][c] for c in range(K)), 'device != host'
    return dict(images=n, classes=K, records=n * 100, host_s=round(host_s, 3),
                device_wall_s=round(min(t[1] for t in times), 4), device_event_s=round(min(t[2] for t in times), 4))


class Gen:
    def __init__(self, n, K, size, seed=1):
        g = torch.Generator().manual_seed(seed)
        self.imgs = [torch.randn(size, size, 3, generator=g) for _ in range(n)]
        rng = np.random.RandomState(seed)
        self.anns = []
        for _ in range(n):
            k = rng.randint(1, 5)
            xy = rng.uniform(0, size - 64, size=(k, 2))
            self.anns.append(np.concatenate([xy, xy + rng.uniform(16, 64, size=(k, 2)), rng.randint(0, K, size=(k, 1))],
                                            axis=1).astype(np.float64))
        self.K = K

    def __len__(self):
        return len(self.imgs)

    def __getitem__(self, i):
        return {'img': self.imgs[i], 'scale': 1.0}

    def load_annotations(self, i):
        return self.anns[i]

    def num_classes(self):
        return self.K

    def label_to_name(self, label):
        return str(label)


def end_to_end(n, batch, size=512, K=20):
    cfg = O.make_config('efficientdet-d0', num_classes=K, W_bifpn=64, D_bifpn=2)
    m = EfficientDet(num_classes=K, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    m.load_state_dict(O.init_state_dict(cfg, seed=1, mode='wellcond'))
    m = m.cuda().eval()
    m.threshold = 0.3
    gen = Gen(n, K, size)
    warm = Gen(batch + 3, K, size, seed=2)
    devnull = open(os.devnull, 'w')
    out, sys.stdout = sys.stdout, devnull
    try:
        evaluation.evaluate(warm, m, batch_size=batch)                 # warm-up: graph capture, allocator, modules
        V.evaluate(V.get_detections(warm, m), V.get_annotations(warm), K)
        torch.cuda.synchronize()
        t = time.perf_counter()
        got = evaluation.evaluate(gen, m, batch_size=batch)
        dev_s = time.perf_counter() - t
        t = time.perf_counter()
        ref = V.evaluate(V.get_detections(gen, m), V.get_annotations(gen), K)
        ref_s = time.perf_counter() - t
    finally:
        sys.stdout = out
    return dict(images=n, size=size, batch=batch, evaluate_img_s=round(n / dev_s, 1), reference_loop_img_s=round(n / ref_s, 1),
                mean_ap_device=float(got[0]), mean_ap_reference_loop=float(ref[0]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=4952)
    ap.add_argument('--classes', type=int, default=20)
    ap.add_argument('--e2e-images', type=int, default=256)
    ap.add_argument('--batch', type=int, default=16)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_eval.py needs a GPU')
    name, q = card()
    res = dict(card=name, nvidia_smi=q, accumulation=accumulation(a.images, a.classes, a.batch),
               end_to_end=end_to_end(a.e2e_images, a.batch))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
