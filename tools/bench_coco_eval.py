"""COCO box evaluation on the device (models.evaluation.COCOAccumulator / evaluate_coco) against the host.

  (a) accumulation of a val2017-sized synthetic set (5,000 images, 80 categories, ~300 detections and ~7 ground truths
      per image, 5 % crowd): COCOAccumulator add() + compute() on the device, timed with a host clock that ends in a
      synchronise; the NumPy oracle (tools/coco_eval_oracle.py) on the host over the first --oracle-images images; and
      pycocotools' COCOeval on the same subset when it is importable.
  (b) evaluate_coco on D0 at 512x512 against the reference-style loop (one image per forward, host collection, the
      oracle's COCOeval), both over --e2e-images images, with the same stats.
Warm-up first, then the device and host sides alternated --repeats times; prints one JSON line with the card's name
and power limit.

usage: python tools/bench_coco_eval.py [--repeats 3] [--oracle-images 200] [--e2e-images 64]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(REPO, 'efficientdet.pytorch_b200'), os.path.join(REPO, 'oracle'),
                os.path.join(REPO, 'tools'), os.path.join(REPO, 'tests'), REPO]
import coco_eval_oracle as O  # noqa: E402


def synthetic(n_img, K=80, dets=300, seed=0):
    from test_coco_eval import _random_set
    return _random_set(n_img=n_img, K=K, seed=seed, C=dets)


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def device_accumulate(inst, ids, lm, scores, labels, boxes, count, scale, batch=16):
    from models.evaluation import COCOAccumulator
    from models._ops import Detections
    dev = torch.device('cuda:0')
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)          # noqa: E731
    S, L, B, Cn = t(scores), t(labels), t(boxes), t(count)                   # detections already on the device
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    acc = COCOAccumulator(inst, ids, lm.__getitem__, num_labels=len(lm), device=dev)
    for i0 in range(0, len(ids), batch):
        i1 = min(len(ids), i0 + batch)
        acc.add(Detections(S[i0:i1], L[i0:i1], B[i0:i1], Cn[i0:i1]), [float(s) for s in scale[i0:i1]])
    out = acc.compute()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def host_oracle(inst, ids, lm, scores, labels, boxes, count, scale, n):
    t0 = time.perf_counter()
    res = []
    for i in range(n):
        res += O.collect(ids[i], scores[i, :count[i]], labels[i, :count[i]], boxes[i, :count[i]], float(scale[i]),
                         lm.__getitem__)
    sub = dict(inst, images=inst['images'][:n])
    keep = set(ids[:n])
    sub['annotations'] = [a for a in inst['annotations'] if a['image_id'] in keep]
    out = O.evaluate(sub, res, ids[:n])
    return time.perf_counter() - t0, out, sub, res


def pycoco(sub, res, ids):
    try:
        from pycocotools.coco import COCO
        from pycocotools.cocoeval import COCOeval
    except ImportError:
        return None
    t0 = time.perf_counter()
    gt = COCO()
    gt.dataset = sub
    gt.createIndex()
    E = COCOeval(gt, gt.loadRes(res), 'bbox')
    E.params.imgIds = list(ids)
    E.evaluate()
    E.accumulate()
    E.summarize()
    return time.perf_counter() - t0


def e2e(n_img, repeats):
    import effdet_oracle as EO
    from models import EfficientDet, evaluation
    from test_coco_eval import _CocoDataset, _reference_evaluate_coco
    K = 80
    from bench import CONFIGS
    d0 = CONFIGS['d0']
    cfg = EO.make_config(d0['net'], K, d0['W'], d0['D'])
    m = EfficientDet(num_classes=K, network=d0['net'], D_bifpn=d0['D'], W_bifpn=d0['W'], is_training=False)
    m.load_state_dict(EO.init_state_dict(cfg, seed=1, mode='wellcond'))
    m = m.to('cuda:0').eval()
    x = EO.synthetic_batch(n_img, size=512, seed=7)[0]
    images = [x[i].permute(1, 2, 0).contiguous() for i in range(n_img)]
    ids = list(range(1000, 1000 + n_img))
    rng = np.random.RandomState(2)
    anns = [{'id': j + 1, 'image_id': ids[j % n_img], 'category_id': 2 * int(rng.randint(K)) + 1,
             'bbox': [float(v) for v in rng.uniform(0, 300, size=2)] + [float(v) for v in rng.uniform(8, 200, size=2)],
             'area': 1000.0, 'iscrowd': 0} for j in range(7 * n_img)]
    inst = {'images': [{'id': i} for i in ids], 'categories': [{'id': 2 * k + 1} for k in range(K)],
            'annotations': anns}
    ds = _CocoDataset(images, [1.0] * n_img, inst, ids, K)
    ref = _reference_evaluate_coco()
    dev_t, host_t, stats = [], [], None
    cwd = os.getcwd()
    with tempfile.TemporaryDirectory() as tmp:
        os.chdir(tmp)
        try:
            for r in range(repeats + 1):
                m.eval()
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                got = evaluation.evaluate_coco(ds, m, batch_size=16, max_records=20000 * n_img)
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                m.eval()
                _, want = ref(ds, m)
                torch.cuda.synchronize()
                t2 = time.perf_counter()
                if r:                                                          # the first round is the warm-up
                    dev_t.append(t1 - t0)
                    host_t.append(t2 - t1)
                stats = (got, want[0])
        finally:
            os.chdir(cwd)
    # random ground truth: a TP decision can sit on the last-bit noise between two network passes
    return dev_t, host_t, float(np.abs(np.asarray(stats[0]) - np.asarray(stats[1])).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--images', type=int, default=5000)
    ap.add_argument('--repeats', type=int, default=3)
    ap.add_argument('--oracle-images', type=int, default=200)
    ap.add_argument('--e2e-images', type=int, default=64)
    a = ap.parse_args()
    from models import _native
    _native.build()
    inst, ids, lm, *arrs = synthetic(a.images)
    records = int(arrs[3].sum())
    device_accumulate(inst, ids, lm, *arrs)                                  # warm-up
    dev_t, host_t, py_t = [], [], []
    for _ in range(a.repeats):
        dt, _ = device_accumulate(inst, ids, lm, *arrs)
        ht, _, sub, res = host_oracle(inst, ids, lm, *arrs, a.oracle_images)
        dev_t.append(dt)
        host_t.append(ht)
        p = pycoco(sub, res, ids[:a.oracle_images])
        if p is not None:
            py_t.append(p)
    e_dev, e_host, e_diff = e2e(a.e2e_images, a.repeats)
    print(json.dumps({'card': card(), 'images': a.images, 'records': records,
                      'device_accumulate_s': [round(v, 4) for v in dev_t],
                      'oracle_images': a.oracle_images, 'oracle_s': [round(v, 3) for v in host_t],
                      'pycocotools_s': [round(v, 3) for v in py_t] or 'not installed',
                      'e2e_images': a.e2e_images, 'evaluate_coco_s': [round(v, 3) for v in e_dev],
                      'reference_loop_s': [round(v, 3) for v in e_host], 'e2e_max_stats_diff': e_diff}))


if __name__ == '__main__':
    main()
