"""Soft-NMS timing against hard NMS, one process, reading the card's name and power limit in the same run.

  post     D0 512x512 bs 32 (bench.py's d0 model, seeded weights) at thresholds 0.05 and 0.01: _ops.detect_batch
           post-processing (candidates + sort + NMS, capped output, no host read) with nms = hard / linear / gaussian,
           the three alternated, CUDA events around each call.
  graph    GraphedDetect replay (network + post-processing) per image at D0 512x512 bs 32, threshold 0.05, per method.
  d7       the D7 1536x1536 bench image (bench.py --config d7: threshold 0.4) post-processed with each method.
  oracle   tools/soft_nms_oracle.py's host time on image 0 of the D0 batch at threshold 0.05, per soft method.

Soft-NMS costs about picks x live candidates, so every row reports candidates (sum and largest image) and rows
written (picks for soft-NMS, kept boxes for hard NMS) beside its time.
  python tools/bench_soft_nms.py [--reps 5] [--no-d7] [--out FILE.json]
"""
import argparse
import json
import os
import subprocess
import sys
import time

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(R, 'efficientdet.pytorch_b200'), os.path.join(R, 'oracle'), os.path.join(R, 'tools'), R]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import bench  # noqa: E402
import effdet_oracle as O  # noqa: E402
import soft_nms_oracle as S  # noqa: E402
from models import EfficientDet, _ops  # noqa: E402
from models.graph_step import GraphedDetect  # noqa: E402

METHODS = (('hard', 0.5), ('linear', 0.5), ('gaussian', 0.5))


def _card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else 'unknown'


def _model(name, threshold):
    c = bench.CONFIGS[name]
    cfg = O.make_config(c['net'], c['K'], c['W'], c['D'])
    m = EfficientDet(num_classes=c['K'], network=c['net'], D_bifpn=c['D'], W_bifpn=c['W'], is_training=False,
                     threshold=threshold, iou_threshold=0.5)
    m.load_state_dict(O.init_state_dict(cfg, seed=0))
    return m.to(torch.device('cuda', 0)).eval(), c


def _event_ms(fn, reps):
    """median device ms of fn over reps calls, CUDA events around each"""
    out = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return float(np.median(out))


def _post_rows(cls, reg, anchors, size, thr, reps, label):
    counts = (cls.max(dim=2)[0] > thr).sum(dim=1).tolist()
    cap = _ops.candidate_cap(None, cls)
    rows, times = {}, {m: [] for m, _ in METHODS}
    for nms, sigma in METHODS:                                     # warm-up and rows written
        d = _ops.detect_batch(cls, reg, anchors, size, size, thr, 0.5, cap=cap, nms=nms, sigma=sigma)
        rows[nms] = int(d.count.clamp(min=0).sum())
    for _ in range(reps):                                          # the methods alternated
        for nms, sigma in METHODS:
            times[nms].append(_event_ms(lambda: _ops.detect_batch(cls, reg, anchors, size, size, thr, 0.5, cap=cap,
                                                                  nms=nms, sigma=sigma), 1))
    return [dict(case=label, threshold=thr, nms=nms, candidates_sum=int(sum(counts)), candidates_max=int(max(counts)),
                 rows=rows[nms], ms=round(float(np.median(times[nms])), 3)) for nms, _ in METHODS]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--no-d7', action='store_true')
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    dev = torch.device('cuda', 0)
    res = dict(card=_card(), post=[], graph=[], d7=[], oracle=[])
    m, c = _model('d0', 0.05)
    x = bench.synthetic(c, 32, seed=1000)[0].to(dev)
    with torch.no_grad():
        cls, reg, anchors = m._raw_predictions(x)
        for thr in (0.05, 0.01):
            res['post'] += _post_rows(cls, reg, anchors, 512, thr, args.reps, 'd0 512 bs32')
        for nms, sigma in METHODS:
            m.nms, m.soft_nms_sigma = nms, sigma
            det = GraphedDetect(m, x, max_candidates=None)
            out = det(x)
            torch.cuda.synchronize()
            ms = _event_ms(lambda: det(x), args.reps)
            res['graph'].append(dict(case='d0 512 bs32 GraphedDetect', threshold=0.05, nms=nms,
                                     rows=int(out.count.clamp(min=0).sum()), ms_per_image=round(ms / 32, 3)))
            del det, out
        cand = [t.cpu().numpy() for t in _ops_candidates(cls[:1], reg[:1], anchors, 512, 0.05)]
        for nms, sigma in METHODS[1:]:
            t0 = time.perf_counter()
            s = S.soft_nms_candidates(*cand, 0, nms, 0.5, sigma, 0.05)[0]
            res['oracle'].append(dict(case='d0 512 image 0 NumPy oracle', threshold=0.05, nms=nms,
                                      candidates=int(cand[3][0]), rows=int(len(s)),
                                      host_ms=round((time.perf_counter() - t0) * 1e3, 1)))
    del m, x, cls, reg
    torch.cuda.empty_cache()
    if not args.no_d7:
        m7, c7 = _model('d7', 0.4)
        x7 = bench.synthetic(c7, 1, seed=1000)[0].to(dev)
        with torch.no_grad():
            cls7, reg7, a7 = m7._raw_predictions(x7)
            res['d7'] = _post_rows(cls7, reg7, a7, 1536, 0.4, max(2, args.reps // 2), 'd7 1536 bench image')
    res['card_after'] = _card()
    print(json.dumps(res, indent=1))
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


def _ops_candidates(cls, reg, anchors, size, thr):
    """effdet_detect_candidates_batch's outputs (boxes, scores, classes, count, keys) for the oracle"""
    N = _ops.N
    B, A, K = cls.shape
    npad = 1 << (A - 1).bit_length()
    boxes = torch.empty((B, A, 4), device=cls.device)
    scores = torch.empty((B, A), device=cls.device)
    classes = torch.empty((B, A), device=cls.device, dtype=torch.int32)
    keys = torch.empty((B, npad), device=cls.device, dtype=torch.int64)
    count = torch.empty((B,), device=cls.device, dtype=torch.int32)
    N.call('effdet_detect_candidates_batch', cls, N.f32(cls.contiguous()), N.f32(reg.contiguous()),
           N.f32(anchors.reshape(-1, 4).contiguous()), N.f32(boxes), N.f32(scores), classes.data_ptr(), keys.data_ptr(),
           count.data_ptr(), B, A, K, npad, float(size), float(size), float(thr))
    return boxes, scores, classes, count, keys


if __name__ == '__main__':
    main()
