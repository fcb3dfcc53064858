"""Time class-aware post-processing on the GPU: the whole detect_batch at cap = A (every anchor may be a candidate) for
every class_nms x nms combination, alternating the modes in one run, with CUDA events.

Workloads: D0 512x512 at B = 32 with K = 20 and 80 at thresholds 0.05 and 0.01, and the D7 1536x1536 bench image
(K = 90, B = 1).  The class scores are seeded random sigmoid outputs, so nearly every pair passes the threshold: these
are worst cases for candidate counts, not a trained model's.  Also reported: GraphedDetect's replay per image (D0,
K = 20, threshold 0.05, seeded weights) in each mode, and the top-k kernels alone as achieved bytes per second (cls
bytes times the passes over cls, over kernel time) against the H100 SXM data sheet's 3.35 TB/s.

usage: python tools/bench_class_nms.py [--reps 5] [--out FILE.json]"""
import argparse
import json
import os
import subprocess
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(REPO, 'efficientdet.pytorch_b200'))
sys.path.insert(0, os.path.join(REPO, 'oracle'))

MODES = ('agnostic', 'per_class', 'multi_label')
METHODS = ('hard', 'linear', 'gaussian')
HBM_TBS = 3.35


def card():
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else 'unknown'


def inputs(B, A, K, seed):
    g = torch.Generator(device='cuda').manual_seed(seed)
    cls = torch.sigmoid(torch.randn((B, A, K), device='cuda', generator=g) - 2.0)
    reg = torch.randn((B, A, 4), device='cuda', generator=g) * 0.1
    return cls, reg


def timed(fn, reps):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    fn()
    torch.cuda.synchronize()
    ev[0].record()
    for _ in range(reps):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    ap.add_argument('--out', default=None, help='also write the results to this JSON file')
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_class_nms needs a GPU')
    from models import _native as N
    from models import _ops
    from models.module import Anchors
    res = dict(card=card(), rows=[], graphed=[], topk=[])
    print('card:', res['card'])
    work = [('D0 512', 32, 512, K, thr) for K in (20, 80) for thr in (0.05, 0.01)] + [('D7 1536', 1, 1536, 90, 0.05)]
    for name, B, S, K, thr in work:
        anchors = Anchors()(torch.zeros((1, 3, S, S), device='cuda'))
        A = anchors.reshape(-1, 4).shape[0]
        cls, reg = inputs(B, A, K, 7)
        times = {}
        for rep in range(args.reps):                     # modes alternate inside each repetition
            for mode in MODES:
                for nms in METHODS:
                    if name.startswith('D7') and nms != 'hard' and mode != 'multi_label':
                        continue                         # Soft-NMS over 400 k+ candidates: minutes per call
                    def run():
                        _ops.detect_batch(cls, reg, anchors, S, S, thr, 0.5, cap=A, nms=nms, class_nms=mode)
                    times.setdefault((mode, nms), []).append(timed(run, 1))
        for (mode, nms), ts in times.items():
            ts = sorted(ts)
            row = dict(work=name, B=B, K=K, threshold=thr, class_nms=mode, nms=nms, ms_median=round(ts[len(ts) // 2], 3),
                       ms_min=round(ts[0], 3), ms_max=round(ts[-1], 3))
            res['rows'].append(row)
            print(json.dumps(row))
        # the top-k kernels alone: passes over cls from the launch sequence's early exits
        kp = _ops.multi_label_slots(A, K, 5000)
        kpad = 1 << (kp - 1).bit_length()
        wsb = _ops._topk_workspace(B, A, K, kp)
        ws = torch.empty((wsb // 8,), device='cuda', dtype=torch.int64)
        o = [torch.empty((B, kp, 4), device='cuda'), torch.empty((B, kp), device='cuda'),
             torch.empty((B, kp), device='cuda', dtype=torch.int32), torch.empty((B, kpad), device='cuda', dtype=torch.int64),
             torch.empty((B,), device='cuda', dtype=torch.int32)]
        an = anchors.reshape(-1, 4).contiguous()

        def topk():
            N.call('effdet_detect_topk_batch', cls, N.f32(cls), N.f32(reg), N.f32(an), B, A, K, float(S), float(S),
                   float(thr), kp, kpad, ws.data_ptr(), wsb, N.f32(o[0]), N.f32(o[1]), o[2].data_ptr(), o[3].data_ptr(),
                   o[4].data_ptr())
        ms = timed(topk, 20)
        # TopkState.resolved (bytes 8..11 of each image's state): r resolved bits took max(1, passes to reach r)
        state = ws.view(torch.uint8)[B * 2048 * 4:].view(B, 32)[:, 8:12].contiguous().view(torch.int32).flatten()
        digits = [0, 11, 22, 32, 43, 54, 64]
        passes = sum(max(1, digits.index(r)) for r in state.tolist()) / B + 1      # histogram passes + compaction
        gbs = cls.numel() * 4 * passes / ms / 1e6
        row = dict(work=name, B=B, K=K, threshold=thr, topk_ms=round(ms, 3), passes_per_image=round(passes, 2),
                   gb_per_s=round(gbs, 1), hbm_frac=round(gbs / (HBM_TBS * 1e3), 3))
        res['topk'].append(row)
        print(json.dumps(row))
        del cls, reg, ws, o
        torch.cuda.empty_cache()
    # GraphedDetect replay per image
    import effdet_oracle as O
    from models import EfficientDet
    from models.graph_step import GraphedDetect
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    m.load_state_dict(O.init_state_dict(cfg, seed=3))
    m = m.cuda().eval()
    m.threshold = 0.05
    x = O.synthetic_batch(32, size=512, seed=8)[0].cuda()
    for mode in MODES:
        m.class_nms = mode
        det = GraphedDetect(m, x, max_candidates=None)
        ms = timed(lambda: det(x), 10)
        row = dict(work='GraphedDetect D0 (W 64, D 2) 512 B32 K20', class_nms=mode, ms_per_image=round(ms / 32, 3),
                   library_launches=det.library_launches)
        res['graphed'].append(row)
        print(json.dumps(row))
        del det
    if args.out:
        with open(args.out, 'w') as f:
            json.dump(res, f, indent=1)


if __name__ == '__main__':
    main()
