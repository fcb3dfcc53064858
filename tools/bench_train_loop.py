"""Time the graphed training micro-step at bench.py's D0 geometry (512x512, batch 32, 80 classes, train mode:
drop-connect on, BatchNorm frozen) with and without the optimizer in the CUDA graph:

  graph_no_optimizer  GraphedTrainStep(model, ...)                                    (bench.py's configuration)
  fused_update_every  GraphedTrainStep(..., optimizer=FusedClipAdamW), update=True on every call
  fused_k4            the same, update=(idx + 1) % 4 == 0                       (--grad_accumulation_steps 4)
  fused_no_update     the same, update=False on every call: the cost of a micro-step between two updates (captured
                      weight packing / BatchNorm folding, the accumulation and the early-exiting optimizer launches)

The configurations are timed in alternating rounds with CUDA events; the card's name and power limit are read in the
same run.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, os.path.join(ROOT, 'efficientdet.pytorch_b200'))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import effdet_oracle as O                            # noqa: E402
from models import EfficientDet                      # noqa: E402
from models.fused_optim import FusedClipAdamW        # noqa: E402
from models.graph_step import GraphedTrainStep       # noqa: E402


def card():
    out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--bs', type=int, default=32)
    ap.add_argument('--size', type=int, default=512)
    ap.add_argument('--steps', type=int, default=20, help='micro-steps per configuration and round (multiple of 4)')
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_train_loop needs a GPU')
    dev = torch.device('cuda:0')
    torch.manual_seed(0)
    cfg = O.make_config('efficientdet-d0', 80, 64, 2)
    sd = O.init_state_dict(cfg, seed=0)
    images, ann = O.synthetic_batch(args.bs, size=args.size, G=8, num_classes=80, seed=1000)
    images, ann = images.to(dev), ann.to(dev)

    def model():
        m = EfficientDet(num_classes=80, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
        m.load_state_dict(sd)
        m = m.to(dev)
        m.train()
        m.is_training = True
        m.freeze_bn()
        return m

    # the graph without an optimizer reads the packed weights its warm-up derived into _ops' cache, which every
    # invalidation (model construction, train(), building a step with an optimizer) drops: build it last
    plain_model, m = model(), model()
    fused = GraphedTrainStep(m, images, ann, optimizer=FusedClipAdamW(m.parameters(), lr=1e-4, max_norm=0.1))
    steps = {'graph_no_optimizer': (GraphedTrainStep(plain_model, images, ann), lambda i: True)}
    steps['fused_update_every'] = (fused, lambda i: True)
    steps['fused_k4'] = (fused, lambda i: (i + 1) % 4 == 0)
    steps['fused_no_update'] = (fused, lambda i: False)
    launches = {'graph_no_optimizer': steps['graph_no_optimizer'][0].library_launches,
                'fused': fused.library_launches}

    def run(name):
        step, update = steps[name]
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            step(images, ann, update=update(i))
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    for name in steps:                                   # warm every configuration once
        run(name)
    times = {name: [] for name in steps}
    for _ in range(args.rounds):
        for name in steps:
            times[name].append(run(name))
    res = {}
    for name, ts in times.items():
        ts = sorted(ts)
        med = ts[len(ts) // 2]
        res[name] = dict(ms_per_micro_step=round(med, 3), img_per_s=round(args.bs * 1000.0 / med, 1),
                         min_ms=round(ts[0], 3), max_ms=round(ts[-1], 3))
    base = res['graph_no_optimizer']['ms_per_micro_step']
    print(json.dumps(dict(card=card(), bs=args.bs, size=args.size, steps=args.steps, rounds=args.rounds,
                          library_launches=launches, configs=res,
                          between_updates_minus_no_optimizer_ms=round(res['fused_no_update']['ms_per_micro_step'] - base, 3),
                          update_minus_no_update_ms=round(res['fused_update_every']['ms_per_micro_step']
                                                          - res['fused_no_update']['ms_per_micro_step'], 3))))


if __name__ == '__main__':
    main()
