"""Cost of the weight EMA (models/ema.py ModelEma, effdet_multi_ema):

  kernel        effdet_multi_ema alone over the D0 and D7 state (every floating-point state-dict entry), CUDA events
                over many launches, against the HBM bound of 3 x 4 bytes per element (read e and s, write e)
  graphed_step  the graphed D0 512x512 bs 32 training step with FusedClipAdamW, without and with ema=, update=True on
                every call, timed in alternating rounds
  eager         one update after an eager step: a timm-style torch._foreach EMA (ModelEmaV3's lerp) against
                ModelEma.update, host time (enqueue, no synchronisation) and device time per update

The card's name and power limit are read in the same run.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, os.path.join(ROOT, 'efficientdet.pytorch_b200'))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import effdet_oracle as O                            # noqa: E402
from models import EfficientDet                      # noqa: E402
from models.ema import ModelEma                      # noqa: E402
from models.fused_optim import FusedClipAdamW        # noqa: E402
from models.graph_step import GraphedTrainStep       # noqa: E402

HBM_GBS = 3350.0                                     # H100 SXM data sheet, 700 W


def card():
    out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def events(fn, iters):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def kernel_leg(net, W, D, iters):
    dev = torch.device('cuda:0')
    m = EfficientDet(num_classes=80, network=net, D_bifpn=D, W_bifpn=W, is_training=True).to(dev)
    ema = ModelEma(m)
    tab = ema._table(m)
    n = sum(t.numel() for t in ema._avg)
    for _ in range(10):
        ema._launch(tab)
    ms = events(lambda: ema._launch(tab), iters)
    gbs = 12.0 * n / ms / 1e6
    res = dict(tensors=len(ema._avg), elements=n, mbytes_moved=round(12.0 * n / 1e6, 1), ctas=tab['nchunks'],
               us=round(ms * 1e3, 2), gb_per_s=round(gbs, 1), hbm_frac=round(gbs / HBM_GBS, 3))
    del ema, m
    torch.cuda.empty_cache()
    return res


def step_leg(bs, size, steps, rounds):
    dev = torch.device('cuda:0')
    sd = O.init_state_dict(O.make_config('efficientdet-d0', 80, 64, 2), seed=0)
    images, ann = O.synthetic_batch(bs, size=size, G=8, num_classes=80, seed=1000)
    images, ann = images.to(dev), ann.to(dev)

    def build(with_ema):
        m = EfficientDet(num_classes=80, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
        m.load_state_dict(sd)
        m = m.to(dev)
        m.train()
        m.is_training = True
        m.freeze_bn()
        opt = FusedClipAdamW(m.parameters(), lr=1e-4, max_norm=0.1)
        return GraphedTrainStep(m, images, ann, optimizer=opt, ema=ModelEma(m) if with_ema else None)

    steps_ = {'no_ema': build(False), 'ema': build(True)}
    launches = {k: s.library_launches for k, s in steps_.items()}

    def run(name):
        return events(lambda: steps_[name](images, ann), steps)

    for name in steps_:
        run(name)
    times = {name: [] for name in steps_}
    for _ in range(rounds):
        for name in steps_:
            times[name].append(run(name))
    res = {}
    for name, ts in times.items():
        ts = sorted(ts)
        res[name] = dict(ms_per_step=round(ts[len(ts) // 2], 3), min_ms=round(ts[0], 3), max_ms=round(ts[-1], 3))
    delta = res['ema']['ms_per_step'] - res['no_ema']['ms_per_step']
    del steps_
    torch.cuda.empty_cache()
    return dict(bs=bs, size=size, steps=steps, rounds=rounds, library_launches=launches, configs=res,
                ema_minus_no_ema_ms=round(delta, 3),
                ema_share=round(delta / res['no_ema']['ms_per_step'], 5))


def eager_leg(iters):
    dev = torch.device('cuda:0')
    sd = O.init_state_dict(O.make_config('efficientdet-d0', 80, 64, 2), seed=0)
    m = EfficientDet(num_classes=80, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
    m.load_state_dict(sd)
    m = m.to(dev)
    m.eval()
    m.is_training = True
    opt = FusedClipAdamW(m.parameters(), lr=1e-4, max_norm=0.1)
    images, ann = O.synthetic_batch(4, size=256, G=8, num_classes=80, seed=1001)
    cl, rl = m([images.to(dev), ann.to(dev)])
    (cl.mean() + rl.mean()).backward()
    opt.step()
    del cl, rl
    ema = ModelEma(m)
    src = [v for v in m.state_dict().values() if v.is_floating_point()]
    shadow = [t.clone() for t in src]
    decay = 0.9998

    def timm():
        with torch.no_grad():
            torch._foreach_lerp_(shadow, src, 1.0 - decay)

    def ours():
        ema.update(m)

    res = {}
    for name, fn in (('timm_foreach', timm), ('model_ema', ours)):
        for _ in range(10):
            fn()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(iters):
            fn()
        host = (time.perf_counter() - t0) / iters
        res[name] = dict(host_us=round(host * 1e6, 1), device_us=round(events(fn, iters) * 1e3, 2))
    res['tensors'] = len(src)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--iters', type=int, default=200, help='launches per kernel / eager timing')
    ap.add_argument('--bs', type=int, default=32)
    ap.add_argument('--size', type=int, default=512)
    ap.add_argument('--steps', type=int, default=20, help='graphed steps per configuration and round')
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_ema needs a GPU')
    torch.manual_seed(0)
    out = dict(card=card())
    out['kernel'] = {'d0': kernel_leg('efficientdet-d0', 64, 2, args.iters),
                     'd7': kernel_leg('efficientdet-d7', 384, 8, args.iters)}
    out['graphed_step'] = step_leg(args.bs, args.size, args.steps, args.rounds)
    out['eager'] = eager_leg(args.iters)
    print(json.dumps(out))


if __name__ == '__main__':
    main()
