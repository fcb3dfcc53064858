"""Throughput and accuracy of the two tensor-core precision modes (EFFDET_B200_PRECISION=bf16x3, the default, and bf16).

One measurement per process, in the mode given on the command line:
  D0 512x512 bs 32 train step exactly as bench.py times it (same seeded batch and init, drop-connect stream seeded with 0,
  3 eager warm-up steps, GraphedTrainStep, 20 timed replays), then D7 1536x1536 bs 1 inference (3 warm-up, 20 timed).
  It writes the img/s, the loss and the seeded gradient sample of the last train step (bench.py's grad_sample) to OUT.
  python tools/bench_precision.py --mode bf16 --out DIR

The driver alternates the two modes, `runs` processes each, and reports the median and range of every rate, the card's
name, power limit and maximum SM clock (nvidia-smi, read in the same call), and how far the bf16 loss and gradient
sample are from the bf16x3 ones:
  python tools/bench_precision.py --driver 5 --out DIR
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def measure(mode, out, steps, warmup):
    sys.path[:0] = [os.path.join(R, 'efficientdet.pytorch_b200'), os.path.join(R, 'oracle'), R]
    import torch
    from models import EfficientDet, _ops
    from models.graph_step import GraphedTrainStep
    import effdet_oracle as O
    import bench
    _ops.PRECISION = mode
    dev = torch.device('cuda', 0)
    res = dict(mode=mode)

    def timed(fn, n):
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1)

    c = bench.CONFIGS['d0']
    torch.manual_seed(0)
    cfg = O.make_config(c['net'], c['K'], c['W'], c['D'])
    model = EfficientDet(num_classes=c['K'], network=c['net'], D_bifpn=c['D'], W_bifpn=c['W'], is_training=True)
    model.load_state_dict(O.init_state_dict(cfg, seed=0))
    model = model.to(dev)
    model.train()
    model.is_training = True
    model.freeze_bn()
    images, ann = bench.synthetic(c, c['bs'], seed=1000)
    images, ann = images.to(dev), ann.to(dev)
    for _ in range(warmup):
        for p in model.parameters():
            p.grad = None
        cl, rl = model([images, ann])
        (cl.mean() + rl.mean()).backward()
    del cl, rl
    step = GraphedTrainStep(model, images, ann, warmup=0)
    for _ in range(2):
        step(images, ann)
    last = {}
    ms = timed(lambda: last.__setitem__('loss', step(images, ann)), steps)
    res['d0_train_img_s'] = c['bs'] * steps * 1000.0 / ms
    res['d0_loss'] = float(last['loss'])
    torch.save(bench.grad_sample(model).cpu(), os.path.join(out, 'grads_%s_%d.pt' % (mode, os.getpid())))
    res['grads'] = 'grads_%s_%d.pt' % (mode, os.getpid())
    del step, model
    torch.cuda.empty_cache()

    c = bench.CONFIGS['d7']
    cfg = O.make_config(c['net'], c['K'], c['W'], c['D'])
    model = EfficientDet(num_classes=c['K'], network=c['net'], D_bifpn=c['D'], W_bifpn=c['W'], is_training=False,
                         threshold=0.4, iou_threshold=0.5)
    model.load_state_dict(O.init_state_dict(cfg, seed=0))
    model = model.to(dev).eval()
    images, _ = bench.synthetic(c, c['bs'], seed=1000)
    images = images.to(dev)
    with torch.no_grad():
        for _ in range(warmup):
            model(images)
        ms = timed(lambda: model(images), steps)
    res['d7_infer_img_s'] = c['bs'] * steps * 1000.0 / ms
    print(json.dumps(res), flush=True)
    return res


def driver(runs, out, steps, warmup):
    import torch
    card = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    results = {'bf16x3': [], 'bf16': []}
    for i in range(runs):
        for mode in ('bf16x3', 'bf16'):
            r = subprocess.run([sys.executable, os.path.abspath(__file__), '--mode', mode, '--out', out, '--steps', str(steps),
                                '--warmup', str(warmup)], capture_output=True, text=True)
            if r.returncode != 0:
                raise RuntimeError('%s run %d failed:\n%s' % (mode, i, r.stdout[-2000:] + r.stderr[-4000:]))
            results[mode].append(json.loads(r.stdout.strip().splitlines()[-1]))
    summary = dict(card=card, runs=runs, steps=steps, warmup=warmup)
    for mode, rs in results.items():
        for k in ('d0_train_img_s', 'd7_infer_img_s'):
            v = [r[k] for r in rs]
            summary['%s %s' % (mode, k)] = dict(median=round(statistics.median(v), 2), min=round(min(v), 2), max=round(max(v), 2))
    # accuracy of bf16 against bf16x3: same batch, same init, same drop-connect draws
    l3 = statistics.median(r['d0_loss'] for r in results['bf16x3'])
    l1 = statistics.median(r['d0_loss'] for r in results['bf16'])
    g3 = torch.load(os.path.join(out, results['bf16x3'][0]['grads']))
    g1 = torch.load(os.path.join(out, results['bf16'][0]['grads']))
    g3b = torch.load(os.path.join(out, results['bf16x3'][-1]['grads']))
    rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())     # noqa: E731
    summary['loss bf16x3'] = l3
    summary['loss bf16'] = l1
    summary['loss rel diff bf16 vs bf16x3'] = abs(l1 - l3) / abs(l3)
    summary['loss spread bf16x3 runs'] = max(r['d0_loss'] for r in results['bf16x3']) - min(r['d0_loss'] for r in results['bf16x3'])
    summary['grad sample rel diff bf16 vs bf16x3'] = rel(g1, g3)
    summary['grad sample rel diff bf16x3 run 1 vs run %d' % runs] = rel(g3b, g3)
    for f in os.listdir(out):
        if f.startswith('grads_'):
            os.remove(os.path.join(out, f))
    print(json.dumps(summary, indent=1))
    with open(os.path.join(out, 'bench_precision.json'), 'w') as fh:
        json.dump(dict(summary=summary, runs=results), fh, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--mode', choices=['bf16x3', 'bf16'])
    ap.add_argument('--driver', type=int, default=0, metavar='RUNS', help='alternate the two modes RUNS times each')
    ap.add_argument('--out', required=True, help='directory for the gradient samples and the summary')
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    if args.driver:
        driver(args.driver, args.out, args.steps, args.warmup)
    else:
        measure(args.mode, args.out, args.steps, args.warmup)


if __name__ == '__main__':
    main()
