"""Time training on ragged DataLoader batches at bench.py's D0 geometry (512x512, 80 classes, Bcap = 32, train mode:
drop-connect on, BatchNorm frozen), no optimizer in the graph, as bench.py runs it:

  (a) step_capacity   GraphedTrainStep(..., max_annotations=256) on batches with VOC-like box counts per image
      step_padded     the default GraphedTrainStep on the same batches, each padded to one fixed G (the largest count)
  (b) loss_*          the FocalLoss kernels alone, forward + backward: the counted pair at Gcap = 256, 1024, 4096 with
                      about 10 boxes per image, against the uncounted pair at G = the largest count
  (c) tail_b7         a capacity-mode replay on a last batch of 7 images (the graph always runs all Bcap images)

Configurations are timed in alternating rounds with CUDA events; the card's name and power limit are read in the same
run.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), '..')
sys.path.insert(0, os.path.join(ROOT, 'efficientdet.pytorch_b200'))
sys.path.insert(0, os.path.join(ROOT, 'oracle'))
import effdet_oracle as O                            # noqa: E402
from models import EfficientDet, _native as N        # noqa: E402
from models.graph_step import GraphedTrainStep       # noqa: E402


def card():
    out = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm',
                          '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    return out or torch.cuda.get_device_name(0)


def ragged(counts, size, K, rng, G=None):
    """a collated batch [B, G, 5]: counts[b] boxes, then -1 rows; G defaults to the largest count"""
    G = G or max(max(counts), 1)
    ann = np.full((len(counts), G, 5), -1.0, np.float32)
    for b, n in enumerate(counts):
        xy = rng.uniform(0, size * 0.8, (n, 2))
        wh = rng.uniform(8, size * 0.25, (n, 2))
        ann[b, :n] = np.concatenate([xy, xy + wh, rng.randint(K, size=(n, 1))], 1)
    return torch.from_numpy(ann)


def timed(fn, n):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(n):
        fn(i)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--bs', type=int, default=32)
    ap.add_argument('--size', type=int, default=512)
    ap.add_argument('--batches', type=int, default=8, help='distinct ragged batches cycled through')
    ap.add_argument('--steps', type=int, default=16, help='micro-steps per configuration and round')
    ap.add_argument('--rounds', type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('bench_ragged_step needs a GPU')
    dev = torch.device('cuda:0')
    K, B = 80, args.bs
    rng = np.random.RandomState(0)
    cfg = O.make_config('efficientdet-d0', K, 64, 2)
    sd = O.init_state_dict(cfg, seed=0)
    # VOC-like: one to a few dozen boxes per image (geometric, mean ~3.3, capped at 40)
    counts = [[int(c) for c in np.minimum(rng.geometric(0.3, size=B), 40)] for _ in range(args.batches)]
    g_fixed = max(max(c) for c in counts)
    images = torch.randn(B, 3, args.size, args.size, generator=torch.Generator().manual_seed(1)).to(dev)
    batches = [ragged(c, args.size, K, rng).to(dev) for c in counts]
    padded = [torch.nn.functional.pad(a, (0, 0, 0, g_fixed - a.shape[1]), value=-1.0) for a in batches]
    tail_ann = ragged(counts[0][:7], args.size, K, rng).to(dev)

    def model():
        m = EfficientDet(num_classes=K, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
        m.load_state_dict(sd)
        m = m.to(dev)
        m.train()
        m.is_training = True
        m.freeze_bn()
        return m

    m_cap, m_pad = model(), model()                  # both built before either graph: construction drops the caches
    cap = GraphedTrainStep(m_cap, images, batches[0], max_annotations=256)
    pad = GraphedTrainStep(m_pad, images, padded[0])
    nb = len(batches)
    runs = {'step_capacity': lambda i: cap(images, batches[i % nb]),
            'step_padded': lambda i: pad(images, padded[i % nb]),
            'tail_b7': lambda i: cap(images[:7], tail_ann)}

    # (b) the loss kernels alone on [B, A, K] predictions, ~10 boxes per image
    A = O.anchors_for(args.size, args.size)[0].shape[0]
    anchors = torch.from_numpy(O.anchors_for(args.size, args.size)[0]).to(dev)
    g = torch.Generator(device=dev).manual_seed(2)
    cls = torch.rand(B, A, K, generator=g, device=dev) * 0.2
    reg = torch.randn(B, A, 4, generator=g, device=dev) * 0.3
    few = [int(c) for c in rng.randint(8, 13, size=B)]
    losses, stats = torch.empty(2, device=dev), torch.empty(B, 4, device=dev)
    assign = torch.empty(B, A, dtype=torch.int32, device=dev)
    dcls, dreg = torch.empty_like(cls), torch.empty_like(reg)
    gout = torch.ones(2, device=dev)
    old = ragged(few, args.size, K, rng).to(dev)
    tables = {}
    for gcap in (256, 1024, 4096):
        t = torch.full((B, gcap, 5), -1.0, device=dev)
        c = torch.empty(1 + B, dtype=torch.int32, device=dev)
        N.call('effdet_pack_annots', t, old.data_ptr(), B, old.shape[1], t.data_ptr(), c.data_ptr(), B, gcap)
        tables[gcap] = (t, c)

    def loss_old(i):
        N.call('effdet_focal_loss_fwd', cls, cls.data_ptr(), reg.data_ptr(), anchors.data_ptr(), old.data_ptr(),
               losses.data_ptr(), assign.data_ptr(), stats.data_ptr(), B, A, K, old.shape[1], 0.25, 2.0)
        N.call('effdet_focal_loss_bwd', cls, cls.data_ptr(), reg.data_ptr(), anchors.data_ptr(), old.data_ptr(),
               gout.data_ptr(), assign.data_ptr(), stats.data_ptr(), dcls.data_ptr(), dreg.data_ptr(), B, A, K,
               old.shape[1], 0.25, 2.0)

    def loss_counted(gcap):
        t, c = tables[gcap]

        def run(i):
            N.call('effdet_focal_loss_counted_fwd', cls, cls.data_ptr(), reg.data_ptr(), anchors.data_ptr(),
                   t.data_ptr(), c.data_ptr(), losses.data_ptr(), assign.data_ptr(), stats.data_ptr(), B, A, K, gcap,
                   0.25, 2.0)
            N.call('effdet_focal_loss_counted_bwd', cls, cls.data_ptr(), reg.data_ptr(), anchors.data_ptr(),
                   t.data_ptr(), c.data_ptr(), gout.data_ptr(), assign.data_ptr(), stats.data_ptr(), dcls.data_ptr(),
                   dreg.data_ptr(), B, A, K, gcap, 0.25, 2.0)
        return run

    runs['loss_uncounted_g%d' % old.shape[1]] = loss_old
    for gcap in tables:
        runs['loss_counted_gcap%d' % gcap] = loss_counted(gcap)

    for name, fn in runs.items():                     # warm-up
        timed(fn, 3)
    times = {name: [] for name in runs}
    for _ in range(args.rounds):
        for name, fn in runs.items():
            times[name].append(timed(fn, args.steps if name.startswith(('step', 'tail')) else 4 * args.steps))
    res = {name: dict(ms_median=round(float(np.median(v)), 4), ms_min=round(float(min(v)), 4)) for name, v in times.items()}
    for name in ('step_capacity', 'step_padded', 'tail_b7'):
        res[name]['img_per_s'] = round((7 if name == 'tail_b7' else B) / res[name]['ms_median'] * 1e3, 1)
    print(json.dumps(dict(card=card(), workload='EfficientDet-D0 %dx%d train, Bcap %d, no optimizer in the graph'
                          % (args.size, args.size, B), fixed_G=g_fixed, uncounted_G=old.shape[1],
                          counts_per_batch=[sum(c) for c in counts], results=res)))


if __name__ == '__main__':
    main()
