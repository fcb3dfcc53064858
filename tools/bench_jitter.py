"""Scale-jitter augmentation (RawCollater(scale_jitter=(0.1, 2.0))) at D0 512^2 batch 32 on seeded VOC-sized (375x500)
and COCO-sized (480x640) uint8 images held in memory (JPEG decoding is not part of any side).

  kernels : effdet_resize_crop_normalize_pad and effdet_collate_pack_annots_crop on jittered batches against
            effdet_resize_normalize_pad and effdet_collate_pack_annots on unjittered batches of the same images, in us
            per launch from CUDA events around CUDA-graph replays of 20 launches, the two sides alternated.
  host    : the host chain the crop kernel replaces, per image: Normalizer (float64) -> flip -> the reference Resizer
            at the drawn L (cv2.resize INTER_LINEAR on the float64 image, zero pad to L x L) -> the S x S window ->
            float32, in ms per image on one core.
  train   : ms per batch of DataLoader(4 workers, pin_memory=True) + the raw GraphedTrainStep, jittered against
            unjittered RawCollater, alternated; and host-side jitter in 4 workers (the host chain above plus the box
            rule, collated to float32 tensors) feeding the tensor capacity-mode GraphedTrainStep.

Prints one JSON line with the card's name, power limit and max SM clock read in the same process.
  python tools/bench_jitter.py [--batches 6] [--reps 2] [--parts kernels,host,train]
"""
import argparse
import json
import os
import sys
import time

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(R, 'efficientdet.pytorch_b200'), os.path.join(R, 'oracle'), os.path.join(R, 'tools')]

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

import effdet_oracle as O  # noqa: E402
import jitter_oracle as J  # noqa: E402
import resize_oracle as RO  # noqa: E402
from bench_raw_input import BS, K, S, Samples, card, train_model  # noqa: E402
from models.fused_optim import FusedClipAdamW  # noqa: E402
from models.graph_step import GraphedTrainStep  # noqa: E402
from models.pipeline import RawCollater, launch_raw_pack, launch_raw_resize  # noqa: E402

JITTER = (0.1, 2.0)


def graph_us(fn, reps=5, per_graph=20):
    """us per call of fn (a capturable launch) from CUDA events around replays of a graph of per_graph calls"""
    fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(per_graph):
            fn()
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / (reps * per_graph)


def bench_kernels(ds, ps, reps=3):
    np.random.seed(11)
    raws = {'plain': RawCollater(S, pixel_scale=ps)(ds.samples[:BS]),
            'jitter': RawCollater(S, pixel_scale=ps, scale_jitter=JITTER)(ds.samples[:BS])}
    out = torch.empty((BS, 3, S, S), device='cuda')
    ann = torch.empty((BS, 64, 5), device='cuda')
    cnt = torch.empty((BS + 1,), dtype=torch.int32, device='cuda')
    blobs = {k: r.blob.cuda() for k, r in raws.items()}
    t = {k: {'resize': [], 'pack': []} for k in raws}
    for _ in range(reps):
        for k, r in raws.items():
            j = r.jitter
            t[k]['resize'].append(graph_us(lambda: launch_raw_resize(out, blobs[k], BS, ps, j)))
            t[k]['pack'].append(graph_us(lambda: launch_raw_pack(blobs[k], BS, ann, cnt, j)))
    L = raws['jitter'].section('resized_hw').numpy().max(axis=1)
    return {'resize_us': {k: [round(v, 1) for v in t[k]['resize']] for k in t},
            'pack_us': {k: [round(v, 2) for v in t[k]['pack']] for k in t},
            'jitter_L_mean': round(float(L.mean()), 1), 'rows': raws['plain'].rows,
            'output_MB': round(4 * BS * 3 * S * S / 1e6, 1)}


def host_jitter(sample, ps):
    """one sample through the host chain with scale jitter: the draws of RawCollater, then Normalizer -> flip ->
    Resizer at L (cv2) -> window -> float32 [3, S, S], and the box rule -> kept float32 rows"""
    im = sample['img']
    h, w = im.shape[:2]
    from models.pipeline import jitter_range, min_common_size
    lo, hi = jitter_range(S, *JITTER)
    L = max(int(np.random.randint(lo, hi + 1)), min_common_size(h, w))
    scale, rh, rw = RO.resizer_geometry(h, w, L)
    y0 = int(np.random.randint(0, max(rh - S, 0) + 1))
    x0 = int(np.random.randint(0, max(rw - S, 0) + 1))
    img = RO.normalize(im, ps)
    if sample.get('flip'):
        img = img[:, ::-1, :]
    full = np.zeros((L, L, 3))
    full[:rh, :rw] = cv2.resize(img, (rw, rh))
    win = np.zeros((S, S, 3))
    part = full[y0:y0 + S, x0:x0 + S]
    win[:part.shape[0], :part.shape[1]] = part
    return (np.ascontiguousarray(win.astype(np.float32).transpose(2, 0, 1)),
            J.crop_boxes(sample['annot'], sample.get('flip'), w, scale, y0, x0, S))


class HostJitterCollater:
    """what a user writes today: scale jitter on the host in the workers, collated to float32 tensors"""

    def __init__(self, ps):
        self.ps = ps

    def __call__(self, samples):
        out = [host_jitter(s, self.ps) for s in samples]
        G = max(1, max(len(b) for _, b in out))
        ann = np.full((len(out), G, 5), -1, np.float32)
        for i, (_, b) in enumerate(out):
            ann[i, :len(b)] = b
        return torch.from_numpy(np.stack([im for im, _ in out])), torch.from_numpy(ann)


def bench_host(ds, ps, n=64):
    np.random.seed(12)
    t0 = time.perf_counter()
    for s in ds.samples[:n]:
        host_jitter(s, ps)
    return {'ms_per_image': round((time.perf_counter() - t0) * 1e3 / n, 2), 'images': n,
            'cv2_threads': cv2.getNumThreads()}


def timed_epoch(loader, call, batches):
    it = iter(loader)
    for _ in range(2):                                                # workers started, first batches warmed
        call(next(it))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(batches):
        call(next(it))
    torch.cuda.synchronize()
    del it
    return (time.perf_counter() - t0) * 1e3 / batches


def bench_train(ds, ps, sd, batches, reps):
    m = train_model(sd)
    cols = {'raw_unjittered': RawCollater(S, pixel_scale=ps),
            'raw_jittered': RawCollater(S, pixel_scale=ps, scale_jitter=JITTER)}
    opts = [FusedClipAdamW(m.parameters(), lr=1e-6, max_norm=0.1) for _ in range(3)]    # one optimizer per graph
    np.random.seed(13)
    steps = {k: GraphedTrainStep(m, col(ds.samples[:BS]), optimizer=opts[i], max_annotations=64)
             for i, (k, col) in enumerate(cols.items())}
    host_col = HostJitterCollater(ps)
    tensor_step = GraphedTrainStep(m, *[t.cuda() for t in host_col(ds.samples[:BS])], optimizer=opts[2],
                                   max_annotations=64)
    res = {k: [] for k in list(cols) + ['host_jitter_tensor_step']}
    for _ in range(reps):
        for k, col in cols.items():
            loader = torch.utils.data.DataLoader(ds, batch_size=BS, shuffle=True, num_workers=4, collate_fn=col,
                                                 pin_memory=True)
            res[k].append(round(timed_epoch(loader, steps[k], batches), 2))
        loader = torch.utils.data.DataLoader(ds, batch_size=BS, shuffle=True, num_workers=4, collate_fn=host_col,
                                             pin_memory=True)
        res['host_jitter_tensor_step'].append(round(timed_epoch(loader, lambda b: tensor_step(*b), batches), 2))
    del steps, tensor_step
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', type=int, default=6)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--parts', default='kernels,host,train', help='comma-separated subset of kernels, host, train')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_jitter.py measures on a GPU'
    torch.cuda.init()                                                  # workers fork after CUDA is initialised
    cfg = O.make_config('efficientdet-d0', num_classes=K, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=5)
    res = {'card': card(), 'cv2': cv2.__version__, 'host_cores': len(os.sched_getaffinity(0)),
           'scale_jitter': JITTER, 'model': 'D0 %d classes, D_bifpn 2, W_bifpn 64, %dx%d, batch %d' % (K, S, S, BS)}
    parts = a.parts.split(',')
    for name, hw, ps in [('voc_375x500', (375, 500), 255), ('coco_480x640', (480, 640), None)]:
        ds = Samples(BS * (a.batches + 2), hw, seed=7)
        res[name] = {}
        if 'kernels' in parts:
            res[name]['kernels'] = bench_kernels(ds, ps)
        if 'host' in parts:
            res[name]['host_chain'] = bench_host(ds, ps)
        if 'train' in parts:
            res[name]['train_ms_per_batch'] = bench_train(ds, ps, sd, a.batches, a.reps)
        print(json.dumps({name: res[name]}), file=sys.stderr)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
