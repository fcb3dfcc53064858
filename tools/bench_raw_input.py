"""Raw batches against the main-process input paths, at D0 512^2 batch 32 on seeded VOC-sized (375x500) and COCO-sized
(480x640) uint8 images held in memory (JPEG decoding is not part of either side).

  train : wall time per batch of DataLoader(4 workers, collate_fn=RawCollater, pin_memory=True) + GraphedTrainStep on
          raw batches, against main-process DeviceCollater(resize=True) + the tensor capacity-mode step, alternated;
          plus where the host time of each step goes (waiting for the loader / collating, and the step call itself).
  eval  : evaluate() img/s with collater=RawCollater and 4 workers, against the unchanged evaluate() on a dataset whose
          __getitem__ runs the reference's eval transform, Normalizer + Resizer with cv2.resize on the float64 image
          (as tools/bench_input.py builds it), with both mAPs.
  pack  : effdet_collate_pack_annots per launch, from CUDA events around 500 launches replayed from a graph.

Prints one JSON line with the card's name, power limit and max SM clock read in the same process.
  python tools/bench_raw_input.py [--batches 8] [--reps 2] [--eval-images 512] [--parts train,eval,pack]
"""
import argparse
import json
import os
import subprocess
import sys
import time

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(R, 'efficientdet.pytorch_b200'), os.path.join(R, 'oracle'), os.path.join(R, 'tools')]

import cv2  # noqa: E402
import numpy as np  # noqa: E402
import torch  # noqa: E402

import effdet_oracle as O  # noqa: E402
import resize_oracle as RO  # noqa: E402
from models import EfficientDet, evaluation  # noqa: E402
from models.fused_optim import FusedClipAdamW  # noqa: E402
from models.graph_step import GraphedTrainStep  # noqa: E402
from models.pipeline import DeviceCollater, RawCollater, launch_raw_pack  # noqa: E402

BS, S, K = 32, 512, 20


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in q.split(','))
        return {'name': name, 'power_limit': power, 'max_sm_clock': clock}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return {'name': torch.cuda.get_device_name(0), 'power_limit': 'not read', 'max_sm_clock': 'not read'}


class Samples(torch.utils.data.Dataset):
    """seeded decoded samples: uint8 [h, w, 3], VOC-like box counts, every other image flipped"""

    def __init__(self, n, hw, seed):
        rng = np.random.RandomState(seed)
        counts = np.minimum(rng.geometric(0.25, size=n), 40)
        images, annots = RO.synthetic_batch(seed, [hw] * n, [int(c) for c in counts])
        self.samples = [dict(img=im, annot=a, flip=bool(i % 2)) for i, (im, a) in enumerate(zip(images, annots))]

    def __len__(self):
        return len(self.samples)

    def __getitem__(self, i):
        return self.samples[i]


class HostChain:
    """the unchanged evaluate()'s input: the reference's eval transform Compose([Normalizer(), Resizer()]) on the host,
    float64 normalisation and cv2.resize, as datasets/augmentation.py runs them"""

    def __init__(self, ds, pixel_scale):
        self.ds, self.pixel_scale = ds, pixel_scale

    def __len__(self):
        return len(self.ds)

    def __getitem__(self, i):
        im = self.ds.samples[i]['img']
        scale, rh, rw = RO.resizer_geometry(im.shape[0], im.shape[1], S)
        new = np.zeros((S, S, 3))
        new[:rh, :rw] = cv2.resize(RO.normalize(im, self.pixel_scale), (rw, rh))
        return {'img': torch.from_numpy(new.astype(np.float32)), 'scale': scale}


class VOCView:
    """the generator interface evaluate() takes, over either input"""

    def __init__(self, base, ds):
        self.base, self.ds = base, ds

    def __len__(self):
        return len(self.base)

    def __getitem__(self, i):
        return self.base[i]

    def load_annotations(self, i):
        return self.ds.samples[i]['annot']

    def num_classes(self):
        return K

    def label_to_name(self, label):
        return str(label)


def train_model(sd):
    m = EfficientDet(num_classes=K, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
    m.load_state_dict(sd)
    m = m.cuda().eval()
    m.is_training = True
    return m


def bench_train(ds, pixel_scale, sd, batches, reps):
    m = train_model(sd)
    col = RawCollater(S, pixel_scale=pixel_scale)
    dcol = DeviceCollater(S, 'cuda:0', resize=True, pixel_scale=pixel_scale)
    opts = [FusedClipAdamW(m.parameters(), lr=1e-6, max_norm=0.1) for _ in range(2)]    # one optimizer per graph
    raw_step = GraphedTrainStep(m, col(ds.samples[:BS]), optimizer=opts[0], max_annotations=64)
    tensor_step = GraphedTrainStep(m, *dcol(ds.samples[:BS]), optimizer=opts[1], max_annotations=64)
    res = {'raw': [], 'tensor': [], 'raw_host': [], 'tensor_host': []}
    for _ in range(reps):
        loader = torch.utils.data.DataLoader(ds, batch_size=BS, shuffle=False, num_workers=4, collate_fn=col,
                                             pin_memory=True)
        it = iter(loader)
        for _ in range(2):                                            # workers started, first batches warmed
            raw_step(next(it))
        torch.cuda.synchronize()
        wait = call = 0.0
        t0 = time.perf_counter()
        for _ in range(batches):
            a = time.perf_counter()
            raw = next(it)
            b = time.perf_counter()
            raw_step(raw)
            wait, call = wait + b - a, call + time.perf_counter() - b
        torch.cuda.synchronize()
        res['raw'].append((time.perf_counter() - t0) * 1e3 / batches)
        res['raw_host'].append({'loader_wait_ms': wait * 1e3 / batches, 'step_call_ms': call * 1e3 / batches})
        del it, loader
        for i in range(2):
            tensor_step(*dcol(ds.samples[i * BS:(i + 1) * BS]))
        torch.cuda.synchronize()
        wait = call = 0.0
        t0 = time.perf_counter()
        for i in range(2, 2 + batches):
            a = time.perf_counter()
            imgs, ann = dcol(ds.samples[i * BS:(i + 1) * BS])
            b = time.perf_counter()
            tensor_step(imgs, ann)
            wait, call = wait + b - a, call + time.perf_counter() - b
        torch.cuda.synchronize()
        res['tensor'].append((time.perf_counter() - t0) * 1e3 / batches)
        res['tensor_host'].append({'collate_ms': wait * 1e3 / batches, 'step_call_ms': call * 1e3 / batches})
    del raw_step, tensor_step
    torch.cuda.empty_cache()
    return {k: [round(v, 2) for v in vs] if k in ('raw', 'tensor') else
            [{kk: round(vv, 2) for kk, vv in d.items()} for d in vs] for k, vs in res.items()}


def bench_eval(ds, pixel_scale, sd, n):
    m = EfficientDet(num_classes=K, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    m.load_state_dict(sd)
    m = m.cuda().eval()
    out = {}
    sub = Samples.__new__(Samples)
    sub.samples = ds.samples[:n]
    for name, gen, kw in [('raw_4_workers', VOCView(sub, sub), dict(collater=RawCollater(S, pixel_scale=pixel_scale),
                                                                      num_workers=4)),
                          ('host_chain', VOCView(HostChain(sub, pixel_scale), sub), {})]:
        evaluation.evaluate(gen, m, batch_size=BS, **kw)             # warm: graph capture, workers, allocator
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        mean_ap, _ = evaluation.evaluate(gen, m, batch_size=BS, **kw)
        dt = time.perf_counter() - t0
        out[name] = {'img_per_s': round(n / dt, 1), 'mAP': float(mean_ap)}
    # the DataLoader alone (4 workers, RawCollater, pinned): how fast raw batches arrive without any GPU work
    loader = torch.utils.data.DataLoader(sub, batch_size=BS, shuffle=False, num_workers=4,
                                         collate_fn=RawCollater(S, pixel_scale=pixel_scale), pin_memory=True)
    t0 = time.perf_counter()
    for _ in loader:
        pass
    out['loader_only_4_workers'] = {'img_per_s': round(n / (time.perf_counter() - t0), 1)}
    return out


def bench_pack(ds, pixel_scale):
    raw = RawCollater(S, pixel_scale=pixel_scale)(ds.samples[:BS])
    blob = raw.blob.cuda()
    ann = torch.empty((BS, 256, 5), device='cuda')
    cnt = torch.empty((BS + 1,), dtype=torch.int32, device='cuda')
    launch_raw_pack(blob, BS, ann, cnt)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()                                         # device time, not the Python launch rate
    with torch.cuda.graph(g):
        for _ in range(100):
            launch_raw_pack(blob, BS, ann, cnt)
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(5):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    return {'us_per_launch': round(e0.elapsed_time(e1) * 1e3 / 500, 2), 'rows': raw.rows, 'Gcap': 256}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--batches', type=int, default=8)
    ap.add_argument('--reps', type=int, default=2)
    ap.add_argument('--eval-images', type=int, default=512)
    ap.add_argument('--parts', default='train,eval,pack', help='comma-separated subset of train, eval, pack')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_raw_input.py measures on a GPU'
    torch.cuda.init()                                                  # workers fork after CUDA is initialised
    cfg = O.make_config('efficientdet-d0', num_classes=K, W_bifpn=64, D_bifpn=2)
    sd = O.init_state_dict(cfg, seed=5)
    res = {'card': card(), 'cv2': cv2.__version__, 'cv2_threads': cv2.getNumThreads(),
           'host_cores': len(os.sched_getaffinity(0)),
           'model': 'D0 %d classes, D_bifpn 2, W_bifpn 64, %dx%d, batch %d' % (K, S, S, BS)}
    for name, hw, ps in [('voc_375x500', (375, 500), 255), ('coco_480x640', (480, 640), None)]:
        ds = Samples(max(BS * (a.batches + 2), a.eval_images), hw, seed=7)
        parts = a.parts.split(',')
        res[name] = {}
        if 'train' in parts:
            res[name]['train_ms_per_batch'] = bench_train(ds, ps, sd, a.batches, a.reps)
        if 'eval' in parts:
            res[name]['evaluate'] = bench_eval(ds, ps, sd, a.eval_images)
        if 'pack' in parts:
            res[name]['pack_kernel'] = bench_pack(ds, ps)
        print(json.dumps({name: res[name]}), file=sys.stderr)
    print(json.dumps(res))


if __name__ == '__main__':
    main()
