"""demo.py's per-frame path: the host chain as demo.py runs it against GraphedFrameDetect, D0 at 512 x 512.

  host chain   the test transform on the CPU (tools/frame_oracle.py's NumPy restatement: albumentations is not a
               dependency), the host->device copy, the eager B = 1 model(img) and the per-box loop as demo.py:86-104
               writes it (two device reads per kept box)
  device path  GraphedFrameDetect: staging + copies, one replay (transform, network, decode, NMS, rescale), two reads

Latency per frame at B = 1 for 480 x 640 and 720 x 1280 frames (host clock around calls that end in a synchronise,
host chain and device path alternated), device-path throughput at B = 8 and 32 (720 x 1280 frames), and the transform
kernel alone (CUDA events over many launches) with its achieved bytes/s (frame bytes in + fp32 out) against the H100
SXM data sheet's 3.35 TB/s.  The model is D0 with 20 classes, seeded weights and the demo's thresholds (0.01, 0.5), so
nearly every anchor is an NMS candidate.  Prints one JSON line with the card's name and power limit read in the same
process.
  python tools/bench_frames.py [--reps 5]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [os.path.join(R, 'efficientdet.pytorch_b200'), os.path.join(R, 'oracle'), os.path.join(R, 'tools')]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import effdet_oracle as O  # noqa: E402
import frame_oracle as F  # noqa: E402
from models import EfficientDet  # noqa: E402
from models.graph_step import GraphedFrameDetect  # noqa: E402
from models.pipeline import launch_frame_transform  # noqa: E402

HBM_TBS = 3.35


def card():
    try:
        q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=60).stdout.strip().splitlines()[0]
        name, power, clock = (s.strip() for s in q.split(','))
        return {'name': name, 'power_limit': power, 'max_sm_clock': clock}
    except (OSError, IndexError, ValueError, subprocess.SubprocessError):
        return {'name': torch.cuda.get_device_name(0), 'power_limit': 'not read', 'max_sm_clock': 'not read'}


def host_chain(model, frame, size=(512, 512)):
    """demo.py's Detect.process without the drawing"""
    img = torch.from_numpy(F.transform([frame], *size)[0]).to('cuda:0').unsqueeze(0)
    with torch.no_grad():
        scores, classification, transformed_anchors = model(img)
        bboxes, labels, bbox_scores = [], [], []
        for j in range(scores.shape[0]):
            bbox = transformed_anchors[[j], :][0].data.cpu().numpy()
            x1 = int(bbox[0] * frame.shape[1] / size[1])
            y1 = int(bbox[1] * frame.shape[0] / size[0])
            x2 = int(bbox[2] * frame.shape[1] / size[1])
            y2 = int(bbox[3] * frame.shape[0] / size[0])
            bboxes.append([x1, y1, x2, y2])
            labels.append(int(classification[[j]]))
            score = np.around(scores[[j]].cpu().numpy(), decimals=2) * 100
            bbox_scores.append(int(score[0]))
    return bboxes, labels, bbox_scores


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def transform_kernel(frames, iters=200):
    """device ms per launch of the transform kernel and achieved bytes/s"""
    flat = np.concatenate([f.reshape(-1) for f in frames])
    offs = np.concatenate([[0], np.cumsum([f.size for f in frames])[:-1]]).astype(np.int64)
    pix = torch.from_numpy(flat).cuda()
    offs = torch.from_numpy(offs).cuda()
    hw = torch.tensor([f.shape[:2] for f in frames], dtype=torch.int32).cuda()
    out = torch.empty((len(frames), 3, 512, 512), device='cuda:0')
    for _ in range(10):
        launch_frame_transform(out, pix, offs, hw)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        launch_frame_transform(out, pix, offs, hw)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / iters
    nbytes = flat.size + 4 * out.numel()
    return {'frames': len(frames), 'size': list(frames[0].shape[:2]), 'ms': round(ms, 4), 'bytes': int(nbytes),
            'tb_per_s': round(nbytes / ms / 1e9, 3), 'hbm_frac': round(nbytes / ms / 1e9 / HBM_TBS, 3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'bench_frames measures on a GPU'
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    model = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    model.load_state_dict(O.init_state_dict(cfg, seed=5))
    model = model.cuda().eval()
    res = {'card': card(), 'model': 'D0 20 classes, 512x512, threshold 0.01, iou 0.5', 'latency_b1': {},
           'throughput': {}, 'transform_kernel': []}
    for h, w in [(480, 640), (720, 1280)]:
        frame = F.synthetic_frames(70, [(h, w)])
        det = GraphedFrameDetect(model, frame)
        host_chain(model, frame[0])
        det(frame)
        hs, ds, kept = [], [], 0
        for _ in range(a.reps):                                   # alternated
            ms, out = timed(lambda: host_chain(model, frame[0]))
            hs.append(ms)
            ms, got = timed(lambda: det(frame))
            ds.append(ms)
            kept = len(got[0][0])
        res['latency_b1']['%dx%d' % (h, w)] = {'host_chain_ms': round(statistics.median(hs), 2),
                                               'device_ms': round(statistics.median(ds), 3), 'kept_boxes': kept,
                                               'host_runs': [round(v, 2) for v in hs],
                                               'device_runs': [round(v, 3) for v in ds]}
        del det
    for B in (8, 32):
        frames = F.synthetic_frames(71, [(720, 1280)] * B)
        det = GraphedFrameDetect(model, frames)
        det(frames)
        ds = [timed(lambda: det(frames))[0] for _ in range(a.reps)]
        res['throughput']['B%d' % B] = {'ms_per_call': round(statistics.median(ds), 3),
                                        'frames_per_s': round(B / statistics.median(ds) * 1e3, 1)}
        del det
    for sizes in ([(480, 640)], [(720, 1280)], [(720, 1280)] * 32, [(1080, 1920)] * 8):
        res['transform_kernel'].append(transform_kernel(F.synthetic_frames(72, sizes)))
    print(json.dumps(res))


if __name__ == '__main__':
    main()
