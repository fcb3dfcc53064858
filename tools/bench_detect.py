"""Inference timing: the CUDA-graph inference step and the batched post-processing, against an earlier build.

One measurement per process, in the source tree given by --tree (default: this one):
  --part eager_vs_graph   D0 512x512 bs 1: eager model(x) against a GraphedDetect replay (+ to_list), ms per image
                          (host clock around calls ending in a synchronise), host issue time of one call (no sync
                          after it), and the replay's library launch count.
  --part post             D0 512x512 bs 32: detect_batch post-processing alone on seeded cls / reg (80 classes), at a
                          threshold giving 1-5 k candidates per image and at one every anchor passes.  Builds without
                          the batched entry points post-process image by image, as their detect_batch did.  Also prints
                          a hash of every output, which must match between builds.
  --part d7_split         D7 1536x1536 bs 1 as bench.py --config d7 sets it up: network, post-processing and whole
                          forward, ms each, a hash of the detections of network outputs shared by all builds (--io),
                          and the device time of each post-processing kernel (torch.profiler, after the timed loops).

The driver alternates this tree and the tree given by --parent (a checkout of an earlier commit whose library has been
built), RUNS processes each for `post` and `d7_split` and RUNS runs of `bench.py --config d7 --dump-outputs` each, and reads the card's name, power limit and maximum SM clock in the same call.  The `chunk_sweep` leg runs this tree
once after the alternated runs: post-processing time, peak memory and output hash per _ops.NMS_CHUNK, on D0 bs 32 with
every anchor a candidate and on the D7 bench image.  `post` and `d7_split` also report the peak memory the
post-processing allocates.
  python tools/bench_detect.py --driver 5 --parent DIR --out DIR [--legs eager_vs_graph,post,d7_split,chunk_sweep,bench]
"""
import argparse
import hashlib
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

R = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _import(tree):
    sys.path[:0] = [os.path.join(tree, 'efficientdet.pytorch_b200'), os.path.join(tree, 'oracle'), tree]
    import torch
    from models import EfficientDet, _ops
    import effdet_oracle as O
    import bench
    return torch, EfficientDet, _ops, O, bench


def _model(torch, EfficientDet, O, bench, name, threshold):
    c = bench.CONFIGS[name]
    cfg = O.make_config(c['net'], c['K'], c['W'], c['D'])
    m = EfficientDet(num_classes=c['K'], network=c['net'], D_bifpn=c['D'], W_bifpn=c['W'], is_training=False,
                     threshold=threshold, iou_threshold=0.5)
    m.load_state_dict(O.init_state_dict(cfg, seed=0))
    return m.to(torch.device('cuda', 0)).eval(), c


def _post(_ops, cls, reg, anchors, h, w, thr):
    """post-processing of every image; builds before the batched entry points ran it image by image"""
    if hasattr(_ops, 'detect_batch'):
        return _ops.detect_batch(cls, reg, anchors, h, w, thr, 0.5)
    return [_ops.detect_image0(cls, reg, anchors, h, w, thr, 0.5, index=i) for i in range(cls.shape[0])]


def _peak_mb(torch, fn):
    """device memory fn allocates at its peak beyond what was allocated before it, MB"""
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return round((torch.cuda.max_memory_allocated() - base) / 1e6, 1)


def _wall(torch, fn, n):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(n):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / n


def _issue(torch, fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    ms = (time.perf_counter() - t0) * 1e3
    torch.cuda.synchronize()
    return ms


def part_eager_vs_graph(tree, iters):
    torch, EfficientDet, _ops, O, bench = _import(tree)
    from models.graph_step import GraphedDetect
    from models import _native
    model, c = _model(torch, EfficientDet, O, bench, 'd0', 0.4)
    x = bench.synthetic(c, 1, seed=1000)[0].to(torch.device('cuda', 0))
    res = dict(part='eager_vs_graph')
    with torch.no_grad():
        for _ in range(5):
            model(x)
        res['eager_ms_per_image'] = _wall(torch, lambda: model(x), iters)
        res['eager_issue_ms'] = statistics.median(_issue(torch, lambda: model(x)) for _ in range(10))
        _native.reset_launch_count()
        model(x)
        res['eager_library_launches'] = _native.launch_count()
    det = GraphedDetect(model, x, max_candidates=8192)
    for _ in range(5):
        det.to_list(det(x))
    res['graph_library_launches'] = det.library_launches
    res['graph_replay_ms_per_image'] = _wall(torch, lambda: det(x), iters)
    res['graph_replay_to_list_ms_per_image'] = _wall(torch, lambda: det.to_list(det(x)), iters)
    res['graph_issue_ms'] = statistics.median(_issue(torch, lambda: det(x)) for _ in range(10))
    with torch.no_grad():
        a, b = model(x), det.to_list(det(x))[0]
    res['detections eager / graph'] = [int(a[0].numel()), int(b[0].numel())]
    return res


def part_post(tree, iters):
    torch, _, _ops, O, _ = _import(tree)
    dev = torch.device('cuda', 0)
    B, K, S = 32, 80, 512
    anchors = torch.from_numpy(O.anchors_for(S, S)).to(dev)
    A = anchors.shape[1]
    g = torch.Generator().manual_seed(7)
    cls = torch.rand(B, A, K, generator=g).to(dev)
    reg = (torch.randn(B, A, 4, generator=g) * 0.3).to(dev)
    res = dict(part='post', B=B, A=A)
    # max of 80 uniform scores > thr with probability 1 - thr^80: 0.99921 -> ~6 %, ~3 k of 49 104 anchors per image
    for name, thr in (('realistic', 0.99921), ('all_anchors', -1.0)):
        out = _post(_ops, cls, reg, anchors, S, S, thr)
        n = int(((cls.max(dim=2)[0] > thr).sum(dim=1)).min()), int(((cls.max(dim=2)[0] > thr).sum(dim=1)).max())
        h = hashlib.sha256()
        for trip in out:
            for t in (trip or []):
                h.update(t.detach().cpu().numpy().tobytes())
        res[name] = dict(threshold=thr, candidates_min_max=n, kept_total=sum(int(t[0].numel()) for t in out if t),
                         ms=_wall(torch, lambda: _post(_ops, cls, reg, anchors, S, S, thr), iters if thr > 0 else 2),
                         peak_mb=_peak_mb(torch, lambda: _post(_ops, cls, reg, anchors, S, S, thr)),
                         sha256=h.hexdigest()[:16])
    return res


def part_d7_split(tree, iters, io):
    """io: file holding the network outputs every build post-processes (written by the first run that finds it
    missing), so the detections' hash compares the post-processing alone: two network passes differ in the last bits"""
    torch, EfficientDet, _ops, O, bench = _import(tree)
    model, c = _model(torch, EfficientDet, O, bench, 'd7', 0.4)
    dev = torch.device('cuda', 0)
    x = bench.synthetic(c, 1, seed=1000)[0].to(dev)
    res = dict(part='d7_split')
    with torch.no_grad():
        for _ in range(2):
            model(x)
        cls, reg, anchors = model._raw_predictions(x)
        if os.path.exists(io):
            cls, reg = [t.to(dev) for t in torch.load(io)]
        else:
            torch.save([cls.cpu(), reg.cpu()], io)
        res['candidates'] = int((cls.max(dim=2)[0] > 0.4).sum())
        res['network_ms'] = _wall(torch, lambda: model._raw_predictions(x), iters)
        res['post_ms'] = _wall(torch, lambda: _post(_ops, cls[:1], reg[:1], anchors, 1536, 1536, 0.4), iters)
        res['post_peak_mb'] = _peak_mb(torch, lambda: _post(_ops, cls[:1], reg[:1], anchors, 1536, 1536, 0.4))
        res['forward_ms'] = _wall(torch, lambda: model(x), iters)
        h = hashlib.sha256()
        for t in _post(_ops, cls[:1], reg[:1], anchors, 1536, 1536, 0.4)[0]:
            h.update(t.cpu().numpy().tobytes())
        res['sha256'] = h.hexdigest()[:16]
        # device time per kernel of one post-processing call, after the timed loops
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            _post(_ops, cls[:1], reg[:1], anchors, 1536, 1536, 0.4)
            torch.cuda.synchronize()
        k = {}
        for e in prof.events():
            if str(e.device_type).endswith('CUDA'):
                k[e.name[:40]] = k.get(e.name[:40], 0.0) + getattr(e, 'device_time_total', 0.0) / 1e3
        res['post_kernel_ms'] = {n: round(v, 3) for n, v in sorted(k.items(), key=lambda kv: -kv[1])[:8]}
    return res


def part_chunk_sweep(tree, iters, io):
    """this tree only: post-processing ms and peak MB per NMS_CHUNK, on D0 512x512 bs 32 with every anchor a candidate
    and on the D7 bench image's network outputs (--io, written by d7_split); the hashes must not depend on the chunk"""
    torch, _, _ops, O, _ = _import(tree)
    dev = torch.device('cuda', 0)
    res = dict(part='chunk_sweep')
    B, K, S = 32, 80, 512
    a0 = torch.from_numpy(O.anchors_for(S, S)).to(dev)
    g = torch.Generator().manual_seed(7)
    cls0 = torch.rand(B, a0.shape[1], K, generator=g).to(dev)
    reg0 = (torch.randn(B, a0.shape[1], 4, generator=g) * 0.3).to(dev)
    cases = [('d0 bs32 all anchors', cls0, reg0, a0, S, -1.0, 2)]
    if io and os.path.exists(io):
        cls7, reg7 = [t.to(dev) for t in torch.load(io)]
        cases.append(('d7 bench image', cls7[:1], reg7[:1], torch.from_numpy(O.anchors_for(1536, 1536)).to(dev), 1536,
                      0.4, iters))
    for chunk in (1024, 2048, 4096, 8192):
        _ops.NMS_CHUNK = chunk
        for name, cls, reg, anchors, s, thr, n in cases:
            run = lambda: _post(_ops, cls, reg, anchors, s, s, thr)  # noqa: E731
            h = hashlib.sha256()
            for trip in run():
                for t in trip:
                    h.update(t.cpu().numpy().tobytes())
            res['%s chunk %d' % (name, chunk)] = dict(ms=_wall(torch, run, n), peak_mb=_peak_mb(torch, run),
                                                     sha256=h.hexdigest()[:16])
    return res


def _run(args):
    r = subprocess.run(args, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('%s failed:\n%s' % (' '.join(args), r.stdout[-2000:] + r.stderr[-4000:]))
    return json.loads(r.stdout.strip().splitlines()[-1])


def driver(runs, parent, out, iters, legs):
    import numpy as np
    card = subprocess.run(['nvidia-smi', '-i', '0', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True).stdout.strip()
    trees = {'parent': os.path.abspath(parent), 'this': R}
    me = os.path.abspath(__file__)
    summary = dict(card=card, runs=runs, iters=iters)
    if 'eager_vs_graph' in legs:
        summary['eager_vs_graph'] = _run([sys.executable, me, '--part', 'eager_vs_graph', '--iters', str(iters)])
    rows = {k: [] for k in trees}
    io = os.path.join(tempfile.mkdtemp(), 'd7_outputs.pt')            # 140 MB: kept out of the output directory
    for i in range(1, runs + 1):
        for k, t in trees.items():
            row = {}
            for part in ('post', 'd7_split'):
                if part in legs:
                    row[part] = _run([sys.executable, me, '--part', part, '--tree', t, '--iters', str(iters),
                                      '--io', io])
            if 'bench' in legs:
                row['bench'] = _run([sys.executable, os.path.join(t, 'bench.py'), '--gpus', '1', '--config', 'd7',
                                     '--steps', '10', '--warmup', '3', '--no-cpu', '--dump-outputs',
                                     os.path.join(out, 'd7_%s_%d' % (k, i))])
            rows[k].append(row)
    med = lambda v: dict(median=round(statistics.median(v), 3), min=round(min(v), 3), max=round(max(v), 3))  # noqa: E731
    for k, rs in rows.items():
        s = {}
        if 'post' in legs:
            for case in ('realistic', 'all_anchors'):
                s['post bs32 %s ms' % case] = med([r['post'][case]['ms'] for r in rs])
                s['post bs32 %s peak MB' % case] = rs[-1]['post'][case].get('peak_mb')
                s['post bs32 %s sha256' % case] = sorted({r['post'][case]['sha256'] for r in rs})
                s['post bs32 %s candidates min/max' % case] = rs[0]['post'][case]['candidates_min_max']
        if 'd7_split' in legs:
            for f in ('network_ms', 'post_ms', 'forward_ms'):
                s['d7 ' + f] = med([r['d7_split'][f] for r in rs])
            s['d7 candidates'] = rs[0]['d7_split']['candidates']
            s['d7 post peak MB'] = rs[-1]['d7_split'].get('post_peak_mb')
            s['d7 post sha256'] = sorted({r['d7_split']['sha256'] for r in rs})
            s['d7 post kernel ms (last run)'] = rs[-1]['d7_split']['post_kernel_ms']
        if 'bench' in legs:
            s['bench d7 img/s'] = med([r['bench']['value'] for r in rs])
        if s:
            summary[k] = s
    if 'chunk_sweep' in legs:
        summary['chunk_sweep'] = _run([sys.executable, me, '--part', 'chunk_sweep', '--iters', str(iters), '--io', io])
    if 'bench' in legs:
        # detections of separate processes differ by the network's fp32 atomics; the post-processing alone is compared
        # bit for bit by the d7_split leg
        for k in trees:
            summary.setdefault(k, {})['bench d7 detections per run'] = [
                int(np.load(os.path.join(out, 'd7_%s_%d' % (k, i), 'scores.npy')).shape[0]) for i in range(1, runs + 1)]
    print(json.dumps(summary, indent=1))
    with open(os.path.join(out, 'bench_detect_%s.json' % '_'.join(legs)), 'w') as fh:
        json.dump(dict(summary=summary, runs=rows), fh, indent=1)
    if os.path.exists(io):
        os.remove(io)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--part', choices=['eager_vs_graph', 'post', 'd7_split', 'chunk_sweep'])
    ap.add_argument('--tree', default=R, help='source tree whose library to measure')
    ap.add_argument('--iters', type=int, default=20)
    ap.add_argument('--driver', type=int, default=0, metavar='RUNS', help='alternate parent and this tree RUNS times')
    ap.add_argument('--parent', help='source tree of the build to compare against (driver)')
    ap.add_argument('--out', help='directory for the dumps and the summary (driver)')
    ap.add_argument('--io', help='d7_split: file of the network outputs every build post-processes')
    ap.add_argument('--legs', default='eager_vs_graph,post,d7_split,bench', help='driver: comma-separated parts to run')
    args = ap.parse_args()
    if args.driver:
        os.makedirs(args.out, exist_ok=True)
        driver(args.driver, args.parent, args.out, args.iters, args.legs.split(','))
    else:
        if args.part in ('d7_split', 'chunk_sweep'):
            res = dict(d7_split=part_d7_split, chunk_sweep=part_chunk_sweep)[args.part](args.tree, args.iters, args.io)
        else:
            res = dict(eager_vs_graph=part_eager_vs_graph, post=part_post)[args.part](args.tree, args.iters)
        print(json.dumps(res), flush=True)


if __name__ == '__main__':
    main()
