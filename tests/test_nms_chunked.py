"""Greedy NMS in column chunks (csrc/detect.cu `effdet_nms_batch_chunked`): the workspace is linear in the candidate cap,
and the keep sets equal the one-chunk NMS (`effdet_nms_batch`) and torchvision's, bit for bit, for every chunk size.

CPU: the entry point's and the workspace function's refusals, and a NumPy restatement of the chunked greedy against
torchvision.ops.nms on the golden boxes and seeded random sets.
GPU: the torchvision goldens and edge cases at chunk boundaries, real D0 outputs with every anchor a candidate against
the one-chunk call, GraphedDetect(max_candidates=None), the memory of D7 post-processing, and evaluate() at its default
MAX_CANDIDATES."""
import os
import sys

import numpy as np
import pytest
import torch

import effdet_oracle as O

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), 'tools'))
import voc_eval_oracle as V  # noqa: E402

G = os.path.join(HERE, 'golden')
gpu = pytest.mark.gpu


def _dev():
    return torch.device('cuda:0')


def _golden():
    st = np.load(os.path.join(G, 'nms_torchvision.npz'))
    return [(st['c%d/boxes' % c], st['c%d/scores' % c], st['c%d/keep' % c]) for c in range(4)]


def _host_keys(scores):
    """sort keys exactly as the candidate kernel builds them: (~order(score)) << 32 | index"""
    u = scores.astype(np.float32).view(np.uint32).astype(np.uint64)
    neg = (u & np.uint64(0x80000000)) != 0
    order = np.where(neg, (~u) & np.uint64(0xffffffff), u | np.uint64(0x80000000))
    inv = (~order) & np.uint64(0xffffffff)
    return (inv << np.uint64(32)) | np.arange(scores.shape[0], dtype=np.uint64)


def _iou_gt(a, b, thr):
    """iou_gt of detect.cu for one box a against boxes b [m,4]: fp32 operations, the comparison in float64"""
    left, right = np.maximum(a[0], b[:, 0]), np.minimum(a[2], b[:, 2])
    top, bottom = np.maximum(a[1], b[:, 1]), np.minimum(a[3], b[:, 3])
    w = np.maximum(right - left, np.float32(0))
    h = np.maximum(bottom - top, np.float32(0))
    inter = w * h
    sa = (a[2] - a[0]) * (a[3] - a[1])
    sb = (b[:, 2] - b[:, 0]) * (b[:, 3] - b[:, 1])
    with np.errstate(divide='ignore', invalid='ignore'):
        ovr = inter / ((sa + sb) - inter)
    return (w > 0) & (h > 0) & (ovr.astype(np.float64) > thr)


def chunked_nms(boxes, scores, thr, chunk):
    """the chunked greedy NMS: per chunk of `chunk` sorted candidates, remove those a box kept by an earlier chunk
    suppresses (cross step), then the greedy inside the chunk.  -> kept indices, best first"""
    boxes = boxes.astype(np.float32)
    order = np.argsort(-scores.astype(np.float32), kind='stable')
    keep = []
    for base in range(0, order.size, chunk):
        idx = order[base:base + chunk]
        cand = boxes[idx]
        removed = np.zeros(idx.size, dtype=bool)
        for k in keep:                                          # cross step: earlier box first
            removed |= _iou_gt(boxes[k], cand, thr)
        for i in range(idx.size):                               # greedy inside the chunk
            if removed[i]:
                continue
            keep.append(int(idx[i]))
            removed[i + 1:] |= _iou_gt(cand[i], cand[i + 1:], thr)
    return np.array(keep, dtype=np.int64)


def _random_set(seed, n=700):
    rng = np.random.RandomState(seed)
    xy = rng.uniform(0, 200, size=(n, 2))
    wh = rng.uniform(4, 60, size=(n, 2))
    return np.concatenate([xy, xy + wh], axis=1).astype(np.float32), rng.uniform(size=n).astype(np.float32)


def _edge_case():
    """256 candidates whose sorted order puts chunk boundaries inside runs of tied scores of overlapping boxes (sorted
    positions 50-78 across 64, 120-135 across 128) and between two boxes with IoU exactly 0.5 (positions 191 | 192 at
    chunk 64 and 192: both kept, IoU is not > 0.5).  The first and the last candidate have IoU just above 0.5, so the
    last one is removed by the cross step of every chunk size below 256.  -> boxes, scores"""
    n = 256
    rng = np.random.RandomState(3)
    boxes = np.zeros((n, 4), np.float32)
    for i in range(n):                                          # disjoint filler boxes on a grid
        x, y = (i % 16) * 100.0, (i // 16) * 100.0
        boxes[i] = [x, y, x + 10, y + 10]
    scores = np.sort(rng.uniform(0.1, 0.9, size=n).astype(np.float32))[::-1].copy()
    for lo, hi, y in ((50, 79, 0.0), (120, 136, 500.0)):      # tie runs of overlapping boxes
        scores[lo:hi] = scores[lo]
        for i in range(lo, hi):
            boxes[i] = [3000 + (i - lo) * 2.0, y, 3000 + (i - lo) * 2.0 + 10, y + 10]
    boxes[191] = [5000, 0, 5003, 1]                             # IoU([0,3],[1,4]) = 2/4 = 0.5 exactly
    boxes[192] = [5001, 0, 5004, 1]
    boxes[255] = [5100, 0, 5103.001, 1]                         # IoU just above 0.5 with position 0's partner below
    boxes[0] = [5101, 0, 5104, 1]
    perm = rng.permutation(n)                                   # anchor order differs from score order
    return boxes[perm], scores[perm]


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def lib():
    from models import _native
    _native.build()
    return _native.load()


def test_chunked_entry_points_refuse_bad_arguments(lib):
    """each refusal returns -1 (EFFDET_ERR_ARG), names the entry point and comes before any device work: the pointers
    are never dereferenced, so these calls run without a GPU"""
    f = 1 << 20                                                 # aligned non-null "pointer"

    def refused(rc, name):
        msg = lib.effdet_last_error().decode()
        assert rc == -1 and name in msg, (rc, msg)

    B, cap, chunk = 2, 1000, 128
    need = lib.effdet_nms_chunked_workspace(B, cap, chunk)
    cw = 2
    assert need == B * (chunk * cw + cw) * 8
    assert lib.effdet_nms_chunked_workspace(B, cap, cap) == B * cap * 16 * 8     # one chunk: effdet_nms_batch's mask
    assert lib.effdet_nms_chunked_workspace(1, 441936, 4096) == (4096 * 64 + 64) * 8
    for args in ((0, cap, chunk), (65536, cap, chunk), (B, 0, 64), (B, cap, 100), (B, cap, 0), (B, cap, 1024 + 64 * 16),
                 (B, 100, 128), (B, 1 << 21, 1 << 21)):
        refused(lib.effdet_nms_chunked_workspace(*args), 'nms_chunked_workspace')

    def nms(*, p=f, cnt=f, B=B, A=2000, npad=2048, cap=cap, chunk=chunk, ws=f, ws_bytes=need, box=f, keep=f):
        return lib.effdet_nms_batch_chunked(box, p, cnt, B, A, npad, cap, chunk, 0.5, ws, ws_bytes, keep, f, 0, None)

    for kw in (dict(p=None), dict(cnt=None), dict(ws=None), dict(keep=None), dict(B=0), dict(B=65536),
               dict(npad=2000), dict(npad=1024), dict(cap=0), dict(A=999, npad=1024), dict(chunk=100), dict(chunk=0),
               dict(chunk=1024 + 64), dict(ws_bytes=need - 1), dict(box=f + 8), dict(ws=f + 8)):
        refused(nms(**kw), 'nms_batch_chunked')


@pytest.mark.parametrize('chunk', [64, 128, 192, None])
def test_numpy_chunked_greedy_equals_torchvision(chunk):
    """the restatement of the chunked greedy equals torchvision.ops.nms on the golden boxes (which cover ties and IoU
    == thr) and on seeded random sets; chunk None = one chunk of all candidates"""
    tv = pytest.importorskip('torchvision')
    for boxes, scores, keep in _golden():
        got = chunked_nms(boxes, scores, 0.5, chunk or boxes.shape[0])
        assert np.array_equal(got, keep), chunk
    for seed in range(3):
        boxes, scores = _random_set(seed)
        for thr in (0.3, 0.5):
            want = tv.ops.nms(torch.from_numpy(boxes), torch.from_numpy(scores), thr).numpy()
            got = chunked_nms(boxes, scores, thr, chunk or boxes.shape[0])
            assert np.array_equal(got, want), (chunk, seed, thr)


def test_numpy_chunked_greedy_edge_case_is_chunk_independent():
    """the boundary case: the restatement gives one keep list for every chunk, equal to the greedy oracle's; the
    exact-0.5 pair keeps both boxes, the pair just above 0.5 (first and last candidate) only the first"""
    boxes, scores = _edge_case()
    want = O.nms_greedy(torch.from_numpy(boxes), torch.from_numpy(scores), 0.5).numpy()
    for chunk in (64, 128, 192, 256):
        assert np.array_equal(chunked_nms(boxes, scores, 0.5, chunk), want), chunk
    order = np.argsort(-scores, kind='stable')
    assert order[191] in want and order[192] in want
    assert order[0] in want and order[255] not in want


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------

def _run_chunked(boxes_d, keys_d, count_d, A, npad, cap, chunk, thr=0.5, fill=-7):
    """effdet_nms_batch_chunked on device tensors -> keep [B,cap] (rows start at `fill`), nkeep [B]"""
    from models import _native as N
    B = boxes_d.shape[0]
    nbytes = int(N.load().effdet_nms_chunked_workspace(B, cap, chunk))
    assert nbytes > 0
    ws = torch.empty(nbytes // 8, dtype=torch.int64, device=boxes_d.device)
    keep = torch.full((B, cap), fill, dtype=torch.int32, device=boxes_d.device)
    nkeep = torch.empty(B, dtype=torch.int32, device=boxes_d.device)
    N.call('effdet_nms_batch_chunked', boxes_d, N.f32(boxes_d), keys_d.data_ptr(), count_d.data_ptr(), B, A, npad, cap,
           chunk, float(thr), ws.data_ptr(), nbytes, keep.data_ptr(), nkeep.data_ptr())
    return keep, nkeep


def _host_batch(cases):
    """[(boxes, scores)] -> device boxes [B,A,4], sorted keys [B,npad], counts [B], A, npad"""
    B, A = len(cases), max(c[0].shape[0] for c in cases)
    npad = 1 << (A - 1).bit_length()
    boxes = np.zeros((B, A, 4), np.float32)
    keys = np.full((B, npad), np.uint64(0xffffffffffffffff), np.uint64)
    counts = np.zeros(B, np.int32)
    for b, (bx, sc) in enumerate(cases):
        n = bx.shape[0]
        boxes[b, :n] = bx
        keys[b, :n] = np.sort(_host_keys(sc))
        counts[b] = n
    d = _dev()
    return (torch.from_numpy(boxes).to(d), torch.from_numpy(keys.view(np.int64)).to(d), torch.from_numpy(counts).to(d),
            A, npad)


@gpu
def test_chunked_keep_sets_equal_torchvision_golden_and_edge_cases():
    """the four torchvision goldens and the chunk-boundary case (tie runs across boundaries, IoU exactly 0.5 and just
    above it) as one batch: every keep list equals the expected one, order included, for chunk 64, 128 and cap = A =
    3000 (one chunk; chunk 4096 is the same single chunk at this size); with cap below the largest count that image reports -1 and nothing is written for it"""
    gold = _golden()
    eb, es = _edge_case()
    cases = [(b, s) for b, s, _ in gold] + [(eb, es)]
    want = [k for _, _, k in gold] + [O.nms_greedy(torch.from_numpy(eb), torch.from_numpy(es), 0.5).numpy()]
    boxes_d, keys_d, count_d, A, npad = _host_batch(cases)
    counts = count_d.cpu().numpy()
    for cap, chunk in ((A, 64), (A, 128), (A, A), (2000, 64), (2000, 2000)):
        keep, nkeep = _run_chunked(boxes_d, keys_d, count_d, A, npad, cap, chunk)
        nk = nkeep.cpu().numpy()
        for b, ref in enumerate(want):
            if counts[b] > cap:
                assert nk[b] == -1 and (keep[b].cpu() == -7).all(), (cap, chunk, b)
                continue
            assert nk[b] == ref.shape[0], (cap, chunk, b, nk[b], ref.shape[0])
            assert np.array_equal(keep[b, :nk[b]].cpu().numpy().astype(np.int64), ref), (cap, chunk, b)


def _candidates(cls, reg, anchors, H, W, thr):
    from models import _native as N
    B, A, K = cls.shape
    npad = 1 << (A - 1).bit_length()
    d = cls.device
    boxes = torch.empty(B, A, 4, device=d)
    scores = torch.empty(B, A, device=d)
    classes = torch.empty(B, A, dtype=torch.int32, device=d)
    keys = torch.empty(B, npad, dtype=torch.int64, device=d)
    count = torch.empty(B, dtype=torch.int32, device=d)
    N.call('effdet_detect_candidates_batch', cls, N.f32(cls), N.f32(reg), N.f32(anchors.view(-1, 4).contiguous()),
           N.f32(boxes), N.f32(scores), classes.data_ptr(), keys.data_ptr(), count.data_ptr(), B, A, K, npad,
           float(W), float(H), float(thr))
    return boxes, keys, count, npad


def _d0_model(size_seed=1, K=80):
    from models import EfficientDet
    cfg = O.make_config('efficientdet-d0', num_classes=K, W_bifpn=64, D_bifpn=2)
    m = EfficientDet(num_classes=K, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    m.load_state_dict(O.init_state_dict(cfg, seed=size_seed, mode='wellcond'))
    return m.to(_dev()).eval()


@gpu
def test_real_d0_every_anchor_chunked_equals_one_chunk():
    """D0 512x512, B = 4, well-conditioned random weights, threshold 0 (every one of the 49 104 anchors of images 0 and 1
    is a candidate; images 2 and 3 have part of their scores zeroed): the chunked NMS at chunk 64 and 4096 equals
    effdet_nms_batch (one chunk, the square mask) bit for bit; with cap below the counts of images 0 and 1 those report
    -1 with nothing written, and images 2 and 3 are unchanged"""
    from models import _native as N
    m = _d0_model()
    x = O.synthetic_batch(4, size=512, seed=41)[0].to(_dev())
    with torch.no_grad():
        cls, reg, anchors = m._raw_predictions(x)
    cls = cls.clone()
    cls[2, :20000] = 0.0
    cls[3, ::2] = 0.0
    boxes, keys, count, npad = _candidates(cls, reg, anchors, 512, 512, 0.0)
    B, A = cls.shape[0], cls.shape[1]
    assert count.tolist() == [A, A, A - 20000, A - (A + 1) // 2]
    cw = (A + 63) // 64
    mask = torch.empty(B * A * cw, dtype=torch.int64, device=_dev())
    ref_keep = torch.full((B, A), -7, dtype=torch.int32, device=_dev())
    ref_n = torch.empty(B, dtype=torch.int32, device=_dev())
    N.call('effdet_nms_batch', boxes, N.f32(boxes), keys.data_ptr(), count.data_ptr(), B, A, npad, A, 0.5,
           mask.data_ptr(), ref_keep.data_ptr(), ref_n.data_ptr())
    del mask
    ref_n = ref_n.cpu()
    assert (ref_n > 0).all()
    print('kept per image', ref_n.tolist())
    for chunk in (64, 4096):
        keep, nkeep = _run_chunked(boxes, keys, count, A, npad, A, chunk)
        assert torch.equal(nkeep.cpu(), ref_n), chunk
        for b in range(B):
            assert torch.equal(keep[b, :ref_n[b]], ref_keep[b, :ref_n[b]]), (chunk, b)
    cap = 30000
    for chunk in (64, 4096):
        keep, nkeep = _run_chunked(boxes, keys, count, A, npad, cap, chunk)
        nk = nkeep.cpu()
        assert nk[0] == -1 and nk[1] == -1 and (keep[:2].cpu() == -7).all(), chunk
        for b in (2, 3):
            assert nk[b] == ref_n[b] and torch.equal(keep[b, :nk[b]], ref_keep[b, :nk[b]]), (chunk, b)


@gpu
def test_graphed_detect_every_anchor_never_overflows():
    """GraphedDetect(max_candidates=None) on D0 256x256 (A = 12 276), B = 3, at a threshold that gives some image more
    than 8192 candidates: no count is -1, the replay equals eager detect_batch on the same network outputs bit for bit,
    and two replays of the captured post-processing on those outputs are bit-identical to it"""
    from models import _ops
    from models.graph_step import GraphedDetect
    m = _d0_model(K=20)
    x = O.synthetic_batch(3, size=256, seed=51)[0].to(_dev())
    with torch.no_grad():
        cls, _, _ = m._raw_predictions(x)
    best = cls.max(dim=2)[0]
    m.threshold = float(torch.sort(best[0], descending=True)[0][9000])
    m.iou_threshold = 0.5
    assert int((best[0] > m.threshold).sum()) > 8192
    det = GraphedDetect(m, x, max_candidates=None)
    out = det(x)
    assert out.scores.shape == (3, cls.shape[1])
    first = [t.clone() for t in out]
    counts = out.count.tolist()
    assert min(counts) >= 0, counts
    eager = _ops.detect_batch(det.cls, det.reg, det.anchors, 256, 256, m.threshold, m.iou_threshold)
    got = det.to_list(out)
    for g_, e in zip(got, eager):
        for a, b in zip(g_, e):
            assert a.dtype == b.dtype and torch.equal(a, b)
    # two network passes differ in the last bits (SE-mean fp32 atomics), so the replay of the post-processing alone is
    # compared: detect_batch with cap = A captured on static network outputs, replayed twice
    cls, reg = det.cls.clone(), det.reg.clone()
    cap = _ops.candidate_cap(None, cls)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        _ops.detect_batch(cls, reg, det.anchors, 256, 256, m.threshold, 0.5, cap=cap)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        post = _ops.detect_batch(cls, reg, det.anchors, 256, 256, m.threshold, 0.5, cap=cap)
    replays = []
    for _ in range(2):
        graph.replay()
        torch.cuda.synchronize()
        replays.append([t.clone() for t in post])
    for a, b, c in zip(replays[0], replays[1], first):
        assert torch.equal(a, b) and torch.equal(a, c)


@gpu
def test_d7_post_processing_memory_is_bounded(monkeypatch):
    """D7 1536x1536 (A = 441 936), B = 1, seeded 80-class scores and box offsets, threshold 0.01: every anchor is a
    candidate, which the square mask would need 24.4 GB for.  Eager detect_batch allocates under 64 MB at its peak, and
    chunk 4096 and chunk 2048 keep the same boxes."""
    from models import _ops
    anchors = torch.from_numpy(O.anchors_for(1536, 1536)).to(_dev())
    A = anchors.shape[1]
    g = torch.Generator().manual_seed(61)
    cls = torch.rand(1, A, 80, generator=g).to(_dev())
    reg = (torch.randn(1, A, 4, generator=g) * 0.3).to(_dev())
    assert int((cls.max(dim=2)[0] > 0.01).sum()) == A
    monkeypatch.setattr(_ops, 'NMS_CHUNK', 4096)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    a = _ops.detect_batch(cls, reg, anchors, 1536, 1536, 0.01, 0.5)[0]
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    print('D7 every anchor: %d kept, peak extra memory %.1f MB' % (a[0].numel(), peak / 1e6))
    assert peak < 64 * 2 ** 20, peak
    monkeypatch.setattr(_ops, 'NMS_CHUNK', 2048)
    b = _ops.detect_batch(cls, reg, anchors, 1536, 1536, 0.01, 0.5)[0]
    for ta, tb in zip(a, b):
        assert torch.equal(ta, tb)


class _Generator:
    """the VOC generator interface of eval.py: images [H,W,3], a scale, annotations [n,5] in image coordinates"""

    def __init__(self, images, annotations, K):
        self.images, self.annotations, self.K = images, annotations, K

    def __len__(self):
        return len(self.images)

    def __getitem__(self, i):
        return {'img': self.images[i], 'scale': 1.0}

    def load_annotations(self, i):
        return self.annotations[i]

    def num_classes(self):
        return self.K

    def label_to_name(self, label):
        return 'class%d' % label


@gpu
def test_evaluate_default_max_candidates_equals_reference_loop():
    """evaluate() at the default MAX_CANDIDATES on 10 D0 256x256 images (batch 4: two graphed batches, an eager
    remainder of 2), at a threshold that gives images more than 8192 candidates, returns the reference loop's mAP.
    Two network passes differ in the last bits, so the ground truth sits on the model's own detections above the
    middle of a wide score gap (TPs) and none below (FPs), as in test_voc_eval."""
    from models import evaluation
    assert evaluation.MAX_CANDIDATES is None
    K, n = 20, 10
    m = _d0_model(K=K)
    x = O.synthetic_batch(n, size=256, seed=71)[0]
    with torch.no_grad():
        cls, _, _ = m._raw_predictions(x.to(_dev()))
    best = cls.max(dim=2)[0]
    m.threshold = float(torch.sort(best[0], descending=True)[0][9000])
    counts = (best > m.threshold).sum(dim=1).tolist()
    assert sum(c > 8192 for c in counts) >= 1, counts
    images = [x[i].permute(1, 2, 0).contiguous() for i in range(n)]
    gen = _Generator(images, [np.zeros((0, 5))] * n, K)
    dets = V.get_detections(gen, m)
    sc = np.unique(np.concatenate([d[c][:, 4] for d in dets for c in range(K)]))
    lo, hi = int(0.3 * sc.size), int(0.7 * sc.size)
    j = lo + int(np.argmax(np.diff(sc[lo:hi])))
    s_star = 0.5 * (sc[j] + sc[j + 1])
    assert sc[j + 1] - sc[j] > 1e-5
    anns = []
    for i in range(n):
        rows = [[1000, 1000, 1010, 1010, 3]]
        for c in range(K):
            rows += [[d[0], d[1], d[2], d[3], c] for d in dets[i][c] if d[4] > s_star]
        anns.append(np.array(rows, np.float64))
    gen = _Generator(images, anns, K)
    want = V.evaluate(V.get_detections(gen, m), V.get_annotations(gen), K, 0.5)
    got = evaluation.evaluate(gen, m, batch_size=4)
    assert got[0] == want[0], (got[0], want[0])
    for c in range(K):
        assert got[1][c] == want[1][c] or (got[1][c][1] == want[1][c][1] == 0), c
