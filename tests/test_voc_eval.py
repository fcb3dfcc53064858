"""VOC mean average precision on the device (csrc/voc_eval.cu, models/evaluation.py) against tools/voc_eval_oracle.py,
which tests/golden/make_eval_golden.py pins to the reference's own eval.py code (tests/golden/voc_eval.npz).

CPU: the oracle equals the fixture, the pairwise-sum model equals np.sum, and the entry points refuse bad arguments.
GPU: the accumulator equals the fixture exactly in any batching, the batched selection equals the per-image one bit for
bit, ties follow the stable order, evaluate() equals the reference loop on a real D0, and add() is sync-free and
capturable."""
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


def _fixture():
    st = np.load(os.path.join(G, 'voc_eval.npz'))
    K, max_det = (int(v) for v in st['config'])
    gts = np.split(st['gt_rows'], np.cumsum(st['gt_counts'])[:-1])
    return st, K, max_det, gts


def _oracle_from_padded(scores, labels, boxes, count, scale, gts, K, thr=0.05, max_det=100, iou=0.5):
    dets = [V.select_detections(scores[i, :count[i]], labels[i, :count[i]], boxes[i, :count[i]], float(scale[i]), thr,
                                max_det, K) for i in range(scores.shape[0])]
    anns = [[g[g[:, 4] == c, :4] for c in range(K)] for g in gts]
    return V.evaluate(dets, anns, K, iou)


def _same(got, want):
    """(mean, {label: (ap, n)}) equal as float64, with the reference's zero for a label without ground truth"""
    assert got[0] == want[0], (got[0], want[0])
    assert sorted(got[1]) == sorted(want[1])
    for c in want[1]:
        assert got[1][c] == want[1][c], (c, got[1][c], want[1][c])
        assert float(got[1][c][0]) == float(want[1][c][0]) and float(got[1][c][1]) == float(want[1][c][1])


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------

def test_oracle_equals_reference_fixture():
    st, K, max_det, gts = _fixture()
    got = _oracle_from_padded(st['scores'], st['labels'].astype(np.int64), st['boxes'], st['count'], st['scale'], gts, K)
    want = (st['mean_ap'][0], {c: ((0, 0) if st['num_annotations'][c] == 0 else (st['ap'][c], st['num_annotations'][c]))
                               for c in range(K)})
    _same(got, want)
    assert st['num_annotations'][5] == 0 and st['num_annotations'][6] > 0 and st['ap'][6] == 0.0


def test_pairwise_sum_model_equals_np_sum():
    """the summation order the AP kernel follows is np.sum's on a contiguous float64 array, at every length up to 299
    and at lengths with several recursion levels, with magnitudes mixed over 16 decades"""
    rng = np.random.RandomState(0)
    for n in list(range(1, 300)) + [1000, 2049, 5000, 20000]:
        a = rng.rand(n) * 10.0 ** rng.randint(-8, 8, size=n)
        assert V.pairwise_sum(a) == np.sum(a), n
    # "first element plus the pairwise sum of the rest" is a different order: it must disagree somewhere
    bad = 0
    for n in range(9, 300):
        a = rng.rand(n) * 10.0 ** rng.randint(-8, 8, size=n)
        bad += (a[0] + V.pairwise_sum(a[1:])) != np.sum(a)
    assert bad > 0


@pytest.fixture(scope='module')
def lib():
    from models import _native
    _native.build()
    return _native.load()


def test_voc_entry_points_refuse_bad_arguments(lib):
    """each refusal returns -1, names the entry point and comes before any device work (never-dereferenced pointers),
    so these calls run without a GPU"""
    f = 1 << 20

    def refused(rc, what):
        msg = lib.effdet_last_error().decode()
        assert rc == -1 and what in msg, (rc, msg)

    def sel(*, sc=f, cnt=f, B=2, C=50, max_det=100, K=20, thr=0.05, box=f):
        return lib.effdet_eval_select_batch(sc, f, box, cnt, f, B, C, thr, max_det, K, f, f, f, f, 0, None)

    refused(sel(max_det=0), 'max_det=0')
    refused(sel(K=0), 'num_classes=0')
    refused(sel(max_det=12300, K=20), "too large")
    refused(sel(sc=None), 'null')
    refused(sel(cnt=None), 'null')
    refused(sel(B=0), 'B=0')
    refused(sel(box=f + 4), 'aligned')
    refused(sel(thr=-0.5), 'score_threshold')

    def match(*, gt=f, ngt=3, B=2, max_det=100, K=20, tp=f):
        return lib.effdet_voc_match(f, f, gt, f, ngt, B, max_det, K, 0.5, tp, f, 0, None)

    refused(match(max_det=0), 'max_det=0')
    refused(match(K=256), 'num_classes=256')
    refused(match(gt=None), 'null')
    refused(match(tp=None), 'null')
    refused(match(B=0), 'B=0')

    assert lib.effdet_voc_ap_workspace(1 << 25, 255) > 0
    assert lib.effdet_voc_ap_workspace((1 << 25) + 1, 20) == -1 and 'records' in lib.effdet_last_error().decode()
    assert lib.effdet_voc_ap_workspace(100, 256) == -1 and 'num_classes=256' in lib.effdet_last_error().decode()
    ws = lib.effdet_voc_ap_workspace(1000, 20)

    def ap(*, d=f, R=1000, K=20, ws_bytes=ws, w=f):
        return lib.effdet_voc_ap(d, f, f, f, R, K, f, f, w, ws_bytes, 0, None)

    refused(ap(R=(1 << 25) + 1), 'records')
    refused(ap(R=0), 'records')
    refused(ap(K=256), 'num_classes=256')
    refused(ap(d=None), 'null')
    refused(ap(ws_bytes=ws - 8), 'workspace')
    refused(ap(w=f + 8), 'aligned')


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------

def _dev():
    return torch.device('cuda:0')


def _detections(st, i0, i1):
    from models._ops import Detections
    d = _dev()
    return Detections(torch.from_numpy(st['scores'][i0:i1]).to(d),
                      torch.from_numpy(st['labels'][i0:i1].astype(np.int64)).to(d),
                      torch.from_numpy(st['boxes'][i0:i1]).to(d), torch.from_numpy(st['count'][i0:i1]).to(d))


@gpu
@pytest.mark.parametrize('batch', [1, 7, 300])
def test_accumulator_equals_fixture(batch):
    from models.evaluation import VOCAccumulator
    st, K, max_det, gts = _fixture()
    n = st['scores'].shape[0]
    acc = VOCAccumulator(K, n, device=_dev())
    for i0 in range(0, n, batch):
        i1 = min(n, i0 + batch)
        acc.add(_detections(st, i0, i1), [float(s) for s in st['scale'][i0:i1]], gts[i0:i1])
    got = acc.compute()
    want = (st['mean_ap'][0], {c: ((0, 0) if st['num_annotations'][c] == 0 else (st['ap'][c], st['num_annotations'][c]))
                               for c in range(K)})
    _same(got, want)
    assert type(got[1][5][0]) is int and type(got[1][0][1]) is float


@gpu
def test_select_batch_bit_exact_against_per_image_selection():
    """random padded detections with count 0, count > max_detections, per-image scales and one overflowed image: every
    image's rows equal select_detections on that image, bit for bit; the overflowed image writes nothing and is flagged"""
    from models import _native as N
    from models.pipeline import select_detections
    rng = np.random.RandomState(5)
    B, C, K, max_det, thr = 6, 300, 20, 100, 0.05
    scores = rng.rand(B, C).astype(np.float32)
    scores[:, 250:] = 0.0
    labels = rng.randint(-1, K + 1, size=(B, C)).astype(np.int64)            # a few labels outside [0, K)
    boxes = (rng.rand(B, C, 4) * 600).astype(np.float32)
    count = np.array([0, 250, 40, 180, -1, 130], np.int32)
    scale = np.array([1.0, 0.7371, 1.25, 0.5, 0.9, 1.6], np.float32)
    d = _dev()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(d)           # noqa: E731
    sc, lb, bx, cn, sl = t(scores), t(labels), t(boxes), t(count), t(scale)
    dets = torch.full((B, max_det, 5), 7.0, device=d)
    labs = torch.full((B, max_det), 7, dtype=torch.int32, device=d)
    offs = torch.full((B, K + 1), 7, dtype=torch.int32, device=d)
    ovf = torch.full((B,), 7, dtype=torch.int32, device=d)
    N.call('effdet_eval_select_batch', sc, N.f32(sc), N.ptr(lb), N.f32(bx), N.ptr(cn), N.ptr(sl), B, C, thr, max_det, K,
           N.f32(dets), N.ptr(labs), N.ptr(offs), N.ptr(ovf))
    assert ovf.tolist() == [0, 0, 0, 0, 1, 0]
    for b in range(B):
        if count[b] < 0:
            assert (labs[b] == -1).all() and (offs[b] == 0).all()
            continue
        n = int(count[b])
        rd, rl, ro = select_detections(sc[b, :n], lb[b, :n], bx[b, :n].contiguous(), float(scale[b]), thr, max_det, K)
        m = int(ro[-1])
        assert torch.equal(offs[b], ro), b
        assert torch.equal(dets[b, :m], rd[:m]) and torch.equal(labs[b, :m], rl[:m]), b
        assert (labs[b, m:] == -1).all(), b
    keep = np.where(scores[1, :250] > thr)[0]                                # count > max_detections: top 100 only,
    top = keep[np.argsort(-scores[1, keep], kind='stable')[:max_det]]       # then labels outside [0, K) dropped
    assert keep.size > max_det and int(offs[1, -1]) == int(((labels[1, top] >= 0) & (labels[1, top] < K)).sum())


@gpu
def test_tied_scores_follow_the_stable_order():
    """scores tied across images and inside an image: the AP equals the oracle's stable order (image, then rank), and
    the stable order differs from a reversed tie order, so the test can see it"""
    from models.evaluation import VOCAccumulator
    K, B, C = 2, 5, 8
    scores = np.zeros((B, C), np.float32)
    labels = np.zeros((B, C), np.int64)
    boxes = np.zeros((B, C, 4), np.float32)
    gts = []
    for i in range(B):
        scores[i, :6] = [0.9, 0.75, 0.75, 0.75, 0.5, 0.5]
        labels[i, :6] = [0, 0, 0, 1, 0, 0]
        for k in range(6):
            boxes[i, k] = [20 * k, 0, 20 * k + 10, 10]
        hit = [0, 1] if i < 2 else [0]                                       # tied records are TPs in images 0, 1 only
        gts.append(np.array([[20 * k, 0, 20 * k + 10, 10, labels[i, k]] for k in hit], np.float64))
    count = np.full(B, 6, np.int32)
    scale = np.ones(B, np.float32)
    want = _oracle_from_padded(scores, labels, boxes, count, scale, gts, K)
    # the same records appended in reverse image order give another AP: ties matter here
    rev = _oracle_from_padded(scores[::-1], labels[::-1], boxes[::-1], count, scale, gts[::-1], K)
    assert rev[1][0][0] != want[1][0][0]
    from models._ops import Detections
    d = _dev()
    acc = VOCAccumulator(K, B, device=d)
    acc.add(Detections(*(torch.from_numpy(a).to(d) for a in (scores, labels, boxes, count))), list(scale), gts)
    _same(acc.compute(), want)


class _Generator:
    """the VOC generator interface eval.py uses: images [H,W,3] float (after Normalizer + Resizer), a scale, and
    annotations [n,5] float64 in original image coordinates"""

    def __init__(self, images, scales, annotations, K):
        self.images, self.scales, self.annotations, self.K = images, scales, annotations, K

    def __len__(self):
        return len(self.images)

    def __getitem__(self, i):
        return {'img': self.images[i], 'scale': self.scales[i]}

    def load_annotations(self, i):
        return self.annotations[i]

    def num_classes(self):
        return self.K

    def label_to_name(self, label):
        return 'class%d' % label


def _d0_case():
    """D0 with the well-conditioned weights of the d0_512_fwd_wellcond fixture, 20 random 256x256 images, and ground
    truth placed on the model's own detections.  Two passes of the network over the same images differ in the last
    bits (the order of the SE-mean fp32 atomics), so the ground truth is laid out to make the result independent of
    that noise: every detection scoring above s* (the middle of a wide gap between neighbouring scores) gets a copy of
    its box (a TP), those below it none (FPs, also when they overlap a copy that is already taken), two boxes per
    image lie outside the image (never matched), and images 3 and 11 have none."""
    from models import EfficientDet
    K = 80
    cfg = O.make_config('efficientdet-d0', num_classes=K, W_bifpn=64, D_bifpn=2)
    m = EfficientDet(num_classes=K, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    m.load_state_dict(O.init_state_dict(cfg, seed=1, mode='wellcond'))
    m = m.to(_dev()).eval()
    m.threshold = 0.3
    x = O.synthetic_batch(20, size=256, seed=31)[0]
    images = [x[i].permute(1, 2, 0).contiguous() for i in range(20)]
    scales = [1.0 if i % 2 else 0.8 for i in range(20)]
    gen = _Generator(images, scales, [np.zeros((0, 5))] * 20, K)
    dets = V.get_detections(gen, m)
    sc = np.unique(np.concatenate([d[c][:, 4] for d in dets for c in range(K)]))
    lo, hi = int(0.3 * sc.size), int(0.7 * sc.size)
    j = lo + int(np.argmax(np.diff(sc[lo:hi])))
    s_star, gap = 0.5 * (sc[j] + sc[j + 1]), sc[j + 1] - sc[j]
    assert gap > 1e-5, gap
    anns = []
    for i in range(20):
        rows = [[1000, 1000, 1010, 1010, c] for c in (7, 57)]
        for c in range(K):
            rows += [[d[0], d[1], d[2], d[3], c] for d in dets[i][c] if d[4] > s_star]
        anns.append(np.array(rows, np.float64) if i not in (3, 11) else np.zeros((0, 5)))
    return m, _Generator(images, scales, anns, K)


def _reference_loop(gen, m):
    return V.evaluate(V.get_detections(gen, m), V.get_annotations(gen), gen.num_classes(), 0.5)


@gpu
def test_evaluate_end_to_end_equals_reference_loop(monkeypatch):
    """models.evaluation.evaluate with batch_size 8 (two graphed batches, an eager remainder of 4) returns the dict and
    mean of the reference loop (one model(image) per image, host selection and accumulation); then again with
    max_candidates small enough that some images overflow NMS and are redone eagerly"""
    from models import evaluation
    m, gen = _d0_case()
    want = _reference_loop(gen, m)
    assert any(want[1][c][1] and 0 < want[1][c][0] < 1 for c in want[1]), want      # TPs and FPs both occur
    got = evaluation.evaluate(gen, m, batch_size=8)
    _same(got, want)
    with torch.no_grad():
        x = torch.stack([gen[i]['img'].permute(2, 0, 1) for i in range(20)]).to(_dev())
        cls, _, _ = m._raw_predictions(x)
    counts = sorted((cls.max(dim=2)[0] > m.threshold).sum(dim=1).tolist())
    cap = counts[10]
    assert counts[0] > 0 and counts[-1] > cap
    monkeypatch.setattr(evaluation, 'MAX_CANDIDATES', cap)
    got = evaluation.evaluate(gen, m, batch_size=8)
    _same(got, want)
    m.is_training = True
    with pytest.raises(RuntimeError, match='inference mode'):
        evaluation.evaluate(gen, m)


@gpu
def test_add_is_sync_free_and_capturable():
    """add() under torch.cuda.set_sync_debug_mode('error') raises nothing; an add() captured in a CUDA graph and replayed
    leaves the accumulator exactly where the eager add() does"""
    from models.evaluation import VOCAccumulator
    st, K, max_det, gts = _fixture()
    B = 16
    dets = _detections(st, 0, B)
    scales = [float(s) for s in st['scale'][:B]]
    torch.cuda.synchronize()
    eager = VOCAccumulator(K, B, device=_dev())
    torch.cuda.set_sync_debug_mode('error')
    try:
        eager.add(dets, scales, gts[:B])
    finally:
        torch.cuda.set_sync_debug_mode(0)
    want = eager.compute()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        VOCAccumulator(K, B, device=_dev()).add(dets, scales, gts[:B])          # warm-up off the capture
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    graphed = VOCAccumulator(K, B, device=_dev())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        graphed.add(dets, scales, gts[:B])
    g.replay()
    torch.cuda.synchronize()
    for a, b in ((graphed.dets, eager.dets), (graphed.labels, eager.labels), (graphed.tp, eager.tp),
                 (graphed.gt_count, eager.gt_count), (graphed.overflow, eager.overflow)):
        assert torch.equal(a, b)
    _same(graphed.compute(), want)
