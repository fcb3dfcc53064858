"""Batched, sync-free inference post-processing (csrc/detect.cu `*_batch` entry points, `_ops.detect_batch`) and the
CUDA-graph inference step (`models/graph_step.py::GraphedDetect`).

GPU tests hold the keep-sets to bit equality (torchvision goldens, the oracle's greedy NMS over the device's own
candidates, B = 1 slices, graph replays).  Whole-network comparisons use the forward-vs-detect_batch tolerance of
test_gpu_parity: two passes over the same images differ by the order of the SE-mean fp32 atomics.  The CPU tests check
the argument refusals and GraphedDetect's preconditions."""
import os

import numpy as np
import pytest
import torch

import effdet_oracle as O

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden')
gpu = pytest.mark.gpu


def _dev():
    return torch.device('cuda:0')


@pytest.fixture(params=['bf16x3', 'fp32'])
def prec(request):
    from models import _ops as ops
    old = ops.PRECISION
    ops.PRECISION = request.param
    yield request.param
    ops.PRECISION = old


def _host_keys(scores):
    """sort keys exactly as the candidate kernel builds them: (~order(score)) << 32 | index."""
    u = scores.astype(np.float32).view(np.uint32).astype(np.uint64)
    neg = (u & np.uint64(0x80000000)) != 0
    order = np.where(neg, (~u) & np.uint64(0xffffffff), u | np.uint64(0x80000000))
    inv = (~order) & np.uint64(0xffffffff)
    return (inv << np.uint64(32)) | np.arange(scores.shape[0], dtype=np.uint64)


def _model(seed, K=20):
    from models import EfficientDet
    cfg = O.make_config('efficientdet-d0', num_classes=K, W_bifpn=64, D_bifpn=2)
    m = EfficientDet(num_classes=K, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    m.load_state_dict(O.init_state_dict(cfg, seed=seed))
    m = m.to(_dev())
    m.eval()
    return m


def _images(B, seed):
    return O.synthetic_batch(B, size=256, seed=seed)[0].to(_dev())


def _threshold(cls, rank=300, images=None):
    """a score threshold that passes at least `rank` candidates in each of the given images"""
    best = cls.max(dim=2)[0]
    images = range(cls.shape[0]) if images is None else images
    return min(float(torch.sort(best[b], descending=True)[0][rank]) for b in images)


def _same_rows(a, b):
    """detections of two network passes over the same image: counts within 1, rows matched at 1e-2 px / 1e-4 score"""
    a = [t.cpu().numpy() for t in a]
    b = [t.cpu().numpy() for t in b]
    assert abs(a[0].shape[0] - b[0].shape[0]) <= 1, (a[0].shape[0], b[0].shape[0])
    used, matched = np.zeros(a[0].shape[0], dtype=bool), 0
    for j in range(b[0].shape[0]):
        if not a[0].shape[0]:
            break
        dist = np.abs(a[2] - b[2][j]).sum(axis=1) + used * 1e9
        k = int(np.argmin(dist))
        if dist[k] < 1e-2 and abs(a[0][k] - b[0][j]) < 1e-4 and a[1][k] == b[1][j]:
            used[k] = True
            matched += 1
    assert matched >= b[0].shape[0] - 1, (matched, b[0].shape[0])


# ------------------------------------------------------------------------------------------------
# kernels
# ------------------------------------------------------------------------------------------------

@gpu
def test_nms_batch_keep_sets_equal_torchvision_golden():
    """the four torchvision golden cases as one batch (one image each, 200 / 1500 / 64 / 3000 candidates): every keep
    list equals torchvision's, order included; with cap below the largest count that image reports -1 and the others
    stay exact"""
    from models import _native as N
    st = np.load(os.path.join(G, 'nms_torchvision.npz'))
    cases = [(st['c%d/boxes' % c], st['c%d/scores' % c], st['c%d/keep' % c]) for c in range(4)]
    B, A = len(cases), max(c[0].shape[0] for c in cases)
    npad = 1 << (A - 1).bit_length()
    boxes = np.zeros((B, A, 4), np.float32)
    keys = np.full((B, npad), np.uint64(0xffffffffffffffff), np.uint64)
    counts = np.zeros(B, np.int32)
    for b, (bx, sc, _) in enumerate(cases):
        n = bx.shape[0]
        boxes[b, :n] = bx
        keys[b, :n] = np.sort(_host_keys(sc))
        counts[b] = n
    d = _dev()
    boxes_d = torch.from_numpy(boxes).to(d)
    keys_d = torch.from_numpy(keys.view(np.int64)).to(d)
    count_d = torch.from_numpy(counts).to(d)
    for cap in (A, 2000):
        cw = (cap + 63) // 64
        mask = torch.empty(B * cap * cw, dtype=torch.int64, device=d)
        keep = torch.full((B, cap), -7, dtype=torch.int32, device=d)
        nkeep = torch.empty(B, dtype=torch.int32, device=d)
        N.call('effdet_nms_batch', boxes_d, N.f32(boxes_d), keys_d.data_ptr(), count_d.data_ptr(), B, A, npad, cap, 0.5,
               mask.data_ptr(), keep.data_ptr(), nkeep.data_ptr())
        nk = nkeep.cpu().numpy()
        for b, (_, _, ref) in enumerate(cases):
            if counts[b] > cap:
                assert nk[b] == -1, (cap, b, nk[b])
                assert (keep[b].cpu() == -7).all()                    # nothing written for an overflowed image
                continue
            assert nk[b] == ref.shape[0], (cap, b, nk[b], ref.shape[0])
            assert np.array_equal(keep[b, :nk[b]].cpu().numpy().astype(np.int64), ref), (cap, b)


@gpu
def test_detect_candidates_sort_and_decode():
    """B = 2 seeded draws, each with a block of exactly tied scores above the threshold: per image, scores and classes
    equal the oracle's class max, boxes its decode + clip, and the sorted key segment (sentinels included) equals the
    host keys, so candidates come best first with ties broken by anchor index"""
    from models import _native as N
    A, K, npad, thr = 5000, 20, 8192, 0.93
    g = torch.Generator().manual_seed(17)
    cls0 = torch.rand(1, A, K, generator=g)
    cls0[0, 100:400] = cls0[0, 100:101]                # exact score ties -> index order must decide
    reg0 = torch.randn(1, A, 4, generator=g) * 0.5
    xy = torch.rand(A, 2, generator=g) * 200
    anchors = torch.cat([xy, xy + torch.rand(A, 2, generator=g) * 60 + 4], dim=1)
    g = torch.Generator().manual_seed(18)
    cls1 = torch.rand(1, A, K, generator=g)
    cls1[0, 2000:2600] = cls1[0, 2000:2001]
    reg1 = torch.randn(1, A, 4, generator=g) * 0.5
    cls, reg = torch.cat([cls0, cls1]), torch.cat([reg0, reg1])
    B, ties = 2, (slice(100, 400), slice(2000, 2600))
    d = _dev()
    boxes = torch.empty(B, A, 4, device=d); scores = torch.empty(B, A, device=d)
    classes = torch.empty(B, A, dtype=torch.int32, device=d); keys = torch.empty(B, npad, dtype=torch.int64, device=d)
    count = torch.empty(B, dtype=torch.int32, device=d)
    cd, rd, ad = cls.to(d), reg.to(d), anchors.to(d)
    N.call('effdet_detect_candidates_batch', cd, N.f32(cd), N.f32(rd), N.f32(ad), N.f32(boxes), N.f32(scores),
           classes.data_ptr(), keys.data_ptr(), count.data_ptr(), B, A, K, npad, 256.0, 224.0, thr)
    ref_boxes = O.clip_boxes(O.decode_boxes(anchors[None], reg), 224, 256)
    for b in range(B):
        ref_s, ref_c = cls[b].max(dim=1)
        assert torch.equal(scores[b].cpu(), ref_s), b
        assert torch.equal(classes[b].cpu().long(), ref_c), b
        assert O.rel_err(boxes[b].cpu(), ref_boxes[b]) < 1e-6, b
        mask = ref_s > thr
        assert bool(mask[ties[b]].all()) and ref_s[ties[b]].unique().numel() == 1, b
        n = int(mask.sum())
        assert int(count[b]) == n and n > 100, b
        hk = _host_keys(ref_s.numpy())
        hk[~mask.numpy()] = np.uint64(0xffffffffffffffff)
        full = np.full(npad, np.uint64(0xffffffffffffffff), dtype=np.uint64)
        full[:A] = hk
        assert np.array_equal(keys[b].cpu().numpy().view(np.uint64), np.sort(full)), b
        order = (keys[b, :n].cpu().numpy().view(np.uint64) & np.uint64(0xffffffff)).astype(np.int64)
        ref_order = torch.nonzero(mask)[:, 0][torch.sort(ref_s[mask], descending=True, stable=True)[1]]
        assert np.array_equal(order, ref_order.numpy()), b


@gpu
def test_real_model_keep_sets_exact_and_batch_equals_slices():
    """D0 256x256, B = 4, random weights, a threshold passing a few hundred candidates and one image with none: every
    keep-set equals the oracle's greedy NMS over the device's own decoded candidates, and the batched call is
    bit-identical to B = 1 calls on each image's slice"""
    from models import _native as N
    from models import _ops as ops
    m = _model(seed=71)
    x = _images(4, seed=72)
    with torch.no_grad():
        cls, reg, anchors = m._raw_predictions(x)
    cls = cls.clone()
    cls[3] = 0.0                                                      # image 3: nothing passes
    thr = _threshold(cls, images=range(3))
    H, W = x.shape[2], x.shape[3]
    dets = ops.detect_batch(cls, reg, anchors, H, W, thr, 0.5)
    assert len(dets) == 4
    # the device's decoded candidates of every anchor
    B, A, K = cls.shape
    npad = 1 << (A - 1).bit_length()
    boxes = torch.empty(B, A, 4, device=_dev())
    scores = torch.empty(B, A, device=_dev())
    classes = torch.empty(B, A, dtype=torch.int32, device=_dev())
    keys = torch.empty(B, npad, dtype=torch.int64, device=_dev())
    count = torch.empty(B, dtype=torch.int32, device=_dev())
    N.call('effdet_detect_candidates_batch', cls, N.f32(cls), N.f32(reg), N.f32(anchors.view(-1, 4).contiguous()),
           N.f32(boxes), N.f32(scores), classes.data_ptr(), keys.data_ptr(), count.data_ptr(), B, A, K, npad,
           float(W), float(H), thr)
    boxes, scores, classes, count = boxes.cpu(), scores.cpu(), classes.cpu(), count.cpu()
    for b in range(B):
        sel = torch.nonzero(scores[b] > thr)[:, 0]
        assert int(count[b]) == sel.numel()
        if b == 3:
            assert sel.numel() == 0 and dets[b][0].numel() == 0 and tuple(dets[b][2].shape) == (0, 4)
            continue
        assert sel.numel() >= 300, sel.numel()
        idx = sel[O.nms_greedy(boxes[b, sel], scores[b, sel], 0.5)]
        got = [t.cpu() for t in dets[b]]
        assert got[1].dtype == torch.int64
        assert torch.equal(got[0], scores[b, idx]) and torch.equal(got[2], boxes[b, idx])
        assert torch.equal(got[1], classes[b, idx].long())
        print('image %d: %d candidates, %d kept' % (b, sel.numel(), idx.numel()))
    for b in range(B):
        one = ops.detect_batch(cls[b:b + 1], reg[b:b + 1], anchors, H, W, thr, 0.5)[0]
        for t1, tb in zip(one, dets[b]):
            assert t1.dtype == tb.dtype and torch.equal(t1, tb), b


@gpu
def test_post_processing_launches_do_not_grow_with_batch():
    from models import _native as N
    from models import _ops as ops
    g = torch.Generator().manual_seed(5)
    A, K = 12276, 20
    anchors = torch.from_numpy(O.anchors_for(256, 256)).to(_dev())
    launches = {}
    for B in (1, 8):
        cls = torch.rand(B, A, K, generator=g).to(_dev())
        reg = (torch.randn(B, A, 4, generator=g) * 0.3).to(_dev())
        ops.detect_batch(cls, reg, anchors, 256, 256, 0.999, 0.5)     # warm-up
        n0 = N.launch_count()
        dets = ops.detect_batch(cls, reg, anchors, 256, 256, 0.999, 0.5)
        launches[B] = N.launch_count() - n0
        assert all(d[0].numel() > 0 for d in dets)
    assert launches[1] == launches[8], launches


@gpu
def test_nms_in_groups_of_images_equals_one_group(monkeypatch):
    """a mask workspace budget below the batch's need runs NMS over consecutive groups of images (offset pointers, one
    shared workspace): the results are bit-identical to the single-group call, eager and with a fixed cap"""
    from models import _ops as ops
    g = torch.Generator().manual_seed(11)
    B, A, K = 5, 12276, 20
    anchors = torch.from_numpy(O.anchors_for(256, 256)).to(_dev())
    cls = torch.rand(B, A, K, generator=g).to(_dev())
    reg = (torch.randn(B, A, 4, generator=g) * 0.3).to(_dev())
    thr = 0.995
    cap = int((cls.max(dim=2)[0] > thr).sum(dim=1).max())
    assert cap > 300
    one = ops.detect_batch(cls, reg, anchors, 256, 256, thr, 0.5)
    fixed = ops.detect_batch(cls, reg, anchors, 256, 256, thr, 0.5, cap=4096)
    per_image = cap * ((cap + 63) // 64) * 8
    for budget in (1, 2 * per_image):                             # groups of 1 image; groups of 2, 2 and 1 images
        monkeypatch.setattr(ops, 'NMS_MASK_BUDGET', budget)
        grouped = ops.detect_batch(cls, reg, anchors, 256, 256, thr, 0.5)
        for a, b in zip(one, grouped):
            for ta, tb in zip(a, b):
                assert torch.equal(ta, tb), budget
        grouped = ops.detect_batch(cls, reg, anchors, 256, 256, thr, 0.5, cap=4096)
        for ta, tb in zip(fixed, grouped):
            assert torch.equal(ta, tb), budget


@gpu
def test_captured_post_processing_replays_bit_identical_to_eager():
    """detect_batch with a fixed cap inside torch.cuda.graph, replayed on two different cls / reg inputs: every output
    bit-identical to the eager call, and its rows equal the eager (cap=None) triples"""
    from models import _ops as ops
    m = _model(seed=81)
    inputs = []
    with torch.no_grad():
        for s in (82, 83):
            cls, reg, anchors = m._raw_predictions(_images(3, seed=s))
            inputs.append((cls.clone(), reg.clone()))
    thr = _threshold(inputs[0][0])
    cap = 8192
    static_cls, static_reg = inputs[0][0].clone(), inputs[0][1].clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        ops.detect_batch(static_cls, static_reg, anchors, 256, 256, thr, 0.5, cap=cap)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = ops.detect_batch(static_cls, static_reg, anchors, 256, 256, thr, 0.5, cap=cap)
    for cls, reg in inputs:
        static_cls.copy_(cls)
        static_reg.copy_(reg)
        graph.replay()
        torch.cuda.synchronize()
        ref = ops.detect_batch(cls, reg, anchors, 256, 256, thr, 0.5, cap=cap)
        for a, b in zip(out, ref):
            assert a.dtype == b.dtype and torch.equal(a, b)
        counts = out.count.tolist()
        eager = ops.detect_batch(cls, reg, anchors, 256, 256, thr, 0.5)
        for b, trip in enumerate(eager):
            assert counts[b] == trip[0].numel() > 0
            assert torch.equal(out.scores[b, :counts[b]], trip[0]) and torch.equal(out.classes[b, :counts[b]], trip[1])
            assert torch.equal(out.boxes[b, :counts[b]], trip[2])
            assert not out.scores[b, counts[b]:].any() and not out.boxes[b, counts[b]:].any()


@gpu
def test_graphed_detect_matches_detect_batch(prec):
    """GraphedDetect on D0 256x256, B = 3: replays on new images match detect_batch, replays follow load_state_dict,
    and with max_candidates below an image's count to_list still equals detect_batch"""
    from models.graph_step import GraphedDetect
    m = _model(seed=91)
    batches = [_images(3, seed=s) for s in (92, 93, 94)]
    with torch.no_grad():
        cls, _, _ = m._raw_predictions(batches[0])
    m.threshold, m.iou_threshold = _threshold(cls, rank=400), 0.5
    det = GraphedDetect(m, batches[0], max_candidates=8192)
    assert det.library_launches > 0
    before = []
    for x in batches[1:]:
        out = det(x)
        assert out.scores.shape == (3, 8192) and out.classes.dtype == torch.int64 and out.boxes.shape == (3, 8192, 4)
        got = det.to_list(out)
        before.append([t.clone() for t in got[0]])
        ref = m.detect_batch(x)
        assert len(got) == 3
        for g_, r in zip(got, ref):
            assert r[0].numel() > 0
            _same_rows(g_, r)
    # in-place weight update: the replay follows it
    cfg = O.make_config('efficientdet-d0', num_classes=20, W_bifpn=64, D_bifpn=2)
    m.load_state_dict(O.init_state_dict(cfg, seed=95))
    got = det.to_list(det(batches[1]))
    ref = m.detect_batch(batches[1])
    for g_, r in zip(got, ref):
        _same_rows(g_, r)
    assert got[0][0].shape != before[0][0].shape or not torch.equal(got[0][0], before[0][0])
    # overflow: an image with more candidates than max_candidates is redone eagerly by to_list
    m.load_state_dict(O.init_state_dict(cfg, seed=91))
    with torch.no_grad():
        cls, _, _ = m._raw_predictions(batches[1])
    counts = (cls.max(dim=2)[0] > m.threshold).sum(dim=1).tolist()
    small = GraphedDetect(m, batches[0], max_candidates=max(counts) // 2)
    out = small(batches[1])
    assert -1 in out.count.tolist()
    got = small.to_list(out)
    ref = m.detect_batch(batches[1])
    for g_, r in zip(got, ref):
        _same_rows(g_, r)
    m.threshold = 0.5
    with pytest.raises(RuntimeError, match='threshold'):
        det(batches[1])


# ------------------------------------------------------------------------------------------------
# CPU: refusals
# ------------------------------------------------------------------------------------------------

@pytest.fixture(scope='module')
def lib():
    from models import _native
    _native.build()
    return _native.load()


def test_batch_entry_points_refuse_bad_arguments(lib):
    """each refusal returns -1 (EFFDET_ERR_ARG), names the entry point, and comes before any device work: the
    pointers below are never dereferenced, so these calls also run without a GPU"""
    f = 1 << 20                                              # aligned non-null "pointer"

    def refused(rc, name):
        msg = lib.effdet_last_error().decode()
        assert rc == -1 and name in msg, (rc, msg)

    def cand(*, p=f, B=2, A=100, K=20, npad=128, box=f):
        return lib.effdet_detect_candidates_batch(p, f, f, box, f, f, f, f, B, A, K, npad, 256.0, 256.0, 0.5, 0, None)

    for kw in (dict(p=None), dict(B=0), dict(npad=96), dict(npad=64), dict(K=0), dict(box=f + 4),
               dict(B=1 << 12, A=1 << 19, npad=1 << 19)):
        refused(cand(**kw), 'detect_candidates_batch')

    def nms(*, p=f, cnt=f, B=2, A=100, npad=128, cap=50, box=f):
        return lib.effdet_nms_batch(box, p, cnt, B, A, npad, cap, 0.5, f, f, f, 0, None)

    for kw in (dict(p=None), dict(cnt=None), dict(B=0), dict(npad=100), dict(npad=64), dict(cap=0), dict(cap=101),
               dict(A=1 << 21, npad=1 << 21, cap=(1 << 21) - 1), dict(box=f + 8)):
        refused(nms(**kw), 'nms_batch')

    def gather(*, p=f, nk=f, B=2, A=100, cap=50, box=f, obox=f):
        return lib.effdet_gather_detections_batch(box, p, f, f, nk, B, A, cap, f, f, obox, 0, None)

    for kw in (dict(p=None), dict(nk=None), dict(B=0), dict(cap=0), dict(cap=101), dict(box=f + 4), dict(obox=f + 4)):
        refused(gather(**kw), 'gather_detections_batch')


def test_graphed_detect_refuses_training_model_and_cpu_images():
    from models import EfficientDet
    from models._native import EffdetNativeError
    from models.graph_step import GraphedDetect
    m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=True)
    x = torch.zeros(1, 3, 128, 128)
    with pytest.raises(EffdetNativeError, match='inference mode'):
        GraphedDetect(m, x)
    m.eval()
    with pytest.raises(EffdetNativeError, match='inference mode'):
        GraphedDetect(m, x)                                  # is_training still set
    m.is_training = False
    m.train()
    with pytest.raises(EffdetNativeError, match='inference mode'):
        GraphedDetect(m, x)                                  # nn.Module training mode
    m.eval()
    with pytest.raises(EffdetNativeError, match='CUDA'):
        GraphedDetect(m, x)


@gpu
def test_graphed_detect_leaves_eager_inference_intact():
    """eager calls straight after building a GraphedDetect (before any replay) see the real weights, not the graph's
    not-yet-computed packed copies; max_candidates above the anchor count is clamped to it (D0 128x128: A = 3069);
    a batch of another shape is refused"""
    from models._native import EffdetNativeError
    from models.graph_step import GraphedDetect
    m = _model(seed=101)
    x = O.synthetic_batch(2, size=128, seed=102)[0].to(_dev())
    with torch.no_grad():
        cls, _, _ = m._raw_predictions(x)
    m.threshold = _threshold(cls, rank=100)
    det = GraphedDetect(m, x)                                    # max_candidates=8192 > A
    ref = m.detect_batch(x)
    with torch.no_grad():
        first = m(x[:1])
    out = det(x)
    assert out.scores.shape == (2, 3069) and out.boxes.shape == (2, 3069, 4)
    got = det.to_list(out)
    for g_, r in zip(got, ref):
        assert r[0].numel() > 0
        _same_rows(g_, r)
    _same_rows(first, got[0])
    with pytest.raises(EffdetNativeError, match='shape'):
        det(x[:1])
