"""Soft-NMS (Bodla et al., ICCV 2017) in detection: tools/soft_nms_oracle.py against a literal transcription of the
paper's Algorithm 1 and against its fixture (tests/golden/make_soft_nms_golden.py), the C entries' refusals, and -- on
the GPU -- effdet_soft_nms_batch against the oracle bit for bit (pick count, anchors, score bits, classes, boxes) on
every fixture case, across each capacity boundary named in csrc/soft_nms.cu, on real network outputs, through
GraphedDetect / GraphedFrameDetect, model(img), and evaluate() / evaluate_coco()."""
import hashlib
import math
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(REPO, 'tools'))
import soft_nms_oracle as S  # noqa: E402

gpu = pytest.mark.gpu
THRESHOLD = 0.05


def _fixture():
    return np.load(os.path.join(HERE, 'golden', 'soft_nms.npz'))


def _case_inputs(st, name):
    """(method, iou_threshold, sigma, threshold, boxes, scores, anchors) of a fixture case, regenerated from its seed"""
    p = name + '/'
    method = str(st[p + 'method'])
    nt, sigma, thr = (float(v) for v in st[p + 'params'])
    seed = int(st[p + 'seed'][0])
    if seed >= 0:
        b, s, a = S.random_candidates(seed, 700, threshold=THRESHOLD)
        h = hashlib.sha256()
        for x in (b, s, a):
            h.update(np.ascontiguousarray(x).tobytes())
        assert np.array_equal(np.frombuffer(h.digest(), np.uint8), st[p + 'input_sha256']), name
    else:
        b, s, a = st[p + 'boxes'], st[p + 'in_scores'], st[p + 'anchors']
    return method, nt, sigma, thr, b, s, a


def literal_soft_nms(boxes, scores, anchors, method, nt, sigma, threshold):
    """Algorithm 1 one candidate at a time, in plain Python on NumPy scalars (no vector operation)"""
    f32 = np.float32
    live = [i for i in range(len(scores)) if f32(scores[i]) > f32(threshold)]
    s = {i: f32(scores[i]) for i in live}
    picks, out = [], []
    while live:
        m = live[0]
        for i in live[1:]:
            if s[i] > s[m] or (s[i] == s[m] and anchors[i] < anchors[m]):
                m = i
        picks.append(int(anchors[m]))
        out.append(s[m])
        live.remove(m)
        bm = [f32(v) for v in boxes[m]]
        for j in list(live):
            bj = [f32(v) for v in boxes[j]]
            w_ = max(f32(min(bm[2], bj[2]) - max(bm[0], bj[0])), f32(0))
            h_ = max(f32(min(bm[3], bj[3]) - max(bm[1], bj[1])), f32(0))
            inter = f32(w_ * h_)
            if inter == 0:
                ov = f32(0)
            else:
                sa = f32(f32(bm[2] - bm[0]) * f32(bm[3] - bm[1]))
                sb = f32(f32(bj[2] - bj[0]) * f32(bj[3] - bj[1]))
                ov = f32(inter / f32(f32(sa + sb) - inter))
            if method == 'linear':
                w = f32(f32(1) - ov) if float(ov) > nt else f32(1)
            else:
                w = f32(math.exp(-(float(ov) * float(ov)) / sigma))
            s[j] = f32(s[j] * w)
            if not s[j] > f32(threshold):
                live.remove(j)
    return np.array(picks, np.int64), np.array(out, np.float32)


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_oracle_equals_fixture_and_literal_algorithm():
    st = _fixture()
    names = [str(n) for n in st['cases']]
    assert len(names) == 19
    assert float(st['gaussian_margin_ulps'][0]) > 1                 # one-ulp exp differences cannot move a weight
    for name in names:
        method, nt, sigma, thr, b, s, a = _case_inputs(st, name)
        pa, ps = S.soft_nms(b, s, a, method, nt, sigma, thr)
        assert np.array_equal(pa, st[name + '/picks']), name
        assert np.array_equal(ps.view(np.uint32), st[name + '/scores'].view(np.uint32)), name
        la, ls = literal_soft_nms(b, s, a, method, nt, sigma, thr)
        assert np.array_equal(pa, la) and np.array_equal(ps.view(np.uint32), ls.view(np.uint32)), name
        assert np.all(np.diff(ps) <= 0) and np.all(ps > np.float32(thr)), name
    # the properties the crafted cases were made for
    pick = lambda n: (st[n + '/picks'], st[n + '/scores'])                          # noqa: E731
    assert np.array_equal(pick('identical_linear')[0], [4, 0])                     # IoU 1: linear weight 0 drops
    ga, gs = pick('identical_gaussian')
    assert np.array_equal(ga, [4, 0, 1, 6])
    assert gs[2] == np.float32(np.float32(0.7) * np.float32(math.exp(-1 / 0.5)))
    assert np.array_equal(pick('iou_half_linear')[1], np.float32([0.9, 0.8, 0.4]))     # IoU 0.5 is not > N_t 0.5
    assert np.array_equal(pick('to_threshold_linear')[0], [0, 2])                  # 0.5 * 0.25 == threshold: dropped
    for m in ('linear', 'gaussian'):
        _, _, _, _, b, s, a = _case_inputs(st, 'disjoint_' + m)
        order = np.lexsort((a, -s))
        assert np.array_equal(pick('disjoint_' + m)[0], a[order])
        assert np.array_equal(pick('disjoint_' + m)[1].view(np.uint32), s[order].view(np.uint32))
    assert pick('empty_linear')[0].size == 0 and np.array_equal(pick('one_gaussian')[0], [17])


@pytest.mark.parametrize('seed', [0, 1, 2])
def test_oracle_equals_literal_algorithm_on_seeded_sets(seed):
    b, s, a = S.random_candidates(seed, 150, size=200.0, clusters=6, threshold=0.1)
    for method, nt, sigma in (('linear', 0.3, 0.5), ('linear', 0.5, 0.5), ('gaussian', 0.5, 0.5),
                              ('gaussian', 0.5, 0.1)):
        pa, ps = S.soft_nms(b, s, a, method, nt, sigma, 0.1)
        la, ls = literal_soft_nms(b, s, a, method, nt, sigma, 0.1)
        assert np.array_equal(pa, la) and np.array_equal(ps.view(np.uint32), ls.view(np.uint32)), (seed, method)


def test_oracle_keep_order_equals_torchvision_when_nothing_overlaps():
    tv = pytest.importorskip('torchvision')
    rng = np.random.default_rng(3)
    g = np.stack(np.meshgrid(np.arange(20), np.arange(20)), -1).reshape(-1, 2).astype(np.float32) * 10
    boxes = np.concatenate([g, g + rng.uniform(1, 9, g.shape).astype(np.float32)], 1)
    scores = rng.uniform(0.1, 1, len(g)).astype(np.float32)
    scores[::7] = scores[3]                                                          # ties
    want = tv.ops.nms(torch.from_numpy(boxes), torch.from_numpy(scores), 0.5).numpy()
    for method in S.METHODS:
        pa, ps = S.soft_nms(boxes, scores, np.arange(len(g)), method, 0.5, 0.5, 0.05)
        assert np.array_equal(pa, want), method
        assert np.array_equal(ps, scores[want])


@pytest.fixture(scope='module')
def lib():
    from models import _native
    _native.build()
    return _native.load()


def test_soft_nms_entry_points_refuse_bad_arguments(lib):
    """each refusal returns -1 (EFFDET_ERR_ARG), names the entry point and comes before any device work: the pointers
    are never dereferenced, so these calls run without a GPU"""
    f = 1 << 20

    def refused(rc, name, what=''):
        msg = lib.effdet_last_error().decode()
        assert rc == -1 and name in msg and what in msg, (rc, msg)

    assert lib.effdet_soft_nms_workspace(4, 32768) == 0
    assert lib.effdet_soft_nms_workspace(4, 32769) == 4 * 32769 * 24
    assert lib.effdet_soft_nms_workspace(1, 32769) == 32769 * 24 + 8                 # rounded up to 16 bytes
    for args in ((0, 100), (65536, 100), (1, 0)):
        refused(lib.effdet_soft_nms_workspace(*args), 'soft_nms_workspace')

    def soft(*, p=f, B=2, A=2000, npad=2048, cap=1000, method=2, nt=0.5, sigma=0.5, ws=f, ws_bytes=0, box=f, obox=f,
             cnt=f):
        return lib.effdet_soft_nms_batch(box, p, p, p, cnt, B, A, npad, cap, method, nt, sigma, 0.05, ws, ws_bytes,
                                         p, p, obox, p, 0, None)

    for kw, what in ((dict(p=None), 'null'), (dict(cnt=None), 'null'), (dict(B=0), 'B=0'), (dict(B=65536), 'B='),
                     (dict(npad=2000), 'npad'), (dict(npad=1024), 'npad'), (dict(cap=0), 'cap'),
                     (dict(cap=2001), 'cap'), (dict(method=0), 'method'), (dict(method=3), 'method'),
                     (dict(method=1, nt=1.5), 'iou_threshold'), (dict(method=1, nt=-0.1), 'iou_threshold'),
                     (dict(sigma=0.0), 'sigma'), (dict(sigma=-1.0), 'sigma'), (dict(sigma=float('nan')), 'sigma'),
                     (dict(sigma=float('inf')), 'sigma'), (dict(box=f + 8), 'aligned'), (dict(obox=f + 8), 'aligned'),
                     (dict(A=40000, npad=65536, cap=40000, ws_bytes=2 * 40000 * 24 - 1), 'workspace'),
                     (dict(A=40000, npad=65536, cap=40000, ws=None, ws_bytes=2 * 40000 * 24), 'workspace')):
        refused(soft(**kw), 'soft_nms_batch', what)


def test_python_refuses_bad_settings_before_any_launch():
    """nms / soft_nms_sigma / a linear iou_threshold are checked on the host before anything reaches the device: these
    calls use CPU tensors and never get to the CUDA check"""
    from models import EfficientDet, _ops
    from models._native import EffdetNativeError
    x = torch.zeros(1, 10, 3)
    for kw, what in ((dict(nms='soft'), "'hard', 'linear', 'gaussian'"), (dict(nms=None), 'nms'),
                     (dict(nms='gaussian', sigma=0), 'soft_nms_sigma'), (dict(nms='gaussian', sigma=-1.0), 'sigma'),
                     (dict(nms='gaussian', sigma=float('nan')), 'sigma'), (dict(nms='linear', sigma='a'), 'sigma'),
                     (dict(nms='linear', iou=1.5), 'iou_threshold')):
        with pytest.raises(EffdetNativeError, match=what):
            _ops.detect_batch(x, x, x, 10, 10, 0.05, kw.get('iou', 0.5), nms=kw['nms'], sigma=kw.get('sigma', 0.5))
    m = EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    assert (m.nms, m.soft_nms_sigma) == ('hard', 0.5)
    assert m.postprocess() == dict(threshold=0.01, iou_threshold=0.5, nms='hard', sigma=0.5)
    m.nms = 'gaussianx'
    with pytest.raises(EffdetNativeError, match='nms'):
        m(torch.zeros(1, 3, 128, 128))
    m.nms, m.soft_nms_sigma = 'gaussian', 0.0
    with pytest.raises(EffdetNativeError, match='soft_nms_sigma'):
        m.detect_batch(torch.zeros(1, 3, 128, 128))
    with pytest.raises(EffdetNativeError, match='nms'):
        EfficientDet(num_classes=20, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, nms='greedy')


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _dev():
    return torch.device('cuda:0')


def _pack(images, cap, A=None):
    """images: list of (boxes [n,4], scores [n], anchors [n]) -> device tensors as effdet_detect_candidates_batch
    leaves them (boxes [B,A,4], scores [B,A], classes [B,A], keys [B,npad] sorted, count [B]), plus A and npad"""
    A = max([cap] + [int(a.max()) + 1 for _, _, a in images if len(a)] + [1]) if A is None else A
    npad = 1 << (A - 1).bit_length()
    B = len(images)
    rng = np.random.default_rng(5)
    boxes = rng.uniform(0, 50, (B, A, 4)).astype(np.float32)
    scores = np.zeros((B, A), np.float32)
    classes = rng.integers(0, 90, (B, A)).astype(np.int32)
    keys = np.full((B, npad), -1, np.int64)
    count = np.zeros(B, np.int32)
    for b, (bx, sc, an) in enumerate(images):
        boxes[b, an] = bx
        scores[b, an] = sc
        order = (np.float32(sc).view(np.uint32).astype(np.uint64) ^ np.uint64(0x80000000))  # positive floats only
        k = ((~order & np.uint64(0xffffffff)) << np.uint64(32)) | an.astype(np.uint64)
        keys[b, :len(an)] = np.sort(k).view(np.int64)
        count[b] = len(an)
    t = lambda x: torch.from_numpy(x).to(_dev())                                     # noqa: E731
    return dict(boxes=t(boxes), scores=t(scores), classes=t(classes), keys=t(keys), count=t(count), A=A, npad=npad)


def _run(p, cap, method, nt, sigma, thr):
    from models import _native as N
    from models import _ops
    B, A = p['boxes'].shape[:2]
    ws_bytes = _ops._soft_nms_workspace(B, cap)
    assert ws_bytes % 16 == 0 and (ws_bytes == 0 or ws_bytes >= B * cap * 24)
    ws = torch.empty((max(ws_bytes, 16),), device=_dev(), dtype=torch.uint8)
    o_s = torch.empty((B, cap), device=_dev())
    o_c = torch.empty((B, cap), device=_dev(), dtype=torch.int64)
    o_b = torch.empty((B, cap, 4), device=_dev())
    o_n = torch.empty((B,), device=_dev(), dtype=torch.int32)
    N.call('effdet_soft_nms_batch', p['boxes'], N.f32(p['boxes']), N.f32(p['scores']), p['classes'].data_ptr(),
           p['keys'].data_ptr(), p['count'].data_ptr(), B, A, p['npad'], cap, _ops.NMS_METHODS[method], nt, sigma, thr,
           ws.data_ptr(), ws_bytes, N.f32(o_s), o_c.data_ptr(), N.f32(o_b), o_n.data_ptr())
    return o_s.cpu().numpy(), o_c.cpu().numpy(), o_b.cpu().numpy(), o_n.cpu().numpy()


def _check(out, p, images, cap, method, nt, sigma, thr):
    """the kernel's padded rows of every image equal the oracle's picks bit for bit"""
    o_s, o_c, o_b, o_n = out
    boxes, classes = p['boxes'].cpu().numpy(), p['classes'].cpu().numpy()
    for b, (bx, sc, an) in enumerate(images):
        if len(an) > cap:
            assert o_n[b] == -1 and not o_s[b].any() and not o_c[b].any() and not o_b[b].any(), b
            continue
        pa, ps = S.soft_nms(bx, sc, an, method, nt, sigma, thr)
        k = len(pa)
        assert o_n[b] == k, (b, o_n[b], k)
        assert np.array_equal(o_s[b, :k].view(np.uint32), ps.view(np.uint32)), b
        assert np.array_equal(o_c[b, :k], classes[b, pa]), b
        assert np.array_equal(o_b[b, :k].view(np.uint32), boxes[b, pa].view(np.uint32)), b
        assert not o_s[b, k:].any() and not o_c[b, k:].any() and not o_b[b, k:].any(), b


@gpu
@pytest.mark.parametrize('cap_extra', [0, 5000])
def test_kernel_equals_oracle_on_fixture_cases(cap_extra):
    """every fixture case as one image of one batch (counts 0 .. 700, the empty images included), at cap = the largest
    count (one CTA per image) and at a cap that gives two-CTA clusters; also with a threshold above some of the
    candidates' scores (only reachable through the C entry), which are then never picked"""
    st = _fixture()
    groups = {}
    for name in (str(n) for n in st['cases']):
        method, nt, sigma, thr, b, s, a = _case_inputs(st, name)
        groups.setdefault((method, nt, sigma, thr), []).append((b, s, a))
    for (method, nt, sigma, thr), images in groups.items():
        cap = max(max(len(a) for _, _, a in images), 1) + cap_extra
        p = _pack(images, cap)
        _check(_run(p, cap, method, nt, sigma, thr), p, images, cap, method, nt, sigma, thr)
        _check(_run(p, cap, method, nt, sigma, 0.5), p, images, cap, method, nt, sigma, 0.5)


def grouped_candidates(seed, n, g=32):
    """n candidates in groups of about g jittered 20x20 boxes (IoU within a group about 0.55 .. 1), the groups far
    apart: each pick decays or drops its group, so the oracle costs about n/g picks"""
    rng = np.random.default_rng(seed)
    groups = max(1, n // g)
    side = int(math.ceil(math.sqrt(groups)))
    gi = rng.integers(0, groups, n)
    c = np.stack([gi % side, gi // side], 1) * 40.0 + 10
    boxes = np.concatenate([c, c + 20], 1) + rng.uniform(-1.5, 1.5, (n, 4))
    scores = rng.uniform(0.1, 1, n).astype(np.float32)
    scores[rng.random(n) < 0.1] = np.float32(0.5)
    return boxes.astype(np.float32), scores


@gpu
@pytest.mark.parametrize('n,cap', [
    (4096, 4096),      # cluster of 1 at its largest
    (4096, 4097),      # cluster of 2, a count that still runs on one CTA
    (4097, 4097),      # cluster of 2 in use
    (8192, 8192),
    (8193, 8193),      # cluster of 4
    (16384, 16384),
    (16385, 16385),    # cluster of 8
    (32768, 32768),    # cluster of 8, slices in shared memory at their largest
    (32768, 32769),    # global workspace allocated, slices still in shared memory
    (32769, 32769),    # slices in the global workspace
])
def test_kernel_equals_oracle_across_capacity_boundaries(n, cap):
    """counts on both sides of each boundary of csrc/soft_nms.cu (single CTA, each cluster size, shared and global
    residency), in a batch with an image that overflows cap, an empty image and, last, the image of n candidates: at
    n == cap it fills the workspace's last slots (B * cap is odd for odd cap)"""
    rng = np.random.default_rng(n + cap)
    A = cap + 7
    images = []
    for i, m in ((2, min(A, cap + 5)), (1, 0), (0, n)):
        bx, sc = grouped_candidates(i + n, m)
        images.append((bx, sc, rng.permutation(A)[:m].astype(np.int64)))
    p = _pack(images, cap, A)
    for method, nt, sigma, thr in (('gaussian', 0.5, 0.1, 0.1), ('linear', 0.3, 0.5, 0.1)):
        _check(_run(p, cap, method, nt, sigma, thr), p, images, cap, method, nt, sigma, thr)


def _d0(seed=3, K=20):
    import effdet_oracle as O
    from models import EfficientDet
    cfg = O.make_config('efficientdet-d0', num_classes=K, W_bifpn=64, D_bifpn=2)
    m = EfficientDet(num_classes=K, network='efficientdet-d0', D_bifpn=2, W_bifpn=64, is_training=False)
    m.load_state_dict(O.init_state_dict(cfg, seed=seed))
    return m.to(_dev()).eval()


def _candidates(cls, reg, anchors, h, w, thr):
    """the device's candidate stage (effdet_detect_candidates_batch, tested on its own in test_detect_batched.py) ->
    NumPy boxes, scores, classes, count, keys"""
    from models import _native as N
    B, A, K = cls.shape
    npad = 1 << (A - 1).bit_length()
    boxes = torch.empty((B, A, 4), device=_dev())
    scores = torch.empty((B, A), device=_dev())
    classes = torch.empty((B, A), device=_dev(), dtype=torch.int32)
    keys = torch.empty((B, npad), device=_dev(), dtype=torch.int64)
    count = torch.empty((B,), device=_dev(), dtype=torch.int32)
    N.call('effdet_detect_candidates_batch', cls, N.f32(cls.contiguous()), N.f32(reg.contiguous()),
           N.f32(anchors.reshape(-1, 4).contiguous()), N.f32(boxes), N.f32(scores), classes.data_ptr(), keys.data_ptr(),
           count.data_ptr(), B, A, K, npad, float(w), float(h), float(thr))
    return [t.cpu().numpy() for t in (boxes, scores, classes, count, keys)]


def _oracle_dets(cls, reg, anchors, h, w, post):
    """the oracle's Soft-NMS of the device candidates of every image -> list of (scores, classes, boxes)"""
    c = _candidates(cls, reg, anchors, h, w, post['threshold'])
    return [S.soft_nms_candidates(*c, b, post['nms'], post['iou_threshold'], post['sigma'], post['threshold'])[:3]
            for b in range(cls.shape[0])]


def _same_dets(got, want):
    for b, ((gs, gc, gb), (ws, wc, wb)) in enumerate(zip(got, want)):
        gs, gc, gb = (t.cpu().numpy() for t in (gs, gc, gb))
        assert len(gs) == len(ws), (b, len(gs), len(ws))
        assert np.array_equal(gs.view(np.uint32), ws.view(np.uint32)), b
        assert np.array_equal(gc, wc) and np.array_equal(gb.view(np.uint32), wb.view(np.uint32)), b
        assert np.all(np.diff(gs) <= 0), b


@gpu
def test_real_network_outputs_equal_oracle():
    """D0 512x512, seeded weights, B = 4, thresholds 0.05 and 0.01, both methods: detect_batch (eager and with a fixed
    cap) equals the oracle on the same network outputs; model(img) equals detect_batch(images)[i]"""
    import effdet_oracle as O
    from models import _ops
    m = _d0()
    x = O.synthetic_batch(4, size=512, seed=8)[0].to(_dev())
    with torch.no_grad():
        cls, reg, anchors = m._raw_predictions(x)
    for thr in (0.05, 0.01):
        counts = (cls.max(dim=2)[0] > thr).sum(dim=1).tolist()
        print('threshold %g: candidates %s' % (thr, counts))
        for nms, sigma in (('linear', 0.5), ('gaussian', 0.5)):
            m.threshold, m.nms, m.soft_nms_sigma = thr, nms, sigma
            post = m.postprocess()
            want = _oracle_dets(cls, reg, anchors, 512, 512, post)
            _same_dets(_ops.detect_batch(cls, reg, anchors, 512, 512, **post), want)
            fixed = _ops.detect_batch(cls, reg, anchors, 512, 512, cap=_ops.candidate_cap(None, cls), **post)
            n = fixed.count.tolist()
            _same_dets([(fixed.scores[b, :n[b]], fixed.classes[b, :n[b]], fixed.boxes[b, :n[b]]) for b in range(4)],
                       want)
    # drop-in: model(img) and model.detect_batch post-process what the network gives them like detect_batch does.  Two
    # network passes differ in the last bits (fp32 atomics), so both see the outputs computed above.
    m.threshold, m.nms = 0.05, 'gaussian'
    m._raw_predictions = lambda images: (cls[:images.shape[0]], reg[:images.shape[0]], anchors)
    want = _ops.detect_batch(cls, reg, anchors, 512, 512, **m.postprocess())
    with torch.no_grad():
        assert all(torch.equal(a, b) for g, w in zip(m.detect_batch(x), want) for a, b in zip(g, w))
        one = m(x[:1])
    assert all(torch.equal(a, b) for a, b in zip(one, _ops.detect_batch(cls[:1], reg[:1], anchors, 512, 512,
                                                                        **m.postprocess())[0]))


@gpu
def test_every_anchor_a_candidate_equals_oracle():
    """one D0 512x512 image with threshold 0, so all 49 104 anchors are candidates: the Gaussian method equals the
    oracle.  The NumPy oracle makes up to 49 104 picks over up to 49 104 live candidates: about a minute on the host."""
    import effdet_oracle as O
    from models import _ops
    m = _d0(seed=4)
    x = O.synthetic_batch(1, size=512, seed=9)[0].to(_dev())
    with torch.no_grad():
        cls, reg, anchors = m._raw_predictions(x)
    post = dict(threshold=0.0, iou_threshold=0.5, nms='gaussian', sigma=0.5)
    assert int((cls.max(dim=2)[0] > 0).sum()) == cls.shape[1] == 49104
    got = _ops.detect_batch(cls, reg, anchors, 512, 512, **post)
    _same_dets(got, _oracle_dets(cls, reg, anchors, 512, 512, post))


@gpu
def test_graphed_detect_replays_equal_eager_and_refuses_changed_settings():
    """GraphedDetect with each soft method replays equal to eager detect_batch on the replay's network outputs (which
    equals the oracle: test_real_network_outputs_equal_oracle), on two different inputs; changing nms or
    soft_nms_sigma after capture raises.  With max_candidates below the images' counts, to_list redoes them eagerly
    with the soft method and still equals detect_batch (a mix of redone and replayed images: the evaluation test)."""
    import effdet_oracle as O
    from models import _ops
    from models.graph_step import GraphedDetect
    from models._native import EffdetNativeError
    m = _d0()
    m.threshold = 0.05
    batches = [O.synthetic_batch(4, size=512, seed=s)[0].to(_dev()) for s in (8, 10)]
    for nms in ('linear', 'gaussian'):
        m.nms = nms
        det = GraphedDetect(m, batches[0], max_candidates=None)
        for x in batches:
            out = det(x)
            got = det.to_list(out)
            want = _ops.detect_batch(det.cls, det.reg, det.anchors, 512, 512, **m.postprocess())
            assert all(torch.equal(a, b) for g, w in zip(got, want) for a, b in zip(g, w)), nms
            assert all(np.all(np.diff(g[0].cpu().numpy()) <= 0) for g in got)
        for attr, value in (('nms', 'hard'), ('soft_nms_sigma', 0.25)):
            old = getattr(m, attr)
            setattr(m, attr, value)
            with pytest.raises(EffdetNativeError, match='post-processing settings changed'):
                det(batches[0])
            setattr(m, attr, old)
        counts = sorted((det.cls.max(dim=2)[0] > m.threshold).sum(dim=1).tolist())
        del det
        small = GraphedDetect(m, batches[1], max_candidates=counts[0] // 2)
        out = small(batches[1])
        assert (out.count == -1).any(), out.count
        want = _ops.detect_batch(small.cls, small.reg, small.anchors, 512, 512, **m.postprocess())
        got = small.to_list(out)
        assert all(torch.equal(a, b) for g, w in zip(got, want) for a, b in zip(g, w)), nms
        del small, out


@gpu
def test_graphed_frame_detect_equals_frame_boxes_of_oracle():
    """GraphedFrameDetect with a soft method returns frame_boxes of the oracle's detections; with max_candidates below
    every frame's count it redoes the frames eagerly and returns frame_boxes of detect_batch's"""
    import frame_oracle as F
    from models import _ops, pipeline
    from models.evaluation import _padded
    from models.graph_step import GraphedFrameDetect
    m = _d0()
    m.threshold, m.nms, m.soft_nms_sigma = 0.05, 'gaussian', 0.3
    frames = F.synthetic_frames(7, [(480, 640), (375, 500)])
    det = GraphedFrameDetect(m, frames)
    got = det(frames)
    for b in range(len(frames)):
        want = _oracle_dets(det.cls[b:b + 1], det.reg[b:b + 1], det.anchors, 512, 512, m.postprocess())[0]
        trip = [torch.from_numpy(np.ascontiguousarray(t)).to(_dev()) for t in want]
        rows, counts = pipeline.frame_boxes(_padded(trip), det._hw[b:b + 1], 512, 512)
        r = rows[0, :int(counts[0])].cpu().numpy()
        assert np.array_equal(got[b][0], r[:, :4]) and np.array_equal(got[b][1], r[:, 4].astype(np.int64))
        assert np.array_equal(got[b][2], r[:, 5]), b
    # frames over max_candidates are redone eagerly (GraphedFrameDetect._redo) with the soft method
    counts = (det.cls.max(dim=2)[0] > m.threshold).sum(dim=1).tolist()
    del det
    det = GraphedFrameDetect(m, frames, max_candidates=min(counts) // 2)
    got = det(frames)
    for b in range(len(frames)):
        trip = _ops.detect_batch(det.cls[b:b + 1], det.reg[b:b + 1], det.anchors, 512, 512, **m.postprocess())[0]
        rows, n = pipeline.frame_boxes(_padded(trip), det._hw[b:b + 1], 512, 512)
        r = rows[0, :int(n[0])].cpu().numpy()
        assert len(r) and np.array_equal(got[b][0], r[:, :4]) and np.array_equal(got[b][2], r[:, 5]), b
        assert np.array_equal(got[b][1], r[:, 4].astype(np.int64)), b


class _Stub(torch.nn.Module):
    """a detector whose raw outputs are fixed elementwise functions of the pixels (deterministic, unlike the
    network's fp32 atomics), with EfficientDet's post-processing settings"""

    def __init__(self, K=4):
        super().__init__()
        from models.module import Anchors
        self.w = torch.nn.Parameter(torch.zeros(1))
        self.K, self.anchors = K, Anchors()
        self.threshold, self.iou_threshold, self.nms, self.soft_nms_sigma = 0.5, 0.5, 'gaussian', 0.5
        self.is_training = False

    def postprocess(self):
        from models import EfficientDet
        return EfficientDet.postprocess(self)

    def _raw_predictions(self, images):
        anchors = self.anchors(images)
        B, A = images.shape[0], anchors.reshape(-1, 4).shape[0]
        flat = images.reshape(B, -1)
        cls = (flat[:, :A * self.K] ** 16).reshape(B, A, self.K).contiguous()
        reg = (flat[:, A * self.K:A * self.K + 4 * A] - 0.5).reshape(B, A, 4).contiguous()
        return cls, reg, anchors


class _Data:
    def __init__(self, n, K, seed=12):
        g = torch.Generator().manual_seed(seed)
        self.images = [torch.rand(256, 256, 3, generator=g) for _ in range(n)]
        self.scales = [1.0 if i % 2 else 0.8 for i in range(n)]
        self.K = K
        rng = np.random.default_rng(seed)
        self.annots = []
        for i in range(n):
            xy = rng.uniform(0, 200, (6, 2))
            wh = rng.uniform(10, 60, (6, 2))
            self.annots.append(np.concatenate([xy, xy + wh, rng.integers(0, K, (6, 1))], 1))
        self.image_ids = list(range(100, 100 + n))
        self.set_name = 'softnms'

    def __len__(self):
        return len(self.images)

    def __getitem__(self, i):
        return {'img': self.images[i], 'scale': self.scales[i]}

    def load_annotations(self, i):
        return self.annots[i]

    def num_classes(self):
        return self.K

    def label_to_name(self, label):
        return 'class%d' % label

    def label_to_coco_label(self, label):
        return label + 1


@gpu
def test_evaluation_with_gaussian_soft_nms_equals_oracles(tmp_path, monkeypatch):
    """evaluate() and evaluate_coco() with model.nms = 'gaussian' (batch_size 4: graphed batches and an eager
    remainder) equal tools/voc_eval_oracle.py / tools/coco_eval_oracle.py on the oracle's Soft-NMS detections, also
    when max_candidates is below half of the images' counts and those images are redone eagerly (_add_batch)"""
    import coco_eval_oracle as C
    import voc_eval_oracle as V
    from models import evaluation
    K, n = 4, 10
    m = _Stub(K).to(_dev()).eval()
    ds = _Data(n, K)
    dets, counts = [], []
    with torch.no_grad():
        for i in range(n):
            x = ds[i]['img'].permute(2, 0, 1)[None].to(_dev())
            cls, reg, anchors = m._raw_predictions(x)
            counts.append(int((cls.max(dim=2)[0] > m.threshold).sum()))
            dets.append(_oracle_dets(cls, reg, anchors, 256, 256, m.postprocess())[0])
    assert sum(len(d[0]) for d in dets) > 100
    sel = [V.select_detections(s, c, b, ds.scales[i], 0.05, 100, K) for i, (s, c, b) in enumerate(dets)]
    want = V.evaluate(sel, V.get_annotations(ds), K, 0.5)
    small = sorted(counts)[n // 2]
    assert sorted(counts)[0] < small < sorted(counts)[-1]
    for cap in (None, small):
        monkeypatch.setattr(evaluation, 'MAX_CANDIDATES', cap)
        got = evaluation.evaluate(ds, m, batch_size=4)
        assert got[0] == want[0], (cap, got[0], want[0])
        assert {c: (float(a), float(k)) for c, (a, k) in got[1].items()} == \
            {c: (float(a), float(k)) for c, (a, k) in want[1].items()}, cap
    anns = []
    for i in range(n):
        for r in ds.annots[i]:
            x1, y1, x2, y2, c = (float(v) for v in r)
            anns.append({'id': len(anns) + 1, 'image_id': ds.image_ids[i], 'category_id': int(c) + 1,
                         'bbox': [x1, y1, x2 - x1, y2 - y1], 'area': (x2 - x1) * (y2 - y1), 'iscrowd': 0})
    inst = {'images': [{'id': i} for i in ds.image_ids], 'categories': [{'id': k + 1} for k in range(K)],
            'annotations': anns}
    ds.coco = C.COCO(inst)
    results = []
    for i, (s, c, b) in enumerate(dets):
        results += C.collect(ds.image_ids[i], s, c, b, ds.scales[i], ds.label_to_coco_label)
    want = C.evaluate(inst, results, ds.image_ids)[0]
    monkeypatch.chdir(tmp_path)
    for cap in (None, small):
        monkeypatch.setattr(evaluation, 'MAX_CANDIDATES', cap)
        m.eval()
        got = evaluation.evaluate_coco(ds, m, batch_size=4)
        assert np.array_equal(np.asarray(got), np.asarray(want)), (cap, got, want)
